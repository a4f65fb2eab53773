"""NonbondedForce parameter changes of a live context, as free-energy work makes them (alchemical decoupling, charging,
exceptions switched on and off, sigma changes), written as parameter offsets of one global parameter "lam": a change is a
base SystemDesc (lam = 0, the parameters the context is made with) plus offsets (name, index, dq, dsigma, deps) of particles
and exceptions (NonbondedForce::addParticleParameterOffset / addExceptionParameterOffset).  The parameters at lam = 1 come
from oracle.port.with_parameter_offsets, the restatement pinned to the Reference platform.

Each change keeps to its own atoms, so that "all" is the union of every change that applies to a system."""
import os
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LAM = "lam"

# PME water (rigid and flexible), PME ions in a triclinic cell, reaction field, a switched LJ fluid with the dispersion
# correction, both non-periodic methods, and a solvated protein
SYSTEMS = ("water_rigid", "water_flexible", "ions_triclinic", "lj_reaction_field", "lj_switch_dispersion", "cluster_nocutoff",
           "cluster_cutoff", "dhfr")
CHANGES = ("decouple", "charge", "exceptions", "sigma")


def system(name):
    from openmm_b200 import systems
    if name == "water_rigid":
        return systems.water_box(7, cutoff=0.9).rounded()
    if name == "water_flexible":
        return systems.water_box(7, cutoff=0.9, rigid=False).rounded()
    if name == "ions_triclinic":
        return systems.random_ions(894, 3.0, cutoff=1.0, triclinic=True).rounded()
    if name == "lj_reaction_field":
        return systems.lj_fluid(7, cutoff=1.0, charged=True).rounded()
    if name == "lj_switch_dispersion":
        d = systems.lj_fluid(7, cutoff=1.0)
        d.use_switch, d.switch_distance, d.use_dispersion = True, 0.85, True
        return d.rounded()
    if name == "cluster_nocutoff":
        return systems.cluster(70).rounded()
    if name == "cluster_cutoff":
        return systems.cluster(70, method=systems.NB_CUTOFF_NONPERIODIC, cutoff=0.9).rounded()
    if name == "dhfr":
        return systems.SystemDesc.load(os.path.join(ROOT, "data", "dhfr.npz")).rounded()
    raise KeyError(name)


def water_oxygens(d):
    """the oxygens of the TIP3P waters (charge -0.834 followed by two hydrogens of 0.417), ascending"""
    q = np.asarray(d.charges)
    o = np.where(np.abs(q + 0.834) < 1e-9)[0]
    o = o[o + 2 < len(q)]
    return o[(np.abs(q[o + 1] - 0.417) < 1e-9) & (np.abs(q[o + 2] - 0.417) < 1e-9)]


def _waters(d, first, last):
    """the atoms of waters first..last-1 (whole molecules), counted from the first water"""
    o = water_oxygens(d)[first:last]
    return np.concatenate([o, o + 1, o + 2])


def _solute_end(d):
    """the first water atom of a solvated solute; 0 in pure water or a system without waters"""
    o = water_oxygens(d)
    return int(o[0]) if len(o) else 0


def _block(d, lo, hi):
    """atoms of the fraction [lo, hi) of a system without waters"""
    return np.arange(int(lo*d.natoms), int(hi*d.natoms))


def _decouple(d, base, p_off, e_off):
    """a block of solute atoms (or whole waters) to charge 0 and half their epsilon; their 1-4 exceptions scaled by 1/2"""
    if _solute_end(d):
        atoms = np.arange(0, 200)                         # the protein's first residues
    elif len(water_oxygens(d)):
        atoms = _waters(d, 10, 18)
    else:
        atoms = _block(d, 0.0, 0.125)
    for i in atoms.tolist():
        p_off.append((LAM, i, -base.charges[i], 0.0, -0.5*base.epsilons[i]))
    inside = np.isin(d.exc_i, atoms) & np.isin(d.exc_j, atoms) & ((d.exc_qq != 0) | (d.exc_eps != 0))
    for e in np.where(inside)[0].tolist():
        e_off.append((LAM, e, -0.5*base.exc_qq[e], 0.0, -0.5*base.exc_eps[e]))
    return True


def _charge(d, base, p_off, e_off):
    """whole waters (or a block of atoms) that have charge 0 in the base get their charges (+-0.4 in a neutral fluid), and
    hydrogens with epsilon 0 get an epsilon of 0.05 at sigma 0.1 nm"""
    if len(water_oxygens(d)):
        atoms = _waters(d, 20, 30)
        q = base.charges[atoms].copy()
    else:
        atoms = _block(d, 0.25, 0.375)
        q = base.charges[atoms].copy()
        q[q == 0] = np.where(np.arange(len(atoms)) % 2 == 0, 0.4, -0.4)[q == 0]
    base.charges[atoms] = 0.0
    for i, qi in zip(atoms.tolist(), q.tolist()):
        p_off.append((LAM, i, qi, 0.0, 0.0))
    hydrogens = []
    if len(water_oxygens(d)):
        o = water_oxygens(d)[30:40]
        hydrogens = np.concatenate([o + 1, o + 2]).tolist()
        hydrogens += [i for i in np.where(base.epsilons == 0)[0].tolist() if i < _solute_end(d)][:10]      # solute hydrogens
    for i in hydrogens:
        assert base.epsilons[i] == 0
        p_off.append((LAM, i, 0.0, 0.1 - base.sigmas[i], 0.05))
    return True


def _exceptions(d, base, p_off, e_off):
    """water O-H exclusions (all parameters zero) become live 1-4 terms; some of a protein's 1-4 terms go to zero"""
    if not len(d.exc_i):
        return False
    if len(water_oxygens(d)):
        o = water_oxygens(d)[40:60]
        live = np.where(np.isin(d.exc_i, o) & (d.exc_j == d.exc_i + 1))[0]
    else:
        live = np.where((d.exc_qq == 0) & (d.exc_eps == 0))[0]
    assert len(live) and (base.exc_qq[live] == 0).all() and (base.exc_eps[live] == 0).all()
    for e in live.tolist():
        e_off.append((LAM, e, -0.05, 0.12 - base.exc_sigma[e], 0.2))
    if _solute_end(d):
        gone = np.where((d.exc_qq != 0) & (d.exc_eps != 0))[0][:60]
        for e in gone.tolist():
            e_off.append((LAM, e, -base.exc_qq[e], 0.0, -base.exc_eps[e]))
    return True


def _sigma(d, base, p_off, e_off):
    """sigma up by 0.03 nm on atoms with an epsilon: the oxygens of some waters, or a block of atoms"""
    if len(water_oxygens(d)):
        atoms = water_oxygens(d)[60:120]
        if _solute_end(d):
            atoms = np.concatenate([atoms, np.arange(200, 400)])          # protein atoms too
    else:
        atoms = _block(d, 0.5, 0.625)
    for i in atoms.tolist():
        if base.epsilons[i] > 0:
            p_off.append((LAM, i, 0.0, 0.03, 0.0))
    return True


_CHANGES = {"decouple": _decouple, "charge": _charge, "exceptions": _exceptions, "sigma": _sigma}


def change(d, name):
    """(base, particle offsets, exception offsets) of change `name` (a key of CHANGES, a tuple of them, or "all": every one
    that applies) to system d, or None when it does not apply (no exceptions)"""
    import copy
    base = copy.copy(d)
    base.charges, base.sigmas, base.epsilons = (np.array(a, dtype=np.float64) for a in (d.charges, d.sigmas, d.epsilons))
    base.exc_qq, base.exc_sigma, base.exc_eps = (np.array(a, dtype=np.float64) for a in (d.exc_qq, d.exc_sigma, d.exc_eps))
    p_off, e_off = [], []
    names = CHANGES if name == "all" else name if isinstance(name, tuple) else (name,)
    applied = [_CHANGES[n](d, base, p_off, e_off) for n in names]
    if not any(applied):
        return None
    return base, p_off, e_off


WITHOUT_EXCEPTIONS = ("ions_triclinic", "lj_reaction_field", "lj_switch_dispersion")


def cases():
    """(system, change) pairs where the change applies (a system without exceptions has no exception change)"""
    return [(s, c) for s in SYSTEMS for c in CHANGES if not (c == "exceptions" and s in WITHOUT_EXCEPTIONS)]


# what updateParametersInContext may change: the Reference platform refuses an exception that turns from excluded (all
# parameters zero) to live or back (ReferenceCalcNonbondedForceKernel::copyParametersToContext)
KEEPS_EXCLUSIONS = ("decouple", "charge", "sigma")


def before_after(system_name, change_name):
    """(A, B, dispersion coefficient of A): the parameters at lam = 0 and lam = 1, and the dispersion coefficient the
    reference uses for both (the one of the parameters' default values, lam = 0)"""
    from oracle import port
    base, p_off, e_off = change(system(system_name), change_name)
    after = port.with_parameter_offsets(base, {LAM: 1.0}, p_off, e_off)
    return base, after, base.dispersion_coefficient()
