"""Energies and energy differences at the kT scale (tests/test_energy_cpu.py, tests/test_gpu_energy.py).

A Monte Carlo barostat accepts a move on w = dE + P dV - N kT ln(V'/V) and a free-energy run evaluates E/kT at every
lambda, so an error in the potential energy matters on the scale of kT, not of the total.  The yardstick is the
double-precision restatement (oracle.port.forces_energy), given exactly the fp32 coordinates the kernels read, split the
way the engine's term masks split the energy:
  direct     = TERM_NB_DIRECT: tile kernel pairs + dispersion correction + 1-4 exceptions + PME exclusion correction
  reciprocal = TERM_NB_RECIP:  PME reciprocal energy + self energy
  bonds, angles, torsions = TERM_BONDS, TERM_ANGLES, TERM_TORSIONS
and evaluated on two ladders: barostat moves of the volume by 1e-4 to 1e-2 (and one anisotropic move), and the
NonbondedForce parameter changes of tests/nonbonded_params_harness.py at lambda = 0 ... 1."""
import copy
import hashlib
import os
import numpy as np
from barostat_harness import barostat_scale
import nonbonded_params_harness as NP
from openmm_b200.engine import TERM_BONDS, TERM_ANGLES, TERM_TORSIONS, TERM_NB_DIRECT, TERM_NB_RECIP

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KT = 0.00831446261815324*300.0               # kJ/mol at 300 K

# oracle parts of each group, and the engine's term mask of each group
GROUPS = {"direct": ("direct", "dispersion", "exceptions14", "exclusion"), "reciprocal": ("reciprocal", "self"),
          "bonds": ("bonds",), "angles": ("angles",), "torsions": ("torsions",)}
MASKS = {"direct": TERM_NB_DIRECT, "reciprocal": TERM_NB_RECIP, "bonds": TERM_BONDS, "angles": TERM_ANGLES, "torsions": TERM_TORSIONS}

# barostat ladder: s^3 - 1 (the relative volume change) of the isotropic moves, and one anisotropic move
VOLUME_STEPS = (1e-4, -1e-4, 1e-3, -1e-3, 1e-2, -1e-2)
ANISO = (1.004, 0.995, 1.003)
RUNGS = tuple("%+g" % v for v in VOLUME_STEPS) + ("aniso",)
LAMBDAS = (0.0, 0.25, 0.5, 0.75, 1.0)
# After these moves of the triclinic ion box the Reference platform's energy is off by 12.2, 12.4 and 0.04 kJ/mol: its voxel
# neighbour list misses pairs inside the cutoff in this cell (as at the reduced-form limits, tests/test_oracle_edges_cpu.py).
# The box sits exactly at a voxel-count boundary: its diagonal lengths are 3.0 nm = 3 cutoffs, and the list's voxel edge
# 0.5*L/floor(L/rc) (ReferenceNeighborList.cpp) changes as soon as a length drops below 3.0 -- which the shrinking moves
# and the anisotropic one (b.y times 0.995) do, and the growing moves do not.
# There the restatement's direct-space energy is pinned to a sum over all 27 images instead
# (tests/test_energy_cpu.py::test_oracle_direct_energy_matches_an_all_image_sum), and comparisons with the Reference
# platform leave these moves out.
REFERENCE_LIST_MISSES = {("ions_triclinic", "-0.001"), ("ions_triclinic", "-0.01"), ("ions_triclinic", "aniso")}


def load(name):
    """A system of the ladders by name: the two proteins, the 24k water box, the triclinic 894-ion box, or a system of
    tests/nonbonded_params_harness.py (lj_switch_dispersion, ...).  Positions are fp32-representable."""
    from openmm_b200 import systems
    if name in ("dhfr", "apoa1"):
        return systems.SystemDesc.load(os.path.join(ROOT, "data", name + ".npz")).rounded()
    if name == "water24k":
        return systems.water_box(20, cutoff=0.9).rounded()
    return NP.system(name)


def pinned_pme(d):
    """d with its PME alpha and grid written out: a context keeps both when its box changes, and so must the oracle."""
    from openmm_b200 import systems
    d = copy.copy(d)
    if d.method == systems.NB_PME:
        alpha, nx, ny, nz = d.pme_parameters()
        d.pme_alpha, d.pme_grid = alpha, (nx, ny, nz)
    return d


def rung_scale(rung):
    """per-axis length factors (sx, sy, sz) of a rung"""
    if rung == "aniso":
        return ANISO
    s = (1.0 + float(rung))**(1.0/3.0)
    return (s, s, s)


def scale_box(box, s):
    """The box after a move: every box vector's x, y and z components times sx, sy and sz (MonteCarloBarostatImpl and
    MonteCarloAnisotropicBarostatImpl::updateContextState)."""
    return np.asarray(box, dtype=np.float64)*np.asarray(s, dtype=np.float64)[None, :]


def fp32(a):
    return np.asarray(a, dtype=np.float64).astype(np.float32).astype(np.float64)


def scaled(d, rung):
    """(desc after the move, (sx, sy, sz)): molecules moved as the reference's barostats move them (barostat_scale), the
    box scaled; positions and box rounded to fp32, so that the kernels and the oracle see the same numbers.  The PME alpha
    and grid stay those of d."""
    d = pinned_pme(d)
    s = rung_scale(rung)
    out = copy.copy(d)
    out.positions = fp32(barostat_scale(d.positions, d.molecules(), d.box, s))
    out.box = fp32(scale_box(d.box, s))
    return out, s


def volume(box):
    return abs(float(np.linalg.det(np.asarray(box, dtype=np.float64))))


def at_lambda(system_name, change_name, lam):
    """(desc with the parameters at lambda, dispersion coefficient): port.with_parameter_offsets of the change, with the
    dispersion coefficient of the parameters' default values (lambda = 0), as the reference keeps it."""
    from oracle import port
    base, p_off, e_off = NP.change(NP.system(system_name), change_name)
    return port.with_parameter_offsets(base, {NP.LAM: lam}, p_off, e_off), base.dispersion_coefficient()


def lambda_changes(system_name):
    return [c for s, c in NP.cases() if s == system_name]


def kernel_positions(eng):
    """The xyz of posq, the fp32 coordinates every force kernel reads, from the checkpoint blob (single: header | posq |
    velm | cellOffset; mixed: header | posq | posqCorr | velmD | cellOffset; posq first in both).  Molecules the list
    build wrapped back into the cell are moved by whole lattice vectors, which leaves the energy as it is."""
    from test_gpu_host_state import HEADER
    npad = eng.stats()["padded_atoms"]
    blob = eng.checkpoint()
    h = np.frombuffer(blob, dtype=HEADER, count=1)[0]
    assert h["magic"] == b"B200MDCK" and h["natoms"] == eng.natoms
    posq = np.frombuffer(blob, dtype=np.float32, count=4*npad, offset=HEADER.itemsize).reshape(npad, 4)
    return posq[:eng.natoms, :3].astype(np.float64)


_ORACLE = {}


def _key(d, x, disp):
    h = hashlib.sha1()
    for a in (x, d.box if d.box is not None else np.zeros(0), d.charges, d.sigmas, d.epsilons, d.exc_qq, d.exc_sigma, d.exc_eps):
        h.update(np.ascontiguousarray(a, dtype=np.float64).tobytes())
    h.update(repr((d.method, d.cutoff, d.use_switch, d.switch_distance, d.use_dispersion, d.rf_dielectric, disp,
                   d.pme_parameters() if d.box is not None else None)).encode())
    return h.hexdigest()


def oracle_parts(d, x=None, dispersion_coefficient=None):
    """{group: energy} of the restatement at positions x (default d.positions), grouped as the engine's term masks group
    it (GROUPS; a group the system lacks is 0).  Cached per configuration: parameters, box, positions, PME parameters."""
    from oracle import port
    from openmm_b200 import systems
    x = np.asarray(d.positions if x is None else x, dtype=np.float64)
    key = _key(d, x, dispersion_coefficient)
    if key not in _ORACLE:
        pme = d.pme_parameters() if d.method == systems.NB_PME else None
        _, _, parts = port.forces_energy(d, positions=x, pme=pme, dispersion_coefficient=dispersion_coefficient)
        _ORACLE[key] = {g: float(sum(parts.get(p, 0.0) for p in ps)) for g, ps in GROUPS.items()}
    return dict(_ORACLE[key])


def engine_parts(eng, d):
    """{group: energy} of the engine, one compute per term mask, for the groups d has"""
    return {g: eng.compute(MASKS[g]) for g in present(d)}


def present(d):
    from openmm_b200 import systems
    out = ["direct"]
    if d.method == systems.NB_PME:
        out.append("reciprocal")
    for g, k in (("bonds", "bond_i"), ("angles", "angle_i"), ("torsions", "tor_i")):
        if len(getattr(d, k)):
            out.append(g)
    return out


def cutoff_edge_energy(d, x, delta):
    """sum of |pair energy| (PME direct-space Coulomb + LJ, no switch) over the pairs whose distance lies within delta of
    the cutoff in an orthorhombic PME box: pairs that two evaluations rounding their displacement differently may count
    on different sides of the cutoff"""
    from scipy.spatial import cKDTree
    from scipy.special import erfc
    from openmm_b200 import systems
    assert d.method == systems.NB_PME and not d.use_switch and not np.count_nonzero(d.box - np.diag(np.diag(d.box)))
    L = np.diag(d.box)
    y = np.mod(x, L)
    y[y >= L] = 0.0
    p = cKDTree(y, boxsize=L).query_pairs(d.cutoff + delta, output_type="ndarray")
    dd = y[p[:, 1]] - y[p[:, 0]]
    r = np.linalg.norm(dd - L*np.round(dd/L), axis=1)
    m = np.abs(r - d.cutoff) < delta
    i, j, r = p[m, 0], p[m, 1], r[m]
    sr6 = (0.5*(d.sigmas[i] + d.sigmas[j])/r)**6
    e = 138.93545764438198*d.charges[i]*d.charges[j]*erfc(d.pme_parameters()[0]*r)/r + 4*np.sqrt(d.epsilons[i]*d.epsilons[j])*(sr6*sr6 - sr6)
    return float(np.abs(e).sum())
