"""The fused integrate kernel on a system that mixes every kind of integration unit: SETTLE waters, SHAKE clusters of a
centre and 1, 2 or 3 hydrogens, free atoms and a massless (frozen) atom, 125 units in all (not a multiple of the 64 units
a block takes).  The kernel maps each unit onto a group of lanes, one lane per atom; Verlet and Langevin runs must
reproduce, bit for bit, the trajectories of the kernel that took one thread per unit (tests/golden/integrate_lanes.npz, written by
tests/golden/make_golden_integrate_lanes.py), keep the constraints and keep the centre-of-mass momentum at zero."""
import os
import numpy as np
import pytest
from conftest import GOLDEN

pytestmark = pytest.mark.gpu

STEPS = 200
DT = 0.002
TOL = {"single": 1e-5, "mixed": 1e-10}
KINDS = {"verlet": 0, "langevin": 1, "langevin_middle": 2}


def mixed_units_system():
    """water_box(5) with every 4th water replaced by a CH3, CH2 or CH group (C-H constrained, 0.109 nm) or an ion, one of
    the ions massless; cm_frequency 1."""
    from openmm_b200 import systems
    w = systems.water_box(5, cutoff=0.7)
    nw = len(w.masses)//3
    dirs = np.array([[1, 1, 1], [1, -1, -1], [-1, 1, -1]], dtype=float)/np.sqrt(3.0)
    m, q, s, e, x = [], [], [], [], []
    exc, con = [], []
    d_oh = 0.09572
    d_hh = 2*d_oh*np.sin(np.radians(104.52)/2)
    replaced = 0
    for k in range(nw):
        o = w.positions[3*k]
        if k % 4 != 3:
            b = len(m)
            m += list(w.masses[3*k:3*k+3]); q += list(w.charges[3*k:3*k+3]); s += list(w.sigmas[3*k:3*k+3])
            e += list(w.epsilons[3*k:3*k+3]); x += list(w.positions[3*k:3*k+3])
            exc += [(b, b+1), (b, b+2), (b+1, b+2)]
            con += [(b, b+1, d_oh), (b, b+2, d_oh), (b+1, b+2, d_hh)]
            continue
        nh = replaced % 4                  # 0: an ion, 1..3: a centre with nh hydrogens
        b = len(m)
        if nh == 0:
            m.append(0.0 if replaced == 8 else 22.99); q.append(0.0); s.append(0.33); e.append(0.5); x.append(o)
        else:
            m.append(12.011); q.append(-0.05*nh); s.append(0.34); e.append(0.36); x.append(o)
            for h in range(nh):
                m.append(1.008); q.append(0.05); s.append(1.0); e.append(0.0); x.append(o + 0.109*dirs[h])
                con.append((b, b+1+h, 0.109))
            atoms = list(range(b, b+1+nh))
            exc += [(i, j) for a, i in enumerate(atoms) for j in atoms[a+1:]]
        replaced += 1
    exc = np.array(exc, dtype=np.int32)
    con_i = np.array([c[0] for c in con], dtype=np.int32)
    con_j = np.array([c[1] for c in con], dtype=np.int32)
    con_d = np.array([c[2] for c in con])
    d = systems.SystemDesc(masses=np.array(m), charges=np.array(q), sigmas=np.array(s), epsilons=np.array(e),
                           positions=np.array(x), box=w.box, method=systems.NB_PME, cutoff=0.7, ewald_tol=w.ewald_tol,
                           exc_i=exc[:, 0].copy(), exc_j=exc[:, 1].copy(), exc_qq=np.zeros(len(exc)),
                           exc_sigma=np.ones(len(exc)), exc_eps=np.zeros(len(exc)), con_i=con_i, con_j=con_j, con_d=con_d,
                           cm_frequency=1, name="mixed_units")
    return d.rounded()


def run(kind, precision, cm_frequency=1):
    """STEPS steps of `kind` from seeded velocities; returns (positions, velocities) as the engine hands them out."""
    from openmm_b200 import Engine
    d = mixed_units_system()
    d.cm_frequency = cm_frequency
    eng = Engine(d, precision=precision)
    eng.set_integrator(KINDS[kind], DT, 300.0, 1.0, 7, TOL[precision])
    v = np.random.default_rng(5).standard_normal((d.natoms, 3))*0.5
    v[d.masses == 0] = 0.0
    eng.set_velocities(v)
    eng.apply_constraints(TOL[precision])
    eng.apply_velocity_constraints(TOL[precision])
    eng.step(STEPS)
    eng.synchronize()
    out = eng.get_positions(), eng.get_velocities()
    eng.close()
    return out


def test_system_has_every_unit_kind():
    """Host-side: the system really holds SETTLE waters, SHAKE clusters of 2, 3 and 4 atoms, free atoms and a massless atom,
    and its unit count is not a multiple of the 64 units of a block."""
    d = mixed_units_system()
    deg = np.bincount(np.concatenate([d.con_i, d.con_j]), minlength=d.natoms)
    centres = [i for i in range(d.natoms) if d.masses[i] == 12.011]
    sizes = sorted(set(int(deg[c]) + 1 for c in centres))
    waters = int((d.masses == 15.9994).sum())
    free = int((deg == 0).sum())
    assert sizes == [2, 3, 4] and waters > 0 and free > 1 and (d.masses == 0).sum() == 1
    units = waters + len(centres) + free
    assert units % 64 != 0


@pytest.mark.parametrize("precision", ["single", "mixed"])
@pytest.mark.parametrize("kind", ["verlet", "langevin"])
def test_trajectory_matches_one_thread_per_unit(kind, precision):
    gold = np.load(os.path.join(GOLDEN, "integrate_lanes.npz"))
    x, v = run(kind, precision)
    key = "%s_%s" % (kind, precision)
    assert np.isfinite(x).all() and np.isfinite(v).all()
    assert np.array_equal(x, gold["x_" + key]), np.abs(x - gold["x_" + key]).max()
    assert np.array_equal(v, gold["v_" + key]), np.abs(v - gold["v_" + key]).max()


def test_langevin_middle_follows_one_thread_per_unit_in_double():
    """LangevinMiddle is not bit-identical to the one-thread-per-unit kernel: after 200 mixed-precision steps positions
    differ by 8e-14 nm (a last-bit difference early on; in fp32 the same difference grows chaotically).  In double it must
    stay at that level."""
    gold = np.load(os.path.join(GOLDEN, "integrate_lanes.npz"))
    x, v = run("langevin_middle", "mixed")
    assert np.abs(x - gold["x_langevin_middle_mixed"]).max() < 1e-11
    assert np.abs(v - gold["v_langevin_middle_mixed"]).max() < 1e-8


@pytest.mark.parametrize("precision", ["single", "mixed"])
@pytest.mark.parametrize("kind", list(KINDS))
def test_constraints_and_centre_of_mass(kind, precision):
    """Every constraint holds to the tolerance, and the removal every step keeps the total momentum at what one step adds
    after the last removal.  For Verlet that is one step's net force (the frozen atom and PME's reciprocal space do not
    sum to zero), far below the momentum of the same run without the removal (initial velocities plus 200 steps of it);
    the Langevin kinds add one step of noise (6 sigma per component)."""
    d = mixed_units_system()
    x, v = run(kind, precision)
    r = np.linalg.norm(x[d.con_i] - x[d.con_j], axis=1)
    bound = 2e-5 if precision == "single" else 1e-9
    assert np.abs(r/d.con_d - 1).max() <= bound
    m = d.masses[:, None]
    p = np.abs((m*v).sum(axis=0)).max()
    if kind == "verlet":
        _, v0 = run(kind, precision, cm_frequency=0)
        p0 = np.abs((m*v0).sum(axis=0)).max()
        assert p <= 0.05*p0, (p, p0)
    else:
        kT = 0.0083144626*300.0
        sigma = np.sqrt((d.masses*kT).sum()*(1.0 - np.exp(-2.0*DT)))
        assert p <= 6.0*sigma, (p, sigma)
