"""GPU tests of CustomAngleForce (a class of k_custom) and CustomCompoundBondForce (k_compound) on the platform: the
reference's own test bodies; DHFR's harmonic angles as custom angles, and its angles and periodic torsions as compound bonds,
against k_bonded's own; a six-particle orientational restraint on DHFR against the double-precision probe and a finite
difference of the device energy; the continuous coordinates a compound bond reads across a molecule wrap; parameter and global
updates without a new step graph; force groups; NVE drift; launch counts; platform fallback."""
import os
import subprocess
import numpy as np
import pytest
from conftest import ROOT

pytestmark = pytest.mark.gpu
PLUGIN = os.path.join(ROOT, "plugin", "libOpenMMB200.so")
REFTESTS = os.path.join(ROOT, "oracle", "_ref", "tests")


@pytest.fixture(scope="module")
def harness():
    import custom_harness
    if not custom_harness.available() or not os.path.exists(PLUGIN):
        pytest.fail("oracle/_ref or the plugin is not built: run __graft_entry__.build() where /root/reference exists")
    custom_harness.omm.load_plugin(PLUGIN)
    return custom_harness


def _dhfr():
    from openmm_b200 import systems
    return systems.SystemDesc.load(os.path.join(ROOT, "data", "dhfr.npz")).rounded()


def _restrained(harness, d=None, **kw):
    from openmm_b200 import systems
    d = _dhfr() if d is None else d
    return harness.compiled(systems.with_orientational_restraint(d, systems.restraint_atoms(d), **kw))


def _group_close(f, e, fr, er, ftol=1e-5, etol=1e-6):
    assert np.abs(f - fr).max() <= ftol*np.abs(fr).max(), np.abs(f - fr).max()/np.abs(fr).max()
    assert abs(e - er) <= etol*abs(er), (e, er)


# ---------------------------------------------------------------------------------------------------- reference test bodies
@pytest.mark.parametrize("name", ["TestB200CustomAngleForce", "TestB200MixedCustomAngleForce", "TestB200CustomCompoundBondForce",
                                  "TestB200MixedCustomCompoundBondForce"])
def test_reference_own_test_bodies_pass(name):
    exe = os.path.join(REFTESTS, name)
    if not os.path.exists(exe):
        pytest.fail("%s not built (make -C plugin reftests where /root/reference exists)" % exe)
    p = subprocess.run([exe], capture_output=True, text=True, timeout=600, env=dict(os.environ, B200_PLUGIN=PLUGIN))
    assert p.returncode == 0 and "Done" in p.stdout, p.stdout[-2000:] + p.stderr[-2000:]


# ---------------------------------------------------------------------------------------------------- against k_bonded
def test_custom_angles_equal_harmonic_angles(harness):
    from openmm_b200 import Engine, engine, systems
    d = _dhfr()
    ref = Engine(d)
    ea = ref.compute(engine.TERM_ANGLES)
    fa = ref.get_forces()
    c = harness.compiled(systems.angles_to_custom(d))
    assert len(c.cangle_prog) == len(d.angle_i) > 0 and len(c.angle_i) == 0
    cus = Engine(c)
    e = cus.compute(engine.TERM_CUSTOM_ANGLES)
    _group_close(cus.get_forces(), e, fa, ea)
    # the class bits select
    assert cus.compute(engine.TERM_CUSTOM_TORSIONS | engine.TERM_CUSTOM_BONDS | engine.TERM_CUSTOM_COMPOUND) == 0.0


def test_compound_angles_and_torsions_equal_k_bonded(harness):
    from openmm_b200 import Engine, engine, systems
    d = _dhfr()
    ref = Engine(d)
    er = ref.compute(engine.TERM_ANGLES | engine.TERM_TORSIONS)
    fr = ref.get_forces()
    c = harness.compiled(systems.torsions_to_compound(systems.angles_to_compound(d)))
    assert len(c.ccompound_expr) == len(d.angle_i) + len(d.tor_i) and len(c.tor_i) == 0 and len(c.angle_i) == 0
    cus = Engine(c)
    e = cus.compute(engine.TERM_CUSTOM_COMPOUND)
    _group_close(cus.get_forces(), e, fr, er)
    assert cus.compute(engine.TERM_CUSTOM_ANGLES) == 0.0
    assert cus.time_phase("custom_compound", 3) > 0


# ---------------------------------------------------------------------------------------------------- the restraint
def _probe_gradient(harness, r, x):
    """energy and gradient [6,3] of the one restraint term at the positions x [6,3], in double, through the host interpreter"""
    from openmm_b200 import systems
    start, par = r.ccompound_prog_start, r.ccompound_params[0]
    vals = [harness.compound_probe(6, bool(r.ccompound_periodic[0]), start, r.ccompound_op, r.ccompound_arg, r.ccompound_imm, len(par), 0, q,
                          x.reshape(-1), np.asarray(r.box), par, ())[0] for q in range(19)]
    return vals[0], np.array(vals[1:]).reshape(6, 3)


def test_restraint_forces_match_the_probe_and_a_finite_difference(harness):
    from openmm_b200 import Engine, engine, systems
    r = _restrained(harness)
    atoms = r.ccompound_atoms[0, :6]
    eng = Engine(r)
    others = engine.TERM_ALL & ~engine.TERM_CUSTOM_COMPOUND
    eng.compute(others, energy=False)
    f_without = eng.get_forces()
    eng.compute(engine.TERM_ALL, energy=False)
    f_with = eng.get_forces()
    mask = np.ones(r.natoms, bool)
    mask[atoms] = False
    assert np.array_equal(f_with[mask], f_without[mask])          # all other atoms unchanged bit for bit
    e = eng.compute(engine.TERM_CUSTOM_COMPOUND)
    f = eng.get_forces()
    assert np.array_equal(f[mask], np.zeros_like(f[mask]))
    x = eng.get_positions()
    ep, grad = _probe_gradient(harness, r, x[atoms])
    assert abs(e - ep) <= 1e-9*abs(ep), (e, ep)
    assert np.abs(f[atoms] + grad).max() <= 1e-6*np.abs(grad).max(), (f[atoms], -grad)
    assert np.abs(grad).max() > 1.0
    # central finite difference of the device energy (fp32 positions: a step of 2^-10 nm is exactly representable here)
    h = 2.0**-10
    for a in atoms[[0, 3]]:
        for k in range(3):
            ee = []
            for s in (+1, -1):
                y = x.copy()
                y[a, k] = np.float32(y[a, k]) + s*h
                eng.set_positions(y)
                ee.append(eng.compute(engine.TERM_CUSTOM_COMPOUND))
            fd = -(ee[0] - ee[1])/(2*h)
            assert abs(fd - f[a, k]) <= 2e-3*np.abs(grad).max(), (a, k, fd, f[a, k])


def test_restraint_is_continuous_across_a_molecule_wrap(harness):
    """a water oxygen far outside the primary cell is one of the restraint's particles: the list build wraps the water back by
    lattice vectors, the restraint still reads the coordinate the user gave"""
    from openmm_b200 import Engine, engine, systems
    d = _dhfr()
    box = np.asarray(d.box)
    ow = max(m[0] for m in d.molecules() if len(m) == 3)
    x = np.array(d.positions)
    x[[ow, ow + 1, ow + 2]] += 2*box[0] - box[1] + box[2]
    d.positions = x.astype(np.float32).astype(np.float64)
    atoms = systems.restraint_atoms(d)
    atoms[5] = ow
    r = harness.compiled(systems.with_orientational_restraint(d, atoms))
    eng = Engine(r)
    e = eng.compute(engine.TERM_CUSTOM_COMPOUND)
    npad = (d.natoms + 31)//32*32
    offsets = np.frombuffer(eng.checkpoint()[-12*npad:], dtype=np.int32).reshape(3, npad)
    assert (offsets[:, ow] != 0).any(), offsets[:, ow]
    ep, _ = _probe_gradient(harness, r, d.positions[atoms])
    # one fp32 rounding of a coordinate up to 16 nm from the origin is all that may differ
    assert abs(e - ep) <= 2e-4*abs(ep), (e, ep)
    # frozen positions, before and after more rebuilds: the same energy
    eng.set_integrator(systems.INT_VERLET, 0.001)
    builds = eng.stats()["list_builds"]
    xs = eng.get_positions()
    eng.set_positions(xs)
    e1 = eng.compute(engine.TERM_CUSTOM_COMPOUND)
    eng.set_positions(xs)
    e2 = eng.compute(engine.TERM_CUSTOM_COMPOUND)
    assert eng.stats()["list_builds"] > builds
    assert abs(e1 - e2) <= 1e-9*abs(e1) and abs(e1 - e) <= 1e-9*abs(e), (e, e1, e2)


# ---------------------------------------------------------------------------------------------------- updates, groups, steps
def test_parameter_and_global_updates_keep_the_step_graph(harness):
    from openmm_b200 import Engine, engine, systems
    d = _dhfr()
    a = systems.angles_to_custom(d)
    a.cangle_energy = ("lam*" + systems.HARMONIC_CUSTOM_ANGLE,)
    a.custom_global_names, a.custom_global_values = ("lam",), np.array([1.0])
    r = _restrained(harness, a)
    eng = Engine(r)
    eng.set_integrator(systems.INT_LANGEVIN_MIDDLE, 0.001, 300.0, 1.0, 7)
    eng.step(3)
    n0 = eng.stats()["graph_instantiations"]
    bits = engine.TERM_CUSTOM_ANGLES | engine.TERM_CUSTOM_COMPOUND
    e0a, e0c = eng.compute(engine.TERM_CUSTOM_ANGLES), eng.compute(engine.TERM_CUSTOM_COMPOUND)
    pa = r.cangle_params.copy()
    pa[:, 0] *= 2.0
    pc = r.ccompound_params.copy()
    pc[:, :3] *= 3.0
    eng.update_custom_angle_params(pa)
    eng.update_custom_compound_params(pc)
    assert abs(eng.compute(engine.TERM_CUSTOM_ANGLES) - 2*e0a) <= 1e-9*abs(e0a)
    assert abs(eng.compute(engine.TERM_CUSTOM_COMPOUND) - 3*e0c) <= 1e-9*abs(e0c)
    eng.set_custom_globals([0.5])
    assert abs(eng.compute(bits) - (e0a + 3*e0c)) <= 1e-9*abs(e0a + 3*e0c)
    eng.step(2)
    assert eng.stats()["graph_instantiations"] == n0
    with pytest.raises(engine.EngineError, match="number of angles has changed"):
        eng.update_custom_angle_params(pa[:-1])
    with pytest.raises(engine.EngineError, match="number of bonds has changed"):
        eng.update_custom_compound_params(np.concatenate([pc, pc]))


def test_two_objects_in_different_force_groups(harness):
    from openmm_b200 import Engine, engine, systems
    d = _dhfr()
    atoms = systems.restraint_atoms(d)
    r = systems.with_orientational_restraint(d, atoms)
    r = harness.compiled(systems.with_orientational_restraint(r, atoms[::-1].copy(), kr=1000.0))
    c = harness.compiled(systems.angles_to_custom(r))
    n = len(c.cangle_prog)
    eng = Engine(c, bonded_groups={"custom_compound": [3, 4], "custom_angles": [5]*(n//2) + [6]*(n - n//2)})
    bits = engine.TERM_CUSTOM_ANGLES | engine.TERM_CUSTOM_COMPOUND
    parts = [eng.compute_groups(bits, 1 << g) for g in (3, 4, 5, 6)]
    assert all(p != 0.0 for p in parts) and parts[0] != parts[1]
    assert abs(sum(parts) - eng.compute(bits)) <= 1e-9*abs(sum(parts))
    assert eng.compute_groups(bits, 1) == 0.0


def _nve_drift(d, steps=2000):
    from openmm_b200 import Engine, systems
    eng = Engine(d)
    eng.set_integrator(systems.INT_VERLET, 0.001)
    eng.set_velocities(np.random.default_rng(3).standard_normal((d.natoms, 3))*0.4)
    eng.step(100)
    e0 = eng.compute() + eng.kinetic_energy()
    eng.step(steps)
    e1 = eng.compute() + eng.kinetic_energy()
    eng.close()
    return abs(e1 - e0)/d.natoms


def test_nve_with_the_restraint_drifts_no_more_than_without(harness):
    d = _dhfr()
    plain, restrained = _nve_drift(d), _nve_drift(_restrained(harness, d))
    print("NVE |dE| per atom over 2,000 steps of 1 fs, kJ/mol: plain %.3e, restrained %.3e" % (plain, restrained))
    # margin: as much again as the unrestrained run's own drift, plus 1e-4 kJ/mol per atom for run-to-run differences
    assert restrained <= 2*plain + 1e-4, (plain, restrained)


def _eval_launches(eng):
    from openmm_b200 import engine
    eng.compute(engine.TERM_ALL, energy=False)
    before = eng.stats()["kernel_launches"]
    eng.compute(engine.TERM_ALL, energy=False)
    return eng.stats()["kernel_launches"] - before


def _step_launches(eng):
    eng.step(1)
    before = eng.stats()["kernel_launches"]
    eng.step(1)
    return eng.stats()["kernel_launches"] - before


def test_launch_counts(harness):
    """custom angles alone launch what custom torsions alone launch (k_custom once); compound bonds one more kernel"""
    from openmm_b200 import Engine, systems
    d = _dhfr()
    counts, steps = {}, {}
    for name, desc in (("plain", d), ("torsions", harness.compiled(systems.periodic_to_custom(d))),
                       ("angles", harness.compiled(systems.angles_to_custom(d))), ("restraint", _restrained(harness, d)),
                       ("angles+restraint", _restrained(harness, systems.angles_to_custom(d)))):
        eng = Engine(desc)
        counts[name] = _eval_launches(eng)
        eng.set_integrator(systems.INT_LANGEVIN_MIDDLE, 0.002, 300.0, 1.0, 7)
        steps[name] = _step_launches(eng)
        eng.close()
    assert counts["angles"] == counts["torsions"] == counts["plain"] + 1, counts
    assert counts["restraint"] == counts["plain"] + 1 and counts["angles+restraint"] == counts["angles"] + 1, counts
    assert steps["angles"] == steps["torsions"] == steps["plain"] + 1 and steps["restraint"] == steps["plain"] + 1, steps
    assert steps["angles+restraint"] == steps["plain"] + 2, steps


# ---------------------------------------------------------------------------------------------------- through the plugin
def test_through_the_plugin_matches_reference_platform(harness):
    from openmm_b200 import systems
    d = _restrained(harness, systems.angles_to_custom(_dhfr()))
    groups = {"custom_angles": 5, "custom_compound": 6}
    ref = harness.Simulation(d, "Reference", pme=d.pme_parameters(), force_groups=groups)
    b200 = harness.Simulation(d, "B200", pme=d.pme_parameters(), force_groups=groups)
    assert b200.platform() == "B200"
    for mask in (1 << 5, 1 << 6, (1 << 5) | (1 << 6)):
        (f, e), (fr, er) = b200.forces_energy(mask), ref.forces_energy(mask)
        _group_close(f, e, fr, er)
    # updateParametersInContext
    pa = d.cangle_params.copy()
    pa[:, 0] *= 0.5
    pc = d.ccompound_params.copy()
    pc[:, 3:] += 0.02
    for s in (ref, b200):
        s.update("cangle", 0, d.cangle_atoms, pa)
        s.update("ccompound", 0, d.ccompound_atoms[:, :6], pc)
    (f, e), (fr, er) = b200.forces_energy((1 << 5) | (1 << 6)), ref.forces_energy((1 << 5) | (1 << 6))
    _group_close(f, e, fr, er)
    with pytest.raises(RuntimeError, match="set of particles in a bond has changed"):
        b200.update("ccompound", 0, d.ccompound_atoms[:, :6][:, ::-1], pc)
    with pytest.raises(RuntimeError, match="number of angles has changed"):
        b200.update("cangle", 0, np.concatenate([d.cangle_atoms, d.cangle_atoms[:1]]), np.concatenate([pa, pa[:1]]))


def _small(energy, particles, names=(), tabulated=False):
    from openmm_b200 import systems
    n, particles = max(particles, 2), min(particles, 8)
    x = np.random.default_rng(1).uniform(0, 1, (n, 3)).astype(np.float32).astype(np.float64)
    bare = systems.SystemDesc(masses=np.full(n, 12.0), charges=np.zeros(n), sigmas=np.full(n, 0.3), epsilons=np.zeros(n), positions=x,
                              box=None, method=systems.NB_NOCUTOFF, use_dispersion=False)
    return systems._add_compound(bare, energy, names, particles, False, np.arange(particles).reshape(1, -1), np.zeros((1, len(names))))


@pytest.mark.parametrize("case,match", [("tabulated", "tabulated functions in a CustomCompoundBondForce"),
                                        ("nine particles", "more than 8 particles per bond"),
                                        ("derivative", "energy parameter derivatives of a CustomCompoundBondForce")])
def test_unsupported_compound_forces_move_the_context_elsewhere(harness, case, match):
    from openmm_b200 import systems
    kw = {}
    if case == "tabulated":
        d, kw = _small("fn(distance(p1,p2))", 2), dict(tabulated=True)
    elif case == "nine particles":
        d = _small("+".join("x%d" % i for i in range(1, 10)), 9)
        d.ccompound_particles, d.ccompound_atoms = np.array([9], dtype=np.int32), np.arange(9).reshape(1, 9)
    else:
        d = _small("lam*distance(p1,p2)", 2)
        d.custom_global_names, d.custom_global_values = ("lam",), np.array([1.0])
        kw = dict(deriv_params={"custom_compound": "lam"})
    s = harness.Simulation(d, "Reference", **kw)
    assert s.default_platform() not in ("", "B200")
    with pytest.raises(RuntimeError, match=match):
        harness.Simulation(d, "B200", **kw)
