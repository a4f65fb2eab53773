"""CustomNonbondedForce on the GPU: the reference's own test bodies in single and mixed precision; DHFR with its Lennard-Jones in
a CustomNonbondedForce of Discrete2DFunction tables (DHFR-LJ-table, and DHFR-NBFIX with overridden pairs and a switching
function) through the plugin against the live Reference platform, fresh and after 200 Langevin steps; the same forces as DHFR
with its Lennard-Jones in the NonbondedForce; force groups, parameter updates, global parameters and box changes through the
long-range correction; reproducibility; and the Systems the platform refuses, which fall back to another platform."""
import os
import subprocess

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PLUGIN = os.path.join(ROOT, "plugin", "libOpenMMB200.so")
REFTESTS = os.path.join(ROOT, "oracle", "_ref", "tests")
FORCE_BAR, ENERGY_BAR = 1e-4, 1e-5


@pytest.fixture(scope="module")
def H():
    import custom_nonbonded_harness
    if not custom_nonbonded_harness.available() or not os.path.exists(PLUGIN):
        pytest.fail("oracle/_ref or the plugin is not built: run __graft_entry__.build() where the reference sources exist")
    custom_nonbonded_harness.omm.load_plugin(PLUGIN)
    return custom_nonbonded_harness


def _pair(H, d, forces, precision="single", **kw):
    pme = d.pme_parameters()
    ref = H.Simulation(d, "Reference", forces=forces, pme=pme, **kw)
    b200 = H.Simulation(d, "B200", forces=forces, pme=pme, props="Precision=" + precision, **kw)
    assert b200.platform() == "B200"
    return ref, b200


def _fp32(x):
    return np.asarray(x, dtype=np.float64).astype(np.float32).astype(np.float64)


def _compare(H, ref, b200, groups=-1, forces=True):
    fr, er = ref.forces_energy(groups)
    fb, eb = b200.forces_energy(groups)
    if forces:
        err = H.force_error(fb, fr)
        assert err < FORCE_BAR, (err, eb, er)
    assert abs(eb - er) <= ENERGY_BAR*max(1.0, abs(er)), (eb, er)
    return fb, eb


# After 200 steps in mixed precision, or on DHFR scaled by 1.01, the NonbondedForce's fp32 PME path alone is 2-3e-4 from the
# Reference platform by force_error (the same with or without a CustomNonbondedForce in the System): there the whole System is
# held to the energy bar and the CustomNonbondedForce's group to both bars.


@pytest.mark.parametrize("name", ["TestB200CustomNonbondedForce", "TestB200MixedCustomNonbondedForce"])
def test_reference_test_bodies(H, name):
    exe = os.path.join(REFTESTS, name)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=900, env=dict(os.environ, B200_PLUGIN=PLUGIN))
    assert r.returncode == 0 and r.stdout.rstrip().endswith("Done"), r.stdout[-3000:] + r.stderr[-2000:]


@pytest.mark.parametrize("precision", ["single", "mixed"])
@pytest.mark.parametrize("nbfix", [False, True])
def test_dhfr_tables_match_reference_fresh_and_aged(H, nbfix, precision):
    """the whole System and the CustomNonbondedForce's group alone, before and after 200 Langevin steps on the GPU"""
    d, f = H.dhfr_lj_table(nbfix)
    ref, b200 = _pair(H, d, [f], precision, integrator=(1, 300.0, 1.0, 0.002))
    _compare(H, ref, b200)
    _compare(H, ref, b200, groups=1 << H.CNB_GROUP)
    b200.step(200)
    # the pair kernel reads the fp32 coordinates (in mixed precision the hi part): the Reference platform gets those
    ref.set_positions(_fp32(b200.state(positions=True)["positions"]))
    _compare(H, ref, b200, forces=False)
    _compare(H, ref, b200, groups=1 << H.CNB_GROUP)


def test_same_forces_as_lennard_jones_in_the_nonbonded_force(H):
    from openmm_b200 import systems
    d, f = H.dhfr_lj_table()
    table = H.Simulation(d, "B200", forces=[f], pme=d.pme_parameters())
    plain = systems.SystemDesc.load(H.DHFR).rounded()
    lj = H.Simulation(plain, "B200", pme=plain.pme_parameters())
    ft, _ = table.forces_energy()
    fl, _ = lj.forces_energy()
    assert H.force_error(ft, fl) < FORCE_BAR


def test_many_types_and_a_global(H):
    """60 random types (a 60 x 60 table) and a global scale in the expression: forces and energies, and the long-range
    correction recomputed when the global changes"""
    d, f = H.dhfr_lj_table()
    rng = np.random.default_rng(3)
    n = 60
    sig, eps = rng.uniform(0.15, 0.4, n), rng.uniform(0.05, 1.0, n)
    s, e = 0.5*(sig[:, None] + sig[None, :]), np.sqrt(eps[:, None]*eps[None, :])
    f.tables = {"acoef": 4*e*s**12, "bcoef": 4*e*s**6}
    f.params = rng.integers(0, n, size=(d.natoms, 1)).astype(np.float64)
    f.energy = "scale*(" + H.LJ_TABLE + ")"
    f.globals = {"scale": 1.0}
    ref, b200 = _pair(H, d, [f])
    _compare(H, ref, b200, groups=1 << H.CNB_GROUP)
    _, e1 = b200.forces_energy(1 << H.CNB_GROUP)
    for sim in (ref, b200):
        sim.set_parameter("scale", 0.5)
    _, e2 = _compare(H, ref, b200, groups=1 << H.CNB_GROUP)
    assert abs(e2 - 0.5*e1) <= ENERGY_BAR*abs(e1)


def test_parameter_update_and_box_change(H):
    d, f = H.dhfr_lj_table(nbfix=True)
    ref, b200 = _pair(H, d, [f])
    _compare(H, ref, b200)
    types = f.params.copy()
    rng = np.random.default_rng(9)
    pick = rng.choice(d.natoms, 500, replace=False)
    types[pick, 0] = rng.integers(0, int(types.max()) + 1, size=500)
    b200.update_custom_nonbonded(0, types)
    # a fresh Reference Context with the new types: the Reference kernel's own update shares the tabulated functions of its
    # copy of the force with the force itself, and both delete them
    f.params = types
    ref = H.Simulation(d, "Reference", forces=[f], pme=d.pme_parameters())
    _compare(H, ref, b200)
    # the long-range correction follows the volume: coefficient/V at the new box
    box = np.asarray(d.box, dtype=np.float64)*1.01
    x = _fp32(np.asarray(d.positions)*1.01)
    for sim in (ref, b200):
        sim.set_box(box)
        sim.set_positions(x)
    _compare(H, ref, b200, forces=False)
    _compare(H, ref, b200, groups=1 << H.CNB_GROUP)


def test_bit_reproducible(H):
    d, f = H.dhfr_lj_table(nbfix=True)
    a = H.Simulation(d, "B200", forces=[f], pme=d.pme_parameters())
    b = H.Simulation(d, "B200", forces=[f], pme=d.pme_parameters())
    g = 1 << H.CNB_GROUP
    fa1, _ = a.forces_energy(g)
    fa2, _ = a.forces_energy(g)
    fb, _ = b.forces_energy(g)
    assert np.array_equal(fa1, fa2) and np.array_equal(fa1, fb)


def _small(H, systems, **kw):
    """four argon-like particles with a NoCutoff NonbondedForce of zero charges, and a matching CustomNonbondedForce"""
    n = 4
    x = np.array([[0, 0, 0], [0.4, 0, 0], [0, 0.5, 0], [0, 0, 0.6]], dtype=np.float64)
    small = systems.SystemDesc(masses=np.full(n, 40.0), charges=np.zeros(n), sigmas=np.full(n, 0.3), epsilons=np.zeros(n),
                               positions=x, method=systems.NB_NOCUTOFF, cutoff=1.0)
    f = H.Force("4*((0.3/r)^12-(0.3/r)^6)*a1*a2", ["a"], np.ones((n, 1)), 0, 1.0, lrc=False, **kw)
    return small, f


@pytest.mark.parametrize("case", ["matching", "interaction_group", "derivative", "continuous", "two_cutoffs", "exclusions",
                                  "method", "too_many_params", "nb_cutoff", "object_exclusions"])
def test_fallback(H, case):
    from openmm_b200 import systems
    d, f = _small(H, systems)
    forces = [f]
    if case == "two_cutoffs":
        d.method = systems.NB_CUTOFF_NONPERIODIC
        f.method = 1
        forces = [f, H.Force("r", [], np.zeros((d.natoms, 0)), 1, 0.9, lrc=False)]
    if case == "exclusions":
        f.exclusions = np.array([[0, 1]], dtype=np.int32)
    if case == "method":
        f.method = 1
    if case == "nb_cutoff":
        d.method, f.method, f.cutoff = systems.NB_CUTOFF_NONPERIODIC, 1, 0.95
    if case == "object_exclusions":
        forces = [f, H.Force("r", [], np.zeros((d.natoms, 0)), 0, 1.0, lrc=False, group=3, exclusions=[[0, 1]])]
    if case == "too_many_params":
        f.names = ["p%d" % k for k in range(9)]
        f.params = np.ones((d.natoms, 9))
        f.energy = "r*(" + "+".join("p%d1*p%d2" % (k, k) for k in range(9)) + ")"
    s = H.Simulation(d, "Reference", forces=forces)
    L, idx = H.lib(), s.cnb_index[0]
    if case == "interaction_group":
        a, b = np.array([0, 1], dtype=np.int32), np.array([2, 3], dtype=np.int32)
        assert L.cnbc_add_interaction_group(s.sys, idx, 2, H._ip(a), 2, H._ip(b)) == 0
    if case == "derivative":
        f2 = H.Force("g*r", [], np.zeros((d.natoms, 0)), 0, 1.0, lrc=False, globals_={"g": 1.0}, group=3)
        idx2 = f2.add_to(s.sys)
        assert L.cnbc_add_derivative(s.sys, idx2, b"g") == 0
    if case == "continuous":
        assert L.cnbc_add_continuous(s.sys, idx, b"smooth") == 0
    platform = s.default_platform()
    if case == "matching":
        assert platform == "B200"
    else:
        assert platform not in ("", "B200"), platform


# ---------------------------------------------------------------- the engine (Python mirror) against the Reference goldens
def _golden(H, nbfix):
    g = np.load(H.GOLDEN)
    k = "nbfix" if nbfix else "lj_table"
    return g[k + "_forces"], float(g[k + "_energy"])


@pytest.mark.parametrize("nbfix", [False, True])
def test_engine_matches_reference_goldens(H, nbfix):
    from openmm_b200 import Engine, engine
    eng = Engine(H.engine_desc(nbfix))
    e = eng.compute(engine.TERM_CUSTOM_NONBONDED)
    f = eng.get_forces()
    fr, er = _golden(H, nbfix)
    assert H.force_error(f, fr) < FORCE_BAR
    assert abs(e - er) <= ENERGY_BAR*abs(er), (e, er)
    # the group mask selects the object's group only
    eng.compute_groups(engine.TERM_CUSTOM_NONBONDED, groups=1 << H.CNB_GROUP)
    assert H.force_error(eng.get_forces(), fr) < FORCE_BAR
    eng.close()


def test_engine_update_keeps_the_step_graph(H):
    """updateParametersInContext's path: new types into the same buffers give the forces of an engine built with those types, to a
    few units of 2^-32 (the two engines' lists put the atoms in different tiles, and each lane's double partial sum is rounded to
    the 2^-32 fixed point on its own); after the original types go back, the steps run on with no new graph instantiation (dynamics is not run with
    the random types, which put large Lennard-Jones spheres on bonded hydrogens)"""
    from openmm_b200 import Engine, engine, systems
    d = H.engine_desc(True)
    eng = Engine(d)
    eng.set_integrator(systems.INT_LANGEVIN_MIDDLE, 0.002, 300.0, 1.0, 7)
    eng.step(20)
    eng.synchronize()
    before = eng.stats()["graph_instantiations"]
    p = d.cnb_params.copy()
    rng = np.random.default_rng(4)
    pick = rng.choice(d.natoms, 500, replace=False)
    p[0, pick, 0] = rng.integers(0, int(p.max()) + 1, size=500)
    eng.update_custom_nonbonded_params(p)
    x = eng.get_positions()
    eng.compute(engine.TERM_CUSTOM_NONBONDED, energy=False)
    f1 = eng.get_forces()
    eng.update_custom_nonbonded_params(d.cnb_params)
    eng.step(20)
    eng.synchronize()
    assert eng.stats()["graph_instantiations"] == before
    eng.close()
    d.cnb_params = p
    d.positions = x
    fresh = Engine(d)
    fresh.compute(engine.TERM_CUSTOM_NONBONDED, energy=False)
    assert H.force_error(f1, fresh.get_forces()) < 64*2.0**-32
    fresh.close()


def test_launch_counts(H):
    """one launch more per evaluation and per step with a CustomNonbondedForce; none without one (the same System without the
    cnb_* fields launches what DHFR launches)"""
    from openmm_b200 import Engine, systems

    def counts(d):
        eng = Engine(d)
        eng.compute()
        a = eng.stats()["kernel_launches"]
        eng.compute()
        per_eval = eng.stats()["kernel_launches"] - a
        eng.set_integrator(systems.INT_VERLET, 0.001)
        eng.step(10)
        eng.synchronize()
        a = eng.stats()["kernel_launches"]
        eng.step(10)
        eng.synchronize()
        per_step = (eng.stats()["kernel_launches"] - a)/10
        eng.close()
        return per_eval, per_step

    with_cnb = counts(H.engine_desc())
    without = counts(H.dhfr_lj_table()[0])
    dhfr = counts(systems.SystemDesc.load(H.DHFR).rounded())
    assert without == dhfr
    assert with_cnb[0] == dhfr[0] + 1 and with_cnb[1] == dhfr[1] + 1, (with_cnb, dhfr)


def test_phase_timing(H):
    from openmm_b200 import Engine
    eng = Engine(H.engine_desc())
    assert eng.time_phase("custom_nonbonded", 3) > 0.0
    eng.close()


def _nve_drift(d, steps=2000, every=100):
    """|drift| per atom of the total energy over `steps` Verlet steps of 1 fs (slope of a fitted line times the span), as the
    generalized Born tests measure it"""
    from openmm_b200 import Engine, systems
    eng = Engine(d)
    eng.set_integrator(systems.INT_VERLET, 0.001)
    eng.set_velocities(np.random.default_rng(3).standard_normal((d.natoms, 3))*0.4)
    eng.apply_velocity_constraints()
    eng.step(100)
    e = []
    for _ in range(steps//every + 1):
        e.append(eng.compute() + eng.kinetic_energy())
        eng.step(every)
    eng.close()
    e = np.array(e)/d.natoms
    return abs(np.polyfit(np.arange(len(e)), e, 1)[0]*(len(e) - 1))


def test_nve_drift_no_worse_than_dhfr(H):
    from openmm_b200 import systems
    plain = _nve_drift(systems.SystemDesc.load(H.DHFR).rounded())
    table = _nve_drift(H.engine_desc())
    print("NVE drift per atom over 2,000 steps of 1 fs, kJ/mol: DHFR %.3e, DHFR-LJ-table %.3e" % (plain, table))
    assert table <= 2*plain + 1e-4, (plain, table)


def test_barostat_moves_see_the_new_volume(H):
    """Monte Carlo barostat moves through the engine calls ApplyMonteCarloBarostatKernel makes (scale the molecules, set the
    scaled box; restore and set the old box on rejection): the group energy, pairs and coefficient/volume, matches the Reference
    platform at each new volume"""
    from openmm_b200 import Engine, engine
    d = H.engine_desc(True)
    eng = Engine(d)
    box0 = np.asarray(d.box, dtype=np.float64)
    eng.set_barostat_molecules()
    _, f = H.dhfr_lj_table(True)
    ref = H.Simulation(d, "Reference", forces=[f], pme=d.pme_parameters())
    for s, accept in ((1.004, False), (0.996, True), (1.002, True)):
        box = eng.get_box()
        eng.scale_coordinates(s, s, s)
        eng.set_box(np.asarray(box)*s)
        e = eng.compute(engine.TERM_CUSTOM_NONBONDED)
        ref.set_box(np.asarray(box)*s)
        ref.set_positions(_fp32(eng.get_positions()))
        _, er = ref.forces_energy(1 << H.CNB_GROUP)
        assert abs(e - er) <= ENERGY_BAR*abs(er), (s, e, er)
        if not accept:
            eng.restore_coordinates()
            eng.set_box(box)
    assert not np.allclose(eng.get_box(), box0)
    eng.close()

