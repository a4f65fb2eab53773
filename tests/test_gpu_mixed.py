"""GPU tests of mixed precision (b200md_set_precision, Engine(precision="mixed"), Precision=mixed on the plugin): positions
as fp32 hi + lo, velocities, integration and constraints in double, forces from the fp32 hi part as in single precision.
Every check here is one that the single-precision state fails or only meets loosely."""
import os
import subprocess
import numpy as np
import pytest
from conftest import relative_force_error, GOLDEN, ROOT

pytestmark = pytest.mark.gpu
PLUGIN = os.path.join(ROOT, "plugin", "libOpenMMB200.so")
REFTESTS = os.path.join(ROOT, "oracle", "_ref", "tests")


def _load(name, rounded=False):
    from openmm_b200 import systems
    d = systems.SystemDesc.load(os.path.join(ROOT, "data", name + ".npz"))
    return d.rounded() if rounded else d


def _constraint_error(x, d):
    return np.abs(np.linalg.norm(x[d.con_i] - x[d.con_j], axis=1)/d.con_d - 1).max()


def test_precision_is_reported_and_validated():
    from openmm_b200 import systems, Engine
    d = systems.water_box(5, cutoff=0.75).rounded()
    assert Engine(d).precision == "single"
    assert Engine(d, precision="mixed").precision == "mixed"
    with pytest.raises(ValueError):
        Engine(d, precision="double")


def test_state_round_trip_keeps_double_values():
    from openmm_b200 import Engine
    d = _load("dhfr")                                   # unrounded: not representable in fp32
    v = np.random.default_rng(1).standard_normal((d.natoms, 3))*0.7
    err = {}
    for p in ("single", "mixed"):
        eng = Engine(d, precision=p)
        eng.set_velocities(v)
        err[p] = (np.abs(eng.get_positions() - d.positions).max(), eng.get_velocities())
    assert err["mixed"][0] < 1e-12
    assert np.array_equal(err["mixed"][1], v)
    assert err["single"][0] > 1e-8 and not np.array_equal(err["single"][1], v)


def test_forces_are_those_of_single_precision_at_the_same_posq():
    from openmm_b200 import Engine
    d = _load("dhfr", rounded=True)
    res = []
    for p in ("single", "single", "mixed"):
        eng = Engine(d, precision=p)
        e = eng.compute()
        res.append((eng.get_forces(), e))
    spread_f = np.abs(res[0][0] - res[1][0]).max()
    spread_e = abs(res[0][1] - res[1][1])
    assert np.abs(res[2][0] - res[0][0]).max() <= spread_f
    assert abs(res[2][1] - res[0][1]) <= max(spread_e, 1e-9*abs(res[0][1]))


def _free_particles():
    """64 particles that feel no force (charge 0, epsilon 0, CutoffPeriodic), every coordinate in [2, 4) nm."""
    from openmm_b200 import systems
    n = 64
    rng = np.random.default_rng(7)
    x = 2.0 + 2.0*rng.random((n, 3))
    return systems.SystemDesc(masses=np.full(n, 12.0), charges=np.zeros(n), sigmas=np.full(n, 0.3), epsilons=np.zeros(n),
                              positions=x, box=np.diag([6.0, 6.0, 6.0]), method=systems.NB_CUTOFF_PERIODIC, cutoff=1.0,
                              use_dispersion=False)


def test_sub_ulp_motion_accumulates():
    """1e-8 nm per step is far below half an fp32 ulp at 2-4 nm (1.2e-7 nm): the single-precision state never moves."""
    from openmm_b200 import systems, Engine
    d = _free_particles()
    v = np.full((d.natoms, 3), 1e-5)
    out = {}
    for p in ("single", "mixed"):
        eng = Engine(d, precision=p)
        eng.set_integrator(systems.INT_VERLET, 0.001, 0.0, 0.0, 0, 1e-6)
        eng.set_velocities(v)
        eng.step(2000)
        out[p] = eng.get_positions()
    x0 = d.positions
    assert np.abs(out["mixed"] - (x0 + v*2.0)).max() < 1e-10
    assert np.array_equal(out["single"], x0.astype(np.float32).astype(np.float64))


@pytest.mark.parametrize("all_bonds", [False, True])
def test_constraints_hold_in_double(all_bonds):
    """DHFR with HBonds (SETTLE + SHAKE clusters) and with AllBonds (CCMA) at tolerance 1e-10: 1e-9 relative after
    applyConstraints and after 200 Langevin steps of 2 fs."""
    from openmm_b200 import systems, Engine
    from test_gpu_parity import _all_bonds
    d = _load("dhfr")
    if all_bonds:
        d = _all_bonds(systems, d)
    eng = Engine(d, precision="mixed")
    eng.set_integrator(systems.INT_LANGEVIN, 0.002, 300.0, 1.0, 5, 1e-10)
    eng.apply_constraints(1e-10)
    assert _constraint_error(eng.get_positions(), d) <= 1e-9
    eng.step(200)
    x = eng.get_positions()
    assert np.isfinite(x).all() and _constraint_error(x, d) <= 1e-9


@pytest.mark.parametrize("kind", [0, 1, 2])
def test_deterministic_integration_matches_reference(kind, capsys):
    """test_gpu_parity.py's trajectory test, in mixed precision, with the same tolerances; prints both precisions'
    deviations."""
    from openmm_b200 import systems, Engine
    ref = np.load(os.path.join(GOLDEN, "reference_platform.npz"))
    d = systems.water_box(6, cutoff=0.9).rounded()
    v = np.random.default_rng(3).standard_normal((d.natoms, 3))*0.3
    key = "integrate%d:" % kind
    dev = {}
    for p in ("single", "mixed"):
        eng = Engine(d, precision=p)
        eng.set_integrator(kind, 0.001, 0.0, 1.0, 7)
        eng.set_velocities(v)
        eng.apply_velocity_constraints()
        eng.step(10)
        eng.compute()
        ke = float(ref[key + "kinetic"])
        dev[p] = (np.abs(eng.get_positions() - (d.positions + ref[key + "dx"])).max(), np.abs(eng.get_velocities() - ref[key + "v"]).max(),
                  abs(eng.kinetic_energy() - ke)/ke)
    with capsys.disabled():
        print("\nintegrate%d max deviation from Reference (x nm, v nm/ps, KE rel): single %.2e %.2e %.2e  mixed %.2e %.2e %.2e"
              % ((kind,) + dev["single"] + dev["mixed"]))
    dx, dv, dke = dev["mixed"]
    assert dx < 5e-6 and dv < 1e-3 and dke < 1e-3


@pytest.mark.parametrize("kind", [0, 1, 2])
def test_ccma_network_follows_reference(kind, capsys):
    from openmm_b200 import systems, Engine
    from test_gpu_parity import _all_bonds
    ref = np.load(os.path.join(GOLDEN, "reference_platform.npz"))
    d = _all_bonds(systems, _load("dhfr", rounded=True))
    v = np.random.default_rng(3).standard_normal((d.natoms, 3))*0.2
    idx = ref["ccma:idx"]
    dev = {}
    for p in ("single", "mixed"):
        eng = Engine(d, precision=p)
        eng.set_integrator(kind, 0.001, 0.0, 1.0, 7, 1e-6)
        eng.apply_constraints(1e-6)
        dx0 = np.abs(eng.get_positions()[idx] - (d.positions[idx] + ref["ccma:dx0"])).max()
        eng.set_velocities(v)
        eng.step(10)
        x = eng.get_positions()
        dev[p] = (dx0, np.abs(x[idx] - (d.positions[idx] + ref["ccma%d:dx" % kind])).max(), _constraint_error(x, d))
    with capsys.disabled():
        print("\nccma%d max deviation from Reference (x0 nm, x nm, constraint rel): single %.2e %.2e %.2e  mixed %.2e %.2e %.2e"
              % ((kind,) + dev["single"] + dev["mixed"]))
    dx0, dx, dc = dev["mixed"]
    assert dx0 < 2e-6 and dx < 5e-5 and dc < 2e-5


def _shifted_positions(d, seed=11):
    """Every 7th molecule moved 2-3 box lengths away: the list build wraps it back into cellOffset."""
    x = d.positions.copy()
    rng = np.random.default_rng(seed)
    for m in d.molecules()[::7]:
        k = rng.integers(-3, 4, 3)
        k[k == 0] = 2
        x[m] += k @ d.box
    return x


def _cell_offsets(eng):
    npad = eng.stats()["padded_atoms"]
    return np.frombuffer(eng.checkpoint()[-12*npad:], dtype=np.int32).reshape(3, npad)[:, :eng.natoms]


def test_wrap_keeps_the_double_coordinates():
    from openmm_b200 import Engine
    d = _load("dhfr")
    x = _shifted_positions(d)
    eng = Engine(d, precision="mixed")
    eng.set_positions(x)
    eng.compute()
    assert (_cell_offsets(eng) != 0).any()
    assert np.abs(eng.get_positions() - x).max() < 1e-11


def test_scale_coordinates_matches_oracle_in_double():
    from barostat_harness import barostat_scale
    from openmm_b200 import Engine
    d = _load("dhfr")
    eng = Engine(d, precision="mixed")
    eng.set_positions(_shifted_positions(d))
    eng.compute()
    mols = d.molecules()
    eng.set_barostat_molecules(mols)
    for s in ((0.98,)*3, (1.02,)*3, (0.99, 1.015, 1.003)):
        x0, f0, blob0 = eng.get_positions(), eng.get_forces(), eng.checkpoint()
        expect = barostat_scale(x0, mols, d.box, s)
        eng.scale_coordinates(*s)
        assert np.abs(eng.get_positions() - expect).max() < 1e-10
        assert not _cell_offsets(eng).any()
        eng.restore_coordinates()
        assert np.array_equal(eng.get_positions(), x0) and np.array_equal(eng.get_forces(), f0)
        assert eng.checkpoint() == blob0


def test_checkpoint_restores_the_state_bit_for_bit():
    from openmm_b200 import systems, Engine, engine
    d = systems.water_box(5, cutoff=0.75).rounded()
    eng = Engine(d, precision="mixed")
    eng.set_integrator(systems.INT_LANGEVIN, 0.002, 300.0, 1.0, 5)
    eng.step(10)
    blob = eng.checkpoint()
    x0, v0 = eng.get_positions(), eng.get_velocities()
    eng.step(10)
    eng.load_checkpoint(blob)
    assert np.array_equal(eng.get_positions(), x0) and np.array_equal(eng.get_velocities(), v0)
    assert eng.checkpoint() == blob
    single = Engine(d)
    with pytest.raises(engine.EngineError, match="precision"):
        single.load_checkpoint(blob)
    with pytest.raises(engine.EngineError, match="precision"):
        eng.load_checkpoint(single.checkpoint())


def test_equal_seeds_give_identical_runs():
    from openmm_b200 import systems, Engine
    d = systems.water_box(6, cutoff=0.9).rounded()
    out = []
    for _ in range(2):
        eng = Engine(d, precision="mixed")
        eng.set_integrator(systems.INT_LANGEVIN_MIDDLE, 0.002, 300.0, 1.0, 9, 1e-6)
        eng.step(50)
        out.append((eng.get_positions(), eng.get_velocities()))
    assert np.array_equal(out[0][0], out[1][0]) and np.array_equal(out[0][1], out[1][1])


def test_nve_energy_drift_verlet(capsys):
    """test_gpu_parity.py::test_nve_energy_drift_verlet in both precisions; the mixed run meets the same bound."""
    from openmm_b200 import systems, Engine
    d = systems.water_box(8, cutoff=0.9).rounded()
    drifts = {}
    for p in ("single", "mixed"):
        eng = Engine(d, precision=p)
        eng.set_integrator(systems.INT_LANGEVIN, 0.002, 300.0, 5.0, 3)
        eng.step(1000)
        eng.set_integrator(systems.INT_VERLET, 0.001, 0, 0, 0, 1e-6)
        dof = 3*d.natoms - len(d.con_i) - 3

        def total():
            return eng.compute() + eng.kinetic_energy()
        e0 = total()
        es = []
        for _ in range(10):
            eng.step(1000)
            es.append(total())
        drifts[p] = (np.array(es) - e0)/dof
    with capsys.disabled():
        print("\nNVE drift per dof over 10 ps (kJ/mol): single %.2e  mixed %.2e" % (np.abs(drifts["single"]).max(), np.abs(drifts["mixed"]).max()))
    assert np.abs(drifts["mixed"]).max() < 0.01, drifts["mixed"]


# ---- through the OpenMM Platform plugin ----
@pytest.fixture(scope="module")
def omm():
    from oracle import omm
    if not omm.available() or not os.path.exists(PLUGIN):
        pytest.fail("oracle/_ref or the plugin is not built: run __graft_entry__.build() where /root/reference exists")
    omm.load_plugin(PLUGIN)
    return omm


def test_plugin_mixed_runs_on_b200_and_matches_reference(omm):
    from openmm_b200 import systems
    d = systems.water_box(6, cutoff=0.9).rounded()
    pme = d.pme_parameters()
    a = omm.Simulation(d, "B200", pme=pme, props="Precision=mixed")
    b = omm.Simulation(d, "Reference", pme=pme)
    assert a.platform() == "B200"
    fa, ea = a.forces_energy()
    fb, eb = b.forces_energy()
    assert relative_force_error(fa, fb) < 1e-4 and abs(ea - eb)/max(1.0, abs(eb)) < 1e-4
    v = np.random.default_rng(3).standard_normal((d.natoms, 3))*0.3
    a = omm.Simulation(d, "B200", integrator=(systems.INT_VERLET, 0, 0, 0.001), pme=pme, props="Precision=mixed")
    b = omm.Simulation(d, "Reference", integrator=(systems.INT_VERLET, 0, 0, 0.001), pme=pme)
    for s in (a, b):
        s.set_velocities(v)
        s.step(10)
    sa, sb = a.state(positions=True, energy=True), b.state(positions=True, energy=True)
    assert np.abs(sa["positions"] - sb["positions"]).max() < 5e-6
    assert abs(sa["potential"] - sb["potential"])/abs(sb["potential"]) < 1e-4
    assert abs(sa["kinetic"] - sb["kinetic"])/sb["kinetic"] < 1e-3


def test_plugin_precision_takes_effect(omm):
    """The sub-ulp motion of test_sub_ulp_motion_accumulates through Context / VerletIntegrator: Precision=mixed moves the
    particles, the default (single) does not."""
    from openmm_b200 import systems
    d = _free_particles()
    v = np.full((d.natoms, 3), 1e-5)
    out = {}
    for props in ("", "Precision=mixed"):
        s = omm.Simulation(d, "B200", integrator=(systems.INT_VERLET, 0, 0, 0.001), props=props)
        s.set_positions(d.positions)
        s.set_velocities(v)
        s.step(2000)
        out[props] = s.state(positions=True)["positions"]
    assert np.abs(out["Precision=mixed"] - (d.positions + v*2.0)).max() < 1e-10
    assert np.abs(out[""] - d.positions).max() < 2.5e-7


def test_plugin_refuses_double_precision(omm):
    from openmm_b200 import systems
    d = systems.water_box(5, cutoff=0.75).rounded()
    with pytest.raises(RuntimeError, match="B200 platform"):
        omm.Simulation(d, "B200", pme=d.pme_parameters(), props="Precision=double")


def test_plugin_fused_step_equals_two_call_path_in_mixed(omm):
    from openmm_b200 import systems
    d = systems.water_box(6, cutoff=0.9).rounded()
    v = np.random.default_rng(4).standard_normal((d.natoms, 3))*0.3
    out = []
    for fused in ("1", "0"):
        os.environ["B200MD_PLUGIN_FUSED"] = fused
        sim = omm.Simulation(d, "B200", integrator=(systems.INT_VERLET, 0, 0, 0.001), pme=d.pme_parameters(), props="Precision=mixed")
        sim.set_velocities(v)
        sim.step(20)
        out.append(sim.state(positions=True)["positions"])
        sim.close()
    os.environ.pop("B200MD_PLUGIN_FUSED", None)
    assert np.abs(out[0] - out[1]).max() < 2e-6          # the bound test_gpu_plugin.py holds single precision to


MIXED_TEST_BINARIES = ["TestB200Mixed" + x for x in ("Settle", "VerletIntegrator", "LangevinIntegrator", "LangevinMiddleIntegrator", "CMMotionRemover",
                                                     "LocalEnergyMinimizer", "MonteCarloBarostat", "MonteCarloAnisotropicBarostat")]


@pytest.mark.parametrize("name", MIXED_TEST_BINARIES)
def test_reference_own_test_bodies_pass_in_mixed_precision(name):
    """The reference's tests/Test<X>.h bodies with Precision=mixed as the platform default (plugin/tests/shim.cpp)."""
    exe = os.path.join(REFTESTS, name)
    if not os.path.exists(exe):
        pytest.fail("%s not built (make -C plugin reftests where /root/reference exists)" % exe)
    env = dict(os.environ, B200_PLUGIN=PLUGIN)
    for attempt in range(2):
        # ASSERT_USUALLY_* assertions get the one rerun the reference's CI gives them (devtools/run-ctest.py:86-118)
        p = subprocess.run([exe], capture_output=True, text=True, timeout=600, env=env)
        if p.returncode == 0 and "Done" in p.stdout:
            break
        if "stochastic" not in p.stdout:
            break
    assert p.returncode == 0 and "Done" in p.stdout, p.stdout[-2000:] + p.stderr[-2000:]
