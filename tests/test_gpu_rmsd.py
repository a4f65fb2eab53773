"""RMSDForce on the GPU: the reference's own test body in single and mixed precision; the golden cases through the plugin; DHFR
with an RMSD over its solute heavy atoms against the Reference platform, before and after 200 LangevinMiddle steps; two
RMSDForce objects in two force groups; updates of the particle set; bit-reproducible forces; the fused and unfused step paths;
zero forces at a perfect alignment; the engine's phase timer and launch counts."""
import os
import subprocess

import numpy as np
import pytest
from conftest import ROOT

pytestmark = pytest.mark.gpu
PLUGIN = os.path.join(ROOT, "plugin", "libOpenMMB200.so")
REFTESTS = os.path.join(ROOT, "oracle", "_ref", "tests")
FORCE_BAR = 1e-4


@pytest.fixture(scope="module")
def H():
    import rmsd_harness
    if not rmsd_harness.available() or not os.path.exists(PLUGIN):
        pytest.fail("oracle/_ref or the plugin is not built: run __graft_entry__.build() where the reference sources exist")
    rmsd_harness.omm.load_plugin(PLUGIN)
    return rmsd_harness


@pytest.fixture(scope="module")
def dhfr():
    from openmm_b200 import systems
    return systems.SystemDesc.load(os.path.join(ROOT, "data", "dhfr.npz")).rounded()


def _restraint(H, d, seed=1):
    """the solute heavy atoms and reference positions a little away from DHFR's own, so that the RMSD is well above 0"""
    from openmm_b200 import systems
    atoms = systems.solute_heavy_atoms(d)
    ref = np.array(d.positions, dtype=np.float64)
    ref[atoms] += np.random.default_rng(seed).normal(0.0, 0.05, (len(atoms), 3))
    return atoms, ref


@pytest.mark.parametrize("name", ["TestB200RMSDForce", "TestB200MixedRMSDForce"])
def test_reference_test_bodies(H, name):
    exe = os.path.join(REFTESTS, name)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=900, env=dict(os.environ, B200_PLUGIN=PLUGIN))
    assert r.returncode == 0 and r.stdout.rstrip().endswith("Done"), r.stdout[-3000:] + r.stderr[-2000:]


@pytest.mark.parametrize("precision", ["single", "mixed"])
def test_golden_cases_through_the_plugin(H, precision):
    """every golden case alone in a System on the B200 platform: the coordinates are fp32 on the device, so the bar is the
    force bar of every other class, and the RMSD agrees to a few fp32 roundings of the coordinates"""
    for name, g in sorted(H.load_golden().items()):
        e, f = H.evaluate(g["positions"], g["reference"], g["particles"], "B200", precision)
        er, fr = float(g["energy"]), g["forces"]
        if name == "rotated_copy":
            assert e < 1e-4 and np.isfinite(f).all(), (name, e)
            continue
        scale = max(1.0, np.abs(g["positions"]).max())
        assert abs(e - er) <= 2e-6*scale, (name, e, er)
        assert H.force_error(f, fr) <= FORCE_BAR, (name, H.force_error(f, fr))


@pytest.mark.parametrize("precision", ["single", "mixed"])
def test_dhfr_rmsd_matches_reference_before_and_after_dynamics(H, dhfr, precision):
    from openmm_b200 import systems
    atoms, ref = _restraint(H, dhfr)
    assert len(atoms) == 1268
    pme = dhfr.pme_parameters()
    spec = [(atoms, ref, H.RMSD_GROUP)]
    b200 = H.Simulation(dhfr, "B200", rmsd=spec, pme=pme, props="Precision=" + precision,
                        integrator=(systems.INT_LANGEVIN_MIDDLE, 300.0, 1.0, 0.002))
    refsim = H.Simulation(dhfr, "Reference", rmsd=spec, pme=pme)
    assert b200.platform() == "B200"
    groups = 1 << H.RMSD_GROUP
    for stage in ("start", "after 200 steps"):
        if stage != "start":
            b200.set_velocities_to_temperature(300.0, 3)
            b200.step(200)
            x = b200.state(positions=True)["positions"]
            refsim.set_positions(x)
        (f, e), (fr, er) = b200.forces_energy(groups), refsim.forces_energy(groups)
        err = H.force_error(f, fr)
        print("DHFR RMSD (%s, %s): %.6f nm vs %.6f, force error %.2e" % (precision, stage, e, er, err))
        assert err <= FORCE_BAR and abs(e - er) <= 1e-5*er, (stage, err, e, er)
        if stage == "start":
            # the whole force field still agrees with the restraint in it.  After mixed-precision dynamics the reported
            # positions carry bits below the fp32 coordinates every force kernel reads, so only the RMSD is compared there
            (fa, ea), (fra, era) = b200.forces_energy(), refsim.forces_energy()
            assert H.force_error(fa, fra) <= FORCE_BAR and abs(ea - era) <= 1e-4*abs(era), (stage, ea, era)


def test_two_objects_in_two_groups(H, dhfr):
    from openmm_b200 import systems
    halves = systems.solute_halves(dhfr)
    ref = np.array(dhfr.positions, dtype=np.float64) + np.random.default_rng(2).normal(0.0, 0.04, (dhfr.natoms, 3))
    spec = [(halves[0], ref, 5), (halves[1], ref, 6)]
    pme = dhfr.pme_parameters()
    b200, refsim = H.Simulation(dhfr, "B200", rmsd=spec, pme=pme), H.Simulation(dhfr, "Reference", rmsd=spec, pme=pme)
    for groups in (1 << 5, 1 << 6, (1 << 5) | (1 << 6)):
        (f, e), (fr, er) = b200.forces_energy(groups), refsim.forces_energy(groups)
        assert H.force_error(f, fr) <= FORCE_BAR and abs(e - er) <= 1e-5*er, (groups, e, er)
    # a new particle set of another size, and a changed reference, for the first object only
    sub = halves[0][::3]
    for sim in (b200, refsim):
        sim.update_rmsd(0, sub, ref*1.01)
    for groups in (1 << 5, (1 << 5) | (1 << 6)):
        (f, e), (fr, er) = b200.forces_energy(groups), refsim.forces_energy(groups)
        assert H.force_error(f, fr) <= FORCE_BAR and abs(e - er) <= 1e-5*er, (groups, e, er)


def test_forces_are_bit_reproducible(H, dhfr):
    atoms, ref = _restraint(H, dhfr)
    s = H.Simulation(dhfr, "B200", rmsd=[(atoms, ref, H.RMSD_GROUP)], pme=dhfr.pme_parameters())
    f1, e1 = s.forces_energy()
    f2, e2 = s.forces_energy()
    assert (f1 == f2).all()
    g1, _ = s.forces_energy(1 << H.RMSD_GROUP)
    g2, _ = s.forces_energy(1 << H.RMSD_GROUP)
    assert (g1 == g2).all()


def test_fused_and_unfused_steps_agree(H, dhfr):
    from openmm_b200 import systems
    atoms, ref = _restraint(H, dhfr)
    v = np.random.default_rng(3).standard_normal((dhfr.natoms, 3))*0.3
    runs = {}
    for fused in ("1", "0"):
        os.environ["B200MD_PLUGIN_FUSED"] = fused
        try:
            s = H.Simulation(dhfr, "B200", rmsd=[(atoms, ref*1.0, H.RMSD_GROUP)], pme=dhfr.pme_parameters(),
                             integrator=(systems.INT_VERLET, 0, 0, 0.001))
        finally:
            os.environ.pop("B200MD_PLUGIN_FUSED", None)
        s.set_velocities(v)
        s.step(50)
        runs[fused] = s.state(positions=True)["positions"]
        s.close()
    # the bound of the other classes' fused/unfused comparisons (test_gpu_cmap_rb.py)
    assert np.abs(runs["1"] - runs["0"]).max() < 5e-6


def test_perfect_alignment_gives_zero_forces(H):
    x = np.array([[1.0, 0.0, 0.0], [-1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [0.0, -1.0, 0.0], [0.0, 0.0, 2.0], [0.0, 0.0, -2.0]])
    for precision in ("single", "mixed"):
        e, f = H.evaluate(x + 3.0, x, np.zeros(0, np.int32), "B200", precision)
        assert e == 0.0 and (f == 0).all(), (e, f)


def test_engine_phase_launch_counts_and_updates(H, dhfr):
    """the RMSD kernels add three launches to an evaluation and to a step, are timed as their own phase, and an update of the
    same size keeps the step graph"""
    import copy
    from openmm_b200 import Engine, engine, systems
    atoms, ref = _restraint(H, dhfr)
    d = copy.copy(dhfr)
    d.rmsd_start, d.rmsd_atoms = np.array([0, len(atoms)], np.int32), atoms
    d.rmsd_ref, d.rmsd_group = ref[atoms], np.zeros(1, np.int32)
    plain, eng = Engine(dhfr, device=0), Engine(d, device=0)
    e_only = eng.compute(engine.TERM_RMSD)
    er = H.Simulation(dhfr, "Reference", rmsd=[(atoms, ref, H.RMSD_GROUP)], pme=dhfr.pme_parameters()).forces_energy(1 << H.RMSD_GROUP)[1]
    assert abs(e_only - er) <= 1e-5*er, (e_only, er)
    for e in (plain, eng):
        e.set_integrator(systems.INT_LANGEVIN_MIDDLE, 0.002, 300.0, 1.0, 7)
        e.step(2)
        e.synchronize()
    counts = []
    for e in (plain, eng):
        before = e.stats()["kernel_launches"]
        e.compute(engine.TERM_ALL, energy=False)
        mid = e.stats()["kernel_launches"]
        e.step(1)
        e.synchronize()
        counts.append((mid - before, e.stats()["kernel_launches"] - mid))
    assert counts[1][0] == counts[0][0] + 3 and counts[1][1] == counts[0][1] + 3, counts
    assert eng.time_phase(engine.PHASES["rmsd"], 20) > 0
    graphs = eng.stats()["graph_instantiations"]
    eng.update_rmsd(d.rmsd_start, atoms, ref[atoms] + 0.01)
    eng.step(5)
    eng.synchronize()
    assert eng.stats()["graph_instantiations"] == graphs
    assert np.isfinite(eng.get_positions()).all()
