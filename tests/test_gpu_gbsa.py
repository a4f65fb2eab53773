"""Generalized Born (GBSAOBCForce) on the GPU: the reference's own test bodies in single and mixed precision; its
HelloSodiumChloride example run unmodified on this platform; DHFR-GBSA and periodic ion boxes against the Reference platform and
the double-precision restatement (tests/gbsa_harness.py); bit-reproducibility with and without the GB stream overlap; force
groups; updateParametersInContext; launch counts; NVE drift and the benchmark's Langevin protocol; platform fallback."""
import os
import subprocess
import tempfile

import numpy as np
import pytest
from conftest import ROOT

pytestmark = pytest.mark.gpu
PLUGIN = os.path.join(ROOT, "plugin", "libOpenMMB200.so")
REFTESTS = os.path.join(ROOT, "oracle", "_ref", "tests")
FORCE_BAR, ENERGY_BAR = 1e-4, 1e-5


@pytest.fixture(scope="module")
def H():
    import gbsa_harness
    if not gbsa_harness.available() or not os.path.exists(PLUGIN):
        pytest.fail("oracle/_ref or the plugin is not built: run __graft_entry__.build() where the reference sources exist")
    gbsa_harness.omm.load_plugin(PLUGIN)
    return gbsa_harness


def _engine_gb(eng):
    from openmm_b200 import engine
    e = eng.compute(engine.TERM_GBSA)
    return eng.get_forces(), e


@pytest.mark.parametrize("name", ["TestB200GBSAOBCForce", "TestB200MixedGBSAOBCForce"])
def test_reference_test_bodies(H, name):
    exe = os.path.join(REFTESTS, name)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=900, env=dict(os.environ, B200_PLUGIN=PLUGIN))
    assert r.returncode == 0 and r.stdout.rstrip().endswith("Done"), r.stdout[-3000:] + r.stderr[-2000:]


def test_hello_sodium_chloride_runs_on_this_platform(H):
    exe = os.path.join(REFTESTS, "HelloSodiumChloride")
    with tempfile.TemporaryDirectory() as tmp:
        os.symlink(PLUGIN, os.path.join(tmp, "libOpenMMB200.so"))
        # the link's $ORIGIN is the temporary directory, so the plugin finds libb200md.so and libOpenMM.so on the library path
        path = os.pathsep.join([os.path.join(ROOT, "openmm_b200"), os.path.join(ROOT, "oracle", "_ref"), os.environ.get("LD_LIBRARY_PATH", "")])
        out = subprocess.run([exe], capture_output=True, text=True, timeout=600,
                             env=dict(os.environ, OPENMM_PLUGIN_DIR=tmp, LD_LIBRARY_PATH=path)).stdout
    assert "Using OpenMM platform B200" in out, out[-2000:]
    frames = [l for l in out.splitlines() if l.startswith("REMARK 250")]
    assert len(frames) > 10
    energies = [float(l.split("energy=")[1].split()[0]) for l in frames]
    assert abs(energies[0] - (-297.971)) <= 0.005, frames[0]
    assert np.isfinite(energies).all()


@pytest.mark.parametrize("method", ["nocutoff", "cutoff"])
def test_dhfr_gbsa_plugin_matches_reference(H, method):
    from openmm_b200 import systems
    d = H.dhfr_gbsa(systems.NB_NOCUTOFF if method == "nocutoff" else systems.NB_CUTOFF_NONPERIODIC).rounded()
    ref, b200 = H.Simulation(d, "Reference"), H.Simulation(d, "B200")
    assert b200.platform() == "B200"
    (f, e), (fr, er) = H.gb_only(b200), H.gb_only(ref)
    err = H.force_error(f, fr)
    print("DHFR-GBSA %s plugin vs Reference: force %.2e, energy %.2e" % (method, err, abs(e - er)/abs(er)))
    assert err <= FORCE_BAR and abs(e - er) <= ENERGY_BAR*abs(er), (err, e, er)


@pytest.mark.parametrize("case", ["dhfr_nocutoff", "dhfr_cutoff", "ion_box_periodic", "ion_box_pme", "ion_box_custom", "hello_nacl",
                                  "ion_box_tri_pmp", "ion_box_tri_mpm"])
def test_engine_matches_the_restatement(H, case):
    from openmm_b200 import Engine, systems
    if case.startswith("ion_box_tri"):
        d = H.triclinic_ion_box(case.split("_")[-1])
    elif case.startswith("dhfr"):
        d = H.dhfr_gbsa(systems.NB_NOCUTOFF if case == "dhfr_nocutoff" else systems.NB_CUTOFF_NONPERIODIC)
    elif case == "ion_box_pme":
        d = H.ion_box(method=systems.NB_PME)
    elif case == "ion_box_periodic":
        d = H.ion_box()
    else:
        d = H.golden_cases()[case]
    d = d.rounded()
    eng = Engine(d)
    f, e = _engine_gb(eng)
    eng.close()
    fr, er = H.obc_forces_energy(d)
    err = H.force_error(f, fr)
    print("%s engine vs restatement: force %.2e, energy %.2e" % (case, err, abs(e - er)/abs(er)))
    assert err <= FORCE_BAR and abs(e - er) <= ENERGY_BAR*abs(er), (err, e, er)


@pytest.mark.parametrize("case", ["ion_box", "ion_box_tri_pmp", "ion_box_tri_mpm"])
def test_periodic_ion_boxes_plugin_matches_reference(H, case):
    """the plugin against the Reference platform on the cubic and the two triclinic periodic ion boxes"""
    d = H.golden_cases()[case].rounded()
    ref, b200 = H.Simulation(d, "Reference"), H.Simulation(d, "B200")
    assert b200.platform() == "B200"
    (f, e), (fr, er) = H.gb_only(b200), H.gb_only(ref)
    err = H.force_error(f, fr)
    print("%s plugin vs Reference: force %.2e, energy %.2e" % (case, err, abs(e - er)/abs(er)))
    assert err <= FORCE_BAR and abs(e - er) <= ENERGY_BAR*abs(er), (err, e, er)


def _to_aged_state(eng, nsteps):
    """Step one step at a time, a compute() after each, until a state after nsteps steps whose list was built neither in
    its last step nor in that compute (test_gpu_oracle_edges._age without the pair counts); returns the steps taken"""
    steps = 0
    while steps < nsteps + 100:
        b0 = eng.stats()["list_builds"]
        eng.step(1)
        steps += 1
        b1 = eng.stats()["list_builds"]
        eng.compute(energy=False)
        if steps >= nsteps and eng.stats()["list_builds"] == b1 == b0:
            return steps
    pytest.fail("no aged state within %d steps" % steps)


def _check_against_restatement_and_fresh(H, eng, d, label, precision="single", fresh_positions=None):
    """GB forces and energy of eng's current state against the restatement at its positions (the fp32 hi part in mixed
    precision) and against a fresh engine at the same positions; returns the force error against the restatement.
    fresh_positions: the engine's own wrapped fp32 coordinates, for atoms that set_positions put whole box lengths out.
    The fresh engine wraps those again and rounds differently, so the two are held to the relative bound of an aged list
    against a fresh one (test_gpu_oracle_edges.AGED_BOUND), not to the 1e-6 absolute bound of identical coordinates."""
    from openmm_b200 import Engine
    import copy
    f, e = _engine_gb(eng)
    x = eng.get_positions()
    xo = x.astype(np.float32).astype(np.float64) if precision == "mixed" else x
    fr, er = H.obc_forces_energy(d, xo)
    err = H.force_error(f, fr)
    d2 = copy.copy(d)
    d2.positions = x if fresh_positions is None else fresh_positions
    fresh = Engine(d2, precision=precision)
    f2, e2 = _engine_gb(fresh)
    fresh.close()
    print("%s: force %.2e, energy %.2e against the restatement; fresh list %.2e, energy %.2e"
          % (label, err, abs(e - er)/abs(er), np.abs(f - f2).max(), abs(e - e2)/abs(e2)))
    assert err <= FORCE_BAR and abs(e - er) <= ENERGY_BAR*abs(er), (err, e, er)
    if fresh_positions is None:
        # same forces as a fresh Context; not to the bit, since that one's list was built at x in another order
        assert np.abs(f - f2).max() < 1e-6 and abs(e - e2) <= 1e-9*abs(e2), (np.abs(f - f2).max(), e, e2)
    else:
        rel = H.force_error(f, f2)
        print("  fresh engine from the wrapped coordinates: force %.2e relative" % rel)
        assert rel < 1.5e-5 and abs(e - e2) <= 1e-8*abs(e2), (rel, e, e2)
    return err


@pytest.mark.parametrize("case", ["dhfr_cutoff", "dhfr_nocutoff", "ion_box_pad002"])
def test_aged_list_matches_the_restatement(H, monkeypatch, record_property, case):
    """GB on the list as it stands after a Langevin run (not rebuilt in the last step): the mask-free pair sweeps rely on
    the aged list still holding every pair within the cutoff once"""
    from openmm_b200 import Engine, systems
    if case == "ion_box_pad002":
        monkeypatch.setenv("B200MD_PAD_FRACTION", "0.02")
        d, dt, nsteps = H.ion_box().rounded(), 0.001, 80
    else:
        d = H.dhfr_gbsa(systems.NB_NOCUTOFF if case == "dhfr_nocutoff" else systems.NB_CUTOFF_NONPERIODIC).rounded()
        dt, nsteps = 0.002, 40
    eng = Engine(d)
    eng.set_integrator(systems.INT_LANGEVIN, dt, 300.0, 1.0, 13)
    eng.set_velocities(np.random.default_rng(13).standard_normal((d.natoms, 3))*np.sqrt(0.0083144626*300.0/np.asarray(d.masses))[:, None])
    eng.apply_velocity_constraints()
    steps = _to_aged_state(eng, nsteps)
    builds = eng.stats()["list_builds"]
    err = _check_against_restatement_and_fresh(H, eng, d, "%s after %d steps, %d list builds" % (case, steps, builds))
    eng.close()
    record_property("force_error", err)
    if case == "ion_box_pad002":
        assert builds > 3


@pytest.mark.parametrize("n", [2, 31, 33, 65])
def test_small_periodic_ion_boxes(H, n):
    """N that leaves the last 32-atom block partly empty, then the same ions moved by 1-3 lattice vectors through
    set_positions (the list build moves them back in fp32)."""
    from openmm_b200 import Engine
    from test_gpu_oracle_edges import _inner_positions
    d = H.ion_box(n=n, edge=2.6, cutoff=1.2, seed=n).rounded()
    eng = Engine(d)
    _check_against_restatement_and_fresh(H, eng, d, "%d ions" % n)
    k = np.random.default_rng(n).integers(-3, 4, (n, 3))
    eng.set_positions(d.positions + k @ d.box)
    eng.compute(energy=False)
    _check_against_restatement_and_fresh(H, eng, d, "%d ions moved by lattice vectors" % n,
                                         fresh_positions=_inner_positions(eng, n))
    eng.close()


def test_mixed_precision_matches_the_restatement(H):
    """DHFR-GBSA in mixed precision after 10 Langevin steps: the pair sweeps read the fp32 hi part of the positions"""
    from openmm_b200 import Engine, systems
    d = H.dhfr_gbsa().rounded()
    eng = Engine(d, precision="mixed")
    assert eng.precision == "mixed"
    eng.set_integrator(systems.INT_LANGEVIN, 0.002, 300.0, 1.0, 17)
    eng.step(10)
    eng.compute(energy=False)
    _check_against_restatement_and_fresh(H, eng, d, "DHFR-GBSA mixed", precision="mixed")
    eng.close()


def _gb_forces(d, overlap):
    from openmm_b200 import Engine
    old = os.environ.pop("B200MD_NO_OVERLAP", None)
    if not overlap:
        os.environ["B200MD_NO_OVERLAP"] = "1"
    try:
        eng = Engine(d)
    finally:
        os.environ.pop("B200MD_NO_OVERLAP", None)
        if old is not None:
            os.environ["B200MD_NO_OVERLAP"] = old
    out = []
    for _ in range(2):
        eng.compute()
        out.append(eng.get_forces())
    eng.close()
    return out


def test_forces_are_bit_reproducible(H):
    d = H.dhfr_gbsa().rounded()
    a = _gb_forces(d, True)
    b = _gb_forces(d, True)
    c = _gb_forces(d, False)
    for f in a[1:] + b + c:
        assert np.array_equal(f, a[0])


def test_force_groups_match_reference(H):
    d = H.dhfr_gbsa().rounded()
    ref, b200 = H.Simulation(d, "Reference"), H.Simulation(d, "B200")
    for groups in (1 << H.GB_GROUP, 0xffffffff & ~(1 << H.GB_GROUP), 0xffffffff):
        (f, e), (fr, er) = b200.forces_energy(groups), ref.forces_energy(groups)
        err = H.force_error(f, fr)
        print("groups %#x: force %.2e, energy %.2e" % (groups, err, abs(e - er)/abs(er)))
        assert err <= FORCE_BAR and abs(e - er) <= ENERGY_BAR*abs(er), (groups, err, e, er)


def test_update_parameters_in_context(H):
    from openmm_b200 import Engine, systems
    d = H.dhfr_gbsa().rounded()
    eng = Engine(d)
    eng.set_integrator(systems.INT_LANGEVIN_MIDDLE, 0.002, 300.0, 1.0, 5)
    eng.step(3)
    eng.synchronize()
    n0 = eng.stats()["graph_instantiations"]
    q, r, s = d.gb_charges*0.9, d.gb_radii*1.05, d.gb_scales
    eng.update_gbsa_params(q, r, s)
    eng.step(3)
    eng.synchronize()
    assert eng.stats()["graph_instantiations"] == n0
    x = eng.get_positions()
    f, e = _engine_gb(eng)
    import copy
    d2 = copy.copy(d)
    d2.gb_charges, d2.gb_radii, d2.positions = q, r, x
    fresh = Engine(d2)
    f2, e2 = _engine_gb(fresh)
    # same forces as a fresh Context; not to the bit, since that one's list was built at x in another order
    assert np.abs(f - f2).max() < 1e-6 and abs(e - e2) <= 1e-9*abs(e2)
    with pytest.raises(Exception, match="number of particles"):
        eng.update_gbsa_params(q[:-1], r[:-1], s[:-1])
    eng.close(); fresh.close()
    # through the plugin: the count change raises, new parameters give the Reference platform's forces
    ref, b200 = H.Simulation(d, "Reference"), H.Simulation(d, "B200")
    for sim in (ref, b200):
        sim.update_gbsa(q, r, s)
    (f, e), (fr, er) = H.gb_only(b200), H.gb_only(ref)
    assert H.force_error(f, fr) <= FORCE_BAR and abs(e - er) <= ENERGY_BAR*abs(er)
    with pytest.raises(RuntimeError, match="number of particles"):
        b200.update_gbsa(np.append(q, 0.0), np.append(r, 0.2), np.append(s, 0.8))


def _launches(eng, step):
    eng.compute(energy=False) if not step else eng.step(1)
    eng.synchronize()
    before = eng.stats()["kernel_launches"]
    eng.compute(energy=False) if not step else eng.step(1)
    eng.synchronize()
    return eng.stats()["kernel_launches"] - before


@pytest.mark.parametrize("step", [False, True])
def test_launch_counts(H, step):
    from openmm_b200 import Engine, systems
    d = H.dhfr_gbsa().rounded()
    counts = []
    for desc in (d, H.without_gbsa(d)):
        eng = Engine(desc)
        eng.set_integrator(systems.INT_VERLET, 0.001)
        counts.append(_launches(eng, step))
        eng.close()
    assert counts[0] - counts[1] == 5, counts
    plain = systems.SystemDesc.load(os.path.join(ROOT, "data", "dhfr.npz")).rounded()
    eng = Engine(plain)
    eng.set_integrator(systems.INT_VERLET, 0.001)
    n = _launches(eng, step)
    eng.close()
    print("launches per %s: DHFR-GBSA %d, without GB %d, DHFR %d" % ("step" if step else "evaluation", counts[0], counts[1], n))


def _nve_drift(d, steps=2000, every=100):
    """|drift| per atom of the total energy over `steps` Verlet steps of 1 fs: the slope of a straight line fitted to the
    energy sampled every `every` steps, times the span.  The end-to-end difference of one run is dominated by the energy's
    fluctuation (DHFR-GBSA: 3-5e-4 kJ/mol per atom standard deviation either way), the fit by the drift."""
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


@pytest.mark.parametrize("method", ["nocutoff", "cutoff"])
def test_nve_with_gb_drifts_no_more_than_without(H, method):
    from openmm_b200 import systems
    d = H.dhfr_gbsa(systems.NB_NOCUTOFF if method == "nocutoff" else systems.NB_CUTOFF_NONPERIODIC).rounded()
    plain, gb = _nve_drift(H.without_gbsa(d)), _nve_drift(d)
    print("NVE drift per atom over 2,000 steps of 1 fs (%s), kJ/mol: without GB %.3e, with GB %.3e" % (method, plain, gb))
    # the centroid test's rule: as much again as the run without GB, plus 1e-4 kJ/mol per atom
    assert gb <= 2*plain + 1e-4, (plain, gb)


def test_benchmark_protocol_stays_finite(H):
    from openmm_b200 import Engine, systems
    d = H.dhfr_gbsa().rounded()
    eng = Engine(d)
    eng.set_integrator(systems.INT_LANGEVIN_MIDDLE, 0.004, 300.0, 91.0, 9)
    eng.step(1000)
    eng.synchronize()
    x = eng.get_positions()
    assert np.isfinite(x).all() and np.isfinite(eng.compute())
    dist = np.linalg.norm(x[d.con_i] - x[d.con_j], axis=1)
    assert np.abs(dist - d.con_d).max() < 1e-4


@pytest.mark.parametrize("case", ["second force", "method", "cutoff", "particles", "matching"])
def test_platform_fallback(H, case):
    from openmm_b200 import systems
    d = H.ion_box(n=64, edge=2.6, cutoff=1.0, method=systems.NB_CUTOFF_NONPERIODIC)

    class Sim(H.Simulation):
        def add_forces(self):
            super().add_forces()
            L = H.lib()
            if case == "second force":
                H.lib().gbc_add_force(self.sys, d.natoms, H._dp(d.gb_charges), H._dp(d.gb_radii), H._dp(d.gb_scales), 1, 1.0, 1.0, 78.5, 2.0, 0)
            elif case == "method":
                self.gb_index = L.gbc_add_force(self.sys, d.natoms, H._dp(d.gb_charges), H._dp(d.gb_radii), H._dp(d.gb_scales), 0, 1.0, 1.0, 78.5, 2.0, 2)
            elif case == "cutoff":
                self.gb_index = L.gbc_add_force(self.sys, d.natoms, H._dp(d.gb_charges), H._dp(d.gb_radii), H._dp(d.gb_scales), 1, 1.1, 1.0, 78.5, 2.0, 2)
            elif case == "particles":
                L.gbc_add_force(self.sys, d.natoms - 1, H._dp(d.gb_charges), H._dp(d.gb_radii), H._dp(d.gb_scales), 1, 1.0, 1.0, 78.5, 2.0, 2)
    import copy
    e = copy.copy(d)
    if case in ("method", "cutoff", "particles"):
        e = H.without_gbsa(d)
    if case == "particles":
        # GBSAOBCForceImpl refuses this on every platform; the plugin refuses it first, with its own message
        with pytest.raises(RuntimeError, match="exactly as many particles"):
            Sim(e, "B200")
        return
    s = Sim(e, "Reference")
    platform = s.default_platform()
    if case == "matching":
        assert platform == "B200"
    else:
        assert platform not in ("", "B200"), platform


def test_engine_refusals(H):
    from openmm_b200 import Engine, EngineError, systems
    d = H.ion_box(n=64, edge=2.6, cutoff=1.0, method=systems.NB_CUTOFF_NONPERIODIC)
    d.gb_method = systems.NB_NOCUTOFF
    with pytest.raises(EngineError, match="NoCutoff needs a NoCutoff nonbonded force"):
        Engine(d)
    d.gb_method = systems.NB_CUTOFF_NONPERIODIC
    d.gb_radii = d.gb_radii.copy()
    d.gb_radii[3] = 0.009
    with pytest.raises(EngineError, match="dielectric offset"):
        Engine(d)
