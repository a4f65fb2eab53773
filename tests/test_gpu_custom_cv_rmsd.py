"""CustomCVForce on the GPU: the reference's own test bodies in single and mixed precision; DHFR with an RMSD restraint over its
solute heavy atoms through a CustomCVForce against the Reference platform, before and after 200 steps; a two-variable bias in
the shape of metadynamics (a centroid distance and a torsion under a Continuous2DFunction) with its variable values, a table
update and a global parameter of a variable; reproducible forces and the fused and unfused step paths; refusals."""
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


def _rmsd_restraint(d):
    from openmm_b200 import systems
    atoms = systems.solute_heavy_atoms(d)
    ref = np.array(d.positions, dtype=np.float64)
    ref[atoms] += np.random.default_rng(1).normal(0.0, 0.05, (len(atoms), 3))
    return {"energy": "0.5*k*max(0, rmsd-r0)^2", "variables": [("rmsd", "rmsd", atoms, ref)],
            "globals": [("k", 5000.0, False), ("r0", 0.02, False)]}


def _metadynamics_bias(d):
    """a centroid distance between the two solute halves and a backbone-like torsion, under a smooth 2-D table"""
    from openmm_b200 import systems
    a, b = systems.solute_halves(d)
    h = systems.solute_heavy_atoms(d)
    x, y = np.meshgrid(np.linspace(0, 1, 24), np.linspace(0, 1, 20), indexing="ij")
    table = (20.0*np.sin(2*np.pi*x)*np.cos(2*np.pi*y) + 5.0*x).T.ravel()     # values[x + xsize*y]
    return {"energy": "bias(dist, phi)", "variables": [("centroid", "dist", a, b, True), ("torsion", "phi", h[10], h[11], h[12], h[13], "shift")],
            "table": ("bias", 24, 20, table, 0.0, 4.0, -np.pi - 0.5, np.pi + 0.5)}


@pytest.mark.parametrize("name", ["TestB200CustomCVForce", "TestB200MixedCustomCVForce"])
def test_reference_test_bodies(H, name):
    exe = os.path.join(REFTESTS, name)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=900, env=dict(os.environ, B200_PLUGIN=PLUGIN))
    assert r.returncode == 0 and r.stdout.rstrip().endswith("Done"), r.stdout[-3000:] + r.stderr[-2000:]


@pytest.mark.parametrize("precision", ["single", "mixed"])
def test_dhfr_rmsd_restraint_matches_reference(H, dhfr, precision):
    from openmm_b200 import systems
    cv, pme = _rmsd_restraint(dhfr), dhfr.pme_parameters()
    b200 = H.CVSimulation(dhfr, "B200", cv=cv, pme=pme, props="Precision=" + precision,
                          integrator=(systems.INT_LANGEVIN_MIDDLE, 300.0, 1.0, 0.002))
    ref = H.CVSimulation(dhfr, "Reference", cv=cv, pme=pme)
    assert b200.platform() == "B200"
    g = 1 << H.CV_GROUP
    for stage in ("start", "after 200 steps"):
        if stage != "start":
            b200.set_velocities_to_temperature(300.0, 3)
            b200.step(200)
            ref.set_positions(b200.state(positions=True)["positions"])
        (f, e), (fr, er) = b200.forces_energy(g), ref.forces_energy(g)
        err = H.force_error(f, fr)
        print("DHFR RMSD restraint (%s, %s): %.6f vs %.6f kJ/mol, force error %.2e" % (precision, stage, e, er, err))
        assert er > 1.0 and err <= FORCE_BAR and abs(e - er) <= 1e-5*abs(er), (stage, err, e, er)
        assert abs(b200.cv_values()[0] - ref.cv_values()[0]) <= 1e-6


def test_metadynamics_shaped_bias(H, dhfr):
    cv, pme = _metadynamics_bias(dhfr), dhfr.pme_parameters()
    b200, ref = H.CVSimulation(dhfr, "B200", cv=cv, pme=pme), H.CVSimulation(dhfr, "Reference", cv=cv, pme=pme)
    g = 1 << H.CV_GROUP

    def check(what):
        (f, e), (fr, er) = b200.forces_energy(g), ref.forces_energy(g)
        v, vr = b200.cv_values(), ref.cv_values()
        assert np.abs(v - vr).max() <= 2e-6, (what, v, vr)
        assert H.force_error(f, fr) <= FORCE_BAR and abs(e - er) <= 1e-5*max(1.0, abs(er)), (what, H.force_error(f, fr), e, er)
        return e
    e0 = check("start")
    name, xs, ys, table, *rng = cv["table"]
    for sim in (b200, ref):
        sim.set_table(name, xs, ys, 2.0*np.asarray(table) + 1.0, *rng)
    e1 = check("table updated")
    assert abs(e1 - (2*e0 + 1)) <= 1e-6*max(1.0, abs(e1))
    for sim in (b200, ref):
        sim.set_parameter("shift", 0.7)
    check("global of a variable")


def test_forces_reproducible_and_step_paths_agree(H, dhfr):
    from openmm_b200 import systems
    cv, pme = _rmsd_restraint(dhfr), dhfr.pme_parameters()
    s = H.CVSimulation(dhfr, "B200", cv=cv, pme=pme)
    f1, _ = s.forces_energy()
    f2, _ = s.forces_energy()
    assert (f1 == f2).all()
    s.close()
    v = np.random.default_rng(3).standard_normal((dhfr.natoms, 3))*0.3
    runs = {}
    for fused in ("1", "0"):
        os.environ["B200MD_PLUGIN_FUSED"] = fused
        try:
            s = H.CVSimulation(dhfr, "B200", cv=cv, pme=pme, integrator=(systems.INT_VERLET, 0, 0, 0.001))
        finally:
            os.environ.pop("B200MD_PLUGIN_FUSED", None)
        s.set_velocities(v)
        s.step(50)
        runs[fused] = s.state(positions=True)["positions"]
        s.close()
    # the two step paths are not bit-equal for any System on this platform, with or without a CustomCVForce: the bound of the
    # other classes' comparisons on DHFR (test_gpu_cmap_rb.py; test_gpu_plugin.py bounds plain water by 2e-6 nm).  The CV's
    # own contribution is bit-reproducible (above).
    print("fused - unfused after 50 steps: %.3e nm" % np.abs(runs["1"] - runs["0"]).max())
    assert np.abs(runs["1"] - runs["0"]).max() < 5e-6


def test_refusals(H, dhfr):
    # a variable of a class without a kernel here: another platform when none is named, a B200 message when B200 is named
    cv = {"energy": "2*v", "variables": [("custom_nonbonded", "v")]}
    s = H.CVSimulation(dhfr, "Reference", cv=cv)
    assert s.try_platform("") not in ("B200", "") and not s.try_platform("").startswith("error")
    assert "B200 platform" in s.try_platform("B200")
    s.close()
    # energy parameter derivatives
    cv = dict(_rmsd_restraint(dhfr))
    cv["globals"] = [("k", 5000.0, True), ("r0", 0.02, False)]
    s = H.CVSimulation(dhfr, "Reference", cv=cv)
    assert "B200 platform" in s.try_platform("B200")
    s.close()


def test_engine_refuses_multi_step_with_cv_forces(dhfr):
    import copy
    from openmm_b200 import Engine, EngineError, systems
    d = copy.copy(dhfr)
    d.cv_count = 2
    eng = Engine(d, device=0)
    eng.set_integrator(systems.INT_LANGEVIN_MIDDLE, 0.002, 300.0, 1.0, 7)
    eng.step(1)
    with pytest.raises(EngineError, match="one step per call"):
        eng.step(2)
    eng.close()
