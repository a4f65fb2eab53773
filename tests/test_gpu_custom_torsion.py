"""GPU tests of CustomTorsionForce on the platform (k_custom_torsion, the expression programs of plugin/custom_translate.h): the
reference's own test bodies; DHFR with its periodic torsions as custom torsions against the periodic torsions; DHFR-CHARMM
(DHFR with CMAP and CharmmPsfFile-form impropers) through the plugin against the live Reference platform, per force group and
periodic; global parameters, parameter updates, the step paths, precision and launch counts; the C-ABI's input checks."""
import ctypes as C
import os
import subprocess
import numpy as np
import pytest
from conftest import relative_force_error, ROOT, GOLDEN

pytestmark = pytest.mark.gpu
PLUGIN = os.path.join(ROOT, "plugin", "libOpenMMB200.so")
REFTESTS = os.path.join(ROOT, "oracle", "_ref", "tests")


@pytest.fixture(scope="module")
def harness():
    """the translator, Lepton and the reference's CustomTorsionForce (tests/custom_harness.py), with the plugin loaded"""
    import custom_harness
    if not custom_harness.available() or not os.path.exists(PLUGIN):
        pytest.fail("oracle/_ref or the plugin is not built: run __graft_entry__.build() where /root/reference exists")
    custom_harness.omm.load_plugin(PLUGIN)
    return custom_harness


def _dhfr():
    from openmm_b200 import systems
    return systems.SystemDesc.load(os.path.join(ROOT, "data", "dhfr.npz")).rounded()


def _maps():
    z = np.load(os.path.join(GOLDEN, "charmm36_cmap.npz"))
    return z["size"], z["energy"], z["coeff"]


@pytest.fixture(scope="module")
def dhfr_charmm(harness):
    """DHFR-CHARMM: DHFR plus the CHARMM36 CMAP maps on its backbone and one CharmmPsfFile-form improper per atom with three
    bonded neighbours, compiled"""
    from openmm_b200 import systems
    d = harness.compiled(systems.with_cmap(systems.with_charmm_impropers(_dhfr()), *_maps()))
    assert len(d.custom_prog) == 522 and len(d.cmap_map) == 157
    return d


def _group_close(f, e, fr, er):
    """one group alone: both sides are double, only the 2^-32 fixed-point force resolution differs"""
    assert np.abs(f - fr).max() <= 1e-6*np.abs(fr).max()
    assert abs(e - er) <= 1e-8*abs(er)


# ---------------------------------------------------------------------------------------------------- reference test bodies
@pytest.mark.parametrize("name", ["TestB200CustomTorsionForce", "TestB200MixedCustomTorsionForce"])
def test_reference_own_test_bodies_pass(name):
    exe = os.path.join(REFTESTS, name)
    if not os.path.exists(exe):
        pytest.fail("%s not built (make -C plugin reftests where /root/reference exists)" % exe)
    p = subprocess.run([exe], capture_output=True, text=True, timeout=600, env=dict(os.environ, B200_PLUGIN=PLUGIN))
    assert p.returncode == 0 and "Done" in p.stdout, p.stdout[-2000:] + p.stderr[-2000:]


def _tiny(harness, **kw):
    """four atoms, one custom torsion with a global parameter"""
    from openmm_b200 import systems
    x = np.array([[0.0, 0.1, 0.0], [0.0, 0.0, 0.0], [0.15, 0.0, 0.0], [0.15, 0.02, 0.13]])
    z = np.zeros(4)
    d = systems.SystemDesc(masses=np.full(4, 12.0), charges=z, sigmas=np.full(4, 0.3), epsilons=z.copy(), positions=x, box=None,
                           method=systems.NB_NOCUTOFF, use_dispersion=False)
    return systems._custom_only(d, ["lam*k*(1+cos(2*theta-theta0))"], [("k", "theta0")], [0], [[0, 1, 2, 3]], [[3.0, 0.4]],
                                ["lam"], [0.5])


def test_energy_parameter_derivatives_move_the_context_elsewhere(harness):
    d = _tiny(harness)
    plain = harness.Simulation(d, "Reference")
    assert plain.default_platform() == "B200"
    s = harness.Simulation(d, "Reference", deriv_params={"custom_torsions": "lam"})
    assert s.default_platform() not in ("", "B200"), harness.lib().cc_last_error()
    with pytest.raises(RuntimeError, match="energy parameter derivatives"):
        harness.Simulation(d, "B200", deriv_params={"custom_torsions": "lam"})


# ---------------------------------------------------------------------------------------------------- engine
def test_custom_periodic_torsions_equal_periodic_torsions_on_the_engine(harness):
    from openmm_b200 import Engine, engine, systems
    d = _dhfr()
    per = Engine(d)
    ep = per.compute(engine.TERM_TORSIONS)
    fp = per.get_forces()
    c = harness.compiled(systems.periodic_to_custom(d))
    assert len(c.custom_prog) == 7310 and len(c.tor_i) == 0
    cus = Engine(c)
    ec = cus.compute(engine.TERM_CUSTOM_TORSIONS)
    _group_close(cus.get_forces(), ec, fp, ep)


# ---------------------------------------------------------------------------------------------------- through the plugin
MASKS = (1 << 5, 1 << 4, (1 << 4) | (1 << 5), 1, 1 | (1 << 5), 0xffffffff)


def test_dhfr_charmm_through_the_plugin_matches_reference_platform(harness, dhfr_charmm):
    d = dhfr_charmm
    pme = d.pme_parameters()
    groups = {"cmap": 4, "custom_torsions": 5}
    ref = harness.Simulation(d, "Reference", pme=pme, force_groups=groups)
    b200 = harness.Simulation(d, "B200", pme=pme, force_groups=groups)
    assert b200.platform() == "B200"
    for mask in MASKS:
        f, e = b200.forces_energy(mask if mask != 0xffffffff else -1)
        fr, er = ref.forces_energy(mask if mask != 0xffffffff else -1)
        if mask & 1:
            assert relative_force_error(f, fr) < 1e-4 and abs(e - er)/abs(er) < 1e-4, mask
        else:
            _group_close(f, e, fr, er)


def _chain(n, rng, start):
    x = [np.asarray(start, float)]
    dvec = np.array([1.0, 0.0, 0.0])
    for _ in range(n - 1):
        while True:
            v = rng.standard_normal(3)
            v /= np.linalg.norm(v)
            if -0.6 < v @ dvec < 0.2:
                break
        dvec = v
        x.append(x[-1] + 0.15*dvec)
    return np.array(x)


def test_periodic_custom_torsions_straddling_a_triclinic_box(harness):
    """two expressions (the CHARMM improper and a periodic torsion with a global) on a chain split across the faces of a
    triclinic cell: only minimum images make it whole; through the engine and through the plugin"""
    from openmm_b200 import Engine, systems
    rng = np.random.default_rng(11)
    box = np.array([[2.5, 0.0, 0.0], [0.625, 2.375, 0.0], [-0.5, 0.75, 2.625]])
    x = _chain(40, rng, start=(2.3, 2.2, 2.4))
    for k in (2, 1, 0):
        x -= np.floor(x[:, k:k+1]/box[k, k])*box[k]
    x = x.astype(np.float32).astype(np.float64)
    z = np.zeros(40)
    bare = systems.SystemDesc(masses=np.full(40, 12.0), charges=z, sigmas=np.full(40, 0.3), epsilons=z.copy(), positions=x, box=box,
                              method=systems.NB_CUTOFF_PERIODIC, cutoff=1.0, use_dispersion=False)
    n = 37
    atoms = np.array([[i, i+1, i+2, i+3] for i in range(n)])
    prog = np.arange(n) % 2
    params = np.stack([rng.uniform(20, 300, n), rng.uniform(-np.pi, np.pi, n)], axis=1)
    d = harness.compiled(systems._custom_only(bare, [systems.CHARMM_IMPROPER, "s*k*0.01*(1+cos(3*theta-theta0))"],
                                              [("k", "theta0"), ("k", "theta0")], prog, atoms, params, ["s"], [1.7]))
    ref = harness.Simulation(d, "Reference", bonded_periodic=True)
    fr, er = ref.forces_energy()
    eng = Engine(d, bonded_groups={"custom_torsions": np.full(n, 0x80)})
    e = eng.compute()
    _group_close(eng.get_forces(), e, fr, er)
    b200 = harness.Simulation(d, "B200", bonded_periodic=True)
    f, e = b200.forces_energy()
    _group_close(f, e, fr, er)


def test_global_parameters_follow_set_parameter(harness):
    """two CustomTorsionForce objects share the global `lam`, which a NonbondedForce offset also reads: after every
    setParameter the energy is the Reference platform's, between steps too"""
    from openmm_b200 import systems
    rng = np.random.default_rng(3)
    x = _chain(12, rng, start=(1.0, 1.0, 1.0)).astype(np.float32).astype(np.float64)
    q = np.where(np.arange(12) % 2, 0.3, -0.3)
    bare = systems.SystemDesc(masses=np.full(12, 12.0), charges=q, sigmas=np.full(12, 0.3), epsilons=np.full(12, 0.2), positions=x,
                              box=None, method=systems.NB_NOCUTOFF, use_dispersion=False)
    atoms = np.array([[i, i+1, i+2, i+3] for i in range(9)])
    d = systems._custom_only(bare, ["lam*k*(1+cos(2*theta-theta0))", "(1-lam)*k*(theta-theta0)^2 + mu*k"],
                             [("k", "theta0"), ("k", "theta0")], np.arange(9) % 2, atoms,
                             np.stack([rng.uniform(1, 10, 9), rng.uniform(-1, 1, 9)], axis=1), ["lam", "mu"], [0.5, 0.1])
    d = harness.compiled(d)
    kw = dict(nb_globals={"lam": 0.5}, particle_offsets=[("lam", 0, 0.2, 0.0, 0.0), ("lam", 3, -0.2, 0.0, 0.0)],
              integrator=(systems.INT_VERLET, 0, 0, 0.001))
    sims = {p: harness.Simulation(d, p, **kw) for p in ("Reference", "B200")}
    for lam, mu in ((0.5, 0.1), (0.2, 0.1), (0.9, -0.4), (0.0, 0.0)):
        for s in sims.values():
            s.set_parameter("lam", lam)
            s.set_parameter("mu", mu)
            s.step(2)
        (f, e), (fr, er) = sims["B200"].forces_energy(), sims["Reference"].forces_energy()
        assert abs(e - er) <= 1e-5*max(1.0, abs(er)), (lam, mu, e, er)
        assert relative_force_error(f, fr) < 1e-4


def test_new_global_values_do_not_instantiate_the_step_graph(harness):
    from openmm_b200 import Engine, engine, systems
    d = harness.compiled(_tiny(harness))
    eng = Engine(d)
    eng.set_integrator(systems.INT_LANGEVIN_MIDDLE, 0.001, 300.0, 1.0, 7)
    eng.step(3)
    n0 = eng.stats()["graph_instantiations"]
    for lam in (0.1, 0.7, 1.3):
        eng.set_custom_globals([lam])
        eng.step(2)
        assert eng.stats()["graph_instantiations"] == n0
        e = eng.compute(engine.TERM_CUSTOM_TORSIONS)
        x = eng.get_positions()
        d2 = harness.compiled(_tiny(harness))
        d2.positions, d2.custom_global_values = x, np.array([lam])
        fresh = Engine(d2)
        assert abs(fresh.compute(engine.TERM_CUSTOM_TORSIONS) - e) <= 1e-12*max(1.0, abs(e))
        fresh.close()
    with pytest.raises(engine.EngineError, match="number of global parameters"):
        eng.set_custom_globals([0.1, 0.2])


def test_update_parameters_in_context(harness, dhfr_charmm):
    d = dhfr_charmm
    pme = d.pme_parameters()
    sims = {p: harness.Simulation(d, p, pme=pme, force_groups={"custom_torsions": 5}) for p in ("Reference", "B200")}
    rng = np.random.default_rng(9)
    new = np.stack([rng.uniform(50, 900, len(d.custom_prog)), rng.uniform(-np.pi, np.pi, len(d.custom_prog))], axis=1)
    for s in sims.values():
        s.update("custom", 0, d.custom_atoms, new)
    (f, e), (fr, er) = sims["B200"].forces_energy(1 << 5), sims["Reference"].forces_energy(1 << 5)
    _group_close(f, e, fr, er)
    b200 = sims["B200"]
    # changed atoms first: the count refusal below leaves the System's force one torsion longer than the Context's
    with pytest.raises(RuntimeError, match="set of particles in a torsion has changed"):
        atoms = d.custom_atoms.copy()
        atoms[3] = atoms[3][::-1]
        b200.update("custom", 0, atoms, new)
    with pytest.raises(RuntimeError, match="number of torsions has changed"):
        b200.update("custom", 0, np.concatenate([d.custom_atoms, d.custom_atoms[:1]]), np.concatenate([new, new[:1]]))


def _plugin_run(harness, d, fused, steps=30):
    from openmm_b200 import systems
    os.environ["B200MD_PLUGIN_FUSED"] = fused
    try:
        s = harness.Simulation(d, "B200", integrator=(systems.INT_LANGEVIN_MIDDLE, 300.0, 1.0, 0.002), pme=d.pme_parameters())
    finally:
        os.environ.pop("B200MD_PLUGIN_FUSED", None)
    s.set_velocities(np.random.default_rng(3).standard_normal((d.natoms, 3))*0.3)
    s.step(steps)
    x = s.state(positions=True)["positions"]
    s.close()
    return x


def test_fused_and_unfused_plugin_steps_agree(harness, dhfr_charmm):
    """LangevinMiddle through the plugin: the fused step graph and B200MD_PLUGIN_FUSED=0 (b200md_compute + integrate_only)
    follow the same trajectory.  The two paths are not bit-equal on a System without custom torsions either (DHFR-CMAP
    here; test_gpu_plugin.py bounds them on water): custom torsions must not widen the gap."""
    from openmm_b200 import systems
    gap = {}
    for name, d in (("dhfr_cmap", systems.with_cmap(_dhfr(), *_maps())), ("dhfr_charmm", dhfr_charmm)):
        x1, x0 = _plugin_run(harness, d, "1"), _plugin_run(harness, d, "0")
        assert np.isfinite(x1).all()
        gap[name] = float(np.abs(x1 - x0).max())
    print("fused - unfused after 30 steps (nm):", gap)
    assert gap["dhfr_charmm"] < 1e-5 and gap["dhfr_charmm"] <= 4*max(gap["dhfr_cmap"], 1e-6), gap


def _step_launches(eng):
    eng.step(1)                      # captures the step graph
    before = eng.stats()["kernel_launches"]
    eng.step(1)
    return eng.stats()["kernel_launches"] - before


# Kernel launches of one LangevinMiddle step of DHFR and of DHFR-CMAP (single and mixed precision), as the engine counted them
# before custom torsions existed: the 12 kernel nodes of the step graph (DESIGN.md section 4)
STEP_LAUNCHES_WITHOUT_CUSTOM_TORSIONS = 12


@pytest.mark.parametrize("precision", ["single", "mixed"])
def test_launches_per_step(harness, dhfr_charmm, precision):
    """custom torsions add exactly one launch per step; a System without them launches what it did before"""
    from openmm_b200 import Engine, systems
    counts = {}
    for name, d in (("dhfr", _dhfr()), ("dhfr_cmap", systems.with_cmap(_dhfr(), *_maps())), ("dhfr_charmm", dhfr_charmm)):
        eng = Engine(d, precision=precision)
        eng.set_integrator(systems.INT_LANGEVIN_MIDDLE, 0.002, 300.0, 1.0, 7)
        counts[name] = _step_launches(eng)
        eng.close()
    assert counts["dhfr"] == counts["dhfr_cmap"] == STEP_LAUNCHES_WITHOUT_CUSTOM_TORSIONS, counts
    assert counts["dhfr_charmm"] == STEP_LAUNCHES_WITHOUT_CUSTOM_TORSIONS + 1, counts


def test_empty_custom_torsion_force_with_a_global(harness):
    """a CustomTorsionForce without torsions whose expression names a global (an empty restraint or alchemical force): every
    setParameter of that global, which a NonbondedForce offset also reads, gives the Reference platform's energy"""
    from openmm_b200 import Engine, engine, systems
    base = _tiny(harness)
    q = np.array([0.4, -0.2, 0.3, -0.5])
    bare = systems.SystemDesc(masses=base.masses, charges=q, sigmas=base.sigmas, epsilons=np.full(4, 0.1), positions=base.positions,
                              box=None, method=systems.NB_NOCUTOFF, use_dispersion=False)
    d = harness.compiled(systems._custom_only(bare, ["lam*k*(1+cos(2*theta-theta0))"], [("k", "theta0")], np.zeros(0),
                                              np.zeros((0, 4)), np.zeros((0, 2)), ["lam"], [0.5]))
    kw = dict(nb_globals={"lam": 0.5}, particle_offsets=[("lam", 0, 0.2, 0.0, 0.0)])
    sims = {p: harness.Simulation(d, p, **kw) for p in ("Reference", "B200")}
    assert sims["B200"].platform() == "B200"
    for lam in (0.5, 0.2, 0.9):
        for s in sims.values():
            s.set_parameter("lam", lam)
        (f, e), (fr, er) = sims["B200"].forces_energy(), sims["Reference"].forces_energy()
        assert abs(e - er) <= 1e-5*max(1.0, abs(er)), (lam, e, er)
        assert relative_force_error(f, fr) < 1e-4
    # the engine: global values and no custom torsions
    eng = Engine(d)
    eng.set_integrator(systems.INT_LANGEVIN_MIDDLE, 0.001, 300.0, 1.0, 7)
    eng.step(2)
    eng.set_custom_globals([0.8])
    eng.step(2)
    assert eng.compute(engine.TERM_CUSTOM_TORSIONS) == 0.0


def test_mixed_precision_run(harness, dhfr_charmm):
    from openmm_b200 import Engine, engine, systems
    d = dhfr_charmm
    single, mixed = Engine(d), Engine(d, precision="mixed")
    es, em = single.compute(engine.TERM_CUSTOM_TORSIONS), mixed.compute(engine.TERM_CUSTOM_TORSIONS)
    _group_close(mixed.get_forces(), em, single.get_forces(), es)
    mixed.set_integrator(systems.INT_LANGEVIN_MIDDLE, 0.002, 300.0, 1.0, 7)
    mixed.step(200)
    x = mixed.get_positions()
    assert np.isfinite(x).all()
    for i, j, dist in zip(d.con_i[::7], d.con_j[::7], d.con_d[::7]):
        assert abs(np.linalg.norm(x[i]-x[j]) - dist) < 1e-5*dist


def test_time_phases(harness, dhfr_charmm):
    from openmm_b200 import Engine, EngineError
    eng = Engine(dhfr_charmm)
    assert eng.time_phase("custom_torsions", 3) > 0 and eng.time_phase("bonded", 3) > 0
    with pytest.raises(EngineError, match="has none"):
        Engine(_dhfr()).time_phase("custom_torsions", 3)


# ---------------------------------------------------------------------------------------------------- C-ABI input checks
def _ints(v):
    return (C.c_int*max(1, len(v)))(*v)


def _dbls(v):
    return (C.c_double*max(1, len(v)))(*v)


GOOD = dict(start=[0, 5, 6], op=[3, 2, 1, 6, 4, 2], arg=[0, 0, 0, 0, 0, 0], stride=1, prog=[0], atoms=[0, 1, 2, 3], nglobals=1)


@pytest.mark.parametrize("case,match", [
    ("negative count", "negative count"), ("atom", "atom index out of range"), ("program index", "program index out of range"),
    ("opcode", "unknown opcode"), ("param", "parameter index out of range"), ("global", "global parameter index out of range"),
    ("underflow", "stack underflow"), ("deep", "deeper than 16"), ("leftover", "exactly one value"),
    ("groups", "group array length"), ("update", "number of torsions"), ("globals after finalize", "number of global parameters"),
])
def test_cabi_refuses_malformed_input(case, match):
    from openmm_b200 import _lib
    L = _lib.load()
    h = C.c_void_p()
    assert L.b200md_create(C.byref(h), 0, 8) == 0
    try:
        g = dict(GOOD)
        n = 1
        if case == "negative count":
            n = -1
        elif case == "atom":
            g["atoms"] = [0, 1, 2, 8]
        elif case == "program index":
            g["prog"] = [1]
        elif case == "opcode":
            g["op"] = g["op"][:3] + [99] + g["op"][4:]
        elif case == "param":
            g["arg"] = [0, 1, 0, 0, 0, 0]
        elif case == "global":
            g["nglobals"] = 0
        elif case == "underflow":
            g["op"], g["start"] = [1, 4, 2], [0, 2, 3]
        elif case == "deep":
            g["op"], g["start"] = [1]*17 + [4]*16 + [2], [0, 33, 34]
        elif case == "leftover":
            g["op"], g["start"] = [1, 1, 2], [0, 2, 3]
        g["arg"] = (g["arg"] + [0]*len(g["op"]))[:len(g["op"])]
        rc = L.b200md_set_custom_torsions(h, 1, _ints(g["start"]), _ints(g["op"]), _ints(g["arg"]), _dbls([0.0]*len(g["op"])), g["stride"],
                                          n, _ints(g["prog"]), _ints(g["atoms"]), _dbls([2.0]))
        if rc == 0 and g["nglobals"]:
            rc = L.b200md_set_custom_globals(h, g["nglobals"], _dbls([0.5]*g["nglobals"]))
        if rc == 0 and case == "groups":
            rc = L.b200md_set_bonded_groups(h, 5, 2, _ints([0, 0]))
        if rc == 0:
            rc = L.b200md_finalize(h)
            assert rc != 0 or case in ("update", "globals after finalize"), L.b200md_last_error(h)
            if case == "update":
                rc = L.b200md_update_custom_torsion_params(h, 2, _dbls([1.0, 2.0]))
            elif case == "globals after finalize":
                rc = L.b200md_set_custom_globals(h, 2, _dbls([0.5, 0.5]))
        assert rc != 0
        assert match in L.b200md_last_error(h).decode()
    finally:
        L.b200md_destroy(h)
