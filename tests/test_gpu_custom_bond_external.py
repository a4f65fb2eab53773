"""GPU tests of CustomBondForce and CustomExternalForce on the platform (k_custom, the expression programs of
plugin/custom_translate.h): the reference's own test bodies; DHFR's harmonic bonds as custom bonds against the bonds; position
restraints on DHFR's solute heavy atoms through the plugin against the live Reference platform, per force group; the continuous
coordinate an external reads after the molecule wrap; global parameters shared with custom torsions, parameter updates,
platform fallback, launch counts, the step paths; the C-ABI's input checks."""
import ctypes as C
import os
import subprocess
import numpy as np
import pytest
from conftest import relative_force_error, ROOT, GOLDEN

pytestmark = pytest.mark.gpu
PLUGIN = os.path.join(ROOT, "plugin", "libOpenMMB200.so")
REFTESTS = os.path.join(ROOT, "oracle", "_ref", "tests")
RESTRAINT_K = 400.0          # kJ/mol/nm^2


@pytest.fixture(scope="module")
def harness():
    """the translator, Lepton and the reference's custom forces (tests/custom_harness.py), with the plugin loaded"""
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


def _restrained(harness, d, periodic=True):
    from openmm_b200 import systems
    atoms = systems.solute_heavy_atoms(d)
    assert len(atoms) == 1268
    return harness.compiled(systems.with_position_restraints(d, atoms, RESTRAINT_K, periodic=periodic))


@pytest.fixture(scope="module")
def dhfr_charmm(harness):
    from openmm_b200 import systems
    return systems.with_cmap(systems.with_charmm_impropers(_dhfr()), *_maps())


def _group_close(f, e, fr, er):
    """one group alone: both sides are double, only the 2^-32 fixed-point force resolution differs"""
    assert np.abs(f - fr).max() <= 1e-6*np.abs(fr).max()
    assert abs(e - er) <= 1e-8*abs(er)


# ---------------------------------------------------------------------------------------------------- reference test bodies
@pytest.mark.parametrize("name", ["TestB200CustomBondForce", "TestB200MixedCustomBondForce", "TestB200CustomExternalForce",
                                  "TestB200MixedCustomExternalForce"])
def test_reference_own_test_bodies_pass(name):
    exe = os.path.join(REFTESTS, name)
    if not os.path.exists(exe):
        pytest.fail("%s not built (make -C plugin reftests where /root/reference exists)" % exe)
    p = subprocess.run([exe], capture_output=True, text=True, timeout=600, env=dict(os.environ, B200_PLUGIN=PLUGIN))
    assert p.returncode == 0 and "Done" in p.stdout, p.stdout[-2000:] + p.stderr[-2000:]


# ---------------------------------------------------------------------------------------------------- engine
def test_custom_bonds_equal_harmonic_bonds_on_the_engine(harness):
    from openmm_b200 import Engine, engine, systems
    d = _dhfr()
    ref = Engine(d)
    eb = ref.compute(engine.TERM_BONDS)
    fb = ref.get_forces()
    c = harness.compiled(systems.bonds_to_custom(d))
    assert len(c.cbond_prog) == 1302 and len(c.bond_i) == 0
    cus = Engine(c)
    ec = cus.compute(engine.TERM_CUSTOM_BONDS)
    _group_close(cus.get_forces(), ec, fb, eb)
    # the class bits select: custom torsions alone see none of the bonds
    assert cus.compute(engine.TERM_CUSTOM_TORSIONS) == 0.0


# ---------------------------------------------------------------------------------------------------- through the plugin
MASKS = (1 << 5, 1 << 4, (1 << 4) | (1 << 5), 1, 1 | (1 << 5), 0xffffffff)


@pytest.mark.parametrize("periodic", [True, False], ids=["periodicdistance", "plain"])
def test_position_restraints_through_the_plugin_match_reference_platform(harness, periodic):
    d = _restrained(harness, _dhfr(), periodic)
    pme = d.pme_parameters()
    groups = {"custom_externals": 5}
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


def test_restraint_reads_the_continuous_coordinate(harness):
    """one DHFR water two box lengths outside the primary cell, its oxygen restrained by the plain form: the list build's
    molecule wrap moves the water back by lattice vectors, and the restraint still sees the coordinate the user sees.  The
    only difference allowed is one fp32 rounding of that coordinate (8 to 16 nm from the origin): 2^-20 nm per component.  A
    restraint reading the raw wrapped coordinate would be two box lengths off."""
    from openmm_b200 import Engine, engine, systems
    d = _dhfr()
    box = np.asarray(d.box)
    ow = max(m[0] for m in d.molecules() if len(m) == 3)
    x = np.array(d.positions)
    mol = [ow, ow + 1, ow + 2]
    x[mol] += 2*box[0] + 2*box[1] - 2*box[2]
    d.positions = x.astype(np.float32).astype(np.float64)
    r = harness.compiled(systems.with_position_restraints(d, [ow], RESTRAINT_K, periodic=False))
    eps = 2.0**-20
    ref = harness.Simulation(r, "Reference", force_groups={"custom_externals": 5})
    fr, er = ref.forces_energy(1 << 5)
    dist = np.linalg.norm(np.array(systems.RESTRAINT_OFFSET))
    de_bound = RESTRAINT_K*(2*dist*np.sqrt(3)*eps + 3*eps*eps)
    b200 = harness.Simulation(r, "B200", force_groups={"custom_externals": 5})
    f, e = b200.forces_energy(1 << 5)
    assert abs(e - er) <= de_bound, (e, er, de_bound)
    assert np.abs(f - fr).max() <= 2*RESTRAINT_K*eps + 1e-6, np.abs(f - fr).max()
    # on the engine, with evidence that the wrap happened: the checkpoint ends with cellOffset [3][npad]
    eng = Engine(r)
    e2 = eng.compute(engine.TERM_CUSTOM_EXTERNALS)
    npad = (d.natoms + 31)//32*32
    offsets = np.frombuffer(eng.checkpoint()[-12*npad:], dtype=np.int32).reshape(3, npad)
    assert (offsets[:, ow] != 0).any(), offsets[:, ow]
    assert abs(e2 - er) <= de_bound
    assert np.abs(eng.get_forces() - fr).max() <= 2*RESTRAINT_K*eps + 1e-6
    assert np.abs(eng.get_positions()[ow] - d.positions[ow]).max() <= eps


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


def _three_classes(harness):
    """12 atoms, one global `lam` read by a custom torsion, a custom bond and a custom external expression"""
    from openmm_b200 import systems
    rng = np.random.default_rng(3)
    x = _chain(12, rng, start=(1.0, 1.0, 1.0)).astype(np.float32).astype(np.float64)
    q = np.where(np.arange(12) % 2, 0.3, -0.3)
    bare = systems.SystemDesc(masses=np.full(12, 12.0), charges=q, sigmas=np.full(12, 0.3), epsilons=np.full(12, 0.2), positions=x,
                              box=None, method=systems.NB_NOCUTOFF, use_dispersion=False)
    d = systems._custom_only(bare, ["lam*k*(1+cos(2*theta-theta0))"], [("k", "theta0")], np.zeros(9),
                             np.array([[i, i+1, i+2, i+3] for i in range(9)]), np.stack([rng.uniform(1, 10, 9), rng.uniform(-1, 1, 9)], axis=1),
                             ["lam"], [0.5])
    d = systems._with_custom_class(d, "cbond", ["(1-lam)*k*(r-r0)^2 + lam*step(r-r0)*k*(r-r0)^2"], [("k", "r0")], np.zeros(11),
                                   np.array([[i, i+1] for i in range(11)]), np.stack([rng.uniform(100, 500, 11), rng.uniform(0.12, 0.18, 11)], axis=1))
    ext = np.arange(0, 12, 2)
    d = systems._with_custom_class(d, "cext", ["lam*k*((x-x0)^2+(y-y0)^2+(z-z0)^2)"], [("k", "x0", "y0", "z0")], np.zeros(len(ext)), ext,
                                   np.concatenate([np.full((len(ext), 1), 300.0), x[ext] + 0.02], axis=1))
    return harness.compiled(d)


def test_one_global_read_by_three_classes_follows_set_parameter(harness):
    from openmm_b200 import systems
    d = _three_classes(harness)
    kw = dict(integrator=(systems.INT_VERLET, 0, 0, 0.001))
    sims = {p: harness.Simulation(d, p, **kw) for p in ("Reference", "B200")}
    assert sims["B200"].platform() == "B200"
    for lam in (0.5, 0.2, 0.9, 0.0):
        for s in sims.values():
            s.set_parameter("lam", lam)
            s.step(2)
        (f, e), (fr, er) = sims["B200"].forces_energy(), sims["Reference"].forces_energy()
        assert abs(e - er) <= 1e-5*max(1.0, abs(er)), (lam, e, er)
        assert relative_force_error(f, fr) < 1e-4


def test_new_global_values_do_not_instantiate_the_step_graph(harness):
    from openmm_b200 import Engine, engine, systems
    d = _three_classes(harness)
    eng = Engine(d)
    eng.set_integrator(systems.INT_LANGEVIN_MIDDLE, 0.001, 300.0, 1.0, 7)
    eng.step(3)
    n0 = eng.stats()["graph_instantiations"]
    for lam in (0.1, 0.7):
        eng.set_custom_globals([lam])
        eng.step(2)
        assert eng.stats()["graph_instantiations"] == n0
        e = eng.compute(engine.TERM_CUSTOM_BONDS | engine.TERM_CUSTOM_EXTERNALS)
        d2 = _three_classes(harness)
        d2.positions, d2.custom_global_values = eng.get_positions(), np.array([lam])
        fresh = Engine(d2)
        assert abs(fresh.compute(engine.TERM_CUSTOM_BONDS | engine.TERM_CUSTOM_EXTERNALS) - e) <= 1e-12*max(1.0, abs(e))
        fresh.close()


def test_update_parameters_in_context(harness):
    d = _three_classes(harness)
    sims = {p: harness.Simulation(d, p) for p in ("Reference", "B200")}
    rng = np.random.default_rng(9)
    nb, ne = len(d.cbond_prog), len(d.cext_prog)
    bonds = np.stack([rng.uniform(100, 900, nb), rng.uniform(0.1, 0.2, nb)], axis=1)
    ext = np.concatenate([rng.uniform(50, 500, (ne, 1)), d.positions[d.cext_atoms] - 0.03], axis=1)
    for s in sims.values():
        s.update("cbond", 0, d.cbond_atoms, bonds)
        s.update("cext", 0, d.cext_atoms, ext)
    (f, e), (fr, er) = sims["B200"].forces_energy(), sims["Reference"].forces_energy()
    assert abs(e - er) <= 1e-5*max(1.0, abs(er)) and relative_force_error(f, fr) < 1e-4
    b200 = sims["B200"]
    with pytest.raises(RuntimeError, match="set of particles in a bond has changed"):
        atoms = d.cbond_atoms.copy()
        atoms[3] = atoms[3][::-1]
        b200.update("cbond", 0, atoms, bonds)
    with pytest.raises(RuntimeError, match="A particle index has changed"):
        atoms = d.cext_atoms.copy()
        atoms[2] += 1
        b200.update("cext", 0, atoms, ext)
    with pytest.raises(RuntimeError, match="number of bonds has changed"):
        b200.update("cbond", 0, np.concatenate([d.cbond_atoms, d.cbond_atoms[:1]]), np.concatenate([bonds, bonds[:1]]))
    with pytest.raises(RuntimeError, match="number of particles has changed"):
        b200.update("cext", 0, np.concatenate([d.cext_atoms, d.cext_atoms[:1]]), np.concatenate([ext, ext[:1]]))


def test_energy_parameter_derivatives_move_the_context_elsewhere(harness):
    d = _three_classes(harness)
    s = harness.Simulation(d, "Reference", deriv_params={"custom_bonds": "lam"})
    assert s.default_platform() not in ("", "B200")
    with pytest.raises(RuntimeError, match="energy parameter derivatives of a CustomBondForce"):
        harness.Simulation(d, "B200", deriv_params={"custom_bonds": "lam"})


def _step_launches(eng):
    eng.step(1)                      # captures the step graph
    before = eng.stats()["kernel_launches"]
    eng.step(1)
    return eng.stats()["kernel_launches"] - before


# Kernel launches of one LangevinMiddle step of DHFR (the 12 kernel nodes of the step graph, DESIGN.md section 4); DHFR-CHARMM
# has one more, k_custom for its impropers
STEP_LAUNCHES_DHFR = 12


@pytest.mark.parametrize("precision", ["single", "mixed"])
def test_launches_per_step(harness, dhfr_charmm, precision):
    """restraints add one launch to DHFR and none to DHFR-CHARMM, whose custom torsions already launch k_custom"""
    from openmm_b200 import Engine, systems
    counts = {}
    charmm = harness.compiled(dhfr_charmm)
    for name, d in (("dhfr", _dhfr()), ("dhfr_restrained", _restrained(harness, _dhfr())), ("dhfr_charmm", charmm),
                    ("dhfr_charmm_restrained", _restrained(harness, charmm))):
        eng = Engine(d, precision=precision)
        eng.set_integrator(systems.INT_LANGEVIN_MIDDLE, 0.002, 300.0, 1.0, 7)
        counts[name] = _step_launches(eng)
        eng.close()
    assert counts["dhfr"] == STEP_LAUNCHES_DHFR and counts["dhfr_charmm"] == STEP_LAUNCHES_DHFR + 1, counts
    assert counts["dhfr_restrained"] == STEP_LAUNCHES_DHFR + 1, counts
    assert counts["dhfr_charmm_restrained"] == counts["dhfr_charmm"], counts


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


def test_fused_and_unfused_plugin_steps_agree(harness):
    """LangevinMiddle through the plugin: the fused step graph and B200MD_PLUGIN_FUSED=0 follow the same trajectory with
    restraints as closely as the custom-torsion test requires (1e-5 nm after 30 steps)"""
    d = _restrained(harness, _dhfr())
    x1, x0 = _plugin_run(harness, d, "1"), _plugin_run(harness, d, "0")
    assert np.isfinite(x1).all()
    gap = float(np.abs(x1 - x0).max())
    print("fused - unfused after 30 steps (nm):", gap)
    assert gap < 1e-5, gap


def test_time_phase_of_restraints_alone(harness):
    from openmm_b200 import Engine
    eng = Engine(_restrained(harness, _dhfr()))
    assert eng.time_phase("custom_torsions", 3) > 0


# ---------------------------------------------------------------------------------------------------- C-ABI input checks
def _ints(v):
    return (C.c_int*max(1, len(v)))(*v)


def _dbls(v):
    return (C.c_double*max(1, len(v)))(*v)


OP_PARAM, OP_MUL, OP_VAR = 2, 6, 42


@pytest.mark.parametrize("call,case,match", [
    ("bonds", "atom", "custom bond: atom index out of range"), ("externals", "atom", "custom external: atom index out of range"),
    ("bonds", "program index", "custom bond: program index out of range"),
    ("externals", "variable", "custom external program: variable index out of range"),
    ("bonds", "variable", "custom bond program: variable index out of range"),
    ("bonds", "update", "The number of bonds has changed"), ("externals", "update", "The number of particles has changed"),
    ("bonds", "kind", "kind must be"),
])
def test_cabi_refuses_malformed_input(call, case, match):
    from openmm_b200 import _lib
    L = _lib.load()
    h = C.c_void_p()
    assert L.b200md_create(C.byref(h), 0, 8) == 0
    try:
        # E = PARAM 0 * VAR 0, then its derivative(s) PARAM 0
        nv = 1 if call == "bonds" else 3
        op, arg = [OP_PARAM, OP_VAR, OP_MUL] + [OP_PARAM]*nv, [0, 0, 0] + [0]*nv
        start = [0, 3] + [4 + k for k in range(nv)]
        atoms, prog = ([0, 1] if call == "bonds" else [3]), [0]
        if case == "atom":
            atoms[-1] = 8
        elif case == "program index":
            prog = [1]
        elif case == "variable":
            arg[1] = nv
        fn = L.b200md_set_custom_bonds if call == "bonds" else L.b200md_set_custom_externals
        rc = fn(h, 1, _ints(start), _ints(op), _ints(arg), _dbls([0.0]*len(op)), 1, 1, _ints(prog), _ints(atoms), _dbls([2.0]))
        if rc == 0 and case == "kind":
            rc = L.b200md_set_bonded_groups(h, 8, 1, _ints([0]))
        if rc == 0:
            assert case == "update", L.b200md_last_error(h)
            assert L.b200md_finalize(h) == 0, L.b200md_last_error(h)
            upd = L.b200md_update_custom_bond_params if call == "bonds" else L.b200md_update_custom_external_params
            rc = upd(h, 2, _dbls([1.0, 2.0]))
        assert rc != 0
        assert match in L.b200md_last_error(h).decode()
    finally:
        L.b200md_destroy(h)
