"""GPU tests of CustomCentroidBondForce on the platform (k_centroid_centers, k_compound at the group centres,
k_centroid_scatter): the reference's own test bodies; DHFR's angles and torsions as centroid bonds over single-atom groups
against the same terms as compound bonds, bit for bit; centre-of-mass and flat-bottom restraints on DHFR against the
double-precision yardstick and a finite difference; reproducibility; continuity across a molecule wrap; updates without a new
step graph; force groups; launch counts; NVE drift; a constant-pressure run through the plugin; platform fallback; the
refusals of the set call."""
import os
import subprocess
import tempfile
import numpy as np
import pytest
from conftest import ROOT

pytestmark = pytest.mark.gpu
PLUGIN = os.path.join(ROOT, "plugin", "libOpenMMB200.so")
REFTESTS = os.path.join(ROOT, "oracle", "_ref", "tests")


@pytest.fixture(scope="module")
def harness():
    import centroid_harness
    if not centroid_harness.available() or not os.path.exists(PLUGIN):
        pytest.fail("oracle/_ref or the plugin is not built: run __graft_entry__.build() where the reference sources exist")
    centroid_harness.omm.load_plugin(PLUGIN)
    return centroid_harness


def _dhfr():
    from openmm_b200 import systems
    return systems.SystemDesc.load(os.path.join(ROOT, "data", "dhfr.npz")).rounded()


def _com_restraint(harness, d=None, weights=False, periodic=False):
    """the two solute halves held at their centre distance plus 0.1 nm, mass weighted or with weights 1, 2, 3, 1, 2, 3, .."""
    from openmm_b200 import systems
    d = _dhfr() if d is None else d
    a, b = systems.solute_halves(d)
    w = None
    if weights:
        w = [1.0 + np.arange(len(a)) % 3, 1.0 + np.arange(len(b)) % 3]
    ww = [np.asarray(d.masses)[a], np.asarray(d.masses)[b]] if w is None else w
    x = np.asarray(d.positions)
    r0 = np.linalg.norm(ww[0] @ x[a]/ww[0].sum() - ww[1] @ x[b]/ww[1].sum()) + 0.1
    return harness.compiled(systems.with_centroid_restraint(d, [a, b], systems.COM_DISTANCE_RESTRAINT, [[2000.0, r0]], ("k", "r0"),
                                                            weights=w, periodic=periodic))


def _flat_bottom(harness, d=None):
    """one half's centre held within 0.05 nm of a point 0.2 nm away, scaled by the global lam"""
    from openmm_b200 import systems
    d = _dhfr() if d is None else d
    a, _ = systems.solute_halves(d)
    m = np.asarray(d.masses)[a]
    c = m @ np.asarray(d.positions)[a]/m.sum() + [0.12, -0.1, 0.12]
    d.custom_global_names, d.custom_global_values = ("lam",), np.array([1.0])
    return harness.compiled(systems.with_centroid_restraint(d, [a], "lam*" + systems.FLAT_BOTTOM_RESTRAINT, [[3000.0, *c, 0.05]],
                                                            ("k", "x0", "y0", "z0", "rflat")))


def _group_close(f, e, fr, er, ftol=1e-5, etol=1e-6):
    assert np.abs(f - fr).max() <= ftol*np.abs(fr).max(), np.abs(f - fr).max()/np.abs(fr).max()
    assert abs(e - er) <= etol*abs(er), (e, er)


# ---------------------------------------------------------------------------------------------------- reference test bodies
@pytest.mark.parametrize("name", ["TestB200CustomCentroidBondForce", "TestB200MixedCustomCentroidBondForce"])
def test_reference_own_test_bodies_pass(name):
    exe = os.path.join(REFTESTS, name)
    if not os.path.exists(exe):
        pytest.fail("%s not built (make -C plugin reftests where the reference sources exist)" % exe)
    p = subprocess.run([exe], capture_output=True, text=True, timeout=600, env=dict(os.environ, B200_PLUGIN=PLUGIN))
    assert p.returncode == 0 and "Done" in p.stdout, p.stdout[-2000:] + p.stderr[-2000:]


# ---------------------------------------------------------------------------------------------------- against compound bonds
def test_single_atom_groups_equal_compound_bonds_bit_for_bit(harness):
    from openmm_b200 import Engine, engine, systems
    d = _dhfr()
    compound = harness.compiled(systems.torsions_to_compound(systems.angles_to_compound(d)))
    centroid = harness.compiled(systems.compound_to_centroid(compound))
    assert len(centroid.ccentroid_expr) == len(d.angle_i) + len(d.tor_i) and len(centroid.ccompound_expr) == 0
    a, b = Engine(compound), Engine(centroid)
    ea, eb = a.compute(engine.TERM_CUSTOM_COMPOUND), b.compute(engine.TERM_CUSTOM_CENTROID)
    fa, fb = a.get_forces(), b.get_forces()
    assert np.array_equal(fa, fb), np.abs(fa - fb).max()
    assert abs(ea - eb) <= 1e-12*abs(ea), (ea, eb)
    assert np.abs(fa).max() > 100.0
    assert b.compute(engine.TERM_CUSTOM_COMPOUND) == 0.0
    assert b.time_phase("custom_centroid", 3) > 0


# ---------------------------------------------------------------------------------------------------- the restraints
CASES = ["com_distance", "flat_bottom", "weighted_periodic"]


def _case(harness, case):
    if case == "com_distance":
        return _com_restraint(harness)
    if case == "flat_bottom":
        return _flat_bottom(harness)
    return _com_restraint(harness, weights=True, periodic=True)


@pytest.mark.parametrize("case", CASES)
def test_restraint_matches_the_yardstick_and_a_finite_difference(harness, case):
    from openmm_b200 import Engine, engine
    r = _case(harness, case)
    atoms = np.unique(r.ccentroid_group_atoms)
    eng = Engine(r)
    eng.compute(engine.TERM_ALL & ~engine.TERM_CUSTOM_CENTROID, energy=False)
    f_without = eng.get_forces()
    eng.compute(engine.TERM_ALL, energy=False)
    f_with = eng.get_forces()
    mask = np.ones(r.natoms, bool)
    mask[atoms] = False
    assert np.array_equal(f_with[mask], f_without[mask])          # all other atoms unchanged bit for bit
    e = eng.compute(engine.TERM_CUSTOM_CENTROID)
    f = eng.get_forces()
    assert np.array_equal(f[mask], np.zeros_like(f[mask]))
    x = eng.get_positions()
    ey, fy = harness.centroid_yardstick(r, x, box=eng.get_box())
    assert abs(e - ey) <= 1e-9*abs(ey) and abs(ey) > 0.1, (e, ey)
    assert np.abs(f - fy).max() <= 1e-6*np.abs(fy).max(), np.abs(f - fy).max()/np.abs(fy).max()
    # central finite difference of the device energy (a step of 2^-10 nm is exactly representable in fp32 here)
    h = 2.0**-10
    big = atoms[np.argsort(-np.abs(fy[atoms]).max(axis=1))[:2]]
    for a in big:
        for k in range(3):
            ee = []
            for s in (+1, -1):
                y = x.copy()
                y[a, k] = np.float32(y[a, k]) + s*h
                eng.set_positions(y)
                ee.append(eng.compute(engine.TERM_CUSTOM_CENTROID))
            fd = -(ee[0] - ee[1])/(2*h)
            assert abs(fd - f[a, k]) <= 2e-3*np.abs(fy).max() + 1e-6, (a, k, fd, f[a, k])


def test_two_evaluations_give_the_same_bits(harness):
    from openmm_b200 import Engine, engine
    eng = Engine(_com_restraint(harness, weights=True, periodic=True))
    out = []
    for _ in range(3):
        eng.compute(engine.TERM_ALL, energy=False)
        out.append(eng.get_forces())
    assert np.array_equal(out[0], out[1]) and np.array_equal(out[0], out[2])


def test_restraint_is_continuous_across_a_molecule_wrap(harness):
    """a water far outside the primary cell joins one group: the list build wraps the water back by lattice vectors, the
    centre still reads the coordinates the user gave"""
    from openmm_b200 import Engine, engine, systems
    d = _dhfr()
    box = np.asarray(d.box)
    ow = max(m[0] for m in d.molecules() if len(m) == 3)
    x = np.array(d.positions)
    x[[ow, ow + 1, ow + 2]] += 2*box[0] - box[1] + box[2]
    d.positions = x.astype(np.float32).astype(np.float64)
    a, b = systems.solute_halves(d)
    r = harness.compiled(systems.with_centroid_restraint(d, [a, np.concatenate([b, [ow, ow + 1, ow + 2]])], systems.COM_DISTANCE_RESTRAINT,
                                                         [[2000.0, 0.5]], ("k", "r0")))
    eng = Engine(r)
    e = eng.compute(engine.TERM_CUSTOM_CENTROID)
    npad = (d.natoms + 31)//32*32
    offsets = np.frombuffer(eng.checkpoint()[-12*npad:], dtype=np.int32).reshape(3, npad)
    assert (offsets[:, ow] != 0).any(), offsets[:, ow]
    ey, _ = harness.centroid_yardstick(r, d.positions)
    # one fp32 rounding of a coordinate up to 16 nm from the origin is all that may differ
    assert abs(e - ey) <= 2e-4*abs(ey), (e, ey)
    builds = eng.stats()["list_builds"]
    xs = eng.get_positions()
    eng.set_positions(xs)
    e1 = eng.compute(engine.TERM_CUSTOM_CENTROID)
    eng.set_positions(xs)
    e2 = eng.compute(engine.TERM_CUSTOM_CENTROID)
    assert eng.stats()["list_builds"] > builds
    assert abs(e1 - e2) <= 1e-9*abs(e1) and abs(e1 - e) <= 1e-9*abs(e), (e, e1, e2)


# ---------------------------------------------------------------------------------------------------- updates, groups, steps
def test_parameter_and_global_updates_keep_the_step_graph(harness):
    from openmm_b200 import Engine, engine, systems
    r = _flat_bottom(harness)
    eng = Engine(r)
    eng.set_integrator(systems.INT_LANGEVIN_MIDDLE, 0.001, 300.0, 1.0, 7)
    eng.step(3)
    n0 = eng.stats()["graph_instantiations"]
    e0 = eng.compute(engine.TERM_CUSTOM_CENTROID)
    assert e0 > 0.1
    p = r.ccentroid_params.copy()
    p[:, 0] *= 3.0
    eng.update_custom_centroid_params(p)
    assert abs(eng.compute(engine.TERM_CUSTOM_CENTROID) - 3*e0) <= 1e-9*abs(e0)
    eng.set_custom_globals([0.5])
    assert abs(eng.compute(engine.TERM_CUSTOM_CENTROID) - 1.5*e0) <= 1e-9*abs(e0)
    eng.step(2)
    assert eng.stats()["graph_instantiations"] == n0
    with pytest.raises(engine.EngineError, match="number of bonds has changed"):
        eng.update_custom_centroid_params(np.concatenate([p, p]))


def test_two_objects_in_different_force_groups(harness):
    from openmm_b200 import Engine, engine
    c = _flat_bottom(harness, _com_restraint(harness))
    eng = Engine(c, bonded_groups={"custom_centroid": [3, 4]})
    parts = [eng.compute_groups(engine.TERM_CUSTOM_CENTROID, 1 << g) for g in (3, 4)]
    assert all(p != 0.0 for p in parts) and parts[0] != parts[1]
    assert abs(sum(parts) - eng.compute(engine.TERM_CUSTOM_CENTROID)) <= 1e-9*abs(sum(parts))
    assert eng.compute_groups(engine.TERM_CUSTOM_CENTROID, 1) == 0.0
    eng.compute(engine.TERM_CUSTOM_CENTROID, energy=False)
    _, fy = harness.centroid_yardstick(c, eng.get_positions())
    assert np.abs(eng.get_forces() - fy).max() <= 1e-6*np.abs(fy).max()


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
    plain, restrained = _nve_drift(d), _nve_drift(_com_restraint(harness, d))
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
    """centroid bonds add their three kernels to an evaluation and to a step; a System without them launches what it did"""
    from openmm_b200 import Engine, systems
    d = _dhfr()
    counts, steps = {}, {}
    for name, desc in (("plain", d), ("restraint", _com_restraint(harness, d))):
        eng = Engine(desc)
        counts[name] = _eval_launches(eng)
        eng.set_integrator(systems.INT_LANGEVIN_MIDDLE, 0.002, 300.0, 1.0, 7)
        steps[name] = _step_launches(eng)
        eng.close()
    assert counts["restraint"] == counts["plain"] + 3, counts
    assert steps["restraint"] == steps["plain"] + 3, steps


# ---------------------------------------------------------------------------------------------------- through the plugin
def test_through_the_plugin_matches_reference_platform(harness):
    d = _flat_bottom(harness, _com_restraint(harness, weights=True))
    groups = {"custom_centroid": 6}
    ref = harness.Simulation(d, "Reference", pme=d.pme_parameters(), force_groups=groups)
    b200 = harness.Simulation(d, "B200", pme=d.pme_parameters(), force_groups=groups)
    assert b200.platform() == "B200"
    (f, e), (fr, er) = b200.forces_energy(1 << 6), ref.forces_energy(1 << 6)
    _group_close(f, e, fr, er)
    p = d.ccentroid_params.copy()
    p[0, 1] += 0.05
    sel = d.ccentroid_expr == 0
    for s in (ref, b200):
        s.update("ccentroid", 0, d.ccentroid_atoms[sel, :2], p[sel, :2])
        s.set_parameter("lam", 0.7)
    (f, e), (fr, er) = b200.forces_energy(1 << 6), ref.forces_energy(1 << 6)
    _group_close(f, e, fr, er)
    with pytest.raises(RuntimeError, match="set of groups in a bond has changed"):
        b200.update("ccentroid", 0, d.ccentroid_atoms[sel, :2][:, ::-1], p[sel, :2])
    with pytest.raises(RuntimeError, match="number of bonds has changed"):
        b200.update("ccentroid", 0, np.concatenate([d.ccentroid_atoms[sel, :2]]*2), np.concatenate([p[sel, :2]]*2))


def test_npt_run_through_the_plugin_matches_reference_at_the_end(harness):
    """LangevinMiddle + MonteCarloBarostat with the two-domain restraint, 200 steps on B200 (the barostat's molecules from
    ContextImpl::getMolecules), then the final positions and box evaluated on both platforms"""
    import barostat_harness
    from oracle import omm
    d = _com_restraint(harness)
    pme = d.pme_parameters()
    groups = {"custom_centroid": 6}
    with tempfile.TemporaryDirectory() as work:
        xml, pos, out = (os.path.join(work, f) for f in ("system.xml", "positions.f64", "out.bin"))
        sim = harness.Simulation(d, "Reference", pme=pme, force_groups=groups)
        assert omm.lib().omm_system_serialize(sim.sys, xml.encode()) == 0
        sim.close()
        np.ascontiguousarray(d.positions, dtype="<f8").tofile(pos)
        r = subprocess.run([barostat_harness.RUN_NPT, xml, pos, out, "--platform", "B200", "--plugin", PLUGIN, "--frequency", "10",
                            "--chunks", "1", "--chunk-steps", "200"], capture_output=True, text=True, timeout=1200, cwd=ROOT)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
        raw = open(out, "rb").read()
    nmol = int(np.frombuffer(raw, "<i4", 1)[0])
    start = np.frombuffer(raw, "<i4", nmol + 1, 4)
    frames = np.frombuffer(raw, "<f8", offset=4*(nmol + 2) + 4*int(start[-1])).reshape(-1, 3 + d.natoms, 3)
    box, x = frames[-1, :3].copy(), frames[-1, 3:].copy()
    assert not np.array_equal(box, np.asarray(d.box))
    import copy
    e2 = copy.copy(d)
    e2.box, e2.positions = box, x
    ref = harness.Simulation(e2, "Reference", pme=pme, force_groups=groups)
    b200 = harness.Simulation(e2, "B200", pme=pme, force_groups=groups)
    (f, e), (fr, er) = b200.forces_energy(1 << 6), ref.forces_energy(1 << 6)
    _group_close(f, e, fr, er)
    (_, e), (_, er) = b200.forces_energy(), ref.forces_energy()
    assert abs(e - er) <= 1e-4*abs(er), (e, er)


def _small(energy, groups_per_bond, names=(), ngroups=None):
    from openmm_b200 import systems
    n = max(groups_per_bond if ngroups is None else ngroups, 2)
    x = np.random.default_rng(1).uniform(0, 1, (n, 3)).astype(np.float32).astype(np.float64)
    bare = systems.SystemDesc(masses=np.full(n, 12.0), charges=np.zeros(n), sigmas=np.full(n, 0.3), epsilons=np.zeros(n), positions=x,
                              box=None, method=systems.NB_NOCUTOFF, use_dispersion=False)
    return systems.with_centroid_restraint(bare, [[g] for g in range(n)], energy, np.zeros((1, len(names))), names,
                                           bonds=[list(range(groups_per_bond))])


@pytest.mark.parametrize("case,match", [("tabulated", "tabulated functions in a CustomCentroidBondForce"),
                                        ("nine groups", "more than 8 groups per bond"),
                                        ("derivative", "energy parameter derivatives of a CustomCentroidBondForce")])
def test_unsupported_centroid_forces_move_the_context_elsewhere(harness, case, match):
    kw = {}
    if case == "tabulated":
        d, kw = _small("fn(distance(g1,g2))", 2), dict(tabulated=True)
    elif case == "nine groups":
        # a desc holds at most 8 groups per bond: nine groups, one bond over the first eight, then widened to all nine
        d = _small("+".join("x%d" % i for i in range(1, 10)), 8, ngroups=9)
        d.ccentroid_groups_per_bond, d.ccentroid_atoms = np.array([9], dtype=np.int32), np.arange(9, dtype=np.int32).reshape(1, 9)
    else:
        d = _small("lam*distance(g1,g2)", 2)
        d.custom_global_names, d.custom_global_values = ("lam",), np.array([1.0])
        kw = dict(deriv_params={"custom_centroid": "lam"})
    s = harness.Simulation(d, "Reference", **kw)
    assert s.default_platform() not in ("", "B200")
    with pytest.raises(RuntimeError, match=match):
        harness.Simulation(d, "B200", **kw)


@pytest.mark.parametrize("case,match", [
    ("group index", "custom centroid bond: group index out of range"),
    ("unused slot", "custom centroid bond: an unused group slot must be -1"),
    ("empty group", "custom centroid bond: a group must hold at least one atom"),
    ("atom index", "custom centroid bond: atom index of a group out of range"),
    ("weight", "custom centroid bond: a group weight is not finite"),
    ("program", "custom centroid program: variable index out of range"),
])
def test_the_set_call_refuses_malformed_input(harness, case, match):
    from openmm_b200 import Engine, engine
    d = harness.compiled(_small("distance(g1,g2)", 2))
    if case == "group index":
        d.ccentroid_atoms = d.ccentroid_atoms.copy(); d.ccentroid_atoms[0, 1] = 2
    elif case == "unused slot":
        d.ccentroid_atoms = d.ccentroid_atoms.copy(); d.ccentroid_atoms[0, 2] = 0
    elif case == "empty group":
        d.ccentroid_group_start = np.array([0, 1, 1], dtype=np.int32)
    elif case == "atom index":
        d.ccentroid_group_atoms = np.array([0, 5], dtype=np.int32)
    elif case == "weight":
        d.ccentroid_group_weights = np.array([1.0, np.nan])
    else:
        d.ccentroid_op, d.ccentroid_arg = d.ccentroid_op.copy(), d.ccentroid_arg.copy()
        d.ccentroid_op[0], d.ccentroid_arg[0] = 42, 6           # VAR 6 of a two-group bond
    with pytest.raises(engine.EngineError, match=match):
        Engine(d)
