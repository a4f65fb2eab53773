"""CPU tests: the plain-C oracle (oracle/md_oracle.c) pinned against the reference's golden vectors and against
fixtures generated from the reference itself (tests/golden/make_golden.py)."""
import json
import os
import numpy as np
import pytest
from conftest import relative_force_error, GOLDEN, ROOT
from openmm_b200 import systems
from oracle import port


def _triclinic_desc():
    g = json.load(open(os.path.join(GOLDEN, "ewald_triclinic_gromacs.json")))
    n = 8
    d = systems.SystemDesc(masses=np.ones(n), charges=np.array(g["charges"]), sigmas=np.array(g["sigmas"]), epsilons=np.array(g["epsilons"]),
                           positions=np.array(g["positions"]), box=np.array(g["box"]), method=systems.NB_PME, cutoff=g["cutoff"],
                           pme_alpha=g["alpha"], pme_grid=tuple(g["grid"]), use_dispersion=False, name="triclinic8")
    return d, g


def test_port_matches_gromacs_golden_triclinic():
    # tests/TestEwald.h:222-271, tolerance 1e-4 there
    d, g = _triclinic_desc()
    f, e, parts = port.forces_energy(d)
    assert relative_force_error(f, np.array(g["expected_forces"])) < 1e-4
    assert abs(e - g["expected_energy"])/abs(g["expected_energy"]) < 1e-4


def test_port_matches_reference_nacl_amorph():
    z = np.load(os.path.join(GOLDEN, "nacl_amorph.npz"))
    n = 894
    L = float(z["box"])
    d = systems.SystemDesc(masses=np.ones(n), charges=z["charges"], sigmas=np.ones(n), epsilons=np.zeros(n), positions=z["positions"],
                           box=np.diag([L, L, L]), method=systems.NB_PME, cutoff=float(z["cutoff"]), ewald_tol=float(z["ewald_tol"]))
    pme = z["pme"]
    f, e, _ = port.forces_energy(d, pme=(float(pme[0]), int(pme[1]), int(pme[2]), int(pme[3])))
    assert relative_force_error(f, z["reference_forces"]) < 1e-9
    assert abs(e - float(z["reference_energy"])) < 1e-6*abs(e)
    assert abs(e - float(z["gromacs_energy"])) < 1e-5*abs(e)     # TestEwald.h:150 quotes -3.82047e5


def test_port_matches_reference_water():
    z = np.load(os.path.join(GOLDEN, "water5_reference.npz"))
    d = systems.water_box(5, cutoff=0.75).rounded()
    assert np.array_equal(d.positions, z["positions"])      # the seeded recipe is reproducible
    pme = z["pme"]
    f, e, _ = port.forces_energy(d, pme=(float(pme[0]), int(pme[1]), int(pme[2]), int(pme[3])))
    assert relative_force_error(f, z["reference_forces"]) < 1e-9
    assert abs(e - float(z["reference_energy"])) < 1e-9*abs(e)


def test_port_fft_matches_numpy():
    rng = np.random.default_rng(0)
    x = rng.standard_normal((6, 5, 7)) + 1j*rng.standard_normal((6, 5, 7))
    assert np.abs(port.fft3d_forward(x) - np.fft.fftn(x)).max() < 1e-11


def test_port_settle_restores_constraints():
    d = systems.water_box(3, cutoff=0.4)
    cl = port.settle_clusters(d)
    assert len(cl[0]) == 27
    rng = np.random.default_rng(1)
    x = d.positions.copy()
    v = rng.standard_normal(x.shape)*0.5
    f = rng.standard_normal(x.shape)*100
    port.step(d, 0, 0.002, 0.0, x, v, f, cl)
    for i, j, dist in zip(d.con_i, d.con_j, d.con_d):
        assert abs(np.linalg.norm(x[i]-x[j]) - dist) < 1e-12
    # centre of mass of each molecule moves as if unconstrained (SETTLE conserves momentum)
    assert np.isfinite(v).all()


def test_dispersion_and_pme_parameter_restatements():
    d = systems.water_box(20)
    alpha, nx, ny, nz = d.pme_parameters()
    assert abs(alpha - 2.9203) < 1e-4 and (nx, ny, nz) == (56, 56, 56)      # SURVEY.md 8(d), probed on the reference
    assert systems.next_fft_size(57) == 60 and systems.fft_size_ok(88) and not systems.fft_size_ok(34)


def test_system_desc_roundtrip(tmp_path):
    d = systems.water_box(2, cutoff=0.3)
    p = str(tmp_path/"w.npz")
    d.save(p)
    e = systems.SystemDesc.load(p)
    assert e.natoms == d.natoms and np.array_equal(e.positions, d.positions) and e.method == d.method and np.array_equal(e.con_i, d.con_i)


# ---- the restatement against the unmodified Reference platform: what it computed for these inputs, stored by
# tests/golden/make_golden.py in reference_platform.npz ----
def _ref():
    return np.load(os.path.join(GOLDEN, "reference_platform.npz"))


def _cases():
    yield "pme_triclinic_ions", systems.random_ions(n=120, box=2.2, cutoff=0.9, triclinic=True).rounded()
    yield "cutoff_periodic_rf", systems.lj_fluid(n_side=5, cutoff=0.8, method=systems.NB_CUTOFF_PERIODIC, charged=True).rounded()
    d = systems.lj_fluid(n_side=5, cutoff=0.8, method=systems.NB_CUTOFF_PERIODIC, charged=True).rounded()
    d.use_switch, d.switch_distance = True, 0.65
    yield "cutoff_periodic_switch", d
    yield "nocutoff_cluster", systems.cluster(n=60).rounded()
    yield "pme_flexible_water_bonded", systems.water_box(3, cutoff=0.45, rigid=False).rounded()


@pytest.mark.parametrize("name", ["pme_triclinic_ions", "cutoff_periodic_rf", "cutoff_periodic_switch", "nocutoff_cluster", "pme_flexible_water_bonded"])
def test_port_matches_live_reference_platform(name):
    """Every branch of the path the GPU parity tests lean on the port for: PME in a triclinic cell, reaction field, the
    switching function, no cutoff, bonded terms + exceptions + exclusion correction (ReferenceKernels.cpp:967-1014)."""
    ref = _ref()
    d = dict(_cases())[name]
    pme = d.pme_parameters() if d.method == systems.NB_PME else None
    f, e, _ = port.forces_energy(d, pme=pme)
    fr, er = ref["port_%s:f" % name], float(ref["port_%s:e" % name])
    assert relative_force_error(f, fr) < 1e-8
    assert abs(e - er) < 1e-8*max(1.0, abs(er))


@pytest.mark.parametrize("kind,friction", [(0, 0.0), (1, 0.0), (1, 5.0), (2, 0.0), (2, 5.0)])
def test_port_integrator_matches_live_reference(kind, friction):
    """Deterministic updates (Verlet; Langevin and LangevinMiddle at zero temperature, with and without friction) with
    SETTLE on positions and -- LangevinMiddle -- on velocities, 5 steps (ReferenceVerletDynamics.cpp,
    ReferenceStochasticDynamics.cpp:89-194, ReferenceLangevinMiddleDynamics.cpp:54-127, ReferenceSETTLEAlgorithm.cpp)."""
    ref = _ref()
    d = systems.water_box(3, cutoff=0.45).rounded()
    pme = d.pme_parameters()
    x = d.positions.copy()
    v = np.zeros_like(x)
    cl = port.settle_clusters(d)
    for _ in range(5):
        f, _, _ = port.forces_energy(d, positions=x, pme=pme)
        port.step(d, kind, 0.002, friction, x, v, f, cl)
    key = "port_integrate%d_%g:" % (kind, friction)
    st = {"positions": ref[key + "x"], "velocities": ref[key + "v"]}
    # measured 4e-9 nm after 5 steps (the port integrates from its own forces, which differ from the reference's at 1e-9)
    assert np.abs(x - st["positions"]).max() < 1e-7
    assert np.abs(v - st["velocities"]).max() < 1e-4
    assert np.abs(v).max() > 0.05            # the molecules did move: the comparison is not of zeros


def test_port_velocity_settle_removes_bond_velocities_for_unequal_masses():
    """ReferenceSETTLEAlgorithm::applyToVelocities (:197-244) allows three different masses; after it the relative velocity
    along every bond of the triangle is zero and the total momentum of the molecule is unchanged."""
    L = port.lib()
    rng = np.random.default_rng(11)
    x = np.array([[0.0, 0.0, 0.0], [0.0957, 0.0, 0.0], [-0.024, 0.0927, 0.0]]) + 0.3
    m = np.array([15.999, 1.008, 2.014])
    v = rng.normal(size=(3, 3))
    p0 = (m[:, None]*v).sum(0)
    a = [np.array([k], dtype=np.int32) for k in range(3)]
    L.orc_settle_velocities(1, port._ip(a[0]), port._ip(a[1]), port._ip(a[2]), port._dp(m), port._dp(x), port._dp(v))
    for i, j in ((0, 1), (1, 2), (2, 0)):
        e = (x[j]-x[i])/np.linalg.norm(x[j]-x[i])
        assert abs(np.dot(v[j]-v[i], e)) < 1e-13
    assert np.abs((m[:, None]*v).sum(0) - p0).max() < 1e-13


def test_port_parameter_offsets_match_live_reference():
    """NonbondedForce global parameters with particle and exception offsets (SURVEY.md section 8 row a2,
    ReferenceKernels.cpp:1077-1121): at the default values and after Context::setParameter, PME with bonded terms.  The two
    exception offsets sit on water O-H exclusions whose base parameters are zero (they must become live 1-4 terms,
    :873-895); the dispersion correction keeps the DEFAULT values (NonbondedForceImpl.cpp:241-258)."""
    ref = _ref()
    d = systems.water_box(3, cutoff=0.45, rigid=False).rounded()
    pme = d.pme_parameters()
    glob = {"lambda_q": 0.25, "lambda_lj": 1.0}
    p_off = [("lambda_q", 0, 0.3, 0.0, 0.0), ("lambda_q", 1, -0.3, 0.0, 0.0), ("lambda_lj", 3, 0.0, 0.02, 0.25), ("lambda_lj", 6, 0.1, -0.01, 0.5),
             ("lambda_q", 6, 0.05, 0.0, 0.0)]
    e_off = [("lambda_lj", 0, 0.04, 0.2, 0.3), ("lambda_q", 4, -0.02, 0.15, 0.1)]
    assert d.exc_qq[0] == 0 and d.exc_eps[0] == 0
    disp = port.with_parameter_offsets(d, glob, p_off, e_off).dispersion_coefficient()
    seen = []
    for k, values in enumerate((glob, {"lambda_q": -0.5, "lambda_lj": 0.4})):
        # the Reference platform after Context::setParameter of each value in turn
        eff = port.with_parameter_offsets(d, values, p_off, e_off)
        f, e, parts = port.forces_energy(eff, pme=pme, dispersion_coefficient=disp)
        fr, er = ref["port_offsets%d:f" % k], float(ref["port_offsets%d:e" % k])
        assert relative_force_error(f, fr) < 1e-8
        assert abs(e - er) < 1e-8*max(1.0, abs(er))
        seen.append(e)
    assert abs(seen[0] - seen[1]) > 1.0                    # the parameters do change the answer
    # and the dispersion term of the second state, computed from ITS parameters, would have been different
    assert abs(port.with_parameter_offsets(d, {"lambda_q": -0.5, "lambda_lj": 0.4}, p_off, e_off).dispersion_coefficient() - disp) > 1e-6*abs(disp)


def test_baseline_config0_hello_sodium_chloride_on_the_reference_platform():
    """BASELINE.json configs[0]: examples/HelloSodiumChloride.cpp as shipped (6 ions, NoCutoff + GBSA-OBC, LangevinMiddle),
    compiled by oracle/Makefile from the source where it lies, on the reference's own Reference platform.  The first frame
    is deterministic: energy -297.971 kcal/mole (SURVEY.md 8c probe)."""
    import subprocess
    exe = os.path.join(ROOT, "oracle", "_ref", "tests", "HelloSodiumChloride")
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref/tests/HelloSodiumChloride not built (needs /root/reference at build time)")
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120).stdout
    assert "Using OpenMM platform Reference" in out
    frames = [l for l in out.splitlines() if l.startswith("REMARK 250")]
    assert len(frames) > 10
    assert "time=0.000 ps; energy=-297.971 kcal/mole" in frames[0]


def _wrapped_chains(seed=3):
    """Eight 4-atom chains (3 bonds, 2 angles, 1 torsion each) in a triclinic cell, every ATOM wrapped into the cell on
    its own, so that bonded terms straddle the faces (the situation of TestPeriodicTorsionForce.h:110-151 testPeriodic)."""
    rng = np.random.default_rng(seed)
    box = np.array([[2.4, 0, 0], [0.5, 2.2, 0], [-0.4, 0.6, 2.0]])
    nmol = 8
    n = 4*nmol
    pos = np.zeros((n, 3))
    for m in range(nmol):
        p = rng.uniform(-0.2, 0.2, 3) + box.sum(0)*rng.uniform(0, 1) * np.array([1, 0, 0]) + rng.uniform(0, 1, 3) @ box
        for a in range(4):
            pos[4*m+a] = p
            p = p + 0.15*rng.normal(size=3)/np.sqrt(3) + np.array([0.1, 0.05, -0.08])
    # wrap atom by atom: c, then b, then a (the order of the reduced cell)
    for a in range(n):
        for axis in (2, 1, 0):
            pos[a] -= np.floor(pos[a, axis]/box[axis, axis])*box[axis]
    mol = np.arange(n)//4
    q = np.tile([0.3, -0.3, 0.2, -0.2], nmol)
    d = systems.SystemDesc(masses=np.full(n, 12.0), charges=q, sigmas=np.full(n, 0.3), epsilons=np.full(n, 0.4), positions=pos, box=box,
                           method=systems.NB_PME, cutoff=0.9)
    first = 4*np.arange(nmol)
    d.bond_i = np.concatenate([first, first+1, first+2]).astype(np.int32)
    d.bond_j = d.bond_i + 1
    d.bond_r0 = np.full(len(d.bond_i), 0.15)
    d.bond_k = np.full(len(d.bond_i), 2.0e5)
    d.angle_i = np.concatenate([first, first+1]).astype(np.int32)
    d.angle_j, d.angle_k = d.angle_i + 1, d.angle_i + 2
    d.angle_t0 = np.full(len(d.angle_i), 1.9)
    d.angle_kk = np.full(len(d.angle_i), 400.0)
    d.tor_i = first.astype(np.int32)
    d.tor_j, d.tor_k, d.tor_l = d.tor_i + 1, d.tor_i + 2, d.tor_i + 3
    d.tor_n = np.tile([1, 2, 3, 2], 2).astype(np.int32)
    d.tor_phase = np.tile([0.0, np.pi, 0.4, 1.1], 2)
    d.tor_kk = np.full(nmol, 8.0)
    ei, ej = np.nonzero((mol[:, None] == mol[None, :]) & (np.arange(n)[:, None] < np.arange(n)[None, :]))
    d.exc_i, d.exc_j = ei.astype(np.int32), ej.astype(np.int32)
    d.exc_qq, d.exc_sigma, d.exc_eps = np.zeros(len(ei)), np.ones(len(ei)), np.zeros(len(ei))
    return d.rounded()


def test_port_periodic_bonded_terms_match_live_reference():
    """Force::usesPeriodicBoundaryConditions on HarmonicBondForce / HarmonicAngleForce / PeriodicTorsionForce: the minimum
    image on every displacement (ReferenceHarmonicBondIxn.cpp:86-89, ReferenceAngleBondIxn.cpp:121-128,
    ReferenceProperDihedralBond.cpp:91-100), in a triclinic cell, with atoms of one molecule on different sides of a face."""
    ref = _ref()
    d = _wrapped_chains()
    pme = d.pme_parameters()
    # the molecules really are split: some bonded neighbours are more than half a cell apart before the minimum image
    raw = np.linalg.norm(d.positions[d.bond_i] - d.positions[d.bond_j], axis=1)
    assert (raw > 1.0).sum() >= 3
    f, e, parts = port.forces_energy(d, pme=pme, bonded_periodic=True)
    fr, er = ref["port_bonded_periodic:f"], float(ref["port_bonded_periodic:e"])
    assert relative_force_error(f, fr) < 1e-8
    assert abs(e - er) < 1e-8*max(1.0, abs(er))
    # and the flag matters: without it both sides agree with each other on a very different answer
    f0, e0, _ = port.forces_energy(d, pme=pme)
    fr0, er0 = ref["port_bonded_nonperiodic:f"], float(ref["port_bonded_nonperiodic:e"])
    assert relative_force_error(f0, fr0) < 1e-8 and abs(e0 - er0) < 1e-8*abs(er0)
    assert e0 > 10*e
