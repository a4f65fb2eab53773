"""CPU companion of tests/test_gpu_energy.py: the ladders of tests/energy_harness.py are what they claim to be, they move
the energy far enough that the GPU comparisons cannot pass vacuously, and -- where oracle/_ref holds the reference
itself -- the restatement's energy differences along them agree with the live Reference platform's to 1e-3 kT."""
import numpy as np
import pytest
import energy_harness as EH
from openmm_b200 import systems

KT = EH.KT
ONE_4PI_EPS0 = 138.93545764438198
BAROSTAT_NAMES = ("dhfr", "water24k", "ions_triclinic", "lj_switch_dispersion")


def test_kt_is_300_kelvin():
    assert KT == pytest.approx(2.494338785, abs=1e-9)


@pytest.mark.parametrize("name", BAROSTAT_NAMES)
def test_barostat_ladder_volumes_positions_and_molecules(name):
    """Each rung changes the volume by its step (the fp32 rounding of the box moves the ratio by < 1e-6); positions and box
    are fp32-representable; every molecule moves as a whole (its internal displacements stay, to fp32 rounding)."""
    d = EH.load(name)
    mols = [m for m in d.molecules() if len(m) > 1]
    v0 = EH.volume(d.box)
    for rung in EH.RUNGS:
        dn, s = EH.scaled(d, rung)
        want = np.prod(EH.ANISO) - 1.0 if rung == "aniso" else float(rung)
        assert abs(EH.volume(dn.box)/v0 - 1.0 - want) < 1e-6, rung
        assert np.array_equal(dn.positions, EH.fp32(dn.positions)) and np.array_equal(dn.box, EH.fp32(dn.box))
        assert dn.pme_parameters() == d.pme_parameters()                        # the grid of the context stays
        for m in mols:
            r0 = d.positions[m] - d.positions[m[0]]
            r1 = dn.positions[m] - dn.positions[m[0]]
            assert np.abs(r1 - r0).max() < 2e-6, (rung, m)
        # molecule centres scale with the box (wrapped into the first cell first)
        c0 = np.array([d.positions[m].mean(0) for m in d.molecules()[:50]])
        c1 = np.array([dn.positions[m].mean(0) for m in d.molecules()[:50]])
        frac0 = np.linalg.solve(d.box.T, c0.T).T
        frac1 = np.linalg.solve(dn.box.T, c1.T).T
        assert np.abs((frac1 - np.floor(frac1)) - (frac0 - np.floor(frac0))).max() < 1e-5


def test_aniso_rung_scales_box_columns():
    """MonteCarloAnisotropicBarostat scales the x, y and z components of every box vector by its own factor."""
    box = np.array([[3.0, 0, 0], [1.0, 2.5, 0], [-0.5, 0.7, 2.0]])
    out = EH.scale_box(box, EH.ANISO)
    assert np.allclose(out[:, 0], box[:, 0]*EH.ANISO[0]) and np.allclose(out[:, 1], box[:, 1]*EH.ANISO[1])
    assert np.allclose(out[:, 2], box[:, 2]*EH.ANISO[2])
    assert len(set(EH.ANISO)) == 3


def _total(p):
    return sum(p.values())


@pytest.mark.parametrize("name", BAROSTAT_NAMES)
def test_one_percent_rungs_move_the_energy_by_more_than_kt(name):
    d = EH.pinned_pme(EH.load(name))
    e0 = _total(EH.oracle_parts(d))
    for rung in ("+0.01", "-0.01"):
        dn, _ = EH.scaled(d, rung)
        de = _total(EH.oracle_parts(dn)) - e0
        print("%s %s: dE %.3f kJ/mol" % (name, rung, de))
        assert abs(de) > KT, (rung, de)


@pytest.mark.parametrize("system_name", ["dhfr", "ions_triclinic"])
def test_lambda_one_moves_the_energy_by_more_than_kt(system_name):
    for change in EH.lambda_changes(system_name):
        d0, disp = EH.at_lambda(system_name, change, 0.0)
        d1, _ = EH.at_lambda(system_name, change, 1.0)
        de = _total(EH.oracle_parts(d1, dispersion_coefficient=disp)) - _total(EH.oracle_parts(d0, dispersion_coefficient=disp))
        print("%s %s: dE %.3f kJ/mol" % (system_name, change, de))
        assert abs(de) > KT, (change, de)


def test_lambda_ladder_interpolates_the_offsets():
    d0, _ = EH.at_lambda("ions_triclinic", "charge", 0.0)
    dh, _ = EH.at_lambda("ions_triclinic", "charge", 0.5)
    d1, _ = EH.at_lambda("ions_triclinic", "charge", 1.0)
    assert not np.array_equal(d0.charges, d1.charges)
    assert np.allclose(dh.charges, 0.5*(d0.charges + d1.charges), atol=1e-15)


def test_kernel_positions_reads_posq_of_a_checkpoint_blob():
    """The reader against a blob laid out as b200md_checkpoint_save writes it (tests/test_gpu_host_state.py::_expected_blob)."""
    from test_gpu_host_state import _expected_blob
    from openmm_b200 import systems
    d = systems.water_box(3, cutoff=0.5).rounded()
    x = d.positions + 0.123456789
    for precision in ("single", "mixed"):
        blob = _expected_blob(d, precision, x, np.zeros_like(x), d.box, 0.0, 0)

        class Fake:
            natoms = d.natoms

            def stats(self):
                return {"padded_atoms": (d.natoms + 31)//32*32}

            def checkpoint(self):
                return blob
        assert np.array_equal(EH.kernel_positions(Fake()), EH.fp32(x))


# ---- the yardstick at the energy-difference level, against the live Reference platform ----
@pytest.fixture(scope="module")
def omm():
    from oracle import omm
    if not omm.available():
        pytest.skip("oracle/_ref has no build of the reference (needs its sources at build time)")
    return omm


def _reference_energy(omm, d, pme):
    sim = omm.Simulation(d, "Reference", pme=pme)
    try:
        return sim.forces_energy()[1]
    finally:
        sim.close()


YARDSTICK = [(n, r) for n in ("water24k", "ions_triclinic", "lj_switch_dispersion") for r in EH.RUNGS] + [("dhfr", "-0.01"), ("dhfr", "aniso")]
@pytest.mark.parametrize("name,rung", YARDSTICK)
def test_oracle_energy_differences_match_live_reference(omm, name, rung):
    """dE of a barostat move, restatement against the Reference platform with the same PME alpha and grid: within 1e-3 kT."""
    d = EH.pinned_pme(EH.load(name))
    pme = d.pme_parameters() if d.method == systems.NB_PME else None
    dn, _ = EH.scaled(d, rung)
    de_orc = _total(EH.oracle_parts(dn)) - _total(EH.oracle_parts(d))
    de_ref = _reference_energy(omm, dn, pme) - _reference_energy(omm, d, pme)
    print("%s %s: dE oracle %.6f, Reference %.6f kJ/mol, difference %.2e kT" % (name, rung, de_orc, de_ref, (de_orc - de_ref)/KT))
    if (name, rung) in EH.REFERENCE_LIST_MISSES:
        assert abs(de_orc - de_ref) > 1e-3*KT         # still wrong there: once it is not, the case joins the others
    else:
        assert abs(de_orc - de_ref) < 1e-3*KT


def _all_image_direct(d, alpha):
    """PME direct space (Coulomb erfc + LJ) of an ion box without exceptions: every pair, every one of the 27 images of
    the cell within the cutoff (the cutoff is under half of every cell width: at most one image counts)"""
    from scipy.special import erfc
    x, q, s, e, rc = d.positions, d.charges, d.sigmas, d.epsilons, d.cutoff
    iu = np.triu_indices(d.natoms, 1)
    dd = (x[None] - x[:, None])[iu]
    qq, sig, eps = (q[:, None]*q[None])[iu], (0.5*(s[:, None] + s[None]))[iu], np.sqrt(e[:, None]*e[None])[iu]
    total, hits = 0.0, np.zeros(len(dd), int)
    for k in np.stack(np.meshgrid(*[np.arange(-1, 2)]*3, indexing="ij"), -1).reshape(-1, 3):
        r = np.linalg.norm(dd + k @ d.box, axis=1)
        m = r < rc
        hits += m
        sr6 = (sig[m]/r[m])**6
        total += np.sum(ONE_4PI_EPS0*qq[m]*erfc(alpha*r[m])/r[m] + 4*eps[m]*(sr6*sr6 - sr6))
    assert hits.max() <= 1
    return total


@pytest.mark.parametrize("rung", (None,) + EH.RUNGS)
def test_oracle_direct_energy_matches_an_all_image_sum(rung):
    from oracle import port
    d = EH.pinned_pme(EH.load("ions_triclinic"))
    assert len(d.exc_i) == 0 and not d.use_switch
    dn = d if rung is None else EH.scaled(d, rung)[0]
    direct = port.forces_energy(dn)[2]["direct"]
    assert abs(direct - _all_image_direct(dn, d.pme_parameters()[0])) < 1e-9*abs(direct)
