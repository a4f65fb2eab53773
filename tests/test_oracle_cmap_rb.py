"""CPU checks behind the GPU tests of RBTorsionForce and CMAPTorsionForce (tests/test_gpu_cmap_rb.py): the exact conversion of
DHFR's periodic torsions to Ryckaert-Bellemans form, the backbone CMAP terms found in DHFR, and the CHARMM36 map fixture."""
import os
import numpy as np
import pytest
from conftest import ROOT, GOLDEN
from openmm_b200 import systems


def _dhfr():
    return systems.SystemDesc.load(os.path.join(ROOT, "data", "dhfr.npz"))


def test_rb_conversion_is_exact_on_the_torsion_energy_surface():
    d = _dhfr()
    r = systems.periodic_to_rb(d)
    assert len(r.rb_i) == len(d.tor_i) == 7310 and len(r.tor_i) == 0
    phi = np.random.default_rng(1).uniform(-np.pi, np.pi, len(d.tor_n))
    e_periodic = d.tor_kk*(1 + np.cos(d.tor_n*phi - d.tor_phase))
    cpsi = np.cos(phi - np.pi)
    e_rb = sum(r.rb_c[:, m]*cpsi**m for m in range(6))
    assert np.abs(e_rb - e_periodic).max() < 1e-10


def test_rb_conversion_refuses_what_it_cannot_convert():
    d = _dhfr()
    d.tor_phase = d.tor_phase.copy()
    d.tor_phase[0] = 0.5
    with pytest.raises(ValueError):
        systems.periodic_to_rb(d)


def test_dhfr_backbone_cmap_pairs_are_torsions_of_the_system():
    d = _dhfr()
    a = systems.backbone_cmap_atoms(d)
    assert a.shape == (157, 8)
    tors = set(zip(d.tor_i.tolist(), d.tor_j.tolist(), d.tor_k.tolist(), d.tor_l.tolist()))
    for row in a.tolist():
        for t in (tuple(row[:4]), tuple(row[4:])):
            assert t in tors or t[::-1] in tors
        assert row[1:4] == row[4:7]                    # phi and psi share N-CA-C


def test_fixture_coefficients_reproduce_the_map_energies_at_the_grid_points():
    z = np.load(os.path.join(GOLDEN, "charmm36_cmap.npz"))
    size, energy, coeff = z["size"], z["energy"], z["coeff"]
    assert len(size) == 8 and (size == 24).all() and coeff.shape == (8*24*24, 16)
    first = 0
    for n in size:
        e = energy[first:first + n*n]
        c = coeff[first:first + n*n]
        # patch s + n*t spans [s, s+1] x [t, t+1] grid cells; c[i*4+j] multiplies da^i db^j
        for s in range(n):
            for t in range(n):
                p = c[s + n*t]
                assert abs(p[0] - e[s + n*t]) < 1e-9*max(1.0, abs(e[s + n*t]))
                corner_a = p[0] + p[4] + p[8] + p[12]                          # da = 1, db = 0
                assert abs(corner_a - e[(s+1) % n + n*t]) < 1e-8*max(1.0, abs(e[(s+1) % n + n*t]))
                corner_b = p[0] + p[1] + p[2] + p[3]                           # da = 0, db = 1
                assert abs(corner_b - e[s + n*((t+1) % n)]) < 1e-8*max(1.0, abs(e[s + n*((t+1) % n)]))
        first += n*n


@pytest.fixture(scope="module")
def harness():
    """Reference-side RB and CMAP forces (tests/cmap_rb_harness.py)"""
    import cmap_rb_harness
    if not cmap_rb_harness.available():
        pytest.skip("oracle/_ref is not built")
    return cmap_rb_harness


def test_fixture_coefficients_are_the_reference_fitter_s(harness):
    z = np.load(os.path.join(GOLDEN, "charmm36_cmap.npz"))
    first = 0
    for n in z["size"]:
        c = harness.coefficients(int(n), z["energy"][first:first + n*n])
        assert np.array_equal(c, z["coeff"][first:first + n*n])
        first += n*n


def test_reference_platform_periodic_and_rb_dhfr_give_the_same_forces(harness):
    d = _dhfr().rounded()
    r = systems.periodic_to_rb(d)
    pme = d.pme_parameters()
    fp, ep = harness.Simulation(d, "Reference", pme=pme).forces_energy()
    fr, er = harness.Simulation(r, "Reference", pme=pme).forces_energy()
    assert np.abs(fr - fp).max() <= 1e-9*np.abs(fp).max()
    assert abs(er - ep) <= 1e-9*abs(ep)
