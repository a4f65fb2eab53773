"""Generalized Born (GBSAOBCForce) without a GPU: the double-precision restatement of OBC II + ACE (tests/gbsa_harness.py)
against the reference's Reference platform (tests/golden/reference_gbsa.npz, written by make_golden_gbsa.py) and against a
finite difference of its own energy; the DHFR implicit-solvent fixture round-trips through SystemDesc."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gbsa_harness as H  # noqa: E402
from openmm_b200 import systems  # noqa: E402

CASES = ("dhfr_nocutoff", "dhfr_cutoff", "hello_nacl", "ion_box", "ion_box_custom", "ion_box_tri_pmp", "ion_box_tri_mpm")


@pytest.mark.parametrize("name", CASES)
def test_restatement_matches_the_reference_platform(name):
    g = np.load(H.GOLDEN)
    d = H.golden_cases()[name]
    f, e = H.obc_forces_energy(d, g[name + "_positions"])
    fr, er = g[name + "_forces"], float(g[name + "_energy"])
    assert abs(e - er) <= 1e-9*abs(er), (e, er)
    scale = np.abs(fr).max()
    assert np.abs(f - fr).max() <= 1e-9*scale, np.abs(f - fr).max()/scale


@pytest.mark.parametrize("method", [systems.NB_NOCUTOFF, systems.NB_CUTOFF_NONPERIODIC])
def test_restatement_forces_are_the_gradient_of_its_energy(method):
    """central differences on a 60-atom piece of DHFR (far from the cutoff: the energy jumps where a pair crosses it)"""
    d = H.dhfr_gbsa(method)
    sel = np.arange(60)
    for k in ("masses", "charges", "sigmas", "epsilons", "gb_charges", "gb_radii", "gb_scales"):
        setattr(d, k, np.asarray(getattr(d, k))[sel])
    d.positions = np.asarray(d.positions)[sel]
    f, _ = H.obc_forces_energy(d)
    h = 1e-6
    num = np.zeros_like(f)
    for i in range(len(sel)):
        for c in range(3):
            x = d.positions.copy()
            x[i, c] += h
            ep = H.obc_forces_energy(d, x)[1]
            x[i, c] -= 2*h
            em = H.obc_forces_energy(d, x)[1]
            num[i, c] = -(ep - em)/(2*h)
    err = np.abs(num - f).max()/np.abs(f).max()
    assert err < 1e-6, err


def test_dhfr_fixture_round_trips(tmp_path):
    d = systems.SystemDesc.load(H.FIXTURE)
    n = d.natoms
    assert n == 2489 and d.box is None
    assert len(d.gb_charges) == len(d.gb_radii) == len(d.gb_scales) == n
    np.testing.assert_array_equal(d.gb_charges, d.charges)
    assert d.method == d.gb_method == systems.NB_CUTOFF_NONPERIODIC and d.cutoff == 2.0
    assert d.rf_dielectric == 1.0
    assert (d.gb_radii > 0.009).all() and len(d.con_i) > 0
    p = tmp_path / "d.npz"
    d.save(str(p))
    e = systems.SystemDesc.load(str(p))
    for k in ("gb_charges", "gb_radii", "gb_scales", "positions", "charges", "con_i", "exc_i"):
        np.testing.assert_array_equal(getattr(e, k), getattr(d, k))
    for k in ("gb_method", "gb_solute_dielectric", "gb_solvent_dielectric", "gb_surface_area_energy", "rf_dielectric", "cutoff", "method"):
        assert getattr(e, k) == getattr(d, k), k
