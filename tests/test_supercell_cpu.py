"""The supercell builder of tests/supercell_harness.py, and the premise of tests/test_gpu_supercell.py checked with the
double-precision restatement itself: every copy of a 2 x 2 x 2 supercell feels the unit cell's forces, and every energy part
of the supercell but the dispersion correction is 8 times the unit cell's."""
import numpy as np
import pytest
import supercell_harness as SC


# the supercells tests/test_gpu_supercell.py runs, and two small ones
BUILT = [("dhfr", 2), ("dhfr", 3), ("dhfr", 4), ("apoa1", 2), ("water23", 3), ("ions_triclinic", 4), ("water_rigid", 2),
         ("water_flexible", 3)]


def test_one_copy_is_the_quantized_unit_cell():
    u = SC.quantized(SC.unit("dhfr"), 1)
    s = SC.supercell(u, 1)
    for f in ("positions", "box", "masses", "charges", "sigmas", "epsilons", "exc_i", "exc_j", "exc_qq", "con_i", "con_j", "con_d",
              "bond_i", "bond_j", "angle_k", "tor_l", "tor_n", "tor_phase"):
        assert np.array_equal(getattr(s, f), getattr(u, f)), f
    assert s.pme_parameters() == u.pme_parameters()


@pytest.mark.parametrize("name,k", BUILT)
def test_supercell_layout(name, k):
    d = SC.unit(name)
    u = SC.quantized(d, k)
    s = SC.supercell(u, k)
    n, m = u.natoms, k**3
    q = SC.quantum(d, k)
    assert q < 1e-5
    # the quantized unit cell moved at most q/2 from d, and keeps d's PME parameters
    assert np.abs(u.positions - d.positions).max() <= 0.5*q and np.abs(u.box - d.box).max() <= 0.5*q
    assert u.pme_parameters() == d.pme_parameters()
    alpha, nx, ny, nz = u.pme_parameters()
    assert s.pme_parameters() == (alpha, k*nx, k*ny, k*nz)
    assert np.array_equal(s.box, k*u.box)
    assert s.natoms == m*n
    for atoms, params in SC.TERM_FIELDS.values():
        for f in atoms + params:
            assert len(getattr(s, f)) == m*len(getattr(u, f)), f
        # every term stays inside its copy, and is the unit cell's term moved by copy * N
        for f in atoms:
            a = SC.copies(getattr(s, f), k)
            assert np.array_equal(a - (np.arange(m)*n)[:, None], np.broadcast_to(getattr(u, f), a.shape)), f
    for i, j in (("exc_i", "exc_j"), ("con_i", "con_j")):
        assert np.array_equal(getattr(s, i)//n, getattr(s, j)//n)
    x = SC.copies(s.positions, k)
    assert np.array_equal(x[0], u.positions)
    assert np.allclose(x - u.positions[None], SC.offsets(u.box, k)[:, None, :], rtol=0, atol=1e-12)
    # every coordinate, every difference of two and the box are multiples of q below 2^24 q: exact in fp32
    assert SC.fp32_exact(s.positions) and SC.fp32_exact(s.box)
    assert np.array_equal(np.round(s.positions/q)*q, s.positions) and np.array_equal(np.round(s.box/q)*q, s.box)
    span = max(np.abs(s.positions).max(), np.abs(s.box).sum(axis=0).max())
    assert 2.0*span < 2.0**24*q


@pytest.mark.parametrize("name", ["ions_triclinic", "water_rigid", "water_flexible"])
def test_molecules_are_copied(name):
    u = SC.quantized(SC.unit(name), 2)
    mols = u.molecules()
    smols = SC.supercell(u, 2).molecules()
    assert len(smols) == 8*len(mols)
    # ordered by their lowest atom: copy c's molecules are the c-th block, each the unit cell's moved by c * N
    n = u.natoms
    for c in range(8):
        assert [list(np.asarray(m) - c*n) for m in smols[c*len(mols):(c + 1)*len(mols)]] == [list(m) for m in mols]


def test_unsupported_terms_and_small_boxes_are_refused():
    import copy
    from openmm_b200 import systems
    d = copy.copy(SC.unit("water_flexible"))
    d.rb_i = np.array([0], dtype=np.int32)
    with pytest.raises(AssertionError):
        SC.supercell(d, 2)
    d = systems.water_box(5, cutoff=0.9).rounded()          # 1.55 nm: the cutoff is above half the width
    with pytest.raises(AssertionError):
        SC.supercell(d, 2)


@pytest.mark.parametrize("name", ["ions_triclinic", "water_flexible"])
def test_every_copy_feels_the_unit_cell_forces(name):
    """The restatement on the 2 x 2 x 2 supercell against the restatement on the unit cell: per copy the forces to 1e-9 of
    the largest force, and every energy part but the dispersion correction, over 8, to 1e-9 of the part (of the self
    energy for the reciprocal part)."""
    from oracle import port
    k = 2
    u = SC.quantized(SC.unit(name), k)
    s = SC.supercell(u, k)
    fu, parts_u = SC.oracle(u)
    fs, _, parts_s = port.forces_energy(s, pme=s.pme_parameters())
    scale = np.linalg.norm(fu, axis=1).max()
    err = max(np.abs(f - fu).max() for f in SC.copies(fs, k))/scale
    print("%s x%d: per-copy force difference %.1e of max |F|" % (name, k, err))
    assert err < 1e-9
    assert set(parts_s) == set(parts_u)
    for p, e in parts_u.items():
        if p == "dispersion":
            continue
        # the reciprocal sum is a small remainder of terms on the scale of the self energy (water: 0.8 against 8e4 kJ/mol)
        scale = max(1.0, abs(e), abs(parts_u["self"]) if p == "reciprocal" else 0.0)
        rel = abs(parts_s[p]/k**3 - e)/scale
        print("  %s %.6f per copy, %.1e" % (p, e, rel))
        assert rel < 1e-9, (p, parts_s[p]/k**3, e)
    # the dispersion correction is the supercell's own, and is not 8 times the unit cell's
    assert parts_s["dispersion"] == pytest.approx(SC.dispersion_energy(s), rel=1e-15)
    expected = SC.expected_groups(u, k, SC.dispersion_energy(s))
    assert expected["direct"] == pytest.approx((parts_s["direct"] + parts_s["dispersion"] + parts_s.get("exceptions14", 0.0)
                                                + parts_s.get("exclusion", 0.0))/k**3, rel=1e-9)
