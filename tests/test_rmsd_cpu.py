"""RMSDForce arithmetic on the CPU: the host probe of the device code (openmm_b200/csrc/rmsd.h) against the Reference
platform's RMSDForce on stored goldens (tests/golden/reference_rmsd.npz), against a central difference of its own energy, and
its Jacobi eigen solve against numpy's eigh on random and nearly degenerate symmetric 4x4 matrices."""
import numpy as np
import pytest

import rmsd_harness as H

G = H.load_golden()


@pytest.mark.parametrize("name", sorted(G))
def test_probe_matches_the_reference_platform(name):
    g = G[name]
    e, f = H.probe_full(g["positions"], g["reference"], g["particles"])
    if name == "rotated_copy":
        # RMSD 0 up to the rounding of sum|x|^2 + sum|r|^2 - 2 lambda, on either side
        assert e < 1e-6 and float(g["energy"]) < 1e-6, (e, float(g["energy"]))
        assert np.abs(f).max() < 1e-6
        return
    assert abs(e - float(g["energy"])) <= 1e-9*max(1.0, abs(float(g["energy"]))), (e, float(g["energy"]))
    assert np.abs(f - g["forces"]).max() <= 1e-9, np.abs(f - g["forces"]).max()
    if len(g["particles"]):
        rest = np.setdiff1d(np.arange(len(f)), g["particles"])
        assert (f[rest] == 0).all()


def test_offsets_do_not_change_the_rmsd():
    a, b, c = G["offset_plus50"], G["offset_minus50"], G["subset_all_listed"]
    ea, _ = H.probe_full(a["positions"], a["reference"], a["particles"])
    eb, _ = H.probe_full(b["positions"], b["reference"], b["particles"])
    ec, _ = H.probe_full(c["positions"], c["reference"], c["particles"])
    assert abs(ea - ec) < 1e-12 and abs(eb - ec) < 1e-12, (ea, eb, ec)


def test_mirror_image_is_not_superposable():
    g = G["mirror"]
    e, _ = H.probe_full(g["positions"], g["reference"], g["particles"])
    assert e > 0.5


@pytest.mark.parametrize("name", ["random_3", "random_20", "random_200", "mirror", "offset_plus50", "subset"])
def test_forces_are_minus_the_gradient(name):
    g = G[name]
    x, ref, particles = np.array(g["positions"]), g["reference"], g["particles"]
    _, f = H.probe_full(x, ref, particles)
    rng = np.random.default_rng(5)
    h = 1e-6
    for a in rng.choice(len(x), min(len(x), 6), replace=False):
        for k in range(3):
            xp, xm = x.copy(), x.copy()
            xp[a, k] += h
            xm[a, k] -= h
            d = (H.probe_full(xp, ref, particles)[0] - H.probe_full(xm, ref, particles)[0])/(2*h)
            assert abs(-d - f[a, k]) <= 1e-6*max(1.0, abs(f[a, k])), (a, k, -d, f[a, k])


def test_perfect_alignment_gives_zero_rmsd_and_zero_forces():
    """Where the mean square deviation is below 1e-20 (here exactly 0: every sum is exact) the RMSD and the forces are 0, as
    on the Reference platform, instead of the 0/0 of the gradient there"""
    x = np.array([[1.0, 0.0, 0.0], [-1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [0.0, -1.0, 0.0], [0.0, 0.0, 2.0], [0.0, 0.0, -2.0]])
    e, f = H.probe(x + 3.0, x)
    assert e == 0.0 and (f == 0).all()


def test_identical_copies_give_finite_forces():
    """An identical copy leaves a mean square deviation of rounding size, of either sign: never a NaN"""
    rng = np.random.default_rng(3)
    for n in (3, 20, 200, 2000):
        for _ in range(5):
            x = rng.uniform(-3.0, 3.0, (n, 3))
            e, f = H.probe(x, x)
            assert 0.0 <= e < 1e-6 and np.isfinite(f).all() and np.abs(f).max() < 1e-6, (n, e)


def _check_eigen(a):
    lam, q, sweeps = H.eigen_probe(a)
    w, v = np.linalg.eigh(a)
    scale = max(1.0, np.abs(w).max())
    assert abs(lam - w[-1]) <= 1e-12*scale, (lam, w)
    assert abs(np.linalg.norm(q) - 1.0) < 1e-12
    # an eigenvector of the largest eigenvalue: A q = lambda q (the eigenvector itself is not unique when it is degenerate)
    assert np.abs(a @ q - lam*q).max() <= 1e-11*scale, (a @ q - lam*q)
    assert sweeps < 64
    return sweeps


def test_jacobi_matches_eigh_on_random_symmetric_matrices():
    rng = np.random.default_rng(7)
    for _ in range(500):
        m = rng.normal(0.0, rng.choice([1e-3, 1.0, 1e3]), (4, 4))
        _check_eigen(m + m.T)


def test_jacobi_matches_eigh_on_nearly_degenerate_matrices():
    rng = np.random.default_rng(8)
    for gap in (0.0, 1e-14, 1e-10, 1e-6):
        for _ in range(100):
            qm, _ = np.linalg.qr(rng.normal(size=(4, 4)))
            w = np.array([rng.uniform(-2, 2), 1.0, 1.0 - gap, rng.uniform(-3, 0.5)])
            _check_eigen(qm @ np.diag(w) @ qm.T)
    _check_eigen(np.eye(4))
    _check_eigen(np.zeros((4, 4)))
    _check_eigen(np.diag([1.0, 3.0, 3.0, 2.0]))
