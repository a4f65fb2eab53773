"""The neighbour-list checker (tests/list_check.py) without a GPU: it accepts a valid list built here in numpy and reports
each single mutation of it as a failure of the invariant it breaks.  This is the evidence that the GPU test of the engine's
list (test_gpu_list_validity.py) fails on a wrong list.  Its exact pair enumeration is itself checked against a dense
all-pairs, 27-image one."""
import copy
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import list_check as LC  # noqa: E402
from openmm_b200 import systems  # noqa: E402


def water(nw=60):
    """the first nw waters of a 4^3 water lattice (PME, rc 0.9 nm) in a 2.1 nm box: 180 atoms, so the last 32-atom block
    holds 20"""
    d = systems.water_box(4, cutoff=0.9)
    keep = np.arange(3*nw)
    m = (d.exc_i < 3*nw) & (d.exc_j < 3*nw)
    e = copy.copy(d)
    for k in ("masses", "charges", "sigmas", "epsilons", "positions"):
        setattr(e, k, np.asarray(getattr(d, k))[keep])
    for k in ("exc_i", "exc_j", "exc_qq", "exc_sigma", "exc_eps"):
        setattr(e, k, np.asarray(getattr(d, k))[m])
    e.box = np.diag([2.1, 2.1, 2.1])          # the padded cutoff stays below half the box
    return e.rounded()


def valid_list(d, seed=3):
    """(sorig, tile_i, tile_j, tile_mask) of an all-pairs list: a shuffled sorted order, per i-block its diagonal tile and
    one tile per j-block above it, the masks from the exclusions (the all-ones mask where a full tile needs none)"""
    n = d.natoms
    nb = (n + 31)//32
    sorig = np.full(32*nb, -1, np.int32)
    sorig[:n] = np.random.default_rng(seed).permutation(n)
    slot = np.empty(n, np.int64)
    slot[sorig[:n]] = np.arange(n)
    excl = {(min(a, b), max(a, b)) for a, b in zip(slot[d.exc_i], slot[d.exc_j])}
    ti, tj, tm = [], [], []
    for ib in range(nb):
        for jb in range(ib, nb):
            cnt = min(32, n - 32*jb)
            j = np.full(32, -1, np.int32)
            j[:cnt] = 32*jb + np.arange(cnt)
            m = np.zeros(32, np.uint32)
            for l in range(32):
                si = 32*ib + l
                if si >= n:
                    continue
                for k in range(cnt):
                    if j[k] > si and (si, j[k]) not in excl:
                        m[l] |= np.uint32(1 << k)
            ti.append(ib)
            tj.append(j)
            tm.append(m)
    return sorig, np.array(ti, np.int32), np.array(tj), np.array(tm, np.uint32)


@pytest.fixture(scope="module")
def case():
    d = water()
    return d, valid_list(d)


def _tile(lst, ib, jb):
    """index of the tile of i-block ib that holds j-block jb"""
    _, ti, tj, _ = lst
    return int(np.nonzero((ti == ib) & (tj[:, 0] >> 5 == jb))[0][0])


def _copy(lst):
    return tuple(a.copy() for a in lst)


def _pair_in(d, lst, need_r, lo, hi):
    """a non-excluded pair with lo < r < hi, as (tile, i lane, j lane)"""
    sorig, ti, tj, tm = lst
    i, j, r = LC.pairs_within(d, d.positions, hi)
    excl = {(min(a, b), max(a, b)) for a, b in zip(d.exc_i, d.exc_j)}
    for a, b, rr in zip(i, j, r):
        if rr > lo and (min(a, b), max(a, b)) not in excl:
            sa, sb = sorted((int(np.nonzero(sorig == a)[0][0]), int(np.nonzero(sorig == b)[0][0])))
            t = _tile(lst, sa >> 5, sb >> 5)
            return t, sa & 31, int(np.nonzero(tj[t] == sb)[0][0])
    raise AssertionError("no pair in (%g, %g)" % (lo, hi))


def test_the_valid_list_passes(case):
    d, lst = case
    rep = LC.check_list(d, d.positions, *lst, need_r=0.99, gb_cutoff=0.9, count_r=0.9)
    n = d.natoms
    i, j, r = LC.pairs_within(d, d.positions, 0.99)
    assert rep["masked"] == n*(n - 1)//2 - len(d.exc_i)
    assert rep["gb_pairs"] == n*(n - 1)//2
    assert rep["required"] > 1000 and rep["gb_required"] == np.count_nonzero(r < 0.9)
    lo, hi = rep["count_bounds"]
    assert lo <= hi and hi - lo <= 2


def test_the_valid_list_passes_all_pairs():
    d = systems.cluster(70)
    lst = valid_list(d)
    rep = LC.check_list(d, d.positions, *lst, need_r=np.inf, gb_cutoff=np.inf)
    assert rep["required"] == 70*69//2 - 3 and rep["gb_required"] == 70*69//2


def _mutate(name, d, lst):
    """(mutated list, need_r, gb_cutoff) for a named single mutation of the valid list"""
    sorig, ti, tj, tm = lst = _copy(lst)
    need_r, gb = 0.99, None
    if name == "pair-removed":
        t, l, k = _pair_in(d, lst, need_r, 0.5, 0.6)
        tm[t, l] &= ~np.uint32(1 << k)
    elif name == "duplicated-j-masked":
        # slot 70 (block 2) also put at the head of i-block 0's tile of the partial block 5, masked there: only GB counts it
        t = _tile(lst, 0, 5)
        tj[t, 1:] = tj[t, :-1]
        tj[t, 0] = 70
        tm[t] = tm[t] << np.uint32(1)
        gb = 0.9
    elif name == "excluded-bit":
        a, b = sorted((int(np.nonzero(sorig == d.exc_i[7])[0][0]), int(np.nonzero(sorig == d.exc_j[7])[0][0])))
        t = _tile(lst, a >> 5, b >> 5)
        tm[t, a & 31] |= np.uint32(1 << int(np.nonzero(tj[t] == b)[0][0]))
    elif name == "diagonal-lower-bit":
        t = _tile(lst, 2, 2)
        tm[t, 9] |= np.uint32(1 << 4)
    elif name == "non-ascending":
        t = _tile(lst, 1, 3)
        tj[t, [5, 6]] = tj[t, [6, 5]]
    elif name == "padding-lane-mask":
        t = _tile(lst, 5, 5)
        tm[t, 25] = 1
    elif name == "j-block-below":
        t = _tile(lst, 3, 4)
        tj[t, 0] = 32*2 + 7
    elif name == "pair-inside-band-edge-dropped":
        # a pair 1e-6 nm inside need_r - band: need_r is placed just beyond it
        t, l, k = _pair_in(d, lst, need_r, 0.8, 0.9)
        x = np.asarray(d.positions)
        si, sj = 32*ti[t] + l, tj[t, k]
        dd = x[sorig[sj]] - x[sorig[si]]
        L = np.diag(d.box)
        r = np.linalg.norm(dd - L*np.round(dd/L))
        need_r = r + LC.BUILD_BAND + 1e-6
        tm[t, l] &= ~np.uint32(1 << k)
    elif name == "duplicated-masked-in":
        # as above, and masked in for an i lane that already sees slot 70 in the tile of block 2
        l = int(np.nonzero(tm[_tile(lst, 0, 2)] & np.uint32(1 << (70 - 64)))[0][0])
        t = _tile(lst, 0, 5)
        tj[t, 1:] = tj[t, :-1]
        tj[t, 0] = 70
        tm[t] = tm[t] << np.uint32(1)
        tm[t, l] |= np.uint32(1)
    elif name == "self-bit":
        t = _tile(lst, 1, 1)
        tm[t, 3] |= np.uint32(1 << 3)
    elif name == "all-ones-partial":
        t = _tile(lst, 0, 5)
        tm[t] = 0xffffffff
    elif name == "empty-lane-bit":
        t = _tile(lst, 0, 5)
        tm[t, 0] |= np.uint32(1 << 25)
    elif name == "sorted-duplicate":
        sorig[10] = sorig[11]
    elif name == "two-diagonals":
        t = _tile(lst, 4, 4)
        lst = (sorig, np.append(ti, ti[t]), np.vstack([tj, tj[t]]), np.vstack([tm, np.zeros(32, np.uint32)]))
        return lst, need_r, gb
    return (sorig, ti, tj, tm), need_r, gb


MUTATIONS = {
    "pair-removed": "kernel-missing",
    "duplicated-j-masked": "gb-duplicate",
    "excluded-bit": "mask-excluded",
    "diagonal-lower-bit": "mask-diagonal",
    "non-ascending": "tile-j-ascending",
    "padding-lane-mask": "mask-padding-lane",
    "j-block-below": "tile-j-block",
    "pair-inside-band-edge-dropped": "kernel-missing",
    "duplicated-masked-in": "kernel-duplicate",
    "self-bit": "mask-self",
    "all-ones-partial": "mask-all-ones",
    "empty-lane-bit": "mask-empty-slot",
    "sorted-duplicate": "sorted-order",
    "two-diagonals": "tile-diagonal",
}


@pytest.mark.parametrize("name", sorted(MUTATIONS))
def test_a_mutation_is_caught_as_its_invariant(case, name):
    d, lst = case
    bad, need_r, gb = _mutate(name, d, lst)
    with pytest.raises(LC.ListError) as e:
        LC.check_list(d, d.positions, *bad, need_r=need_r, gb_cutoff=gb)
    print(e.value)
    assert e.value.invariant == MUTATIONS[name], str(e.value)


def test_a_masked_duplicate_is_invisible_to_the_tile_kernel_view(case):
    """the duplicated j slot, masked in its second tile, is a GB-only failure: without the GB view the list passes"""
    d, lst = case
    bad, need_r, _ = _mutate("duplicated-j-masked", d, lst)
    LC.check_list(d, d.positions, *bad, need_r=need_r)


def test_a_pair_inside_the_band_may_be_dropped(case):
    d, lst = case
    bad, need_r, _ = _mutate("pair-inside-band-edge-dropped", d, lst)
    rep = LC.check_list(d, d.positions, *bad, need_r=need_r - 2e-6)
    assert rep["band"] >= 1


def _dense_pairs(d, x, r):
    """all pairs closer than r, minimum over the 27 images of the plain difference (no reduction), for small systems"""
    x = np.asarray(x, dtype=np.float64)
    dd = x[None, :, :] - x[:, None, :]
    if LC.is_periodic(d):
        box = np.asarray(d.box, dtype=np.float64)
        dd = LC._reduce(dd, box)
        sh = np.stack(np.meshgrid([-1, 0, 1], [-1, 0, 1], [-1, 0, 1], indexing="ij"), -1).reshape(-1, 3) @ box
        dist = np.sqrt(((dd[:, :, None, :] + sh)**2).sum(-1).min(-1))
    else:
        dist = np.linalg.norm(dd, axis=-1)
    i, j = np.nonzero((dist < r) & np.triu(np.ones(dist.shape, bool), 1))
    return i, j, dist[i, j]


@pytest.mark.parametrize("kind", ["orthorhombic", "over_half_box", "triclinic", "nonperiodic", "far"])
def test_pair_enumeration_matches_a_dense_one(kind):
    if kind == "orthorhombic":
        d, r = water(), 0.99
    elif kind == "over_half_box":
        # the padded cutoff of a 2.05 nm box at rc 1 nm reaches past half the box: each pair still once, at its minimum image
        d, r = systems.random_ions(97, 2.05, cutoff=1.0), 1.1
    elif kind == "triclinic":
        d, r = systems.random_ions(300, 3.0, cutoff=1.0, triclinic=True), 1.1
    elif kind == "nonperiodic":
        d, r = systems.cluster(200, method=systems.NB_CUTOFF_NONPERIODIC), 0.9
    else:
        # molecules several box lengths outside the cell
        d, r = water(), 0.99
        d.positions = d.positions + np.repeat(np.random.default_rng(2).integers(-3, 4, (60, 3)), 3, axis=0) @ d.box
    x = np.asarray(d.positions)
    a = LC.pairs_within(d, x, r)
    b = _dense_pairs(d, x, r)
    ka, kb = a[0]*d.natoms + a[1], b[0]*d.natoms + b[1]
    oa, ob = np.argsort(ka), np.argsort(kb)
    assert np.array_equal(ka[oa], kb[ob]) and len(ka) > 100
    np.testing.assert_allclose(a[2][oa], b[2][ob], rtol=0, atol=1e-12)
