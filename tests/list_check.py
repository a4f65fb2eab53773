"""A plain reference of the neighbour-list contract: check_list() takes what Engine.get_list() returns and the positions in
double, and checks the list against an exact enumeration of the pairs (numpy / scipy, no GPU).

The invariants are those the list's consumers rely on (nonbonded.cu, gbsa.cu), not those of the builder:
  1. sorted order   sorig[:natoms] is a permutation of the atoms, sorig[natoms:] == -1 (k_fold_sorted, brick_atom, gb_tiles)
  2. tile shape     tile_i in [0, nblocks); the non-negative j slots of a tile form a strictly ascending prefix with -1
                    after it (flush_tile bisects in it); every j slot is < natoms; a tile of i-block ib holds j slots of
                    block ib (the diagonal tile) or of blocks > ib; each i-block has exactly one diagonal tile, holding
                    ib*32 + arange(count)
  3. masks          bit k of tile_mask[t, l] lets i lane l see j lane k (k_pair, k_count_pairs); a padding i lane
                    (slot >= natoms) has mask 0; no bit for an excluded pair, an empty j lane (-1) or i == j; the diagonal
                    tile keeps only j lanes above the i lane; an all-ones tile (tileMask -1) is full and not diagonal
  4. tile kernel    every (i, j) pair with its bit set appears at most once, and every non-excluded pair closer than
                    need_r appears (so exactly once)
  5. GB             (gb_cutoff given; the mask is ignored, as k_gb_born / k_gb_pairs / k_gb_chain ignore it) the pairs
                    (si, sj) with sj > si, si < natoms and sj >= 0 of all tiles hold every pair within gb_cutoff,
                    excluded pairs included, exactly once; no pair appears twice, whatever its distance

Pairs within `band` of need_r are skipped: fp32 may decide them either way.  A freshly built list holds every pair within
the padded cutoff rc*(1 + pad) (B200MD_PAD_FRACTION, default 0.1), up to the build's 1e-5 relative margin on r^2; an
aged list still holds every pair within rc (the displacement check rebuilds it after a move of half the padding).

Pairs are compared as sorted-slot keys si*npad + sj (si < sj), a chunk of i-blocks at a time, so that ApoA1-sized lists
stay at about 2 GB of peak memory."""
import numpy as np

from openmm_b200 import systems

PERIODIC_METHODS = (systems.NB_CUTOFF_PERIODIC, systems.NB_PME)
BUILD_BAND = 2e-5           # nm, around need_r = rc*(1 + pad) at a build
AGED_BAND = 1e-6            # nm, around need_r = rc on an aged list (tests/test_gpu_oracle_edges.py _pair_count_bounds)
COUNT_BAND = 1e-6           # nm, around count_r for the pairs_in_cutoff bounds (at least 2^-22 of the largest coordinate:
                            # k_count_pairs takes the distance of wrapped fp32 positions, ApoA1's reach 10.9 nm)
LANES = np.arange(32)


class ListError(AssertionError):
    """A broken list invariant; `invariant` names it (the test of the checker asserts on it)."""

    def __init__(self, invariant, message):
        super().__init__("%s: %s" % (invariant, message))
        self.invariant = invariant


def is_periodic(desc):
    return desc.box is not None and desc.method in PERIODIC_METHODS


def _reduce(d, box):
    """Wrap displacements d [..., 3] into the reduced cell (c, b, a order, as ReferenceForce::getDeltaRPeriodic)."""
    a, b, c = box
    d = d - np.floor(d[..., 2:3]/c[2] + 0.5)*c
    d = d - np.floor(d[..., 1:2]/b[1] + 0.5)*b
    return d - np.floor(d[..., 0:1]/a[0] + 0.5)*a


def pairs_within(desc, x, r, chunk=256):
    """(i, j, dist) of every atom pair i < j (user order) closer than r, minimum image in periodic systems: a periodic
    k-d tree in orthorhombic boxes, the least of the 27 images of the reduced displacement in triclinic ones, a plain
    k-d tree without periodicity.  r = inf enumerates all pairs."""
    from scipy.spatial import cKDTree
    x = np.asarray(x, dtype=np.float64)
    n = len(x)
    if not np.isfinite(r):
        i, j = np.triu_indices(n, 1)
        return i, j, np.linalg.norm(x[j] - x[i], axis=1)
    if not is_periodic(desc):
        p = cKDTree(x).query_pairs(r, output_type="ndarray")
        i, j = p.min(axis=1), p.max(axis=1)
        return i, j, np.linalg.norm(x[j] - x[i], axis=1)
    box = np.asarray(desc.box, dtype=np.float64)
    if not np.count_nonzero(box - np.diag(np.diag(box))):
        L = np.diag(box)
        y = np.mod(x, L)
        y[y >= L] = 0.0
        p = cKDTree(y, boxsize=L).query_pairs(r, output_type="ndarray")
        i, j = p.min(axis=1), p.max(axis=1)
        d = x[j] - x[i]
        return i, j, np.linalg.norm(d - L*np.round(d/L), axis=1)
    shifts = np.stack(np.meshgrid([-1, 0, 1], [-1, 0, 1], [-1, 0, 1], indexing="ij"), -1).reshape(-1, 3) @ box
    out = []
    for i0 in range(0, n, chunk):
        rows = np.arange(i0, min(n, i0 + chunk))
        d = _reduce(x[None, :, :] - x[rows, None, :], box)
        dist = np.sqrt((((d[:, :, None, :] + shifts[None, None]))**2).sum(-1).min(-1))
        ii, jj = np.nonzero((dist < r) & (np.arange(n)[None, :] > rows[:, None]))
        out.append((rows[ii], jj, dist[ii, jj]))
    return tuple(np.concatenate(a) for a in zip(*out))


def _keys(si, sj, npad):
    lo, hi = np.minimum(si, sj), np.maximum(si, sj)
    return lo.astype(np.int64)*npad + hi


def _first(mask):
    """index tuple of the first True of an array"""
    return tuple(int(v) for v in np.argwhere(mask)[0])


def check_list(desc, x, sorig, tile_i, tile_j, tile_mask, need_r, gb_cutoff=None, band=BUILD_BAND, count_r=None,
               chunk_tiles=1 << 15):
    """Check a neighbour list (Engine.get_list()) of desc at positions x [natoms, 3] against the invariants of the module
    docstring; need_r is the distance within which every non-excluded pair must be listed (rc*(1 + pad) at a build, rc on
    an aged list), inf for NoCutoff.  Raises ListError on the first broken invariant, naming the tile, lanes and atoms.
    Returns a report: tiles, masked (masked-in pairs), required (non-excluded pairs closer than need_r - band), band
    (pairs within band of need_r, skipped), and with gb_cutoff gb_pairs / gb_required; with count_r, count_bounds = the
    (lo, hi) range of masked-in pairs closer than count_r (up to the count band), which k_count_pairs reports."""
    n = desc.natoms
    sorig = np.asarray(sorig).astype(np.int64)
    ti = np.asarray(tile_i).astype(np.int64)
    tj = np.asarray(tile_j).astype(np.int64)
    tm = np.asarray(tile_mask).astype(np.uint32)
    npad = len(sorig)
    nblocks = (n + 31)//32
    T = len(ti)
    # ---- 1. sorted order
    if npad != 32*nblocks:
        raise ListError("sorted-order", "%d sorted slots for %d atoms (want %d)" % (npad, n, 32*nblocks))
    head = sorig[:n]
    if (head < 0).any() or (head >= n).any():
        s = _first((head < 0) | (head >= n))[0]
        raise ListError("sorted-order", "slot %d holds atom %d" % (s, head[s]))
    seen = np.bincount(head, minlength=n)
    if (seen != 1).any():
        a = _first(seen != 1)[0]
        raise ListError("sorted-order", "atom %d is in %d slots" % (a, seen[a]))
    if (sorig[n:] != -1).any():
        s = n + _first(sorig[n:] != -1)[0]
        raise ListError("sorted-order", "padding slot %d holds %d, not -1" % (s, sorig[s]))
    slot_of = np.empty(n, dtype=np.int64)
    slot_of[head] = np.arange(n)
    # ---- 2. tile shape
    if tj.shape != (T, 32) or tm.shape != (T, 32):
        raise ListError("tile-shape", "tile arrays of shape %s, %s for %d tiles" % (tj.shape, tm.shape, T))
    if T and ((ti < 0) | (ti >= nblocks)).any():
        t = _first((ti < 0) | (ti >= nblocks))[0]
        raise ListError("tile-i-range", "tile %d has i-block %d of %d" % (t, ti[t], nblocks))
    valid = tj >= 0
    if (tj < -1).any():
        t, k = _first(tj < -1)
        raise ListError("tile-j-prefix", "tile %d lane %d holds j slot %d" % (t, k, tj[t, k]))
    if T and (~valid[:, 0]).any():
        t = _first(~valid[:, 0])[0]
        raise ListError("tile-j-prefix", "tile %d (i-block %d) has no j slot" % (t, ti[t]))
    hole = valid[:, 1:] & ~valid[:, :-1]
    if hole.any():
        t, k = _first(hole)
        raise ListError("tile-j-prefix", "tile %d: j lane %d is -1 but lane %d holds slot %d" % (t, k, k + 1, tj[t, k + 1]))
    down = valid[:, 1:] & (tj[:, 1:] <= tj[:, :-1])
    if down.any():
        t, k = _first(down)
        raise ListError("tile-j-ascending", "tile %d: j lane %d holds slot %d after slot %d" % (t, k + 1, tj[t, k + 1], tj[t, k]))
    if (tj >= n).any():
        t, k = _first(tj >= n)
        raise ListError("tile-j-range", "tile %d lane %d holds slot %d >= %d atoms" % (t, k, tj[t, k], n))
    jb = np.where(valid, tj >> 5, nblocks)
    low = valid & (jb < ti[:, None])
    if low.any():
        t, k = _first(low)
        raise ListError("tile-j-block", "tile %d of i-block %d: j lane %d holds slot %d (atom %d) of block %d"
                        % (t, ti[t], k, tj[t, k], sorig[tj[t, k]], jb[t, k]))
    diag = (jb == ti[:, None]).any(axis=1)
    count = np.minimum(32, n - 32*ti)
    want = np.where(LANES[None, :] < count[:, None], 32*ti[:, None] + LANES[None, :], -1)
    wrong = diag & (tj != want).any(axis=1)
    if wrong.any():
        t = _first(wrong)[0]
        k = _first(tj[t] != want[t])[0]
        raise ListError("tile-diagonal", "diagonal tile %d of i-block %d: lane %d holds %d, not %d" % (t, ti[t], k, tj[t, k], want[t, k]))
    ndiag = np.bincount(ti[diag], minlength=nblocks)
    if (ndiag != 1).any():
        b = _first(ndiag != 1)[0]
        raise ListError("tile-diagonal", "i-block %d has %d diagonal tiles" % (b, ndiag[b]))
    # ---- the pairs the list must hold
    r_gb = None if gb_cutoff is None else min(gb_cutoff, need_r - band)
    r_max = need_r + band
    count_band = max(COUNT_BAND, 2.0**-22*float(np.abs(x).max() if desc.box is None else np.abs(desc.box).max()))
    if count_r is not None:
        r_max = max(r_max, count_r + count_band)
    i, j, dist = pairs_within(desc, x, r_max)
    keys = _keys(slot_of[i], slot_of[j], npad)
    excl = np.zeros(0, dtype=np.int64)
    if len(desc.exc_i):
        excl = np.unique(_keys(slot_of[np.asarray(desc.exc_i)], slot_of[np.asarray(desc.exc_j)], npad))
    excluded = np.isin(keys, excl)
    report = {"tiles": T, "masked": 0, "band": int(np.count_nonzero(np.abs(dist - need_r) <= band))}
    need = np.sort(keys[~excluded & (dist < need_r - band)])
    report["required"] = len(need)
    if count_r is not None:
        report["count_bounds"] = (int(np.count_nonzero(~excluded & (dist < count_r - count_band))),
                                  int(np.count_nonzero(~excluded & (dist < count_r + count_band))))
    need_gb = None
    if r_gb is not None:
        need_gb = np.sort(keys[dist < r_gb])
        report["gb_required"], report["gb_pairs"] = len(need_gb), 0
    # ---- 3.-5., a chunk of i-blocks at a time (every listed pair lies in the tiles of its lower slot's block)
    order = np.argsort(ti, kind="stable")
    tcount = np.bincount(ti, minlength=nblocks)
    tend = np.cumsum(tcount)
    b0 = 0
    while b0 < nblocks:
        b1 = max(b0 + 1, int(np.searchsorted(tend, (tend[b0 - 1] if b0 else 0) + chunk_tiles, side="right")))
        b1 = min(b1, nblocks)
        sel = order[(tend[b0 - 1] if b0 else 0):tend[b1 - 1]]
        klo, khi = 32*b0*npad, 32*b1*npad
        report["masked"] += _check_chunk(sel, ti[sel], tj[sel], tm[sel], valid[sel], diag[sel], n, npad, sorig, excl,
                                         need[(need >= klo) & (need < khi)], need_gb if need_gb is None else
                                         need_gb[(need_gb >= klo) & (need_gb < khi)], report)
        b0 = b1
    return report


def _pair_name(key, npad, sorig):
    si, sj = divmod(int(key), npad)
    return "slots %d, %d (atoms %d, %d)" % (si, sj, sorig[si], sorig[sj])


def _check_chunk(tid, ti, tj, tm, valid, diag, n, npad, sorig, excl, need, need_gb, report):
    si = 32*ti[:, None] + LANES[None, :]                                   # [C, 32] i slot of each lane
    pad_lane = (si >= n) & (tm != 0)
    if pad_lane.any():
        c, l = _first(pad_lane)
        raise ListError("mask-padding-lane", "tile %d i lane %d (slot %d >= %d atoms) has mask %#010x" % (tid[c], l, si[c, l], n, tm[c, l]))
    ones = (tm == 0xffffffff).all(axis=1) & (diag | ~valid.all(axis=1))
    if ones.any():
        c = _first(ones)[0]
        raise ListError("mask-all-ones", "tile %d (i-block %d, %d j slots%s) has the all-ones mask"
                        % (tid[c], ti[c], valid[c].sum(), ", diagonal" if diag[c] else ""))
    bits = ((tm[:, :, None] >> LANES[None, None, :].astype(np.uint32)) & 1).astype(bool)    # [C, i lane, j lane]
    empty = bits & ~valid[:, None, :]
    if empty.any():
        c, l, k = _first(empty)
        raise ListError("mask-empty-slot", "tile %d: i lane %d (atom %d) has the bit of empty j lane %d" % (tid[c], l, sorig[si[c, l]], k))
    sj = tj[:, None, :]
    same = bits & (sj == si[:, :, None])
    if same.any():
        c, l, k = _first(same)
        raise ListError("mask-self", "tile %d: i lane %d and j lane %d are both slot %d (atom %d)" % (tid[c], l, k, si[c, l], sorig[si[c, l]]))
    lower = bits & (sj < si[:, :, None])
    if lower.any():
        c, l, k = _first(lower)
        raise ListError("mask-diagonal", "tile %d (i-block %d): i lane %d (slot %d) sees j lane %d (slot %d) below it"
                        % (tid[c], ti[c], l, si[c, l], k, tj[c, k]))
    c, l, k = np.nonzero(bits)
    keys = si[c, l].astype(np.int64)*npad + tj[c, k]
    hit = np.isin(keys, excl)
    if hit.any():
        h = _first(hit)[0]
        raise ListError("mask-excluded", "tile %d: i lane %d, j lane %d, excluded pair %s is masked in" % (tid[c[h]], l[h], k[h], _pair_name(keys[h], npad, sorig)))
    _unique_and_complete("kernel", keys, need, tid[c], l, k, npad, sorig)
    if need_gb is not None:
        gb = valid[:, None, :] & (sj > si[:, :, None]) & (si[:, :, None] < n)
        c, l, k = np.nonzero(gb)
        gkeys = si[c, l].astype(np.int64)*npad + tj[c, k]
        _unique_and_complete("gb", gkeys, need_gb, tid[c], l, k, npad, sorig)
        report["gb_pairs"] += len(gkeys)
    return len(keys)


def _unique_and_complete(view, keys, need, tiles, ilane, jlane, npad, sorig):
    o = np.argsort(keys, kind="stable")
    ks = keys[o]
    dup = np.nonzero(ks[1:] == ks[:-1])[0]
    if len(dup):
        a, b = o[dup[0]], o[dup[0] + 1]
        raise ListError(view + "-duplicate", "pair %s in tile %d (i lane %d, j lane %d) and tile %d (i lane %d, j lane %d)"
                        % (_pair_name(ks[dup[0]], npad, sorig), tiles[a], ilane[a], jlane[a], tiles[b], ilane[b], jlane[b]))
    pos = np.searchsorted(ks, need)
    found = (pos < len(ks)) & (ks[np.minimum(pos, max(len(ks) - 1, 0))] == need) if len(ks) else np.zeros(len(need), bool)
    if not found.all():
        m = need[_first(~found)[0]]
        raise ListError(view + "-missing", "pair %s (i-block %d) is not in the list; %d such pairs"
                        % (_pair_name(m, npad, sorig), int(m)//npad//32, int(np.count_nonzero(~found))))
