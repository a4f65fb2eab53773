"""GPU tests that the neighbour-list build emits the list it always emitted.  The tile kernel's fp32 sums depend on which
j atoms share a tile and in which lane order, so the list is part of what the forces are: a faster build must produce the
same sorted order and the same tiles, tile for tile.  Only where a tile lands in the slot pools (and where its mask lands
in the mask pool) may change, since the tile kernel adds its tiles with order-free int64 atomics.

The list is compared in a canonical form: the sorted order (`sorig`), then every tile's i-block, 32 j-slots and 32 mask
words, with the tiles sorted by (i-block, j-slots).  tests/golden/list_hashes.json holds the SHA-256 of that form and the
tile and masked-tile counts per case, from the build before the list kernels were reorganised
(tests/golden/make_golden_list.py)."""
import hashlib
import json
import os
import numpy as np
import pytest
from conftest import ROOT, GOLDEN

pytestmark = pytest.mark.gpu


def _far_molecules(systems):
    """PME water with every third water moved by 2-4 box lengths per axis: the list build wraps those molecules back."""
    d = systems.water_box(7, cutoff=0.9)
    nw = d.natoms//3
    k = np.random.default_rng(9).choice([-4, -3, -2, 2, 3, 4], size=(nw, 3))*(np.arange(nw) % 3 == 0)[:, None]
    d.positions = d.positions + np.repeat(k @ d.box, 3, axis=0)
    return d.rounded()


def _many_exclusions(systems):
    """PME water in which the oxygen of every fifth water also excludes its 40 nearest atoms of other waters: more than the
    24 partners a lane caches per i-block, so the masks also take the uncached look-up."""
    d = systems.water_box(8, cutoff=0.9)
    x = d.positions
    ei, ej = [d.exc_i], [d.exc_j]
    for a in range(0, d.natoms, 15):
        r = np.linalg.norm(x - x[a], axis=1)
        r[a - a % 3:a - a % 3 + 3] = np.inf
        nbr = np.argsort(r, kind="stable")[:40]
        ei.append(np.full(len(nbr), a, np.int32))
        ej.append(nbr.astype(np.int32))
    d.exc_i, d.exc_j = np.concatenate(ei).astype(np.int32), np.concatenate(ej).astype(np.int32)
    n = len(d.exc_i)
    d.exc_qq, d.exc_sigma, d.exc_eps = np.zeros(n), np.ones(n), np.zeros(n)
    return d.rounded()


def system(name):
    from openmm_b200 import systems
    if name in ("dhfr", "dhfr_200_steps"):
        return systems.SystemDesc.load(os.path.join(ROOT, "data", "dhfr.npz")).rounded()
    if name == "apoa1":
        return systems.SystemDesc.load(os.path.join(ROOT, "data", "apoa1.npz")).rounded()
    if name == "ions_triclinic":
        return systems.random_ions(894, 3.0, cutoff=1.0, triclinic=True).rounded()
    if name == "water_partial_block":
        return systems.water_box(7, cutoff=0.9).rounded()       # 1,029 atoms: the last block is partial
    if name == "cluster_nocutoff":
        return systems.cluster(70).rounded()
    if name == "many_exclusions":
        return _many_exclusions(systems)
    if name == "far_molecules":
        return _far_molecules(systems)
    raise KeyError(name)


# DHFR (8 warps per i-block), ApoA1 (4), a triclinic box (27-image box test, no exact cull), an atom count that is not a
# multiple of 32, no cutoff, more exclusions than a lane caches, molecules to wrap, and a list rebuilt during a run
CASES = ["dhfr", "apoa1", "ions_triclinic", "water_partial_block", "cluster_nocutoff", "many_exclusions", "far_molecules",
         "dhfr_200_steps"]


def canonical(eng):
    """(SHA-256 of the canonical list, tiles, masked tiles)"""
    sorig, ti, tj, tm = eng.get_list()
    order = np.lexsort(tuple(tj[:, k] for k in range(31, -1, -1)) + (ti,))
    rec = np.concatenate([ti[order, None].astype("<i4").view("<u4"), tj[order].astype("<i4").view("<u4"),
                          tm[order].astype("<u4")], axis=1)
    h = hashlib.sha256(sorig.astype("<i4").tobytes())
    h.update(np.ascontiguousarray(rec).tobytes())
    masked = int((tm != 0xffffffff).any(axis=1).sum())
    return h.hexdigest(), len(ti), masked


def build(name):
    """(engine, canonical list) of the case"""
    from openmm_b200 import Engine, systems
    eng = Engine(system(name))
    eng.compute(energy=False)
    if name == "dhfr_200_steps":
        eng.set_integrator(systems.INT_LANGEVIN, 0.002, 300.0, 1.0, 11)
        eng.step(200)
        eng.synchronize()
    return eng, canonical(eng)


@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(GOLDEN, "list_hashes.json")) as f:
        return json.load(f)


@pytest.mark.parametrize("name", CASES)
def test_list_is_identical(golden, name):
    eng, (digest, tiles, masked) = build(name)
    st = eng.stats()
    assert st["overflow"] == 0
    assert (tiles, masked) == (golden[name]["tiles"], golden[name]["masked_tiles"])
    assert (st["num_tiles"], st["num_mask_tiles"]) == (tiles, masked)
    if name == "dhfr_200_steps":
        assert st["list_builds"] == golden[name]["list_builds"] > 3
    assert digest == golden[name]["sha256"]


def test_canonical_form_sees_the_dealing():
    """Two j-slots swapped between tiles of one i-block (as a different dealing of candidate blocks to warps would do)
    change the canonical form, while reordering the tiles does not."""
    class Fake:
        def __init__(self, lst):
            self.lst = lst

        def get_list(self):
            return self.lst
    sorig = np.arange(64, dtype=np.int32)
    ti = np.array([0, 0, 1], np.int32)
    tj = np.stack([np.arange(32), np.arange(32, 64), np.arange(32, 64)]).astype(np.int32)
    tm = np.full((3, 32), 0xffffffff, np.uint32)
    base = canonical(Fake((sorig, ti, tj, tm)))
    assert canonical(Fake((sorig, ti[::-1].copy(), tj[::-1].copy(), tm[::-1].copy()))) == base
    tj2 = tj.copy()
    tj2[0, 5], tj2[1, 7] = tj[1, 7], tj[0, 5]
    assert canonical(Fake((sorig, ti, tj2, tm)))[0] != base[0]
