"""GPU tests that the engine's neighbour list is right, not only that it is the list it always was (test_gpu_list_identity):
the list of Engine.get_list() against an exact enumeration of the pairs, through the checker of tests/list_check.py.

At a build every non-excluded pair closer than the padded cutoff rc*(1 + pad) must be masked in exactly once (the pairs
between rc and rc + padding are the ones the displacement check relies on, and no force test at a fresh build looks at
them); on an aged list every pair closer than rc.  For systems with a GB force the mask-free view of k_gb_born, k_gb_pairs
and k_gb_chain is checked as well: every pair within the GB cutoff exactly once, excluded pairs included, no pair twice.
stats()["pairs_in_cutoff"] (k_count_pairs) must equal the checker's count of masked-in pairs closer than rc, up to the
pairs within fp32 reach of rc (1e-6 nm; 2.6e-6 nm in ApoA1's 10.9 nm box)."""
import copy
import os
import time

import numpy as np
import pytest
from conftest import ROOT

pytestmark = pytest.mark.gpu
PAD = 0.1                   # B200MD_PAD_FRACTION's default (engine.cu)


@pytest.fixture
def LC():
    import list_check
    return list_check


def _build_case(name):
    """(SystemDesc, has a GB force) of a build case"""
    from openmm_b200 import systems
    import test_gpu_list_identity as LI
    import test_gpu_oracle_edges as OE
    if name in ("dhfr", "apoa1", "ions_triclinic", "cluster_nocutoff", "many_exclusions", "water_partial_block", "far_molecules"):
        return LI.system(name), False
    if name == "water24k":
        return systems.water_box(20, cutoff=0.9).rounded(), False
    if name.startswith("triclinic_"):
        return OE.triclinic_limit_ions(systems, name.split("_")[1]), False
    if name.startswith("ions"):
        n = int(name[4:])
        return OE.ions_in_box(systems, n, np.diag([2.05]*3), 1.0, seed=n), False
    if name.startswith("shift_"):
        off, on = OE.shift_box_pair(systems)
        return (off if name == "shift_off" else on), False
    if name.startswith("water_L"):
        # 8^3 waters on a lattice stretched to the box edge L: 0.5*L - rc - padding runs from 0.16 to 0.51 nm, across the
        # largest block half-extent the exact cull compares it with
        L = float(name[7:])
        return systems.water_box(8, cutoff=0.9, spacing=L/8).rounded(), False
    if name in ("overflow_cluster", "water_slab", "dense_cluster", "far_and_neutral_water"):
        return getattr(OE, name)(systems), False
    if name.startswith("dhfr_gbsa"):
        import gbsa_harness as H
        return H.dhfr_gbsa(systems.NB_NOCUTOFF if name.endswith("nocutoff") else systems.NB_CUTOFF_NONPERIODIC).rounded(), True
    raise KeyError(name)


SWEEP = ["water_L%.1f" % L for L in np.arange(2.3, 3.05, 0.1)]
BUILD_CASES = (["dhfr", "apoa1", "water24k", "ions_triclinic", "triclinic_pmp", "triclinic_mpm"]
               + ["ions%d" % n for n in (2, 31, 32, 33, 63, 65, 97)]
               + ["shift_off", "shift_on"] + SWEEP
               + ["overflow_cluster", "cluster_nocutoff", "water_slab", "dense_cluster", "far_and_neutral_water", "many_exclusions",
                  "water_partial_block", "far_molecules", "dhfr_gbsa_cutoff", "dhfr_gbsa_nocutoff"])


def _need_r(d, pad=PAD):
    from openmm_b200 import systems
    return np.inf if d.method == systems.NB_NOCUTOFF else d.cutoff*(1.0 + pad)


def check_engine(LC, eng, d, need_r, band, gb=False):
    """check_list on the engine's current list at its positions, and stats()["pairs_in_cutoff"] against the checker's
    count; returns the checker's report"""
    from openmm_b200 import systems
    x = eng.get_positions()
    if eng.precision == "mixed":
        x = x.astype(np.float32).astype(np.float64)              # the list and the pair kernels read the fp32 hi part
    nocut = d.method == systems.NB_NOCUTOFF
    gb_cutoff = (np.inf if nocut else d.cutoff) if gb else None
    rep = LC.check_list(d, x, *eng.get_list(), need_r=need_r, gb_cutoff=gb_cutoff, band=band,
                        count_r=None if nocut else d.cutoff)
    st = eng.stats()
    assert st["overflow"] == 0 and st["num_tiles"] == rep["tiles"]
    if nocut:
        assert st["pairs_in_cutoff"] == rep["masked"] == rep["required"]
    else:
        lo, hi = rep["count_bounds"]
        assert lo <= st["pairs_in_cutoff"] <= hi, (st["pairs_in_cutoff"], lo, hi)
    return rep


@pytest.mark.parametrize("name", BUILD_CASES)
def test_built_list_holds_every_pair_within_the_padded_cutoff(LC, monkeypatch, record_property, name):
    from openmm_b200 import Engine
    monkeypatch.delenv("B200MD_PAD_FRACTION", raising=False)
    d, gb = _build_case(name)
    eng = Engine(d)
    eng.compute(energy=False)
    t0 = time.perf_counter()
    rep = check_engine(LC, eng, d, _need_r(d), LC.BUILD_BAND, gb=gb)
    wall = time.perf_counter() - t0
    eng.close()
    print("%s: %d tiles, %d masked-in pairs, %d required, %d in the band%s; checked in %.1f s"
          % (name, rep["tiles"], rep["masked"], rep["required"], rep["band"],
             ", GB %d of %d required" % (rep["gb_pairs"], rep["gb_required"]) if gb else "", wall))
    record_property("check_seconds", wall)
    assert rep["masked"] > 0


def _age_and_check(LC, eng, d, nsteps):
    """Step one step at a time with a compute() after each (test_gpu_oracle_edges._age); every state whose compute() did
    not rebuild the list is checked at need_r = rc (the freshly built ones are what the build cases check).  Returns the
    number of aged states checked."""
    aged = 0
    for _ in range(nsteps):
        eng.step(1)
        b1 = eng.stats()["list_builds"]
        eng.compute(energy=False)
        if eng.stats()["list_builds"] == b1:
            check_engine(LC, eng, d, d.cutoff, LC.AGED_BAND)
            aged += 1
    return aged


@pytest.mark.parametrize("name,T", [("dhfr", 300.0), ("water24k", 600.0)])
def test_aged_list_holds_every_pair_within_the_cutoff(LC, monkeypatch, record_property, name, T):
    """80 Langevin steps of 0.5 fs at padding 0.02 (the list is rebuilt every few steps): every state is checked"""
    from openmm_b200 import Engine, systems
    import test_gpu_oracle_edges as OE
    monkeypatch.setenv("B200MD_PAD_FRACTION", "0.02")
    d, _ = _build_case(name)
    eng = Engine(d)
    eng.set_integrator(systems.INT_LANGEVIN, 0.0005, T, 1.0, 3)
    eng.set_velocities(OE._thermal_velocities(d, T, 3))
    eng.apply_velocity_constraints()
    eng.compute(energy=False)
    aged = _age_and_check(LC, eng, d, 80)
    builds = eng.stats()["list_builds"]
    eng.close()
    print("%s at %g K: %d aged states checked, %d list builds" % (name, T, aged, builds))
    record_property("aged_states", aged)
    assert aged > 20 and builds > 5


def test_list_after_molecules_moved_by_lattice_vectors(LC, monkeypatch):
    from openmm_b200 import Engine, systems
    import test_gpu_oracle_edges as OE
    monkeypatch.delenv("B200MD_PAD_FRACTION", raising=False)
    d, _ = _build_case("water24k")
    eng = Engine(d)
    eng.set_integrator(systems.INT_LANGEVIN, 0.002, 300.0, 1.0, 7)
    eng.set_velocities(OE._thermal_velocities(d, 300.0, 7))
    eng.step(10)
    x = eng.get_positions()
    rng = np.random.default_rng(7)
    mols = d.molecules()
    k = rng.choice([-3, -2, 2, 3], size=(len(mols), 3))*(rng.random(len(mols)) < 0.5)[:, None]
    for m, km in zip(mols, k):
        x[m] += km @ d.box
    eng.set_positions(x)
    b0 = eng.stats()["list_builds"]
    eng.compute(energy=False)
    rebuilt = eng.stats()["list_builds"] > b0
    check_engine(LC, eng, d, _need_r(d) if rebuilt else d.cutoff, LC.BUILD_BAND if rebuilt else LC.AGED_BAND)
    for _ in range(5):
        eng.step(1)
        eng.compute(energy=False)
    check_engine(LC, eng, d, d.cutoff, LC.AGED_BAND)
    eng.close()


@pytest.mark.parametrize("scale", [0.99, 1.01])
def test_list_after_a_barostat_move(LC, monkeypatch, scale):
    """scale_coordinates, then set_box with the scaled box (as MonteCarloBarostatImpl does): the list of the scaled state"""
    from openmm_b200 import Engine, systems
    monkeypatch.delenv("B200MD_PAD_FRACTION", raising=False)
    d = systems.SystemDesc.load(os.path.join(ROOT, "data", "dhfr.npz")).rounded()
    eng = Engine(d)
    eng.compute(energy=False)
    eng.set_barostat_molecules()
    eng.scale_coordinates(scale, scale, scale)
    eng.set_box(d.box*scale)
    b0 = eng.stats()["list_builds"]
    eng.compute(energy=False)
    rebuilt = eng.stats()["list_builds"] > b0
    s = copy.copy(d)
    s.box = eng.get_box()
    check_engine(LC, eng, s, _need_r(s) if rebuilt else s.cutoff, LC.BUILD_BAND if rebuilt else LC.AGED_BAND)
    eng.close()
