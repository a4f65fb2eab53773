"""The engine at up to 1.5 M atoms: periodic supercells of DHFR, ApoA1, water and the triclinic ion box (tests/supercell_harness.py)
against the double-precision restatement on their unit cells, and against the engine on the unit cell.

In exact arithmetic every copy of an atom in a k x k x k supercell (the unit cell's alpha, k times its grid and box) feels the
force its atom feels in the unit cell, and the coordinates are quantized so that the device reads exactly that geometry.  This
reaches what no smaller system does: tile pools of millions of tiles and their int tile / mask indices, the list build's
grid-wide cell scan over ~1e5 cells, the line-batched FFT (any grid edge above 160 points), brick spreads of tens of thousands
of CTAs, and fp32 coordinates of 20-26 nm in the tile kernel's differences and minimum images.

  case               atoms       box         grid   FFT
  dhfr_x2            188,464     12.4 nm     112^3  slab
  dhfr_x3            636,066     18.7 nm     168^3  line-batched (radix 8, 3, 7)
  dhfr_x4          1,507,712     24.9 nm     224^3  line-batched
  apoa1_x2           737,792     21.8 nm     176^3  line-batched (radix 11)
  water23_x3         985,527     21.4 nm     192^3  line-batched (bench.py's water1m: its atom count and box)
  ions_triclinic_x4   57,216     12 nm tri.  100^3  slab"""
import copy
import time
import numpy as np
import pytest
from conftest import relative_force_error
import energy_harness as EH
import supercell_harness as SC

pytestmark = pytest.mark.gpu
TOL = 1e-4                      # test_gpu_parity.py: the reference's ASSERT_EQUAL_VEC form
KT = EH.KT
BONDED_REL = 1e-9
CASES = {"dhfr_x2": ("dhfr", 2), "dhfr_x3": ("dhfr", 3), "dhfr_x4": ("dhfr", 4), "apoa1_x2": ("apoa1", 2),
         "water23_x3": ("water23", 3), "ions_triclinic_x4": ("ions_triclinic", 4)}
# Per-copy bounds in kJ/mol on the direct and reciprocal groups against the oracle: the unit cell's own bounds of
# tests/test_gpu_energy.py (test_gpu_energy.part_bounds) for the systems it measures; for the 23^3 water box twice the worst
# per-copy error measured on an H100 SXM (80 GB HBM3, 700 W power limit): direct -1.1729 kJ/mol (the unit cell of 24,000
# atoms measures 0.76: the tile kernel's fp32 bias grows with the atom count), reciprocal < 1e-4 (floored at
# test_gpu_energy.PART_FLOOR).
WATER23_BOUNDS = (2.35, 0.005)
# The direct-space forces of each copy against the engine on the unit cell: the pair terms are evaluated from the same exact
# displacements, and only the fp32 sums of the tile kernel differ, because a tile groups different j atoms in the two lists.
# Twice the worst measured over the cases, 1.08e-5 on apoa1_x2 (1.4e-6 to 4.2e-6 on the others; H100 SXM, 700 W).
DIRECT_ENGINE_BOUND = 2.2e-5
# A pair whose distance lies within an fp32 rounding of the cutoff may be counted on the other side of it by the tile kernel
# than by the oracle (test_gpu_energy.py EDGE_DELTA): the quantized coordinates make every displacement exact, but r^2 is
# still summed in fp32 (~1e-7 nm along the pair at the cutoff) and rc^2 rounded to fp32.  Such a pair changes its atoms'
# forces by up to ~0.3 kJ/mol/nm (DHFR: 0.23 at the 3.8e-6 nm quantum of dhfr_x3 and dhfr_x4, 4.4e-4 of the atom's force),
# and whether one exists depends on the quantum: an atom above TOL is allowed the forces of its pairs within EDGE_DELTA of
# the cutoff (supercell_harness.excess_over_edge).
EDGE_DELTA = 5e-7
# ApoA1: beyond the cutoff-edge pairs two atoms of every copy stay 1.20e-4 off (H100 SXM, 700 W), in every copy alike, so it
# is the geometry of the quantized cell and not the supercell; ApoA1 is the system whose atoms with ~1 kJ/mol/nm net forces
# are differences of ~100 kJ/mol/nm direct and reciprocal sums (test_gpu_parity.test_real_benchmark_systems_parity).  Twice
# the measured value.
FORCE_BOUNDS = {"apoa1_x2": 2.4e-4}
_CASES = {}


def _case(name):
    """(quantized unit cell, supercell, k, supercell dispersion energy) of a case, built once per module"""
    if name not in _CASES:
        unit_name, k = CASES[name]
        u = SC.quantized(SC.unit(unit_name), k)
        s = SC.supercell(u, k)
        _CASES[name] = (u, s, k, SC.dispersion_energy(s))
    return _CASES[name]


def _bounds(name):
    unit_name = CASES[name][0]
    if unit_name == "water23":
        return WATER23_BOUNDS
    from test_gpu_energy import part_bounds
    return part_bounds(unit_name)


def _engine(d, precision="single"):
    from openmm_b200 import Engine
    return Engine(d, precision=precision)


@pytest.mark.parametrize("name", list(CASES))
def test_copies_match_the_unit_cell_oracle(name, record_property):
    """Every copy's forces against the oracle's on the unit cell, and every energy group over k^3 against the unit cell's."""
    u, s, k, disp = _case(name)
    t0 = time.perf_counter()
    fo, _ = SC.oracle(u)
    r = SC.expected_groups(u, k, disp)
    t1 = time.perf_counter()
    eng = _engine(s)
    total = eng.compute()
    f = eng.get_forces()
    e = EH.engine_parts(eng, s)
    st = eng.stats()
    eng.close()
    t2 = time.perf_counter()
    alpha, nx, ny, nz = u.pme_parameters()
    assert st["pme_grid"] == [k*nx, k*ny, k*nz]
    assert st["overflow"] == 0
    errs = [relative_force_error(fc, fo) for fc in SC.copies(f, k)]
    worst = max(errs)
    edge = [SC.excess_over_edge(u, u.positions, fc, fo, TOL, EDGE_DELTA) for fc in SC.copies(f, k)]
    worst_edge, edge_atoms = max(e[0] for e in edge), max(e[1] for e in edge)
    part_errs = {g: e[g]/k**3 - r[g] for g in e}
    total_err = total/k**3 - sum(r[g] for g in e)
    print("%s: %d atoms, grid %s, %d tiles; per-copy force error against the oracle %.2e (median %.2e; %.2e beyond the forces "
          "of the pairs at the cutoff of %d atoms); per-copy parts %s; total %+.4f kJ/mol (%+.3f kT); oracle %.1f s, engine %.1f s"
          % (name, s.natoms, st["pme_grid"], st["num_tiles"], worst, float(np.median(errs)), worst_edge, edge_atoms,
             ", ".join("%s %+.4f" % kv for kv in part_errs.items()), total_err, total_err/KT, t1 - t0, t2 - t1))
    record_property("force_error", worst)
    record_property("force_error_beyond_cutoff_edge", worst_edge)
    record_property("total_error_kj", total_err)
    record_property("seconds", t2 - t0)
    for g, err in part_errs.items():
        record_property(g + "_error_kj", err)
    assert worst_edge < FORCE_BOUNDS.get(name, TOL), (worst, worst_edge)
    direct_bound, recip_bound = _bounds(name)
    for g, err in part_errs.items():
        if g == "direct":
            assert abs(err) <= direct_bound, (g, err, direct_bound)
        elif g == "reciprocal":
            assert abs(err) <= recip_bound, (g, err, recip_bound)
        else:
            assert abs(err) <= BONDED_REL*max(1.0, abs(r[g])), (g, err)
    assert abs(total_err) <= KT, total_err


@pytest.mark.parametrize("name", list(CASES))
def test_copies_match_the_unit_cell_engine(name, record_property):
    """The bonded terms of every copy bit for bit those of the engine on the unit cell; the direct-space forces up to the
    order of the tile kernel's fp32 sums; k^3 times the unit cell's pairs inside the cutoff."""
    from openmm_b200.engine import TERM_BONDS, TERM_ANGLES, TERM_TORSIONS, TERM_NB_DIRECT
    u, s, k, _ = _case(name)
    t0 = time.perf_counter()
    eu, es = _engine(u), _engine(s)
    out = {}
    if len(u.bond_i) or len(u.angle_i) or len(u.tor_i):
        # each term's doubles come from the same exact differences and its forces are summed in int64 fixed point, so the
        # order does not matter; the energies are double atomics (a few ulps apart)
        mask = TERM_BONDS | TERM_ANGLES | TERM_TORSIONS
        ebu, ebs = eu.compute(mask), es.compute(mask)
        fbu, fbs = eu.get_forces(), es.get_forces()
        differing = sum(int(not np.array_equal(fc, fbu)) for fc in SC.copies(fbs, k))
        out["bonded_copies_differing"] = differing
        out["bonded_energy_difference"] = ebs - k**3*ebu
        assert differing == 0, "%d of %d copies' bonded forces differ from the unit cell's" % (differing, k**3)
        assert abs(ebs - k**3*ebu) <= 1e-12*abs(ebs), (ebs, k**3*ebu)
    eu.compute(TERM_NB_DIRECT)
    es.compute(TERM_NB_DIRECT)
    fdu, fds = eu.get_forces(), es.get_forces()
    out["direct_error"] = max(relative_force_error(fc, fdu) for fc in SC.copies(fds, k))
    pu, ps = eu.stats()["pairs_in_cutoff"], es.stats()["pairs_in_cutoff"]
    out["pairs_unit"], out["pairs_super"] = pu, ps
    assert es.stats()["overflow"] == 0 and eu.stats()["overflow"] == 0
    eu.close()
    es.close()
    out["seconds"] = time.perf_counter() - t0
    print("%s: %s" % (name, ", ".join("%s %s" % kv for kv in out.items())))
    for kv in out.items():
        record_property(*kv)
    assert out["direct_error"] < DIRECT_ENGINE_BOUND, out["direct_error"]
    # k_count_pairs sees the same exact displacements in both engines
    assert ps == k**3*pu, (ps, pu)


def test_supercell_list_is_valid(monkeypatch, record_property):
    """The list the engine builds for DHFR x 2 holds every non-excluded pair within the padded cutoff exactly once
    (tests/list_check.py, as test_gpu_list_validity.check_engine runs it)."""
    import list_check as LC
    from test_gpu_list_validity import check_engine, _need_r
    monkeypatch.delenv("B200MD_PAD_FRACTION", raising=False)
    _, s, _, _ = _case("dhfr_x2")
    eng = _engine(s)
    eng.compute(energy=False)
    t0 = time.perf_counter()
    rep = check_engine(LC, eng, s, _need_r(s), LC.BUILD_BAND)
    wall = time.perf_counter() - t0
    eng.close()
    print("dhfr_x2: %d tiles, %d masked-in pairs, %d required, %d in the band; checked in %.1f s"
          % (rep["tiles"], rep["masked"], rep["required"], rep["band"], wall))
    record_property("check_seconds", wall)
    assert rep["masked"] > 0


AGED_BOUND = 1.5e-5             # test_gpu_oracle_edges.AGED_BOUND
# The aged list and the fresh one may put a pair within an fp32 rounding of its displacement of the cutoff on different
# sides (the single-image shift is added to whichever atom a tile holds; test_gpu_energy.py).  In the 24.9 nm box a shifted
# coordinate stays below 64 nm, so each component rounds by at most 1.9e-6 nm, 3.3e-6 nm along the pair: an atom above
# AGED_BOUND is allowed the forces of its pairs within AGED_EDGE_DELTA of the cutoff.
AGED_EDGE_DELTA = 4e-6
# Beyond those pairs the 24.9 nm DHFR x 4 measures 1.72e-5 (H100 SXM, 700 W) where DHFR at 6.2 nm stays under AGED_BOUND:
# the fp32 coordinates there round four times as coarsely.  Twice the measured value.
AGED_BOUND_AT_SCALE = 3.5e-5
STEPS = 200


@pytest.mark.parametrize("name,precision", [("dhfr_x4", "single"), ("dhfr_x2", "mixed")])
def test_bench_protocol_at_scale(name, precision, record_property):
    """bench.py's protocol on a supercell: Langevin at 300 K, 1/ps, 2 fs, constraint tolerance 1e-5, thermal velocities, 200
    steps; then the forces on the list as it stands (not rebuilt on the last step) against a fresh engine at the same inner
    positions, every HBonds constraint of a sample, and a finite state without overflow."""
    from openmm_b200 import systems
    from test_gpu_oracle_edges import _thermal_velocities
    _, s, _, _ = _case(name)
    t0 = time.perf_counter()
    eng = _engine(s, precision)
    eng.set_integrator(systems.INT_LANGEVIN, 0.002, 300.0, 1.0, 17, 1e-5)
    eng.set_velocities(_thermal_velocities(s, 300.0, 17))
    eng.apply_velocity_constraints()
    builds0 = eng.stats()["list_builds"]
    eng.step(STEPS - 1)
    steps = STEPS - 1
    while True:                     # one step at a time until a state whose last step and compute() both kept the list
        b0 = eng.stats()["list_builds"]
        eng.step(1)
        steps += 1
        b1 = eng.stats()["list_builds"]
        eng.compute(energy=False)
        if eng.stats()["list_builds"] == b1 == b0:
            break
        assert steps < STEPS + 100, "no aged state"
    f = eng.get_forces()
    x = eng.get_positions()
    st = eng.stats()
    fresh_d = copy.copy(s)
    fresh_d.positions = EH.kernel_positions(eng)
    eng.close()
    fresh = _engine(fresh_d, precision)
    fresh.compute(energy=False)
    ff = fresh.get_forces()
    fresh.close()
    err_fresh = relative_force_error(f, ff)
    err_edge, edge_atoms = SC.excess_over_edge(s, fresh_d.positions, f, ff, AGED_BOUND, AGED_EDGE_DELTA)
    sel = slice(None, None, 97)
    con_err = float(np.abs(np.linalg.norm(x[s.con_i[sel]] - x[s.con_j[sel]], axis=1) - s.con_d[sel]).max())
    wall = time.perf_counter() - t0
    res = {"steps": steps, "list_builds": st["list_builds"] - builds0, "fresh_list": err_fresh, "fresh_list_beyond_cutoff_edge": err_edge,
           "atoms_above_bound": edge_atoms, "constraint": con_err, "seconds": wall}
    print("%s %s: %s" % (name, precision, ", ".join("%s %s" % kv for kv in res.items())))
    for kv in res.items():
        record_property(*kv)
    assert np.isfinite(x).all() and np.isfinite(f).all() and st["overflow"] == 0
    assert err_edge < AGED_BOUND_AT_SCALE, (err_fresh, err_edge)
    assert con_err < 2e-5, con_err
    assert res["list_builds"] < steps
