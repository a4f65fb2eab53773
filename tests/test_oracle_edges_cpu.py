"""CPU companion of tests/test_gpu_oracle_edges.py.  Where oracle/_ref holds the reference itself, the C restatement
(oracle/md_oracle.c) is pinned to the live Reference platform on the new edge systems, so that the GPU tests rest on a
pinned oracle; everywhere, the host-side facts those GPU tests rely on are checked."""
import numpy as np
import pytest
from conftest import relative_force_error
from openmm_b200 import systems
from oracle import port
import test_gpu_oracle_edges as edges


def _live_cases():
    yield "pme_switch_water", edges.pme_switch_water(systems)
    # Only the (-, +, -) limit: in the (+, -, +) cell (b.x = a/2, c.x = -a/2, c.y = b/2) the Reference platform's voxel
    # neighbour list (ReferenceNeighborList.cpp, the shifted x / y voxel windows of the periodic search) misses pairs inside
    # the cutoff -- 4e-2 relative on the forces and 0.7 kJ/mol at cutoff 1.09 nm, still 1e-2 at 0.8 nm -- although for every
    # pair within the cutoff the three-step minimum image it and the oracle use is the nearest image
    # (test_triclinic_limit_boxes_are_reduced_form).  The GPU tests compare both cells with the all-pairs oracle.
    yield "triclinic_limit_mpm", edges.triclinic_limit_ions(systems, "mpm")
    for g in edges.ODD_GRIDS:
        yield "odd_grid_%d_%d_%d" % g, edges.odd_grid_ions(systems, g)
    yield "close_contact_ions", edges.close_contact_ions(systems)


@pytest.mark.parametrize("name", [n for n, _ in _live_cases()])
def test_oracle_matches_live_reference_on_edge_systems(name):
    """PME with a switching function, the reduced-form triclinic limits, odd / anisotropic PME grids with a large alpha,
    and the close-contact ions at alpha 4.4 nm^-1: the restatement against the Reference platform on the same alpha and grid."""
    from oracle import omm
    if not omm.available():
        pytest.skip("oracle/_ref has no build of the reference (needs its sources at build time)")
    d = dict(_live_cases())[name]
    pme = d.pme_parameters()
    f, e, _ = port.forces_energy(d, pme=pme)
    sim = omm.Simulation(d, "Reference", pme=pme)
    try:
        assert sim.pme_parameters()[1:] == tuple(pme[1:]) and abs(sim.pme_parameters()[0] - pme[0]) < 1e-12
        fr, er = sim.forces_energy()
    finally:
        sim.close()
    assert relative_force_error(f, fr) < 1e-8
    assert abs(e - er) < 1e-8*max(1.0, abs(er))


@pytest.mark.parametrize("sign", sorted(edges.TRICLINIC_LIMITS))
def test_triclinic_limit_boxes_are_reduced_form(sign):
    """OpenMM's reduced form (a along x, b in the xy plane, |b.x|, |c.x| <= a.x/2, |c.y| <= b.y/2), met with equality, and a
    cutoff within 10 % of half the smallest distance between opposite faces (and no more than half of a.x, b.y, c.z)."""
    d = edges.triclinic_limit_ions(systems, sign)
    a, b, c = d.box
    assert a[1] == a[2] == b[2] == 0
    assert abs(b[0]) == a[0]/2 and abs(c[0]) == a[0]/2 and abs(c[1]) == b[1]/2
    w = edges.cell_widths(d.box).min()
    assert 0.45*w < d.cutoff < 0.5*w
    assert d.cutoff <= 0.5*min(a[0], b[1], c[2])
    # the three-step minimum image (c, then b, then a; ReferenceForce::getDeltaRPeriodic) finds the nearest of the 125
    # images for every pair within the cutoff, so the all-pairs oracle counts every interacting pair exactly once
    x = d.positions
    dd = x[None] - x[:, None]
    r3 = dd.copy()
    for axis in (2, 1, 0):
        r3 -= np.floor(r3[..., axis]/d.box[axis][axis] + 0.5)[..., None]*d.box[axis]
    r3 = np.linalg.norm(r3, axis=-1)
    best = np.full(r3.shape, np.inf)
    for s in np.stack(np.meshgrid(*[np.arange(-2, 3)]*3, indexing="ij"), -1).reshape(-1, 3):
        best = np.minimum(best, np.linalg.norm(dd + s @ d.box, axis=-1))
    inside = best < d.cutoff
    np.fill_diagonal(inside, False)
    assert inside.sum() > 1000 and np.abs(r3[inside] - best[inside]).max() < 1e-9


def test_shift_mode_margins():
    """The single-image mode of the tile kernel needs 0.5*minL - rc - padding >= (largest block half extent) > 0; padding is
    0.1*rc by default (engine.cu padFrac)."""
    off, on = edges.shift_box_pair(systems)
    assert off.natoms == 3*6**3 and on.natoms == 3*16**3 and off.cutoff == on.cutoff
    assert off.box[0][0] >= 2*off.cutoff                                 # a valid periodic box, ...
    assert 0.5*off.box[0][0] - off.cutoff - 0.1*off.cutoff < 0           # ... too small for the single-image mode
    assert 0.5*on.box[0][0] - on.cutoff - 0.1*on.cutoff > 1.4


def test_overflow_cluster_fills_one_tile_beyond_the_close_pair_queue():
    """Non-periodic systems keep the identity order, so atoms 0-31 form one block: more than CLOSE_QCAP = 96 of its
    pairs (all 496) are closer than the 0.36 nm close-pair distance."""
    d = edges.overflow_cluster(systems)
    assert d.natoms >= 40 and d.box is None
    x = d.positions[:32]
    r = np.linalg.norm(x[:, None] - x[None], axis=-1)[np.triu_indices(32, 1)]
    assert (r < 0.36).sum() > 96 and (r < 0.36).all()
    assert np.ptp(d.positions, axis=0).max() <= 0.2
    assert r.min() > 0.02                                                  # no pair closer than the LJ sigma


def test_close_contact_ions_geometry():
    d = edges.close_contact_ions(systems)
    x = d.positions
    pair = np.linalg.norm(x[0::2] - x[1::2], axis=1)
    assert pair.min() >= 0.15 - 1e-6 and pair.max() <= 0.36 + 1e-6
    r = np.linalg.norm(x[:, None] - x[None], axis=-1)
    np.fill_diagonal(r, np.inf)
    r[np.arange(0, d.natoms, 2), np.arange(1, d.natoms, 2)] = np.inf
    r[np.arange(1, d.natoms, 2), np.arange(0, d.natoms, 2)] = np.inf
    assert r.min() > 0.18                                                  # other ions stay clear of the close pairs
    assert abs(d.pme_parameters()[0] - 4.38) < 0.01 and d.cutoff == 0.6


def test_odd_grids_factor_into_supported_radices():
    for g in edges.ODD_GRIDS:
        assert all(systems.fft_size_ok(n) for n in g), g
    assert any(g[2] % 2 for g in edges.ODD_GRIDS) and any(g[2] % 2 == 0 for g in edges.ODD_GRIDS)
    assert any(len(set(n % 2 for n in g)) == 2 for g in edges.ODD_GRIDS)


def test_edge_builders_keep_molecules_and_inputs_exact():
    slab = edges.water_slab(systems)
    assert slab.natoms % 3 == 0 and len(slab.con_i) == slab.natoms and slab.positions[:, 2].max() < 0.5*slab.box[2][2] + 0.2
    far = edges.far_and_neutral_water(systems)
    L = far.box[0][0]
    assert (np.abs(far.positions) > 2*L).any() and (far.charges == 0).sum() > 0 and (far.epsilons[0::3] == 0).sum() > 0
    for d in (slab, far, edges.dense_cluster(systems), edges.overflow_cluster(systems)):
        assert np.array_equal(d.positions, d.positions.astype(np.float32).astype(np.float64))


def test_forces_only_cases_cover_every_reference_case():
    """The forces-only GPU parity test is parametrized by name: it must name every case of the Reference-platform parity
    tests, so that a case added there does not go without a forces-only check."""
    from test_gpu_parity import reference_cases
    assert sorted(edges._reference_case_names()) == sorted(reference_cases(systems))
