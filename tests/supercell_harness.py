"""Periodic supercells: a system tiled k x k x k against its unit cell (tests/test_supercell_cpu.py, tests/test_gpu_supercell.py).

Copy (i, j, l) of a periodic system, moved by i a + j b + l c, in the box k (a, b, c) with the unit cell's Ewald alpha and k
times its PME grid, feels in exact arithmetic exactly the forces its atom feels in the unit cell:
  direct space  every atom has the same neighbours, because the cutoff is below half of every unit cell width;
  reciprocal    the charge grid repeats with period n, so only wave vectors that are multiples of k survive, and at those the
                B-spline moduli and the influence function are the unit cell's divided by k^3: the potential grid, and every
                reciprocal force, is the unit cell's.
Every energy part is k^3 times the unit cell's except the dispersion correction, whose coefficient averages over the pairs
i <= j (NonbondedForceImpl::calcDispersionCorrection) and so does not scale as k^6: the supercell is held to its own.
The O(N^2) oracle therefore needs to run only on the unit cell, while the engine runs the supercell of up to 1.5 M atoms.

quantized() rounds the unit cell's positions and box to a power-of-two quantum q such that every supercell coordinate, and
every difference of two, is an integer multiple of q below 2^24 q: exact in fp32.  The device then reads exactly the geometry
the oracle evaluates, moved by whole lattice vectors, and every displacement a kernel forms (an fp32 difference of two
coordinates, a k L image shift, the bonded kernels' fp32 coordinates subtracted in double) is exact: what remains is the
device's own rounding."""
import hashlib
import math
import numpy as np
import energy_harness as EH

# per-atom and per-term fields a supercell tiles, and the atom index fields it offsets by copy * N
ATOM_FIELDS = ("masses", "charges", "sigmas", "epsilons")
TERM_FIELDS = {"exc": (("exc_i", "exc_j"), ("exc_qq", "exc_sigma", "exc_eps")),
               "con": (("con_i", "con_j"), ("con_d",)),
               "bond": (("bond_i", "bond_j"), ("bond_r0", "bond_k")),
               "angle": (("angle_i", "angle_j", "angle_k"), ("angle_t0", "angle_kk")),
               "tor": (("tor_i", "tor_j", "tor_k", "tor_l"), ("tor_n", "tor_phase", "tor_kk"))}
# terms a supercell does not replicate
UNSUPPORTED = ("rb_i", "cmap_map", "custom_prog", "cbond_prog", "cext_prog", "cangle_prog", "ccompound_expr", "ccentroid_expr",
               "gb_charges")


def unit(name):
    """A unit cell by name: the two proteins, the triclinic 894-ion box, the 7^3 water boxes (rigid or flexible) and the 23^3
    water box whose 3^3 supercell has the atom count and box of bench.py's water1m; positions fp32-representable."""
    from openmm_b200 import systems
    if name == "water23":
        return systems.water_box(23, cutoff=0.9).rounded()
    if name in ("dhfr", "apoa1", "ions_triclinic", "water_rigid", "water_flexible"):
        return EH.load(name)
    raise KeyError(name)


def _check_unit(d):
    from openmm_b200 import systems
    assert d.box is not None and d.method in (systems.NB_PME, systems.NB_CUTOFF_PERIODIC), "a supercell needs a periodic system"
    for f in UNSUPPORTED:
        assert len(getattr(d, f)) == 0, "supercells do not replicate %s" % f
    widths = np.diag(np.asarray(d.box, dtype=np.float64))      # reduced form: the perpendicular widths are a_x, b_y, c_z
    assert d.cutoff < 0.5*widths.min(), "the cutoff must be below half of every unit cell width"


def offsets(box, k):
    """[k^3, 3] lattice shifts i a + j b + l c of the copies, (i, j, l) in that order (l fastest)"""
    ijl = np.stack(np.meshgrid(*[np.arange(k)]*3, indexing="ij"), -1).reshape(-1, 3).astype(np.float64)
    return ijl @ np.asarray(box, dtype=np.float64)


def quantum(d, k):
    """The power of two q for which every coordinate of the k^3 supercell of d, every difference of two and the supercell box
    are integer multiples of q below 2^24 q once d's positions and box are multiples of q"""
    x = np.asarray(d.positions, dtype=np.float64)
    box = np.abs(np.asarray(d.box, dtype=np.float64))
    reach = max(np.abs(x).max() + (k - 1)*box.sum(axis=0).max(), k*box.sum(axis=0).max())
    return 2.0**math.ceil(math.log2(2.0*reach/2.0**24))


def quantized(d, k):
    """d with its PME alpha and grid pinned (those of d) and its positions and box rounded to quantum(d, k)"""
    _check_unit(d)
    out = EH.pinned_pme(d)
    q = quantum(d, k)
    out.positions = np.round(np.asarray(d.positions, dtype=np.float64)/q)*q
    out.box = np.round(np.asarray(d.box, dtype=np.float64)/q)*q
    return out


def supercell(d, k):
    """The k x k x k supercell of d: copy (i, j, l) of every atom at x + i a + j b + l c, copies in that order; per-atom and
    per-term arrays tiled, atom indices of exceptions, constraints, bonds, angles and torsions offset by copy * N; box k * box,
    the unit cell's PME alpha and k times its grid."""
    import copy
    from openmm_b200 import systems
    _check_unit(d)
    n, m = d.natoms, k**3
    s = copy.copy(d)
    s.positions = (np.asarray(d.positions, dtype=np.float64)[None, :, :] + offsets(d.box, k)[:, None, :]).reshape(m*n, 3)
    for f in ATOM_FIELDS:
        setattr(s, f, np.tile(np.asarray(getattr(d, f)), m))
    shift = (np.arange(m, dtype=np.int64)*n)[:, None]
    for atoms, params in TERM_FIELDS.values():
        for f in atoms:
            a = np.asarray(getattr(d, f), dtype=np.int64)
            setattr(s, f, (a[None, :] + shift).reshape(-1).astype(np.int32))
        for f in params:
            setattr(s, f, np.tile(np.asarray(getattr(d, f)), m))
    s.box = k*np.asarray(d.box, dtype=np.float64)
    if d.method == systems.NB_PME:
        alpha, nx, ny, nz = d.pme_parameters()
        s.pme_alpha, s.pme_grid = alpha, (k*nx, k*ny, k*nz)
    s.name = "%s_x%d" % (d.name, k)
    return s


def copies(a, k):
    """[k^3, N, ...]: a per-atom array of the supercell split by copy"""
    a = np.asarray(a)
    return a.reshape(k**3, -1, *a.shape[1:])


def fp32_exact(a):
    a = np.asarray(a, dtype=np.float64)
    return bool(np.array_equal(a.astype(np.float32).astype(np.float64), a))


_ORACLE = {}


def _key(d):
    h = hashlib.sha1()
    for a in (d.positions, d.box, d.charges, d.sigmas, d.epsilons, d.exc_i, d.exc_j, d.exc_qq, d.exc_sigma, d.exc_eps, d.bond_i,
              d.bond_r0, d.bond_k, d.angle_i, d.angle_t0, d.angle_kk, d.tor_i, d.tor_kk, d.tor_phase):
        h.update(np.ascontiguousarray(a, dtype=np.float64).tobytes())
    h.update(repr((d.natoms, d.method, d.cutoff, d.use_switch, d.switch_distance, d.use_dispersion, d.pme_parameters())).encode())
    return h.hexdigest()


def oracle(d):
    """(forces [N, 3], raw parts) of the restatement on d at d.positions, cached per configuration"""
    from oracle import port
    from openmm_b200 import systems
    key = _key(d)
    if key not in _ORACLE:
        pme = d.pme_parameters() if d.method == systems.NB_PME else None
        f, _, parts = port.forces_energy(d, pme=pme)
        _ORACLE[key] = (f, dict(parts))
    f, parts = _ORACLE[key]
    return f.copy(), dict(parts)


def dispersion_energy(d):
    return d.dispersion_coefficient()/EH.volume(d.box) if d.use_dispersion else 0.0


def expected_groups(u, k, super_dispersion):
    """{group: energy per copy} (energy_harness.GROUPS) the k^3 supercell of the unit cell u should have: the oracle's groups
    of u, with u's dispersion energy replaced by super_dispersion / k^3 (dispersion_energy of the supercell)"""
    _, parts = oracle(u)
    out = {g: float(sum(parts.get(p, 0.0) for p in ps)) for g, ps in EH.GROUPS.items()}
    out["direct"] += super_dispersion/k**3 - parts.get("dispersion", 0.0)
    return out


def cutoff_edge_forces(d, x, atoms, delta):
    """[len(atoms)] the sum of |pair force| (PME direct-space Coulomb + LJ, no switch) over the pairs of each of `atoms` whose
    distance lies within delta of the cutoff at positions x (orthorhombic box): pairs that an fp32 evaluation may count on
    the other side of the cutoff than the double-precision one.  Excluded pairs count too, which only widens the allowance."""
    from scipy.spatial import cKDTree
    from scipy.special import erfc
    box = np.asarray(d.box, dtype=np.float64)
    assert not np.count_nonzero(box - np.diag(np.diag(box))), "orthorhombic boxes only"
    L = np.diag(box)
    y = np.mod(np.asarray(x, dtype=np.float64), L)
    y[y >= L] = 0.0
    alpha = d.pme_parameters()[0]
    tree = cKDTree(y, boxsize=L)
    out = np.zeros(len(atoms))
    for n, (a, nbr) in enumerate(zip(atoms, tree.query_ball_point(y[np.asarray(atoms)], d.cutoff + delta))):
        j = np.array([b for b in nbr if b != a], dtype=np.int64)
        if not len(j):
            continue
        dd = y[j] - y[a]
        r = np.linalg.norm(dd - L*np.round(dd/L), axis=1)
        m = np.abs(r - d.cutoff) < delta
        j, r = j[m], r[m]
        qq = 138.93545764438198*d.charges[a]*d.charges[j]
        fc = qq*(erfc(alpha*r)/r + 2*alpha/math.sqrt(math.pi)*np.exp(-(alpha*r)**2))/r
        sr6 = (0.5*(d.sigmas[a] + d.sigmas[j])/r)**6
        flj = 24*np.sqrt(d.epsilons[a]*d.epsilons[j])*(2*sr6*sr6 - sr6)/r
        out[n] = float(np.abs(fc + flj).sum())
    return out


def excess_over_edge(d, x, f, fref, tol, delta):
    """(worst |dF_i|_inf / max(1, |F_ref,i|) after each atom's excess over tol is reduced by its cutoff_edge_forces, number of
    atoms above tol): the relative force error of conftest.relative_force_error, allowing every atom the forces of its pairs
    within delta of the cutoff.  Only the atoms above tol are looked at (x, f, fref: the same atoms, positions x)."""
    df = np.abs(f - fref).max(axis=1)
    norm = np.maximum(1.0, np.linalg.norm(fref, axis=1))
    over = np.nonzero(df > tol*norm)[0]
    rel = df/norm
    if len(over):
        rel[over] = np.maximum(0.0, (df[over] - cutoff_edge_forces(d, x, over, delta))/norm[over])
    return float(rel.max()), int(len(over))
