"""GPU tests of the kernels a run actually executes, against the plain-C double-precision oracle (oracle/md_oracle.c,
oracle.port.forces_energy, same PME alpha and grid as the engine) and, where it has a stored result, the Reference platform
(tests/golden/reference_platform.npz):
 1. the forces-only instantiations (compute(energy=False): k_pair<false, *>, k_fft_x_conv<false>, k_bonded<false>), which
    every MD step runs, against the Reference platform and against the energy path of the same engine;
 2. forces after the neighbour list has aged inside a run of Langevin steps (rebuild check, per-step sposq refresh, molecule
    wrap, single-image SHIFT mode), against the oracle and against a freshly built engine;
 3. shapes and edges: partly empty 32-atom blocks, SHIFT mode on and off, PME with a switching function, the switched
    close-pair path, more close pairs in one tile than the per-warp queue holds, reduced-form triclinic limits,
    inhomogeneous density, zero-charge / zero-epsilon atoms and molecules far outside the cell;
 4. PME on odd and anisotropic grids, slab and line-batched FFT.
Inputs are fp32-representable.  Tolerance: 1e-4 on forces in the ASSERT_EQUAL_VEC form, 1e-5 relative (floor 1) on energy.
The builders of the edge systems are shared with tests/test_oracle_edges_cpu.py, which pins the oracle itself to the live
Reference platform on them and checks the host-side claims made here."""
import copy
import numpy as np
import pytest
from conftest import relative_force_error

pytestmark = pytest.mark.gpu
TOL = 1e-4
ETOL = 1e-5
# forces-only against the energy path of the same engine and inputs, relative_force_error.  They differ only where the
# arithmetic differs: the close pairs of the forces-only PME tile kernel take the Ewald screening term from the fp32
# rational fit ewald_g instead of erfc/exp in double (nonbonded.cu close_pair_double).  The other methods, the reciprocal
# part and the bonded terms run the same arithmetic in both instantiations and are held to bit-identical forces (measured
# exactly 0).  PME direct space, measured on an H100 SXM (80 GB HBM3, 400 W power limit): at most 5.7e-7 (ApoA1; DHFR
# 4.5e-7, water 1.1-1.5e-7), 1.8e-7 on the close-contact ions at alpha 4.4 nm^-1.
FORCES_ONLY_BOUND = 2e-6
# aged list against a freshly built one at the same fp32 positions: the two lists order the atoms differently, so only
# the fp32 summation order differs.  Measured on the same H100: at most 5.7e-6 (the 24k water box at 600 K; DHFR 4.2e-6
# at padding 0.3), the same size as the aged forces' distance from the oracle (up to 7.2e-6).
AGED_BOUND = 1.5e-5
MOLAR_KT = 0.00831446261815324


@pytest.fixture(scope="module")
def mods():
    import os
    from conftest import GOLDEN
    from openmm_b200 import systems, Engine, engine
    from oracle import port
    return systems, Engine, engine, np.load(os.path.join(GOLDEN, "reference_platform.npz")), port


# ---------------------------------------------------------------- system builders (also used by the CPU companion)
def subset(d, keep):
    """d restricted to the atoms `keep` (closed under molecules); every term whose atoms are all kept survives, renumbered."""
    keep = np.asarray(keep)
    new = -np.ones(d.natoms, dtype=np.int64)
    new[keep] = np.arange(len(keep))
    s = copy.copy(d)
    for k in ("masses", "charges", "sigmas", "epsilons", "positions"):
        setattr(s, k, np.asarray(getattr(d, k))[keep])
    for idx, vals in ((("exc_i", "exc_j"), ("exc_qq", "exc_sigma", "exc_eps")), (("bond_i", "bond_j"), ("bond_r0", "bond_k")),
                      (("angle_i", "angle_j", "angle_k"), ("angle_t0", "angle_kk")),
                      (("tor_i", "tor_j", "tor_k", "tor_l"), ("tor_n", "tor_phase", "tor_kk")), (("con_i", "con_j"), ("con_d",))):
        m = np.ones(len(getattr(d, idx[0])), bool)
        for k in idx:
            m &= new[getattr(d, k)] >= 0
        for k in idx:
            setattr(s, k, new[getattr(d, k)][m].astype(np.int32))
        for k in vals:
            setattr(s, k, np.asarray(getattr(d, k))[m])
    return s


def ions_in_box(systems, n, box, cutoff, seed=0, method=None):
    """n +-1 ions on a jittered lattice of the (possibly triclinic) cell `box` (rows a, b, c), as systems.random_ions."""
    rng = np.random.default_rng(seed)
    m = int(np.ceil(n**(1.0/3.0)))
    sites = np.stack(np.meshgrid(*[np.arange(m)]*3, indexing="ij"), -1).reshape(-1, 3)
    sites = sites[rng.permutation(len(sites))[:n]]
    frac = (sites + 0.5 + 0.5*(rng.random((n, 3)) - 0.5))/m
    q = np.where(np.arange(n) % 2 == 0, 1.0, -1.0)
    box = np.asarray(box, dtype=float)
    return systems.SystemDesc(masses=np.where(q > 0, 22.99, 35.45), charges=q, sigmas=np.where(q > 0, 0.23, 0.32),
                              epsilons=np.where(q > 0, 0.0115897, 0.4184), positions=frac @ box, box=box,
                              method=systems.NB_PME if method is None else method, cutoff=cutoff, name="ions%d" % n).rounded()


def close_contact_ions(systems):
    """64 +-1 ion pairs 0.15-0.36 nm apart, pair centres on a jittered 0.55 nm lattice (other ions >= 0.19 nm away), PME
    cutoff 0.6 nm so alpha = sqrt(-ln(2*5e-4))/0.6 = 4.4 nm^-1: every close pair of the tile kernel carries an Ewald
    screening term of up to a fifth of its Coulomb force."""
    rng = np.random.default_rng(21)
    m, h = 4, 0.55
    c = (np.stack(np.meshgrid(*[np.arange(m)]*3, indexing="ij"), -1).reshape(-1, 3) + 0.5)*h + 0.02*(rng.random((m**3, 3)) - 0.5)
    u = rng.normal(size=(m**3, 3))
    u /= np.linalg.norm(u, axis=1)[:, None]
    r = rng.uniform(0.15, 0.36, m**3)
    pos = np.empty((2*m**3, 3))
    pos[0::2] = c - 0.5*r[:, None]*u
    pos[1::2] = c + 0.5*r[:, None]*u
    n = len(pos)
    q = np.tile([1.0, -1.0], m**3)
    L = m*h
    return systems.SystemDesc(masses=np.full(n, 20.0), charges=q, sigmas=np.full(n, 0.1), epsilons=np.full(n, 0.1), positions=pos,
                              box=np.diag([L, L, L]), method=systems.NB_PME, cutoff=0.6, name="close_ions").rounded()


def pme_switch_water(systems):
    d = systems.water_box(8, cutoff=0.9).rounded()
    d.use_switch, d.switch_distance = True, 0.75
    return d


def lj_short_switch(systems):
    """Cutoff-periodic LJ fluid switched from 0.3 nm: every close pair (< 0.36 nm) of the tile kernel is inside the switch."""
    d = systems.lj_fluid(8, cutoff=1.0).rounded()
    d.use_switch, d.switch_distance = True, 0.3
    return d


TRICLINIC_LIMITS = {"pmp": (1.5, -1.5, 1.5), "mpm": (-1.5, 1.5, -1.5)}


def triclinic_limit_box(sign):
    """a = 3, b.x = +-a/2, c.x = -+a/2, c.y = +-b/2: the edges of OpenMM's reduced form."""
    bx, cx, cy = TRICLINIC_LIMITS[sign]
    return np.array([[3.0, 0, 0], [bx, 3.0, 0], [cx, cy, 3.0]])


def cell_widths(box):
    """Distances between opposite faces of the cell."""
    a, b, c = box
    v = abs(np.dot(a, np.cross(b, c)))
    return np.array([v/np.linalg.norm(np.cross(b, c)), v/np.linalg.norm(np.cross(c, a)), v/np.linalg.norm(np.cross(a, b))])


def triclinic_limit_ions(systems, sign):
    box = triclinic_limit_box(sign)
    rc = 0.49*cell_widths(box).min()            # 1.09 nm: close to half the smallest width (2.23 nm)
    return ions_in_box(systems, 300, box, round(rc, 2), seed=8)


def overflow_cluster(systems):
    """48 weakly charged (+-0.05 e), small-sigma atoms on a jittered 4x4x3 lattice of 0.06 nm inside a 0.2 nm cube
    (diagonal 0.346 nm < 0.36 nm): all 496 pairs of the first 32-atom block are close pairs of ONE tile, far more than
    the 96 the per-warp queue takes (CLOSE_QCAP); the rest stay on the fp32 path."""
    rng = np.random.default_rng(4)
    g = np.stack(np.meshgrid(np.arange(4), np.arange(4), np.arange(3), indexing="ij"), -1).reshape(-1, 3)
    pos = 0.01 + (g + 0.5)*0.06 - 0.02 + 0.02*rng.random(g.shape)
    n = len(pos)
    q = np.where(np.arange(n) % 2 == 0, 0.05, -0.05)
    return systems.SystemDesc(masses=np.full(n, 12.0), charges=q, sigmas=np.full(n, 0.02), epsilons=np.full(n, 0.1), positions=pos,
                              box=None, method=systems.NB_CUTOFF_NONPERIODIC, cutoff=1.0, name="overflow48").rounded()


def water_slab(systems):
    """A 3.73 nm water box with the waters of the upper half of the box removed."""
    d = systems.water_box(12, cutoff=0.9)
    L = d.box[2][2]
    keep_w = np.nonzero(d.positions[0::3, 2] < 0.5*L)[0]
    return subset(d, (3*keep_w[:, None] + np.arange(3)).reshape(-1)).rounded()


def dense_cluster(systems):
    """A 648-atom water droplet (1.86 nm cube at water density) alone in a 5 nm PME box."""
    d = systems.water_box(6, cutoff=0.9)
    d.box = np.diag([5.0, 5.0, 5.0])
    d.positions = d.positions + 1.0
    return d.rounded()


def far_and_neutral_water(systems):
    """PME water with zero-charge waters, zero-epsilon oxygens (the hydrogens have epsilon 0 anyway), and every third water
    moved by 2-4 lattice vectors per axis (positions stay fp32-representable)."""
    d = systems.water_box(7, cutoff=0.9)
    nw = d.natoms//3
    rng = np.random.default_rng(9)
    d.charges = d.charges.copy()
    d.epsilons = d.epsilons.copy()
    for w in range(0, nw, 4):
        d.charges[3*w:3*w+3] = 0.0
    d.epsilons[0::15] = 0.0
    k = rng.choice([-4, -3, -2, 2, 3, 4], size=(nw, 3))*(np.arange(nw) % 3 == 0)[:, None]
    d.positions = d.positions + np.repeat(k @ d.box, 3, axis=0)
    return d.rounded()


ODD_GRIDS = [(25, 27, 33), (27, 40, 21), (22, 26, 28)]
ODD_BOX = (3.1, 3.7, 4.3)
ODD_ALPHA = 4.0


def odd_grid_ions(systems, grid):
    """600 ions in a 3.1 x 3.7 x 4.3 nm box, PME with alpha 4.0 nm^-1 on an explicit grid.  The large alpha puts weight on
    the highest frequencies (the kz = nz/2 plane of an even nz included)."""
    d = ions_in_box(systems, 600, np.diag(ODD_BOX), 1.0, seed=13)
    d.pme_alpha, d.pme_grid = ODD_ALPHA, tuple(grid)
    return d


def shift_box_pair(systems):
    """(off, on): the same water lattice (0.3107 nm spacing) in a box too small and a box large enough for the single-image
    SHIFT mode of the tile kernel (nonbonded.cu k_pair: 0.5*minL - rc - padding >= max block half extent)."""
    return systems.water_box(6, cutoff=0.9).rounded(), systems.water_box(16, cutoff=0.9).rounded()


# ---------------------------------------------------------------- helpers
def _oracle(port, d, positions=None):
    f, e, _ = port.forces_energy(d, positions=positions)
    return f, e


def _cutoff_edge_atoms(d, x, eps=2e-7):
    """Atoms of pairs whose distance lies within eps of the cutoff (orthorhombic periodic boxes).  The fp32 tile kernel
    and the double oracle may classify such a pair differently -- a 0.1 kJ/mol/nm difference for one O-H pair at 0.9 nm
    (measured: a pair at 0.8999999961 nm in the 16^3 water box).  The seeded 16^3 and 20^3 water boxes have two and one
    pairs that close to the cutoff, so these atoms are left out of the force comparison."""
    from scipy.spatial import cKDTree
    from openmm_b200 import systems
    if d.box is None or d.method not in (systems.NB_CUTOFF_PERIODIC, systems.NB_PME) or np.count_nonzero(d.box - np.diag(np.diag(d.box))):
        return np.zeros(0, dtype=np.int64)
    L = np.diag(d.box)
    t = cKDTree(np.mod(x, L), boxsize=L)
    edge = t.query_pairs(d.cutoff + eps, output_type="ndarray")
    if len(edge) == 0:
        return np.zeros(0, dtype=np.int64)
    dd = x[edge[:, 1]] - x[edge[:, 0]]
    r = np.linalg.norm(dd - L*np.round(dd/L), axis=1)
    return np.unique(edge[np.abs(r - d.cutoff) < eps].reshape(-1))


def _force_error(d, x, f, fo):
    """relative_force_error over the atoms that are not in a pair at the cutoff (at most a few)."""
    skip = _cutoff_edge_atoms(d, x)
    assert len(skip) <= max(16, d.natoms//1000)
    keep = np.setdiff1d(np.arange(d.natoms), skip)
    return relative_force_error(f[keep], fo[keep])


def _energy_close(e, er, tol=ETOL):
    return abs(e - er)/max(1.0, abs(er)) < tol


def _both(Engine, d, **kw):
    """(forces-only forces, energy-path forces, energy) of one engine."""
    eng = Engine(d, **kw)
    eng.compute(energy=False)
    f0 = eng.get_forces()
    e = eng.compute()
    f1 = eng.get_forces()
    assert eng.stats()["overflow"] == 0
    return f0, f1, e, eng


def _against_oracle(mods, d, tol=TOL, etol=ETOL):
    systems, Engine, _, _, port = mods
    f0, f1, e, eng = _both(Engine, d)
    # the state the engine holds: a molecule more than a box length away is moved back by whole lattice vectors in fp32
    x = eng.get_positions()
    fo, eo = _oracle(port, d, x)
    err0, err1 = _force_error(d, x, f0, fo), _force_error(d, x, f1, fo)
    print("%s: forces-only %.2e, energy path %.2e, energy %.2e" % (d.name, err0, err1, abs(e - eo)/max(1.0, abs(eo))))
    assert err0 < tol, err0
    assert err1 < tol, err1
    assert _energy_close(e, eo, etol), (e, eo)
    return f0, f1, e, eng


# ---------------------------------------------------------------- 1. forces-only parity
def _reference_case_names():
    return ["nocutoff_cluster", "cutoff_nonperiodic", "cutoff_periodic_lj", "reaction_field", "pme_water_rigid", "pme_water_flexible",
            "pme_ions_cubic", "pme_ions_triclinic", "water24k", "switch_dispersion", "pme_grid_radix_11", "exceptions_14_torsions",
            "dhfr", "apoa1"]


@pytest.mark.parametrize("name", _reference_case_names())
def test_forces_only_matches_reference_platform(mods, name):
    """compute(energy=False) -- the instantiations the step graph runs -- against the Reference platform's forces, at the
    tolerance of the energy path; and term class by term class against compute(energy=True) on the same engine."""
    from test_gpu_parity import reference_cases
    systems, Engine, engine, ref, _ = mods
    d = reference_cases(systems)[name]
    idx = ref[name + ":idx"]
    assert abs(d.positions.sum() - float(ref[name + ":xsum"])) < 1e-9*d.natoms
    eng = Engine(d)
    eng.compute(energy=False)
    assert relative_force_error(eng.get_forces()[idx], ref[name + ":f"]) < TOL
    classes = {"direct": engine.TERM_NB_DIRECT}
    if d.method == systems.NB_PME:
        classes["reciprocal"] = engine.TERM_NB_RECIP
    if len(d.bond_i) + len(d.angle_i) + len(d.tor_i):
        classes["bonded"] = engine.TERM_BONDS | engine.TERM_ANGLES | engine.TERM_TORSIONS
    for cls, terms in classes.items():
        eng.compute(terms, energy=False)
        f0 = eng.get_forces()
        eng.compute(terms)
        err = relative_force_error(f0, eng.get_forces())
        print("%s %s: forces-only vs energy path %.2e" % (name, cls, err))
        if cls == "direct" and d.method == systems.NB_PME:
            assert err < FORCES_ONLY_BOUND, (cls, err)
        else:
            assert err == 0.0, (cls, err)           # same arithmetic in both instantiations: measured bit-identical
    assert eng.stats()["overflow"] == 0


def test_forces_only_close_contact_ions(mods):
    """The close pairs of the forces-only PME kernel evaluate the Ewald screening with the fp32 fit ewald_g: at alpha 4.4
    nm^-1 and 0.15-0.36 nm that term is large, so an error of the fit shows against the oracle and the energy path."""
    systems, Engine, _, _, port = mods
    d = close_contact_ions(systems)
    assert abs(d.pme_parameters()[0] - 4.38) < 0.01
    f0, f1, e, _ = _against_oracle(mods, d)
    err = relative_force_error(f0, f1)
    print("close_contact_ions: forces-only vs energy path %.2e" % err)
    assert err < FORCES_ONLY_BOUND, err


# ---------------------------------------------------------------- 2. aged neighbour list
def _thermal_velocities(d, T, seed):
    rng = np.random.default_rng(seed)
    return rng.standard_normal((d.natoms, 3))*np.sqrt(MOLAR_KT*T/np.asarray(d.masses))[:, None]


def _exclusion_pairs(d):
    if len(d.exc_i) == 0:
        return np.zeros((0, 2), dtype=np.int64)
    return np.unique(np.sort(np.stack([d.exc_i, d.exc_j], 1).astype(np.int64), axis=1), axis=0)


def _pair_count_bounds(d, x, excl, eps=1e-6):
    """(lo, hi) for stats()["pairs_in_cutoff"], the number of non-excluded pairs inside the cutoff that the current list
    evaluates (k_count_pairs, from the per-step refreshed sorted positions).  A valid list holds every pair closer than
    rc - eps; a pair within eps of the cutoff may go either way in fp32 (the fp32 box length alone is 2e-7 nm off at
    6 nm).  Orthorhombic periodic boxes."""
    from scipy.spatial import cKDTree
    L = np.diag(d.box)
    y = np.mod(x, L)
    y[y >= L] = 0.0
    t = cKDTree(y, boxsize=L)
    n = (t.count_neighbors(t, np.array([d.cutoff - eps, d.cutoff + eps])) - d.natoms)//2
    dd = x[excl[:, 1]] - x[excl[:, 0]]
    r = np.linalg.norm(dd - L*np.round(dd/L), axis=1)
    return int(n[0] - np.count_nonzero(r < d.cutoff - eps)), int(n[1] - np.count_nonzero(r < d.cutoff + eps))


def _age(eng, d, nsteps, count_every_step, precision):
    """Step one step at a time, with a compute() after each (it runs the same displacement check the next step would,
    at the same positions).  Whenever that compute did not rebuild the list -- the list is aged, up to the state just
    before its next rebuild -- and count_every_step is set, the pairs the list evaluates are counted against an exact
    count of the pairs inside the cutoff: a rebuild that comes too late loses pairs that have just crossed into the
    cutoff.  Stops at the first aged state after nsteps steps whose last step did not rebuild either, so that the
    forces of that compute() are those of the aged list.  Returns (steps, list builds, aged states counted)."""
    excl = _exclusion_pairs(d)
    steps = counted = 0
    while steps < nsteps + 100:
        b0 = eng.stats()["list_builds"]
        eng.step(1)
        steps += 1
        b1 = eng.stats()["list_builds"]
        eng.compute(energy=False)
        st = eng.stats()
        aged = st["list_builds"] == b1
        last = steps >= nsteps and aged and b1 == b0
        if aged and (count_every_step or last):
            x = eng.get_positions()
            if precision == "mixed":
                x = x.astype(np.float32).astype(np.float64)        # the pair kernel reads the fp32 hi part
            lo, hi = _pair_count_bounds(d, x, excl)
            assert lo <= st["pairs_in_cutoff"] <= hi, ("pairs inside the cutoff missing from the aged list", steps, st["pairs_in_cutoff"], lo, hi)
            counted += 1
        if last:
            return steps, st["list_builds"], counted
    pytest.fail("no aged state within %d steps" % steps)


def _inner_positions(eng, natoms):
    """The engine's internal (wrapped) fp32 coordinates, from a single-precision checkpoint blob: header (112 bytes, magic
    B200MDCK, version 2) | posq | velm | cellOffset (engine.cu, b200md_checkpoint_save)."""
    npad = eng.stats()["padded_atoms"]
    blob = eng.checkpoint()
    hdr = 112
    assert eng.precision == "single" and blob[:8] == b"B200MDCK"
    assert int.from_bytes(blob[8:12], "little") == 2 and int.from_bytes(blob[12:16], "little") == natoms
    assert len(blob) == hdr + 2*16*npad + 3*4*npad
    return np.frombuffer(blob, dtype=np.float32, count=4*npad, offset=hdr).reshape(npad, 4)[:natoms, :3].astype(np.float64)


def _aged_check(mods, d, T=300.0, nsteps=40, dt=0.002, precision="single", shift_molecules=False, seed=1, count_every_step=False):
    systems, Engine, _, _, port = mods
    eng = Engine(d, precision=precision)
    eng.set_integrator(systems.INT_LANGEVIN, dt, T, 1.0, seed)
    eng.set_velocities(_thermal_velocities(d, T, seed))
    eng.apply_velocity_constraints()
    if shift_molecules:
        # whole molecules moved by 2-3 lattice vectors per axis: the next list build wraps them back (wrap_molecule)
        eng.step(10)
        x = eng.get_positions()
        rng = np.random.default_rng(seed)
        mols = d.molecules()
        k = rng.choice([-3, -2, 2, 3], size=(len(mols), 3))*(rng.random(len(mols)) < 0.5)[:, None]
        for m, km in zip(mols, k):
            x[m] += km @ d.box
        eng.set_positions(x)
    steps, builds, counted = _age(eng, d, nsteps, count_every_step, precision)
    f = eng.get_forces()
    x = eng.get_positions()
    # mixed precision: the forces come from the fp32 hi part of the positions
    xo = x.astype(np.float32).astype(np.float64) if precision == "mixed" else x
    fo, _ = _oracle(port, d, xo)
    err_oracle = _force_error(d, x, f, fo)
    fresh_d = copy.copy(d)
    fresh_d.positions = _inner_positions(eng, d.natoms) if shift_molecules else x
    fresh = Engine(fresh_d, precision=precision)
    fresh.compute(energy=False)
    err_fresh = relative_force_error(f, fresh.get_forces())
    print("%s T=%g %s shift=%s: %d steps, %d list builds, %d aged states counted; oracle %.2e, fresh list %.2e"
          % (d.name, T, precision, shift_molecules, steps, builds, counted, err_oracle, err_fresh))
    assert np.isfinite(x).all() and eng.stats()["overflow"] == 0
    assert err_oracle < TOL, err_oracle
    assert err_fresh < AGED_BOUND, err_fresh
    return {"steps": steps, "list_builds": builds, "aged_states_counted": counted, "oracle": err_oracle, "fresh_list": err_fresh}


def _record(record_property, res):
    for k, v in res.items():
        record_property(k, v)


def _system(mods, name):
    import os
    from conftest import ROOT
    systems = mods[0]
    if name == "dhfr":
        return systems.SystemDesc.load(os.path.join(ROOT, "data", "dhfr.npz")).rounded()
    return systems.water_box(20, cutoff=0.9).rounded()


@pytest.mark.parametrize("pad", ["0.02", None, "0.3"])
@pytest.mark.parametrize("name", ["dhfr", "water24k"])
def test_aged_list_matches_oracle(mods, monkeypatch, record_property, name, pad):
    """Langevin at 300 K with B200MD_PAD_FRACTION 0.02, the default (0.1) and 0.3: forces on the list as it stands after
    the run (not rebuilt on the last step) against the oracle and against a freshly built list.  At 0.02 the list is
    rebuilt every few steps, and the pairs it evaluates are counted in every aged state of an 80-step run: a rebuild that
    comes late drops pairs that have just crossed into the cutoff."""
    if pad is not None:
        monkeypatch.setenv("B200MD_PAD_FRACTION", pad)
    # at 0.02 (half padding 0.009 nm) the fastest hydrogen crosses half the padding in one 2 fs step: 0.5 fs steps let the
    # list live a few steps
    tight = pad == "0.02"
    res = _aged_check(mods, _system(mods, name), nsteps=80 if tight else 40, dt=0.0005 if tight else 0.002, count_every_step=tight)
    _record(record_property, res)
    if tight:
        assert res["list_builds"] > 5 and res["aged_states_counted"] > 20     # the check fired, and most states were aged
    assert res["list_builds"] < res["steps"]


def test_aged_list_hot(mods, record_property):
    _record(record_property, _aged_check(mods, _system(mods, "water24k"), T=600.0, seed=3))


def test_aged_list_mixed_precision(mods, record_property):
    _record(record_property, _aged_check(mods, _system(mods, "dhfr"), precision="mixed", seed=5))


def test_aged_list_after_molecules_moved_by_lattice_vectors(mods, record_property):
    _record(record_property, _aged_check(mods, _system(mods, "water24k"), shift_molecules=True, seed=7))


def approaching_blocks(systems, step=0.0005, margin=0.00025):
    """Two 32-atom blocks (4 x 4 x 2 lattices of 0.1 nm, atoms 0-31 and 32-63: a non-periodic system keeps the identity
    order) whose facing layers start rc + padding + margin apart (cutoff 0.9 nm, default padding 0.09 nm), so the list
    built at the start has no tile between them.  Neutral, epsilon 0: no forces, and with velocities +-step/dt along x
    every atom moves exactly `step` per Verlet step."""
    rc, pad = 0.9, 0.09
    g = np.stack(np.meshgrid(np.arange(2), np.arange(4), np.arange(4), indexing="ij"), -1).reshape(-1, 3)*0.1
    gap = rc + pad + margin
    pos = np.concatenate([g, g + np.array([0.1 + gap, 0.0, 0.0])])
    n = len(pos)
    d = systems.SystemDesc(masses=np.ones(n), charges=np.zeros(n), sigmas=np.full(n, 0.3), epsilons=np.zeros(n), positions=pos,
                           box=None, method=systems.NB_CUTOFF_NONPERIODIC, cutoff=rc, name="approaching_blocks").rounded()
    return d, gap


def test_rebuild_comes_before_a_pair_enters_the_cutoff(mods):
    """The list is rebuilt once an atom has moved half the padding (k_check_gather): two atoms that approach each other
    head on can then not have closed more than the padding.  Two blocks approach at 2 x 0.5 pm per step from 0.25 pm
    outside the padded cutoff, so their facing pairs cross the cutoff at step 91, and the check fires at step 90 or 91
    (every atom has moved 0.045 nm = padding/2 at step 90).  Every step, the pairs the list evaluates are counted against
    the exact count: a check that fired later (say at a full padding) would leave the crossing pairs out of the list for
    90 steps."""
    systems, Engine, _, _, _ = mods
    d, gap = approaching_blocks(systems)
    dt, step = 0.001, 0.0005
    eng = Engine(d)
    eng.set_integrator(systems.INT_VERLET, dt, 0.0, 0.0, 0)
    v = np.zeros((d.natoms, 3))
    v[:32, 0], v[32:, 0] = step/dt, -step/dt
    eng.set_velocities(v)
    eng.compute(energy=False)
    st = eng.stats()
    assert st["num_tiles"] == 2 and st["pairs_in_cutoff"] == 2*(32*31//2)      # no tile between the two blocks yet
    builds0, crossed = st["list_builds"], 0
    for k in range(1, 131):
        eng.step(1)
        eng.compute(energy=False)
        x = eng.get_positions()
        r = np.linalg.norm(x[:, None] - x[None], axis=-1)[np.triu_indices(d.natoms, 1)]
        st = eng.stats()
        assert st["pairs_in_cutoff"] == np.count_nonzero(r < d.cutoff), (k, st["pairs_in_cutoff"], np.count_nonzero(r < d.cutoff))
        crossed = max(crossed, np.count_nonzero(r < d.cutoff) - 2*(32*31//2))
    assert np.abs(eng.get_forces()).max() == 0.0
    assert crossed >= 16 and st["list_builds"] > builds0                        # pairs did cross; the list was rebuilt


# ---------------------------------------------------------------- 3. shapes and edges
@pytest.mark.parametrize("n", [2, 31, 32, 33, 63, 65, 97])
def test_ion_boxes_with_partial_blocks(mods, n):
    """N that leaves the last 32-atom block partly empty (padding atoms: sorig = -1, jidx < 0, charge 0), in a cubic PME box
    just above twice the cutoff (1.0 nm)."""
    systems = mods[0]
    _against_oracle(mods, ions_in_box(systems, n, np.diag([2.05]*3), 1.0, seed=n))


@pytest.mark.parametrize("which", ["off", "on"])
def test_shift_mode_forced_off_and_on(mods, which):
    """The same water lattice with and without the single-image SHIFT mode.  The tile kernel takes it when
    0.5*minL - rc - padding >= maxHalf (padding = 0.1*rc = 0.09 nm by default, maxHalf = the largest 32-atom block half
    extent, > 0).  Off: 6^3 waters, L = 1.8642 nm, 0.5*L - 0.9 - 0.09 = -0.058 < 0 whatever maxHalf is.  On: 16^3 waters,
    L = 4.9712 nm, margin 1.496 nm, more than any block of water at this density spans (a 32-atom block is ~0.32 nm^3).
    Neither box tests the padding term of the margin: that needs 0.5*L - rc between maxHalf and maxHalf + padding, and
    maxHalf is known only on the device.  Even in such a box, a margin without the term picks a wrong image only for a
    pair whose atoms have moved, since the build, far enough past their blocks' recorded extents to reach half a box from
    the block centre.  Dropping the term therefore passes every test here."""
    systems = mods[0]
    off, on = shift_box_pair(systems)
    _against_oracle(mods, off if which == "off" else on)


def test_pme_with_switching_function(mods):
    _against_oracle(mods, pme_switch_water(mods[0]))


def test_switched_close_pairs(mods):
    _against_oracle(mods, lj_short_switch(mods[0]))


@pytest.mark.parametrize("name", ["reaction_field", "cutoff_nonperiodic", "nocutoff_cluster"])
def test_non_pme_methods_forces_only(mods, name):
    from test_gpu_parity import reference_cases
    _against_oracle(mods, reference_cases(mods[0])[name])


@pytest.mark.parametrize("sign", sorted(TRICLINIC_LIMITS))
def test_triclinic_reduced_form_limits(mods, sign):
    _against_oracle(mods, triclinic_limit_ions(mods[0], sign))


def test_close_pair_queue_overflow(mods, monkeypatch):
    """~500 close pairs in one tile: the first 96 go through the double-precision queue, the rest stay in the fp32 loop.
    No pair may be lost or counted twice: the energy equals that of a run with the close-pair path switched off
    (B200MD_CLOSE_NM=0, every pair in fp32)."""
    systems, Engine, _, _, _ = mods
    d = overflow_cluster(systems)
    f0, f1, e, _ = _against_oracle(mods, d)
    monkeypatch.setenv("B200MD_CLOSE_NM", "0")
    g0, g1, e_fp32, _ = _both(Engine, d)
    print("overflow48: energy %.9g, fp32-only %.9g" % (e, e_fp32))
    assert _energy_close(e, e_fp32), (e, e_fp32)
    assert relative_force_error(f0, g0) < TOL


@pytest.mark.parametrize("name", ["slab", "cluster"])
def test_inhomogeneous_density(mods, name):
    systems = mods[0]
    _against_oracle(mods, water_slab(systems) if name == "slab" else dense_cluster(systems))


def test_zero_parameters_and_far_molecules(mods):
    _against_oracle(mods, far_and_neutral_water(mods[0]))


# ---------------------------------------------------------------- 4. PME on odd and anisotropic grids
@pytest.mark.parametrize("noslab", [False, True])
@pytest.mark.parametrize("grid", ODD_GRIDS)
def test_pme_odd_grids_reciprocal(mods, monkeypatch, grid, noslab):
    """Reciprocal space alone (TERM_NB_RECIP) against orc_pme_reciprocal + orc_self_energy on the same alpha and grid, with
    the slab FFT and (B200MD_FFT_NOSLAB) the line-batched one: odd nz has no Nyquist plane in the Hermitian weights of
    k_fft_x_conv, even nz has one."""
    systems, Engine, engine, _, port = mods
    if noslab:
        monkeypatch.setenv("B200MD_FFT_NOSLAB", "1")
    d = odd_grid_ions(systems, grid)
    eng = Engine(d)
    assert eng.stats()["pme_grid"] == list(grid)
    eng.compute(engine.TERM_NB_RECIP, energy=False)
    f0 = eng.get_forces()
    e = eng.compute(engine.TERM_NB_RECIP)
    f1 = eng.get_forces()
    L = port.lib()
    pos, q, box = port._d(d.positions), port._d(d.charges), port._d(d.box).reshape(9)
    fo = np.zeros((d.natoms, 3))
    eo = L.orc_pme_reciprocal(d.natoms, port._dp(pos), port._dp(q), port._dp(box), ODD_ALPHA, grid[0], grid[1], grid[2], port._dp(fo))
    eo += L.orc_self_energy(d.natoms, port._dp(q), ODD_ALPHA)
    err0, err1 = relative_force_error(f0, fo), relative_force_error(f1, fo)
    print("grid %s noslab=%s: forces-only %.2e, energy path %.2e, energy %.2e" % (grid, noslab, err0, err1, abs(e - eo)/abs(eo)))
    assert err0 < TOL and err1 < TOL, (err0, err1)
    assert abs(e - eo)/abs(eo) < ETOL, (e, eo)
