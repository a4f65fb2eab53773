"""The Langevin random force, on the CPU: the restated generator (orc_philox4x32_10 / orc_gauss3 in oracle/md_oracle.c, the
engine's engine.h philox / gauss3 in plain C) against the published Philox4x32-10 known answers and for the statistics of
its normals, and the oracle's stochastic step (orc_langevin_step) against its zero-temperature form, its constraint
tolerance and -- where oracle/_ref holds the reference -- the velocity distribution the Reference platform produces."""
import numpy as np
import pytest
from scipy import stats
from openmm_b200 import systems
from oracle import port

SEED = 20240611
KT300 = port.BOLTZ*300.0


def test_philox_known_answers():
    """The three Random123 known-answer vectors of philox4x32-10 (kat_vectors: zero counter and key; all ones; the pi
    digits)."""
    kat = [(([0, 0, 0, 0], [0, 0]), [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]),
           (([0xffffffff]*4, [0xffffffff]*2), [0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd]),
           (([0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344], [0xa4093822, 0x299f31d0]), [0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1])]
    for (ctr, key), want in kat:
        assert port.philox4x32_10(ctr, key).tolist() == want


def test_gauss3_is_the_keyed_philox_stream():
    """gauss3(seed, atom, step) is the Box-Muller transform of Philox on counter (atom, step_lo, step_hi, 0x5eed5eed) and key
    (seed, 0xb200b200), with 24-bit uniforms formed as the engine forms them."""
    for seed, atom, step in ((7, 0, 0), (1, 12345, 2**32 + 17), (0xffffffff, 999, 2**40 - 1)):
        r = port.philox4x32_10([atom, step & 0xffffffff, step >> 32, 0x5eed5eed], [seed, 0xb200b200]).astype(np.float64)
        u1, u2 = (np.floor(r[0]/256) + 1)/2**24, np.floor(r[1]/256)/2**24
        u3, u4 = (np.floor(r[2]/256) + 1)/2**24, np.floor(r[3]/256)/2**24
        m1, m2 = np.sqrt(-2*np.log(u1)), np.sqrt(-2*np.log(u3))
        want = [m1*np.cos(2*np.pi*u2), m1*np.sin(2*np.pi*u2), m2*np.cos(2*np.pi*u4)]
        assert np.allclose(port.gauss3(seed, [atom], step)[0], want, rtol=1e-14, atol=1e-14)
    assert np.array_equal(port.gauss3(-1, [3], 5), port.gauss3(0xffffffff, [3], 5))     # the seed is taken as unsigned


@pytest.fixture(scope="module")
def draws():
    """20,000 atoms x 50 steps of one fixed seed: [steps, atoms, 3]."""
    atoms = np.arange(20000)
    return np.stack([port.gauss3(SEED, atoms, s) for s in range(50)])


def _corr(a, b):
    return float(np.corrcoef(a.ravel(), b.ravel())[0, 1])


def test_generator_moments_and_distribution(draws):
    """Per component: mean 0 and variance 1 within 5 standard errors of 10^6 samples, and a KS test against N(0,1)."""
    n = draws.shape[0]*draws.shape[1]
    for c in range(3):
        g = draws[..., c].ravel()
        assert abs(g.mean()) < 5/np.sqrt(n)
        assert abs(g.var() - 1) < 5*np.sqrt(2.0/n)
        assert stats.kstest(g, "norm").pvalue > 0.01
    assert np.abs(draws).max() < 6.5


def test_generator_correlations(draws):
    """No correlation between components, neighbouring atoms, consecutive steps or consecutive seeds (|r| within 5 standard
    errors, 5e-3 at 10^6 samples)."""
    lim = 5e-3
    for a, b in ((0, 1), (0, 2), (1, 2)):
        assert abs(_corr(draws[..., a], draws[..., b])) < lim
    assert abs(_corr(draws[:, :-1], draws[:, 1:])) < lim
    assert abs(_corr(draws[:-1], draws[1:])) < lim
    atoms = np.arange(20000)
    other = np.stack([port.gauss3(SEED + 1, atoms, s) for s in range(5)])
    assert abs(_corr(draws[:5], other)) < 2*lim


def test_high_word_of_the_step_counter_is_used():
    """Steps 2^32 - 1 and 2^32 give unrelated draws, and so do steps 0 and 2^32, which differ only in the counter's high
    word."""
    atoms = np.arange(20000)
    lo = port.gauss3(SEED, atoms, 2**32 - 1)
    hi = port.gauss3(SEED, atoms, 2**32)
    zero = port.gauss3(SEED, atoms, 0)
    lim = 5/np.sqrt(lo.size)
    assert abs(_corr(lo, hi)) < lim and abs(_corr(zero, hi)) < lim
    assert not np.any(hi == zero)


# ---- the oracle's stochastic step ----
def _network_system():
    from test_gpu_integrate_lanes import mixed_units_system
    return with_general_networks(mixed_units_system())


def with_general_networks(d):
    """d with two general constraint networks made out of its X-H_n clusters (neither SETTLE nor SHAKE can take them): the
    first CH3 centre gets a fourth partner, the nearest sodium ion (a CH4-like centre), and the first CH2 and the first CH are
    joined into an H-C-C-H2 chain by a C-C constraint; both new constraints at the current distance."""
    import copy
    d = copy.copy(d)
    deg = np.bincount(np.concatenate([d.con_i, d.con_j]), minlength=d.natoms)
    by_n = {}
    for c in np.flatnonzero(d.masses == 12.011):
        by_n.setdefault(int(deg[c]), int(c))
    x = d.positions
    ions = np.flatnonzero(d.masses == 22.99)
    ion = int(ions[np.argmin(np.linalg.norm(x[ions] - x[by_n[3]], axis=1))])
    add = [(by_n[3], ion), (by_n[2], by_n[1])]
    d.con_i = np.concatenate([d.con_i, [a for a, _ in add]]).astype(np.int32)
    d.con_j = np.concatenate([d.con_j, [b for _, b in add]]).astype(np.int32)
    d.con_d = np.concatenate([d.con_d, [np.linalg.norm(x[a] - x[b]) for a, b in add]])
    return d


@pytest.mark.parametrize("kind", [0, 1, 2])
def test_langevin_step_without_noise_is_orc_step(kind):
    """orc_step is orc_langevin_step with no random force and SETTLE the only constraints: bit for bit."""
    d = systems.water_box(3, cutoff=0.45).rounded()
    f, _, _ = port.forces_energy(d, pme=d.pme_parameters())
    cl = port.settle_clusters(d)
    v0 = np.random.default_rng(2).standard_normal((d.natoms, 3))*0.3
    xa, va = d.positions.copy(), v0.copy()
    xb, vb = d.positions.copy(), v0.copy()
    port.step(d, kind, 0.002, 5.0, xa, va, f, cl)
    port.langevin_step(d, kind, 0.002, 5.0, 300.0, xb, vb, f, gauss=None)
    assert np.array_equal(xa, xb) and np.array_equal(va, vb)


@pytest.mark.parametrize("kind", [1, 2])
def test_langevin_step_keeps_shake_and_general_constraints(kind):
    """SETTLE waters, X-H_n clusters and the general networks at 300 K and 10/ps: after each step every non-water constraint
    holds to the CCMA tolerance 1e-12 (plus rounding) and every water to SETTLE's rounding."""
    d = _network_system()
    split = port.constraint_split(d)
    assert len(split[1][0]) > 0
    pme = d.pme_parameters()
    x, v = d.positions.copy(), np.zeros((d.natoms, 3))
    settled = np.zeros(d.natoms, bool)
    for a in split[0][:3]:
        settled[a] = True
    water = settled[d.con_i] & settled[d.con_j]
    for s in range(3):
        f, _, _ = port.forces_energy(d, positions=x, pme=pme)
        x0 = x.copy()
        it = port.langevin_step(d, kind, 0.002, 10.0, 300.0, x, v, f, gauss=port.gauss3(SEED, np.arange(d.natoms), s), split=split)
        assert it > 0
        err = np.abs(np.linalg.norm(x[d.con_i] - x[d.con_j], axis=1)/d.con_d - 1)
        assert err[~water].max() < 2e-12 and err[water].max() < 1e-12
        m = d.masses == 0
        assert np.array_equal(x[m], x0[m]) and not v[m].any()
    assert np.abs(v).max() > 0.5          # the atoms did move


def ideal_gas(n=2000, seed=3):
    """n atoms with zero charges and epsilons (forces exactly 0) at random positions in a periodic box; masses of four
    classes and a fifth class of massless atoms, assigned in turn."""
    rng = np.random.default_rng(seed)
    L = 4.0
    classes = np.array([1.008, 12.011, 39.948, 131.29, 0.0])
    return systems.SystemDesc(masses=classes[np.arange(n) % 5], charges=np.zeros(n), sigmas=np.full(n, 0.3), epsilons=np.zeros(n),
                              positions=rng.random((n, 3))*L, box=np.diag([L, L, L]).astype(float), method=systems.NB_CUTOFF_PERIODIC,
                              cutoff=1.0, use_dispersion=False, name="ideal_gas%d" % n)


def assert_gas_variance(d, v, kT, vscale, nsteps):
    """Per massive class: <v^2> = kT/m (1 - vscale^(2n)) within 4 standard errors (3 * class size samples of a centred
    normal); massless atoms have v = 0."""
    for m in np.unique(d.masses):
        sel = d.masses == m
        if m == 0:
            assert not v[sel].any()
            continue
        want = kT/m*(1 - vscale**(2*nsteps))
        got = (v[sel]**2).mean()
        assert abs(got - want) < 4*want*np.sqrt(2.0/v[sel].size), (m, got, want)


@pytest.mark.parametrize("kind", [1, 2])
def test_oracle_and_reference_platform_give_the_analytic_velocity_variance(kind):
    """An ideal gas from v = 0: after n steps each velocity component is N(0, kT/m (1 - vscale^(2n))) for Langevin and
    LangevinMiddle alike.  The oracle with the restated noise and the live Reference platform (its own generator) must both
    give that variance per mass class; massless atoms stay where they are."""
    d = ideal_gas()
    dt, fr, T, nsteps = 0.002, 10.0, 300.0, 20
    vscale = np.exp(-dt*fr)
    x, v = d.positions.copy(), np.zeros((d.natoms, 3))
    zero = np.zeros((d.natoms, 3))
    split = port.constraint_split(d)
    for s in range(nsteps):
        port.langevin_step(d, kind, dt, fr, T, x, v, zero, gauss=port.gauss3(SEED, np.arange(d.natoms), s), split=split)
    assert_gas_variance(d, v, port.BOLTZ*T, vscale, nsteps)
    assert np.array_equal(x[d.masses == 0], d.positions[d.masses == 0])
    from oracle import omm
    if not omm.available():
        pytest.skip("oracle/_ref has no reference build: the Reference platform half needs it")
    sim = omm.Simulation(d, "Reference", integrator=(kind, T, fr, dt), seed=SEED)
    sim.set_velocities(np.zeros((d.natoms, 3)))
    sim.step(nsteps)
    st = sim.state(positions=True, velocities=True)
    assert_gas_variance(d, st["velocities"], port.BOLTZ*T, vscale, nsteps)
    assert np.array_equal(st["positions"][d.masses == 0], d.positions[d.masses == 0])
