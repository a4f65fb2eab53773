"""The Langevin random force on the device, held to the restated generator (oracle port.gauss3 = engine.h gauss3) and the
oracle's stochastic step (port.langevin_step).  The stream contract: the normals of atom a in the step that starts with
counter s are gauss3(seed, a, s), in every kernel and call path, and the counter advances by one per step.

(a) an ideal gas (forces exactly 0) gives v' = vscale v + s_m g per atom and step, so g can be recovered and compared;
(b) the same for every call path that steps the engine and every way the counter is carried or set;
(c) every integration unit kind (SETTLE, SHAKE X-H_n, general CCMA networks, free and massless atoms) against the oracle's
    stochastic step, each tolerance checked to lie 50x below the smallest kick of its case;
(d) 400 graph steps from v = 0 give the analytic velocity variance per mass class."""
import os
import struct
import numpy as np
import pytest
from conftest import ROOT

pytestmark = pytest.mark.gpu

DT, TEMP, FRICTION, SEED = 0.002, 300.0, 10.0, 918273
KT = 0.00831446261815324*TEMP
VSCALE = np.exp(-DT*FRICTION)
KINDS = {"langevin": 1, "langevin_middle": 2}
# g recovered from one step: fp32 velocities and the fp32 Box-Muller of the engine against the double restatement
# (measured on an H100: 2.9e-6 single, 4.0e-7 mixed; a mis-keyed draw is O(1) off)
GTOL = {"single": 1e-5, "mixed": 1e-6}


def gas(n=1000, cm_frequency=0, seed=11):
    """n atoms (not a multiple of 32 or 64) with zero charges and epsilons on randomly chosen, jittered sites of a lattice
    (no close pairs; the tile sort does not keep the user order); masses of four classes in turn and one massless atom."""
    from openmm_b200 import systems
    rng = np.random.default_rng(seed)
    L, side = 3.2, 16
    sites = np.stack(np.meshgrid(*[np.arange(side)]*3, indexing="ij"), -1).reshape(-1, 3)[rng.permutation(side**3)[:n]]
    x = (sites + 0.5 + 0.6*(rng.random((n, 3)) - 0.5))*(L/side)
    m = np.array([1.008, 12.011, 39.948, 131.29])[np.arange(n) % 4]
    m[137] = 0.0
    return systems.SystemDesc(masses=m, charges=np.zeros(n), sigmas=np.full(n, 0.3), epsilons=np.zeros(n),
                              positions=x.astype(np.float32).astype(np.float64), box=np.diag([L, L, L]),
                              method=systems.NB_CUTOFF_PERIODIC, cutoff=1.0, use_dispersion=False, cm_frequency=cm_frequency,
                              name="gas%d" % n)


def thermal(masses, seed=4):
    v = np.random.default_rng(seed).standard_normal((len(masses), 3))*np.sqrt(KT/np.where(masses > 0, masses, 1.0))[:, None]
    v[masses == 0] = 0.0
    return v


def header(eng):
    """(stepCount, rngStep) of the checkpoint: the 112-byte header holds the int64 stepCount at byte 24 and the unsigned
    64-bit rngStep (the noise counter) at byte 104 (engine.cu CkptHeader)."""
    blob = eng.checkpoint()
    assert blob[:8] == b"B200MDCK" and struct.unpack_from("<i", blob, 12)[0] == eng.natoms
    return struct.unpack_from("<q", blob, 24)[0], struct.unpack_from("<Q", blob, 104)[0]


def kick(m):
    """Per-atom noise amplitude s_m = sqrt(kT/m (1 - vscale^2)) (both kinds), 0 for massless atoms."""
    return np.where(m > 0, np.sqrt(KT/np.where(m > 0, m, 1.0)*(1 - VSCALE**2)), 0.0)


def predict(kind, m, x, v, seed, s0, nsteps, step_count=0, cm_frequency=0):
    """The free-gas trajectory the stream contract prescribes: nsteps steps from (x, v) with counters s0, s0+1, ..; the
    centre-of-mass velocity of the massive atoms is removed before each step whose stepCount is a multiple of cm_frequency."""
    x, v = x.copy(), v.copy()
    live = m > 0
    sm = kick(m)[:, None]
    atoms = np.arange(len(m))
    for k in range(nsteps):
        if cm_frequency and (step_count + k) % cm_frequency == 0:
            v[live] -= (m[live, None]*v[live]).sum(axis=0)/m[live].sum()
        g = port().gauss3(seed, atoms, s0 + k)
        if kind == 1:
            v[live] = VSCALE*v[live] + sm[live]*g[live]
            x[live] += v[live]*DT
        else:
            x[live] += 0.5*DT*v[live]
            v[live] = VSCALE*v[live] + sm[live]*g[live]
            x[live] += 0.5*DT*v[live]
    return x, v


def port():
    from oracle import port as p
    return p


class Stream:
    """An engine on the gas, and the checks that each way of stepping it draws the prescribed normals."""

    def __init__(self, kind, precision="single", seed=SEED, cm_frequency=0):
        from openmm_b200 import Engine
        self.kind, self.precision, self.seed, self.cm = kind, precision, seed, cm_frequency
        self.d = gas(cm_frequency=cm_frequency)
        self.m = self.d.masses
        self.eng = Engine(self.d, precision=precision)
        self.eng.set_integrator(kind, DT, TEMP, FRICTION, seed, 1e-6)
        self.eng.set_velocities(thermal(self.m))

    def check(self, action, nsteps, expect_counter=None):
        """Run action (nsteps steps) and compare positions and velocities with predict(); returns the counter after."""
        eng = self.eng
        count, s0 = header(eng)
        if expect_counter is not None:
            assert s0 == expect_counter
        x0, v0 = eng.get_positions(), eng.get_velocities()
        action()
        x1, v1 = eng.get_positions(), eng.get_velocities()
        xp, vp = predict(self.kind, self.m, x0, v0, self.seed, s0, nsteps, count, self.cm)
        live = self.m > 0
        # velocities in units of the atom's kick: a draw of the wrong atom, step, seed or component is O(1) off
        err = float((np.abs(v1 - vp)[live]/kick(self.m)[live, None]).max())
        assert err < GTOL[self.precision]*nsteps, (err, nsteps)
        assert np.abs(x1 - xp).max() < (2e-6 if self.precision == "single" else 1e-9)*nsteps
        assert np.array_equal(x1[~live], x0[~live]) and not v1[~live].any()
        count1, s1 = header(eng)
        assert s1 == s0 + nsteps and count1 == count + nsteps
        return s1


# ---- (a) ----
@pytest.mark.parametrize("precision", ["single", "mixed"])
@pytest.mark.parametrize("kind", list(KINDS))
def test_noise_recovered_from_free_atoms(kind, precision):
    """Every atom's g recovered from v' = vscale v + s_m g equals gauss3(seed, user atom, counter), step by step."""
    st = Stream(KINDS[kind], precision)
    eng, m = st.eng, st.m
    live = m > 0
    sm = kick(m)[:, None]
    worst = 0.0
    for k in range(6):
        count, s = header(eng)
        assert count == k and s == k
        x0, v0 = eng.get_positions(), eng.get_velocities()
        eng.step(1)
        x1, v1 = eng.get_positions(), eng.get_velocities()
        g = (v1[live] - VSCALE*v0[live])/sm[live]
        want = port().gauss3(SEED, np.flatnonzero(live), s)
        worst = max(worst, float(np.abs(g - want).max()))
        assert np.abs(g - want).max() < GTOL[precision]
        assert np.array_equal(x1[~live], x0[~live]) and not v1[~live].any()
    print("noise %s %s: max |g - gauss3| = %.2e" % (kind, precision, worst))


# ---- (b) ----
@pytest.mark.parametrize("kind", list(KINDS))
def test_one_stream_whatever_the_call_path(kind):
    """step(1) xN, step(16) (two replays of the 8-step graph), compute + b200md_integrate_only, set_integrator again
    mid-run, checkpoint -> load, and a counter patched to 2^32 - 2 stepped across the high word: one stream, no gap, no
    reuse."""
    st = Stream(KINDS[kind])
    eng = st.eng
    s = 0
    for _ in range(3):
        s = st.check(lambda: eng.step(1), 1, s)
    s = st.check(lambda: eng.step(16), 16, s)

    def two_call():
        eng.compute(energy=False)
        eng._ck(eng.lib.b200md_integrate_only(eng.h))
    for _ in range(2):
        s = st.check(two_call, 1, s)
    eng.set_integrator(KINDS[kind], DT, TEMP, FRICTION, SEED, 1e-6)
    s = st.check(lambda: eng.step(1), 1, s)
    blob = eng.checkpoint()
    s_blob = s
    s = st.check(lambda: eng.step(3), 3, s)
    eng.load_checkpoint(blob)
    s = st.check(lambda: eng.step(2), 2, s_blob)
    patched = bytearray(eng.checkpoint())
    struct.pack_into("<Q", patched, 104, 2**32 - 2)
    eng.load_checkpoint(bytes(patched))
    for k in range(4):
        s = st.check(lambda: eng.step(1), 1, 2**32 - 2 + k)
    assert s == 2**32 + 2
    s = st.check(lambda: eng.step(8), 8, s)


@pytest.mark.parametrize("cm_frequency", [0, 1, 3])
def test_one_stream_with_centre_of_mass_removal(cm_frequency):
    """cm_frequency 0, 1 (removal fused into the integrate kernel) and 3 (removal outside the step graph): the removal changes
    the velocities, never the draws."""
    st = Stream(KINDS["langevin_middle"], cm_frequency=cm_frequency)
    eng = st.eng
    s = 0
    for _ in range(4):
        s = st.check(lambda: eng.step(1), 1, s)
    s = st.check(lambda: eng.step(8), 8, s)
    s = st.check(lambda: eng.step(5), 5, s)


@pytest.mark.parametrize("seed", [1, 2**31 - 1, -1])
def test_one_stream_for_every_seed(seed):
    """The seed keys the generator as a 32-bit unsigned value (-1 is 0xffffffff)."""
    st = Stream(KINDS["langevin"], seed=seed)
    eng = st.eng
    s = st.check(lambda: eng.step(1), 1, 0)
    st.check(lambda: eng.step(8), 8, s)


@pytest.mark.parametrize("kind", list(KINDS))
def test_plugin_forwards_the_integrator_seed(kind):
    """LangevinIntegrator / LangevinMiddleIntegrator with an explicit seed on platform B200 (lazy forces + fused step): step k
    of the Context draws gauss3(seed, atom, k)."""
    from oracle import omm
    plugin = os.path.join(ROOT, "plugin", "libOpenMMB200.so")
    if not omm.available() or not os.path.exists(plugin):
        pytest.fail("oracle/_ref or the plugin is not built: run __graft_entry__.build() where the reference sources exist")
    omm.load_plugin(plugin)
    d = gas()
    seed = 424242
    sim = omm.Simulation(d, "B200", integrator=(KINDS[kind], TEMP, FRICTION, DT), seed=seed)
    assert sim.platform() == "B200"
    sim.set_velocities(thermal(d.masses))
    live = d.masses > 0
    sm = kick(d.masses)[:, None]
    for k in range(4):
        v0 = sim.state(velocities=True)["velocities"]
        sim.step(1)
        v1 = sim.state(velocities=True)["velocities"]
        g = (v1[live] - VSCALE*v0[live])/sm[live]
        assert np.abs(g - port().gauss3(seed, np.flatnonzero(live), k)).max() < GTOL["single"]
    sim.close()


# ---- (c) ----
def network_system():
    from test_gpu_integrate_lanes import mixed_units_system
    from test_oracle_langevin_cpu import with_general_networks
    return with_general_networks(mixed_units_system())


def dhfr_all_bonds():
    from openmm_b200 import systems
    from test_gpu_parity import _all_bonds
    return _all_bonds(systems, systems.SystemDesc.load(os.path.join(ROOT, "data", "dhfr.npz")).rounded())


# (velocity nm/ps, position nm) per atom against the oracle step.  Measured on an H100, max over the steps of a case: single
# 8e-5 nm/ps and 2e-7 nm, mixed 1.1e-7 nm/ps and 2.2e-10 nm (DHFR included).  The smallest kick of a case is 5.5e-2 nm/ps
# (DHFR's sulphur), 1.1e-4 nm per step, so 50x below it are 1.1e-3 nm/ps and 2.2e-6 nm.
UNIT_TOL = {"single": (1e-3, 2e-6), "mixed": (1e-6, 1e-9)}
CON_TOL = {"single": 1e-6, "mixed": 1e-10}


def run_against_oracle(d, kind, precision, nsteps=5, seed=SEED):
    from openmm_b200 import Engine
    p = port()
    eng = Engine(d, precision=precision)
    tol_v, tol_x = UNIT_TOL[precision]
    live = d.masses > 0
    smin = float(kick(d.masses)[live].min())
    # the tolerance can never admit a wrong draw: 50x below the smallest kick of the case and its displacement
    assert 50*tol_v <= smin and 50*tol_x <= smin*DT, (tol_v, tol_x, smin)
    eng.set_integrator(kind, DT, TEMP, FRICTION, seed, CON_TOL[precision])
    eng.set_velocities(thermal(d.masses))
    eng.apply_constraints(CON_TOL[precision])
    eng.apply_velocity_constraints(CON_TOL[precision])
    split = p.constraint_split(d)
    ev = ex = 0.0
    for _ in range(nsteps):
        x, v = eng.get_positions(), eng.get_velocities()
        eng.compute(energy=False)
        f = eng.get_forces()
        _, s = header(eng)
        eng.step(1)
        if d.cm_frequency == 1:
            v[live] -= (d.masses[live, None]*v[live]).sum(axis=0)/d.masses[live].sum()
        it = p.langevin_step(d, kind, DT, FRICTION, TEMP, x, v, f, gauss=p.gauss3(seed, np.arange(d.natoms), s), split=split)
        assert it >= 0
        ex = max(ex, float(np.abs(eng.get_positions() - x).max()))
        ev = max(ev, float(np.abs(eng.get_velocities() - v).max()))
    print("units %s kind %d %s cm %d: |dx| %.2e nm (tol %.0e), |dv| %.2e nm/ps (tol %.0e), smallest kick %.3e nm/ps"
          % (d.name, kind, precision, d.cm_frequency, ex, tol_x, ev, tol_v, smin))
    eng.close()
    assert ex < tol_x and ev < tol_v


@pytest.mark.parametrize("precision", ["single", "mixed"])
@pytest.mark.parametrize("kind", list(KINDS))
def test_every_unit_kind_follows_the_oracle_stochastic_step(kind, precision):
    """SETTLE, SHAKE with 2, 3 and 4 atoms, two general networks (k_ccma_step), free and massless atoms at 300 K, 10/ps:
    5 consecutive steps, each from the engine's own state, against port.langevin_step with the restated noise."""
    d = network_system()
    d.cm_frequency = 0
    run_against_oracle(d, KINDS[kind], precision)


@pytest.mark.parametrize("kind", list(KINDS))
def test_every_unit_kind_with_centre_of_mass_removal(kind):
    """The same with the removal every step (fused into both kernels): the oracle subtracts sum(m v)/sum(m) first."""
    d = network_system()
    d.cm_frequency = 1
    run_against_oracle(d, KINDS[kind], "mixed")


@pytest.mark.parametrize("kind", list(KINDS))
def test_dhfr_all_bonds_follows_the_oracle_stochastic_step(kind):
    """DHFR under AllBonds: the 2,500-constraint protein network in k_ccma_step at real size, with 7,000 SETTLE waters."""
    run_against_oracle(dhfr_all_bonds(), KINDS[kind], "mixed", nsteps=3)


# ---- (d) ----
@pytest.mark.parametrize("precision", ["single", "mixed"])
@pytest.mark.parametrize("kind", list(KINDS))
def test_long_run_velocity_variance(kind, precision):
    """400 steps from v = 0 through the 8-step graph: per mass class <v^2> = kT/m (1 - vscale^800) within 4 standard errors
    (fixed by the seed: the test cannot be flaky); the massless atom never moves."""
    from openmm_b200 import Engine
    from test_oracle_langevin_cpu import assert_gas_variance
    d = gas(n=4000 - 37)
    eng = Engine(d, precision=precision)
    eng.set_integrator(KINDS[kind], DT, TEMP, FRICTION, SEED, 1e-6)
    eng.set_velocities(np.zeros((d.natoms, 3)))
    eng.step(400)
    v, x = eng.get_velocities(), eng.get_positions()
    assert header(eng)[1] == 400
    assert_gas_variance(d, v, KT, VSCALE, 400)
    assert np.array_equal(x[d.masses == 0], d.positions[d.masses == 0])
