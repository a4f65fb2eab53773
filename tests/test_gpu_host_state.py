"""The engine's host-side handling of the per-atom state, held to explicit expectations: the checkpoint blob's exact layout in
both precisions, the barostat's save/restore, time_phase leaving the state as it found it, and which calls make the next
evaluation rebuild the neighbour list."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

PRECISIONS = ["single", "mixed"]
ONE_4PI_EPS0 = 138.93545764438198
HEADER = np.dtype([("magic", "S8"), ("version", "<i4"), ("natoms", "<i4"), ("time", "<f8"), ("step_count", "<i8"),
                   ("box", "<f8", (9,)), ("step_counter", "<u8")])
DT = 0.002


def _system():
    """375 TIP3P atoms (padded to 384); the last water is massless (its constraints are then ignored: three free atoms)."""
    from openmm_b200 import systems
    d = systems.water_box(5, cutoff=0.75).rounded()
    d.masses = d.masses.copy()
    d.masses[-3:] = 0.0
    return d


def _velocities(d):
    v = np.random.default_rng(3).standard_normal((d.natoms, 3))*0.5
    v[d.masses == 0] = 0.0
    return v


def _engine(d, precision):
    from openmm_b200 import systems, Engine
    eng = Engine(d, precision=precision)
    eng.set_integrator(systems.INT_LANGEVIN, DT, 300.0, 1.0, 7)
    eng.set_velocities(_velocities(d))
    return eng


def _expected_blob(d, precision, x, v, box, time, step_count):
    """header | posq (xyz, w = q sqrt(ONE_4PI_EPS0)) | posqCorr (mixed: fp32 low parts) | velm (fp32, w = 1/mass) or velmD
    (double) | cellOffset (zeros)"""
    n, npad = d.natoms, (d.natoms + 31)//32*32
    h = np.zeros(1, HEADER)
    h["magic"], h["version"], h["natoms"] = b"B200MDCK", 3 if precision == "mixed" else 2, n
    h["time"], h["step_count"], h["box"], h["step_counter"] = time, step_count, np.asarray(box).ravel(), step_count
    hi = x.astype(np.float32)
    posq = np.zeros((npad, 4), np.float32)
    posq[:n, :3] = hi
    posq[:n, 3] = (d.charges*np.sqrt(ONE_4PI_EPS0)).astype(np.float32)
    invm = np.divide(1.0, d.masses, out=np.zeros(n), where=d.masses > 0)
    parts = [h.tobytes(), posq.tobytes()]
    if precision == "mixed":
        corr = np.zeros((npad, 4), np.float32)
        corr[:n, :3] = (x - hi.astype(np.float64)).astype(np.float32)
        velm = np.zeros((npad, 4), np.float64)
        parts.append(corr.tobytes())
    else:
        velm = np.zeros((npad, 4), np.float32)
    velm[:n, :3] = v
    velm[:n, 3] = invm
    parts += [velm.tobytes(), np.zeros(3*npad, np.int32).tobytes()]
    return b"".join(parts)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_checkpoint_layout(precision):
    d = _system()
    eng = _engine(d, precision)
    x = d.positions + np.random.default_rng(4).uniform(-0.01, 0.01, d.positions.shape)
    v = _velocities(d)
    box = d.box*1.001
    eng.set_positions(x)
    eng.set_velocities(v)
    eng.set_box(box)
    blob = eng.checkpoint()
    assert len(blob) == 112 + (76 if precision == "mixed" else 44)*384
    assert blob == _expected_blob(d, precision, x, v, box, 0.0, 0)
    # after some steps: the blob describes the state the engine reports, and load -> save reproduces it
    eng.step(13)
    x, v = eng.get_positions(), eng.get_velocities()
    blob = eng.checkpoint()
    assert blob == _expected_blob(d, precision, x, v, box, eng.time(), 13)
    assert eng.lib.b200md_get_step_count(eng.h) == 13
    fresh = _engine(d, precision)
    fresh.load_checkpoint(blob)
    assert fresh.checkpoint() == blob
    assert np.array_equal(fresh.get_positions(), x) and np.array_equal(fresh.get_velocities(), v)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_barostat_restore_returns_the_saved_state(precision):
    d = _system()
    eng = _engine(d, precision)
    eng.step(10)
    eng.compute(energy=False)
    eng.set_barostat_molecules()
    x0, v0, f0, blob0 = eng.get_positions(), eng.get_velocities(), eng.get_forces(), eng.checkpoint()
    eng.scale_coordinates(1.01, 1.01, 1.01)
    assert not np.array_equal(eng.get_positions(), x0)
    assert np.array_equal(eng.get_velocities(), v0)
    eng.compute(energy=False)
    assert not np.array_equal(eng.get_forces(), f0)
    eng.restore_coordinates()
    assert np.array_equal(eng.get_positions(), x0) and np.array_equal(eng.get_forces(), f0)
    assert eng.checkpoint() == blob0


_TRAJECTORY = {}


def _trajectory(precision):
    """(positions, velocities) after 20 steps from the state _engine sets up"""
    if precision not in _TRAJECTORY:
        eng = _engine(_system(), precision)
        eng.step(20)
        _TRAJECTORY[precision] = eng.get_positions(), eng.get_velocities()
    return _TRAJECTORY[precision]


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("phase", ["pair", "pme_spread", "pme_fft_conv", "pme_gather", "integrate", "list_build", "bonded"])
def test_time_phase_leaves_the_state_alone(phase, precision):
    d = _system()
    eng = _engine(d, precision)
    x0, v0, blob0 = eng.get_positions(), eng.get_velocities(), eng.checkpoint()
    eng.time_phase(phase, reps=3)
    assert np.array_equal(eng.get_positions(), x0) and np.array_equal(eng.get_velocities(), v0)
    assert eng.checkpoint() == blob0              # the step counter in the header included
    eng.step(20)
    x, v = _trajectory(precision)
    assert np.array_equal(eng.get_positions(), x) and np.array_equal(eng.get_velocities(), v)


PREPARE_LIST_LAUNCHES = 3      # the synchronous list pass of a dirty list: the displacement check and the two build kernels


def _launches(eng, call):
    """kernel launches the engine counts for `call`"""
    before = eng.stats()["kernel_launches"]
    call()
    return eng.stats()["kernel_launches"] - before


@pytest.mark.parametrize("precision", PRECISIONS)
def test_timed_list_build_adds_no_rebuild_to_the_next_step(precision):
    """time_phase("list_build") raises the device's rebuild flag only: it must not mark the list dirty, which would put a
    synchronous list pass in front of the next step."""
    eng = _engine(_system(), precision)
    eng.step(1)                # captures the step graph; the list is clean from here on
    steady = _launches(eng, lambda: eng.step(1))
    eng.time_phase("list_build", reps=3)
    builds = eng.stats()["list_builds"]
    assert _launches(eng, lambda: eng.step(1)) == steady
    assert eng.stats()["list_builds"] == builds       # the positions have not moved since the last timed build


@pytest.mark.parametrize("call", ["set_positions", "set_box", "update_nonbonded_params", "load_checkpoint"])
def test_state_changes_rebuild_the_list(call):
    d = _system()
    eng = _engine(d, "single")
    eng.compute(energy=False)          # the tile pools are sized by now
    x, blob = eng.get_positions(), eng.checkpoint()
    clean = _launches(eng, lambda: eng.compute(energy=False))
    builds = eng.stats()["list_builds"]
    if call == "set_positions":
        eng.set_positions(x)
    elif call == "set_box":
        eng.set_box(d.box)
    elif call == "update_nonbonded_params":
        eng.update_nonbonded_params(d)          # the same parameters again
    else:
        eng.load_checkpoint(blob)
    # the list is marked dirty (a synchronous list pass first) and the device's rebuild flag is raised (one build)
    assert _launches(eng, lambda: eng.compute(energy=False)) == clean + PREPARE_LIST_LAUNCHES
    assert eng.stats()["list_builds"] == builds + 1
