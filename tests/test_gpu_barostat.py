"""GPU tests of the Monte Carlo barostat: ApplyMonteCarloBarostatKernel (olla/include/openmm/kernels.h:1425-1459) through the
C-ABI (b200md_scale_coordinates / b200md_restore_coordinates, k_scale_molecules) and through the OpenMM Platform plugin, where
the reference's own MonteCarloBarostatImpl drives it."""
import os
import subprocess
import numpy as np
import pytest
from conftest import relative_force_error, GOLDEN, ROOT

pytestmark = pytest.mark.gpu
PLUGIN = os.path.join(ROOT, "plugin", "libOpenMMB200.so")
REFTESTS = os.path.join(ROOT, "oracle", "_ref", "tests")
BAROSTAT_SCALE = 1.02          # the move stored in tests/golden/reference_barostat.npz (tests/golden/make_golden_barostat.py)


def _load(name):
    from openmm_b200 import systems
    return systems.SystemDesc.load(os.path.join(ROOT, "data", name + ".npz")).rounded()


def _cell_offsets(eng):
    """cellOffset of every atom, read from the checkpoint blob (its last 3*npad int32)."""
    npad = eng.stats()["padded_atoms"]
    return np.frombuffer(eng.checkpoint()[-12*npad:], dtype=np.int32).reshape(3, npad)[:, :eng.natoms]


def _shifted_engine(d):
    """An engine whose every 7th molecule sits 2-3 box lengths away, so that the list build wraps it back and keeps the lattice
    vectors in cellOffset."""
    from openmm_b200 import Engine
    x = d.positions.copy()
    rng = np.random.default_rng(11)
    for m in d.molecules()[::7]:
        k = rng.integers(-3, 4, 3)
        k[k == 0] = 2
        x[m] += k @ d.box
    eng = Engine(d)
    eng.set_positions(x)
    eng.compute()
    assert (_cell_offsets(eng) != 0).any()
    return eng


@pytest.mark.parametrize("name", ["dhfr", "apoa1"])
def test_scale_coordinates_matches_oracle(name):
    from barostat_harness import barostat_scale
    d = _load(name)
    eng = _shifted_engine(d)
    mols = d.molecules()
    eng.set_barostat_molecules(mols)
    for s in ((0.98,)*3, (1.02,)*3, (0.99, 1.015, 1.003)):
        x0 = eng.get_positions()
        expect = barostat_scale(x0, mols, d.box, s)
        eng.scale_coordinates(*s)
        x1 = eng.get_positions()
        # fp32 positions: one rounding of a coordinate of up to ~12 nm is 5e-7 nm
        assert np.abs(x1 - expect).max() < 2e-6, (s, np.abs(x1 - expect).max())
        assert not _cell_offsets(eng).any()
        eng.restore_coordinates()
        assert np.array_equal(eng.get_positions(), x0)


@pytest.mark.parametrize("name", ["dhfr", "apoa1"])
def test_forces_in_the_scaled_box_match_reference(name):
    """After scale_coordinates + set_box(scaled box) the forces and energy are the Reference platform's at the same coordinates
    (stored sample, the metric of tests/test_gpu_parity.py)."""
    from openmm_b200 import Engine
    ref = np.load(os.path.join(GOLDEN, "reference_barostat.npz"))
    d = _load(name)
    eng = Engine(d)
    eng.compute()
    eng.set_barostat_molecules()
    eng.scale_coordinates(BAROSTAT_SCALE, BAROSTAT_SCALE, BAROSTAT_SCALE)
    eng.set_box(d.box*BAROSTAT_SCALE)
    idx = ref[name + ":idx"]
    x = eng.get_positions()
    assert np.abs(x[idx] - ref[name + ":x"]).max() < 2e-6
    e = eng.compute()
    f = eng.get_forces()
    er = float(ref[name + ":e"])
    assert relative_force_error(f[idx], ref[name + ":f"]) < 1e-4
    assert abs(e - er)/max(1.0, abs(er)) < 1e-4
    assert eng.stats()["overflow"] == 0


def test_rejected_move_restores_state_bit_for_bit():
    from openmm_b200 import systems
    d = _load("dhfr")
    eng = _shifted_engine(d)
    eng.set_barostat_molecules()
    eng.set_integrator(systems.INT_LANGEVIN_MIDDLE, 0.002, 300.0, 1.0, 3, 1e-5)
    eng.step(20)
    e0 = eng.compute()
    x0, f0, blob0 = eng.get_positions(), eng.get_forces(), eng.checkpoint()
    box = d.box.copy()
    for s in (1.02, 0.98):
        eng.scale_coordinates(s, s, s)
        eng.set_box(box*s)
        assert eng.compute() != e0
        eng.restore_coordinates()
        assert np.array_equal(eng.get_forces(), f0)          # the saved force buffer
        eng.set_box(box)
        # forces are int64 fixed point and repeat exactly; the energy is a sum of double atomics, equal to rounding
        assert abs(eng.compute() - e0) < 1e-9*abs(e0)
        assert np.array_equal(eng.get_positions(), x0) and np.array_equal(eng.get_forces(), f0)
        assert eng.checkpoint() == blob0                     # posq, velocities, cellOffset, step counter: every byte


def _npt(d, steps, frequency, seed, attempts_log=None):
    """MonteCarloBarostatImpl::updateContextState (MonteCarloBarostatImpl.cpp:64-121) over the C-ABI, with numpy's RNG."""
    from openmm_b200 import Engine, systems
    kT = 0.00831446261815324*300.0
    pressure = 1.0*6.02214076e23*1e-25
    eng = Engine(d)
    eng.set_integrator(systems.INT_LANGEVIN_MIDDLE, 0.002, 300.0, 1.0, seed, 1e-5)
    eng.set_barostat_molecules()
    nmol = len(d.molecules())
    rng = np.random.default_rng(seed)
    box = d.box.copy()
    volume_scale = 0.01*np.prod(np.diag(box))
    accepted = rejected = 0
    for _ in range(steps//frequency):
        eng.step(frequency)
        e0 = eng.compute()
        v = np.prod(np.diag(box))
        dv = volume_scale*2*(rng.random() - 0.5)
        s = ((v + dv)/v)**(1/3)
        eng.scale_coordinates(s, s, s)
        eng.set_box(box*s)
        e1 = eng.compute()
        w = e1 - e0 + pressure*dv - nmol*kT*np.log((v + dv)/v)
        if w > 0 and rng.random() > np.exp(-w/kT):
            eng.restore_coordinates()
            eng.set_box(box)
            rejected += 1
        else:
            box = box*s
            accepted += 1
        if attempts_log is not None:
            attempts_log.append(eng.stats()["graph_instantiations"])
    return eng, box, accepted, rejected


def test_npt_is_deterministic_and_does_not_instantiate_graphs():
    from openmm_b200 import systems
    d = systems.water_box(10, cutoff=0.9).rounded()
    runs = []
    for _ in range(2):
        log = []
        eng, box, acc, rej = _npt(d, 200, 5, 9, log)
        runs.append((eng.get_positions(), box))
        assert acc > 0 and rej > 0
        # the box changes at every attempt: the step graph is updated in place, never instantiated again
        assert log[-1] == log[0] <= 2, log
        eng.close()
    assert np.array_equal(runs[0][0], runs[1][0]) and np.array_equal(runs[0][1], runs[1][1])


# The DHFR box (6.22 nm, 241 nm^3) holds ~3 % more volume than the system has at 1 bar: 7,023 TIP3P waters take ~210 nm^3 and
# the 18 kDa protein ~22 nm^3.  Within 20 ps of NPT the volume falls by 2.5-3 % (measured on an H100, the C-ABI and the plugin
# path alike), so the bound is the physical range: it shrinks, by less than 5 %.
def _dhfr_volume_ok(v, v0):
    return 0.95 < v/v0 < 1.0


def test_dhfr_npt_run():
    d = _load("dhfr")
    eng, box, acc, rej = _npt(d, 10000, 25, 5)
    v0, v1 = np.prod(np.diag(d.box)), np.prod(np.diag(box))
    assert acc > 0 and rej > 0
    assert _dhfr_volume_ok(v1, v0)
    x = eng.get_positions()
    assert np.abs(np.linalg.norm(x[d.con_i] - x[d.con_j], axis=1) - d.con_d).max() < 1e-5
    assert eng.stats()["overflow"] == 0


# ---- through the plugin: the reference's MonteCarloBarostatImpl drives ApplyMonteCarloBarostatKernel (plugin/examples/run_npt.cpp) ----
@pytest.fixture(scope="module")
def npt():
    from oracle import omm
    from barostat_harness import RUN_NPT, run_npt
    if not omm.available() or not os.path.exists(PLUGIN) or not os.path.exists(RUN_NPT):
        pytest.fail("oracle/_ref, the plugin or run_npt is not built: run __graft_entry__.build() where /root/reference exists")
    return run_npt


def test_plugin_npt_runs_on_b200_and_repeats_exactly(npt, tmp_path):
    from openmm_b200 import systems
    d = systems.water_box(10, cutoff=0.9).rounded()
    runs = [npt(d, str(tmp_path/str(k)), pme=d.pme_parameters(), seed=3, frequency=5, barostat_seed=17, chunks=4, chunk_steps=50)
            for k in range(2)]
    line, mols, boxes, frames = runs[0]
    assert line["platform"] == "B200"
    assert mols == d.molecules()
    assert len({b[0, 0] for b in boxes}) > 1                                # moves were accepted
    assert np.array_equal(boxes, runs[1][2]) and np.array_equal(frames, runs[1][3])


def test_plugin_dhfr_npt(npt, tmp_path):
    d = _load("dhfr")
    line, _, boxes, frames = npt(d, str(tmp_path), pme=d.pme_parameters(), seed=5, frequency=25, barostat_seed=5, chunks=100, chunk_steps=100)
    assert line["platform"] == "B200"
    volumes = boxes[:, 0, 0]*boxes[:, 1, 1]*boxes[:, 2, 2]
    v0 = np.prod(np.diag(d.box))
    assert len(set(volumes.tolist())) > 1                                 # moves were accepted
    assert _dhfr_volume_ok(volumes[-1], v0) and volumes.min()/v0 > 0.95
    x = frames[-1]
    assert np.abs(np.linalg.norm(x[d.con_i] - x[d.con_j], axis=1) - d.con_d).max() < 1e-5


@pytest.mark.parametrize("name", ["TestB200MonteCarloBarostat", "TestB200MonteCarloAnisotropicBarostat"])
def test_reference_barostat_test_bodies_pass_on_b200_platform(name):
    """tests/TestMonteCarloBarostat.h and TestMonteCarloAnisotropicBarostat.h of the reference against our platform
    (plugin/Makefile lists the functions); ASSERT_USUALLY_* failures get the one rerun the reference's CI gives them."""
    exe = os.path.join(REFTESTS, name)
    if not os.path.exists(exe):
        pytest.fail("%s not built (make -C plugin reftests where /root/reference exists)" % exe)
    env = dict(os.environ, B200_PLUGIN=PLUGIN)
    for attempt in range(2):
        p = subprocess.run([exe], capture_output=True, text=True, timeout=1200, env=env)
        if p.returncode == 0 and "Done" in p.stdout:
            break
        if "stochastic" not in p.stdout:
            break
    assert p.returncode == 0 and "Done" in p.stdout, p.stdout[-2000:] + p.stderr[-2000:]
