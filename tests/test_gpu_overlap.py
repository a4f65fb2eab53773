"""The single-GPU step runs the reciprocal-space chain and the bonded terms beside the tile kernel, as graph nodes of a higher
priority and with CTAs shaped to fit the slots the tile kernel hands back.  Where and when those kernels run must not change
a bit of the trajectory: every force goes into the int64 fixed-point buffer, the charge grid is an exact integer sum, and each
FFT butterfly is computed the same way whichever thread takes it."""
import os
import subprocess
import sys
import numpy as np
import pytest
from conftest import ROOT

pytestmark = pytest.mark.gpu


def _load(name):
    from openmm_b200 import systems
    return systems.SystemDesc.load(os.path.join(ROOT, "data", name + ".npz")).rounded()


def _run(d, env, monkeypatch, steps=200):
    from openmm_b200 import systems, Engine
    for k in ("B200MD_NO_OVERLAP", "B200MD_USE_GRAPH"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    eng = Engine(d)                     # the schedule switches are read when the context is created
    eng.set_integrator(systems.INT_LANGEVIN, 0.002, 300.0, 1.0, 7, 1e-5)
    st0 = eng.stats()
    eng.step(steps)
    eng.synchronize()
    out = eng.get_positions(), eng.get_velocities(), eng.stats()["list_builds"] - st0["list_builds"]
    eng.close()
    return out


def test_schedule_does_not_change_the_trajectory(monkeypatch):
    """200 Langevin steps of DHFR, list rebuilds included: the default overlapped graph, one stream, and no graph agree bit
    for bit."""
    d = _load("dhfr")
    x0, v0, builds = _run(d, {}, monkeypatch)
    assert builds > 1, "the run must include list rebuilds"
    for env in ({"B200MD_NO_OVERLAP": "1"}, {"B200MD_USE_GRAPH": "0"}):
        x, v, _ = _run(d, env, monkeypatch)
        assert np.array_equal(x, x0), env
        assert np.array_equal(v, v0), env


_RECIP = """
import os, sys
sys.path.insert(0, %r)
import numpy as np
from openmm_b200 import systems, Engine
from openmm_b200.engine import TERM_NB_RECIP
d = systems.SystemDesc.load(os.path.join(%r, "data", "dhfr.npz")).rounded()
eng = Engine(d)
eng.set_integrator(systems.INT_LANGEVIN, 0.002, 300.0, 1.0, 7, 1e-5)
eng.step(50)
eng.compute(TERM_NB_RECIP, energy=False)
np.save(sys.argv[1], eng.get_forces())
"""


def test_fft_cta_shape_does_not_change_reciprocal_forces(tmp_path):
    """Reciprocal-space forces with the single-GPU FFT CTAs and with 512-thread ones are identical.  The thread counts are
    read once per process, so each shape runs in a process of its own."""
    forces = []
    for k, threads in enumerate((None, "512")):
        env = dict(os.environ)
        env.pop("B200MD_FFT_THREADS", None)
        env.pop("B200MD_FFTX_THREADS", None)
        if threads:
            env["B200MD_FFT_THREADS"] = threads
        path = str(tmp_path / ("f%d.npy" % k))
        subprocess.run([sys.executable, "-c", _RECIP % (ROOT, ROOT), path], env=env, cwd=ROOT, check=True, timeout=600)
        forces.append(np.load(path))
    assert np.abs(forces[0]).max() > 0
    assert np.array_equal(forces[0], forces[1])
