"""The kernels a force evaluation and a step enqueue, counted per call: Engine.stats()'s kernel_launches and graph_instantiations
for the step in every schedule and precision, compute() of each term class with and without the energy, a bonded group mask,
custom torsions, a cutoff System without PME and the stand-alone reciprocal-space context.  The counts pin the schedule that
enqueue_forces builds: a branch that runs where it did not, or stops running, changes them."""
import ctypes as C
import os
import numpy as np
import pytest
from conftest import ROOT
from openmm_b200.engine import TERM_ALL as ALL, TERM_CUSTOM_TORSIONS as CUSTOM, TERM_NB_DIRECT as DIRECT, TERM_NB_RECIP as RECIP

pytestmark = pytest.mark.gpu

BONDED = ALL & ~(DIRECT | RECIP)


def _dhfr():
    from openmm_b200 import systems
    return systems.SystemDesc.load(os.path.join(ROOT, "data", "dhfr.npz")).rounded()


def _engine(d, env=None, precision="single"):
    """an Engine made with the schedule switches in `env` (they are read when the context is created)"""
    from openmm_b200 import systems, Engine
    keys = ("B200MD_NO_OVERLAP", "B200MD_USE_GRAPH")
    saved = {k: os.environ.pop(k, None) for k in keys}
    os.environ.update(env or {})
    try:
        eng = Engine(d, precision=precision)
    finally:
        for k in keys:
            os.environ.pop(k, None)
            if saved[k] is not None:
                os.environ[k] = saved[k]
    eng.set_integrator(systems.INT_LANGEVIN, 0.002, 300.0, 1.0, 7, 1e-5)
    return eng


def _counts(stats, calls):
    """(kernel launches, graph instantiations) that each call adds"""
    out = []
    for call in calls:
        s0 = stats()
        call()
        s1 = stats()
        out.append((s1["kernel_launches"] - s0["kernel_launches"], s1["graph_instantiations"] - s0["graph_instantiations"]))
    return out


def _steps(eng):
    """the first step (list pass, one-step graph), a captured step, the eight-step graph twice and a remainder of three"""
    return _counts(eng.stats, [lambda n=n: eng.step(n) for n in (1, 1, 16, 3)])


def _computes(eng, calls):
    eng.compute(ALL, energy=False)          # the list pass of the new positions
    return _counts(eng.stats, calls)


def step_counts(precision, env):
    eng = _engine(_dhfr(), env, precision)
    try:
        return _steps(eng)
    finally:
        eng.close()


def compute_counts():
    eng = _engine(_dhfr())
    try:
        calls = [lambda t=t, e=e: eng.compute(t, energy=e) for t in (DIRECT, RECIP, BONDED, ALL) for e in (False, True)]
        calls.append(lambda: eng.compute_groups(ALL, 0x2))
        return _computes(eng, calls)
    finally:
        eng.close()


def custom_torsion_counts():
    import custom_harness as harness
    from openmm_b200 import systems
    if not harness.available():
        pytest.fail("oracle/_ref is not built: run __graft_entry__.build() where /root/reference exists")
    eng = _engine(harness.compiled(systems.with_charmm_impropers(_dhfr())))
    try:
        calls = [lambda: eng.compute(CUSTOM, energy=True), lambda: eng.compute(ALL, energy=True),
                 lambda: eng.compute_groups(ALL, 0x1)]
        return _computes(eng, calls) + _steps(eng)
    finally:
        eng.close()


def cutoff_periodic_counts():
    from openmm_b200 import systems
    eng = _engine(systems.water_box(8, cutoff=0.9, method=systems.NB_CUTOFF_PERIODIC).rounded())
    try:
        calls = [lambda e=e: eng.compute(ALL, energy=e) for e in (False, True)] + [lambda: eng.compute(RECIP, energy=True)]
        return _computes(eng, calls) + _steps(eng)
    finally:
        eng.close()


def standalone_pme_counts():
    """b200md_pme_create / b200md_pme_exec, as the CalcPmeReciprocalForce kernel calls them; the first call finalizes"""
    from openmm_b200 import _lib, systems
    lib = _lib.load()
    d = systems.water_box(6, cutoff=0.9).rounded()
    alpha, nx, ny, nz = d.pme_parameters()
    h = C.c_void_p()
    assert lib.b200md_pme_create(C.byref(h), 0, d.natoms, nx, ny, nz, alpha) == 0, lib.b200md_last_error(None)
    try:
        posq = np.zeros((d.natoms, 4), np.float32)
        posq[:, :3], posq[:, 3] = d.positions, d.charges
        box = np.ascontiguousarray(d.box, dtype=np.float64).ravel()
        force = np.zeros((d.natoms, 4), np.float32)
        e = C.c_double()
        fp, dp = C.POINTER(C.c_float), C.POINTER(C.c_double)

        def stats():
            s = _lib.Stats()
            assert lib.b200md_get_stats(h, C.byref(s)) == 0
            return {"kernel_launches": s.kernel_launches, "graph_instantiations": s.graph_instantiations}

        def run(energy):
            rc = lib.b200md_pme_exec(h, posq.ctypes.data_as(fp), box.ctypes.data_as(dp), energy, force.ctypes.data_as(fp), C.byref(e))
            assert rc == 0, lib.b200md_last_error(h)
        return _counts(stats, [lambda x=x: run(x) for x in (1, 0, 1)])
    finally:
        lib.b200md_destroy(h)


# (kernel launches, graph instantiations) per call, measured on one H100 80GB HBM3.  A DHFR step is the 12 kernel nodes of
# DESIGN.md section 4; the first call adds the synchronous list pass of the new positions (3).  The schedule switches move
# kernels between streams, not in or out of the step.
_STEP = [(15, 1), (12, 0), (192, 1), (36, 0)]
_STEP_NO_GRAPH = [(15, 0), (12, 0), (192, 0), (36, 0)]
EXPECTED = {
    **{("step", p, "graph"): _STEP for p in ("single", "mixed")},
    **{("step", p, "no_overlap"): _STEP for p in ("single", "mixed")},
    **{("step", p, "no_graph"): _STEP_NO_GRAPH for p in ("single", "mixed")},
    # DIRECT, RECIP, BONDED, ALL, each without and with the energy; then ALL restricted to bonded group 1
    "compute": [(6, 0), (6, 0), (5, 0), (5, 0), (1, 0), (1, 0), (11, 0), (11, 0), (11, 0)],
    # CUSTOM, ALL, ALL in group 0 only; then the steps (a 13th node: k_custom_torsion)
    "custom_torsions": [(1, 0), (12, 0), (12, 0), (13, 1), (13, 0), (208, 1), (39, 0)],
    # ALL without and with the energy, RECIP (nothing to run); then the steps
    "cutoff_periodic": [(6, 0), (6, 0), (0, 0), (7, 1), (7, 0), (112, 1), (21, 0)],
    # with, without, with the energy
    "standalone_pme": [(6, 0), (5, 0), (5, 0)],
}


@pytest.mark.parametrize("precision", ["single", "mixed"])
@pytest.mark.parametrize("schedule", ["graph", "no_overlap", "no_graph"])
def test_step(precision, schedule):
    env = {"graph": {}, "no_overlap": {"B200MD_NO_OVERLAP": "1"}, "no_graph": {"B200MD_USE_GRAPH": "0"}}[schedule]
    assert step_counts(precision, env) == EXPECTED["step", precision, schedule]


def test_compute():
    assert compute_counts() == EXPECTED["compute"]


def test_custom_torsions():
    assert custom_torsion_counts() == EXPECTED["custom_torsions"]


def test_cutoff_periodic():
    assert cutoff_periodic_counts() == EXPECTED["cutoff_periodic"]


def test_standalone_pme():
    assert standalone_pme_counts() == EXPECTED["standalone_pme"]
