"""GPU tests of NonbondedForce parameter changes in a live context (b200md_update_nonbonded_params, which
updateParametersInContext and Context::setParameter of parameter offsets both reach).  The update rewrites every copy of
the parameters the kernels read -- the fp32 charges in posq.w and sigma/epsilon pairs of the tile kernel, the double
charges and pairs of the close-pair path and of PME, the exception table with its PME exclusion products, the self
energy -- and the next list build re-sorts them.  Each change (tests/nonbonded_params_harness.py) is checked against the
double-precision restatement, against a context made with the new parameters, and across a round trip, MD steps and
checkpoints; then through the OpenMM plugin against the Reference platform in the same process.

A checkpoint holds no force-field parameters (ContextImpl::loadCheckpoint restores the state and the global parameter
values): a context that loads one keeps its current parameters, whatever they were when the checkpoint was written."""
import os
import numpy as np
import pytest
from conftest import relative_force_error, ROOT
import nonbonded_params_harness as H

pytestmark = pytest.mark.gpu
PRECISIONS = ["single", "mixed"]
PLUGIN = os.path.join(ROOT, "plugin", "libOpenMMB200.so")
_ORACLE = {}


def _oracle(key, d, disp):
    """(forces, energy) of the restatement, cached per key (the protein takes seconds)"""
    from oracle import port
    if key not in _ORACLE:
        f, e, _ = port.forces_energy(d, dispersion_coefficient=disp)
        _ORACLE[key] = f, e
    return _ORACLE[key]


def _evaluate(eng):
    e = eng.compute()
    return eng.get_forces(), e


# ---- the C ABI against the restatement and against a freshly made context ----
@pytest.mark.parametrize("system_name,change_name", H.cases())
def test_update_matches_oracle(system_name, change_name):
    """After the update the forces and energy are those of the new parameters; the dispersion correction keeps the
    coefficient of the parameters' default values, as the reference does for parameter offsets."""
    from openmm_b200 import Engine
    a, b, disp = H.before_after(system_name, change_name)
    eng = Engine(a)
    f0, e0 = _evaluate(eng)
    eng.update_nonbonded_params(b, disp)
    f, e = _evaluate(eng)
    fr, er = _oracle((system_name, change_name, "B"), b, disp)
    _, er0 = _oracle((system_name, change_name, "A"), a, disp)
    assert abs(er - er0) > 1.0 and abs(e - e0) > 1.0          # the change shows: the comparison below is not of the old state
    assert relative_force_error(f, fr) < 1e-4
    assert abs(e - er)/max(1.0, abs(er)) < 1e-5
    assert eng.stats()["overflow"] == 0


@pytest.mark.parametrize("system_name,change_name", H.cases())
def test_update_matches_a_fresh_context(system_name, change_name):
    """Fixed-point force sums do not depend on order: an updated context and one made with the new parameters, at the same
    positions, give the same forces bit for bit."""
    from openmm_b200 import Engine
    a, b, _ = H.before_after(system_name, change_name)
    eng = Engine(a)
    eng.compute()
    eng.update_nonbonded_params(b)
    f, e = _evaluate(eng)
    ff, ef = _evaluate(Engine(b))
    assert np.array_equal(f, ff)
    assert e == pytest.approx(ef, rel=1e-12)


@pytest.mark.parametrize("system_name,change_name", H.cases())
def test_round_trip_restores_the_forces(system_name, change_name):
    from openmm_b200 import Engine
    a, b, _ = H.before_after(system_name, change_name)
    eng = Engine(a)
    f0, e0 = _evaluate(eng)
    eng.update_nonbonded_params(b)
    f1, _ = _evaluate(eng)
    assert not np.array_equal(f1, f0)
    eng.update_nonbonded_params(a)
    f, e = _evaluate(eng)
    assert np.array_equal(f, f0)
    assert e == pytest.approx(e0, rel=1e-12)


def _langevin(d, precision):
    from openmm_b200 import Engine, systems
    eng = Engine(d, precision=precision)
    eng.set_integrator(systems.INT_LANGEVIN_MIDDLE, 0.002, 300.0, 1.0, 5)
    return eng


@pytest.mark.parametrize("precision", PRECISIONS)
def test_update_in_the_middle_of_a_run(precision):
    """20 LangevinMiddle steps with A, a checkpoint, the update to B and 20 more steps: the same trajectory as a context
    made with B that loads the checkpoint (the random force is keyed on the step counter, which the checkpoint carries).
    A context that stays at A goes elsewhere, so the update did reach the captured step graph."""
    a, b, _ = H.before_after("water_rigid", "all")
    x = _langevin(a, precision)
    x.step(20)
    blob = x.checkpoint()
    x.update_nonbonded_params(b)
    x.step(20)
    y = _langevin(b, precision)
    y.load_checkpoint(blob)
    y.step(20)
    assert np.array_equal(x.get_positions(), y.get_positions())
    assert np.array_equal(x.get_velocities(), y.get_velocities())
    z = _langevin(a, precision)
    z.load_checkpoint(blob)
    z.step(20)
    assert not np.array_equal(x.get_positions(), z.get_positions())


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("system_name", ["water_rigid", "dhfr"])
def test_checkpoint_across_an_update(system_name, precision):
    """A checkpoint written with A (its posq.w holds the charges of A, and 0 for the waters that are uncharged in A), the
    update to B, then the checkpoint loaded: the context evaluates B, as one made with B does and as the restatement does."""
    from openmm_b200 import Engine
    a, b, _ = H.before_after(system_name, "all")
    assert ((a.charges == 0) & (b.charges != 0)).sum() >= 30
    eng = Engine(a, precision=precision)
    blob = eng.checkpoint()
    eng.update_nonbonded_params(b)
    eng.load_checkpoint(blob)
    f, e = _evaluate(eng)
    ff, ef = _evaluate(Engine(b, precision=precision))
    assert np.array_equal(f, ff)
    assert e == pytest.approx(ef, rel=1e-12)
    fr, er = _oracle((system_name, "all", "B own dispersion"), b, b.dispersion_coefficient())
    assert relative_force_error(f, fr) < 1e-4
    assert abs(e - er)/max(1.0, abs(er)) < 1e-5


def test_refused_update_leaves_the_context_intact():
    """An update with another number of exceptions is refused before anything is changed."""
    import copy
    from openmm_b200 import Engine
    from openmm_b200.engine import EngineError
    a, b, disp = H.before_after("water_rigid", "exceptions")
    eng = Engine(a)
    f0, e0 = _evaluate(eng)
    bad = copy.copy(b)
    for k in ("exc_i", "exc_j", "exc_qq", "exc_sigma", "exc_eps"):
        setattr(bad, k, getattr(b, k)[:-1])
    with pytest.raises(EngineError, match="number of exceptions"):
        eng.update_nonbonded_params(bad, disp)
    f, e = _evaluate(eng)
    assert np.array_equal(f, f0) and e == pytest.approx(e0, rel=1e-12)
    fr, er = _oracle(("water_rigid", "exceptions", "A"), a, disp)
    assert relative_force_error(f, fr) < 1e-4 and abs(e - er)/max(1.0, abs(er)) < 1e-5
    eng.update_nonbonded_params(b, disp)         # and a correct update still goes through
    f, e = _evaluate(eng)
    fr, er = _oracle(("water_rigid", "exceptions", "B"), b, disp)
    assert relative_force_error(f, fr) < 1e-4 and abs(e - er)/max(1.0, abs(er)) < 1e-5


# ---- the plugin against the Reference platform in the same process ----
@pytest.fixture(scope="module")
def omm():
    from oracle import omm
    if not omm.available() or not os.path.exists(PLUGIN):
        pytest.fail("oracle/_ref or the plugin is not built: run __graft_entry__.build() where /root/reference exists")
    omm.load_plugin(PLUGIN)
    return omm


def _offset_water(rigid):
    """The global parameters and offsets of test_oracle.py::test_port_parameter_offsets_match_live_reference on a larger
    box.  The two exceptions with offsets are water O-H exclusions; their base sigma is 0.1 nm here instead of 1 nm (the
    base parameters stay zero, so they still become live 1-4 terms only through the offsets): at 1.2 nm and 0.096 nm apart a
    Lennard-Jones term is 1e13 kJ/mol, past the engine's fixed-point force range."""
    from openmm_b200 import systems
    d = systems.water_box(6, cutoff=0.9, rigid=rigid).rounded()
    d.exc_sigma = d.exc_sigma.copy()
    d.exc_sigma[[0, 4]] = 0.1
    glob = {"lambda_q": 0.25, "lambda_lj": 1.0}
    p_off = [("lambda_q", 0, 0.3, 0.0, 0.0), ("lambda_q", 1, -0.3, 0.0, 0.0), ("lambda_lj", 3, 0.0, 0.02, 0.25), ("lambda_lj", 6, 0.1, -0.01, 0.5),
             ("lambda_q", 6, 0.05, 0.0, 0.0)]
    e_off = [("lambda_lj", 0, 0.04, 0.02, 0.3), ("lambda_q", 4, -0.02, 0.015, 0.1)]
    return d, dict(nb_globals=glob, particle_offsets=p_off, exception_offsets=e_off, pme=d.pme_parameters())


def _pair(omm, d, props="", **kw):
    return omm.Simulation(d, "B200", props=props, **kw), omm.Simulation(d, "Reference", **kw)


def _agree(a, b):
    fa, ea = a.forces_energy()
    fb, eb = b.forces_energy()
    assert relative_force_error(fa, fb) < 1e-4
    assert abs(ea - eb)/max(1.0, abs(eb)) < 1e-5
    return eb


SWEEP = [(0.25, 1.0), (-0.5, 0.4), (1.0, 0.0), (0.0, 0.7), (0.25, 1.0)]


def test_plugin_set_parameter_sweep(omm):
    d, kw = _offset_water(rigid=False)
    a, b = _pair(omm, d, **kw)
    energies = []
    for q, lj in SWEEP:
        for s in (a, b):
            s.set_parameter("lambda_q", q)
            s.set_parameter("lambda_lj", lj)
        energies.append(_agree(a, b))
    assert min(abs(np.diff(energies[:-1]))) > 1.0
    assert energies[-1] == pytest.approx(energies[0], rel=1e-12)


def test_plugin_verlet_run_with_changing_parameters(omm):
    """lambda changes every 5 steps of Integrator::step, which replays one captured step graph with lazy forces: the graph
    must see each change."""
    from openmm_b200 import systems
    d, kw = _offset_water(rigid=True)
    v = np.random.default_rng(3).standard_normal((d.natoms, 3))*0.3
    a, b = _pair(omm, d, integrator=(systems.INT_VERLET, 0, 0, 0.001), **kw)
    for s in (a, b):
        s.set_velocities(v)
    for q, lj in SWEEP[1:]:
        for s in (a, b):
            s.set_parameter("lambda_q", q)
            s.set_parameter("lambda_lj", lj)
            s.step(5)
    sa, sb = a.state(positions=True, energy=True), b.state(positions=True, energy=True)
    assert np.abs(sa["positions"] - sb["positions"]).max() < 5e-6
    assert abs(sa["potential"] - sb["potential"])/abs(sb["potential"]) < 1e-4


@pytest.mark.parametrize("precision", PRECISIONS)
def test_plugin_update_parameters_in_context(omm, precision):
    a_desc, b_desc, _ = H.before_after("water_flexible", H.KEEPS_EXCLUSIONS)
    a, b = _pair(omm, a_desc, props="Precision=" + precision, pme=a_desc.pme_parameters())
    e0 = _agree(a, b)
    for s in (a, b):
        s.update_nonbonded(b_desc)
    assert abs(_agree(a, b) - e0) > 1.0


@pytest.mark.parametrize("precision", PRECISIONS)
def test_plugin_checkpoint_then_update_then_load(omm, precision):
    """createCheckpoint, updateParametersInContext, loadCheckpoint: the Reference platform evaluates the new parameters."""
    a_desc, b_desc, _ = H.before_after("water_flexible", H.KEEPS_EXCLUSIONS)
    a, b = _pair(omm, a_desc, props="Precision=" + precision, pme=a_desc.pme_parameters())
    e0 = _agree(a, b)
    blobs = [s.checkpoint() for s in (a, b)]
    for s, blob in zip((a, b), blobs):
        s.update_nonbonded(b_desc)
        s.load_checkpoint(blob)
    assert abs(_agree(a, b) - e0) > 1.0


@pytest.mark.parametrize("precision", PRECISIONS)
def test_plugin_checkpoint_across_a_parameter_change(omm, precision):
    """setParameter(B), createCheckpoint (the platform has not uploaded B yet: that waits for the next evaluation),
    getState (uploads B), loadCheckpoint (lambda comes back as B, the value already uploaded): the state of B."""
    base, p_off, e_off = H.change(H.system("water_flexible"), "all")
    a, b = _pair(omm, base, props="Precision=" + precision, pme=base.pme_parameters(), nb_globals={H.LAM: 0.0},
                 particle_offsets=p_off, exception_offsets=e_off)
    e0 = _agree(a, b)
    for s in (a, b):
        s.set_parameter(H.LAM, 1.0)
    blobs = [s.checkpoint() for s in (a, b)]
    e1 = _agree(a, b)
    assert abs(e1 - e0) > 1.0
    for s, blob in zip((a, b), blobs):
        s.load_checkpoint(blob)
    assert _agree(a, b) == pytest.approx(e1, rel=1e-12)
