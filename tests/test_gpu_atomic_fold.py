"""GPU tests of the brick path of the PME charge spread (B200MD_PME_BRICK): the charge grid is an int64 sum, so spreading
through shared-memory bricks in sorted atom order must give the same grid bits, hence the same forces, as the user-order
kernel, whether a brick fits or not (B200MD_PME_BRICK_POINTS forces the global-memory fallback).  The reciprocal-space
energy is summed with double atomics, whose order varies from run to run, so it is compared to 1e-13 relative."""
import os
import numpy as np
import pytest
from conftest import ROOT

pytestmark = pytest.mark.gpu


def _system(name):
    from openmm_b200 import systems
    if name == "water24k":
        return systems.water_box(20, cutoff=0.9).rounded()
    if name == "ions_triclinic":
        return systems.random_ions(894, 3.0, cutoff=1.0, triclinic=True).rounded()
    if name == "dhfr_zero_charges":
        d = systems.SystemDesc.load(os.path.join(ROOT, "data", "dhfr.npz")).rounded()
        d.charges = d.charges.copy()
        d.charges[::7] = 0.0
        return d
    return systems.SystemDesc.load(os.path.join(ROOT, "data", name + ".npz")).rounded()


def _engine(monkeypatch, d, brick, points=None, precision="single"):
    from openmm_b200 import Engine
    monkeypatch.setenv("B200MD_PME_BRICK", "1" if brick else "0")
    if points is None:
        monkeypatch.delenv("B200MD_PME_BRICK_POINTS", raising=False)
    else:
        monkeypatch.setenv("B200MD_PME_BRICK_POINTS", str(points))
    return Engine(d, precision=precision)


def _recip(monkeypatch, d, brick, points=None, positions=None):
    from openmm_b200.engine import TERM_NB_RECIP
    eng = _engine(monkeypatch, d, brick, points)
    if positions is not None:
        eng.set_positions(positions)
    e = eng.compute(TERM_NB_RECIP)
    return eng.get_forces(), e


SYSTEMS = ["water24k", "dhfr", "apoa1", "ions_triclinic", "dhfr_zero_charges"]


@pytest.mark.parametrize("name", SYSTEMS)
@pytest.mark.parametrize("points", [None, 64])
def test_reciprocal_forces_and_energy_are_identical(monkeypatch, name, points):
    d = _system(name)
    f0, e0 = _recip(monkeypatch, d, False)
    f1, e1 = _recip(monkeypatch, d, True, points)
    assert np.abs(f0).max() > 0
    assert np.array_equal(f0, f1)
    assert e1 == pytest.approx(e0, rel=1e-13)


def test_molecules_shifted_by_lattice_vectors(monkeypatch):
    d = _system("dhfr")
    rng = np.random.default_rng(3)
    x = d.positions.copy()
    for mol in d.molecules():
        x[mol] += rng.integers(-2, 3, 3) @ d.box
    for points in (None, 64):
        f0, e0 = _recip(monkeypatch, d, False, positions=x)
        f1, e1 = _recip(monkeypatch, d, True, points, positions=x)
        assert np.array_equal(f0, f1)
        assert e1 == pytest.approx(e0, rel=1e-13)


@pytest.mark.parametrize("name", ["dhfr", "ions_triclinic"])
def test_full_compute_is_identical(monkeypatch, name):
    d = _system(name)
    res = []
    for brick in (False, True):
        eng = _engine(monkeypatch, d, brick)
        e = eng.compute()
        res.append((eng.get_forces(), e))
    assert np.array_equal(res[0][0], res[1][0])
    assert res[1][1] == pytest.approx(res[0][1], rel=1e-13)


@pytest.mark.parametrize("precision", ["single", "mixed"])
def test_langevin_trajectory_is_identical(monkeypatch, precision):
    from openmm_b200 import systems
    d = _system("dhfr")
    # no centre-of-mass removal: its momentum sum is a double atomicAdd over blocks, whose order (and hence last bit) varies
    # from run to run, and in mixed precision that bit reaches the double velocities
    d.cm_frequency = 0
    out = []
    for brick in (False, True):
        eng = _engine(monkeypatch, d, brick, precision=precision)
        eng.set_velocities(np.random.default_rng(5).standard_normal((d.natoms, 3))*0.3)
        eng.set_integrator(systems.INT_LANGEVIN, 0.002, 300.0, 1.0, 11)
        eng.step(200)
        eng.synchronize()
        assert eng.stats()["list_builds"] > 1
        out.append((eng.get_positions(), eng.get_velocities()))
    assert np.array_equal(out[0][0], out[1][0])
    assert np.array_equal(out[0][1], out[1][1])
