"""GPU tests of the tile kernel's sorted-order force accumulation: k_pair adds its forces into a buffer laid out in the
current neighbour list's sorted order, and k_fold_sorted, launched right behind it, adds that buffer into the user-order
force buffer and zeroes it.  Fixed-point addition is exact and does not depend on order, so the forces must be
bit-identical to those of the user-order accumulation (tests/golden/tile_forces.npz, make_golden_tile_forces.py) and
repeat exactly across evaluations, list rebuilds, MD steps and rejected barostat moves.  Energies are sums of double
atomics whose order varies from run to run: compared to 1e-12 relative."""
import os
import numpy as np
import pytest
from conftest import ROOT, GOLDEN

pytestmark = pytest.mark.gpu

# name -> (energy evaluated, precision).  Together they run the forces-only and the energy tile kernel, the single-image
# (SHIFT) and the per-pair minimum-image path, the switching function, PME, reaction field and no cutoff, and atom
# counts that are not a multiple of 32.
CASES = {"dhfr": (False, "single"),
         "ions_triclinic": (True, "single"),
         "water": (True, "single"),
         "water_switch": (True, "single"),
         "water_mixed": (False, "mixed"),
         "cluster_nocutoff": (True, "single"),
         "lj_reaction_field": (True, "single")}


def system(name):
    from openmm_b200 import systems
    if name == "dhfr":
        return systems.SystemDesc.load(os.path.join(ROOT, "data", "dhfr.npz")).rounded()
    if name == "ions_triclinic":
        return systems.random_ions(894, 3.0, cutoff=1.0, triclinic=True).rounded()
    if name in ("water", "water_mixed"):
        return systems.water_box(6, cutoff=0.9).rounded()
    if name == "water_switch":
        d = systems.water_box(6, cutoff=0.9).rounded()
        d.use_switch, d.switch_distance = True, 0.8
        return d
    if name == "cluster_nocutoff":
        return systems.cluster(70).rounded()
    if name == "lj_reaction_field":
        return systems.lj_fluid(7, cutoff=1.0, charged=True).rounded()
    raise KeyError(name)


def run(name):
    """(engine, forces, energy or None) of one evaluation of every term at the stored positions."""
    from openmm_b200 import Engine
    energy, precision = CASES[name]
    eng = Engine(system(name), precision=precision)
    e = eng.compute(energy=energy)
    return eng, eng.get_forces(), e


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN, "tile_forces.npz"))


@pytest.mark.parametrize("name", sorted(CASES))
def test_forces_match_user_order_accumulation(golden, name):
    eng, f, e = run(name)
    assert np.abs(f).max() > 0
    assert np.array_equal(f, golden["f_" + name])
    if e is not None:
        assert e == pytest.approx(float(golden["e_" + name]), rel=1e-12)


@pytest.mark.parametrize("name", sorted(CASES))
def test_repeated_evaluation_is_identical(name):
    # an undrained sorted buffer would add the direct-space forces of the first evaluation to the second
    eng, f0, _ = run(name)
    energy = CASES[name][0]
    for _ in range(2):
        eng.compute(energy=energy)
        assert np.array_equal(eng.get_forces(), f0)


def test_forced_rebuild_at_same_positions_is_identical():
    eng, f0, _ = run("dhfr")
    eng.set_positions(system("dhfr").positions)          # marks the list dirty: the next evaluation rebuilds it
    eng.compute(energy=False)
    assert eng.stats()["list_builds"] >= 2
    assert np.array_equal(eng.get_forces(), f0)


@pytest.mark.parametrize("precision", ["single", "mixed"])
def test_forces_after_steps_match_a_fresh_context(precision):
    """After graph-captured MD steps (the fused step path, which never reads forces back) the sorted buffer must be empty:
    an evaluation there equals one in a new context at the same positions and with a list built at them."""
    from openmm_b200 import Engine, systems
    d = system("dhfr")
    eng = Engine(d, precision=precision)
    eng.set_integrator(systems.INT_LANGEVIN, 0.002, 300.0, 1.0, 11)
    eng.step(25)
    eng.synchronize()
    x = eng.get_positions()
    eng.set_positions(x)
    eng.compute(energy=False)
    f = eng.get_forces()
    fresh = Engine(d, precision=precision)
    fresh.set_positions(x)
    fresh.compute(energy=False)
    assert np.array_equal(f, fresh.get_forces())


def test_rejected_barostat_move_is_identical():
    eng, f0, _ = run("dhfr")
    d = system("dhfr")
    eng.set_barostat_molecules()
    for s in (1.02, 0.98):
        eng.scale_coordinates(s, s, s)
        eng.set_box(d.box*s)
        eng.compute(energy=False)
        assert not np.array_equal(eng.get_forces(), f0)
        eng.restore_coordinates()
        eng.set_box(d.box)
        eng.compute(energy=False)
        assert np.array_equal(eng.get_forces(), f0)
