"""The NonbondedForce parameter changes the GPU tests make (tests/nonbonded_params_harness.py), checked on the CPU against
the double-precision restatement: every change moves the energy by more than 1 kJ/mol, so that no GPU comparison after an
update can pass because nothing changed, and each change does what its name says."""
import numpy as np
import pytest
import nonbonded_params_harness as H


@pytest.mark.parametrize("system_name,change_name", H.cases() + [(s, "all") for s in H.SYSTEMS])
def test_change_moves_the_energy(system_name, change_name):
    from oracle import port
    a, b, disp = H.before_after(system_name, change_name)
    _, ea, _ = port.forces_energy(a, dispersion_coefficient=disp)
    _, eb, _ = port.forces_energy(b, dispersion_coefficient=disp)
    assert abs(eb - ea) > 1.0
    assert len(b.exc_i) == len(a.exc_i) and (b.exc_i == a.exc_i).all() and (b.exc_j == a.exc_j).all()


@pytest.mark.parametrize("system_name", ["water_rigid", "ions_triclinic", "dhfr"])
def test_changes_touch_what_they_name(system_name):
    d = H.system(system_name)
    a, b, _ = H.before_after(system_name, "charge")
    charged = (a.charges == 0) & (b.charges != 0)
    assert charged.sum() >= 30 and (b.charges[charged] == d.charges[charged]).all()     # the base's zero charges come back
    a, b, _ = H.before_after(system_name, "decouple")
    off = (a.charges != 0) & (b.charges == 0)
    assert off.sum() >= 24 and np.allclose(b.epsilons[off], 0.5*a.epsilons[off])
    if system_name in H.WITHOUT_EXCEPTIONS:
        return
    a, b, _ = H.before_after(system_name, "exceptions")
    live = (a.exc_qq == 0) & (a.exc_eps == 0) & (b.exc_eps > 0)
    assert live.sum() >= 20
    if system_name == "dhfr":
        assert ((a.exc_eps > 0) & (b.exc_qq == 0) & (b.exc_eps == 0)).sum() == 60
