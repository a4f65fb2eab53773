"""The double-precision restatement of the barostat move (tests/barostat_harness.py: barostat_scale) against the live Reference
platform (oracle/_ref/libOpenMM.so, driven by plugin/examples/run_npt.cpp; both are built where the reference sources are
present).  Every particle has mass 0, so a VerletIntegrator moves nothing and any change of the positions in a step comes from
the barostat (frequency 1)."""
import os
import numpy as np
import pytest
from barostat_harness import RUN_NPT, barostat_scale, run_npt


@pytest.fixture(scope="module")
def omm():
    from oracle import omm
    if not omm.available() or not os.path.exists(RUN_NPT):
        pytest.skip("oracle/_ref (libOpenMM.so, tests/run_npt) is not built: no reference sources")
    return omm


def _chains(box, seed):
    """Chains of 1-5 bonded atoms, bonds straddling box faces, some molecules several box lengths outside the box."""
    from openmm_b200 import systems
    rng = np.random.default_rng(seed)
    x, bi, bj = [], [], []
    for m in range(40):
        n = int(rng.integers(1, 6))
        start = rng.random(3) @ box + (rng.integers(-3, 4, 3) @ box if m % 3 == 0 else 0)
        for k in range(n):
            if k:
                bi.append(len(x) - 1)
                bj.append(len(x))
            x.append(start + 0.15*k*np.array([1.0, 0.3, -0.2]))
    n = len(x)
    return systems.SystemDesc(masses=np.zeros(n), charges=np.zeros(n), sigmas=np.full(n, 0.3), epsilons=np.zeros(n),
                              positions=np.array(x), box=box, method=systems.NB_CUTOFF_PERIODIC, cutoff=0.5, use_dispersion=False,
                              bond_i=np.array(bi, np.int32), bond_j=np.array(bj, np.int32), bond_r0=np.full(len(bi), 0.15),
                              bond_k=np.full(len(bi), 1000.0))


@pytest.mark.parametrize("triclinic", [False, True])
def test_barostat_scale_matches_reference_platform(omm, tmp_path, triclinic):
    box = np.array([[2.5, 0, 0], [0.4, 2.2, 0], [-0.3, 0.6, 2.0]]) if triclinic else np.diag([2.5, 2.2, 2.0])
    d = _chains(box, 3 + int(triclinic))
    # triclinic: MonteCarloAnisotropicBarostat (every axis its own factor); rectangular: MonteCarloBarostat
    _, mols, boxes, frames = run_npt(d, str(tmp_path), platform="Reference", integrator="verlet", dt=0.001, temperature=300,
                                     barostat=2 if triclinic else 1, frequency=1, barostat_seed=11, chunks=30, chunk_steps=1)
    assert mols == d.molecules()
    accepted = 0
    for k in range(1, len(frames)):
        b0, b1, x0, x1 = boxes[k-1], boxes[k], frames[k-1], frames[k]
        if np.array_equal(b1, b0):
            assert np.array_equal(x1, x0)
            continue
        accepted += 1
        s = (b1[0, 0]/b0[0, 0], b1[1, 1]/b0[1, 1], b1[2, 2]/b0[2, 2])
        assert np.abs(barostat_scale(x0, mols, b0, s) - x1).max() < 1e-12
    assert accepted >= 1
