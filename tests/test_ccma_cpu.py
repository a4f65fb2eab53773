"""CPU tests of the general-constraint (CCMA) path, no GPU needed:
 * oracle/md_oracle.c:orc_ccma restates ReferenceCCMAAlgorithm::applyConstraints and is pinned against the Reference platform
   (Context::applyConstraints on the real DHFR protein under constraints=AllBonds, stored in tests/golden/reference_platform.npz);
 * the matrix the ENGINE builds on the host (b200md_ccma_setup_probe: coupling matrix as the reference builds it, inverse
   approximated from the constraints within three bonds) makes that iteration converge as fast as an exact inverse would need
   to, and to the same positions as the reference's own sparse-QR matrix."""
import ctypes as C
import os
import numpy as np
import pytest
from conftest import ROOT, GOLDEN
from openmm_b200 import systems, _lib
from oracle import port

D, I, F = C.POINTER(C.c_double), C.POINTER(C.c_int), C.POINTER(C.c_float)


def _probe(mass, ci, cj, cd, ang=None):
    lib = _lib.load()
    mass = np.ascontiguousarray(mass, np.float64); ci = np.ascontiguousarray(ci, np.int32); cj = np.ascontiguousarray(cj, np.int32)
    cd = np.ascontiguousarray(cd, np.float64)
    ai, aj, ak, t0 = [np.ascontiguousarray(a, t) for a, t in zip(ang if ang is not None else ([0], [0], [0], [0.0]), (np.int32, np.int32, np.int32, np.float64))]
    na = 0 if ang is None else len(ai)
    ncomp, nccma = C.c_int(), C.c_int()
    n = len(ci)
    order = np.zeros(max(n, 1), np.int32); row = np.zeros(n + 1, np.int32)
    cap = 64*max(n, 1)
    col = np.zeros(cap, np.int32); val = np.zeros(cap, np.float32)
    nnz = lib.b200md_ccma_setup_probe(len(mass), mass.ctypes.data_as(D), n, ci.ctypes.data_as(I), cj.ctypes.data_as(I), cd.ctypes.data_as(D),
                                      na, ai.ctypes.data_as(I), aj.ctypes.data_as(I), ak.ctypes.data_as(I), t0.ctypes.data_as(D),
                                      C.byref(ncomp), C.byref(nccma), order.ctypes.data_as(I), row.ctypes.data_as(I), col.ctypes.data_as(I), val.ctypes.data_as(F), cap)
    assert nnz >= 0, nnz
    k = nccma.value
    return ncomp.value, order[:k].copy(), row[:k+1].copy(), col[:nnz].copy(), val[:nnz].astype(np.float64)


def _iterate(order, row, col, val, ci, cj, cd, invm, x, xp, tol=1e-6, vel=False):
    L = port.lib()
    ai = np.ascontiguousarray(np.asarray(ci)[order], np.int32); aj = np.ascontiguousarray(np.asarray(cj)[order], np.int32)
    d = np.ascontiguousarray(np.asarray(cd)[order], np.float64)
    xp = np.ascontiguousarray(xp, np.float64).copy()
    it = L.orc_ccma(len(ai), ai.ctypes.data_as(I), aj.ctypes.data_as(I), d.ctypes.data_as(D), np.ascontiguousarray(invm, np.float64).ctypes.data_as(D),
                    np.ascontiguousarray(x, np.float64).ctypes.data_as(D), xp.ctypes.data_as(D), np.ascontiguousarray(row, np.int32).ctypes.data_as(I),
                    np.ascontiguousarray(col, np.int32).ctypes.data_as(I), np.ascontiguousarray(val, np.float64).ctypes.data_as(D), int(vel), tol, 150)
    return it, xp


def test_chain_classification_components_and_convergence():
    """TestVerletIntegrator::testConstrainedChain shape: a 100-particle chain is ONE component of 99 coupled constraints; a rigid
    water and an X-H3 cluster beside it stay with SETTLE / SHAKE."""
    n = 100
    rng = np.random.default_rng(0)
    x = np.zeros((n + 7, 3))
    for i in range(1, n):
        dlt = rng.standard_normal(3); x[i] = x[i-1] + dlt/np.linalg.norm(dlt)
    x[n:n+3] = [[50, 0, 0], [50.0957, 0, 0], [49.976, 0.0927, 0]]
    x[n+3:n+7] = [[60, 0, 0], [60.109, 0, 0], [59.964, 0.103, 0], [59.964, -0.051, 0.089]]
    ci = list(range(n-1)) + [n, n, n+1] + [n+3, n+3, n+3]
    cj = list(range(1, n)) + [n+1, n+2, n+2] + [n+4, n+5, n+6]
    cd = [1.0]*(n-1) + [0.0957, 0.0957, float(np.linalg.norm(x[n+1]-x[n+2]))] + [0.109]*3
    mass = np.ones(n + 7); mass[n] = 16; mass[n+3] = 12
    ncomp, order, row, col, val = _probe(mass, ci, cj, cd)
    assert ncomp == 1 and sorted(order) == list(range(n-1))
    # every row has its diagonal near 1/(1 - coupling^2...) and a few neighbours; no angle information -> bare chain couplings are zero
    assert all(row[k+1] > row[k] for k in range(len(order)))
    xp = x.copy(); xp[:n] += 0.02*rng.standard_normal((n, 3))
    it, xc = _iterate(order, row, col, val, ci, cj, cd, 1/mass, x, xp)
    assert it < 40
    dist = np.linalg.norm(xc[np.array(ci[:n-1])] - xc[np.array(cj[:n-1])], axis=1)
    assert np.abs(dist - 1).max() < 2e-6


@pytest.mark.parametrize("vel", [False, True])
def test_dhfr_allbonds_matrix_and_iteration_against_the_live_reference(vel):
    d = systems.SystemDesc.load(os.path.join(ROOT, "data", "dhfr.npz"))
    have = set((min(i, j), max(i, j)) for i, j in zip(d.con_i, d.con_j))
    ci, cj, cd = list(d.con_i), list(d.con_j), list(d.con_d)
    for i, j, r0 in zip(d.bond_i, d.bond_j, d.bond_r0):
        if (min(i, j), max(i, j)) not in have:
            ci.append(int(i)); cj.append(int(j)); cd.append(float(r0))
    d.con_i, d.con_j, d.con_d = np.array(ci, np.int32), np.array(cj, np.int32), np.array(cd)
    ncomp, order, row, col, val = _probe(d.masses, ci, cj, cd, (d.angle_i, d.angle_j, d.angle_k, d.angle_t0))
    nprot = len(order)
    assert ncomp >= 1 and 2000 < nprot < 3000                      # the protein's bonds; the waters stay with SETTLE
    nnz_per_row = (row[1:] - row[:-1])
    assert nnz_per_row.min() >= 1 and nnz_per_row.mean() < 20     # sparse: entries below the reference's 0.02 cut-off are dropped
    # the Reference platform projects the PDB structure onto the constraints (ReferenceConstraints -> SETTLE + CCMA with ITS
    # matrix, tolerance 1e-7); stored for the protein atoms as the displacement from the input positions
    x0 = np.array(d.positions, dtype=np.float64)
    dx = np.load(os.path.join(GOLDEN, "reference_platform.npz"))["ccma_cpu:dx"]
    xref = x0.copy()
    xref[:len(dx)] += dx
    assert max(np.array(ci)[order].max(), np.array(cj)[order].max()) < len(dx)
    if vel:
        # velocities: project random velocities with the restated iteration and check the constraint velocities vanish
        v = np.random.default_rng(2).standard_normal(x0.shape)
        it, vc = _iterate(order, row, col, val, ci, cj, cd, 1/np.asarray(d.masses), xref, v, tol=1e-7, vel=True)
        a, b = np.array(ci)[order], np.array(cj)[order]
        rel = np.einsum("ij,ij->i", vc[a] - vc[b], xref[a] - xref[b])/np.array(cd)[order]**2
        assert it < 30 and np.abs(rel).max() < 1e-5
    else:
        it, xc = _iterate(order, row, col, val, ci, cj, cd, 1/np.asarray(d.masses), x0, x0, tol=1e-7)
        prot = np.unique(np.concatenate([np.array(ci)[order], np.array(cj)[order]]))
        assert it < 30                                              # an exact inverse needs ~5-10 on this structure
        assert np.abs(xc[prot] - xref[prot]).max() < 2e-6           # same solution as the reference's sparse-QR matrix
