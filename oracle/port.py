"""oracle/port.py -- TEST INFRASTRUCTURE, not product code.

ctypes binding of oracle/_ref/liboracle-<sha1 of md_oracle.c>.so (md_oracle.c, the plain-C restatement of the reference algorithm).
forces_energy(desc) evaluates a SystemDesc exactly the way ReferenceCalcNonbondedForceKernel::execute
(ReferenceKernels.cpp:967-1014) + the bonded kernels do.  Only tests/, smoke() and bench.py's cpu_baseline may use it.
"""
import ctypes as C
import hashlib
import os
import subprocess
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
with open(os.path.join(_HERE, "md_oracle.c"), "rb") as _src:
    _TAG = hashlib.sha1(_src.read()).hexdigest()[:16]
# named after the source's content (oracle/Makefile `port`): a library built from another version is never loaded
_LIB = os.path.join(_HERE, "_ref", "liboracle-%s.so" % _TAG)
_lib = None
D = C.POINTER(C.c_double)
I = C.POINTER(C.c_int)


def build():
    subprocess.check_call(["make", "-s", "-C", _HERE, "port", "ORC_TAG=" + _TAG])


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB):
            build()
        L = C.CDLL(_LIB)
        L.orc_direct.restype = C.c_double
        L.orc_direct.argtypes = [C.c_int, D, D, D, D, D, C.c_int, C.c_double, C.c_double, C.c_double, C.c_int, C.c_double, I, I, D]
        L.orc_self_energy.restype = C.c_double
        L.orc_self_energy.argtypes = [C.c_int, D, C.c_double]
        L.orc_exclusion_correction.restype = C.c_double
        L.orc_exclusion_correction.argtypes = [C.c_int, I, I, D, D, D, C.c_int, C.c_double, D]
        L.orc_exceptions14.restype = C.c_double
        L.orc_exceptions14.argtypes = [C.c_int, I, I, D, D, D, D, D]
        L.orc_pme_reciprocal.restype = C.c_double
        L.orc_pme_reciprocal.argtypes = [C.c_int, D, D, D, C.c_double, C.c_int, C.c_int, C.c_int, D]
        L.orc_bonds_pbc.restype = C.c_double
        L.orc_bonds_pbc.argtypes = [C.c_int, I, I, D, D, D, D, D]
        L.orc_angles_pbc.restype = C.c_double
        L.orc_angles_pbc.argtypes = [C.c_int, I, I, I, D, D, D, D, D]
        L.orc_torsions_pbc.restype = C.c_double
        L.orc_torsions_pbc.argtypes = [C.c_int, I, I, I, I, I, D, D, D, D, D]
        L.orc_settle.restype = None
        L.orc_settle.argtypes = [C.c_int, I, I, I, D, D, D, D, D]
        L.orc_settle_velocities.restype = None
        L.orc_settle_velocities.argtypes = [C.c_int, I, I, I, D, D, D]
        L.orc_step.restype = None
        L.orc_step.argtypes = [C.c_int, C.c_int, C.c_double, C.c_double, D, D, D, D, C.c_int, I, I, I, D, D]
        L.orc_fft3d_forward.restype = None
        L.orc_fft3d_forward.argtypes = [C.c_int, C.c_int, C.c_int, D, D]
        L.orc_ccma.restype = C.c_int
        L.orc_ccma.argtypes = [C.c_int, I, I, D, D, D, D, I, I, D, C.c_int, C.c_double, C.c_int]
        U = C.POINTER(C.c_uint32)
        L.orc_philox4x32_10.restype = None
        L.orc_philox4x32_10.argtypes = [U, U, U]
        L.orc_gauss3.restype = None
        L.orc_gauss3.argtypes = [C.c_uint32, C.c_int, C.c_uint64, D]
        L.orc_gauss3_atoms.restype = None
        L.orc_gauss3_atoms.argtypes = [C.c_uint32, C.c_int, I, C.c_uint64, D]
        L.orc_langevin_step.restype = C.c_int
        L.orc_langevin_step.argtypes = [C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, D, D, D, D, D, C.c_int, I, I, I, D, D,
                                        C.c_int, I, I, D, C.c_double]
        L.orc_num_threads.restype = C.c_int
        _lib = L
    return _lib


def _d(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def _i(a):
    return np.ascontiguousarray(a, dtype=np.int32)


def _dp(a):
    return a.ctypes.data_as(D)


def _ip(a):
    return a.ctypes.data_as(I)


def exclusion_csr(n, ei, ej):
    ex = [[] for _ in range(n)]
    for a, b in zip(np.asarray(ei).tolist(), np.asarray(ej).tolist()):
        ex[a].append(b)
        ex[b].append(a)
    start = np.zeros(n+1, dtype=np.int32)
    lst = []
    for k in range(n):
        s = sorted(set(ex[k]))
        start[k+1] = start[k] + len(s)
        lst.extend(s)
    return start, np.array(lst if lst else [0], dtype=np.int32)


def with_parameter_offsets(desc, values, particle_offsets=(), exception_offsets=()):
    """The SystemDesc the force field sees when the global parameters have `values` (ReferenceCalcNonbondedForceKernel::
    computeParameters, ReferenceKernels.cpp:1077-1121): every offset (name, index, dq, dsigma, deps) adds value*scale to the
    base charge / sigma / epsilon of its particle, or to chargeProd / sigma / epsilon of its exception.  An exception that
    has an offset stays a 1-4 even when its base parameters are zero (:873-895); here every exception is evaluated anyway.
    NOT affected by the current values: the dispersion coefficient, which the reference computes once from the parameters'
    DEFAULT values (NonbondedForceImpl.cpp:241-258; ReferenceKernels.cpp:962) -- pass that one to forces_energy()."""
    import copy
    d = copy.copy(desc)
    d.charges, d.sigmas, d.epsilons = _d(desc.charges).copy(), _d(desc.sigmas).copy(), _d(desc.epsilons).copy()
    d.exc_qq, d.exc_sigma, d.exc_eps = _d(desc.exc_qq).copy(), _d(desc.exc_sigma).copy(), _d(desc.exc_eps).copy()
    for name, idx, dq, ds, de in particle_offsets:
        d.charges[idx] += values[name]*dq
        d.sigmas[idx] += values[name]*ds
        d.epsilons[idx] += values[name]*de
    for name, idx, dq, ds, de in exception_offsets:
        d.exc_qq[idx] += values[name]*dq
        d.exc_sigma[idx] += values[name]*ds
        d.exc_eps[idx] += values[name]*de
    return d


def forces_energy(desc, positions=None, pme=None, terms=None, bonded_periodic=False, dispersion_coefficient=None):
    """(forces [N,3], energy, parts) of a SystemDesc; pme = (alpha, nx, ny, nz) overrides desc.pme_parameters();
    bonded_periodic: the bonded forces use the minimum image (Force::usesPeriodicBoundaryConditions);
    dispersion_coefficient: overrides desc.dispersion_coefficient() (parameter offsets: see with_parameter_offsets)."""
    L = lib()
    n = desc.natoms
    pos = _d(desc.positions if positions is None else positions)
    q, sig, eps = _d(desc.charges), _d(desc.sigmas), _d(desc.epsilons)
    box = _d(desc.box).reshape(9) if desc.box is not None else _d(np.eye(3)).reshape(9)
    f = np.zeros((n, 3))
    parts = {}
    start, lst = exclusion_csr(n, desc.exc_i, desc.exc_j)
    alpha = 0.0
    if desc.method == 4:
        alpha, nx, ny, nz = pme if pme is not None else desc.pme_parameters()
    parts["direct"] = L.orc_direct(n, _dp(pos), _dp(q), _dp(sig), _dp(eps), _dp(box), desc.method, desc.cutoff, alpha, desc.rf_dielectric,
                                   int(desc.use_switch), desc.switch_distance, _ip(start), _ip(lst), _dp(f))
    if desc.method in (2, 4) and desc.use_dispersion:
        parts["dispersion"] = (desc.dispersion_coefficient() if dispersion_coefficient is None else dispersion_coefficient)/(box[0]*box[4]*box[8])
    ne = len(desc.exc_i)
    ei, ej = _i(desc.exc_i), _i(desc.exc_j)
    if ne:
        parts["exceptions14"] = L.orc_exceptions14(ne, _ip(ei), _ip(ej), _dp(_d(desc.exc_qq)), _dp(_d(desc.exc_sigma)), _dp(_d(desc.exc_eps)), _dp(pos), _dp(f))
    if desc.method == 4:
        parts["self"] = L.orc_self_energy(n, _dp(q), alpha)
        parts["reciprocal"] = L.orc_pme_reciprocal(n, _dp(pos), _dp(q), _dp(box), alpha, nx, ny, nz, _dp(f))
        if ne:
            parts["exclusion"] = L.orc_exclusion_correction(ne, _ip(ei), _ip(ej), _dp(pos), _dp(q), _dp(box), 0, alpha, _dp(f))
    bbox = _dp(box) if bonded_periodic else None          # NULL = plain displacements
    if len(desc.bond_i):
        parts["bonds"] = L.orc_bonds_pbc(len(desc.bond_i), _ip(_i(desc.bond_i)), _ip(_i(desc.bond_j)), _dp(_d(desc.bond_r0)), _dp(_d(desc.bond_k)), _dp(pos),
                                         bbox, _dp(f))
    if len(desc.angle_i):
        parts["angles"] = L.orc_angles_pbc(len(desc.angle_i), _ip(_i(desc.angle_i)), _ip(_i(desc.angle_j)), _ip(_i(desc.angle_k)),
                                           _dp(_d(desc.angle_t0)), _dp(_d(desc.angle_kk)), _dp(pos), bbox, _dp(f))
    if len(desc.tor_i):
        parts["torsions"] = L.orc_torsions_pbc(len(desc.tor_i), _ip(_i(desc.tor_i)), _ip(_i(desc.tor_j)), _ip(_i(desc.tor_k)), _ip(_i(desc.tor_l)),
                                               _ip(_i(desc.tor_n)), _dp(_d(desc.tor_phase)), _dp(_d(desc.tor_kk)), _dp(pos), bbox, _dp(f))
    return f, float(sum(parts.values())), parts


def settle_clusters(desc):
    """(a0, a1, a2, d1, d2) for 3-atom rigid molecules described by desc's constraints (ReferenceConstraints.cpp:69-146)."""
    n = desc.natoms
    adj = [dict() for _ in range(n)]
    for a, b, d in zip(desc.con_i.tolist(), desc.con_j.tolist(), desc.con_d.tolist()):
        adj[a][b] = d
        adj[b][a] = d
    done = np.zeros(n, bool)
    out = []
    for a in range(n):
        if done[a] or len(adj[a]) != 2:
            continue
        b, c = list(adj[a])
        if len(adj[b]) != 2 or len(adj[c]) != 2 or c not in adj[b]:
            continue
        dab, dac, dbc = np.float32(adj[a][b]), np.float32(adj[a][c]), np.float32(adj[b][c])
        if dab == dac:
            out.append((a, b, c, adj[a][b], adj[b][c]))
        elif dab == dbc:
            out.append((b, a, c, adj[a][b], adj[a][c]))
        elif dac == dbc:
            out.append((c, a, b, adj[a][c], adj[a][b]))
        else:
            continue
        done[[a, b, c]] = True
    arr = np.array(out) if out else np.zeros((0, 5))
    return _i(arr[:, 0]), _i(arr[:, 1]), _i(arr[:, 2]), _d(arr[:, 3]), _d(arr[:, 4])


def step(desc, kind, dt, friction, x, v, forces, clusters):
    """One deterministic (zero-temperature) Verlet (0) / Langevin (1) / LangevinMiddle (2) step with SETTLE; x, v modified in place."""
    L = lib()
    a0, a1, a2, d1, d2 = clusters
    L.orc_step(kind, desc.natoms, dt, friction, _dp(_d(desc.masses)), _dp(_d(forces)), _dp(x), _dp(v), len(a0), _ip(a0), _ip(a1), _ip(a2), _dp(d1), _dp(d2))


BOLTZ = 0.00831446261815324          # kJ/mol/K, as md_oracle.c and the engine


def philox4x32_10(ctr, key):
    """Philox4x32-10 of a 4-word counter and a 2-word key (orc_philox4x32_10), as 4 uint32."""
    c, k, out = (np.ascontiguousarray(np.asarray(a, dtype=np.uint64) & 0xffffffff, dtype=np.uint32) for a in (ctr, key, np.zeros(4)))
    U = C.POINTER(C.c_uint32)
    lib().orc_philox4x32_10(c.ctypes.data_as(U), k.ctypes.data_as(U), out.ctypes.data_as(U))
    return out


def gauss3(seed, atoms, step):
    """[n, 3]: the three normals the engine draws for each of `atoms` in the step that starts with counter `step`
    (engine.h gauss3, restated by orc_gauss3).  The seed is taken as the engine takes it, cast to 32-bit unsigned."""
    a = _i(np.atleast_1d(atoms))
    g = np.empty((len(a), 3))
    lib().orc_gauss3_atoms(int(seed) & 0xffffffff, len(a), _ip(a), int(step), _dp(g))
    return g


def constraint_split(desc):
    """(SETTLE clusters as settle_clusters(desc), (ai, aj, dist) of every other constraint): the Reference platform's split
    of a System's constraints into rigid waters and one CCMA system (ReferenceConstraints.cpp:69-184)."""
    cl = settle_clusters(desc)
    settled = np.zeros(desc.natoms, bool)
    for a in cl[:3]:
        settled[a] = True
    rest = ~(settled[desc.con_i] & settled[desc.con_j])
    return cl, (_i(desc.con_i[rest]), _i(desc.con_j[rest]), _d(desc.con_d[rest]))


def langevin_step(desc, kind, dt, friction, temperature, x, v, forces, gauss=None, split=None, tol=1e-12):
    """One Verlet (0) / Langevin (1) / LangevinMiddle (2) step with the random force `gauss` [n, 3] (None: none) at
    `temperature`; SETTLE for the rigid waters, CCMA in double to `tol` for every other constraint (split: constraint_split(desc),
    computed when not given).  x, v modified in place; returns the most CCMA iterations a solve used (-1: no convergence)."""
    L = lib()
    (a0, a1, a2, d1, d2), (ai, aj, dist) = split or constraint_split(desc)
    assert x.dtype == np.float64 and v.dtype == np.float64 and x.flags.c_contiguous and v.flags.c_contiguous
    g = None if gauss is None else _d(gauss)
    return L.orc_langevin_step(kind, desc.natoms, dt, friction, BOLTZ*temperature, _dp(_d(desc.masses)), _dp(_d(forces)),
                               None if g is None else _dp(g), _dp(x), _dp(v), len(a0), _ip(a0), _ip(a1), _ip(a2), _dp(d1), _dp(d2),
                               len(ai), _ip(ai), _ip(aj), _dp(dist), tol)


def fft3d_forward(x):
    L = lib()
    re = _d(x.real).copy()
    im = _d(x.imag).copy() if np.iscomplexobj(x) else np.zeros_like(re)
    nx, ny, nz = x.shape
    L.orc_fft3d_forward(nx, ny, nz, _dp(re), _dp(im))
    return re + 1j*im
