"""Test harness of the RMSDForce and CustomCVForce tests: the golden cases, the engine's host probes of the RMSD arithmetic
(b200md_rmsd_probe, b200md_rmsd_eigen_probe), and the reference's RMSDForce and CustomCVForce over
oracle/_ref/tests/librmsd_capi.so (plugin/tests/rmsd_capi.cpp): added to an oracle.omm.Simulation, or evaluated alone on a
named platform."""
import ctypes as C
import os

import numpy as np

from oracle import omm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "oracle", "_ref", "tests", "librmsd_capi.so")
GOLDEN = os.path.join(ROOT, "tests", "golden", "reference_rmsd.npz")
RMSD_GROUP = 5
_lib = None
D, I, P = C.POINTER(C.c_double), C.POINTER(C.c_int), C.c_void_p


def available():
    return os.path.exists(LIB) and omm.available()


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(LIB)
        L.rmc_add_force.argtypes = [P, C.c_int, I, C.c_int, D, C.c_int]
        L.rmc_add_force.restype = C.c_int
        L.rmc_update.argtypes = [P, C.c_int, P, C.c_int, I, C.c_int, D]
        L.rmc_update.restype = C.c_int
        L.rmc_default_platform.argtypes = [P]
        L.rmc_default_platform.restype = C.c_char_p
        L.rmc_evaluate.argtypes = [C.c_int, D, D, C.c_int, I, C.c_char_p, C.c_char_p, D, D]
        L.rmc_evaluate.restype = C.c_int
        L.rmc_last_error.restype = C.c_char_p
        S = C.c_char_p
        for name, args in (("rmc_add_cv_force", [P, S, C.c_int]), ("rmc_cv_add_rmsd", [P, C.c_int, S, C.c_int, I, C.c_int, D]),
                           ("rmc_cv_add_centroid_distance", [P, C.c_int, S, C.c_int, I, C.c_int, I, C.c_int]),
                           ("rmc_cv_add_torsion", [P, C.c_int, S, C.c_int, C.c_int, C.c_int, C.c_int, S]),
                           ("rmc_cv_add_custom_nonbonded", [P, C.c_int, S, C.c_int]),
                           ("rmc_cv_add_global", [P, C.c_int, S, C.c_double, C.c_int]),
                           ("rmc_cv_set_table2d", [P, C.c_int, S, C.c_int, C.c_int, D, C.c_double, C.c_double, C.c_double, C.c_double]),
                           ("rmc_cv_update", [P, C.c_int, P]), ("rmc_cv_values", [P, C.c_int, P, D])):
            getattr(L, name).argtypes = args
            getattr(L, name).restype = C.c_int
        L.rmc_try_platform.argtypes = [P, S]
        L.rmc_try_platform.restype = C.c_char_p
        _lib = L
    return _lib


def _f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def _i32(a):
    return np.ascontiguousarray(a, dtype=np.int32)


def _dp(a):
    return a.ctypes.data_as(D)


def _ip(a):
    return a.ctypes.data_as(I)


# ---------------------------------------------------------------- the cases
def _rotation(axis, angle):
    a = np.asarray(axis, dtype=np.float64)
    a = a/np.linalg.norm(a)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(angle)*K + (1 - np.cos(angle))*K @ K


def golden_cases():
    """name -> (positions [n, 3], reference positions [n, 3], particles (empty: all)), every one seeded"""
    rng = np.random.default_rng(2004)
    out = {}
    for n in (3, 20, 200, 2000):
        ref = rng.uniform(0.0, 4.0, (n, 3))
        out["random_%d" % n] = (ref + rng.normal(0.0, 0.15, (n, 3)), ref, np.zeros(0, np.int32))
    ref = rng.uniform(-1.5, 1.5, (60, 3))
    out["mirror"] = (ref*np.array([-1.0, 1.0, 1.0]), ref, np.zeros(0, np.int32))
    out["rotated_copy"] = (ref @ _rotation((1, 2, 3), 1.1).T + np.array([0.1, -11.3, 1.5]), ref, np.zeros(0, np.int32))
    x = ref + rng.normal(0.0, 0.1, ref.shape)
    for tag, shift in (("plus50", 50.0), ("minus50", -50.0)):
        out["offset_" + tag] = (x @ _rotation((0, 1, 1), -0.7).T + shift, ref, np.zeros(0, np.int32))
    sub = np.sort(rng.choice(60, 25, replace=False)).astype(np.int32)
    out["subset"] = (x, ref, sub)
    out["subset_all_listed"] = (x, ref, np.arange(60, dtype=np.int32))
    return out


def load_golden():
    g = np.load(GOLDEN)
    names = sorted({k.rsplit("_", 1)[0] for k in g.files})
    return {n: {k: g[n + "_" + k] for k in ("positions", "reference", "particles", "energy", "forces")} for n in names}


# ---------------------------------------------------------------- the engine's host probes
def probe(pos, ref):
    """(rmsd, forces) of the listed positions against their reference positions, by the device arithmetic run on the host"""
    from openmm_b200 import _lib as elib
    L = elib.load()
    pos, ref = _f64(pos), _f64(ref)
    e = np.zeros(1)
    f = np.zeros_like(pos)
    assert L.b200md_rmsd_probe(len(pos), _dp(pos), _dp(ref), _dp(e), _dp(f)) == 0
    return float(e[0]), f


def probe_full(pos, ref, particles):
    """probe() of an RMSDForce over `particles` (empty: all) of a System: its energy and the forces on every particle"""
    p = np.arange(len(pos)) if len(particles) == 0 else np.asarray(particles)
    e, fp = probe(np.asarray(pos)[p], np.asarray(ref)[p])
    f = np.zeros((len(pos), 3))
    f[p] = fp
    return e, f


def eigen_probe(a):
    """(largest eigenvalue, unit eigenvector, sweeps) of the symmetric 4x4 matrix a by the device's Jacobi iteration"""
    from openmm_b200 import _lib as elib
    L = elib.load()
    a = _f64(a).reshape(16)
    lam, q = np.zeros(1), np.zeros(4)
    sweeps = L.b200md_rmsd_eigen_probe(_dp(a), _dp(lam), _dp(q))
    return float(lam[0]), q, sweeps


# ---------------------------------------------------------------- the reference
def evaluate(pos, ref, particles, platform="Reference", precision=""):
    """(energy, forces) of one RMSDForce alone in a System of unit masses, on the named platform"""
    pos, ref, p = _f64(pos), _f64(ref), _i32(particles)
    e = np.zeros(1)
    f = np.zeros_like(pos)
    if lib().rmc_evaluate(len(pos), _dp(pos), _dp(ref), len(p), _ip(p), platform.encode(), precision.encode(), _dp(e), _dp(f)) != 0:
        raise RuntimeError(lib().rmc_last_error().decode())
    return float(e[0]), f


class Simulation(omm.Simulation):
    """oracle.omm.Simulation plus one RMSDForce per entry of rmsd = [(particles, reference positions [natoms, 3], group)]"""

    def __init__(self, desc, platform="Reference", rmsd=(), **kw):
        self.rmsd_specs = list(rmsd)
        super().__init__(desc, platform, **kw)

    def add_forces(self):
        super().add_forces()
        self.rmsd_index = []
        for particles, ref, group in self.rmsd_specs:
            p, r = _i32(particles), _f64(ref)
            k = lib().rmc_add_force(self.sys, len(p), _ip(p), len(r), _dp(r), int(group))
            if k < 0:
                raise RuntimeError(lib().rmc_last_error().decode())
            self.rmsd_index.append(k)

    def update_rmsd(self, which, particles, ref):
        p, r = _i32(particles), _f64(ref)
        if lib().rmc_update(self.sys, self.rmsd_index[which], self.ctx, len(p), _ip(p), len(r), _dp(r)) != 0:
            raise RuntimeError(lib().rmc_last_error().decode())

    def default_platform(self):
        return lib().rmc_default_platform(self.sys).decode()


CV_GROUP = 7


class CVSimulation(omm.Simulation):
    """oracle.omm.Simulation plus one CustomCVForce in force group CV_GROUP: energy = cv["energy"]; cv["variables"] a list of
    ("rmsd", name, particles, reference [natoms, 3]), ("centroid", name, group1, group2, periodic), ("torsion", name, a, b, c, d,
    global name or ""), ("custom_nonbonded", name); cv["globals"] [(name, value, derivative)]; cv["table"] (name, xsize, ysize,
    values, xmin, xmax, ymin, ymax) or None"""

    def __init__(self, desc, platform="Reference", cv=None, **kw):
        self.cv = cv
        super().__init__(desc, platform, **kw)

    def _cvck(self, rc):
        if rc < 0:
            raise RuntimeError(lib().rmc_last_error().decode() or self.L.omm_last_error().decode())
        return rc

    def add_forces(self):
        super().add_forces()
        L, cv = lib(), self.cv
        self.cv_index = self._cvck(L.rmc_add_cv_force(self.sys, cv["energy"].encode(), CV_GROUP))
        for v in cv["variables"]:
            kind, name = v[0], v[1].encode()
            if kind == "rmsd":
                p, r = _i32(v[2]), _f64(v[3])
                self._cvck(L.rmc_cv_add_rmsd(self.sys, self.cv_index, name, len(p), _ip(p), len(r), _dp(r)))
            elif kind == "centroid":
                g1, g2 = _i32(v[2]), _i32(v[3])
                self._cvck(L.rmc_cv_add_centroid_distance(self.sys, self.cv_index, name, len(g1), _ip(g1), len(g2), _ip(g2), int(v[4])))
            elif kind == "torsion":
                self._cvck(L.rmc_cv_add_torsion(self.sys, self.cv_index, name, *[int(a) for a in v[2:6]], v[6].encode()))
            else:
                self._cvck(L.rmc_cv_add_custom_nonbonded(self.sys, self.cv_index, name, self.n))
        for name, value, deriv in cv.get("globals", ()):
            self._cvck(L.rmc_cv_add_global(self.sys, self.cv_index, name.encode(), value, int(deriv)))
        if cv.get("table") is not None:
            self.set_table(*cv["table"], update=False)

    def set_table(self, name, xsize, ysize, values, xmin, xmax, ymin, ymax, update=True):
        v = _f64(values)
        self._cvck(lib().rmc_cv_set_table2d(self.sys, self.cv_index, name.encode(), xsize, ysize, _dp(v), xmin, xmax, ymin, ymax))
        if update:
            self._cvck(lib().rmc_cv_update(self.sys, self.cv_index, self.ctx))

    def cv_values(self):
        out = np.zeros(32)
        n = self._cvck(lib().rmc_cv_values(self.sys, self.cv_index, self.ctx, _dp(out)))
        return out[:n]

    def try_platform(self, platform=""):
        """platform empty: the platform a Context of this System gets; else "" if one can be made on it, or the error"""
        return lib().rmc_try_platform(self.sys, platform.encode()).decode()


def force_error(f, ref):
    """max over atoms of max|df| / max(1, |f_ref|)"""
    return float((np.abs(f - ref).max(axis=1)/np.maximum(1.0, np.linalg.norm(ref, axis=1))).max())
