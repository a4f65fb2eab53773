"""Reference-side harness of the RB torsion and CMAP tests: the reference's own RBTorsionForce and CMAPTorsionForce, added to
the System an oracle/omm.py Simulation builds, and the reference's CMAP spline fitter (CMAPTorsionForceImpl::
calcMapDerivatives).  ctypes over oracle/_ref/tests/libcmap_rb_capi.so (plugin/tests/cmap_rb_capi.cpp)."""
import ctypes as C
import os
import numpy as np
from oracle import omm

LIB = os.path.join(omm.REF_DIR, "tests", "libcmap_rb_capi.so")
_lib = None


def available():
    return omm.available() and os.path.exists(LIB)


def lib():
    global _lib
    if _lib is None:
        omm.lib()                                   # libOpenMM.so, loaded globally
        L = C.CDLL(LIB)
        P, D, I = C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_int)
        L.cmap_rb_add_rb_torsions.restype = C.c_int
        L.cmap_rb_add_rb_torsions.argtypes = [P, C.c_int, I, I, I, I, D, C.c_int, C.c_int]
        L.cmap_rb_add_cmap.restype = C.c_int
        L.cmap_rb_add_cmap.argtypes = [P, C.c_int, I, D, C.c_int, I, I, C.c_int, C.c_int]
        L.cmap_rb_coefficients.restype = None
        L.cmap_rb_coefficients.argtypes = [C.c_int, D, D]
        _lib = L
    return _lib


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def _ip(a):
    return a.ctypes.data_as(C.POINTER(C.c_int))


def coefficients(size, energy):
    """[size^2, 16] bicubic coefficients of one map, from the reference's fitter"""
    out = np.zeros((size*size, 16))
    lib().cmap_rb_coefficients(int(size), _dp(np.ascontiguousarray(energy, dtype=np.float64)), _dp(out))
    return out


class Simulation(omm.Simulation):
    """omm.Simulation of desc plus its RB torsions and CMAP terms (desc.rb_*, desc.cmap_*).  force_groups = {"rb_torsions": g,
    "cmap": g} puts those forces in group g; bonded_periodic also applies to them."""

    def __init__(self, desc, platform="Reference", integrator=(0, 0.0, 0.0, 0.001), seed=7, constraint_tol=1e-5,
                 force_groups=None, bonded_periodic=False, **kw):
        self.force_groups, self.bonded_periodic = force_groups or {}, bonded_periodic
        super().__init__(desc, platform, integrator=integrator, seed=seed, constraint_tol=constraint_tol,
                         bonded_periodic=bonded_periodic, **kw)

    def add_forces(self):
        desc, groups, per = self.desc, self.force_groups, int(self.bonded_periodic)
        i32 = lambda a: np.ascontiguousarray(a, dtype=np.int32)
        f64 = lambda a: np.ascontiguousarray(a, dtype=np.float64)
        if len(desc.rb_i):
            lib().cmap_rb_add_rb_torsions(self.sys, len(desc.rb_i), _ip(i32(desc.rb_i)), _ip(i32(desc.rb_j)), _ip(i32(desc.rb_k)),
                                          _ip(i32(desc.rb_l)), _dp(f64(desc.rb_c)), per, groups.get("rb_torsions", 0))
        if len(desc.cmap_map):
            lib().cmap_rb_add_cmap(self.sys, len(desc.cmap_size), _ip(i32(desc.cmap_size)), _dp(f64(desc.cmap_energy)), len(desc.cmap_map),
                                   _ip(i32(desc.cmap_map)), _ip(i32(desc.cmap_atoms)), per, groups.get("cmap", 0))
