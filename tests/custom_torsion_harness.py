"""Harness of the custom-torsion tests: the plugin's expression translator (plugin/custom_translate.h), Lepton's own evaluation of
the same expressions, and the reference's CustomTorsionForce added to the System an oracle/omm.py Simulation builds.  ctypes
over oracle/_ref/tests/libcustom_torsion_capi.so (plugin/tests/custom_torsion_capi.cpp)."""
import copy
import ctypes as C
import os
import numpy as np
from oracle import omm
import cmap_rb_harness

LIB = os.path.join(omm.REF_DIR, "tests", "libcustom_torsion_capi.so")
_lib = None


class Refused(ValueError):
    """an expression the platform does not run (the plugin's validateSystem refuses it)"""


def available():
    return omm.available() and os.path.exists(LIB)


def lib():
    global _lib
    if _lib is None:
        omm.lib()                                   # libOpenMM.so, loaded globally
        L = C.CDLL(LIB)
        P, D, I, S = C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_int), C.c_char_p
        L.ct_last_error.restype = S
        L.ct_last_error.argtypes = []
        L.ct_translate.restype = C.c_int
        L.ct_translate.argtypes = [S, S, S, C.c_int, I, I, D, I, I]
        L.ct_lepton_eval.restype = C.c_int
        L.ct_lepton_eval.argtypes = [S, C.c_int, C.c_double, S, D, S, D, D]
        L.ct_add_custom_torsions.restype = C.c_int
        L.ct_add_custom_torsions.argtypes = [P, S, S, S, D, C.c_int, I, D, C.c_int, C.c_int, S]
        L.ct_update_custom_torsions.restype = C.c_int
        L.ct_update_custom_torsions.argtypes = [P, C.c_int, P, C.c_int, I, D]
        L.ct_default_platform.restype = S
        L.ct_default_platform.argtypes = [P]
        _lib = L
    return _lib


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def _ip(a):
    return a.ctypes.data_as(C.POINTER(C.c_int))


def _names(seq):
    return ",".join(seq).encode()


def translate(energy, params=(), globals_=()):
    """(op, arg, imm, n_energy): the energy program followed by the dE/dtheta program, as the plugin makes them; global slot s
    is globals_[s]"""
    cap = 4096
    op, arg, imm = np.zeros(cap, np.int32), np.zeros(cap, np.int32), np.zeros(cap)
    ne, nd = C.c_int(), C.c_int()
    rc = lib().ct_translate(energy.encode(), _names(params), _names(globals_), cap, _ip(op), _ip(arg), _dp(imm), C.byref(ne), C.byref(nd))
    if rc == -2:
        raise Refused(lib().ct_last_error().decode())
    if rc != 0:
        raise ValueError(lib().ct_last_error().decode())
    n = ne.value + nd.value
    return op[:n].copy(), arg[:n].copy(), imm[:n].copy(), ne.value


def lepton(energy, deriv, theta, params=(), pvals=(), globals_=(), gvals=()):
    """ExpressionProgram::evaluate of the energy (deriv False) or dE/dtheta (deriv True)"""
    out = C.c_double()
    pv, gv = np.ascontiguousarray(pvals, dtype=np.float64).reshape(-1), np.ascontiguousarray(gvals, dtype=np.float64).reshape(-1)
    if lib().ct_lepton_eval(energy.encode(), int(deriv), float(theta), _names(params), _dp(pv), _names(globals_), _dp(gv), C.byref(out)) != 0:
        raise ValueError(lib().ct_last_error().decode())
    return out.value


def compiled(desc):
    """desc with custom_prog_start / op / arg / imm: the programs of its expressions, from the plugin's translator"""
    d = copy.copy(desc)
    start, op, arg, imm = [0], [], [], []
    for p, energy in enumerate(desc.custom_energy):
        o, a, i, ne = translate(energy, desc.custom_param_names[p], desc.custom_global_names)
        op += o.tolist()
        arg += a.tolist()
        imm += i.tolist()
        start += [start[-1] + ne, start[-1] + len(o)]
    d.custom_prog_start = np.array(start if desc.custom_energy else [], dtype=np.int32)
    d.custom_op, d.custom_arg, d.custom_imm = np.array(op, np.int32), np.array(arg, np.int32), np.array(imm, np.float64)
    return d


class Simulation(cmap_rb_harness.Simulation):
    """cmap_rb_harness.Simulation of desc plus one CustomTorsionForce per expression of desc (each declares every global of
    desc.custom_global_names, with desc.custom_global_values as defaults).  force_groups["custom_torsions"] puts them in a
    group; bonded_periodic also applies to them; deriv_param asks for the energy derivative by that global."""

    def __init__(self, desc, platform="Reference", integrator=(0, 0.0, 0.0, 0.001), seed=7, constraint_tol=1e-5,
                 force_groups=None, bonded_periodic=False, deriv_param="", **kw):
        super().__init__(desc, platform, integrator=integrator, seed=seed, constraint_tol=constraint_tol,
                         force_groups=force_groups, bonded_periodic=bonded_periodic, **kw)
        self.custom_forces = []
        if not desc.custom_energy:          # a CustomTorsionForce without torsions is still added
            return
        self.L.omm_context_destroy(self.ctx)
        self.ctx = None
        self.L.omm_integrator_destroy(self.integ)
        kind, T, fric, dt = integrator
        self.integ = self.L.omm_integrator_create(kind, T, fric, dt, seed, constraint_tol)
        gv = np.ascontiguousarray(desc.custom_global_values, dtype=np.float64)
        group = (force_groups or {}).get("custom_torsions", 0)
        for p, energy in enumerate(desc.custom_energy):
            sel = np.nonzero(np.asarray(desc.custom_prog) == p)[0]
            atoms = np.ascontiguousarray(np.asarray(desc.custom_atoms)[sel], dtype=np.int32)
            npar = len(desc.custom_param_names[p])
            pv = np.ascontiguousarray(np.asarray(desc.custom_params)[sel][:, :npar], dtype=np.float64)
            self.custom_forces.append(lib().ct_add_custom_torsions(self.sys, energy.encode(), _names(desc.custom_param_names[p]),
                                                                   _names(desc.custom_global_names), _dp(gv), len(sel), _ip(atoms), _dp(pv),
                                                                   int(bonded_periodic), group, deriv_param.encode()))
        props = kw.get("props", "")
        self.ctx = self.L.omm_context_create(self.sys, self.integ, platform.encode(), props.encode())
        if not self.ctx:
            raise RuntimeError("Context creation failed: " + self.L.omm_last_error().decode())
        self.set_positions(desc.positions)

    def default_platform(self):
        """the platform a Context of this System gets when none is named"""
        return lib().ct_default_platform(self.sys).decode()

    def update_custom_torsions(self, p, atoms, params):
        """CustomTorsionForce p gets these torsions (atoms [n,4], params [n, its parameters]), then updateParametersInContext"""
        a = np.ascontiguousarray(atoms, dtype=np.int32)
        v = np.ascontiguousarray(params, dtype=np.float64)
        if lib().ct_update_custom_torsions(self.sys, self.custom_forces[p], self.ctx, len(a), _ip(a), _dp(v)) != 0:
            raise RuntimeError(lib().ct_last_error().decode())
