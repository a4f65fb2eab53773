"""Harness of the custom-bond and custom-external tests: the plugin's expression translator (plugin/custom_translate.h) for the
three classes, Lepton's own evaluation of the same expressions with the Reference platform's periodicdistance, and the
reference's CustomBondForce and CustomExternalForce added to the System a custom_torsion_harness Simulation builds.  ctypes
over oracle/_ref/tests/libcustom_terms_capi.so (plugin/tests/custom_terms_capi.cpp)."""
import copy
import ctypes as C
import os
import numpy as np
import custom_torsion_harness
from custom_torsion_harness import omm, Refused, _dp, _ip, _names

LIB = os.path.join(omm.REF_DIR, "tests", "libcustom_terms_capi.so")
TORSION, BOND, EXTERNAL = 0, 1, 2
NUM_VARS = {TORSION: 1, BOND: 1, EXTERNAL: 3}
_lib = None


def available():
    return custom_torsion_harness.available() and os.path.exists(LIB)


def lib():
    global _lib
    if _lib is None:
        omm.lib()
        L = C.CDLL(LIB)
        P, D, I, S = C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_int), C.c_char_p
        L.cterm_last_error.restype = S
        L.cterm_last_error.argtypes = []
        L.cterm_translate.restype = C.c_int
        L.cterm_translate.argtypes = [C.c_int, S, S, S, C.c_int, I, I, D, I]
        L.cterm_lepton_eval.restype = C.c_int
        L.cterm_lepton_eval.argtypes = [C.c_int, S, C.c_int, D, D, S, D, S, D, D]
        L.cterm_add_custom_bonds.restype = C.c_int
        L.cterm_add_custom_bonds.argtypes = [P, S, S, S, D, C.c_int, I, D, C.c_int, C.c_int, S]
        L.cterm_add_custom_externals.restype = C.c_int
        L.cterm_add_custom_externals.argtypes = [P, S, S, S, D, C.c_int, I, D, C.c_int]
        for name in ("cterm_update_custom_bonds", "cterm_update_custom_externals"):
            getattr(L, name).restype = C.c_int
            getattr(L, name).argtypes = [P, C.c_int, P, C.c_int, I, D]
        _lib = L
    return _lib


def translate(cls, energy, params=(), globals_=()):
    """(op, arg, imm, starts): the energy program and one derivative program per variable of class cls, as the plugin makes
    them; starts = the prog_start of this one expression"""
    cap = 8192
    op, arg, imm = np.zeros(cap, np.int32), np.zeros(cap, np.int32), np.zeros(cap)
    counts = np.zeros(8, np.int32)
    n = lib().cterm_translate(cls, energy.encode(), _names(params), _names(globals_), cap, _ip(op), _ip(arg), _dp(imm), _ip(counts))
    if n == -2:
        raise Refused(lib().cterm_last_error().decode())
    if n < 0:
        raise ValueError(lib().cterm_last_error().decode())
    starts = np.concatenate([[0], np.cumsum(counts[:n])]).astype(np.int32)
    return op[:starts[-1]].copy(), arg[:starts[-1]].copy(), imm[:starts[-1]].copy(), starts


def lepton(cls, energy, which, variables, box=np.eye(3), params=(), pvals=(), globals_=(), gvals=()):
    """ExpressionProgram::evaluate of the energy (which 0) or its derivative by variable which-1"""
    out = C.c_double()
    v, b = np.ascontiguousarray(variables, dtype=np.float64), np.ascontiguousarray(box, dtype=np.float64).reshape(9)
    pv, gv = np.ascontiguousarray(pvals, dtype=np.float64).reshape(-1), np.ascontiguousarray(gvals, dtype=np.float64).reshape(-1)
    if not len(pv):
        pv = np.zeros(1)
    if not len(gv):
        gv = np.zeros(1)
    if lib().cterm_lepton_eval(cls, energy.encode(), int(which), _dp(v), _dp(b), _names(params), _dp(pv), _names(globals_), _dp(gv),
                               C.byref(out)) != 0:
        raise ValueError(lib().cterm_last_error().decode())
    return out.value


def compiled(desc):
    """desc with the programs of its custom torsions, bonds and externals, from the plugin's translator"""
    d = custom_torsion_harness.compiled(desc)
    for prefix, cls in (("cbond", BOND), ("cext", EXTERNAL)):
        start, op, arg, imm = [0], [], [], []
        for p, energy in enumerate(getattr(desc, prefix + "_energy")):
            o, a, i, s = translate(cls, energy, getattr(desc, prefix + "_param_names")[p], desc.custom_global_names)
            op += o.tolist()
            arg += a.tolist()
            imm += i.tolist()
            start += (start[-1] + s[1:]).tolist()
        setattr(d, prefix + "_prog_start", np.array(start if getattr(desc, prefix + "_energy") else [], dtype=np.int32))
        setattr(d, prefix + "_op", np.array(op, np.int32))
        setattr(d, prefix + "_arg", np.array(arg, np.int32))
        setattr(d, prefix + "_imm", np.array(imm, np.float64))
    return d


class Simulation(custom_torsion_harness.Simulation):
    """custom_torsion_harness.Simulation of desc plus one CustomBondForce per desc.cbond_energy and one CustomExternalForce per
    desc.cext_energy (each declares every global of desc.custom_global_names).  force_groups["custom_bonds"] and
    ["custom_externals"] put them in a group; bonded_periodic also applies to the bonds; deriv_param asks for the energy
    derivative by that global of the bonds."""

    def __init__(self, desc, platform="Reference", integrator=(0, 0.0, 0.0, 0.001), seed=7, constraint_tol=1e-5,
                 force_groups=None, bonded_periodic=False, deriv_param="", **kw):
        super().__init__(desc, platform, integrator=integrator, seed=seed, constraint_tol=constraint_tol, force_groups=force_groups,
                         bonded_periodic=bonded_periodic, **kw)
        self.cbond_forces, self.cext_forces = [], []
        if not desc.cbond_energy and not desc.cext_energy:
            return
        if self.ctx:
            self.L.omm_context_destroy(self.ctx)
            self.ctx = None
        self.L.omm_integrator_destroy(self.integ)
        kind, T, fric, dt = integrator
        self.integ = self.L.omm_integrator_create(kind, T, fric, dt, seed, constraint_tol)
        gv = np.ascontiguousarray(desc.custom_global_values, dtype=np.float64)
        if not len(gv):
            gv = np.zeros(1)
        groups = force_groups or {}
        for prefix in ("cbond", "cext"):
            for p, energy in enumerate(getattr(desc, prefix + "_energy")):
                sel = np.nonzero(np.asarray(getattr(desc, prefix + "_prog")) == p)[0]
                atoms = np.ascontiguousarray(np.asarray(getattr(desc, prefix + "_atoms"))[sel], dtype=np.int32)
                names = getattr(desc, prefix + "_param_names")[p]
                pv = np.ascontiguousarray(np.asarray(getattr(desc, prefix + "_params"))[sel][:, :len(names)], dtype=np.float64)
                if not pv.size:
                    pv = np.zeros(1)
                if prefix == "cbond":
                    self.cbond_forces.append(lib().cterm_add_custom_bonds(
                        self.sys, energy.encode(), _names(names), _names(desc.custom_global_names), _dp(gv), len(sel), _ip(atoms), _dp(pv),
                        int(bonded_periodic), groups.get("custom_bonds", 0), deriv_param.encode()))
                else:
                    self.cext_forces.append(lib().cterm_add_custom_externals(
                        self.sys, energy.encode(), _names(names), _names(desc.custom_global_names), _dp(gv), len(sel), _ip(atoms), _dp(pv),
                        groups.get("custom_externals", 0)))
        props = kw.get("props", "")
        self.ctx = self.L.omm_context_create(self.sys, self.integ, platform.encode(), props.encode())
        if not self.ctx:
            raise RuntimeError("Context creation failed: " + self.L.omm_last_error().decode())
        self.set_positions(desc.positions)

    def update(self, prefix, p, atoms, params):
        """Force p of the class ("cbond" or "cext") gets these terms, then updateParametersInContext"""
        a = np.ascontiguousarray(atoms, dtype=np.int32)
        v = np.ascontiguousarray(params, dtype=np.float64)
        call = lib().cterm_update_custom_bonds if prefix == "cbond" else lib().cterm_update_custom_externals
        forces = self.cbond_forces if prefix == "cbond" else self.cext_forces
        if call(self.sys, forces[p], self.ctx, len(a), _ip(a), _dp(v)) != 0:
            raise RuntimeError(lib().cterm_last_error().decode())


def probe(cls, start, op, arg, imm, stride, nglobals, which, variables, box, params, globals_):
    """b200md_custom_term_probe: (value, None) or (None, message)"""
    from openmm_b200 import _lib

    def ints(a):
        a = np.ascontiguousarray(a, dtype=np.int32)
        return a, a.ctypes.data_as(C.POINTER(C.c_int))

    def dbls(a):
        a = np.ascontiguousarray(a, dtype=np.float64).reshape(-1)
        if not len(a):
            a = np.zeros(1)
        return a, a.ctypes.data_as(C.POINTER(C.c_double))
    keep = [ints(start), ints(op), ints(arg), dbls(imm), dbls(variables), dbls(box), dbls(params), dbls(globals_)]
    out, msg = C.c_double(), C.create_string_buffer(256)
    nprog = (len(start) - 1)//(1 + NUM_VARS[cls])
    rc = _lib.load().b200md_custom_term_probe(cls, nprog, keep[0][1], keep[1][1], keep[2][1], keep[3][1], stride, nglobals, which,
                                              keep[4][1], keep[5][1], keep[6][1], keep[7][1], C.byref(out), msg, 256)
    return (out.value, None) if rc == 0 else (None, msg.value.decode())
