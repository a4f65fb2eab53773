"""Harness of the custom-angle and custom-compound-bond tests: the plugin's expression translator (plugin/custom_translate.h)
for the two classes, Lepton's own evaluation of the same expressions with the Reference platform's point functions, and the
reference's CustomAngleForce and CustomCompoundBondForce added to the System a custom_terms_harness Simulation builds.
ctypes over oracle/_ref/tests/libcustom_compound_capi.so (plugin/tests/custom_compound_capi.cpp)."""
import ctypes as C
import os
import numpy as np
import custom_terms_harness
from custom_terms_harness import omm, Refused, _dp, _ip, _names

LIB = os.path.join(omm.REF_DIR, "tests", "libcustom_compound_capi.so")
ANGLE = 3
_lib = None


def available():
    return custom_terms_harness.available() and os.path.exists(LIB)


def lib():
    global _lib
    if _lib is None:
        omm.lib()
        L = C.CDLL(LIB)
        P, D, I, S = C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_int), C.c_char_p
        L.ccomp_last_error.restype = S
        L.ccomp_last_error.argtypes = []
        L.ccomp_translate.restype = C.c_int
        L.ccomp_translate.argtypes = [C.c_int, S, S, S, C.c_int, C.c_int, I, I, D, I]
        L.ccomp_lepton_eval.restype = C.c_int
        L.ccomp_lepton_eval.argtypes = [C.c_int, S, C.c_int, D, D, C.c_int, S, D, S, D, D]
        L.ccomp_add_custom_angles.restype = C.c_int
        L.ccomp_add_custom_angles.argtypes = [P, S, S, S, D, C.c_int, I, D, C.c_int, C.c_int, S]
        L.ccomp_add_compound.restype = C.c_int
        L.ccomp_add_compound.argtypes = [P, C.c_int, S, S, S, D, C.c_int, I, D, C.c_int, C.c_int, C.c_int, S]
        for name in ("ccomp_update_custom_angles", "ccomp_update_compound"):
            getattr(L, name).restype = C.c_int
            getattr(L, name).argtypes = [P, C.c_int, P, C.c_int, I, D]
        _lib = L
    return _lib


def translate(nparticles, energy, params=(), globals_=(), tabulated=False):
    """(op, arg, imm, starts): the programs of a CustomAngleForce expression (nparticles 0: energy, dE/dtheta) or of a
    CustomCompoundBondForce of nparticles particles per bond (energy, then the derivatives by x1, y1, z1, x2, ..), as the
    plugin makes them; starts = the prog_start of this one expression"""
    cap = 65536
    op, arg, imm = np.zeros(cap, np.int32), np.zeros(cap, np.int32), np.zeros(cap)
    counts = np.zeros(32, np.int32)
    n = lib().ccomp_translate(nparticles, energy.encode(), _names(params), _names(globals_), int(tabulated), cap, _ip(op), _ip(arg),
                              _dp(imm), _ip(counts))
    if n == -2:
        raise Refused(lib().ccomp_last_error().decode())
    if n < 0:
        raise ValueError(lib().ccomp_last_error().decode())
    starts = np.concatenate([[0], np.cumsum(counts[:n])]).astype(np.int32)
    return op[:starts[-1]].copy(), arg[:starts[-1]].copy(), imm[:starts[-1]].copy(), starts


def _vec(a):
    a = np.ascontiguousarray(a, dtype=np.float64).reshape(-1)
    return a if len(a) else np.zeros(1)


def lepton(nparticles, energy, which, variables, box=np.eye(3), periodic=False, params=(), pvals=(), globals_=(), gvals=()):
    """ExpressionProgram::evaluate of the energy (which 0) or its derivative by variable which-1, a compound bond's with the
    Reference platform's point functions"""
    out = C.c_double()
    if lib().ccomp_lepton_eval(nparticles, energy.encode(), int(which), _dp(_vec(variables)), _dp(_vec(box)), int(periodic), _names(params),
                               _dp(_vec(pvals)), _names(globals_), _dp(_vec(gvals)), C.byref(out)) != 0:
        raise ValueError(lib().ccomp_last_error().decode())
    return out.value


def probe(nparticles, periodic, start, op, arg, imm, stride, nglobals, which, variables, box, params, globals_):
    """b200md_custom_compound_probe (nparticles > 0) or b200md_custom_term_probe of the angle class: (value, None) or
    (None, message)"""
    from openmm_b200 import _lib as native
    ints = [np.ascontiguousarray(a, dtype=np.int32) for a in (start, op, arg)]
    dbls = [_vec(a) for a in (imm, variables, box, params, globals_)]
    out, msg = C.c_double(), C.create_string_buffer(256)
    head = (nparticles, int(periodic)) if nparticles > 0 else (ANGLE, (len(start) - 1)//2)
    call = native.load().b200md_custom_compound_probe if nparticles > 0 else native.load().b200md_custom_term_probe
    rc = call(*head, _ip(ints[0]), _ip(ints[1]), _ip(ints[2]), _dp(dbls[0]), stride, nglobals, which, _dp(dbls[1]), _dp(dbls[2]),
              _dp(dbls[3]), _dp(dbls[4]), C.byref(out), msg, 256)
    return (out.value, None) if rc == 0 else (None, msg.value.decode())


def compiled(desc):
    """desc with the programs of all its custom classes, from the plugin's translator"""
    d = custom_terms_harness.compiled(desc)
    for prefix in ("cangle", "ccompound"):
        start, op, arg, imm = [0], [], [], []
        for p, energy in enumerate(getattr(desc, prefix + "_energy")):
            nparticles = int(desc.ccompound_particles[p]) if prefix == "ccompound" else 0
            o, a, i, s = translate(nparticles, energy, getattr(desc, prefix + "_param_names")[p], desc.custom_global_names)
            op += o.tolist()
            arg += a.tolist()
            imm += i.tolist()
            start += (start[-1] + s[1:]).tolist()
        setattr(d, prefix + "_prog_start", np.array(start if getattr(desc, prefix + "_energy") else [], dtype=np.int32))
        setattr(d, prefix + "_op", np.array(op, np.int32))
        setattr(d, prefix + "_arg", np.array(arg, np.int32))
        setattr(d, prefix + "_imm", np.array(imm, np.float64))
    return d


class Simulation(custom_terms_harness.Simulation):
    """custom_terms_harness.Simulation of desc plus one CustomAngleForce per desc.cangle_energy and one CustomCompoundBondForce
    per desc.ccompound_energy (each declares every global of desc.custom_global_names).  force_groups["custom_angles"] and
    ["custom_compound"] put them in a group; bonded_periodic also applies to the angles; tabulated gives every compound force a
    tabulated function; deriv_param asks for the energy derivative by that global of the compound forces."""

    def __init__(self, desc, platform="Reference", integrator=(0, 0.0, 0.0, 0.001), seed=7, constraint_tol=1e-5,
                 force_groups=None, bonded_periodic=False, tabulated=False, compound_deriv_param="", **kw):
        bare = platform if not (desc.cangle_energy or desc.ccompound_energy) else "Reference"
        super().__init__(desc, bare, integrator=integrator, seed=seed, constraint_tol=constraint_tol, force_groups=force_groups,
                         bonded_periodic=bonded_periodic, **kw)
        self.cangle_forces, self.ccompound_forces = [], []
        if not desc.cangle_energy and not desc.ccompound_energy:
            return
        if self.ctx:
            self.L.omm_context_destroy(self.ctx)
            self.ctx = None
        self.L.omm_integrator_destroy(self.integ)
        kind, T, fric, dt = integrator
        self.integ = self.L.omm_integrator_create(kind, T, fric, dt, seed, constraint_tol)
        gv = _vec(desc.custom_global_values)
        groups = force_groups or {}
        for p, energy in enumerate(desc.cangle_energy):
            sel = np.nonzero(np.asarray(desc.cangle_prog) == p)[0]
            atoms = np.ascontiguousarray(np.asarray(desc.cangle_atoms)[sel], dtype=np.int32)
            names = desc.cangle_param_names[p]
            pv = _vec(np.asarray(desc.cangle_params)[sel][:, :len(names)])
            self.cangle_forces.append(lib().ccomp_add_custom_angles(
                self.sys, energy.encode(), _names(names), _names(desc.custom_global_names), _dp(gv), len(sel), _ip(atoms), _dp(pv),
                int(bonded_periodic), groups.get("custom_angles", 0), b""))
        for p, energy in enumerate(desc.ccompound_energy):
            sel = np.nonzero(np.asarray(desc.ccompound_expr) == p)[0]
            w = int(desc.ccompound_particles[p])
            atoms = np.ascontiguousarray(np.asarray(desc.ccompound_atoms)[sel][:, :w], dtype=np.int32)
            names = desc.ccompound_param_names[p]
            pv = _vec(np.asarray(desc.ccompound_params)[sel][:, :len(names)])
            self.ccompound_forces.append(lib().ccomp_add_compound(
                self.sys, w, energy.encode(), _names(names), _names(desc.custom_global_names), _dp(gv), len(sel), _ip(atoms), _dp(pv),
                int(desc.ccompound_periodic[p]), groups.get("custom_compound", 0), int(tabulated), compound_deriv_param.encode()))
        props = kw.get("props", "")
        self.ctx = self.L.omm_context_create(self.sys, self.integ, platform.encode(), props.encode())
        if not self.ctx:
            raise RuntimeError("Context creation failed: " + self.L.omm_last_error().decode())
        self.set_positions(desc.positions)

    def update(self, prefix, p, atoms, params):
        """Force p of the class ("cangle" or "ccompound") gets these terms, then updateParametersInContext"""
        if prefix not in ("cangle", "ccompound"):
            return super().update(prefix, p, atoms, params)
        a = np.ascontiguousarray(atoms, dtype=np.int32)
        v = np.ascontiguousarray(params, dtype=np.float64)
        call = lib().ccomp_update_custom_angles if prefix == "cangle" else lib().ccomp_update_compound
        forces = self.cangle_forces if prefix == "cangle" else self.ccompound_forces
        if call(self.sys, forces[p], self.ctx, len(a), _ip(a), _dp(v)) != 0:
            raise RuntimeError(lib().ccomp_last_error().decode())
