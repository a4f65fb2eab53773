"""Harness of the custom-force tests, for every custom class (TORSION, BOND, EXTERNAL, ANGLE, COMPOUND): the plugin's
expression translator (plugin/custom_translate.h), Lepton's own evaluation of the same expressions with the Reference
platform's periodicdistance and point functions, the engine's program probes, and the reference's custom Force classes added
to the System a cmap_rb_harness Simulation builds.  ctypes over oracle/_ref/tests/libcustom_capi.so (plugin/tests/custom_capi.cpp)."""
import copy
import ctypes as C
import os
import numpy as np
from oracle import omm
import cmap_rb_harness

LIB = os.path.join(omm.REF_DIR, "tests", "libcustom_capi.so")
TORSION, BOND, EXTERNAL, ANGLE, COMPOUND = 0, 1, 2, 3, 4
NUM_VARS = {TORSION: 1, BOND: 1, EXTERNAL: 3, ANGLE: 1}
# the custom classes of a SystemDesc: field prefix, class, the field of each term's expression, the key of force_groups
CLASSES = (("custom", TORSION, "custom_prog", "custom_torsions"), ("cbond", BOND, "cbond_prog", "custom_bonds"),
           ("cext", EXTERNAL, "cext_prog", "custom_externals"), ("cangle", ANGLE, "cangle_prog", "custom_angles"),
           ("ccompound", COMPOUND, "ccompound_expr", "custom_compound"))
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
        P, D, I, S, N = C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_int), C.c_char_p, C.c_int
        L.cc_last_error.restype = S
        L.cc_last_error.argtypes = []
        L.cc_translate.restype = N
        L.cc_translate.argtypes = [N, N, S, S, S, N, N, I, I, D, I]
        L.cc_lepton_eval.restype = N
        L.cc_lepton_eval.argtypes = [N, N, S, N, D, D, N, S, D, S, D, D]
        L.cc_add_force.restype = N
        L.cc_add_force.argtypes = [P, N, N, S, S, S, D, N, I, D, N, N, N, S]
        L.cc_update_force.restype = N
        L.cc_update_force.argtypes = [P, N, N, P, N, I, D]
        L.cc_default_platform.restype = S
        L.cc_default_platform.argtypes = [P]
        _lib = L
    return _lib


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def _ip(a):
    return a.ctypes.data_as(C.POINTER(C.c_int))


def _names(seq):
    return ",".join(seq).encode()


def _vec(a):
    a = np.ascontiguousarray(a, dtype=np.float64).reshape(-1)
    return a if len(a) else np.zeros(1)


def translate(cls, energy, params=(), globals_=(), nparticles=0, tabulated=False):
    """(op, arg, imm, starts): the energy program and one derivative program per variable of an expression of class cls (a
    compound bond of nparticles particles per bond: the derivatives by x1, y1, z1, x2, ..), as the plugin makes them; starts =
    the prog_start of this one expression.  tabulated gives a compound force a tabulated function."""
    cap = 65536
    op, arg, imm = np.zeros(cap, np.int32), np.zeros(cap, np.int32), np.zeros(cap)
    counts = np.zeros(32, np.int32)
    n = lib().cc_translate(cls, nparticles, energy.encode(), _names(params), _names(globals_), int(tabulated), cap, _ip(op), _ip(arg), _dp(imm),
                           _ip(counts))
    if n == -2:
        raise Refused(lib().cc_last_error().decode())
    if n < 0:
        raise ValueError(lib().cc_last_error().decode())
    starts = np.concatenate([[0], np.cumsum(counts[:n])]).astype(np.int32)
    return op[:starts[-1]].copy(), arg[:starts[-1]].copy(), imm[:starts[-1]].copy(), starts


def lepton(cls, energy, which, variables, box=np.eye(3), params=(), pvals=(), globals_=(), gvals=(), nparticles=0, periodic=False):
    """ExpressionProgram::evaluate of the energy (which 0) or its derivative by variable which-1, with the Reference
    platform's periodicdistance (externals) and point functions (compound bonds, periodic or not)"""
    out = C.c_double()
    if lib().cc_lepton_eval(cls, nparticles, energy.encode(), int(which), _dp(_vec(variables)), _dp(_vec(box)), int(periodic), _names(params),
                            _dp(_vec(pvals)), _names(globals_), _dp(_vec(gvals)), C.byref(out)) != 0:
        raise ValueError(lib().cc_last_error().decode())
    return out.value


def _probe(call, head, start, op, arg, imm, tail, dbls):
    """call(*head, start, op, arg, imm, *tail, *dbls, out, msg, 256), one of the engine's probes: (value, None) or (None, message)"""
    ints = [np.ascontiguousarray(a, dtype=np.int32) for a in (start, op, arg)]
    dbls = [_vec(a) for a in (imm,) + tuple(dbls)]
    out, msg = C.c_double(), C.create_string_buffer(256)
    rc = call(*head, *[_ip(a) for a in ints], _dp(dbls[0]), *tail, *[_dp(a) for a in dbls[1:]], C.byref(out), msg, 256)
    return (out.value, None) if rc == 0 else (None, msg.value.decode())


def program_probe(start, op, arg, imm, stride, nglobals, which, theta, params, globals_):
    """b200md_custom_program_probe (a custom-torsion program set)"""
    from openmm_b200 import _lib as native
    return _probe(native.load().b200md_custom_program_probe, (len(start)//2,), start, op, arg, imm, (stride, nglobals, which, theta),
                  (params, globals_))


def term_probe(cls, start, op, arg, imm, stride, nglobals, which, variables, box, params, globals_):
    """b200md_custom_term_probe (a program set of class cls)"""
    from openmm_b200 import _lib as native
    return _probe(native.load().b200md_custom_term_probe, (cls, (len(start) - 1)//(1 + NUM_VARS[cls])), start, op, arg, imm,
                  (stride, nglobals, which), (variables, box, params, globals_))


def compound_probe(nparticles, periodic, start, op, arg, imm, stride, nglobals, which, variables, box, params, globals_):
    """b200md_custom_compound_probe (one compound-bond expression of nparticles particles)"""
    from openmm_b200 import _lib as native
    return _probe(native.load().b200md_custom_compound_probe, (nparticles, int(periodic)), start, op, arg, imm, (stride, nglobals, which),
                  (variables, box, params, globals_))


def compiled(desc):
    """desc with the programs of all its custom classes (<prefix>_prog_start / _op / _arg / _imm), from the plugin's translator"""
    d = copy.copy(desc)
    for prefix, cls, _, _ in CLASSES:
        start, op, arg, imm = [0], [], [], []
        energies = getattr(desc, prefix + "_energy")
        for p, energy in enumerate(energies):
            nparticles = int(desc.ccompound_particles[p]) if cls == COMPOUND else 0
            o, a, i, s = translate(cls, energy, getattr(desc, prefix + "_param_names")[p], desc.custom_global_names, nparticles)
            op += o.tolist()
            arg += a.tolist()
            imm += i.tolist()
            start += (start[-1] + s[1:]).tolist()
        setattr(d, prefix + "_prog_start", np.array(start if energies else [], dtype=np.int32))
        setattr(d, prefix + "_op", np.array(op, np.int32))
        setattr(d, prefix + "_arg", np.array(arg, np.int32))
        setattr(d, prefix + "_imm", np.array(imm, np.float64))
    return d


class Simulation(cmap_rb_harness.Simulation):
    """cmap_rb_harness.Simulation of desc plus one custom Force per expression of every custom class of desc (each declares
    every global of desc.custom_global_names, with desc.custom_global_values as defaults; a Force without terms is still
    added), all in the System before its Context is made.  force_groups["custom_torsions"], ["custom_bonds"],
    ["custom_externals"], ["custom_angles"] and ["custom_compound"] put them in a group; bonded_periodic also applies to the
    torsions, bonds and angles (a compound force is periodic as desc.ccompound_periodic says).  deriv_params, keyed alike,
    asks the forces of a class (not the externals) for the energy derivative by that global; tabulated gives every compound
    force a tabulated function."""

    def __init__(self, desc, platform="Reference", integrator=(0, 0.0, 0.0, 0.001), seed=7, constraint_tol=1e-5,
                 force_groups=None, bonded_periodic=False, deriv_params=None, tabulated=False, **kw):
        self.deriv_params = deriv_params or {}
        self.tabulated = tabulated
        self.forces = {prefix: [] for prefix, _, _, _ in CLASSES}
        super().__init__(desc, platform, integrator=integrator, seed=seed, constraint_tol=constraint_tol, force_groups=force_groups,
                         bonded_periodic=bonded_periodic, **kw)

    def add_forces(self):
        super().add_forces()
        desc = self.desc
        gv = _vec(desc.custom_global_values)
        for prefix, cls, expr_field, group in CLASSES:
            for p, energy in enumerate(getattr(desc, prefix + "_energy")):
                sel = np.nonzero(np.asarray(getattr(desc, expr_field)) == p)[0]
                atoms = np.asarray(getattr(desc, prefix + "_atoms"))[sel]
                nparticles, periodic = 0, int(self.bonded_periodic)
                if cls == COMPOUND:
                    nparticles, periodic = int(desc.ccompound_particles[p]), int(desc.ccompound_periodic[p])
                    atoms = atoms[:, :nparticles]
                atoms = np.ascontiguousarray(atoms, dtype=np.int32)
                names = getattr(desc, prefix + "_param_names")[p]
                pv = _vec(np.asarray(getattr(desc, prefix + "_params"))[sel][:, :len(names)])
                self.forces[prefix].append(lib().cc_add_force(
                    self.sys, cls, nparticles, energy.encode(), _names(names), _names(desc.custom_global_names), _dp(gv), len(sel), _ip(atoms),
                    _dp(pv), periodic, self.force_groups.get(group, 0), int(self.tabulated), self.deriv_params.get(group, "").encode()))

    def default_platform(self):
        """the platform a Context of this System gets when none is named"""
        return lib().cc_default_platform(self.sys).decode()

    def update(self, prefix, p, atoms, params):
        """Force p of the class with this field prefix ("custom", "cbond", "cext", "cangle" or "ccompound") gets these terms
        (atoms [n, its atoms per term], params [n, its parameters]), then updateParametersInContext"""
        cls = {c[0]: c[1] for c in CLASSES}[prefix]
        a = np.ascontiguousarray(atoms, dtype=np.int32)
        v = np.ascontiguousarray(params, dtype=np.float64)
        if lib().cc_update_force(self.sys, cls, self.forces[prefix][p], self.ctx, len(a), _ip(a), _dp(v)) != 0:
            raise RuntimeError(lib().cc_last_error().decode())
