"""Harness of the custom centroid bond tests: the plugin's translator of CustomCentroidBondForce expressions
(plugin/custom_translate.h), the reference's CustomCentroidBondForce with its groups and weights added to the System a
custom_harness Simulation builds, computeNormalizedWeights, and the double-precision yardstick of a centroid bond.  ctypes
over oracle/_ref/tests/libcentroid_capi.so (plugin/tests/centroid_capi.cpp); everything else is custom_harness's."""
import ctypes as C
import os
import numpy as np
import custom_harness
from custom_harness import COMPOUND, Refused, compound_probe, omm     # noqa: F401  (re-exported for the tests)

LIB = os.path.join(omm.REF_DIR, "tests", "libcentroid_capi.so")
CENTROID = 5
_lib = None


def available():
    return custom_harness.available() and os.path.exists(LIB)


def lib():
    global _lib
    if _lib is None:
        omm.lib()                                   # libOpenMM.so, loaded globally
        L = C.CDLL(LIB)
        P, D, I, S, N = C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_int), C.c_char_p, C.c_int
        L.ccc_last_error.restype = S
        L.ccc_last_error.argtypes = []
        L.ccc_translate.restype = N
        L.ccc_translate.argtypes = [N, S, S, S, N, N, I, I, D, I]
        L.ccc_add_force.restype = N
        L.ccc_add_force.argtypes = [P, N, S, S, S, D, N, I, I, D, I, N, I, D, N, N, N, S]
        L.ccc_update_force.restype = N
        L.ccc_update_force.argtypes = [P, N, P, N, I, D]
        L.ccc_normalized_weights.restype = N
        L.ccc_normalized_weights.argtypes = [P, N, D]
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


def _i32(a):
    return np.ascontiguousarray(a, dtype=np.int32)


def translate(cls, energy, params=(), globals_=(), nparticles=0, tabulated=False):
    """(op, arg, imm, starts) as custom_harness.translate; class CENTROID: a CustomCentroidBondForce expression of nparticles
    groups per bond (the derivatives by x1, y1, z1, x2, .. of the group centres)"""
    if cls != CENTROID:
        return custom_harness.translate(cls, energy, params, globals_, nparticles, tabulated)
    cap = 65536
    op, arg, imm = np.zeros(cap, np.int32), np.zeros(cap, np.int32), np.zeros(cap)
    counts = np.zeros(32, np.int32)
    n = lib().ccc_translate(nparticles, energy.encode(), _names(params), _names(globals_), int(tabulated), cap, _ip(op), _ip(arg), _dp(imm),
                            _ip(counts))
    if n == -2:
        raise Refused(lib().ccc_last_error().decode())
    if n < 0:
        raise ValueError(lib().ccc_last_error().decode())
    starts = np.concatenate([[0], np.cumsum(counts[:n])]).astype(np.int32)
    return op[:starts[-1]].copy(), arg[:starts[-1]].copy(), imm[:starts[-1]].copy(), starts


def compiled(desc):
    """custom_harness.compiled(desc) plus the programs of its centroid bonds (ccentroid_prog_start / _op / _arg / _imm)"""
    d = custom_harness.compiled(desc)
    start, op, arg, imm = [0], [], [], []
    for p, energy in enumerate(desc.ccentroid_energy):
        o, a, i, s = translate(CENTROID, energy, desc.ccentroid_param_names[p], desc.custom_global_names, int(desc.ccentroid_groups_per_bond[p]))
        op += o.tolist()
        arg += a.tolist()
        imm += i.tolist()
        start += (start[-1] + s[1:]).tolist()
    d.ccentroid_prog_start = np.array(start if desc.ccentroid_energy else [], dtype=np.int32)
    d.ccentroid_op = np.array(op, np.int32)
    d.ccentroid_arg = np.array(arg, np.int32)
    d.ccentroid_imm = np.array(imm, np.float64)
    return d


class Simulation(custom_harness.Simulation):
    """custom_harness.Simulation plus one CustomCentroidBondForce per centroid expression of desc, each holding every group of
    desc (ccentroid_group_*; a mass-weighted group without weights), declaring every global of desc.custom_global_names, and
    periodic as desc.ccentroid_periodic says.  force_groups["custom_centroid"] puts them in a group, deriv_params["custom_centroid"]
    asks them for the energy derivative by that global, tabulated gives them a tabulated function."""

    def add_forces(self):
        super().add_forces()
        desc = self.desc
        self.forces["ccentroid"] = []
        gv = _vec(desc.custom_global_values)
        start = _i32(desc.ccentroid_group_start)
        for p, energy in enumerate(desc.ccentroid_energy):
            n = int(desc.ccentroid_groups_per_bond[p])
            sel = np.nonzero(np.asarray(desc.ccentroid_expr) == p)[0]
            groups = _i32(np.asarray(desc.ccentroid_atoms)[sel][:, :n])
            names = desc.ccentroid_param_names[p]
            pv = _vec(np.asarray(desc.ccentroid_params)[sel][:, :len(names)])
            index = lib().ccc_add_force(self.sys, n, energy.encode(), _names(names), _names(desc.custom_global_names), _dp(gv), len(start) - 1,
                                        _ip(start), _ip(_i32(desc.ccentroid_group_atoms)), _dp(_vec(desc.ccentroid_group_weights)),
                                        _ip(_i32(desc.ccentroid_group_mass)), len(sel), _ip(groups), _dp(pv), int(desc.ccentroid_periodic[p]),
                                        self.force_groups.get("custom_centroid", 0), int(self.tabulated),
                                        self.deriv_params.get("custom_centroid", "").encode())
            if index < 0:
                raise RuntimeError(lib().ccc_last_error().decode())
            self.forces["ccentroid"].append(index)

    def normalized_weights(self, p=0):
        """CustomCentroidBondForceImpl::computeNormalizedWeights of centroid force p: every group's weights, one after the other"""
        out = np.zeros(max(1, len(self.desc.ccentroid_group_atoms)))
        n = lib().ccc_normalized_weights(self.sys, self.forces["ccentroid"][p], _dp(out))
        if n < 0:
            raise RuntimeError(lib().ccc_last_error().decode())
        return out[:n]

    def update(self, prefix, p, atoms, params):
        """custom_harness.Simulation.update; prefix "ccentroid": centroid force p gets the bonds (groups [n, its groups per bond],
        params [n, its parameters]), then updateParametersInContext"""
        if prefix != "ccentroid":
            return super().update(prefix, p, atoms, params)
        g, v = _i32(atoms), np.ascontiguousarray(params, dtype=np.float64)
        if lib().ccc_update_force(self.sys, self.forces["ccentroid"][p], self.ctx, len(g), _ip(g), _dp(v)) != 0:
            raise RuntimeError(lib().ccc_last_error().decode())


def centroid_yardstick(desc, x, weights=None, box=None, globals_=None):
    """Energy and forces [natoms, 3] of the centroid bonds of a compiled desc at the positions x, in double: the group centres
    from the normalised weights (desc.ccentroid_group_weights, or `weights` in the same order, e.g. from
    Simulation.normalized_weights), every program of a bond through b200md_custom_compound_probe at the centres of its groups
    (a centroid bond's programs are a compound bond's), and -w times the derivatives by a centre on each atom of the group"""
    x = np.asarray(x, dtype=np.float64)
    w = np.asarray(desc.ccentroid_group_weights if weights is None else weights, dtype=np.float64)
    start, atoms = np.asarray(desc.ccentroid_group_start), np.asarray(desc.ccentroid_group_atoms)
    centres = np.array([w[start[g]:start[g+1]] @ x[atoms[start[g]:start[g+1]]] for g in range(len(start) - 1)]).reshape(-1, 3)
    box = np.asarray(desc.box if box is None else box, dtype=np.float64) if (box is not None or desc.box is not None) else np.eye(3)
    gv = desc.custom_global_values if globals_ is None else globals_
    first = np.concatenate([[0], np.cumsum(1 + 3*np.asarray(desc.ccentroid_groups_per_bond))])
    energy, forces = 0.0, np.zeros_like(x)
    for i, p in enumerate(desc.ccentroid_expr):
        n = int(desc.ccentroid_groups_per_bond[p])
        groups = desc.ccentroid_atoms[i, :n]
        q0 = first[p]
        start_p = desc.ccentroid_prog_start[q0:q0 + 2 + 3*n] - desc.ccentroid_prog_start[q0]
        code = slice(desc.ccentroid_prog_start[q0], desc.ccentroid_prog_start[q0 + 1 + 3*n])
        par = np.asarray(desc.ccentroid_params[i])
        vals = []
        for which in range(1 + 3*n):
            v, msg = compound_probe(n, bool(desc.ccentroid_periodic[p]), start_p, desc.ccentroid_op[code], desc.ccentroid_arg[code],
                                    desc.ccentroid_imm[code], len(par), len(gv), which, centres[groups].reshape(-1), box, par, gv)
            assert msg is None, msg
            vals.append(v)
        energy += vals[0]
        grad = np.array(vals[1:]).reshape(n, 3)
        for k, g in enumerate(groups):
            np.add.at(forces, atoms[start[g]:start[g+1]], -np.outer(w[start[g]:start[g+1]], grad[k]))
    return energy, forces
