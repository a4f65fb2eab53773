"""Test harness of the CustomNonbondedForce tests: DHFR with its Lennard-Jones moved into a CustomNonbondedForce of
Discrete2DFunction tables, exactly as the reference's LennardJonesGenerator (app/forcefield.py) builds every charmm36.xml System,
and the reference's Simulation with such a force added, over oracle/_ref/tests/libcustom_nonbonded_capi.so
(plugin/tests/custom_nonbonded_capi.cpp).

DHFR-LJ-table: the (sigma, epsilon) pairs of data/dhfr.npz merged into types; acoef = 4 eps sigma^12 and bcoef = 4 eps sigma^6
of the Lorentz-Berthelot combination of every pair of types; the NonbondedForce's epsilons zeroed, its exceptions (and their 1-4
Lennard-Jones) kept; the exceptions as the exclusions; the long-range correction on; PME with a 0.9 nm cutoff.  DHFR-NBFIX: the
same with a few pairs of types overridden (the tables are then no longer Lorentz-Berthelot) and a switching function at 0.8 nm.

Engine-level: engine_desc() puts such a force into a SystemDesc's cnb_* fields, with the programs of the plugin's translator
(translate()) and the long-range coefficient the Reference platform's goldens store (tests/golden/reference_custom_nonbonded.npz,
tests/golden/make_golden_custom_nonbonded.py)."""
import ctypes as C
import os

import numpy as np

from openmm_b200 import systems
from oracle import omm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "oracle", "_ref", "tests", "libcustom_nonbonded_capi.so")
DHFR = os.path.join(ROOT, "data", "dhfr.npz")
GOLDEN = os.path.join(ROOT, "tests", "golden", "reference_custom_nonbonded.npz")
LJ_TABLE = "acoef(type1, type2)/r^12 - bcoef(type1, type2)/r^6"
CNB_GROUP = 2
CUTOFF_PERIODIC = 2          # CustomNonbondedForce::CutoffPeriodic
_lib = None


def available():
    return os.path.exists(LIB) and omm.available()


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(LIB)
        D, I, P, S = C.POINTER(C.c_double), C.c_int, C.c_void_p, C.c_char_p
        IP = C.POINTER(C.c_int)
        L.cnbc_add_force.argtypes = [P, S, I, S, D, I, C.c_double, C.c_double, I, I, I, IP, IP, S, IP, IP, D, S, D]
        L.cnbc_add_force.restype = I
        L.cnbc_update.argtypes = [P, I, P, D]
        L.cnbc_update.restype = I
        L.cnbc_add_interaction_group.argtypes = [P, I, I, IP, I, IP]
        L.cnbc_add_derivative.argtypes = [P, I, S]
        L.cnbc_add_continuous.argtypes = [P, I, S]
        L.cnbc_last_error.restype = S
        L.cnbc_add_table.argtypes = [P, I, S, I, I, I, I, D]
        L.cnbc_translate.argtypes = [P, I, I, IP, IP, IP, D, IP, IP, IP, IP, D, I]
        L.cnbc_lepton.argtypes = [P, I, I, C.c_double, D, D, D]
        L.cnbc_lrc.argtypes = [P, I, P, D]
        L.cnbc_default_platform.argtypes = [P]
        L.cnbc_default_platform.restype = S
        _lib = L
    return _lib


def _dp(a):
    return np.ascontiguousarray(a, dtype=np.float64).ctypes.data_as(C.POINTER(C.c_double))


def _ip(a):
    return np.ascontiguousarray(a, dtype=np.int32).ctypes.data_as(C.POINTER(C.c_int))


class Force:
    """One CustomNonbondedForce: expression, per-particle parameters params[n][k] named names, method, cutoff, switching distance
    (None: off), long-range correction, group, exclusions (pairs), square tables {name: matrix} and globals {name: default}."""

    def __init__(self, energy, names, params, method, cutoff, switch=None, lrc=True, group=CNB_GROUP, exclusions=(), tables=None, globals_=None):
        self.energy, self.names = energy, list(names)
        self.params = np.asarray(params, dtype=np.float64).reshape(len(params), len(self.names))
        self.method, self.cutoff, self.switch, self.lrc, self.group = method, cutoff, switch, lrc, group
        self.exclusions = np.asarray(exclusions, dtype=np.int32).reshape(-1, 2)
        self.tables = dict(tables or {})
        self.globals = dict(globals_ or {})

    def add_to(self, sys):
        names = list(self.tables)
        mats = [np.asarray(self.tables[k], dtype=np.float64) for k in names]
        sizes = np.array([m.shape[0] for m in mats] or [0], dtype=np.int32)
        start = np.concatenate([[0], np.cumsum([m.size for m in mats])]).astype(np.int32)
        values = np.concatenate([m.T.ravel() for m in mats] or [np.zeros(1)])      # x (the first argument) fastest
        g = list(self.globals)
        idx = lib().cnbc_add_force(sys, self.energy.encode(), len(self.params), ",".join(self.names).encode(), _dp(self.params),
                                   self.method, self.cutoff, -1.0 if self.switch is None else self.switch, int(self.lrc), self.group,
                                   len(self.exclusions), _ip(self.exclusions[:, 0]), _ip(self.exclusions[:, 1]),
                                   ",".join(names).encode(), _ip(sizes), _ip(start), _dp(values), ",".join(g).encode(),
                                   _dp(np.array([self.globals[k] for k in g] or [0.0])))
        if idx < 0:
            raise RuntimeError(lib().cnbc_last_error().decode())
        return idx


class Simulation(omm.Simulation):
    """oracle.omm.Simulation plus the CustomNonbondedForce objects of `forces` (keyword argument)."""

    def __init__(self, desc, platform="Reference", forces=(), **kw):
        self.cnb_forces = list(forces)
        super().__init__(desc, platform, **kw)

    def add_forces(self):
        super().add_forces()
        self.cnb_index = [f.add_to(self.sys) for f in self.cnb_forces]

    def default_platform(self):
        return lib().cnbc_default_platform(self.sys).decode()

    def lrc(self, k=0):
        """CustomNonbondedForceImpl::calcLongRangeCorrection of force k in this Context"""
        c = np.zeros(1)
        if lib().cnbc_lrc(self.sys, self.cnb_index[k], self.ctx, _dp(c)) != 0:
            raise RuntimeError(lib().cnbc_last_error().decode())
        return float(c[0])

    def update_custom_nonbonded(self, k, params):
        self.cnb_forces[k].params = np.asarray(params, dtype=np.float64)
        if lib().cnbc_update(self.sys, self.cnb_index[k], self.ctx, _dp(self.cnb_forces[k].params)) != 0:
            raise RuntimeError(lib().cnbc_last_error().decode())


# ---------------------------------------------------------------- the plugin's translator and Lepton (no Context)
class Standalone:
    """One CustomNonbondedForce in a System of n particles, for translate() and lepton()"""

    def __init__(self, force, n):
        self.L = omm.lib()
        self.sys = self.L.omm_system_create(n, _dp(np.ones(n)))
        self.index = force.add_to(self.sys)

    def add_table(self, name, table):
        t = np.asarray(table, dtype=np.float64)
        shape = list(t.shape) + [1]*(3 - t.ndim)
        if lib().cnbc_add_table(self.sys, self.index, name.encode(), t.ndim, *shape, _dp(t.transpose().ravel())) != 0:
            raise RuntimeError(lib().cnbc_last_error().decode())

    def translate(self, cap=4096, vcap=1 << 20):
        """(prog_start, op, arg, imm, dims [t, 4], start, values) of translateNonbonded, or raises with its message"""
        op, arg, imm = np.zeros(cap, np.int32), np.zeros(cap, np.int32), np.zeros(cap)
        start, nops, nt = np.zeros(3, np.int32), np.zeros(1, np.int32), np.zeros(1, np.int32)
        dims, tstart, values = np.zeros(4*64, np.int32), np.zeros(65, np.int32), np.zeros(vcap)
        if lib().cnbc_translate(self.sys, self.index, cap, _ip(nops), _ip(op), _ip(arg), _dp(imm), _ip(start), _ip(nt), _ip(dims),
                                _ip(tstart), _dp(values), vcap) != 0:
            raise RuntimeError(lib().cnbc_last_error().decode())
        n, t = int(nops[0]), int(nt[0])
        return start, op[:n], arg[:n], imm[:n], dims[:4*t].reshape(t, 4), tstart[:t + 1], values[:tstart[t]]

    def lepton(self, which, r, p1, p2):
        """Lepton's energy (which 0) or dE/dr (which 1), the tables the Reference platform's functions"""
        out = np.zeros(1)
        if lib().cnbc_lepton(self.sys, self.index, which, r, _dp(np.asarray(p1, float)), _dp(np.asarray(p2, float)), _dp(out)) != 0:
            raise RuntimeError(lib().cnbc_last_error().decode())
        return float(out[0])

    def close(self):
        self.L.omm_system_destroy(self.sys)


def engine_desc(nbfix=False):
    """DHFR-LJ-table (or DHFR-NBFIX) as a SystemDesc of the Python mirror: the NonbondedForce with zero epsilons and the
    CustomNonbondedForce in the cnb_* fields, its programs from the plugin's translator, its long-range coefficient from the
    goldens"""
    d, f = dhfr_lj_table(nbfix)
    s = Standalone(f, d.natoms)
    start, op, arg, imm, dims, tstart, values = s.translate()
    s.close()
    g = np.load(GOLDEN)
    d.cnb_method, d.cnb_cutoff = systems.NB_CUTOFF_PERIODIC, f.cutoff
    d.cnb_excl = f.exclusions.astype(np.int32)
    d.cnb_prog_start, d.cnb_op, d.cnb_arg, d.cnb_imm = start, op, arg, imm
    d.cnb_nparams = np.array([len(f.names)], np.int32)
    d.cnb_switch = np.array([-1.0 if f.switch is None else f.switch])
    d.cnb_group = np.array([CNB_GROUP], np.int32)
    d.cnb_lrc = np.array([float(g[("nbfix" if nbfix else "lj_table") + "_lrc"])])
    d.cnb_params = f.params[None, :, :].copy()
    d.cnb_table_dims, d.cnb_table_start, d.cnb_table_values = dims, tstart, values
    return d


# ---------------------------------------------------------------- systems
def lj_types(sigmas, epsilons):
    """LennardJonesGenerator's merge: the distinct (sigma, epsilon) pairs as types, the type of every atom, and the
    Lorentz-Berthelot acoef and bcoef tables of every pair of types"""
    pairs, types = np.unique(np.stack([sigmas, epsilons], axis=1), axis=0, return_inverse=True)
    s = 0.5*(pairs[:, 0, None] + pairs[None, :, 0])
    e = np.sqrt(pairs[:, 1, None]*pairs[None, :, 1])
    return types.ravel(), 4.0*e*s**12, 4.0*e*s**6


def dhfr_lj_table(nbfix=False):
    """(desc, force): DHFR with its LJ in a CustomNonbondedForce of tables (DHFR-LJ-table), or DHFR-NBFIX with nbfix"""
    d = systems.SystemDesc.load(DHFR).rounded()
    types, acoef, bcoef = lj_types(d.sigmas, d.epsilons)
    if nbfix:
        # a few overridden pairs of types (both orders), as CHARMM36's NBFIX entries make them
        rng = np.random.default_rng(5)
        for a, b in rng.choice(acoef.shape[0], size=(6, 2)):
            acoef[a, b] = acoef[b, a] = 1.3*acoef[a, b]
            bcoef[a, b] = bcoef[b, a] = 0.8*bcoef[a, b]
    force = Force(LJ_TABLE, ["type"], types[:, None].astype(np.float64), CUTOFF_PERIODIC, float(d.cutoff),
                  switch=0.8 if nbfix else None, exclusions=np.stack([d.exc_i, d.exc_j], axis=1),
                  tables={"acoef": acoef, "bcoef": bcoef})
    d.epsilons = np.zeros_like(d.epsilons)
    return d, force


def force_error(f, ref):
    """max over atoms of max|df| / max(1, |f_ref|)"""
    return float((np.abs(f - ref).max(axis=1)/np.maximum(1.0, np.linalg.norm(ref, axis=1))).max())
