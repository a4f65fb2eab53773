"""oracle/omm.py -- TEST INFRASTRUCTURE, not product code.

ctypes harness over oracle/_ref/libomm_capi.so, i.e. over the UNMODIFIED reference OpenMM (oracle/_ref/libOpenMM.so
built by oracle/Makefile from /root/reference).  Builds an OpenMM System from an openmm_b200.systems.SystemDesc and
runs it on a named Platform ("Reference" = the parity oracle, "CPU" = the speed baseline, "B200" = our plugin).
Only tests/, __graft_entry__.smoke() and bench.py may import this module.
"""
import ctypes as C
import os
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
REF_DIR = os.path.join(_HERE, "_ref")
_lib = None
_plugins = set()


def available():
    return os.path.exists(os.path.join(REF_DIR, "libomm_capi.so")) and os.path.exists(os.path.join(REF_DIR, "libOpenMM.so"))


def lib():
    global _lib
    if _lib is None:
        C.CDLL(os.path.join(REF_DIR, "libOpenMM.so"), mode=C.RTLD_GLOBAL)
        L = C.CDLL(os.path.join(REF_DIR, "libomm_capi.so"), mode=C.RTLD_GLOBAL)
        P, D, I = C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_int)
        sig = {
            "omm_last_error": (C.c_char_p, []), "omm_load_plugin": (C.c_int, [C.c_char_p]), "omm_num_platforms": (C.c_int, []),
            "omm_platform_name": (C.c_char_p, [C.c_int]),
            "omm_system_create": (P, [C.c_int, D]), "omm_system_destroy": (None, [P]), "omm_system_set_box": (None, [P, D, D, D]),
            "omm_system_add_constraints": (None, [P, C.c_int, I, I, D]), "omm_system_add_force": (C.c_int, [P, P]),
            "omm_system_serialize": (C.c_int, [P, C.c_char_p]),
            "omm_nonbonded_create": (P, [C.c_int, D, D, D]), "omm_nonbonded_add_exceptions": (None, [P, C.c_int, I, I, D, D, D]),
            "omm_nonbonded_create_exceptions_from_bonds": (None, [P, C.c_int, I, I, C.c_double, C.c_double]),
            "omm_nonbonded_num_exceptions": (C.c_int, [P]), "omm_nonbonded_get_exceptions": (None, [P, I, I, D, D, D]),
            "omm_force_destroy": (None, [P]),
            "omm_nonbonded_set_method": (None, [P, C.c_int, C.c_double, C.c_double]), "omm_nonbonded_set_pme": (None, [P, C.c_double, C.c_int, C.c_int, C.c_int]),
            "omm_nonbonded_set_switch": (None, [P, C.c_int, C.c_double]), "omm_nonbonded_set_dispersion": (None, [P, C.c_int]),
            "omm_nonbonded_set_rf_dielectric": (None, [P, C.c_double]), "omm_nonbonded_set_recip_group": (None, [P, C.c_int]),
            "omm_nonbonded_set_exceptions_periodic": (None, [P, C.c_int]), "omm_force_set_group": (None, [P, C.c_int]),
            "omm_bonds_create": (P, [C.c_int, I, I, D, D]), "omm_angles_create": (P, [C.c_int, I, I, I, D, D]),
            "omm_torsions_create": (P, [C.c_int, I, I, I, I, I, D, D]), "omm_cmmotion_create": (P, [C.c_int]),
            "omm_bonded_set_periodic": (None, [P, C.c_int, C.c_int]),
            "omm_nonbonded_add_global": (C.c_int, [P, C.c_char_p, C.c_double]),
            "omm_nonbonded_add_particle_offset": (C.c_int, [P, C.c_char_p, C.c_int, C.c_double, C.c_double, C.c_double]),
            "omm_nonbonded_add_exception_offset": (C.c_int, [P, C.c_char_p, C.c_int, C.c_double, C.c_double, C.c_double]),
            "omm_context_set_parameter": (C.c_int, [P, C.c_char_p, C.c_double]),
            "omm_integrator_create": (P, [C.c_int, C.c_double, C.c_double, C.c_double, C.c_int, C.c_double]),
            "omm_integrator_destroy": (None, [P]), "omm_integrator_step": (C.c_int, [P, C.c_int]),
            "omm_context_create": (P, [P, P, C.c_char_p, C.c_char_p]), "omm_context_destroy": (None, [P]),
            "omm_context_set_positions": (C.c_int, [P, C.c_int, D]), "omm_context_set_velocities": (C.c_int, [P, C.c_int, D]),
            "omm_context_set_box": (C.c_int, [P, D, D, D]), "omm_context_set_velocities_to_temperature": (C.c_int, [P, C.c_double, C.c_int]),
            "omm_context_apply_constraints": (C.c_int, [P, C.c_double]),
            "omm_context_get_state": (C.c_int, [P, C.c_int, D, D, D, D, C.c_int, C.c_int]),
            "omm_context_get_pme": (C.c_int, [P, P, D, I, I, I]), "omm_context_get_time": (C.c_double, [P]),
            "omm_context_platform": (C.c_char_p, [P]), "omm_context_checkpoint_roundtrip": (C.c_int, [P]),
        }
        for name, (res, args) in sig.items():
            f = getattr(L, name)
            f.restype, f.argtypes = res, args
        _lib = L
    return _lib


# parameter updates and checkpoints through a buffer (plugin/tests/nonbonded_capi.cpp, built by plugin/Makefile `all`
# against the headers oracle/Makefile stages, so that it builds wherever oracle/_ref/ is present)
NB_LIB = os.path.join(REF_DIR, "tests", "libnonbonded_capi.so")
_nb_lib = None


def nb_lib():
    global _nb_lib
    if _nb_lib is None:
        lib()
        L = C.CDLL(NB_LIB)
        P, D, I = C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_int)
        sig = {
            "nbc_last_error": (C.c_char_p, []), "nbc_set_particles": (C.c_int, [P, C.c_int, D, D, D]),
            "nbc_set_exceptions": (C.c_int, [P, C.c_int, I, I, D, D, D]), "nbc_update_in_context": (C.c_int, [P, P]),
            "nbc_create_checkpoint": (C.c_longlong, [P, C.c_char_p, C.c_longlong]),
            "nbc_load_checkpoint": (C.c_int, [P, C.c_char_p, C.c_longlong]),
        }
        for name, (res, args) in sig.items():
            f = getattr(L, name)
            f.restype, f.argtypes = res, args
        _nb_lib = L
    return _nb_lib


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def _ip(a):
    return a.ctypes.data_as(C.POINTER(C.c_int))


def _f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def _i32(a):
    return np.ascontiguousarray(a, dtype=np.int32)


def load_plugin(path):
    L = lib()
    path = os.path.abspath(path)
    if path in _plugins:
        return
    if L.omm_load_plugin(path.encode()) != 0:
        raise RuntimeError("plugin load failed: " + L.omm_last_error().decode())
    _plugins.add(path)


def platforms():
    L = lib()
    return [L.omm_platform_name(i).decode() for i in range(L.omm_num_platforms())]


def exceptions_from_bonds(charges, sigmas, epsilons, bond_i, bond_j, coulomb14, lj14):
    """NonbondedForce::createExceptionsFromBonds of the reference itself (NonbondedForce.cpp:207-248)."""
    L = lib()
    n = len(charges)
    nb = L.omm_nonbonded_create(n, _dp(_f64(charges)), _dp(_f64(sigmas)), _dp(_f64(epsilons)))
    bi, bj = _i32(bond_i), _i32(bond_j)
    L.omm_nonbonded_create_exceptions_from_bonds(nb, len(bi), _ip(bi), _ip(bj), coulomb14, lj14)
    ne = L.omm_nonbonded_num_exceptions(nb)
    i, j = np.zeros(ne, np.int32), np.zeros(ne, np.int32)
    qq, sg, ep = np.zeros(ne), np.zeros(ne), np.zeros(ne)
    L.omm_nonbonded_get_exceptions(nb, _ip(i), _ip(j), _dp(qq), _dp(sg), _dp(ep))
    L.omm_force_destroy(nb)
    return i, j, qq, sg, ep


class Simulation:
    """System + Integrator + Context on one platform, from a SystemDesc."""

    def __init__(self, desc, platform="Reference", integrator=(0, 0.0, 0.0, 0.001), seed=7, constraint_tol=1e-5,
                 pme=None, props="", recip_group=None, bonded_periodic=False, nb_globals=None, particle_offsets=(), exception_offsets=(),
                 bonded_group=None):
        """integrator = (kind, temperature, friction, dt); pme = (alpha, nx, ny, nz) to pin the PME parameters;
        bonded_periodic: setUsesPeriodicBoundaryConditions(true) on the three bonded forces; bonded_group: the force group of
        the three bonded forces (default 0, the NonbondedForce's); nb_globals = {name: default},
        particle_offsets = [(name, particle, dq, dsigma, deps)], exception_offsets = [(name, exception index, dqq, dsigma, deps)]
        (NonbondedForce parameter offsets)."""
        L = lib()
        self.L = L
        self.n = desc.natoms
        self.desc = desc
        self.sys = L.omm_system_create(self.n, _dp(_f64(desc.masses)))
        if desc.box is not None:
            b = _f64(desc.box)
            L.omm_system_set_box(self.sys, _dp(b[0]), _dp(b[1]), _dp(b[2]))
        if len(desc.con_i):
            L.omm_system_add_constraints(self.sys, len(desc.con_i), _ip(_i32(desc.con_i)), _ip(_i32(desc.con_j)), _dp(_f64(desc.con_d)))
        nb = L.omm_nonbonded_create(self.n, _dp(_f64(desc.charges)), _dp(_f64(desc.sigmas)), _dp(_f64(desc.epsilons)))
        self.nb = nb
        if len(desc.exc_i):
            L.omm_nonbonded_add_exceptions(nb, len(desc.exc_i), _ip(_i32(desc.exc_i)), _ip(_i32(desc.exc_j)), _dp(_f64(desc.exc_qq)),
                                           _dp(_f64(desc.exc_sigma)), _dp(_f64(desc.exc_eps)))
        L.omm_nonbonded_set_method(nb, desc.method, desc.cutoff, desc.ewald_tol)
        L.omm_nonbonded_set_switch(nb, int(desc.use_switch), desc.switch_distance)
        L.omm_nonbonded_set_dispersion(nb, int(desc.use_dispersion))
        L.omm_nonbonded_set_rf_dielectric(nb, desc.rf_dielectric)
        if pme is not None:
            L.omm_nonbonded_set_pme(nb, pme[0], pme[1], pme[2], pme[3])
        if recip_group is not None:
            L.omm_nonbonded_set_recip_group(nb, recip_group)
        for name, default in (nb_globals or {}).items():
            L.omm_nonbonded_add_global(nb, name.encode(), default)
        for name, idx, dq, ds, de in particle_offsets:
            L.omm_nonbonded_add_particle_offset(nb, name.encode(), int(idx), dq, ds, de)
        for name, idx, dq, ds, de in exception_offsets:
            L.omm_nonbonded_add_exception_offset(nb, name.encode(), int(idx), dq, ds, de)
        L.omm_system_add_force(self.sys, nb)
        if len(desc.bond_i):
            f = L.omm_bonds_create(len(desc.bond_i), _ip(_i32(desc.bond_i)), _ip(_i32(desc.bond_j)), _dp(_f64(desc.bond_r0)), _dp(_f64(desc.bond_k)))
            L.omm_bonded_set_periodic(f, 0, int(bonded_periodic))
            if bonded_group is not None:
                L.omm_force_set_group(f, bonded_group)
            L.omm_system_add_force(self.sys, f)
        if len(desc.angle_i):
            f = L.omm_angles_create(len(desc.angle_i), _ip(_i32(desc.angle_i)), _ip(_i32(desc.angle_j)), _ip(_i32(desc.angle_k)),
                                    _dp(_f64(desc.angle_t0)), _dp(_f64(desc.angle_kk)))
            L.omm_bonded_set_periodic(f, 1, int(bonded_periodic))
            if bonded_group is not None:
                L.omm_force_set_group(f, bonded_group)
            L.omm_system_add_force(self.sys, f)
        if len(desc.tor_i):
            f = L.omm_torsions_create(len(desc.tor_i), _ip(_i32(desc.tor_i)), _ip(_i32(desc.tor_j)), _ip(_i32(desc.tor_k)), _ip(_i32(desc.tor_l)),
                                      _ip(_i32(desc.tor_n)), _dp(_f64(desc.tor_phase)), _dp(_f64(desc.tor_kk)))
            L.omm_bonded_set_periodic(f, 2, int(bonded_periodic))
            if bonded_group is not None:
                L.omm_force_set_group(f, bonded_group)
            L.omm_system_add_force(self.sys, f)
        if desc.cm_frequency:
            L.omm_system_add_force(self.sys, L.omm_cmmotion_create(desc.cm_frequency))
        self.add_forces()
        kind, T, fric, dt = integrator
        self.integ = L.omm_integrator_create(kind, T, fric, dt, seed, constraint_tol)
        self.ctx = L.omm_context_create(self.sys, self.integ, platform.encode(), props.encode())
        if not self.ctx:
            raise RuntimeError("Context creation failed: " + L.omm_last_error().decode())
        self.set_positions(desc.positions)

    def add_forces(self):
        """Subclasses add more forces to self.sys here: the Context is made after it."""

    def set_parameter(self, name, value):
        self._ck(self.L.omm_context_set_parameter(self.ctx, name.encode(), value))

    def _ck(self, rc):
        if rc != 0:
            raise RuntimeError(self.L.omm_last_error().decode())

    def set_positions(self, x):
        self._ck(self.L.omm_context_set_positions(self.ctx, self.n, _dp(_f64(x))))

    def set_box(self, box):
        """Context::setPeriodicBoxVectors, as MonteCarloBarostatImpl calls it after scaling the coordinates"""
        b = _f64(box)
        self._ck(self.L.omm_context_set_box(self.ctx, _dp(b[0]), _dp(b[1]), _dp(b[2])))

    def set_velocities(self, v):
        self._ck(self.L.omm_context_set_velocities(self.ctx, self.n, _dp(_f64(v))))

    def set_velocities_to_temperature(self, T, seed=1):
        self._ck(self.L.omm_context_set_velocities_to_temperature(self.ctx, T, seed))

    def state(self, positions=False, velocities=False, forces=False, energy=False, groups=-1, enforce_periodic=False):
        n = self.n
        p = np.empty((n, 3)) if positions else None
        v = np.empty((n, 3)) if velocities else None
        f = np.empty((n, 3)) if forces else None
        e = np.empty(2) if energy else None
        nul = C.POINTER(C.c_double)()
        self._ck(self.L.omm_context_get_state(self.ctx, n, _dp(p) if positions else nul, _dp(v) if velocities else nul,
                                              _dp(f) if forces else nul, _dp(e) if energy else nul, groups, int(enforce_periodic)))
        out = {}
        if positions:
            out["positions"] = p
        if velocities:
            out["velocities"] = v
        if forces:
            out["forces"] = f
        if energy:
            out["potential"], out["kinetic"] = float(e[0]), float(e[1])
        return out

    def forces_energy(self, groups=-1):
        s = self.state(forces=True, energy=True, groups=groups)
        return s["forces"], s["potential"]

    def step(self, n=1):
        self._ck(self.L.omm_integrator_step(self.integ, n))

    def apply_constraints(self, tol=1e-5):
        self._ck(self.L.omm_context_apply_constraints(self.ctx, tol))

    def pme_parameters(self):
        a = C.c_double()
        nx, ny, nz = C.c_int(), C.c_int(), C.c_int()
        self._ck(self.L.omm_context_get_pme(self.ctx, self.nb, C.byref(a), C.byref(nx), C.byref(ny), C.byref(nz)))
        return a.value, nx.value, ny.value, nz.value

    def platform(self):
        return self.L.omm_context_platform(self.ctx).decode()

    def checkpoint_roundtrip(self):
        self._ck(self.L.omm_context_checkpoint_roundtrip(self.ctx))

    def _nbck(self, rc):
        if rc != 0:
            raise RuntimeError(nb_lib().nbc_last_error().decode())

    def update_nonbonded(self, desc):
        """desc's per-atom and per-exception parameters as the NonbondedForce's new base values (same particles and
        exceptions; the parameter offsets stay), then NonbondedForce::updateParametersInContext."""
        L = nb_lib()
        self._nbck(L.nbc_set_particles(self.nb, self.n, _dp(_f64(desc.charges)), _dp(_f64(desc.sigmas)), _dp(_f64(desc.epsilons))))
        if len(desc.exc_i):
            self._nbck(L.nbc_set_exceptions(self.nb, len(desc.exc_i), _ip(_i32(desc.exc_i)), _ip(_i32(desc.exc_j)), _dp(_f64(desc.exc_qq)),
                                            _dp(_f64(desc.exc_sigma)), _dp(_f64(desc.exc_eps))))
        self._nbck(L.nbc_update_in_context(self.nb, self.ctx))

    def checkpoint(self):
        """Context::createCheckpoint, as bytes"""
        L = nb_lib()
        n = L.nbc_create_checkpoint(self.ctx, None, 0)
        if n < 0:
            raise RuntimeError(L.nbc_last_error().decode())
        buf = C.create_string_buffer(n)
        if L.nbc_create_checkpoint(self.ctx, buf, n) != n:
            raise RuntimeError(L.nbc_last_error().decode() or "the checkpoint changed size")
        return buf.raw

    def load_checkpoint(self, blob):
        self._nbck(nb_lib().nbc_load_checkpoint(self.ctx, blob, len(blob)))

    def close(self):
        if getattr(self, "ctx", None):
            self.L.omm_context_destroy(self.ctx)
            self.L.omm_integrator_destroy(self.integ)
            self.L.omm_system_destroy(self.sys)
            self.ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
