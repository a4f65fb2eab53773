"""Engine: Python handle on a b200md context (one CUDA device).  Mirrors the kernel interfaces the OpenMM plugin
forwards (olla/include/openmm/kernels.h): UpdateStateData get/set, CalcForcesAndEnergy, Integrate*Step."""
import ctypes as C
import numpy as np
from . import _lib
from .systems import SystemDesc, NB_PME

TERM_BONDS, TERM_ANGLES, TERM_TORSIONS, TERM_NB_DIRECT, TERM_NB_RECIP = 1, 2, 4, 8, 16
TERM_RB_TORSIONS, TERM_CMAP, TERM_CUSTOM_TORSIONS, TERM_ALL = 32, 64, 128, 255
# kinds of b200md_set_bonded_groups
BONDED_KINDS = {"bonds": 0, "angles": 1, "torsions": 2, "rb_torsions": 3, "cmap": 4, "custom_torsions": 5}
PHASES = {"pair": 0, "pme_spread": 1, "pme_fft_conv": 2, "pme_gather": 3, "integrate": 4, "list_build": 5, "bonded": 6,
          "custom_torsions": 7}


class EngineError(RuntimeError):
    pass


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def _ip(a):
    return a.ctypes.data_as(C.POINTER(C.c_int))


def _f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def _i32(a):
    return np.ascontiguousarray(a, dtype=np.int32)


PRECISIONS = {"single": 0, "mixed": 1}


class Engine:
    def __init__(self, desc: SystemDesc, device=0, comm=None, precision="single", bonded_groups=None):
        """comm = (rank, world, unique_id_bytes) for the multi-GPU force decomposition.  precision: "single" (fp32 state) or
        "mixed" (positions as fp32 hi + lo, velocities, integration and constraints in double; single GPU only).
        bonded_groups = {kind: group byte per term} with kind a key of BONDED_KINDS: bits 0-4 the force group, bit 7 the
        term takes minimum-image difference vectors (Force::setUsesPeriodicBoundaryConditions)."""
        if precision not in PRECISIONS:
            raise ValueError("precision must be one of %s, not %r" % (sorted(PRECISIONS), precision))
        self.lib = _lib.load()
        self.desc = desc
        self.natoms = desc.natoms
        self._precision = precision
        h = C.c_void_p()
        if self.lib.b200md_create(C.byref(h), device, self.natoms) != 0:
            raise EngineError(self.lib.b200md_last_error(None).decode())
        self.h = h
        self._bonded_groups = bonded_groups or {}
        try:
            self._define(desc, comm)
        except Exception:
            self.close()
            raise

    def _ck(self, rc):
        if rc != 0:
            raise EngineError(self.lib.b200md_last_error(self.h).decode())

    def _define(self, d, comm):
        L = self.lib
        if comm is not None:
            rank, world, uid = comm
            buf = C.create_string_buffer(bytes(uid), 128)
            self._ck(L.b200md_comm_init(self.h, rank, world, C.cast(buf, C.c_void_p)))
        self._ck(L.b200md_set_precision(self.h, PRECISIONS[self._precision]))
        self._ck(L.b200md_set_masses(self.h, _dp(_f64(d.masses))))
        nd = _lib.NonbondedDesc()
        nd.method = d.method
        nd.cutoff = d.cutoff
        nd.use_switch = int(d.use_switch)
        nd.switch_distance = d.switch_distance
        nd.rf_dielectric = d.rf_dielectric
        if d.method == NB_PME:
            alpha, nx, ny, nz = d.pme_parameters()
            nd.ewald_alpha = alpha
            nd.grid[0], nd.grid[1], nd.grid[2] = nx, ny, nz
        nd.dispersion_coefficient = d.dispersion_coefficient()
        nd.exceptions_periodic = 0
        self._ck(L.b200md_set_nonbonded(self.h, C.byref(nd), _dp(_f64(d.charges)), _dp(_f64(d.sigmas)), _dp(_f64(d.epsilons))))
        if len(d.exc_i):
            self._ck(L.b200md_set_exceptions(self.h, len(d.exc_i), _ip(_i32(d.exc_i)), _ip(_i32(d.exc_j)), _dp(_f64(d.exc_qq)),
                                             _dp(_f64(d.exc_sigma)), _dp(_f64(d.exc_eps))))
        if len(d.bond_i):
            self._ck(L.b200md_set_bonds(self.h, len(d.bond_i), _ip(_i32(d.bond_i)), _ip(_i32(d.bond_j)), _dp(_f64(d.bond_r0)), _dp(_f64(d.bond_k))))
        if len(d.angle_i):
            self._ck(L.b200md_set_angles(self.h, len(d.angle_i), _ip(_i32(d.angle_i)), _ip(_i32(d.angle_j)), _ip(_i32(d.angle_k)),
                                         _dp(_f64(d.angle_t0)), _dp(_f64(d.angle_kk))))
        if len(d.tor_i):
            self._ck(L.b200md_set_torsions(self.h, len(d.tor_i), _ip(_i32(d.tor_i)), _ip(_i32(d.tor_j)), _ip(_i32(d.tor_k)), _ip(_i32(d.tor_l)),
                                           _ip(_i32(d.tor_n)), _dp(_f64(d.tor_phase)), _dp(_f64(d.tor_kk))))
        if len(d.rb_i):
            self._ck(L.b200md_set_rb_torsions(self.h, len(d.rb_i), _ip(_i32(d.rb_i)), _ip(_i32(d.rb_j)), _ip(_i32(d.rb_k)), _ip(_i32(d.rb_l)),
                                              _dp(_f64(d.rb_c))))
        if len(d.cmap_map):
            self._ck(L.b200md_set_cmap(self.h, len(d.cmap_size), _ip(_i32(d.cmap_size)), _dp(_f64(d.cmap_coeff)), len(d.cmap_map),
                                       _ip(_i32(d.cmap_map)), _ip(_i32(d.cmap_atoms))))
        if len(d.custom_prog):
            if not len(d.custom_op):
                raise EngineError("custom torsions without programs: compile desc.custom_energy into custom_op / custom_arg / "
                                  "custom_imm / custom_prog_start first (the plugin's expression translator)")
            params = _f64(d.custom_params).reshape(len(d.custom_prog), -1)
            self._ck(L.b200md_set_custom_torsions(self.h, len(d.custom_prog_start)//2, _ip(_i32(d.custom_prog_start)), _ip(_i32(d.custom_op)),
                                                  _ip(_i32(d.custom_arg)), _dp(_f64(d.custom_imm)), params.shape[1], len(d.custom_prog),
                                                  _ip(_i32(d.custom_prog)), _ip(_i32(d.custom_atoms)), _dp(params)))
        if len(d.custom_global_values):
            self._ck(L.b200md_set_custom_globals(self.h, len(d.custom_global_values), _dp(_f64(d.custom_global_values))))
        for kind, g in self._bonded_groups.items():
            g = _i32(g)
            self._ck(L.b200md_set_bonded_groups(self.h, BONDED_KINDS[kind], len(g), _ip(g)))
        if len(d.con_i):
            self._ck(L.b200md_set_constraints(self.h, len(d.con_i), _ip(_i32(d.con_i)), _ip(_i32(d.con_j)), _dp(_f64(d.con_d))))
        if d.cm_frequency:
            self._ck(L.b200md_set_cm_remover(self.h, d.cm_frequency))
        if d.box is not None:
            b = _f64(d.box)
            self._ck(L.b200md_set_box(self.h, _dp(b[0]), _dp(b[1]), _dp(b[2])))
        self._ck(L.b200md_finalize(self.h))
        self.set_positions(d.positions)

    @property
    def precision(self):
        """"single" or "mixed", as the library reports it."""
        p = self.lib.b200md_get_precision(self.h)
        return {v: k for k, v in PRECISIONS.items()}[p]

    # ---- UpdateStateDataKernel ----
    def set_positions(self, x):
        x = _f64(x)
        assert x.shape == (self.natoms, 3)
        self._ck(self.lib.b200md_set_positions(self.h, _dp(x)))

    def get_positions(self):
        x = np.empty((self.natoms, 3))
        self._ck(self.lib.b200md_get_positions(self.h, _dp(x)))
        return x

    def set_velocities(self, v):
        v = _f64(v)
        self._ck(self.lib.b200md_set_velocities(self.h, _dp(v)))

    def get_velocities(self):
        v = np.empty((self.natoms, 3))
        self._ck(self.lib.b200md_get_velocities(self.h, _dp(v)))
        return v

    def get_forces(self):
        f = np.empty((self.natoms, 3))
        self._ck(self.lib.b200md_get_forces(self.h, _dp(f)))
        return f

    def set_box(self, box):
        b = _f64(box)
        self._ck(self.lib.b200md_set_box(self.h, _dp(b[0]), _dp(b[1]), _dp(b[2])))

    def get_box(self):
        a, b, c = np.empty(3), np.empty(3), np.empty(3)
        self._ck(self.lib.b200md_get_box(self.h, _dp(a), _dp(b), _dp(c)))
        return np.array([a, b, c])

    # ---- ApplyMonteCarloBarostatKernel ----
    def set_barostat_molecules(self, molecules=None):
        """The molecules the barostat scales as rigid groups (default: desc.molecules(), as ContextImpl::getMolecules())."""
        mols = self.desc.molecules() if molecules is None else molecules
        start = np.zeros(len(mols) + 1, dtype=np.int32)
        start[1:] = np.cumsum([len(m) for m in mols])
        atoms = _i32([a for m in mols for a in m] or [0])
        self._ck(self.lib.b200md_set_barostat_molecules(self.h, len(mols), _ip(start), _ip(atoms)))

    def scale_coordinates(self, sx, sy, sz):
        """Save positions and forces, then wrap every molecule's centre into the first periodic box and scale it.  The box
        itself is unchanged: set_box(scaled box) follows, as in MonteCarloBarostatImpl::updateContextState."""
        self._ck(self.lib.b200md_scale_coordinates(self.h, sx, sy, sz))

    def restore_coordinates(self):
        """Positions and forces as before the last scale_coordinates (a rejected move); set_box(old box) follows."""
        self._ck(self.lib.b200md_restore_coordinates(self.h))

    # ---- CalcForcesAndEnergyKernel ----
    def compute(self, terms=TERM_ALL, energy=True):
        """Forces (get_forces()) and, if energy, the potential energy of the selected terms."""
        if energy:
            e = C.c_double()
            self._ck(self.lib.b200md_compute(self.h, terms, 1, C.byref(e)))
            return e.value
        self._ck(self.lib.b200md_compute(self.h, terms, 1, None))
        return None

    def compute_groups(self, terms=TERM_ALL, groups=0xffffffff):
        """compute() restricted to the bonded terms whose force group is in the `groups` bit mask; returns the energy."""
        e = C.c_double()
        self._ck(self.lib.b200md_compute_groups(self.h, terms, groups, 1, C.byref(e)))
        return e.value

    # ---- Calc{RBTorsion,CMAPTorsion}ForceKernel::copyParametersToContext ----
    def update_rb_torsion_params(self, c):
        c = _f64(c)
        self._ck(self.lib.b200md_update_rb_torsion_params(self.h, len(c), _dp(c)))

    def update_cmap_params(self, size, coeff, cmap_map):
        size, coeff, cmap_map = _i32(size), _f64(coeff), _i32(cmap_map)
        self._ck(self.lib.b200md_update_cmap_params(self.h, len(size), _ip(size), _dp(coeff), len(cmap_map), _ip(cmap_map)))

    # ---- CalcCustomTorsionForceKernel::copyParametersToContext and the global parameters of its expressions ----
    def update_custom_torsion_params(self, params):
        """New per-torsion parameters [n, param_stride] for the same torsions and expressions."""
        p = _f64(params)
        self._ck(self.lib.b200md_update_custom_torsion_params(self.h, len(p), _dp(p)))

    def set_custom_globals(self, values):
        """The values of the global parameter slots the expressions read (the number of slots is fixed at definition)."""
        v = _f64(values)
        self._ck(self.lib.b200md_set_custom_globals(self.h, len(v), _dp(v)))

    # ---- Integrate*StepKernel ----
    def set_integrator(self, kind, dt, temperature=300.0, friction=1.0, seed=7, constraint_tol=1e-5):
        self._ck(self.lib.b200md_set_integrator(self.h, kind, dt, temperature, friction, seed, constraint_tol))

    def step(self, n=1):
        self._ck(self.lib.b200md_step(self.h, n))

    def kinetic_energy(self):
        e = C.c_double()
        self._ck(self.lib.b200md_kinetic_energy(self.h, C.byref(e)))
        return e.value

    def apply_constraints(self, tol=1e-5):
        self._ck(self.lib.b200md_apply_constraints(self.h, tol))

    def apply_velocity_constraints(self, tol=1e-5):
        self._ck(self.lib.b200md_apply_velocity_constraints(self.h, tol))

    def synchronize(self):
        self._ck(self.lib.b200md_synchronize(self.h))

    def time(self):
        return self.lib.b200md_get_time(self.h)

    def checkpoint(self):
        n = self.lib.b200md_checkpoint_save(self.h, None, 0)
        buf = C.create_string_buffer(n)
        if self.lib.b200md_checkpoint_save(self.h, C.cast(buf, C.c_void_p), n) != n:
            raise EngineError(self.lib.b200md_last_error(self.h).decode())
        return buf.raw

    def load_checkpoint(self, blob):
        buf = C.create_string_buffer(blob, len(blob))
        self._ck(self.lib.b200md_checkpoint_load(self.h, C.cast(buf, C.c_void_p), len(blob)))

    # ---- introspection ----
    def stats(self):
        s = _lib.Stats()
        self._ck(self.lib.b200md_get_stats(self.h, C.byref(s)))
        return {k: (list(getattr(s, k)) if k == "pme_grid" else getattr(s, k)) for k, _ in s._fields_}

    def time_phase(self, phase, reps=20):
        ms = C.c_double()
        self._ck(self.lib.b200md_time_phase(self.h, PHASES[phase] if isinstance(phase, str) else phase, reps, C.byref(ms)))
        return ms.value

    def stream(self):
        return self.lib.b200md_cuda_stream(self.h)

    def close(self):
        if getattr(self, "h", None):
            self.lib.b200md_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def fft3d_r2c(x, device=0):
    """The bespoke 3-D FFT alone: real [nx,ny,nz] -> complex [nx,ny,nz//2+1] (unnormalised, e^{-2 pi i jk/n})."""
    lib = _lib.load()
    x = np.ascontiguousarray(x, dtype=np.float32)
    nx, ny, nz = x.shape
    out = np.empty((nx, ny, nz//2+1, 2), dtype=np.float32)
    fp = C.POINTER(C.c_float)
    if lib.b200md_fft3d_r2c(device, nx, ny, nz, x.ctypes.data_as(fp), out.ctypes.data_as(fp)) != 0:
        raise EngineError(lib.b200md_last_error(None).decode())
    return out[..., 0] + 1j*out[..., 1]


def fft3d_c2r(c, nz, device=0):
    lib = _lib.load()
    nx, ny, nzc = c.shape
    assert nzc == nz//2+1
    inp = np.ascontiguousarray(np.stack([c.real, c.imag], -1), dtype=np.float32)
    out = np.empty((nx, ny, nz), dtype=np.float32)
    fp = C.POINTER(C.c_float)
    if lib.b200md_fft3d_c2r(device, nx, ny, nz, inp.ctypes.data_as(fp), out.ctypes.data_as(fp)) != 0:
        raise EngineError(lib.b200md_last_error(None).decode())
    return out
