"""Engine: Python handle on a b200md context (one CUDA device).  Mirrors the kernel interfaces the OpenMM plugin
forwards (olla/include/openmm/kernels.h): UpdateStateData get/set, CalcForcesAndEnergy, Integrate*Step."""
import ctypes as C
import numpy as np
from . import _lib
from .systems import SystemDesc, NB_PME

TERM_BONDS, TERM_ANGLES, TERM_TORSIONS, TERM_NB_DIRECT, TERM_NB_RECIP = 1, 2, 4, 8, 16
TERM_RB_TORSIONS, TERM_CMAP, TERM_CUSTOM_TORSIONS = 32, 64, 128
TERM_CUSTOM_BONDS, TERM_CUSTOM_EXTERNALS, TERM_CUSTOM_ANGLES, TERM_CUSTOM_COMPOUND = 256, 512, 1024, 2048
TERM_CUSTOM_CENTROID, TERM_GBSA, TERM_RMSD, TERM_CV_FORCES, TERM_CUSTOM_NONBONDED = 4096, 8192, 16384, 32768, 65536
TERM_ALL = 131071
# kinds of b200md_set_bonded_groups
BONDED_KINDS = {"bonds": 0, "angles": 1, "torsions": 2, "rb_torsions": 3, "cmap": 4, "custom_torsions": 5, "custom_bonds": 6,
                "custom_externals": 7, "custom_angles": 9, "custom_compound": 10, "custom_centroid": 11}
PHASES = {"pair": 0, "pme_spread": 1, "pme_fft_conv": 2, "pme_gather": 3, "integrate": 4, "list_build": 5, "bonded": 6,
          "custom_torsions": 7, "custom_compound": 8, "custom_centroid": 9, "gbsa": 10, "list_prep": 11, "list_tiles": 12,
          "rmsd": 13, "custom_nonbonded": 14}


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
        # the custom classes: field prefix, field of each term's expression, programs per expression (E and dE/dtheta, E and
        # dE/dr, E and dE/dx, dE/dy, dE/dz, E and dE/dtheta; a compound bond's E and its derivatives by every coordinate of its
        # particles, whose number and periodic flag per expression its call also takes; a centroid bond's likewise, by the
        # coordinates of its group centres, and its call also takes the groups), what messages call the terms
        for prefix, expr_field, nprog, name, call in (
                ("custom", "_prog", 2, "custom torsions", L.b200md_set_custom_torsions),
                ("cbond", "_prog", 2, "custom bonds", L.b200md_set_custom_bonds),
                ("cext", "_prog", 4, "custom externals", L.b200md_set_custom_externals),
                ("cangle", "_prog", 2, "custom angles", L.b200md_set_custom_angles),
                ("ccompound", "_expr", None, "custom compound bonds", L.b200md_set_custom_compound),
                ("ccentroid", "_expr", None, "custom centroid bonds", L.b200md_set_custom_centroid)):
            expr = getattr(d, prefix + expr_field)
            if not len(expr):
                continue
            start, op, arg, imm = (getattr(d, prefix + k) for k in ("_prog_start", "_op", "_arg", "_imm"))
            if not len(op):
                raise EngineError("%s without programs: compile desc.%s_energy into %s_op / %s_arg / %s_imm / %s_prog_start first (the "
                                  "plugin's expression translator)" % (name, prefix, prefix, prefix, prefix, prefix))
            params = _f64(getattr(d, prefix + "_params")).reshape(len(expr), -1)
            atoms = _i32(getattr(d, prefix + "_atoms")).reshape(len(expr), -1)
            tail = ()
            if nprog is None:
                npart = getattr(d, prefix + ("_groups_per_bond" if prefix == "ccentroid" else "_particles"))
                head = (len(npart), _ip(_i32(npart)), _ip(_i32(getattr(d, prefix + "_periodic"))))
            else:
                head = ((len(start) - 1)//nprog,)
            if prefix == "ccentroid":
                gs = _i32(d.ccentroid_group_start)
                tail = (len(gs) - 1, _ip(gs), _ip(_i32(d.ccentroid_group_atoms)), _dp(_f64(d.ccentroid_group_weights)))
            self._ck(call(self.h, *head, _ip(_i32(start)), _ip(_i32(op)), _ip(_i32(arg)), _dp(_f64(imm)), params.shape[1], len(expr),
                          _ip(_i32(expr)), _ip(atoms), _dp(params), *tail))
        if len(d.custom_global_values):
            self._ck(L.b200md_set_custom_globals(self.h, len(d.custom_global_values), _dp(_f64(d.custom_global_values))))
        for kind, g in self._bonded_groups.items():
            g = _i32(g)
            self._ck(L.b200md_set_bonded_groups(self.h, BONDED_KINDS[kind], len(g), _ip(g)))
        if len(d.gb_charges):
            self._ck(L.b200md_set_gbsa(self.h, int(d.gb_method), float(d.cutoff), float(d.gb_solute_dielectric),
                                       float(d.gb_solvent_dielectric), float(d.gb_surface_area_energy), _dp(_f64(d.gb_charges)),
                                       _dp(_f64(d.gb_radii)), _dp(_f64(d.gb_scales))))
        if len(d.cnb_group):
            p = np.ascontiguousarray(d.cnb_params, dtype=np.float64)
            ex = _i32(np.asarray(d.cnb_excl).reshape(-1, 2))
            self._ck(L.b200md_set_custom_nonbonded(self.h, int(d.cnb_method), float(d.cnb_cutoff), len(d.cnb_group), _ip(_i32(d.cnb_prog_start)),
                                                   _ip(_i32(d.cnb_op)), _ip(_i32(d.cnb_arg)), _dp(_f64(d.cnb_imm)), _ip(_i32(d.cnb_nparams)),
                                                   p.shape[2], _dp(p), _dp(_f64(d.cnb_switch)), _ip(_i32(d.cnb_group)), len(ex),
                                                   _ip(_i32(ex[:, 0])), _ip(_i32(ex[:, 1]))))
            dims = _i32(np.asarray(d.cnb_table_dims).reshape(-1, 4))
            self._ck(L.b200md_set_custom_tables(self.h, len(dims), _ip(dims), _ip(_i32(d.cnb_table_start)), _dp(_f64(d.cnb_table_values))))
            if len(d.cnb_lrc):
                self._ck(L.b200md_set_custom_nonbonded_lrc(self.h, len(d.cnb_lrc), _dp(_f64(d.cnb_lrc))))
        if d.cv_count:
            self._ck(L.b200md_set_cv_forces(self.h, int(d.cv_count)))
        if len(d.rmsd_group):
            self._ck(L.b200md_set_rmsd(self.h, len(d.rmsd_group), _ip(_i32(d.rmsd_start)), _ip(_i32(d.rmsd_atoms)),
                                       _dp(_f64(d.rmsd_ref)), _ip(_i32(d.rmsd_group))))
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

    # ---- CalcNonbondedForceKernel::copyParametersToContext (and Context::setParameter of its parameter offsets) ----
    def update_nonbonded_params(self, desc, dispersion_coefficient=None):
        """The per-atom charges, sigmas and epsilons and the per-exception (chargeProd, sigma, epsilon) of `desc` for the same
        atoms and exceptions.  dispersion_coefficient defaults to desc.dispersion_coefficient(), as at definition; parameter
        offsets pass the one of the parameters' default values instead (NonbondedForceImpl::calcDispersionCorrection)."""
        q, sig, eps = _f64(desc.charges), _f64(desc.sigmas), _f64(desc.epsilons)
        eqq, esig, eeps = _f64(desc.exc_qq), _f64(desc.exc_sigma), _f64(desc.exc_eps)
        if not (len(q) == len(sig) == len(eps) == self.natoms):
            raise ValueError("update_nonbonded_params: charges, sigmas and epsilons need one value per atom (%d)" % self.natoms)
        if not (len(eqq) == len(esig) == len(eeps) == len(desc.exc_i)):
            raise ValueError("update_nonbonded_params: exc_qq, exc_sigma and exc_eps need one value per exception")
        disp = desc.dispersion_coefficient() if dispersion_coefficient is None else dispersion_coefficient
        self._ck(self.lib.b200md_update_nonbonded_params(self.h, _dp(q), _dp(sig), _dp(eps), len(eqq), _dp(eqq), _dp(esig), _dp(eeps),
                                                         float(disp)))

    # ---- Calc{RBTorsion,CMAPTorsion}ForceKernel::copyParametersToContext ----
    def update_rb_torsion_params(self, c):
        c = _f64(c)
        self._ck(self.lib.b200md_update_rb_torsion_params(self.h, len(c), _dp(c)))

    def update_cmap_params(self, size, coeff, cmap_map):
        size, coeff, cmap_map = _i32(size), _f64(coeff), _i32(cmap_map)
        self._ck(self.lib.b200md_update_cmap_params(self.h, len(size), _ip(size), _dp(coeff), len(cmap_map), _ip(cmap_map)))

    # ---- CalcCustom{Torsion,Bond,External,Angle,CompoundBond,CentroidBond}ForceKernel::copyParametersToContext and the globals ----
    def _update_custom(self, call, params):
        p = _f64(params)
        self._ck(call(self.h, len(p), _dp(p)))

    def update_custom_torsion_params(self, params):
        """New per-torsion parameters [n, param_stride] for the same torsions and expressions."""
        self._update_custom(self.lib.b200md_update_custom_torsion_params, params)

    def update_custom_bond_params(self, params):
        """New per-bond parameters [n, param_stride] for the same custom bonds and expressions."""
        self._update_custom(self.lib.b200md_update_custom_bond_params, params)

    def update_custom_external_params(self, params):
        """New per-particle parameters [n, param_stride] for the same custom externals and expressions."""
        self._update_custom(self.lib.b200md_update_custom_external_params, params)

    def update_custom_angle_params(self, params):
        """New per-angle parameters [n, param_stride] for the same custom angles and expressions."""
        self._update_custom(self.lib.b200md_update_custom_angle_params, params)

    def update_custom_compound_params(self, params):
        """New per-bond parameters [n, param_stride] for the same custom compound bonds and expressions."""
        self._update_custom(self.lib.b200md_update_custom_compound_params, params)

    def update_custom_centroid_params(self, params):
        """New per-bond parameters [n, param_stride] for the same custom centroid bonds, groups and expressions."""
        self._update_custom(self.lib.b200md_update_custom_centroid_params, params)

    # ---- CalcGBSAOBCForceKernel::copyParametersToContext ----
    def update_gbsa_params(self, charges, radii, scales):
        """New per-atom charges, radii and scale factors of the generalized Born force (one per atom, as before)."""
        q, r, s = _f64(charges), _f64(radii), _f64(scales)
        if not (len(q) == len(r) == len(s)):
            raise ValueError("update_gbsa_params: charges, radii and scales differ in length")
        self._ck(self.lib.b200md_update_gbsa_params(self.h, len(q), _dp(q), _dp(r), _dp(s)))

    # ---- CalcCustomNonbondedForceKernel::copyParametersToContext ----
    def update_custom_nonbonded_params(self, params):
        """New per-particle parameters [objects, N, stride] of the custom nonbonded objects, into the same device buffers."""
        p = np.ascontiguousarray(params, dtype=np.float64)
        self._ck(self.lib.b200md_update_custom_nonbonded_params(self.h, p.shape[1], _dp(p)))

    def set_custom_nonbonded_lrc(self, coefficients):
        """The long-range coefficient of every custom nonbonded object (energy += coefficient/volume)."""
        c = _f64(coefficients)
        self._ck(self.lib.b200md_set_custom_nonbonded_lrc(self.h, len(c), _dp(c)))

    # ---- CalcRMSDForceKernel::copyParametersToContext ----
    def update_rmsd(self, start, atoms, ref):
        """New particle lists and reference positions ([entries, 3]) for the same number of RMSD forces."""
        start, atoms, ref = _i32(start), _i32(atoms), _f64(ref)
        self._ck(self.lib.b200md_update_rmsd(self.h, len(start) - 1, _ip(start), _ip(atoms), _dp(ref)))

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

    def get_list(self):
        """(sorig [padded atoms], tile_i [T], tile_j [T, 32], tile_mask [T, 32] uint32) of the current neighbour list; the
        tiles in the order of the slot pools, which depends on the order in which they were emitted"""
        n = C.c_int64()
        sorig = np.empty(self.stats()["padded_atoms"], dtype=np.int32)
        self._ck(self.lib.b200md_get_list(self.h, _ip(sorig), 0, None, None, None, C.byref(n)))
        t = n.value
        ti, tj, tm = np.empty(t, np.int32), np.empty((t, 32), np.int32), np.empty((t, 32), np.uint32)
        self._ck(self.lib.b200md_get_list(self.h, None, t, _ip(ti), _ip(tj), tm.ctypes.data_as(C.POINTER(C.c_uint)), C.byref(n)))
        return sorig, ti, tj, tm

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
