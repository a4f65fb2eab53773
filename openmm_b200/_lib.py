"""ctypes binding of libb200md.so (C-ABI: include/b200md.h).  No fallback: a missing library is a hard error."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("B200MD_LIB", os.path.join(_HERE, "libb200md.so"))      # B200MD_LIB: experiment builds (csrc/Makefile `dbl`)


class NonbondedDesc(C.Structure):
    _fields_ = [("method", C.c_int), ("cutoff", C.c_double), ("use_switch", C.c_int), ("switch_distance", C.c_double),
                ("rf_dielectric", C.c_double), ("ewald_alpha", C.c_double), ("grid", C.c_int*3),
                ("dispersion_coefficient", C.c_double), ("exceptions_periodic", C.c_int)]


class Stats(C.Structure):
    _fields_ = [("natoms", C.c_int64), ("padded_atoms", C.c_int64), ("num_blocks", C.c_int64), ("num_tiles", C.c_int64),
                ("num_mask_tiles", C.c_int64), ("list_builds", C.c_int64), ("force_evals", C.c_int64),
                ("kernel_launches", C.c_int64), ("pairs_in_cutoff", C.c_int64), ("pme_grid", C.c_int*3),
                ("ewald_alpha", C.c_double), ("overflow", C.c_int),
                ("graph_instantiations", C.c_int64)]


_P = C.c_void_p
_D = C.POINTER(C.c_double)
_I = C.POINTER(C.c_int)
_F = C.POINTER(C.c_float)

# name -> (restype, argtypes); this table must list every symbol declared in include/b200md.h
SIGNATURES = {
    "b200md_create": (C.c_int, [C.POINTER(_P), C.c_int, C.c_int]),
    "b200md_destroy": (None, [_P]),
    "b200md_last_error": (C.c_char_p, [_P]),
    "b200md_version": (C.c_char_p, []),
    "b200md_set_masses": (C.c_int, [_P, _D]),
    "b200md_set_nonbonded": (C.c_int, [_P, C.POINTER(NonbondedDesc), _D, _D, _D]),
    "b200md_set_exceptions": (C.c_int, [_P, C.c_int, _I, _I, _D, _D, _D]),
    "b200md_set_bonds": (C.c_int, [_P, C.c_int, _I, _I, _D, _D]),
    "b200md_set_angles": (C.c_int, [_P, C.c_int, _I, _I, _I, _D, _D]),
    "b200md_set_torsions": (C.c_int, [_P, C.c_int, _I, _I, _I, _I, _I, _D, _D]),
    "b200md_set_rb_torsions": (C.c_int, [_P, C.c_int, _I, _I, _I, _I, _D]),
    "b200md_set_cmap": (C.c_int, [_P, C.c_int, _I, _D, C.c_int, _I, _I]),
    "b200md_set_custom_torsions": (C.c_int, [_P, C.c_int, _I, _I, _I, _D, C.c_int, C.c_int, _I, _I, _D]),
    "b200md_set_custom_bonds": (C.c_int, [_P, C.c_int, _I, _I, _I, _D, C.c_int, C.c_int, _I, _I, _D]),
    "b200md_set_custom_externals": (C.c_int, [_P, C.c_int, _I, _I, _I, _D, C.c_int, C.c_int, _I, _I, _D]),
    "b200md_set_custom_angles": (C.c_int, [_P, C.c_int, _I, _I, _I, _D, C.c_int, C.c_int, _I, _I, _D]),
    "b200md_set_custom_compound": (C.c_int, [_P, C.c_int, _I, _I, _I, _I, _I, _D, C.c_int, C.c_int, _I, _I, _D]),
    "b200md_set_custom_centroid": (C.c_int, [_P, C.c_int, _I, _I, _I, _I, _I, _D, C.c_int, C.c_int, _I, _I, _D, C.c_int, _I, _I, _D]),
    "b200md_set_custom_globals": (C.c_int, [_P, C.c_int, _D]),
    "b200md_set_bonded_groups": (C.c_int, [_P, C.c_int, C.c_int, _I]),
    "b200md_set_constraints": (C.c_int, [_P, C.c_int, _I, _I, _D]),
    "b200md_check_constraints": (C.c_int, [C.c_int, _D, C.c_int, _I, _I, _D, C.c_char_p, C.c_int]),
    "b200md_ccma_setup_probe": (C.c_int, [C.c_int, _D, C.c_int, _I, _I, _D, C.c_int, _I, _I, _I, _D, _I, _I, _I, _I, _I, _F, C.c_int]),
    "b200md_set_cm_remover": (C.c_int, [_P, C.c_int]),
    "b200md_remove_cm_motion": (C.c_int, [_P]),
    "b200md_set_precision": (C.c_int, [_P, C.c_int]),
    "b200md_get_precision": (C.c_int, [_P]),
    "b200md_finalize": (C.c_int, [_P]),
    "b200md_update_nonbonded_params": (C.c_int, [_P, _D, _D, _D, C.c_int, _D, _D, _D, C.c_double]),
    "b200md_update_bonded_params": (C.c_int, [_P, C.c_int, C.c_int, _D, _D, _I]),
    "b200md_update_rb_torsion_params": (C.c_int, [_P, C.c_int, _D]),
    "b200md_update_cmap_params": (C.c_int, [_P, C.c_int, _I, _D, C.c_int, _I]),
    "b200md_update_custom_torsion_params": (C.c_int, [_P, C.c_int, _D]),
    "b200md_update_custom_bond_params": (C.c_int, [_P, C.c_int, _D]),
    "b200md_update_custom_external_params": (C.c_int, [_P, C.c_int, _D]),
    "b200md_update_custom_angle_params": (C.c_int, [_P, C.c_int, _D]),
    "b200md_update_custom_compound_params": (C.c_int, [_P, C.c_int, _D]),
    "b200md_update_custom_centroid_params": (C.c_int, [_P, C.c_int, _D]),
    "b200md_set_gbsa": (C.c_int, [_P, C.c_int, C.c_double, C.c_double, C.c_double, C.c_double, _D, _D, _D]),
    "b200md_update_gbsa_params": (C.c_int, [_P, C.c_int, _D, _D, _D]),
    "b200md_set_custom_nonbonded": (C.c_int, [_P, C.c_int, C.c_double, C.c_int, _I, _I, _I, _D, _I, C.c_int, _D, _D, _I, C.c_int, _I, _I]),
    "b200md_set_custom_tables": (C.c_int, [_P, C.c_int, _I, _I, _D]),
    "b200md_update_custom_nonbonded_params": (C.c_int, [_P, C.c_int, _D]),
    "b200md_set_custom_nonbonded_lrc": (C.c_int, [_P, C.c_int, _D]),
    "b200md_custom_nonbonded_probe": (C.c_int, [C.c_int, _I, _I, _I, _D, C.c_int, C.c_int, C.c_int, C.c_double, _D, _D, C.c_int, _I, _I,
                                                _D, _D, C.c_char_p, C.c_int]),
    "b200md_set_rmsd": (C.c_int, [_P, C.c_int, _I, _I, _D, _I]),
    "b200md_update_rmsd": (C.c_int, [_P, C.c_int, _I, _I, _D]),
    "b200md_rmsd_probe": (C.c_int, [C.c_int, _D, _D, _D, _D]),
    "b200md_set_cv_forces": (C.c_int, [_P, C.c_int]),
    "b200md_cv_copy_state": (C.c_int, [_P, _P]),
    "b200md_cv_snapshot_forces": (C.c_int, [_P, _P, C.c_int]),
    "b200md_set_cv_coefficients": (C.c_int, [_P, C.c_int, _D]),
    "b200md_rmsd_eigen_probe": (C.c_int, [_D, _D, _D]),
    "b200md_custom_program_probe": (C.c_int, [C.c_int, _I, _I, _I, _D, C.c_int, C.c_int, C.c_int, C.c_double, _D, _D, _D,
                                              C.c_char_p, C.c_int]),
    "b200md_custom_term_probe": (C.c_int, [C.c_int, C.c_int, _I, _I, _I, _D, C.c_int, C.c_int, C.c_int, _D, _D, _D, _D, _D,
                                           C.c_char_p, C.c_int]),
    "b200md_custom_compound_probe": (C.c_int, [C.c_int, C.c_int, _I, _I, _I, _D, C.c_int, C.c_int, C.c_int, _D, _D, _D, _D, _D,
                                               C.c_char_p, C.c_int]),
    "b200md_set_box": (C.c_int, [_P, _D, _D, _D]),
    "b200md_get_box": (C.c_int, [_P, _D, _D, _D]),
    "b200md_set_barostat_molecules": (C.c_int, [_P, C.c_int, _I, _I]),
    "b200md_scale_coordinates": (C.c_int, [_P, C.c_double, C.c_double, C.c_double]),
    "b200md_restore_coordinates": (C.c_int, [_P]),
    "b200md_set_positions": (C.c_int, [_P, _D]),
    "b200md_get_positions": (C.c_int, [_P, _D]),
    "b200md_set_velocities": (C.c_int, [_P, _D]),
    "b200md_get_velocities": (C.c_int, [_P, _D]),
    "b200md_get_forces": (C.c_int, [_P, _D]),
    "b200md_set_time": (C.c_int, [_P, C.c_double]),
    "b200md_get_time": (C.c_double, [_P]),
    "b200md_get_step_count": (C.c_int64, [_P]),
    "b200md_checkpoint_save": (C.c_int64, [_P, _P, C.c_int64]),
    "b200md_checkpoint_load": (C.c_int, [_P, _P, C.c_int64]),
    "b200md_compute": (C.c_int, [_P, C.c_int, C.c_int, _D]),
    "b200md_compute_groups": (C.c_int, [_P, C.c_int, C.c_uint, C.c_int, _D]),
    "b200md_set_integrator": (C.c_int, [_P, C.c_int, C.c_double, C.c_double, C.c_double, C.c_int, C.c_double]),
    "b200md_step": (C.c_int, [_P, C.c_int]),
    "b200md_integrate_only": (C.c_int, [_P]),
    "b200md_kinetic_energy": (C.c_int, [_P, _D]),
    "b200md_apply_constraints": (C.c_int, [_P, C.c_double]),
    "b200md_apply_velocity_constraints": (C.c_int, [_P, C.c_double]),
    "b200md_synchronize": (C.c_int, [_P]),
    "b200md_comm_unique_id": (C.c_int, [_P]),
    "b200md_ownership_probe": (C.c_int, [C.c_int, _D, C.c_int, _I, _I, _D, C.c_int, _I, _I]),
    "b200md_comm_init": (C.c_int, [_P, C.c_int, C.c_int, _P]),
    "b200md_get_stats": (C.c_int, [_P, C.POINTER(Stats)]),
    "b200md_time_phase": (C.c_int, [_P, C.c_int, C.c_int, _D]),
    "b200md_get_list": (C.c_int, [_P, _I, C.c_int64, _I, _I, C.POINTER(C.c_uint), C.POINTER(C.c_int64)]),
    "b200md_fft3d_r2c": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, _F, _F]),
    "b200md_fft3d_c2r": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, _F, _F]),
    "b200md_pme_create": (C.c_int, [C.POINTER(_P), C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_double]),
    "b200md_pme_exec": (C.c_int, [_P, _F, _D, C.c_int, _F, _D]),
    "b200md_cuda_stream": (_P, [_P]),
}

_lib = None


def load():
    """Load libb200md.so; raises (never falls back) when the CUDA extension has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError("libb200md.so is missing (%s): build it with `python -c 'import __graft_entry__ as g; g.build()'`. "
                               "openmm_b200 has no CPU fallback." % LIB_PATH)
        lib = C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib
