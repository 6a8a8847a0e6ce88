"""ctypes binding of libmollyb200.so (include/mollyb200.h). No torch types cross this boundary."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("MOLLYB200_LIB") or os.path.join(_HERE, "libmollyb200.so")  # override: tuning variants

MB_LJ, MB_COULOMB, MB_CRF, MB_EWALD_REAL = 0, 1, 2, 3
MB_CUT_NONE, MB_CUT_DISTANCE, MB_CUT_SHIFTED_POTENTIAL, MB_CUT_SHIFTED_FORCE = 0, 1, 2, 3
MB_CUT_CUBIC_SPLINE, MB_CUT_POLYNOMIAL = 4, 5
MB_MIX_LORENTZ, MB_MIX_GEOMETRIC = 0, 1
MB_VC_NONE, MB_VC_IMMEDIATE, MB_VC_BERENDSEN, MB_VC_VRESCALE = 0, 1, 2, 3
MB_OK, MB_ERR_INVALID, MB_ERR_CUDA, MB_ERR_CAPACITY, MB_ERR_STATE, MB_ERR_NOGPU = 0, -1, -2, -3, -4, -5

EXPORTED = [
    "mb_last_error", "mb_device_count", "mb_ctx_create", "mb_ctx_destroy", "mb_set_atoms", "mb_set_atoms_soa",
    "mb_set_box", "mb_set_inters", "mb_set_exceptions", "mb_set_neighbor_policy", "mb_forces", "mb_energy",
    "mb_forces_energy", "mb_simulate_vv", "mb_remove_cm_motion", "mb_kinetic_energy", "mb_rebuild_neighbors",
    "mb_stats", "mb_synchronize", "mb_set_capacity_scale", "mb_set_launch_config", "mb_comm_unique_id",
    "mb_comm_init", "mb_decomp_plan", "mb_set_profiling", "mb_set_specific", "mb_forces_energy_all", "mb_set_pme", "mb_pme_plan",
    "mb_set_lj_dispersion_correction", "mb_random_velocities", "mb_kinetic_energy_tensor", "mb_set_box_triclinic",
    "mb_simulate_vv_log", "mb_minimize_sd", "mb_set_velocity_coupling", "mb_simulate_langevin",
    "mb_simulate_nose_hoover", "mb_set_specific_levels", "mb_simulate_mts", "mb_set_implicit_solvent",
    "mb_simulate_langevin_splitting", "mb_simulate_verlet", "mb_simulate_stormer_verlet", "mb_simulate_overdamped_langevin",
    "mb_set_dpd", "mb_forces_energy_vel", "mb_simulate_dpd_vv", "mb_simulate_group",
]
MB_GB_MAX_NECK_CLASSES = 32
# specific interaction kinds of mb_set_specific (include/mollyb200.h)
(MB_SPECIFIC_HARMONIC_BOND, MB_SPECIFIC_HARMONIC_ANGLE, MB_SPECIFIC_PERIODIC_TORSION, MB_SPECIFIC_POSITION_RESTRAINT,
 MB_SPECIFIC_MORSE_BOND, MB_SPECIFIC_FENE_BOND, MB_SPECIFIC_COSINE_ANGLE, MB_SPECIFIC_UREY_BRADLEY, MB_SPECIFIC_HARMONIC_TORSION,
 MB_SPECIFIC_RB_TORSION, MB_SPECIFIC_N_KINDS) = range(11)
MB_MTS_MAX_LEVELS = 8
# integrator kinds of mb_simulate_group, one per mb_simulate_* entry (include/mollyb200.h)
(MB_INTEG_VV, MB_INTEG_LANGEVIN, MB_INTEG_NOSE_HOOVER, MB_INTEG_MTS, MB_INTEG_LANGEVIN_SPLITTING, MB_INTEG_VERLET,
 MB_INTEG_STORMER_VERLET, MB_INTEG_OVERDAMPED_LANGEVIN, MB_INTEG_DPD_VV) = range(9)
MB_SPLIT_MAX_OPS = 32


class MBInter(C.Structure):
    _fields_ = [
        ("kind", C.c_int32), ("cutoff_kind", C.c_int32), ("r_cut", C.c_double), ("r_act", C.c_double),
        ("weight_special", C.c_double), ("coulomb_const", C.c_double), ("solvent_dielectric", C.c_double),
        ("ewald_alpha", C.c_double), ("sigma_mix", C.c_int32), ("eps_mix", C.c_int32), ("approx_erfc", C.c_int32),
        ("use_neighbors", C.c_int32),
    ]


class MBGbsa(C.Structure):
    _fields_ = [
        ("dist_cutoff", C.c_double), ("offset", C.c_double), ("probe_radius", C.c_double), ("sa_factor", C.c_double),
        ("factor_solute", C.c_double), ("factor_solvent", C.c_double), ("kappa", C.c_double), ("neck_scale", C.c_double),
        ("neck_cut", C.c_double), ("use_ace", C.c_int32), ("n_neck_classes", C.c_int32),
    ]


class MBStats(C.Structure):
    _fields_ = [
        ("n_atoms", C.c_int64), ("n_rebuilds", C.c_int64), ("n_force_evals", C.c_int64), ("n_steps", C.c_int64),
        ("n_list_entries", C.c_int64), ("n_pairs_in_list", C.c_int64), ("n_bricks", C.c_int32),
        ("n_cells", C.c_int32 * 3), ("brick_dims", C.c_int32 * 3), ("halo_capacity", C.c_int32),
        ("list_stride", C.c_int32), ("max_neighbors", C.c_int32), ("max_halo", C.c_int32), ("path", C.c_int32),
        ("violations", C.c_int32), ("r_list", C.c_double), ("kernel_launches", C.c_int64),
        ("force_ms", C.c_double), ("vv_ms", C.c_double), ("rebuild_ms", C.c_double),
        ("force_launches", C.c_int64), ("vv_launches", C.c_int64), ("rebuild_launches", C.c_int64),
        ("graph_mode", C.c_int32), ("n_prunes", C.c_int32), ("peer_transport", C.c_int32), ("reserved_", C.c_int32),
    ]


class MBVVParams(C.Structure):
    _fields_ = [
        ("dt", C.c_double), ("n_steps", C.c_int64), ("init_step", C.c_int64), ("remove_cm_every", C.c_int32),
        ("andersen_kT", C.c_double), ("andersen_prob", C.c_double), ("rng_ctr1", C.c_uint64), ("rng_key", C.c_uint64),
    ]


class MBDpd(C.Structure):
    _fields_ = [
        ("a", C.c_double), ("gamma", C.c_double), ("sigma", C.c_double), ("r_c", C.c_double), ("dt", C.c_double),
        ("key", C.c_uint64), ("use_neighbors", C.c_int32),
    ]


class MBDpdVVParams(C.Structure):
    _fields_ = [
        ("dt", C.c_double), ("n_steps", C.c_int64), ("init_step", C.c_int64), ("remove_cm_every", C.c_int32),
        ("lambda_", C.c_double),
    ]


class MBLangevinParams(C.Structure):
    _fields_ = [
        ("dt", C.c_double), ("n_steps", C.c_int64), ("init_step", C.c_int64), ("remove_cm_every", C.c_int32),
        ("kT", C.c_double), ("friction", C.c_double), ("rng_ctr1", C.c_uint64), ("rng_key", C.c_uint64),
    ]


class MBNoseHooverParams(C.Structure):
    _fields_ = [
        ("dt", C.c_double), ("n_steps", C.c_int64), ("init_step", C.c_int64), ("remove_cm_every", C.c_int32),
        ("kT", C.c_double), ("damping", C.c_double),
    ]


class MBMTSParams(C.Structure):
    _fields_ = [
        ("dt", C.c_double), ("n_steps", C.c_int64), ("init_step", C.c_int64), ("remove_cm_every", C.c_int32),
        ("n_levels", C.c_int32), ("fractions", C.c_int32 * MB_MTS_MAX_LEVELS), ("langevin", C.c_int32), ("reserved_", C.c_int32),
        ("kT", C.c_double), ("friction", C.c_double), ("rng_ctr1", C.c_uint64), ("rng_key", C.c_uint64),
    ]


class MBSplittingParams(C.Structure):
    _fields_ = [
        ("dt", C.c_double), ("n_steps", C.c_int64), ("init_step", C.c_int64), ("remove_cm_every", C.c_int32),
        ("kT", C.c_double), ("friction", C.c_double), ("rng_ctr1", C.c_uint64), ("rng_key", C.c_uint64),
        ("n_ops", C.c_int32), ("ops", C.c_char * MB_SPLIT_MAX_OPS),
    ]


class MBStormerParams(C.Structure):
    _fields_ = [("dt", C.c_double), ("n_steps", C.c_int64), ("init_step", C.c_int64)]


class MBVCoupling(C.Structure):
    _fields_ = [("kind", C.c_int32), ("n_steps", C.c_int32), ("kT", C.c_double), ("tau", C.c_double)]


class MBLog(C.Structure):
    _fields_ = [
        ("energy_every", C.c_int64), ("coords_every", C.c_int64), ("vels_every", C.c_int64), ("log_initial", C.c_int32),
        ("reserved_", C.c_int32), ("energies", C.c_void_p), ("coords", C.c_void_p), ("vels", C.c_void_p),
        ("energy_capacity", C.c_int64), ("coords_capacity", C.c_int64), ("vels_capacity", C.c_int64),
        ("n_energies", C.c_int64), ("n_coords", C.c_int64), ("n_vels", C.c_int64),
    ]


class MBSDParams(C.Structure):
    _fields_ = [
        ("step_size", C.c_double), ("max_steps", C.c_int64), ("tol", C.c_double), ("init_step", C.c_int64),
        ("trace", C.c_void_p), ("trace_capacity", C.c_int64), ("n_iterations", C.c_int64), ("energy", C.c_double),
        ("max_force", C.c_double), ("final_step_size", C.c_double), ("converged", C.c_int32), ("reserved_", C.c_int32),
    ]


class MollyB200Error(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"libmollyb200 error {code}: {msg}")
        self.code = code


class MBGroupMember(C.Structure):
    _fields_ = [("ctx", C.c_void_p), ("coords", C.c_void_p), ("vels", C.c_void_p), ("kind", C.c_int32),
                ("params", C.c_void_p), ("log", C.c_void_p), ("status", C.c_int32)]


_lib = None


def load():
    """Load libmollyb200.so. Fails loudly if it has not been built: there is no fallback path."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build it with `python __graft_entry__.py` (nvcc, sm_90a). "
            "mollyb200 has no CPU or PyTorch fallback.")
    L = C.CDLL(LIB_PATH)
    vp, i32, i64, dbl = C.c_void_p, C.c_int32, C.c_int64, C.c_double
    L.mb_last_error.restype = C.c_char_p
    L.mb_device_count.restype = C.c_int
    L.mb_ctx_create.argtypes = [C.c_int, C.c_int, vp, C.POINTER(vp)]
    L.mb_ctx_destroy.argtypes = [vp]
    L.mb_ctx_destroy.restype = None
    L.mb_set_atoms.argtypes = [vp, i64, vp]
    L.mb_set_atoms_soa.argtypes = [vp, i64, vp, vp, vp, vp]
    L.mb_set_box.argtypes = [vp, C.POINTER(dbl)]
    L.mb_set_inters.argtypes = [vp, C.c_int, C.POINTER(MBInter)]
    L.mb_set_exceptions.argtypes = [vp, i64, vp, vp, i64, vp, vp]
    L.mb_set_neighbor_policy.argtypes = [vp, dbl, C.c_int]
    L.mb_forces.argtypes = [vp, vp, vp, vp, i64]
    L.mb_energy.argtypes = [vp, vp, vp, i64]
    L.mb_forces_energy.argtypes = [vp, vp, vp, vp, vp, i64]
    L.mb_simulate_vv.argtypes = [vp, vp, vp, C.POINTER(MBVVParams)]
    L.mb_simulate_vv_log.argtypes = [vp, vp, vp, C.POINTER(MBVVParams), C.POINTER(MBLog)]
    L.mb_simulate_langevin.argtypes = [vp, vp, vp, C.POINTER(MBLangevinParams), C.POINTER(MBLog)]
    L.mb_simulate_nose_hoover.argtypes = [vp, vp, vp, C.POINTER(MBNoseHooverParams), C.POINTER(MBLog)]
    L.mb_simulate_mts.argtypes = [vp, vp, vp, C.POINTER(MBMTSParams), C.POINTER(MBLog)]
    L.mb_simulate_langevin_splitting.argtypes = [vp, vp, vp, C.POINTER(MBSplittingParams), C.POINTER(MBLog)]
    L.mb_simulate_verlet.argtypes = [vp, vp, vp, C.POINTER(MBVVParams), C.POINTER(MBLog)]
    L.mb_simulate_stormer_verlet.argtypes = [vp, vp, vp, C.POINTER(MBStormerParams), C.POINTER(MBLog)]
    L.mb_simulate_overdamped_langevin.argtypes = [vp, vp, vp, C.POINTER(MBLangevinParams), C.POINTER(MBLog)]
    L.mb_set_dpd.argtypes = [vp, C.POINTER(MBDpd)]
    L.mb_forces_energy_vel.argtypes = [vp, vp, vp, vp, vp, i64]
    L.mb_simulate_dpd_vv.argtypes = [vp, vp, vp, C.POINTER(MBDpdVVParams), C.POINTER(MBLog)]
    L.mb_simulate_group.argtypes = [i32, C.POINTER(MBGroupMember)]
    L.mb_set_specific_levels.argtypes = [vp, C.c_int, i64, vp]
    L.mb_minimize_sd.argtypes = [vp, vp, C.POINTER(MBSDParams)]
    L.mb_set_velocity_coupling.argtypes = [vp, C.POINTER(MBVCoupling)]
    L.mb_remove_cm_motion.argtypes = [vp, vp]
    L.mb_kinetic_energy.argtypes = [vp, vp, C.POINTER(dbl)]
    L.mb_rebuild_neighbors.argtypes = [vp, vp]
    L.mb_stats.argtypes = [vp, C.POINTER(MBStats)]
    L.mb_synchronize.argtypes = [vp]
    L.mb_set_capacity_scale.argtypes = [vp, dbl]
    L.mb_set_launch_config.argtypes = [vp, C.POINTER(i32), i32]
    L.mb_comm_unique_id.argtypes = [vp]
    L.mb_comm_init.argtypes = [vp, vp, C.c_int, C.c_int]
    L.mb_set_specific.argtypes = [vp, C.c_int, i64, vp, vp]
    L.mb_set_pme.argtypes = [vp, C.c_double, C.c_double, C.c_int, C.c_double, i64, vp, vp]
    L.mb_pme_plan.argtypes = [vp, C.c_double, C.c_double, C.c_int, vp, vp, vp, C.c_int]
    L.mb_forces_energy_all.argtypes = [vp, vp, vp, vp, i64]
    L.mb_set_lj_dispersion_correction.argtypes = [vp, dbl]
    L.mb_set_implicit_solvent.argtypes = [vp, C.POINTER(MBGbsa), vp, vp, vp, vp, vp, vp, vp, vp]
    L.mb_random_velocities.argtypes = [vp, vp, dbl, C.c_uint64, C.c_uint64]
    L.mb_kinetic_energy_tensor.argtypes = [vp, vp, C.POINTER(dbl)]
    L.mb_decomp_plan.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, C.POINTER(i32), vp, C.POINTER(i32), C.c_int]
    L.mb_set_profiling.argtypes = [vp, C.c_int]
    for name in EXPORTED:
        fn = getattr(L, name)
        if name not in ("mb_last_error", "mb_ctx_destroy", "mb_device_count"):
            fn.restype = C.c_int
    _lib = L
    return L


def check(rc):
    if rc != MB_OK:
        raise MollyB200Error(rc, load().mb_last_error().decode())
