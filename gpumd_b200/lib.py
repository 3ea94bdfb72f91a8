"""ctypes loader for libb200md.so (the C-ABI declared in include/b200md.h).

There is NO fallback: if the shared library is missing or no CUDA device is present, every entry
point raises.  PyTorch is used only as the owner of device memory and streams.
"""
import ctypes as C
from pathlib import Path

import os

PKG = Path(__file__).resolve().parent
# B200MD_LIB: a diagnostic build of the same library (gpumd_b200.build.build_lib(variant=...))
LIB_PATH = Path(os.environ.get("B200MD_LIB") or PKG / "libb200md.so")

_dp = C.POINTER(C.c_double)
_ip = C.POINTER(C.c_int)
_vp = C.c_void_p

# name -> (restype, argtypes); mirrors include/b200md.h one to one
SIGNATURES = {
    "b200md_last_error": (C.c_char_p, []),
    "b200md_launch_count": (C.c_longlong, []),
    "b200md_nep_create": (C.c_int, [C.c_char_p, C.c_int, C.POINTER(_vp)]),
    "b200md_nep_destroy": (None, [_vp]),
    "b200md_nep_info": (C.c_int, [_vp, C.c_int]),
    "b200md_nep_rc": (C.c_double, [_vp]),
    "b200md_nep_symbol": (C.c_char_p, [_vp, C.c_int]),
    "b200md_nep_compute": (C.c_int, [_vp, C.c_int, _dp, _ip, _vp, _vp, _vp, _vp, _vp, _vp]),
    "b200md_nep_compute_host": (C.c_int, [_vp, C.c_int, _dp, _ip, _vp, _vp, _vp, _vp, _vp]),
    "b200md_nep_export_neighbors": (C.c_int, [_vp, C.c_int, _vp, _vp, C.c_int, _vp, _vp, _vp]),
    "b200md_transpose_int": (C.c_int, [C.c_int, C.c_int, _vp, _vp, _vp]),
    "b200md_nep_export_descriptors": (C.c_int, [_vp, _vp, _vp]),
    "b200md_nep_export_schedule": (C.c_int, [_vp, _ip, _vp, _vp, _vp]),
    "b200md_nep_export_tiles": (C.c_int, [_vp, _vp, _vp, _vp]),
    "b200md_nep_export_mlp": (C.c_int, [_vp, _vp, _vp, _vp]),
    "b200md_nep_check": (C.c_int, [_vp, _vp]),
    "b200md_nep_profile": (C.c_int, [_vp, C.c_int]),
    "b200md_nep_profile_read": (C.c_int, [_vp, C.c_int, C.POINTER(C.c_float), _ip]),
    "b200md_nep_stage_name": (C.c_char_p, [C.c_int]),
    "b200md_nep_mean_neighbors": (C.c_int, [_vp, _dp]),
    "b200md_lj_create": (C.c_int, [C.c_char_p, C.c_int, C.POINTER(_vp)]),
    "b200md_lj_destroy": (None, [_vp]),
    "b200md_lj_rc": (C.c_double, [_vp]),
    "b200md_lj_info": (C.c_int, [_vp, C.c_int]),
    "b200md_lj_symbol": (C.c_char_p, [_vp, C.c_int]),
    "b200md_lj_compute": (C.c_int, [_vp, C.c_int, _dp, _ip, _vp, _vp, _vp, _vp, _vp, _vp]),
    "b200md_lj_check": (C.c_int, [_vp, _vp]),
    "b200md_lj_invalidate": (C.c_int, [_vp, C.c_int, _vp]),
    "b200md_tersoff_create": (C.c_int, [C.c_char_p, C.c_int, C.POINTER(_vp)]),
    "b200md_tersoff_destroy": (None, [_vp]),
    "b200md_tersoff_rc": (C.c_double, [_vp]),
    "b200md_tersoff_info": (C.c_int, [_vp, C.c_int]),
    "b200md_tersoff_symbol": (C.c_char_p, [_vp, C.c_int]),
    "b200md_tersoff_compute": (C.c_int, [_vp, C.c_int, _dp, _ip, _vp, _vp, _vp, _vp, _vp, _vp]),
    "b200md_tersoff_invalidate": (C.c_int, [_vp, C.c_int, _vp]),
    "b200md_tersoff_check": (C.c_int, [_vp, _vp]),
    "b200md_eam_create": (C.c_int, [C.c_char_p, C.c_int, C.POINTER(_vp)]),
    "b200md_eam_destroy": (None, [_vp]),
    "b200md_eam_rc": (C.c_double, [_vp]),
    "b200md_eam_info": (C.c_int, [_vp, C.c_int]),
    "b200md_eam_symbol": (C.c_char_p, [_vp, C.c_int]),
    "b200md_eam_compute": (C.c_int, [_vp, C.c_int, _dp, _ip, _vp, _vp, _vp, _vp, _vp, _vp]),
    "b200md_eam_invalidate": (C.c_int, [_vp, C.c_int, _vp]),
    "b200md_eam_check": (C.c_int, [_vp, _vp]),
    "b200md_compute_heat": (C.c_int, [C.c_int, C.c_int, _vp, _vp, _vp, C.c_int, _vp]),
    "b200md_apply_pbc": (C.c_int, [C.c_int, _dp, _ip, _vp, _vp]),
    "b200md_zero_properties": (C.c_int, [C.c_int, _vp, _vp, _vp, _vp]),
    "b200md_velocity_verlet": (C.c_int, [C.c_int, C.c_int, C.c_double, _vp, _vp, _vp, _vp, _vp]),
    "b200md_velocity_verlet_groups": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_double, _vp, _vp, _vp, _vp, _vp,
                                                C.c_int, C.c_int, _dp, _vp]),
    "b200md_thermo_scratch_bytes": (C.c_longlong, [C.c_int]),
    "b200md_find_thermo": (C.c_int, [C.c_int, C.c_int, C.c_double, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "b200md_scale_velocity": (C.c_int, [C.c_int, C.c_double, _vp, _vp]),
    "b200md_berendsen_temperature": (C.c_int, [C.c_int, C.c_int, C.c_double, C.c_double, _vp, _vp, _vp]),
    "b200md_nhc_create": (C.c_int, [C.c_longlong, C.c_double, C.c_double, C.c_double, C.POINTER(_vp)]),
    "b200md_nhc_destroy": (None, [_vp]),
    "b200md_nhc_half_step": (C.c_int, [_vp, C.c_int, C.c_int, C.c_double, _vp, _vp, _vp]),
    "b200md_bdp_create": (C.c_int, [C.c_longlong, C.c_double, C.c_double, C.c_uint, C.POINTER(_vp)]),
    "b200md_bdp_destroy": (None, [_vp]),
    "b200md_bdp_step": (C.c_int, [_vp, C.c_int, C.c_int, _vp, _vp, _vp]),
    "b200md_hac_create": (C.c_int, [C.c_int, C.c_int, C.c_int, C.POINTER(_vp)]),
    "b200md_hac_destroy": (None, [_vp]),
    "b200md_hac_sample": (C.c_int, [_vp, C.c_int, C.c_int, C.c_int, _vp, _vp, _vp]),
    "b200md_hac_finish": (C.c_int, [_vp, C.c_double, C.c_double, C.c_double, _dp, _dp, _vp]),
    "b200md_hac_series": (C.c_int, [_vp, _dp, _vp]),
    "b200md_hnemd_drive_scratch_bytes": (C.c_longlong, [C.c_int]),
    "b200md_hnemd_drive": (C.c_int, [C.c_int, C.c_int, _dp, _vp, _vp, _vp, _vp]),
    "b200md_hnemd_create": (C.c_int, [C.c_int, _dp, C.POINTER(_vp)]),
    "b200md_hnemd_destroy": (None, [_vp]),
    "b200md_hnemd_sample": (C.c_int, [_vp, C.c_int, C.c_int, C.c_int, _vp, _vp, _vp]),
    "b200md_hnemd_take": (C.c_int, [_vp, C.c_double, C.c_double, _dp, _dp, _vp]),
    "b200md_hnemd_drive_add": (C.c_int, [C.c_int, C.c_int, _dp, _vp, _vp, _vp, _vp, _vp]),
    "b200md_hnemd_drive_correct": (C.c_int, [C.c_int, C.c_int, C.c_double, _vp, _vp, _vp]),
    "b200md_hnemd_heat_row_scratch_bytes": (C.c_longlong, [C.c_int]),
    "b200md_hnemd_heat_row": (C.c_int, [C.c_int, C.c_int, _vp, _vp, _vp, C.c_int, _vp, _vp, _vp]),
    "b200md_hnemd_kappa": (C.c_int, [C.c_int, C.c_double, C.c_double, _dp, _dp, _dp]),
    "b200md_shc_create": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _ip, _ip, C.POINTER(_vp)]),
    "b200md_shc_destroy": (None, [_vp]),
    "b200md_shc_sample": (C.c_int, [_vp, C.c_int, C.c_int, C.c_int, _vp, _vp, _vp]),
    "b200md_shc_finish": (C.c_int, [_vp, C.c_double, C.c_int, C.c_double, _dp, _dp, _dp, _dp, _vp]),
    "b200md_dos_create": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_double, C.c_double, C.c_int, C.c_int, _ip,
                                    _ip, C.c_int, _vp, C.POINTER(_vp)]),
    "b200md_dos_destroy": (None, [_vp]),
    "b200md_dos_sample": (C.c_int, [_vp, C.c_int, C.c_int, C.c_int, _vp, _vp]),
    "b200md_dos_finish": (C.c_int, [_vp, _dp, _dp, _vp]),
    "b200md_sdc_create": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_double, C.c_int, _ip, _ip, C.POINTER(_vp)]),
    "b200md_sdc_destroy": (None, [_vp]),
    "b200md_sdc_sample": (C.c_int, [_vp, C.c_int, C.c_int, C.c_int, _vp, _vp]),
    "b200md_sdc_finish": (C.c_int, [_vp, _dp, _dp, _vp]),
    "b200md_msd_create": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_double, C.c_int, _ip, _ip, C.POINTER(_vp)]),
    "b200md_msd_destroy": (None, [_vp]),
    "b200md_msd_sample": (C.c_int, [_vp, C.c_int, C.c_int, C.c_int, _vp, _vp]),
    "b200md_msd_finish": (C.c_int, [_vp, _dp, _dp, _vp]),
    "b200md_rdf_create": (C.c_int, [C.c_double, C.c_int, C.c_int, _ip, _ip, C.c_int, C.POINTER(_vp)]),
    "b200md_rdf_destroy": (None, [_vp]),
    "b200md_rdf_sample": (C.c_int, [_vp, _dp, _ip, _vp, _vp, C.c_int, _vp]),
    "b200md_rdf_finish": (C.c_int, [_vp, C.c_int, _dp, _vp]),
    "b200md_unwrap_begin": (C.c_int, [C.c_int, _vp, _vp, _vp]),
    "b200md_unwrap_end": (C.c_int, [C.c_int, _vp, _vp, _vp, _vp]),
    "b200md_heat_bath_create":(C.c_int, [C.c_int, C.c_int, C.c_int, _ip, _ip, C.c_int, C.c_int, C.c_double,
                                          C.c_double, C.c_double, C.c_double, C.c_ulonglong, C.c_ulonglong,
                                          C.POINTER(_vp)]),
    "b200md_heat_bath_destroy": (None, [_vp]),
    "b200md_heat_bath_half": (C.c_int, [_vp, C.c_int, C.c_int, C.c_int, _vp, _vp, _vp]),
    "b200md_heat_bath_energy": (C.c_int, [_vp, _dp, _vp]),
    "b200md_heat_bath_state": (C.c_int, [_vp, _dp, _vp]),
    "b200md_group_compute_create": (C.c_int, [C.c_int, C.c_int, _ip, _ip, C.c_uint, C.POINTER(_vp)]),
    "b200md_group_compute_destroy": (None, [_vp]),
    "b200md_group_compute_columns": (C.c_int, [_vp]),
    "b200md_group_compute_sample": (C.c_int, [_vp, C.c_int, C.c_int, _vp, _vp, _vp, _vp, _vp, _vp]),
    "b200md_group_compute_take": (C.c_int, [_vp, C.c_int, _dp, _vp]),
    "b200md_langevin_create": (C.c_int, [C.c_int, C.c_ulonglong, C.POINTER(_vp)]),
    "b200md_langevin_destroy": (None, [_vp]),
    "b200md_langevin_apply": (C.c_int, [_vp, C.c_int, C.c_int, C.c_double, C.c_double, _vp, _vp, _vp]),
    "b200md_baoab_operator": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_double, _vp, _vp, _vp, _vp, _vp,
                                        C.c_int, _vp]),
    "b200md_berendsen_pressure": (C.c_int, [C.c_int, C.c_int, C.c_int, _dp, _dp, _ip, _dp, _ip, _dp, _vp,
                                            _vp, _vp]),
    "b200md_apply_pbc_strided": (C.c_int, [C.c_int, C.c_int, _dp, _ip, _vp, _vp]),
    "b200md_velocity_verlet_strided": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_double, _vp, _vp, _vp, _vp, _vp]),
    "b200md_find_thermo_strided": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_double, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "b200md_halo_pack": (C.c_int, [C.c_int, _vp, C.c_int, _vp, _dp, _vp, _vp]),
    "b200md_nep_invalidate": (C.c_int, [_vp, C.c_int, _vp]),
    "b200md_nep_set_owned": (C.c_int, [_vp, C.c_int]),
    "b200md_nep_set_accumulate": (C.c_int, [_vp, C.c_int]),
    "b200md_nep_set_active_region": (C.c_int, [_vp, _dp, _dp]),
    "b200md_minimizer_create": (C.c_int, [C.c_int, C.c_int, C.c_double, C.c_int, C.c_int, C.c_int,
                                          C.POINTER(_vp)]),
    "b200md_minimizer_destroy": (None, [_vp]),
    "b200md_minimizer_velocity": (_vp, [_vp]),
    "b200md_minimizer_set_record": (C.c_int, [_vp, _dp, _vp]),
    "b200md_minimizer_sd_begin": (C.c_int, [_vp, C.c_int, _vp, _vp, _vp, _vp, _vp, _vp, _vp, C.c_int, _dp, _vp]),
    "b200md_minimizer_sd_step": (C.c_int, [_vp, C.c_int, _vp, _vp, _vp, _vp, _vp, _vp, _vp, C.c_int, _dp, _vp]),
    "b200md_minimizer_fire_step": (C.c_int, [_vp, C.c_int, _dp, _vp, _vp, _vp, _vp, _dp, _vp]),
    "b200md_phonon_create": (C.c_int, [C.c_int, C.c_int, C.c_int, _dp, C.c_double, C.POINTER(_vp)]),
    "b200md_phonon_destroy": (None, [_vp]),
    "b200md_phonon_begin": (C.c_int, [_vp, C.c_int, _dp, _ip, C.c_double, _vp, _vp, _vp]),
    "b200md_phonon_step": (C.c_int, [_vp, C.c_int, _vp, _vp, _vp]),
    "b200md_phonon_dynamical": (C.c_int, [_vp, _vp]),
    "b200md_phonon_eig": (C.c_int, [_vp, _vp]),
    "b200md_phonon_read": (C.c_int, [_vp, C.c_int, _dp, _vp]),
    "b200md_jacobi_eig": (C.c_int, [C.c_int, C.c_int, C.c_int, _vp, _vp, _vp, _vp, _vp, _vp]),
    "b200md_tc_selftest": (C.c_int, [C.c_int, C.c_int, C.c_int, _vp, _vp, _vp, _vp]),
}

_LIB = None


class B200mdError(RuntimeError):
    pass


def load():
    """dlopen libb200md.so and bind every symbol include/b200md.h declares."""
    global _LIB
    if _LIB is None:
        if not LIB_PATH.exists():
            raise B200mdError(
                f"{LIB_PATH} is missing: build it with `python -m gpumd_b200.build` "
                "(libb200md has no CPU fallback)")
        L = C.CDLL(str(LIB_PATH))
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(L, name)  # AttributeError if the symbol is not exported
            fn.restype = res
            fn.argtypes = args
        _LIB = L
    return _LIB


def check(rc):
    if rc != 0:
        raise B200mdError(f"libb200md error {rc}: {load().b200md_last_error().decode()}")
