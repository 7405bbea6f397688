"""ctypes binding of libodcuda.so (C-ABI declared in include/odcuda.h).

The library is the product: there is no CPU fallback.  Importing this module without the
built shared object raises immediately with build instructions.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get('ODCUDA_LIB') or os.path.join(_HERE, 'libodcuda.so')   # ODCUDA_LIB: tuning builds only

OD_EULER, OD_RK2, OD_RK4 = 0, 1, 2
OD_T_LERP, OD_T_FIRST, OD_T_SECOND, OD_T_MISSING = 0, 1, 2, 3
OD_LON_0_360, OD_LON_PM180 = 0, 1
OD_OPT_TILE = 1
OD_OPT_SPEC = 2
OD_MATH_EXACT, OD_MATH_FAST, OD_MATH_SERIES = 0, 1, 2
OD_MIX_ENVIRONMENT, OD_MIX_LARGE1994, OD_MIX_SUNDBY1983, OD_MIX_CONSTANT = 0, 1, 2, 3
OD_MAX_LEVELS = 128
OD_MAX_GROUPS = 64
OD_MAX_CHAIN = 2
SCHEMES = {'euler': OD_EULER, 'runge-kutta': OD_RK2, 'runge-kutta4': OD_RK4}


class ProjDesc(C.Structure):
    _fields_ = [('kind', C.c_int32), ('has_lat_ts', C.c_int32), ('a', C.c_double), ('lat_0', C.c_double),
                ('lon_0', C.c_double), ('lat_ts', C.c_double), ('k_0', C.c_double), ('x_0', C.c_double), ('y_0', C.c_double),
                ('es', C.c_double), ('lat_1', C.c_double), ('lat_2', C.c_double)]


class GroupDesc(C.Structure):
    _fields_ = [('ncomp', C.c_int32), ('nx', C.c_int32), ('ny', C.c_int32), ('nz', C.c_int32),
                ('lon_mode', C.c_int32), ('n_slots', C.c_int32), ('wrap_x', C.c_int32), ('global_x', C.c_int32),
                ('x0', C.c_double), ('xspan', C.c_double), ('y0', C.c_double), ('yspan', C.c_double),
                ('xmin', C.c_double), ('xmax', C.c_double), ('ymin', C.c_double), ('ymax', C.c_double),
                ('fallback', C.c_float * 2), ('proj', ProjDesc), ('rotate_vectors', C.c_int32), ('pad_', C.c_int32)]


class TimeSample(C.Structure):
    _fields_ = [('slot_a', C.c_int32), ('slot_b', C.c_int32), ('mode', C.c_int32), ('pad_', C.c_int32),
                ('w', C.c_double)]


class HostIO(C.Structure):
    _fields_ = [('h_lon', C.c_void_p), ('h_lat', C.c_void_p), ('h_z', C.c_void_p),
                ('h_out_lon', C.c_void_p), ('h_out_lat', C.c_void_p), ('chunks', C.c_int32), ('pad_', C.c_int32),
                ('h_out_z', C.c_void_p)]


class AdvectArgs(C.Structure):
    _fields_ = [('scheme', C.c_int32), ('group_uv', C.c_int32),
                ('t_start', TimeSample), ('t_mid', TimeSample), ('t_end', TimeSample),
                ('dt', C.c_double), ('n', C.c_int64),
                ('d_lon', C.c_void_p), ('d_lat', C.c_void_p), ('d_z', C.c_void_p),
                ('d_factor', C.c_void_p), ('factor_f64', C.c_int32), ('pos_f32', C.c_int32),
                ('d_moving', C.c_void_p), ('d_k1_u', C.c_void_p), ('d_k1_v', C.c_void_p),
                ('truncate_below', C.c_double),
                ('d_env_u', C.c_void_p), ('d_env_v', C.c_void_p), ('z_f64', C.c_int32), ('pad3_', C.c_int32), ('d_noise_cur', C.c_void_p), ('noise_kinds', C.c_int32),
                ('fast', C.c_int32),
                ('n_chain', C.c_int32), ('chain_group', C.c_int32 * 2), ('pad4_', C.c_int32), ('chain_t', (TimeSample * 3) * 2)]


class StepArgs(C.Structure):
    _fields_ = [('cur', AdvectArgs),
                ('group_wind', C.c_int32), ('wdf_f64', C.c_int32), ('t_wind', TimeSample),
                ('d_wdf', C.c_void_p), ('wind_drift_depth', C.c_double),
                ('group_w', C.c_int32), ('w_at_surface', C.c_int32), ('t_w', TimeSample),
                ('d_z_inout', C.c_void_p),
                ('d_rand_x', C.c_void_p), ('d_rand_y', C.c_void_p), ('d_diffusivity', C.c_void_p),
                ('diffusivity_const', C.c_float), ('z_inout_f64', C.c_int32), ('d_noise_wind', C.c_void_p)]


class MixArgs(C.Structure):
    _fields_ = [('group_k', C.c_int32), ('ntimes', C.c_int32), ('t_k', TimeSample), ('n', C.c_int64),
                ('d_lon', C.c_void_p), ('d_lat', C.c_void_p), ('d_z_in', C.c_void_p), ('d_z_out', C.c_void_p),
                ('d_moving', C.c_void_p), ('d_terminal_velocity', C.c_void_p), ('d_ids', C.c_void_p),
                ('d_rand', C.c_void_p), ('d_sea_floor', C.c_void_p), ('dt_mix', C.c_double),
                ('sea_floor_const', C.c_double), ('seed', C.c_uint64), ('step_index', C.c_int32),
                ('z_in_f64', C.c_int32), ('tv_f64', C.c_int32), ('mix_at_surface', C.c_int32),
                ('pos_f32', C.c_int32), ('model', C.c_int32), ('nlev', C.c_int32), ('seafloor_action', C.c_int32),
                ('d_wind_speed', C.c_void_p), ('d_mld', C.c_void_p), ('mld_const', C.c_double),
                ('background', C.c_double), ('k_const', C.c_double), ('d_status', C.c_void_p), ('d_moving_out', C.c_void_p),
                ('seafloor_code', C.c_int32), ('iter0', C.c_int32), ('h_n_deactivated', C.POINTER(C.c_int64)),
                ('skip_surface_stick', C.c_int32), ('pad3_', C.c_int32)]


class LeewayArgs(C.Structure):
    _fields_ = [('group_wind', C.c_int32), ('group_cur', C.c_int32), ('t_wind', TimeSample), ('t_cur', TimeSample),
                ('n', C.c_int64), ('d_lon', C.c_void_p), ('d_lat', C.c_void_p), ('d_dw_slope', C.c_void_p),
                ('d_dw_offset', C.c_void_p), ('d_dw_eps', C.c_void_p), ('d_cw_slope', C.c_void_p),
                ('d_cw_offset', C.c_void_p), ('d_cw_eps', C.c_void_p), ('d_orientation', C.c_void_p),
                ('d_capsized', C.c_void_p), ('d_jibe_probability', C.c_void_p), ('d_moving', C.c_void_p),
                ('d_status', C.c_void_p), ('d_ids', C.c_void_p), ('d_rand', C.c_void_p), ('dt', C.c_double),
                ('seed', C.c_uint64), ('capsize_fraction', C.c_float), ('jp_f64', C.c_int32), ('pos_f32', C.c_int32),
                ('step_index', C.c_int32), ('missing_code', C.c_int32), ('pad_', C.c_int32),
                ('capsize_on', C.c_int32), ('capsize_from', C.c_int32), ('wind_threshold', C.c_float),
                ('wind_sigma', C.c_float), ('d_rand_capsize', C.c_void_p),
                ('d_noise_cur', C.c_void_p), ('d_noise_wind', C.c_void_p), ('noise_kinds', C.c_int32), ('pad2_', C.c_int32)]


class StokesArgs(C.Structure):
    _fields_ = [('n', C.c_int64), ('d_lon', C.c_void_p), ('d_lat', C.c_void_p), ('d_z', C.c_void_p),
                ('d_us', C.c_void_p), ('d_vs', C.c_void_p), ('d_hs', C.c_void_p), ('d_xwind', C.c_void_p),
                ('d_ywind', C.c_void_p), ('d_moving', C.c_void_p), ('dt', C.c_double), ('z_f64', C.c_int32),
                ('hs_mode', C.c_int32), ('profile', C.c_int32), ('pad_', C.c_int32), ('factor', C.c_double), ('d_factor', C.c_void_p),
                ('factor_f64', C.c_int32), ('pad2_', C.c_int32), ('d_swell_dir', C.c_void_p), ('d_swell_period', C.c_void_p),
                ('d_swell_hs', C.c_void_p), ('d_windsea_dir', C.c_void_p), ('d_windsea_period', C.c_void_p), ('d_windsea_hs', C.c_void_p)]


class AnalyticDesc(C.Structure):
    _fields_ = [('kind', C.c_int32), ('lon_mode', C.c_int32), ('proj', ProjDesc),
                ('xmin', C.c_double), ('xmax', C.c_double), ('ymin', C.c_double), ('ymax', C.c_double),
                ('par', C.c_double * 4), ('rot_delta', C.c_double), ('fallback', C.c_float * 2)]


class AnalyticAdvectArgs(C.Structure):
    _fields_ = [('scheme', C.c_int32), ('math', C.c_int32), ('factor_f64', C.c_int32), ('pos_f32', C.c_int32),
                ('t_start', C.c_double), ('t_mid', C.c_double), ('t_end', C.c_double), ('dt', C.c_double),
                ('n', C.c_int64), ('d_lon', C.c_void_p), ('d_lat', C.c_void_p), ('d_factor', C.c_void_p),
                ('d_moving', C.c_void_p), ('d_k1_u', C.c_void_p), ('d_k1_v', C.c_void_p),
                ('d_env_u', C.c_void_p), ('d_env_v', C.c_void_p)]


class HistoryArgs(C.Structure):
    _fields_ = [('n', C.c_int64), ('n_total', C.c_int64), ('col', C.c_int32), ('ncols', C.c_int32),
                ('z_f64', C.c_int32), ('pad_', C.c_int32), ('d_ids', C.c_void_p), ('d_lon', C.c_void_p), ('d_lat', C.c_void_p),
                ('d_z', C.c_void_p), ('d_status', C.c_void_p), ('d_buf_lon', C.c_void_p), ('d_buf_lat', C.c_void_p),
                ('d_buf_z', C.c_void_p), ('d_buf_status', C.c_void_p)]


class BuoyancyArgs(C.Structure):
    _fields_ = [('n', C.c_int64), ('d_z_in', C.c_void_p), ('d_z_out', C.c_void_p), ('d_terminal_velocity', C.c_void_p),
                ('d_sea_floor', C.c_void_p), ('d_status', C.c_void_p), ('d_moving', C.c_void_p), ('dt', C.c_double),
                ('sea_surface_height', C.c_float), ('z_f64', C.c_int32), ('tv_f64', C.c_int32), ('seafloor_code', C.c_int32),
                ('h_n_deactivated', C.POINTER(C.c_int64))]


class BookkeepArgs(C.Structure):
    _fields_ = [('n', C.c_int64), ('d_lon', C.c_void_p), ('d_lat', C.c_void_p), ('d_z', C.c_void_p), ('d_age', C.c_void_p),
                ('d_status', C.c_void_p), ('d_moving', C.c_void_p), ('d_ids', C.c_void_p), ('dt_age', C.c_double),
                ('max_age', C.c_double), ('west', C.c_double), ('east', C.c_double), ('south', C.c_double), ('north', C.c_double),
                ('outside_code', C.c_int32), ('retired_code', C.c_int32), ('z_f64', C.c_int32), ('age_f64', C.c_int32),
                ('pos_f32', C.c_int32), ('only_deactivated', C.c_int32), ('n_total', C.c_int64), ('col', C.c_int32), ('ncols', C.c_int32),
                ('d_buf_lon', C.c_void_p), ('d_buf_lat', C.c_void_p), ('d_buf_z', C.c_void_p), ('d_buf_status', C.c_void_p),
                ('h_counts', C.POINTER(C.c_int64))]


class CoastArgs(C.Structure):
    _fields_ = [('n', C.c_int64), ('d_mask', C.c_void_p), ('d_lon', C.c_void_p), ('d_lat', C.c_void_p), ('d_z', C.c_void_p),
                ('d_age', C.c_void_p), ('d_status', C.c_void_p), ('d_moving', C.c_void_p), ('d_ids', C.c_void_p),
                ('d_prev_lon', C.c_void_p), ('d_prev_lat', C.c_void_p), ('n_total', C.c_int64), ('id_base', C.c_int32),
                ('action', C.c_int32), ('ssh', C.c_float), ('stranded_code', C.c_int32), ('seeded_code', C.c_int32), ('missing_code', C.c_int32),
                ('check_seeded', C.c_int32), ('z_f64', C.c_int32), ('age_f64', C.c_int32), ('h_counts', C.POINTER(C.c_int64))]


OD_INTERP_POS_F32, OD_INTERP_NO_FALLBACK, OD_INTERP_Z_F64, OD_INTERP_NO_ROTATE, OD_INTERP_OUT_F64, OD_INTERP_NEAREST = 1, 2, 4, 8, 16, 32
OD_PACK_MAX_COLS, OD_PACK_MAX_WORLD = 16, 64


class PackArgs(C.Structure):
    _fields_ = [('n', C.c_int64), ('d_lon', C.c_void_p), ('h_bounds', C.POINTER(C.c_double)), ('world', C.c_int32), ('ncols', C.c_int32),
                ('d_cols', C.c_void_p * OD_PACK_MAX_COLS), ('col_bytes', C.c_int32 * OD_PACK_MAX_COLS), ('rec_bytes', C.c_int32),
                ('pad_', C.c_int32), ('d_records', C.c_void_p), ('d_perm', C.c_void_p), ('h_counts', C.POINTER(C.c_int64))]


OD_PROJ_STERE_SPHERE = 1
OD_PROJ_MERC, OD_PROJ_LCC, OD_PROJ_STERE_ELLPS, OD_PROJ_OB_TRAN = 2, 3, 4, 5
OD_ANALYTIC_DOUBLE_GYRE = 1

# every symbol include/odcuda.h declares: (restype, argtypes)
_P = C.c_void_p
SYMBOLS = {
    'od_abi_version': (C.c_int, []),
    'od_create': (C.c_int, [C.c_int, C.POINTER(_P)]),
    'od_destroy': (None, [_P]),
    'od_last_error': (C.c_char_p, [_P]),
    'od_set_stream': (C.c_int, [_P, _P]),
    'od_sync': (C.c_int, [_P]),
    'od_set_option': (C.c_int, [_P, C.c_int, C.c_int]),
    'od_device_sm_count': (C.c_int, [_P]),
    'od_group_define': (C.c_int, [_P, C.c_int, C.POINTER(GroupDesc), C.POINTER(C.c_double)]),
    'od_group_free': (C.c_int, [_P, C.c_int]),
    'od_group_upload': (C.c_int, [_P, C.c_int, C.c_int, C.c_int, _P, C.c_int]),
    'od_group_fill_nan': (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int64)]),
    'od_group_slot_ptr': (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.POINTER(_P)]),
    'od_group_touch': (C.c_int, [_P, C.c_int, C.c_int]),
    'od_group_set_fallback': (C.c_int, [_P, C.c_int, C.c_float, C.c_float]),
    'od_group_set_window': (C.c_int, [_P, C.c_int, C.POINTER(GroupDesc)]),
    'od_bbox': (C.c_int, [_P, C.c_int64, _P, _P, C.POINTER(C.c_double)]),
    'od_interp': (C.c_int, [_P, C.c_int, C.POINTER(TimeSample), C.c_int64, _P, _P, _P, C.c_int, _P, _P]),
    'od_geod_fwd': (C.c_int, [_P, C.c_int64, _P, _P, _P, _P]),
    'od_update_positions': (C.c_int, [_P, C.c_int64, _P, _P, _P, _P, C.c_int, _P, C.c_double]),
    'od_advect_current': (C.c_int, [_P, C.POINTER(AdvectArgs)]),
    'od_advect_current_host': (C.c_int, [_P, C.POINTER(AdvectArgs), C.POINTER(HostIO)]),
    'od_step_oceandrift_host': (C.c_int, [_P, C.POINTER(StepArgs), C.POINTER(HostIO)]),
    'od_step_oceandrift': (C.c_int, [_P, C.POINTER(StepArgs)]),
    'od_leeway_step': (C.c_int, [_P, C.POINTER(LeewayArgs)]),
    'od_analytic_interp': (C.c_int, [_P, C.POINTER(AnalyticDesc), C.c_double, C.c_int64, _P, _P, C.c_int, _P, _P]),
    'od_history_scatter': (C.c_int, [_P, C.POINTER(HistoryArgs)]),
    'od_analytic_advect': (C.c_int, [_P, C.POINTER(AnalyticDesc), C.POINTER(AnalyticAdvectArgs)]),
    'od_minmax_f32': (C.c_int, [_P, C.c_int64, _P, _P, C.POINTER(C.c_float), C.POINTER(C.c_float)]),
    'od_stokes_drift': (C.c_int, [_P, C.POINTER(StokesArgs)]),
    'od_vertical_mixing': (C.c_int, [_P, C.POINTER(MixArgs)]),
    'od_vertical_buoyancy': (C.c_int, [_P, C.POINTER(BuoyancyArgs)]),
    'od_bookkeeping': (C.c_int, [_P, C.POINTER(BookkeepArgs)]),
    'od_coastline': (C.c_int, [_P, C.POINTER(CoastArgs)]),
    'od_store_previous': (C.c_int, [_P, C.c_int64, _P, _P, _P, C.c_int32, C.c_int64, _P, _P]),
    'od_store_previous_env': (C.c_int, [_P, C.c_int64, _P, _P, _P, C.c_int32, C.c_double, C.c_int32, C.c_int64, _P, _P]),
    'od_vertical_advection_corrected': (C.c_int, [_P, C.c_int64, _P, C.c_int32, _P, _P, _P, _P, C.c_float, _P, C.c_int32,
                                                  C.c_double]),
    'od_pack_by_owner': (C.c_int, [_P, C.POINTER(PackArgs)]),
    'od_unpack_records': (C.c_int, [_P, C.c_int64, _P, C.c_int32, C.POINTER(_P), C.POINTER(C.c_int32), C.c_int32]),
    'od_sort_by_cell': (C.c_int, [_P, C.c_int, C.c_int64, _P, _P, _P, _P]),
    'od_partition_active': (C.c_int, [_P, C.c_int64, _P, _P, C.POINTER(C.c_int64)]),
    'od_permute': (C.c_int, [_P, C.c_int64, _P, _P, _P, C.c_int]),
    'od_unpermute': (C.c_int, [_P, C.c_int64, _P, _P, _P, C.c_int]),
    'od_launch_count': (C.c_int64, [_P]),
}

_lib = None


def load():
    """Load libodcuda.so (once).  Fails loudly when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            'opendrift_b200: %s is missing. This package has no CPU fallback; build the CUDA '
            'extension first:  python -c "import __graft_entry__ as g; g.build()"  '
            '(or python -m opendrift_b200.build).' % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    for name, (restype, argtypes) in SYMBOLS.items():
        fn = getattr(lib, name)          # AttributeError if the library lacks a declared symbol
        fn.restype = restype
        fn.argtypes = argtypes
    if lib.od_abi_version() != 1:
        raise RuntimeError('libodcuda.so ABI version mismatch')
    _lib = lib
    return lib
