"""ctypes binding of the C-ABI in include/dbw_render.h (the drop-in boundary).  There is NO CPU fallback: if the
shared library is missing or a call fails, this raises."""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# DBW_RENDER_LIB: explicit path of another build of the same library (kernel experiments); never a fallback
LIB_PATH = os.environ.get('DBW_RENDER_LIB') or os.path.join(_HERE, 'libdbw_render.so')

ABI_VERSION = 8


class DbwRenderSettings(ctypes.Structure):
    _fields_ = [
        ('n_views', ctypes.c_int32), ('height', ctypes.c_int32), ('width', ctypes.c_int32),
        ('faces_per_pixel', ctypes.c_int32), ('n_verts', ctypes.c_int32), ('n_faces', ctypes.c_int32),
        ('n_maps', ctypes.c_int32), ('alpha_view_stride', ctypes.c_int32),
        ('fx', ctypes.c_float), ('fy', ctypes.c_float), ('px', ctypes.c_float), ('py', ctypes.c_float),
        ('sigma', ctypes.c_float), ('blur_radius', ctypes.c_float), ('z_clip', ctypes.c_float),
        ('proj_eps', ctypes.c_float), ('background', ctypes.c_float * 3),
        ('clip_inside', ctypes.c_int32), ('perspective_correct', ctypes.c_int32),
        ('clip_barycentric', ctypes.c_int32), ('detach_bary', ctypes.c_int32), ('verts_are_ndc', ctypes.c_int32),
        ('n_map_floats', ctypes.c_int32), ('maps_are_texels4', ctypes.c_int32), ('save_fragment_state', ctypes.c_int32),
        ('alpha_group', ctypes.c_int32), ('n_static_faces', ctypes.c_int32), ('view_rows', ctypes.c_void_p),
    ]


class DbwSceneGeometry(ctypes.Structure):
    _fields_ = [('n_blocks', ctypes.c_int32), ('verts_per_block', ctypes.c_int32), ('n_ground_verts', ctypes.c_int32),
                ('reserved', ctypes.c_int32)] \
             + [(n, ctypes.c_void_p) for n in ('sq_eta', 'sq_omega', 'sq_eps', 'S', 'R_6d', 'T', 'ground_verts',
                                               'R_6d_ground', 'T_ground')] \
             + [('ratio_block_scene', ctypes.c_float), ('scale_min', ctypes.c_float), ('S_world', ctypes.c_float),
                ('R_world', ctypes.c_float * 9), ('T_world', ctypes.c_float * 3)]


class DbwLossEpilogue(ctypes.Structure):
    _fields_ = [('env_rgba', ctypes.c_void_p), ('target', ctypes.c_void_p), ('g_env', ctypes.c_void_p), ('rec', ctypes.c_void_p),
                ('loss_partials', ctypes.c_void_p), ('n_partials', ctypes.c_int32), ('inv_count', ctypes.c_float),
                ('env_alpha_unread', ctypes.c_int32)]


class DbwTexJob(ctypes.Structure):
    _fields_ = [('textures', ctypes.c_void_p), ('atlas', ctypes.c_void_p), ('g_textures', ctypes.c_void_p),
                ('n_maps', ctypes.c_int32), ('txt_size', ctypes.c_int32), ('p_left', ctypes.c_int32), ('p_right', ctypes.c_int32),
                ('decimate', ctypes.c_int32), ('stage', ctypes.c_int32)]


class DbwEvalGrid(ctypes.Structure):
    _fields_ = [('origin', ctypes.c_double * 3), ('cell', ctypes.c_double), ('dims', ctypes.c_int64 * 3),
                ('block', ctypes.c_int32), ('reserved', ctypes.c_int32)]


class DbwLpipsNet(ctypes.Structure):
    _fields_ = [('conv_w', ctypes.c_void_p * 13), ('conv_b', ctypes.c_void_p * 13), ('lin_w', ctypes.c_void_p * 5),
                ('shift', ctypes.c_void_p), ('scale', ctypes.c_void_p), ('prepared', ctypes.c_void_p)]


class DbwLpipsTargetCache(ctypes.Structure):
    _fields_ = [('arena', ctypes.c_void_p), ('N', ctypes.c_int64), ('H', ctypes.c_int32), ('W', ctypes.c_int32),
                ('normalize', ctypes.c_int32)]


class DbwVggLossOptions(ctypes.Structure):
    _fields_ = [('levels', ctypes.c_int32), ('normalize_input', ctypes.c_int32), ('normalize_features', ctypes.c_int32),
                ('sum_channels', ctypes.c_int32)]


class DbwMapDesc(ctypes.Structure):
    _fields_ = [('offset', ctypes.c_int32), ('height', ctypes.c_int32), ('width', ctypes.c_int32),
                ('reserved', ctypes.c_int32)]


EXPORTS = ['dbw_abi_version', 'dbw_debug_generic_kernel_only', 'dbw_debug_keep_unread_outputs', 'dbw_sizeof_settings', 'dbw_last_error', 'dbw_workspace_bytes', 'dbw_render_forward', 'dbw_render_backward',
           'dbw_render_forward_loss', 'dbw_render_forward_loss_grad', 'dbw_render_backward_deferred',
           'dbw_composite_mse', 'dbw_composite_mse_backward', 'dbw_render_forward_host', 'dbw_host_arena_release', 'dbw_launch_count',
           'dbw_timing_enable', 'dbw_timing_read', 'dbw_timing_reset', 'dbw_scene_geometry_forward', 'dbw_scene_geometry_backward',
           'dbw_opacity_forward', 'dbw_opacity_backward', 'dbw_texture_prep_forward_multi', 'dbw_texture_prep_backward_multi',
           'dbw_comm_create', 'dbw_comm_buffer', 'dbw_comm_ipc_handle', 'dbw_comm_connect', 'dbw_comm_all_reduce', 'dbw_comm_error', 'dbw_comm_destroy',
           'dbw_eval_sample_setup', 'dbw_eval_sample_count', 'dbw_eval_sample_write', 'dbw_eval_cell_keys',
           'dbw_eval_cell_ranges', 'dbw_eval_downsample_workspace_bytes', 'dbw_eval_radius_downsample', 'dbw_eval_nn_distance',
           'dbw_knn_forward', 'dbw_knn_backward',
           'dbw_lpips_workspace_bytes', 'dbw_lpips_prepare_weights', 'dbw_lpips_forward', 'dbw_lpips_backward',
           'dbw_lpips_conv3x3', 'dbw_lpips_conv_first', 'dbw_lpips_dgrad_last', 'dbw_lpips_maxpool', 'dbw_lpips_maxpool_backward',
           'dbw_lpips_head_forward', 'dbw_lpips_head_backward',
           'dbw_lpips_cache_bytes', 'dbw_lpips_cache_targets', 'dbw_lpips_forward_cached', 'dbw_lpips_backward_cached',
           'dbw_vgg_loss_workspace_bytes', 'dbw_vgg_loss_forward', 'dbw_vgg_loss_backward']

_lib = None


class DbwError(RuntimeError):
    pass


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise DbwError(f'{LIB_PATH} not found: build it with `python -c "import __graft_entry__ as g; g.build()"` '
                           f'or `make -C differentiable-blocksworld_b200/csrc` (there is no CPU fallback)')
        L = ctypes.CDLL(LIB_PATH)
        vp, sz = ctypes.c_void_p, ctypes.c_size_t
        L.dbw_abi_version.restype = ctypes.c_int
        L.dbw_sizeof_settings.restype = ctypes.c_size_t
        L.dbw_last_error.restype = ctypes.c_char_p
        L.dbw_launch_count.restype = ctypes.c_uint64
        L.dbw_workspace_bytes.argtypes = [ctypes.POINTER(DbwRenderSettings), ctypes.POINTER(sz), ctypes.POINTER(sz)]
        L.dbw_render_forward.argtypes = [ctypes.POINTER(DbwRenderSettings)] + [vp] * 12 + [sz, vp, vp, vp]
        L.dbw_render_backward.argtypes = [ctypes.POINTER(DbwRenderSettings)] + [vp] * 10 + [sz] + [vp] * 8 + [sz, vp]
        L.dbw_render_forward_loss.argtypes = [ctypes.POINTER(DbwRenderSettings)] + [vp] * 12 + [sz, ctypes.POINTER(DbwLossEpilogue), vp]
        L.dbw_render_forward_loss_grad.argtypes = [ctypes.POINTER(DbwRenderSettings)] + [vp] * 10 + [sz, ctypes.POINTER(DbwLossEpilogue),
                                                                                               ctypes.c_int32, vp, sz, vp]
        L.dbw_render_backward_deferred.argtypes = [ctypes.POINTER(DbwRenderSettings)] + [vp] * 5 + [sz] + [vp] * 7 + [sz, vp]
        L.dbw_composite_mse.argtypes = [ctypes.c_int32] * 3 + [vp] * 3 + [ctypes.c_float] + [vp] * 5
        L.dbw_composite_mse_backward.argtypes = [ctypes.c_int32] * 3 + [vp] * 3 + [ctypes.c_float] + [vp] * 5
        L.dbw_render_forward_host.argtypes = [ctypes.POINTER(DbwRenderSettings)] + [vp] * 5 + [sz] + [vp] * 6
        L.dbw_host_arena_release.restype = None
        L.dbw_scene_geometry_forward.argtypes = [ctypes.POINTER(DbwSceneGeometry), vp, ctypes.c_int32, vp, vp]
        L.dbw_scene_geometry_backward.argtypes = [ctypes.POINTER(DbwSceneGeometry)] + [vp] * 9
        L.dbw_opacity_forward.argtypes = [vp, vp, ctypes.c_float, ctypes.c_float, vp, ctypes.c_int32, ctypes.c_int32, vp, vp, vp, vp]
        L.dbw_opacity_backward.argtypes = [vp, vp, ctypes.c_float, ctypes.c_float, vp, vp, ctypes.c_int32, vp, vp]
        L.dbw_comm_create.argtypes = [ctypes.c_int32, ctypes.c_int32, sz, ctypes.POINTER(vp)]
        L.dbw_comm_buffer.argtypes = [vp, ctypes.POINTER(vp)]
        L.dbw_comm_ipc_handle.argtypes = [vp, vp]
        L.dbw_comm_connect.argtypes = [vp, vp]
        L.dbw_comm_all_reduce.argtypes = [vp, vp, sz, vp]
        L.dbw_comm_error.argtypes = [vp, ctypes.POINTER(ctypes.c_int32)]
        L.dbw_comm_destroy.argtypes = [vp]
        L.dbw_debug_generic_kernel_only.restype = None
        L.dbw_debug_generic_kernel_only.argtypes = [ctypes.c_int]
        L.dbw_debug_keep_unread_outputs.restype = None
        L.dbw_debug_keep_unread_outputs.argtypes = [ctypes.c_int]
        L.dbw_texture_prep_forward_multi.argtypes = [ctypes.POINTER(DbwTexJob), ctypes.c_int32, vp]
        L.dbw_texture_prep_backward_multi.argtypes = [ctypes.POINTER(DbwTexJob), ctypes.c_int32, vp]
        L.dbw_timing_enable.restype = None
        L.dbw_timing_reset.restype = None
        L.dbw_timing_read.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_int)]
        i64, gp = ctypes.c_int64, ctypes.POINTER(DbwEvalGrid)
        L.dbw_eval_sample_setup.argtypes = [vp, vp, i64, vp, vp, vp]
        L.dbw_eval_sample_count.argtypes = [vp, vp, i64, i64, vp, vp]
        L.dbw_eval_sample_write.argtypes = [vp, vp, i64, i64, vp, vp, vp, vp]
        L.dbw_eval_cell_keys.argtypes = [vp, i64, gp, vp, vp]
        L.dbw_eval_cell_ranges.argtypes = [vp, vp, i64, gp, vp, vp, vp]
        L.dbw_eval_downsample_workspace_bytes.argtypes = [i64, ctypes.POINTER(sz)]
        L.dbw_eval_radius_downsample.argtypes = [vp] * 5 + [i64, ctypes.c_double, ctypes.c_int32, vp,
                                                            ctypes.POINTER(ctypes.c_int32), vp, sz, vp]
        L.dbw_eval_nn_distance.argtypes = [vp, i64, vp, vp, gp, ctypes.c_double, vp, vp]
        L.dbw_knn_forward.argtypes = [vp] * 4 + [i64] * 3 + [ctypes.c_int32] + [vp] * 3
        L.dbw_knn_backward.argtypes = [vp] * 6 + [i64] * 3 + [ctypes.c_int32] + [vp] * 3
        i32, np_ = ctypes.c_int32, ctypes.POINTER(DbwLpipsNet)
        L.dbw_lpips_workspace_bytes.argtypes = [i64, i32, i32, i32, ctypes.POINTER(sz), ctypes.POINTER(sz)]
        L.dbw_lpips_prepare_weights.argtypes = [np_, vp]
        L.dbw_lpips_forward.argtypes = [np_, vp, vp, i64, i32, i32, i32, i32, i32, vp, vp, vp, sz, vp]
        L.dbw_lpips_backward.argtypes = [np_, vp, i64, i32, i32, i32, i32, vp, vp, sz, vp]
        L.dbw_lpips_conv3x3.argtypes = [vp] * 5 + [i64] + [i32] * 5 + [vp]
        L.dbw_lpips_conv_first.argtypes = [vp] * 5 + [i32, vp, i64, i32, i32, vp]
        L.dbw_lpips_dgrad_last.argtypes = [vp] * 3 + [i32, vp, i64, i32, i32, vp]
        L.dbw_lpips_maxpool.argtypes = [vp, vp, i64, i32, i32, i32, vp]
        L.dbw_lpips_maxpool_backward.argtypes = [vp, vp, vp, i64, i32, i32, i32, vp]
        L.dbw_lpips_head_forward.argtypes = [vp] * 3 + [i64] + [i32] * 5 + [vp, vp, vp]
        L.dbw_lpips_head_backward.argtypes = [vp] * 3 + [i64] + [i32] * 5 + [vp, vp, i32, vp, vp]
        cp = ctypes.POINTER(DbwLpipsTargetCache)
        L.dbw_lpips_cache_bytes.argtypes = [i32, i32, ctypes.POINTER(sz)]
        L.dbw_lpips_cache_targets.argtypes = [np_, vp, cp, i64, vp, sz, vp]
        L.dbw_lpips_forward_cached.argtypes = [np_, cp, vp, vp, i64, i32, i32, i32, i32, i32, vp, vp, vp, vp, vp, sz, vp]
        L.dbw_lpips_backward_cached.argtypes = [np_, cp, vp, vp, i64, i32, i32, i32, i32, vp, vp, sz, vp]
        op = ctypes.POINTER(DbwVggLossOptions)
        L.dbw_vgg_loss_workspace_bytes.argtypes = [i64, i32, i32, op, i32, ctypes.POINTER(sz)]
        L.dbw_vgg_loss_forward.argtypes = [np_, op, vp, vp, i64, i32, i32, i32, vp, vp, sz, vp]
        L.dbw_vgg_loss_backward.argtypes = [np_, op, vp, i64, i32, i32, vp, vp, sz, vp]
        if L.dbw_sizeof_settings() != ctypes.sizeof(DbwRenderSettings):
            raise DbwError('DbwRenderSettings layout mismatch between the library and its ctypes mirror')
        if L.dbw_abi_version() != ABI_VERSION:
            raise DbwError(f'ABI mismatch: library {L.dbw_abi_version()} != binding {ABI_VERSION}')
        _lib = L
    return _lib


def check(rc, what):
    if rc != 0:
        raise DbwError(f'{what} failed: {lib().dbw_last_error().decode()}')


def launch_count():
    return int(lib().dbw_launch_count())


def kernel_time_ms(kind, K=0):
    """(total ms, launches) of the raster kernel `kind` (0 forward, 1 backward) recorded since the last reset."""
    tot, n = ctypes.c_double(0), ctypes.c_int(0)
    check(lib().dbw_timing_read(kind, K, ctypes.byref(tot), ctypes.byref(n)), 'dbw_timing_read')
    return tot.value, n.value
