"""ctypes binding of csrc/libgast_b200.so (C ABI: include/gast_b200.h).

There is no fallback: if the shared library is missing or fails to load, importing the
engine raises with the build command.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get('GAST_B200_LIB') or os.path.join(os.path.dirname(_HERE), 'csrc', 'libgast_b200.so')
# (GAST_B200_LIB: alternative build of the same library, used only for A/B experiments)

GAST_MAX_STAGES = 8
KIND_MODEL, KIND_BLOCK, KIND_LOCAL, KIND_MGLOBAL, KIND_SEMCH, KIND_GLOBAL_HEAD = range(6)

# every symbol include/gast_b200.h declares
SYMBOLS = ['gast_create', 'gast_destroy', 'gast_bind', 'gast_prepare', 'gast_out_frames',
           'gast_receptive_field', 'gast_workspace_bytes', 'gast_forward', 'gast_forward_mpjpe',
           'gast_last_launch_count', 'gast_last_tc_launch_count', 'gast_set_timing',
           'gast_get_timings', 'gast_set_gemm_core', 'gast_set_precision', 'gast_set_train_precision',
           'gast_set_activation_dtype',
           'gast_last_wgrad_tc_launch_count', 'gast_debug_gemm', 'gast_debug_wgrad', 'gast_debug_set_gemm_audit',
           'gast_debug_gemm_audit_skips', 'gast_debug_set_kernel_audit', 'gast_debug_kernel_audit_skips',
           'gast_bind_grads',
           'gast_train_workspace_bytes', 'gast_forward_train', 'gast_backward', 'gast_backward_input',
           'gast_eval_backward_workspace_bytes', 'gast_eval_backward', 'gast_chunked_workspace_bytes',
           'gast_forward_chunked', 'gast_eval_backward_chunked', 'gast_set_dropout_state', 'gast_tta_prepare', 'gast_tta_merge',
           'gast_stream_state_bytes', 'gast_stream_workspace_bytes', 'gast_stream_push',
           'gast_stream_latency', 'gast_stream_push_ex', 'gast_stream_chunk_workspace_bytes', 'gast_stream_push_chunk',
           'gast_stream_peek', 'gast_stream_subset_workspace_bytes', 'gast_stream_push_subset', 'gast_stream_peek_subset',
           'gast_stream_device_workspace_bytes', 'gast_stream_push_device', 'gast_stream_peek_device',
           'gast_stream_snapshot_floats', 'gast_stream_move_workspace_bytes', 'gast_stream_export',
           'gast_stream_import', 'gast_chunk_gather', 'gast_keypoints_convert', 'gast_h36m_coco_format', 'gast_revise_kpts',
           'gast_revise_skes_workspace_bytes', 'gast_revise_skes', 'gast_revise_skes_real_time_workspace_bytes',
           'gast_revise_skes_real_time', 'gast_normalize_screen', 'gast_camera_to_world', 'gast_world_to_camera',
           'gast_project_to_2d', 'gast_project_to_2d_backward', 'gast_normalize_screen_segments',
           'gast_mpjpe_workspace_bytes', 'gast_mpjpe', 'gast_p_mpjpe', 'gast_pose_metrics_workspace_bytes',
           'gast_pose_metrics', 'gast_render_geometry', 'gast_render_frames', 'gast_downsample_frames',
           'gast_person_crops', 'gast_heatmap_decode', 'gast_letterbox', 'gast_person_detections',
           'gast_sort_state_bytes', 'gast_sort_init', 'gast_sort_update', 'gast_track_records', 'gast_record_inverse',
           'gast_live_slots', 'gast_live_inputs', 'gast_live_place',
           'gast_adam_chunk', 'gast_adam_step', 'gast_chunk_gather_indexed',
           'gast_adam_step_table', 'gast_adam_step_indexed', 'gast_epoch_loss_accumulate',
           'gast_last_error', 'gast_version']


class GastCfg(C.Structure):
    _fields_ = [
        ('kind', C.c_int32), ('num_joints', C.c_int32), ('in_features', C.c_int32),
        ('channels', C.c_int32), ('channels_out', C.c_int32), ('num_stages', C.c_int32),
        ('filter_widths', C.c_int32 * GAST_MAX_STAGES),
        ('causal', C.c_int32), ('dense', C.c_int32), ('strided', C.c_int32),
        ('heads', C.c_int32), ('semch_shared_e', C.c_int32), ('semch_bias', C.c_int32),
        ('sym_nnz', C.c_int32), ('con_nnz', C.c_int32),
        ('sym_rows', C.POINTER(C.c_int32)), ('sym_cols', C.POINTER(C.c_int32)),
        ('con_rows', C.POINTER(C.c_int32)), ('con_cols', C.POINTER(C.c_int32)),
        ('device', C.c_int32),
    ]


class GemmAuditSeg(C.Structure):
    """gast_gemm_audit_seg: one K-segment of a GEMM launch's A operand"""
    _fields_ = [('base', C.c_void_p), ('tap_stride', C.c_int64), ('ld', C.c_int32), ('K', C.c_int32),
                ('Kc', C.c_int32), ('T_out', C.c_int32), ('T_in', C.c_int32), ('t_mul', C.c_int32),
                ('t_off', C.c_int32)]


class GemmAudit(C.Structure):
    """gast_gemm_audit: what one GEMM launch receives (gast_debug_set_gemm_audit)"""
    _fields_ = [('index', C.c_int64), ('epi', C.c_int32), ('core', C.c_int32), ('tc_form', C.c_int32),
                ('tma_mask', C.c_int32), ('nseg', C.c_int32), ('seg', GemmAuditSeg * 3), ('W', C.c_void_p),
                ('ldw', C.c_int32), ('N', C.c_int32), ('F', C.c_int32), ('J', C.c_int32), ('fpt', C.c_int32),
                ('ld_out', C.c_int32), ('out', C.c_void_p), ('bias', C.c_void_p), ('relu', C.c_int32),
                ('res_ld', C.c_int32), ('res', C.c_void_p), ('res_T_out', C.c_int32), ('res_T_in', C.c_int32),
                ('res_t_mul', C.c_int32), ('res_t_off', C.c_int32), ('coef', C.c_void_p * 2), ('shift', C.c_void_p),
                ('C', C.c_int32), ('tiles_per_mask', C.c_int32), ('nbr_row_ptr', (C.c_uint8 * 36) * 2),
                ('nbr_col', (C.c_uint8 * 164) * 2), ('ab', C.c_void_p), ('ck', C.c_void_p), ('bg', C.c_void_p),
                ('heads', C.c_int32), ('Cg', C.c_int32)]


GemmAuditFn = C.CFUNCTYPE(C.c_int32, C.c_int32, C.POINTER(GemmAudit), C.c_void_p)


class KernelAudit(C.Structure):
    """gast_kernel_audit: what one expand, row-dot, attention-mix or shrink launch receives
    (gast_debug_set_kernel_audit)"""
    _fields_ = [('index', C.c_int64), ('gemm_index', C.c_int64), ('kind', C.c_int32), ('variant', C.c_int32),
                ('fpb', C.c_int32), ('block', C.c_int32), ('in_type', C.c_int32), ('out_type', C.c_int32),
                ('x', C.c_void_p), ('We', C.c_void_p), ('be', C.c_void_p), ('U', C.c_void_p), ('cab', C.c_void_p),
                ('ab', C.c_void_p), ('Ck', C.c_void_p), ('Ws', C.c_void_p), ('target', C.c_void_p),
                ('loss', C.c_void_p), ('out', C.c_void_p), ('rows', C.c_int64), ('K', C.c_int32), ('ld', C.c_int32),
                ('J', C.c_int32), ('T', C.c_int32), ('T0', C.c_int32), ('stride', C.c_int32), ('taps', C.c_int32),
                ('Fin', C.c_int32), ('heads', C.c_int32), ('Cg', C.c_int32)]


KernelAuditFn = C.CFUNCTYPE(C.c_int32, C.c_int32, C.POINTER(KernelAudit), C.c_void_p)

_lib = None


def load():
    """Load the library once; raise loudly when it is absent (no CPU / torch fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            'gast_b200: %s not found. Build it with `python __graft_entry__.py build` '
            '(or gast-net-3dposeestimation_b200/csrc/build.sh). There is no fallback path.' % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    vp = C.c_void_p
    lib.gast_create.argtypes = [C.POINTER(vp), C.POINTER(GastCfg)]
    lib.gast_create.restype = C.c_int
    lib.gast_destroy.argtypes = [vp]
    lib.gast_destroy.restype = None
    lib.gast_bind.argtypes = [vp, C.c_int32, C.POINTER(C.c_char_p), C.POINTER(vp), C.POINTER(C.c_int64)]
    lib.gast_bind.restype = C.c_int
    lib.gast_prepare.argtypes = [vp, vp]
    lib.gast_prepare.restype = C.c_int
    lib.gast_out_frames.argtypes = [vp, C.c_int32, C.c_int32]
    lib.gast_out_frames.restype = C.c_int32
    lib.gast_receptive_field.argtypes = [vp]
    lib.gast_receptive_field.restype = C.c_int32
    lib.gast_workspace_bytes.argtypes = [vp, C.c_int32, C.c_int32, C.c_int32]
    lib.gast_workspace_bytes.restype = C.c_size_t
    lib.gast_forward.argtypes = [vp, vp, vp, C.c_int32, C.c_int32, C.c_int32, vp, C.c_size_t, vp]
    lib.gast_forward.restype = C.c_int
    lib.gast_forward_mpjpe.argtypes = [vp, vp, vp, vp, vp, C.c_int32, C.c_int32, C.c_int32, vp, C.c_size_t, vp]
    lib.gast_forward_mpjpe.restype = C.c_int
    lib.gast_last_launch_count.argtypes = [vp]
    lib.gast_last_launch_count.restype = C.c_int32
    lib.gast_last_tc_launch_count.argtypes = [vp]
    lib.gast_last_tc_launch_count.restype = C.c_int32
    lib.gast_set_timing.argtypes = [vp, C.c_int32]
    lib.gast_set_timing.restype = C.c_int
    lib.gast_get_timings.argtypes = [vp, C.c_int32, C.POINTER(C.c_float), C.POINTER(C.c_int32)]
    lib.gast_get_timings.restype = C.c_int32
    lib.gast_set_gemm_core.argtypes = [vp, C.c_int32]
    lib.gast_set_gemm_core.restype = C.c_int
    lib.gast_set_precision.argtypes = [vp, C.c_int32]
    lib.gast_set_precision.restype = C.c_int
    lib.gast_set_activation_dtype.argtypes = [vp, C.c_int32]
    lib.gast_set_activation_dtype.restype = C.c_int
    lib.gast_set_train_precision.argtypes = [vp, C.c_int32]
    lib.gast_set_train_precision.restype = C.c_int
    lib.gast_last_wgrad_tc_launch_count.argtypes = [vp]
    lib.gast_last_wgrad_tc_launch_count.restype = C.c_int32
    lib.gast_debug_gemm.argtypes = [vp, vp, vp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                    C.POINTER(C.c_float), vp]
    lib.gast_debug_gemm.restype = C.c_int
    lib.gast_debug_wgrad.argtypes = [vp, vp, vp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                     C.POINTER(C.c_float), vp]
    lib.gast_debug_wgrad.restype = C.c_int
    lib.gast_debug_set_gemm_audit.argtypes = [vp, GemmAuditFn, vp]
    lib.gast_debug_set_gemm_audit.restype = C.c_int
    lib.gast_debug_gemm_audit_skips.argtypes = [vp]
    lib.gast_debug_gemm_audit_skips.restype = C.c_int64
    lib.gast_debug_set_kernel_audit.argtypes = [vp, KernelAuditFn, vp]
    lib.gast_debug_set_kernel_audit.restype = C.c_int
    lib.gast_debug_kernel_audit_skips.argtypes = [vp]
    lib.gast_debug_kernel_audit_skips.restype = C.c_int64
    lib.gast_bind_grads.argtypes = [vp, C.c_int32, C.POINTER(C.c_char_p), C.POINTER(vp), C.POINTER(C.c_int64)]
    lib.gast_bind_grads.restype = C.c_int
    lib.gast_train_workspace_bytes.argtypes = [vp, C.c_int32, C.c_int32, C.c_float]
    lib.gast_train_workspace_bytes.restype = C.c_size_t
    lib.gast_forward_train.argtypes = [vp, vp, vp, C.c_int32, C.c_int32, C.c_float, C.c_uint64, vp, C.c_size_t, vp]
    lib.gast_forward_train.restype = C.c_int
    lib.gast_backward.argtypes = [vp, vp, vp, C.c_size_t, vp]
    lib.gast_backward.restype = C.c_int
    lib.gast_backward_input.argtypes = [vp, vp, vp, C.c_int32, vp, C.c_size_t, vp]
    lib.gast_backward_input.restype = C.c_int
    lib.gast_eval_backward_workspace_bytes.argtypes = [vp, C.c_int32, C.c_int32, C.c_int32]
    lib.gast_eval_backward_workspace_bytes.restype = C.c_size_t
    lib.gast_eval_backward.argtypes = [vp, vp, vp, vp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, vp, C.c_size_t, vp]
    lib.gast_eval_backward.restype = C.c_int
    lib.gast_chunked_workspace_bytes.argtypes = [vp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32]
    lib.gast_chunked_workspace_bytes.restype = C.c_size_t
    lib.gast_forward_chunked.argtypes = [vp, vp, vp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, vp, C.c_size_t, vp]
    lib.gast_forward_chunked.restype = C.c_int
    lib.gast_eval_backward_chunked.argtypes = [vp, vp, vp, vp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, vp,
                                               C.c_size_t, vp]
    lib.gast_eval_backward_chunked.restype = C.c_int
    lib.gast_set_dropout_state.argtypes = [vp, vp]
    lib.gast_set_dropout_state.restype = C.c_int
    lib.gast_stream_state_bytes.argtypes = [vp, C.c_int32]
    lib.gast_stream_state_bytes.restype = C.c_size_t
    lib.gast_stream_workspace_bytes.argtypes = [vp, C.c_int32]
    lib.gast_stream_workspace_bytes.restype = C.c_size_t
    lib.gast_stream_push.argtypes = [vp, vp, C.c_int64, vp, vp, C.c_int32, vp, vp, C.c_size_t, vp]
    lib.gast_stream_push.restype = C.c_int
    lib.gast_stream_push_ex.argtypes = [vp, vp, C.c_int64, vp, vp, C.c_int32, vp, vp, vp, C.c_size_t, vp]
    lib.gast_stream_push_ex.restype = C.c_int
    lib.gast_stream_chunk_workspace_bytes.argtypes = [vp, C.c_int32, C.c_int32]
    lib.gast_stream_chunk_workspace_bytes.restype = C.c_size_t
    lib.gast_stream_push_chunk.argtypes = [vp, vp, C.c_int64, vp, vp, C.c_int32, C.c_int32, vp, vp, vp, C.c_size_t, vp]
    lib.gast_stream_push_chunk.restype = C.c_int
    lib.gast_stream_peek.argtypes = [vp, vp, C.c_int64, vp, C.c_int32, C.c_int32, vp, C.c_size_t, vp]
    lib.gast_stream_peek.restype = C.c_int
    lib.gast_stream_subset_workspace_bytes.argtypes = [vp, C.c_int32, C.c_int32]
    lib.gast_stream_subset_workspace_bytes.restype = C.c_size_t
    lib.gast_stream_push_subset.argtypes = [vp, vp, C.c_int32, vp, vp, C.c_int32, C.c_int32, vp, vp, vp, vp, vp,
                                            C.c_size_t, vp]
    lib.gast_stream_push_subset.restype = C.c_int
    lib.gast_stream_peek_subset.argtypes = [vp, vp, C.c_int32, vp, vp, C.c_int32, C.c_int32, vp, vp, C.c_size_t, vp]
    lib.gast_stream_peek_subset.restype = C.c_int
    lib.gast_stream_device_workspace_bytes.argtypes = [vp, C.c_int32, C.c_int32]
    lib.gast_stream_device_workspace_bytes.restype = C.c_size_t
    lib.gast_stream_push_device.argtypes = [vp, vp, C.c_int32, vp, vp, C.c_int32, vp, vp, vp, vp, vp, C.c_size_t, vp]
    lib.gast_stream_push_device.restype = C.c_int
    lib.gast_stream_peek_device.argtypes = [vp, vp, C.c_int32, vp, vp, C.c_int32, vp, vp, C.c_size_t, vp]
    lib.gast_stream_peek_device.restype = C.c_int
    lib.gast_stream_snapshot_floats.argtypes = [vp]
    lib.gast_stream_snapshot_floats.restype = C.c_size_t
    lib.gast_stream_move_workspace_bytes.argtypes = [vp, C.c_int32]
    lib.gast_stream_move_workspace_bytes.restype = C.c_size_t
    for fn in ('gast_stream_export', 'gast_stream_import'):
        getattr(lib, fn).argtypes = [vp, vp, C.c_int32, vp, vp, C.c_int32, vp, vp, C.c_size_t, vp]
        getattr(lib, fn).restype = C.c_int
    lib.gast_stream_latency.argtypes = [vp]
    lib.gast_stream_latency.restype = C.c_int32
    ip = C.POINTER(C.c_int32)
    lib.gast_tta_prepare.argtypes = [vp, vp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, ip, ip, vp]
    lib.gast_tta_prepare.restype = C.c_int
    lib.gast_tta_merge.argtypes = [vp, vp, C.c_int32, C.c_int32, C.c_int32, ip, ip, vp]
    lib.gast_tta_merge.restype = C.c_int
    fp = C.POINTER(C.c_float)
    lib.gast_chunk_gather.argtypes = [vp, vp, vp, vp, C.c_int32, vp, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                      C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, ip, ip, C.c_int32, ip, ip,
                                      vp, vp, vp, vp]
    lib.gast_chunk_gather.restype = C.c_int
    lib.gast_keypoints_convert.argtypes = [vp, vp, vp, C.c_int32, C.c_int32, C.c_int32, vp]
    lib.gast_keypoints_convert.restype = C.c_int
    lib.gast_h36m_coco_format.argtypes = [vp, vp, C.c_int32, C.c_int32, vp, vp, vp, vp, vp]
    lib.gast_h36m_coco_format.restype = C.c_int
    lib.gast_revise_kpts.argtypes = [vp, vp, vp, C.c_int32, C.c_int32, C.c_int32, vp, vp]
    lib.gast_revise_kpts.restype = C.c_int
    lib.gast_revise_skes_workspace_bytes.argtypes = [C.c_int32, C.c_int32]
    lib.gast_revise_skes_workspace_bytes.restype = C.c_size_t
    lib.gast_revise_skes.argtypes = [vp, vp, C.POINTER(C.c_int64), C.c_int32, C.c_int32, C.c_int32, C.c_int32, vp, vp, vp,
                                     C.c_size_t, vp]
    lib.gast_revise_skes.restype = C.c_int
    lib.gast_revise_skes_real_time_workspace_bytes.argtypes = [C.c_int32]
    lib.gast_revise_skes_real_time_workspace_bytes.restype = C.c_size_t
    lib.gast_revise_skes_real_time.argtypes = [vp, vp, C.c_int32, C.c_int32, C.c_int32, C.c_double, vp, vp, C.c_size_t, vp]
    lib.gast_revise_skes_real_time.restype = C.c_int
    lib.gast_normalize_screen.argtypes = [vp, vp, C.c_int64, C.c_float, C.c_float, C.c_int32, vp]
    lib.gast_normalize_screen.restype = C.c_int
    lib.gast_camera_to_world.argtypes = [vp, vp, C.c_int64, fp, fp, vp]
    lib.gast_camera_to_world.restype = C.c_int
    lib.gast_world_to_camera.argtypes = [vp, C.c_int64, C.c_int32, vp, vp, vp, C.c_int32, C.c_int64, C.c_int32, vp, vp]
    lib.gast_world_to_camera.restype = C.c_int
    lib.gast_project_to_2d.argtypes = [vp, C.c_int64, vp, vp, C.c_int32, vp, vp]
    lib.gast_project_to_2d.restype = C.c_int
    lib.gast_project_to_2d_backward.argtypes = [vp, C.c_int64, vp, vp, C.c_int32, vp, vp, vp]
    lib.gast_project_to_2d_backward.restype = C.c_int
    lib.gast_normalize_screen_segments.argtypes = [vp, C.c_int64, C.c_int32, C.c_int32, vp, vp, vp, C.c_int32, C.c_int64,
                                                   C.c_int32, vp, vp]
    lib.gast_normalize_screen_segments.restype = C.c_int
    lib.gast_mpjpe_workspace_bytes.argtypes = []
    lib.gast_mpjpe_workspace_bytes.restype = C.c_size_t
    lib.gast_mpjpe.argtypes = [vp, vp, C.c_int64, C.c_int32, vp, vp, C.c_float, vp, vp]
    lib.gast_mpjpe.restype = C.c_int
    lib.gast_p_mpjpe.argtypes = [vp, vp, C.c_int32, C.c_int32, vp, vp]
    lib.gast_p_mpjpe.restype = C.c_int
    lib.gast_pose_metrics_workspace_bytes.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_int64]
    lib.gast_pose_metrics_workspace_bytes.restype = C.c_size_t
    lib.gast_pose_metrics.argtypes = [vp, vp, C.c_int64, C.c_int32, C.POINTER(C.c_int64), C.c_int32, fp, C.c_int32,
                                      C.c_int32, C.c_int32, vp, vp, vp, C.c_size_t, vp]
    lib.gast_pose_metrics.restype = C.c_int
    lib.gast_render_geometry.argtypes = [C.c_int32, C.c_float, C.c_int32, C.c_int32, C.c_float, C.c_float, C.c_float,
                                         C.c_float, C.c_int32, fp]
    lib.gast_render_geometry.restype = C.c_int
    lib.gast_render_frames.argtypes = [vp, C.c_int64, C.c_int32, C.c_int32, vp, C.c_int32, C.c_int64, vp, C.c_int64,
                                       C.c_int32, C.c_int32, ip, C.POINTER(C.c_uint8), ip, C.c_int32, C.c_int32,
                                       C.c_int32, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int32,
                                       C.c_int64, C.c_int32, vp, vp]
    lib.gast_render_frames.restype = C.c_int
    lib.gast_downsample_frames.argtypes = [vp, C.c_int64, C.c_int64, C.c_int32, C.c_int32, vp, vp]
    lib.gast_downsample_frames.restype = C.c_int
    lib.gast_person_crops.argtypes = [vp, C.c_int64, C.c_int32, C.c_int32, vp, vp, C.c_int32, C.c_int32, C.c_int32,
                                      C.c_int32, vp, vp]
    lib.gast_person_crops.restype = C.c_int
    lib.gast_heatmap_decode.argtypes = [vp, vp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, vp, vp, vp]
    lib.gast_heatmap_decode.restype = C.c_int
    lib.gast_letterbox.argtypes = [vp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                   vp, vp]
    lib.gast_letterbox.restype = C.c_int
    lib.gast_person_detections.argtypes = [vp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, vp, C.c_float, C.c_float,
                                           C.c_int32, C.c_int32, vp, vp, vp, vp, vp, vp]
    lib.gast_person_detections.restype = C.c_int
    lib.gast_sort_state_bytes.argtypes = [C.c_int32, C.c_int32]
    lib.gast_sort_state_bytes.restype = C.c_size_t
    lib.gast_sort_init.argtypes = [vp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, vp, vp]
    lib.gast_sort_init.restype = C.c_int
    lib.gast_sort_update.argtypes = [vp, C.c_int32, C.c_int32, C.c_int32, vp, vp, C.c_int32, C.c_int32, vp, vp, vp, vp]
    lib.gast_sort_update.restype = C.c_int
    lib.gast_track_records.argtypes = [vp, vp, vp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                       C.c_int32, C.c_int32, vp, vp, vp, vp, vp, vp, vp]
    lib.gast_track_records.restype = C.c_int
    lib.gast_record_inverse.argtypes = [vp, C.c_int32, vp, C.c_int32, C.c_int32, vp, vp]
    lib.gast_record_inverse.restype = C.c_int
    # the live tick (DESIGN.md §8.10)
    lib.gast_live_slots.argtypes = [vp, vp, vp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                    C.c_int32, C.c_int32, C.c_int32, vp, vp, vp, vp, vp, vp, vp]
    lib.gast_live_slots.restype = C.c_int
    lib.gast_live_inputs.argtypes = [vp, vp, vp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, vp, vp, vp, vp, vp, vp,
                                     vp, vp]
    lib.gast_live_inputs.restype = C.c_int
    lib.gast_live_place.argtypes = [vp, vp, vp, C.c_int32, C.c_int32, C.c_double, vp, vp]
    lib.gast_live_place.restype = C.c_int
    lib.gast_adam_chunk.argtypes = []
    lib.gast_adam_chunk.restype = C.c_int32
    lib.gast_adam_step.argtypes = [vp, C.c_int32, vp, vp, vp, C.c_double, C.c_double, C.c_double, C.c_double,
                                   C.c_double, C.c_int64, vp]
    lib.gast_adam_step.restype = C.c_int
    lib.gast_chunk_gather_indexed.argtypes = [vp, vp, vp, vp, C.c_int32, vp, C.c_int64, C.c_int32, vp, C.c_int32,
                                              C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                              C.c_int32, C.c_int32, ip, ip, C.c_int32, ip, ip, vp, vp, vp, vp]
    lib.gast_chunk_gather_indexed.restype = C.c_int
    lib.gast_adam_step_table.argtypes = [C.c_double, C.c_double, C.c_double, C.c_int64, C.c_int32, vp]
    lib.gast_adam_step_table.restype = C.c_int
    lib.gast_adam_step_indexed.argtypes = [vp, C.c_int32, vp, vp, vp, C.c_double, C.c_double, C.c_double, C.c_double,
                                           vp, C.c_int64, vp, vp]
    lib.gast_adam_step_indexed.restype = C.c_int
    lib.gast_epoch_loss_accumulate.argtypes = [vp, C.c_int64, vp, vp, C.c_int64, vp, vp]
    lib.gast_epoch_loss_accumulate.restype = C.c_int
    lib.gast_last_error.argtypes = []
    lib.gast_last_error.restype = C.c_char_p
    lib.gast_version.argtypes = []
    lib.gast_version.restype = C.c_char_p
    _lib = lib
    return lib


def last_error():
    return load().gast_last_error().decode('utf-8', 'replace')
