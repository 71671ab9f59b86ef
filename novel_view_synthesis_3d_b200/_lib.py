"""ctypes binding of libxunet_b200.so (include/xunet_b200.h).  There is NO fallback: if the CUDA
library is missing or fails to load, importing the compute path raises."""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

# XUNET_LIB=<path> loads another build of the same library (same-call A/B of a kernel change against the previous build)
LIB_PATH = Path(os.environ['XUNET_LIB']).resolve() if os.environ.get('XUNET_LIB') else Path(__file__).resolve().parent / 'libxunet_b200.so'
MAX_LEVELS = 8
GRAD_NORM_SCRATCH = 1024       # XUNET_GRAD_NORM_SCRATCH: doubles of scratch xunet_grad_global_norm needs
SAMPLER_DYN_MAX_PER = 256 * 256 * 3     # XUNET_SAMPLER_DYN_MAX_PER: values per view xunet_sampler_step_dynamic takes
DTYPE_F32, DTYPE_BF16 = 0, 1
PIXELS_U8, PIXELS_F32 = 0, 1            # XUNET_PIXELS_*: storage of an xunet_srn_store's views
RAYS = {'v3d130_ij': 0, 'opencv_uv': 1}


class XunetConfig(C.Structure):
    _fields_ = [('ch', C.c_int), ('n_levels', C.c_int), ('ch_mult', C.c_int * MAX_LEVELS), ('emb_ch', C.c_int),
                ('num_res_blocks', C.c_int), ('n_attn_resolutions', C.c_int),
                ('attn_resolutions', C.c_int * MAX_LEVELS), ('attn_heads', C.c_int), ('dropout', C.c_float),
                ('use_pos_emb', C.c_int), ('use_ref_pose_emb', C.c_int), ('ray_convention', C.c_int)]


class XunetBatch(C.Structure):
    _fields_ = [(k, C.c_void_p) for k in ('x', 'z', 'logsnr', 'R1', 't1', 'R2', 't2', 'K', 'cond_mask', 'rays')]


class XunetInputGrads(C.Structure):
    _fields_ = [(k, C.c_void_p) for k in ('dx', 'dz', 'd_rays', 'dR1', 'dt1', 'dR2', 'dt2', 'dK')]


LAUNCH_CONV, LAUNCH_ATTN = 0, 1
KERNEL_NONE, KERNEL_SIMT, KERNEL_TC, KERNEL_CIN3, KERNEL_COUT3 = -1, 0, 1, 2, 3


class XunetLaunchInfo(C.Structure):
    _fields_ = [('kind', C.c_int), ('leaf', C.c_int)] + \
        [(k, C.c_int) for k in ('N', 'Hi', 'Wi', 'Ci', 'Ho', 'Wo', 'Co', 'ksize', 'stride', 'nseg', 'residual')] + \
        [('alpha', C.c_float), ('fwd', C.c_int), ('dgrad', C.c_int), ('wgrad', C.c_int), ('emits_stats', C.c_int),
         ('bwd_alpha', C.c_float), ('accumulate', C.c_int), ('gn_mode', C.c_int)] + \
        [(k, C.c_int) for k in ('L', 'C', 'heads', 'cross', 'impl')]


PLAN_OP_LOGSNR, PLAN_OP_POSE, PLAN_OP_EMB, PLAN_OP_RESAMPLE, PLAN_OP_CONCAT, PLAN_OP_ATTN_RESIDUAL, PLAN_OP_LOSS = range(7)
RS_NONE, RS_DOWN, RS_UP = 0, 1, 2


class XunetOpInfo(C.Structure):
    _fields_ = [(k, C.c_int) for k in ('kind', 'B', 'S', 'E', 'N', 'H', 'W', 'C', 'C2')] + \
        [('copies', (C.c_int * 5) * 4), ('rs', C.c_int), ('fwd_pool', C.c_int), ('fwd_scale', C.c_float), ('gscale', C.c_float),
         ('bwd_pool', C.c_int), ('bwd_scale', C.c_float), ('alpha', C.c_float)] + \
        [(k, C.c_int) for k in ('acc_x', 'acc_r', 'need_grad', 'need_grad_r', 'write_dpe', 'pos_emb', 'ref_pose_emb',
                                'ray_convention')]


class XunetSrnStore(C.Structure):
    _fields_ = [('pixels', C.c_void_p), ('pixel_kind', C.c_int), ('S', C.c_int), ('n_items', C.c_longlong),
                ('n_instances', C.c_int), ('R', C.c_void_p), ('t', C.c_void_p), ('K', C.c_void_p), ('first', C.c_void_p),
                ('count', C.c_void_p), ('item_inst', C.c_void_p)]


# void fn(void* user, long long elem_offset, long long n_elems)  -- the data-parallel gradient-bucket hook
BUCKET_FN = C.CFUNCTYPE(None, C.c_void_p, C.c_longlong, C.c_longlong)


# name -> (restype, argtypes): every symbol include/xunet_b200.h declares
SYMBOLS = {
    'xunet_last_error': (C.c_char_p, []),
    'xunet_version': (C.c_int, []),
    'xunet_create': (C.c_int, [C.POINTER(XunetConfig), C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_void_p)]),
    'xunet_destroy': (None, [C.c_void_p]),
    'xunet_param_count': (C.c_longlong, [C.c_void_p]),
    'xunet_param_leaves': (C.c_int, [C.c_void_p]),
    'xunet_param_leaf': (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_int),
                                   C.POINTER(C.c_longlong * 5), C.POINTER(C.c_longlong)]),
    'xunet_workspace_bytes': (C.c_longlong, [C.c_void_p]),
    'xunet_tap_count': (C.c_int, [C.c_void_p]),
    'xunet_tap': (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_int * 4),
                            C.POINTER(C.c_longlong), C.POINTER(C.c_int), C.POINTER(C.c_longlong)]),
    'xunet_plan_launch_count': (C.c_int, [C.c_void_p]),
    'xunet_plan_launch': (C.c_int, [C.c_void_p, C.c_int, C.POINTER(XunetLaunchInfo)]),
    'xunet_plan_op_count': (C.c_int, [C.c_void_p]),
    'xunet_plan_op': (C.c_int, [C.c_void_p, C.c_int, C.POINTER(XunetOpInfo)]),
    'xunet_forward': (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(XunetBatch), C.c_int, C.c_void_p, C.c_void_p,
                                C.c_void_p, C.c_void_p]),
    'xunet_set_static_conditioning': (C.c_int, [C.c_void_p, C.c_int]),
    'xunet_set_feature_cache': (C.c_int, [C.c_void_p, C.c_int]),
    'xunet_backward': (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(XunetBatch), C.c_void_p, C.c_void_p, C.c_void_p,
                                 C.c_void_p, C.c_void_p, C.c_void_p]),
    'xunet_backward_accumulate': (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(XunetBatch), C.c_void_p, C.c_void_p,
                                            C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    'xunet_backward_mse': (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(XunetBatch)] + [C.c_void_p] * 6 +
                           [C.c_int, C.c_void_p]),
    'xunet_backward_vjp': (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(XunetBatch)] + [C.c_void_p] * 4 +
                           [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    'xunet_backward_vjp_inputs': (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(XunetBatch)] + [C.c_void_p] * 4 +
                                  [C.c_int, C.POINTER(XunetInputGrads), C.c_void_p]),
    'xunet_set_grad_bucket_callback': (C.c_int, [C.c_void_p, BUCKET_FN, C.c_void_p, C.c_longlong]),
    'xunet_grad_bucket_count': (C.c_int, [C.c_void_p]),
    'xunet_count_kernels': (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(XunetBatch), C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    'xunet_adam_step': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong, C.c_longlong,
                                  C.c_void_p, C.c_double, C.c_double, C.c_double, C.c_double, C.c_double, C.c_void_p]),
    'xunet_adam_ema_step': (C.c_int, [C.c_void_p] * 5 + [C.c_longlong, C.c_longlong, C.c_void_p] + [C.c_double] * 6 +
                            [C.c_void_p]),
    'xunet_grad_global_norm': (C.c_int, [C.c_void_p, C.c_longlong, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p]),
    'xunet_adam_clip_step': (C.c_int, [C.c_void_p] * 5 + [C.c_longlong, C.c_longlong, C.c_void_p] + [C.c_double] * 6 +
                             [C.c_void_p, C.c_double, C.c_longlong, C.c_void_p, C.c_void_p]),
    'xunet_adam_posthoc_step': (C.c_int, [C.c_void_p] * 6 + [C.c_longlong, C.c_longlong, C.c_void_p] + [C.c_double] * 7 +
                                [C.c_void_p, C.c_double, C.c_longlong, C.c_void_p, C.c_void_p]),
    'xunet_sampler_step_table': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong, C.c_float, C.c_void_p, C.c_void_p,
                                           C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    'xunet_sampler_step_multistep': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong, C.c_float] +
                                     [C.c_void_p] * 6 + [C.c_int, C.c_void_p]),
    'xunet_sampler_step_dynamic': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong, C.c_float] + [C.c_void_p] * 4 +
                                   [C.c_int, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    'xunet_forward_diffusion': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_ulonglong, C.c_void_p, C.c_void_p, C.c_float,
                                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_longlong,
                                          C.c_void_p]),
    'xunet_forward_diffusion_v': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_ulonglong, C.c_void_p, C.c_void_p,
                                            C.c_float] + [C.c_void_p] * 6 + [C.c_int, C.c_longlong, C.c_void_p]),
    'xunet_srn_batch': (C.c_int, [C.POINTER(XunetSrnStore), C.c_void_p, C.c_ulonglong] + [C.c_int] * 5 +
                        [C.c_void_p, C.c_void_p, C.c_float, C.c_void_p, C.POINTER(XunetBatch)] + [C.c_void_p] * 5),
    'xunet_srn_batch_v': (C.c_int, [C.POINTER(XunetSrnStore), C.c_void_p, C.c_ulonglong] + [C.c_int] * 5 +
                          [C.c_void_p, C.c_void_p, C.c_float, C.c_void_p, C.POINTER(XunetBatch)] + [C.c_void_p] * 6),
    'xunet_srn_batch_distill': (C.c_int, [C.POINTER(XunetSrnStore), C.c_void_p, C.c_ulonglong] + [C.c_int] * 5 +
                                [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.POINTER(XunetBatch), C.POINTER(XunetBatch),
                                 C.c_int] + [C.c_void_p] * 4),
    'xunet_distill_teacher_step': (C.c_int, [C.c_void_p, C.c_float, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_longlong,
                                             C.POINTER(XunetBatch), C.c_void_p]),
    'xunet_distill_target': (C.c_int, [C.c_void_p, C.c_float, C.c_int] + [C.c_void_p] * 5 + [C.c_int, C.c_longlong,
                                                                                             C.c_void_p, C.c_void_p]),
    'xunet_cd_teacher_step': (C.c_int, [C.c_void_p, C.c_float, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_longlong] +
                              [C.c_void_p] * 4),
    'xunet_cd_target': (C.c_int, [C.c_void_p] * 5 + [C.c_int, C.c_longlong, C.c_void_p, C.c_void_p]),
    'xunet_sampler_step_cond': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong] + [C.c_void_p] * 4 +
                                [C.c_int, C.c_double] + [C.c_void_p] * 4),
    'xunet_sampler_step_guide': (C.c_int, [C.c_void_p] * 4 + [C.c_longlong, C.c_float] + [C.c_void_p] * 4 +
                                 [C.c_int, C.c_double] + [C.c_void_p] * 4),
    'xunet_dropout_mask': (C.c_int, [C.c_void_p, C.c_longlong, C.c_int, C.c_ulonglong, C.c_float, C.c_void_p]),
    'xunet_image_metrics': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p]),
    'xunet_field_render': (C.c_int, [C.c_void_p, C.c_int, C.c_float] + [C.c_void_p] * 4 + [C.c_int, C.c_int] + [C.c_float] * 3 +
                           [C.c_void_p, C.c_void_p]),
    'xunet_field_loss_grad': (C.c_int, [C.c_void_p, C.c_int, C.c_float] + [C.c_void_p] * 5 + [C.c_int, C.c_int] +
                              [C.c_float] * 3 + [C.c_int, C.c_void_p, C.c_ulonglong, C.c_float, C.c_float] + [C.c_void_p] * 3 +
                              [C.c_longlong, C.c_void_p]),
    'xunet_field_image_grad': (C.c_int, [C.c_void_p, C.c_int, C.c_float, C.c_void_p, C.c_double] + [C.c_void_p] * 4 +
                               [C.c_int, C.c_int] + [C.c_float] * 5 + [C.c_void_p] * 3),
    'xunet_pose_draw': (C.c_int, [C.c_void_p] + [C.c_int] * 6 + [C.c_void_p, C.c_ulonglong, C.c_void_p, C.c_void_p, C.c_int] +
                        [C.c_void_p] * 5),
    'xunet_pose_loss': (C.c_int, [C.c_void_p, C.c_void_p] + [C.c_int] * 3 + [C.c_void_p] * 4 + [C.c_longlong, C.c_void_p]),
    'xunet_pose_tangent': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                     C.c_void_p]),
    'xunet_pose_retract': (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 5),
    'xunet_lift_draw': (C.c_int, [C.c_int] * 3 + [C.c_void_p, C.c_ulonglong] + [C.c_double] * 6 + [C.c_void_p] * 6),
    'xunet_lift_noise': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_ulonglong] + [C.c_void_p] * 6),
    'xunet_lift_grad': (C.c_int, [C.c_void_p] * 6 + [C.c_int, C.c_int, C.c_float, C.c_int, C.c_float, C.c_float, C.c_double] +
                        [C.c_void_p] * 7 + [C.c_longlong, C.c_void_p]),
    'xunet_op_conv': (C.c_int, [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p] +
                      [C.c_int] * 8 + [C.c_float, C.c_void_p]),
    'xunet_op_conv_dgrad': (C.c_int, [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p] + [C.c_int] * 8 +
                            [C.c_float, C.c_int, C.c_void_p]),
    'xunet_op_conv_wgrad': (C.c_int, [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p] +
                            [C.c_int] * 8 + [C.c_float, C.c_void_p]),
    'xunet_op_attention': (C.c_int, [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p] +
                           [C.c_int] * 5 + [C.c_void_p]),
    'xunet_op_attention_bwd': (C.c_int, [C.c_int, C.c_int] + [C.c_void_p] * 7 + [C.c_int] * 5 + [C.c_void_p]),
    'xunet_op_conv_stats': (C.c_int, [C.c_int, C.c_int] + [C.c_void_p] * 6 + [C.c_int] * 6 + [C.c_float, C.c_void_p]),
    'xunet_op_attention_stats': (C.c_int, [C.c_int, C.c_int] + [C.c_void_p] * 5 + [C.c_int] * 5 + [C.c_void_p]),
    'xunet_op_groupnorm': (C.c_int, [C.c_int] + [C.c_void_p] * 3 + [C.c_int] + [C.c_void_p] * 6 + [C.c_int] * 6 +
                           [C.c_float, C.c_int, C.c_void_p, C.c_int, C.c_void_p]),
    'xunet_op_conv_dgrad_groupnorm': (C.c_int, [C.c_int] + [C.c_void_p] * 4 + [C.c_int] + [C.c_void_p] * 2 +
                                      [C.c_float, C.c_int, C.c_void_p, C.c_int] + [C.c_void_p] * 2 + [C.c_int] * 7 +
                                      [C.c_float, C.c_void_p]),
    'xunet_op_groupnorm_bwd': (C.c_int, [C.c_int] + [C.c_void_p] * 13 + [C.c_float] + [C.c_int] * 6 +
                               [C.c_float, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    'xunet_op_logsnr_emb': (C.c_int, [C.c_void_p] * 8 + [C.c_int, C.c_int, C.c_void_p]),
    'xunet_op_logsnr_emb_bwd': (C.c_int, [C.c_void_p] * 9 + [C.c_int, C.c_int, C.c_int, C.c_void_p]),
    'xunet_op_pose_emb': (C.c_int, [C.c_int] + [C.c_void_p] * 11 + [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    'xunet_op_pose_emb_bwd': (C.c_int, [C.c_int] + [C.c_void_p] * 4 + [C.c_int, C.c_int, C.c_int, C.c_void_p]),
    'xunet_op_film_emb': (C.c_int, [C.c_int] + [C.c_void_p] * 3 + [C.c_int] * 3 + [C.c_void_p]),
    'xunet_op_film_emb_bwd': (C.c_int, [C.c_int] + [C.c_void_p] * 5 + [C.c_int] * 4 + [C.c_void_p]),
    'xunet_op_resample': (C.c_int, [C.c_int, C.c_void_p, C.c_void_p] + [C.c_int] * 5 + [C.c_float, C.c_int, C.c_void_p]),
    'xunet_op_copy_channels': (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_longlong] + [C.c_int] * 6 + [C.c_void_p]),
    'xunet_op_scale_add': (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_longlong, C.c_float, C.c_int, C.c_void_p]),
    'xunet_op_loss': (C.c_int, [C.c_int] + [C.c_void_p] * 5 + [C.c_int, C.c_int, C.c_void_p]),
}

_lib = None


def load():
    """Load the CUDA library; raises (never falls back) if it is absent or lacks a symbol."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise RuntimeError(f'{LIB_PATH} is missing: build it with `python -m novel_view_synthesis_3d_b200.build` '
                           f'(or __graft_entry__.build()); there is no CPU/PyTorch fallback for the X-UNet path')
    lib = C.CDLL(str(LIB_PATH))
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)   # AttributeError if the .so does not export it
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc: int, what: str = ''):
    if rc != 0:
        raise RuntimeError(f'{what}: {load().xunet_last_error().decode()}')
