"""ctypes binding of libccb200.so (include/ccb200.h).

The product path has NO CPU fallback: importing works without the library (so the package can be
inspected), but the first op call raises if ``cc_b200/libccb200.so`` is missing, and every op
refuses non-CUDA tensors.  The only exception is the *test hook* ``use_library(path)``, which the
GPU-less unit tests use to point the binding at the CPU execution-model simulator build of the same
kernel sources (tests/sim); that library reports ``ccb_is_simulator() == 1``.
"""
import ctypes as C
import os
import torch

MAX_LEVELS = 8
MAX_REFS = 4
SSIM_TAPS = 13

PHOTO_RIGID, PHOTO_FLOW, PHOTO_CONSENSUS = 0, 1, 2
ROT_EULER, ROT_QUAT = 0, 1
PAD_ZEROS, PAD_BORDER, PAD_NONE = 0, 1, 2
SMOOTH_EDGE, SMOOTH_SECOND = 0, 1
BCE_ONES, BCE_CONSENSUS = 0, 1

_P = C.c_void_p
_LP = _P * MAX_LEVELS
_LRP = (_P * MAX_REFS) * MAX_LEVELS
_LI = C.c_int * MAX_LEVELS


class PhotoDesc(C.Structure):
    _fields_ = [
        ('mode', C.c_int), ('B', C.c_int), ('R', C.c_int), ('H', C.c_int), ('W', C.c_int),
        ('nlevels', C.c_int), ('h', _LI), ('w', _LI),
        ('has_mask', C.c_int), ('has_occ', C.c_int), ('rotation_mode', C.c_int), ('padding_mode', C.c_int),
        ('wssim', C.c_float), ('qch', C.c_float), ('lambda_oob', C.c_float), ('wrig', C.c_float),
        ('one_minus_wssim', C.c_float),
        ('taps', C.c_float * SSIM_TAPS),
        ('tgt', _LP), ('ref', _LRP), ('depth', _LP), ('flow', _LRP), ('mask', _LP),
        ('pose', _P), ('K', _P), ('Kinv', _P),
        ('dmaps', _LP), ('gmask', _LP), ('vo', _LP), ('scal', _P),
        ('partials', _P), ('loss', _P), ('target', _LP),
        ('grad_out', _P), ('d_depth', _LP), ('d_flow', _LRP), ('d_mask', _LP), ('d_pose', _P),
        ('pose_partials', _P),
    ]


class SmoothDesc(C.Structure):
    _fields_ = [
        ('kind', C.c_int), ('B', C.c_int), ('C', C.c_int), ('nlevels', C.c_int), ('h', _LI), ('w', _LI),
        ('img', _LP), ('pred', _LP), ('partials', _P), ('loss', _P), ('grad_out', _P), ('d_pred', _LP),
    ]


class BceDesc(C.Structure):
    _fields_ = [
        ('kind', C.c_int), ('B', C.c_int), ('C', C.c_int), ('nlevels', C.c_int), ('h', _LI), ('w', _LI),
        ('thresh', C.c_float), ('wbce', C.c_float),
        ('mask', _LP), ('census_bwd', _LP), ('census_fwd', _LP), ('target_bwd', _LP), ('target_fwd', _LP),
        ('partials', _P), ('loss', _P), ('grad_out', _P), ('d_mask', _LP),
    ]


class ConvDesc(C.Structure):
    _fields_ = [(n, C.c_int) for n in ('B', 'Ci', 'Hi', 'Wi', 'Co', 'Ho', 'Wo', 'kh', 'kw', 'stride', 'pad', 'act')] + \
               [('slope', C.c_float), ('impl', C.c_int), ('wcache', C.c_void_p)]


ACT_NONE, ACT_RELU, ACT_LEAKY, ACT_SIGMOID = 0, 1, 2, 3
CONV_FPROP, CONV_DGRAD, CONV_WGRAD = 0, 1, 2
IMPL_AUTO, IMPL_FFMA, IMPL_TC = 0, 1, 2

_lib = None
_is_sim = False
DEFAULT_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'libccb200.so')

_I, _F, _LL = C.c_int, C.c_float, C.c_longlong
_SIGS = {
    'ccb_last_error_string': (C.c_char_p, []),
    'ccb_version': (_I, []),
    'ccb_is_simulator': (_I, []),
    'ccb_image_pyramid': (_I, [_P, _I, _I, _I, _I, C.POINTER(_P), _P]),
    'ccb_photo_partials_floats': (_LL, [C.POINTER(PhotoDesc)]),
    'ccb_photo_pose_partials_floats': (_LL, [C.POINTER(PhotoDesc)]),
    'ccb_photo_loss_fwd': (_I, [C.POINTER(PhotoDesc), _P]),
    'ccb_photo_loss_bwd': (_I, [C.POINTER(PhotoDesc), _P]),
    'ccb_consensus_targets': (_I, [C.POINTER(PhotoDesc), _P]),
    'ccb_inverse_warp_fwd': (_I, [_P, _P, _P, _I, _P, _P, _I, _I, _I, _I, _I, _P, _P]),
    'ccb_inverse_warp_bwd': (_I, [_P, _P, _P, _I, _P, _P, _I, _I, _I, _I, _I, _P, _P, _P, _P, _P]),
    'ccb_warp_pose_partials_floats': (_LL, [_I, _I, _I]),
    'ccb_flow_warp_fwd': (_I, [_P, _P, _I, _I, _I, _I, _I, _P, _P]),
    'ccb_flow_warp_bwd': (_I, [_P, _P, _I, _I, _I, _I, _I, _P, _P, _P, _P, _P]),
    'ccb_pose2flow_fwd': (_I, [_P, _P, _I, _P, _P, _I, _I, _I, _I, _I, _P, _P]),
    'ccb_pose2flow_bwd': (_I, [_P, _P, _I, _P, _P, _I, _I, _I, _I, _I, _P, _P, _P, _P, _P]),
    'ccb_ssim_fwd': (_I, [_P, _P, _I, _I, _I, C.POINTER(_F), _P, _P]),
    'ccb_ssim_bwd': (_I, [_P, _P, _I, _I, _I, C.POINTER(_F), _P, _P, _P, _P, _P]),
    'ccb_smooth_partials_floats': (_LL, [C.POINTER(SmoothDesc)]),
    'ccb_smooth_fwd': (_I, [C.POINTER(SmoothDesc), _P]),
    'ccb_smooth_bwd': (_I, [C.POINTER(SmoothDesc), _P]),
    'ccb_bce_partials_floats': (_LL, [C.POINTER(BceDesc)]),
    'ccb_bce_fwd': (_I, [C.POINTER(BceDesc), _P]),
    'ccb_bce_bwd': (_I, [C.POINTER(BceDesc), _P]),
    'ccb_conv_workspace_floats': (_LL, [C.POINTER(ConvDesc), _I]),
    'ccb_conv2d_fprop': (_I, [C.POINTER(ConvDesc), _P, _P, _P, _P, _P, _P, _LL, _P]),
    'ccb_conv2d_dgrad': (_I, [C.POINTER(ConvDesc), _P, _P, _P, _P, _P, _P, _LL, _P]),
    'ccb_conv2d_wgrad': (_I, [C.POINTER(ConvDesc), _P, _P, _P, _P, _LL, _P]),
    'ccb_act_bwd_bias_workspace_floats': (_LL, [_I, _I, _I]),
    'ccb_act_bwd_bias': (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _F, _P, _LL, _P]),
    'ccb_debug_last_conv_kernel': (C.c_char_p, []),
    'ccb_debug_tc_plan': (_I, [_I, C.POINTER(_I)]),
    'ccb_wcache_create': (C.c_void_p, []),
    'ccb_wcache_destroy': (None, [C.c_void_p]),
    'ccb_wcache_plan_floats': (_LL, [C.c_void_p]),
    'ccb_wcache_table_bytes': (_LL, [C.c_void_p]),
    'ccb_wcache_commit': (_I, [C.c_void_p, _P, _LL, _P, _LL, _P]),
    'ccb_wcache_refresh': (_I, [C.c_void_p, _P]),
    'ccb_wcache_stats': (None, [C.c_void_p, C.POINTER(C.c_longlong * 4)]),
    'ccb_corr81_fwd_workspace_floats': (_LL, [_I, _I, _I, _I]),
    'ccb_corr81_fwd': (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _P, _LL, _P]),
    'ccb_corr81_bwd': (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _P, _P]),
    'ccb_corr441d_fwd': (_I, [_P, _P, _P, _I, _I, _I, _I, _P]),
    'ccb_corr441d_bwd': (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _P]),
    'ccb_featwarp_fwd': (_I, [_P, _P, _I, _I, _I, _I, _P, _P]),
    'ccb_featwarp_bwd': (_I, [_P, _P, _I, _I, _I, _I, _P, _P, _P, _P, _P]),
    'ccb_bn_workspace_floats': (_LL, [_I, _I, _I]),
    'ccb_bn_fwd': (_I, [_P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _F, _F, _I, _P, _P]),
    'ccb_bn_bwd': (_I, [_P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _P, _P]),
    'ccb_upsample2x_fwd': (_I, [_P, _P, _I, _I, _I, _P]),
    'ccb_upsample2x_bwd': (_I, [_P, _P, _I, _I, _I, _P]),
    'ccb_adam_step': (_I, [_P, _P, _P, _P, _LL, _P, _F, _F, _F, _F, _F, _P]),
    'ccb_adam_step_ranges': (_I, [_P, _P, _P, _P, _P, _I, _LL, _P, _I, _P, _F, _F, _F, _F, _F, _P]),
    'ccb_launch_count': (_LL, []),
    'ccb_flow_metrics_workspace_bytes': (_LL, [_I, _I, _I]),
    'ccb_flow_metrics': (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _F, _F, _F, _P, _P, _P, _P]),
    'ccb_depth_errors_workspace_bytes': (_LL, [_I, _I, _I]),
    'ccb_depth_errors': (_I, [_P, _P, _I, _I, _I, _I, _P, _P, _P]),
    'ccb_mask_iou_workspace_bytes': (_LL, [_I, _I, _I, _I, _I]),
    'ccb_mask_iou': (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _F, _I, _P, _P, _LL, _P, _P]),
    'ccb_prep_frames': (_I, [_P, C.POINTER(_P), _P, _P, _I, _I, _I, _I, _I, _I, _P]),
    'ccb_prep_frames_unit': (_I, [_P, C.POINTER(_P), _P, _P, _I, _I, _I, _I, _I, _I, _P]),
    'ccb_rotate_frames_u8': (_I, [_P, _P, _P, _I, _I, _I, _I, _P]),
    'ccb_resize_u8_workspace_bytes': (_LL, [_I, _I, _I, _I, _I]),
    'ccb_resize_u8': (_I, [_P, _P, _I, _I, _I, _I, _I, _P, _LL, _P]),
    'ccb_normalize_local_workspace_bytes': (_LL, [_I, _I, _I]),
    'ccb_normalize_local': (_I, [C.POINTER(_P), _I, _I, _I, _I, _P, _P, _LL, _P]),
}
# entry points added by later translation units register themselves here (conv, nets, optimiser ...)
EXTRA_SIGS = {}


def _bind(lib):
    sigs = dict(_SIGS)
    sigs.update(EXTRA_SIGS)
    for name, (res, args) in sigs.items():
        fn = getattr(lib, name)          # AttributeError => header/library mismatch: fail loudly
        fn.restype = res
        fn.argtypes = args


def use_library(path):
    """Load a specific build of the library (test hook; see module docstring)."""
    global _lib, _is_sim
    lib = C.CDLL(path)
    _bind(lib)
    _lib = lib
    _is_sim = bool(lib.ccb_is_simulator())
    return lib


def lib():
    if _lib is None:
        if not os.path.exists(DEFAULT_PATH):
            raise RuntimeError(
                'cc_b200: %s is missing - build the sm_90a extension first '
                '(python -c "import __graft_entry__ as g; g.build()"); there is no CPU fallback.' % DEFAULT_PATH)
        use_library(DEFAULT_PATH)
    return _lib


def is_simulator():
    lib()
    return _is_sim


def check(rc, what=''):
    if rc != 0:
        msg = lib().ccb_last_error_string()
        raise RuntimeError('libccb200 %s failed (status %d): %s' % (what, rc, msg.decode() if msg else ''))


def ptr(t, name='tensor', dtype=torch.float32):
    """Device pointer of a contiguous tensor of `dtype` (fp32 unless stated; None -> NULL)."""
    if t is None:
        return None
    if t.dtype != dtype:
        raise TypeError('cc_b200: %s must be %s, got %s' % (name, dtype, t.dtype))
    if not t.is_contiguous():
        raise ValueError('cc_b200: %s must be contiguous' % name)
    if not t.is_cuda and not is_simulator():
        raise RuntimeError('cc_b200: %s is on %s - the sm_90a kernels need CUDA tensors (no CPU fallback)'
                           % (name, t.device))
    return t.data_ptr()


def scatter_workspace(t):
    """Fixed-point accumulators (+1 word) for the image gradient of a warp of `t` (ccb_flow_warp_bwd / ccb_featwarp_bwd)."""
    return torch.empty(t.numel() + 1, dtype=torch.int64, device=t.device)


def stream(t=None):
    if t is not None and t.is_cuda:
        return torch.cuda.current_stream(t.device).cuda_stream
    return None


def contig(t):
    return t if t.is_contiguous() else t.contiguous()
