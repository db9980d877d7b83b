"""ctypes binding of libccb200.so (include/ccb200.h, include/ccb200_debug.h).

Every op reaches the library through ``call(name, *args)``, which converts each argument as the header declares that
parameter (``_SIGS``) and raises on a non-zero status.  tests/test_cabi_symbols.py holds ``_SIGS`` and the descriptor
Structures to the headers.

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
        ('partials', _P), ('partials_floats', C.c_longlong), ('loss', _P), ('target', _LP),
        ('grad_out', _P), ('d_depth', _LP), ('d_flow', _LRP), ('d_mask', _LP), ('d_pose', _P),
        ('pose_partials', _P), ('pose_partials_floats', C.c_longlong),
    ]


class SmoothDesc(C.Structure):
    _fields_ = [
        ('kind', C.c_int), ('B', C.c_int), ('C', C.c_int), ('nlevels', C.c_int), ('h', _LI), ('w', _LI),
        ('img', _LP), ('pred', _LP), ('partials', _P), ('partials_floats', C.c_longlong), ('loss', _P), ('grad_out', _P),
        ('d_pred', _LP),
    ]


class BceDesc(C.Structure):
    _fields_ = [
        ('kind', C.c_int), ('B', C.c_int), ('C', C.c_int), ('nlevels', C.c_int), ('h', _LI), ('w', _LI),
        ('thresh', C.c_float), ('wbce', C.c_float),
        ('mask', _LP), ('census_bwd', _LP), ('census_fwd', _LP), ('target_bwd', _LP), ('target_fwd', _LP),
        ('partials', _P), ('partials_floats', C.c_longlong), ('loss', _P), ('grad_out', _P), ('d_mask', _LP),
    ]


class ConvDesc(C.Structure):
    _fields_ = [(n, C.c_int) for n in ('B', 'Ci', 'Hi', 'Wi', 'Co', 'Ho', 'Wo', 'kh', 'kw', 'stride', 'pad', 'act')] + \
               [('slope', C.c_float), ('impl', C.c_int), ('wcache', C.c_void_p)]


STRUCTS = {'ccb_photo_desc': PhotoDesc, 'ccb_smooth_desc': SmoothDesc, 'ccb_bce_desc': BceDesc, 'ccb_conv_desc': ConvDesc}

ACT_NONE, ACT_RELU, ACT_LEAKY, ACT_SIGMOID = 0, 1, 2, 3
CONV_FPROP, CONV_DGRAD, CONV_WGRAD = 0, 1, 2
IMPL_AUTO, IMPL_FFMA, IMPL_TC = 0, 1, 2

_lib = None
_is_sim = False
DEFAULT_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'libccb200.so')

# Every prototype of the headers: (return, parameter types), each type written as the header writes it.  A pointer is a
# device pointer unless marked 'host'; 'handle void*' is the weight-cache handle.  The return STATUS is an int
# ccb_status that call() checks; any other return is handed back as it is.
STATUS = 'status'
_SIGS = {
    'ccb_last_error_string': ('const char*', ''),
    'ccb_version': ('int', ''),
    'ccb_is_simulator': ('int', ''),
    'ccb_image_pyramid': (STATUS, 'const float*, int, int, int, int, float* const*, ccb_stream_t'),
    'ccb_photo_partials_floats': ('long long', 'const ccb_photo_desc*'),
    'ccb_photo_pose_partials_floats': ('long long', 'const ccb_photo_desc*'),
    'ccb_photo_loss_fwd': (STATUS, 'const ccb_photo_desc*, ccb_stream_t'),
    'ccb_photo_loss_bwd': (STATUS, 'const ccb_photo_desc*, ccb_stream_t'),
    'ccb_consensus_targets': (STATUS, 'const ccb_photo_desc*, ccb_stream_t'),
    'ccb_inverse_warp_fwd': (STATUS, 'const float*, const float*, const float*, int, const float*, const float*, '
                                     'int, int, int, int, int, float*, ccb_stream_t'),
    'ccb_inverse_warp_bwd': (STATUS, 'const float*, const float*, const float*, int, const float*, const float*, '
                                     'int, int, int, int, int, const float*, float*, float*, float*, long long, '
                                     'ccb_stream_t'),
    'ccb_warp_pose_partials_floats': ('long long', 'int, int, int'),
    'ccb_flow_warp_fwd': (STATUS, 'const float*, const float*, int, int, int, int, int, float*, ccb_stream_t'),
    'ccb_flow_warp_bwd': (STATUS, 'const float*, const float*, int, int, int, int, int, const float*, float*, '
                                  'float*, unsigned long long*, long long, ccb_stream_t'),
    'ccb_pose2flow_fwd': (STATUS, 'const float*, const float*, int, const float*, const float*, int, int, int, int, '
                                  'int, float*, ccb_stream_t'),
    'ccb_pose2flow_bwd': (STATUS, 'const float*, const float*, int, const float*, const float*, int, int, int, int, '
                                  'int, const float*, float*, float*, float*, long long, ccb_stream_t'),
    'ccb_ssim_fwd': (STATUS, 'const float*, const float*, int, int, int, host const float*, float*, ccb_stream_t'),
    'ccb_ssim_bwd_workspace_floats': ('long long', 'int, int, int'),
    'ccb_ssim_bwd': (STATUS, 'const float*, const float*, int, int, int, host const float*, const float*, float*, '
                             'float*, float*, long long, ccb_stream_t'),
    'ccb_smooth_partials_floats': ('long long', 'const ccb_smooth_desc*'),
    'ccb_smooth_fwd': (STATUS, 'const ccb_smooth_desc*, ccb_stream_t'),
    'ccb_smooth_bwd': (STATUS, 'const ccb_smooth_desc*, ccb_stream_t'),
    'ccb_bce_partials_floats': ('long long', 'const ccb_bce_desc*'),
    'ccb_bce_fwd': (STATUS, 'const ccb_bce_desc*, ccb_stream_t'),
    'ccb_bce_bwd': (STATUS, 'const ccb_bce_desc*, ccb_stream_t'),
    'ccb_wcache_create': ('void*', ''),
    'ccb_wcache_destroy': ('void', 'handle void*'),
    'ccb_wcache_plan_floats': ('long long', 'handle void*'),
    'ccb_wcache_table_bytes': ('long long', 'handle void*'),
    'ccb_wcache_commit': (STATUS, 'handle void*, float*, long long, void*, long long, ccb_stream_t'),
    'ccb_wcache_refresh': (STATUS, 'handle void*, ccb_stream_t'),
    'ccb_wcache_stats': ('void', 'handle void*, host long long*'),
    'ccb_conv_workspace_floats': ('long long', 'const ccb_conv_desc*, int'),
    'ccb_conv2d_fprop': (STATUS, 'const ccb_conv_desc*, const float*, const float*, const float*, const float*, '
                                 'float*, float*, long long, ccb_stream_t'),
    'ccb_conv2d_dgrad': (STATUS, 'const ccb_conv_desc*, const float*, const float*, const float*, const float*, '
                                 'float*, float*, long long, ccb_stream_t'),
    'ccb_conv2d_wgrad': (STATUS, 'const ccb_conv_desc*, const float*, const float*, float*, float*, long long, '
                                 'ccb_stream_t'),
    'ccb_act_bwd_bias_workspace_floats': ('long long', 'int, int, int'),
    'ccb_act_bwd_bias': (STATUS, 'const float*, const float*, float*, float*, int, int, int, int, float, float*, '
                                 'long long, ccb_stream_t'),
    'ccb_corr81_fwd_workspace_floats': ('long long', 'int, int, int, int'),
    'ccb_corr81_fwd': (STATUS, 'const float*, const float*, float*, int, int, int, int, int, float*, long long, '
                               'ccb_stream_t'),
    'ccb_corr81_bwd_workspace_floats': ('long long', 'int, int, int, int'),
    'ccb_corr81_bwd': (STATUS, 'const float*, const float*, const float*, float*, float*, int, int, int, int, int, '
                               'float*, long long, ccb_stream_t'),
    'ccb_corr441d_fwd': (STATUS, 'const float*, const float*, float*, int, int, int, int, ccb_stream_t'),
    'ccb_corr441d_bwd': (STATUS, 'const float*, const float*, const float*, const float*, float*, float*, int, int, '
                                 'int, int, ccb_stream_t'),
    'ccb_featwarp_fwd': (STATUS, 'const float*, const float*, int, int, int, int, float*, ccb_stream_t'),
    'ccb_featwarp_bwd': (STATUS, 'const float*, const float*, int, int, int, int, const float*, float*, float*, '
                                 'unsigned long long*, long long, ccb_stream_t'),
    'ccb_bn_workspace_floats': ('long long', 'int, int, int'),
    'ccb_bn_fwd': (STATUS, 'const float*, const float*, const float*, float*, float*, float*, float*, int, int, int, '
                           'float, float, int, float*, long long, ccb_stream_t'),
    'ccb_bn_bwd': (STATUS, 'const float*, const float*, const float*, const float*, float*, float*, float*, int, '
                           'int, int, float*, long long, ccb_stream_t'),
    'ccb_upsample2x_fwd': (STATUS, 'const float*, float*, int, int, int, ccb_stream_t'),
    'ccb_upsample2x_bwd': (STATUS, 'const float*, float*, int, int, int, ccb_stream_t'),
    'ccb_adam_step_ranges': (STATUS, 'float*, const float*, float*, float*, const long long*, int, long long, '
                                     'const int*, int, float*, float, float, float, float, float, ccb_stream_t'),
    'ccb_flow_metrics_workspace_bytes': ('long long', 'int, int, int'),
    'ccb_flow_metrics': (STATUS, 'const float*, const float*, const float*, const float*, int, int, int, int, int, '
                                 'int, int, int, float, float, float, float*, void*, long long, float*, ccb_stream_t'),
    'ccb_depth_errors_workspace_bytes': ('long long', 'int, int, int'),
    'ccb_depth_errors': (STATUS, 'const float*, const float*, int, int, int, int, void*, long long, float*, '
                                 'ccb_stream_t'),
    'ccb_mask_iou_workspace_bytes': ('long long', 'int, int, int, int, int'),
    'ccb_mask_iou': (STATUS, 'const float*, const float*, const float*, const float*, const float*, int, int, int, '
                             'int, int, int, float, int, float*, void*, long long, long long*, ccb_stream_t'),
    'ccb_flow_submit': (STATUS, 'const float*, const float*, const float*, int, int, int, int, int, int, float, float*, '
                                'float*, unsigned short*, float*, ccb_stream_t'),
    'ccb_flow_eval_workspace_bytes': ('long long', 'int, int, int, int, int'),
    'ccb_flow_eval': (STATUS, 'const float*, const float*, const float*, const float*, const float*, int, int, int, int, '
                              'int, int, float, float, float, float, float*, void*, long long, float*, ccb_stream_t'),
    'ccb_flow_color_workspace_bytes': ('long long', 'int, int, int, int'),
    'ccb_flow_color': (STATUS, 'const float*, int, int, int, int, void*, long long, unsigned char*, ccb_stream_t'),
    'ccb_kitti_flow_errors_workspace_bytes': ('long long', 'int, int, int'),
    'ccb_kitti_flow_errors': (STATUS, 'const unsigned short*, const unsigned short*, int, int, int, void*, long long, '
                                      'double*, long long*, ccb_stream_t'),
    'ccb_velo_depth_workspace_bytes': ('long long', 'int, int, int'),
    'ccb_velo_depth': (STATUS, 'const float*, const long long*, const double*, long long, int, int, int, void*, long long, '
                               'double*, ccb_stream_t'),
    'ccb_spline_zoom_workspace_bytes': ('long long', 'int, int, int'),
    'ccb_spline_zoom': (STATUS, 'const float*, int, int, int, int, int, float, float, void*, long long, float*, ccb_stream_t'),
    'ccb_eigen_depth_errors_workspace_bytes': ('long long', 'int, int, int'),
    'ccb_eigen_depth_errors': (STATUS, 'const double*, const float*, int, int, int, double, double, host const double*, '
                                       'const float*, const double*, int, void*, long long, double*, ccb_stream_t'),
    'ccb_bytescale_u8_workspace_bytes': ('long long', 'int, int, int'),
    'ccb_bytescale_u8': (STATUS, 'const unsigned char*, int, int, int, void*, long long, unsigned char*, ccb_stream_t'),
    'ccb_make3d_depth_errors_workspace_bytes': ('long long', 'int, int, int'),
    'ccb_make3d_depth_errors': (STATUS, 'const double*, const float*, int, int, int, double, double, void*, long long, '
                                        'double*, ccb_stream_t'),
    'ccb_pose_errors': (STATUS, 'const float*, int, int, int, const double*, double*, double*, ccb_stream_t'),
    'ccb_prep_frames': (STATUS, 'const unsigned char*, float* const*, const float*, const int*, int, int, int, int, '
                                'int, int, ccb_stream_t'),
    'ccb_prep_frames_unit': (STATUS, 'const unsigned char*, float* const*, const float*, const int*, int, int, int, '
                                     'int, int, int, ccb_stream_t'),
    'ccb_rotate_frames_u8': (STATUS, 'const unsigned char*, const double*, unsigned char*, int, int, int, int, '
                                     'ccb_stream_t'),
    'ccb_resize_u8_workspace_bytes': ('long long', 'int, int, int, int, int'),
    'ccb_resize_u8': (STATUS, 'const unsigned char*, unsigned char*, int, int, int, int, int, void*, long long, '
                              'ccb_stream_t'),
    'ccb_normalize_local_workspace_bytes': ('long long', 'int, int, int'),
    'ccb_normalize_local': (STATUS, 'float* const*, int, int, int, int, float*, void*, long long, ccb_stream_t'),
    'ccb_launch_count': ('long long', ''),
    'ccb_debug_last_conv_kernel': ('const char*', ''),
    'ccb_debug_tc_plan': (STATUS, 'int, host int*'),
    'ccb_debug_conv_plan': (STATUS, 'const ccb_conv_desc*, int, host int*'),
}

_SCALARS = {'int': C.c_int, 'long long': C.c_longlong, 'float': C.c_float, 'double': C.c_double}
_DTYPES = {'float': torch.float32, 'double': torch.float64, 'int': torch.int32, 'long long': torch.int64,
           'unsigned long long': torch.int64, 'unsigned char': torch.uint8, 'unsigned short': torch.uint16, 'void': None}
_RESTYPES = {STATUS: C.c_int, 'int': C.c_int, 'long long': C.c_longlong, 'void*': C.c_void_p, 'const char*': C.c_char_p,
             'void': None}


def _where(name, pos):
    return name if pos is None else '%s argument %d' % (name, pos)


def ptr(t, name='tensor', dtype=torch.float32, pos=None):
    """Device pointer of a contiguous tensor of `dtype` (fp32 unless stated; None: any dtype; t None -> NULL).
    `pos`: the position of the argument of entry point `name` that `t` is for (error messages)."""
    if t is None:
        return None
    if dtype is not None and t.dtype != dtype:
        raise TypeError('cc_b200: %s must be %s, got %s' % (_where(name, pos), dtype, t.dtype))
    if not t.is_contiguous():
        raise ValueError('cc_b200: %s must be contiguous' % _where(name, pos))
    if not t.is_cuda and not is_simulator():
        raise RuntimeError('cc_b200: %s is on %s - the sm_90a kernels need CUDA tensors (no CPU fallback)'
                           % (_where(name, pos), t.device))
    return t.data_ptr()


def stream(t=None):
    """The current stream of tensor `t`'s device (NULL for a CPU tensor: the simulator)."""
    if t is not None and t.is_cuda:
        return torch.cuda.current_stream(t.device).cuda_stream
    return None


def _param(decl):
    """(ctypes argtype, conversion (arg, entry point, position) -> ctypes value, None: as it is) of a declared parameter."""
    if decl in _SCALARS:
        return _SCALARS[decl], None
    if decl == 'ccb_stream_t':
        return C.c_void_p, lambda t, name, pos: stream(t)
    if decl == 'handle void*':
        return C.c_void_p, None
    if decl == 'float* const*':             # host array of device pointers, given as a list of fp32 tensors
        return C.POINTER(C.c_void_p), lambda ts, name, pos: (C.c_void_p * len(ts))(*[ptr(t, name, pos=pos) for t in ts])
    base = decl.replace('const ', '').rstrip('*')
    if base.startswith('host '):            # host array: an input given as a list of values, an output as a ctypes array
        ct = _SCALARS[base[len('host '):]]
        if 'const ' in decl:
            return C.POINTER(ct), lambda a, name, pos: (ct * len(a))(*a)
        return C.POINTER(ct), None
    if base in STRUCTS:
        return C.POINTER(STRUCTS[base]), lambda d, name, pos: C.byref(d)
    dtype = _DTYPES[base]
    return C.c_void_p, lambda t, name, pos: ptr(t, name, dtype, pos)


_CALLS = {name: (ret, [_param(p) for p in params.split(', ') if p]) for name, (ret, params) in _SIGS.items()}


def _bind(lib):
    for name, (ret, params) in _CALLS.items():
        fn = getattr(lib, name)          # AttributeError => header/library mismatch: fail loudly
        fn.restype = _RESTYPES[ret]
        fn.argtypes = [argtype for argtype, _ in params]


def call(name, *args):
    """Entry point `name` on `args`, each converted as its parameter is declared: a tensor -> device pointer (checked like
    ptr()), None -> NULL, a list of tensors -> host array of their pointers, a descriptor -> byref, and in the stream
    slot a tensor -> its device's current stream.  A non-zero status raises RuntimeError.  The function is looked up
    on every call and called with positional arguments (tools swap lib() for a proxy that times the calls)."""
    ret, params = _CALLS[name]
    if len(args) != len(params):
        raise TypeError('cc_b200: %s takes %d arguments, got %d' % (name, len(params), len(args)))
    fn = getattr(lib(), name)
    rc = fn(*[a if conv is None else conv(a, name, i) for i, ((_, conv), a) in enumerate(zip(params, args))])
    if ret == STATUS:
        check(rc, name)
    return rc


def check(rc, what=''):
    """Raise RuntimeError for a non-zero ccb_status `rc` of entry point `what`, with ccb_last_error_string()."""
    if rc != 0:
        msg = lib().ccb_last_error_string()
        raise RuntimeError('libccb200 %s failed (status %d): %s' % (what, rc, msg.decode() if msg else ''))


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


def device():
    """The device the library's kernels run on: the CPU for the simulator build, else the current CUDA device."""
    return torch.device('cpu') if is_simulator() else torch.device('cuda')


def workspace(query, *args, like):
    """(scratch buffer, its size) for the entry point whose size query `query` is, called on `args`: fp32 for a
    `*_floats` query, uint8 for `*_bytes`, on `like`'s device; (None, 0) where nothing is needed.  A query's -1
    (invalid sizes) raises."""
    n = call(query, *args)
    if n < 0:
        raise RuntimeError('cc_b200: %s returned -1: invalid sizes' % query)
    dtype = torch.float32 if query.endswith('_floats') else torch.uint8
    return (torch.empty(n, dtype=dtype, device=like.device) if n else None), n


def scatter_workspace(t):
    """(fixed-point accumulators, their size in words) for the image gradient of a warp of `t` (ccb_flow_warp_bwd /
    ccb_featwarp_bwd): the gradient's element count + 1, as include/ccb200.h states."""
    n = t.numel() + 1
    return torch.empty(n, dtype=torch.int64, device=t.device), n


def f32(t):
    """`t` detached, as contiguous fp32: how every op hands a tensor to the kernels."""
    return t.detach().float().contiguous()
