"""ctypes binding of libnlt_b200.so (the C ABI declared in include/nlt_b200.h).

The product path has NO CPU fallback: if the shared library is missing or a
tensor is not a CUDA fp32 contiguous tensor, this module raises.
"""
import contextlib
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'csrc', 'libnlt_b200.so')
NLT_MAX_SEG = 4

ACT_CODES = {None: 0, 'none': 0, 'relu': 1, 'leakyrelu': 2, 'elu': 3}


class GConvDesc(C.Structure):
    _fields_ = [
        ('N', C.c_int32), ('Hin', C.c_int32), ('Win', C.c_int32),
        ('Hout', C.c_int32), ('Wout', C.c_int32),
        ('kh', C.c_int32), ('kw', C.c_int32), ('stride', C.c_int32),
        ('pad_t', C.c_int32), ('pad_l', C.c_int32),
        ('transposed', C.c_int32), ('nseg', C.c_int32),
        ('seg_ptr', C.c_void_p * NLT_MAX_SEG),
        ('seg_sub', C.c_void_p * NLT_MAX_SEG),
        ('seg_C', C.c_int32 * NLT_MAX_SEG),
        ('seg_bcast', C.c_int32 * NLT_MAX_SEG),
        ('Cout', C.c_int32),
        ('w', C.c_void_p),
        ('w_tap_stride', C.c_int64), ('w_c_stride', C.c_int64),
        ('w_n_stride', C.c_int64),
    ]


class PwTerm(C.Structure):
    """nlt_pw_term (include/nlt_b200.h): pointwise term fused into a pointwise op's epilogue."""
    _fields_ = [('x', C.c_void_p), ('K', C.c_int32), ('w', C.c_void_p),
                ('w_k_stride', C.c_int64), ('w_n_stride', C.c_int64)]


class LpipsWeights(C.Structure):
    """nlt_lpips_weights (include/nlt_b200.h): device pointers to the LPIPS AlexNet constants."""
    _fields_ = [('scale', C.c_void_p), ('shift', C.c_void_p), ('w', C.c_void_p * 5), ('b', C.c_void_p * 5),
                ('lin', C.c_void_p * 5)]


class NativeError(RuntimeError):
    pass


_lib = None

_SIGS = {
    'nlt_version': (C.c_char_p, []),
    'nlt_last_error': (C.c_char_p, []),
    'nlt_set_option': (C.c_int, [C.c_char_p, C.c_int]),
    'nlt_get_option': (C.c_int, [C.c_char_p, C.POINTER(C.c_int)]),
    'nlt_launch_count': (C.c_uint64, []),
    'nlt_tc_launch_count': (C.c_uint64, []),
    'nlt_kernel_launch_count': (C.c_uint64, [C.c_char_p]),
    'nlt_gconv_fwd': (C.c_int, [C.POINTER(GConvDesc), C.c_void_p, C.c_int, C.c_float, C.c_void_p, C.c_int,
                                C.c_void_p, C.c_void_p]),
    'nlt_gconv_fwd_fused_supported': (C.c_int, [C.POINTER(GConvDesc), C.POINTER(PwTerm), C.c_void_p, C.c_void_p]),
    'nlt_gconv_fwd_fused': (C.c_int, [C.POINTER(GConvDesc), C.POINTER(PwTerm), C.c_void_p, C.c_int, C.c_float,
                                      C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    'nlt_gconv_fwd_workspace_bytes': (C.c_int64, [C.POINTER(GConvDesc)]),
    'nlt_gconv_fwd_ws': (C.c_int, [C.POINTER(GConvDesc), C.c_void_p, C.c_int, C.c_float, C.c_void_p, C.c_int,
                                   C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    'nlt_gconv_fwd_pack_bytes': (C.c_int64, [C.POINTER(GConvDesc), C.c_float, C.c_int]),
    'nlt_gconv_pack_weights': (C.c_int, [C.POINTER(GConvDesc), C.c_void_p, C.c_int64, C.c_void_p]),
    'nlt_gconv_fwd_packed': (C.c_int, [C.POINTER(GConvDesc), C.c_void_p, C.c_int, C.c_float, C.c_void_p, C.c_int,
                                       C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    'nlt_gconv_wgrad_workspace_bytes': (C.c_int64, [C.POINTER(GConvDesc)]),
    'nlt_gconv_wgrad': (C.c_int, [C.POINTER(GConvDesc), C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                  C.c_int64, C.c_void_p]),
    'nlt_barron_loss_workspace_bytes': (C.c_int64, [C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    'nlt_barron_loss': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                  C.c_float, C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    'nlt_kmean_fwd': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p]),
    'nlt_kmean_bwd': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int64, C.c_float, C.c_void_p,
                                C.c_int, C.c_void_p, C.c_void_p]),
    'nlt_uv2cam_fwd': (C.c_int, [C.c_void_p] * 4 + [C.c_int32] * 6 + [C.c_void_p] * 6),
    'nlt_uv2cam_bwd': (C.c_int, [C.c_void_p] * 2 + [C.c_int32] * 5 + [C.c_void_p] * 2),
    'nlt_uv2cam_bwd_workspace_bytes': (C.c_int64, [C.c_int32] * 3),
    'nlt_uv2cam_bwd_det': (C.c_int, [C.c_void_p] * 2 + [C.c_int32] * 5 + [C.c_void_p] * 3),
    'nlt_resize_bilinear_fwd': (C.c_int, [C.c_void_p] + [C.c_int32] * 6 + [C.c_void_p] * 2),
    'nlt_resize_bilinear_bwd': (C.c_int, [C.c_void_p] + [C.c_int32] * 6 + [C.c_void_p] * 2),
    'nlt_l2_loss_workspace_bytes': (C.c_int64, [C.c_int32, C.c_int64]),
    'nlt_l2_loss': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_float, C.c_void_p, C.c_void_p,
                              C.c_void_p, C.c_void_p]),
    'nlt_l1_loss_workspace_bytes': (C.c_int64, [C.c_int32, C.c_int64]),
    'nlt_l1_loss': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_float, C.c_void_p, C.c_void_p,
                              C.c_void_p, C.c_void_p]),
    'nlt_ssim_loss_workspace_bytes': (C.c_int64, [C.c_int32] * 3),
    'nlt_ssim_loss': (C.c_int, [C.c_void_p, C.c_void_p] + [C.c_int32] * 3 + [C.c_float] * 2 + [C.c_void_p] * 4),
    'nlt_lpips_loss_workspace_bytes': (C.c_int64, [C.c_int32] * 3),
    'nlt_lpips_loss': (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(LpipsWeights)] + [C.c_int32] * 3
                       + [C.c_float] + [C.c_void_p] * 3 + [C.c_int64, C.c_void_p]),
    'nlt_amsgrad_step': (C.c_int, [C.c_void_p] * 5 + [C.c_int64, C.c_int32] + [C.c_float] * 5 + [C.c_void_p]),
    'nlt_amsgrad_step_dev': (C.c_int, [C.c_void_p] * 5 + [C.c_int64, C.c_void_p] + [C.c_float] * 5 + [C.c_void_p]),
    'nlt_pixelnorm_fwd': (C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_int, C.c_void_p, C.c_void_p]),
    'nlt_pixelnorm_bwd': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p]),
    'nlt_instnorm_workspace_bytes': (C.c_int64, [C.c_int32] * 3),
    'nlt_instnorm_fwd': (C.c_int, [C.c_void_p] * 3 + [C.c_int32] * 3 + [C.c_int, C.c_float] + [C.c_void_p] * 5),
    'nlt_instnorm_bwd': (C.c_int, [C.c_void_p] * 5 + [C.c_int32] * 3 + [C.c_void_p] * 3 + [C.c_int] + [C.c_void_p] * 2),
    'nlt_pool2x2_fwd': (C.c_int, [C.c_void_p] + [C.c_int32] * 4 + [C.c_int, C.c_void_p, C.c_void_p]),
    'nlt_pool2x2_bwd': (C.c_int, [C.c_void_p] * 2 + [C.c_int32] * 4 + [C.c_int, C.c_float, C.c_void_p, C.c_int]
                        + [C.c_void_p] * 2),
    'nlt_upsample2x_bilinear_fwd': (C.c_int, [C.c_void_p] + [C.c_int32] * 4 + [C.c_void_p] * 2),
    'nlt_upsample2x_bilinear_bwd': (C.c_int, [C.c_void_p] + [C.c_int32] * 4 + [C.c_float, C.c_void_p, C.c_int]
                                    + [C.c_void_p] * 2),
    'nlt_u8_to_f32': (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    'nlt_ksum_acc': (C.c_int, [C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p]),
    'nlt_scale': (C.c_int, [C.c_void_p, C.c_int64, C.c_float, C.c_void_p]),
    'nlt_mul': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
}


def exported_symbols():
    """Names every build of the library must export (tests check this)."""
    return sorted(_SIGS)


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise NativeError(
                'CUDA extension %s is missing; run `python -c "import __graft_entry__ as g; g.build()"` '
                '(there is no CPU fallback)' % LIB_PATH)
        handle = C.CDLL(LIB_PATH)
        for name, (res, args) in _SIGS.items():
            fn = getattr(handle, name)
            fn.restype = res
            fn.argtypes = args
        _lib = handle
    return _lib


def check(rc):
    if rc != 0:
        raise NativeError('nlt_b200 error %d: %s' % (rc, lib().nlt_last_error().decode()))


def ptr(t):
    """Device pointer of a CUDA fp32 contiguous tensor (None -> NULL)."""
    if t is None:
        return None
    if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()):
        raise NativeError('expected a contiguous CUDA float32 tensor, got %s %s contiguous=%s' % (
            t.device, t.dtype, t.is_contiguous()))
    return t.data_ptr()


def stream():
    return torch.cuda.current_stream().cuda_stream


def launch_count():
    """Kernels launched by the library so far (bench.py's gpu_launches)."""
    return int(lib().nlt_launch_count())


def kernel_launch_count(name):
    """Launches of the kernel the library reports as `name` so far."""
    return int(lib().nlt_kernel_launch_count(name.encode()))


def tc_launch_count():
    """wgmma tensor-core kernel launches so far."""
    return int(lib().nlt_tc_launch_count())


def set_option(name, value):
    """Sets a process-wide kernel switch (the option table of csrc/nlt_gconv.cu), e.g. 'tc': 1 = wgmma 3xTF32 kernels
    where eligible (default), 0 = fp32-FMA kernels only."""
    check(lib().nlt_set_option(name.encode(), int(value)))


def get_option(name):
    """Current value of a kernel switch: what set_option stored, else its environment value or default."""
    v = C.c_int()
    check(lib().nlt_get_option(name.encode(), C.byref(v)))
    return v.value


@contextlib.contextmanager
def options(**kv):
    """Sets the named switches for the duration of the block and restores their previous values on exit."""
    saved = {k: get_option(k) for k in kv}
    try:
        for k, v in kv.items():
            set_option(k, v)
        yield
    finally:
        for k, v in saved.items():
            set_option(k, v)
