"""ctypes binding of libkfac_b200.so (C ABI declared in include/kfac_b200.h).

There is NO CPU fallback: if the shared library is missing this module raises
at import of the symbols, and every compute entry point raises if no sm_90
device is current.
"""
from __future__ import annotations

import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'csrc', 'libkfac_b200.so')

c_void_p, c_int, c_float, c_size_t, c_int64 = C.c_void_p, C.c_int, C.c_float, C.c_size_t, C.c_int64

KFAC_OK, KFAC_ERR_BAD_ARG, KFAC_ERR_NOT_READY, KFAC_ERR_CUDA = 0, -1, -2, -3
KFAC_ERR_WORKSPACE, KFAC_ERR_NO_CONVERGE, KFAC_ERR_UNSUPPORTED = -4, -5, -6
KFAC_EIGEN, KFAC_INVERSE = 1, 2

DTYPE_CODE = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}


class EmaItem(C.Structure):
    _fields_ = [('factor', c_void_p), ('batch', c_void_p), ('d', c_int),
                ('first', c_int), ('inv_count', c_float)]


class EighItem(C.Structure):
    _fields_ = [('F', c_void_p), ('Q', c_void_p), ('QT', c_void_p), ('d', c_void_p), ('n', c_int), ('ldq', c_int), ('V0T', c_void_p)]


class PrecondItem(C.Structure):
    _fields_ = [('wgrad', c_void_p), ('bgrad', c_void_p), ('grad_dtype', c_int),
                ('g', c_int), ('a', c_int),
                ('qa', c_void_p), ('qaT', c_void_p), ('qg', c_void_p), ('qgT', c_void_p),
                ('dgda', c_void_p), ('da', c_void_p), ('dg', c_void_p),
                ('a_inv', c_void_p), ('g_inv', c_void_p),
                ('ldqa', c_int), ('ldqg', c_int), ('ld_dgda', c_int),
                ('P', c_void_p), ('ldp', c_int),
                ('peer_P', C.POINTER(c_void_p)), ('n_peers', c_int)]


class GradItem(C.Structure):
    _fields_ = [('P', c_void_p), ('wgrad', c_void_p), ('bgrad', c_void_p),
                ('grad_dtype', c_int), ('g', c_int), ('a', c_int), ('ldp', c_int)]


# name -> (restype, argtypes); must list EVERY symbol of include/kfac_b200.h
SIGNATURES = {
    'kfac_version': (c_int, []),
    'kfac_last_error': (C.c_char_p, []),
    'kfac_device_arch': (c_int, []),
    'kfac_launch_count': (C.c_longlong, []),
    'kfac_factor_linear_workspace_bytes': (c_size_t, [c_int64, c_int, c_int]),
    'kfac_factor_linear': (c_int, [c_void_p, c_int, c_int64, c_int, c_int, c_float, c_void_p, c_void_p, c_size_t, c_void_p]),
    'kfac_factor_conv2d_input_workspace_bytes': (c_size_t, [c_int] * 11),
    'kfac_factor_conv2d_input': (c_int, [c_void_p, c_int] + [c_int] * 11 + [c_float, c_void_p, c_void_p, c_size_t, c_void_p]),
    'kfac_factor_conv2d_gradout_workspace_bytes': (c_size_t, [c_int, c_int, c_int, c_int]),
    'kfac_factor_conv2d_gradout': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p, c_void_p, c_size_t, c_void_p]),
    'kfac_factor_ema': (c_int, [C.POINTER(EmaItem), c_int, c_float, c_void_p]),
    'kfac_eigh_workspace_bytes': (c_size_t, [C.POINTER(c_int), c_int]),
    'kfac_eigh_batched': (c_int, [C.POINTER(EighItem), c_int, c_void_p, c_size_t, c_int, c_float, c_void_p]),
    'kfac_eigh_status': (c_int, [c_void_p, c_void_p, c_void_p]),
    'kfac_dgda': (c_int, [c_void_p, c_void_p, c_int, c_int, c_float, c_void_p, c_int, c_void_p]),
    'kfac_inverse_from_eigh': (c_int, [c_void_p, c_int, c_void_p, c_int, c_float, c_void_p, c_int, c_void_p, c_size_t, c_void_p]),
    'kfac_transpose': (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_void_p]),
    'kfac_precondition_workspace_bytes': (c_size_t, [C.POINTER(PrecondItem), c_int]),
    'kfac_precondition': (c_int, [C.POINTER(PrecondItem), c_int, c_int, c_float, c_void_p, c_size_t, c_void_p]),
    'kfac_grad_workspace_bytes': (c_size_t, [c_int]),
    'kfac_grad_scale': (c_int, [C.POINTER(GradItem), c_int, c_float, c_float, c_void_p, c_size_t, c_void_p, c_void_p]),
    'kfac_grad_update': (c_int, [C.POINTER(GradItem), c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
    'kfac_peer_alloc': (c_int, [c_size_t, C.POINTER(c_void_p), c_void_p]),
    'kfac_peer_open': (c_int, [c_void_p, C.POINTER(c_void_p)]),
    'kfac_peer_close': (c_int, [c_void_p]),
    'kfac_peer_free': (c_int, [c_void_p]),
    'kfac_triu_pack': (c_int, [c_void_p, c_int, c_void_p, c_void_p]),
    'kfac_triu_unpack': (c_int, [c_void_p, c_int, c_void_p, c_void_p]),
    'kfac_scale_inplace': (c_int, [c_void_p, c_int64, c_float, c_void_p]),
    'kfac_gemm_tn_tc': (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_int64, c_int, c_int, c_int,
                                c_float, c_int, c_int, c_void_p]),
    'kfac_gemm_f32': (c_int, [c_void_p, c_int64, c_int64, c_void_p, c_int64, c_int64, c_void_p, c_int64,
                              c_int, c_int, c_int, c_float, c_float, c_void_p]),
}

_lib = None


class KFACNativeError(RuntimeError):
    """The native library is missing or a native call failed."""


def load():
    """Load libkfac_b200.so (loudly) and declare every prototype."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise KFACNativeError(
            f'{LIB_PATH} not found: build it with `python -c "import __graft_entry__ as g; g.build()"` '
            '(nvcc, sm_90a). kfac_b200 has no CPU / PyTorch fallback.')
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is missing
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def last_error() -> str:
    return load().kfac_last_error().decode()


def check(rc: int, what: str = '') -> None:
    """Map kfac_status to the Python exception types of the reference."""
    if rc == KFAC_OK:
        return
    msg = f'{what}: {last_error()}' if what else last_error()
    if rc == KFAC_ERR_BAD_ARG:
        raise ValueError(msg)
    if rc == KFAC_ERR_NOT_READY:
        raise RuntimeError(msg)
    raise KFACNativeError(f'{msg} (status {rc})')


def ld4(n: int) -> int:
    """Leading dimension used for arena matrices: multiple of 4 floats (16 B) so
    TMA tensor maps can address them."""
    return (n + 3) & ~3


def stream_ptr() -> int:
    return torch.cuda.current_stream().cuda_stream


def require_device(t: torch.Tensor) -> None:
    if not t.is_cuda:
        raise KFACNativeError(
            'kfac_b200 runs on CUDA (sm_90a) tensors only; got a tensor on '
            f'{t.device}. There is no CPU fallback.')
