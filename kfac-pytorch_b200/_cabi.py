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
KFAC_EKFAC_KEEP, KFAC_EKFAC_EMA, KFAC_EKFAC_RESET, KFAC_EKFAC_SEED = 0, 1, 2, 3

KFAC_EIGH_MAX_N = 8192   # largest factor dimension the eigensolver takes

KFAC_ITEM_DENSE, KFAC_ITEM_EMBEDDING, KFAC_ITEM_DIAG_G, KFAC_ITEM_TIED, KFAC_ITEM_DIAG_A = 0, 1, 2, 3, 4

DTYPE_CODE = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}
INDEX_DTYPE_CODE = {torch.int32: 3, torch.int64: 4}
KFAC_BAG_SUM, KFAC_BAG_MEAN = 0, 1


class ConvGeometry(C.Structure):
    """kfac_conv_geometry: every per-axis array in (D, H, W) order."""
    _fields_ = [('batch', c_int), ('C', c_int), ('input', c_int * 3), ('kernel', c_int * 3), ('stride', c_int * 3),
                ('dilation', c_int * 3), ('pad_before', c_int * 3), ('pad_after', c_int * 3)]


class ConvTransposeGeometry(C.Structure):
    """kfac_conv_transpose_geometry: torch's parameters of a transposed convolution, every per-axis array in (D, H, W)
    order."""
    _fields_ = [('batch', c_int), ('C', c_int), ('input', c_int * 3), ('kernel', c_int * 3), ('stride', c_int * 3),
                ('dilation', c_int * 3), ('padding', c_int * 3), ('output_padding', c_int * 3)]


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
                ('peer_P', C.POINTER(c_void_p)), ('n_peers', c_int), ('kind', c_int),
                ('dh', c_void_p), ('tied_damping', c_float), ('wgrad_taps', c_int), ('pi', c_void_p)]


class PiItem(C.Structure):
    """kfac_pi_item: the factors of one layer (ld 0: a vector factor) and its pi slot."""
    _fields_ = [('A', c_void_p), ('G', c_void_p), ('pi', c_void_p), ('a', c_int), ('g', c_int), ('lda', c_int),
                ('ldg', c_int)]


class TiedItem(C.Structure):
    _fields_ = [('Q', c_void_p), ('QT', c_void_p), ('e', c_void_p), ('H', c_void_p), ('C', c_void_p),
                ('UT', c_void_p), ('M', c_void_p), ('MT', c_void_p), ('d', c_int), ('ld', c_int)]


KFAC_NORM_BATCH, KFAC_NORM_LAYER, KFAC_NORM_RMS = 0, 1, 2
# GroupNorm / InstanceNorm*: the statistics of kfac_factor_group_norm (not a kind kfac_factor_norm takes)
KFAC_NORM_GROUP = 3


class NormItem(C.Structure):
    _fields_ = [('F', c_void_p), ('wgrad', c_void_p), ('bgrad', c_void_p), ('grad_dtype', c_int),
                ('C', c_int), ('k', c_int), ('P', c_void_p)]


class GradItem(C.Structure):
    _fields_ = [('P', c_void_p), ('wgrad', c_void_p), ('bgrad', c_void_p),
                ('grad_dtype', c_int), ('g', c_int), ('a', c_int), ('ldp', c_int), ('wgrad_taps', c_int)]


class SequenceRows(C.Structure):
    """kfac_sequence_rows: the source rows of a recurrent sub-layer's positions (time-major or packed)."""
    _fields_ = [('x', c_void_p), ('ldx', c_int64), ('col0', c_int),
                ('h0', c_void_p), ('ldh', c_int64), ('shift', c_int),
                ('mul', c_void_p), ('ldm', c_int64), ('mul_col0', c_int),
                ('T', c_int), ('B', c_int), ('offsets', c_void_p)]


class EkfacStatItem(C.Structure):
    _fields_ = [('X', c_void_p), ('G', c_void_p), ('qaT', c_void_p), ('qgT', c_void_p), ('S_batch', c_void_p),
                ('N', c_int64), ('a', c_int), ('g', c_int),
                ('ldx', c_int), ('ldg', c_int), ('ldqa', c_int), ('ldqg', c_int), ('lds', c_int)]


class EkfacUpdateItem(C.Structure):
    _fields_ = [('S', c_void_p), ('S_batch', c_void_p), ('dg', c_void_p), ('da', c_void_p), ('dgda', c_void_p),
                ('g', c_int), ('a', c_int), ('ld', c_int), ('drop_a', c_void_p), ('drop_g', c_void_p)]


# name -> (restype, argtypes); must list EVERY symbol of include/kfac_b200.h
SIGNATURES = {
    'kfac_version': (c_int, []),
    'kfac_last_error': (C.c_char_p, []),
    'kfac_device_arch': (c_int, []),
    'kfac_launch_count': (C.c_longlong, []),
    'kfac_factor_linear_workspace_bytes': (c_size_t, [c_int64, c_int, c_int]),
    'kfac_factor_linear': (c_int, [c_void_p, c_int, c_int64, c_int, c_int, c_float, c_void_p, c_void_p, c_size_t, c_void_p]),
    'kfac_factor_linear_strided_workspace_bytes': (c_size_t, [c_int64, c_int, c_int64, c_int]),
    'kfac_factor_linear_strided': (c_int, [c_void_p, c_int, c_int64, c_int, c_int64, c_int, c_float, c_void_p, c_void_p,
                                           c_size_t, c_void_p]),
    'kfac_factor_conv2d_input_workspace_bytes': (c_size_t, [c_int] * 11),
    'kfac_factor_conv2d_input': (c_int, [c_void_p, c_int] + [c_int] * 11 + [c_float, c_void_p, c_void_p, c_size_t, c_void_p]),
    'kfac_factor_conv_input_workspace_bytes': (c_size_t, [C.POINTER(ConvGeometry), c_int, c_size_t]),
    'kfac_factor_conv_input': (c_int, [c_void_p, c_int, C.POINTER(ConvGeometry), c_int, c_float, c_void_p, c_void_p,
                                       c_size_t, c_void_p]),
    'kfac_factor_conv_transpose_input_workspace_bytes': (c_size_t, [C.POINTER(ConvTransposeGeometry), c_int, c_size_t]),
    'kfac_factor_conv_transpose_input': (c_int, [c_void_p, c_int, C.POINTER(ConvTransposeGeometry), c_int, c_float,
                                                 c_void_p, c_void_p, c_size_t, c_void_p]),
    'kfac_factor_conv2d_gradout_workspace_bytes': (c_size_t, [c_int, c_int, c_int, c_int]),
    'kfac_factor_conv2d_gradout': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p, c_void_p, c_size_t, c_void_p]),
    'kfac_factor_ema': (c_int, [C.POINTER(EmaItem), c_int, c_float, c_void_p]),
    'kfac_factor_ema_guarded_workspace_bytes': (c_size_t, [c_int]),
    'kfac_factor_ema_guarded': (c_int, [C.POINTER(EmaItem), c_int, c_float, C.POINTER(c_void_p), c_void_p,
                                        c_void_p, c_size_t, c_void_p]),
    'kfac_factor_embedding_workspace_bytes': (c_size_t, [c_int]),
    'kfac_factor_embedding': (c_int, [c_void_p, c_int, c_int64, c_int, c_float, c_void_p, c_void_p, c_size_t,
                                      c_void_p]),
    'kfac_factor_embedding_bag_workspace_bytes': (c_size_t, [c_int64, c_int64, c_int]),
    'kfac_factor_embedding_bag': (c_int, [c_void_p, c_void_p, c_int, c_int64, c_int64, c_int64, c_int, c_void_p, c_int,
                                          c_int, c_float, c_void_p, c_void_p, c_size_t, c_void_p]),
    'kfac_factor_ema_diag': (c_int, [C.POINTER(EmaItem), c_int, c_float, c_void_p]),
    'kfac_factor_ema_diag_guarded_workspace_bytes': (c_size_t, [c_int]),
    'kfac_factor_ema_diag_guarded': (c_int, [C.POINTER(EmaItem), c_int, c_float, C.POINTER(c_void_p), c_void_p,
                                             c_void_p, c_size_t, c_void_p]),
    'kfac_factor_linear_diag_workspace_bytes': (c_size_t, [c_int64, c_int]),
    'kfac_factor_linear_diag': (c_int, [c_void_p, c_int, c_int64, c_int, c_float, c_void_p, c_void_p, c_size_t,
                                        c_void_p]),
    'kfac_factor_linear_diag_ones': (c_int, [c_void_p, c_int, c_int64, c_int, c_int, c_float, c_void_p, c_void_p,
                                             c_size_t, c_void_p]),
    'kfac_factor_conv_input_diag_workspace_bytes': (c_size_t, [C.POINTER(ConvGeometry)]),
    'kfac_factor_conv_input_diag': (c_int, [c_void_p, c_int, C.POINTER(ConvGeometry), c_int, c_float, c_void_p,
                                            c_void_p, c_size_t, c_void_p]),
    'kfac_diag_snapshot': (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    'kfac_factor_norm_workspace_bytes': (c_size_t, [c_int, c_int64, c_int, c_int64]),
    'kfac_factor_norm': (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int64, c_int, c_int64, c_int, C.c_double,
                                 c_float, c_void_p, c_void_p, c_size_t, c_void_p]),
    'kfac_factor_group_norm_workspace_bytes': (c_size_t, [c_int64, c_int, c_int64, c_int]),
    'kfac_factor_group_norm': (c_int, [c_void_p, c_int, c_void_p, c_int, c_int64, c_int, c_int64, c_int, c_int,
                                       C.c_double, c_float, c_void_p, c_void_p, c_size_t, c_void_p]),
    'kfac_norm_precondition_workspace_bytes': (c_size_t, [c_int]),
    'kfac_norm_precondition': (c_int, [C.POINTER(NormItem), c_int, c_float, c_void_p, c_size_t, c_void_p]),
    'kfac_eigh_workspace_bytes': (c_size_t, [C.POINTER(c_int), c_int]),
    'kfac_eigh_batched': (c_int, [C.POINTER(EighItem), c_int, c_void_p, c_size_t, c_int, c_float, c_void_p]),
    'kfac_eigh_status': (c_int, [c_void_p, c_void_p, c_void_p]),
    'kfac_dgda': (c_int, [c_void_p, c_void_p, c_int, c_int, c_float, c_void_p, c_int, c_void_p]),
    'kfac_inverse_from_eigh': (c_int, [c_void_p, c_int, c_void_p, c_int, c_float, c_void_p, c_int, c_void_p, c_size_t, c_void_p]),
    'kfac_pi': (c_int, [C.POINTER(PiItem), c_int, c_void_p]),
    'kfac_dgda_pi': (c_int, [c_void_p, c_void_p, c_int, c_int, c_float, c_void_p, c_void_p, c_int, c_void_p]),
    'kfac_inverse_from_eigh_pi': (c_int, [c_void_p, c_int, c_void_p, c_int, c_float, c_void_p, c_int, c_void_p, c_int,
                                          c_void_p, c_size_t, c_void_p]),
    'kfac_transpose': (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_void_p]),
    'kfac_precondition_workspace_bytes': (c_size_t, [C.POINTER(PrecondItem), c_int]),
    'kfac_precondition': (c_int, [C.POINTER(PrecondItem), c_int, c_int, c_float, c_void_p, c_size_t, c_void_p]),
    'kfac_tied_workspace_bytes': (c_size_t, [C.POINTER(TiedItem), c_int]),
    'kfac_tied_whiten': (c_int, [C.POINTER(TiedItem), c_int, c_float, c_void_p, c_size_t, c_void_p]),
    'kfac_tied_basis': (c_int, [C.POINTER(TiedItem), c_int, c_float, c_void_p, c_size_t, c_void_p]),
    'kfac_grad_workspace_bytes': (c_size_t, [c_int]),
    'kfac_grad_scale': (c_int, [C.POINTER(GradItem), c_int, c_float, c_float, c_void_p, c_size_t, c_void_p, c_void_p]),
    'kfac_grad_update': (c_int, [C.POINTER(GradItem), c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
    'kfac_rows_linear': (c_int, [c_void_p, c_int, c_int64, c_int, c_int, c_float, c_void_p, c_void_p, c_int, c_void_p]),
    'kfac_rows_linear_strided': (c_int, [c_void_p, c_int, c_int64, c_int, c_int64, c_int, c_float, c_void_p, c_void_p,
                                         c_int, c_void_p]),
    'kfac_rows_conv2d_input': (c_int, [c_void_p, c_int] + [c_int] * 11 + [c_float, c_void_p, c_int, c_void_p]),
    'kfac_rows_conv_input': (c_int, [c_void_p, c_int, C.POINTER(ConvGeometry), c_int, c_float, c_void_p, c_int,
                                     c_void_p]),
    'kfac_rows_conv_transpose_input': (c_int, [c_void_p, c_int, C.POINTER(ConvTransposeGeometry), c_int, c_float,
                                               c_void_p, c_int, c_void_p]),
    'kfac_rows_conv2d_gradout': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p, c_void_p, c_int,
                                         c_void_p]),
    'kfac_reduce_rows_linear': (c_int, [c_void_p, c_int, c_int64, c_int64, c_int, c_int, c_float, c_void_p, c_void_p,
                                        c_int, c_void_p]),
    'kfac_reduce_rows_linear_strided': (c_int, [c_void_p, c_int, c_int64, c_int64, c_int, c_int64, c_int64, c_int,
                                                c_float, c_void_p, c_void_p, c_int, c_void_p]),
    'kfac_reduce_rows_conv2d_input': (c_int, [c_void_p, c_int] + [c_int] * 11 + [c_float, c_void_p, c_int, c_void_p]),
    'kfac_reduce_rows_conv_input': (c_int, [c_void_p, c_int, C.POINTER(ConvGeometry), c_int, c_float, c_void_p, c_int,
                                            c_void_p]),
    'kfac_reduce_rows_conv_transpose_input': (c_int, [c_void_p, c_int, C.POINTER(ConvTransposeGeometry), c_int,
                                                      c_float, c_void_p, c_int, c_void_p]),
    'kfac_reduce_rows_conv2d_gradout': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p,
                                                c_void_p, c_int, c_void_p]),
    'kfac_rows_sequence': (c_int, [C.POINTER(SequenceRows), c_int, c_int, c_int, c_float, c_void_p, c_void_p, c_int,
                                   c_void_p]),
    'kfac_reduce_rows_sequence': (c_int, [C.POINTER(SequenceRows), c_int, c_int, c_int, c_float, c_float, c_void_p,
                                          c_void_p, c_int, c_void_p]),
    'kfac_ekfac_statistics_workspace_bytes': (c_size_t, [C.POINTER(EkfacStatItem), c_int]),
    'kfac_ekfac_statistics': (c_int, [C.POINTER(EkfacStatItem), c_int, c_void_p, c_size_t, c_void_p]),
    'kfac_ekfac_update_workspace_bytes': (c_size_t, [c_int]),
    'kfac_ekfac_update': (c_int, [C.POINTER(EkfacUpdateItem), c_int, c_float, c_int, c_float, c_void_p, c_void_p,
                                  c_size_t, c_void_p]),
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
