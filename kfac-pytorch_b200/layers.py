"""Module adapters and per-layer K-FAC state.

Mirrors the reference's `ModuleHelper` family (kfac/layers/modules.py:13-237)
and the state carried by `KFACBaseLayer` / `KFACEigenLayer` /
`KFACInverseLayer` (kfac/layers/base.py:19, eigen.py:20, inverse.py:20), but
the layer object here is only a *descriptor*: every tensor it exposes is a view
into a contiguous HBM arena owned by the preconditioner, and all arithmetic
happens in libkfac_b200.so.
"""
from __future__ import annotations

import ctypes as C
import math
import re
from typing import Any, Callable

import torch

from kfac_b200 import _cabi
from kfac_b200.attention import KFACMultiheadAttention
from kfac_b200.recurrent import SWAPPED as RECURRENT_SWAPPED


class FactorRows:
    """The rows one call of a layer forms a factor's statistics of: n rows (B under K-FAC-reduce) of d features.

    write(out_ptr, ld, grad_scale, loss_scale) writes them in fp32 at out_ptr with row stride ld, divided by grad_scale
    and by the device float at loss_scale (or None).  direct(acc, grad_scale, scratch), when given, adds their
    statistics to acc reading the layer's tensor in place (the expand entry points); without it the rows are written
    and the statistics formed of them (ModuleHelper._accumulate_rows).  A slotted class: every factor hook builds one,
    so it is kept cheap to construct."""
    __slots__ = ('n', 'd', 'write', 'direct')

    def __init__(self, n: int, d: int, write: Callable[[int, int, float, int | None], None],
                 direct: Callable[[torch.Tensor, float, Any], None] | None = None) -> None:
        self.n, self.d, self.write, self.direct = n, d, write, direct


class ModuleHelper:
    """Geometry + native dispatch for one supported module type."""

    diagonal_a = False      # True: A is kept as a vector (embeddings; Linear and convolutions in diagonal_a_layers)
    diagonal_g = False      # True: G is approximated by its diagonal and kept as a vector (diagonal_g_layers)
    embedding = False       # True: an nn.Embedding or EmbeddingBag (a diagonal A, its input indices, P is (V, d))
    counts_a = False        # True: A counts the input indices, so it is finite whatever the forward values
    norm = False            # True: exact per-channel Fisher blocks instead of two factors (precondition_norms)
    call_kwargs = False     # True: the A hook passes every call's arguments to bind_call (output_size)
    # 0: the weight gradient is the row-major (g, a - has_bias) gradient matrix; T > 0: it is (C_in, g, T), a transposed
    # convolution's, with grad-matrix element (r, ci * T + t) at [ci, r, t] (kfac_precond_item.wgrad_taps)
    wgrad_taps = 0

    def __init__(self, module: torch.nn.Module, reduce: bool = False, diagonal_a: bool = False):
        self.module = module
        # K-FAC-reduce (kfac_approx='reduce', Linear and Conv2d only): a call with R > 1 shared positions per example
        # forms its statistics from one row per example; R = 1 takes the expand path
        self.reduce = reduce
        # diagonal_a_layers (Linear, Conv2d, Conv1d / Conv3d): A is approximated by diag(A), the diagonal of the dense
        # A of the same rows, kept as a vector of a_dim floats
        self.diagonal_a = diagonal_a or type(self).diagonal_a

    def __repr__(self) -> str:
        return f'{self.__class__.__name__}({repr(self.module)})'

    @property
    def a_factor_shape(self) -> tuple[int, int]:
        raise NotImplementedError

    @property
    def g_factor_shape(self) -> tuple[int, int]:
        raise NotImplementedError

    @property
    def device(self) -> torch.device:
        return next(self.module.parameters()).device

    def has_bias(self) -> bool:
        return getattr(self.module, 'bias', None) is not None

    def has_symmetric_factors(self) -> bool:
        return True

    def get_weight_grad(self) -> torch.Tensor:
        return self.module.weight.grad

    def get_bias_grad(self) -> torch.Tensor:
        return self.module.bias.grad

    def get_grad(self) -> torch.Tensor:
        """(out, in*kh*kw [+1]) gradient matrix; torch glue for inspection /
        tests only -- the hot path reads weight.grad / bias.grad in place."""
        g = self.module.weight.grad.reshape(self.module.weight.grad.size(0), -1)
        if self.has_bias():
            g = torch.cat([g, self.module.bias.grad.view(-1, 1)], 1)
        return g

    def prepare_input(self, x: torch.Tensor) -> torch.Tensor:
        """The tensor accumulate_a, num_rows_a and write_rows_a of one call read, formed once per call."""
        return x

    # the declaration of one call's factor rows: each kind decides here, once per side, between K-FAC-reduce and
    # expand, the row count and the scale of the rows
    def rows_a(self, x: torch.Tensor) -> FactorRows:
        raise NotImplementedError

    def rows_g(self, g: torch.Tensor) -> FactorRows:
        raise NotImplementedError

    # native accumulation of the factor statistics of one micro-batch
    def accumulate_a(self, x: torch.Tensor, acc: torch.Tensor, scratch) -> None:
        rows = self.rows_a(_detached(x))
        if rows.direct is not None:
            rows.direct(acc, 1.0, scratch)
        else:
            self._accumulate_rows(rows, acc, 1.0, scratch, self.diagonal_a)

    def accumulate_g(self, g: torch.Tensor, acc: torch.Tensor, grad_scale: float, scratch) -> None:
        rows = self.rows_g(_detached(g))
        if rows.direct is not None:
            rows.direct(acc, grad_scale, scratch)
        else:
            self._accumulate_rows(rows, acc, grad_scale, scratch, self.diagonal_g)

    # EKFAC row writers: the rows x_r / g_r of one micro-batch (exactly the rows the A / G statistics are formed of),
    # written sample-major in fp32 into `out`, a buffer of at least num_rows_{a,g} x ld4(d) floats
    def num_rows_a(self, x: torch.Tensor) -> int:
        return self.rows_a(x).n

    def num_rows_g(self, g: torch.Tensor) -> int:
        return self.rows_g(g).n

    def write_rows_a(self, x: torch.Tensor, out: torch.Tensor) -> None:
        rows = self.rows_a(_detached(x))
        rows.write(out.data_ptr(), _cabi.ld4(rows.d), 1.0, None)

    def write_rows_g(self, g: torch.Tensor, out: torch.Tensor, grad_scale: float, loss_scale: int | None) -> None:
        """loss_scale: device pointer of a float the rows are divided by (the AMP loss scale), or None."""
        rows = self.rows_g(_detached(g))
        rows.write(out.data_ptr(), _cabi.ld4(rows.d), grad_scale, loss_scale)

    @staticmethod
    def _accumulate_rows(rows: FactorRows, acc: torch.Tensor, grad_scale: float, scratch, diagonal: bool) -> None:
        """acc += the statistics of one call's rows without a direct statistic: the rows written in fp32 (ld = d) at
        the start of the scratch buffer and the Linear statistics call on them at 1 / (n * grad_scale^2) (the column
        sums of squares for a diagonal G)."""
        n, d = rows.n, rows.d
        if n == 0:
            return
        lib = _cabi.load()
        row_bytes = (n * d * 4 + 255) // 256 * 256
        need = (lib.kfac_factor_linear_diag_workspace_bytes(n, d) if diagonal
                else lib.kfac_factor_linear_workspace_bytes(n, d, 0))
        ptr = scratch.get(row_bytes + need, acc.device).data_ptr()
        rows.write(ptr, d, 1.0, None)
        ws = ptr + row_bytes if need else None
        scale = 1.0 / (n * grad_scale * grad_scale)
        f32 = _cabi.DTYPE_CODE[torch.float32]
        if diagonal:
            _cabi.check(lib.kfac_factor_linear_diag(ptr, f32, n, d, scale, acc.data_ptr(), ws, need,
                                                    _cabi.stream_ptr()), 'kfac_factor_linear_diag')
        else:
            _cabi.check(lib.kfac_factor_linear(ptr, f32, n, d, 0, scale, acc.data_ptr(), ws, need, _cabi.stream_ptr()),
                        'kfac_factor_linear')


_NATIVE_INPUT_DTYPES = (torch.float32, torch.float16, torch.bfloat16)


def cast_for_factor(t: torch.Tensor, factor_dtype: torch.dtype | None) -> torch.Tensor:
    """The reference casts the activation / grad-output to `factor_dtype` before the statistics are formed
    (kfac/layers/base.py:350,364).  Here the statistics are always ACCUMULATED and STORED in float32:
      * float16 / bfloat16: the input is rounded to that dtype (same input rounding as the reference),
        the products are accumulated in fp32 (at least as accurate as the reference's half GEMM);
      * float32 / float64 / None: the input is used as is (float64 inputs are cast to float32 at the
        boundary -- the native library has no fp64 path; documented deviation)."""
    if factor_dtype in (torch.float16, torch.bfloat16) and t.dtype != factor_dtype:
        t = t.to(factor_dtype)
    if t.dtype not in _NATIVE_INPUT_DTYPES:
        t = t.to(torch.float32)
    return t


def _dtype_code(t: torch.Tensor) -> int:
    try:
        return _cabi.DTYPE_CODE[t.dtype]
    except KeyError:
        raise ValueError(f'unsupported activation/gradient dtype {t.dtype}') from None


def _detached(t: torch.Tensor) -> torch.Tensor:
    _cabi.require_device(t)
    return t.detach()


def _dense(t: torch.Tensor) -> torch.Tensor:
    return t if t.is_contiguous() else t.contiguous()


def _workspace(scratch, need: int, device: torch.device) -> int | None:
    """Device pointer of `need` bytes of the scratch buffer (None for none)."""
    ws = scratch.get(need, device)
    return ws.data_ptr() if ws is not None else None


class LinearModuleHelper(ModuleHelper):
    """torch.nn.Linear: A = [x,1]^T[x,1]/rows, G = g^T g/rows (modules.py:100-141).

    Under K-FAC-reduce, dimension 0 is the example dimension (B; an unbatched 1-D input is one example) and every
    dimension between it and the last is shared (R = numel / (B * features) positions).  For R > 1 each example gives
    one row: the mean of its R A rows, and the sum of its R G rows divided by sqrt(R)."""

    @property
    def a_factor_shape(self):
        d = self.module.weight.size(1) + int(self.has_bias())
        return (d,) if self.diagonal_a else (d, d)

    @property
    def g_factor_shape(self):
        d = self.module.weight.size(0)
        return (d, d)

    def _positions(self, t: torch.Tensor) -> tuple[int, int] | None:
        """(B, R) when this call takes the K-FAC-reduce path (reduce on and R > 1), else None."""
        if not self.reduce or t.numel() == 0:
            return None
        B = t.size(0) if t.dim() > 1 else 1
        R = t.numel() // (B * t.size(-1))
        return (B, R) if R > 1 else None

    def rows_a(self, x):
        return self._rows(x, 'a')

    def rows_g(self, g):
        return self._rows(g, 'g')

    def _rows(self, t: torch.Tensor, side: str) -> FactorRows:
        """The rows of one tap of side 'a' (ones column included) or 'g': every position, or under K-FAC-reduce the
        mean of each example's R A rows and the sum of its R G rows divided by sqrt(R)."""
        feat = t.size(-1)
        ones = int(self.has_bias()) if side == 'a' else 0
        pos = self._positions(t)
        if pos is not None:
            B, R = pos
            per = 1.0 / R if side == 'a' else 1.0 / math.sqrt(R)

            def write_reduced(out, ld, grad_scale, loss_scale):
                c = _dense(t)
                _cabi.check(_cabi.load().kfac_reduce_rows_linear(c.data_ptr(), _dtype_code(c), B, R, feat, ones,
                                                                 1.0 / grad_scale * per, loss_scale, out, ld,
                                                                 _cabi.stream_ptr()), 'kfac_reduce_rows_linear')
            return FactorRows(B, feat + ones, write_reduced)
        rows = t.numel() // feat

        def write(out, ld, grad_scale, loss_scale):
            c = _dense(t)
            _cabi.check(_cabi.load().kfac_rows_linear(c.data_ptr(), _dtype_code(c), rows, feat, ones,
                                                      1.0 / grad_scale, loss_scale, out, ld, _cabi.stream_ptr()),
                        'kfac_rows_linear')

        if side == 'a' and self.diagonal_a:
            def direct(acc, grad_scale, scratch):
                if rows == 0:
                    return
                lib = _cabi.load()
                c = _dense(t)
                need = lib.kfac_factor_linear_diag_workspace_bytes(rows, feat)
                _cabi.check(lib.kfac_factor_linear_diag_ones(c.data_ptr(), _dtype_code(c), rows, feat, ones,
                                                             1.0 / (rows * grad_scale * grad_scale), acc.data_ptr(),
                                                             _workspace(scratch, need, c.device), need,
                                                             _cabi.stream_ptr()), 'kfac_factor_linear_diag_ones')
        elif side == 'g' and self.diagonal_g:
            def direct(acc, grad_scale, scratch):
                if rows == 0:
                    return
                lib = _cabi.load()
                c = _dense(t)
                need = lib.kfac_factor_linear_diag_workspace_bytes(rows, feat)
                _cabi.check(lib.kfac_factor_linear_diag(c.data_ptr(), _dtype_code(c), rows, feat,
                                                        1.0 / (rows * grad_scale * grad_scale), acc.data_ptr(),
                                                        _workspace(scratch, need, c.device), need,
                                                        _cabi.stream_ptr()), 'kfac_factor_linear_diag')
        else:
            def direct(acc, grad_scale, scratch):
                lib = _cabi.load()
                c = _dense(t)
                need = lib.kfac_factor_linear_workspace_bytes(rows, feat, ones)
                _cabi.check(lib.kfac_factor_linear(c.data_ptr(), _dtype_code(c), rows, feat, ones,
                                                   1.0 / (rows * grad_scale * grad_scale), acc.data_ptr(),
                                                   _workspace(scratch, need, c.device), need, _cabi.stream_ptr()),
                            'kfac_factor_linear')
        return FactorRows(rows, feat + ones, write, direct)


class Conv2dModuleHelper(ModuleHelper):
    """torch.nn.Conv2d (modules.py:144-237).  Like the reference, dilation and
    groups are ignored; feature order is (C_in, kh, kw) [+ ones]."""

    @property
    def a_factor_shape(self):
        m = self.module
        d = m.in_channels * m.kernel_size[0] * m.kernel_size[1] + int(self.has_bias())
        return (d,) if self.diagonal_a else (d, d)

    @property
    def g_factor_shape(self):
        return (self.module.out_channels, self.module.out_channels)

    def _geometry(self, x):
        m = self.module
        pad = m.padding
        if isinstance(pad, str):
            raise ValueError('string padding modes are not supported by K-FAC conv factors')
        B, Cc, H, W = x.shape
        return (B, Cc, H, W, m.kernel_size[0], m.kernel_size[1], m.stride[0], m.stride[1],
                pad[0], pad[1])

    @staticmethod
    def _spatial(geo) -> int:
        B, _, H, W, kh, kw, sh, sw, ph, pw = geo
        return ((H + 2 * ph - kh) // sh + 1) * ((W + 2 * pw - kw) // sw + 1)

    def rows_a(self, x):
        geo = self._geometry(x)
        B, Cc, H, W, kh, kw, sh, sw, ph, pw = geo
        arr = lambda v: (C.c_int * 3)(*v)  # noqa: E731
        diag = (_cabi.ConvGeometry(B, Cc, arr((1, H, W)), arr((1, kh, kw)), arr((1, sh, sw)), arr((1, 1, 1)),
                                   arr((0, ph, pw)), arr((0, ph, pw))) if self.diagonal_a else None)
        return _conv_input_rows(self, x, 'conv2d_input', geo, (), B, self._spatial(geo), Cc * kh * kw, diag)

    def rows_g(self, g):
        return _conv_gradout_rows(g, *g.shape, self.reduce)


# The rows of a convolution (modules.py:170-192): the B * S output positions, the A and G rows scaled by 1/S, so the
# statistics are the plain sums scaled by 1/(B*S) * 1/S^2.  Under K-FAC-reduce (S > 1) one row per example, the mean
# of its S A rows and the sum of its S G rows divided by sqrt(S), the rows carrying the 1/S of the expand rows: scale
# 1/S^2 (A) and S^-3/2 (G) on the plain window sums.
def _conv_input_rows(helper: ModuleHelper, x: torch.Tensor, entry: str, geo: tuple, ws_args: tuple, B: int,
                     S: int, patch: int, diag: _cabi.ConvGeometry | None = None) -> FactorRows:
    """A rows of a convolution (`patch` = C_in * taps features before the ones column) through the native entries
    kfac_factor_{entry}, kfac_rows_{entry} and kfac_reduce_rows_{entry}, which take the geometry arguments `geo` (and
    `ws_args` after the ones column in the workspace query).  A diagonal A (`diag`: the geometry as a
    kfac_conv_geometry) takes kfac_factor_conv_input_diag in expand mode, and the diagonal statistics of the reduced
    rows under K-FAC-reduce."""
    ones = int(helper.has_bias())
    d = patch + ones
    if helper.reduce and S > 1:
        def write_reduced(out, ld, grad_scale, loss_scale):
            c, fn = _dense(x), f'kfac_reduce_rows_{entry}'
            _cabi.check(getattr(_cabi.load(), fn)(c.data_ptr(), _dtype_code(c), *geo, ones, 1.0 / (float(S) * S),
                                                  out, ld, _cabi.stream_ptr()), fn)
        return FactorRows(B, d, write_reduced)

    def write(out, ld, grad_scale, loss_scale):
        c, fn = _dense(x), f'kfac_rows_{entry}'
        _cabi.check(getattr(_cabi.load(), fn)(c.data_ptr(), _dtype_code(c), *geo, ones, 1.0 / S, out, ld,
                                              _cabi.stream_ptr()), fn)

    if diag is not None:
        def direct_diag(acc, grad_scale, scratch):
            lib = _cabi.load()
            c = _dense(x)
            need = lib.kfac_factor_conv_input_diag_workspace_bytes(C.byref(diag))
            _cabi.check(lib.kfac_factor_conv_input_diag(c.data_ptr(), _dtype_code(c), C.byref(diag), ones,
                                                        1.0 / (float(B) * float(S) ** 3), acc.data_ptr(),
                                                        _workspace(scratch, need, c.device), need, _cabi.stream_ptr()),
                        'kfac_factor_conv_input_diag')
        return FactorRows(B * S, d, write, direct_diag)

    def direct(acc, grad_scale, scratch):
        lib = _cabi.load()
        c, fn = _dense(x), f'kfac_factor_{entry}'
        need = getattr(lib, fn + '_workspace_bytes')(*geo, ones, *ws_args)
        # ws_bytes = need, not the scratch buffer's size: the chunking, and so the bits, depend on it
        _cabi.check(getattr(lib, fn)(c.data_ptr(), _dtype_code(c), *geo, ones, 1.0 / (float(B) * float(S) ** 3),
                                     acc.data_ptr(), _workspace(scratch, need, c.device), need, _cabi.stream_ptr()), fn)
    return FactorRows(B * S, d, write, direct)


def _conv_gradout_rows(g: torch.Tensor, B: int, Cc: int, Ho: int, Wo: int, reduce: bool) -> FactorRows:
    """G rows of a convolution whose output gradient g is read as (B, Cc, Ho, Wo)."""
    S = Ho * Wo
    if reduce and S > 1:
        def write_reduced(out, ld, grad_scale, loss_scale):
            c = _dense(g)
            _cabi.check(_cabi.load().kfac_reduce_rows_conv2d_gradout(c.data_ptr(), _dtype_code(c), B, Cc, Ho, Wo,
                                                                     1.0 / grad_scale / float(S) ** 1.5, loss_scale,
                                                                     out, ld, _cabi.stream_ptr()),
                        'kfac_reduce_rows_conv2d_gradout')
        return FactorRows(B, Cc, write_reduced)

    def write(out, ld, grad_scale, loss_scale):
        c = _dense(g)
        _cabi.check(_cabi.load().kfac_rows_conv2d_gradout(c.data_ptr(), _dtype_code(c), B, Cc, Ho, Wo,
                                                          1.0 / (float(S) * grad_scale), loss_scale, out, ld,
                                                          _cabi.stream_ptr()), 'kfac_rows_conv2d_gradout')

    def direct(acc, grad_scale, scratch):
        lib = _cabi.load()
        c = _dense(g)
        need = lib.kfac_factor_conv2d_gradout_workspace_bytes(B, Cc, Ho, Wo)
        _cabi.check(lib.kfac_factor_conv2d_gradout(c.data_ptr(), _dtype_code(c), B, Cc, Ho, Wo,
                                                   1.0 / (float(B) * float(S) ** 3 * grad_scale * grad_scale),
                                                   acc.data_ptr(), _workspace(scratch, need, c.device), need,
                                                   _cabi.stream_ptr()), 'kfac_factor_conv2d_gradout')
    return FactorRows(B * S, Cc, write, direct)


# Largest im2col chunk of a Conv1d / Conv3d factor call: a video layer's im2col is tens of times its input (r2plus1d_18
# layer1 on 8 x 16 x 112^2 clips: 401 k rows x 576 features, 0.93 GB), so the matrix is formed a few examples at a time
CONV_ND_WORKSPACE_BYTES = 1 << 30
# most taps (kd * kh * kw) of a kernel whose K-FAC-reduce window sums the native kernel forms
REDUCE_MAX_TAPS = 2048


class ConvNdModuleHelper(ModuleHelper):
    """torch.nn.Conv1d / Conv3d (an extension beyond the reference, opt-in through `precondition_conv_nd`).

    The statistics are those of a Conv2d layer (modules.py:170-192) on the N-d lattice: rows = B * S positions
    (S = Lo or Do * Ho * Wo), the A and G rows scaled by 1/S, A's feature order (C_in, kd, kh, kw) [+ ones], the order
    of weight.reshape(out, -1).  Unlike Conv2d the geometry is honoured exactly: dilation on every axis, and per-axis
    (before, after) padding from `_reversed_padding_repeated_twice` (integers, 'valid', or 'same' with torch's
    asymmetric split).  A `padding_mode` other than 'zeros' pads the input with F.pad as the module's forward does,
    and the statistics are formed with zero padding 0.  An unbatched input is one example.  A Conv1d is the N-d case
    D = kd = 1, H = kh = 1.  Under K-FAC-reduce R = S with the Conv2d constants.  The A-side methods read the tensor
    prepare_input made of the call's input (batched, contiguous, padded for a non-'zeros' padding_mode)."""

    keyword = 'precondition_conv_nd'
    # the native input-side entries: kfac_factor_{entry}, kfac_rows_{entry}, kfac_reduce_rows_{entry}
    entry = 'conv_input'

    def __init__(self, module: torch.nn.Module, reduce: bool = False, diagonal_a: bool = False):
        super().__init__(module, reduce=reduce, diagonal_a=diagonal_a)
        self.nd = len(module.kernel_size)
        # output extents of the recent A calls: the G call checks its output gradient against them
        self._extents: list[tuple[int, ...]] = []

    def check(self, name: str) -> None:
        """Raise for what this helper cannot precondition (called at registration)."""
        m = self.module
        what = None
        taps = math.prod(m.kernel_size)
        if m.groups != 1:
            what = f'groups={m.groups} (grouped and depthwise convolutions are not supported)'
        elif self.diagonal_a and m.out_channels > _cabi.KFAC_EIGH_MAX_N:
            what = f'a G factor of {m.out_channels}, beyond the eigensolver\'s {_cabi.KFAC_EIGH_MAX_N}'
        elif self.diagonal_a and taps > REDUCE_MAX_TAPS:
            what = f'a kernel of {taps} taps, beyond the {REDUCE_MAX_TAPS} of the diagonal A statistics'
        elif not self.diagonal_a and max(self.a_factor_shape[0], m.out_channels) > _cabi.KFAC_EIGH_MAX_N:
            what = (f'factors of {self.a_factor_shape[0]} (A) and {m.out_channels} (G), beyond the eigensolver\'s '
                    f'{_cabi.KFAC_EIGH_MAX_N}')
        elif self.reduce and taps > REDUCE_MAX_TAPS:
            what = (f'a kernel of {taps} taps, beyond the {REDUCE_MAX_TAPS} of the K-FAC-reduce window sums '
                    "(kfac_approx='reduce')")
        if what is not None:
            raise ValueError(f'{self.keyword}: "{name}" ({m.__class__.__name__}) has {what}; add it to skip_layers')

    @property
    def a_factor_shape(self):
        d = self.module.in_channels * math.prod(self.module.kernel_size) + int(self.has_bias())
        return (d,) if self.diagonal_a else (d, d)

    @property
    def g_factor_shape(self):
        return (self.module.out_channels, self.module.out_channels)

    def _pads(self) -> tuple[list[int], list[int]]:
        """Per-axis (before, after) zero padding of the statistics, each in (D, H, W) order."""
        before, after = [0, 0, 0], [0, 0, 0]
        if self.module.padding_mode == 'zeros':
            rp = self.module._reversed_padding_repeated_twice
            for k in range(self.nd):            # rp lists (before, after) from the last axis to the first
                before[2 - k], after[2 - k] = rp[2 * k], rp[2 * k + 1]
        return before, after

    def _geometry(self, shape: torch.Size) -> tuple[_cabi.ConvGeometry, tuple[int, ...]]:
        """Native geometry and output extents of an input of `shape` (batched, padded as by prepare_input)."""
        m = self.module
        lead = [1] * (3 - self.nd)
        ins = lead + list(shape[2:])
        ker, st, dil = (lead + list(v) for v in (m.kernel_size, m.stride, m.dilation))
        before, after = self._pads()
        out = [(ins[a] + before[a] + after[a] - dil[a] * (ker[a] - 1) - 1) // st[a] + 1 for a in range(3)]
        geo = _cabi.ConvGeometry(shape[0], shape[1], (C.c_int * 3)(*ins), (C.c_int * 3)(*ker), (C.c_int * 3)(*st),
                                 (C.c_int * 3)(*dil), (C.c_int * 3)(*before), (C.c_int * 3)(*after))
        return geo, tuple(out[3 - self.nd:])

    def _batched(self, t: torch.Tensor) -> torch.Tensor:
        return t.unsqueeze(0) if t.dim() == self.nd + 1 else t

    def prepare_input(self, x: torch.Tensor) -> torch.Tensor:
        """The batched, contiguous input the statistics read, padded here for a non-'zeros' padding_mode (once per
        call: EKFAC's row writer reads the same tensor)."""
        _cabi.require_device(x)
        self._input_geometry(x.shape)       # refuses an input with an empty output
        x = self._batched(x.detach())
        m = self.module
        if m.padding_mode != 'zeros':
            x = torch.nn.functional.pad(x, m._reversed_padding_repeated_twice, mode=m.padding_mode)
        return x if x.is_contiguous() else x.contiguous()

    def _input_geometry(self, x_shape: torch.Size):
        """(geometry, S) of a raw (unpadded, possibly unbatched) input shape."""
        shape = list(x_shape) if len(x_shape) == self.nd + 2 else [1] + list(x_shape)
        if self.module.padding_mode != 'zeros':
            rp = self.module._reversed_padding_repeated_twice
            for k in range(self.nd):
                shape[-1 - k] += rp[2 * k] + rp[2 * k + 1]
        geo, out = self._geometry(torch.Size(shape))
        if min(out) <= 0:
            raise ValueError(f'{self.module.__class__.__name__}: input of shape {tuple(x_shape)} gives an empty output')
        return geo, math.prod(out), out

    def _prepared_geometry(self, x: torch.Tensor) -> tuple[_cabi.ConvGeometry, int]:
        """(geometry, S) of a prepare_input tensor; its output extent is recorded for the G call's check."""
        geo, out = self._geometry(x.shape)
        if not self._extents or self._extents[-1] != out:
            self._extents = (self._extents + [out])[-8:]
        return geo, math.prod(out)

    def rows_a(self, x):
        geo, S = self._prepared_geometry(x)
        return _conv_input_rows(self, x, self.entry, (C.byref(geo),), (CONV_ND_WORKSPACE_BYTES,), geo.batch, S,
                                geo.C * math.prod(self.module.kernel_size), geo if self.diagonal_a else None)

    def rows_g(self, g):
        """The output gradient read as (B, C, 1, S); its extent must be one an A call of this window computed."""
        g = self._batched(g)
        out = tuple(g.shape[2:])
        if self._extents and out not in self._extents:
            raise ValueError(f'{self.module.__class__.__name__}: output gradient extent {out} does not match the '
                             f'output extent {self._extents[-1]} computed from the input and the padding')
        return _conv_gradout_rows(g, g.size(0), g.size(1), 1, math.prod(out), self.reduce)


class ConvTransposeModuleHelper(ConvNdModuleHelper):
    """torch.nn.ConvTranspose1d / 2d / 3d with groups = 1 (an extension beyond the reference, opt-in through
    `precondition_conv_transpose`).

    y[b, co, o] = bias[co] + sum_{ci, k, i: o = i s - p + k d} x[b, ci, i] W[ci, co, k], so each output position o has
    the patch a(o)[ci, k] = x[b, ci, (o + p - k d) / s] when s divides (o + p - k d) on every axis and the quotient is
    an input position, 0 otherwise, and y[:, o] = Wmat a(o) + bias with Wmat[co, ci K + k] = W[ci, co, k].  The rows are
    the B * S output positions (S the product of the output extents), A and G rows scaled by 1/S as for a Conv2d layer,
    A's feature order (C_in, kd, kh, kw) [+ ones] and G C_out x C_out; under K-FAC-reduce R = S.  The G side, the
    extent check of the output gradient and the reduce constants are those of ConvNdModuleHelper.

    The weight gradient (C_in, C_out, k...) is not Wmat's layout: `wgrad_taps` = K tells the native precondition,
    kl-clip and write-back to address it in place.  The output padding of a call is torch's (`output_size` passed
    positionally or as a keyword, through bind_call); the padding mode is always 'zeros'."""

    keyword = 'precondition_conv_transpose'
    entry = 'conv_transpose_input'
    call_kwargs = True

    def __init__(self, module: torch.nn.Module, reduce: bool = False):
        super().__init__(module, reduce=reduce)
        self._call_op = list(module.output_padding)    # output padding of the call bind_call saw last

    @property
    def wgrad_taps(self) -> int:
        return math.prod(self.module.kernel_size)

    def get_grad(self) -> torch.Tensor:
        m = self.module
        w = m.weight.grad.reshape(m.in_channels, m.out_channels, -1).permute(1, 0, 2).reshape(m.out_channels, -1)
        return torch.cat([w, m.bias.grad.view(-1, 1)], 1) if self.has_bias() else w

    def bind_call(self, args: tuple, kwargs: dict) -> None:
        """Take the output padding of a forward call (module(x), module(x, output_size) or module(x,
        output_size=...)), derived as the module's forward derives it."""
        m = self.module
        output_size = args[1] if len(args) > 1 else kwargs.get('output_size')
        self._call_op = list(m._output_padding(args[0], output_size, m.stride, m.padding, m.kernel_size, self.nd,
                                               m.dilation))

    def _geometry(self, shape: torch.Size) -> tuple[_cabi.ConvTransposeGeometry, tuple[int, ...]]:
        """Native geometry and output extents of a batched input of `shape` with the bound call's output padding."""
        m = self.module
        lead, zero = [1] * (3 - self.nd), [0] * (3 - self.nd)
        ins = lead + list(shape[2:])
        ker, st, dil = (lead + list(v) for v in (m.kernel_size, m.stride, m.dilation))
        pad, op = zero + list(m.padding), zero + list(self._call_op)
        out = [(ins[a] - 1) * st[a] - 2 * pad[a] + dil[a] * (ker[a] - 1) + op[a] + 1 for a in range(3)]
        arr = lambda v: (C.c_int * 3)(*v)  # noqa: E731
        geo = _cabi.ConvTransposeGeometry(shape[0], shape[1], arr(ins), arr(ker), arr(st), arr(dil), arr(pad), arr(op))
        return geo, tuple(out[3 - self.nd:])

    def output_extent(self, x_shape: torch.Size) -> tuple[int, ...]:
        """Output extents of a (possibly unbatched) input of `x_shape` under the bound call's output padding."""
        shape = list(x_shape) if len(x_shape) == self.nd + 2 else [1] + list(x_shape)
        return self._geometry(torch.Size(shape))[1]

    def prepare_input(self, x: torch.Tensor) -> torch.Tensor:
        """The batched, contiguous input the statistics read."""
        _cabi.require_device(x)
        if min(self.output_extent(x.shape)) <= 0:
            raise ValueError(f'{self.module.__class__.__name__}: input of shape {tuple(x.shape)} gives an empty output')
        x = self._batched(x.detach())
        return x if x.is_contiguous() else x.contiguous()


class EmbeddingModuleHelper(LinearModuleHelper):
    """torch.nn.Embedding (an extension beyond the reference, opt-in through `precondition_embeddings`).

    An embedding is a Linear layer whose input rows are one-hot vectors e_idx, so A = (1/N) sum_r e_r e_r^T is
    DIAGONAL: the token frequencies counts / N, kept as a vector of V floats (`a_factor_shape` is (V,)).  Every
    index position is one row, `padding_idx` positions included (their gradient row is zero, so their P row is
    zero), which keeps N = idx.numel() known on the host.  G is formed from the grad-output rows exactly like a
    Linear layer's (never K-FAC-reduced).  The gradient and P use the weight's own layout (V x d)."""

    diagonal_a = True
    embedding = True
    counts_a = True

    @property
    def a_factor_shape(self):
        return (self.module.num_embeddings,)

    @property
    def g_factor_shape(self):
        d = self.module.embedding_dim
        return (d, d)

    def has_bias(self) -> bool:
        return False

    def accumulate_a(self, x, acc, scratch):
        """acc += the index histogram of one call / N."""
        x = _detached(x)
        try:
            code = _cabi.INDEX_DTYPE_CODE[x.dtype]
        except KeyError:
            raise ValueError(f'unsupported embedding index dtype {x.dtype}') from None
        x = _dense(x)
        V = self.module.num_embeddings
        n = x.numel()
        if n == 0:
            return
        lib = _cabi.load()
        need = lib.kfac_factor_embedding_workspace_bytes(V)
        _cabi.check(lib.kfac_factor_embedding(x.data_ptr(), code, n, V, 1.0 / n, acc.data_ptr(),
                                              _workspace(scratch, need, x.device), need, _cabi.stream_ptr()),
                    'kfac_factor_embedding')


class EmbeddingBagModuleHelper(EmbeddingModuleHelper):
    """torch.nn.EmbeddingBag with mode 'sum' or 'mean' (an extension beyond the reference, opt-in through
    `precondition_embedding_bags`).

    Bag b pools its entries into the row c_b in R^V of a Linear layer, output_b = W^T c_b and weight.grad = C^T g:
    c_bv = sum of the per-sample weights (or 1) of its entries equal to v ('sum'), or n_bv / L_b ('mean', L_b the
    bag's non-padding entries; an empty bag is a zero row), `padding_idx` entries left out.  A = (1/B) C^T C is V x V
    and not diagonal once a bag holds two distinct tokens; its diagonal (1/B) sum_b c_bv^2 is kept, a vector of V
    floats, exact for bags of one index (where it is nn.Embedding's A).  Every bag, empty or not, is one row (N = B),
    also under K-FAC-reduce.  G is formed from the rows of the (B, d) output gradient like a Linear layer's.  The
    gradient and P use the weight's layout (V x d).  The call's `offsets` and `per_sample_weights` reach the A
    statistic through bind_call."""

    call_kwargs = True
    counts_a = False

    def __init__(self, module: torch.nn.Module):
        super().__init__(module)
        self._call: tuple[torch.Tensor | None, torch.Tensor | None] = (None, None)

    def bind_call(self, args: tuple, kwargs: dict) -> None:
        """Take the offsets and per-sample weights of a forward call, positional or keyword."""
        offsets = args[1] if len(args) > 1 else kwargs.get('offsets')
        weights = args[2] if len(args) > 2 else kwargs.get('per_sample_weights')
        self._call = (offsets, weights)

    def accumulate_a(self, x, acc, scratch):
        """acc += the diagonal of the pooled rows' C^T C / B for the call bind_call saw."""
        offsets, weights = self._call
        self._call = (None, None)
        m = self.module
        x = _detached(x)
        if x.dim() == 2:
            B, offsets = x.size(0), None
        elif x.dim() == 1 and offsets is not None:
            offsets = _detached(offsets)
            B = offsets.numel() - int(m.include_last_offset)
            if offsets.dtype != x.dtype:        # torch promotes mixed index and offset dtypes to int64
                x, offsets = x.long(), offsets.long()
            offsets = _dense(offsets)
        else:
            raise ValueError(f'EmbeddingBag: input of shape {tuple(x.shape)} (1-D input needs offsets)')
        try:
            code = _cabi.INDEX_DTYPE_CODE[x.dtype]
        except KeyError:
            raise ValueError(f'unsupported embedding bag index dtype {x.dtype}') from None
        x = _dense(x)
        n = x.numel()
        if n == 0 or B <= 0:
            return
        wcode = 0
        if weights is not None:
            weights = _dense(cast_for_factor(_detached(weights), None))
            wcode = _dtype_code(weights)
        V = m.num_embeddings
        mode = {'sum': _cabi.KFAC_BAG_SUM, 'mean': _cabi.KFAC_BAG_MEAN}[m.mode]
        lib = _cabi.load()
        need = lib.kfac_factor_embedding_bag_workspace_bytes(n, B, V)
        _cabi.check(lib.kfac_factor_embedding_bag(x.data_ptr(), offsets.data_ptr() if offsets is not None else None,
                                                  code, n, B, -1 if m.padding_idx is None else m.padding_idx, mode,
                                                  weights.data_ptr() if weights is not None else None, wcode, V,
                                                  1.0 / B, acc.data_ptr(), _workspace(scratch, need, x.device), need,
                                                  _cabi.stream_ptr()), 'kfac_factor_embedding_bag')


class DiagonalGLinearModuleHelper(LinearModuleHelper):
    """torch.nn.Linear with G approximated by its diagonal (an extension beyond the reference, opt-in through
    `diagonal_g_layers`), for layers with too many outputs for a dense G: an LM head of V = 50257 outputs would need
    a V x V factor (10 GB) beyond the eigensolver.  diag(G) = (1/N) sum_r g_r^2 is kept as a vector of V floats
    (`g_factor_shape` is (V,)); it is its own eigendecomposition (Qg = I).  A, the gradient, P and the G rows are
    those of a Linear layer; `diagonal_g` selects the diagonal statistics of the G rows."""

    diagonal_g = True

    @property
    def g_factor_shape(self):
        return (self.module.weight.size(0),)


class NormModuleHelper(ModuleHelper):
    """torch.nn.BatchNorm1d / BatchNorm2d / LayerNorm / RMSNorm (opt-in through `precondition_norms`) and GroupNorm /
    InstanceNorm1d / 2d / 3d (opt-in through `precondition_group_norms`) with an affine part (an extension beyond the
    reference).

    The affine part y = s * xhat + b is a depthwise layer with bias on the normalized input, so each channel c is a
    one-input layer with rows a_r = (xhat_rc, 1) (or (xhat_rc) for a scale-only layer) and g_r = dL/dy_rc.  Instead
    of a Kronecker factorization the exact per-channel block of the row-level Fisher is kept,
        F_c = (1/N) sum_r g_rc^2 a_r a_r^T,
    packed as k = 3 floats (F_ss, F_sb, F_bb) or k = 1 (`g_factor_shape` is (C, k)); there is no A factor.
    P_c = (F_c + damping I)^-1 (weight.grad[c], bias.grad[c]) is stored as C x (1 + has_bias), the layout of a
    Linear layer's P with the weight in column 0 and the bias in the last column.

    Rows and xhat:
      * BatchNorm2d, BatchNorm1d on (B, C, L): the B * S positions (S = H * W or L) with a_r and g_r scaled by 1/S,
        as a Conv2d layer's rows; xhat from the biased batch statistics of each channel plus eps;
      * BatchNorm1d on (B, C), LayerNorm, RMSNorm: every leading position is a row, unscaled, as for nn.Linear;
        xhat from the statistics of each row over `normalized_shape` (mean and biased variance plus eps, or
        x / sqrt(mean(x^2) + eps); when the module's eps is None, torch's: finfo(float32).eps for fp16, bf16 and
        fp32 inputs, finfo(float64).eps for fp64 inputs);
      * GroupNorm, InstanceNorm* (kind KFAC_NORM_GROUP): the rows of BatchNorm (B * S positions scaled by 1/S; S = 1
        and unscaled for a GroupNorm on (B, C)); xhat from the mean and biased variance plus eps of each example's
        group of C / `groups` channels (`groups` = num_groups, or C for an InstanceNorm).  An unbatched
        InstanceNorm input is one example.
    xhat is recomputed from the layer input, so a gain near zero does not affect it."""

    norm = True

    def __init__(self, module: torch.nn.Module):
        super().__init__(module)
        self.groups = 0             # the number of groups of a KFAC_NORM_GROUP layer
        if isinstance(module, (torch.nn.BatchNorm1d, torch.nn.BatchNorm2d)):
            self.kind = _cabi.KFAC_NORM_BATCH
        elif isinstance(module, torch.nn.LayerNorm):
            self.kind = _cabi.KFAC_NORM_LAYER
        elif isinstance(module, torch.nn.RMSNorm):
            self.kind = _cabi.KFAC_NORM_RMS
        else:
            self.kind = _cabi.KFAC_NORM_GROUP
            self.groups = module.num_groups if isinstance(module, torch.nn.GroupNorm) else module.num_features

    @property
    def channels(self) -> int:
        return self.module.weight.numel()

    @property
    def k(self) -> int:
        """Packed entries of one block: 3 (F_ss, F_sb, F_bb) with a bias, 1 (F_ss) without."""
        return 3 if self.has_bias() else 1

    @property
    def a_factor_shape(self):
        """(width of a_r,): only its length is used (the columns of P); no A factor is stored."""
        return (1 + int(self.has_bias()),)

    @property
    def g_factor_shape(self):
        return (self.channels, self.k)

    def get_grad(self) -> torch.Tensor:
        g = self.module.weight.grad.reshape(-1, 1)
        if self.has_bias():
            g = torch.cat([g, self.module.bias.grad.reshape(-1, 1)], 1)
        return g

    def eps_for(self, x: torch.Tensor) -> float:
        """The module's eps; for eps=None (RMSNorm) the machine epsilon of torch's computation type: that of float32
        for fp16, bf16 and fp32 inputs, that of float64 for fp64 inputs."""
        eps = self.module.eps
        if eps is None:
            return float(torch.finfo(torch.float64 if x.dtype == torch.float64 else torch.float32).eps)
        return float(eps)

    def accumulate_norm(self, x: torch.Tensor, g: torch.Tensor, acc: torch.Tensor, grad_scale: float, eps: float,
                        scratch) -> None:
        """acc (C x k) += the window's share of F_c for one call: x the layer input, g the gradient of its output."""
        _cabi.require_device(x)
        _cabi.require_device(g)
        x = x.detach()
        g = g.detach()
        x = x if x.is_contiguous() else x.contiguous()
        g = g if g.is_contiguous() else g.contiguous()
        if x.shape != g.shape:
            raise ValueError(f'normalization layer: input {tuple(x.shape)} and output gradient {tuple(g.shape)} differ')
        C = self.channels
        if x.numel() == 0:
            return
        lib = _cabi.load()
        if self.kind == _cabi.KFAC_NORM_GROUP:
            # an InstanceNorm input without the batch dimension is one example, detected as the module's forward does
            unbatched = (not isinstance(self.module, torch.nn.GroupNorm)
                         and x.dim() == self.module._get_no_batch_dim())
            xb = x.unsqueeze(0) if unbatched else x
            if xb.dim() < 2 or xb.size(1) != C or (not isinstance(self.module, torch.nn.GroupNorm)
                                                   and xb.dim() != self.module._get_no_batch_dim() + 1):
                raise ValueError(f'{self.module.__class__.__name__} input of shape {tuple(x.shape)} for {C} channels')
            B, S = xb.size(0), x.numel() // (xb.size(0) * C)
            # the rows of BatchNorm: N = B * S, a_r and g_r scaled by 1/S (as a Conv2d layer's): 1 / (N * S^4)
            scale = 1.0 / (float(B) * float(S) ** 5 * grad_scale * grad_scale)
            need = lib.kfac_factor_group_norm_workspace_bytes(B, C, S, self.groups)
            ws = scratch.get(need, x.device)
            _cabi.check(lib.kfac_factor_group_norm(x.data_ptr(), _dtype_code(x), g.data_ptr(), _dtype_code(g), B, C,
                                                   S, self.groups, self.k, eps, scale, acc.data_ptr(), ws.data_ptr(),
                                                   need, _cabi.stream_ptr()), 'kfac_factor_group_norm')
            return
        if self.kind == _cabi.KFAC_NORM_BATCH:
            if x.dim() not in (2, 3, 4) or x.size(1) != C:
                raise ValueError(f'BatchNorm input of shape {tuple(x.shape)} for {C} channels')
            rows, S = x.size(0), x.numel() // (x.size(0) * C)
            # N = B * S rows, a_r and g_r scaled by 1/S (as a Conv2d layer's): 1 / (N * S^4)
            scale = 1.0 / (float(rows) * float(S) ** 5 * grad_scale * grad_scale)
        else:
            rows, S = x.numel() // C, 1
            scale = 1.0 / (float(rows) * grad_scale * grad_scale)
        need = lib.kfac_factor_norm_workspace_bytes(self.kind, rows, C, S)
        ws = scratch.get(need, x.device)
        _cabi.check(lib.kfac_factor_norm(x.data_ptr(), _dtype_code(x), g.data_ptr(), _dtype_code(g), self.kind, rows,
                                         C, S, self.k, eps, scale, acc.data_ptr(), ws.data_ptr(), need,
                                         _cabi.stream_ptr()), 'kfac_factor_norm')


def _strided_rows(t: torch.Tensor, ordered: bool) -> tuple[torch.Tensor, int]:
    """(rows tensor, row stride) of a (..., features) tensor whose rows are `features` unit-stride elements at one row
    stride: the tensor itself, or -- when `ordered` is False, i.e. only sums over the rows are formed -- its
    transpose(0, 1) (the contiguous batch-first input behind a sequence-first view).  Any other layout is made
    contiguous."""
    feat = t.size(-1)
    for c in ((t,) if ordered or t.dim() != 3 else (t, t.transpose(0, 1))):
        if c.stride(-1) != 1 and feat > 1:
            continue
        try:
            r = c.view(-1, feat)
        except RuntimeError:
            continue
        ld = r.stride(0) if r.size(0) > 1 else feat
        if ld >= feat:
            return r, ld
    return t.contiguous().view(-1, feat), feat


class SequenceFirstLinearHelper(LinearModuleHelper):
    """A Linear layer keyed by an object that is not its own module, whose taps see (L, B, features) tensors in a
    sequence-first layout, read in place through the strided native entry points.  Under K-FAC-reduce the example
    dimension is B (dimension 1); an unbatched call is one example."""

    def get_grad(self):
        g = self.get_weight_grad()
        return torch.cat([g, self.get_bias_grad().view(-1, 1)], 1) if self.has_bias() else g

    def _positions(self, t):
        """(B, R) = (t.size(1), t.size(0)) of an (L, B, features) tap under K-FAC-reduce with R > 1, else None."""
        if not self.reduce or t.numel() == 0 or t.size(0) == 1:
            return None
        return (t.size(1), t.size(0))

    def _rows(self, t, side):
        """The rows of one tap, read in place through the strided entry points."""
        feat = t.size(-1)
        ones = int(self.has_bias()) if side == 'a' else 0
        pos = self._positions(t)
        if pos is not None:
            B, R = pos
            per = 1.0 / R if side == 'a' else 1.0 / math.sqrt(R)

            def write_reduced(out, ld, grad_scale, loss_scale):
                c = t if t.stride(-1) == 1 else t.contiguous()
                _cabi.check(_cabi.load().kfac_reduce_rows_linear_strided(
                    c.data_ptr(), _dtype_code(c), B, R, feat, c.stride(1), c.stride(0), ones, 1.0 / grad_scale * per,
                    loss_scale, out, ld, _cabi.stream_ptr()), 'kfac_reduce_rows_linear_strided')
            return FactorRows(B, feat + ones, write_reduced)

        def write(out, ld, grad_scale, loss_scale):
            # the A and G rows of EKFAC are paired row by row: both in the (L, B) order of the taps
            r, ldr = _strided_rows(t, ordered=True)
            _cabi.check(_cabi.load().kfac_rows_linear_strided(r.data_ptr(), _dtype_code(r), r.size(0), feat, ldr,
                                                              ones, 1.0 / grad_scale, loss_scale, out, ld,
                                                              _cabi.stream_ptr()), 'kfac_rows_linear_strided')

        def direct(acc, grad_scale, scratch):
            r, ldr = _strided_rows(t, ordered=False)
            rows = r.size(0)
            if rows == 0:
                return
            lib = _cabi.load()
            need = lib.kfac_factor_linear_strided_workspace_bytes(rows, feat, ldr, ones)
            _cabi.check(lib.kfac_factor_linear_strided(r.data_ptr(), _dtype_code(r), rows, feat, ldr, ones,
                                                       1.0 / (rows * grad_scale * grad_scale), acc.data_ptr(),
                                                       _workspace(scratch, need, r.device), need, _cabi.stream_ptr()),
                        'kfac_factor_linear_strided')
        return FactorRows(t.numel() // feat, feat + ones, write, direct)


class AttentionProjectionHelper(SequenceFirstLinearHelper):
    """One projection of a `torch.nn.MultiheadAttention` (an extension beyond the reference, opt-in through
    `precondition_attention`), preconditioned as the `torch.nn.Linear` it is mathematically:

        'q'    Linear(E, E) on query        rows [0, E) of in_proj_weight / in_proj_bias, or q_proj_weight
        'k'    Linear(kdim, E) on key       rows [E, 2E), or k_proj_weight
        'v'    Linear(vdim, E) on value     rows [2E, 3E), or v_proj_weight
        'out'  Linear(E, E) on the concatenated head outputs: out_proj.weight / out_proj.bias

    The gradients are row-slice views, contiguous like a Linear layer's, so the write-back runs in place.  The
    statistics come from taps inside `kfac_b200.attention.KFACMultiheadAttention`, which see (L, B, features) tensors
    in the sequence-first layout of torch's attention path: views of the batch-first input, column blocks of a packed
    projection's gradient.  They are read in place through the strided native entry points.  Under K-FAC-reduce the
    example dimension is the attention's batch dimension B (dimension 1 here); an unbatched call is one example."""

    def __init__(self, attn: torch.nn.MultiheadAttention, which: str, reduce: bool = False):
        super().__init__(attn, reduce=reduce)
        self.attn = attn
        self.which = which
        E = attn.embed_dim
        if which == 'out':
            self.weight, self.bias, self.rows = attn.out_proj.weight, attn.out_proj.bias, None
        else:
            i = 'qkv'.index(which)
            self.rows = (i * E, (i + 1) * E)
            self.weight = attn.in_proj_weight if attn._qkv_same_embed_dim else getattr(attn, f'{which}_proj_weight')
            self.bias = attn.in_proj_bias

    def __repr__(self) -> str:
        return f'{self.__class__.__name__}({self.which}, in_features={self.in_features}, out_features={self.attn.embed_dim})'

    def parameters(self):
        """The projection's own parameters (the whole packed in_proj_weight / in_proj_bias for q, k and v)."""
        return iter([p for p in (self.weight, self.bias) if p is not None])

    @property
    def in_features(self) -> int:
        return {'q': self.attn.embed_dim, 'k': self.attn.kdim, 'v': self.attn.vdim, 'out': self.attn.embed_dim}[self.which]

    def has_bias(self) -> bool:
        return self.bias is not None

    @property
    def a_factor_shape(self):
        d = self.in_features + int(self.has_bias())
        return (d, d)

    @property
    def g_factor_shape(self):
        return (self.attn.embed_dim, self.attn.embed_dim)

    def _slice(self, t: torch.Tensor | None, weight: bool) -> torch.Tensor | None:
        if t is None or self.rows is None or (weight and not self.attn._qkv_same_embed_dim):
            return t
        return t[self.rows[0]:self.rows[1]]

    def get_weight_grad(self):
        return self._slice(self.weight.grad, True)

    def get_bias_grad(self):
        return self._slice(self.bias.grad, False)


class RecurrentSubLayerHelper(SequenceFirstLinearHelper):
    """One sub-layer of a `torch.nn.RNN`, `LSTM` or `GRU` (an extension beyond the reference, opt-in through
    `precondition_recurrent`), preconditioned as the `torch.nn.Linear` it is mathematically, time steps being the
    positions of a weight-shared layer:

        'ih_l{k}{sfx}'   weight_ih_l{k}{sfx}, bias_ih_l{k}{sfx}   A: the layer input x_t    G: d(W_ih x_t + b_ih)
        'hh_l{k}{sfx}'   weight_hh_l{k}{sfx}, bias_hh_l{k}{sfx}   A: h_{t-1} (h0 first)     G: d(W_hh h_{t-1} + b_hh)

    For RNN and LSTM the two G rows of a position are equal; for GRU the hidden one is [dr, dz, r * dn].  The two biases
    have the same gradient (RNN, LSTM) and each is preconditioned by its own layer with its own ones column, as the
    two-Linear twin of the module does.

    The statistics come from taps inside `kfac_b200.recurrent`, which see time-major (T, B, features) tensors or the
    (N, features) data of a PackedSequence; each statistics call is preceded by the `SequenceTap` of its rows
    (`tap_a` / `tap_g`).  Unpacked input rows and the RNN / LSTM hidden G rows take the sequence-first Linear path.
    The hidden-state rows, the GRU hidden G rows and the per-sequence K-FAC-reduce rows of packed input go through
    `kfac_rows_sequence` / `kfac_reduce_rows_sequence` into scratch rows and the existing statistics call.  Under
    K-FAC-reduce the example dimension is the module's batch dimension, with R_b = T or the length of sequence b."""

    def __init__(self, rnn: torch.nn.Module, layer: int, direction: int, side: str, reduce: bool = False):
        super().__init__(rnn, reduce=reduce)
        self.rnn = rnn
        self.side = side
        self.suffix = f'{side}_l{layer}' + ('_reverse' if direction else '')
        self.tap_a = self.tap_g = None

    def __repr__(self) -> str:
        return f'{self.__class__.__name__}({self.suffix}, {tuple(self.weight.shape)}, bias={self.has_bias()})'

    @property
    def weight(self) -> torch.Tensor:
        return getattr(self.rnn, 'weight_' + self.suffix)

    @property
    def bias(self) -> torch.Tensor | None:
        return getattr(self.rnn, 'bias_' + self.suffix) if self.rnn.bias else None

    def parameters(self):
        return iter([p for p in (self.weight, self.bias) if p is not None])

    def has_bias(self) -> bool:
        return bool(self.rnn.bias)

    @property
    def a_factor_shape(self):
        d = self.weight.size(1) + int(self.has_bias())
        return (d, d)

    @property
    def g_factor_shape(self):
        d = self.weight.size(0)
        return (d, d)

    def get_weight_grad(self):
        return self.weight.grad

    def get_bias_grad(self):
        return self.bias.grad

    # ---- the rows of one tap
    def _reduced(self, tap) -> bool:
        return self.reduce and tap.T > 1

    def _native(self, tap) -> bool:
        """Whether the rows go through the sequence writers (else the sequence-first Linear path reads them)."""
        return tap.h0 is not None or tap.mul is not None or (tap.offsets is not None and self._reduced(tap))

    @staticmethod
    def _first(t: torch.Tensor, tap) -> torch.Tensor:
        """A packed (N, features) tap as the one-position (1, N, features) sequence-first tensor of its rows."""
        return t.unsqueeze(0) if tap.offsets is not None else t

    def _sequence_call(self, t, tap, side, scale, loss_scale, out_ptr, ld, reduced):
        t = t if t.is_contiguous() else t.contiguous()
        feat = (self.a_factor_shape[0] - int(self.has_bias())) if side == 'a' else self.g_factor_shape[0]

        def like(u):         # h0 and r in the dtype of the rows (factor_dtype casts those)
            return None if u is None else u.to(t.dtype).contiguous()
        h0, mul = like(tap.h0), like(tap.mul)
        src = _cabi.SequenceRows(t.data_ptr(), t.size(-1), tap.col0,
                                 h0.data_ptr() if h0 is not None else None, h0.size(-1) if h0 is not None else 0,
                                 tap.shift, mul.data_ptr() if mul is not None else None,
                                 mul.size(-1) if mul is not None else 0, tap.mul_col0, tap.T, tap.B,
                                 tap.offsets.data_ptr() if tap.offsets is not None else None)
        ones = int(self.has_bias()) if side == 'a' else 0
        lib = _cabi.load()
        if reduced:
            _cabi.check(lib.kfac_reduce_rows_sequence(C.byref(src), _dtype_code(t), feat, ones, scale,
                                                      1.0 if side == 'a' else 0.5, loss_scale, out_ptr, ld,
                                                      _cabi.stream_ptr()), 'kfac_reduce_rows_sequence')
        else:
            _cabi.check(lib.kfac_rows_sequence(C.byref(src), _dtype_code(t), feat, ones, scale, loss_scale, out_ptr,
                                               ld, _cabi.stream_ptr()), 'kfac_rows_sequence')

    def _rows(self, t, side):
        """The rows of the tap `tap_a` / `tap_g` describes."""
        tap = self.tap_a if side == 'a' else self.tap_g
        if not self._native(tap):
            return super()._rows(self._first(t, tap), side)
        reduced = self._reduced(tap)
        n = tap.B if reduced else t.numel() // t.size(-1)
        d = (self.a_factor_shape if side == 'a' else self.g_factor_shape)[0]
        return FactorRows(n, d, lambda out, ld, grad_scale, loss_scale: self._sequence_call(
            t, tap, side, 1.0 / grad_scale, loss_scale, out, ld, reduced))


LINEAR_TYPES: tuple[type, ...] = (torch.nn.Linear,)
CONV2D_TYPES: tuple[type, ...] = (torch.nn.Conv2d,)
CONV_ND_TYPES: tuple[type, ...] = (torch.nn.Conv1d, torch.nn.Conv3d)
CONV_TRANSPOSE_TYPES: tuple[type, ...] = (torch.nn.ConvTranspose1d, torch.nn.ConvTranspose2d, torch.nn.ConvTranspose3d)
EMBEDDING_TYPES: tuple[type, ...] = (torch.nn.Embedding,)
EMBEDDING_BAG_TYPES: tuple[type, ...] = (torch.nn.EmbeddingBag,)
# SyncBatchNorm (global statistics) and BatchNorm3d are in neither tuple; GroupNorm and InstanceNorm* are registered
# through their own keyword (precondition_group_norms)
NORM_TYPES: tuple[type, ...] = (torch.nn.BatchNorm1d, torch.nn.BatchNorm2d, torch.nn.LayerNorm, torch.nn.RMSNorm)
GROUP_NORM_TYPES: tuple[type, ...] = (torch.nn.GroupNorm, torch.nn.InstanceNorm1d, torch.nn.InstanceNorm2d,
                                      torch.nn.InstanceNorm3d)
# registered through their own keyword (precondition_recurrent), as two Linear layers per layer and direction
RECURRENT_TYPES: tuple[type, ...] = (torch.nn.RNN, torch.nn.LSTM, torch.nn.GRU)


def get_module_helper(module: torch.nn.Module, embeddings: bool = False,
                      diagonal_g: bool = False, norms: bool = False, reduce: bool = False,
                      conv_nd: bool = False, conv_transpose: bool = False,
                      group_norms: bool = False, diagonal_a: bool = False,
                      embedding_bags: bool = False) -> ModuleHelper | None:
    """reduce: K-FAC-reduce statistics for Linear (dense and diagonal-G), Conv2d and (with conv_nd) Conv1d / Conv3d
    and (with conv_transpose) ConvTranspose1d / 2d / 3d layers; embeddings, embedding bags and normalization layers keep
    their own statistics.  diagonal_a: a diagonal A for a Linear, Conv2d or (with conv_nd) Conv1d / Conv3d layer; the
    other kinds ignore it (register_modules refuses them)."""
    if isinstance(module, LINEAR_TYPES):
        if diagonal_g:
            return DiagonalGLinearModuleHelper(module, reduce=reduce)
        return LinearModuleHelper(module, reduce=reduce, diagonal_a=diagonal_a)
    if isinstance(module, CONV2D_TYPES):
        return Conv2dModuleHelper(module, reduce=reduce, diagonal_a=diagonal_a)
    if conv_nd and isinstance(module, CONV_ND_TYPES):
        return ConvNdModuleHelper(module, reduce=reduce, diagonal_a=diagonal_a)
    if conv_transpose and isinstance(module, CONV_TRANSPOSE_TYPES):
        return ConvTransposeModuleHelper(module, reduce=reduce)
    if embeddings and isinstance(module, EMBEDDING_TYPES):
        return EmbeddingModuleHelper(module)
    if embedding_bags and isinstance(module, EMBEDDING_BAG_TYPES):
        return EmbeddingBagModuleHelper(module)
    if norms and isinstance(module, NORM_TYPES) and getattr(module, 'weight', None) is not None:
        return NormModuleHelper(module)      # affine=False / elementwise_affine=False: nothing to precondition
    if group_norms and isinstance(module, GROUP_NORM_TYPES) and getattr(module, 'weight', None) is not None:
        return NormModuleHelper(module)      # affine=False: nothing to precondition
    return None


class KFACLayer:
    """Per-layer descriptor.  Attribute names follow the reference layer
    classes (`a_factor`, `g_factor`, `qa`, `qg`, `da`, `dg`, `dgda`, `a_inv`,
    `g_inv`, `grad`) so tests and tools written against them keep working."""

    def __init__(self, module: ModuleHelper, *, method, prediv_eigenvalues: bool = True,
                 grad_scaler: Callable[[], float] | Any | None = None,
                 factor_dtype: torch.dtype | None = None,
                 inv_dtype: torch.dtype = torch.float32,
                 symmetry_aware: bool = False) -> None:
        self.module = module
        self.method = method
        self.prediv_eigenvalues = prediv_eigenvalues
        # a torch.amp.GradScaler (torch.cuda.amp.GradScaler is a subclass) is kept as is: the G hook snapshots its
        # scale on the device into `_g_scale_slot` (no host sync).  Other objects with get_scale() and plain callables
        # are called on the host in every G hook.
        if (grad_scaler is not None and not isinstance(grad_scaler, torch.amp.GradScaler)
                and hasattr(grad_scaler, 'get_scale')):
            grad_scaler = grad_scaler.get_scale
        self.grad_scaler = grad_scaler
        self._g_scale_slot = None               # device float: loss scale of the open G window (bound by the preconditioner)
        self.factor_dtype = factor_dtype
        self.inv_dtype = inv_dtype
        self.symmetry_aware = symmetry_aware
        self.symmetric_factors = module.has_symmetric_factors()
        self.a_dim = module.a_factor_shape[0]
        self.g_dim = module.g_factor_shape[0]
        # A is a vector of a_dim floats (embeddings, diagonal_a_layers)
        self.diag_a = module.diagonal_a
        # an nn.Embedding or EmbeddingBag: its input is indices, and P has the weight's layout (a x g), not (g x a)
        self.embedding = module.embedding
        # G is a vector of g_dim floats (diagonal_g_layers); P keeps the dense layout (g x a)
        self.diag_g = module.diagonal_g
        # normalization layer (precondition_norms): no A factor, G holds the C x k blocks, P is C x a_dim
        # (a_dim = 1 + has_bias); it is preconditioned locally on every rank, outside the work assignment
        self.norm = module.norm
        # tied pair (precondition_tied_embeddings): the embedding holds its head in `tied_head` and carries the pair's
        # placement, second-order data and P; the head holds the embedding in `tied_embedding` and keeps only its
        # factors
        self.tied_head: KFACLayer | None = None
        self.tied_embedding: KFACLayer | None = None
        # pi-adjusted damping (set by the preconditioner): the damping is split between A and G by their trace norms
        self.pi_damping = False
        self.index = -1
        # arena views (bound by the preconditioner)
        self._a_view = self._g_view = None
        self._a_batch_view = self._g_batch_view = None
        self._has_a = self._has_g = False       # running average exists
        self._a_count = self._g_count = 0       # accumulated micro-batches
        self._a_pending = self._g_pending = False
        self._inv = {}                          # name -> storage (rows x ld4(cols)) of qa, qg, da, dg, dgda, a_inv, g_inv
        self._inv_cols = {}                     # name -> logical column count
        self._p_store = None
        self._inv_ready = set()
        self._p_view = None
        self._grad_ready = False
        # EKFAC (bound by the preconditioner): S and S_batch (g x ld4(a) arena views), grow-only row buffers, the
        # rows written in the open factor window, and the guarded EMA's drop flags of that window (device pointers)
        self._S = self._S_batch = None
        self._rows_x = self._rows_g = None
        self._rows_n_a = self._rows_n_g = 0
        self._drop_a = self._drop_g = None

    def __repr__(self) -> str:
        return f'{self.__class__.__name__}({repr(self.module)})'

    @property
    def device_grad_scaler(self) -> bool:
        """True when the loss scale is read on the device (a torch.amp.GradScaler)."""
        return isinstance(self.grad_scaler, torch.amp.GradScaler)

    # -------- reference-compatible read accessors (views into the arenas)
    def _as_factor_dtype(self, t):
        fd = self.factor_dtype
        return t if (t is None or fd in (None, torch.float32)) else t.to(fd)

    @property
    def a_factor(self):
        """Running average A (fp32 arena view; a cast copy when `factor_dtype` is not float32)."""
        return self._as_factor_dtype(self._a_view if self._has_a else None)

    @property
    def g_factor(self):
        return self._as_factor_dtype(self._g_view if self._has_g else None)

    def _inv_get(self, key):
        if key not in self._inv_ready:
            return None
        t = self._inv[key]
        t = t[:, :self._inv_cols[key]] if t.dim() == 2 else t
        # second-order data is stored in fp32; `inv_dtype=float64` readers get a cast copy (eigen.py:319-320)
        return t if self.inv_dtype == torch.float32 else t.to(self.inv_dtype)

    qa = property(lambda self: self._inv_get('qa'))
    qg = property(lambda self: self._inv_get('qg'))
    da = property(lambda self: self._inv_get('da'))
    dg = property(lambda self: self._inv_get('dg'))
    dgda = property(lambda self: self._inv_get('dgda'))
    a_inv = property(lambda self: self._inv_get('a_inv'))
    g_inv = property(lambda self: self._inv_get('g_inv'))

    @property
    def a_factor_shape(self) -> tuple[int, ...]:
        if self.norm:
            return ()           # a normalization layer has no A factor
        return (self.a_dim,) if self.diag_a else (self.a_dim, self.a_dim)

    @property
    def g_factor_shape(self) -> tuple[int, ...]:
        if self.norm:
            return self.module.g_factor_shape
        return (self.g_dim,) if self.diag_g else (self.g_dim, self.g_dim)

    @property
    def diag_side(self) -> str | None:
        """'a' or 'g': the factor kept as a vector (the other one is dense); None for a dense layer."""
        return 'a' if self.diag_a else 'g' if self.diag_g else None

    @property
    def dense_side(self) -> str | None:
        """The dense factor of a diagonal layer ('g' for an embedding or a diagonal-A layer, 'a' for a diagonal-G
        layer)."""
        return {'a': 'g', 'g': 'a'}.get(self.diag_side)

    @property
    def p_shape(self) -> tuple[int, int]:
        """Logical shape of P: (g, a), or the weight layout (a, g) = (V, d) of an embedding."""
        return (self.a_dim, self.g_dim) if self.embedding else (self.g_dim, self.a_dim)

    @property
    def grad(self):
        """Preconditioned gradient P (g x a; V x d for an embedding) while it is pending write-back."""
        return self._p_view if self._grad_ready else None

    def state_dict(self) -> dict[str, torch.Tensor | None]:
        a, g = self.a_factor, self.g_factor
        return {'A': a.clone() if a is not None else None, 'G': g.clone() if g is not None else None}

    def load_state_dict(self, state_dict: dict[str, torch.Tensor | None]) -> None:
        if 'A' not in state_dict or 'G' not in state_dict:
            raise KeyError("KFACLayer state_dict must contain keys 'A' and 'G'")
        if self.diag_side:
            for key, want in (('A', self.a_factor_shape), ('G', self.g_factor_shape)):
                t = state_dict[key]
                if t is not None and tuple(t.shape) != want:
                    kind = ('embedding' if self.embedding else 'diagonal-A layer' if self.diag_a
                            else 'diagonal-G layer')
                    raise ValueError(f'{kind} factor {key} has shape {tuple(t.shape)}, expected {want}')
        elif not self.norm:
            # a vector (a diagonal factor's entry) would broadcast into a dense factor
            for key, want in (('A', self.a_factor_shape), ('G', self.g_factor_shape)):
                t = state_dict[key]
                if t is not None and t.dim() != len(want):
                    raise ValueError(f'factor {key} has shape {tuple(t.shape)}, expected {want}')
        if self.norm:
            if state_dict['A'] is not None:
                raise ValueError('a normalization layer has no A factor (expected None)')
            t = state_dict['G']
            if t is not None and tuple(t.shape) != self.g_factor_shape:
                raise ValueError(f'normalization layer block G has shape {tuple(t.shape)}, '
                                 f'expected {self.g_factor_shape}')
        if state_dict['A'] is not None:
            self._a_view.copy_(state_dict['A'].to(torch.float32))
            self._has_a = True
        if state_dict['G'] is not None:
            self._g_view.copy_(state_dict['G'].to(torch.float32))
            self._has_g = True

    def memory_usage(self) -> dict[str, int]:
        b = 4
        a_numel = 0 if self.norm else self.a_dim if self.diag_a else self.a_dim * self.a_dim
        g_numel = math.prod(self.g_factor_shape)
        out = {
            'a_factors': a_numel * b if self._has_a else 0,
            'g_factors': g_numel * b if self._has_g else 0,
            'a_batch': a_numel * b if self._a_count else 0,
            'g_batch': g_numel * b if self._g_count else 0,
            'a_inverses': 0, 'g_inverses': 0,
        }
        for k in self._inv_ready:
            bucket = 'a_inverses' if k in ('qa', 'da', 'a_inv') else 'g_inverses'
            out[bucket] += self._inv[k].numel() * b
        if self._S is not None:
            out['ekfac'] = sum(t.numel() * b for t in (self._S, self._S_batch, self._rows_x, self._rows_g)
                               if t is not None)
        return out

    def reset_batch(self) -> None:
        if self._a_batch_view is not None:
            self._a_batch_view.zero_()
        if self._g_batch_view is not None:
            self._g_batch_view.zero_()
        self._a_count = self._g_count = 0
        self._a_pending = self._g_pending = False
        self._rows_n_a = self._rows_n_g = 0
        self._drop_a = self._drop_g = None


def any_match(query: str, patterns: list[str]) -> bool:
    return any(re.compile(p).search(query) for p in patterns)


def register_modules(model: torch.nn.Module, skip_layers: list[str], precondition_embeddings: bool = False,
                     diagonal_g_layers: list[str] | None = None, precondition_norms: bool = False,
                     kfac_approx: str = 'expand', precondition_attention: bool = False,
                     precondition_conv_nd: bool = False, precondition_conv_transpose: bool = False,
                     precondition_group_norms: bool = False, precondition_recurrent: bool = False,
                     diagonal_a_layers: list[str] | None = None, precondition_embedding_bags: bool = False,
                     **layer_kwargs: Any) -> dict[torch.nn.Module, tuple[str, KFACLayer]]:
    """Leaf-module discovery with regex skip on name and class name
    (kfac/layers/register.py:57-95).  precondition_embeddings: also register torch.nn.Embedding
    modules (not in the reference).  diagonal_g_layers: regexes on name and class name; a registered
    torch.nn.Linear that matches keeps a diagonal G (not in the reference); any other registered
    module that matches is an error.  precondition_norms: also register BatchNorm1d/2d, LayerNorm and
    RMSNorm modules with affine parameters (not in the reference; `layer.norm`).  kfac_approx: 'expand'
    or 'reduce' (K-FAC-reduce statistics for the Linear and Conv2d layers; not in the reference).
    precondition_attention: register every torch.nn.MultiheadAttention as four projections named
    `{name}.q_proj`, `.k_proj`, `.v_proj` and `.out_proj`, keyed by their AttentionProjectionHelper
    (not in the reference); the `out_proj` leaf of an attention is then never registered as a Linear.
    precondition_conv_nd: also register torch.nn.Conv1d and Conv3d modules (not in the reference); grouped ones and
    ones whose factors exceed the eigensolver are an error.  precondition_conv_transpose: also register
    torch.nn.ConvTranspose1d, 2d and 3d modules (not in the reference), with the same errors.
    precondition_group_norms: also register GroupNorm and InstanceNorm1d/2d/3d modules with affine parameters (not in
    the reference; `layer.norm`).  precondition_recurrent: register every torch.nn.RNN, LSTM and GRU as two Linear
    layers per layer k and direction, `{name}.ih_l{k}{sfx}` and `{name}.hh_l{k}{sfx}`, keyed by their
    RecurrentSubLayerHelper (not in the reference).  diagonal_a_layers: regexes on name and class name; a registered
    torch.nn.Linear, Conv2d or (precondition_conv_nd) Conv1d / Conv3d that matches keeps a diagonal A and may have an A
    above the eigensolver's limit (not in the reference); any other registered module that matches, a match of
    diagonal_g_layers too and a G above the limit are errors.  precondition_embedding_bags: also register
    torch.nn.EmbeddingBag modules (not in the reference).  `layer.index` counts the other layers and the
    normalization layers separately."""
    diagonal_g_layers = diagonal_g_layers or []
    diagonal_a_layers = diagonal_a_layers or []
    layers: dict[torch.nn.Module, tuple[str, KFACLayer]] = {}
    counts = [0, 0]
    out_projs = ({id(m.out_proj) for m in model.modules() if isinstance(m, torch.nn.MultiheadAttention)}
                 if precondition_attention else set())
    for name, module in model.named_modules():
        if precondition_attention and isinstance(module, torch.nn.MultiheadAttention):
            for helper in _attention_projections(name, module, skip_layers, diagonal_g_layers, kfac_approx,
                                                 diagonal_a_layers):
                layer = KFACLayer(helper, **layer_kwargs)
                layer.index = counts[0]
                counts[0] += 1
                layers[helper] = (f'{name}.{helper.which}_proj', layer)
            continue
        if precondition_recurrent and isinstance(module, RECURRENT_TYPES):
            for helper in _recurrent_sublayers(name, module, skip_layers, diagonal_g_layers, kfac_approx,
                                               diagonal_a_layers):
                layer = KFACLayer(helper, **layer_kwargs)
                layer.index = counts[0]
                counts[0] += 1
                layers[helper] = (f'{name}.{helper.suffix}', layer)
            continue
        if len(list(module.children())) != 0 or id(module) in out_projs:
            continue
        if any_match(name, skip_layers) or any_match(module.__class__.__name__, skip_layers):
            continue
        if not all(p.requires_grad for p in module.parameters()):
            continue
        diag_g = any_match(name, diagonal_g_layers) or any_match(module.__class__.__name__, diagonal_g_layers)
        diag_a = any_match(name, diagonal_a_layers) or any_match(module.__class__.__name__, diagonal_a_layers)
        helper = get_module_helper(module, embeddings=precondition_embeddings, diagonal_g=diag_g,
                                   norms=precondition_norms, reduce=kfac_approx == 'reduce',
                                   conv_nd=precondition_conv_nd, conv_transpose=precondition_conv_transpose,
                                   group_norms=precondition_group_norms, diagonal_a=diag_a and not diag_g,
                                   embedding_bags=precondition_embedding_bags)
        if helper is None:
            continue
        if diag_g and not helper.diagonal_g:
            raise ValueError(f'diagonal_g_layers matches "{name}" ({module.__class__.__name__}): only torch.nn.Linear '
                             'layers can keep a diagonal G (add it to skip_layers or narrow the pattern)')
        if diag_a:
            _check_diagonal_a(name, module, helper, diag_g)
        if isinstance(helper, ConvNdModuleHelper):
            helper.check(name)
        assert module not in layers
        layer = KFACLayer(helper, **layer_kwargs)
        layer.index = counts[helper.norm]
        counts[helper.norm] += 1
        layers[module] = (name, layer)
    # a projection weight that another registered module also owns would have its gradient preconditioned twice (the
    # projections of one attention share in_proj_weight / in_proj_bias by design)
    owners: dict[int, list[tuple[Any, str]]] = {}
    for key, (name, _) in layers.items():
        owner = (key.attn if isinstance(key, AttentionProjectionHelper) else key.rnn
                 if isinstance(key, RecurrentSubLayerHelper) else key)
        for p in key.parameters():
            owners.setdefault(id(p), []).append((owner, name))
    for key, (name, _) in layers.items():
        if isinstance(key, AttentionProjectionHelper):
            for p in key.parameters():
                other = next((n for o, n in owners[id(p)] if o is not key.attn), None)
                if other is not None:
                    raise ValueError(f'attention projection "{name}" shares a weight with "{other}": two layers '
                                     'would precondition one gradient; add one of them to skip_layers')
        if isinstance(key, RecurrentSubLayerHelper):
            for p in key.parameters():
                other = next((n for o, n in owners[id(p)] if o is not key.rnn), None)
                if other is not None:
                    raise ValueError(f'recurrent sub-layer "{name}" shares a weight with "{other}": two layers would '
                                     'precondition one gradient; add one of them to skip_layers')
    return layers


def _check_diagonal_a(name: str, module: torch.nn.Module, helper: ModuleHelper, diag_g: bool) -> None:
    """Refuse a diagonal_a_layers match that cannot keep a diagonal A."""
    cls = module.__class__.__name__
    if diag_g:
        raise ValueError(f'diagonal_a_layers and diagonal_g_layers both match "{name}" ({cls}): a layer keeps at most '
                         'one diagonal factor (add it to skip_layers or narrow a pattern)')
    if helper.embedding or not helper.diagonal_a:
        raise ValueError(f'diagonal_a_layers matches "{name}" ({cls}): only torch.nn.Linear, Conv2d and (with '
                         'precondition_conv_nd) Conv1d / Conv3d layers can keep a diagonal A (add it to skip_layers or '
                         'narrow the pattern)')
    g = helper.g_factor_shape[0]
    if g > _cabi.KFAC_EIGH_MAX_N:
        raise ValueError(f'diagonal_a_layers matches "{name}" ({cls}), whose G factor of {g} exceeds '
                         f'KFAC_EIGH_MAX_N = {_cabi.KFAC_EIGH_MAX_N}; add it to skip_layers')


def _attention_projections(name: str, module: torch.nn.MultiheadAttention, skip_layers: list[str],
                           diagonal_g_layers: list[str], kfac_approx: str,
                           diagonal_a_layers: list[str]) -> list[AttentionProjectionHelper]:
    """The registered projections of one attention: none when skip_layers matches its name or class or one of its
    parameters is frozen, else those whose name `{name}.{q,k,v,out}_proj` skip_layers does not match."""
    cls = module.__class__.__name__
    if any_match(name, skip_layers) or any_match(cls, skip_layers):
        return []
    if not all(p.requires_grad for p in module.parameters()):
        return []
    if type(module) not in (torch.nn.MultiheadAttention, KFACMultiheadAttention):
        raise ValueError(f'precondition_attention: "{name}" is a {cls}, a subclass of torch.nn.MultiheadAttention '
                         'whose forward cannot be tapped; add it to skip_layers')
    for flag, what in ((module.bias_k is not None, 'add_bias_kv=True'), (module.add_zero_attn, 'add_zero_attn=True')):
        if flag:
            raise ValueError(f'precondition_attention does not support {what} (attention "{name}"); add it to '
                             'skip_layers')
    helpers = []
    for which in ('q', 'k', 'v', 'out'):
        pname = f'{name}.{which}_proj'
        if any_match(pname, skip_layers):
            continue
        if any_match(name, diagonal_g_layers) or any_match(cls, diagonal_g_layers) or any_match(pname,
                                                                                               diagonal_g_layers):
            raise ValueError(f'diagonal_g_layers matches the attention projection "{pname}": attention projections '
                             'cannot keep a diagonal G (add it to skip_layers or narrow the pattern)')
        if any(any_match(q, diagonal_a_layers) for q in (name, cls, pname)):
            raise ValueError(f'diagonal_a_layers matches the attention projection "{pname}": attention projections '
                             'cannot keep a diagonal A (add it to skip_layers or narrow the pattern)')
        helpers.append(AttentionProjectionHelper(module, which, reduce=kfac_approx == 'reduce'))
    return helpers


def _recurrent_sublayers(name: str, module: torch.nn.Module, skip_layers: list[str], diagonal_g_layers: list[str],
                         kfac_approx: str, diagonal_a_layers: list[str]) -> list[RecurrentSubLayerHelper]:
    """The registered sub-layers of one RNN / LSTM / GRU: none when skip_layers matches its name or class or one of its
    parameters is frozen, else those whose name `{name}.{ih,hh}_l{k}{sfx}` skip_layers does not match."""
    cls = module.__class__.__name__
    if any_match(name, skip_layers) or any_match(cls, skip_layers):
        return []
    if not all(p.requires_grad for p in module.parameters()):
        return []
    if type(module) not in RECURRENT_SWAPPED and type(module) not in RECURRENT_SWAPPED.values():
        base = module.mode.split('_')[0]
        raise ValueError(f'precondition_recurrent: "{name}" is a {cls}, a subclass of torch.nn.{base} whose forward '
                         'cannot be tapped; add it to skip_layers')
    if getattr(module, 'proj_size', 0) > 0:
        raise ValueError(f'precondition_recurrent does not support proj_size > 0 (LSTM "{name}"); add it to skip_layers')
    helpers = []
    for k in range(module.num_layers):
        for d in range(2 if module.bidirectional else 1):
            for side in ('ih', 'hh'):
                helper = RecurrentSubLayerHelper(module, k, d, side, reduce=kfac_approx == 'reduce')
                sname = f'{name}.{helper.suffix}'
                if any_match(sname, skip_layers):
                    continue
                if any(any_match(q, diagonal_g_layers) for q in (name, cls, sname)):
                    raise ValueError(f'diagonal_g_layers matches the recurrent sub-layer "{sname}": recurrent layers '
                                     'cannot keep a diagonal G (add it to skip_layers or narrow the pattern)')
                if any(any_match(q, diagonal_a_layers) for q in (name, cls, sname)):
                    raise ValueError(f'diagonal_a_layers matches the recurrent sub-layer "{sname}": recurrent layers '
                                     'cannot keep a diagonal A (add it to skip_layers or narrow the pattern)')
                n = max(helper.a_factor_shape[0], helper.g_factor_shape[0])
                if n > _cabi.KFAC_EIGH_MAX_N:
                    raise ValueError(f'recurrent sub-layer "{sname}" has a factor of {n} > KFAC_EIGH_MAX_N = '
                                     f'{_cabi.KFAC_EIGH_MAX_N}; add it to skip_layers')
                helpers.append(helper)
    return helpers
