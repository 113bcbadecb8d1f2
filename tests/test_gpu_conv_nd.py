"""Conv1d / Conv3d layers (`precondition_conv_nd=True`) on the GPU:

  * the three N-d input kernels (factor, EKFAC rows, K-FAC-reduce rows) against an fp64 im2col built from F.pad and
    Tensor.unfold, over 1-D and 3-D geometries with strides, dilation and asymmetric padding, in fp32, fp16 and bf16,
    with and without the ones column; a workspace forcing several im2col chunks against one chunk;
  * twins, bitwise: a Conv1d layer and its Conv2d twin with kernel (1, k), and a Conv3d layer with kd = 1, D = 1 and its
    Conv2d twin, give identical A, G and preconditioned gradients under EIGEN, INVERSE and EKFAC (K-FAC-reduce: fp32
    tolerance);
  * a dilated TCN and a small 3-D conv net against an fp64 restatement (factors -> eigh -> P) under EIGEN, INVERSE and
    EKFAC, expand and reduce, with a schedule and accumulation_steps; unbatched inputs and the non-'zeros' padding modes;
  * fp16 autocast with a GradScaler and a dropped overflow window; other layers unaffected by the keyword; two ranks
    (tests/dist_conv_nd.py).
"""
import ctypes
import math
import os
import socket
import subprocess
import sys
import zlib

import pytest
import torch
from torch import nn
from torch.nn import functional as F

from conftest import rel_fro

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda')
DTYPES = [torch.float32, torch.float16, torch.bfloat16]


@pytest.fixture(scope='module')
def lib():
    from kfac_b200 import _cabi
    return _cabi.load()


def S():
    return torch.cuda.current_stream().cuda_stream


def _ld4(n):
    return (n + 3) & ~3


def _code(dtype):
    from kfac_b200 import _cabi
    return _cabi.DTYPE_CODE[dtype]


# ---------------------------------------------------------------------------------------------- kernels
# (B, C, in, kernel, stride, dilation, pad_before, pad_after), per axis in (D, H, W) order
GEOS = [
    (3, 2, (1, 1, 4003), (1, 1, 7), (1, 1, 3), (1, 1, 2), (0, 0, 5), (0, 0, 4)),       # long 1-D, asymmetric padding
    (2, 1, (1, 1, 16000), (1, 1, 10), (1, 1, 5), (1, 1, 1), (0, 0, 0), (0, 0, 0)),     # the wav2vec2 stem
    (2, 5, (1, 1, 37), (1, 1, 4), (1, 1, 1), (1, 1, 3), (0, 0, 4), (0, 0, 5)),         # 'same', even kernel
    (2, 3, (5, 7, 9), (3, 3, 3), (1, 1, 1), (1, 1, 1), (1, 1, 1), (1, 1, 1)),
    (2, 4, (6, 10, 11), (1, 3, 3), (1, 2, 2), (1, 1, 1), (0, 1, 1), (0, 1, 1)),
    (3, 6, (7, 5, 6), (3, 1, 1), (1, 1, 1), (2, 1, 1), (2, 0, 0), (2, 0, 0)),
    (2, 3, (9, 11, 13), (2, 2, 2), (2, 2, 2), (2, 2, 2), (1, 0, 2), (0, 1, 1)),
    (2, 64, (3, 5, 7), (1, 1, 1), (1, 1, 1), (1, 1, 1), (0, 0, 0), (0, 0, 0)),         # 1 x 1 x 1: packed (35 % 4)
    (2, 16, (2, 4, 6), (1, 1, 1), (1, 1, 1), (1, 1, 1), (0, 0, 0), (0, 0, 0)),         # 1 x 1 x 1: in place
    (2, 3, (1, 1, 29), (1, 1, 3), (1, 3, 2), (1, 1, 1), (0, 1, 1), (0, 1, 1)),         # H = 1, the output row is padding
    (2, 3, (1, 2, 9), (1, 2, 3), (3, 1, 1), (1, 1, 1), (1, 0, 1), (1, 0, 1)),          # D = 1, the output plane is padding
]


def _geo(g):
    from kfac_b200 import _cabi
    B, C, ins, k, s, d, pb, pa = g
    arr = lambda v: (ctypes.c_int * 3)(*v)  # noqa: E731
    return _cabi.ConvGeometry(B, C, arr(ins), arr(k), arr(s), arr(d), arr(pb), arr(pa))


def _out(g):
    _, _, ins, k, s, d, pb, pa = g
    return [(ins[a] + pb[a] + pa[a] - d[a] * (k[a] - 1) - 1) // s[a] + 1 for a in range(3)]


def _im2col64(x, g):
    """(B, S, C*kd*kh*kw) fp64 im2col of x (B, C, D, H, W) from F.pad and Tensor.unfold."""
    _, _, _, k, s, d, pb, pa = g
    x = F.pad(x.double(), (pb[2], pa[2], pb[1], pa[1], pb[0], pa[0]))
    for a in range(3):
        x = x.unfold(2 + a, d[a] * (k[a] - 1) + 1, s[a])
    x = x[..., ::d[0], ::d[1], ::d[2]]
    B, C = x.shape[:2]
    return x.permute(0, 2, 3, 4, 1, 5, 6, 7).reshape(B, -1, C * k[0] * k[1] * k[2])


def _input(g, dtype):
    B, C, ins = g[:3]
    gen = torch.Generator(device=DEV).manual_seed(zlib.crc32(repr(g).encode()))
    return (torch.randn(B, C, *ins, device=DEV, generator=gen) + 0.3).to(dtype)


def _factor(lib, x, geo, ones, scale, ws_bytes, d):
    acc = torch.zeros(d, d, device=DEV)
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=DEV)
    rc = lib.kfac_factor_conv_input(x.data_ptr(), _code(x.dtype), ctypes.byref(geo), ones, scale, acc.data_ptr(),
                                    ws.data_ptr(), ws_bytes, S())
    assert rc == 0, lib.kfac_last_error()
    torch.cuda.synchronize()
    return acc


@pytest.mark.parametrize('ones', [0, 1])
@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('g', GEOS, ids=lambda g: f'{g[2]}-k{g[3]}s{g[4]}d{g[5]}')
def test_input_kernels_against_fp64(lib, g, dtype, ones):
    x = _input(g, dtype)
    geo = _geo(g)
    B = g[0]
    U = _im2col64(x, g)
    Sp = U.shape[1]
    assert Sp == math.prod(_out(g))
    if ones:
        U = torch.cat([U, U.new_ones(B, Sp, 1)], 2)
    d = U.shape[2]
    rows = U.reshape(B * Sp, d)
    # factor: scale * X^T X
    need = lib.kfac_factor_conv_input_workspace_bytes(ctypes.byref(geo), ones, 1 << 30)
    acc = _factor(lib, x, geo, ones, 1.0 / (B * Sp), need, d)
    assert rel_fro(acc, rows.T @ rows / (B * Sp)) <= 1e-5
    assert torch.equal(acc, _factor(lib, x, geo, ones, 1.0 / (B * Sp), need, d))
    # EKFAC rows, sample-major, scale 1/S
    ld = _ld4(d)
    out = torch.full((B * Sp, ld), float('nan'), device=DEV)
    assert lib.kfac_rows_conv_input(x.data_ptr(), _code(dtype), ctypes.byref(geo), ones, 1.0 / Sp, out.data_ptr(), ld,
                                    S()) == 0, lib.kfac_last_error()
    torch.cuda.synchronize()
    assert rel_fro(out[:, :d], rows / Sp) <= 1e-6 and not out[:, d:].any()
    # K-FAC-reduce rows: per-example window sums
    for ldr in (d, ld):
        red = torch.full((B, ldr), float('nan'), device=DEV)
        assert lib.kfac_reduce_rows_conv_input(x.data_ptr(), _code(dtype), ctypes.byref(geo), ones, 0.5,
                                               red.data_ptr(), ldr, S()) == 0, lib.kfac_last_error()
        torch.cuda.synchronize()
        assert rel_fro(red[:, :d], U.sum(1) * 0.5) <= 1e-6 and not red[:, d:].any()
        again = torch.empty_like(red)
        assert lib.kfac_reduce_rows_conv_input(x.data_ptr(), _code(dtype), ctypes.byref(geo), ones, 0.5,
                                               again.data_ptr(), ldr, S()) == 0
        torch.cuda.synchronize()
        assert torch.equal(red, again)


@pytest.mark.parametrize('g', [GEOS[0], GEOS[3], GEOS[6]], ids=['1d', '3d', '3d-s2d2'])
def test_chunked_im2col(lib, g):
    """A workspace of one or two examples' im2col gives the factor of one chunk (fp32 tolerance), the same bits on a
    repeat call, and the workspace query sizes chunks from its byte limit."""
    g = (5,) + g[1:]
    x = _input(g, torch.float32)
    geo = _geo(g)
    d = g[1] * math.prod(g[3]) + 1
    Sp = math.prod(_out(g))
    whole = lib.kfac_factor_conv_input_workspace_bytes(ctypes.byref(geo), 1, 1 << 30)
    one = lib.kfac_factor_conv_input_workspace_bytes(ctypes.byref(geo), 1, 0)       # at least one example
    two = lib.kfac_factor_conv_input_workspace_bytes(ctypes.byref(geo), 1, 2 * _ld4(Sp) * d * 4 + 64)
    # the query stays under its cap unless one example's matrix and partials alone exceed it
    assert one <= two <= max(2 * _ld4(Sp) * d * 4 + 64, one) and one < whole
    ref = _factor(lib, x, geo, 1, 1.0 / (5 * Sp), whole, d)
    for ws in (one, two, one + 1024):
        got = _factor(lib, x, geo, 1, 1.0 / (5 * Sp), ws, d)
        assert rel_fro(got, ref) <= 1e-5, (ws, rel_fro(got, ref))
        assert torch.equal(got, _factor(lib, x, geo, 1, 1.0 / (5 * Sp), ws, d))
    # one example's matrix fits but not its SYRK partials: one example per chunk, the SYRK unsplit
    pack1 = _ld4(Sp) * d * 4
    assert pack1 < one
    got = _factor(lib, x, geo, 1, 1.0 / (5 * Sp), pack1, d)
    assert rel_fro(got, ref) <= 1e-5 and torch.equal(got, _factor(lib, x, geo, 1, 1.0 / (5 * Sp), pack1, d))
    # the query fits matrix and partials under its cap
    assert lib.kfac_factor_conv_input_workspace_bytes(ctypes.byref(geo), 1, two) <= two
    # too small for one example's matrix
    acc = torch.zeros(d, d, device=DEV)
    assert lib.kfac_factor_conv_input(x.data_ptr(), 0, ctypes.byref(geo), 1, 1.0, acc.data_ptr(), None, 0, S()) != 0


@pytest.mark.parametrize('g2', [(3, 5, 13, 11, 3, 5, 2, 1, 1, 2), (2, 4, 1, 23, 1, 3, 3, 2, 1, 1)],
                         ids=['3x5', 'single-row-padded'])
def test_conv2d_entries_are_the_depth_one_geometry(lib, g2):
    """The Conv2d entry points give the bits of the N-d ones on the depth-1, dilation-1 geometry, including a height-1
    input whose one output row lies in the padding (its window sums are 0)."""
    B, C, H, W, kh, kw, sh, sw, ph, pw = g2
    g = (B, C, (1, H, W), (1, kh, kw), (1, sh, sw), (1, 1, 1), (0, ph, pw), (0, ph, pw))
    geo = _geo(g)
    for dtype in DTYPES:
        x = _input(g, dtype)
        d = C * kh * kw + 1
        need = lib.kfac_factor_conv2d_input_workspace_bytes(B, C, H, W, kh, kw, sh, sw, ph, pw, 1)
        ws = torch.empty(need, dtype=torch.uint8, device=DEV)
        a2 = torch.zeros(d, d, device=DEV)
        assert lib.kfac_factor_conv2d_input(x.data_ptr(), _code(dtype), B, C, H, W, kh, kw, sh, sw, ph, pw, 1, 0.25,
                                            a2.data_ptr(), ws.data_ptr(), need, S()) == 0
        assert torch.equal(a2, _factor(lib, x, geo, 1, 0.25, need, d))
        Sp = math.prod(_out(g))
        r2, rn = (torch.empty(B * Sp, _ld4(d), device=DEV) for _ in range(2))
        assert lib.kfac_rows_conv2d_input(x.data_ptr(), _code(dtype), B, C, H, W, kh, kw, sh, sw, ph, pw, 1, 0.5,
                                          r2.data_ptr(), _ld4(d), S()) == 0
        assert lib.kfac_rows_conv_input(x.data_ptr(), _code(dtype), ctypes.byref(geo), 1, 0.5, rn.data_ptr(), _ld4(d),
                                        S()) == 0
        q2, qn = (torch.empty(B, d, device=DEV) for _ in range(2))
        assert lib.kfac_reduce_rows_conv2d_input(x.data_ptr(), _code(dtype), B, C, H, W, kh, kw, sh, sw, ph, pw, 1, 0.5,
                                                 q2.data_ptr(), d, S()) == 0
        assert lib.kfac_reduce_rows_conv_input(x.data_ptr(), _code(dtype), ctypes.byref(geo), 1, 0.5, qn.data_ptr(), d,
                                               S()) == 0
        torch.cuda.synchronize()
        assert torch.equal(r2, rn) and torch.equal(q2, qn)
        U = _im2col64(x, g)
        want = torch.cat([U.sum(1), U.new_full((B, 1), U.shape[1])], 1) * 0.5
        assert rel_fro(q2, want) <= 1e-6
        if g2[2] == 1 and g2[6] > 2 * g2[8]:
            assert not q2[:, :-1].any()         # the one output row lies in the padding


@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('shape', [(2, 1, 16000, 10, 5), (3, 2, 4003, 7, 3), (2, 8, 37, 4, 1)], ids=str)
def test_single_row_kernel_is_bitwise_the_general_one(lib, shape, dtype):
    """A single-row input (1-D kernel) gives the bits of the general kernel on the same row inside a two-row input whose
    second row no window touches (kh = 1, sh = 2: Ho = 1)."""
    B, C, W, kw, sw = shape
    g1 = (B, C, (1, 1, W), (1, 1, kw), (1, 1, sw), (1, 1, 1), (0, 0, 2), (0, 0, 1))
    g2 = (B, C, (1, 2, W), (1, 1, kw), (1, 2, sw), (1, 1, 1), (0, 0, 2), (0, 0, 1))
    x2 = _input(g2, dtype)
    x1 = x2[:, :, :, :1].contiguous()
    d = C * kw + 1
    outs = []
    for x, g in ((x1, g1), (x2, g2)):
        o = torch.empty(B, d, device=DEV)
        assert lib.kfac_reduce_rows_conv_input(x.data_ptr(), _code(dtype), ctypes.byref(_geo(g)), 1, 0.25, o.data_ptr(),
                                               d, S()) == 0, lib.kfac_last_error()
        outs.append(o)
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1])


def test_reject_bad_geometry(lib):
    x = torch.zeros(64, device=DEV)
    out = torch.zeros(64, device=DEV)
    bad = [(1, 1, (1, 1, 3), (1, 1, 5), (1, 1, 1), (1, 1, 1), (0, 0, 0), (0, 0, 0)),    # empty output
           (1, 1, (1, 1, 8), (1, 1, 3), (1, 1, 0), (1, 1, 1), (0, 0, 0), (0, 0, 0)),    # stride 0
           (1, 1, (1, 1, 8), (1, 1, 3), (1, 1, 1), (1, 1, 0), (0, 0, 0), (0, 0, 0))]    # dilation 0
    for g in bad:
        geo = _geo(g)
        assert lib.kfac_factor_conv_input_workspace_bytes(ctypes.byref(geo), 0, 1 << 20) == 0
        assert lib.kfac_rows_conv_input(x.data_ptr(), 0, ctypes.byref(geo), 0, 1.0, out.data_ptr(), 4, S()) != 0
        assert lib.kfac_reduce_rows_conv_input(x.data_ptr(), 0, ctypes.byref(geo), 0, 1.0, out.data_ptr(), 4, S()) != 0


# ---------------------------------------------------------------------------------------------- twins
def _twin_models(kind):
    torch.manual_seed(5)
    if kind == '1d':
        nd = nn.Conv1d(4, 6, 5, stride=2, padding=2)
        tw = nn.Conv2d(4, 6, (1, 5), stride=(1, 2), padding=(0, 2))
        x = lambda gen: torch.randn(8, 4, 301, generator=gen)  # noqa: E731
        to2d = lambda t: t.unsqueeze(2)  # noqa: E731
    else:
        nd = nn.Conv3d(4, 6, (1, 3, 3), stride=(1, 2, 2), padding=(0, 1, 1))
        tw = nn.Conv2d(4, 6, 3, stride=2, padding=1)
        x = lambda gen: torch.randn(8, 4, 1, 23, 17, generator=gen)  # noqa: E731
        to2d = lambda t: t.squeeze(2)  # noqa: E731
    with torch.no_grad():
        tw.weight.copy_(nd.weight.view_as(tw.weight))
        tw.bias.copy_(nd.bias)
    return nn.Sequential(nd).to(DEV), nn.Sequential(tw).to(DEV), x, to2d


@pytest.mark.parametrize('approx', ['expand', 'reduce'])
@pytest.mark.parametrize('method', ['eigen', 'inverse', 'ekfac'])
@pytest.mark.parametrize('kind', ['1d', '3d'])
def test_twin_of_conv2d(kind, method, approx):
    from kfac_b200.preconditioner import KFACPreconditioner
    nd, tw, xs, to2d = _twin_models(kind)
    kw = dict(compute_method=method, kfac_approx=approx, damping=0.003, factor_update_steps=1,
              inv_update_steps=1 if method == 'ekfac' else 2)
    p_nd = KFACPreconditioner(nd, precondition_conv_nd=True, **kw)
    p_tw = KFACPreconditioner(tw, **kw)
    (_, l_nd), = p_nd._layers.values()
    (_, l_tw), = p_tw._layers.values()
    gen = torch.Generator().manual_seed(2)
    for s in range(4):
        x = xs(gen).to(DEV)
        nd.zero_grad()
        tw.zero_grad()
        y_tw = tw(to2d(x))
        R = torch.randn(y_tw.shape, generator=gen).to(DEV)
        (y_tw * R).sum().backward()                                  # the output gradient is R, exactly
        (nd(x).view_as(y_tw) * R).sum().backward()
        with torch.no_grad():                                        # the same weight gradient for both
            nd[0].weight.grad.copy_(tw[0].weight.grad.view_as(nd[0].weight))
            nd[0].bias.grad.copy_(tw[0].bias.grad)
        p_nd.step()
        p_tw.step()
        torch.cuda.synchronize()
        pairs = [(l_nd.a_factor, l_tw.a_factor), (l_nd.g_factor, l_tw.g_factor),
                 (nd[0].weight.grad.flatten(), tw[0].weight.grad.flatten()), (nd[0].bias.grad, tw[0].bias.grad)]
        for i, (u, v) in enumerate(pairs):
            if approx == 'expand':
                assert torch.equal(u, v), (s, i)
            else:
                assert rel_fro(u, v) <= 1e-5, (s, i, rel_fro(u, v))
        with torch.no_grad():
            for p, q in zip(nd.parameters(), tw.parameters()):
                p.copy_(q.view_as(p) - 0.05 * q.grad.view_as(p))
                q.sub_(0.05 * q.grad)


# ---------------------------------------------------------------------------------------------- module level
class _Rec:
    """Every call's input and output gradient of every registered layer (lists in hook order)."""

    def __init__(self, layers):
        self.inp, self.gout = {}, {}
        for m in layers:
            m.register_forward_pre_hook(lambda mod, i: self.inp.setdefault(mod, []).append(i[0].detach().clone()))
            m.register_full_backward_hook(lambda mod, gi, go: self.gout.setdefault(mod, []).append(go[0].detach().clone()))

    def clear(self):
        self.inp, self.gout = {}, {}


def _rows64(m, x, g, reduce):
    """fp64 rows (X, G) of one call, restated from the definition: the module's padding applied with F.pad, the
    dilated windows cut with Tensor.unfold, rows scaled by 1/S (reduce: the per-example mean of X, sum of G / sqrt(S))."""
    if isinstance(m, nn.Linear):
        x, g = x.double().reshape(-1, x.shape[-1]), g.double().reshape(-1, g.shape[-1])
        X = torch.cat([x, x.new_ones(x.shape[0], 1)], 1) if m.bias is not None else x
        return X, g
    nd = len(m.kernel_size)
    x, g = x.double(), g.double()
    if x.dim() == nd + 1:
        x, g = x.unsqueeze(0), g.unsqueeze(0)
    x = F.pad(x, m._reversed_padding_repeated_twice, mode='constant' if m.padding_mode == 'zeros' else m.padding_mode)
    for a in range(nd):
        x = x.unfold(2 + a, m.dilation[a] * (m.kernel_size[a] - 1) + 1, m.stride[a])
    x = x[(Ellipsis,) + tuple(slice(None, None, d) for d in m.dilation)]
    B, C = x.shape[:2]
    Sp = math.prod(x.shape[2:2 + nd])
    assert Sp == math.prod(g.shape[2:])
    X = x.permute(0, *range(2, 2 + nd), 1, *range(2 + nd, 2 + 2 * nd)).reshape(B, Sp, -1) / Sp
    if m.bias is not None:
        X = torch.cat([X, X.new_full((B, Sp, 1), 1.0 / Sp)], 2)
    G = g.flatten(2).transpose(1, 2) / Sp
    if reduce and Sp > 1:
        return X.mean(1), G.sum(1) / math.sqrt(Sp)
    return X.reshape(B * Sp, -1), G.reshape(B * Sp, -1)


def _grad_matrix(module):
    g = module.weight.grad.reshape(module.weight.grad.size(0), -1)
    if module.bias is not None:
        g = torch.cat([g, module.bias.grad.view(-1, 1)], 1)
    return g.detach().double()


def _run(model, batches, loss_fn, method, approx, steps, ius=1, acc=1, damping=0.003, alpha=0.9, tol=1e-3, kw=None,
         fus=1):
    """Train `steps` steps and check every registered layer's A, G (and S under EKFAC) and preconditioned gradient
    against fp64 after each; factors are formed every `fus` steps, second-order data every `ius` steps."""
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    pre = KFACPreconditioner(model, compute_method=method, kfac_approx=approx, factor_update_steps=fus,
                             inv_update_steps=ius, damping=damping,
                             factor_decay=alpha, kl_clip=None, accumulation_steps=acc, precondition_conv_nd=True,
                             **(kw or {}))
    rec = _Rec(pre._layers)
    A, G, Sm, snap = {}, {}, {}, {}
    opt = torch.optim.SGD(model.parameters(), lr=0.01)
    reduce = approx == 'reduce'
    for s in range(steps):
        opt.zero_grad()
        calls = {m: [] for m in pre._layers}
        for k in range(acc):
            rec.clear()
            x, y = batches(s * acc + k)
            loss_fn(model(x), y).backward()
            for m in pre._layers:
                calls[m].append(list(zip(rec.inp[m], reversed(rec.gout[m]))))
        grads = {name: _grad_matrix(m) for m, (name, _) in pre._layers.items()}
        pre.step()
        torch.cuda.synchronize()
        for m, (name, layer) in pre._layers.items():
            eye = lambda n: torch.eye(n, dtype=torch.float64, device=DEV)  # noqa: E731
            if s % fus == 0:
                wa, wg = 0.0, 0.0
                for mb in calls[m]:
                    for xx, gg in mb:
                        X, Gr = _rows64(m, xx, gg, reduce)
                        wa = wa + X.T @ X / X.shape[0] / acc
                        wg = wg + Gr.T @ Gr / Gr.shape[0] / acc
                A[name] = alpha * A.get(name, eye(wa.shape[0])) + (1 - alpha) * wa
                G[name] = alpha * G.get(name, eye(wg.shape[0])) + (1 - alpha) * wg
            assert rel_fro(layer.a_factor, A[name]) <= 1e-5, (s, name, 'A', rel_fro(layer.a_factor, A[name]))
            assert rel_fro(layer.g_factor, G[name]) <= 1e-5, (s, name, 'G', rel_fro(layer.g_factor, G[name]))
            if s % ius == 0:
                da, qa = torch.linalg.eigh(A[name])
                dg, qg = torch.linalg.eigh(G[name])
                snap[name] = (A[name], G[name], da.clamp(min=0), qa, dg.clamp(min=0), qg)
            An, Gn, da, qa, dg, qg = snap[name]
            grad = grads[name]
            if method == 'inverse':
                want = (torch.linalg.inv(Gn + damping * eye(Gn.shape[0])) @ grad
                        @ torch.linalg.inv(An + damping * eye(An.shape[0])))
            elif method == 'eigen':
                want = qg @ ((qg.T @ grad @ qa) / (torch.outer(dg, da) + damping)) @ qa.T
            else:
                Qa, Qg = layer.qa.double(), layer.qg.double()
                if s % fus == 0:
                    X, Gr = _rows64(m, *calls[m][0][0], reduce)
                    Sb = ((Gr @ Qg) ** 2).T @ ((X @ Qa) ** 2) / X.shape[0]
                    Sm[name] = Sb if s % ius == 0 else alpha * Sm[name] + (1 - alpha) * Sb
                assert rel_fro(layer._S[:, :layer.a_dim], Sm[name]) < 1e-4, (s, name, 'S')
                want = Qg @ ((Qg.T @ grad @ Qa) / (Sm[name] + damping)) @ Qa.T
            e = rel_fro(_grad_matrix(m), want)
            assert e < tol, (s, name, 'P', e)
        opt.step()
    return pre


class _TCN(nn.Module):
    """Dilated causal-free TCN: 'same' padding with an even kernel (asymmetric), dilation, stride."""

    def __init__(self, mode='zeros'):
        super().__init__()
        self.c1 = nn.Conv1d(3, 16, 3, dilation=2, padding='same', padding_mode=mode)
        self.c2 = nn.Conv1d(16, 16, 4, dilation=3, padding='same', bias=False)
        self.c3 = nn.Conv1d(16, 12, 5, stride=2, dilation=2, padding=3, padding_mode=mode)
        self.fc = nn.Linear(12, 5)

    def forward(self, x):
        x = torch.tanh(self.c3(torch.tanh(self.c2(torch.tanh(self.c1(x))))))
        return self.fc(x.mean(-1))


class _Vid(nn.Module):
    def __init__(self, mode='zeros'):
        super().__init__()
        self.c1 = nn.Conv3d(3, 8, 3, padding=1, padding_mode=mode)
        self.c2 = nn.Conv3d(8, 8, (1, 3, 3), stride=(1, 2, 2), padding=(0, 1, 1), bias=False)
        self.c3 = nn.Conv3d(8, 10, (3, 1, 1), dilation=(2, 1, 1), padding='same', padding_mode=mode)
        self.c4 = nn.Conv3d(10, 12, 2, stride=2, dilation=2)
        self.fc = nn.Linear(12, 5)

    def forward(self, x):
        x = torch.tanh(self.c4(torch.tanh(self.c3(torch.tanh(self.c2(torch.tanh(self.c1(x))))))))
        return self.fc(x.flatten(-3).mean(-1))


def _batches(shape, n, seed=3):
    gen = torch.Generator().manual_seed(seed)
    data = [(torch.randn(*shape, generator=gen).to(DEV), torch.randint(0, 5, shape[:1], generator=gen).to(DEV))
            for _ in range(n)]
    return lambda s: data[s]


NETS = {'tcn': (_TCN, (6, 3, 50)), 'vid': (_Vid, (4, 3, 6, 10, 9))}


@pytest.mark.parametrize('approx', ['expand', 'reduce'])
@pytest.mark.parametrize('method', ['eigen', 'inverse', 'ekfac'])
@pytest.mark.parametrize('net', list(NETS))
def test_module_against_fp64(net, method, approx):
    cls, shape = NETS[net]
    torch.manual_seed(3)
    ius = 1 if method == 'ekfac' else 2
    _run(cls().to(DEV), _batches(shape, 4), nn.CrossEntropyLoss(), method, approx, steps=4, ius=ius)


@pytest.mark.parametrize('approx', ['expand', 'reduce'])
@pytest.mark.parametrize('net', list(NETS))
def test_accumulation_steps(net, approx):
    cls, shape = NETS[net]
    torch.manual_seed(4)
    _run(cls().to(DEV), _batches(shape, 6), nn.CrossEntropyLoss(), 'eigen', approx, steps=3, ius=2, acc=2)


@pytest.mark.parametrize('method', ['eigen', 'inverse', 'ekfac'])
@pytest.mark.parametrize('net', list(NETS))
def test_factor_and_inverse_schedule(net, method):
    """factor_update_steps=2 with inv_update_steps=4 (EKFAC: 2): no statistics at odd steps, stale data between."""
    cls, shape = NETS[net]
    torch.manual_seed(9)
    _run(cls().to(DEV), _batches(shape, 6), nn.CrossEntropyLoss(), method, 'expand', steps=6, fus=2,
         ius=2 if method == 'ekfac' else 4)


@pytest.mark.parametrize('mode', ['reflect', 'replicate', 'circular'])
@pytest.mark.parametrize('net', list(NETS))
def test_padding_modes(net, mode):
    cls, shape = NETS[net]
    torch.manual_seed(5)
    for method in ('eigen', 'ekfac'):
        _run(cls(mode).to(DEV), _batches(shape, 3), nn.CrossEntropyLoss(), method, 'expand', steps=3)


@pytest.mark.parametrize('approx', ['expand', 'reduce'])
@pytest.mark.parametrize('net', list(NETS))
def test_unbatched_input(net, approx):
    cls, shape = NETS[net]
    torch.manual_seed(6)
    data = _batches(shape[1:], 3)
    loss = lambda out, y: (out * torch.arange(5.0, device=DEV)).sum()  # noqa: E731
    for method in ('eigen', 'ekfac'):
        _run(cls().to(DEV), data, loss, method, approx, steps=3)


# ---------------------------------------------------------------------------------------------- AMP, other layers
@pytest.mark.parametrize('method', ['eigen', 'ekfac'])
@pytest.mark.parametrize('net', list(NETS))
def test_amp_grad_scaler(net, method):
    from kfac_b200.preconditioner import KFACPreconditioner
    cls, shape = NETS[net]
    torch.manual_seed(0)
    base = cls().to(DEV)
    data = _batches((16,) + shape[1:], 4, seed=0)
    runs = {}
    for amp in (False, True):
        m = cls().to(DEV)
        m.load_state_dict(base.state_dict())
        scaler = torch.amp.GradScaler('cuda', init_scale=2.0 ** 10, growth_interval=10 ** 9, enabled=amp)
        pre = KFACPreconditioner(m, compute_method=method, damping=0.003, precondition_conv_nd=True,
                                 grad_scaler=scaler if amp else None)
        opt = torch.optim.SGD(m.parameters(), lr=0.0)
        facs = []
        for s in range(4):
            m.zero_grad()
            if amp and s == 2:
                scaler.update(new_scale=2.0 ** 60)       # the scaled loss overflows fp16: every G window is dropped
                before = {n: l.g_factor.clone() for n, l in pre._layers.values()}
                skipped = pre.skipped_factor_updates
            with torch.autocast('cuda', dtype=torch.float16, enabled=amp):
                loss = nn.functional.cross_entropy(m(data(s)[0]), data(s)[1])
            scaler.scale(loss).backward()
            scaler.unscale_(opt)
            pre.step()
            torch.cuda.synchronize()
            if amp and s == 2:
                assert pre.skipped_factor_updates - skipped >= len(pre._layers)
                for n, l in pre._layers.values():
                    assert torch.equal(l.g_factor, before[n]), n
                    assert torch.isfinite(l.a_factor).all()
            if amp:
                scaler.update(new_scale=2.0 ** 10)
            facs.append({n: (l.a_factor.clone(), l.g_factor.clone()) for n, l in pre._layers.values()})
        runs[amp] = facs
    for s in (0, 1):
        for n in runs[False][s]:
            for u, v in zip(runs[True][s][n], runs[False][s][n]):
                assert rel_fro(u, v) <= 2e-2, (s, n, rel_fro(u, v))


def test_factor_dtype_bf16():
    torch.manual_seed(7)
    from kfac_b200.preconditioner import KFACPreconditioner
    m = _TCN().to(DEV)
    pre = KFACPreconditioner(m, precondition_conv_nd=True, factor_dtype=torch.bfloat16, damping=0.003)
    rec = _Rec(pre._layers)
    x, y = _batches((6, 3, 50), 1)(0)
    nn.functional.cross_entropy(m(x), y).backward()
    pre.step()
    torch.cuda.synchronize()
    for mod, (name, l) in pre._layers.items():
        X, _ = _rows64(mod, rec.inp[mod][0].bfloat16(), rec.gout[mod][0], False)
        want = 0.95 * torch.eye(X.shape[1], dtype=torch.float64, device=DEV) + 0.05 * X.T @ X / X.shape[0]
        assert rel_fro(l._a_view[:, :l.a_dim], want) <= 1e-5, name


@pytest.mark.parametrize('method', ['eigen', 'inverse', 'ekfac'])
def test_other_layers_unaffected(method):
    """With the new layers skipped, every other layer's preconditioned gradient is bitwise that of the keyword off."""
    from kfac_b200.preconditioner import KFACPreconditioner

    class Net(nn.Module):
        def __init__(self):
            super().__init__()
            self.c1 = nn.Conv1d(3, 8, 3, padding=1)
            self.c2 = nn.Conv2d(8, 8, 3, padding=1)
            self.fc = nn.Linear(8, 5)

        def forward(self, x):
            h = torch.tanh(self.c1(x)).unsqueeze(2)
            return self.fc(torch.tanh(self.c2(h)).mean((2, 3)))

    torch.manual_seed(8)
    base = Net().to(DEV)
    data = _batches((6, 3, 20), 3)
    out = []
    for kw in ({}, dict(precondition_conv_nd=True, skip_layers=['c1'])):
        m = Net().to(DEV)
        m.load_state_dict(base.state_dict())
        pre = KFACPreconditioner(m, compute_method=method, damping=0.003, **kw)
        assert [n for n, _ in pre._layers.values()] == ['c2', 'fc']
        grads = []
        for s in range(3):
            m.zero_grad()
            nn.functional.cross_entropy(m(data(s)[0]), data(s)[1]).backward()
            pre.step()
            grads.append([p.grad.clone() for p in m.parameters()])
        out.append(grads)
    for a, b in zip(*out):
        assert all(torch.equal(u, v) for u, v in zip(a, b))


# ---------------------------------------------------------------------------------------------- two ranks
def _run_dist(backend):
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    script = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'dist_conv_nd.py')
    out = subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node=2',
                          '--master-addr', '127.0.0.1', '--master-port', str(port), script, '--backend', backend],
                         capture_output=True, text=True, timeout=900)
    print(out.stdout[-3000:])
    assert out.returncode == 0, out.stderr[-4000:]
    assert out.stdout.count('dist_conv_nd ok') == 2, out.stdout[-2000:]


def test_two_ranks_gloo():
    _run_dist('gloo')


def test_two_ranks_nccl():
    if torch.cuda.device_count() < 2:
        pytest.skip('needs >= 2 GPUs')
    _run_dist('nccl')
