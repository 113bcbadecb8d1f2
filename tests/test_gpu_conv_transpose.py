"""ConvTranspose1d / 2d / 3d layers (`precondition_conv_transpose=True`) on the GPU:

  * an fp64 oracle of the patches a(o) restated from the definition (output o reads input (o + p - k d) / s through tap k
    where s divides it), itself checked against autograd: y = Wmat a + bias and sum_o g a^T = the permuted weight.grad;
  * the three transposed input kernels (factor, EKFAC rows, K-FAC-reduce rows) against it, over 1-D, 2-D and 3-D
    geometries with s in {1, 2, 3}, d in {1, 2}, output padding, s > k and p > d (k - 1), in fp32, fp16 and bf16, with
    and without the ones column; chunked against whole-batch workspaces; the off-phase blocks of A exact zeros;
  * a DCGAN-style generator, a 1-D upsampler and a 3-D decoder against an fp64 restatement (factors -> eigh -> P) under
    EIGEN, INVERSE and EKFAC, expand and reduce, with kl_clip (nu against fp64), accumulation and schedules, unbatched
    inputs and output_size passed as a keyword, a GradScaler under fp16 autocast and factor_dtype=bf16;
  * a stride-1 ConvTranspose2d against its Conv2d twin; other layers unaffected; two ranks
    (tests/dist_conv_transpose.py).
"""
import ctypes
import itertools
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


# ---------------------------------------------------------------------------------------------- fp64 oracle
def _tap_index(L, Lo, k, s, d, p, device):
    """(Lo, k) input index that output o reads through tap k; L (a zero appended to the axis) where s does not divide
    o + p - k d or the quotient is not an input position."""
    t = torch.arange(Lo, device=device)[:, None] + p - torch.arange(k, device=device)[None, :] * d
    i = torch.div(t, s, rounding_mode='floor')
    ok = (t >= 0) & (t % s == 0) & (i < L)
    return torch.where(ok, i, torch.full_like(i, L))


def _patches64(x, k, s, d, p, out):
    """(B, S, C*kd*kh*kw) fp64 patches of x (B, C, D, H, W), per-axis parameters in (D, H, W) order, out the output
    extents: a(o)[ci, k] = x[b, ci, (o + p - k d) / s] where s divides o + p - k d on every axis and the quotient is an
    input position, else 0."""
    x = F.pad(x.double(), (0, 1, 0, 1, 0, 1))
    B, C = x.shape[:2]
    I = [_tap_index(x.shape[2 + a] - 1, out[a], k[a], s[a], d[a], p[a], x.device) for a in range(3)]
    P = x[:, :, I[0][:, None, None, :, None, None], I[1][None, :, None, None, :, None], I[2][None, None, :, None, None, :]]
    return P.permute(0, 2, 3, 4, 1, 5, 6, 7).reshape(B, math.prod(out), C * math.prod(k))


def _lead(v, nd, fill=1):
    return [fill] * (3 - nd) + list(v)


def _module_patches64(m, x, out):
    """fp64 patches of a batched call of the transposed convolution m whose output extent is `out`."""
    nd = len(m.kernel_size)
    x5 = x.reshape(x.shape[:2] + (1,) * (3 - nd) + x.shape[2:])
    return _patches64(x5, _lead(m.kernel_size, nd), _lead(m.stride, nd), _lead(m.dilation, nd), _lead(m.padding, nd, 0),
                      _lead(out, nd))


def _wmat(m, w):
    """Wmat[co, ci K + k] = w[ci, co, k] of a (C_in, C_out, k...) tensor."""
    return w.reshape(m.in_channels, m.out_channels, -1).permute(1, 0, 2).reshape(m.out_channels, -1)


ORACLE_CASES = [
    (nn.ConvTranspose1d, dict(kernel_size=16, stride=8, padding=4), (2, 3, 9), None),
    (nn.ConvTranspose1d, dict(kernel_size=3, stride=3, dilation=2, padding=1, output_padding=2), (2, 3, 7), None),
    (nn.ConvTranspose1d, dict(kernel_size=2, stride=3), (2, 3, 6), [17]),                      # s > k, output_size
    (nn.ConvTranspose1d, dict(kernel_size=3, padding=5), (2, 3, 14), None),                   # p > d (k - 1)
    (nn.ConvTranspose2d, dict(kernel_size=4, stride=2, padding=1), (2, 3, 5, 6), [11, 12]),
    (nn.ConvTranspose2d, dict(kernel_size=(3, 2), stride=(2, 3), dilation=(2, 1), padding=(4, 0), output_padding=(1, 2)),
     (2, 3, 6, 5), None),
    (nn.ConvTranspose3d, dict(kernel_size=(3, 1, 2), stride=(2, 1, 3), dilation=(2, 1, 1), padding=(1, 0, 1),
                              output_padding=(1, 0, 2)), (2, 2, 3, 4, 4), None),
]


@pytest.mark.parametrize('case', range(len(ORACLE_CASES)))
def test_oracle_against_autograd(case):
    """The fp64 patches reproduce the module's output, and sum_o g(o) a(o)^T is the weight gradient permuted to Wmat."""
    cls, kw, shape, size = ORACLE_CASES[case]
    torch.manual_seed(case)
    m = cls(shape[1], 4, **kw).double().to(DEV)
    x = torch.randn(*shape, dtype=torch.float64, device=DEV)
    y = m(x, output_size=size) if size is not None else m(x)
    nd = len(m.kernel_size)
    out = tuple(y.shape[2:])
    U = _module_patches64(m, x, out)                                        # (B, S, C_in K)
    W = _wmat(m, m.weight.detach())
    want_y = U @ W.T + m.bias.detach()                                      # (B, S, C_out)
    assert torch.allclose(y.flatten(2).transpose(1, 2), want_y, rtol=0, atol=1e-12)
    g = torch.randn_like(y)
    y.backward(g)
    Gr = g.flatten(2).transpose(1, 2).reshape(-1, y.shape[1])
    dW = Gr.T @ U.reshape(-1, U.shape[2])
    assert torch.allclose(dW, _wmat(m, m.weight.grad), rtol=0, atol=1e-10)
    assert len(out) == nd


# ---------------------------------------------------------------------------------------------- kernels
# (B, C, in, kernel, stride, dilation, padding, output_padding), per axis in (D, H, W) order
GEOS = [
    (3, 2, (1, 1, 257), (1, 1, 16), (1, 1, 8), (1, 1, 1), (0, 0, 4), (0, 0, 0)),   # MelGAN-style x8 upsampler
    (2, 3, (1, 1, 40), (1, 1, 3), (1, 1, 3), (1, 1, 2), (0, 0, 1), (0, 0, 2)),     # s = 3, d = 2, op = 2
    (2, 4, (1, 1, 31), (1, 1, 2), (1, 1, 3), (1, 1, 1), (0, 0, 0), (0, 0, 1)),     # s > k: outputs without a tap
    (2, 3, (1, 1, 29), (1, 1, 3), (1, 1, 1), (1, 1, 1), (0, 0, 5), (0, 0, 0)),     # p > d (k - 1)
    (2, 5, (1, 7, 9), (1, 4, 4), (1, 2, 2), (1, 1, 1), (0, 1, 1), (0, 0, 0)),      # DCGAN
    (2, 3, (1, 6, 5), (1, 3, 2), (1, 2, 3), (1, 2, 1), (0, 4, 0), (0, 1, 2)),      # p > d (k - 1) on H, s > k on W
    (2, 3, (3, 4, 5), (2, 2, 2), (2, 2, 2), (1, 1, 1), (0, 0, 0), (0, 0, 0)),      # 3-D x2
    (2, 2, (3, 5, 4), (3, 1, 2), (2, 1, 3), (2, 1, 1), (1, 0, 1), (1, 0, 2)),      # 3-D mixed, op
    (2, 64, (2, 3, 5), (1, 1, 1), (1, 1, 1), (1, 1, 1), (0, 0, 0), (0, 0, 0)),     # 1 x 1 x 1: packed (30 % 4)
    (2, 16, (1, 3, 4), (1, 1, 1), (1, 1, 1), (1, 1, 1), (0, 0, 0), (0, 0, 0)),     # 1 x 1 x 1: in place
]


def _geo(g):
    from kfac_b200 import _cabi
    B, C, ins, k, s, d, p, op = g
    arr = lambda v: (ctypes.c_int * 3)(*v)  # noqa: E731
    return _cabi.ConvTransposeGeometry(B, C, arr(ins), arr(k), arr(s), arr(d), arr(p), arr(op))


def _out(g):
    _, _, ins, k, s, d, p, op = g
    return [(ins[a] - 1) * s[a] - 2 * p[a] + d[a] * (k[a] - 1) + op[a] + 1 for a in range(3)]


def _input(g, dtype):
    B, C, ins = g[:3]
    gen = torch.Generator(device=DEV).manual_seed(zlib.crc32(repr(g).encode()))
    return (torch.randn(B, C, *ins, device=DEV, generator=gen) + 0.3).to(dtype)


def _oracle(x, g):
    _, _, _, k, s, d, p, _ = g
    return _patches64(x, k, s, d, p, _out(g))


def _factor(lib, x, geo, ones, scale, ws_bytes, d):
    acc = torch.zeros(d, d, device=DEV)
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=DEV)
    rc = lib.kfac_factor_conv_transpose_input(x.data_ptr(), _code(x.dtype), ctypes.byref(geo), ones, scale,
                                              acc.data_ptr(), ws.data_ptr(), ws_bytes, S())
    assert rc == 0, lib.kfac_last_error()
    torch.cuda.synchronize()
    return acc


@pytest.mark.parametrize('ones', [0, 1])
@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('g', GEOS, ids=lambda g: f'{g[2]}-k{g[3]}s{g[4]}d{g[5]}p{g[6]}op{g[7]}')
def test_input_kernels_against_fp64(lib, g, dtype, ones):
    x = _input(g, dtype)
    geo = _geo(g)
    B = g[0]
    U = _oracle(x, g)
    Sp = U.shape[1]
    if ones:
        U = torch.cat([U, U.new_ones(B, Sp, 1)], 2)
    d = U.shape[2]
    rows = U.reshape(B * Sp, d)
    need = lib.kfac_factor_conv_transpose_input_workspace_bytes(ctypes.byref(geo), ones, 1 << 30)
    acc = _factor(lib, x, geo, ones, 1.0 / (B * Sp), need, d)
    assert rel_fro(acc, rows.T @ rows / (B * Sp)) <= 1e-5
    assert torch.equal(acc, _factor(lib, x, geo, ones, 1.0 / (B * Sp), need, d))
    ld = _ld4(d)
    out = torch.full((B * Sp, ld), float('nan'), device=DEV)
    assert lib.kfac_rows_conv_transpose_input(x.data_ptr(), _code(dtype), ctypes.byref(geo), ones, 1.0 / Sp,
                                              out.data_ptr(), ld, S()) == 0, lib.kfac_last_error()
    torch.cuda.synchronize()
    assert rel_fro(out[:, :d], rows / Sp) <= 1e-6 and not out[:, d:].any()
    for ldr in (d, ld):
        red = torch.full((B, ldr), float('nan'), device=DEV)
        assert lib.kfac_reduce_rows_conv_transpose_input(x.data_ptr(), _code(dtype), ctypes.byref(geo), ones, 0.5,
                                                         red.data_ptr(), ldr, S()) == 0, lib.kfac_last_error()
        torch.cuda.synchronize()
        assert rel_fro(red[:, :d], U.sum(1) * 0.5) <= 1e-6 and not red[:, d:].any()
        again = torch.empty_like(red)
        assert lib.kfac_reduce_rows_conv_transpose_input(x.data_ptr(), _code(dtype), ctypes.byref(geo), ones, 0.5,
                                                         again.data_ptr(), ldr, S()) == 0
        torch.cuda.synchronize()
        assert torch.equal(red, again)


@pytest.mark.parametrize('g', [GEOS[0], GEOS[4], GEOS[7]], ids=['1d', '2d', '3d'])
def test_chunked_im2col(lib, g):
    """A workspace of one or two examples' im2col gives the factor of one chunk (fp32 tolerance), the same bits on a
    repeat call, and the workspace query sizes chunks from its byte limit."""
    g = (5,) + g[1:]
    x = _input(g, torch.float32)
    geo = _geo(g)
    d = g[1] * math.prod(g[3]) + 1
    Sp = math.prod(_out(g))
    q = lambda cap: lib.kfac_factor_conv_transpose_input_workspace_bytes(ctypes.byref(geo), 1, cap)  # noqa: E731
    whole, one, two = q(1 << 30), q(0), q(2 * _ld4(Sp) * d * 4 + 64)
    assert one <= two <= max(2 * _ld4(Sp) * d * 4 + 64, one) and one < whole
    ref = _factor(lib, x, geo, 1, 1.0 / (5 * Sp), whole, d)
    for ws in (one, two, one + 1024):
        got = _factor(lib, x, geo, 1, 1.0 / (5 * Sp), ws, d)
        assert rel_fro(got, ref) <= 1e-5, (ws, rel_fro(got, ref))
        assert torch.equal(got, _factor(lib, x, geo, 1, 1.0 / (5 * Sp), ws, d))
    pack1 = _ld4(Sp) * d * 4          # one example's matrix without its SYRK partials: the SYRK unsplit
    assert pack1 < one
    got = _factor(lib, x, geo, 1, 1.0 / (5 * Sp), pack1, d)
    assert rel_fro(got, ref) <= 1e-5 and torch.equal(got, _factor(lib, x, geo, 1, 1.0 / (5 * Sp), pack1, d))
    acc = torch.zeros(d, d, device=DEV)
    assert lib.kfac_factor_conv_transpose_input(x.data_ptr(), 0, ctypes.byref(geo), 1, 1.0, acc.data_ptr(), None, 0,
                                                S()) != 0


@pytest.mark.parametrize('g', [(4, 6, (1, 1, 50), (1, 1, 16), (1, 1, 8), (1, 1, 1), (0, 0, 4), (0, 0, 0)),
                               (4, 8, (1, 9, 9), (1, 4, 4), (1, 2, 2), (1, 1, 1), (0, 1, 1), (0, 0, 0)),
                               (2, 4, (1, 8, 7), (1, 3, 5), (1, 3, 2), (1, 1, 1), (0, 2, 1), (0, 1, 1)),
                               (2, 3, (4, 5, 6), (2, 3, 2), (2, 3, 2), (1, 1, 1), (0, 1, 0), (1, 2, 1))],
                         ids=['1d-s8', '2d-s2', '2d-s3x2', '3d'])
def test_off_phase_blocks_are_exact_zeros(lib, g):
    """With dilation 1, two taps whose phases k mod s differ on an axis never feed the same output: those entries of A
    (without the ones column) are exact fp32 zeros, and the on-phase blocks are not."""
    x = _input(g, torch.float32)
    geo = _geo(g)
    k, s = g[3], g[4]
    need = lib.kfac_factor_conv_transpose_input_workspace_bytes(ctypes.byref(geo), 0, 1 << 30)
    A = _factor(lib, x, geo, 0, 1.0, need, g[1] * math.prod(k)).cpu()
    phase = torch.tensor([tuple(t[a] % s[a] for a in range(3)) for t in itertools.product(*(range(n) for n in k))])
    same = (phase[:, None, :] == phase[None, :, :]).all(-1).repeat(g[1], g[1])
    assert not same.all() and (A[~same] == 0).all()
    assert (A.diagonal() > 0).all()


def test_reject_bad_geometry(lib):
    x = torch.zeros(64, device=DEV)
    out = torch.zeros(64, device=DEV)
    bad = [(1, 1, (1, 1, 3), (1, 1, 1), (1, 1, 1), (1, 1, 1), (0, 0, 2), (0, 0, 0)),     # empty output
           (1, 1, (1, 1, 8), (1, 1, 3), (1, 1, 2), (1, 1, 1), (0, 0, 0), (0, 0, 2)),     # op = s
           (1, 1, (1, 1, 8), (1, 1, 3), (1, 1, 2), (1, 1, 3), (0, 0, 0), (0, 0, 3)),     # op = max(s, d)
           (1, 1, (1, 1, 8), (1, 1, 3), (1, 1, 0), (1, 1, 1), (0, 0, 0), (0, 0, 0)),     # stride 0
           (1, 1, (1, 1, 8), (1, 1, 3), (1, 1, 1), (1, 1, 1), (0, 0, -1), (0, 0, 0)),    # negative padding
           (512, 1, (1, 1024, 1024), (1, 4, 4), (1, 4, 4), (1, 1, 1), (0, 0, 0), (0, 0, 0))]   # 2^33 rows
    for g in bad:
        geo = _geo(g)
        assert lib.kfac_factor_conv_transpose_input_workspace_bytes(ctypes.byref(geo), 0, 1 << 20) == 0
        acc = torch.zeros(4, device=DEV)
        assert lib.kfac_factor_conv_transpose_input(x.data_ptr(), 0, ctypes.byref(geo), 0, 1.0, acc.data_ptr(), None, 0,
                                                    S()) == -1
        assert lib.kfac_rows_conv_transpose_input(x.data_ptr(), 0, ctypes.byref(geo), 0, 1.0, out.data_ptr(), 4,
                                                  S()) == -1
        assert lib.kfac_reduce_rows_conv_transpose_input(x.data_ptr(), 0, ctypes.byref(geo), 0, 1.0, out.data_ptr(),
                                                         4, S()) == -1


# ---------------------------------------------------------------------------------------------- module level
class _Rec:
    """Every call's input, output gradient and output extent of every registered layer (lists in hook order)."""

    def __init__(self, layers):
        self.inp, self.gout = {}, {}
        for m in layers:
            m.register_forward_pre_hook(lambda mod, i: self.inp.setdefault(mod, []).append(i[0].detach().clone()))
            m.register_full_backward_hook(lambda mod, gi, go: self.gout.setdefault(mod, []).append(go[0].detach().clone()))

    def clear(self):
        self.inp, self.gout = {}, {}


def _rows64(m, x, g, reduce):
    """fp64 rows (X, G) of one call, restated from the definition: patches a(o) / S with the ones column 1 / S, and
    g(o) / S (reduce: the per-example mean of X, sum of G / sqrt(S)).  The output padding is the one the output
    gradient's extent shows."""
    if isinstance(m, nn.Linear):
        x, g = x.double().reshape(-1, x.shape[-1]), g.double().reshape(-1, g.shape[-1])
        X = torch.cat([x, x.new_ones(x.shape[0], 1)], 1) if m.bias is not None else x
        return X, g
    nd = len(m.kernel_size)
    x, g = x.double(), g.double()
    if x.dim() == nd + 1:
        x, g = x.unsqueeze(0), g.unsqueeze(0)
    U = _module_patches64(m, x, tuple(g.shape[2:]))
    B, Sp = U.shape[:2]
    X = U / Sp
    if m.bias is not None:
        X = torch.cat([X, X.new_full((B, Sp, 1), 1.0 / Sp)], 2)
    G = g.flatten(2).transpose(1, 2) / Sp
    if reduce and Sp > 1:
        return X.mean(1), G.sum(1) / math.sqrt(Sp)
    return X.reshape(B * Sp, -1), G.reshape(B * Sp, -1)


def _grad_matrix(helper):
    return helper.get_grad().detach().double()


def _run(model, batches, method, approx, steps, ius=1, acc=1, damping=0.003, alpha=0.9, tol=1e-3, kw=None, fus=1,
         kl_clip=None, lr=0.1):
    """Train `steps` steps of the loss sum(model(x) * y) and check every registered layer's A, G (and S under EKFAC)
    and preconditioned gradient against fp64 after each, and nu against fp64 under kl_clip; factors are formed every
    `fus` steps, second-order data every `ius` steps."""
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    pre = KFACPreconditioner(model, compute_method=method, kfac_approx=approx, factor_update_steps=fus,
                             inv_update_steps=ius, damping=damping, factor_decay=alpha, kl_clip=kl_clip, lr=lr,
                             accumulation_steps=acc, precondition_conv_transpose=True, **(kw or {}))
    rec = _Rec(pre._layers)
    A, G, Sm, snap = {}, {}, {}, {}
    opt = torch.optim.SGD(model.parameters(), lr=0.01)
    reduce = approx == 'reduce'
    eye = lambda n: torch.eye(n, dtype=torch.float64, device=DEV)  # noqa: E731
    for s in range(steps):
        opt.zero_grad()
        calls = {m: [] for m in pre._layers}
        for k in range(acc):
            rec.clear()
            x, y = batches(s * acc + k)
            (model(x) * y).sum().backward()
            for m in pre._layers:
                calls[m].append(list(zip(rec.inp[m], reversed(rec.gout[m]))))
        grads = {name: _grad_matrix(l.module) for name, l in pre._layers.values()}
        pre.step()
        torch.cuda.synchronize()
        wants = {}
        for m, (name, layer) in pre._layers.items():
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
            wants[name] = (layer, want)
        nu = 1.0
        if kl_clip is not None:
            vg = sum(float((want * grads[name]).sum()) for name, (_, want) in wants.items()) * lr * lr
            nu = min(1.0, math.sqrt(kl_clip / abs(vg)))
            assert nu < 1.0
            assert abs(float(pre.last_grad_scale) - nu) <= 1e-3 * nu, (s, float(pre.last_grad_scale), nu)
        for name, (layer, want) in wants.items():
            e = rel_fro(_grad_matrix(layer.module), nu * want)
            assert e < tol, (s, name, 'P', e)
        opt.step()
    return pre


class _Generator(nn.Module):
    """DCGAN-style: z (B, 8, 1, 1) -> 4 x 4 -> 8 x 8 -> 16 x 16 images, the first layer without a bias."""

    def __init__(self):
        super().__init__()
        self.g1 = nn.ConvTranspose2d(8, 12, 4, 1, 0, bias=False)
        self.g2 = nn.ConvTranspose2d(12, 6, 4, 2, 1)
        self.g3 = nn.ConvTranspose2d(6, 3, 4, 2, 1)

    def forward(self, z):
        return torch.tanh(self.g3(torch.tanh(self.g2(torch.tanh(self.g1(z))))))


class _Upsampler(nn.Module):
    """1-D x8 / x2 / x3 upsampling: a MelGAN-style stage, a dilated one, and s > k with output padding."""

    def __init__(self):
        super().__init__()
        self.u1 = nn.ConvTranspose1d(6, 8, 16, stride=8, padding=4)
        self.u2 = nn.ConvTranspose1d(8, 6, 3, stride=2, dilation=2, padding=3, output_padding=1)
        self.u3 = nn.ConvTranspose1d(6, 2, 2, stride=3, output_padding=2, bias=False)

    def forward(self, x):
        return self.u3(torch.tanh(self.u2(torch.tanh(self.u1(x)))))


class _Decoder3d(nn.Module):
    """A 3-D segmentation decoder stage: x2 on every axis, x2 in-plane with output padding, then a 1 x 1 x 1 head."""

    def __init__(self):
        super().__init__()
        self.d1 = nn.ConvTranspose3d(4, 6, 2, stride=2)
        self.d2 = nn.ConvTranspose3d(6, 4, 3, stride=(1, 2, 2), padding=1, output_padding=(0, 1, 1))
        self.d3 = nn.ConvTranspose3d(4, 2, 1)

    def forward(self, x):
        return self.d3(torch.tanh(self.d2(torch.tanh(self.d1(x)))))


class _UNetUp(nn.Module):
    """U-Net decoder steps that call their upsampling layer with output_size=skip.shape (a keyword), batched or not:
    output padding (1, 1), then (1, 0)."""

    def __init__(self):
        super().__init__()
        self.up1 = nn.ConvTranspose2d(6, 4, 2, stride=2)
        self.up2 = nn.ConvTranspose2d(4, 3, 3, stride=2, padding=1)

    def forward(self, x):
        lead = x.shape[:-3]
        h = torch.tanh(self.up1(x, output_size=lead + (4, 11, 13)))
        return self.up2(h, output_size=lead + (3, 22, 25))


NETS = {'dcgan': (_Generator, (6, 8, 1, 1)), 'audio': (_Upsampler, (3, 6, 11)), 'vol': (_Decoder3d, (2, 4, 2, 3, 3)),
        'unet': (_UNetUp, (3, 6, 5, 6))}


def _batches(model, shape, n, seed=3):
    """n batches (x, y): inputs of `shape` and loss weights y of the model's output shape (formed before the model is
    hooked)."""
    gen = torch.Generator().manual_seed(seed)
    xs = [torch.randn(*shape, generator=gen).to(DEV) for _ in range(n)]
    with torch.no_grad():
        out = model(xs[0]).shape
    data = [(x, torch.randn(*out, generator=gen).to(DEV)) for x in xs]
    return lambda s: data[s]


@pytest.mark.parametrize('approx', ['expand', 'reduce'])
@pytest.mark.parametrize('method', ['eigen', 'inverse', 'ekfac'])
@pytest.mark.parametrize('net', ['dcgan', 'audio', 'vol'])
def test_module_against_fp64(net, method, approx):
    cls, shape = NETS[net]
    torch.manual_seed(3)
    m = cls().to(DEV)
    _run(m, _batches(m, shape, 4), method, approx, steps=4, ius=1 if method == 'ekfac' else 2)


@pytest.mark.parametrize('method', ['eigen', 'inverse', 'ekfac'])
@pytest.mark.parametrize('net', ['dcgan', 'audio'])
def test_kl_clip(net, method):
    """nu is formed from the permuted weight gradients and is checked against fp64 with every P."""
    cls, shape = NETS[net]
    torch.manual_seed(11)
    m = cls().to(DEV)
    _run(m, _batches(m, shape, 3), method, 'expand', steps=3, kl_clip=1e-8)


@pytest.mark.parametrize('approx', ['expand', 'reduce'])
@pytest.mark.parametrize('net', ['dcgan', 'vol'])
def test_accumulation_steps(net, approx):
    cls, shape = NETS[net]
    torch.manual_seed(4)
    m = cls().to(DEV)
    _run(m, _batches(m, shape, 6), 'eigen', approx, steps=3, ius=2, acc=2)


@pytest.mark.parametrize('method', ['eigen', 'inverse', 'ekfac'])
@pytest.mark.parametrize('net', ['audio', 'vol'])
def test_factor_and_inverse_schedule(net, method):
    """factor_update_steps=2 with inv_update_steps=4 (EKFAC: 2): no statistics at odd steps, stale data between."""
    cls, shape = NETS[net]
    torch.manual_seed(9)
    m = cls().to(DEV)
    _run(m, _batches(m, shape, 6), method, 'expand', steps=6, fus=2, ius=2 if method == 'ekfac' else 4)


@pytest.mark.parametrize('approx', ['expand', 'reduce'])
@pytest.mark.parametrize('unbatched', [False, True])
def test_output_size_keyword(unbatched, approx):
    """U-Net steps that pass output_size as a keyword, which sets their output padding."""
    cls, shape = NETS['unet']
    torch.manual_seed(6)
    m = cls().to(DEV)
    for method in ('eigen', 'ekfac'):
        _run(m, _batches(m, shape[1:] if unbatched else shape, 3), method, approx, steps=3)


@pytest.mark.parametrize('approx', ['expand', 'reduce'])
@pytest.mark.parametrize('net', ['audio', 'vol'])
def test_unbatched_input(net, approx):
    cls, shape = NETS[net]
    torch.manual_seed(6)
    m = cls().to(DEV)
    for method in ('eigen', 'ekfac'):
        _run(m, _batches(m, shape[1:], 3), method, approx, steps=3)


@pytest.mark.parametrize('method', ['eigen', 'ekfac'])
@pytest.mark.parametrize('net', ['dcgan', 'audio'])
def test_amp_grad_scaler(net, method):
    """fp16 autocast with a GradScaler: the factors follow the fp32 run, and a window whose scaled loss overflows fp16
    is dropped for every layer."""
    from kfac_b200.preconditioner import KFACPreconditioner
    cls, shape = NETS[net]
    torch.manual_seed(0)
    base = cls().to(DEV)
    data = _batches(base, (16,) + shape[1:], 4, seed=0)
    runs = {}
    for amp in (False, True):
        m = cls().to(DEV)
        m.load_state_dict(base.state_dict())
        scaler = torch.amp.GradScaler('cuda', init_scale=2.0 ** 10, growth_interval=10 ** 9, enabled=amp)
        pre = KFACPreconditioner(m, compute_method=method, damping=0.003, precondition_conv_transpose=True,
                                 grad_scaler=scaler if amp else None)
        opt = torch.optim.SGD(m.parameters(), lr=0.0)
        facs = []
        for s in range(4):
            m.zero_grad()
            if amp and s == 2:
                scaler.update(new_scale=2.0 ** 60)
                before = {n: l.g_factor.clone() for n, l in pre._layers.values()}
                skipped = pre.skipped_factor_updates
            with torch.autocast('cuda', dtype=torch.float16, enabled=amp):
                loss = (m(data(s)[0]).float() * data(s)[1]).mean()
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
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(7)
    m = _Upsampler().to(DEV)
    x, y = _batches(m, (3, 6, 11), 1)(0)
    pre = KFACPreconditioner(m, precondition_conv_transpose=True, factor_dtype=torch.bfloat16, damping=0.003)
    rec = _Rec(pre._layers)
    (m(x) * y).sum().backward()
    pre.step()
    torch.cuda.synchronize()
    for mod, (name, l) in pre._layers.items():
        X, _ = _rows64(mod, rec.inp[mod][0].bfloat16(), rec.gout[mod][0], False)
        want = 0.95 * torch.eye(X.shape[1], dtype=torch.float64, device=DEV) + 0.05 * X.T @ X / X.shape[0]
        assert rel_fro(l._a_view[:, :l.a_dim], want) <= 1e-5, name


# ---------------------------------------------------------------------------------------------- twins, other layers
@pytest.mark.parametrize('method', ['eigen', 'inverse'])
@pytest.mark.parametrize('padding', [0, 1])
def test_stride_one_twin_of_conv2d(padding, method):
    """A stride-1 ConvTranspose2d is the Conv2d with padding k - 1 - p and the flipped, transposed weight: the factors
    and P agree after the tap permutation (fp32 tolerance)."""
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(2)
    k = 3
    ct = nn.ConvTranspose2d(4, 6, k, padding=padding).to(DEV)
    cv = nn.Conv2d(4, 6, k, padding=k - 1 - padding).to(DEV)
    with torch.no_grad():
        cv.weight.copy_(ct.weight.flip(2, 3).transpose(0, 1))
        cv.bias.copy_(ct.bias)
    # feature ci * 9 + kh * 3 + kw of the transposed layer is feature ci * 9 + (2 - kh) * 3 + (2 - kw) of the Conv2d
    perm = torch.tensor([ci * 9 + (2 - kh) * 3 + (2 - kw) for ci, kh, kw in itertools.product(range(4), range(k),
                                                                                              range(k))] + [36])
    kw = dict(compute_method=method, damping=0.003, inv_update_steps=1)
    p_ct = KFACPreconditioner(nn.Sequential(ct), precondition_conv_transpose=True, **kw)
    p_cv = KFACPreconditioner(nn.Sequential(cv), **kw)
    (_, l_ct), = p_ct._layers.values()
    (_, l_cv), = p_cv._layers.values()
    gen = torch.Generator().manual_seed(4)
    for s in range(3):
        x = torch.randn(5, 4, 9, 10, generator=gen).to(DEV)
        ct.zero_grad()
        cv.zero_grad()
        y, y_cv = ct(x), cv(x)
        assert rel_fro(y_cv, y) <= 1e-6
        R = torch.randn(y.shape, generator=gen).to(DEV)
        (y * R).sum().backward()
        (y_cv * R).sum().backward()
        with torch.no_grad():       # the same gradient matrix for both
            ct.weight.grad.copy_(cv.weight.grad.transpose(0, 1).flip(2, 3))
        assert torch.equal(l_ct.module.get_grad()[:, :36], l_cv.module.get_grad()[:, perm[:36]])
        p_ct.step()
        p_cv.step()
        torch.cuda.synchronize()
        assert rel_fro(l_ct.a_factor, l_cv.a_factor[perm][:, perm]) <= 1e-6
        assert rel_fro(l_ct.g_factor, l_cv.g_factor) <= 1e-6
        assert rel_fro(l_ct.module.get_grad(), l_cv.module.get_grad()[:, perm]) <= 1e-4


@pytest.mark.parametrize('method', ['eigen', 'inverse', 'ekfac'])
def test_other_layers_unaffected(method):
    """With the transposed layers skipped, the Conv2d and Linear layers' preconditioned gradients are bitwise those of
    the keyword off; with them registered, the transposed layers' own gradients are preconditioned."""
    from kfac_b200.preconditioner import KFACPreconditioner

    class Net(nn.Module):
        def __init__(self):
            super().__init__()
            self.up = nn.ConvTranspose2d(3, 6, 4, stride=2, padding=1)
            self.c = nn.Conv2d(6, 8, 3, padding=1)
            self.fc = nn.Linear(8, 5)

        def forward(self, x):
            return self.fc(torch.tanh(self.c(torch.tanh(self.up(x)))).mean((2, 3)))

    torch.manual_seed(8)
    base = Net().to(DEV)
    gen = torch.Generator().manual_seed(1)
    data = [(torch.randn(6, 3, 5, 5, generator=gen).to(DEV), torch.randint(0, 5, (6,), generator=gen).to(DEV))
            for _ in range(3)]
    out = []
    for kw, names in (({}, ['c', 'fc']), (dict(precondition_conv_transpose=True, skip_layers=['up']), ['c', 'fc']),
                      (dict(precondition_conv_transpose=True), ['up', 'c', 'fc'])):
        m = Net().to(DEV)
        m.load_state_dict(base.state_dict())
        pre = KFACPreconditioner(m, compute_method=method, damping=0.003, **kw)
        assert [n for n, _ in pre._layers.values()] == names
        grads = []
        for x, y in data:
            m.zero_grad()
            nn.functional.cross_entropy(m(x), y).backward()
            raw = m.up.weight.grad.clone()
            pre.step()
            grads.append([p.grad.clone() for p in m.parameters()])
            assert torch.equal(m.up.weight.grad, raw) == ('up' not in names)
        out.append(grads)
    for a, b in zip(out[0], out[1]):
        assert all(torch.equal(u, v) for u, v in zip(a, b))


# ---------------------------------------------------------------------------------------------- two ranks
def _run_dist(backend):
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    script = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'dist_conv_transpose.py')
    out = subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node=2',
                          '--master-addr', '127.0.0.1', '--master-port', str(port), script, '--backend', backend],
                         capture_output=True, text=True, timeout=900)
    print(out.stdout[-3000:])
    assert out.returncode == 0, out.stderr[-4000:]
    assert out.stdout.count('dist_conv_transpose ok') == 2, out.stdout[-2000:]


def test_two_ranks_gloo():
    _run_dist('gloo')


def test_two_ranks_nccl():
    if torch.cuda.device_count() < 2:
        pytest.skip('needs >= 2 GPUs')
    _run_dist('nccl')
