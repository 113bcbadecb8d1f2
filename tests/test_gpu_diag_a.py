"""Diagonal-A Linear and convolution layers (`diagonal_a_layers=[...]`) on the GPU, everything against fp64:

  * kfac_factor_conv_input_diag against the diagonal of an fp64 im2col Gram matrix: 1-D / 2-D / 3-D geometries with
    strides, dilations and asymmetric 'same' padding, with and without the ones column, fp32 / fp16 / bf16 inputs,
    accumulated into a live vector, batch 1 and a wide case (C = 1280, 3 x 3); the same bits on a repeat, agreement
    with diag(kfac_factor_conv_input) on the same input, a too-small workspace rejected;
  * kfac_factor_linear_diag_ones the same way, and bit-equal to kfac_factor_linear_diag on the features;
  * kfac_precondition with diagonal-A items (g in {64, 769, 4096}, a in {1000, 9217, 14337}, with and without bias,
    fp32 / fp16 / bf16 gradients) mixed with dense, embedding and diagonal-G items, eigen and inverse: P against fp64,
    the same bits on a repeat and with peer stores, and the other items' P bit-identical without the diagonal-A items;
  * models: a SwiGLU block whose down_proj has 8200 inputs, a conv net with Conv2d(1024, 64, 3) (A = 9217) and
    Conv1d / Conv3d layers under precondition_conv_nd, under eigen and inverse, expand and reduce, integer and callable
    schedules and accumulation_steps=2: every layer's written gradient against fp64 from the factors the
    preconditioner holds, the diagonal A factors against fp64 restatements, and the first step's dense layers
    bit-identical to a run with the diagonal-A layers skipped;
  * the kl-clip scale, a state_dict round trip, an fp16 overflow under a GradScaler, hooks without host syncs, and two
    ranks (tests/dist_diag_a.py).
"""
import copy
import ctypes as C
import os
import subprocess
import sys

import pytest
import torch
from torch import nn
from torch.nn import functional as F

from conftest import rel_fro

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda')


@pytest.fixture(scope='module')
def lib():
    from kfac_b200 import _cabi
    return _cabi.load()


def S():
    return torch.cuda.current_stream().cuda_stream


def bits(x):
    return x.contiguous().view(torch.int32 if x.element_size() == 4 else torch.int16)


# ---------------------------------------------------------------------------------------------- factor kernels
def _geometry(B, Cc, ins, ker, st, dil, before, after):
    from kfac_b200 import _cabi
    arr = lambda v: (C.c_int * 3)(*v)  # noqa: E731
    return _cabi.ConvGeometry(B, Cc, arr(ins), arr(ker), arr(st), arr(dil), arr(before), arr(after))


def _im2col64(x, ker, st, dil, before, after):
    """fp64 im2col rows (B * S, C * taps) of x (B, C, D, H, W), features in the order (C, kd, kh, kw)."""
    x = x.double()
    x = F.pad(x, (before[2], after[2], before[1], after[1], before[0], after[0]))
    B, Cc = x.shape[:2]
    u = x
    for ax in range(3):          # unfold every axis: (B, C, Do, Ho, Wo, kd, kh, kw)
        size = dil[ax] * (ker[ax] - 1) + 1
        u = u.unfold(2 + ax, size, st[ax])[..., ::dil[ax]]
    Do, Ho, Wo = u.shape[2:5]
    return u.permute(0, 2, 3, 4, 1, 5, 6, 7).reshape(B * Do * Ho * Wo, Cc * ker[0] * ker[1] * ker[2]), Do * Ho * Wo


def _conv_diag(lib, x, geo, ones, scale, live, need=None):
    from kfac_b200 import _cabi
    if need is None:
        need = lib.kfac_factor_conv_input_diag_workspace_bytes(C.byref(geo))
    acc = live.clone()
    ws = torch.full((max(need, 1),), 255, dtype=torch.uint8, device=DEV)
    rc = lib.kfac_factor_conv_input_diag(x.data_ptr(), _cabi.DTYPE_CODE[x.dtype], C.byref(geo), ones, scale,
                                         acc.data_ptr(), ws.data_ptr(), need, S())
    torch.cuda.synchronize()
    return rc, acc


CONV_CASES = {   # (B, C, (D, H, W), kernel, stride, dilation, pad_before, pad_after)
    'conv1d': (4, 8, (1, 1, 97), (1, 1, 5), (1, 1, 2), (1, 1, 3), (0, 0, 6), (0, 0, 6)),
    'conv1d_same': (3, 16, (1, 1, 50), (1, 1, 4), (1, 1, 1), (1, 1, 1), (0, 0, 1), (0, 0, 2)),
    'conv2d': (5, 12, (1, 13, 11), (1, 3, 3), (1, 2, 1), (1, 1, 2), (0, 1, 2), (0, 1, 2)),
    'conv2d_same': (2, 7, (1, 9, 10), (1, 2, 4), (1, 1, 1), (1, 2, 1), (0, 1, 1), (0, 1, 2)),
    'conv3d': (2, 6, (5, 7, 6), (3, 3, 2), (2, 1, 1), (1, 2, 1), (1, 2, 0), (1, 2, 1)),
    'batch1': (1, 33, (1, 16, 16), (1, 3, 3), (1, 1, 1), (1, 1, 1), (0, 1, 1), (0, 1, 1)),
    'wide': (4, 1280, (1, 16, 16), (1, 3, 3), (1, 1, 1), (1, 1, 1), (0, 1, 1), (0, 1, 1)),
}


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16, torch.bfloat16])
@pytest.mark.parametrize('ones', [0, 1])
@pytest.mark.parametrize('case', list(CONV_CASES))
def test_factor_conv_input_diag(lib, case, ones, dtype):
    B, Cc, ins, ker, st, dil, before, after = CONV_CASES[case]
    gen = torch.Generator(device=DEV).manual_seed(len(case) + ones)
    x = (torch.randn(B, Cc, *ins, device=DEV, generator=gen) * 2).to(dtype)
    geo = _geometry(B, Cc, ins, ker, st, dil, before, after)
    rows, Sp = _im2col64(x, ker, st, dil, before, after)
    d = rows.shape[1] + ones
    live = torch.rand(d, device=DEV, generator=gen)
    scale = 1.0 / (B * Sp ** 3)
    rc, acc = _conv_diag(lib, x, geo, ones, scale, live)
    assert rc == 0, lib.kfac_last_error()
    ref = live.double().clone()
    ref[:rows.shape[1]] += scale * (rows ** 2).sum(0)
    if ones:
        ref[-1] += scale * rows.shape[0]
    assert float(((acc.double() - ref).abs() / ref.abs()).max()) <= 1e-6, case
    _, again = _conv_diag(lib, x, geo, ones, scale, live)
    assert torch.equal(bits(acc), bits(again))
    need = lib.kfac_factor_conv_input_diag_workspace_bytes(C.byref(geo))
    rc, _ = _conv_diag(lib, x, geo, ones, scale, live, need=need - 4)
    assert rc != 0
    if case != 'wide':           # the dense factor of the same call: its diagonal to fp32 rounding
        from kfac_b200 import _cabi
        dense = torch.zeros(d, d, device=DEV)
        need = lib.kfac_factor_conv_input_workspace_bytes(C.byref(geo), ones, 1 << 30)
        ws = torch.empty(max(need, 1), dtype=torch.uint8, device=DEV)
        assert lib.kfac_factor_conv_input(x.data_ptr(), _cabi.DTYPE_CODE[x.dtype], C.byref(geo), ones, scale,
                                          dense.data_ptr(), ws.data_ptr(), need, S()) == 0
        zero = torch.zeros(d, device=DEV)
        _, diag = _conv_diag(lib, x, geo, ones, scale, zero)
        assert float(((diag - dense.diagonal()).abs() / dense.diagonal().abs()).max()) <= 1e-5


def _linear_diag_ones(lib, x, ones, live, scale, need=None):
    from kfac_b200 import _cabi
    rows, V = x.shape
    if need is None:
        need = lib.kfac_factor_linear_diag_workspace_bytes(rows, V)
    acc = live.clone()
    ws = torch.full((max(need, 1),), 255, dtype=torch.uint8, device=DEV)
    rc = lib.kfac_factor_linear_diag_ones(x.data_ptr(), _cabi.DTYPE_CODE[x.dtype], rows, V, ones, scale,
                                          acc.data_ptr(), ws.data_ptr(), need, S())
    torch.cuda.synchronize()
    return rc, acc


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16, torch.bfloat16])
@pytest.mark.parametrize('rows,V', [(1, 10), (4096, 1001), (333, 14336)])
def test_factor_linear_diag_ones(lib, dtype, rows, V):
    from kfac_b200 import _cabi
    gen = torch.Generator(device=DEV).manual_seed(rows + V)
    x = (torch.randn(rows, V, device=DEV, generator=gen) * 3).to(dtype)
    live = torch.rand(V + 1, device=DEV, generator=gen)
    scale = 1.0 / rows
    rc, acc = _linear_diag_ones(lib, x, 1, live, scale)
    assert rc == 0, lib.kfac_last_error()
    ref = live.double().clone()
    ref[:V] += scale * (x.double() ** 2).sum(0)
    ref[V] += scale * rows
    assert float(((acc.double() - ref).abs() / ref.abs()).max()) <= 1e-6
    _, again = _linear_diag_ones(lib, x, 1, live, scale)
    assert torch.equal(bits(acc), bits(again))
    rc, _ = _linear_diag_ones(lib, x, 1, live, scale, need=lib.kfac_factor_linear_diag_workspace_bytes(rows, V) - 4)
    assert rc != 0
    # the features are kfac_factor_linear_diag's bits; without ones the bias entry is left alone
    need = lib.kfac_factor_linear_diag_workspace_bytes(rows, V)
    plain = live[:V].clone()
    ws = torch.empty(need, dtype=torch.uint8, device=DEV)
    assert lib.kfac_factor_linear_diag(x.data_ptr(), _cabi.DTYPE_CODE[x.dtype], rows, V, scale, plain.data_ptr(),
                                       ws.data_ptr(), need, S()) == 0
    torch.cuda.synchronize()
    assert torch.equal(bits(plain), bits(acc[:V]))
    _, no_ones = _linear_diag_ones(lib, x, 0, live, scale)
    assert torch.equal(bits(no_ones[:V]), bits(acc[:V])) and torch.equal(no_ones[V], live[V])
    if V <= 1001:                # the dense factor's diagonal to fp32 rounding
        dense = torch.zeros(V + 1, V + 1, device=DEV)
        need = lib.kfac_factor_linear_workspace_bytes(rows, V, 1)
        ws = torch.empty(max(need, 1), dtype=torch.uint8, device=DEV)
        assert lib.kfac_factor_linear(x.data_ptr(), _cabi.DTYPE_CODE[x.dtype], rows, V, 1, scale, dense.data_ptr(),
                                      ws.data_ptr(), need, S()) == 0
        _, diag = _linear_diag_ones(lib, x, 1, torch.zeros(V + 1, device=DEV), scale)
        assert float(((diag - dense.diagonal()).abs() / dense.diagonal().abs()).max()) <= 1e-5


# ---------------------------------------------------------------------------------------------- precondition
def _stored(x):
    from kfac_b200 import _cabi
    out = torch.full((x.shape[0], _cabi.ld4(x.shape[1])), float('nan'), device=DEV)
    out[:, :x.shape[1]] = x
    return out


def test_precondition_diag_a_items(lib):
    from kfac_b200 import _cabi
    damping = float(torch.tensor(0.003, dtype=torch.float32))
    gen = torch.Generator(device=DEV).manual_seed(17)

    def basis(n):
        q, _ = torch.linalg.qr(torch.randn(n, n, dtype=torch.float64, device=DEV, generator=gen))
        return q.float(), (torch.rand(n, dtype=torch.float64, device=DEV, generator=gen) ** 4).float()

    def inv(q, d):
        return ((q.double() / (d.double() + damping)) @ q.double().t()).float()

    dense = [(256, 129, 1, torch.float32), (64, 577, 1, torch.float16), (10, 21, 1, torch.bfloat16)]
    embs = [(1000, 48, torch.float16)]
    diag_g = [(10007, 769, 1, torch.float32)]
    # diagonal A (g, a, bias, dtype)
    diag_a = [(64, 14337, 1, torch.float16), (769, 9217, 0, torch.bfloat16), (4096, 1000, 1, torch.float32),
              (4096, 14337, 1, torch.bfloat16), (769, 1000, 0, torch.float32), (64, 9217, 1, torch.float32),
              (4096, 9217, 0, torch.float16)]
    D, E, GD, AD = [], [], [], []
    for g, a, bias, dtype in dense:
        qa, da = basis(a)
        qg, dg = basis(g)
        D.append(dict(g=g, a=a, dtype=dtype, w=torch.randn(g, a - bias, device=DEV, generator=gen).to(dtype),
                      b=torch.randn(g, device=DEV, generator=gen).to(dtype), qa=_stored(qa), qaT=_stored(qa.t()),
                      qg=_stored(qg), qgT=_stored(qg.t()), da=da, dg=dg, a_inv=_stored(inv(qa, da)),
                      g_inv=_stored(inv(qg, dg))))
    for V, d, dtype in embs:
        qg, dg = basis(d)
        E.append(dict(V=V, d=d, dtype=dtype, w=torch.randn(V, d, device=DEV, generator=gen).to(dtype),
                      av=torch.rand(V, device=DEV, generator=gen) * 1e-3, qg=_stored(qg), qgT=_stored(qg.t()), dg=dg,
                      g_inv=_stored(inv(qg, dg))))
    for V, a, bias, dtype in diag_g:
        qa, da = basis(a)
        GD.append(dict(V=V, a=a, dtype=dtype, w=torch.randn(V, a - bias, device=DEV, generator=gen).to(dtype),
                       b=torch.randn(V, device=DEV, generator=gen).to(dtype),
                       dgv=torch.rand(V, device=DEV, generator=gen) * 1e-2, qa=_stored(qa), qaT=_stored(qa.t()),
                       da=da, a_inv=_stored(inv(qa, da))))
    for g, a, bias, dtype in diag_a:
        qg, dg = basis(g)
        av = torch.rand(a, device=DEV, generator=gen) ** 2 * 1e-2
        av[::7] = 0                                                      # inputs without curvature
        w = torch.randn(g, a - bias, device=DEV, generator=gen).to(dtype)
        b = torch.randn(g, device=DEV, generator=gen).to(dtype) if bias else None
        grad = torch.cat([w.double(), b.double()[:, None]], 1) if bias else w.double()
        qg64, g_inv = qg.double(), inv(qg, dg)
        ref_e = qg64 @ ((qg64.t() @ grad) / (dg.double()[:, None] * av.double()[None, :] + damping))
        ref_i = (g_inv.double() @ grad) / (av.double()[None, :] + damping)
        AD.append(dict(g=g, a=a, dtype=dtype, w=w, b=b, av=av, qg=_stored(qg), qgT=_stored(qg.t()), dg=dg,
                       g_inv=_stored(g_inv), ref_e=ref_e.float(), ref_i=ref_i.float()))
        del grad, ref_e, ref_i

    def precondition(method, with_diag, peers=False):
        e = method == _cabi.KFAC_EIGEN
        others = [('d', l) for l in D] + [('e', l) for l in E] + [('g', l) for l in GD]
        if with_diag:           # interleaved: the order of the items must not matter
            layers, da_ = [], [('a', l) for l in AD]
            while others or da_:
                for src in (da_, others):
                    if src:
                        layers.append(src.pop(0))
        else:
            layers = others
        items = (_cabi.PrecondItem * len(layers))()
        Ps, keep = [], []
        for i, (kind, l) in enumerate(layers):
            p = lambda k, use: l[k].data_ptr() if use else None  # noqa: E731,B023
            if kind == 'd':
                g, a = l['g'], l['a']
                P = torch.full((g, _cabi.ld4(a)), float('nan'), device=DEV)
                items[i] = _cabi.PrecondItem(l['w'].data_ptr(), l['b'].data_ptr(), _cabi.DTYPE_CODE[l['dtype']], g, a,
                                             p('qa', e), p('qaT', e), p('qg', e), p('qgT', e), None, p('da', e),
                                             p('dg', e), p('a_inv', not e), p('g_inv', not e), _cabi.ld4(a),
                                             _cabi.ld4(g), _cabi.ld4(a), P.data_ptr(), _cabi.ld4(a))
                Ps.append((kind, l, P[:, :a], None))
            elif kind == 'e':
                V, d = l['V'], l['d']
                P = torch.full((V, _cabi.ld4(d)), float('nan'), device=DEV)
                items[i] = _cabi.PrecondItem(l['w'].data_ptr(), None, _cabi.DTYPE_CODE[l['dtype']], d, V,
                                             None, None, p('qg', e), p('qgT', e), None, l['av'].data_ptr(), p('dg', e),
                                             None, p('g_inv', not e), 0, _cabi.ld4(d), 0, P.data_ptr(), _cabi.ld4(d),
                                             None, 0, _cabi.KFAC_ITEM_EMBEDDING)
                Ps.append((kind, l, P[:, :d], None))
            elif kind == 'g':
                V, a = l['V'], l['a']
                P = torch.full((V, _cabi.ld4(a)), float('nan'), device=DEV)
                items[i] = _cabi.PrecondItem(l['w'].data_ptr(), l['b'].data_ptr(), _cabi.DTYPE_CODE[l['dtype']], V, a,
                                             p('qa', e), p('qaT', e), None, None, None, p('da', e),
                                             l['dgv'].data_ptr(), p('a_inv', not e), None, _cabi.ld4(a), 0, 0,
                                             P.data_ptr(), _cabi.ld4(a), None, 0, _cabi.KFAC_ITEM_DIAG_G)
                Ps.append((kind, l, P[:, :a], None))
            else:
                g, a = l['g'], l['a']
                P = torch.full((g, _cabi.ld4(a)), float('nan'), device=DEV)
                items[i] = _cabi.PrecondItem(l['w'].data_ptr(), l['b'].data_ptr() if l['b'] is not None else None,
                                             _cabi.DTYPE_CODE[l['dtype']], g, a, None, None, p('qg', e), p('qgT', e),
                                             None, l['av'].data_ptr(), p('dg', e), None, p('g_inv', not e), 0,
                                             _cabi.ld4(g), 0, P.data_ptr(), _cabi.ld4(a), None, 0,
                                             _cabi.KFAC_ITEM_DIAG_A)
                peer = None
                if peers:                # a second local buffer stands in for a peer's P entry
                    peer = torch.full_like(P, float('nan'))
                    arr = (C.c_void_p * 1)(peer.data_ptr())
                    keep.append(arr)
                    items[i].peer_P = arr
                    items[i].n_peers = 1
                Ps.append((kind, l, P[:, :a], peer))
        need = lib.kfac_precondition_workspace_bytes(items, len(layers))
        ws = torch.full((need,), 255, dtype=torch.uint8, device=DEV)
        rc = lib.kfac_precondition(items, len(layers), method, damping, ws.data_ptr(), need, S())
        assert rc == 0, lib.kfac_last_error()
        torch.cuda.synchronize()
        del ws
        return Ps

    for method, key in ((_cabi.KFAC_EIGEN, 'ref_e'), (_cabi.KFAC_INVERSE, 'ref_i')):
        P1 = precondition(method, True)
        for kind, l, P, _ in P1:
            if kind == 'a':
                err = rel_fro(P, l[key])
                assert err < 1e-3, (method, l['g'], l['a'], l['dtype'], err)
        P2 = precondition(method, True)
        for (_, _, p1, _), (_, _, p2, _) in zip(P1, P2):
            assert torch.equal(bits(p1), bits(p2))
        del P2
        P3 = precondition(method, True, peers=True)
        for (kind, _, p1, _), (_, _, p3, peer) in zip(P1, P3):
            assert torch.equal(bits(p1), bits(p3))
            if kind == 'a':
                assert torch.equal(bits(peer[:, :p1.shape[1]]), bits(p1))
        del P3
        alone = {id(l): P for _, l, P, _ in precondition(method, False)}
        for kind, l, P, _ in P1:
            if kind != 'a':
                assert torch.equal(bits(P), bits(alone[id(l)])), (method, kind)
        del P1, alone


def test_precondition_rejects_incomplete_diag_a_item(lib):
    from kfac_b200 import _cabi
    w = torch.zeros(12, 99, device=DEV)
    b = torch.zeros(12, device=DEV)
    qg = torch.eye(12, device=DEV)
    av = torch.ones(100, device=DEV)
    P = torch.zeros(12, 100, device=DEV)
    rcs = []
    for method, (q, qT, dg, a) in ((_cabi.KFAC_EIGEN, (qg, qg, None, av)), (_cabi.KFAC_EIGEN, (qg, None, b, av)),
                                   (_cabi.KFAC_INVERSE, (None, None, b, av)), (_cabi.KFAC_INVERSE, (qg, None, b, None))):
        items = (_cabi.PrecondItem * 1)()
        ptr = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
        items[0] = _cabi.PrecondItem(w.data_ptr(), b.data_ptr(), 0, 12, 100, None, None, ptr(q), ptr(qT), None, ptr(a),
                                     ptr(dg), None, ptr(q) if method == _cabi.KFAC_INVERSE else None, 0, 12, 0,
                                     P.data_ptr(), 100, None, 0, _cabi.KFAC_ITEM_DIAG_A)
        need = lib.kfac_precondition_workspace_bytes(items, 1)
        ws = torch.zeros(need, dtype=torch.uint8, device=DEV)
        rcs.append(lib.kfac_precondition(items, 1, method, 0.1, ws.data_ptr(), need, S()))
    assert rcs == [_cabi.KFAC_ERR_NOT_READY] * 4


# ---------------------------------------------------------------------------------------------- module level
D_MLP, H_MLP = 128, 8200      # down_proj: A = 8201 > KFAC_EIGH_MAX_N (with its bias)


class SwiGLU(nn.Module):
    """inp -> SwiGLU MLP (gate / up in diagonal_g_layers, G = 8200) -> head; inp and head are dense."""

    def __init__(self):
        super().__init__()
        self.inp = nn.Linear(32, D_MLP)
        self.gate = nn.Linear(D_MLP, H_MLP, bias=False)
        self.up = nn.Linear(D_MLP, H_MLP, bias=False)
        self.down = nn.Linear(H_MLP, D_MLP)
        self.head = nn.Linear(D_MLP, 16)

    def forward(self, x):
        h = self.inp(x)
        return self.head(self.down(F.silu(self.gate(h)) * self.up(h)))


class ConvNet(nn.Module):
    """stem (dense, G = 1024) -> Conv2d(1024, 64, 3) (A = 9217) -> fc (dense)."""

    def __init__(self):
        super().__init__()
        self.stem = nn.Conv2d(3, 1024, 1)
        self.wide = nn.Conv2d(1024, 64, 3, padding=1)
        self.fc = nn.Linear(64, 10)

    def forward(self, x):
        return self.fc(self.wide(torch.relu(self.stem(x))).mean((2, 3)))


class NdNet(nn.Module):
    """Conv1d and Conv3d (precondition_conv_nd): both diagonal in the tests, small enough to compare with dense."""

    def __init__(self):
        super().__init__()
        self.c1 = nn.Conv1d(4, 16, 5, padding='same', dilation=2)
        self.c3 = nn.Conv3d(2, 8, 3, stride=2, padding=1)
        self.fc = nn.Linear(24, 10)

    def forward(self, xs):
        x1, x3 = xs
        return self.fc(torch.cat([self.c1(x1).mean(2), self.c3(x3).mean((2, 3, 4))], 1))


def _data(name, step):
    g = torch.Generator().manual_seed(step)
    if name == 'swiglu':
        x = torch.randn(4, 16, 32, generator=g).to(DEV)
        return x, torch.randint(0, 16, (4, 16), generator=g).to(DEV)
    if name == 'conv':
        return torch.randn(2, 3, 8, 8, generator=g).to(DEV), torch.randint(0, 10, (2,), generator=g).to(DEV)
    x = (torch.randn(3, 4, 40, generator=g).to(DEV), torch.randn(3, 2, 6, 7, 5, generator=g).to(DEV))
    return x, torch.randint(0, 10, (3,), generator=g).to(DEV)


MODELS = {'swiglu': (SwiGLU, dict(diagonal_a_layers=['down'], diagonal_g_layers=['gate', 'up'])),
          'conv': (ConvNet, dict(diagonal_a_layers=['wide'])),
          'nd': (NdNet, dict(diagonal_a_layers=['c1', 'c3'], precondition_conv_nd=True))}


def _loss(name, model, x, y):
    out = model(x)
    return F.cross_entropy(out.flatten(0, -2) if name == 'swiglu' else out, y.flatten())


def _grad_matrix(m):
    g = m.weight.grad.double().reshape(m.weight.shape[0], -1)
    bias = getattr(m, 'bias', None)
    return torch.cat([g, bias.grad.double()[:, None]], 1) if bias is not None else g


def _eigh(Fm):
    d, q = torch.linalg.eigh(Fm.double())
    return q, d.clamp(min=0)


def _inv(Fm, damping):
    return torch.linalg.inv(Fm.double() + damping * torch.eye(Fm.shape[0], dtype=torch.float64, device=Fm.device))


def p_ref(l, method, grad, A, G, damping):
    """fp64 P of a dense, diagonal-A (A a vector) or diagonal-G (G a vector) Linear / conv layer."""
    if l.diag_a:
        if method == 'inverse':
            return (_inv(G, damping) @ grad) / (A.double()[None, :] + damping)
        qg, dg = _eigh(G)
        return qg @ ((qg.t() @ grad) / (dg[:, None] * A.double()[None, :] + damping))
    if l.diag_g:
        if method == 'inverse':
            return (grad / (G.double()[:, None] + damping)) @ _inv(A, damping)
        qa, da = _eigh(A)
        return ((grad @ qa) / (G.double()[:, None] * da[None, :] + damping)) @ qa.t()
    if method == 'inverse':
        return _inv(G, damping) @ grad @ _inv(A, damping)
    qa, da = _eigh(A)
    qg, dg = _eigh(G)
    return qg @ ((qg.t() @ grad @ qa) / (dg[:, None] * da[None, :] + damping)) @ qa.t()


def _a_rows64(m, x, reduce):
    """fp64 A rows of one call of a Linear or Conv2d (ones column included; conv rows scaled by 1/S, reduce rows)."""
    x = x.double()
    if isinstance(m, nn.Linear):
        if reduce and x.dim() > 2:
            x = x.mean(tuple(range(1, x.dim() - 1)))
        r = x.reshape(-1, x.shape[-1])
        return torch.cat([r, torch.ones(r.shape[0], 1, dtype=r.dtype, device=r.device)], 1) if m.bias is not None else r
    u = F.unfold(x, m.kernel_size, padding=m.padding, stride=m.stride)          # (B, C k k, S)
    Sp = u.shape[2]
    u = torch.cat([u, torch.ones(u.shape[0], 1, Sp, dtype=u.dtype, device=u.device)], 1) if m.bias is not None else u
    if reduce and Sp > 1:
        return u.mean(2) / Sp
    return u.transpose(1, 2).reshape(-1, u.shape[1]) / Sp


SCHEDULES = {'every': (1, 1, 1), 'f2i4': (2, 4, 1), 'accum2': (1, 2, 2),
             'callable': (lambda s: 1 if s < 3 else 2, lambda s: 2 if s < 3 else 4, 1)}


@pytest.mark.parametrize('approx', ['expand', 'reduce'])
@pytest.mark.parametrize('schedule', list(SCHEDULES))
@pytest.mark.parametrize('method', ['eigen', 'inverse'])
@pytest.mark.parametrize('name', list(MODELS))
def test_model_against_fp64(name, method, schedule, approx):
    """Every layer's written gradient (kl-clip off: exactly P) against fp64 from the factors the preconditioner holds
    at its inverse steps, and the diagonal A of the Linear / Conv2d layers against an fp64 restatement of its EMA
    (the N-d ones against a dense twin in test_nd_diagonal_is_the_dense_diagonal)."""
    from kfac_b200.preconditioner import KFACPreconditioner
    cls, kw = MODELS[name]
    fus, ius, acc = SCHEDULES[schedule]
    damping, alpha = 0.003, 0.9
    torch.manual_seed(0)
    model = cls().to(DEV)
    pre = KFACPreconditioner(model, factor_update_steps=fus, inv_update_steps=ius, accumulation_steps=acc,
                             damping=damping, factor_decay=alpha, kl_clip=None, compute_method=method,
                             kfac_approx=approx, **kw)
    layers = {m: l for m, (_, l) in pre._layers.items()}
    diag = {m: l for m, l in layers.items() if l.diag_a}
    assert diag and all(l.a_factor_shape == (l.a_dim,) for l in diag.values())
    seen = {}
    for m in diag:
        m.register_forward_pre_hook(lambda mod, inp: seen.setdefault(mod, []).append(inp[0].detach()))
    opt = torch.optim.SGD(model.parameters(), lr=0.05)
    A_ref, snap = {}, {}
    for s in range(6):
        is_factor = s % pre.factor_update_steps == 0
        is_inv = s % pre.inv_update_steps == 0
        opt.zero_grad()
        seen.clear()
        for k in range(acc):          # accumulation_steps micro-batches of one step
            x, y = _data(name, 10 * s + k)
            (_loss(name, model, x, y) / acc).backward()
        grads = {m: _grad_matrix(m) for m in layers}
        pre.step()
        torch.cuda.synchronize()
        if is_factor and name != 'nd':
            for m in diag:
                win = sum(((r := _a_rows64(m, xi, approx == 'reduce')) ** 2).sum(0) / r.shape[0]
                          for xi in seen[m]) / len(seen[m])
                A_ref[m] = alpha * (torch.ones_like(win) if m not in A_ref else A_ref[m]) + (1 - alpha) * win
                assert rel_fro(layers[m].a_factor, A_ref[m]) < 1e-5, (s, pre._layers[m][0])
        if is_inv:
            snap = {m: (l.a_factor.double(), l.g_factor.double()) for m, l in layers.items()}
            for l in diag.values():
                assert l.qa is None and l.a_inv is None and l.dgda is None and torch.equal(l.da, l.a_factor)
                assert (l.qg is not None) if method == 'eigen' else (l.g_inv is not None)
        for m, l in layers.items():
            A, G = snap[m]
            ref = p_ref(l, method, grads[m], A, G, damping)
            got = _grad_matrix(m)
            assert rel_fro(got, ref) < 1e-3, (s, pre._layers[m][0], rel_fro(got, ref))
        opt.step()


@pytest.mark.parametrize('approx', ['expand', 'reduce'])
def test_nd_diagonal_is_the_dense_diagonal(approx):
    """The diagonal A of Conv1d / Conv3d layers equals the diagonal of the dense A their twin forms, to fp32 rounding,
    over a few factor steps."""
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(0)
    m_diag = NdNet().to(DEV)
    m_dense = copy.deepcopy(m_diag)
    p_diag = KFACPreconditioner(m_diag, precondition_conv_nd=True, diagonal_a_layers=['c1', 'c3'], kfac_approx=approx)
    p_dense = KFACPreconditioner(m_dense, precondition_conv_nd=True, kfac_approx=approx)
    for s in range(3):
        for model, pre in ((m_diag, p_diag), (m_dense, p_dense)):
            model.zero_grad()
            x, y = _data('nd', s)
            _loss('nd', model, x, y).backward()
            pre.step()
    torch.cuda.synchronize()
    for name in ('c1', 'c3'):
        la = p_diag._layers[getattr(m_diag, name)][1]
        ld = p_dense._layers[getattr(m_dense, name)][1]
        assert la.a_factor.shape == (la.a_dim,) and ld.a_factor.shape == (la.a_dim, la.a_dim)
        assert torch.allclose(la.a_factor, ld.a_factor.diagonal(), rtol=1e-5, atol=0), name
        assert torch.equal(la.g_factor, ld.g_factor), name


@pytest.mark.parametrize('name', ['swiglu', 'conv'])
@pytest.mark.parametrize('method', ['eigen', 'inverse'])
def test_first_step_other_gradients_unchanged(name, method):
    """Same weights, same batch, kl-clip off: the dense layers get the same bits with the diagonal-A layers skipped
    and with them diagonal (the diagonal-G layers share their eigensolver call with the diagonal-A layers' G)."""
    from kfac_b200.preconditioner import KFACPreconditioner
    cls, kw = MODELS[name]
    torch.manual_seed(0)
    m_diag = cls().to(DEV)
    m_skip = copy.deepcopy(m_diag)
    skip = dict(kw, skip_layers=kw['diagonal_a_layers'])
    del skip['diagonal_a_layers']
    out = []
    for model, k in ((m_diag, kw), (m_skip, skip)):
        pre = KFACPreconditioner(model, kl_clip=None, compute_method=method, **k)
        x, y = _data(name, 0)
        _loss(name, model, x, y).backward()
        pre.step()
        torch.cuda.synchronize()
        out.append({n: p.grad.clone() for n, p in model.named_parameters()})
    dense = ('inp', 'head') if name == 'swiglu' else ('stem', 'fc')
    for n in out[0]:
        if n.split('.')[0] in dense:
            assert torch.equal(bits(out[0][n]), bits(out[1][n])), n
    wide = 'down' if name == 'swiglu' else 'wide'
    assert not torch.equal(out[0][f'{wide}.weight'], out[1][f'{wide}.weight'])


def test_kl_clip_includes_the_diagonal_a_layer():
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(0)
    m_p = SwiGLU().to(DEV)
    m_c = copy.deepcopy(m_p)
    x, y = _data('swiglu', 1)
    lr = 0.1
    res = []
    for model, kl in ((m_p, None), (m_c, 1e-3)):
        pre = KFACPreconditioner(model, kl_clip=kl, lr=lr, **MODELS['swiglu'][1])
        _loss('swiglu', model, x, y).backward()
        grads = {n: p.grad.double().clone() for n, p in model.named_parameters()}
        pre.step()
        torch.cuda.synchronize()
        res.append((pre, grads, {n: p.grad.clone() for n, p in model.named_parameters()}))
    _, grads, P = res[0]
    vg = sum(float((P[n].double() * grads[n]).sum()) for n in P)
    nu_ref = min(1.0, (1e-3 / abs(vg * lr * lr)) ** 0.5)
    pre_c, _, written = res[1]
    nu = pre_c._compute_grad_scale()
    assert nu_ref < 1.0 and abs(nu - nu_ref) <= 1e-5 * nu_ref, (nu, nu_ref)
    down = sum(float((P[n].double() * grads[n]).sum()) for n in ('down.weight', 'down.bias')) / vg
    assert down > 1e-6
    for n in P:
        assert torch.equal(written[n], pre_c.last_grad_scale * P[n]), n


def test_state_dict_round_trip():
    from kfac_b200.preconditioner import KFACPreconditioner
    kw = MODELS['conv'][1]
    torch.manual_seed(0)
    m1 = ConvNet().to(DEV)
    pre1 = KFACPreconditioner(m1, kl_clip=None, inv_update_steps=2, **kw)
    opt = torch.optim.SGD(m1.parameters(), lr=0.05)
    for s in range(3):
        x, y = _data('conv', s)
        opt.zero_grad()
        _loss('conv', m1, x, y).backward()
        pre1.step()
        opt.step()
    sd = pre1.state_dict()
    assert sd['layers']['wide']['A'].shape == (9217,) and sd['layers']['wide']['G'].shape == (64, 64)
    mem = pre1.memory_usage()
    assert mem['a_factors'] == 4 * (4 * 4 + 9217 + 65 * 65)
    m2 = ConvNet().to(DEV)
    m2.load_state_dict(m1.state_dict())
    pre2 = KFACPreconditioner(m2, kl_clip=None, inv_update_steps=2, **kw)
    pre2.load_state_dict(sd)
    for model, pre in ((m1, pre1), (m2, pre2)):
        model.zero_grad()
        x, y = _data('conv', 3)
        _loss('conv', model, x, y).backward()
        pre.step()
    torch.cuda.synchronize()
    for (n, p1), (_, p2) in zip(m1.named_parameters(), m2.named_parameters()):
        assert torch.equal(p1.grad, p2.grad), n
    bad = copy.deepcopy(sd)
    bad['layers']['wide']['A'] = torch.ones(9217, 9217, device=DEV)
    with pytest.raises(ValueError, match=r'diagonal-A layer factor A has shape \(9217, 9217\), expected \(9217,\)'):
        KFACPreconditioner(ConvNet().to(DEV), **kw).load_state_dict(bad)
    small = SwiGLU().to(DEV)
    pre = KFACPreconditioner(small, **MODELS['swiglu'][1])
    sd = pre.state_dict()
    sd['layers']['inp']['A'] = torch.ones(33, device=DEV)        # a vector into a dense A
    with pytest.raises(ValueError, match=r'factor A has shape \(33,\), expected \(33, 33\)'):
        pre.load_state_dict(sd)


def test_fp16_overflow_drops_the_windows():
    """An injected fp16 overflow under a GradScaler: every G window is dropped and counted once; the diagonal A
    windows (finite) go through the guarded vector EMA and are kept; training stays finite."""
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(0)
    model = SwiGLU().to(DEV)
    scaler = torch.amp.GradScaler('cuda', init_scale=2.0 ** 10)
    pre = KFACPreconditioner(model, grad_scaler=scaler, damping=0.003, **MODELS['swiglu'][1])
    layers = {m: l for m, (_, l) in pre._layers.items()}
    ld = layers[model.down]
    opt = torch.optim.SGD(model.parameters(), lr=0.01)
    for step in range(5):
        x, y = _data('swiglu', step)
        opt.zero_grad()
        if step == 2:
            scaler.update(new_scale=2.0 ** 60)
            before = {m: l.g_factor.clone() for m, l in layers.items()}
            a_before = ld.a_factor.clone()
        with torch.autocast('cuda', dtype=torch.float16):
            loss = _loss('swiglu', model, x, y).float()
        scaler.scale(loss).backward()
        scaler.unscale_(opt)
        pre.step()
        torch.cuda.synchronize()
        if step == 2:
            for m, l in layers.items():
                assert torch.equal(l.g_factor, before[m]), pre._layers[m][0]
            assert pre.skipped_factor_updates == len(layers)
            assert not torch.equal(ld.a_factor, a_before)
        elif step > 2:
            for p in model.parameters():
                assert torch.isfinite(p.grad).all(), step
        scaler.step(opt)
        scaler.update(new_scale=2.0 ** 10) if step == 2 else scaler.update()
    assert torch.isfinite(ld.g_factor).all() and torch.isfinite(ld.a_factor).all()


@pytest.mark.parametrize('name', list(MODELS))
def test_no_host_sync_in_hooks(name):
    from kfac_b200.preconditioner import KFACPreconditioner
    cls, kw = MODELS[name]
    torch.manual_seed(0)
    model = cls().to(DEV)
    scaler = torch.amp.GradScaler('cuda', init_scale=2.0 ** 10)
    pre = KFACPreconditioner(model, grad_scaler=scaler, **kw)
    opt = torch.optim.SGD(model.parameters(), lr=0.01)
    for s in range(2):
        x, y = _data(name, s)
        opt.zero_grad()
        torch.cuda.synchronize()
        if s == 1:
            torch.cuda.set_sync_debug_mode('error')
        try:
            with torch.autocast('cuda', dtype=torch.float16):
                loss = _loss(name, model, x, y).float()
            scaler.scale(loss).backward()
        finally:
            torch.cuda.set_sync_debug_mode(0)
        scaler.unscale_(opt)
        pre.step()
        scaler.step(opt)
        scaler.update()
    torch.cuda.synchronize()
    for _, l in pre._layers.values():
        assert l._a_count == 0 and l._has_a


# ---------------------------------------------------------------------------------------------- two ranks
def _run_dist(backend):
    import socket
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    script = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'dist_diag_a.py')
    out = subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node=2',
                          '--master-addr', '127.0.0.1', '--master-port', str(port), script, '--backend', backend],
                         capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, (out.stdout[-3000:], out.stderr[-3000:])
    assert out.stdout.count('dist_diag_a ok') == 2, out.stdout[-2000:]


def test_two_ranks_gloo():
    """Two ranks over gloo (they may share one GPU), COMM_OPT and MEM_OPT: P identical on both ranks and equal to
    fp64 on the concatenated batch."""
    _run_dist('gloo')


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='NCCL needs one GPU per rank')
def test_two_ranks_nccl():
    _run_dist('nccl')
