"""pi-adjusted damping (`pi_damping=True`) on the GPU, everything against the fp64 restatement of
tests/test_pi_damping_host.py:

  * kfac_pi: dense factors with padded leading dimensions (n up to 8192), vectors (V = 50257), many items in one call
    (more than one launch's worth), zero, negative and non-finite traces (pi = 1), and the same bits on a repeat;
  * kfac_dgda_pi and kfac_inverse_from_eigh_pi, the latter bit-equal to kfac_inverse_from_eigh at damping gamma;
  * kfac_precondition with pi items of every kind (dense eigen with and without dgda, inverse, embedding, diagonal-G,
    diagonal-A, a transposed convolution's wgrad_taps) at SIMT-fallback sizes and with split reductions (> 1024),
    fp32 / fp16 / bf16 gradients; pi items mixed with NULL-pi items (whose P keeps its bits) and peer stores (P's bits);
    a tied item with pi rejected;
  * scale invariance bit for bit: factors (A, G) and (4^k A, G / 4^k) give the same P bits under pi_damping (eigen
    with and without dgda, inverse; a bias-free dense layer and a diagonal-G layer), and different bits without it;
  * models (a conv net with BatchNorm and a diagonal-A layer, an embedding -> attention -> diagonal-G head, an LSTM)
    under eigen (dgda on and off) and inverse, integer and callable damping, inv_update_steps=3: every written gradient
    against fp64 from the factors of the last inverse step, pi frozen between inverse steps, the normalization layers'
    gradients bit-identical to a run without the keyword, and step() without host syncs;
  * a short training run whose loss decreases under both methods, and two ranks (tests/dist_pi_damping.py).
"""
import ctypes as C
import math
import os
import socket
import subprocess
import sys

import pytest
import torch
from torch import nn
from torch.nn import functional as F

from conftest import rel_fro
from test_pi_damping_host import f32, gammas, pi_ref, precondition_ref

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda')
DAMPING = 0.003


@pytest.fixture(scope='module')
def lib():
    from kfac_b200 import _cabi
    return _cabi.load()


def S():
    return torch.cuda.current_stream().cuda_stream


def bits(x):
    return x.contiguous().view(torch.int32 if x.element_size() == 4 else torch.int16)


def _pi_call(lib, facs):
    """kfac_pi over [(A storage, G storage, a, g, lda, ldg)]: the pi tensor (NaN-filled before the call)"""
    from kfac_b200 import _cabi
    out = torch.full((len(facs),), float('nan'), device=DEV)
    items = (_cabi.PiItem * len(facs))()
    for i, (A, G, a, g, lda, ldg) in enumerate(facs):
        items[i] = _cabi.PiItem(A.data_ptr(), G.data_ptr(), out.data_ptr() + 4 * i, a, g, lda, ldg)
    assert lib.kfac_pi(items, len(facs), S()) == 0, lib.kfac_last_error()
    torch.cuda.synchronize()
    return out


def _dense(n, gen, ld=None, scale=1.0):
    """A factor's storage (n x ld, NaN in the padding) and its logical (n x n) matrix"""
    ld = ld or n + 3
    x = torch.randn(2 * n + 8, n, device=DEV, generator=gen)
    Fm = (x.t() @ x / x.shape[0] * scale).float()
    st = torch.full((n, ld), float('nan'), device=DEV)
    st[:, :n] = Fm
    return st, Fm


def _close_pi(got, ref):
    return abs(got - ref) <= 2.0 ** -22 * abs(ref)


def test_pi_against_fp64_traces(lib):
    gen = torch.Generator(device=DEV).manual_seed(1)
    facs, refs = [], []
    for n, m in ((1, 3), (3, 129), (129, 2049), (2049, 4608), (4608, 8192), (8192, 1)):
        A, Am = _dense(n, gen, scale=0.01)
        G, Gm = _dense(m, gen, ld=m + (4 if m > 1 else 0), scale=3e-7)
        facs.append((A, G, n, m, A.shape[1], G.shape[1]))
        refs.append(pi_ref(Am, Gm))
        del Am, Gm
    f = torch.rand(50257, device=DEV, generator=gen) / 50257          # an embedding's token frequencies
    G, Gm = _dense(768, gen, scale=1e-8)
    facs.append((f, G, 50257, 768, 0, G.shape[1]))
    refs.append(pi_ref(f, Gm))
    head = torch.rand(50257, device=DEV, generator=gen) * 1e-9       # a diagonal-G head
    A, Am = _dense(769, gen)
    facs.append((A, head, 769, 50257, A.shape[1], 0))
    refs.append(pi_ref(Am, head))
    got = _pi_call(lib, facs)
    for i, r in enumerate(refs):
        assert _close_pi(float(got[i]), r), (i, float(got[i]), r)
    assert torch.equal(bits(got), bits(_pi_call(lib, facs)))
    del facs


def test_pi_many_items_and_degenerate_traces(lib):
    gen = torch.Generator(device=DEV).manual_seed(2)
    facs, refs = [], []
    for i in range(1000):                               # more items than one launch takes
        a, g = 1 + i % 37, 1 + (7 * i) % 53
        if i % 3 == 0:                                  # a vector factor
            A = Am = torch.rand(a, device=DEV, generator=gen) * 10 ** (i % 7 - 3)
            lda = 0
        else:
            A, Am = _dense(a, gen, ld=a + i % 5, scale=10 ** (i % 5 - 2))
            lda = A.shape[1]
        G, Gm = _dense(g, gen, ld=g, scale=10 ** (i % 9 - 6))
        facs.append((A, G, a, g, lda, g))
        refs.append(pi_ref(Am, Gm))
    nan, inf = float('nan'), float('inf')
    degenerate = [torch.zeros(5, device=DEV), -torch.ones(5, device=DEV), torch.tensor([1.0, inf], device=DEV),
                  torch.tensor([nan, 1.0], device=DEV), torch.tensor([inf, -inf], device=DEV)]
    ok = torch.rand(6, device=DEV, generator=gen) + 0.5
    for v in degenerate:
        facs += [(v, ok, v.numel(), 6, 0, 0), (ok, v, 6, v.numel(), 0, 0)]
        refs += [1.0, 1.0]
    got = _pi_call(lib, facs)
    for i, r in enumerate(refs):
        assert _close_pi(float(got[i]), r), (i, float(got[i]), r)
    assert torch.equal(bits(got), bits(_pi_call(lib, facs)))
    assert float(got[-1]) == 1.0 and float(got[-10]) == 1.0


def test_dgda_pi_and_inverse_pi(lib):
    gen = torch.Generator(device=DEV).manual_seed(3)
    from kfac_b200 import _cabi
    s = f32(math.sqrt(f32(DAMPING)))
    for g, a, p in ((10, 21, 0.37), (769, 1025, 3.5), (64, 4097, 1.0)):
        dg = torch.rand(g, device=DEV, generator=gen) ** 3
        da = torch.rand(a, device=DEV, generator=gen) ** 3 * 5
        pi = torch.tensor([p], device=DEV)
        out = torch.full((g, _cabi.ld4(a) + 4), float('nan'), device=DEV)
        assert lib.kfac_dgda_pi(dg.data_ptr(), da.data_ptr(), g, a, s, pi.data_ptr(), out.data_ptr(), out.shape[1],
                                S()) == 0
        ga, gg = gammas(p, DAMPING)
        ref = 1.0 / ((dg.double()[:, None] + gg) * (da.double()[None, :] + ga))
        assert float(((out[:, :a].double() - ref).abs() / ref).max()) < 1e-6
        assert torch.all(out[:, a:] == 0)
    for n in (40, 700, 1500):
        q, _ = torch.linalg.qr(torch.randn(n, n, dtype=torch.float64, device=DEV, generator=gen))
        d = (torch.rand(n, device=DEV, generator=gen) ** 4).float()
        ld = _cabi.ld4(n)
        Q = torch.zeros(n, ld, device=DEV)
        Q[:, :n] = q.float()
        ws = torch.empty(n * ld, device=DEV)
        for side, p in ((1, 0.25), (-1, 0.25), (1, 7.0)):
            pi = torch.tensor([p], device=DEV)
            inv = torch.full((n, ld), float('nan'), device=DEV)
            assert lib.kfac_inverse_from_eigh_pi(Q.data_ptr(), ld, d.data_ptr(), n, s, pi.data_ptr(), side,
                                                 inv.data_ptr(), ld, ws.data_ptr(), ws.numel() * 4, S()) == 0
            gam = gammas(p, DAMPING)[0 if side == 1 else 1]
            ref = (Q[:, :n].double() / (d.double() + gam)) @ Q[:, :n].double().t()
            assert rel_fro(inv[:, :n], ref) < 1e-5, (n, side)
            same = torch.full_like(inv, float('nan'))
            assert lib.kfac_inverse_from_eigh(Q.data_ptr(), ld, d.data_ptr(), n, gam, same.data_ptr(), ld,
                                              ws.data_ptr(), ws.numel() * 4, S()) == 0
            torch.cuda.synchronize()
            assert torch.equal(bits(inv[:, :n]), bits(same[:, :n]))
    pi = torch.ones(1, device=DEV)
    assert lib.kfac_inverse_from_eigh_pi(Q.data_ptr(), ld, d.data_ptr(), n, s, pi.data_ptr(), 0, inv.data_ptr(), ld,
                                         ws.data_ptr(), ws.numel() * 4, S()) == _cabi.KFAC_ERR_BAD_ARG


# ------------------------------------------------------------------------------------------- kfac_precondition
def _stored(x):
    from kfac_b200 import _cabi
    out = torch.full((x.shape[0], _cabi.ld4(x.shape[1])), float('nan'), device=DEV)
    out[:, :x.shape[1]] = x
    return out


def _basis(n, gen, scale):
    q, _ = torch.linalg.qr(torch.randn(n, n, dtype=torch.float64, device=DEV, generator=gen))
    return q.float(), ((torch.rand(n, dtype=torch.float64, device=DEV, generator=gen) ** 4) * scale).float()


def _damped64(q, d, gam):
    return (q.double() / (d.double() + gam)) @ q.double().t()


# (kind, g, a, bias, dtype, taps): a = the gradient matrix's columns (bias included); an embedding is (d, V)
SPECS = [('dense', 256, 129, 1, torch.float32, 0), ('dense', 10, 21, 1, torch.bfloat16, 0),
         ('dense', 1100, 65, 0, torch.float16, 0), ('dense', 72, 1037, 1, torch.float32, 0),
         ('taps', 40, 8 * 9 + 1, 1, torch.float32, 9), ('taps', 96, 16 * 4, 0, torch.bfloat16, 4),
         ('emb', 48, 1000, 0, torch.float16, 0), ('emb', 1030, 300, 0, torch.float32, 0),
         ('diag_g', 10007, 769, 1, torch.float32, 0), ('diag_g', 20, 33, 0, torch.bfloat16, 0),
         ('diag_a', 769, 9217, 1, torch.bfloat16, 0), ('diag_a', 1500, 100, 0, torch.float16, 0),
         ('diag_a', 12, 40, 1, torch.float32, 0)]


def _make_layers(gen, method):
    """Each spec's gradient, second-order data (with its own pi) and fp64 P"""
    eigen = method == 'eigen'
    out = []
    for i, (kind, g, a, bias, dtype, taps) in enumerate(SPECS):
        p = (0.3, 2.0, 17.0, 1.0)[i % 4]
        ga, gg = gammas(p, DAMPING)
        L = dict(kind=kind, g=g, a=a, dtype=dtype, taps=taps, pi=torch.tensor([p], device=DEV))
        aw = a - bias
        if kind == 'emb':
            L['w'] = torch.randn(a, g, device=DEV, generator=gen).to(dtype)   # (V, d)
            L['b'] = None
            grad = L['w'].double().t()
        elif kind == 'taps':
            L['w'] = torch.randn(aw // taps, g, taps, device=DEV, generator=gen).to(dtype)
            L['b'] = torch.randn(g, device=DEV, generator=gen).to(dtype) if bias else None
            grad = L['w'].double().permute(1, 0, 2).reshape(g, aw)
        else:
            L['w'] = torch.randn(g, aw, device=DEV, generator=gen).to(dtype)
            L['b'] = torch.randn(g, device=DEV, generator=gen).to(dtype) if bias else None
            grad = L['w'].double()
        if L['b'] is not None:
            grad = torch.cat([grad, L['b'].double()[:, None]], 1)
        # factors: dense ones as a basis and eigenvalues, diagonal ones as vectors; a different scale on each side
        if kind in ('dense', 'taps', 'diag_g'):
            qa, da = _basis(a, gen, 2.0)
            L.update(qa=_stored(qa), qaT=_stored(qa.t()), da=da, a_inv=_stored(_damped64(qa, da, ga).float()))
            MA = _damped64(qa, da, ga)
        else:
            av = torch.rand(a, device=DEV, generator=gen) ** 2 * 1e-3
            av[::7] = 0
            L['da'] = av
            MA = 1.0 / (av.double() + ga)
        if kind in ('dense', 'taps', 'emb', 'diag_a'):
            qg, dg = _basis(g, gen, 1e-5)
            L.update(qg=_stored(qg), qgT=_stored(qg.t()), dg=dg, g_inv=_stored(_damped64(qg, dg, gg).float()))
            MG = _damped64(qg, dg, gg)
        else:
            dgv = torch.rand(g, device=DEV, generator=gen) * 1e-6
            L['dg'] = dgv
            MG = 1.0 / (dgv.double() + gg)
        if kind in ('dense', 'taps') and i % 2 == 0:     # dgda formed with pi (the outer-product path)
            L['dgda'] = _stored((1.0 / ((L['dg'].double()[:, None] + gg) * (L['da'].double()[None, :] + ga))).float())
        ref = (MG[:, None] * grad if MG.dim() == 1 else MG @ grad)
        ref = ref * MA[None, :] if MA.dim() == 1 else ref @ MA
        L['ref'] = (ref.t() if kind == 'emb' else ref).float()
        out.append(L)
    return out


def _precondition(lib, layers, method, use_pi, peers=False):
    """One kfac_precondition over `layers` (use_pi[i]: item i carries its pi): the P tensors and peer copies"""
    from kfac_b200 import _cabi
    e = method == 'eigen'
    kinds = {'dense': _cabi.KFAC_ITEM_DENSE, 'taps': _cabi.KFAC_ITEM_DENSE, 'emb': _cabi.KFAC_ITEM_EMBEDDING,
             'diag_g': _cabi.KFAC_ITEM_DIAG_G, 'diag_a': _cabi.KFAC_ITEM_DIAG_A}
    items = (_cabi.PrecondItem * len(layers))()
    out, keep = [], []
    for i, L in enumerate(layers):
        ptr = lambda k: L[k].data_ptr() if k in L and L[k] is not None else None  # noqa: E731,B023
        rows, cols = (L['a'], L['g']) if L['kind'] == 'emb' else (L['g'], L['a'])
        P = torch.full((rows, _cabi.ld4(cols)), float('nan'), device=DEV)
        it = _cabi.PrecondItem()
        it.wgrad, it.bgrad, it.grad_dtype = ptr('w'), ptr('b'), _cabi.DTYPE_CODE[L['dtype']]
        it.g, it.a, it.kind, it.wgrad_taps = L['g'], L['a'], kinds[L['kind']], L['taps']
        for f in ('qa', 'qaT', 'qg', 'qgT'):
            setattr(it, f, ptr(f) if e else None)
        it.a_inv, it.g_inv = (None, None) if e else (ptr('a_inv'), ptr('g_inv'))
        it.da, it.dg = ptr('da'), ptr('dg')
        it.dgda = ptr('dgda') if e and use_pi[i] else None
        it.ldqa, it.ldqg, it.ld_dgda = _cabi.ld4(L['a']), _cabi.ld4(L['g']), _cabi.ld4(L['a'])
        it.P, it.ldp = P.data_ptr(), P.shape[1]
        it.pi = L['pi'].data_ptr() if use_pi[i] else None
        peer = None
        if peers:                         # a second local buffer stands in for a peer's P entry
            peer = torch.full_like(P, float('nan'))
            arr = (C.c_void_p * 1)(peer.data_ptr())
            keep.append(arr)
            it.peer_P, it.n_peers = arr, 1
        items[i] = it
        out.append((P[:, :cols], peer))
    need = lib.kfac_precondition_workspace_bytes(items, len(layers))
    ws = torch.full((need,), 255, dtype=torch.uint8, device=DEV)
    rc = lib.kfac_precondition(items, len(layers), _cabi.KFAC_EIGEN if e else _cabi.KFAC_INVERSE, DAMPING,
                               ws.data_ptr(), need, S())
    assert rc == 0, lib.kfac_last_error()
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize('method', ['eigen', 'inverse'])
def test_precondition_pi_items_against_fp64(lib, method):
    gen = torch.Generator(device=DEV).manual_seed(5)
    layers = _make_layers(gen, method)
    n = len(layers)
    got = _precondition(lib, layers, method, [True] * n)
    for L, (P, _) in zip(layers, got):
        err = rel_fro(P, L['ref'])
        assert err < 1e-3, (method, L['kind'], L['g'], L['a'], L['dtype'], err)
    again = _precondition(lib, layers, method, [True] * n, peers=True)
    for (p1, _), (p2, peer) in zip(got, again):
        assert torch.equal(bits(p1), bits(p2)) and torch.equal(bits(peer[:, :p1.shape[1]]), bits(p1))
    # pi items mixed with NULL-pi items: the NULL items keep the bits of a call without the pi items
    mixed = [i % 2 == 0 for i in range(n)]
    with_pi = _precondition(lib, layers, method, mixed, peers=True)
    alone_layers = [L for L, m in zip(layers, mixed) if not m]
    alone = iter(_precondition(lib, alone_layers, method, [False] * len(alone_layers)))
    for L, m, (P, peer), (p1, _) in zip(layers, mixed, with_pi, got):
        assert torch.equal(bits(peer[:, :P.shape[1]]), bits(P))
        if m:
            assert torch.equal(bits(P), bits(p1))
        else:
            assert torch.equal(bits(P), bits(next(alone)[0]))


def test_precondition_rejects_a_tied_item_with_pi(lib):
    from kfac_b200 import _cabi
    V, d = 100, 16
    w, P = torch.zeros(V, d, device=DEV), torch.full((V, d), 7.0, device=DEV)
    q, vec, pi = torch.eye(d, device=DEV), torch.ones(V, device=DEV), torch.ones(1, device=DEV)
    it = _cabi.PrecondItem(w.data_ptr(), None, 0, d, V, qg=q.data_ptr(), qgT=q.data_ptr(), da=vec.data_ptr(),
                           dg=vec.data_ptr(), ldqg=d, P=P.data_ptr(), ldp=d, kind=_cabi.KFAC_ITEM_TIED,
                           dh=vec.data_ptr(), tied_damping=0.5, pi=pi.data_ptr())
    items = (_cabi.PrecondItem * 1)(it)
    need = lib.kfac_precondition_workspace_bytes(items, 1)
    ws = torch.empty(need, dtype=torch.uint8, device=DEV)
    n0 = lib.kfac_launch_count()
    assert lib.kfac_precondition(items, 1, _cabi.KFAC_EIGEN, 1e-3, ws.data_ptr(), need, S()) == _cabi.KFAC_ERR_BAD_ARG
    assert 'pi' in _cabi.last_error() and lib.kfac_launch_count() == n0
    torch.cuda.synchronize()
    assert torch.all(P == 7.0)


# ------------------------------------------------------------------------------------------- scale invariance
def _spd(n, gen, top):
    """A symmetric positive definite factor whose largest entry is `top`"""
    x = torch.randn(3 * n, n, dtype=torch.float64, device=DEV, generator=gen)
    Fm = x.t() @ x / (3 * n)
    return (Fm / Fm.abs().max() * top).float()


@pytest.mark.parametrize('method,prediv', [('eigen', True), ('eigen', False), ('inverse', False)])
def test_scale_invariance_bit_for_bit(method, prediv):
    """The largest entries of every factor, scaled or not, lie outside [1/16, 1): kfac_eigh_batched then gives the
    same basis and 4^k times the eigenvalues, pi becomes 4^k pi, and every product of P sees the same bits.  Without
    the keyword the inverse method's P differs; the eigen method's division by dg x da + damping damps the product
    and does not depend on the split either."""
    from kfac_b200.preconditioner import KFACPreconditioner
    gen = torch.Generator(device=DEV).manual_seed(9)
    A0, G0, A1 = _spd(96, gen, 1.5), _spd(80, gen, 24.0), _spd(80, gen, 1.25)
    G1 = (torch.rand(300, device=DEV, generator=gen) * 8 + 16).float()       # a diagonal G, largest in [16, 32)
    w0 = torch.randn(80, 96, device=DEV, generator=gen)
    w1 = torch.randn(300, 80, device=DEV, generator=gen)

    def run(k, pi_damping):
        c = 4.0 ** k
        model = nn.Sequential(nn.Linear(96, 80, bias=False), nn.Linear(80, 300, bias=False)).to(DEV)
        pre = KFACPreconditioner(model, damping=DAMPING, kl_clip=None, inv_update_steps=1000, compute_method=method,
                                 compute_eigenvalue_outer_product=prediv, diagonal_g_layers=['1'],
                                 pi_damping=pi_damping)
        pre.load_state_dict({'steps': 1, 'layers': {'0': {'A': A0 * c, 'G': G0 / c}, '1': {'A': A1 * c, 'G': G1 / c}}})
        model[0].weight.grad, model[1].weight.grad = w0.clone(), w1.clone()
        pre.step()
        torch.cuda.synchronize()
        return [model[0].weight.grad.clone(), model[1].weight.grad.clone()]

    base = run(0, True)
    for k in (1, 2):
        for p, q in zip(base, run(k, True)):
            assert torch.equal(bits(p), bits(q)), k
    if method == 'inverse':
        # (A + damping I)^-1 and (G + damping I)^-1 see the split; the eigen method's dg x da + damping does not
        off = [run(0, False), run(1, False)]
        for p, q in zip(*off):
            assert not torch.equal(bits(p), bits(q))


# ------------------------------------------------------------------------------------------- models
class ConvNet(nn.Module):
    def __init__(self):
        super().__init__()
        self.conv1 = nn.Conv2d(3, 8, 3, padding=1)
        self.bn = nn.BatchNorm2d(8)
        self.conv2 = nn.Conv2d(8, 16, 3, stride=2)
        self.fc = nn.Linear(16 * 7 * 7, 10)

    def forward(self, x):
        return self.fc(F.relu(self.conv2(F.relu(self.bn(self.conv1(x))))).flatten(1))


class EmbAttn(nn.Module):
    def __init__(self):
        super().__init__()
        self.emb = nn.Embedding(300, 32)
        self.attn = nn.MultiheadAttention(32, 4, batch_first=True)
        self.head = nn.Linear(32, 1000)

    def forward(self, x):
        h = self.emb(x)
        return self.head(h + self.attn(h, h, h, need_weights=False)[0])


class LSTMNet(nn.Module):
    def __init__(self):
        super().__init__()
        self.lstm = nn.LSTM(12, 24)
        self.fc = nn.Linear(24, 5)

    def forward(self, x):
        return self.fc(self.lstm(x)[0][-1])


MODELS = {
    'conv': (ConvNet, dict(precondition_norms=True, diagonal_a_layers=['fc'])),
    'emb_attn': (EmbAttn, dict(precondition_embeddings=True, precondition_attention=True, diagonal_g_layers=['^head$'])),
    'lstm': (LSTMNet, dict(precondition_recurrent=True)),
}


def _data(name, step):
    g = torch.Generator().manual_seed(100 + step)
    if name == 'conv':
        return torch.randn(16, 3, 16, 16, generator=g), torch.randint(0, 10, (16,), generator=g)
    if name == 'emb_attn':
        return torch.randint(0, 300, (8, 12), generator=g), torch.randint(0, 1000, (8, 12), generator=g)
    return torch.randn(7, 16, 12, generator=g), torch.randint(0, 5, (16,), generator=g)


def _loss(model, x, y):
    out = model(x.to(DEV))
    return F.cross_entropy(out.reshape(-1, out.shape[-1]), y.to(DEV).reshape(-1))


def _grad_matrix(l):
    """The layer's gradient as the (g, a) matrix [wgrad | bgrad] (an embedding's as (d, V)) in fp64"""
    m = l.module
    w = m.get_weight_grad().double()
    if l.embedding:
        return w.t()
    w = w.reshape(l.g_dim, -1)
    return torch.cat([w, m.get_bias_grad().double()[:, None]], 1) if m.has_bias() else w


SCHEDULES = {'int': DAMPING, 'callable': lambda step: DAMPING * (1 + step)}


@pytest.mark.parametrize('schedule', list(SCHEDULES))
@pytest.mark.parametrize('method,prediv', [('eigen', True), ('eigen', False), ('inverse', False)])
@pytest.mark.parametrize('name', list(MODELS))
def test_model_against_fp64(name, method, prediv, schedule):
    from kfac_b200.preconditioner import KFACPreconditioner
    cls, kw = MODELS[name]
    damping = SCHEDULES[schedule]
    runs = {}
    # deterministic cuDNN kernels: both runs get the same raw gradients, so the normalization layers' P can be compared
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    for on in (True, False):
        torch.manual_seed(0)
        model = cls().to(DEV)
        pre = KFACPreconditioner(model, damping=damping, kl_clip=None, inv_update_steps=3, compute_method=method,
                                 compute_eigenvalue_outer_product=prediv, pi_damping=on, **kw)
        layers = {n: l for n, l in pre._layers.values()}
        norm_grads, snap = [], None
        for step in range(5):
            x, y = _data(name, step)
            model.zero_grad()
            _loss(model, x, y).backward()        # the weights stay: every step sees the same model
            grads = {n: _grad_matrix(l) for n, l in layers.items()}
            lam = damping(step) if callable(damping) else damping
            if step > 0:
                torch.cuda.synchronize()
                torch.cuda.set_sync_debug_mode('error')
            try:
                pre.step()
            finally:
                torch.cuda.set_sync_debug_mode(0)
            torch.cuda.synchronize()
            norm_grads.append([p.grad.clone() for m in model.modules() if isinstance(m, nn.BatchNorm2d)
                               for p in m.parameters()])
            if not on:
                continue
            if step % 3 == 0:                     # an inverse step: the factors it decomposed, pi and its damping
                snap = {n: (l.a_factor.clone(), l.g_factor.clone(), float(l._inv['pi'][0])) for n, l in layers.items()}
                lam_inv = lam
            for n, l in layers.items():
                A, G, pi = snap[n]
                assert float(l._inv['pi'][0]) == pi, (n, step)          # frozen until the next inverse step
                assert _close_pi(pi, pi_ref(A, G)), (n, pi, pi_ref(A, G))
                if l.diag_side is None:
                    lam_a = lam_g = lam_inv if (method == 'inverse' or prediv) else lam
                elif method == 'eigen':
                    lam_a = lam_g = lam
                else:       # the dense side's inverse is formed at the inverse step, the diagonal side divides now
                    lam_a, lam_g = (lam, lam_inv) if l.diag_side == 'a' else (lam_inv, lam)
                ref = precondition_ref(grads[n], A, G, pi, lam_a, lam_g)
                err = rel_fro(_grad_matrix(l), ref)
                assert err < 1e-3, (name, method, prediv, schedule, step, n, err)
        runs[on] = norm_grads
        pre.close()
    torch.backends.cudnn.deterministic = False
    for a, b in zip(runs[True], runs[False]):
        for p, q in zip(a, b):
            assert torch.equal(bits(p), bits(q))


@pytest.mark.parametrize('method', ['eigen', 'inverse'])
def test_training_loss_decreases(method):
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(0)
    model = ConvNet().to(DEV)
    pre = KFACPreconditioner(model, damping=0.01, inv_update_steps=5, compute_method=method, pi_damping=True,
                             **MODELS['conv'][1])
    opt = torch.optim.SGD(model.parameters(), lr=0.05, momentum=0.9)
    g = torch.Generator().manual_seed(0)
    x, y = torch.randn(64, 3, 16, 16, generator=g), torch.randint(0, 10, (64,), generator=g)
    losses = []
    for _ in range(30):
        opt.zero_grad()
        loss = _loss(model, x, y)
        loss.backward()
        pre.step()
        opt.step()
        losses.append(float(loss.detach()))
    assert all(math.isfinite(v) for v in losses)
    assert sum(losses[-5:]) / 5 < 0.5 * sum(losses[:5]) / 5, losses


# ------------------------------------------------------------------------------------------- two ranks
def _run_dist(backend):
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    script = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'dist_pi_damping.py')
    out = subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node=2',
                          '--master-addr', '127.0.0.1', '--master-port', str(port), script, '--backend', backend],
                         capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, (out.stdout[-3000:], out.stderr[-3000:])
    assert out.stdout.count('dist_pi_damping ok') == 2, out.stdout[-2000:]


def test_two_ranks_gloo():
    """Two ranks over gloo (they may share one GPU): COMM_OPT and MEM_OPT under eigen and inverse, and
    colocate_factors=False under inverse."""
    _run_dist('gloo')


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='NCCL needs one GPU per rank')
def test_two_ranks_nccl():
    _run_dist('nccl')
