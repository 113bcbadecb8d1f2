"""K-FAC-reduce (`kfac_approx='reduce'`) on the GPU, everything against fp64:

  * the three reduce-row kernels against fp64 sums (relative error <= 1e-6), the same bits on a repeat call, and the
    per-example sum of the existing kfac_rows_* writer's rows;
  * R = 1 (a Linear on (B, d)) is bit-identical to expand under EIGEN, INVERSE and EKFAC;
  * a sequence Linear stack and resnet32 under EIGEN, INVERSE and EKFAC, callable schedules, factor_update_steps=2 /
    inv_update_steps=4, accumulation_steps=2 and a module called twice in a window: A, G and P (S for EKFAC, with the
    GPU's own eigenbases) against an fp64 restatement of the definition from the captured inputs and output gradients;
  * a GPT-shaped model with embeddings, norms and a diagonal-G head: the embedding and norm layers are bit-identical
    with reduce on and off, and the head's diagonal G matches fp64;
  * fp16 autocast with a GradScaler (an overflow step is dropped), EKFAC's row-buffer memory, a training run, and two
    ranks (tests/dist_reduce.py).
"""
import math
import os
import socket
import subprocess
import sys
import zlib

import pytest
import torch
from torch import nn

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
def _reduce_linear(lib, x, ones, scale, ls, ld):
    B, R, F = x.shape
    out = torch.full((B, ld), float('nan'), device=DEV)
    rc = lib.kfac_reduce_rows_linear(x.data_ptr(), _code(x.dtype), B, R, F, ones, scale,
                                     ls.data_ptr() if ls is not None else None, out.data_ptr(), ld, S())
    assert rc == 0, lib.kfac_last_error()
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize('F', [1, 5, 64, 769, 4096])
@pytest.mark.parametrize('R', [1, 7, 128, 2048])
@pytest.mark.parametrize('B', [1, 3, 32])
@pytest.mark.parametrize('dtype', DTYPES)
def test_reduce_rows_linear(lib, dtype, B, R, F):
    gen = torch.Generator(device=DEV).manual_seed(zlib.crc32(f'{dtype}/{B}/{R}/{F}'.encode()))
    x = (torch.randn(B, R, F, device=DEV, generator=gen) + 0.5).to(dtype)
    ref_sum = x.double().sum(1)                                        # fp64 of the same rounded inputs
    ls = torch.tensor([512.0], device=DEV)
    for ones, scale, with_ls in ((1, 1.0 / R, False), (0, 0.3, True), (1, 2.0, True), (0, 1.0, False)):
        d = F + ones
        ld = _ld4(d) if ones else d
        out = _reduce_linear(lib, x, ones, scale, ls if with_ls else None, ld)
        div = 512.0 if with_ls else 1.0
        want = ref_sum * scale / div
        if ones:
            want = torch.cat([want, want.new_full((B, 1), scale * R / div)], 1)
        assert rel_fro(out[:, :d], want) <= 1e-6, (ones, scale, with_ls, rel_fro(out[:, :d], want))
        assert not out[:, d:].any()
        assert torch.equal(out, _reduce_linear(lib, x, ones, scale, ls if with_ls else None, ld))
    if B * R * F <= 1 << 22:
        # the per-example sum of the expand rows of kfac_rows_linear
        ld = _ld4(F + 1)
        rows = torch.empty(B * R, ld, device=DEV)
        assert lib.kfac_rows_linear(x.data_ptr(), _code(dtype), B * R, F, 1, 1.0, ls.data_ptr(), rows.data_ptr(), ld,
                                    S()) == 0
        out = _reduce_linear(lib, x, 1, 1.0, ls, ld)
        assert rel_fro(out, rows.double().view(B, R, ld).sum(1)) <= 1e-6


CONV_GEOS = [
    # (B, C, H, W, kh, kw, sh, sw, ph, pw, bias): the geometries of test_rows_conv_against_unfold, then more
    (2, 3, 7, 7, 3, 3, 1, 1, 1, 1, True),
    (3, 5, 7, 7, 1, 1, 1, 1, 0, 0, False),
    (2, 4, 9, 8, 3, 3, 2, 2, 1, 1, False),
    (2, 6, 8, 8, 1, 1, 2, 2, 0, 0, True),
    (1, 3, 11, 13, 7, 7, 2, 2, 3, 3, False),
    (2, 64, 6, 6, 3, 3, 1, 1, 1, 1, True),
    (4, 3, 224, 224, 7, 7, 2, 2, 3, 3, False),    # the ResNet stem
    (3, 16, 56, 56, 1, 1, 2, 2, 0, 0, True),      # 1x1 / s2 downsample
    (5, 33, 7, 7, 3, 3, 1, 1, 1, 1, True),        # 3x3 on a 7x7 map
    (2, 4, 12, 10, 2, 5, 3, 1, 1, 2, True),       # non-square kernel, strides and padding
    (3, 7, 1, 1, 3, 3, 1, 1, 1, 1, True),         # H = W = 1
    (2, 2, 1, 1, 5, 5, 4, 4, 2, 2, False),        # a window wider than the map
]


def _reduce_conv_input(lib, x, geo, scale, ld):
    B, C, H, W, kh, kw, sh, sw, ph, pw, bias = geo
    out = torch.full((B, ld), float('nan'), device=DEV)
    rc = lib.kfac_reduce_rows_conv2d_input(x.data_ptr(), _code(x.dtype), B, C, H, W, kh, kw, sh, sw, ph, pw, int(bias),
                                           scale, out.data_ptr(), ld, S())
    assert rc == 0, lib.kfac_last_error()
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('geo', CONV_GEOS, ids=lambda g: 'x'.join(map(str, g[:4])) + f'-k{g[4]}{g[5]}s{g[6]}{g[7]}p{g[8]}{g[9]}')
def test_reduce_rows_conv_input(lib, geo, dtype):
    B, C, H, W, kh, kw, sh, sw, ph, pw, bias = geo
    gen = torch.Generator(device=DEV).manual_seed(zlib.crc32(repr(geo).encode()))
    x = (torch.randn(B, C, H, W, device=DEV, generator=gen) + 0.3).to(dtype)
    Ho, Wo = (H + 2 * ph - kh) // sh + 1, (W + 2 * pw - kw) // sw + 1
    Sp = Ho * Wo
    d = C * kh * kw + int(bias)
    # the per-example mean of F.unfold, scaled like the expand rows (1/S): the A row of K-FAC-reduce
    u = torch.nn.functional.unfold(x.double(), (kh, kw), padding=(ph, pw), stride=(sh, sw))     # B, C*kh*kw, S
    want = u.sum(2) / (Sp * Sp)
    if bias:
        want = torch.cat([want, want.new_full((B, 1), 1.0 / Sp)], 1)
    out = _reduce_conv_input(lib, x, geo, 1.0 / (Sp * Sp), _ld4(d))
    assert rel_fro(out[:, :d], want) <= 1e-6, rel_fro(out[:, :d], want)
    assert not out[:, d:].any()
    assert torch.equal(out, _reduce_conv_input(lib, x, geo, 1.0 / (Sp * Sp), _ld4(d)))
    # the per-example sum of kfac_rows_conv2d_input's rows
    if B * Sp * _ld4(d) <= 1 << 24:
        rows = torch.empty(B * Sp, _ld4(d), device=DEV)
        assert lib.kfac_rows_conv2d_input(x.data_ptr(), _code(dtype), B, C, H, W, kh, kw, sh, sw, ph, pw, int(bias),
                                          0.5, rows.data_ptr(), _ld4(d), S()) == 0
        out = _reduce_conv_input(lib, x, geo, 0.5, d)
        assert rel_fro(out, rows.double().view(B, Sp, -1).sum(1)[:, :d]) <= 1e-6


@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('hw', [(1, 1), (7, 7), (56, 56), (112, 112)])
def test_reduce_rows_conv_gradout(lib, hw, dtype):
    Ho, Wo = hw
    B, C = 6, 67
    gen = torch.Generator(device=DEV).manual_seed(zlib.crc32(f'{hw}/{dtype}'.encode()))
    g = torch.randn(B, C, Ho, Wo, device=DEV, generator=gen).to(dtype)
    ls = torch.tensor([64.0], device=DEV)
    Sp = Ho * Wo

    def run(scale, with_ls, ld):
        out = torch.full((B, ld), float('nan'), device=DEV)
        rc = lib.kfac_reduce_rows_conv2d_gradout(g.data_ptr(), _code(dtype), B, C, Ho, Wo, scale,
                                                 ls.data_ptr() if with_ls else None, out.data_ptr(), ld, S())
        assert rc == 0, lib.kfac_last_error()
        torch.cuda.synchronize()
        return out
    scale = Sp ** -1.5
    for with_ls in (False, True):
        out = run(scale, with_ls, _ld4(C))
        want = g.double().sum((2, 3)) * scale / (64.0 if with_ls else 1.0)
        assert rel_fro(out[:, :C], want) <= 1e-6
        assert not out[:, C:].any()
        assert torch.equal(out, run(scale, with_ls, _ld4(C)))
    rows = torch.empty(B * Sp, _ld4(C), device=DEV)
    assert lib.kfac_rows_conv2d_gradout(g.data_ptr(), _code(dtype), B, C, Ho, Wo, 0.25, ls.data_ptr(),
                                        rows.data_ptr(), _ld4(C), S()) == 0
    assert rel_fro(run(0.25, True, _ld4(C)), rows.double().view(B, Sp, -1).sum(1)) <= 1e-6


def test_reduce_rows_reject_bad_arguments(lib):
    x = torch.zeros(2, 3, 4, device=DEV)
    out = torch.zeros(64, device=DEV)
    assert lib.kfac_reduce_rows_linear(x.data_ptr(), 0, 2, 3, 4, 1, 1.0, None, out.data_ptr(), 4, S()) != 0   # ld < d
    assert lib.kfac_reduce_rows_linear(x.data_ptr(), 7, 2, 3, 4, 0, 1.0, None, out.data_ptr(), 4, S()) != 0   # dtype
    assert lib.kfac_reduce_rows_conv2d_input(x.data_ptr(), 0, 1, 1, 2, 2, 5, 5, 1, 1, 0, 0, 0, 1.0, out.data_ptr(), 25,
                                             S()) != 0                                                         # no output
    assert lib.kfac_reduce_rows_conv2d_gradout(x.data_ptr(), 0, 2, 3, 2, 2, 1.0, None, out.data_ptr(), 2, S()) != 0


# ---------------------------------------------------------------------------------------------- R = 1
@pytest.mark.parametrize('method', ['eigen', 'inverse', 'ekfac'])
def test_r1_is_bitwise_expand(method):
    from kfac_b200.preconditioner import KFACPreconditioner
    from oracle.models import TinyModel
    torch.manual_seed(0)
    base = TinyModel().to(DEV)
    runs = []
    for approx in ('expand', 'reduce'):
        m = TinyModel().to(DEV)
        m.load_state_dict(base.state_dict())
        pre = KFACPreconditioner(m, compute_method=method, kfac_approx=approx, damping=0.003,
                                 factor_update_steps=1, inv_update_steps=2)
        opt = torch.optim.SGD(m.parameters(), lr=0.05)
        gen = torch.Generator().manual_seed(1)
        snap = []
        for s in range(4):
            x, y = torch.rand(8, 10, generator=gen).to(DEV), torch.rand(8, 10, generator=gen).to(DEV)
            opt.zero_grad()
            torch.nn.functional.mse_loss(m(x), y, reduction='sum').backward()
            pre.step()
            torch.cuda.synchronize()
            snap.append({n: [l.a_factor.clone(), l.g_factor.clone(), l._p_view.clone()]
                         + [t.clone() for t in (l.qa, l.qg, l.dgda, l.a_inv, l.g_inv) if t is not None]
                         + [p.grad.clone() for p in l.module.module.parameters()]
                         + ([l._S.clone()] if l._S is not None else [])
                         for n, l in pre._layers.values()})
            opt.step()
        runs.append(snap)
    for s, (a, b) in enumerate(zip(*runs)):
        for n in a:
            assert len(a[n]) == len(b[n])
            for i, (u, v) in enumerate(zip(a[n], b[n])):
                assert torch.equal(u, v), (s, n, i)


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


def _reduced_rows(module, x, g, grad_scale=1.0):
    """fp64 K-FAC-reduce rows (x_b, g_b) of one call, restated from the expand rows' definition."""
    x, g = x.double(), g.double() / grad_scale
    if isinstance(module, nn.Conv2d):
        Sp = g.shape[2] * g.shape[3]
        u = torch.nn.functional.unfold(x, module.kernel_size, padding=module.padding, stride=module.stride) / Sp
        if module.bias is not None:
            u = torch.cat([u, u.new_full((u.shape[0], 1, u.shape[2]), 1.0 / Sp)], 1)
        X = u.mean(2)
        G = (g / Sp).flatten(2).sum(2) / math.sqrt(Sp)
        return X, G
    B = x.shape[0] if x.dim() > 1 else 1
    xr, gr = x.reshape(B, -1, x.shape[-1]), g.reshape(B, -1, g.shape[-1])
    if module.bias is not None:
        xr = torch.cat([xr, xr.new_ones(*xr.shape[:2], 1)], 2)
    R = xr.shape[1]
    if R == 1:
        return xr[:, 0], gr[:, 0]
    return xr.mean(1), gr.sum(1) / math.sqrt(R)


def _grad_matrix(module):
    g = module.weight.grad.reshape(module.weight.grad.size(0), -1)
    if module.bias is not None:
        g = torch.cat([g, module.bias.grad.view(-1, 1)], 1)
    return g.detach().double()


class _Fp64:
    """fp64 factors (EMA from I, windows of `acc` calls in hook order), second-order data and EKFAC S."""

    def __init__(self, acc=1, diag_g=()):
        self.A, self.G, self.snap, self.S = {}, {}, {}, {}
        self.acc = acc
        self.diag_g = set(diag_g)

    def _ema(self, store, name, stats, alpha):
        for w in range(0, len(stats), self.acc):
            win = sum(stats[w:w + self.acc]) / len(stats[w:w + self.acc])
            prev = store.get(name)
            if prev is None:
                prev = torch.ones_like(win) if win.dim() == 1 else torch.eye(win.shape[0], dtype=win.dtype,
                                                                               device=win.device)
            store[name] = alpha * prev + (1 - alpha) * win

    def factors(self, pre, calls, alpha):
        """calls[m]: per micro-batch, the (input, output gradient) pairs of its calls in forward order.  The A hooks
        run in forward order, the G hooks of a micro-batch in reverse."""
        for m, (name, _) in pre._layers.items():
            A, Gs = [], []
            for mb in calls[m]:
                for x, g in mb:
                    X, _ = _reduced_rows(m, x, g)
                    A.append(X.T @ X / X.shape[0])
                for x, g in reversed(mb):
                    _, G = _reduced_rows(m, x, g)
                    Gs.append((G * G).sum(0) / G.shape[0] if name in self.diag_g else G.T @ G / G.shape[0])
            self._ema(self.A, name, A, alpha)
            self._ema(self.G, name, Gs, alpha)

    def invert(self, pre, damping):
        for _, (name, _) in pre._layers.items():
            A, G = self.A[name], self.G[name]
            da, qa = torch.linalg.eigh(A)
            if G.dim() == 1:
                dg, qg = G, None
            else:
                dg, qg = torch.linalg.eigh(G)
            self.snap[name] = dict(A=A, G=G, da=da.clamp(min=0), qa=qa, dg=dg.clamp(min=0), qg=qg, damping=damping)

    def precondition(self, name, grad, method):
        s = self.snap[name]
        lam = s['damping']
        if method == 'inverse':
            eye = lambda n: torch.eye(n, dtype=grad.dtype, device=grad.device)  # noqa: E731
            ginv = torch.diag(1 / (s['G'] + lam)) if s['G'].dim() == 1 else torch.linalg.inv(s['G'] + lam * eye(grad.shape[0]))
            return ginv @ grad @ torch.linalg.inv(s['A'] + lam * eye(grad.shape[1]))
        qa, qg = s['qa'], s['qg']
        v = grad @ qa if qg is None else qg.T @ grad @ qa
        v = v / (torch.outer(s['dg'], s['da']) + lam if method == 'eigen' else self.S[name] + lam)
        return (v if qg is None else qg @ v) @ qa.T


def _run(model, batches, loss_fn, method, steps, fus=1, ius=1, acc=1, damping=0.003, alpha=0.9, kw=None,
         calls_per_step=1):
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    kw = kw or {}
    pre = KFACPreconditioner(model, compute_method=method, kfac_approx='reduce', factor_update_steps=fus,
                             inv_update_steps=ius, damping=damping, factor_decay=alpha, kl_clip=None,
                             accumulation_steps=acc, **kw)
    rec = _Rec(pre._layers)
    ref = _Fp64(acc, diag_g=kw.get('diagonal_g_layers') or ())
    opt = torch.optim.SGD(model.parameters(), lr=0.01)
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
        f, i = (fus(s) if callable(fus) else fus), (ius(s) if callable(ius) else ius)
        if s % f == 0:
            ref.factors(pre, calls, alpha)
        if s % i == 0:
            ref.invert(pre, damping)
        for m, (name, layer) in pre._layers.items():
            assert rel_fro(layer.a_factor, ref.A[name]) <= 1e-5, (s, name, 'A', rel_fro(layer.a_factor, ref.A[name]))
            assert rel_fro(layer.g_factor, ref.G[name]) <= 1e-5, (s, name, 'G', rel_fro(layer.g_factor, ref.G[name]))
            if method == 'ekfac':
                Qa, Qg = layer.qa.double(), layer.qg.double()
                if s % f == 0:
                    X, G = _reduced_rows(m, *calls[m][0][0])
                    Sb = ((G @ Qg) ** 2).T @ ((X @ Qa) ** 2) / X.shape[0]
                    ref.S[name] = Sb if s % i == 0 else alpha * ref.S[name] + (1 - alpha) * Sb
                elif s % i == 0:
                    ref.S[name] = torch.outer(layer.dg.double(), layer.da.double())
                assert rel_fro(layer._S[:, :layer.a_dim], ref.S[name]) < 1e-4, (s, name, 'S')
                want = Qg @ ((Qg.T @ grads[name] @ Qa) / (ref.S[name] + damping)) @ Qa.T
            else:
                want = ref.precondition(name, grads[name], method)
            e = rel_fro(_grad_matrix(m), want)
            assert e < 1e-3, (s, name, 'P', e)
        opt.step()
    return pre


class _Seq(nn.Module):
    def __init__(self):
        super().__init__()
        self.l1 = nn.Linear(24, 130)
        self.l2 = nn.Linear(130, 70, bias=False)
        self.l3 = nn.Linear(70, 5)

    def forward(self, x):
        return self.l3(torch.tanh(self.l2(torch.tanh(self.l1(x))))).mean(1)


def _seq_batches(n, seed=3):
    gen = torch.Generator().manual_seed(seed)
    data = [(torch.randn(6, 40, 24, generator=gen).to(DEV), torch.randint(0, 5, (6,), generator=gen).to(DEV))
            for _ in range(n)]
    return lambda s: data[s]


def _img_batches(n, seed=4):
    gen = torch.Generator().manual_seed(seed)
    data = [(torch.randn(8, 3, 32, 32, generator=gen).to(DEV), torch.randint(0, 10, (8,), generator=gen).to(DEV))
            for _ in range(n)]
    return lambda s: data[s]


@pytest.mark.parametrize('method', ['eigen', 'inverse', 'ekfac'])
def test_sequence_linear_stack(method):
    torch.manual_seed(3)
    _run(_Seq().to(DEV), _seq_batches(4), nn.CrossEntropyLoss(), method, steps=4, ius=2 if method != 'ekfac' else 1)


@pytest.mark.parametrize('method', ['eigen', 'inverse', 'ekfac'])
def test_resnet32(method):
    from oracle.models import resnet32
    torch.manual_seed(4)
    _run(resnet32().to(DEV), _img_batches(2), nn.CrossEntropyLoss(), method, steps=2)


@pytest.mark.parametrize('method', ['eigen', 'inverse', 'ekfac'])
def test_schedules(method):
    """factor_update_steps=2, inv_update_steps=4 over 6 steps, then callables (factor 2, inverse 3)."""
    torch.manual_seed(5)
    _run(_Seq().to(DEV), _seq_batches(6, 5), nn.CrossEntropyLoss(), method, steps=6, fus=2, ius=4)
    torch.manual_seed(5)
    _run(_Seq().to(DEV), _seq_batches(7, 6), nn.CrossEntropyLoss(), method, steps=7, fus=lambda s: 2,
         ius=lambda s: 3 if method != 'ekfac' else 2)


@pytest.mark.parametrize('method', ['eigen', 'inverse'])
def test_accumulation_steps(method):
    from oracle.models import resnet32
    torch.manual_seed(6)
    _run(_Seq().to(DEV), _seq_batches(6, 7), nn.CrossEntropyLoss(), method, steps=3, acc=2)
    torch.manual_seed(6)
    _run(resnet32().to(DEV), _img_batches(4, 8), nn.CrossEntropyLoss(), method, steps=2, acc=2)


def test_module_called_twice():
    class Twice(nn.Module):
        def __init__(self):
            super().__init__()
            self.inp = nn.Linear(24, 32)
            self.shared = nn.Linear(32, 32)
            self.out = nn.Linear(32, 5)

        def forward(self, x):
            h = torch.tanh(self.inp(x))
            h = torch.tanh(self.shared(h))
            h = torch.tanh(self.shared(h[:, :20]))       # a second call with another R
            return self.out(h).mean(1)
    torch.manual_seed(7)
    _run(Twice().to(DEV), _seq_batches(3, 9), nn.CrossEntropyLoss(), 'eigen', steps=3)


# ---------------------------------------------------------------------------------------------- other layers
class _GPT(nn.Module):
    def __init__(self, V=300, D=64):
        super().__init__()
        from workloads import NeoXBlock
        self.emb = nn.Embedding(V, D)
        self.ln = nn.LayerNorm(D)
        self.block = NeoXBlock(D)
        self.rms = nn.RMSNorm(D)
        self.head = nn.Linear(D, V, bias=False)

    def forward(self, idx):
        return self.head(self.rms(self.block(self.ln(self.emb(idx)))))


def test_other_layers_untouched_and_diag_head():
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(8)
    base = _GPT().to(DEV)
    gen = torch.Generator().manual_seed(8)
    data = [(torch.randint(0, 300, (4, 16), generator=gen).to(DEV), torch.randint(0, 300, (4, 16), generator=gen).to(DEV))
            for _ in range(3)]
    kw = dict(precondition_embeddings=True, precondition_norms=True, diagonal_g_layers=['head'], kl_clip=None,
              damping=0.003, factor_decay=0.9)
    out = {}
    for approx in ('expand', 'reduce'):
        m = _GPT().to(DEV)
        m.load_state_dict(base.state_dict())
        pre = KFACPreconditioner(m, kfac_approx=approx, **kw)
        rec = _Rec([mod for mod, (n, _) in pre._layers.items() if n == 'head'])
        heads = []
        snaps = []
        for s in range(3):
            rec.clear()
            m.zero_grad()
            idx, y = data[s]
            nn.functional.cross_entropy(m(idx).flatten(0, 1), y.flatten()).backward()
            pre.step()
            torch.cuda.synchronize()
            snaps.append({n: [t.clone() for t in (l.a_factor, l.g_factor, l._p_view) if t is not None]
                          for n, l in list(pre._layers.values()) + list(pre._norm_layers.values())
                          if l.diag_a or l.norm})
            head = next(mod for mod, (n, _) in pre._layers.items() if n == 'head')
            _, G = _reduced_rows(head, rec.inp[head][0], rec.gout[head][0])
            heads.append(((G * G).sum(0) / G.shape[0], pre._layers[head][1].g_factor.clone()))
        out[approx] = (snaps, heads)
    for a, b in zip(out['expand'][0], out['reduce'][0]):
        assert list(a) == list(b) == ['emb', 'ln', 'rms']
        for n in a:
            for u, v in zip(a[n], b[n]):
                assert torch.equal(u, v), n
    # the reduce head's diag(G): EMA from ones of the fp64 reduced rows
    want = None
    for Gb, got in out['reduce'][1]:
        want = 0.9 * (torch.ones_like(Gb) if want is None else want) + 0.1 * Gb
        assert rel_fro(got, want) <= 1e-5


# ---------------------------------------------------------------------------------------------- AMP
class _ConvNet(nn.Module):
    def __init__(self):
        super().__init__()
        self.conv1 = nn.Conv2d(3, 32, 3, padding=1)
        self.conv2 = nn.Conv2d(32, 64, 3, stride=2, padding=1, bias=False)
        self.fc1 = nn.Linear(64, 80)
        self.fc2 = nn.Linear(80, 10)

    def forward(self, x):
        x = torch.relu(self.conv2(torch.relu(self.conv1(x))))
        return self.fc2(torch.relu(self.fc1(x.mean((2, 3)))))


@pytest.mark.parametrize('method', ['eigen', 'ekfac'])
def test_amp_grad_scaler(method):
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(0)
    base = _ConvNet().to(DEV)
    gen = torch.Generator().manual_seed(0)
    data = [(torch.randn(16, 3, 16, 16, generator=gen).to(DEV), torch.randint(0, 10, (16,), generator=gen).to(DEV))
            for _ in range(4)]
    runs = {}
    for amp in (False, True):
        m = _ConvNet().to(DEV)
        m.load_state_dict(base.state_dict())
        scaler = torch.amp.GradScaler('cuda', init_scale=2.0 ** 10, growth_interval=10 ** 9, enabled=amp)
        pre = KFACPreconditioner(m, kfac_approx='reduce', compute_method=method, damping=0.003,
                                 grad_scaler=scaler if amp else None)
        opt = torch.optim.SGD(m.parameters(), lr=0.0)
        facs = []
        for s in range(4):
            m.zero_grad()
            if amp and s == 2:
                scaler.update(new_scale=2.0 ** 60)       # the scaled loss overflows fp16: every G window is dropped
                before = {n: l.g_factor.clone() for n, l in pre._layers.values()}
            with torch.autocast('cuda', dtype=torch.float16, enabled=amp):
                loss = nn.functional.cross_entropy(m(data[s][0]), data[s][1])
            scaler.scale(loss).backward()
            scaler.unscale_(opt)
            pre.step()
            torch.cuda.synchronize()
            if amp and s == 2:
                assert pre.skipped_factor_updates >= len(pre._layers)
                for n, l in pre._layers.values():
                    assert torch.equal(l.g_factor, before[n]), n
                    assert torch.isfinite(l.a_factor).all()
            if amp:
                scaler.update(new_scale=2.0 ** 10)
            facs.append({n: (l.a_factor.clone(), l.g_factor.clone()) for n, l in pre._layers.values()})
        runs[amp] = facs
    # before the overflow the fp16 factors follow the fp32 ones within the AMP tolerance
    for s in (0, 1):
        for n in runs[False][s]:
            for u, v in zip(runs[True][s][n], runs[False][s][n]):
                assert rel_fro(u, v) <= 2e-2, (s, n, rel_fro(u, v))


# ---------------------------------------------------------------------------------------------- memory, training
def test_ekfac_row_buffers():
    from kfac_b200.preconditioner import KFACPreconditioner
    use = {}
    for approx in ('expand', 'reduce'):
        torch.manual_seed(0)
        m = _Seq().to(DEV)
        pre = KFACPreconditioner(m, compute_method='ekfac', kfac_approx=approx)
        x = torch.randn(6, 40, 24, device=DEV)
        nn.functional.cross_entropy(m(x), torch.zeros(6, dtype=torch.long, device=DEV)).backward()
        pre.step()
        use[approx] = {n: (l._rows_x.numel(), l._rows_g.numel(), l.memory_usage()['ekfac'])
                       for n, l in pre._layers.values()}
        if approx == 'reduce':
            for n, l in pre._layers.values():
                assert l._rows_x.numel() == 6 * _ld4(l.a_dim) and l._rows_g.numel() == 6 * _ld4(l.g_dim), n
                s_bytes = 2 * l._S.numel() * 4
                assert l.memory_usage()['ekfac'] == s_bytes + 4 * 6 * (_ld4(l.a_dim) + _ld4(l.g_dim))
            total = sum(v[2] for v in use[approx].values())
            assert pre.memory_usage()['ekfac'] == total + pre._ekfac_scratch.buf.numel()
    for n in use['expand']:
        assert use['expand'][n][0] == 40 * use['reduce'][n][0] and use['expand'][n][1] == 40 * use['reduce'][n][1]


def test_training_loss_decreases():
    from kfac_b200.preconditioner import KFACPreconditioner
    for method in ('eigen', 'ekfac'):
        torch.manual_seed(42)
        m = _Seq().to(DEV)
        opt = torch.optim.SGD(m.parameters(), lr=0.05)
        pre = KFACPreconditioner(m, lr=0.05, compute_method=method, kfac_approx='reduce')
        x, y = torch.randn(16, 20, 24, device=DEV), torch.randint(0, 5, (16,), device=DEV)
        losses = []
        for _ in range(30):
            opt.zero_grad()
            loss = nn.functional.cross_entropy(m(x), y)
            loss.backward()
            pre.step()
            opt.step()
            losses.append(loss.item())
        assert losses[-1] < 0.8 * losses[0], (method, losses[0], losses[-1])


# ---------------------------------------------------------------------------------------------- two ranks
def _run_dist(backend):
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    script = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'dist_reduce.py')
    out = subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node=2',
                          '--master-addr', '127.0.0.1', '--master-port', str(port), script, '--backend', backend],
                         capture_output=True, text=True, timeout=900)
    print(out.stdout[-3000:])
    assert out.returncode == 0, out.stderr[-4000:]
    assert out.stdout.count('dist_reduce ok') == 2, out.stdout[-2000:]


def test_two_ranks_gloo():
    _run_dist('gloo')


def test_two_ranks_nccl():
    if torch.cuda.device_count() < 2:
        pytest.skip('needs >= 2 GPUs')
    _run_dist('nccl')
