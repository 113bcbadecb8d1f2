"""Diagonal-G Linear layers (`diagonal_g_layers=[...]`) on the GPU, everything against fp64:

  * kfac_factor_linear_diag against scale * sum_r x[r, j]^2 for fp32/fp16/bf16 inputs, rows from 1 to 10^5,
    V in {10, 1001, 50257}, accumulated into a live batch vector; the same bits on a repeat, the diagonal of
    kfac_factor_linear on the same input, a too-small workspace rejected;
  * kfac_factor_ema_diag_guarded bit-equal to kfac_factor_ema_diag on batch * u, and its drop rules;
  * kfac_precondition with diagonal-G items (V in {10007, 50257}, a in {49, 769, 2049}, with and without bias, fp32/
    fp16/bf16 gradients) mixed with dense and embedding items, eigen and inverse: P against fp64, the same bits on a
    repeat, and the other items' P bit-identical with and without the diagonal-G items;
  * an LM (Embedding -> NeoX block -> Linear(d, V) head, V = 10007 > KFAC_EIGH_MAX_N) with the head diagonal, with
    and without precondition_embeddings, under integer and callable schedules: every layer's gradient against an
    fp64 restatement, and the first step's other gradients bit-identical to a run with the head skipped;
  * the kl-clip scale, a state_dict round trip, an fp16 overflow under a GradScaler, a non-finite head G without a
    grad_scaler, hooks without host syncs, and two ranks (tests/dist_diag_g.py).
"""
import copy
import os
import subprocess
import sys

import pytest
import torch
from torch import nn

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
def _linear_diag(lib, x, live, scale, need=None):
    from kfac_b200 import _cabi
    rows, V = x.shape
    if need is None:
        need = lib.kfac_factor_linear_diag_workspace_bytes(rows, V)
    acc = live.clone()
    ws = torch.full((max(need, 1),), 255, dtype=torch.uint8, device=DEV)
    rc = lib.kfac_factor_linear_diag(x.data_ptr(), _cabi.DTYPE_CODE[x.dtype], rows, V, scale, acc.data_ptr(),
                                     ws.data_ptr(), need, S())
    torch.cuda.synchronize()
    return rc, acc


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16, torch.bfloat16])
@pytest.mark.parametrize('rows,V,offset', [(1, 10, 0), (100003, 10, 1), (37, 1001, 3), (100003, 1001, 0),
                                           (1, 50257, 0), (333, 50257, 1), (4096, 50257, 2)])
def test_factor_linear_diag(lib, dtype, rows, V, offset):
    """offset: the matrix starts that many elements into its allocation, so no row is 16-byte aligned."""
    gen = torch.Generator(device=DEV).manual_seed(rows + V)
    buf = (torch.randn(rows * V + offset, device=DEV, generator=gen) * 3).to(dtype)
    x = buf[offset:].view(rows, V)
    x[0, :3] = 0
    live = torch.rand(V, device=DEV, generator=gen)           # a batch vector that already holds a window
    scale = 1.0 / rows
    rc, acc = _linear_diag(lib, x, live, scale)
    assert rc == 0, lib.kfac_last_error()
    ref = live.double() + scale * (x.double() ** 2).sum(0)
    assert float(((acc.double() - ref).abs() / ref.abs()).max()) <= 1e-6
    _, again = _linear_diag(lib, x, live, scale)
    assert torch.equal(bits(acc), bits(again))
    need = lib.kfac_factor_linear_diag_workspace_bytes(rows, V)
    rc, _ = _linear_diag(lib, x, live, scale, need=need - 4)
    assert rc != 0


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
@pytest.mark.parametrize('V', [10, 1001])
def test_factor_linear_diag_is_the_diagonal_of_the_dense_factor(lib, dtype, V):
    from kfac_b200 import _cabi
    rows = 4096
    gen = torch.Generator(device=DEV).manual_seed(V)
    x = torch.randn(rows, V, device=DEV, generator=gen).to(dtype)
    _, diag = _linear_diag(lib, x, torch.zeros(V, device=DEV), 1.0 / rows)
    dense = torch.zeros(V, V, device=DEV)
    need = lib.kfac_factor_linear_workspace_bytes(rows, V, 0)
    ws = torch.empty(max(need, 1), dtype=torch.uint8, device=DEV)
    assert lib.kfac_factor_linear(x.data_ptr(), _cabi.DTYPE_CODE[dtype], rows, V, 0, 1.0 / rows, dense.data_ptr(),
                                  ws.data_ptr(), need, S()) == 0
    torch.cuda.synchronize()
    ref = (x.double() ** 2).sum(0) / rows
    # the two agree to 1e-6 beyond the dense factor's own error (its tensor-core path rounds to 3xTF32)
    dense_err, diag_err = rel_fro(torch.diagonal(dense), ref), rel_fro(diag, ref)
    assert diag_err <= 1e-6
    assert rel_fro(diag, torch.diagonal(dense)) <= 1e-6 + dense_err, (diag_err, dense_err)


def _ema_diag(lib, fac0, bat0, firsts, inv_counts, alpha, scales=None, guarded=False):
    import ctypes as C

    from kfac_b200 import _cabi
    fac = [f.clone() for f in fac0]
    bat = [b.clone() for b in bat0]
    n = len(fac)
    items = (_cabi.EmaItem * n)()
    for i in range(n):
        items[i] = _cabi.EmaItem(fac[i].data_ptr(), bat[i].data_ptr(), fac[i].numel(), firsts[i], inv_counts[i])
    skipped = torch.zeros(1, dtype=torch.int64, device=DEV)
    if guarded:
        ptrs = (C.c_void_p * n)(*[s.data_ptr() if s is not None else None for s in scales]) if scales else None
        need = lib.kfac_factor_ema_diag_guarded_workspace_bytes(n)
        ws = torch.full((need,), 255, dtype=torch.uint8, device=DEV)
        rc = lib.kfac_factor_ema_diag_guarded(items, n, alpha, ptrs, skipped.data_ptr(), ws.data_ptr(), need, S())
        assert lib.kfac_factor_ema_diag_guarded(items, n, alpha, ptrs, skipped.data_ptr(), ws.data_ptr(), need - 4,
                                                S()) != 0
    else:
        rc = lib.kfac_factor_ema_diag(items, n, alpha, S())
    assert rc == 0, lib.kfac_last_error()
    torch.cuda.synchronize()
    return fac, bat, int(skipped.item())


def test_ema_diag_guarded(lib):
    gen = torch.Generator(device=DEV).manual_seed(7)
    alpha = float(torch.tensor(0.95, dtype=torch.float32))
    dims = [3, 1000, 10007, 50257] + [17 * k + 1 for k in range(40)]       # 44 items: two launches of up to 40
    firsts = [i % 3 == 0 for i in range(len(dims))]
    inv_counts = [1.0 / (1 + i % 4) for i in range(len(dims))]
    fac0 = [torch.rand(d, device=DEV, generator=gen) for d in dims]
    bat0 = [torch.rand(d, device=DEV, generator=gen) * 1e4 for d in dims]
    # NULL scales: the bits of the unguarded EMA
    ref, _, _ = _ema_diag(lib, fac0, bat0, firsts, inv_counts, alpha)
    got, bat, skipped = _ema_diag(lib, fac0, bat0, firsts, inv_counts, alpha, guarded=True)
    assert skipped == 0 and all(torch.equal(bits(a), bits(b)) for a, b in zip(got, ref))
    assert not any(bool(b.any()) for b in bat)
    # power-of-two scales (a GradScaler's): the bits of the unguarded EMA on batch * (1/s)^2
    svals = [2.0 ** (3 * (i % 5)) for i in range(len(dims))]
    scales = [torch.tensor([s], device=DEV) for s in svals]
    scales[1] = None
    u = [(1.0 / s) ** 2 if sc is not None else 1.0 for s, sc in zip(svals, scales)]
    ref, _, _ = _ema_diag(lib, fac0, [b * torch.tensor(ui, device=DEV) for b, ui in zip(bat0, u)], firsts, inv_counts,
                          alpha)
    got, _, skipped = _ema_diag(lib, fac0, bat0, firsts, inv_counts, alpha, scales=scales, guarded=True)
    assert skipped == 0 and all(torch.equal(bits(a), bits(b)) for a, b in zip(got, ref))
    # dropped windows: inf, NaN, 2e15, and a scale too small for the window (1e10 * 2^40 > 1e15); the first of them
    # is a first window and becomes ones
    bad = [b.clone() for b in bat0]
    bad[0][1] = float('inf')
    bad[2][500] = float('nan')
    bad[3][50256] = 2e15
    bad[4][0] = 1e10
    drop = {0, 2, 3, 4}
    scales = [None] * len(dims)
    scales[4] = torch.tensor([2.0 ** -20], device=DEV)
    good_ref, _, _ = _ema_diag(lib, fac0, bat0, firsts, inv_counts, alpha)
    got, bat, skipped = _ema_diag(lib, fac0, bad, firsts, inv_counts, alpha, scales=scales, guarded=True)
    assert skipped == len(drop)
    assert firsts[0] and torch.equal(got[0], torch.ones_like(got[0]))
    for i in range(len(dims)):
        assert not bool(bat[i].any()), i
        if i in drop and i != 0:
            assert torch.equal(got[i], torch.ones_like(got[i]) if firsts[i] else fac0[i]), i
        elif i not in drop:
            assert torch.equal(bits(got[i]), bits(good_ref[i])), i


# ---------------------------------------------------------------------------------------------- precondition
def _stored(x):
    from kfac_b200 import _cabi
    out = torch.full((x.shape[0], _cabi.ld4(x.shape[1])), float('nan'), device=DEV)
    out[:, :x.shape[1]] = x
    return out


def test_precondition_diag_g_items(lib):
    from kfac_b200 import _cabi
    damping = float(torch.tensor(0.003, dtype=torch.float32))
    gen = torch.Generator(device=DEV).manual_seed(13)

    def basis(n):
        q, _ = torch.linalg.qr(torch.randn(n, n, dtype=torch.float64, device=DEV, generator=gen))
        return q.float(), (torch.rand(n, dtype=torch.float64, device=DEV, generator=gen) ** 4).float()

    def inv(q, d):
        return ((q.double() / (d.double() + damping)) @ q.double().t()).float()

    # dense (g, a, bias, dtype): Linear-, Conv- and SIMT-sized; embedding (V, d, dtype); diagonal G (V, a, bias, dtype)
    dense = [(256, 129, 1, torch.float32), (64, 577, 1, torch.float16), (10, 21, 1, torch.bfloat16)]
    embs = [(1000, 48, torch.float16), (50257, 768, torch.float32)]
    diags = [(10007, 49, 1, torch.float16), (50257, 769, 0, torch.float32), (10007, 2049, 1, torch.bfloat16),
             (50257, 49, 0, torch.bfloat16), (10007, 769, 1, torch.float32), (50257, 2049, 1, torch.float32)]
    D, E, G = [], [], []
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
    for V, a, bias, dtype in diags:
        qa, da = basis(a)
        dgv = torch.rand(V, device=DEV, generator=gen) ** 2 * 1e-2
        dgv[::7] = 0                                                     # outputs without curvature
        w = torch.randn(V, a - bias, device=DEV, generator=gen).to(dtype)
        b = torch.randn(V, device=DEV, generator=gen).to(dtype) if bias else None
        grad = torch.cat([w.double(), b.double()[:, None]], 1) if bias else w.double()
        qa64, a_inv = qa.double(), inv(qa, da)
        ref_e = ((grad @ qa64) / (dgv.double()[:, None] * da.double()[None, :] + damping)) @ qa64.t()
        ref_i = (grad / (dgv.double()[:, None] + damping)) @ a_inv.double()
        G.append(dict(V=V, a=a, dtype=dtype, w=w, b=b, dgv=dgv, qa=_stored(qa), qaT=_stored(qa.t()), da=da,
                      a_inv=_stored(a_inv), ref_e=ref_e.float(), ref_i=ref_i.float()))
        del grad, ref_e, ref_i

    def precondition(method, with_diag):
        e = method == _cabi.KFAC_EIGEN
        others = [('d', l) for l in D] + [('e', l) for l in E]
        if with_diag:           # interleaved: the order of the items must not matter
            layers, dg_ = [], [('g', l) for l in G]
            while others or dg_:
                for src in (dg_, others):
                    if src:
                        layers.append(src.pop(0))
        else:
            layers = others
        items = (_cabi.PrecondItem * len(layers))()
        Ps = []
        for i, (kind, l) in enumerate(layers):
            p = lambda k, use: l[k].data_ptr() if use else None  # noqa: E731,B023
            if kind == 'd':
                g, a = l['g'], l['a']
                P = torch.full((g, _cabi.ld4(a)), float('nan'), device=DEV)
                items[i] = _cabi.PrecondItem(l['w'].data_ptr(), l['b'].data_ptr(), _cabi.DTYPE_CODE[l['dtype']], g, a,
                                             p('qa', e), p('qaT', e), p('qg', e), p('qgT', e), None, p('da', e),
                                             p('dg', e), p('a_inv', not e), p('g_inv', not e), _cabi.ld4(a),
                                             _cabi.ld4(g), _cabi.ld4(a), P.data_ptr(), _cabi.ld4(a))
                Ps.append((kind, l, P[:, :a]))
            elif kind == 'e':
                V, d = l['V'], l['d']
                P = torch.full((V, _cabi.ld4(d)), float('nan'), device=DEV)
                items[i] = _cabi.PrecondItem(l['w'].data_ptr(), None, _cabi.DTYPE_CODE[l['dtype']], d, V,
                                             None, None, p('qg', e), p('qgT', e), None, l['av'].data_ptr(), p('dg', e),
                                             None, p('g_inv', not e), 0, _cabi.ld4(d), 0, P.data_ptr(), _cabi.ld4(d),
                                             None, 0, _cabi.KFAC_ITEM_EMBEDDING)
                Ps.append((kind, l, P[:, :d]))
            else:
                V, a = l['V'], l['a']
                P = torch.full((V, _cabi.ld4(a)), float('nan'), device=DEV)
                items[i] = _cabi.PrecondItem(l['w'].data_ptr(), l['b'].data_ptr() if l['b'] is not None else None,
                                             _cabi.DTYPE_CODE[l['dtype']], V, a, p('qa', e), p('qaT', e), None, None,
                                             None, p('da', e), l['dgv'].data_ptr(), p('a_inv', not e), None,
                                             _cabi.ld4(a), 0, 0, P.data_ptr(), _cabi.ld4(a), None, 0,
                                             _cabi.KFAC_ITEM_DIAG_G)
                Ps.append((kind, l, P[:, :a]))
        need = lib.kfac_precondition_workspace_bytes(items, len(layers))
        ws = torch.full((need,), 255, dtype=torch.uint8, device=DEV)
        rc = lib.kfac_precondition(items, len(layers), method, damping, ws.data_ptr(), need, S())
        assert rc == 0, lib.kfac_last_error()
        torch.cuda.synchronize()
        del ws
        return Ps

    for method, key in ((_cabi.KFAC_EIGEN, 'ref_e'), (_cabi.KFAC_INVERSE, 'ref_i')):
        P1 = precondition(method, True)
        for kind, l, P in P1:
            if kind == 'g':
                err = rel_fro(P, l[key])
                assert err < 1e-3, (method, l['V'], l['a'], l['dtype'], err)
        P2 = precondition(method, True)
        for (_, _, p1), (_, _, p2) in zip(P1, P2):
            assert torch.equal(bits(p1), bits(p2))
        del P2
        alone = {id(l): P for _, l, P in precondition(method, False)}
        for kind, l, P in P1:
            if kind != 'g':
                assert torch.equal(bits(P), bits(alone[id(l)])), (method, kind)
        del P1, alone


def test_precondition_rejects_incomplete_diag_g_item(lib):
    from kfac_b200 import _cabi
    w = torch.zeros(100, 8, device=DEV)
    b = torch.zeros(100, device=DEV)
    qa = torch.eye(12, device=DEV)
    P = torch.zeros(100, 12, device=DEV)
    need_items = []
    # eigen without dg, eigen without qaT, inverse without a_inv
    for method, item in ((_cabi.KFAC_EIGEN, (qa, qa, None, qa.diagonal().contiguous())),
                         (_cabi.KFAC_EIGEN, (qa, None, b, qa.diagonal().contiguous())),
                         (_cabi.KFAC_INVERSE, (None, None, b, None))):
        q, qT, dg, da = item
        items = (_cabi.PrecondItem * 1)()
        items[0] = _cabi.PrecondItem(w.data_ptr(), b.data_ptr(), 0, 100, 9,
                                     q.data_ptr() if q is not None else None, qT.data_ptr() if qT is not None else None,
                                     None, None, None, da.data_ptr() if da is not None else None,
                                     dg.data_ptr() if dg is not None else None, None, None, 12, 0, 0, P.data_ptr(), 12,
                                     None, 0, _cabi.KFAC_ITEM_DIAG_G)
        need = lib.kfac_precondition_workspace_bytes(items, 1)
        ws = torch.zeros(need, dtype=torch.uint8, device=DEV)
        need_items.append(lib.kfac_precondition(items, 1, method, 0.1, ws.data_ptr(), need, S()))
    assert need_items == [_cabi.KFAC_ERR_NOT_READY] * 3


# ---------------------------------------------------------------------------------------------- module level
V_LM, D_LM, B_LM, T_LM = 10007, 64, 4, 64


class LM(nn.Module):
    def __init__(self):
        super().__init__()
        from workloads import NeoXBlock
        self.emb = nn.Embedding(V_LM, D_LM)
        self.block = NeoXBlock(D_LM)
        self.head = nn.Linear(D_LM, V_LM)

    def forward(self, idx):
        return self.head(self.block(self.emb(idx)))


def _batch(step):
    g = torch.Generator().manual_seed(step)
    idx = torch.randint(0, V_LM, (B_LM, T_LM), generator=g)
    idx[0, 10:40] = 17
    dev = torch.device('cuda', torch.cuda.current_device())
    return idx.to(dev), torch.randint(0, V_LM, (B_LM, T_LM), generator=g).to(dev)


def _grad_matrix(m):
    g = m.weight.grad.double().reshape(m.weight.shape[0], -1)
    bias = getattr(m, 'bias', None)
    return torch.cat([g, bias.grad.double()[:, None]], 1) if bias is not None else g


def _eigh(F):
    d, q = torch.linalg.eigh(F.double())
    return q, d.clamp(min=0)


def _inv(F, damping):
    return torch.linalg.inv(F.double() + damping * torch.eye(F.shape[0], dtype=torch.float64, device=F.device))


def p_ref(l, method, grad, A, G, damping):
    """fp64 P of a dense, embedding (A a vector) or diagonal-G (G a vector) layer."""
    if l.diag_g:
        if method == 'inverse':
            return (grad / (G.double()[:, None] + damping)) @ _inv(A, damping)
        qa, da = _eigh(A)
        return ((grad @ qa) / (G.double()[:, None] * da[None, :] + damping)) @ qa.t()
    if l.diag_a:
        if method == 'inverse':
            return (grad / (A.double()[:, None] + damping)) @ _inv(G, damping)
        qg, dg = _eigh(G)
        return ((grad @ qg) / (A.double()[:, None] * dg[None, :] + damping)) @ qg.t()
    if method == 'inverse':
        return _inv(G, damping) @ grad @ _inv(A, damping)
    qa, da = _eigh(A)
    qg, dg = _eigh(G)
    return qg @ ((qg.t() @ grad @ qa) / (dg[:, None] * da[None, :] + damping)) @ qa.t()


def keep_logits_grad(model, seen):
    def hook(module, input_, output):        # returns None: the output is left as it is
        output.register_hook(lambda g: seen.__setitem__('g', g.detach()))
    model.head.register_forward_hook(hook)


SCHEDULES = {'every': (1, 1), 'f2i4': (2, 4),
             'callable': (lambda s: 1 if s < 3 else 2, lambda s: 2 if s < 3 else 4)}


@pytest.mark.parametrize('emb', [False, True])
@pytest.mark.parametrize('schedule', list(SCHEDULES))
@pytest.mark.parametrize('method', ['eigen', 'inverse'])
def test_lm_against_fp64(method, schedule, emb):
    """Every layer's written gradient (kl-clip off: exactly P) against fp64.  The head's G is restated as
    diag(g^T g / N) from the logits gradient; every other factor is the one the preconditioner holds at its inverse
    steps."""
    from kfac_b200.preconditioner import KFACPreconditioner
    fus, ius = SCHEDULES[schedule]
    damping, alpha = 0.003, 0.9
    torch.manual_seed(0)
    model = LM().to(DEV)
    pre = KFACPreconditioner(model, diagonal_g_layers=['head'], precondition_embeddings=emb, factor_update_steps=fus,
                             inv_update_steps=ius, damping=damping, factor_decay=alpha, kl_clip=None,
                             compute_method=method)
    layers = {m: l for m, (_, l) in pre._layers.items()}
    lh = layers[model.head]
    assert lh.diag_g and lh.g_dim == V_LM and len(layers) == 5 + emb
    seen = {}
    keep_logits_grad(model, seen)
    opt = torch.optim.SGD(model.parameters(), lr=0.05)
    G_ref = None
    snap = {}
    for s in range(6):
        is_factor = s % pre.factor_update_steps == 0
        is_inv = s % pre.inv_update_steps == 0
        idx, y = _batch(s)
        opt.zero_grad()
        nn.functional.cross_entropy(model(idx).flatten(0, 1), y.flatten()).backward()
        grads = {m: _grad_matrix(m) for m in layers}
        pre.step()
        torch.cuda.synchronize()
        if is_factor:
            g = seen['g'].double().reshape(-1, V_LM)
            g_b = (g * g).sum(0) / g.shape[0]
            G_ref = alpha * (torch.ones_like(g_b) if G_ref is None else G_ref) + (1 - alpha) * g_b
        assert lh.g_factor.shape == (V_LM,) and rel_fro(lh.g_factor, G_ref) < 1e-5, s
        if is_inv:
            snap = {m: (l.a_factor.double(), G_ref.clone() if l.diag_g else l.g_factor.double())
                    for m, l in layers.items()}
            assert lh.qg is None and lh.g_inv is None and lh.dgda is None
            assert torch.equal(lh.dg, lh.g_factor)
            assert (lh.qa is not None) if method == 'eigen' else (lh.a_inv is not None)
        for m, l in layers.items():
            A, G = snap[m]
            ref = p_ref(l, method, grads[m], A, G, damping)
            got = _grad_matrix(m)
            assert rel_fro(got, ref) < 1e-3, (s, pre._layers[m][0], rel_fro(got, ref))
        opt.step()


@pytest.mark.parametrize('emb', [False, True])
@pytest.mark.parametrize('method', ['eigen', 'inverse'])
def test_first_step_other_gradients_unchanged(method, emb):
    """Same weights, same batch, kl-clip off: every layer but the head (and the embedding, whose G shares its
    eigensolver call with the head's A) gets the same bits with the head skipped and with the head diagonal."""
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(0)
    m_diag = LM().to(DEV)
    m_skip = copy.deepcopy(m_diag)
    out = []
    for model, kw in ((m_diag, dict(diagonal_g_layers=['head'])), (m_skip, dict(skip_layers=['head']))):
        pre = KFACPreconditioner(model, kl_clip=None, compute_method=method, precondition_embeddings=emb, **kw)
        idx, y = _batch(0)
        nn.functional.cross_entropy(model(idx).flatten(0, 1), y.flatten()).backward()
        pre.step()
        torch.cuda.synchronize()
        out.append({n: p.grad.clone() for n, p in model.named_parameters()})
    for n in out[0]:
        if n.startswith('block'):
            assert torch.equal(bits(out[0][n]), bits(out[1][n])), n
    assert not torch.equal(out[0]['head.weight'], out[1]['head.weight'])


def test_kl_clip_includes_the_head():
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(0)
    m_p = LM().to(DEV)
    m_c = copy.deepcopy(m_p)
    idx, y = _batch(1)
    lr = 0.1
    res = []
    for model, kl in ((m_p, None), (m_c, 1e-3)):
        pre = KFACPreconditioner(model, diagonal_g_layers=['head'], kl_clip=kl, lr=lr)
        nn.functional.cross_entropy(model(idx).flatten(0, 1), y.flatten()).backward()
        grads = {n: p.grad.double().clone() for n, p in model.named_parameters()}
        pre.step()
        torch.cuda.synchronize()
        res.append((pre, grads, {n: p.grad.clone() for n, p in model.named_parameters()}))
    _, grads, P = res[0]
    P = {n: p for n, p in P.items() if not n.startswith('emb')}     # the embedding is not registered here
    vg = sum(float((P[n].double() * grads[n]).sum()) for n in P)
    nu_ref = min(1.0, (1e-3 / abs(vg * lr * lr)) ** 0.5)
    pre_c, _, written = res[1]
    nu = pre_c._compute_grad_scale()
    assert nu_ref < 1.0 and abs(nu - nu_ref) <= 1e-5 * nu_ref, (nu, nu_ref)
    head = sum(float((P[n].double() * grads[n]).sum()) for n in ('head.weight', 'head.bias')) / vg
    assert head > 1e-6
    for n in P:
        assert torch.equal(written[n], pre_c.last_grad_scale * P[n]), n


def test_state_dict_round_trip():
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(0)
    m1 = LM().to(DEV)
    pre1 = KFACPreconditioner(m1, diagonal_g_layers=['head'], kl_clip=None, inv_update_steps=2)
    opt = torch.optim.SGD(m1.parameters(), lr=0.05)
    for s in range(3):
        idx, y = _batch(s)
        opt.zero_grad()
        nn.functional.cross_entropy(m1(idx).flatten(0, 1), y.flatten()).backward()
        pre1.step()
        opt.step()
    sd = pre1.state_dict()
    assert sd['layers']['head']['G'].shape == (V_LM,) and sd['layers']['head']['A'].shape == (D_LM + 1, D_LM + 1)
    assert pre1.memory_usage()['g_factors'] >= V_LM * 4
    m2 = LM().to(DEV)
    m2.load_state_dict(m1.state_dict())
    pre2 = KFACPreconditioner(m2, diagonal_g_layers=['head'], kl_clip=None, inv_update_steps=2)
    pre2.load_state_dict(sd)
    for model, pre in ((m1, pre1), (m2, pre2)):
        model.zero_grad()
        idx, y = _batch(3)
        nn.functional.cross_entropy(model(idx).flatten(0, 1), y.flatten()).backward()
        pre.step()
    torch.cuda.synchronize()
    for (n, p1), (_, p2) in zip(m1.named_parameters(), m2.named_parameters()):
        assert torch.equal(p1.grad, p2.grad), n
    bad = copy.deepcopy(sd)
    bad['layers']['head']['G'] = torch.ones(V_LM, V_LM, device=DEV)
    with pytest.raises(ValueError, match='shape'):
        KFACPreconditioner(LM().to(DEV), diagonal_g_layers=['head']).load_state_dict(bad)


def test_fp16_overflow_drops_the_head_window():
    """An injected fp16 overflow under a GradScaler: every G window is dropped and counted once -- the head's
    through the guarded vector EMA -- and training stays finite."""
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(0)
    model = LM().to(DEV)
    scaler = torch.amp.GradScaler('cuda', init_scale=2.0 ** 10)
    pre = KFACPreconditioner(model, diagonal_g_layers=['head'], grad_scaler=scaler, damping=0.003)
    layers = {m: l for m, (_, l) in pre._layers.items()}
    lh = layers[model.head]
    opt = torch.optim.SGD(model.parameters(), lr=0.01)
    for step in range(5):
        idx, y = _batch(step)
        opt.zero_grad()
        if step == 2:
            scaler.update(new_scale=2.0 ** 60)
            before = {m: l.g_factor.clone() for m, l in layers.items()}
        with torch.autocast('cuda', dtype=torch.float16):
            loss = nn.functional.cross_entropy(model(idx).flatten(0, 1).float(), y.flatten())
        scaler.scale(loss).backward()
        scaler.unscale_(opt)
        pre.step()
        torch.cuda.synchronize()
        if step == 1:
            assert pre.skipped_factor_updates == 0 and lh.g_factor.shape == (V_LM,)
        if step == 2:
            for m, l in layers.items():
                assert torch.equal(l.g_factor, before[m]), pre._layers[m][0]
            assert pre.skipped_factor_updates == len(layers)
        elif step > 2:
            for p in model.parameters():
                assert torch.isfinite(p.grad).all(), step
        scaler.step(opt)
        if step == 2:
            scaler.update(new_scale=2.0 ** 10)
        else:
            scaler.update()
    assert torch.isfinite(lh.g_factor).all() and torch.isfinite(lh.a_factor).all()


def test_non_finite_head_g_raises_at_next_step():
    from kfac_b200 import _cabi
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(0)
    model = LM().to(DEV)
    pre = KFACPreconditioner(model, diagonal_g_layers=['head'], factor_update_steps=2, inv_update_steps=1)
    lh = pre._layers[model.head][1]

    def step(s):
        idx, y = _batch(s)
        model.zero_grad()
        nn.functional.cross_entropy(model(idx).flatten(0, 1), y.flatten()).backward()
        pre.step()
        torch.cuda.synchronize()

    step(0)
    step(1)                       # no factor update: the snapshot of the factor below is the one checked
    lh._g_view[V_LM // 2] = float('inf')
    step(2)                       # a factor step: the window is finite, the factor stays inf; the inverse snapshots it
    with pytest.raises(_cabi.KFACNativeError, match='non-finite'):
        step(3)


def test_no_host_sync_in_hooks():
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(0)
    model = LM().to(DEV)
    scaler = torch.amp.GradScaler('cuda', init_scale=2.0 ** 10)
    pre = KFACPreconditioner(model, diagonal_g_layers=['head'], precondition_embeddings=True, grad_scaler=scaler)
    opt = torch.optim.SGD(model.parameters(), lr=0.01)
    for s in range(2):
        idx, y = _batch(s)
        opt.zero_grad()
        torch.cuda.synchronize()
        if s == 1:
            torch.cuda.set_sync_debug_mode('error')
        try:
            with torch.autocast('cuda', dtype=torch.float16):
                loss = nn.functional.cross_entropy(model(idx).flatten(0, 1).float(), y.flatten())
            scaler.scale(loss).backward()
        finally:
            torch.cuda.set_sync_debug_mode(0)
        scaler.unscale_(opt)
        pre.step()
        scaler.step(opt)
        scaler.update()
    torch.cuda.synchronize()
    assert pre._layers[model.head][1]._g_count == 0 and pre._layers[model.head][1]._has_g


# ---------------------------------------------------------------------------------------------- two ranks
def _run_dist(backend):
    import socket
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    script = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'dist_diag_g.py')
    out = subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node=2',
                          '--master-addr', '127.0.0.1', '--master-port', str(port), script, '--backend', backend],
                         capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, (out.stdout[-3000:], out.stderr[-3000:])
    assert out.stdout.count('dist_diag_g ok') == 2, out.stdout[-2000:]


def test_two_ranks_gloo():
    """Two ranks over gloo (they may share one GPU), COMM_OPT and MEM_OPT: P identical on both ranks and equal to
    fp64 on the concatenated batch."""
    _run_dist('gloo')


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='NCCL needs one GPU per rank')
def test_two_ranks_nccl():
    _run_dist('nccl')
