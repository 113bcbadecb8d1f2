"""Embedding preconditioning (`precondition_embeddings=True`) on the GPU, everything against fp64:

  * kfac_factor_embedding against bincount / N, accumulated into a live batch, the same bits on a repeat;
  * kfac_factor_ema_diag against an fp64 evaluation of the EMA (within 1 ulp), and against the diagonal of the
    dense EMA bit for bit;
  * kfac_precondition with embedding items of V in {1000, 50257} and d in {48, 768} in one call with Linear- and
    Conv-shaped dense items, eigen (dense items with dgda and with da/dg) and inverse: P against fp64, the same
    bits on a repeat, and the dense items' P bit-identical with and without the embedding items;
  * a small LM (Embedding -> NeoX block -> untied Linear head) over several steps with integer and callable
    schedules: every layer's P against an fp64 restatement, and the first step's non-embedding gradients
    bit-identical with the keyword on and off;
  * the kl-clip scale, a state_dict round trip, an fp16 overflow under a GradScaler, hooks without host syncs,
    and two ranks (tests/dist_embedding.py).
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
@pytest.mark.parametrize('dtype', [torch.int32, torch.int64])
def test_factor_embedding_counts(lib, dtype):
    from kfac_b200 import _cabi
    V = 50257
    gen = torch.Generator(device=DEV).manual_seed(3)
    idx = torch.randint(0, V, (8, 512), device=DEV, generator=gen, dtype=dtype)
    idx[0, :100] = 7                      # a frequent token
    idx[1, :3] = V - 1
    N = idx.numel()
    alpha = float(torch.tensor(1.0 / N, dtype=torch.float32))
    live = torch.rand(V, device=DEV, generator=gen)          # a batch vector that already holds a window
    need = lib.kfac_factor_embedding_workspace_bytes(V)
    assert need >= V * 4

    def run():
        acc = live.clone()
        ws = torch.full((need,), 255, dtype=torch.uint8, device=DEV)
        rc = lib.kfac_factor_embedding(idx.data_ptr(), _cabi.INDEX_DTYPE_CODE[dtype], N, V, alpha, acc.data_ptr(),
                                       ws.data_ptr(), need, S())
        assert rc == 0, lib.kfac_last_error()
        torch.cuda.synchronize()
        return acc

    acc = run()
    counts = torch.bincount(idx.flatten().long(), minlength=V)
    ref = live.double() + counts.double() / N
    assert float((acc.double() - ref).abs().max()) <= 1e-6
    # one rounding of alpha * count, one of the sum
    assert torch.equal(acc, live + torch.tensor(alpha, device=DEV) * counts.float())
    assert torch.equal(bits(acc), bits(run()))
    # a call with too small a workspace is rejected
    assert lib.kfac_factor_embedding(idx.data_ptr(), _cabi.INDEX_DTYPE_CODE[dtype], N, V, alpha, acc.data_ptr(),
                                     acc.data_ptr(), need - 4, S()) != 0


def test_ema_diag(lib):
    from kfac_b200 import _cabi
    gen = torch.Generator(device=DEV).manual_seed(5)
    alpha = float(torch.tensor(0.95, dtype=torch.float32))
    dims, firsts, inv_counts = (1000, 300, 50257), (1, 0, 0), (1.0, 0.25, 1.0)
    fac0 = [torch.rand(d, device=DEV, generator=gen) for d in dims]
    bat0 = [torch.rand(d, device=DEV, generator=gen) * 1e-2 for d in dims]

    def run():
        fac = [f.clone() for f in fac0]
        bat = [b.clone() for b in bat0]
        items = (_cabi.EmaItem * len(dims))()
        for i, d in enumerate(dims):
            items[i] = _cabi.EmaItem(fac[i].data_ptr(), bat[i].data_ptr(), d, firsts[i], inv_counts[i])
        assert lib.kfac_factor_ema_diag(items, len(dims), alpha, S()) == 0, lib.kfac_last_error()
        torch.cuda.synchronize()
        return fac, bat

    fac, bat = run()
    for i in range(len(dims)):
        f = torch.ones_like(fac0[i]).double() if firsts[i] else fac0[i].double()
        ref = alpha * f + (1 - alpha) * bat0[i].double() * inv_counts[i]
        ulp = (torch.nextafter(fac[i], torch.tensor(float('inf'), device=DEV)) - fac[i]).double()
        assert bool(((fac[i].double() - ref).abs() <= ulp).all()), i
        assert not bool(bat[i].any())
    fac2, _ = run()
    for a, b in zip(fac, fac2):
        assert torch.equal(bits(a), bits(b))
    # the diagonal of the dense EMA on diag(batch), bit for bit
    d = dims[1]
    F = torch.diag(fac0[1]).contiguous()
    B = torch.diag(bat0[1]).contiguous()
    items = (_cabi.EmaItem * 1)(_cabi.EmaItem(F.data_ptr(), B.data_ptr(), d, 0, inv_counts[1]))
    assert lib.kfac_factor_ema(items, 1, alpha, S()) == 0
    torch.cuda.synchronize()
    assert torch.equal(bits(torch.diagonal(F).contiguous()), bits(fac[1]))


# ---------------------------------------------------------------------------------------------- precondition
def _stored(x):
    from kfac_b200 import _cabi
    out = torch.full((x.shape[0], _cabi.ld4(x.shape[1])), float('nan'), device=DEV)
    out[:, :x.shape[1]] = x
    return out


@pytest.mark.parametrize('prediv', [True, False])
def test_precondition_embedding_items(lib, prediv):
    """Embedding items mixed with dense items in one call.  prediv: the dense items' eigen epilogue (dgda or
    dg x da); the embedding items always use the vector form."""
    from kfac_b200 import _cabi
    damping = float(torch.tensor(0.003, dtype=torch.float32))
    gen = torch.Generator(device=DEV).manual_seed(11)

    def basis(n):
        q, _ = torch.linalg.qr(torch.randn(n, n, dtype=torch.float64, device=DEV, generator=gen))
        return q.float(), (torch.rand(n, dtype=torch.float64, device=DEV, generator=gen) ** 4).float()

    # dense: (g, a, bias, dtype) -- a Linear layer, a 3x3 Conv2d layer, a small one on the SIMT path
    dense = [(256, 129, 1, torch.float32), (64, 577, 1, torch.float16), (10, 21, 1, torch.bfloat16)]
    # embedding: (V, d, dtype)
    embs = [(1000, 48, torch.float16), (50257, 768, torch.float32), (1000, 768, torch.bfloat16), (50257, 48, torch.float32)]
    D, E = [], []
    for g, a, bias, dtype in dense:
        qa, da = basis(a)
        qg, dg = basis(g)
        w = torch.randn(g, a - bias, device=DEV, generator=gen).to(dtype)
        b = torch.randn(g, device=DEV, generator=gen).to(dtype)
        dgda = (1.0 / (dg.double()[:, None] * da.double()[None, :] + damping)).float()
        a_inv = ((qa.double() / (da.double() + damping)) @ qa.double().t()).float()
        g_inv = ((qg.double() / (dg.double() + damping)) @ qg.double().t()).float()
        D.append(dict(g=g, a=a, dtype=dtype, w=w, b=b, qa=_stored(qa), qaT=_stored(qa.t()), qg=_stored(qg),
                      qgT=_stored(qg.t()), dgda=_stored(dgda), da=da, dg=dg, a_inv=_stored(a_inv), g_inv=_stored(g_inv)))
    for V, d, dtype in embs:
        qg, dg = basis(d)
        counts = torch.randint(0, 40, (V,), device=DEV, generator=gen).double()
        counts[torch.rand(V, device=DEV, generator=gen) < 0.3] = 0       # tokens never seen
        av = (counts / counts.sum()).float()
        w = torch.randn(V, d, device=DEV, generator=gen)
        w[av == 0] = 0                                                     # ... have zero gradient rows
        w = w.to(dtype)
        g_inv = ((qg.double() / (dg.double() + damping)) @ qg.double().t()).float()
        grad, qg64 = w.double(), qg.double()
        ref_e = ((grad @ qg64) / (av.double()[:, None] * dg.double()[None, :] + damping)) @ qg64.t()
        ref_i = (grad / (av.double()[:, None] + damping)) @ g_inv.double()
        E.append(dict(V=V, d=d, dtype=dtype, w=w, av=av, qg=_stored(qg), qgT=_stored(qg.t()), dg=dg,
                      g_inv=_stored(g_inv), ref_e=ref_e, ref_i=ref_i))

    def precondition(method, with_emb):
        e = method == _cabi.KFAC_EIGEN
        layers = [('d', l) for l in D] + ([('e', l) for l in E] if with_emb else [])
        # embeddings first and in between: the order of the items must not matter either
        if with_emb:
            layers = [layers[3], layers[0], layers[4], layers[1], layers[5], layers[2], layers[6]]
        items = (_cabi.PrecondItem * len(layers))()
        Ps = []
        for i, (kind, l) in enumerate(layers):
            if kind == 'd':
                g, a = l['g'], l['a']
                P = torch.full((g, _cabi.ld4(a)), float('nan'), device=DEV)
                p = lambda k, use: l[k].data_ptr() if use else None  # noqa: E731,B023
                items[i] = _cabi.PrecondItem(l['w'].data_ptr(), l['b'].data_ptr(), _cabi.DTYPE_CODE[l['dtype']], g, a,
                                             p('qa', e), p('qaT', e), p('qg', e), p('qgT', e), p('dgda', e and prediv),
                                             p('da', e and not prediv), p('dg', e and not prediv),
                                             p('a_inv', not e), p('g_inv', not e), _cabi.ld4(a), _cabi.ld4(g),
                                             _cabi.ld4(a), P.data_ptr(), _cabi.ld4(a))
                Ps.append((kind, l, P[:, :a]))
            else:
                V, d = l['V'], l['d']
                P = torch.full((V, _cabi.ld4(d)), float('nan'), device=DEV)
                p = lambda k, use: l[k].data_ptr() if use else None  # noqa: E731,B023
                items[i] = _cabi.PrecondItem(l['w'].data_ptr(), None, _cabi.DTYPE_CODE[l['dtype']], d, V,
                                             None, None, p('qg', e), p('qgT', e), None, l['av'].data_ptr(), p('dg', e),
                                             None, p('g_inv', not e), 0, _cabi.ld4(d), 0, P.data_ptr(), _cabi.ld4(d),
                                             None, 0, _cabi.KFAC_ITEM_EMBEDDING)
                Ps.append((kind, l, P[:, :d]))
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
            if kind == 'e':
                assert rel_fro(P, l[key]) < 1e-3, (method, l['V'], l['d'], rel_fro(P, l[key]))
                assert not bool(P[l['av'] == 0].any())          # zero gradient rows stay zero
        P2 = precondition(method, True)
        for (_, _, p1), (_, _, p2) in zip(P1, P2):
            assert torch.equal(bits(p1), bits(p2))
        dense_only = {id(l): P for _, l, P in precondition(method, False)}
        for kind, l, P in P1:
            if kind == 'd':
                assert torch.equal(bits(P), bits(dense_only[id(l)])), (method, l['g'], l['a'])
        del P1, P2


def test_precondition_rejects_incomplete_embedding_item(lib):
    from kfac_b200 import _cabi
    w = torch.zeros(100, 8, device=DEV)
    P = torch.zeros(100, 8, device=DEV)
    items = (_cabi.PrecondItem * 1)()
    items[0] = _cabi.PrecondItem(w.data_ptr(), None, 0, 8, 100, None, None, None, None, None, None, None, None, None,
                                 0, 8, 0, P.data_ptr(), 8, None, 0, _cabi.KFAC_ITEM_EMBEDDING)
    need = lib.kfac_precondition_workspace_bytes(items, 1)
    ws = torch.zeros(need, dtype=torch.uint8, device=DEV)
    assert lib.kfac_precondition(items, 1, _cabi.KFAC_INVERSE, 0.1, ws.data_ptr(), need, S()) == _cabi.KFAC_ERR_NOT_READY


# ---------------------------------------------------------------------------------------------- module level
V_LM, D_LM, B_LM, T_LM = 1000, 192, 4, 64


class LM(nn.Module):
    def __init__(self):
        super().__init__()
        from workloads import NeoXBlock
        self.emb = nn.Embedding(V_LM, D_LM, padding_idx=0)
        self.block = NeoXBlock(D_LM)
        self.head = nn.Linear(D_LM, V_LM)

    def forward(self, idx):
        return self.head(self.block(self.emb(idx)))


def _batch(step):
    g = torch.Generator().manual_seed(step)
    idx = torch.randint(0, V_LM, (B_LM, T_LM), generator=g)
    idx[:, :5] = 0                                       # padding positions are rows too
    idx[0, 10:40] = 17                                   # a frequent token
    dev = torch.device('cuda', torch.cuda.current_device())
    return idx.to(dev), torch.randint(0, V_LM, (B_LM, T_LM), generator=g).to(dev)


def _grad_matrix(m):
    g = m.weight.grad.double().reshape(m.weight.shape[0], -1)
    bias = getattr(m, 'bias', None)                      # nn.Embedding has none
    return torch.cat([g, bias.grad.double()[:, None]], 1) if bias is not None else g


def _eigh(F):
    d, q = torch.linalg.eigh(F.double())
    return q, d.clamp(min=0)


def _p_dense(method, grad, A, G, damping):
    if method == 'inverse':
        ia = torch.linalg.inv(A.double() + damping * torch.eye(A.shape[0], dtype=torch.float64, device=grad.device))
        ig = torch.linalg.inv(G.double() + damping * torch.eye(G.shape[0], dtype=torch.float64, device=grad.device))
        return ig @ grad @ ia
    qa, da = _eigh(A)
    qg, dg = _eigh(G)
    return qg @ ((qg.t() @ grad @ qa) / (dg[:, None] * da[None, :] + damping)) @ qa.t()


def _p_embedding(method, grad, a, G, damping):
    if method == 'inverse':
        ig = torch.linalg.inv(G.double() + damping * torch.eye(G.shape[0], dtype=torch.float64, device=grad.device))
        return (grad / (a.double()[:, None] + damping)) @ ig
    qg, dg = _eigh(G)
    return ((grad @ qg) / (a.double()[:, None] * dg[None, :] + damping)) @ qg.t()


SCHEDULES = {'every': (1, 1), 'f2i4': (2, 4),
             'callable': (lambda s: 1 if s < 3 else 2, lambda s: 2 if s < 3 else 4)}


@pytest.mark.parametrize('schedule', list(SCHEDULES))
@pytest.mark.parametrize('method,prediv', [('eigen', True), ('eigen', False), ('inverse', False)])
def test_lm_against_fp64(schedule, method, prediv):
    """Every layer's written gradient (kl-clip off: exactly P) against fp64.  The embedding's factors are restated
    from the indices and grad-outputs (which also shows the output hook fires); the dense layers' P is formed in
    fp64 from the factors the preconditioner holds at its inverse steps."""
    from kfac_b200.preconditioner import KFACPreconditioner
    fus, ius = SCHEDULES[schedule]
    damping, alpha = 0.003, 0.9
    torch.manual_seed(0)
    model = LM().to(DEV)
    pre = KFACPreconditioner(model, precondition_embeddings=True, factor_update_steps=fus, inv_update_steps=ius,
                             damping=damping, factor_decay=alpha, kl_clip=None, compute_method=method,
                             compute_eigenvalue_outer_product=prediv)
    layers = {m: l for m, (_, l) in pre._layers.items()}
    assert layers[model.emb].diag_a and len(layers) == 6
    seen = {}

    def keep_grad_output(module, input_, output):   # returns None: the output is left as it is
        output.register_hook(lambda g: seen.__setitem__('g', g.detach()))
    model.emb.register_forward_hook(keep_grad_output)
    opt = torch.optim.SGD(model.parameters(), lr=0.05)
    A_ref = G_ref = None
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
            N = idx.numel()
            a_b = torch.bincount(idx.flatten(), minlength=V_LM).double() / N
            g = seen['g'].double().reshape(N, D_LM)
            g_b = g.t() @ g / N
            if A_ref is None:      # the first window is seeded with ones / identity
                A_ref, G_ref = torch.ones_like(a_b), torch.eye(D_LM, dtype=torch.float64, device=DEV)
            A_ref = alpha * A_ref + (1 - alpha) * a_b
            G_ref = alpha * G_ref + (1 - alpha) * g_b
        le = layers[model.emb]
        assert le.a_factor.shape == (V_LM,) and rel_fro(le.a_factor, A_ref) < 1e-6, s
        assert rel_fro(le.g_factor, G_ref) < 1e-5, s
        if is_inv:
            snap = {m: (A_ref.clone(), G_ref.clone()) if l.diag_a else (l.a_factor.double(), l.g_factor.double())
                    for m, l in layers.items()}
            assert le.qa is None and le.a_inv is None and le.dgda is None
            assert torch.equal(le.da, le.a_factor) if method == 'eigen' else le.g_inv is not None
        for m, l in layers.items():
            A, G = snap[m]
            if l.diag_a:
                ref = _p_embedding(method, grads[m], A, G, damping)
            else:
                ref = _p_dense(method, grads[m], A, G, damping)
            got = _grad_matrix(m)
            assert rel_fro(got, ref) < 1e-3, (s, pre._layers[m][0], rel_fro(got, ref))
        assert not bool(model.emb.weight.grad[0].any())          # the padding row stays zero
        opt.step()


@pytest.mark.parametrize('method', ['eigen', 'inverse'])
def test_first_step_dense_gradients_unchanged(method):
    """Same weights, same batch, kl-clip off: the gradients written for the non-embedding layers are the same bits
    with and without the keyword (later steps differ: the embedding itself is then updated differently)."""
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(0)
    m_on = LM().to(DEV)
    m_off = copy.deepcopy(m_on)
    out = []
    for model, flag in ((m_on, True), (m_off, False)):
        pre = KFACPreconditioner(model, precondition_embeddings=flag, kl_clip=None, compute_method=method)
        assert any(l.diag_a for _, l in pre._layers.values()) == flag
        idx, y = _batch(0)
        nn.functional.cross_entropy(model(idx).flatten(0, 1), y.flatten()).backward()
        pre.step()
        torch.cuda.synchronize()
        out.append({n: p.grad.clone() for n, p in model.named_parameters()})
    for n in out[0]:
        if not n.startswith('emb'):
            assert torch.equal(bits(out[0][n]), bits(out[1][n])), n
    assert not torch.equal(out[0]['emb.weight'], out[1]['emb.weight'])


def test_kl_clip_includes_the_embedding():
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(0)
    m_p = LM().to(DEV)
    m_c = copy.deepcopy(m_p)
    idx, y = _batch(1)
    lr = 0.1
    res = []
    for model, kl in ((m_p, None), (m_c, 1e-3)):
        pre = KFACPreconditioner(model, precondition_embeddings=True, kl_clip=kl, lr=lr)
        nn.functional.cross_entropy(model(idx).flatten(0, 1), y.flatten()).backward()
        grads = {n: p.grad.double().clone() for n, p in model.named_parameters()}
        pre.step()
        torch.cuda.synchronize()
        res.append((pre, grads, {n: p.grad.clone() for n, p in model.named_parameters()}))
    _, grads, P = res[0]                                   # kl-clip off: the written gradients are P
    vg = sum(float((P[n].double() * grads[n]).sum()) for n in P)
    nu_ref = min(1.0, (1e-3 / abs(vg * lr * lr)) ** 0.5)
    pre_c, _, written = res[1]
    nu = pre_c._compute_grad_scale()
    assert nu_ref < 1.0 and abs(nu - nu_ref) <= 1e-5 * nu_ref, (nu, nu_ref)
    emb_share = float((P['emb.weight'].double() * grads['emb.weight']).sum()) / vg
    assert emb_share > 1e-6                                # the embedding's term is part of the sum
    nu_t = pre_c.last_grad_scale
    for n in P:
        assert torch.equal(written[n], nu_t * P[n]), n


def test_state_dict_round_trip():
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(0)
    m1 = LM().to(DEV)
    pre1 = KFACPreconditioner(m1, precondition_embeddings=True, kl_clip=None, inv_update_steps=2)
    opt = torch.optim.SGD(m1.parameters(), lr=0.05)
    for s in range(3):
        idx, y = _batch(s)
        opt.zero_grad()
        nn.functional.cross_entropy(m1(idx).flatten(0, 1), y.flatten()).backward()
        pre1.step()
        opt.step()
    sd = pre1.state_dict()
    assert sd['layers']['emb']['A'].shape == (V_LM,) and sd['layers']['emb']['G'].shape == (D_LM, D_LM)
    m2 = LM().to(DEV)                  # (a deep copy of m1 would copy pre1's hooks with it)
    m2.load_state_dict(m1.state_dict())
    pre2 = KFACPreconditioner(m2, precondition_embeddings=True, kl_clip=None, inv_update_steps=2)
    pre2.load_state_dict(sd)
    # step 3 is no inverse step: pre1 uses the inverses of step 2, pre2 those the load formed from the same factors
    for model, pre in ((m1, pre1), (m2, pre2)):
        model.zero_grad()
        idx, y = _batch(3)
        nn.functional.cross_entropy(model(idx).flatten(0, 1), y.flatten()).backward()
        pre.step()
    torch.cuda.synchronize()
    for (n, p1), (_, p2) in zip(m1.named_parameters(), m2.named_parameters()):
        assert torch.equal(p1.grad, p2.grad), n
    bad = copy.deepcopy(sd)
    bad['layers']['emb']['A'] = torch.ones(V_LM + 1, device=DEV)
    with pytest.raises(ValueError, match='shape'):
        KFACPreconditioner(LM().to(DEV), precondition_embeddings=True).load_state_dict(bad)


def test_fp16_overflow_keeps_factors():
    """An injected fp16 overflow under a GradScaler: the G windows are dropped (G unchanged), the embedding's A
    window of counts is kept, and training stays finite."""
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(0)
    model = LM().to(DEV)
    scaler = torch.amp.GradScaler('cuda', init_scale=2.0 ** 10)
    pre = KFACPreconditioner(model, precondition_embeddings=True, grad_scaler=scaler, damping=0.003)
    layers = {m: l for m, (_, l) in pre._layers.items()}
    le = layers[model.emb]
    opt = torch.optim.SGD(model.parameters(), lr=0.01)
    for step in range(5):
        idx, y = _batch(step)
        opt.zero_grad()
        if step == 2:
            scaler.update(new_scale=2.0 ** 60)
            before = {m: (l.a_factor.clone(), l.g_factor.clone()) for m, l in layers.items()}
        with torch.autocast('cuda', dtype=torch.float16):
            loss = nn.functional.cross_entropy(model(idx).flatten(0, 1).float(), y.flatten())
        scaler.scale(loss).backward()
        scaler.unscale_(opt)
        pre.step()
        torch.cuda.synchronize()
        if step == 2:
            for m, l in layers.items():
                assert torch.equal(l.g_factor, before[m][1]), pre._layers[m][0]
            assert not torch.equal(le.a_factor, before[model.emb][0])       # the counts window was taken
            assert pre.skipped_factor_updates == len(layers)
        elif step > 2:
            for p in model.parameters():
                assert torch.isfinite(p.grad).all(), step
        scaler.step(opt)
        if step == 2:
            scaler.update(new_scale=2.0 ** 10)
        else:
            scaler.update()
    for l in layers.values():
        assert torch.isfinite(l.a_factor).all() and torch.isfinite(l.g_factor).all()


def test_no_host_sync_in_hooks():
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(0)
    model = LM().to(DEV)
    scaler = torch.amp.GradScaler('cuda', init_scale=2.0 ** 10)
    pre = KFACPreconditioner(model, precondition_embeddings=True, grad_scaler=scaler)
    opt = torch.optim.SGD(model.parameters(), lr=0.01)

    def fwd_bwd(step):
        idx, y = _batch(step)
        with torch.autocast('cuda', dtype=torch.float16):
            loss = nn.functional.cross_entropy(model(idx).flatten(0, 1).float(), y.flatten())
        scaler.scale(loss).backward()

    fwd_bwd(0)
    scaler.unscale_(opt)
    pre.step()
    scaler.step(opt)
    scaler.update()
    opt.zero_grad()
    idx, y = _batch(1)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        with torch.autocast('cuda', dtype=torch.float16):
            loss = nn.functional.cross_entropy(model(idx).flatten(0, 1).float(), y.flatten())
        scaler.scale(loss).backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert pre._layers[model.emb][1]._g_count == 1 and pre._layers[model.emb][1]._a_count == 1


# ---------------------------------------------------------------------------------------------- two ranks
def _run_dist(backend):
    import socket
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    script = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'dist_embedding.py')
    out = subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node=2',
                          '--master-addr', '127.0.0.1', '--master-port', str(port), script, '--backend', backend],
                         capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, (out.stdout[-3000:], out.stderr[-3000:])
    assert out.stdout.count('dist_embedding ok') == 2, out.stdout[-2000:]


def test_two_ranks_gloo():
    """Two ranks over gloo (they may share one GPU), COMM_OPT and MEM_OPT: P identical on both ranks and equal to
    fp64 on the concatenated batch."""
    _run_dist('gloo')


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='NCCL needs one GPU per rank')
def test_two_ranks_nccl():
    _run_dist('nccl')
