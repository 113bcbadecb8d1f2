"""Embedding-bag preconditioning (`precondition_embedding_bags=True`) on the GPU, everything against fp64:

  * kfac_factor_embedding_bag against an fp64 restatement from the dense pooled rows C, for 1-D indices with offsets
    (with and without include_last_offset) and 2-D indices, int32 and int64, sum and mean, with and without
    padding_idx, empty bags and fp32 / fp16 / bf16 per-sample weights; integer cases exact, the same bits on a
    repeat, and bags of one index giving the bits of kfac_factor_embedding;
  * a text-classifier-shaped model (mean bag + Linear) and a small DLRM-shaped model (weighted sum bags + MLPs) over
    several steps: every layer's P against fp64 under eigen (with and without compute_eigenvalue_outer_product),
    inverse and pi_damping;
  * the dense layers' P bit-identical with the bag registered and with it in skip_layers; a bag of one-index bags
    with the A and G bits of an nn.Embedding on those indices;
  * a state_dict round trip, an fp16 overflow under a GradScaler, a non-finite per-sample weight with and without a
    GradScaler, the bag's statistics without host syncs, and two ranks (tests/dist_embedding_bag.py).
"""
import copy
import os
import subprocess
import sys

import pytest
import torch
from torch import nn

from conftest import rel_fro
from test_gpu_embedding import _grad_matrix, _p_dense, _p_embedding
from test_pi_damping_host import pi_ref, precondition_ref

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


# ---------------------------------------------------------------------------------------------- fp64 restatement
def pooled_rows(idx, offsets, B, V, mode, weights=None, padding_idx=None):
    """The (B, V) pooled rows C of one call in fp64: torch's bag semantics restated from the indices (with
    include_last_offset the last offset is not read: the last bag ends at the last index, as in torch)."""
    if idx.dim() == 2:
        bag = torch.arange(B, device=idx.device).repeat_interleave(idx.size(1))
        idx = idx.flatten()
    else:
        bag = torch.searchsorted(offsets[:B].long(), torch.arange(idx.numel(), device=idx.device), right=True) - 1
    keep = bag >= 0
    if padding_idx is not None:
        keep &= idx != padding_idx
    w = weights.double().flatten() if weights is not None else torch.ones(idx.numel(), dtype=torch.float64,
                                                                          device=idx.device)
    C = torch.zeros(B, V, dtype=torch.float64, device=idx.device)
    C.index_put_((bag[keep], idx[keep].long()), w[keep], accumulate=True)
    if mode == 'mean':
        L = torch.zeros(B, dtype=torch.float64, device=idx.device).index_add_(0, bag[keep], w[keep] * 0 + 1)
        C /= L.clamp(min=1)[:, None]
    return C


def bag_a(C):
    """The diagonal A of the pooled rows: (1/B) sum_b c_bv^2."""
    return (C * C).sum(0) / C.shape[0]


def random_bags(gen, B, V, lo, hi, frequent=None, padding_idx=None):
    """1-D indices and offsets of B bags of lo..hi entries; `frequent` opens 90 % of the non-empty bags."""
    lens = torch.randint(lo, hi + 1, (B,), generator=gen)
    idx = torch.randint(0, V, (int(lens.sum()),), generator=gen)
    offsets = torch.cat([torch.zeros(1, dtype=torch.long), lens.cumsum(0)[:-1]])
    if frequent is not None:
        for b in range(B):
            if lens[b] > 0 and b % 10:
                idx[offsets[b]] = frequent
    if padding_idx is not None:
        idx[::7] = padding_idx
    return idx.to(DEV), offsets.to(DEV)


# ---------------------------------------------------------------------------------------------- the kernel
def _call(lib, idx, offsets, B, mode, weights, padding_idx, include_last, V, alpha, acc):
    from kfac_b200 import _cabi
    need = lib.kfac_factor_embedding_bag_workspace_bytes(idx.numel(), B, V)
    ws = torch.full((max(need, 1),), 255, dtype=torch.uint8, device=DEV)
    rc = lib.kfac_factor_embedding_bag(idx.data_ptr(), offsets.data_ptr() if offsets is not None else None,
                                       _cabi.INDEX_DTYPE_CODE[idx.dtype], idx.numel(), B,
                                       -1 if padding_idx is None else padding_idx,
                                       {'sum': _cabi.KFAC_BAG_SUM, 'mean': _cabi.KFAC_BAG_MEAN}[mode],
                                       weights.data_ptr() if weights is not None else None,
                                       _cabi.DTYPE_CODE[weights.dtype] if weights is not None else 0, V, alpha,
                                       acc.data_ptr(), ws.data_ptr(), need, S())
    assert rc == 0, lib.kfac_last_error()
    torch.cuda.synchronize()
    return acc


CASES = {'sum': ('sum', None), 'mean': ('mean', None), 'w_int': ('sum', 'int'), 'w_f32': ('sum', torch.float32),
         'w_f16': ('sum', torch.float16), 'w_bf16': ('sum', torch.bfloat16)}


@pytest.mark.parametrize('case', list(CASES))
@pytest.mark.parametrize('padding_idx', [None, 5])
@pytest.mark.parametrize('dtype', [torch.int32, torch.int64])
@pytest.mark.parametrize('form', ['offsets', 'include_last_offset', '2d'])
def test_factor_embedding_bag_against_fp64(lib, form, dtype, padding_idx, case):
    mode, wdtype = CASES[case]
    V, B = 5000, 300
    gen = torch.Generator().manual_seed(sum(map(ord, form + case)))
    include_last = form == 'include_last_offset'
    if form == '2d':
        idx = torch.randint(0, V, (B, 24), generator=gen)
        idx[::3, :5] = 7                                      # repeats inside a bag
        if padding_idx is not None:
            idx[1] = padding_idx                              # a bag of padding only: an empty row
            idx[:, -3:] = padding_idx
        idx, offsets = idx.to(DEV), None
    else:
        idx, offsets = random_bags(gen, B, V, 0, 60, frequent=7, padding_idx=padding_idx)
        idx[40:50] = 11                                       # a token repeated inside a bag
        if include_last:                                      # B + 1 offsets, the last one ending the last bag
            offsets = torch.cat([offsets, torch.tensor([idx.numel()], device=DEV)])
    idx = idx.to(dtype)
    offsets = offsets.to(dtype) if offsets is not None else None
    weights = None
    if wdtype == 'int':
        weights = torch.randint(-3, 4, (idx.numel(),), generator=gen).float().to(DEV)
    elif wdtype is not None:
        weights = (torch.rand(idx.numel(), generator=gen) * 2 - 0.5).to(wdtype).to(DEV)
    C = pooled_rows(idx, offsets, B, V, mode, weights, padding_idx)
    s_ref = (C * C).sum(0)
    zero = torch.zeros(V, device=DEV)
    s = _call(lib, idx, offsets, B, mode, weights, padding_idx, include_last, V, 1.0, zero.clone())
    if mode == 'sum' and wdtype in (None, 'int'):
        assert torch.equal(s, s_ref.float())                  # integer sums are exact
    else:
        assert bool(((s.double() - s_ref).abs() <= s_ref.abs() * 2.0 ** -24 * (1 + 1e-9)).all()), case
    # into a live batch: one rounding of alpha * s, one of the sum; the same bits on a repeat
    live = torch.rand(V, device=DEV)
    alpha = float(torch.tensor(1.0 / B, dtype=torch.float32))
    acc = _call(lib, idx, offsets, B, mode, weights, padding_idx, include_last, V, alpha, live.clone())
    assert torch.equal(acc, live + torch.tensor(alpha, device=DEV) * s)
    again = _call(lib, idx, offsets, B, mode, weights, padding_idx, include_last, V, alpha, live.clone())
    assert torch.equal(bits(acc), bits(again))


def test_factor_embedding_bag_long_runs_and_rejections(lib):
    """One token in each of 40k bags (a run of 40k pairs), and the arguments the call refuses."""
    from kfac_b200 import _cabi
    V, B = 1000, 40000
    gen = torch.Generator().manual_seed(1)
    idx, offsets = random_bags(gen, B, V, 1, 6, frequent=3)
    w = torch.rand(idx.numel(), generator=gen).to(DEV)
    s = _call(lib, idx, offsets, B, 'sum', w, None, False, V, 1.0, torch.zeros(V, device=DEV))
    s_ref = (pooled_rows(idx, offsets, B, V, 'sum', w) ** 2).sum(0)
    assert rel_fro(s, s_ref) < 1e-6
    need = lib.kfac_factor_embedding_bag_workspace_bytes(idx.numel(), B, V)
    acc = torch.zeros(V, device=DEV)
    ws = torch.empty(need, dtype=torch.uint8, device=DEV)
    args = lambda mode, wp, n_ws: (idx.data_ptr(), offsets.data_ptr(), _cabi.INDEX_DTYPE_CODE[idx.dtype],  # noqa
                                   idx.numel(), B, -1, mode, wp, 0, V, 1.0, acc.data_ptr(), ws.data_ptr(), n_ws, S())
    assert lib.kfac_factor_embedding_bag(*args(_cabi.KFAC_BAG_SUM, None, need - 1)) == _cabi.KFAC_ERR_WORKSPACE
    assert lib.kfac_factor_embedding_bag(*args(_cabi.KFAC_BAG_MEAN, w.data_ptr(), need)) == _cabi.KFAC_ERR_BAD_ARG
    assert lib.kfac_factor_embedding_bag(*args(2, None, need)) == _cabi.KFAC_ERR_BAD_ARG


@pytest.mark.parametrize('mode', ['sum', 'mean'])
@pytest.mark.parametrize('dtype', [torch.int32, torch.int64])
def test_bags_of_one_index_give_the_embedding_bits(lib, mode, dtype):
    from kfac_b200 import _cabi
    V = 50257
    gen = torch.Generator(device=DEV).manual_seed(3)
    idx = torch.randint(0, V, (4096,), device=DEV, generator=gen, dtype=dtype)
    idx[:300] = 7
    N = idx.numel()
    alpha = float(torch.tensor(1.0 / N, dtype=torch.float32))
    live = torch.rand(V, device=DEV, generator=gen)
    got = _call(lib, idx, torch.arange(N, device=DEV, dtype=dtype), N, mode, None, None, False, V, alpha, live.clone())
    want = live.clone()
    need = lib.kfac_factor_embedding_workspace_bytes(V)
    ws = torch.empty(need, dtype=torch.uint8, device=DEV)
    assert lib.kfac_factor_embedding(idx.data_ptr(), _cabi.INDEX_DTYPE_CODE[dtype], N, V, alpha, want.data_ptr(),
                                     ws.data_ptr(), need, S()) == 0
    torch.cuda.synchronize()
    assert torch.equal(bits(got), bits(want))


# ---------------------------------------------------------------------------------------------- models
V_TC, D_TC, B_TC = 3000, 32, 64


class TextClassifier(nn.Module):
    """The text classifier of PyTorch's text-classification tutorial: a mean bag over the vocabulary and a Linear."""

    def __init__(self, V=V_TC, d=D_TC, classes=4, padding_idx=0):
        super().__init__()
        self.bag = nn.EmbeddingBag(V, d, mode='mean', padding_idx=padding_idx)
        self.fc = nn.Linear(d, classes)

    def forward(self, idx, offsets):
        return self.fc(self.bag(idx, offsets))


def mlp(sizes, last_relu):
    layers = []
    for i in range(len(sizes) - 1):
        layers.append(nn.Linear(sizes[i], sizes[i + 1]))
        if i < len(sizes) - 2 or last_relu:
            layers.append(nn.ReLU())
    return nn.Sequential(*layers)


class DLRM(nn.Module):
    """A DLRM-shaped recommender: a bottom MLP on the dense features, one weighted sum bag per sparse feature, and a
    top MLP on their concatenation."""

    def __init__(self, V=2000, d=16, tables=3, bottom=(13, 32), top=(32,)):
        super().__init__()
        self.bottom = mlp(bottom + (d,), True)
        self.tables = nn.ModuleList(nn.EmbeddingBag(V, d, mode='sum') for _ in range(tables))
        self.top = mlp((d * (tables + 1),) + top + (1,), False)

    def forward(self, dense, sparse):
        z = [self.bottom(dense)] + [t(i, o, per_sample_weights=w) for t, (i, o, w) in zip(self.tables, sparse)]
        return self.top(torch.cat(z, 1)).squeeze(1)


def tc_batch(step, B=B_TC, V=V_TC):
    gen = torch.Generator().manual_seed(step)
    idx, offsets = random_bags(gen, B, V, 0, 40, frequent=17, padding_idx=0)
    return idx, offsets, torch.randint(0, 4, (B,), generator=gen).to(DEV)


def dlrm_batch(step, model, B=64):
    gen = torch.Generator().manual_seed(100 + step)
    sparse = []
    for t in model.tables:
        idx, offsets = random_bags(gen, B, t.num_embeddings, 1, 12, frequent=1)
        sparse.append((idx, offsets, torch.rand(idx.numel(), generator=gen).to(DEV)))
    return torch.randn(B, 13, generator=gen).to(DEV), sparse, torch.randint(0, 2, (B,), generator=gen).float().to(DEV)


def _bag_inputs(model, batch):
    """The bag modules of a model and the (idx, offsets, weights) each is called with."""
    if isinstance(model, TextClassifier):
        return {model.bag: (batch[0], batch[1], None)}
    return dict(zip(model.tables, batch[1]))


def _loss(model, batch):
    if isinstance(model, TextClassifier):
        return nn.functional.cross_entropy(model(batch[0], batch[1]), batch[2])
    return nn.functional.binary_cross_entropy_with_logits(model(batch[0], batch[1]), batch[2])


def _batch_for(model, step):
    return tc_batch(step) if isinstance(model, TextClassifier) else dlrm_batch(step, model)


def _keep_grad_outputs(bags):
    seen = {}
    for m in bags:
        def hook(module, input_, output, m=m):          # returns None: the output is left as it is
            output.register_hook(lambda g: seen.__setitem__(m, g.detach()))
        m.register_forward_hook(hook)
    return seen


@pytest.mark.parametrize('model_cls', [TextClassifier, DLRM])
@pytest.mark.parametrize('method,prediv,pi', [('eigen', True, False), ('eigen', False, False),
                                              ('inverse', False, False), ('eigen', True, True),
                                              ('inverse', False, True)])
def test_models_against_fp64(model_cls, method, prediv, pi):
    """Every layer's written gradient (kl-clip off: exactly P) against fp64 over five steps (inverse every second
    step).  The bags' factors are restated from their inputs and output gradients; the dense layers' P is formed in
    fp64 from the factors the preconditioner holds at its inverse steps."""
    from kfac_b200.preconditioner import KFACPreconditioner
    damping, alpha = 0.003, 0.9
    torch.manual_seed(0)
    model = model_cls().to(DEV)
    pre = KFACPreconditioner(model, precondition_embedding_bags=True, inv_update_steps=2, damping=damping,
                             factor_decay=alpha, kl_clip=None, compute_method=method,
                             compute_eigenvalue_outer_product=prediv, pi_damping=pi)
    layers = {m: l for m, (_, l) in pre._layers.items()}
    bags = [m for m in layers if isinstance(m, nn.EmbeddingBag)]
    assert bags and all(layers[m].diag_a for m in bags)
    seen = _keep_grad_outputs(bags)
    opt = torch.optim.SGD(model.parameters(), lr=0.05)
    ref = {m: None for m in bags}
    snap = {}
    for s in range(5):
        batch = _batch_for(model, s)
        opt.zero_grad()
        _loss(model, batch).backward()
        grads = {m: _grad_matrix(m) for m in layers}
        pre.step()
        torch.cuda.synchronize()
        for m, (idx, offsets, w) in _bag_inputs(model, batch).items():
            B = offsets.numel()
            a_b = bag_a(pooled_rows(idx, offsets, B, m.num_embeddings, m.mode, w, m.padding_idx))
            g = seen[m].double()
            g_b = g.t() @ g / B
            if ref[m] is None:                    # the first window is seeded with ones / identity
                ref[m] = (torch.ones_like(a_b), torch.eye(g.shape[1], dtype=torch.float64, device=DEV))
            A_ref, G_ref = ref[m]
            ref[m] = (alpha * A_ref + (1 - alpha) * a_b, alpha * G_ref + (1 - alpha) * g_b)
            assert layers[m].a_factor.shape == (m.num_embeddings,)
            assert rel_fro(layers[m].a_factor, ref[m][0]) < 1e-6, s
            assert rel_fro(layers[m].g_factor, ref[m][1]) < 1e-5, s
        if s % 2 == 0:
            snap = {m: ref[m] if m in ref else (l.a_factor.double(), l.g_factor.double()) for m, l in layers.items()}
        for m, l in layers.items():
            A, G = snap[m]
            if pi:
                gm = grads[m].t() if l.embedding else grads[m]
                want = precondition_ref(gm, A, G, pi_ref(A, G), damping, damping)
                want = want.t() if l.embedding else want
            elif l.embedding:
                want = _p_embedding(method, grads[m], A, G, damping)
            else:
                want = _p_dense(method, grads[m], A, G, damping)
            got = _grad_matrix(m)
            assert rel_fro(got, want) < 1e-3, (s, pre._layers[m][0], rel_fro(got, want))
        opt.step()


@pytest.mark.parametrize('model_cls', [TextClassifier, DLRM])
@pytest.mark.parametrize('method', ['eigen', 'inverse'])
def test_dense_layers_keep_their_bits(model_cls, method):
    """Same weights, same batch, kl-clip off: the dense layers' P is the same bits with the bags registered and with
    them in skip_layers (later steps differ: the bags are then updated differently)."""
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(0)
    m_on = model_cls().to(DEV)
    m_off = copy.deepcopy(m_on)
    out = []
    for model, skip in ((m_on, []), (m_off, ['EmbeddingBag'])):
        pre = KFACPreconditioner(model, precondition_embedding_bags=True, skip_layers=skip, kl_clip=None,
                                 compute_method=method)
        assert any(l.diag_a for _, l in pre._layers.values()) == (not skip)
        _loss(model, _batch_for(model, 0)).backward()
        pre.step()
        torch.cuda.synchronize()
        out.append({n: p.grad.clone() for n, p in model.named_parameters()})
    for n in out[0]:
        if 'bag' in n or 'tables' in n:
            assert not torch.equal(out[0][n], out[1][n]), n
        else:
            assert torch.equal(bits(out[0][n]), bits(out[1][n])), n


@pytest.mark.parametrize('mode', ['sum', 'mean'])
def test_one_index_bags_match_an_embedding(mode):
    """A bag of one-index bags has the A and G bits of an nn.Embedding on those indices."""
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(0)
    V, d, N = 500, 24, 256
    emb_model = nn.Sequential(nn.Embedding(V, d), nn.Tanh(), nn.Linear(d, 3)).to(DEV)
    bag_model = nn.Sequential(nn.EmbeddingBag(V, d, mode=mode), nn.Tanh(), nn.Linear(d, 3)).to(DEV)
    bag_model.load_state_dict(emb_model.state_dict())
    pe = KFACPreconditioner(emb_model, precondition_embeddings=True)
    pb = KFACPreconditioner(bag_model, precondition_embedding_bags=True)
    for s in range(2):
        gen = torch.Generator().manual_seed(s)
        idx = torch.randint(0, V, (N,), generator=gen).to(DEV)
        idx[:40] = 9
        y = torch.randint(0, 3, (N,), generator=gen).to(DEV)
        for model, pre, call in ((emb_model, pe, lambda m: m[0](idx)),
                                 (bag_model, pb, lambda m: m[0](idx, torch.arange(N, device=DEV)))):
            model.zero_grad()
            nn.functional.cross_entropy(model[2](model[1](call(model))), y).backward()
            pre.step()
        torch.cuda.synchronize()
        le, lb = pe._layers[emb_model[0]][1], pb._layers[bag_model[0]][1]
        assert torch.equal(bits(le.a_factor), bits(lb.a_factor)), s
        assert torch.equal(bits(le.g_factor), bits(lb.g_factor)), s


def test_state_dict_round_trip():
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(0)
    m1 = DLRM().to(DEV)
    pre1 = KFACPreconditioner(m1, precondition_embedding_bags=True, kl_clip=None, inv_update_steps=2)
    opt = torch.optim.SGD(m1.parameters(), lr=0.05)
    for s in range(3):
        opt.zero_grad()
        _loss(m1, dlrm_batch(s, m1)).backward()
        pre1.step()
        opt.step()
    sd = pre1.state_dict()
    assert sd['layers']['tables.0']['A'].shape == (2000,) and sd['layers']['tables.0']['G'].shape == (16, 16)
    m2 = DLRM().to(DEV)
    m2.load_state_dict(m1.state_dict())
    pre2 = KFACPreconditioner(m2, precondition_embedding_bags=True, kl_clip=None, inv_update_steps=2)
    pre2.load_state_dict(sd)
    # step 3 is no inverse step: pre1 uses the inverses of step 2, pre2 those the load formed from the same factors
    for model, pre in ((m1, pre1), (m2, pre2)):
        model.zero_grad()
        _loss(model, dlrm_batch(3, model)).backward()
        pre.step()
    torch.cuda.synchronize()
    for (n, p1), (_, p2) in zip(m1.named_parameters(), m2.named_parameters()):
        assert torch.equal(p1.grad, p2.grad), n
    mem = pre2.memory_usage()
    assert mem['total'] > 0
    bad = copy.deepcopy(sd)
    bad['layers']['tables.1']['A'] = torch.ones(2001, device=DEV)
    with pytest.raises(ValueError, match='shape'):
        KFACPreconditioner(DLRM().to(DEV), precondition_embedding_bags=True).load_state_dict(bad)


def _huge_weight(model, batch):
    """Give entry 0 of table 0 the weight 1e10 and zero its token's row: its c^2 = 1e20 leaves the forward pass as it
    is and makes the bag's A window exceed 1e15, the bound above which a window or snapshot counts as not finite."""
    idx, _, w = batch[1][0]
    w[0] = 1e10
    with torch.no_grad():
        model.tables[0].weight[idx[0]] = 0


def _amp_step(model, pre, scaler, opt, batch):
    with torch.autocast('cuda', dtype=torch.float16):
        loss = _loss(model, batch)
    scaler.scale(loss.float()).backward()
    scaler.unscale_(opt)
    pre.step()


def test_fp16_overflow_keeps_factors():
    """An injected fp16 overflow under a GradScaler: the G windows are dropped (G unchanged) and the bags' finite A
    windows are taken.  A per-sample weight whose square exceeds what a window may hold (on a zero row, so the forward
    pass is unchanged) drops that bag's A window (A unchanged) and nothing else's."""
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(0)
    model = DLRM().to(DEV)
    scaler = torch.amp.GradScaler('cuda', init_scale=2.0 ** 10)
    pre = KFACPreconditioner(model, precondition_embedding_bags=True, grad_scaler=scaler, damping=0.003)
    layers = {m: l for m, (_, l) in pre._layers.items()}
    bag = layers[model.tables[0]]
    opt = torch.optim.SGD(model.parameters(), lr=0.01)
    for step in range(6):
        batch = dlrm_batch(step, model)
        opt.zero_grad()
        if step == 2:
            scaler.update(new_scale=2.0 ** 60)
        if step == 4:
            _huge_weight(model, batch)
        if step in (2, 4):
            before = {m: (l.a_factor.clone(), l.g_factor.clone()) for m, l in layers.items()}
            skipped = pre.skipped_factor_updates
        _amp_step(model, pre, scaler, opt, batch)
        torch.cuda.synchronize()
        if step == 2:
            for m, l in layers.items():
                assert torch.equal(l.g_factor, before[m][1]), pre._layers[m][0]
            assert not torch.equal(bag.a_factor, before[model.tables[0]][0])    # a finite A window is taken
            assert pre.skipped_factor_updates - skipped == len(layers)
        if step == 4:
            assert torch.equal(bag.a_factor, before[model.tables[0]][0])
            assert pre.skipped_factor_updates - skipped == 1
        for l in layers.values():
            assert torch.isfinite(l.a_factor).all() and torch.isfinite(l.g_factor).all(), step
        scaler.step(opt)
        if step == 2:
            scaler.update(new_scale=2.0 ** 10)
        else:
            scaler.update()


def test_non_finite_weight_without_scaler_raises():
    """Without a GradScaler a per-sample weight whose window is not finite reaches the bag's A, and the next step()
    raises."""
    from kfac_b200 import _cabi
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(0)
    model = DLRM().to(DEV)
    pre = KFACPreconditioner(model, precondition_embedding_bags=True, damping=0.003)

    def step(s, huge=False):
        batch = dlrm_batch(s, model)
        if huge:
            _huge_weight(model, batch)
        model.zero_grad()
        _loss(model, batch).backward()
        pre.step()
        torch.cuda.synchronize()

    step(0)
    step(1, huge=True)            # the window enters the factor; the inverse step snapshots it
    with pytest.raises(_cabi.KFACNativeError, match='non-finite'):
        step(2)


def test_no_host_sync_in_bag_statistics():
    """The bag's A and G statistics (bind_call, the A kernel, the G rows) run without a host sync."""
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(0)
    model = DLRM().to(DEV)
    scaler = torch.amp.GradScaler('cuda', init_scale=2.0 ** 10)
    pre = KFACPreconditioner(model, precondition_embedding_bags=True, grad_scaler=scaler)
    opt = torch.optim.SGD(model.parameters(), lr=0.01)
    _amp_step(model, pre, scaler, opt, dlrm_batch(0, model))
    scaler.step(opt)
    scaler.update()
    opt.zero_grad()
    layer = pre._layers[model.tables[0]][1]
    helper = layer.module
    calls = []
    for name in ('bind_call', 'accumulate_a', 'accumulate_g'):
        def strict(*args, f=getattr(helper, name), name=name, **kw):
            calls.append(name)
            torch.cuda.set_sync_debug_mode('error')
            try:
                return f(*args, **kw)
            finally:
                torch.cuda.set_sync_debug_mode(0)
        setattr(helper, name, strict)
    batch = dlrm_batch(1, model)
    torch.cuda.synchronize()
    with torch.autocast('cuda', dtype=torch.float16):
        loss = _loss(model, batch)
    scaler.scale(loss.float()).backward()
    torch.cuda.synchronize()
    assert calls == ['bind_call', 'accumulate_a', 'accumulate_g']
    assert layer._g_count == 1 and layer._a_count == 1


# ---------------------------------------------------------------------------------------------- two ranks
def _run_dist(backend):
    import socket
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    script = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'dist_embedding_bag.py')
    out = subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node=2',
                          '--master-addr', '127.0.0.1', '--master-port', str(port), script, '--backend', backend],
                         capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, (out.stdout[-3000:], out.stderr[-3000:])
    assert out.stdout.count('dist_embedding_bag ok') == 2, out.stdout[-2000:]


def test_two_ranks_gloo():
    """Two ranks over gloo (they may share one GPU), COMM_OPT and MEM_OPT: P identical on both ranks and equal to
    fp64 on the concatenated batch."""
    _run_dist('gloo')


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='NCCL needs one GPU per rank')
def test_two_ranks_nccl():
    _run_dist('nccl')
