"""GPU tests of tied embedding / LM-head pairs (`precondition_tied_embeddings=True`), against fp64:
  * kfac_tied_whiten / kfac_tied_basis: M^T (E + tI) M = I and M^T (H + tI) M = diag(mu) for d on both sides of the
    eigensolver's n = 128 switch and of the K > 1024 split, with well-conditioned and cond ~ 1e6 factors; C exactly
    symmetric; the same bits on a repeat;
  * kfac_precondition with KFAC_ITEM_TIED items among dense, embedding and diagonal-G items: P against the per-row
    fp64 solve of (f_v + t)(E + tI) + (h_v + t)(H + tI), for fp32 / fp16 / bf16 gradients; the other items' P
    bit-identical with and without the tied items;
  * a nanoGPT-shaped model with a tied embedding / head: the weight's gradient against the fp64 formula built from
    the pair's own snapshots, every other gradient bit-identical to a run with the head skipped, eigen and inverse,
    integer and callable schedules; a state_dict round trip; an fp16 overflow under a GradScaler; hooks without host
    syncs; the keyword on without a pair gives the bits of the keyword off; two ranks (tests/dist_tied.py).
"""
import copy
import ctypes as C
import os
import subprocess
import sys

import pytest
import torch
from torch import nn

from conftest import rel_fro

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda')
KW = dict(precondition_embeddings=True, diagonal_g_layers=['head'], precondition_tied_embeddings=True)


@pytest.fixture(scope='module')
def lib():
    from kfac_b200 import _cabi
    return _cabi.load()


def S():
    return torch.cuda.current_stream().cuda_stream


def bits(x):
    return x.contiguous().view(torch.int32 if x.element_size() == 4 else torch.int16)


def ld4(n):
    return (n + 3) & ~3


def spd(d, cond, seed, scale=1.0):
    """fp64 SPD matrix with eigenvalues log-spaced over [scale / cond, scale]."""
    gen = torch.Generator().manual_seed(seed)
    q, _ = torch.linalg.qr(torch.randn(d, d, generator=gen, dtype=torch.float64))
    ev = scale * torch.logspace(-torch.log10(torch.tensor(float(cond))).item(), 0, d, dtype=torch.float64)
    return (q * ev) @ q.T


def _eigh(lib, F):
    """The library's eigendecomposition of fp32 F (d x d, ld = d): Q, QT (ld4), eigenvalues."""
    from kfac_b200 import _cabi
    d = F.shape[0]
    Q = torch.zeros(d, ld4(d), device=DEV)
    QT = torch.zeros(d, ld4(d), device=DEV)
    e = torch.zeros(d, device=DEV)
    item = (_cabi.EighItem * 1)(_cabi.EighItem(F.data_ptr(), Q.data_ptr(), QT.data_ptr(), e.data_ptr(), d, ld4(d),
                                               None))
    ns = (C.c_int * 1)(d)
    need = lib.kfac_eigh_workspace_bytes(ns, 1)
    ws = torch.empty(need, dtype=torch.uint8, device=DEV)
    assert lib.kfac_eigh_batched(item, 1, ws.data_ptr(), need, 0, 0.0, S()) == 0, lib.kfac_last_error()
    return Q, QT, e


def tied_data(lib, E, H, t):
    """M (d x ld4), M^T, mu and C of fp32 factors E, H through the library's path (eigh, whiten, eigh, basis)."""
    from kfac_b200 import _cabi
    d = E.shape[0]
    E, H = E.float().contiguous().to(DEV), H.float().contiguous().to(DEV)
    Q, QT, e = _eigh(lib, E)
    Cm = torch.zeros(d, d, device=DEV)
    M = torch.zeros(d, ld4(d), device=DEV)
    MT = torch.zeros(d, ld4(d), device=DEV)
    item = _cabi.TiedItem(Q.data_ptr(), QT.data_ptr(), e.data_ptr(), H.data_ptr(), Cm.data_ptr(), None, None, None,
                          d, ld4(d))
    items = (_cabi.TiedItem * 1)(item)
    need = lib.kfac_tied_workspace_bytes(items, 1)
    ws = torch.full((need,), 255, dtype=torch.uint8, device=DEV)
    assert lib.kfac_tied_whiten(items, 1, t, ws.data_ptr(), need - 4, S()) != 0
    assert lib.kfac_tied_whiten(items, 1, t, ws.data_ptr(), need, S()) == 0, lib.kfac_last_error()
    C_out = Cm.clone()
    U, UT, mu = _eigh(lib, Cm)
    items[0].UT, items[0].M, items[0].MT = UT.data_ptr(), M.data_ptr(), MT.data_ptr()
    assert lib.kfac_tied_basis(items, 1, t, ws.data_ptr(), need, S()) == 0, lib.kfac_last_error()
    torch.cuda.synchronize()
    return M, MT, mu, C_out


# ---------------------------------------------------------------------------------------------- whitening
@pytest.mark.parametrize('d', [48, 129, 768, 1025])
@pytest.mark.parametrize('cond', [10.0, 1e6])
def test_tied_whiten_diagonalises_both_factors(lib, d, cond):
    # lambda_max(E) = 1: the damping bounds cond(E + tI) by 101 and the condition number of M by about 10
    t = 1e-2
    E = spd(d, cond, seed=d)
    H = spd(d, cond, seed=d + 1, scale=0.5)
    M, MT, mu, Cm = tied_data(lib, E, H, t)
    assert torch.equal(bits(Cm), bits(Cm.T))                       # the eigensolver sees an exact symmetric input
    assert torch.equal(bits(MT[:, :d]), bits(M[:, :d].T.contiguous()))
    assert torch.all(torch.isfinite(M)) and torch.all(mu > 0)
    Md = M[:, :d].double().cpu()
    I = torch.eye(d, dtype=torch.float64)
    err_e = rel_fro(Md.T @ (E + t * I) @ Md, I)
    err_h = rel_fro(Md.T @ (H + t * I) @ Md, torch.diag(mu.double().cpu()))
    print(f'd={d} cond={cond:g}: E {err_e:.2e}  H {err_h:.2e}')
    assert err_e <= 1e-4 and err_h <= 1e-4, (err_e, err_h)
    again = tied_data(lib, E, H, t)
    for x, y in zip((M, MT, mu, Cm), again):
        assert torch.equal(bits(x), bits(y))


# ---------------------------------------------------------------------------------------------- precondition
def _f_h(V, seed):
    gen = torch.Generator().manual_seed(seed)
    f = torch.rand(V, generator=gen, dtype=torch.float64) ** 4
    f[::7] = 0.0                                                    # tokens that never occur
    h = torch.rand(V, generator=gen, dtype=torch.float64) * 1e-2
    return (f / f.sum()).float(), h.float()


def _ref_rows(grad, E, H, f, h, t, rows):
    """Per-row fp64 solve of (f_v + t)(E + tI) + (h_v + t)(H + tI), not through M."""
    d = E.shape[0]
    I = torch.eye(d, dtype=torch.float64, device=DEV)
    Eh, Hh = (E.double().to(DEV) + t * I), (H.double().to(DEV) + t * I)
    out = []
    for chunk in rows.split(256):
        fv = f.double().to(DEV)[chunk].view(-1, 1, 1) + t
        hv = h.double().to(DEV)[chunk].view(-1, 1, 1) + t
        F = fv * Eh + hv * Hh
        out.append(torch.linalg.solve(F, grad.double().to(DEV)[chunk].unsqueeze(-1)).squeeze(-1))
    return torch.cat(out)


def _tied_item(grad, M, MT, mu, f, h, t, P):
    from kfac_b200 import _cabi
    V, d = grad.shape
    return _cabi.PrecondItem(grad.data_ptr(), None, _cabi.DTYPE_CODE[grad.dtype], d, V, None, None, M.data_ptr(),
                             MT.data_ptr(), None, f.data_ptr(), mu.data_ptr(), None, None, 0, ld4(d), 0, P.data_ptr(),
                             ld4(d), None, 0, _cabi.KFAC_ITEM_TIED, h.data_ptr(), t)


def _other_items(lib, gen):
    """A dense, an embedding and a diagonal-G item with arbitrary (orthogonal) eigen data, and their outputs."""
    from kfac_b200 import _cabi

    def orth(n):
        q = torch.linalg.qr(torch.randn(n, n, generator=gen, dtype=torch.float64))[0].float()
        Q = torch.zeros(n, ld4(n))
        Q[:, :n] = q
        QT = torch.zeros(n, ld4(n))
        QT[:, :n] = q.T
        return Q.to(DEV), QT.to(DEV)

    keep = []
    items = []
    # dense: g = 96, a = 130 (with a bias)
    g, a = 96, 130
    w = torch.randn(g, a - 1, generator=gen).to(DEV)
    b = torch.randn(g, generator=gen).to(DEV)
    qa, qaT = orth(a)
    qg, qgT = orth(g)
    da, dg = torch.rand(a, generator=gen).to(DEV), torch.rand(g, generator=gen).to(DEV)
    P = torch.zeros(g, ld4(a), device=DEV)
    keep += [w, b, qa, qaT, qg, qgT, da, dg, P]
    items.append((_cabi.PrecondItem(w.data_ptr(), b.data_ptr(), 0, g, a, qa.data_ptr(), qaT.data_ptr(), qg.data_ptr(),
                                    qgT.data_ptr(), None, da.data_ptr(), dg.data_ptr(), None, None, ld4(a), ld4(g), 0,
                                    P.data_ptr(), ld4(a), None, 0), P))
    # embedding: V = 3000, d = 64
    V, d = 3000, 64
    w = torch.randn(V, d, generator=gen).to(DEV)
    q, qT = orth(d)
    fa, ev = torch.rand(V, generator=gen).to(DEV), torch.rand(d, generator=gen).to(DEV)
    P = torch.zeros(V, ld4(d), device=DEV)
    keep += [w, q, qT, fa, ev, P]
    items.append((_cabi.PrecondItem(w.data_ptr(), None, 0, d, V, None, None, q.data_ptr(), qT.data_ptr(), None,
                                    fa.data_ptr(), ev.data_ptr(), None, None, 0, ld4(d), 0, P.data_ptr(), ld4(d), None,
                                    0, _cabi.KFAC_ITEM_EMBEDDING), P))
    # diagonal-G: V = 2000, a = 65 (with a bias)
    V, a = 2000, 65
    w = torch.randn(V, a - 1, generator=gen).to(DEV)
    b = torch.randn(V, generator=gen).to(DEV)
    q, qT = orth(a)
    ea, hg = torch.rand(a, generator=gen).to(DEV), torch.rand(V, generator=gen).to(DEV)
    P = torch.zeros(V, ld4(a), device=DEV)
    keep += [w, b, q, qT, ea, hg, P]
    items.append((_cabi.PrecondItem(w.data_ptr(), b.data_ptr(), 0, V, a, q.data_ptr(), qT.data_ptr(), None, None,
                                    None, ea.data_ptr(), hg.data_ptr(), None, None, ld4(a), 0, 0, P.data_ptr(), ld4(a),
                                    None, 0, _cabi.KFAC_ITEM_DIAG_G), P))
    return items, keep


def _precondition(lib, items, method=1, damping=0.003):
    from kfac_b200 import _cabi
    arr = (_cabi.PrecondItem * len(items))(*items)
    need = lib.kfac_precondition_workspace_bytes(arr, len(items))
    ws = torch.full((need,), 255, dtype=torch.uint8, device=DEV)
    rc = lib.kfac_precondition(arr, len(items), method, damping, ws.data_ptr(), need, S())
    assert rc == 0, lib.kfac_last_error()
    torch.cuda.synchronize()


@pytest.mark.parametrize('V,d', [(1000, 96), (50257, 768)])
@pytest.mark.parametrize('dtype', [torch.float32, torch.float16, torch.bfloat16])
def test_precondition_tied_items_against_fp64(lib, V, d, dtype):
    t = 3e-3
    gen = torch.Generator().manual_seed(V + d)
    E = spd(d, 1e4, seed=V, scale=0.2)
    H = spd(d, 1e3, seed=V + 1, scale=2.0)
    f, h = _f_h(V, seed=d)
    fD, hD = f.to(DEV), h.to(DEV)
    M, MT, mu, _ = tied_data(lib, E, H, t)
    grad = torch.randn(V, d, generator=gen).to(dtype).to(DEV)
    grad[::7] = 0                                                    # the rows of absent tokens
    P = torch.full((V, ld4(d)), float('nan'), device=DEV)
    others, keep = _other_items(lib, gen)
    tied = _tied_item(grad, M, MT, mu, fD, hD, t, P)
    _precondition(lib, [it for it, _ in others] + [tied])
    mixed = P.clone()
    with_tied = [p.clone() for _, p in others]
    _precondition(lib, [it for it, _ in others])
    for (_, p), q in zip(others, with_tied):
        assert torch.equal(bits(p), bits(q))
    for method in (1, 2):                                            # the call's method is not used by tied items
        P.fill_(float('nan'))
        _precondition(lib, [tied], method=method)
        assert torch.equal(bits(P), bits(mixed))
    rows = torch.arange(V) if V <= 1000 else torch.randperm(V, generator=gen)[:512]
    ref = _ref_rows(grad, E, H, f, h, t, rows.to(DEV))
    err = rel_fro(P[:, :d][rows.to(DEV)], ref)
    print(f'V={V} d={d} {dtype}: rel-fro {err:.2e}')
    assert err <= 1e-3, err
    assert torch.all(P[::7, :d] == 0)


# ---------------------------------------------------------------------------------------------- model
V_SMALL = 1000


class Block(nn.Module):
    """GPT-NeoX block: x + attn(ln1(x)) + mlp(ln2(x)), causal attention written with Linear layers."""

    def __init__(self, d, heads=4):
        super().__init__()
        self.ln1, self.ln2 = nn.LayerNorm(d), nn.LayerNorm(d)
        self.qkv, self.proj = nn.Linear(d, 3 * d), nn.Linear(d, d)
        self.fc, self.out = nn.Linear(d, 4 * d), nn.Linear(4 * d, d)
        self.heads = heads

    def forward(self, x):
        B, T, d = x.shape
        q, k, v = self.qkv(self.ln1(x)).view(B, T, 3, self.heads, d // self.heads).permute(2, 0, 3, 1, 4)
        a = nn.functional.scaled_dot_product_attention(q, k, v, is_causal=True).transpose(1, 2).reshape(B, T, d)
        return x + self.proj(a) + self.out(nn.functional.gelu(self.fc(self.ln2(x))))


class NanoGPT(nn.Module):
    def __init__(self, V=V_SMALL, d=64, tie=True):
        super().__init__()
        self.emb = nn.Embedding(V, d)
        self.pos = nn.Parameter(torch.randn(16, d) * 0.02)
        self.block = Block(d)
        self.ln = nn.LayerNorm(d)
        self.head = nn.Linear(d, V, bias=False)
        if tie:
            self.head.weight = self.emb.weight

    def forward(self, idx):
        return self.head(self.ln(self.block(self.emb(idx) + self.pos[:idx.shape[1]])))


def _batch(step, V, B=8, T=16):
    gen = torch.Generator().manual_seed(100 + step)
    idx = torch.randint(0, V, (B, T), generator=gen)
    idx[:, 0] = 3                                                    # one frequent token
    return idx.to(DEV), torch.randint(0, V, (B, T), generator=gen).to(DEV)


def _loss(model, idx, y):
    logits = model(idx)
    return nn.functional.cross_entropy(logits.flatten(0, 1).float(), y.flatten())


def _p_ref(grad, emb_layer, E, H, t):
    """fp64 P of the pair from the snapshots the layer holds and the factors of its last inverse step."""
    I = torch.eye(E.shape[0], dtype=torch.float64, device=DEV)
    f = emb_layer._inv['da'].double()
    h = emb_layer._inv['dh'].double()
    Eh, Hh = E.double() + t * I, H.double() + t * I
    out = []
    for chunk in torch.arange(grad.shape[0], device=DEV).split(500):
        F = (f[chunk] + t).view(-1, 1, 1) * Eh + (h[chunk] + t).view(-1, 1, 1) * Hh
        out.append(torch.linalg.solve(F, grad.double()[chunk].unsqueeze(-1)).squeeze(-1))
    return torch.cat(out)


SCHEDULES = {
    'int': dict(factor_update_steps=1, inv_update_steps=2, damping=0.003),
    'callable': dict(factor_update_steps=lambda s: 1 if s < 3 else 2, inv_update_steps=lambda s: 1 if s < 2 else 3,
                     damping=lambda s: 0.003 if s < 2 else 0.01),
}


@pytest.mark.parametrize('V', [V_SMALL, 10007])
@pytest.mark.parametrize('method', ['eigen', 'inverse'])
@pytest.mark.parametrize('schedule', ['int', 'callable'])
def test_model_tied_pair(V, method, schedule):
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(0)
    tied = NanoGPT(V).to(DEV)
    skip = copy.deepcopy(tied)
    kw = dict(kl_clip=None, compute_method=method, **SCHEDULES[schedule])
    pre = KFACPreconditioner(tied, **kw, **KW)
    ref = KFACPreconditioner(skip, skip_layers=['head'], **kw, **KW)
    emb = pre._layers[tied.emb][1]
    assert emb.tied_head is pre._layers[tied.head][1]
    worst = 0.0
    E = H = None
    for step in range(6):
        idx, y = _batch(step, V)
        for m in (tied, skip):
            m.zero_grad()
            _loss(m, idx, y).backward()
        g = tied.emb.weight.grad.clone()
        new_basis = pre.steps % pre.inv_update_steps == 0
        pre.step()
        ref.step()
        if new_basis:
            E, H = emb.g_factor.clone(), emb.tied_head.a_factor.clone()
        want = _p_ref(g, emb, E, H, emb._tied_damping)
        err = rel_fro(tied.emb.weight.grad, want)
        worst = max(worst, err)
        assert err <= 1e-3, (step, err)
        # every other gradient has the bits of the run with the head skipped
        for (n, p), (_, q) in zip(tied.named_parameters(), skip.named_parameters()):
            if n != 'emb.weight':
                assert torch.equal(bits(p.grad), bits(q.grad)), (step, n)
        # plain SGD on identical updates keeps the two models' other weights equal
        with torch.no_grad():
            for (n, p), (_, q) in zip(tied.named_parameters(), skip.named_parameters()):
                p -= 0.05 * p.grad
                q -= 0.05 * (p.grad if n == 'emb.weight' else q.grad)
    print(f'V={V} {method} {schedule}: worst rel-fro of the tied gradient {worst:.2e}')
    mem = pre.memory_usage()
    assert mem['g_inverses'] >= 4 * (2 * 64 * 64 + 64 + V)


def test_state_dict_round_trip():
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(1)
    model = NanoGPT().to(DEV)
    twin = copy.deepcopy(model)                                      # before hooks hold the preconditioner
    pre = KFACPreconditioner(model, kl_clip=None, **KW)
    for step in range(2):
        idx, y = _batch(step, V_SMALL)
        model.zero_grad()
        _loss(model, idx, y).backward()
        pre.step()
    sd = pre.state_dict()
    assert sd['layers']['emb']['A'].shape == (V_SMALL,) and sd['layers']['emb']['G'].shape == (64, 64)
    assert sd['layers']['head']['A'].shape == (64, 64) and sd['layers']['head']['G'].shape == (V_SMALL,)
    # the shapes of the untied members: a run with the head skipped and one with the embedding skipped
    for skip in ('head', 'emb'):
        other = KFACPreconditioner(NanoGPT().to(DEV), kl_clip=None, skip_layers=[skip], **KW)
        keep = 'emb' if skip == 'head' else 'head'
        layer = next(l for n, l in other._layers.values() if n == keep)
        assert layer.a_factor_shape == tuple(sd['layers'][keep]['A'].shape)
        assert layer.g_factor_shape == tuple(sd['layers'][keep]['G'].shape)
    pre2 = KFACPreconditioner(twin, kl_clip=None, **KW)
    pre2.load_state_dict(sd)
    pre._compute_inverses()
    e1, e2 = pre._layers[model.emb][1], pre2._layers[twin.emb][1]
    for key in ('tq', '_tqT', 'tmu', 'da', 'dh'):
        assert torch.equal(bits(e1._inv[key]), bits(e2._inv[key])), key
    idx, y = _batch(5, V_SMALL)
    for m, p in ((model, pre), (twin, pre2)):
        m.zero_grad()
        _loss(m, idx, y).backward()
    pre._inv_update_steps = pre2._inv_update_steps = 100            # no inverse step: the loaded data is used
    pre.step()
    pre2.step()
    assert torch.equal(bits(model.emb.weight.grad), bits(twin.emb.weight.grad))


def test_fp16_overflow_under_grad_scaler_and_no_host_sync():
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(2)
    model = NanoGPT().to(DEV)
    scaler = torch.amp.GradScaler('cuda', init_scale=2.0 ** 40)
    pre = KFACPreconditioner(model, grad_scaler=scaler, **KW)
    opt = torch.optim.SGD(model.parameters(), lr=0.01)
    for step in range(5):
        idx, y = _batch(step, V_SMALL)
        opt.zero_grad()
        if step >= 2:
            torch.cuda.set_sync_debug_mode('error')
        try:
            with torch.autocast('cuda', dtype=torch.float16):
                loss = _loss(model, idx, y)
            scaler.scale(loss).backward()
        finally:
            torch.cuda.set_sync_debug_mode(0)
        scaler.unscale_(opt)
        pre.step()
        scaler.step(opt)
        scaler.update(2.0 ** 10 if step == 0 else None)              # only the first step overflows
    torch.cuda.synchronize()
    assert pre.skipped_factor_updates >= 1
    emb = pre._layers[model.emb][1]
    for t in (emb.g_factor, emb.a_factor, emb.tied_head.a_factor, emb.tied_head.g_factor, emb._inv['tq'],
              emb._inv['tmu']):
        assert torch.all(torch.isfinite(t))
    assert torch.all(torch.isfinite(model.emb.weight))


def test_keyword_on_without_a_pair_gives_the_bits_of_the_keyword_off():
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(3)
    a = NanoGPT(tie=False).to(DEV)
    b = copy.deepcopy(a)
    pa = KFACPreconditioner(a, precondition_embeddings=True, diagonal_g_layers=['head'])
    pb = KFACPreconditioner(b, **KW)
    for step in range(3):
        idx, y = _batch(step, V_SMALL)
        for m, p in ((a, pa), (b, pb)):
            m.zero_grad()
            _loss(m, idx, y).backward()
            p.step()
        for p, q in zip(a.parameters(), b.parameters()):
            assert torch.equal(bits(p.grad), bits(q.grad))


# ---------------------------------------------------------------------------------------------- two ranks
def _run_dist(backend):
    import socket
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    script = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'dist_tied.py')
    out = subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node=2',
                          '--master-addr', '127.0.0.1', '--master-port', str(port), script, '--backend', backend],
                         capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, (out.stdout[-3000:], out.stderr[-3000:])
    assert out.stdout.count('dist_tied ok') == 2, out.stdout[-2000:]


def test_two_ranks_gloo():
    """Two ranks over gloo (they may share one GPU), COMM_OPT and MEM_OPT, eigen and inverse: the same gradients on
    both ranks."""
    _run_dist('gloo')


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='NCCL needs one GPU per rank')
def test_two_ranks_nccl():
    _run_dist('nccl')
