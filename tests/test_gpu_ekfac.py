"""EKFAC (compute_method='ekfac'): the row writers, kfac_ekfac_statistics and kfac_ekfac_update against fp64, the
preconditioner against an fp64 restatement of the method that uses the GPU's own eigenbases, and its behaviour.

Definition restated here (never in the product).  For a row r of a layer (a flattened Linear input row, or one
spatial position of a Conv2d im2col), x_r enters A (ones column appended, conv rows scaled by 1/S_sp) and g_r enters
G (conv rows scaled by 1/S_sp, AMP rows unscaled by 1/s).  With N rows,
    S_batch = (1/N) sum_r (Qg^T g_r x_r^T Qa)^2          (element-wise square of the projected per-row gradient)
    P       = Qg [ (Qg^T grad Qa) / (S + damping) ] Qa^T
S follows the schedule: EMA with factor_decay on factor steps, S_batch on inverse steps with a window, dg x da for a
new basis without one."""
import copy
import ctypes as C

import pytest
import torch

from conftest import rel_fro
from kfac_b200 import _cabi

DEV = torch.device('cuda:0')
gpu = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------- constructor (CPU)
def test_constructor_validation():
    from kfac_b200.enums import ComputeMethod, DistributedStrategy
    from kfac_b200.preconditioner import KFACPreconditioner as K
    from oracle.models import TinyModel
    assert ComputeMethod.EIGEN.value == 1 and ComputeMethod.INVERSE.value == 2 and ComputeMethod.EKFAC.value == 3
    p = K(TinyModel(), compute_method='ekfac')
    assert p.compute_method == ComputeMethod.EKFAC
    assert all(l.method == ComputeMethod.EKFAC for _, l in p._layers.values())
    # compute_eigenvalue_outer_product is ignored, colocate_factors keeps its rules
    K(TinyModel(), compute_method='ekfac', compute_eigenvalue_outer_product=True, colocate_factors=False)
    with pytest.raises(ValueError, match='COMM_OPT'):
        K(TinyModel(), compute_method='ekfac', grad_worker_fraction=DistributedStrategy.MEM_OPT)
    with pytest.raises(ValueError, match='COMM_OPT'):
        K(TinyModel(), compute_method=ComputeMethod.EKFAC, grad_worker_fraction=DistributedStrategy.HYBRID_OPT)
    with pytest.raises(ValueError, match='accumulation_steps'):
        K(TinyModel(), compute_method='ekfac', accumulation_steps=2)
    with pytest.raises(ValueError, match='multiple'):
        K(TinyModel(), compute_method='ekfac', factor_update_steps=2, inv_update_steps=3)
    # callables are accepted (an inverse step that is not a factor step seeds S with dg x da)
    K(TinyModel(), compute_method='ekfac', factor_update_steps=lambda s: 2, inv_update_steps=lambda s: 3)
    # no side effects on the other methods: the same arguments stay accepted there
    for method in ('eigen', 'inverse'):
        K(TinyModel(), compute_method=method, accumulation_steps=2, compute_eigenvalue_outer_product=False)
        K(TinyModel(), compute_method=method, grad_worker_fraction=DistributedStrategy.HYBRID_OPT,
          compute_eigenvalue_outer_product=False)
        with pytest.warns(UserWarning):
            K(TinyModel(), compute_method=method, factor_update_steps=2, inv_update_steps=3)


# ---------------------------------------------------------------------------------------------- kernels
def _ld4(n):
    return (n + 3) & ~3


def _rows_ref(x, conv=None, ones=False, scale=1.0):
    """fp64 rows of an input: conv = (kh, kw, sh, sw, ph, pw) -> F.unfold order (C, kh, kw)."""
    x = x.double()
    if conv is None:
        r = x.reshape(-1, x.size(-1))
    else:
        kh, kw, sh, sw, ph, pw = conv
        u = torch.nn.functional.unfold(x, (kh, kw), padding=(ph, pw), stride=(sh, sw))   # B, C*kh*kw, L
        r = u.transpose(1, 2).reshape(-1, u.size(1))
    if ones:
        r = torch.cat([r, r.new_ones(r.size(0), 1)], 1)
    return r * scale


def _padded(rows, d):
    """(N, ld4(d)) view of a flat row buffer, padding columns included."""
    return rows.view(-1, _ld4(d))


@gpu
@pytest.mark.parametrize('dtype', [torch.float32, torch.float16, torch.bfloat16])
@pytest.mark.parametrize('geo', [
    # (B, C, H, W, kh, kw, sh, sw, ph, pw, bias)
    (2, 3, 7, 7, 3, 3, 1, 1, 1, 1, True),
    (3, 5, 7, 7, 1, 1, 1, 1, 0, 0, False),       # 1x1 / stride 1 on a 7x7 map: the gather
    (2, 4, 9, 8, 3, 3, 2, 2, 1, 1, False),        # stride 2
    (2, 6, 8, 8, 1, 1, 2, 2, 0, 0, True),         # 1x1 stride 2 (downsample)
    (1, 3, 11, 13, 7, 7, 2, 2, 3, 3, False),      # 7x7 stem geometry
    (2, 64, 6, 6, 3, 3, 1, 1, 1, 1, True),        # d = 577
])
def test_rows_conv_against_unfold(geo, dtype):
    lib = _cabi.load()
    B, Cc, H, W, kh, kw, sh, sw, ph, pw, bias = geo
    torch.manual_seed(0)
    x = torch.randn(B, Cc, H, W, device=DEV).to(dtype)
    d = Cc * kh * kw + int(bias)
    Ho, Wo = (H + 2 * ph - kh) // sh + 1, (W + 2 * pw - kw) // sw + 1
    N = B * Ho * Wo
    out = torch.full((N * _ld4(d),), float('nan'), device=DEV)
    _cabi.check(lib.kfac_rows_conv2d_input(x.data_ptr(), _cabi.DTYPE_CODE[dtype], B, Cc, H, W, kh, kw, sh, sw, ph, pw,
                                           int(bias), 1.0 / (Ho * Wo), out.data_ptr(), _ld4(d), _cabi.stream_ptr()))
    want = _rows_ref(x.cpu(), (kh, kw, sh, sw, ph, pw), bias, 1.0 / (Ho * Wo))
    got = _padded(out, d).cpu().double()
    assert got[:, :d].sub(want).abs().max().item() <= 1e-7 * want.abs().max().item()
    assert not got[:, d:].any()
    # grad-output rows, divided by a device loss scale
    g = torch.randn(B, Cc, Ho, Wo, device=DEV).to(dtype)
    ls = torch.tensor([8.0], device=DEV)
    out = torch.full((N * _ld4(Cc),), float('nan'), device=DEV)
    _cabi.check(lib.kfac_rows_conv2d_gradout(g.data_ptr(), _cabi.DTYPE_CODE[dtype], B, Cc, Ho, Wo, 1.0 / (Ho * Wo),
                                             ls.data_ptr(), out.data_ptr(), _ld4(Cc), _cabi.stream_ptr()))
    want = g.cpu().double().permute(0, 2, 3, 1).reshape(-1, Cc) / (Ho * Wo) / 8.0
    got = _padded(out, Cc).cpu().double()
    assert got[:, :Cc].sub(want).abs().max().item() <= 1e-7 * want.abs().max().item()
    assert not got[:, Cc:].any()


@gpu
@pytest.mark.parametrize('dtype', [torch.float32, torch.float16, torch.bfloat16])
def test_rows_linear(dtype):
    lib = _cabi.load()
    torch.manual_seed(1)
    x = torch.randn(3, 5, 13, device=DEV).to(dtype)
    for ones, scale in ((1, 1.0), (0, 0.25)):
        d = 13 + ones
        out = torch.full((15 * _ld4(d),), float('nan'), device=DEV)
        _cabi.check(lib.kfac_rows_linear(x.data_ptr(), _cabi.DTYPE_CODE[dtype], 15, 13, ones, scale, None,
                                         out.data_ptr(), _ld4(d), _cabi.stream_ptr()))
        got = _padded(out, d).cpu().double()
        assert torch.equal(got[:, :d], _rows_ref(x.cpu(), None, bool(ones), scale))
        assert not got[:, d:].any()


def _eigbasis(d, seed):
    g = torch.Generator().manual_seed(seed)
    q, _ = torch.linalg.qr(torch.randn(d, d, generator=g, dtype=torch.float64))
    return q


def _stat_case(N, a, g, seed):
    gen = torch.Generator().manual_seed(seed)
    X = torch.randn(N, a, generator=gen, dtype=torch.float64)
    G = torch.randn(N, g, generator=gen, dtype=torch.float64) * 1e-3
    return dict(N=N, a=a, g=g, X=X, G=G, Qa=_eigbasis(a, seed + 1), Qg=_eigbasis(g, seed + 2))


def _dev_rows(t):
    n, d = t.shape
    out = torch.zeros(n, _ld4(d), device=DEV)
    out[:, :d] = t.float().to(DEV)
    return out


def _run_statistics(cases):
    lib = _cabi.load()
    items = (_cabi.EkfacStatItem * len(cases))()
    keep = []
    outs = []
    for i, c in enumerate(cases):
        X, G = _dev_rows(c['X']), _dev_rows(c['G'])
        qaT, qgT = _dev_rows(c['Qa'].T.contiguous()), _dev_rows(c['Qg'].T.contiguous())
        S = torch.full((c['g'], _ld4(c['a'])), float('nan'), device=DEV)
        keep += [X, G, qaT, qgT]
        outs.append(S)
        items[i] = _cabi.EkfacStatItem(X.data_ptr(), G.data_ptr(), qaT.data_ptr(), qgT.data_ptr(), S.data_ptr(),
                                       c['N'], c['a'], c['g'], _ld4(c['a']), _ld4(c['g']), _ld4(c['a']), _ld4(c['g']),
                                       _ld4(c['a']))
    need = lib.kfac_ekfac_statistics_workspace_bytes(items, len(cases))
    ws = torch.empty(need, dtype=torch.uint8, device=DEV)
    _cabi.check(lib.kfac_ekfac_statistics(items, len(cases), ws.data_ptr(), need, _cabi.stream_ptr()))
    torch.cuda.synchronize()
    return outs


@gpu
def test_statistics_against_fp64():
    """One call over tiny, SIMT-class, unaligned, wide and N >= 1e5 items (split chains on both engines)."""
    cases = [_stat_case(4, 10, 20, 0),              # tiny (SIMT)
             _stat_case(3000, 37, 50, 10),          # SIMT-class, unaligned a
             _stat_case(100_352, 20, 48, 20),       # SIMT-class with a long reduction (chunked)
             _stat_case(100_352, 65, 64, 30),       # tensor cores, N >= 1e5 (split into chains of 512 rows)
             _stat_case(2048, 1155, 130, 40),       # a > 1024: projection accumulated over column chunks, then squared
             _stat_case(777, 131, 97, 50)]          # unaligned N and a on the tensor cores
    outs = _run_statistics(cases)
    for c, S in zip(cases, outs):
        xh = c['X'] @ c['Qa']
        gh = c['G'] @ c['Qg']
        want = torch.einsum('ri,rj->ij', gh * gh, xh * xh) / c['N']
        got = S[:, :c['a']].cpu().double()
        e = rel_fro(got, want)
        assert e <= 1e-5, (c['N'], c['a'], c['g'], e)
        assert (got >= 0).all()
    # two calls give the same bits
    again = _run_statistics(cases)
    for S, T in zip(outs, again):
        assert torch.equal(S[:, :S.shape[1]].nan_to_num(0.0), T.nan_to_num(0.0))


def _update(items_spec, alpha, mode, damping, skipped=None):
    lib = _cabi.load()
    items = (_cabi.EkfacUpdateItem * len(items_spec))()
    for i, t in enumerate(items_spec):
        items[i] = _cabi.EkfacUpdateItem(t['S'].data_ptr(), t['Sb'].data_ptr(), t['dg'].data_ptr(), t['da'].data_ptr(),
                                         t['dgda'].data_ptr(), t['g'], t['a'], _ld4(t['a']),
                                         t['drop_a'].data_ptr() if t.get('drop_a') is not None else None,
                                         t['drop_g'].data_ptr() if t.get('drop_g') is not None else None)
    need = lib.kfac_ekfac_update_workspace_bytes(len(items_spec))
    ws = torch.empty(need, dtype=torch.uint8, device=DEV)
    _cabi.check(lib.kfac_ekfac_update(items, len(items_spec), alpha, mode, damping,
                                      skipped.data_ptr() if skipped is not None else None, ws.data_ptr(), need,
                                      _cabi.stream_ptr()))
    torch.cuda.synchronize()


def _update_items(seed):
    gen = torch.Generator().manual_seed(seed)
    out = []
    for g, a in ((3, 5), (64, 65), (130, 577)):
        S = torch.rand(g, _ld4(a), generator=gen)
        S[:, a:] = 0
        Sb = torch.rand(g, _ld4(a), generator=gen)
        Sb[:, a:] = 0
        out.append(dict(g=g, a=a, S=S.to(DEV), Sb=Sb.to(DEV), dg=torch.rand(g, generator=gen).to(DEV),
                        da=torch.rand(a, generator=gen).to(DEV),
                        dgda=torch.full((g, _ld4(a)), float('nan'), device=DEV)))
    return out


@gpu
def test_update_modes():
    lam, alpha = 0.003, 0.9
    K = _cabi
    for mode in (K.KFAC_EKFAC_KEEP, K.KFAC_EKFAC_EMA, K.KFAC_EKFAC_RESET, K.KFAC_EKFAC_SEED):
        items = _update_items(mode)
        S0 = [t['S'].double().cpu() for t in items]
        _update(items, alpha, mode, lam)
        for t, s0 in zip(items, S0):
            a = t['a']
            Sb, dg, da = t['Sb'].double().cpu(), t['dg'].double().cpu(), t['da'].double().cpu()
            want = {K.KFAC_EKFAC_KEEP: s0, K.KFAC_EKFAC_EMA: alpha * s0 + (1 - alpha) * Sb,
                    K.KFAC_EKFAC_RESET: Sb}.get(mode)
            if want is None:
                want = torch.outer(dg, da)
            want = want[:, :a]
            assert rel_fro(t['S'][:, :a], want) < 1e-6, mode
            assert rel_fro(t['dgda'][:, :a], 1.0 / (want + lam)) < 1e-6, mode
            assert not t['dgda'][:, a:].any()
        if mode == K.KFAC_EKFAC_SEED:
            # the bits kfac_dgda gives: the eigen method's dgda for S = dg x da
            for t in items:
                ref = torch.empty_like(t['dgda'])
                _cabi.check(_cabi.load().kfac_dgda(t['dg'].data_ptr(), t['da'].data_ptr(), t['g'], t['a'], lam,
                                                   ref.data_ptr(), _ld4(t['a']), _cabi.stream_ptr()))
                torch.cuda.synchronize()
                assert torch.equal(ref, t['dgda'])


@gpu
def test_update_drops_bad_windows():
    K = _cabi
    lam = 0.01
    for mode in (K.KFAC_EKFAC_EMA, K.KFAC_EKFAC_RESET):
        items = _update_items(7)
        items[0]['Sb'][1, 2] = float('inf')                      # a non-finite S_batch entry
        items[1]['Sb'][3, 4] = 2e15                              # over range
        items[2]['drop_g'] = torch.ones(1, dtype=torch.int32, device=DEV)   # a G window the guarded EMA dropped
        keep = _update_items(7)[2]
        keep['S'], keep['Sb'] = items[2]['S'].clone(), items[2]['Sb'].clone()
        keep['drop_a'] = torch.zeros(1, dtype=torch.int32, device=DEV)
        S0 = [t['S'].clone() for t in items]
        skipped = torch.zeros(1, dtype=torch.int64, device=DEV)
        _update(items + [keep], 0.5, mode, lam, skipped)
        assert skipped.item() == 2, mode    # items 0 and 1 (S_batch alone); item 2 was counted by the guarded EMA
        for t, s0 in zip(items, S0):
            a = t['a']
            want = s0 if mode == K.KFAC_EKFAC_EMA else torch.outer(t['dg'], t['da'])   # reset falls back to the seed
            assert torch.equal(t['S'][:, :a], want[:, :a]), mode
            assert torch.isfinite(t['dgda']).all()
        assert not torch.equal(keep['S'], items[2]['S'])        # an unflagged item is updated


# ---------------------------------------------------------------------------------------------- module level
class _Rec:
    """Records every layer's inputs and grad-outputs of the current step (hooks registered after the
    preconditioner's, on the same modules)."""

    def __init__(self, pre):
        self.inp, self.gout = {}, {}
        for m in pre._layers:
            m.register_forward_pre_hook(lambda mod, i: self.inp.__setitem__(mod, i[0].detach().clone()))
            m.register_full_backward_hook(lambda mod, gi, go: self.gout.__setitem__(mod, go[0].detach().clone()))

    def clear(self):
        self.inp, self.gout = {}, {}


def _layer_rows(module, x, gout, grad_scale=1.0):
    """fp64 (x_r, g_r) of one layer (the definition above)."""
    if isinstance(module, torch.nn.Conv2d):
        Ho, Wo = gout.shape[2], gout.shape[3]
        X = _rows_ref(x.cpu(), (module.kernel_size[0], module.kernel_size[1], module.stride[0], module.stride[1],
                                module.padding[0], module.padding[1]), module.bias is not None, 1.0 / (Ho * Wo))
        G = gout.cpu().double().permute(0, 2, 3, 1).reshape(-1, gout.shape[1]) / (Ho * Wo)
    else:
        X = _rows_ref(x.cpu(), None, module.bias is not None)
        G = gout.cpu().double().reshape(-1, gout.shape[-1])
    return X, G / grad_scale


def _s_batch_per_row(X, G, Qa, Qg):
    """(1/N) sum_r (Qg^T g_r x_r^T Qa)^2, by explicit per-row outer products (chunked)."""
    acc = torch.zeros(Qg.shape[0], Qa.shape[0], dtype=torch.float64)
    for r0 in range(0, X.shape[0], 256):
        per_row = torch.einsum('ri,rj->rij', G[r0:r0 + 256], X[r0:r0 + 256])     # g_r x_r^T
        acc += ((Qg.T @ per_row @ Qa) ** 2).sum(0)
    return acc / X.shape[0]


class _Oracle:
    """fp64 EKFAC state per layer, driven by the GPU's own bases."""

    def __init__(self):
        self.S = {}

    def step(self, pre, rec, factor_step, inverse_step, alpha, damping, grads):
        out = {}
        for m, (name, layer) in pre._layers.items():
            Qa, Qg = layer.qa.double().cpu(), layer.qg.double().cpu()
            if factor_step:
                X, G = _layer_rows(m, rec.inp[m], rec.gout[m])
                Sb = _s_batch_per_row(X, G, Qa, Qg)
                self.S[name] = Sb if inverse_step else alpha * self.S[name] + (1 - alpha) * Sb
            elif inverse_step:
                self.S[name] = torch.outer(layer.dg.double().cpu(), layer.da.double().cpu())
            gr = grads[name]
            out[name] = Qg @ ((Qg.T @ gr @ Qa) / (self.S[name] + damping)) @ Qa.T
        return out


def _grad_matrix(module):
    g = module.weight.grad.reshape(module.weight.grad.size(0), -1)
    if module.bias is not None:
        g = torch.cat([g, module.bias.grad.view(-1, 1)], 1)
    return g.detach().double().cpu()


def _run_module(model, make_batch, loss_fn, steps, fus=1, ius=1, damping=0.003, alpha=0.95):
    """fus / ius: ints or callables of the step, as the preconditioner takes them."""
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    pre = KFACPreconditioner(model, compute_method='ekfac', factor_update_steps=fus, inv_update_steps=ius,
                             damping=damping, factor_decay=alpha, kl_clip=None)
    rec = _Rec(pre)
    oracle = _Oracle()
    opt = torch.optim.SGD(model.parameters(), lr=0.01)
    worst = 0.0
    for s in range(steps):
        rec.clear()
        opt.zero_grad()
        x, y = make_batch(s)
        loss_fn(model(x), y).backward()
        grads = {name: _grad_matrix(m) for m, (name, _) in pre._layers.items()}
        pre.step()
        torch.cuda.synchronize()
        f, i = (fus(s) if callable(fus) else fus), (ius(s) if callable(ius) else ius)
        want = oracle.step(pre, rec, s % f == 0, s % i == 0, alpha, damping, grads)
        for m, (name, layer) in pre._layers.items():
            assert rel_fro(layer._S[:, :layer.a_dim], oracle.S[name]) < 1e-4, (s, name)
            # kl_clip=None: the gradient written back is P itself
            e = rel_fro(_grad_matrix(m), want[name])
            worst = max(worst, e)
            assert e < 1e-3, (s, name, e)
        opt.step()
    return pre, worst


@gpu
def test_tiny_model_against_fp64():
    from oracle.models import TinyModel
    torch.manual_seed(0)
    gen = torch.Generator().manual_seed(1)
    data = [(torch.rand(8, 10, generator=gen).to(DEV), torch.rand(8, 10, generator=gen).to(DEV)) for _ in range(4)]
    _run_module(TinyModel().to(DEV), lambda s: data[s % 4], torch.nn.MSELoss(reduction='sum'), steps=4)


@gpu
def test_schedule_ema_reset_seed():
    """factor_update_steps=2, inv_update_steps=4 over 9 steps: reset (0, 4, 8), EMA (2, 6), the stored S (odd)."""
    from oracle.models import TinyModel
    torch.manual_seed(0)
    gen = torch.Generator().manual_seed(2)
    data = [(torch.rand(8, 10, generator=gen).to(DEV), torch.rand(8, 10, generator=gen).to(DEV)) for _ in range(9)]
    _run_module(TinyModel().to(DEV), lambda s: data[s], torch.nn.MSELoss(reduction='sum'), steps=9, fus=2, ius=4,
                alpha=0.8)


@gpu
def test_callable_schedule_seeds_in_step():
    """Callables: factor steps 0, 2, 4, 6, inverse steps 0, 3, 6.  Step 3 is an inverse step without a window, so
    step() seeds S with dg x da of the new bases; steps 2 and 4 are EMA steps, 0 and 6 resets."""
    from oracle.models import TinyModel
    torch.manual_seed(0)
    gen = torch.Generator().manual_seed(8)
    data = [(torch.rand(8, 10, generator=gen).to(DEV), torch.rand(8, 10, generator=gen).to(DEV)) for _ in range(7)]
    _run_module(TinyModel().to(DEV), lambda s: data[s], torch.nn.MSELoss(reduction='sum'), steps=7,
                fus=lambda s: 2, ius=lambda s: 3, alpha=0.8)


@gpu
def test_sequence_linear_stack_against_fp64():
    class Seq(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.l1 = torch.nn.Linear(24, 130)
            self.l2 = torch.nn.Linear(130, 70, bias=False)
            self.l3 = torch.nn.Linear(70, 5)

        def forward(self, x):
            return self.l3(torch.tanh(self.l2(torch.tanh(self.l1(x))))).mean(1)
    torch.manual_seed(3)
    gen = torch.Generator().manual_seed(3)
    data = [(torch.randn(6, 40, 24, generator=gen).to(DEV), torch.randint(0, 5, (6,), generator=gen).to(DEV))
            for _ in range(3)]
    _run_module(Seq().to(DEV), lambda s: data[s], torch.nn.CrossEntropyLoss(), steps=3)


@gpu
def test_conv_stack_against_fp64():
    """ResNet-32-like: 3x3 convs with stride 2, 1x1 shortcuts, BatchNorm, a Linear head."""
    from oracle.models import resnet32
    torch.manual_seed(4)
    gen = torch.Generator().manual_seed(4)
    data = [(torch.randn(8, 3, 32, 32, generator=gen).to(DEV), torch.randint(0, 10, (8,), generator=gen).to(DEV))
            for _ in range(2)]
    _run_module(resnet32().to(DEV), lambda s: data[s], torch.nn.CrossEntropyLoss(), steps=2)


# ---------------------------------------------------------------------------------------------- behaviour
@gpu
def test_second_forward_in_a_window_raises():
    from kfac_b200.preconditioner import KFACPreconditioner
    from oracle.models import TinyModel
    m = TinyModel().to(DEV)
    KFACPreconditioner(m, compute_method='ekfac')
    x = torch.rand(4, 10, device=DEV)
    m(x)
    with pytest.raises(RuntimeError, match='second time'):
        m(x)


@gpu
def test_first_step_after_load_equals_eigen():
    """After load_state_dict, S = dg x da: the first P is the eigen method's P."""
    from kfac_b200.preconditioner import KFACPreconditioner
    from oracle.models import TinyModel
    torch.manual_seed(5)
    m = TinyModel().to(DEV)
    kw = dict(factor_update_steps=2, inv_update_steps=4, damping=0.003)
    p = KFACPreconditioner(m, compute_method='ekfac', **kw)
    x, y = torch.rand(8, 10, device=DEV), torch.rand(8, 10, device=DEV)
    crit = torch.nn.MSELoss(reduction='sum')
    for _ in range(3):
        m.zero_grad()
        crit(m(x), y).backward()
        p.step()
    sd = p.state_dict()
    assert set(sd['layers']['linear1']) == {'A', 'G'}          # the reference's schema: no S
    outs = []
    for method in ('ekfac', 'eigen'):
        m2 = TinyModel().to(DEV)
        m2.load_state_dict(m.state_dict())
        p2 = KFACPreconditioner(m2, compute_method=method, **kw)
        m2.zero_grad()
        crit(m2(x), y).backward()           # a window is open when the state is loaded: EKFAC discards its rows
        p2.load_state_dict(sd)
        if method == 'ekfac':
            for _, l in p2._layers.values():
                assert l._rows_n_a == 0 and l._rows_n_g == 0
                assert torch.equal(l._S[:, :l.a_dim], torch.outer(l.dg, l.da))
        m2.zero_grad()
        crit(m2(x), y).backward()           # step 3: neither a factor nor an inverse step
        p2.step()
        torch.cuda.synchronize()
        outs.append({n: l._p_view.clone() for n, l in p2._layers.values()})
    # the seed gives the eigen method's dgda bit for bit; this step refreshes it as 1 / (S + damping) from the
    # stored S = dg x da, which may differ in the last bit
    for n in outs[0]:
        assert rel_fro(outs[0][n], outs[1][n]) < 1e-6, n


@gpu
def test_training_loss_decreases():
    from kfac_b200.preconditioner import KFACPreconditioner
    from oracle.models import TinyModel
    torch.manual_seed(42)
    m = TinyModel().to(DEV)
    opt = torch.optim.SGD(m.parameters(), lr=0.001)
    p = KFACPreconditioner(m, lr=0.001, compute_method='ekfac')
    x, y = torch.rand(4, 10, device=DEV), torch.rand(4, 10, device=DEV)
    crit = torch.nn.MSELoss(reduction='sum')
    losses = []
    for _ in range(20):
        opt.zero_grad()
        loss = crit(m(x), y)
        loss.backward()
        p.step()
        opt.step()
        losses.append(loss.item())
    assert losses[0] > losses[-1]
    mem = p.memory_usage()
    assert mem['ekfac'] > 0 and mem['total'] >= mem['ekfac']


@gpu
def test_grad_scaler_overflow_leaves_S_unchanged():
    """fp16 autocast with a GradScaler: an overflow window on a factor step that is not an inverse step keeps S and
    is counted once per dropped factor window; the G rows are unscaled by the device loss scale."""
    from kfac_b200.preconditioner import KFACPreconditioner

    class Net(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.l1 = torch.nn.Linear(16, 64)
            self.l2 = torch.nn.Linear(64, 8)

        def forward(self, x):
            return self.l2(torch.relu(self.l1(x)))
    torch.manual_seed(6)
    model = Net().to(DEV)
    scaler = torch.amp.GradScaler('cuda', init_scale=2.0 ** 10, growth_interval=10 ** 9)
    pre = KFACPreconditioner(model, grad_scaler=scaler, compute_method='ekfac', inv_update_steps=4, damping=0.003)
    opt = torch.optim.SGD(model.parameters(), lr=0.01)
    finite = {}
    for m in pre._layers:
        m.register_full_backward_hook(lambda mod, gi, go: finite.__setitem__(mod, bool(torch.isfinite(go[0]).all())))
    gen = torch.Generator().manual_seed(6)
    for step in range(4):
        x = torch.randn(32, 16, generator=gen).to(DEV)
        y = torch.randint(0, 8, (32,), generator=gen).to(DEV)
        opt.zero_grad()
        if step == 2:
            scaler.update(new_scale=2.0 ** 60)
            before = {n: l._S.clone() for n, l in pre._layers.values()}
            skipped = pre.skipped_factor_updates
        with torch.autocast('cuda', dtype=torch.float16):
            loss = torch.nn.functional.cross_entropy(model(x), y)
        scaler.scale(loss).backward()
        scaler.unscale_(opt)
        pre.step()
        torch.cuda.synchronize()
        if step == 2:
            bad = [m for m in pre._layers if not finite[m]]
            assert bad, 'the injected loss scale did not overflow fp16'
            for m, (n, l) in pre._layers.items():
                if m in bad:
                    assert torch.equal(l._S, before[n]), n
                assert torch.isfinite(l._S).all() and torch.isfinite(l.dgda).all()
            assert pre.skipped_factor_updates - skipped == len(bad)
        scaler.step(opt)
        scaler.update(new_scale=2.0 ** 10) if step == 2 else scaler.update()
    for _, l in pre._layers.values():
        assert torch.isfinite(l._S).all()


@gpu
def test_guarded_ema_drop_flags_reach_their_layer():
    """With a grad_scaler, the G window of l1 is dropped by the guarded EMA for an over-range entry (|g| ~ 1e8, so
    G ~ 1e16 > 1e15) while its S_batch stays finite (its inputs are ~ 1e-12): S of l1 is kept because of the EMA's drop
    flag alone.  l2's window in the same step is kept, and the drop is counted once."""
    from kfac_b200.preconditioner import KFACPreconditioner

    class Two(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.l1 = torch.nn.Linear(16, 8, bias=False)
            self.l2 = torch.nn.Linear(16, 8, bias=False)

        def forward(self, x1, x2):
            return self.l1(x1), self.l2(x2)
    torch.manual_seed(9)
    model = Two().to(DEV)
    scaler = torch.amp.GradScaler('cuda', init_scale=1.0, growth_interval=10 ** 9)
    pre = KFACPreconditioner(model, grad_scaler=scaler, compute_method='ekfac', inv_update_steps=4, damping=0.003)
    opt = torch.optim.SGD(model.parameters(), lr=0.01)
    gen = torch.Generator().manual_seed(9)
    l1, l2 = pre._layers[model.l1][1], pre._layers[model.l2][1]
    for step, c in enumerate((1.0, 1e8)):
        x1 = (torch.randn(32, 16, generator=gen) * 1e-12).to(DEV)
        x2 = torch.randn(32, 16, generator=gen).to(DEV)
        t1, t2 = torch.randn(32, 8, generator=gen).to(DEV), torch.randn(32, 8, generator=gen).to(DEV)
        if step == 1:
            before = (l1._S.clone(), l2._S.clone(), pre.skipped_factor_updates)
        opt.zero_grad()
        o1, o2 = model(x1, x2)
        scaler.scale(c * (o1 * t1).sum() + (o2 * t2).sum()).backward()
        scaler.unscale_(opt)
        pre.step()
        scaler.step(opt)
        scaler.update()
    torch.cuda.synchronize()
    assert torch.isfinite(l1._S_batch).all() and l1._S_batch.abs().max() <= 1e15   # the scan would keep this window
    assert torch.equal(l1._S, before[0])
    assert not torch.equal(l2._S, before[1])
    assert pre.skipped_factor_updates - before[2] == 1


@gpu
def test_grad_scaler_rows_are_unscaled():
    """fp32 with a GradScaler at 2^10 gives the S of the same run without a loss scale (the G rows are divided by the
    scale read on the device; a power of two changes no bits)."""
    from kfac_b200.preconditioner import KFACPreconditioner
    from oracle.models import TinyModel
    torch.manual_seed(7)
    base = TinyModel().to(DEV)
    x, y = torch.rand(8, 10, device=DEV), torch.rand(8, 10, device=DEV)
    S = []
    for use_scaler in (False, True):
        m = copy.deepcopy(base)
        scaler = torch.amp.GradScaler('cuda', init_scale=2.0 ** 10, growth_interval=10 ** 9) if use_scaler else None
        p = KFACPreconditioner(m, compute_method='ekfac', grad_scaler=scaler, factor_update_steps=1,
                               inv_update_steps=2)
        opt = torch.optim.SGD(m.parameters(), lr=0.01)
        for _ in range(3):
            opt.zero_grad()
            loss = torch.nn.functional.mse_loss(m(x), y, reduction='sum')
            if scaler is None:
                loss.backward()
                p.step()
                opt.step()
            else:
                scaler.scale(loss).backward()
                scaler.unscale_(opt)
                p.step()
                scaler.step(opt)
                scaler.update()
        torch.cuda.synchronize()
        S.append([l._S.clone() for _, l in p._layers.values()])
    for a, b in zip(*S):
        assert rel_fro(b, a) < 1e-6


@gpu
def test_eigen_method_has_no_ekfac_state():
    """The eigen method never allocates or touches EKFAC state."""
    from kfac_b200.preconditioner import KFACPreconditioner
    from oracle.models import TinyModel
    m = TinyModel().to(DEV)
    p = KFACPreconditioner(m)
    m(torch.rand(4, 10, device=DEV)).sum().backward()
    p.step()
    assert not hasattr(p, '_s_arena') and 'ekfac' not in p.memory_usage()
    assert all(l._rows_x is None and l._S is None for _, l in p._layers.values())


def _run_dist(backend):
    import os
    import socket
    import subprocess
    import sys
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    script = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'dist_ekfac.py')
    out = subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node=2',
                          '--master-addr', '127.0.0.1', '--master-port', str(port), script, '--backend', backend],
                         capture_output=True, text=True, timeout=600)
    print(out.stdout[-3000:])
    assert out.returncode == 0 and 'DIST EKFAC OK' in out.stdout, (out.stdout[-3000:], out.stderr[-3000:])


@gpu
def test_multi_gpu_ranks_agree():
    """tests/dist_ekfac.py on two GPUs (NCCL): identical S and P on every rank, both against fp64 on the concatenated
    rows of the two shards over an EMA / reset schedule."""
    if torch.cuda.device_count() < 2:
        pytest.skip('needs >= 2 GPUs')
    _run_dist('nccl')


@gpu
def test_two_ranks_gloo():
    """The same check with two ranks over gloo (they may share one GPU): the all-reduce of S_batch and the
    broadcast of the bases through the preconditioner's communicator."""
    _run_dist('gloo')
