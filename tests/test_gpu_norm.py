"""Normalization layers (`precondition_norms=True`) on the GPU, everything against fp64:

  * kfac_factor_norm for BatchNorm2d (56 x 56, 7 x 7 and 1 x 1 maps, odd C), BatchNorm1d on 2-D and 3-D inputs,
    LayerNorm with 1-D and 2-D normalized_shape, with and without bias, RMSNorm with eps set and eps=None; x and g
    each in fp32/fp16/bf16, inputs centred and with |mean| = 100 std: relative Frobenius error <= 1e-5 and the same
    bits on a repeat (fp64 is formed from the same rounded inputs);
  * kfac_norm_precondition against an fp64 2 x 2 (1 x 1) solve, many items in one launch;
  * a small CNN (BatchNorm2d / BatchNorm1d) and a NeoX-style block (LayerNorm / RMSNorm) for 5 steps under EIGEN,
    INVERSE and EKFAC, with callable schedules and with accumulation_steps=2: the written norm gradients against an
    fp64 restatement from the captured inputs and output gradients;
  * with the keyword off and on (kl-clip off) every other layer's factors, second-order data, P and written gradient
    are bit-identical, and the norm gradients are untouched when off; with kl-clip on the written gradients are
    nu * P with nu over all layers;
  * eval(), a module called twice in a window, torch.utils.checkpoint, an fp16 GradScaler overflow, a non-finite
    block without a grad_scaler, a state_dict round trip, memory_usage(), and two ranks (tests/dist_norm.py).
"""
import copy
import os
import subprocess
import sys
import zlib

import pytest
import torch
from torch import nn
from torch.utils.checkpoint import checkpoint

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


def bits(x):
    return x.contiguous().view(torch.int32 if x.element_size() == 4 else torch.int16)


# ---------------------------------------------------------------------------------------------- fp64 restatement
def ref_blocks(module, x, g, k):
    """(C, k) fp64 block of one call of `module` (the scaled sums the statistics kernel adds)."""
    x, g = x.double(), g.double()
    if isinstance(module, (nn.BatchNorm1d, nn.BatchNorm2d)):
        B, C = x.shape[:2]
        xv, gv = x.reshape(B, C, -1), g.reshape(B, C, -1)
        Sp = xv.shape[2]
        mu = xv.mean((0, 2), keepdim=True)
        var = xv.var((0, 2), unbiased=False, keepdim=True)
        xh = (xv - mu) / torch.sqrt(var + module.eps)
        scale, dims = 1.0 / (B * Sp * float(Sp) ** 4), (0, 2)
    else:
        D = module.weight.numel()
        xv, gv = x.reshape(-1, D), g.reshape(-1, D)
        if isinstance(module, nn.LayerNorm):
            xh = (xv - xv.mean(1, keepdim=True)) / torch.sqrt(xv.var(1, unbiased=False, keepdim=True) + module.eps)
        else:
            # torch's eps=None: the machine epsilon of the computation type (float32 for fp16 / bf16 / fp32)
            eps = torch.finfo(torch.float32).eps if module.eps is None else module.eps
            xh = xv / torch.sqrt((xv * xv).mean(1, keepdim=True) + eps)
        scale, dims = 1.0 / xv.shape[0], (0,)
    g2 = gv * gv
    ss = (g2 * xh * xh).sum(dims)
    if k == 1:
        return (ss * scale)[:, None]
    return torch.stack([ss, (g2 * xh).sum(dims), g2.sum(dims)], 1) * scale


def ref_solve(F, grad, damping):
    """P = (F + damping I)^-1 grad per channel; F (C, k), grad (C, np)."""
    F, grad = F.double(), grad.double()
    if F.shape[1] == 1:
        return grad / (F + damping)
    M = torch.stack([torch.stack([F[:, 0] + damping, F[:, 1]], 1), torch.stack([F[:, 1], F[:, 2] + damping], 1)], 1)
    return torch.linalg.solve(M, grad.unsqueeze(2)).squeeze(2)


# ---------------------------------------------------------------------------------------------- statistics kernel
CASES = {
    'bn2d_56': (lambda: nn.BatchNorm2d(7), (4, 7, 56, 56)),
    'bn2d_7': (lambda: nn.BatchNorm2d(33, eps=1e-3), (16, 33, 7, 7)),
    'bn2d_1': (lambda: nn.BatchNorm2d(65), (32, 65, 1, 1)),
    'bn1d_2d': (lambda: nn.BatchNorm1d(129), (64, 129)),
    'bn1d_3d': (lambda: nn.BatchNorm1d(17), (8, 17, 100)),
    'ln_1d': (lambda: nn.LayerNorm(768), (3, 100, 768)),
    'ln_2d': (lambda: nn.LayerNorm((6, 7)), (5, 11, 6, 7)),
    'ln_nobias': (lambda: nn.LayerNorm(257, bias=False), (300, 257)),
    'rms_eps': (lambda: nn.RMSNorm(96, eps=1e-5), (7, 50, 96)),
    'rms_none': (lambda: nn.RMSNorm(64), (123, 64)),
}


def _stats(lib, helper, x, g, live, eps):
    from kfac_b200 import _cabi
    acc = live.clone()
    C = helper.channels
    if helper.kind == _cabi.KFAC_NORM_BATCH:
        rows, Sp = x.shape[0], x.numel() // (x.shape[0] * C)
        scale = 1.0 / (rows * float(Sp) ** 5)
    else:
        rows, Sp = x.numel() // C, 1
        scale = 1.0 / rows
    need = lib.kfac_factor_norm_workspace_bytes(helper.kind, rows, C, Sp)
    ws = torch.full((need,), 255, dtype=torch.uint8, device=DEV)
    rc = lib.kfac_factor_norm(x.data_ptr(), _cabi.DTYPE_CODE[x.dtype], g.data_ptr(), _cabi.DTYPE_CODE[g.dtype],
                              helper.kind, rows, C, Sp, helper.k, eps, scale, acc.data_ptr(), ws.data_ptr(), need, S())
    assert rc == 0, lib.kfac_last_error()
    assert lib.kfac_factor_norm(x.data_ptr(), _cabi.DTYPE_CODE[x.dtype], g.data_ptr(), _cabi.DTYPE_CODE[g.dtype],
                                helper.kind, rows, C, Sp, helper.k, eps, scale, acc.data_ptr(), ws.data_ptr(), need - 8,
                                S()) != 0
    torch.cuda.synchronize()
    return acc


@pytest.mark.parametrize('offset', [0.0, 100.0])
@pytest.mark.parametrize('g_dtype', DTYPES)
@pytest.mark.parametrize('x_dtype', DTYPES)
@pytest.mark.parametrize('case', list(CASES))
def test_factor_norm_against_fp64(lib, case, x_dtype, g_dtype, offset):
    from kfac_b200.layers import NormModuleHelper
    make, shape = CASES[case]
    module = make().to(DEV)
    helper = NormModuleHelper(module)
    gen = torch.Generator(device=DEV).manual_seed(zlib.crc32(f'{case}/{offset}'.encode()))
    C = helper.channels
    # per-channel (BatchNorm) or per-row (LayerNorm / RMSNorm) scales and means, std 1 .. 3
    x = torch.randn(shape, device=DEV, generator=gen) * (1 + 2 * torch.rand(shape, device=DEV, generator=gen)) + offset
    x = x.to(x_dtype)
    g = torch.randn(shape, device=DEV, generator=gen).to(g_dtype)
    ref = ref_blocks(module, x, g, helper.k)
    acc = _stats(lib, helper, x, g, torch.zeros(C, helper.k, device=DEV), helper.eps_for(x))
    err = rel_fro(acc, ref)
    assert err <= 1e-5, err
    # accumulated into a batch buffer that already holds a window of the same magnitude
    live = torch.rand(C, helper.k, device=DEV, generator=gen) * float(ref.abs().max())
    acc = _stats(lib, helper, x, g, live, helper.eps_for(x))
    assert rel_fro(acc, live.double() + ref) <= 1e-5
    assert torch.equal(bits(acc), bits(_stats(lib, helper, x, g, live, helper.eps_for(x))))


@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('case', ['rms_none', 'rms_eps', 'ln_1d', 'bn2d_7', 'bn1d_2d'])
def test_xhat_is_the_modules_own_normalization(lib, case, dtype):
    """With weight 1 and bias 0 the module's forward output is x-hat itself, so the block formed by the kernel must be
    the one of module(x) -- computed here from the module's output, not from a restated formula.  Small activations
    (rms 0.02, the scale of an embedding output) make the eps of RMSNorm(eps=None) matter: torch uses the float32
    machine epsilon for fp16 / bf16 inputs, not the input dtype's."""
    from kfac_b200.layers import NormModuleHelper
    make, shape = CASES[case]
    module = make().to(DEV).to(dtype).train()
    with torch.no_grad():
        module.weight.fill_(1.0)
        if getattr(module, 'bias', None) is not None:
            module.bias.zero_()
    helper = NormModuleHelper(module)
    gen = torch.Generator(device=DEV).manual_seed(zlib.crc32(f'xhat/{case}'.encode()))
    x = (torch.randn(shape, device=DEV, generator=gen) * 0.02).to(dtype)
    g = torch.randn(shape, device=DEV, generator=gen).to(dtype)
    with torch.no_grad():
        xh = module(x).double()            # rounded to `dtype` by the module
    acc = _stats(lib, helper, x, g, torch.zeros(helper.channels, helper.k, device=DEV), helper.eps_for(x))
    C, gd = helper.channels, g.double()
    if isinstance(module, (nn.BatchNorm1d, nn.BatchNorm2d)):
        B = shape[0]
        xv, gv = xh.reshape(B, C, -1), gd.reshape(B, C, -1)
        Sp = xv.shape[2]
        scale, dims = 1.0 / (B * Sp * float(Sp) ** 4), (0, 2)
    else:
        xv, gv = xh.reshape(-1, C), gd.reshape(-1, C)
        scale, dims = 1.0 / xv.shape[0], (0,)
    g2 = gv * gv
    ref = [(g2 * xv * xv).sum(dims) * scale]
    if helper.k == 3:
        ref += [(g2 * xv).sum(dims) * scale, g2.sum(dims) * scale]
    ref = torch.stack(ref, 1)
    # the module's output carries the rounding of `dtype` (2^-8 relative for bf16)
    tol = {torch.float32: 1e-5, torch.float16: 2e-3, torch.bfloat16: 1e-2}[dtype]
    assert rel_fro(acc, ref) <= tol, rel_fro(acc, ref)


def test_factor_norm_rejects_bad_arguments(lib):
    from kfac_b200 import _cabi
    x = torch.zeros(4, 8, device=DEV)
    acc = torch.zeros(8, 3, device=DEV)
    ws = torch.zeros(1 << 16, dtype=torch.uint8, device=DEV)
    args = dict(kind=_cabi.KFAC_NORM_LAYER, rows=4, C=8, S=1, k=3)

    def call(**kw):
        a = {**args, **kw}
        return lib.kfac_factor_norm(x.data_ptr(), 0, x.data_ptr(), 0, a['kind'], a['rows'], a['C'], a['S'], a['k'],
                                    1e-5, 1.0, acc.data_ptr(), ws.data_ptr(), ws.numel(), S())
    assert call() == 0
    assert call(k=2) != 0
    assert call(kind=_cabi.KFAC_NORM_RMS) != 0         # RMSNorm has no bias
    assert call(S=2) != 0                              # LayerNorm rows are not spatial
    assert call(kind=7) != 0


# ---------------------------------------------------------------------------------------------- precondition
def test_norm_precondition_against_fp64(lib):
    from kfac_b200 import _cabi
    gen = torch.Generator(device=DEV).manual_seed(3)
    damping = 1e-3
    specs = [(7, 3, torch.float32), (1000, 1, torch.float16), (65, 3, torch.bfloat16), (33, 1, torch.float32),
             (4097, 3, torch.float16)] * 3
    keep, items = [], (_cabi.NormItem * len(specs))()
    for i, (C, k, dtype) in enumerate(specs):
        if k == 3:
            a, b = torch.rand(C, device=DEV, generator=gen), torch.randn(C, device=DEV, generator=gen)
            c = torch.rand(C, device=DEV, generator=gen)
            F = torch.stack([a * a + 1e-4, a * b, b * b + c * 1e-2], 1) * 10 ** (4 * torch.rand(C, 1, device=DEV,
                                                                                              generator=gen) - 4)
        else:
            F = torch.rand(C, 1, device=DEV, generator=gen) ** 3
        w = torch.randn(C, device=DEV, generator=gen).to(dtype)
        b = torch.randn(C, device=DEV, generator=gen).to(dtype) if k == 3 else None
        P = torch.full((C, 2 if k == 3 else 1), float('nan'), device=DEV)
        keep.append((F, w, b, P))
        items[i] = _cabi.NormItem(F.data_ptr(), w.data_ptr(), b.data_ptr() if b is not None else None,
                                  _cabi.DTYPE_CODE[dtype], C, k, P.data_ptr())
    need = lib.kfac_norm_precondition_workspace_bytes(len(specs))
    ws = torch.empty(need, dtype=torch.uint8, device=DEV)
    launches = lib.kfac_launch_count()
    assert lib.kfac_norm_precondition(items, len(specs), damping, ws.data_ptr(), need, S()) == 0
    assert lib.kfac_launch_count() - launches == 1
    torch.cuda.synchronize()
    first = [P.clone() for *_, P in keep]
    for F, w, b, P in keep:
        grad = torch.stack([w, b], 1) if b is not None else w[:, None]
        assert rel_fro(P, ref_solve(F, grad, damping)) <= 1e-5
    assert lib.kfac_norm_precondition(items, len(specs), damping, ws.data_ptr(), need, S()) == 0
    torch.cuda.synchronize()
    assert all(torch.equal(bits(a), bits(P)) for a, (*_, P) in zip(first, keep))
    assert lib.kfac_norm_precondition(items, len(specs), damping, ws.data_ptr(), need - 1, S()) != 0
    bad = (_cabi.NormItem * 1)(_cabi.NormItem(keep[0][0].data_ptr(), keep[0][1].data_ptr(), None, 0, 7, 3,
                                              keep[0][3].data_ptr()))
    assert lib.kfac_norm_precondition(bad, 1, damping, ws.data_ptr(), need, S()) != 0    # k = 3 needs bgrad


# ---------------------------------------------------------------------------------------------- models
class CNN(nn.Module):
    def __init__(self):
        super().__init__()
        self.conv1 = nn.Conv2d(3, 8, 3, padding=1)
        self.bn1 = nn.BatchNorm2d(8)
        self.conv2 = nn.Conv2d(8, 15, 3, stride=2, padding=1)
        self.bn2 = nn.BatchNorm2d(15)
        self.fc = nn.Linear(15, 32)
        self.bn3 = nn.BatchNorm1d(32)
        self.head = nn.Linear(32, 10)

    def forward(self, x):
        h = torch.relu(self.bn1(self.conv1(x)))
        h = torch.relu(self.bn2(self.conv2(h))).mean((2, 3))
        return self.head(torch.relu(self.bn3(self.fc(h))))


class NeoX(nn.Module):
    """Parallel-residual block: x + attn(ln1(x)) + mlp(ln2(x)), then a bias-free final LayerNorm and a head."""

    def __init__(self, d=64, heads=4, ckpt=None):
        super().__init__()
        self.heads, self.ckpt = heads, ckpt
        self.ln1 = nn.LayerNorm(d)
        self.qkv = nn.Linear(d, 3 * d)
        self.proj = nn.Linear(d, d)
        self.ln2 = nn.RMSNorm(d)
        self.fc1 = nn.Linear(d, 4 * d)
        self.fc2 = nn.Linear(4 * d, d)
        self.lnf = nn.LayerNorm(d, bias=False)
        self.head = nn.Linear(d, 10)

    def block(self, x):
        B, T, d = x.shape
        q, k, v = self.qkv(self.ln1(x)).view(B, T, 3, self.heads, d // self.heads).unbind(2)
        a = nn.functional.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2),
                                                       is_causal=True)
        return x + self.proj(a.transpose(1, 2).reshape(B, T, d)) + self.fc2(nn.functional.gelu(self.fc1(self.ln2(x))))

    def forward(self, x):
        if self.ckpt is None:
            x = self.block(x)
        else:
            # the reentrant variant only differentiates through inputs that require grad
            x = checkpoint(self.block, x.detach().requires_grad_(self.ckpt), use_reentrant=self.ckpt)
        return self.head(self.lnf(x))


def make_model(kind, **kw):
    return (CNN() if kind == 'cnn' else NeoX(**kw)).to(DEV)


def batch(kind, step, micro=0, B=8):
    gen = torch.Generator(device=DEV).manual_seed(1000 * step + micro)
    if kind == 'cnn':
        x = torch.randn(B, 3, 4, 4, device=DEV, generator=gen)
    else:
        x = torch.randn(B, 16, 64, device=DEV, generator=gen) + 3.0
    return x, torch.randn(B, *((16, 10) if kind == 'neox' else (10,)), device=DEV, generator=gen)


def loss_of(model, x, y):
    return (model(x) - y).square().sum()


def capture(model):
    """Record (input, output gradient) of every call of every norm module, per module."""
    calls = {}
    for m in model.modules():
        if isinstance(m, (nn.BatchNorm1d, nn.BatchNorm2d, nn.LayerNorm, nn.RMSNorm)):
            calls[m] = []

            def fh(mod, inp, out):
                if not mod.training or not out.requires_grad:
                    return
                rec = {'x': inp[0].detach().clone()}
                calls[mod].append(rec)
                out.register_hook(lambda g: rec.__setitem__('g', g.detach().clone()))
            m.register_forward_hook(fh)
    return calls


def _norm_grad(m):
    g = m.weight.grad.reshape(-1, 1)
    bias = getattr(m, 'bias', None)         # RMSNorm has none
    return torch.cat([g, bias.grad.reshape(-1, 1)], 1) if bias is not None else g


@pytest.mark.parametrize('kind', ['cnn', 'neox'])
@pytest.mark.parametrize('method,schedule,accum', [('eigen', 'int', 1), ('inverse', 'int', 1), ('ekfac', 'int', 1),
                                                   ('eigen', 'callable', 1), ('inverse', 'callable', 2),
                                                   ('ekfac', 'callable', 1), ('eigen', 'int', 2)])
def test_module_level_against_fp64(kind, method, schedule, accum):
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(0)
    model = make_model(kind)
    alpha = 0.9
    if schedule == 'int':
        fus, ius, damp = 1, 2, 1e-3
    else:
        fus = lambda s: 1 if s < 2 else 2          # noqa: E731
        ius = lambda s: 2 if s < 2 else 4          # noqa: E731
        damp = lambda s: 1e-3 * (1 + s)            # noqa: E731
    pre = KFACPreconditioner(model, precondition_norms=True, kl_clip=None, factor_decay=alpha,
                             factor_update_steps=fus, inv_update_steps=ius, damping=damp, compute_method=method,
                             accumulation_steps=accum)
    val = lambda v, s: v(s) if callable(v) else v   # noqa: E731
    calls = capture(model)
    norms = {m: l for m, (_, l) in pre._norm_layers.items()}
    assert len(norms) == 3
    F = {m: None for m in norms}
    snap = {}
    for s in range(5):         # the weights stay put (kl-clip is off); the batches differ
        model.zero_grad()
        for c in calls.values():
            c.clear()
        for mb in range(accum):
            loss_of(model, *batch(kind, s, mb)).backward()
        grads = {m: _norm_grad(m).clone() for m in norms}
        windows = {}
        for m, l in norms.items():
            if s % val(fus, s) == 0:
                windows[m] = sum(ref_blocks(m, c['x'], c['g'], l.module.k)
                                 for c in calls[m]) / len(calls[m])
                # the open window itself (the BatchNorm2d windows are small next to the identity seed of the EMA)
                assert l._g_count == accum
                assert rel_fro(l._g_batch_view / l._g_count, windows[m]) <= 1e-5, (s, l)
            else:
                assert l._g_count == 0 and not bool(l._g_batch_view.any())
        pre.step()
        torch.cuda.synchronize()
        for m, l in norms.items():
            if m in windows:
                seed = torch.zeros_like(windows[m])
                seed[:, 0] = seed[:, -1] = 1.0
                F[m] = alpha * (seed if F[m] is None else F[m]) + (1 - alpha) * windows[m]
            if s % val(ius, s) == 0:
                snap[m] = F[m].clone()
            assert rel_fro(l.g_factor, F[m]) <= 1e-5, (s, l)
            got = _norm_grad(m)
            ref = ref_solve(snap[m], grads[m], val(damp, s))
            assert rel_fro(got, ref) <= 1e-4, (s, l, rel_fro(got, ref))


def _other_state(pre):
    out = {}
    for name, l in pre._layers.values():
        for key in ('a_factor', 'g_factor', 'qa', 'qg', 'da', 'dg', 'dgda', 'a_inv', 'g_inv'):
            t = getattr(l, key)
            if t is not None:
                out[(name, key)] = t.clone()
        out[(name, 'P')] = l._p_view.clone()
    return out


@pytest.mark.parametrize('kind', ['cnn', 'neox'])
@pytest.mark.parametrize('method', ['eigen', 'inverse', 'ekfac'])
def test_other_layers_bit_identical_with_the_keyword(kind, method):
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(0)
    m_off = make_model(kind)
    m_on = copy.deepcopy(m_off)
    kw = dict(kl_clip=None, damping=1e-3, inv_update_steps=2, compute_method=method)
    p_off = KFACPreconditioner(m_off, **kw)
    p_on = KFACPreconditioner(m_on, precondition_norms=True, **kw)
    norm_params = {n for n, mod in m_off.named_modules() if isinstance(mod, (nn.BatchNorm1d, nn.BatchNorm2d,
                                                                              nn.LayerNorm, nn.RMSNorm))}
    for s in range(3):      # the same weights at every step: the batches differ, the factors evolve
        for model in (m_off, m_on):
            model.zero_grad()
            loss_of(model, *batch(kind, s)).backward()
        raw = {n: p.grad.clone() for n, p in m_off.named_parameters()}
        p_off.step()
        p_on.step()
        torch.cuda.synchronize()
        a, b = _other_state(p_off), _other_state(p_on)
        assert a.keys() == b.keys()
        for key in a:
            assert torch.equal(bits(a[key]), bits(b[key])), (s, key)
        for (n, p), (_, q) in zip(m_off.named_parameters(), m_on.named_parameters()):
            if n.rsplit('.', 1)[0] in norm_params:
                assert torch.equal(p.grad, raw[n]), n          # keyword off: untouched
                assert not torch.equal(q.grad, raw[n]), n      # keyword on: preconditioned
            else:
                assert torch.equal(bits(p.grad), bits(q.grad)), (s, n)


def test_kl_clip_over_all_layers():
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(0)
    model = make_model('neox')
    kl_clip, lr = 1e-3, 0.1
    pre = KFACPreconditioner(model, precondition_norms=True, kl_clip=kl_clip, lr=lr, damping=1e-3)
    loss_of(model, *batch('neox', 0)).backward()
    layers = pre._layers | pre._norm_layers
    raw = {m: l.module.get_grad().clone() for m, (_, l) in layers.items()}
    pre.step()
    torch.cuda.synchronize()
    P = {m: l._p_view.double() for m, (_, l) in layers.items()}
    vg = sum(float((P[m] * raw[m].double()).sum()) for m in layers) * lr * lr
    nu = min(1.0, (kl_clip / abs(vg)) ** 0.5)
    assert nu < 1.0 and abs(pre._compute_grad_scale() - nu) <= 1e-6 * nu
    for m, (_, l) in layers.items():
        assert rel_fro(l.module.get_grad(), nu * P[m]) <= 1e-6, l


# ---------------------------------------------------------------------------------------------- lifecycle
def test_eval_accumulates_nothing():
    from kfac_b200.preconditioner import KFACPreconditioner
    model = make_model('cnn')
    pre = KFACPreconditioner(model, precondition_norms=True)
    loss_of(model, *batch('cnn', 0)).backward()
    pre.step()
    model.eval()
    model.zero_grad()
    loss_of(model, *batch('cnn', 1)).backward()
    torch.cuda.synchronize()
    for _, l in pre._norm_layers.values():
        assert l._g_count == 0 and not l._g_pending and not bool(l._g_batch_view.any())


def test_module_called_twice_in_a_window():
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(0)
    ln, lin = nn.LayerNorm(32).to(DEV), nn.Linear(32, 32).to(DEV)
    model = nn.ModuleDict({'ln': ln, 'lin': lin})
    calls = capture(model)
    pre = KFACPreconditioner(model, precondition_norms=True, factor_decay=0.5, kl_clip=None)
    x = torch.randn(16, 32, device=DEV) * 2 + 1
    out = ln(lin(ln(x)))
    out.square().sum().backward()
    assert len(calls[ln]) == 2
    l = pre._norm_layers[ln][1]
    assert l._g_count == 2
    pre.step()
    torch.cuda.synchronize()
    w = sum(ref_blocks(ln, c['x'], c['g'], 3) for c in calls[ln]) / 2
    seed = torch.zeros_like(w)
    seed[:, 0] = seed[:, 2] = 1
    assert rel_fro(l.g_factor, 0.5 * seed + 0.5 * w) <= 1e-6


@pytest.mark.parametrize('reentrant', [False, True])
def test_checkpoint_pairs_the_recomputed_call(reentrant):
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(0)
    plain = make_model('neox')
    ck = copy.deepcopy(plain)
    ck.ckpt = reentrant
    p1 = KFACPreconditioner(plain, precondition_norms=True, kl_clip=None)
    p2 = KFACPreconditioner(ck, precondition_norms=True, kl_clip=None)
    for s in range(2):
        for model in (plain, ck):
            model.zero_grad()
            loss_of(model, *batch('neox', s)).backward()
        p1.step()
        p2.step()
        torch.cuda.synchronize()
        for (m1, (n, l1)), (m2, (_, l2)) in zip(p1._norm_layers.items(), p2._norm_layers.items()):
            assert l2._g_count == 0 and l2._has_g
            assert rel_fro(l2.g_factor, l1.g_factor) <= 1e-6, (s, n)
            assert rel_fro(_norm_grad(m2), _norm_grad(m1)) <= 1e-5, (s, n)


def test_fp16_overflow_drops_the_norm_windows():
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(0)
    model = make_model('cnn')
    scaler = torch.amp.GradScaler('cuda', init_scale=2.0 ** 10)
    pre = KFACPreconditioner(model, precondition_norms=True, grad_scaler=scaler, damping=1e-3)
    layers = {m: l for m, (_, l) in (pre._layers | pre._norm_layers).items()}
    opt = torch.optim.SGD(model.parameters(), lr=0.01)
    for step in range(5):
        opt.zero_grad()
        if step == 2:
            scaler.update(new_scale=2.0 ** 60)
            before = {m: l.g_factor.clone() for m, l in layers.items()}
        x, y = batch('cnn', step)
        with torch.autocast('cuda', dtype=torch.float16):
            loss = (model(x).float() - y).square().sum()
        scaler.scale(loss).backward()
        scaler.unscale_(opt)
        pre.step()
        torch.cuda.synchronize()
        if step == 1:
            assert pre.skipped_factor_updates == 0
        if step == 2:
            for m, l in layers.items():
                assert torch.equal(l.g_factor, before[m]), l
            assert pre.skipped_factor_updates == len(layers)
        elif step > 2:
            for p in model.parameters():
                assert torch.isfinite(p.grad).all(), step
        scaler.step(opt)
        scaler.update(new_scale=2.0 ** 10) if step == 2 else scaler.update()
    for _, l in pre._norm_layers.values():
        assert torch.isfinite(l.g_factor).all()


def test_non_finite_block_raises_at_next_step():
    from kfac_b200 import _cabi
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(0)
    model = make_model('neox')
    pre = KFACPreconditioner(model, precondition_norms=True, factor_update_steps=2, inv_update_steps=1)
    l = pre._norm_layers[model.ln2][1]

    def step(s):
        model.zero_grad()
        loss_of(model, *batch('neox', s)).backward()
        pre.step()
        torch.cuda.synchronize()

    step(0)
    step(1)
    l._g_view[3, 0] = float('inf')
    step(2)                    # the factor stays inf; the inverse step snapshots it
    with pytest.raises(_cabi.KFACNativeError, match='non-finite'):
        step(3)


def test_state_dict_round_trip_and_memory_usage():
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(0)
    m1 = make_model('cnn')
    m2, mo = copy.deepcopy(m1), copy.deepcopy(m1)
    p1 = KFACPreconditioner(m1, precondition_norms=True, kl_clip=None)
    for s in range(2):
        m1.zero_grad()
        loss_of(m1, *batch('cnn', s)).backward()
        p1.step()
    sd = p1.state_dict()
    for name, l in p1._norm_layers.values():
        assert sd['layers'][name]['A'] is None and sd['layers'][name]['G'].shape == (l.g_dim, l.module.k)
    p2 = KFACPreconditioner(m2, precondition_norms=True, kl_clip=None)
    p2.load_state_dict(sd)
    for (_, l1), (_, l2) in zip(p1._norm_layers.values(), p2._norm_layers.values()):
        assert torch.equal(l1.g_factor, l2.g_factor) and torch.equal(l1.dg, l2.dg)
    # the next step of both gives the same norm gradients (same weights, same batch)
    for m, p in ((m1, p1), (m2, p2)):
        m.zero_grad()
        loss_of(m, *batch('cnn', 5)).backward()
        p.step()
    torch.cuda.synchronize()
    for mod1, mod2 in zip(p1._norm_layers, p2._norm_layers):
        assert torch.equal(_norm_grad(mod1), _norm_grad(mod2))
    # memory_usage: the same keys, the blocks counted under g_factors / g_inverses
    po = KFACPreconditioner(mo, kl_clip=None)
    mo.zero_grad()
    loss_of(mo, *batch('cnn', 5)).backward()
    po.step()
    on, of = p1.memory_usage(), po.memory_usage()
    assert on.keys() == of.keys()
    blocks = sum(l.g_dim * l.module.k * 4 for _, l in p1._norm_layers.values())
    assert on['g_factors'] - of['g_factors'] == blocks and on['g_inverses'] - of['g_inverses'] == blocks
    assert on['a_factors'] == of['a_factors']


# ---------------------------------------------------------------------------------------------- two ranks
def _run_dist(backend):
    import socket
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    script = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'dist_norm.py')
    out = subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node=2',
                          '--master-addr', '127.0.0.1', '--master-port', str(port), script, '--backend', backend],
                         capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, (out.stdout[-3000:], out.stderr[-3000:])
    assert out.stdout.count('dist_norm ok') == 2, out.stdout[-2000:]


def test_two_ranks_gloo():
    _run_dist('gloo')


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='NCCL needs one GPU per rank')
def test_two_ranks_nccl():
    _run_dist('nccl')
