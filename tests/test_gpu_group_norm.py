"""GroupNorm and InstanceNorm layers (`precondition_group_norms=True`) on the GPU, everything against fp64:

  * kfac_factor_group_norm for GroupNorm(32, 256) on 16 x 16 (a block per plane) and GroupNorm(32, 512) on 16 x 16
    at batch 12 (a warp per plane), GroupNorm(32, 96) on 7 x 7 (Cg = 3), GroupNorm(1, 64),
    GroupNorm(8, 64) on (B, C) and (B, C, L), a GroupNorm on a 3-D map, InstanceNorm1d / 2d / 3d (one of them
    unbatched) and S = 4097; x and g each in fp32/fp16/bf16, inputs centred and with |mean| = 100 std: relative
    Frobenius error <= 1e-5 and the same bits on a repeat, with and without a live accumulator; the argument checks;
  * xhat is the module's own: with weight 1 and bias 0 the block formed from module(x) is the kernel's;
  * a small diffusion-U-Net-shaped model (GroupNorm, a time embedding, a ConvTranspose2d upsample) and an
    InstanceNorm2d generator for 5 steps under EIGEN, INVERSE and EKFAC, with callable schedules and with
    accumulation_steps=2: the written norm gradients against an fp64 restatement from the captured inputs and output
    gradients;
  * with the keyword off and on (kl-clip off) every other layer's factors, second-order data, P and written gradient
    are bit-identical and the GroupNorm gradients are untouched when off; with `precondition_norms` as well, the
    BatchNorm / LayerNorm blocks and P are those of `precondition_norms` alone, bit for bit;
  * eval(), an fp16 GradScaler overflow, a state_dict round trip, memory_usage(), and two ranks
    (tests/dist_group_norm.py).
"""
import copy
import os
import subprocess
import sys
import zlib

import pytest
import torch
from torch import nn

from conftest import rel_fro
from test_gpu_norm import DTYPES, _norm_grad, bits, ref_solve

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda')
GROUP_NORM_TYPES = (nn.GroupNorm, nn.InstanceNorm1d, nn.InstanceNorm2d, nn.InstanceNorm3d)


@pytest.fixture(scope='module')
def lib():
    from kfac_b200 import _cabi
    return _cabi.load()


def S():
    return torch.cuda.current_stream().cuda_stream


@pytest.fixture
def deterministic_convs():
    """cuDNN's default conv backward algorithms need not give the same bits twice, so two copies of a model would not
    receive the same raw gradients; the comparisons of bits between runs take the deterministic ones."""
    old = torch.backends.cudnn.deterministic
    torch.backends.cudnn.deterministic = True
    yield
    torch.backends.cudnn.deterministic = old


# ---------------------------------------------------------------------------------------------- fp64 restatement
def _groups(module):
    return module.num_groups if isinstance(module, nn.GroupNorm) else module.num_features


def _batched(module, t):
    """An unbatched InstanceNorm input is one example."""
    if not isinstance(module, nn.GroupNorm) and t.dim() == module._get_no_batch_dim():
        return t.unsqueeze(0)
    return t


def ref_group_blocks(module, x, g, k=3):
    """(C, k) fp64 block of one call of `module`: group_norm decomposed in float64, the rows of BatchNorm."""
    x, g = _batched(module, x.double()), _batched(module, g.double())
    B, C = x.shape[:2]
    G = _groups(module)
    xg = x.reshape(B, G, -1)
    mu = xg.mean(2, keepdim=True)
    var = xg.var(2, unbiased=False, keepdim=True)
    xh = ((xg - mu) / torch.sqrt(var + module.eps)).reshape(B, C, -1)
    gv = g.reshape(B, C, -1)
    Sp = xh.shape[2]
    scale = 1.0 / (B * Sp * float(Sp) ** 4)
    g2 = gv * gv
    ss = (g2 * xh * xh).sum((0, 2))
    if k == 1:
        return (ss * scale)[:, None]
    return torch.stack([ss, (g2 * xh).sum((0, 2)), g2.sum((0, 2))], 1) * scale


# ---------------------------------------------------------------------------------------------- statistics kernel
CASES = {
    'gn32_256_16x16': (lambda: nn.GroupNorm(32, 256), (4, 256, 16, 16)),
    'gn32_96_7x7': (lambda: nn.GroupNorm(32, 96, eps=1e-3), (8, 96, 7, 7)),
    'gn32_512_16x16_many': (lambda: nn.GroupNorm(32, 512), (12, 512, 16, 16)),   # 6144 planes: a warp each
    'gn1_64': (lambda: nn.GroupNorm(1, 64), (4, 64, 8, 8)),
    'gn8_64_flat': (lambda: nn.GroupNorm(8, 64), (32, 64)),
    'gn8_64_seq': (lambda: nn.GroupNorm(8, 64), (6, 64, 37)),
    'gn_3d': (lambda: nn.GroupNorm(4, 16), (2, 16, 5, 6, 7)),
    'in1d': (lambda: nn.InstanceNorm1d(12, affine=True), (5, 12, 300)),
    'in2d': (lambda: nn.InstanceNorm2d(24, affine=True), (3, 24, 9, 11)),
    'in2d_unbatched': (lambda: nn.InstanceNorm2d(8, affine=True), (8, 20, 20)),
    'in3d': (lambda: nn.InstanceNorm3d(6, affine=True), (2, 6, 4, 8, 8)),
    'gn_4097': (lambda: nn.GroupNorm(4, 8), (3, 8, 4097)),
}


def _stats(lib, helper, x, g, live, eps):
    from kfac_b200 import _cabi
    acc = live.clone()
    C = helper.channels
    xb = _batched(helper.module, x)
    B, Sp = xb.shape[0], x.numel() // (xb.shape[0] * C)
    scale = 1.0 / (B * float(Sp) ** 5)
    need = lib.kfac_factor_group_norm_workspace_bytes(B, C, Sp, helper.groups)
    ws = torch.full((need,), 255, dtype=torch.uint8, device=DEV)
    args = (x.data_ptr(), _cabi.DTYPE_CODE[x.dtype], g.data_ptr(), _cabi.DTYPE_CODE[g.dtype], B, C, Sp, helper.groups,
            helper.k, eps, scale, acc.data_ptr(), ws.data_ptr())
    assert lib.kfac_factor_group_norm(*args, need, S()) == 0, lib.kfac_last_error()
    assert lib.kfac_factor_group_norm(*args, need - 8, S()) != 0
    torch.cuda.synchronize()
    return acc


@pytest.mark.parametrize('offset', [0.0, 100.0])
@pytest.mark.parametrize('g_dtype', DTYPES)
@pytest.mark.parametrize('x_dtype', DTYPES)
@pytest.mark.parametrize('case', list(CASES))
def test_factor_group_norm_against_fp64(lib, case, x_dtype, g_dtype, offset):
    from kfac_b200.layers import NormModuleHelper
    make, shape = CASES[case]
    module = make().to(DEV)
    helper = NormModuleHelper(module)
    gen = torch.Generator(device=DEV).manual_seed(zlib.crc32(f'{case}/{offset}'.encode()))
    C = helper.channels
    # per-element scales (std 1 .. 3) and a common offset
    x = torch.randn(shape, device=DEV, generator=gen) * (1 + 2 * torch.rand(shape, device=DEV, generator=gen)) + offset
    x = x.to(x_dtype)
    g = torch.randn(shape, device=DEV, generator=gen).to(g_dtype)
    ref = ref_group_blocks(module, x, g, helper.k)
    acc = _stats(lib, helper, x, g, torch.zeros(C, helper.k, device=DEV), helper.eps_for(x))
    err = rel_fro(acc, ref)
    assert err <= 1e-5, err
    assert torch.equal(bits(acc), bits(_stats(lib, helper, x, g, torch.zeros(C, helper.k, device=DEV),
                                              helper.eps_for(x))))
    # accumulated into a batch buffer that already holds a window of the same magnitude
    live = torch.rand(C, helper.k, device=DEV, generator=gen) * float(ref.abs().max())
    acc = _stats(lib, helper, x, g, live, helper.eps_for(x))
    assert rel_fro(acc, live.double() + ref) <= 1e-5
    assert torch.equal(bits(acc), bits(_stats(lib, helper, x, g, live, helper.eps_for(x))))


@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('case', ['gn32_96_7x7', 'gn1_64', 'gn8_64_flat', 'in2d_unbatched', 'in1d'])
def test_xhat_is_the_modules_own_normalization(lib, case, dtype):
    """With weight 1 and bias 0 the module's forward output is x-hat itself, so the block formed by the kernel must be
    the one of module(x), computed here from the module's output and not from a restated formula."""
    from kfac_b200.layers import NormModuleHelper
    make, shape = CASES[case]
    module = make().to(DEV).to(dtype).train()
    with torch.no_grad():
        module.weight.fill_(1.0)
        module.bias.zero_()
    helper = NormModuleHelper(module)
    gen = torch.Generator(device=DEV).manual_seed(zlib.crc32(f'xhat/{case}'.encode()))
    x = (torch.randn(shape, device=DEV, generator=gen) * 0.02 + 0.01).to(dtype)
    g = torch.randn(shape, device=DEV, generator=gen).to(dtype)
    with torch.no_grad():
        xh = _batched(module, module(x).double())            # rounded to `dtype` by the module
    acc = _stats(lib, helper, x, g, torch.zeros(helper.channels, helper.k, device=DEV), helper.eps_for(x))
    C, gd = helper.channels, _batched(module, g.double())
    B = xh.shape[0]
    xv, gv = xh.reshape(B, C, -1), gd.reshape(B, C, -1)
    Sp = xv.shape[2]
    scale = 1.0 / (B * Sp * float(Sp) ** 4)
    g2 = gv * gv
    ref = torch.stack([(g2 * xv * xv).sum((0, 2)), (g2 * xv).sum((0, 2)), g2.sum((0, 2))], 1) * scale
    # the module's output carries the rounding of `dtype` (2^-8 relative for bf16)
    tol = {torch.float32: 1e-5, torch.float16: 2e-3, torch.bfloat16: 1e-2}[dtype]
    assert rel_fro(acc, ref) <= tol, rel_fro(acc, ref)


def test_factor_group_norm_rejects_bad_arguments(lib):
    x = torch.zeros(4, 8, 3, device=DEV)
    acc = torch.zeros(8, 3, device=DEV)
    ws = torch.zeros(1 << 16, dtype=torch.uint8, device=DEV)
    args = dict(B=4, C=8, S=3, groups=4, k=3, x_dtype=0, g_dtype=0)

    def call(**kw):
        a = {**args, **kw}
        return lib.kfac_factor_group_norm(x.data_ptr(), a['x_dtype'], x.data_ptr(), a['g_dtype'], a['B'], a['C'],
                                          a['S'], a['groups'], a['k'], 1e-5, 1.0, acc.data_ptr(), ws.data_ptr(),
                                          ws.numel(), S())
    assert call() == 0
    assert call(k=1) == 0
    assert call(k=2) != 0
    assert call(groups=3) != 0                          # 3 does not divide 8 channels
    assert call(groups=0) != 0
    assert call(x_dtype=7) != 0 and call(g_dtype=7) != 0
    assert call(S=1 << 28) != 0                         # 4 * 8 * 2^28 = 2^33 elements
    assert call(S=0) != 0
    assert lib.kfac_factor_group_norm_workspace_bytes(4, 8, 3, 3) == 0
    assert lib.kfac_factor_group_norm_workspace_bytes(4, 8, 3, 4) > 0
    torch.cuda.synchronize()


@pytest.mark.parametrize('module,shape', [
    (nn.GroupNorm(2, 4), (3, 5, 6)), (nn.InstanceNorm2d(4, affine=True), (2, 4, 5)),
    (nn.InstanceNorm1d(4, affine=True), (2, 3, 4, 5)), (nn.InstanceNorm3d(4, affine=True), (3, 4, 5))],
    ids=lambda v: repr(v))
def test_helper_checks_the_input_shape(module, shape):
    from kfac_b200.layers import NormModuleHelper
    helper = NormModuleHelper(module)
    x = torch.zeros(shape, device=DEV)
    with pytest.raises(ValueError, match='input of shape'):
        helper.accumulate_norm(x, x, torch.zeros(4, 3, device=DEV), 1.0, 1e-5, None)


# ---------------------------------------------------------------------------------------------- models
class UNet(nn.Module):
    """Diffusion-U-Net-shaped: conv -> GroupNorm -> SiLU -> conv with a time embedding added in between, a strided
    conv down, a ConvTranspose2d up and a final conv.  A LayerNorm on the time input (for `precondition_norms`)."""

    def __init__(self):
        super().__init__()
        self.conv_in = nn.Conv2d(3, 32, 3, padding=1)
        self.t_ln = nn.LayerNorm(16)
        self.temb = nn.Linear(16, 32)
        self.gn1 = nn.GroupNorm(8, 32)
        self.conv1 = nn.Conv2d(32, 32, 3, padding=1)
        self.gn2 = nn.GroupNorm(1, 32)
        self.down = nn.Conv2d(32, 32, 3, stride=2, padding=1)
        self.gn3 = nn.GroupNorm(32, 32)
        self.up = nn.ConvTranspose2d(32, 16, 4, stride=2, padding=1)
        self.out = nn.Conv2d(16, 3, 3, padding=1)

    def forward(self, x, t):
        h = self.conv_in(x)
        h = self.conv1(nn.functional.silu(self.gn1(h + self.temb(self.t_ln(t))[:, :, None, None])))
        h = self.down(nn.functional.silu(self.gn2(h)))
        return self.out(nn.functional.silu(self.up(nn.functional.silu(self.gn3(h)))))


class Generator(nn.Module):
    """pix2pix / CycleGAN-shaped block: conv -> InstanceNorm2d -> ReLU, a strided conv with BatchNorm2d (for
    `precondition_norms`), a ConvTranspose2d up -> InstanceNorm2d, and a final conv."""

    def __init__(self):
        super().__init__()
        self.c1 = nn.Conv2d(3, 16, 7, padding=3)
        self.in1 = nn.InstanceNorm2d(16, affine=True)
        self.c2 = nn.Conv2d(16, 32, 3, stride=2, padding=1)
        self.bn2 = nn.BatchNorm2d(32)
        self.up = nn.ConvTranspose2d(32, 16, 3, stride=2, padding=1, output_padding=1)
        self.in3 = nn.InstanceNorm2d(16, affine=True)
        self.c4 = nn.Conv2d(16, 3, 7, padding=3)

    def forward(self, x, t=None):
        h = torch.relu(self.in1(self.c1(x)))
        h = torch.relu(self.bn2(self.c2(h)))
        h = torch.relu(self.in3(self.up(h)))
        return torch.tanh(self.c4(h))


def make_model(kind):
    return (UNet() if kind == 'unet' else Generator()).to(DEV)


def batch(kind, step, micro=0, B=8):
    gen = torch.Generator(device=DEV).manual_seed(1000 * step + micro)
    x = torch.randn(B, 3, 16, 16, device=DEV, generator=gen) + (2.0 if kind == 'unet' else 0.0)
    t = torch.randn(B, 16, device=DEV, generator=gen)
    return x, t, torch.randn(B, 3, 16, 16, device=DEV, generator=gen)


def loss_of(model, x, t, y):
    return (model(x, t) - y).square().sum()


def capture(model, types=GROUP_NORM_TYPES):
    """Record (input, output gradient) of every call of every GroupNorm / InstanceNorm module, per module."""
    calls = {}
    for m in model.modules():
        if isinstance(m, types):
            calls[m] = []

            def fh(mod, inp, out):
                if not mod.training or not out.requires_grad:
                    return
                rec = {'x': inp[0].detach().clone()}
                calls[mod].append(rec)
                out.register_hook(lambda g: rec.__setitem__('g', g.detach().clone()))
            m.register_forward_hook(fh)
    return calls


def make_pre(model, **kw):
    from kfac_b200.preconditioner import KFACPreconditioner
    return KFACPreconditioner(model, precondition_conv_transpose=True, **kw)


@pytest.mark.parametrize('kind', ['unet', 'gen'])
@pytest.mark.parametrize('method,schedule,accum', [('eigen', 'int', 1), ('inverse', 'int', 1), ('ekfac', 'int', 1),
                                                   ('eigen', 'callable', 1), ('inverse', 'callable', 2),
                                                   ('ekfac', 'callable', 1), ('eigen', 'int', 2)])
def test_module_level_against_fp64(kind, method, schedule, accum):
    torch.manual_seed(0)
    model = make_model(kind)
    alpha = 0.9
    if schedule == 'int':
        fus, ius, damp = 1, 2, 1e-3
    else:
        fus = lambda s: 1 if s < 2 else 2          # noqa: E731
        ius = lambda s: 2 if s < 2 else 4          # noqa: E731
        damp = lambda s: 1e-3 * (1 + s)            # noqa: E731
    pre = make_pre(model, precondition_group_norms=True, kl_clip=None, factor_decay=alpha, factor_update_steps=fus,
                   inv_update_steps=ius, damping=damp, compute_method=method, accumulation_steps=accum)
    val = lambda v, s: v(s) if callable(v) else v   # noqa: E731
    calls = capture(model)
    norms = {m: l for m, (_, l) in pre._norm_layers.items()}
    assert set(norms) == set(calls) and len(norms) == (3 if kind == 'unet' else 2)
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
                windows[m] = sum(ref_group_blocks(m, c['x'], c['g'], l.module.k) for c in calls[m]) / len(calls[m])
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


def _state(layers):
    out = {}
    for name, l in layers.values():
        for key in ('a_factor', 'g_factor', 'qa', 'qg', 'da', 'dg', 'dgda', 'a_inv', 'g_inv'):
            t = getattr(l, key)
            if t is not None:
                out[(name, key)] = t.clone()
        out[(name, 'P')] = l._p_view.clone()
    return out


@pytest.mark.parametrize('kind', ['unet', 'gen'])
@pytest.mark.parametrize('method', ['eigen', 'inverse', 'ekfac'])
@pytest.mark.parametrize('norms', [False, True])
def test_other_layers_bit_identical_with_the_keyword(kind, method, norms, deterministic_convs):
    """Off and on: the dense layers (and, with precondition_norms on both, the BatchNorm / LayerNorm layers) keep
    their factors, second-order data, P and written gradients bit for bit; the GroupNorm / InstanceNorm gradients are
    untouched when off and preconditioned when on."""
    torch.manual_seed(0)
    m_off = make_model(kind)
    m_on = copy.deepcopy(m_off)
    kw = dict(kl_clip=None, damping=1e-3, inv_update_steps=2, compute_method=method, precondition_norms=norms)
    p_off = make_pre(m_off, **kw)
    p_on = make_pre(m_on, precondition_group_norms=True, **kw)
    assert len(p_on._norm_layers) == len(p_off._norm_layers) + (3 if kind == 'unet' else 2)
    assert len(p_off._norm_layers) == (1 if norms else 0)
    group_params = {n for n, mod in m_off.named_modules() if isinstance(mod, GROUP_NORM_TYPES)}
    for s in range(3):      # the same weights at every step: the batches differ, the factors evolve
        for model in (m_off, m_on):
            model.zero_grad()
            loss_of(model, *batch(kind, s)).backward()
        raw = {n: p.grad.clone() for n, p in m_off.named_parameters()}
        for n, q in m_on.named_parameters():
            assert torch.equal(bits(q.grad), bits(raw[n])), (s, n)     # the same raw gradients to start from
        p_off.step()
        p_on.step()
        torch.cuda.synchronize()
        a, b = _state(p_off._layers), _state(p_on._layers)
        assert a.keys() == b.keys()
        for key in a:
            assert torch.equal(bits(a[key]), bits(b[key])), (s, key)
        if norms:              # the BatchNorm / LayerNorm layer of precondition_norms
            (name, l_off), = p_off._norm_layers.values()
            l_on = {n: l for n, l in p_on._norm_layers.values()}[name]
            for key in ('g_factor', 'dg'):
                assert torch.equal(bits(getattr(l_off, key)), bits(getattr(l_on, key))), (s, name, key)
            assert torch.equal(bits(l_off._p_view), bits(l_on._p_view)), (s, name)
        for (n, p), (_, q) in zip(m_off.named_parameters(), m_on.named_parameters()):
            if n.rsplit('.', 1)[0] in group_params:
                assert torch.equal(p.grad, raw[n]), n          # keyword off: untouched
                assert not torch.equal(q.grad, raw[n]), n      # keyword on: preconditioned
            else:
                assert torch.equal(bits(p.grad), bits(q.grad)), (s, n)


# ---------------------------------------------------------------------------------------------- lifecycle
def test_eval_accumulates_nothing():
    model = make_model('unet')
    pre = make_pre(model, precondition_group_norms=True)
    loss_of(model, *batch('unet', 0)).backward()
    pre.step()
    model.eval()
    model.zero_grad()
    loss_of(model, *batch('unet', 1)).backward()
    torch.cuda.synchronize()
    for _, l in pre._norm_layers.values():
        assert l._g_count == 0 and not l._g_pending and not bool(l._g_batch_view.any())


@pytest.mark.parametrize('amp', [torch.float16, torch.bfloat16])
def test_autocast_blocks_against_fp64(amp):
    """Under autocast a GroupNorm receives a half-precision x and returns fp32, so its output gradient is fp32."""
    torch.manual_seed(0)
    model = make_model('unet')
    pre = make_pre(model, precondition_group_norms=True, kl_clip=None, factor_decay=0.5)
    calls = capture(model)
    x, t, y = batch('unet', 0)
    with torch.autocast('cuda', dtype=amp):
        out = model(x, t)
    (out.float() - y).square().sum().backward()
    for m, (_, l) in pre._norm_layers.items():
        (c,) = calls[m]
        assert c['x'].dtype == amp and c['g'].dtype == torch.float32
        assert rel_fro(l._g_batch_view, ref_group_blocks(m, c['x'], c['g'])) <= 1e-5
    pre.step()
    torch.cuda.synchronize()


def test_fp16_overflow_drops_the_norm_windows():
    torch.manual_seed(0)
    model = make_model('gen')
    scaler = torch.amp.GradScaler('cuda', init_scale=2.0 ** 10)
    pre = make_pre(model, precondition_group_norms=True, grad_scaler=scaler, damping=1e-3)
    layers = {m: l for m, (_, l) in (pre._layers | pre._norm_layers).items()}
    opt = torch.optim.SGD(model.parameters(), lr=0.01)
    for step in range(5):
        opt.zero_grad()
        if step == 2:
            scaler.update(new_scale=2.0 ** 60)
            before = {m: l.g_factor.clone() for m, l in layers.items()}
        x, t, y = batch('gen', step)
        with torch.autocast('cuda', dtype=torch.float16):
            out = model(x, t)
        loss = (out.float() - y).square().mean()     # a sum over the 6144 outputs would overflow fp16 at 2^10
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


def test_state_dict_round_trip_and_memory_usage(deterministic_convs):
    torch.manual_seed(0)
    m1 = make_model('unet')
    m2, mo = copy.deepcopy(m1), copy.deepcopy(m1)
    p1 = make_pre(m1, precondition_group_norms=True, kl_clip=None)
    for s in range(2):
        m1.zero_grad()
        loss_of(m1, *batch('unet', s)).backward()
        p1.step()
    sd = p1.state_dict()
    for name, l in p1._norm_layers.values():
        assert sd['layers'][name]['A'] is None and sd['layers'][name]['G'].shape == (l.g_dim, l.module.k)
    p2 = make_pre(m2, precondition_group_norms=True, kl_clip=None)
    p2.load_state_dict(sd)
    for (_, l1), (_, l2) in zip(p1._norm_layers.values(), p2._norm_layers.values()):
        assert torch.equal(l1.g_factor, l2.g_factor) and torch.equal(l1.dg, l2.dg)
    # the next step of both gives the same norm gradients (same weights, same batch)
    for m, p in ((m1, p1), (m2, p2)):
        m.zero_grad()
        loss_of(m, *batch('unet', 5)).backward()
        p.step()
    torch.cuda.synchronize()
    for mod1, mod2 in zip(p1._norm_layers, p2._norm_layers):
        assert torch.equal(_norm_grad(mod1), _norm_grad(mod2))
    # memory_usage: the same keys, the blocks counted under g_factors / g_inverses
    po = make_pre(mo, kl_clip=None)
    mo.zero_grad()
    loss_of(mo, *batch('unet', 5)).backward()
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
    script = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'dist_group_norm.py')
    out = subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node=2',
                          '--master-addr', '127.0.0.1', '--master-port', str(port), script, '--backend', backend],
                         capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, (out.stdout[-3000:], out.stderr[-3000:])
    assert out.stdout.count('dist_group_norm ok') == 2, out.stdout[-2000:]


def test_two_ranks_gloo():
    _run_dist('gloo')


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='NCCL needs one GPU per rank')
def test_two_ranks_nccl():
    _run_dist('nccl')
