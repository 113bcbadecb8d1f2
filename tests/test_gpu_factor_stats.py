"""The factor statistics (acc += scale * X^T X) and their EMA against fp64, at transformer and ResNet-50 widths,
accumulating into live factor buffers.

* kfac_factor_linear / kfac_factor_linear_strided, kfac_factor_conv2d_gradout and kfac_factor_conv2d_input on each
  of their dispatch paths: packed feature-major (a transpose or im2col first) or read as stored, and one split
  (the SYRK's read-modify-write epilogue, or the SIMT kernel's +=) or split partials added by cov_reduce_kernel.  A
  Python copy of the split plans (cov_tc_splits, cov_simt_splits, linear_pack_bytes, gradout_ws) names the path of
  each case on this device, and the kfac_launch_count() delta of the call confirms it, so that a change to the
  dispatch cannot silently turn one case into a copy of another;
* kfac_factor_ema over ResNet-50's 108 factors plus edge widths, three launches of up to 40 items;
* a Linear and a Conv2d layer trained one step with accumulation_steps=2 through the preconditioner.

Every statistic starts from a non-symmetric fp32 acc0 inside a larger arena whose other entries are canaries, with
a workspace of NaN bytes.  Each entry is checked against the dot-product bound
    |acc - (acc0 + scale X^T X)| <= u (c K scale (|X|^T |X|) + |acc0|),     u = 2^-24,
K the length of the reduction and c one constant per path (SIMT FMA chains, 3xTF32 wgmma, split partials), with the
reference formed in fp64 from the input values as stored (after rounding to fp16 / bf16).  A wrong block, however
small, or an add that became a store, fails this bound where it would hide in a Frobenius norm."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
# c of the bound per path: one split on the SIMT kernel (FMA chains), one split on the 3xTF32 wgmma SYRK, and split
# partials (either engine).  The worst ratios over this file's cases on an H100 80GB HBM3 (132 SMs, 700 W) were
# 0.066, 0.126 and 0.059; each c leaves less than 10x headroom above its path's worst ratio
C_PATH = {'simt': 0.5, 'tc': 1.0, 'split': 0.5}
CANARY = 0x7FBADBAD                                   # a NaN pattern no kernel writes
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
DTYPE_CODE = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}


@pytest.fixture(scope='module')
def lib():
    from kfac_b200 import _cabi
    return _cabi.load()


@pytest.fixture(scope='module')
def dev():
    assert torch.cuda.is_available()
    return torch.device('cuda:0')


@pytest.fixture(scope='module')
def sms(dev):
    n = torch.cuda.get_device_properties(dev).multi_processor_count
    print(f'{torch.cuda.get_device_name(dev)}: {n} SMs')
    return n


def S():
    return torch.cuda.current_stream().cuda_stream


def f32(x):
    """x rounded to fp32, as a Python float (the value a c_float argument carries)."""
    return float(np.float32(x))


# ---- the split plans of csrc/factor.cu ----------------------------------------------------------------------------

def ceil_div(a, b):
    return -(-a // b)


def ld4(n):
    return (n + 3) // 4 * 4


def tc_normalize_splits(splits, kb_total):
    splits = max(1, min(splits, kb_total))
    return ceil_div(kb_total, ceil_div(kb_total, splits))


def cov_tc_splits(d, rows, batch, sms):
    nt = ceil_div(d, 128)
    ntiles = nt * (nt + 1) // 2
    kb_total = ceil_div(rows, 32) * batch
    splits = max(1, min(sms // ntiles, kb_total // 8)) if ntiles < sms else 1
    return tc_normalize_splits(splits, kb_total)


def cov_simt_splits(d, rows, batch, sms):
    nt = ceil_div(d, 64)
    tiles = nt * (nt + 1) // 2
    return max(1, min(ceil_div(sms * 3, tiles), ceil_div(rows * batch, 64)))


def cov_ws(pack, d, rows, batch, sms):
    """CovWs: (pack bytes, offset of the split partials, total bytes)."""
    slab_off = (pack + 255) // 256 * 256 if pack else 0
    s = max(cov_tc_splits(d, rows, batch, sms), cov_simt_splits(d, rows, batch, sms))
    return pack, slab_off, (slab_off + s * d * d * 4 if s > 1 else pack)


def linear_pack_bytes(rows, features, ones):
    return 0 if rows < 512 or features < 128 else ld4(rows) * (features + ones) * 4


def gradout_ws(B, Cc, Ho, Wo, sms):
    if (Ho * Wo) % 4 == 0 or Cc < 64:
        return cov_ws(0, Cc, Ho * Wo, B, sms)
    rows = B * Ho * Wo
    return cov_ws(ld4(rows) * Cc * 4, Cc, rows, 1, sms)


def launch_cov(d, rows, batch, ld, f32_input, feature_major, slab, sms):
    """(engine, splits) of launch_cov: the wgmma SYRK on fp32 feature-major data it can address, else the SIMT kernel."""
    if feature_major and f32_input and d >= 64 and rows * batch >= 256 and ld % 4 == 0:
        return 'tc', cov_tc_splits(d, rows, batch, sms) if slab else 1
    return 'simt', cov_simt_splits(d, rows, batch, sms) if slab else 1


def has_slab(w, ws_bytes):
    _, slab_off, total = w
    return ws_bytes > 0 and total > slab_off and ws_bytes >= total


def path_name(packed, splits):
    return ('pack' if packed else 'direct') + ('+split' if splits > 1 else '+one')


def launches(path):
    """transpose / im2col (pack), the SYRK or SIMT kernel, cov_reduce_kernel (split)."""
    return path.startswith('pack') + 1 + path.endswith('split')


def linear_path(rows, feat, ones, dtype, ws_bytes, sms):
    d = feat + ones
    pack = linear_pack_bytes(rows, feat, ones)
    w = cov_ws(pack, d, rows, 1, sms)
    if pack and ws_bytes >= pack:
        engine, splits = launch_cov(d, rows, 1, ld4(rows), True, True, has_slab(w, ws_bytes), sms)
    else:
        engine, splits = launch_cov(d, rows, 1, feat, dtype == torch.float32, False, has_slab(w, ws_bytes), sms)
    return path_name(pack and ws_bytes >= pack, splits), engine


def gradout_path(B, Cc, Ho, Wo, dtype, ws_bytes, sms):
    w = gradout_ws(B, Cc, Ho, Wo, sms)
    pack = w[0]
    if pack and ws_bytes >= pack:
        rows = B * Ho * Wo
        engine, splits = launch_cov(Cc, rows, 1, ld4(rows), True, True, has_slab(w, ws_bytes), sms)
    else:
        engine, splits = launch_cov(Cc, Ho * Wo, B, Ho * Wo, dtype == torch.float32, True, has_slab(w, ws_bytes), sms)
    return path_name(pack and ws_bytes >= pack, splits), engine


# ---- live buffers and the bound -----------------------------------------------------------------------------------

def nan_ws(nbytes, dev):
    return torch.full((max(nbytes, 1),), 255, dtype=torch.uint8, device=dev)     # all-ones bytes: NaN floats


def canary_arena(n, pad, dev):
    """A flat fp32 arena of pad + n + pad canaries; returns (arena, the n entries after the first pad)."""
    arena = torch.full((2 * pad + n,), CANARY, dtype=torch.int32, device=dev).view(torch.float32)
    return arena, arena[pad:pad + n]


def assert_canaries(arena, pad, n, what):
    # booleans formed before the assert: pytest would explain a failed `tensor == value` element by element
    bits = arena.view(torch.int32)
    before, after = bool((bits[:pad] == CANARY).all()), bool((bits[pad + n:] == CANARY).all())
    assert before, (what, 'written before the block')
    assert after, (what, 'written after the block')


def check_statistic(lib, call, X64, scale, ws_bytes, dev, expect_path, engine, what):
    """Run call(acc_ptr, ws_ptr, ws_bytes) twice from the same live acc0 and a NaN workspace; check its launch count,
    the element-wise bound, the canaries around acc and that both calls give the same bits.  Prints the worst ratio
    of the error to u K scale (|X|^T |X|), the c this case needs."""
    K, d = X64.shape
    s = f32(scale)
    ref = s * (X64.t() @ X64)
    absX = X64.abs()
    bound_unit = U * K * s * (absX.t() @ absX)
    del absX
    g = torch.Generator(device=dev).manual_seed(K * 7919 + d)
    acc0 = torch.randn(d, d, device=dev, generator=g) * f32(ref.diagonal().abs().mean().item())   # not symmetric
    pad = 2 * d + 64
    runs = []
    for _ in range(2):
        arena, block = canary_arena(d * d, pad, dev)
        acc = block.view(d, d)
        acc.copy_(acc0)
        ws = nan_ws(ws_bytes, dev)
        torch.cuda.synchronize()
        n0 = lib.kfac_launch_count()
        rc = call(acc.data_ptr(), ws.data_ptr() if ws_bytes else None, ws_bytes)
        n1 = lib.kfac_launch_count()
        torch.cuda.synchronize()
        assert rc == 0, (what, lib.kfac_last_error())
        assert n1 - n0 == launches(expect_path), (what, expect_path, 'launches', n1 - n0)
        assert_canaries(arena, pad, d * d, what)
        runs.append(arena.view(torch.int32).clone())
    assert torch.equal(runs[0], runs[1]), (what, 'not the same bits in a repeat call')
    got = runs[0][pad:pad + d * d].view(torch.float32).view(d, d)
    finite = bool(torch.isfinite(got).all())
    assert finite, what
    excess = (got.double() - (acc0.double() + ref)).abs() - U * acc0.double().abs()
    ratio = float((excess / bound_unit).max())
    c = C_PATH['split' if expect_path.endswith('split') else engine]
    print(f'{what}: {expect_path} ({engine}), {launches(expect_path)} launches, worst ratio {ratio:.3g} (c = {c})')
    assert ratio <= c, (what, expect_path, engine, ratio, c)


# ---- kfac_factor_linear / kfac_factor_linear_strided ---------------------------------------------------------------

# (rows, features, ones, workspace, path on a 132- or 114-SM part); workspace 'full' is the size the query returns,
# 'pack' only the packed matrix (no room for the split partials)
LINEAR_CASES = [
    (2048, 1024, 1, 'full', 'pack+split'),
    (4096, 2048, 1, 'full', 'pack+one'),        # d = 2049: GPT-NeoX / ResNet-50 fc widths, odd d
    (8192, 3072, 1, 'full', 'pack+one'),        # d = 3073
    (1024, 4096, 0, 'full', 'pack+one'),        # d = 4096, even
    (600, 8191, 1, 'full', 'pack+one'),         # d = 8192 from an odd feature count
    (2048, 1024, 1, 'pack', 'pack+one'),
    (511, 200, 1, 'full', 'direct+split'),      # one row short of packing: the sample-major SIMT kernel
    (300, 2048, 1, 'full', 'direct+one'),
]


@pytest.mark.parametrize('strided', [False, True])
@pytest.mark.parametrize('dtype', DTYPES, ids=['f32', 'f16', 'bf16'])
@pytest.mark.parametrize('rows,feat,ones,ws_kind,path', LINEAR_CASES)
def test_linear_statistic_matches_fp64(lib, dev, sms, rows, feat, ones, ws_kind, path, dtype, strided):
    code = DTYPE_CODE[dtype]
    ldx = feat + 5 if strided else feat
    g = torch.Generator(device=dev).manual_seed(rows * 31 + feat)
    xs = torch.randn(rows, ldx, device=dev, generator=g).to(dtype)
    x = xs[:, :feat]
    need = (lib.kfac_factor_linear_strided_workspace_bytes(rows, feat, ldx, ones) if strided
            else lib.kfac_factor_linear_workspace_bytes(rows, feat, ones))
    ws_bytes = need if ws_kind == 'full' else linear_pack_bytes(rows, feat, ones)
    got_path, engine = linear_path(rows, feat, ones, dtype, ws_bytes, sms)
    assert got_path == path, ('the dispatch copy puts this case elsewhere', got_path)
    X64 = x.double()
    if ones:
        X64 = torch.cat([X64, X64.new_ones(rows, 1)], 1)
    scale = 1.0 / rows

    def call(acc, ws, nbytes):
        if strided:
            return lib.kfac_factor_linear_strided(xs.data_ptr(), code, rows, feat, ldx, ones, scale, acc, ws, nbytes,
                                                  S())
        return lib.kfac_factor_linear(xs.data_ptr(), code, rows, feat, ones, scale, acc, ws, nbytes, S())
    check_statistic(lib, call, X64, scale, ws_bytes, dev, path, engine,
                    f'linear{"_strided" if strided else ""} {rows}x{feat}+{ones} {dtype} ws={ws_kind}')


def test_linear_statistic_boundaries(lib, dev):
    """rows = 0 changes nothing and launches nothing; rows >= 2^31 is refused before anything is launched."""
    from kfac_b200 import _cabi
    d, feat = 65, 64
    x = torch.randn(8, feat, device=dev)
    pad = 2 * d + 64
    arena, block = canary_arena(d * d, pad, dev)
    block.copy_(torch.randn(d * d, device=dev))
    before = arena.view(torch.int32).clone()
    ws = nan_ws(1 << 20, dev)
    torch.cuda.synchronize()
    n0 = lib.kfac_launch_count()
    assert lib.kfac_factor_linear(x.data_ptr(), 0, 0, feat, 1, 1.0, block.data_ptr(), ws.data_ptr(), 1 << 20, S()) == 0
    assert lib.kfac_factor_linear_strided(x.data_ptr(), 0, 0, feat, feat + 3, 1, 1.0, block.data_ptr(), None, 0,
                                          S()) == 0
    for rows in (1 << 31, (1 << 31) + 7):
        assert lib.kfac_factor_linear(x.data_ptr(), 0, rows, feat, 1, 1.0, block.data_ptr(), ws.data_ptr(), 1 << 20,
                                      S()) == _cabi.KFAC_ERR_BAD_ARG
    assert lib.kfac_launch_count() == n0
    torch.cuda.synchronize()
    assert torch.equal(arena.view(torch.int32), before)


# ---- kfac_factor_conv2d_gradout ------------------------------------------------------------------------------------

# (B, C, Ho, Wo, path with the queried workspace on a 132- or 114-SM part).  Without a workspace every case is read as
# stored in one split.  (B, C, 1, S): a Conv1d gradient.
GRADOUT_CASES = [
    (32, 512, 14, 14, 'direct+split'),          # ResNet-50 layer 3
    (32, 256, 56, 56, 'direct+split'),          # ResNet-50 layer 1
    (32, 2048, 7, 7, 'pack+one'),               # ResNet-50 layer 4: rows of 49 floats are packed
    (16, 2048, 7, 7, 'pack+one'),
    (16, 256, 1, 100, 'direct+split'),          # Conv1d, S = 100: read as stored
    (8, 128, 1, 75, 'pack+split'),              # Conv1d, S = 75: packed
]


@pytest.mark.parametrize('with_ws', [True, False])
@pytest.mark.parametrize('dtype', DTYPES, ids=['f32', 'f16', 'bf16'])
@pytest.mark.parametrize('B,Cc,Ho,Wo,path', GRADOUT_CASES)
def test_conv2d_gradout_statistic_matches_fp64(lib, dev, sms, B, Cc, Ho, Wo, path, dtype, with_ws):
    code = DTYPE_CODE[dtype]
    g = torch.Generator(device=dev).manual_seed(B * Cc + Ho * Wo)
    gr = torch.randn(B, Cc, Ho, Wo, device=dev, generator=g).to(dtype)
    ws_bytes = lib.kfac_factor_conv2d_gradout_workspace_bytes(B, Cc, Ho, Wo) if with_ws else 0
    got_path, engine = gradout_path(B, Cc, Ho, Wo, dtype, ws_bytes, sms)
    assert got_path == (path if with_ws else 'direct+one'), ('the dispatch copy puts this case elsewhere', got_path)
    X64 = gr.double().permute(0, 2, 3, 1).reshape(-1, Cc)
    scale = 1.0 / (B * float(Ho * Wo) ** 3)

    def call(acc, ws, nbytes):
        return lib.kfac_factor_conv2d_gradout(gr.data_ptr(), code, B, Cc, Ho, Wo, scale, acc, ws, nbytes, S())
    check_statistic(lib, call, X64, scale, ws_bytes, dev, got_path, engine,
                    f'conv2d_gradout {B}x{Cc}x{Ho}x{Wo} {dtype} ws={with_ws}')


# ---- kfac_factor_conv2d_input --------------------------------------------------------------------------------------

def test_conv2d_input_statistic_accumulates_at_resnet_layer4(lib, dev, sms):
    """ResNet-50's layer-4 3x3 conv (B = 32, C = 512, 7 x 7 maps, pad 1): d = 4608 through im2col and one SYRK split
    into a live slot.  The geometry x dtype matrix is test_gpu_conv_nd.py's."""
    from oracle import kfac_oracle as O
    B, Cc, H, W = 32, 512, 7, 7
    d, rows = Cc * 9, B * H * W
    g = torch.Generator(device=dev).manual_seed(4608)
    x = torch.randn(B, Cc, H, W, device=dev, generator=g)
    ws_bytes = lib.kfac_factor_conv2d_input_workspace_bytes(B, Cc, H, W, 3, 3, 1, 1, 1, 1, 0)
    assert ws_bytes == ld4(rows) * d * 4
    engine, splits = launch_cov(d, rows, 1, ld4(rows), True, True, False, sms)
    assert (engine, splits) == ('tc', 1)
    X64 = O.conv2d_patches(x.double(), (3, 3), (1, 1), (1, 1)).reshape(rows, d)
    scale = 1.0 / (B * float(H * W) ** 3)

    def call(acc, ws, nbytes):
        return lib.kfac_factor_conv2d_input(x.data_ptr(), 0, B, Cc, H, W, 3, 3, 1, 1, 1, 1, 0, scale, acc, ws, nbytes,
                                            S())
    check_statistic(lib, call, X64, scale, ws_bytes, dev, 'pack+one', engine, 'conv2d_input 32x512x7x7 k3 p1')


# ---- kfac_factor_ema -----------------------------------------------------------------------------------------------

def resnet50_factor_dims():
    from workloads import resnet50
    dims = []
    for m in resnet50().modules():
        if isinstance(m, torch.nn.Conv2d):
            dims += [m.in_channels * m.kernel_size[0] * m.kernel_size[1] + (m.bias is not None), m.out_channels]
        elif isinstance(m, torch.nn.Linear):
            dims += [m.in_features + (m.bias is not None), m.out_features]
    return dims


def test_ema_over_resnet50_factors_matches_fp64(lib, dev):
    """ResNet-50's 108 factors plus d = 1, 31, 33 and 4097 back to back in one arena: three launches of up to 40
    items, each decoding its own items and tile pairs.  Each factor against alpha f + (1 - alpha) inv_count (b + b^T)
    / 2 in fp64 within 2 ulp (2^-23 relative) of the magnitudes involved; every batch zeroed; the canaries before and
    after the items unchanged."""
    from kfac_b200 import _cabi
    dims = resnet50_factor_dims()
    assert len(dims) == 108
    for at, d in ((0, 1), (45, 31), (85, 33), (len(dims), 4097)):
        dims.insert(at, d)
    n = len(dims)
    assert n > 80                                    # three launches
    offs = np.concatenate([[0], np.cumsum([d * d for d in dims])]).tolist()
    total, pad = offs[-1], 4096
    alpha = f32(0.95)
    g = torch.Generator(device=dev).manual_seed(108)
    fac_arena, fac = canary_arena(total, pad, dev)
    bat_arena, bat = canary_arena(total, pad, dev)
    fac.copy_(torch.randn(total, device=dev, generator=g))
    bat.copy_(torch.randn(total, device=dev, generator=g))
    items = (_cabi.EmaItem * n)()
    firsts, inv_counts = [], []
    for i, d in enumerate(dims):
        first = int(i % 3 == 0)
        inv_count = f32(1.0 / (1 + i % 3 if i % 2 else 1 + (i + 1) % 3))
        if first:
            fac[offs[i]:offs[i + 1]].fill_(float('nan'))     # a first window does not read the factor
        firsts.append(first)
        inv_counts.append(inv_count)
        items[i] = _cabi.EmaItem(fac.data_ptr() + 4 * offs[i], bat.data_ptr() + 4 * offs[i], d, first, inv_count)
    assert set(inv_counts) == {f32(1.0), f32(0.5), f32(1.0 / 3)} and 0 < sum(firsts) < n
    fac0, bat0 = fac.clone(), bat.clone()
    torch.cuda.synchronize()
    n0 = lib.kfac_launch_count()
    assert lib.kfac_factor_ema(items, n, alpha, S()) == 0, lib.kfac_last_error()
    assert lib.kfac_launch_count() - n0 == ceil_div(n, 40)
    torch.cuda.synchronize()
    assert_canaries(fac_arena, pad, total, 'factor arena')
    assert_canaries(bat_arena, pad, total, 'batch arena')
    zeroed = bool((bat == 0).all())
    assert zeroed, 'a batch was not zeroed'
    worst = 0.0
    for i, d in enumerate(dims):
        b = bat0[offs[i]:offs[i + 1]].view(d, d).double()
        f = (torch.eye(d, dtype=torch.float64, device=dev) if firsts[i]
             else fac0[offs[i]:offs[i + 1]].view(d, d).double())
        beta = (1.0 - alpha) * inv_counts[i] / 2
        ref = alpha * f + beta * (b + b.t())
        mag = alpha * f.abs() + beta * (b.abs() + b.t().abs())
        got = fac[offs[i]:offs[i + 1]].view(d, d).double()
        ratio = float(((got - ref).abs() / (2.0 ** -23 * mag)).max())
        worst = max(worst, ratio)
        assert ratio <= 2.0, (i, d, firsts[i], inv_counts[i], ratio)
    print(f'kfac_factor_ema, {n} items of d <= {max(dims)}: worst error {worst:.3g} ulp (2^-23 relative)')


# ---- through the preconditioner ------------------------------------------------------------------------------------

class _WideNet(torch.nn.Module):
    """A ResNet-50 layer-4 3 x 3 conv on 7 x 7 maps beside a transformer-width Linear on (4, 256, 2048) tokens."""

    def __init__(self):
        super().__init__()
        self.conv = torch.nn.Conv2d(512, 512, 3, padding=1)
        self.fc = torch.nn.Linear(2048, 2304)

    def forward(self, x, t):
        return 0.5 * self.conv(x).square().sum() + 0.5 * self.fc(t).square().sum()


def test_preconditioner_factors_at_one_split_widths(dev):
    """One step with accumulation_steps=2 in fp32: A and G of the Linear (d = 2049, 2304) and the Conv2d (d = 4609,
    512) against the oracle's statistics and EMA of the inputs and output gradients the layers saw, in fp64.  The
    second micro-batch adds into the live window slot of each factor."""
    from kfac_b200.preconditioner import KFACPreconditioner
    from oracle import kfac_oracle as O
    torch.manual_seed(11)
    model = _WideNet().to(dev)
    alpha = 0.95
    pre = KFACPreconditioner(model, factor_decay=alpha, accumulation_steps=2, damping=0.003)
    seen = {model.conv: ([], []), model.fc: ([], [])}
    hooks = []
    for m, (xs, gs) in seen.items():
        hooks.append(m.register_forward_pre_hook(lambda mod, inp, xs=xs: xs.append(inp[0].detach().double())))
        hooks.append(m.register_full_backward_hook(lambda mod, gi, go, gs=gs: gs.append(go[0].detach().double())))
    for _ in range(2):
        model(torch.randn(32, 512, 7, 7, device=dev), torch.randn(4, 256, 2048, device=dev)).backward()
    pre.step()
    torch.cuda.synchronize()
    for h in hooks:
        h.remove()
    conv = lambda x: O.conv2d_a_factor(x, (3, 3), (1, 1), (1, 1), True)   # noqa: E731
    checks = [('conv A', model.conv, 'a', conv, 32 * 49), ('conv G', model.conv, 'g', O.conv2d_g_factor, 32 * 49),
              ('fc A', model.fc, 'a', lambda x: O.linear_a_factor(x, True), 1024),
              ('fc G', model.fc, 'g', O.linear_g_factor, 1024)]
    c = max(C_PATH.values())
    a32 = f32(alpha)
    for what, m, side, stat, K in checks:
        inputs = seen[m][0 if side == 'a' else 1]
        assert len(inputs) == 2
        window = sum(stat(t) for t in inputs)
        abs_window = sum(stat(t.abs()) for t in inputs)
        ref = O.ema_update(None, window.cpu(), 2, a32).to(dev)
        eye = torch.eye(ref.shape[0], dtype=torch.float64, device=dev)
        # the statistics, the fp32 scale of each call and the add of the second call, then the EMA's roundings
        bound = ((1 - a32) / 2 * U * (c * K + 3) * abs_window
                 + 4 * U * (a32 * eye + (1 - a32) / 2 * abs_window))
        layer = pre._layers[m][1]
        got = (layer.a_factor if side == 'a' else layer.g_factor).double()
        assert got.shape == ref.shape, what
        ratio = float(((got - ref).abs() / bound).max())
        print(f'preconditioner {what} (d = {ref.shape[0]}): worst error / bound {ratio:.3g}')
        assert ratio <= 1.0, (what, ratio)
