"""EKFAC's kernels (csrc/ekfac.cu) at ResNet-50 and transformer widths against fp64.

* the row writers (kfac_rows_*) bit for bit at model shapes: each value is fp32(x) * s with s = scale or
  fl32(scale / *loss_scale), which torch restates exactly;
* kfac_ekfac_statistics over every dispatch path of stat_layout in one call: projections in one launch (EPI_SQUARE),
  projections chained over column chunks (K = a or g > 1024) and squared by one pass, S_batch split into chains of
  <= 512 rows on the tensor cores, SIMT-class S_batch in chunks of 4096 rows, and the SIMT fallback of each problem.
  A Python copy of stat_layout names the path of each case, pins the workspace bytes on the host, and gives the
  kfac_launch_count() delta of the call;
* kfac_ekfac_update in each mode over the S_batch of those cases, and its scan of bad S_batch entries;
* the preconditioner (compute_method='ekfac') on a GPT-NeoX-125M block and a ResNet-50 layer-4 bottleneck, against an
  fp64 restatement of the method that uses the GPU's own bases.

The statistics start from rows as stored (fp32, post-ReLU X with exact zeros, G near 2^-20, a few dead units whose
basis block is the identity) in row buffers longer than N whose stale rows are NaN, with bases rounded to fp32 (not
exactly orthogonal), a NaN-byte workspace and S_batch inside a canary arena.  Each entry is checked against
    |S - S_ref| <= c u (L_x + L_g + L_s) S_abs,       u = 2^-24,
    S_abs = (1/N) ((|G||Qg|)^2)^T ((|X||Qa|)^2),
with S_ref and S_abs in fp64 from the operands as stored, L_* the longest chain plus the number of chains of each
product, and c one constant per path.  The entries of dead units have S_abs = 0 and must be exactly 0.  A dropped
column chunk or a block squared twice fails this bound where it would hide in a Frobenius norm."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_fro
from kfac_b200 import _cabi

U = 2.0 ** -24
# c of the bound per path of an item: S_batch on the tensor cores in one chain ('tc') or split into chains of <= 512
# rows ('tc-split'), either with a projection chained over column chunks ('chunked'), S_batch on the SIMT engine in
# one chain ('simt') or in chunks of 4096 rows ('simt-chunks').  The worst ratios over this file's cases on an H100
# 80GB HBM3 (132 SMs, 700 W) were 5.7e-4, 3.9e-4, 8.3e-5, 7.3e-4 and 9.3e-5; each c leaves less than 10x headroom
# above its path's worst ratio
C_PATH = {'tc': 4e-3, 'tc-split': 3e-3, 'chunked': 6e-4, 'simt': 5e-3, 'simt-chunks': 6e-4}
CANARY = 0x7FBADBAD                                   # a NaN pattern no kernel writes
CHAIN, SIMT_CHAIN = 512, 4096                         # ekfac.cu
SQDEV_BYTES = 16                                      # ekfac.cu SqDev: a pointer and a long long
FAKE = 0x7f0000100000                                 # a 256-byte aligned stand-in for a device pointer


def gpu(f):
    """A test that needs an H100: marked, and skipped where there is no CUDA device."""
    return pytest.mark.gpu(pytest.mark.skipif(not torch.cuda.is_available(), reason='needs a CUDA device')(f))


def S():
    return torch.cuda.current_stream().cuda_stream


def f32(x):
    """x rounded to fp32, as a Python float (the value a c_float argument carries)."""
    return float(np.float32(x))


def ceil_div(a, b):
    return -(-a // b)


def ld4(n):
    return (n + 3) // 4 * 4


def align256(n):
    return (n + 255) // 256 * 256


def bits(t):
    return t.contiguous().view(torch.int32)


# ---- the plan of kfac_ekfac_statistics (stat_layout, column_chunk and launch_grouped_gemm) -------------------------

def chain_splits(K):
    return ceil_div(K, 512) if K > 1024 else 1


def tc_ok(M, N, K, lda, ldb):
    """grouped_gemm_tc_ok for 16-byte aligned operands (workspace regions, arena entries and row buffers)."""
    return M >= 64 and N >= 64 and K >= 32 and lda % 4 == 0 and ldb % 4 == 0


def column_chunk(K, n, c):
    """(k0, k): chunk c of n over K columns, in whole k-blocks of 32."""
    cs = (ceil_div(K, n) + 31) // 32 * 32
    k0 = min(K, c * cs)
    return k0, max(0, min(K, k0 + cs) - k0)


def grouped_ws_bytes(count):
    fn = _cabi.load().kfac_stage_grouped_gemm_ws_bytes      # grouped_gemm_ws_bytes (a test entry of gemm_grouped.cu)
    fn.restype, fn.argtypes = C.c_size_t, [C.c_int]
    return fn(count)


class Spec:
    """One statistics item: its shape, its leading dimensions and the plan its name claims."""

    def __init__(self, name, a, g, N, wide, **expect):
        self.name, self.a, self.g, self.N = name, a, g, N
        # wide: row buffers, bases and S_batch with leading dimensions past ld4
        self.ldx, self.ldg = ld4(a) + 8 * wide, ld4(g) + 4 * wide
        self.ldqa, self.ldqg = ld4(a) + 4 * wide, ld4(g)
        self.lds = ld4(a) + 12 * wide
        self.expect = dict(ch_x=1, ch_g=1, sp_s=1, simt_s=False, tc_x=True, tc_g=True, tc_s=True)
        self.expect.update(expect)

    def __repr__(self):
        return f'{self.name} (a={self.a}, g={self.g}, N={self.N})'


def stat_plan(specs):
    """stat_layout: per item ch_x, ch_g (column chunks of each projection), sp_s (chains of S_batch), simt_s and the
    engine of each product; and the workspace bytes of the call."""
    off = 0

    def take(nbytes):
        nonlocal off
        o, off = off, align256(off + nbytes)
        return o
    n_s = 0
    for s in specs:
        tc = tc_ok(s.g, s.a, s.N, ld4(s.N), ld4(s.N))
        n_s += ceil_div(s.N, SIMT_CHAIN) if (not tc and s.N > 2 * SIMT_CHAIN) else 1
    take(grouped_ws_bytes(max(2 * len(specs), n_s)))
    take(SQDEV_BYTES * 2 * len(specs))
    for s in specs:
        take(s.a * ld4(s.N) * 4)
        take(s.g * ld4(s.N) * 4)
    plans = []
    for s in specs:
        p = dict(tc_x=tc_ok(s.a, s.N, s.a, s.ldqa, s.ldx), tc_g=tc_ok(s.g, s.N, s.g, s.ldqg, s.ldg),
                 tc_s=tc_ok(s.g, s.a, s.N, ld4(s.N), ld4(s.N)), sp_s=1, simt_s=False)
        p['ch_x'] = chain_splits(s.a) if p['tc_x'] else 1
        p['ch_g'] = chain_splits(s.g) if p['tc_g'] else 1
        chain = CHAIN if p['tc_s'] else SIMT_CHAIN
        if s.N > 2 * chain:
            p['sp_s'], p['simt_s'] = ceil_div(s.N, chain), not p['tc_s']
            take(p['sp_s'] * s.g * s.lds * 4)
        plans.append(p)
    return plans, off


def path_of(p):
    if p['ch_x'] > 1 or p['ch_g'] > 1:
        return 'chunked'
    if p['simt_s']:
        return 'simt-chunks'
    if not p['tc_s']:
        return 'simt'
    return 'tc-split' if p['sp_s'] > 1 else 'tc'


def engine_splits(K, splits):
    """(chain length, chains) of a tensor-core product split `splits` ways over K (launch_grouped_gemm)."""
    kb_total = ceil_div(K, 32)
    per = ceil_div(kb_total, splits)
    return per * 32, ceil_div(kb_total, per)


def chain_terms(s, p):
    """L_x + L_g + L_s: the longest chain plus the number of chains of each product of the item."""
    def proj(d, ch):
        return d + 1 if ch == 1 else column_chunk(d, ch, 0)[1] + ch
    if p['simt_s']:
        ls = SIMT_CHAIN + p['sp_s']
    elif p['sp_s'] > 1:
        ls = sum(engine_splits(s.N, p['sp_s']))
    else:
        ls = s.N + 1
    return proj(s.a, p['ch_x']) + proj(s.g, p['ch_g']) + ls


def grouped_launches(probs):
    """Launches of launch_grouped_gemm over (tensor cores?, splits) problems: one per SIMT problem, the wgmma kernel,
    and the reduce pass of the split problems."""
    tcs = [sp for tc, sp in probs if tc]
    return sum(not tc for tc, _ in probs) + bool(tcs) + any(sp > 1 for sp in tcs)


def stat_launches(specs, plans):
    rounds = max(max(p['ch_x'], p['ch_g']) for p in plans)
    n = 0
    for c in range(rounds):
        probs = []
        for s, p in zip(specs, plans):
            for d, ldq, ldr, ch in ((s.a, s.ldqa, s.ldx, p['ch_x']), (s.g, s.ldqg, s.ldg, p['ch_g'])):
                if c >= ch:
                    continue
                k = d if ch == 1 else column_chunk(d, ch, c)[1]
                if k:
                    probs.append((tc_ok(d, s.N, k, ldq, ldr), 1))
        n += grouped_launches(probs)
    n += rounds > 1                                       # square_all_kernel
    probs = []
    for s, p in zip(specs, plans):
        if p['simt_s']:
            probs += [(False, 1)] * p['sp_s']
            n += 1                                        # chunk_sum_kernel
        else:
            probs.append((p['tc_s'], p['sp_s']))
    return n + grouped_launches(probs)


def stat_specs():
    """The cases of the statistics call; odd ones take leading dimensions past ld4."""
    cases = [
        ('stem 7x7', 147, 64, 401408, dict(sp_s=784)),
        ('layer1 3x3', 576, 64, 100352, dict(sp_s=196)),
        ('layer4 3x3', 4608, 512, 1568, dict(ch_x=9, sp_s=4)),
        ('layer4 1x1 expand', 512, 2048, 1568, dict(ch_g=4, sp_s=4)),
        ('fc at batch 32', 2049, 1000, 32, dict(tc_x=False, tc_g=False)),      # SIMT projections, K = 2049 / 1000
        ('neox qkv', 769, 2304, 4096, dict(ch_g=5, sp_s=8)),
        ('neox mlp up', 769, 3072, 4096, dict(ch_g=6, sp_s=8)),
        ('neox mlp down', 3073, 768, 4096, dict(ch_x=7, sp_s=8)),
        ('both chunked', 2049, 1025, 1500, dict(ch_x=5, ch_g=3, sp_s=3)),
        ('a = 1024', 1024, 96, 600, {}),
        ('a = 1025', 1025, 96, 600, dict(ch_x=3)),                           # chunks of 352, 352 and 321 columns
        ('N = 1024', 160, 96, 1024, {}),
        ('N = 1025', 160, 96, 1025, dict(sp_s=3)),
        ('SIMT N = 8192', 100, 48, 8192, dict(tc_g=False, tc_s=False)),      # one SIMT chain of 8192 rows
        ('SIMT N = 8193', 100, 48, 8193, dict(tc_g=False, tc_s=False, sp_s=3, simt_s=True)),   # 4096 + 4096 + 1
        ('tiny N = 31', 80, 72, 31, dict(tc_x=False, tc_g=False, tc_s=False)),
        ('unaligned N = 777', 131, 97, 777, {}),
    ]
    return [Spec(name, a, g, N, i % 2 == 1, **e) for i, (name, a, g, N, e) in enumerate(cases)]


def fake_items(specs):
    items = (_cabi.EkfacStatItem * len(specs))()
    for i, s in enumerate(specs):
        items[i] = _cabi.EkfacStatItem(FAKE, FAKE, FAKE, FAKE, FAKE, s.N, s.a, s.g, s.ldx, s.ldg, s.ldqa, s.ldqg, s.lds)
    return items


# ---- 1. the plan, on the host ---------------------------------------------------------------------------------------

def test_plan_names_each_case_and_matches_the_workspace_query():
    lib = _cabi.load()
    specs = stat_specs()
    plans, total = stat_plan(specs)
    for s, p in zip(specs, plans):
        assert {k: p[k] for k in s.expect} == s.expect, ('the plan puts this case elsewhere', s, p)
    assert {path_of(p) for p in plans} == set(C_PATH)
    assert lib.kfac_ekfac_statistics_workspace_bytes(fake_items(specs), len(specs)) == total
    for s in specs:                                   # each item alone, as the bit-for-bit check calls it
        assert lib.kfac_ekfac_statistics_workspace_bytes(fake_items([s]), 1) == stat_plan([s])[1], s
    for sub in (specs[::2], specs[1::2], specs[-5:]):
        assert lib.kfac_ekfac_statistics_workspace_bytes(fake_items(sub), len(sub)) == stat_plan(sub)[1]
    # the boundaries the names claim
    assert [column_chunk(1025, 3, c)[1] for c in range(3)] == [352, 352, 321]
    assert [min(SIMT_CHAIN, 8193 - c * SIMT_CHAIN) for c in range(3)] == [4096, 4096, 1]
    assert sum(column_chunk(4608, 9, c)[1] for c in range(9)) == 4608
    # nine rounds of projections: the first holds every projection (tensor-core and SIMT, chunked or not), the later
    # ones the chunks of the seven chunked items, which end in different rounds
    assert sorted(max(p['ch_x'], p['ch_g']) for p in plans if path_of(p) == 'chunked') == [3, 4, 5, 5, 6, 7, 9]


# ---- 2. row writers, bit for bit -------------------------------------------------------------------------------------

DTYPES = {'f32': torch.float32, 'f16': torch.float16, 'bf16': torch.bfloat16}


def run_rows(call, n, d, ld, want, what):
    """call(out_ptr) into a NaN-filled buffer longer than n rows; the n x ld rows must be the bits of `want` (n x d)
    with exact zeros in [d, ld), and nothing may be written past them."""
    tail = 4099
    out = torch.full((n * ld + tail,), CANARY, dtype=torch.int32, device='cuda').view(torch.float32)
    rc = call(out.data_ptr())
    assert rc == 0, (what, _cabi.last_error())
    torch.cuda.synchronize()
    got = out[:n * ld].view(n, ld)
    same = torch.equal(bits(got[:, :d]), bits(want))
    assert same, (what, 'not the bits of fp32(x) * s')
    zero = bool((bits(got[:, d:]) == 0).all())
    assert zero, (what, 'padding columns are not exact zeros')
    untouched = bool((bits(out[n * ld:]) == CANARY).all())
    assert untouched, (what, 'written past N rows')


CONV_INPUT_CASES = [
    # (name, B, C, H, W, k, stride, pad): ResNet-50 at batch 32
    ('stem 7x7/s2', 32, 3, 224, 224, 7, 2, 3),          # C = 3, N = 401408
    ('layer1 3x3', 32, 64, 56, 56, 3, 1, 1),
    ('layer4 3x3', 32, 512, 7, 7, 3, 1, 1),              # a = 4608: 144 tile columns (145 with the ones column)
    ('downsample 1x1/s2', 32, 1024, 14, 14, 1, 2, 0),
]


@gpu
@pytest.mark.parametrize('dtype', list(DTYPES), ids=list(DTYPES))
@pytest.mark.parametrize('ones', [0, 1])
@pytest.mark.parametrize('case', CONV_INPUT_CASES, ids=[c[0] for c in CONV_INPUT_CASES])
def test_rows_conv2d_input_bits(case, ones, dtype):
    lib = _cabi.load()
    name, B, Cc, H, W, k, st, p = case
    g = torch.Generator(device='cuda').manual_seed(B * Cc + H)
    x = F.relu(torch.randn(B, Cc, H, W, device='cuda', generator=g)).to(DTYPES[dtype])
    Ho, Wo = (H + 2 * p - k) // st + 1, (W + 2 * p - k) // st + 1
    n, a = B * Ho * Wo, Cc * k * k
    d = a + ones
    ld = ld4(d) if ones else ld4(d) + 4
    scale = f32(1.0 / (Ho * Wo))
    s = torch.tensor(scale, dtype=torch.float32, device='cuda')
    u = F.unfold(x.float(), (k, k), padding=(p, p), stride=(st, st))          # B, C k k, Ho Wo
    want = torch.empty(n, d, device='cuda')
    want[:, :a] = u.transpose(1, 2).reshape(n, a) * s
    del u
    if ones:
        want[:, a] = s
    run_rows(lambda out: lib.kfac_rows_conv2d_input(x.data_ptr(), _cabi.DTYPE_CODE[x.dtype], B, Cc, H, W, k, k, st, st,
                                                    p, p, ones, scale, out, ld, S()),
             n, d, ld, want, f'conv2d_input {name} ones={ones} {dtype}')


@gpu
@pytest.mark.parametrize('dtype', list(DTYPES), ids=list(DTYPES))
def test_rows_conv2d_gradout_bits_with_device_loss_scale(dtype):
    """112 x 112 maps (ResNet-50's stem output) unscaled by a loss scale read on the device: s = fl32(scale / ls)."""
    lib = _cabi.load()
    B, Cc, Ho, Wo = 32, 64, 112, 112
    n = B * Ho * Wo
    gen = torch.Generator(device='cuda').manual_seed(112)
    gr = (torch.randn(B, Cc, Ho, Wo, device='cuda', generator=gen) * 3000.0).to(DTYPES[dtype])
    ls = torch.tensor([3000.0], device='cuda')
    scale = f32(1.0 / (Ho * Wo))
    s = torch.tensor(scale, dtype=torch.float32, device='cuda') / ls[0]
    want = gr.float().permute(0, 2, 3, 1).reshape(n, Cc) * s
    for ld in (Cc, Cc + 8):
        run_rows(lambda out: lib.kfac_rows_conv2d_gradout(gr.data_ptr(), _cabi.DTYPE_CODE[gr.dtype], B, Cc, Ho, Wo,
                                                          scale, ls.data_ptr(), out, ld, S()),
                 n, Cc, ld, want, f'conv2d_gradout 112x112 {dtype} ld={ld}')


LINEAR_ROW_CASES = [
    # (name, rows, ldx, col0, features, ones, loss scale): slices of a fused QKV output and GPT-NeoX MLP rows
    ('qkv slice k', 4096, 3 * 768, 768, 768, 1, None),
    ('qkv slice v, grad', 4096, 3 * 768, 1536, 768, 0, 3000.0),
    ('mlp up input', 4096, 768, 0, 768, 1, None),
    ('mlp down input', 4096, 3072, 0, 3072, 1, None),
    ('mlp up grad', 4096, 3072, 0, 3072, 0, 3000.0),
]


@gpu
@pytest.mark.parametrize('dtype', ['f16', 'bf16'])
@pytest.mark.parametrize('case', LINEAR_ROW_CASES, ids=[c[0] for c in LINEAR_ROW_CASES])
def test_rows_linear_strided_bits(case, dtype):
    lib = _cabi.load()
    name, rows, ldx, col0, feat, ones, lsv = case
    gen = torch.Generator(device='cuda').manual_seed(rows + ldx + col0)
    buf = torch.randn(rows, ldx, device='cuda', generator=gen).to(DTYPES[dtype])
    x = buf[:, col0:col0 + feat]
    d = feat + ones
    ld = ld4(d) + 4 * ones
    scale = f32(1.0 / rows if ones else 0.7)
    s = torch.tensor(scale, dtype=torch.float32, device='cuda')
    ls = None
    if lsv is not None:
        ls = torch.tensor([lsv], device='cuda')
        s = s / ls[0]
    want = torch.empty(rows, d, device='cuda')
    want[:, :feat] = x.float() * s
    if ones:
        want[:, feat] = s
    run_rows(lambda out: lib.kfac_rows_linear_strided(x.data_ptr(), _cabi.DTYPE_CODE[x.dtype], rows, feat, ldx, ones,
                                                      scale, ls.data_ptr() if ls is not None else None, out, ld, S()),
             rows, d, ld, want, f'linear_strided {name} {dtype}')


# ---- 3. kfac_ekfac_statistics against fp64 ---------------------------------------------------------------------------

def dead_units(d):
    return sorted({0, d // 2, d - 1})


def basis_T(d, ld, gen):
    """Q^T (d x ld, fp32) of a random orthogonal basis in fp64 whose dead units keep an identity block."""
    dead = dead_units(d)
    live = torch.tensor([i for i in range(d) if i not in dead], device='cuda')
    q = torch.eye(d, dtype=torch.float64, device='cuda')
    r, _ = torch.linalg.qr(torch.randn(len(live), len(live), dtype=torch.float64, device='cuda', generator=gen))
    q[live[:, None], live[None, :]] = r
    out = torch.zeros(d, ld, device='cuda')
    out[:, :d] = q.t().float()
    return out


def row_buffer(N, d, ld, values):
    """N + 37 rows of ld floats: the first N hold `values` (zeros in the padding columns), the rest are stale NaN."""
    buf = torch.full((N + 37, ld), float('nan'), device='cuda')
    buf[:N] = 0.0
    buf[:N, :d] = values
    return buf


class StatRun:
    """The cases of stat_specs on the device, S_batch of each inside one canary arena, and the full call's result."""

    def __init__(self, lib):
        self.lib = lib
        self.specs = stat_specs()
        self.plans = stat_plan(self.specs)[0]
        self.X, self.G, self.qaT, self.qgT, self.offs = [], [], [], [], []
        off = 256
        for i, s in enumerate(self.specs):
            gen = torch.Generator(device='cuda').manual_seed(7000 + i)
            x = F.relu(torch.randn(s.N, s.a, device='cuda', generator=gen))                 # post-ReLU: exact zeros
            x[:, dead_units(s.a)] = 0.0
            self.X.append(row_buffer(s.N, s.a, s.ldx, x))
            del x
            gr = torch.randn(s.N, s.g, device='cuda', generator=gen) * 2.0 ** -20
            gr[:, dead_units(s.g)] = 0.0
            self.G.append(row_buffer(s.N, s.g, s.ldg, gr))
            del gr
            self.qaT.append(basis_T(s.a, s.ldqa, gen))
            self.qgT.append(basis_T(s.g, s.ldqg, gen))
            self.offs.append(off)
            off = align256(4 * (off + s.g * s.lds) + 4 * 100) // 4       # 100+ canaries between blocks
        self.arena_len = off + 256

    def items(self, idx, arena):
        items = (_cabi.EkfacStatItem * len(idx))()
        for j, i in enumerate(idx):
            s = self.specs[i]
            items[j] = _cabi.EkfacStatItem(self.X[i].data_ptr(), self.G[i].data_ptr(), self.qaT[i].data_ptr(),
                                           self.qgT[i].data_ptr(), arena.data_ptr() + 4 * self.offs[i], s.N, s.a,
                                           s.g, s.ldx, s.ldg, s.ldqa, s.ldqg, s.lds)
        return items

    def arena(self):
        return torch.full((self.arena_len,), CANARY, dtype=torch.int32, device='cuda').view(torch.float32)

    def call(self, idx, ws_bytes=None):
        """kfac_ekfac_statistics over the items idx into a fresh arena with a NaN-byte workspace: (rc, arena bits,
        launches)."""
        arena = self.arena()
        items = self.items(idx, arena)
        need = self.lib.kfac_ekfac_statistics_workspace_bytes(items, len(idx))
        nbytes = need if ws_bytes is None else ws_bytes(need)
        ws = torch.full((max(nbytes, 1),), 255, dtype=torch.uint8, device='cuda')
        torch.cuda.synchronize()
        n0 = self.lib.kfac_launch_count()
        rc = self.lib.kfac_ekfac_statistics(items, len(idx), ws.data_ptr(), nbytes, S())
        n1 = self.lib.kfac_launch_count()
        torch.cuda.synchronize()
        del ws
        return rc, bits(arena).clone(), n1 - n0

    def block(self, arena_bits, i):
        s = self.specs[i]
        return arena_bits[self.offs[i]:self.offs[i] + s.g * s.lds].view(s.g, s.lds)

    def reference(self, i):
        """(S_ref, S_abs) in fp64 from the operands as stored."""
        s = self.specs[i]
        out = []
        for rows, qT, d in ((self.X[i], self.qaT[i], s.a), (self.G[i], self.qgT[i], s.g)):
            r = rows[:s.N, :d].double()
            q = qT[:, :d].double().t()                        # Q[k, f] = Q^T[f, k]
            out.append(((r @ q).square_(), (r.abs() @ q.abs()).square_()))
            del r, q
        (xh, xa), (gh, ga) = out
        return (gh.t() @ xh) / s.N, (ga.t() @ xa) / s.N


@pytest.fixture(scope='module')
def stat_run():
    lib = _cabi.load()
    run = StatRun(lib)
    run.full = run.call(list(range(len(run.specs))))
    return run


@gpu
def test_statistics_against_fp64(stat_run):
    """Every case in one call: the launches the plan gives, the canaries outside each block, the padding columns of
    S_batch 0 or untouched, S_batch >= 0 and each entry within its path's bound."""
    run = stat_run
    rc, arena, launches = run.full
    assert rc == 0, _cabi.last_error()
    assert launches == stat_launches(run.specs, run.plans), launches
    inside = torch.zeros(run.arena_len, dtype=torch.bool, device='cuda')
    for i, s in enumerate(run.specs):
        inside[run.offs[i]:run.offs[i] + s.g * s.lds] = True
    canaries = bool((arena[~inside] == CANARY).all())
    assert canaries, 'written outside the S_batch blocks'
    worst = {}
    for i, s in enumerate(run.specs):
        blk = run.block(arena, i)
        pad = blk[:, s.a:]
        pad_ok = bool(((pad == 0) | (pad == CANARY)).all())
        assert pad_ok, (s, 'padding columns of S_batch hold neither 0 nor what was there')
        got = blk[:, :s.a].contiguous().view(torch.float32).double()
        finite = bool(torch.isfinite(got).all())
        assert finite, s
        nonneg = bool((got >= 0).all())
        assert nonneg, (s, 'S_batch < 0')
        ref, sabs = run.reference(i)
        dead = sabs == 0
        assert bool(dead.any()), s                        # the dead units
        exact = bool((got[dead] == 0).all())
        assert exact, (s, 'an entry of a dead unit is not 0')
        path = path_of(run.plans[i])
        unit = U * chain_terms(s, run.plans[i]) * sabs
        ratio = float(((got - ref).abs()[~dead] / unit[~dead]).max())
        del ref, sabs, unit, got
        worst[path] = max(worst.get(path, 0.0), ratio)
        print(f'{s}: {path} {run.plans[i]}, L = {chain_terms(s, run.plans[i])}, worst ratio {ratio:.3g} '
              f'(c = {C_PATH[path]})')
        assert ratio <= C_PATH[path], (s, path, ratio)
    print('worst ratio per path on', torch.cuda.get_device_name(), worst)


@gpu
def test_statistics_same_bits_again_and_alone(stat_run):
    """A second call gives the same bits, and each item alone gives the bits it has in the full list."""
    run = stat_run
    rc, arena, _ = run.full
    assert rc == 0
    rc2, again, _ = run.call(list(range(len(run.specs))))
    assert rc2 == 0, _cabi.last_error()
    assert torch.equal(arena, again), 'not the same bits in a repeat call'
    del again
    for i, s in enumerate(run.specs):
        rc1, alone, n = run.call([i])
        assert rc1 == 0, (s, _cabi.last_error())
        assert n == stat_launches([s], [run.plans[i]]), (s, n)
        assert torch.equal(run.block(alone, i), run.block(arena, i)), (s, 'other bits alone than in the list')


@gpu
def test_statistics_short_workspace_touches_nothing(stat_run):
    run = stat_run
    before = bits(run.arena()).clone()
    rc, arena, launches = run.call(list(range(len(run.specs))), ws_bytes=lambda need: need - 1)
    assert rc == _cabi.KFAC_ERR_WORKSPACE, rc
    assert launches == 0
    assert torch.equal(arena, before)


# ---- 4. kfac_ekfac_update at width ----------------------------------------------------------------------------------

def ulps(a, b):
    """Distance in units in the last place between non-negative fp32 tensors."""
    return (bits(a).long() - bits(b).long()).abs()


class UpdateSet:
    """The S_batch of the statistics call as update items, with a previous S (padding columns canaries) and
    eigenvalues whose products are of S's magnitude."""

    def __init__(self, run):
        _, arena, _ = run.full
        self.specs = run.specs
        self.Sb = [run.block(arena, i).clone().view(torch.float32) for i in range(len(run.specs))]
        self.S0, self.dg, self.da = [], [], []
        for i, s in enumerate(self.specs):
            gen = torch.Generator(device='cuda').manual_seed(9000 + i)
            s0 = torch.full((s.g, s.lds), CANARY, dtype=torch.int32, device='cuda').view(torch.float32)
            s0[:, :s.a] = self.Sb[i][:, :s.a] * (0.5 + 1.5 * torch.rand(s.g, s.a, device='cuda', generator=gen))
            self.S0.append(s0)
            mag = float(self.Sb[i][:, :s.a].mean()) ** 0.5
            self.dg.append(mag * (0.1 + torch.rand(s.g, device='cuda', generator=gen)))
            self.da.append(mag * (0.1 + torch.rand(s.a, device='cuda', generator=gen)))
        self.damping = f32(float(torch.stack([b[:, :s.a].mean() for b, s in zip(self.Sb, self.specs)]).mean()))

    def run(self, lib, mode, alpha, skipped=None, Sb=None):
        Sb = Sb or self.Sb
        s_new = [t.clone() for t in self.S0]
        dgda = [torch.full_like(t, float('nan')) for t in self.S0]
        items = (_cabi.EkfacUpdateItem * len(self.specs))()
        for i, s in enumerate(self.specs):
            items[i] = _cabi.EkfacUpdateItem(s_new[i].data_ptr(), Sb[i].data_ptr(), self.dg[i].data_ptr(),
                                             self.da[i].data_ptr(), dgda[i].data_ptr(), s.g, s.a, s.lds, None, None)
        need = lib.kfac_ekfac_update_workspace_bytes(len(self.specs))
        ws = torch.full((need,), 255, dtype=torch.uint8, device='cuda')
        rc = lib.kfac_ekfac_update(items, len(self.specs), alpha, mode, self.damping,
                                   skipped.data_ptr() if skipped is not None else None, ws.data_ptr(), need, S())
        assert rc == 0, _cabi.last_error()
        torch.cuda.synchronize()
        return s_new, dgda

    def want_S(self, i, mode, alpha):
        """S by the mode's formula in fp64, rounded to fp32."""
        a = self.specs[i].a
        K = _cabi
        if mode == K.KFAC_EKFAC_KEEP:
            return self.S0[i][:, :a]
        if mode == K.KFAC_EKFAC_RESET:
            return self.Sb[i][:, :a]
        if mode == K.KFAC_EKFAC_SEED:
            return torch.outer(self.dg[i].double(), self.da[i].double()).float()
        return (alpha * self.S0[i][:, :a].double() + (1.0 - alpha) * self.Sb[i][:, :a].double()).float()


@pytest.fixture(scope='module')
def update_set(stat_run):
    return UpdateSet(stat_run)


@gpu
@pytest.mark.parametrize('mode', ['keep', 'ema', 'reset', 'seed'])
def test_update_modes_at_width(stat_run, update_set, mode):
    """All items in one call into a NaN dgda: S within 1 ulp of its formula, dgda within 1 ulp of 1 / (S + damping)
    from the kernel's own S, the padding columns of dgda 0 and of S untouched; the seed gives kfac_dgda's bits."""
    lib = _cabi.load()
    K = _cabi
    code = {'keep': K.KFAC_EKFAC_KEEP, 'ema': K.KFAC_EKFAC_EMA, 'reset': K.KFAC_EKFAC_RESET, 'seed': K.KFAC_EKFAC_SEED}
    m = code[mode]
    up = update_set
    alpha = f32(0.95)
    skipped = torch.zeros(1, dtype=torch.int64, device='cuda')
    s_new, dgda = up.run(lib, m, alpha, skipped)
    assert skipped.item() == 0
    worst_s = worst_d = 0
    for i, s in enumerate(up.specs):
        a = s.a
        exact_S = m != K.KFAC_EKFAC_EMA
        e = int(ulps(s_new[i][:, :a], up.want_S(i, m, alpha)).max())
        worst_s = max(worst_s, e)
        assert e <= (0 if exact_S else 1), (s, mode, 'S off by', e)
        kept = torch.equal(bits(s_new[i][:, a:]), bits(up.S0[i][:, a:]))
        assert kept, (s, mode, 'padding columns of S written')
        den = (torch.outer(up.dg[i].double(), up.da[i].double()) if m == K.KFAC_EKFAC_SEED
               else s_new[i][:, :a].double()) + up.damping
        e = int(ulps(dgda[i][:, :a], (1.0 / den).float()).max())
        worst_d = max(worst_d, e)
        assert e <= 1, (s, mode, 'dgda off by', e)
        zero = bool((bits(dgda[i][:, a:]) == 0).all())
        assert zero, (s, mode, 'padding columns of dgda are not 0')
        if m == K.KFAC_EKFAC_SEED:
            ref = torch.full_like(dgda[i], float('nan'))
            assert lib.kfac_dgda(up.dg[i].data_ptr(), up.da[i].data_ptr(), s.g, a, up.damping, ref.data_ptr(), s.lds,
                                 S()) == 0
            torch.cuda.synchronize()
            assert torch.equal(bits(ref), bits(dgda[i])), (s, 'seed is not the bits of kfac_dgda')
    print(f'update {mode}: worst S {worst_s} ulp, worst dgda {worst_d} ulp')


@gpu
@pytest.mark.parametrize('mode', ['ema', 'reset'])
def test_update_scan_drops_only_the_flagged_item(stat_run, update_set, mode):
    """An inf in the last entry (g-1, a-1) of the largest item drops its window (counted once); NaN in the padding
    columns of another item's S_batch is not an entry and drops nothing."""
    lib = _cabi.load()
    K = _cabi
    m = K.KFAC_EKFAC_EMA if mode == 'ema' else K.KFAC_EKFAC_RESET
    up = update_set
    alpha = f32(0.95)
    Sb = [t.clone() for t in up.Sb]
    big = max(range(len(up.specs)), key=lambda i: up.specs[i].g * up.specs[i].a)
    s = up.specs[big]
    Sb[big][s.g - 1, s.a - 1] = float('inf')
    padded = next(i for i, t in enumerate(up.specs) if t.lds > t.a and i != big)
    Sb[padded][:, up.specs[padded].a:] = float('nan')
    skipped = torch.zeros(1, dtype=torch.int64, device='cuda')
    s_new, dgda = up.run(lib, m, alpha, skipped, Sb)
    assert skipped.item() == 1
    for i, t in enumerate(up.specs):
        a = t.a
        if i == big:
            want = up.S0[i][:, :a] if m == K.KFAC_EKFAC_EMA else up.want_S(i, K.KFAC_EKFAC_SEED, alpha)
            assert torch.equal(bits(s_new[i][:, :a]), bits(want)), (t, 'a dropped window changed S')
        else:
            e = int(ulps(s_new[i][:, :a], up.want_S(i, m, alpha)).max())
            assert e <= (1 if m == K.KFAC_EKFAC_EMA else 0), (t, mode, 'not updated', e)
        finite = bool(torch.isfinite(dgda[i][:, :a]).all())
        assert finite, t


# ---- 5. the preconditioner at bench widths --------------------------------------------------------------------------

class _Rec:
    """Every layer's input and output gradient of the current step (hooks after the preconditioner's)."""

    def __init__(self, pre):
        self.inp, self.gout = {}, {}
        for m in pre._layers:
            m.register_forward_pre_hook(lambda mod, i: self.inp.__setitem__(mod, i[0].detach().clone()))
            m.register_full_backward_hook(lambda mod, gi, go: self.gout.__setitem__(mod, go[0].detach().clone()))


def _rows64(module, x, gout):
    """fp64 (x_r, g_r) of one layer on the device: conv rows scaled by 1 / (Ho Wo), the ones column for a bias."""
    if isinstance(module, torch.nn.Conv2d):
        Ho, Wo = gout.shape[2], gout.shape[3]
        u = F.unfold(x.double(), module.kernel_size, padding=module.padding, stride=module.stride)
        X = u.transpose(1, 2).reshape(-1, u.shape[1])
        G = gout.double().permute(0, 2, 3, 1).reshape(-1, gout.shape[1])
        sp = float(Ho * Wo)
    else:
        X = x.double().reshape(-1, x.shape[-1])
        G = gout.double().reshape(-1, gout.shape[-1])
        sp = 1.0
    if module.bias is not None:
        X = torch.cat([X, X.new_ones(X.shape[0], 1)], 1)
    return X / sp, G / sp


class _Oracle:
    """fp64 EKFAC state per layer, driven by the GPU's own bases; S_batch by the matrix formula."""

    def __init__(self):
        self.S = {}

    def step(self, pre, rec, inverse_step, alpha, damping, grads):
        out = {}
        for m, (name, layer) in pre._layers.items():
            Qa, Qg = layer.qa.double(), layer.qg.double()
            X, G = _rows64(m, rec.inp[m], rec.gout[m])
            Sb = ((G @ Qg).square().t() @ (X @ Qa).square()) / X.shape[0]
            self.S[name] = Sb if inverse_step else alpha * self.S[name] + (1 - alpha) * Sb
            out[name] = Qg @ ((Qg.t() @ grads[name] @ Qa) / (self.S[name] + damping)) @ Qa.t()
        return out


def _grad_matrix(module):
    g = module.weight.grad.reshape(module.weight.grad.size(0), -1)
    if module.bias is not None:
        g = torch.cat([g, module.bias.grad.view(-1, 1)], 1)
    return g.detach().double()


def _run_three_steps(model, make_batch, rows, damping, alpha=0.95):
    """factor_update_steps=1, inv_update_steps=2 over 3 steps on new batches: reset, EMA, reset.  The weights stay put
    (with a small damping the preconditioned step is large enough to blow the activations past the scan's 1e15), and
    the loss is a mean over the `rows` samples or tokens; no window may be dropped."""
    from kfac_b200.preconditioner import KFACPreconditioner
    pre = KFACPreconditioner(model, compute_method='ekfac', factor_update_steps=1, inv_update_steps=2,
                             damping=damping, factor_decay=alpha, kl_clip=None)
    rec = _Rec(pre)
    oracle = _Oracle()
    a32 = f32(alpha)
    for step in range(3):
        model.zero_grad()
        out = model(make_batch(step))
        (0.5 * out.square().sum() / rows).backward()
        grads = {name: _grad_matrix(m) for m, (name, _) in pre._layers.items()}
        pre.step()
        torch.cuda.synchronize()
        assert pre.skipped_factor_updates == 0, step
        want = oracle.step(pre, rec, step % 2 == 0, a32, damping, grads)
        for m, (name, layer) in pre._layers.items():
            es = rel_fro(layer._S[:, :layer.a_dim], oracle.S[name])
            ep = rel_fro(_grad_matrix(m), want[name])          # kl_clip=None: the gradient written back is P
            print(f'step {step} {name} (a = {layer.a_dim}, g = {layer.g_dim}): S {es:.2e}, P {ep:.2e}')
            assert es < 1e-4, (step, name, es)
            assert ep < 1e-3, (step, name, ep)
    return pre


@gpu
def test_neox_block_at_bench_width():
    """A GPT-NeoX-125M block (d = 768, ffn = 3072) on 4 x 1024 tokens: a = 769 / 3073, g = 2304 / 768 / 3072."""
    from workloads import NeoXBlock
    torch.manual_seed(12)
    model = NeoXBlock(768).cuda()
    gen = torch.Generator(device='cuda').manual_seed(12)
    xs = [torch.randn(4, 1024, 768, device='cuda', generator=gen) for _ in range(3)]
    pre = _run_three_steps(model, lambda s: xs[s], rows=4096, damping=1e-5)
    assert len(pre._layers) == 4


@gpu
def test_resnet50_layer4_bottleneck_at_bench_width():
    """A ResNet-50 layer-4 bottleneck (2048 -> 512 -> 512 -> 2048) on 7 x 7 maps at batch 32: N = 1568 rows, a = 2048
    / 4608 / 512."""
    from workloads import _Bottleneck
    torch.manual_seed(13)
    model = _Bottleneck(2048, 512, 1).cuda()
    gen = torch.Generator(device='cuda').manual_seed(13)
    xs = [F.relu(torch.randn(32, 2048, 7, 7, device='cuda', generator=gen)) for _ in range(3)]
    pre = _run_three_steps(model, lambda s: xs[s], rows=32, damping=1e-6)
    assert len(pre._layers) == 3
