"""The kernels of an inverse step after the eigensolver, against fp64 at the widths models reach.

* kfac_inverse_from_eigh (the inverse method's (F + damping I)^-1 from Q and d): from fp32 inputs against fp64, on the
  SIMT and the tensor-core path, below and above the width (1024) where the reduction runs as chains of <= 512; the
  same bits in every call; nothing written outside the result;
* the eigensolver followed by kfac_inverse_from_eigh against torch.linalg.inv(F64 + damping I) at bench widths;
* kfac_transpose (the K-major copy a rank builds from a received eigenbasis): bit for bit, and equal to the QT the
  eigensolver writes for the same Q;
* kfac_diag_snapshot (the snapshot and status check of a vector factor): bit for bit over several passes of its
  grid-stride loop, and the status bit for every kind of rejected entry;
* kfac_dgda at a bench shape;
* the whole preconditioner with compute_method='inverse' on an MLP whose factors are wider than 1024.

Every output buffer and every workspace starts as NaN (workspaces: bytes of 255).  All kernel calls go through the C
ABI, the way the preconditioner makes them."""
import copy
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import rel_fro
from kfac_like import kfac_like_sequence

pytestmark = pytest.mark.gpu

NAN = float('nan')


@pytest.fixture(scope='module')
def lib():
    from kfac_b200 import _cabi
    return _cabi.load()


@pytest.fixture(scope='module')
def dev():
    assert torch.cuda.is_available()
    return torch.device('cuda:0')


@pytest.fixture
def no_tf32():
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def S():
    return torch.cuda.current_stream().cuda_stream


def ld4(n):
    return (n + 3) // 4 * 4


def bits(x):
    return x.contiguous().view(torch.int32)


def f32(x):
    """x rounded to fp32, as a Python float (the value a c_float argument carries)."""
    return float(np.float32(x))


def nan_ws(nbytes, dev):
    return torch.full((nbytes,), 255, dtype=torch.uint8, device=dev)     # all-ones bytes: NaN floats


def stored(x, ld):
    """(r, c) fp32 in storage with leading dimension ld and NaN padding columns."""
    r, c = x.shape
    out = torch.full((r, ld), NAN, device=x.device)
    out[:, :c] = x
    return out


def assert_nan_outside(buf, rows, cols, what):
    """Columns [cols, ld) of the first `rows` rows and every row after them are still NaN."""
    assert torch.isnan(buf[:rows, cols:]).all(), (what, 'padding columns written')
    assert torch.isnan(buf[rows:]).all(), (what, 'rows past the result written')


def run_eigh(lib, dev, F):
    """One kfac_eigh_batched call: Q and QT (n x ld4(n), NaN outside n x n) and d."""
    from kfac_b200 import _cabi
    n = F.shape[0]
    ld = ld4(n)
    Q = torch.full((n, ld), NAN, device=dev)
    QT = torch.full((n, ld), NAN, device=dev)
    d = torch.full((n,), NAN, device=dev)
    Fd = F.to(dev).contiguous()
    items = (_cabi.EighItem * 1)(_cabi.EighItem(Fd.data_ptr(), Q.data_ptr(), QT.data_ptr(), d.data_ptr(), n, ld, None))
    ns = (C.c_int * 1)(n)
    need = lib.kfac_eigh_workspace_bytes(ns, 1)
    ws = nan_ws(need, dev)
    assert lib.kfac_eigh_batched(items, 1, ws.data_ptr(), need, 0, 0.0, S()) == 0, lib.kfac_last_error()
    host = torch.zeros(1, dtype=torch.int32).pin_memory()
    assert lib.kfac_eigh_status(ws.data_ptr(), host.data_ptr(), S()) == 0
    torch.cuda.synchronize()
    assert int(host.item()) == 0, n
    return Q, QT, d


# ---- kfac_inverse_from_eigh from fp32 inputs -------------------------------------------------------------------------

# SIMT path (n < 64), first tensor-core size, the last unsplit reduction (1024), the first split one (1025), n mod 4 = 1,
# the bench widths (ResNet-50 2049 / 4608, GPT-NeoX-125M 3073) and KFAC_EIGH_MAX_N
INV_SIZES = [1, 3, 63, 64, 65, 129, 1000, 1024, 1025, 1153, 2049, 3073, 4608, 8192]
_bases = {}


def basis(n, dev):
    """fp32 orthogonal Q (QR of an fp64 Gaussian, rounded) and fp32 d >= 0 spread over 1 .. 1e-7 in random order, an
    eighth of it exactly 0."""
    if n not in _bases:
        g = torch.Generator(device=dev).manual_seed(1000 + n)
        q, _ = torch.linalg.qr(torch.randn(n, n, dtype=torch.float64, device=dev, generator=g))
        d = torch.logspace(0, -7, n, dtype=torch.float64, device=dev)
        d = d[torch.randperm(n, device=dev, generator=g)]
        d[torch.randperm(n, device=dev, generator=g)[:n // 8]] = 0.0
        _bases.clear()                  # one size at a time: n = 8192 alone takes 0.8 GB in fp64
        _bases[n] = (q.float().contiguous(), d.float().contiguous())
    return _bases[n]


def ref_inverse(Q, d, damping):
    """(Q diag(1 / (d + damping)) Q^T) in fp64 from the fp32 inputs."""
    Q64 = Q.double()
    return (Q64 / (d.double() + damping)) @ Q64.t()


def call_inverse(lib, Qs, ldq, d, n, damping, ld_inv, ws_offset=0, ws_bytes=None):
    """kfac_inverse_from_eigh into a NaN-filled (n + 1) x ld_inv buffer (one row past the result) with a NaN-filled
    workspace of ws_bytes (default n * ldq floats) at byte offset ws_offset; returns (rc, buffer)."""
    dev = Qs.device
    need = n * ldq * 4 if ws_bytes is None else ws_bytes
    ws = nan_ws(need + ws_offset + 16, dev)
    inv = torch.full((n + 1, ld_inv), NAN, device=dev)
    rc = lib.kfac_inverse_from_eigh(Qs.data_ptr(), ldq, d.data_ptr(), n, damping, inv.data_ptr(), ld_inv,
                                    ws.data_ptr() + ws_offset, need, S())
    torch.cuda.synchronize()
    return rc, inv


def check_inverse(inv, ref, n, what):
    """The tolerances of the wgmma engine's fp64 tests (test_gpu_tc_gemm.py), and nothing written outside n x n."""
    got = inv[:n, :n].double()
    e = float((got - ref).norm() / ref.norm())
    e_max = float((got - ref).abs().max() / ref.abs().max())
    assert e < 3e-6 + 4e-9 * n, (what, 'rel-fro', e)
    assert e_max < 2e-5 + 1e-8 * n, (what, 'max entry', e_max)
    assert_nan_outside(inv, n, n, what)


@pytest.mark.parametrize('n', INV_SIZES)
def test_inverse_from_eigh_matches_fp64(lib, dev, n):
    Q, d = basis(n, dev)
    dmax = float(d.max())
    for rel in (1e-3, 1e-7):
        damping = f32(rel * dmax)
        ref = ref_inverse(Q, d, damping)
        for ldq in (ld4(n), ld4(n) + 8):
            Qs = stored(Q, ldq)
            for ld_inv in (ldq, n + 1):             # n + 1 is odd: the scalar stores of the epilogue
                what = (n, rel, ldq, ld_inv)
                rc, inv = call_inverse(lib, Qs, ldq, d, n, damping, ld_inv)
                assert rc == 0, (what, lib.kfac_last_error())
                check_inverse(inv, ref, n, what)


def test_inverse_from_eigh_simt_at_split_width(lib, dev):
    """n = 1025 on the SIMT engine: rows of ldq = 1025 floats are not 16-byte aligned, and so is a workspace at a
    4-byte offset; both must give the damped inverse with nothing written outside it."""
    n = 1025
    Q, d = basis(n, dev)
    damping = f32(1e-3 * float(d.max()))
    ref = ref_inverse(Q, d, damping)
    for ldq, off in ((n, 0), (ld4(n), 4)):
        rc, inv = call_inverse(lib, stored(Q, ldq), ldq, d, n, damping, ldq, ws_offset=off)
        assert rc == 0, lib.kfac_last_error()
        check_inverse(inv, ref, n, ('simt', ldq, off))


@pytest.mark.parametrize('n', [1025, 2049, 3073, 4608])
def test_inverse_from_eigh_is_deterministic(lib, dev, n):
    """Split reductions: three calls give the same bits."""
    Q, d = basis(n, dev)
    Qs = stored(Q, ld4(n))
    damping = f32(1e-3 * float(d.max()))
    runs = []
    for _ in range(3):
        rc, inv = call_inverse(lib, Qs, ld4(n), d, n, damping, ld4(n))
        assert rc == 0, lib.kfac_last_error()
        runs.append(bits(inv[:n, :n]))
    assert torch.equal(runs[0], runs[1]) and torch.equal(runs[0], runs[2]), n


def test_inverse_from_eigh_rejects(lib, dev):
    from kfac_b200 import _cabi
    n = 1025
    Q, d = basis(n, dev)
    ldq = ld4(n)
    Qs = stored(Q, ldq)
    # a workspace one byte short of n * ldq floats: refused before anything is launched
    rc, inv = call_inverse(lib, Qs, ldq, d, n, 0.01, ldq, ws_bytes=n * ldq * 4 - 1)
    assert rc == _cabi.KFAC_ERR_WORKSPACE
    assert torch.isnan(inv).all()
    inv = torch.full((n, ldq), NAN, device=dev)
    ws = nan_ws(n * ldq * 4, dev)
    assert lib.kfac_inverse_from_eigh(Qs.data_ptr(), ldq, d.data_ptr(), n, 0.01, inv.data_ptr(), ldq, None,
                                      n * ldq * 4, S()) == _cabi.KFAC_ERR_WORKSPACE
    for ldq_, ld_inv, n_ in ((n - 1, ldq, n), (ldq, n - 1, n), (ldq, ldq, 0)):
        assert lib.kfac_inverse_from_eigh(Qs.data_ptr(), ldq_, d.data_ptr(), n_, 0.01, inv.data_ptr(), ld_inv,
                                          ws.data_ptr(), n * ldq * 4, S()) == _cabi.KFAC_ERR_BAD_ARG, (ldq_, ld_inv, n_)
    torch.cuda.synchronize()
    assert torch.isnan(inv).all()


# ---- eigensolver + damped inverse -------------------------------------------------------------------------------------

@pytest.mark.parametrize('n', [1025, 2304, 3073, 4608])
def test_eigh_then_inverse_matches_fp64_inverse(lib, dev, no_tf32, n):
    """What the inverse method computes for one factor (inverse.py:186-213 of the reference) at the widths of
    ResNet-50 and GPT-NeoX-125M, against torch.linalg.inv(F64 + damping I)."""
    *_, F = kfac_like_sequence(n, n // 3, 3, dev, seed=n)
    F64 = F.double()
    damping = f32(1e-3 * float(torch.linalg.eigvalsh(F64).max()))
    Q, _, d = run_eigh(lib, dev, F)
    ld = ld4(n)
    rc, inv = call_inverse(lib, Q, ld, d, n, damping, ld)
    assert rc == 0, lib.kfac_last_error()
    ref = torch.linalg.inv(F64 + damping * torch.eye(n, dtype=torch.float64, device=dev))
    e = rel_fro(inv[:n, :n], ref)
    print(f'n={n}: eigh + inverse vs fp64 inverse {e:.2e}')
    assert e < 1e-3, (n, e)
    assert_nan_outside(inv, n, n, n)


# ---- kfac_transpose ---------------------------------------------------------------------------------------------------

def special_values(rows, cols, dev, seed):
    """Gaussian fp32 with -0.0, subnormals and a NaN with a payload mixed in (a transpose moves bits)."""
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn(rows, cols, device=dev, generator=g)
    flat = bits(x).view(-1)
    k = flat.numel()
    picks = torch.randint(0, k, (min(k, 12),), device=dev, generator=g)
    specials = torch.tensor([-2 ** 31, 1, 0x007fffff, -2 ** 31 + 5, 0x7fc0dead, -0x003ff453], dtype=torch.int32,
                            device=dev)          # -0.0, subnormals (+ and -), quiet NaNs with payloads (+ and -)
    flat[picks] = specials[torch.arange(picks.numel(), device=dev) % specials.numel()]
    return x


@pytest.mark.parametrize('rows,cols', [(1, 1), (1, 37), (37, 1), (31, 33), (32, 32), (100, 257), (1025, 1025),
                                       (4608, 3073)])
def test_transpose_bitwise(lib, dev, rows, cols):
    x = special_values(rows, cols, dev, rows * 7 + cols)
    want = bits(x.t())
    for ld_src in (ld4(cols), ld4(cols) + 8):
        src = stored(x, ld_src)
        for ld_dst in (ld4(rows), ld4(rows) + 4):
            dst = torch.full((cols + 1, ld_dst), NAN, device=dev)
            assert lib.kfac_transpose(src.data_ptr(), ld_src, dst.data_ptr(), ld_dst, rows, cols, S()) == 0, \
                lib.kfac_last_error()
            torch.cuda.synchronize()
            what = (rows, cols, ld_src, ld_dst)
            assert torch.equal(bits(dst[:cols, :rows]), want), what
            assert_nan_outside(dst, cols, rows, what)


def test_transpose_rejects(lib, dev):
    from kfac_b200 import _cabi
    src = torch.randn(40, 36, device=dev)
    dst = torch.full((36, 40), NAN, device=dev)
    s, t = src.data_ptr(), dst.data_ptr()
    for args in ((s, 36, t, 40, 0, 36), (s, 36, t, 40, 40, 0), (s, 35, t, 40, 40, 36), (s, 36, t, 39, 40, 36),
                 (None, 36, t, 40, 40, 36), (s, 36, None, 40, 40, 36), (s, 36, t, 40, -1, 36)):
        assert lib.kfac_transpose(*args, S()) == _cabi.KFAC_ERR_BAD_ARG, args[1:]
    torch.cuda.synchronize()
    assert torch.isnan(dst).all()


@pytest.mark.parametrize('n', [129, 1025, 3073])
def test_transpose_of_eigenbasis_is_the_solvers_qt(lib, dev, no_tf32, n):
    """A rank that receives Q by broadcast builds QT with kfac_transpose; it must hold the bits the eigensolver wrote
    to QT on the rank that decomposed the factor, so that both precondition with the same data."""
    *_, F = kfac_like_sequence(n, n // 3, 2, dev, seed=n + 1)
    Q, QT, _ = run_eigh(lib, dev, F)
    ld = ld4(n)
    dst = torch.full((n, ld), NAN, device=dev)
    assert lib.kfac_transpose(Q.data_ptr(), ld, dst.data_ptr(), ld, n, n, S()) == 0, lib.kfac_last_error()
    torch.cuda.synchronize()
    assert torch.isfinite(QT[:, :n]).all()
    assert torch.equal(bits(dst[:, :n]), bits(QT[:, :n])), n


# ---- kfac_diag_snapshot -----------------------------------------------------------------------------------------------

F32_1E15 = f32(1e15)
BAD_VALUES = {'+inf': float('inf'), '-inf': float('-inf'), 'nan': None,
              'next above 1e15': float(np.nextafter(np.float32(1e15), np.float32(np.inf))), '-2e15': -2e15}


def one_grid(dev):
    """Elements one launch of a grid-stride kernel covers in one pass: grid_for caps the grid at SMs * 16 blocks of
    256 threads."""
    return torch.cuda.get_device_properties(dev).multi_processor_count * 16 * 256


def snapshot(lib, src, preset):
    dev = src.device
    dst = torch.full_like(src, NAN)
    status = torch.full((1,), preset, dtype=torch.int32, device=dev)
    assert lib.kfac_diag_snapshot(src.data_ptr(), dst.data_ptr(), src.numel(), status.data_ptr(), S()) == 0
    torch.cuda.synchronize()
    return dst, int(status.item())


@pytest.mark.parametrize('n', [1, 257, 4099, 3_000_017])
def test_diag_snapshot(lib, dev, n):
    g = torch.Generator(device=dev).manual_seed(n)
    src = torch.rand(n, device=dev, generator=g) * 10.0 ** torch.randint(-30, 12, (n,), device=dev, generator=g)
    sb = bits(src)
    # clean entries of every kind: -0.0, subnormals, +-1e15 exactly (the largest accepted magnitude)
    clean = [(0, -2 ** 31), (n // 2, 1), (n // 3, 0x007fffff), (n - 1, int(bits(torch.tensor([-F32_1E15])).item())),
             (n // 5, int(bits(torch.tensor([F32_1E15])).item()))]
    for i, b in clean:
        sb[i] = b
    assert torch.isfinite(src).all() and float(src.abs().max()) <= F32_1E15
    for preset in (0, 1):
        dst, status = snapshot(lib, src, preset)
        assert torch.equal(bits(dst), sb), (n, 'clean', preset)
        assert status == preset, (n, 'clean', preset, status)
    cover = one_grid(dev)
    places = sorted({i for i in (0, n - 1, cover + 3) if i < n})
    if n > 2 * cover:
        assert cover + 3 in places          # an entry only a later pass of the grid-stride loop reaches
    payload_nan = 0x7fc0beef
    for name, v in BAD_VALUES.items():
        for i in places:
            keep = int(sb[i].item())
            if v is None:
                sb[i] = payload_nan
            else:
                src[i] = v
            want = bits(src).clone()
            for preset in (0, 1):
                dst, status = snapshot(lib, src, preset)
                assert torch.equal(bits(dst), want), (n, name, i, preset)
                assert status == preset | 2, (n, name, i, preset, status)    # ORed in, never overwritten
            sb[i] = keep


# ---- kfac_dgda --------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('ld_out', [3076, 3080])
def test_dgda_bench_shape(lib, dev, ld_out):
    g_dim, a_dim = 4608, 3073
    gen = torch.Generator(device=dev).manual_seed(ld_out)
    dg = torch.rand(g_dim, device=dev, generator=gen) ** 4
    da = torch.rand(a_dim, device=dev, generator=gen) ** 4 * 30.0
    dg[:7] = 0.0
    da[-5:] = 0.0
    damping = f32(0.003)
    out = torch.full((g_dim + 1, ld_out), NAN, device=dev)
    assert lib.kfac_dgda(dg.data_ptr(), da.data_ptr(), g_dim, a_dim, damping, out.data_ptr(), ld_out, S()) == 0
    torch.cuda.synchronize()
    ref = 1.0 / (dg.double()[:, None] * da.double()[None, :] + damping)
    err = float(((out[:g_dim, :a_dim].double() - ref).abs() / ref).max())
    assert err <= 2.0 ** -21, err            # 4 ulp
    assert torch.equal(out[:g_dim, a_dim:], torch.zeros(g_dim, ld_out - a_dim, device=dev))
    assert torch.isnan(out[g_dim]).all()


# ---- the preconditioner, inverse method, factors wider than 1024 ------------------------------------------------------

class _WideMlp(torch.nn.Module):
    """A factors of 1101, 1031 and 1501, G factors of 1030, 1500 and 300.  The sin(4 x) units keep the hidden A
    factors well conditioned (see _Mlp in test_gpu_eigh_scale.py)."""

    def __init__(self):
        super().__init__()
        self.l1 = torch.nn.Linear(1100, 1030)
        self.l2 = torch.nn.Linear(1030, 1500)
        self.l3 = torch.nn.Linear(1500, 300)

    def forward(self, x):
        return self.l3(torch.sin(4 * self.l2(torch.sin(4 * self.l1(x)))))


def _train(model, batches, damping):
    """Steps of SGD on the preconditioned gradients; per step and layer: the factors, the inverses, P, the gradient
    matrix [wgrad | bgrad] before and after the preconditioner (fp32 copies)."""
    from kfac_b200.preconditioner import KFACPreconditioner
    pre = KFACPreconditioner(model, damping=damping, compute_method='inverse')
    opt = torch.optim.SGD(model.parameters(), lr=0.05)
    mse = torch.nn.MSELoss(reduction='sum')
    modules = [model.l1, model.l2, model.l3]
    record = []
    for x, y in batches:
        opt.zero_grad()
        (0.05 * mse(model(x), y)).backward()
        grads = [torch.cat([m.weight.grad, m.bias.grad[:, None]], 1).clone() for m in modules]
        pre.step()
        torch.cuda.synchronize()
        step = {}
        for m, grad in zip(modules, grads):
            _, layer = pre._layers[m]
            step[m] = dict(A=layer.a_factor.clone(), G=layer.g_factor.clone(), a_inv=layer.a_inv.clone(),
                           g_inv=layer.g_inv.clone(), P=layer._p_view.clone(), grad=grad,
                           out=torch.cat([m.weight.grad, m.bias.grad[:, None]], 1).clone())
        record.append(step)
        opt.step()
    return record


def test_inverse_method_wide_layers(dev, no_tf32):
    torch.manual_seed(23)
    model = _WideMlp().to(dev)
    model2 = copy.deepcopy(model)
    gen = torch.Generator(device=dev).manual_seed(24)
    batches = [(torch.randn(4, 512, 1100, device=dev, generator=gen), torch.randn(4, 512, 300, device=dev, generator=gen))
               for _ in range(3)]
    damping = 0.003
    lam = f32(damping)
    rec1 = _train(model, batches, damping)
    dims = [(r['A'].shape[0], r['G'].shape[0]) for r in rec1[0].values()]
    assert dims == [(1101, 1030), (1031, 1500), (1501, 300)], dims
    for s, step in enumerate(rec1):
        for li, r in enumerate(step.values()):
            A64, G64 = r['A'].double(), r['G'].double()
            a_inv = torch.linalg.inv(A64 + lam * torch.eye(A64.shape[0], dtype=torch.float64, device=dev))
            g_inv = torch.linalg.inv(G64 + lam * torch.eye(G64.shape[0], dtype=torch.float64, device=dev))
            ref = g_inv @ r['grad'].double() @ a_inv
            e = rel_fro(r['P'], ref)
            print(f'step {s} layer {li}: P vs fp64 {e:.2e}, a_inv {rel_fro(r["a_inv"], a_inv):.2e}, '
                  f'g_inv {rel_fro(r["g_inv"], g_inv):.2e}')
            assert e < 1e-3, (s, li, e)
    # the same batches on a copy of the initial model: the same bits.  Step by step, the factors of a step come
    # first, so that a difference that starts in the model's own kernels is not taken for one of the preconditioner's
    # (and one that starts in the preconditioner shows before the next step's factors inherit it).
    rec2 = _train(model2, batches, damping)
    for s, (st1, st2) in enumerate(zip(rec1, rec2)):
        for key in ('A', 'G', 'a_inv', 'g_inv', 'P', 'out'):
            for li, (r1, r2) in enumerate(zip(st1.values(), st2.values())):
                assert torch.equal(bits(r1[key]), bits(r2[key])), (s, key, li)
