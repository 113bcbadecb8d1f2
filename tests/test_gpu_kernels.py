"""GPU parity tests of every C-ABI entry point against the CPU oracle.

All calls go through the C ABI (ctypes) exactly as the product path does.
Tolerances: fp32 arithmetic -> rel-Frobenius <= 1e-5 for factor statistics,
<= 1e-3 for anything downstream of the eigensolver (the bar of BASELINE.json).
"""
import ctypes as C

import pytest
import torch

from conftest import rel_fro

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def lib():
    from kfac_b200 import _cabi
    return _cabi.load()


@pytest.fixture(scope='module')
def dev():
    assert torch.cuda.is_available()
    return torch.device('cuda:0')


def S():
    return torch.cuda.current_stream().cuda_stream


def test_device_is_hopper(lib):
    assert lib.kfac_device_arch() == 90


@pytest.mark.parametrize('M,N,K', [(1, 1, 1), (7, 5, 3), (64, 64, 64), (100, 130, 257), (20, 577, 64), (300, 33, 1000)])
@pytest.mark.parametrize('ta,tb', [(False, False), (True, False), (False, True), (True, True)])
def test_gemm_f32(lib, dev, M, N, K, ta, tb):
    torch.manual_seed(M * 1000 + N * 10 + K)
    A = torch.randn(K, M, device=dev).t() if ta else torch.randn(M, K, device=dev)
    B = torch.randn(N, K, device=dev).t() if tb else torch.randn(K, N, device=dev)
    Cm = torch.randn(M, N, device=dev)
    ref = 0.5 * (A.double() @ B.double()) + 2.0 * Cm.double()
    rc = lib.kfac_gemm_f32(A.data_ptr(), A.stride(0), A.stride(1), B.data_ptr(), B.stride(0), B.stride(1),
                           Cm.data_ptr(), N, M, N, K, 0.5, 2.0, S())
    assert rc == 0
    torch.cuda.synchronize()
    assert rel_fro(Cm, ref) < 1e-5


@pytest.mark.parametrize('rows,feat,ones,dtype', [(1, 3, 1, torch.float32), (4, 10, 0, torch.float32), (33, 21, 1, torch.float32),
                                                   (1000, 65, 1, torch.float32), (5000, 130, 0, torch.float32),
                                                   (257, 64, 1, torch.bfloat16), (257, 64, 0, torch.float16),
                                                   (2048, 768, 1, torch.float32), (1030, 130, 0, torch.float32),
                                                   (4096, 256, 1, torch.bfloat16)])
def test_factor_linear(lib, dev, rows, feat, ones, dtype):
    from oracle import kfac_oracle as O
    torch.manual_seed(rows + feat)
    x = torch.randn(rows, feat).to(dtype)
    d = feat + ones
    acc = torch.zeros(d, d, device=dev)
    xd = x.to(dev)
    need = lib.kfac_factor_linear_workspace_bytes(rows, feat, ones)
    ws = torch.empty(max(need, 1), dtype=torch.uint8, device=dev)
    assert lib.kfac_factor_linear(xd.data_ptr(), {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}[dtype],
                                  rows, feat, ones, 1.0 / rows, acc.data_ptr(), ws.data_ptr() if need else None, need,
                                  S()) == 0
    acc2 = torch.zeros_like(acc)
    assert lib.kfac_factor_linear(xd.data_ptr(), {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}[dtype],
                                  rows, feat, ones, 1.0 / rows, acc2.data_ptr(), ws.data_ptr() if need else None, need,
                                  S()) == 0
    torch.cuda.synchronize()
    ref = O.linear_a_factor(x.float(), bool(ones))
    got = 0.5 * (acc + acc.t())
    assert rel_fro(got, ref) < 2e-5
    assert torch.equal(acc, acc.t()) or rel_fro(acc, acc.t()) < 1e-6
    assert torch.equal(acc, acc2)        # the same bits in every call


def test_get_cov_reference_vector_on_gpu(lib, dev):
    # exact vector of the reference's tests/layers/utils_test.py
    a = torch.tensor([[1., 2, 3], [4, 5, 6], [7, 8, 9]], device=dev)
    acc = torch.zeros(3, 3, device=dev)
    assert lib.kfac_factor_linear(a.data_ptr(), 0, 3, 3, 0, 1.0 / 3, acc.data_ptr(), None, 0, S()) == 0
    torch.cuda.synchronize()
    assert torch.allclose(acc.cpu(), torch.tensor([[22., 26, 30], [26, 31, 36], [30, 36, 42]]), rtol=1e-6)


CONV_GEOS = [  # B, C, H, W, kh, kw, sh, sw, ph, pw, bias
    (2, 3, 8, 8, 3, 3, 1, 1, 1, 1, 1),
    (3, 6, 12, 12, 3, 3, 2, 2, 1, 1, 0),
    (2, 8, 6, 6, 1, 1, 1, 1, 0, 0, 0),
    (2, 8, 6, 6, 1, 1, 1, 1, 0, 0, 1),
    (2, 8, 7, 7, 1, 1, 2, 2, 0, 0, 0),
    (2, 3, 17, 15, 7, 7, 2, 2, 3, 3, 0),
    (4, 16, 9, 9, 2, 2, 1, 1, 0, 0, 1),     # reference modules_test geometry k2 s1 p0 bias
    (1, 5, 10, 6, 3, 2, 2, 1, 1, 0, 0),
    (8, 64, 14, 14, 3, 3, 1, 1, 1, 1, 0),
    (8, 256, 7, 7, 1, 1, 1, 1, 0, 0, 0),    # 1x1 on 7x7 maps: rows of 49 floats are packed for the tensor-core SYRK
    (4, 128, 7, 7, 1, 1, 1, 1, 0, 0, 1),
]


@pytest.mark.parametrize('geo', CONV_GEOS)
def test_factor_conv2d_input(lib, dev, geo):
    from oracle import kfac_oracle as O
    B, Cc, H, W, kh, kw, sh, sw, ph, pw, bias = geo
    torch.manual_seed(sum(geo))
    x = torch.randn(B, Cc, H, W)
    ref = O.conv2d_a_factor(x, (kh, kw), (sh, sw), (ph, pw), bool(bias))
    Ho, Wo = (H + 2 * ph - kh) // sh + 1, (W + 2 * pw - kw) // sw + 1
    d = Cc * kh * kw + bias
    assert ref.shape == (d, d)
    acc = torch.zeros(d, d, device=dev)
    need = lib.kfac_factor_conv2d_input_workspace_bytes(B, Cc, H, W, kh, kw, sh, sw, ph, pw, bias)
    ws = torch.empty(max(need, 1), dtype=torch.uint8, device=dev)
    xd = x.to(dev)
    scale = 1.0 / (B * float(Ho * Wo) ** 3)
    assert lib.kfac_factor_conv2d_input(xd.data_ptr(), 0, B, Cc, H, W, kh, kw, sh, sw, ph, pw, bias, scale,
                                        acc.data_ptr(), ws.data_ptr(), need, S()) == 0
    torch.cuda.synchronize()
    assert rel_fro(0.5 * (acc + acc.t()), ref) < 2e-5


@pytest.mark.parametrize('B,Cc,Ho,Wo', [(2, 6, 8, 8), (3, 10, 3, 3), (4, 64, 14, 14), (2, 130, 5, 7), (1, 1, 1, 1),
                                        (8, 256, 7, 7), (32, 512, 7, 7)])
@pytest.mark.parametrize('with_ws', [True, False])
def test_factor_conv2d_gradout(lib, dev, B, Cc, Ho, Wo, with_ws):
    from oracle import kfac_oracle as O
    torch.manual_seed(B + Cc)
    g = torch.randn(B, Cc, Ho, Wo)
    ref = O.conv2d_g_factor(g)
    acc = torch.zeros(Cc, Cc, device=dev)
    gd = g.to(dev)
    scale = 1.0 / (B * float(Ho * Wo) ** 3)
    need = lib.kfac_factor_conv2d_gradout_workspace_bytes(B, Cc, Ho, Wo) if with_ws else 0
    # maps whose rows are not 16-byte multiples are packed (feature-major, rows padded to 4); the workspace also
    # holds the split partials of the SYRK
    packed = (B * Ho * Wo + 3) // 4 * 4 * Cc * 4 if (Ho * Wo) % 4 != 0 and Cc >= 64 else 0
    assert not with_ws or need >= packed
    ws = torch.empty(max(need, 1), dtype=torch.uint8, device=dev)
    acc2 = torch.zeros_like(acc)
    for out in (acc, acc2):
        assert lib.kfac_factor_conv2d_gradout(gd.data_ptr(), 0, B, Cc, Ho, Wo, scale, out.data_ptr(),
                                              ws.data_ptr() if need else None, need, S()) == 0
    torch.cuda.synchronize()
    assert rel_fro(0.5 * (acc + acc.t()), ref) < 2e-5
    assert torch.equal(acc, acc2)        # the same bits in every call


def test_factor_ema(lib, dev):
    from kfac_b200 import _cabi
    from oracle import kfac_oracle as O
    torch.manual_seed(0)
    ds = [3, 64, 65, 200]
    items = (_cabi.EmaItem * len(ds))()
    keep = []
    for i, d in enumerate(ds):
        batch = torch.randn(d, d)
        batch = batch @ batch.t()
        fac = torch.randn(d, d)
        fac = fac + fac.t()
        first = i % 2
        count = 1 + i
        fd, bd = fac.to(dev), (batch * count).to(dev)
        items[i] = _cabi.EmaItem(fd.data_ptr(), bd.data_ptr(), d, first, 1.0 / count)
        ref = O.ema_update(None if first else fac, batch * count, count, 0.9)
        keep.append((fd, bd, ref))
    assert lib.kfac_factor_ema(items, len(ds), 0.9, S()) == 0
    torch.cuda.synchronize()
    for fd, bd, ref in keep:
        assert rel_fro(fd, ref) < 1e-6
        assert float(bd.abs().max()) == 0.0


def make_psd(n, kind, seed):
    g = torch.Generator().manual_seed(seed)
    Q, _ = torch.linalg.qr(torch.randn(n, n, generator=g, dtype=torch.float64))
    if kind == 'geo':
        lam = torch.logspace(0, -7, n, dtype=torch.float64)
    elif kind == 'lowrank':
        r = min(8, n)
        lam = torch.cat([torch.linspace(5, 0.5, r, dtype=torch.float64), torch.full((n - r,), 0.95, dtype=torch.float64)])
    elif kind == 'cluster':
        lam = torch.cat([torch.ones(n // 2, dtype=torch.float64), torch.full((n - n // 2,), 1e-4, dtype=torch.float64)])
    elif kind == 'ident':
        return (0.73 * torch.eye(n, dtype=torch.float64)).float()
    else:
        X = torch.randn(4 * n, n, generator=g, dtype=torch.float64).clamp(min=0)
        return (X.t() @ X / X.shape[0]).float()
    return ((Q * lam) @ Q.t()).float()


def run_eigh(lib, dev, mats):
    from kfac_b200 import _cabi
    items = (_cabi.EighItem * len(mats))()
    ns = (C.c_int * len(mats))()
    outs = []
    for i, F in enumerate(mats):
        n = F.shape[0]
        Fd = F.to(dev).contiguous()
        ld = _cabi.ld4(n)
        Qs = torch.zeros(n, ld, device=dev)
        QTs = torch.zeros(n, ld, device=dev)
        d = torch.empty(n, device=dev)
        items[i] = _cabi.EighItem(Fd.data_ptr(), Qs.data_ptr(), QTs.data_ptr() if i % 2 == 0 else None,
                                  d.data_ptr(), n, ld)
        ns[i] = n
        outs.append((Fd, Qs[:, :n], d, QTs[:, :n] if i % 2 == 0 else None))
    need = lib.kfac_eigh_workspace_bytes(ns, len(mats))
    ws = torch.empty(max(need, 1), dtype=torch.uint8, device=dev)
    rc = lib.kfac_eigh_batched(items, len(mats), ws.data_ptr(), need, 0, 0.0, S())
    assert rc == 0, lib.kfac_last_error()
    torch.cuda.synchronize()
    return outs


def check_eigh(F, Q, d, damping=1e-3, tol=1e-3):
    n = F.shape[0]
    F64, Q64, d64 = F.double().cpu(), Q.double().cpu(), d.double().cpu()
    assert torch.isfinite(Q64).all() and torch.isfinite(d64).all()
    assert float(d64.min()) >= 0.0
    orth = (Q64.t() @ Q64 - torch.eye(n, dtype=torch.float64)).abs().max().item()
    assert orth < 2e-4, ('orthogonality', n, orth)
    w, V = torch.linalg.eigh(F64)
    scale = max(float(w.abs().max()), 1e-30)
    assert (torch.sort(d64).values - w.clamp(min=0)).abs().max().item() / scale < 5e-5
    f_ref = (V / (w.clamp(min=0) + damping * scale)) @ V.t()
    f_got = (Q64 / (d64 + damping * scale)) @ Q64.t()
    e = rel_fro(f_got, f_ref)
    assert e < tol, ('functional', n, e)
    return e


@pytest.mark.parametrize('kind', ['geo', 'lowrank', 'cluster', 'cov', 'ident'])
def test_eigh_batched_sizes(lib, dev, kind):
    sizes = [1, 2, 5, 10, 27, 64, 65, 100, 128, 129, 144, 200, 288, 576]
    mats = [make_psd(n, kind, 17 * n + 3) for n in sizes]
    outs = run_eigh(lib, dev, mats)
    worst = 0.0
    for F, Q, d, QT in outs:
        worst = max(worst, check_eigh(F, Q, d))
        if QT is not None:
            assert torch.equal(QT, Q.t())
    print(kind, 'worst functional error', worst)


def test_eigh_tc_class(lib, dev):
    # mid sizes (384..640) and the first sizes of the large class (768, 800, 1000)
    mats = [make_psd(384, 'cov', 1), make_psd(500, 'lowrank', 2), make_psd(576, 'cluster', 3), make_psd(640, 'ident', 4),
            make_psd(768, 'cov', 7), make_psd(800, 'cluster', 8), make_psd(1000, 'lowrank', 9)]
    for F, Q, d, _ in run_eigh(lib, dev, mats):
        check_eigh(F, Q, d)


def test_eigh_large(lib, dev):
    mats = [make_psd(1152, 'cov', 5), make_psd(1024, 'geo', 6)]
    for F, Q, d, _ in run_eigh(lib, dev, mats):
        check_eigh(F, Q, d)


def test_eigh_rejects_oversized(lib, dev):
    """Dimensions beyond KFAC_EIGH_MAX_N (8192) are refused up front with KFAC_ERR_UNSUPPORTED, not solved wrongly."""
    from kfac_b200 import _cabi
    n = 8193
    ns = (C.c_int * 1)(n)
    need = lib.kfac_eigh_workspace_bytes(ns, 1)
    ws = torch.empty(max(need, 1), dtype=torch.uint8, device=dev)
    ld = _cabi.ld4(n)
    F = torch.eye(n, device=dev)
    Q = torch.zeros(n, ld, device=dev)
    d = torch.empty(n, device=dev)
    items = (_cabi.EighItem * 1)(_cabi.EighItem(F.data_ptr(), Q.data_ptr(), None, d.data_ptr(), n, ld, None))
    rc = lib.kfac_eigh_batched(items, 1, ws.data_ptr(), need, 0, 0.0, S())
    assert rc != 0 and b'exceeds the supported dimension' in lib.kfac_last_error()


def test_eigh_reports_non_finite_input(lib, dev):
    """A factor with an Inf (AMP overflow step) must not yield a silently wrong eigenbasis: the status word of
    the workspace reports it (torch.linalg.eigh raises in the reference, kfac/layers/eigen.py:310)."""
    from kfac_b200 import _cabi
    for n in (40, 300):
        F = make_psd(n, 'cov', n).to(dev).contiguous()
        F[n // 2, n // 3] = float('inf')
        F[n // 3, n // 2] = float('inf')
        ld = _cabi.ld4(n)
        Q = torch.zeros(n, ld, device=dev)
        d = torch.empty(n, device=dev)
        items = (_cabi.EighItem * 1)(_cabi.EighItem(F.data_ptr(), Q.data_ptr(), None, d.data_ptr(), n, ld, None))
        ns = (C.c_int * 1)(n)
        need = lib.kfac_eigh_workspace_bytes(ns, 1)
        ws = torch.empty(need, dtype=torch.uint8, device=dev)
        assert lib.kfac_eigh_batched(items, 1, ws.data_ptr(), need, 0, 0.0, S()) == 0
        host = torch.zeros(1, dtype=torch.int32).pin_memory()
        assert lib.kfac_eigh_status(ws.data_ptr(), host.data_ptr(), S()) == 0
        torch.cuda.synchronize()
        assert int(host.item()) != 0, n


def test_dgda_and_inverse(lib, dev):
    from oracle import kfac_oracle as O
    torch.manual_seed(3)
    dg, da = torch.rand(37), torch.rand(130)
    out = torch.empty(37, 130, device=dev)
    out = torch.empty(37, 132, device=dev)
    assert lib.kfac_dgda(dg.to(dev).data_ptr(), da.to(dev).data_ptr(), 37, 130, 0.003, out.data_ptr(), 132, S()) == 0
    torch.cuda.synchronize()
    assert rel_fro(out[:, :130], O.eigen_dgda(dg, da, 0.003)) < 1e-6
    for n in (10, 64, 200):
        F = make_psd(n, 'cov', n)
        (Fd, Q, d, _), = run_eigh(lib, dev, [F])
        from kfac_b200 import _cabi
        ld = _cabi.ld4(n)
        inv = torch.empty(n, ld, device=dev)
        ws = torch.empty(n * ld, device=dev)
        assert lib.kfac_inverse_from_eigh(Q.data_ptr(), ld, d.data_ptr(), n, 0.01, inv.data_ptr(), ld,
                                          ws.data_ptr(), n * ld * 4, S()) == 0
        torch.cuda.synchronize()
        assert rel_fro(inv[:, :n], O.damped_inverse(F, 0.01)) < 1e-3


@pytest.mark.parametrize('g,a,bias,method', [(20, 10, 0, 'eigen'), (10, 21, 1, 'eigen'), (64, 577, 1, 'eigen'), (256, 1153, 1, 'eigen'), (512, 1024, 0, 'eigen'), (384, 640, 0, 'inverse'),
                                              (130, 65, 0, 'eigen_noprediv'), (16, 145, 1, 'inverse'), (200, 300, 0, 'inverse')])
def test_precondition_and_update(lib, dev, g, a, bias, method):
    from kfac_b200 import _cabi
    from oracle import kfac_oracle as O
    torch.manual_seed(g * a)
    A, G = make_psd(a, 'cov', a), make_psd(g, 'cov', g + 1)
    wgrad = torch.randn(g, a - bias)
    bgrad = torch.randn(g) if bias else None
    grad = O.grad_matrix(wgrad, bgrad)
    da, qa = O.eigen_decompose(A)
    dg, qg = O.eigen_decompose(G)
    damping = 0.003
    dgda = O.eigen_dgda(dg, da, damping)
    t = lambda x: x.to(dev).contiguous() if x is not None else None  # noqa: E731

    def pad(x):   # (rows, cols) -> storage with ld4(cols)
        out = torch.zeros(x.shape[0], _cabi.ld4(x.shape[1]), device=dev)
        out[:, :x.shape[1]] = x.to(dev)
        return out
    wd, bd = t(wgrad), t(bgrad)
    lda_, ldg_ = _cabi.ld4(a), _cabi.ld4(g)
    Ps = torch.zeros(g, lda_, device=dev)
    P = Ps[:, :a]
    a_inv_ref, g_inv_ref = O.damped_inverse(A, damping), O.damped_inverse(G, damping)
    keep = dict(qa=pad(qa), qaT=pad(qa.t()), qg=pad(qg), qgT=pad(qg.t()), dgda=pad(dgda), da=t(da), dg=t(dg),
                a_inv=pad(a_inv_ref), g_inv=pad(g_inv_ref))
    p = lambda k, use: keep[k].data_ptr() if use else None  # noqa: E731
    e, pre, inv = method.startswith('eigen'), method == 'eigen', method == 'inverse'
    items = (_cabi.PrecondItem * 1)()
    items[0] = _cabi.PrecondItem(wd.data_ptr(), bd.data_ptr() if bias else None, 0, g, a,
                                 p('qa', e), p('qaT', e), p('qg', e), p('qgT', e), p('dgda', pre),
                                 p('da', e and not pre), p('dg', e and not pre),
                                 p('a_inv', inv), p('g_inv', inv), lda_, ldg_, lda_, Ps.data_ptr(), lda_)
    need = lib.kfac_precondition_workspace_bytes(items, 1)
    ws = torch.empty(need, dtype=torch.uint8, device=dev)
    rc = lib.kfac_precondition(items, 1, 2 if inv else 1, damping, ws.data_ptr(), need, S())
    assert rc == 0, lib.kfac_last_error()
    torch.cuda.synchronize()
    if inv:
        ref = O.precondition_inverse(grad, a_inv_ref, g_inv_ref)
    elif pre:
        ref = O.precondition_eigen(grad, qa, qg, dgda=dgda)
    else:
        ref = O.precondition_eigen(grad, qa, qg, da=da, dg=dg, damping=damping)
    assert rel_fro(P, ref) < 1e-4

    # kl-clip scale + in-place write back
    gi = (_cabi.GradItem * 1)()
    gi[0] = _cabi.GradItem(Ps.data_ptr(), wd.data_ptr(), bd.data_ptr() if bias else None, 0, g, a, lda_)
    vg = torch.zeros(1, dtype=torch.float64, device=dev)
    nu = torch.zeros(1, device=dev)
    gneed = lib.kfac_grad_workspace_bytes(1)
    gws = torch.empty(gneed, dtype=torch.uint8, device=dev)
    assert lib.kfac_grad_scale(gi, 1, 0.001, 0.1, gws.data_ptr(), gneed, nu.data_ptr(), S()) == 0
    assert lib.kfac_grad_update(gi, 1, nu.data_ptr(), gws.data_ptr(), gneed, S()) == 0
    torch.cuda.synchronize()
    ref_scale = O.grad_scale([ref], [grad], 0.1, 0.001)
    assert abs(float(nu) - ref_scale) <= 1e-4 * ref_scale
    new = O.grad_matrix(wd.cpu(), bd.cpu() if bias else None)
    assert rel_fro(new, ref_scale * ref) < 2e-4


def test_not_ready_maps_to_runtime_error(lib, dev):
    from kfac_b200 import _cabi
    w = torch.randn(4, 4, device=dev)
    P = torch.empty(4, 4, device=dev)
    items = (_cabi.PrecondItem * 1)()
    items[0] = _cabi.PrecondItem(w.data_ptr(), None, 0, 4, 4, None, None, None, None, None, None, None, None, None,
                                 4, 4, 4, P.data_ptr(), 4)
    ws = torch.empty(4096, dtype=torch.uint8, device=dev)
    rc = lib.kfac_precondition(items, 1, 1, 0.1, ws.data_ptr(), 4096, S())
    assert rc == _cabi.KFAC_ERR_NOT_READY
    with pytest.raises(RuntimeError):
        _cabi.check(rc)
    with pytest.raises(ValueError):
        _cabi.check(lib.kfac_dgda(None, None, 0, 0, 0.1, None, 0, S()))


@pytest.mark.parametrize('n', [1, 2, 5, 64, 257])
def test_triu_pack_unpack(lib, dev, n):
    torch.manual_seed(n)
    F = torch.randn(n, n)
    F = F + F.t()
    Fd = F.to(dev)
    packed = torch.empty(n * (n + 1) // 2, device=dev)
    assert lib.kfac_triu_pack(Fd.data_ptr(), n, packed.data_ptr(), S()) == 0
    idx = torch.triu_indices(n, n)
    torch.cuda.synchronize()
    assert torch.equal(packed.cpu(), F[idx[0], idx[1]])   # kfac/distributed.py:422-433 order
    out = torch.zeros(n, n, device=dev)
    assert lib.kfac_triu_unpack(packed.data_ptr(), n, out.data_ptr(), S()) == 0
    torch.cuda.synchronize()
    assert torch.equal(out.cpu(), F)
    assert lib.kfac_scale_inplace(out.data_ptr(), n * n, 0.5, S()) == 0
    torch.cuda.synchronize()
    assert torch.equal(out.cpu(), 0.5 * F)


def test_eigh_accepts_v0t(lib, dev):
    """ABI compatibility: `V0T` (warm start of the round-1 iterative solver, may alias QT) is accepted and ignored."""
    from kfac_b200 import _cabi
    torch.manual_seed(0)
    for n in (200, 576, 1024):
        F1 = make_psd(n, 'cov', n)
        F2 = (0.95 * F1 + 0.05 * make_psd(n, 'cov', n + 7)).contiguous()
        ld = _cabi.ld4(n)
        Q = torch.zeros(n, ld, device=dev)
        QT = torch.zeros(n, ld, device=dev)
        d = torch.empty(n, device=dev)
        ns = (C.c_int * 1)(n)
        need = lib.kfac_eigh_workspace_bytes(ns, 1)
        ws = torch.empty(need, dtype=torch.uint8, device=dev)
        for F, warm in ((F1, None), (F2, QT)):
            Fd = F.to(dev)
            items = (_cabi.EighItem * 1)(_cabi.EighItem(Fd.data_ptr(), Q.data_ptr(), QT.data_ptr(), d.data_ptr(), n, ld,
                                                       warm.data_ptr() if warm is not None else None))
            assert lib.kfac_eigh_batched(items, 1, ws.data_ptr(), need, 0, 0.0, S()) == 0, lib.kfac_last_error()
            torch.cuda.synchronize()
            check_eigh(Fd, Q[:, :n], d)
            assert torch.equal(QT[:, :n], Q[:, :n].t())
