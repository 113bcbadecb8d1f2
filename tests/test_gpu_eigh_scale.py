"""kfac_eigh_batched at the magnitudes K-FAC factors reach: power-of-two scale equivariance and fp64 accuracy.

Per-batch G factors of a trained network have entries around 1e-12 (a ResNet-50 backward with cross-entropy gives
2.6e-13 .. 1e-10 for every layer wider than 128), so the solver must be as accurate there as at norm 1, the way LAPACK's
ssyevd (torch.linalg.eigh) is.  Every input here is an fp32 matrix whose largest entry lies in [1, 2) and whose
non-zero entries are at least 2^-30 of it, so F * 2^k is exact for k in [-90, 40]: the solver brings each factor into
[1, 2) by an exact power of two (factors whose largest entry is in [1/16, 1) are solved as they are), and the tests ask
for the same Q bits and 2^k times the same eigenvalues at every scale outside that band."""
import copy
import ctypes as C

import pytest
import torch

from conftest import rel_fro

pytestmark = pytest.mark.gpu

SIZES = [40, 100, 128, 129, 300, 1000, 1025, 2049]   # both Jacobi classes, first direct size, merge boundaries, two levels
SCALES = [-90, -60, -40, -20, -10, 0, 10, 40]   # k in [-4, -1] is the unscaled band
KINDS = ['cov', 'geo', 'lowrank', 'steady', 'dead']
TINY = 2.0 ** -126      # smallest normal fp32
SUB_ULP = 2.0 ** -149   # spacing of the fp32 subnormals


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


def exact_scalable(F64):
    """fp64 symmetric -> fp32 with max|F| in [1, 2) and every entry below 2^-30 max set to 0 (symmetry is kept: the
    rounding and the cut act on each entry alone)."""
    F = F64.float()
    _, e = torch.frexp(F.abs().max())
    F = F * 2.0 ** (1 - int(e))
    F[F.abs() < 2.0 ** -30 * F.abs().max()] = 0.0
    assert torch.equal(F, F.t())
    assert 1.0 <= float(F.abs().max()) < 2.0
    for k in range(-90, 41):
        assert torch.equal((F * 2.0 ** k) * 2.0 ** -k, F), k
    return F.contiguous()


def factor(n, kind, seed):
    g = torch.Generator().manual_seed(seed)
    f64 = torch.float64
    if kind in ('geo', 'lowrank'):
        Q, _ = torch.linalg.qr(torch.randn(n, n, generator=g, dtype=f64))
        if kind == 'geo':
            lam = torch.logspace(0, -7, n, dtype=f64)
        else:
            r = min(8, n)
            lam = torch.cat([torch.linspace(5, 0.5, r, dtype=f64), torch.full((n - r,), 0.95, dtype=f64)])
        F = (Q * lam) @ Q.t()
        return exact_scalable((F + F.t()) / 2)
    if kind == 'cov':
        X = torch.randn(4 * n, n, generator=g, dtype=f64).clamp(min=0)
        return exact_scalable(X.t() @ X / X.shape[0])
    # steady-state G: the batch statistic X^T X / m of m < n rows, no identity part (rank-deficient); graded feature
    # scales and a shared mixing like the rows of a backward pass
    m = max(8, n // 3)
    mix = torch.randn(n, n, generator=g, dtype=f64) / n ** 0.5
    X = torch.relu(torch.randn(m, n, generator=g, dtype=f64) @ mix + 0.3) * torch.logspace(0, -2, n, dtype=f64)
    if kind == 'dead':      # about a quarter of the units never receive a gradient
        X[:, dead_units(n, seed)] = 0.0
    else:
        assert kind == 'steady', kind
    return exact_scalable(X.t() @ X / m)


def dead_units(n, seed):
    g = torch.Generator().manual_seed(seed + 1)
    return torch.randperm(n, generator=g)[:n // 4]


def solve(lib, dev, mats):
    """One kfac_eigh_batched call over `mats` (device fp32); returns [(Q, QT, d)] and the status word."""
    from kfac_b200 import _cabi
    items = (_cabi.EighItem * len(mats))()
    ns = (C.c_int * len(mats))(*[F.shape[0] for F in mats])
    outs = []
    for i, F in enumerate(mats):
        n = F.shape[0]
        ld = _cabi.ld4(n)
        Q = torch.full((n, ld), float('nan'), device=dev)
        QT = torch.full((n, ld), float('nan'), device=dev)
        d = torch.full((n,), float('nan'), device=dev)
        items[i] = _cabi.EighItem(F.data_ptr(), Q.data_ptr(), QT.data_ptr(), d.data_ptr(), n, ld, None)
        outs.append((Q[:, :n], QT[:, :n], d))
    need = lib.kfac_eigh_workspace_bytes(ns, len(mats))
    ws = torch.empty(need, dtype=torch.uint8, device=dev)
    assert lib.kfac_eigh_batched(items, len(mats), ws.data_ptr(), need, 0, 0.0, S()) == 0, lib.kfac_last_error()
    host = torch.zeros(1, dtype=torch.int32).pin_memory()
    assert lib.kfac_eigh_status(ws.data_ptr(), host.data_ptr(), S()) == 0
    torch.cuda.synchronize()
    return outs, int(host.item())


def assert_scaled_copy(out, ref, k, what):
    """out is the solve of 2^k F, ref the solve of F: the same Q / QT bits, d = 2^k d_ref exactly where both are
    normal floats or zero, within one subnormal ulp elsewhere."""
    Q, QT, d = out
    Q0, QT0, d0 = ref
    assert torch.equal(Q, Q0), (what, k, 'Q', float((Q - Q0).abs().max()))
    assert torch.equal(QT, QT0), (what, k, 'QT')
    want = d0.double() * 2.0 ** k
    got = d.double()
    normal = ((want == 0) | (want.abs() >= TINY)) & ((got == 0) | (got.abs() >= TINY))
    assert torch.equal(got[normal], want[normal]), (what, k, 'd', float((got - want)[normal].abs().max()))
    rest = (got - want)[~normal]
    assert rest.numel() == 0 or float(rest.abs().max()) <= SUB_ULP, (what, k, 'd subnormal')


def accuracy(F, w, V, Q, d):
    """Scale-relative errors of (Q, d) against the fp64 eigendecomposition (w, V) of F (all fp64, one device)."""
    n = F.shape[0]
    scale = float(w.abs().max())
    orth = float((Q.t() @ Q - torch.eye(n, dtype=Q.dtype, device=Q.device)).abs().max())
    ev = float((torch.sort(d).values - w.clamp(min=0)).abs().max()) / scale
    f_ref = (V / (w.clamp(min=0) + 1e-3 * scale)) @ V.t()
    f_got = (Q / (d + 1e-3 * scale)) @ Q.t()
    func = float((f_got - f_ref).norm() / f_ref.norm())
    res = float((F @ Q - Q * d).norm() / F.norm())
    return orth, ev, func, res


def check_accuracy(F, ref64, out, k, what):
    Q, _, d = out
    assert torch.isfinite(Q).all() and torch.isfinite(d).all(), (what, k)
    assert float(d.min()) >= 0.0
    w, V = ref64
    orth, ev, func, res = accuracy(F.double(), w, V, Q.double(), d.double() * 2.0 ** -k)
    print(f'{what} k={k}: orth {orth:.1e} eig {ev:.1e} damped inverse {func:.1e} residual {res:.1e}')
    assert orth < 2e-4, (what, k, 'orthogonality', orth)
    assert ev < 5e-5, (what, k, 'eigenvalues', ev)
    assert func < 1e-3, (what, k, 'damped inverse', func)
    assert res < 1e-4, (what, k, 'residual', res)


_cache = {}


def scaled_solves(lib, dev, kind):
    """For one spectrum: the inputs over SIZES, their fp64 eigendecompositions and one call per scale in SCALES."""
    if kind not in _cache:
        mats = [factor(n, kind, 1000 * i + 17).to(dev) for i, n in enumerate(SIZES)]
        ref64 = [torch.linalg.eigh(F.double()) for F in mats]
        runs = {}
        for k in SCALES:
            outs, status = solve(lib, dev, [F * 2.0 ** k for F in mats])
            runs[k] = (outs, status)
        _cache[kind] = (mats, ref64, runs)
    return _cache[kind]


@pytest.mark.parametrize('kind', KINDS)
def test_scale_equivariance(lib, dev, kind):
    mats, _, runs = scaled_solves(lib, dev, kind)
    outs0, _ = runs[0]
    for k in SCALES:
        outs, status = runs[k]
        assert status == 0, (kind, k, status)
        for F, out, ref in zip(mats, outs, outs0):
            assert_scaled_copy(out, ref, k, (kind, F.shape[0]))


@pytest.mark.parametrize('kind', KINDS)
def test_accuracy_at_every_scale(lib, dev, kind):
    mats, ref64, runs = scaled_solves(lib, dev, kind)
    failures = []
    for k in SCALES:
        outs, _ = runs[k]
        for F, r, out in zip(mats, ref64, outs):
            try:
                check_accuracy(F, r, out, k, (kind, F.shape[0]))
            except AssertionError as e:
                failures.append(str(e))
    assert not failures, '\n'.join(failures)


@pytest.mark.parametrize('n,kind', [(2304, 'steady'), (4608, 'steady'), (2304, 'geo'), (4608, 'cov')])
def test_large_sizes(lib, dev, n, kind):
    F = factor(n, kind, n).to(dev)
    ref64 = torch.linalg.eigh(F.double())
    (out0,), status0 = solve(lib, dev, [F])
    (out,), status = solve(lib, dev, [F * 2.0 ** -40])
    assert status0 == 0 and status == 0
    check_accuracy(F, ref64, out0, 0, (kind, n))
    check_accuracy(F, ref64, out, -40, (kind, n))
    assert_scaled_copy(out, out0, -40, (kind, n))


@pytest.mark.parametrize('kind', ['cov', 'dead'])
def test_scales_mixed_in_one_call(lib, dev, kind):
    """Every item carries its own exponent: a batch of factors of very different magnitudes (the A and G factors of
    one step) gives each the bits it gets alone at k = 0."""
    mats, _, runs = scaled_solves(lib, dev, kind)
    outs0, _ = runs[0]
    ks = [-80, -62, -47, -31, -16, -5, 14, 30]     # spread over [-80, 30], outside the unscaled band k in [-4, -1]
    assert len(ks) == len(SIZES)
    for ks_i in (ks, ks[::-1]):
        outs, status = solve(lib, dev, [F * 2.0 ** k for F, k in zip(mats, ks_i)])
        assert status == 0
        for F, k, out, ref in zip(mats, ks_i, outs, outs0):
            assert_scaled_copy(out, ref, k, (kind, F.shape[0], 'mixed'))


def test_zero_factors(lib, dev):
    ns = [64, 100, 300, 1025]
    outs, status = solve(lib, dev, [torch.zeros(n, n, device=dev) for n in ns])
    assert status == 0
    for n, (Q, QT, d) in zip(ns, outs):
        assert torch.equal(d, torch.zeros_like(d)), n
        assert torch.isfinite(Q).all(), n
        Q64 = Q.double()
        assert float((Q64.t() @ Q64 - torch.eye(n, dtype=torch.float64, device=dev)).abs().max()) < 2e-4, n
        assert torch.equal(QT, Q.t()), n


def test_dead_units_at_small_scale(lib, dev):
    """Units without gradient give zero rows and columns; at 2^-60 their directions must still come out as (near)
    zero eigenvalues rather than as deflated diagonal entries."""
    ns = [129, 300, 1025]
    mats = [factor(n, 'dead', n) for n in ns]
    outs, status = solve(lib, dev, [F.to(dev) * 2.0 ** -60 for F in mats])
    assert status == 0
    for n, F, (Q, _, d) in zip(ns, mats, outs):
        dead = dead_units(n, n)
        assert float(F[dead].abs().max()) == 0.0
        w = torch.linalg.eigvalsh(F.double())
        dd = torch.sort(d.double().cpu() * 2.0 ** 60).values
        top = float(w.abs().max())
        assert float(dd[:len(dead)].max()) <= 1e-6 * top, (n, float(dd[:len(dead)].max()) / top)
        # the dead coordinates are (numerically) outside the span of the eigenvectors with non-negligible eigenvalues
        big = dd > 1e-2 * top
        Qs = Q.double().cpu()[:, torch.argsort(d.cpu())][:, big]
        assert float(Qs[dead].abs().max()) < 1e-3, n


def test_rejected_entries_at_small_scale(lib, dev):
    """Entries the input rule replaces by 0 (non-finite, |x| > 1e15) do not take part in the normalising exponent:
    the solve equals the solve of the matrix with those entries zeroed, and the status word reports them."""
    ns = [40, 128, 300, 1025]
    clean, dirty = [], []
    for n in ns:
        F = factor(n, 'cov', 3 * n).to(dev) * 2.0 ** -60
        i, j, p, q = n // 5, n // 2, n // 3, n - 2
        F[i, j] = F[j, i] = 0.0
        F[p, q] = F[q, p] = 0.0
        clean.append(F)
        G = F.clone()
        G[i, j] = G[j, i] = float('inf')
        G[p, q] = G[q, p] = 1e16
        dirty.append(G)
    outs_c, status_c = solve(lib, dev, clean)
    outs_d, status_d = solve(lib, dev, dirty)
    assert status_c == 0
    assert status_d & 2, status_d
    for n, out, ref in zip(ns, outs_d, outs_c):
        assert_scaled_copy(out, ref, 0, (n, 'rejected entries'))


# ---- the whole preconditioner on factors that are the batch statistics (a decayed EMA)

class _Mlp(torch.nn.Module):
    """Every A and G dimension is above 128: all factors go through the direct solver.  The sin(4 x) units keep the
    hidden A factors well conditioned (condition numbers near 60; tanh gives 3e4), so the inverse method's A stays
    invertible when the damping shrinks with G."""

    def __init__(self):
        super().__init__()
        self.l1 = torch.nn.Linear(160, 300)
        self.l2 = torch.nn.Linear(300, 257)
        self.l3 = torch.nn.Linear(257, 140)

    def forward(self, x):
        return self.l3(torch.sin(4 * self.l2(torch.sin(4 * self.l1(x)))))


# The EMA starts from I; a decay of 2^-100 leaves exactly the batch statistic in fp32 at both loss scales (2^-60, the
# value one would reach for first, is not absorbed by entries of 1e-12).
_DECAY = 2.0 ** -100


def _precondition(method, loss_scale, damping):
    from kfac_b200.preconditioner import KFACPreconditioner
    from oracle.kfac_oracle import OraclePreconditioner
    dev = torch.device('cuda:0')
    torch.manual_seed(5)
    ref_model = _Mlp()
    gpu_model = copy.deepcopy(ref_model).to(dev)
    x, y = torch.randn(512, 160), torch.randn(512, 140)
    kw = dict(damping=damping, factor_decay=lambda s: _DECAY, compute_method=method)
    ref = OraclePreconditioner(ref_model, **kw)
    pre = KFACPreconditioner(gpu_model, **kw)
    mse = torch.nn.MSELoss(reduction='sum')
    (loss_scale * mse(ref_model(x), y)).backward()
    (loss_scale * mse(gpu_model(x.to(dev)), y.to(dev))).backward()
    for p, q in zip(ref_model.parameters(), gpu_model.parameters()):
        q.grad.copy_(p.grad.to(dev))
    ref.step()
    pre.step()
    torch.cuda.synchronize()
    refs = {L.name: L for L in ref.layers.values()}
    out = {}
    for name, layer in pre._layers.values():
        R = refs[name]
        assert min(layer.a_factor.shape[0], layer.g_factor.shape[0]) > 128
        e = rel_fro(layer._p_view, R.P)
        print(f'{method} loss scale {loss_scale:.3e} {name}: max|G| {float(R.G.abs().max()):.2e} P vs oracle {e:.2e}')
        out[name] = (layer._p_view.detach().clone(), R.G.clone(), e)
    return out


@pytest.mark.parametrize('method', ['eigen', 'inverse'])
def test_preconditioner_at_steady_state_magnitudes(method):
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        # a loss scale 2^s that puts the largest entry of the smallest G factor in [1, 4): every G factor of the first
        # run lies above the band [1/16, 1) the solver leaves unscaled, so the second run must give its bits
        probe = _precondition(method, 1.0, 1e-3)
        gmin = min(float(G.abs().max()) for _, G, _ in probe.values())
        _, e = torch.frexp(torch.tensor(gmin, dtype=torch.float64))
        s = (2 - int(e)) // 2
        damping = 1e-3
        first = _precondition(method, 2.0 ** s, damping)
        assert 1.0 <= min(float(G.abs().max()) for _, G, _ in first.values()) < 4.0
        second = _precondition(method, 2.0 ** (s - 20), damping * 2.0 ** -40)
        for name in first:
            P1, G1, e1 = first[name]
            P2, G2, e2 = second[name]
            assert torch.equal(G2, G1 * 2.0 ** -40), name      # the factors themselves scale exactly
            assert e1 < 1e-3, (method, name, 'first run vs oracle', e1)
            assert e2 < 1e-3, (method, name, 'second run vs oracle', e2)
            if method == 'eigen':
                # 1 / (dg da + damping) scales by exactly 2^40 and the gradient by 2^-20; the inverse method damps A
                # with the same (here 2^-40 smaller) value, so its two runs solve different problems
                d = rel_fro(P2 * 2.0 ** -20, P1)
                print(f'{name}: second run * 2^-20 vs first run {d:.2e}, bit-identical {torch.equal(P2 * 2.0 ** -20, P1)}')
                assert d < 1e-6, (name, d)
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old
