"""Mixed precision with a dynamic loss scale: the guarded EMA (kfac_factor_ema_guarded) and the GradScaler path of the
preconditioner.

  * the guarded EMA gives the bits of kfac_factor_ema (on batch / s^2) for every window it keeps, and drops windows
    with non-finite or huge entries (factor unchanged, or I for a first window);
  * a torch.amp.GradScaler read on the device gives the same factors and gradients as a host callable returning the
    same scale, and adds no host sync to the hooks;
  * an fp16 overflow step no longer poisons the G factors; without a grad_scaler it still raises."""
import ctypes as C
import os
import socket
import subprocess
import sys

import pytest
import torch

from kfac_b200 import _cabi

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda:0')
DIMS = (3, 64, 65, 200, 1000)


def _items(factors, batches, firsts, counts):
    items = (_cabi.EmaItem * len(factors))()
    for i, (f, b, first, n) in enumerate(zip(factors, batches, firsts, counts)):
        items[i] = _cabi.EmaItem(f.data_ptr(), b.data_ptr(), f.shape[0], first, 1.0 / n)
    return items


def _ema(factors, batches, firsts, counts, alpha):
    lib = _cabi.load()
    _cabi.check(lib.kfac_factor_ema(_items(factors, batches, firsts, counts), len(factors), alpha,
                                    _cabi.stream_ptr()), 'kfac_factor_ema')


def _ema_guarded(factors, batches, firsts, counts, alpha, scales, skipped, ws_bytes=None):
    """scales: None (NULL array) or a list of device float tensors / None (NULL entries)."""
    lib = _cabi.load()
    n = len(factors)
    arr = None
    if scales is not None:
        arr = (C.c_void_p * n)(*[s.data_ptr() if s is not None else None for s in scales])
    need = lib.kfac_factor_ema_guarded_workspace_bytes(n)
    ws = torch.empty(max(need, 1), dtype=torch.uint8, device=DEV)
    _cabi.check(lib.kfac_factor_ema_guarded(_items(factors, batches, firsts, counts), n, alpha, arr,
                                            skipped.data_ptr() if skipped is not None else None, ws.data_ptr(),
                                            need if ws_bytes is None else ws_bytes, _cabi.stream_ptr()),
                'kfac_factor_ema_guarded')


def _problem(n_items=44, seed=0):
    g = torch.Generator(device='cpu').manual_seed(seed)
    dims = [DIMS[i % len(DIMS)] for i in range(n_items)]
    factors, batches, firsts, counts = [], [], [], []
    for i, d in enumerate(dims):
        x = torch.randn(d, d, generator=g)
        factors.append((x @ x.T / d).to(DEV))
        batches.append(torch.randn(d, d, generator=g).to(DEV) * 3.0)   # not symmetric: the EMA symmetrises
        firsts.append((i // len(DIMS)) % 2)
        counts.append(1 + i % 3)
    return factors, batches, firsts, counts


def _clone(ts):
    return [t.clone() for t in ts]


def test_guarded_ema_equals_ema():
    """> 40 items (two launches of each kernel), d in {3, 64, 65, 200, 1000}, first = 0 and 1."""
    factors, batches, firsts, counts = _problem()
    assert len(factors) > 40 and set(firsts) == {0, 1}
    alpha = 0.95
    # reference: the unguarded EMA
    rf, rb = _clone(factors), _clone(batches)
    _ema(rf, rb, firsts, counts, alpha)
    # NULL scale array and an array of NULL entries
    for scales in (None, [None] * len(factors)):
        gf, gb = _clone(factors), _clone(batches)
        skipped = torch.zeros(1, dtype=torch.int64, device=DEV)
        _ema_guarded(gf, gb, firsts, counts, alpha, scales, skipped)
        torch.cuda.synchronize()
        for i in range(len(factors)):
            assert torch.equal(gf[i], rf[i]), (i, factors[i].shape)
            assert torch.equal(gb[i], rb[i]) and not gb[i].any()
        assert skipped.item() == 0
    # loss scales 2^k: the unguarded EMA on batch / 2^(2k); NULL entries mixed in
    ks = [(-3, 0, 5, 10, 16, 24, None)[i % 7] for i in range(len(factors))]
    scales = [torch.tensor([2.0 ** k], device=DEV) if k is not None else None for k in ks]
    rf, rb = _clone(factors), [b / 2.0 ** (2 * k) if k is not None else b.clone() for b, k in zip(batches, ks)]
    _ema(rf, rb, firsts, counts, alpha)
    runs = []
    for _ in range(2):      # a repeat call gives the same bits
        gf, gb = _clone(factors), _clone(batches)
        skipped = torch.zeros(1, dtype=torch.int64, device=DEV)
        _ema_guarded(gf, gb, firsts, counts, alpha, scales, skipped)
        torch.cuda.synchronize()
        for i in range(len(factors)):
            assert torch.equal(gf[i], rf[i]), (i, ks[i], factors[i].shape)
            assert not gb[i].any()
        assert skipped.item() == 0
        runs.append(gf)
    for a, b in zip(*runs):
        assert torch.equal(a, b)


def test_guarded_ema_drops_bad_windows():
    factors, batches, firsts, counts = _problem(n_items=46, seed=1)
    alpha = 0.9
    # items 3 (d = 200), 7 (d = 65) and 44 (d = 1000, first window) are tripped: inf, NaN, 2e15;
    # item 41 holds 1e15 (kept)
    bad = {3: float('inf'), 7: float('nan'), 44: 2e15}
    firsts[3], firsts[7], firsts[44] = 0, 0, 1
    for i, v in bad.items():
        d = factors[i].shape[0]
        batches[i][d // 2, d - 1] = v
    batches[41][0, 0] = 1e15
    scales = [None] * len(factors)
    scales[7] = torch.tensor([4.0], device=DEV)          # a scale does not save a NaN
    scales[41] = torch.tensor([1.0], device=DEV)
    ref_b = _clone(batches)
    ref_b[7] = ref_b[7] / 16.0
    rf = _clone(factors)
    _ema(rf, ref_b, firsts, counts, alpha)
    gf, gb = _clone(factors), _clone(batches)
    skipped = torch.zeros(1, dtype=torch.int64, device=DEV)
    _ema_guarded(gf, gb, firsts, counts, alpha, scales, skipped)
    torch.cuda.synchronize()
    assert skipped.item() == len(bad)
    for i in range(len(factors)):
        assert not gb[i].any(), i
        if i in bad:
            want = torch.eye(factors[i].shape[0], device=DEV) if firsts[i] else factors[i]
            assert torch.equal(gf[i], want), i
        else:
            assert torch.equal(gf[i], rf[i]), i
    assert torch.isfinite(torch.cat([f.flatten() for f in gf])).all()
    # the counter accumulates over calls; a small enough scale trips a finite window
    gb[0].fill_(1.0)
    big = torch.tensor([2.0 ** -30], device=DEV)         # 1 / s^2 = 2^60 > 1e15
    before = gf[0].clone()
    _ema_guarded(gf[:1], gb[:1], [0], [1], alpha, [big], skipped)
    torch.cuda.synchronize()
    assert skipped.item() == len(bad) + 1 and torch.equal(gf[0], before) and not gb[0].any()


def test_guarded_ema_rejects_small_workspace():
    factors, batches, firsts, counts = _problem(n_items=2)
    before = _clone(factors)
    with pytest.raises(_cabi.KFACNativeError):
        _ema_guarded(factors, batches, firsts, counts, 0.9, None, None, ws_bytes=3)
    torch.cuda.synchronize()
    for a, b in zip(factors, before):
        assert torch.equal(a, b)


# ------------------------------------------------------------------ preconditioner
class _Net(torch.nn.Module):
    """Conv and Linear layers whose factors take the SIMT and the tensor-core SYRK paths."""

    def __init__(self):
        super().__init__()
        self.conv1 = torch.nn.Conv2d(3, 32, 3, padding=1)
        self.conv2 = torch.nn.Conv2d(32, 64, 3, stride=2, padding=1, bias=False)
        self.conv3 = torch.nn.Conv2d(64, 96, 1)
        self.fc1 = torch.nn.Linear(96, 80)
        self.fc2 = torch.nn.Linear(80, 10)

    def forward(self, x):
        x = torch.relu(self.conv1(x))
        x = torch.relu(self.conv2(x))
        x = torch.relu(self.conv3(x))
        x = torch.nn.functional.adaptive_avg_pool2d(x, 1).flatten(1)
        return self.fc2(torch.relu(self.fc1(x)))


def _data(seed=0):
    g = torch.Generator(device='cpu').manual_seed(seed)
    return torch.randn(16, 3, 16, 16, generator=g).to(DEV), torch.randint(0, 10, (16,), generator=g).to(DEV)


def _scaler(scale=2.0 ** 10):
    return torch.amp.GradScaler('cuda', init_scale=scale, growth_interval=10 ** 9)


def _forward_backward(model, scaler, x, y, extra=1.0):
    with torch.autocast('cuda', dtype=torch.float16):
        loss = torch.nn.functional.cross_entropy(model(x), y)
    (scaler.scale(loss) * extra).backward()


def _layers(pre):
    return [layer for _, layer in pre._layers.values()]


def test_device_scale_matches_host_scale():
    """A GradScaler read on the device and a callable returning the same scale give the same bits."""
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(0)
    model = _Net().to(DEV)
    scaler = _scaler()
    dev_pre = KFACPreconditioner(model, grad_scaler=scaler, damping=0.003)
    host_pre = KFACPreconditioner(model, grad_scaler=lambda: 1024.0, damping=0.003)
    opt = torch.optim.SGD(model.parameters(), lr=0.01)
    for step in range(4):
        x, y = _data(step)
        opt.zero_grad()
        _forward_backward(model, scaler, x, y)
        scaler.unscale_(opt)
        raw = [p.grad.clone() for p in model.parameters()]
        dev_pre.step()
        dev_grads = [p.grad.clone() for p in model.parameters()]
        for p, g in zip(model.parameters(), raw):
            p.grad.copy_(g)
        host_pre.step()
        torch.cuda.synchronize()
        for a, b in zip(_layers(dev_pre), _layers(host_pre)):
            assert torch.equal(a.a_factor, b.a_factor), (step, 'A')
            assert torch.equal(a.g_factor, b.g_factor), (step, 'G')
        for p, g in zip(model.parameters(), dev_grads):
            assert torch.isfinite(g).all()
            assert torch.equal(p.grad, g), step
        scaler.step(opt)
        scaler.update()
    assert scaler.get_scale() == 1024.0
    assert dev_pre.skipped_factor_updates == 0 and host_pre.skipped_factor_updates == 0


def _hooks_sync_free(grad_scaler_of):
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(0)
    model = _Net().to(DEV)
    scaler = _scaler()
    pre = KFACPreconditioner(model, grad_scaler=grad_scaler_of(scaler))
    opt = torch.optim.SGD(model.parameters(), lr=0.01)
    x, y = _data()
    _forward_backward(model, scaler, x, y)      # warm-up step
    scaler.unscale_(opt)
    pre.step()
    scaler.step(opt)
    scaler.update()
    opt.zero_grad()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        _forward_backward(model, scaler, x, y)   # a factor-update step: every hook runs
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


def test_no_host_sync_in_hooks():
    _hooks_sync_free(lambda scaler: scaler)
    # the check can see a sync: GradScaler.get_scale() is an .item()
    with pytest.raises(RuntimeError):
        _hooks_sync_free(lambda scaler: (lambda: scaler.get_scale()))


def _overflow_run(with_scaler):
    """Train with factor = inv = 1; step 2 forces an fp16 overflow (loss scale 2^60), then restores 2^10."""
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(0)
    model = _Net().to(DEV)
    scaler = _scaler()
    pre = KFACPreconditioner(model, grad_scaler=scaler if with_scaler else None, damping=0.003)
    finite = {}

    def watch(module, grad_input, grad_output):
        finite[module] = torch.isfinite(grad_output[0]).all()
    for module in pre._layers:
        module.register_full_backward_hook(watch)
    opt = torch.optim.SGD(model.parameters(), lr=0.01)
    out = {}
    for step in range(6):
        x, y = _data(step)
        opt.zero_grad()
        if step == 2:
            scaler.update(new_scale=2.0 ** 60)
            out['before'] = {m: l.g_factor.clone() for m, (_, l) in pre._layers.items()}
        _forward_backward(model, scaler, x, y)
        scaler.unscale_(opt)
        pre.step()
        torch.cuda.synchronize()
        if step == 2:
            out['overflowed'] = [m for m in pre._layers if not bool(finite[m])]
            out['after'] = {m: l.g_factor.clone() for m, (_, l) in pre._layers.items()}
        elif step > 2:
            for p in model.parameters():
                assert torch.isfinite(p.grad).all(), step
        scaler.step(opt)
        if step == 2:
            scaler.update(new_scale=2.0 ** 10)
        else:
            scaler.update()
    return pre, out


def test_overflow_step_is_skipped():
    pre, out = _overflow_run(with_scaler=True)
    assert out['overflowed'], 'the injected loss scale did not overflow fp16'
    for m in out['overflowed']:
        assert torch.equal(out['after'][m], out['before'][m])
    assert pre.skipped_factor_updates == len(out['overflowed'])
    for layer in _layers(pre):
        assert torch.isfinite(layer.a_factor).all() and torch.isfinite(layer.g_factor).all()


def test_overflow_without_grad_scaler_still_raises():
    with pytest.raises(_cabi.KFACNativeError):
        _overflow_run(with_scaler=False)


def test_two_ranks_drop_the_same_windows():
    """An overflow on rank 0 only: after the all-reduce of the statistics both ranks drop the same windows."""
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip('needs >= 2 GPUs')
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    script = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'dist_amp.py')
    out = subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node=2',
                          '--master-addr', '127.0.0.1', '--master-port', str(port), script],
                         capture_output=True, text=True, timeout=600)
    print(out.stdout[-3000:])
    assert out.returncode == 0 and 'DIST AMP OK' in out.stdout, out.stderr[-3000:]
