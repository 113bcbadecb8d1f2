"""Cost of the GradScaler path on ResNet-50 (batch 32, fp16 autocast, one GPU).

    python tests/amp_overhead.py [--iters N] [--out DIR]

Two numbers, each for the two variants measured alternately in one process:
  * forward + backward of a factor-update step, with the loss scale read on the device from a
    torch.amp.GradScaler vs a callable `lambda: scaler.get_scale()` (a host sync in every G hook);
  * the EMA of all 108 factors, kfac_factor_ema_guarded (drop-flag scan + guarded EMA) vs kfac_factor_ema,
    timed with CUDA events.
The card's name and power limit are printed with the numbers (and written to DIR/amp_overhead.json).
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from kfac_b200 import _cabi  # noqa: E402
from kfac_b200.preconditioner import KFACPreconditioner  # noqa: E402
from workloads import resnet50  # noqa: E402


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        q = torch.cuda.get_device_name() + ', power limit unknown'
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    torch.manual_seed(0)
    x = torch.randn(32, 3, 224, 224, device=dev)
    y = torch.randint(0, 1000, (32,), device=dev)
    runs = {}
    for name in ('device_scale', 'host_get_scale'):
        model = resnet50().to(dev)
        scaler = torch.amp.GradScaler('cuda', init_scale=2.0 ** 10, growth_interval=10 ** 9)
        gs = scaler if name == 'device_scale' else (lambda s=scaler: s.get_scale())
        pre = KFACPreconditioner(model, grad_scaler=gs, factor_update_steps=1, inv_update_steps=10 ** 6,
                                 damping=0.001)
        opt = torch.optim.SGD(model.parameters(), lr=0.01)
        runs[name] = (model, scaler, pre, opt)

    def fwd_bwd(model, scaler):
        with torch.autocast('cuda', dtype=torch.float16):
            loss = torch.nn.functional.cross_entropy(model(x), y)
        scaler.scale(loss).backward()

    def finish(model, scaler, pre, opt):
        scaler.unscale_(opt)
        pre.step()
        scaler.step(opt)
        scaler.update()
        opt.zero_grad()

    for r in runs.values():             # warm-up: inverses, workspaces, cuDNN plans
        for _ in range(3):
            fwd_bwd(r[0], r[1])
            finish(*r)
    torch.cuda.synchronize()
    times = {k: [] for k in runs}
    for _ in range(args.iters):
        for name, r in runs.items():    # alternate the variants
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fwd_bwd(r[0], r[1])
            torch.cuda.synchronize()
            times[name].append((time.perf_counter() - t0) * 1e3)
            finish(*r)

    # EMA of every factor of the first preconditioner: guarded vs unguarded, CUDA events
    model, scaler, pre, opt = runs['device_scale']
    lib = _cabi.load()
    todo = [(l._a_view, l._a_batch_view, None) for _, l in pre._layers.values()]
    todo += [(l._g_view, l._g_batch_view, l._g_scale_slot) for _, l in pre._layers.values()]
    items = (_cabi.EmaItem * len(todo))()
    scales = (C.c_void_p * len(todo))()
    for i, (f, b, s) in enumerate(todo):
        items[i] = _cabi.EmaItem(f.data_ptr(), b.data_ptr(), f.shape[0], 0, 1.0)
        scales[i] = s.data_ptr() if s is not None else None
    need = lib.kfac_factor_ema_guarded_workspace_bytes(len(todo))
    ws = torch.empty(need, dtype=torch.uint8, device=dev)
    skipped = torch.zeros(1, dtype=torch.int64, device=dev)
    stream = _cabi.stream_ptr()

    def ema():
        _cabi.check(lib.kfac_factor_ema(items, len(todo), 0.95, stream))

    def guarded():
        _cabi.check(lib.kfac_factor_ema_guarded(items, len(todo), 0.95, scales, skipped.data_ptr(), ws.data_ptr(),
                                                need, stream))
    ema_ms = {'ema': [], 'ema_guarded': []}
    for fn in (ema, guarded):
        fn()
    for _ in range(args.iters):
        for key, fn in (('ema', ema), ('ema_guarded', guarded)):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            e1.synchronize()
            ema_ms[key].append(e0.elapsed_time(e1))
    factor_bytes = sum(f.numel() * 4 for f, _, _ in todo)

    def summary(v):
        return {'median_ms': statistics.median(v), 'min_ms': min(v), 'max_ms': max(v), 'n': len(v)}
    out = {'card': card(), 'workload': 'ResNet-50, batch 32, 224x224, fp16 autocast, factor_update_steps=1',
           'fwd_bwd': {k: summary(v) for k, v in times.items()},
           'ema_all_factors': {k: summary(v) for k, v in ema_ms.items()},
           'factors': len(todo), 'factor_mb': factor_bytes / 1e6, 'skipped': int(skipped.item())}
    print(json.dumps(out, indent=1))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'amp_overhead.json'), 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
