"""Cost of EKFAC over the eigen method on ResNet-50 (batch 32, fp32, one GPU).

    python tests/ekfac_overhead.py [--iters N] [--out DIR]

Numbers, with the two methods measured alternately in one process:
  * forward + backward + step() of a factor step that is not an inverse step (factor_update_steps=1), wall clock
    around work that ends in a device synchronise;
  * kfac_ekfac_statistics + kfac_ekfac_update alone over all layers, CUDA events;
  * the memory of the row buffers, of S / S_batch and of the statistics workspace.
The card's name, power limit and maximum SM clock are printed with the numbers (and written to DIR/ekfac_overhead.json).
"""
import argparse
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
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        q = torch.cuda.get_device_name() + ', power limit unknown'
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    torch.manual_seed(0)
    x = torch.randn(32, 3, 224, 224, device=dev)
    y = torch.randint(0, 1000, (32,), device=dev)
    runs = {}
    for method in ('eigen', 'ekfac'):
        torch.manual_seed(0)
        model = resnet50().to(dev)
        pre = KFACPreconditioner(model, compute_method=method, factor_update_steps=1, inv_update_steps=10 ** 6,
                                 damping=0.001)
        opt = torch.optim.SGD(model.parameters(), lr=0.01)
        runs[method] = (model, pre, opt)

    def one_step(model, pre, opt):
        opt.zero_grad()
        torch.nn.functional.cross_entropy(model(x), y).backward()
        pre.step()
        opt.step()

    for r in runs.values():              # warm-up: inverses, workspaces, cuDNN plans
        for _ in range(3):
            one_step(*r)
    torch.cuda.synchronize()
    times = {k: [] for k in runs}
    for _ in range(args.iters):
        for name, r in runs.items():     # alternate the methods
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            one_step(*r)
            torch.cuda.synchronize()
            times[name].append((time.perf_counter() - t0) * 1e3)

    # the EKFAC phase alone: refill the windows with one forward + backward, then time statistics + update
    model, pre, opt = runs['ekfac']
    ek = [l for _, l in pre._layer_list()]
    phase_ms = []
    for _ in range(args.iters):
        opt.zero_grad()
        torch.nn.functional.cross_entropy(model(x), y).backward()
        pre._flush_factor_updates()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        pre._ekfac_update(new_basis=False)
        e1.record()
        e1.synchronize()
        phase_ms.append(e0.elapsed_time(e1))
    opt.zero_grad()
    rows_bytes = sum(l._rows_x.numel() * 4 + l._rows_g.numel() * 4 for l in ek)
    s_bytes = sum(l._S.numel() * 4 * 2 for l in ek)
    ws_bytes = pre._ekfac_scratch.buf.numel()
    flop = 0
    for l in ek:
        n = l._rows_x.numel() // _cabi.ld4(l.a_dim)
        flop += 2 * n * (l.a_dim ** 2 + l.g_dim ** 2) + 2 * n * l.g_dim * l.a_dim

    def summary(v):
        return {'median_ms': statistics.median(v), 'min_ms': min(v), 'max_ms': max(v), 'n': len(v)}
    out = {'card': card(),
           'workload': 'ResNet-50, batch 32, 224x224, fp32, factor_update_steps=1 (no inverse step timed)',
           'step': {k: summary(v) for k, v in times.items()},
           'ekfac_statistics_and_update': summary(phase_ms),
           'ekfac_algorithmic_gflop': flop / 1e9,
           'row_buffers_gb': rows_bytes / 1e9, 'S_and_S_batch_mb': s_bytes / 1e6,
           'statistics_workspace_gb': ws_bytes / 1e9,
           'max_memory_allocated_gb': torch.cuda.max_memory_allocated() / 1e9}
    print(json.dumps(out, indent=1))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'ekfac_overhead.json'), 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
