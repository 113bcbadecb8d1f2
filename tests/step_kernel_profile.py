"""Per-kernel breakdown of bench-shaped ResNet-50 K-FAC steps (diagnostic, not a pytest).

Builds the benchmark's workload on its own (ResNet-50, batch 32 of 224 x 224, factor and inverse updates every
step, SGD lr 0.1 with momentum, eight distinct random batches cycled), warms up, then records a few steps with
torch.profiler (CUDA activities) and writes the kernels sorted by total device time:

    python tests/step_kernel_profile.py OUT_DIR [--steps 3] [--warmup 3]

OUT_DIR/kernels.md   name, launches, total ms, ms per step, share of the summed kernel time
OUT_DIR/kernels.json the same rows, plus the card, its power limit and the wall time per profiled step
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
from collections import defaultdict

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader',
                            '-i', '0'], capture_output=True, text=True, timeout=30)
        return q.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return 'unknown'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('out')
    ap.add_argument('--steps', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)

    from kfac_b200.preconditioner import KFACPreconditioner
    from workloads import resnet50

    assert torch.cuda.is_available(), 'step_kernel_profile.py needs a CUDA device'
    dev = torch.device('cuda:0')
    torch.manual_seed(0)
    model = resnet50().to(dev)
    pre = KFACPreconditioner(model, factor_update_steps=1, inv_update_steps=1, damping=0.001, factor_decay=0.95,
                             kl_clip=0.001, lr=0.1)
    opt = torch.optim.SGD(model.parameters(), lr=0.1, momentum=0.9)
    crit = torch.nn.CrossEntropyLoss()
    torch.manual_seed(1)
    batches = [(torch.randn(32, 3, 224, 224, device=dev), torch.randint(0, 1000, (32,), device=dev)) for _ in range(8)]
    it = {'i': 0}

    def step():
        x, y = batches[it['i'] % len(batches)]
        it['i'] += 1
        opt.zero_grad(set_to_none=True)
        crit(model(x), y).backward()
        pre.step()
        opt.step()

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        t0 = time.perf_counter()
        for _ in range(args.steps):
            step()
        torch.cuda.synchronize()
        wall = (time.perf_counter() - t0) * 1e3 / args.steps

    launches, total_us = defaultdict(int), defaultdict(float)
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        launches[ev.name] += 1
        total_us[ev.name] += ev.time_range.elapsed_us()
    summed = sum(total_us.values())
    rows = sorted(({'name': n, 'launches': launches[n], 'total_ms': total_us[n] / 1e3,
                    'ms_per_step': total_us[n] / 1e3 / args.steps, 'share': total_us[n] / summed}
                   for n in total_us), key=lambda r: -r['total_ms'])
    info = {'card': card(), 'steps': args.steps, 'wall_ms_per_step_profiled': wall,
            'kernel_ms_per_step': summed / 1e3 / args.steps, 'kernels': rows}
    with open(os.path.join(args.out, 'kernels.json'), 'w') as f:
        json.dump(info, f, indent=1)
    with open(os.path.join(args.out, 'kernels.md'), 'w') as f:
        f.write(f"card: {info['card']}; {args.steps} profiled steps, {wall:.1f} ms wall per step under the profiler, "
                f"{info['kernel_ms_per_step']:.1f} ms of kernels per step\n\n")
        f.write('| kernel | launches | total ms | ms / step | share |\n|---|---|---|---|---|\n')
        for r in rows:
            name = r['name'] if len(r['name']) <= 110 else r['name'][:107] + '...'
            f.write(f"| `{name}` | {r['launches']} | {r['total_ms']:.2f} | {r['ms_per_step']:.2f} | "
                    f"{100 * r['share']:.1f} % |\n")
    print(open(os.path.join(args.out, 'kernels.md')).read()[:6000])


if __name__ == '__main__':
    main()
