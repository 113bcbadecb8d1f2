"""Cost of pi-adjusted damping on ResNet-50 (batch 32, fp32, one GPU).

    python tests/pi_damping_overhead.py [--iters N] [--out DIR]

Two preconditioners on two copies of the model, pi_damping=False and True, measured alternately in one process:
  * step() at an inverse step and at a step that is not one (the forward and backward pass run before and are not
    timed), wall clock around work that ends in a device synchronise, medians over --iters;
  * the lone kfac_pi launch over all layers, CUDA events, median over 200 launches.
Prints one JSON line with the card's name, power limit and maximum SM clock (also written to DIR/pi_damping_overhead.json).
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
    dev = torch.device('cuda')
    g = torch.Generator().manual_seed(0)
    x = torch.randn(32, 3, 224, 224, generator=g).to(dev)
    y = torch.randint(0, 1000, (32,), generator=g).to(dev)
    runs = {}
    for on in (False, True):
        torch.manual_seed(0)
        model = resnet50().to(dev)
        # inv_update_steps=2: even steps are inverse steps, odd ones are not
        pre = KFACPreconditioner(model, damping=0.003, inv_update_steps=2, pi_damping=on)
        runs[on] = (model, pre)
    times = {(on, inv): [] for on in (False, True) for inv in (True, False)}
    ce = torch.nn.CrossEntropyLoss()
    for it in range(2 * (args.iters + 2)):
        inv = it % 2 == 0
        for on in ((False, True) if it % 4 < 2 else (True, False)):
            model, pre = runs[on]
            model.zero_grad()
            ce(model(x), y).backward()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            pre.step()
            torch.cuda.synchronize()
            if it >= 4:                          # the first two steps of each kind warm up
                times[(on, inv)].append((time.perf_counter() - t0) * 1e3)
    # the lone kfac_pi launch over all layers of the pi_damping preconditioner
    _, pre = runs[True]
    lib = _cabi.load()
    layers = [l for l in pre._layouts if l.pi_damping]
    items = (_cabi.PiItem * len(layers))()
    for i, l in enumerate(layers):
        items[i] = _cabi.PiItem(l._a_view.data_ptr(), l._g_view.data_ptr(), l._inv['pi'].data_ptr(), l.a_dim, l.g_dim,
                                0 if l.diag_a else l.a_dim, 0 if l.diag_g else l.g_dim)
    stream = _cabi.stream_ptr()
    for _ in range(20):
        _cabi.check(lib.kfac_pi(items, len(layers), stream), 'kfac_pi')
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(200)]
    for a, b in ev:
        a.record()
        _cabi.check(lib.kfac_pi(items, len(layers), stream), 'kfac_pi')
        b.record()
    torch.cuda.synchronize()
    pi_us = statistics.median(a.elapsed_time(b) for a, b in ev) * 1e3
    med = {f'{"pi" if on else "base"}_{"inverse" if inv else "plain"}_step_ms': round(statistics.median(v), 3)
           for (on, inv), v in times.items()}
    out = dict(workload='resnet50 batch 32 fp32', card=card(), layers=len(layers), iters=args.iters,
               kfac_pi_us=round(pi_us, 2), **med)
    print(json.dumps(out))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'pi_damping_overhead.json'), 'w') as f:
            json.dump(out, f, indent=1)
    for _, pre in runs.values():
        pre.close()


if __name__ == '__main__':
    main()
