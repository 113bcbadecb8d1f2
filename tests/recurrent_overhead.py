"""Cost of `precondition_recurrent`, one GPU.

    python tests/recurrent_overhead.py [--iters N] [--out DIR]

Workloads: a 2-layer bidirectional nn.LSTM with input 1024 and H = 1024 (layer-1 ih A 2049, G 4096), T = 128, B = 32,
fp32, and a GRU of the same shape (G 3072); eigen method, factor_update_steps=1.  Configurations alternate in one
process:
  * stock      the module without a preconditioner (cuDNN);
  * restated   the restated forward with no-op taps (no preconditioner, no statistics);
  * recurrent  KFACPreconditioner(precondition_recurrent=True): 8 sub-layers.
Reported (medians, wall clock around work that ends in a device synchronise): forward + backward at a factor step;
step() with an inverse step (inv_update_steps=1) and without one (inv_update_steps=10**6); memory_usage()['total'].
The sequence row writers are timed alone with CUDA events on this workload's shapes (the forward hidden-state gather of
one direction, the GRU hidden G rows) against the bytes floor at the data-sheet 3.35 TB/s of the H100 SXM.  The card's
name, power limit and maximum SM clock are printed with the numbers (and written to DIR/recurrent_overhead.json).
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys
import time

import torch
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from attention_overhead import event_ms  # noqa: E402
from embedding_overhead import card  # noqa: E402
from kfac_b200 import _cabi, recurrent  # noqa: E402
from kfac_b200.preconditioner import KFACPreconditioner  # noqa: E402

HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet
I, H, LAYERS, T, B = 1024, 1024, 2, 128, 32


def kernels(dev):
    lib = _cabi.load()
    stream = _cabi.stream_ptr()
    N = T * B
    out = {}
    y = torch.randn(T, B, 2 * H, device=dev)
    h0 = torch.randn(B, H, device=dev)
    g = torch.randn(T, B, 3 * H, device=dev)
    r = torch.rand(T, B, H, device=dev)
    gather = _cabi.SequenceRows(y.data_ptr(), 2 * H, 0, h0.data_ptr(), H, 1, None, 0, 0, T, B, None)
    gru = _cabi.SequenceRows(g.data_ptr(), 3 * H, 0, None, 0, 0, r.data_ptr(), H, 2 * H, T, B, None)
    rows_a = torch.empty(N, H + 1, device=dev)
    rows_g = torch.empty(N, 3 * H, device=dev)
    red = torch.empty(B, H + 1, device=dev)
    cases = {
        'rows_sequence hidden gather': (lambda: _cabi.check(lib.kfac_rows_sequence(
            C.byref(gather), 0, H, 1, 1.0, None, rows_a.data_ptr(), H + 1, stream)), N * H * 4 * 2),
        'rows_sequence gru hidden G': (lambda: _cabi.check(lib.kfac_rows_sequence(
            C.byref(gru), 0, 3 * H, 0, 1.0, None, rows_g.data_ptr(), 3 * H, stream)), N * 4 * H * 4 + N * 3 * H * 4),
        'reduce_rows_sequence hidden gather': (lambda: _cabi.check(lib.kfac_reduce_rows_sequence(
            C.byref(gather), 0, H, 1, 1.0, 1.0, None, red.data_ptr(), H + 1, stream)), N * H * 4),
    }
    for name, (fn, nbytes) in cases.items():
        ms = event_ms(fn, 100)
        floor = nbytes / HBM_BYTES_PER_S * 1e3
        out[name] = {'ms': ms, 'floor_ms': floor, 'share': floor / ms}
    return out


def make_model(mode, dev):
    torch.manual_seed(0)
    cls = nn.LSTM if mode == 'LSTM' else nn.GRU
    return cls(I, H, num_layers=LAYERS, bidirectional=True).to(dev)


class _NoTaps:
    """Stands in for the preconditioner inside the recurrent module: the restated forward with no-op taps."""

    def __init__(self, keys):
        self.keys = keys

    def _active_recurrent_taps(self, module):
        return self.keys

    def _recurrent_input(self, key, x, tap):
        pass

    def _recurrent_grad_output(self, key, g, tap):
        pass


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    info = card()
    print(info, flush=True)
    result = {'card': info, 'kernels': kernels(dev), 'ms': {}, 'spread_ms': {}, 'memory_usage_total_bytes': {}}
    x = torch.randn(T, B, I, device=dev)

    def fwd_bwd(model):
        model.zero_grad(set_to_none=False)
        model(x)[0].pow(2).mean().backward()

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3

    keys = [f'{s}_l{k}{sfx}' for k in range(LAYERS) for sfx in ('', '_reverse') for s in ('ih', 'hh')]
    no_taps = _NoTaps({k: type('Key', (), {'suffix': k})() for k in keys})
    for mode in ('LSTM', 'GRU'):
        models = {cfg: make_model(mode, dev) for cfg in ('stock', 'restated')}
        recurrent.bind(models['restated'], no_taps)
        pres = {}
        for inv in ('inverse', 'no_inverse'):
            models[inv] = make_model(mode, dev)
            pres[inv] = KFACPreconditioner(models[inv], inv_update_steps=1 if inv == 'inverse' else 10 ** 6,
                                           damping=0.003, precondition_recurrent=True)
        samples = {}
        for _ in range(2 + args.iters):
            for cfg, model in models.items():
                name = cfg if cfg in ('stock', 'restated') else f'recurrent {cfg}'
                samples.setdefault(f'{mode} {name} fwd+bwd', []).append(timed(lambda: fwd_bwd(model)))
                if cfg in pres:
                    samples.setdefault(f'{mode} {name} step', []).append(timed(pres[cfg].step))
        result['ms'].update({k: statistics.median(v[2:]) for k, v in samples.items()})
        result['spread_ms'].update({k: (min(v[2:]), max(v[2:])) for k, v in samples.items()})
        result['memory_usage_total_bytes'][mode] = pres['inverse'].memory_usage()['total']
        del models, pres
        torch.cuda.empty_cache()
    print(json.dumps(result, indent=1), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'recurrent_overhead.json'), 'w') as f:
            json.dump(result, f, indent=1)


if __name__ == '__main__':
    main()
