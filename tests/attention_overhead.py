"""Cost of `precondition_attention`, one GPU.

    python tests/attention_overhead.py [--iters N] [--out DIR]

Workload: a GPT-2-small-shaped nn.TransformerEncoder (12 batch-first layers, E = 768, 12 heads, feed-forward 3072,
dropout 0), batch 8 x 128 tokens, fp32, eigen method, factor_update_steps=1, SDPA on its default backend.  Three
configurations alternate in one process:
  * bare      the model without a preconditioner;
  * skipped   KFACPreconditioner(skip_layers=['self_attn']): the 24 feed-forward Linear layers;
  * attention KFACPreconditioner(precondition_attention=True): those plus 4 projections per block (72 layers).
Reported (medians, wall clock around work that ends in a device synchronise):
  * forward + backward at a factor step, and for `attention` the same with the taps replaced by no-ops (the cost of
    the restated forward alone, against the stock forward of `skipped` / `bare`);
  * step() with an inverse step (inv_update_steps=1) and without one (inv_update_steps=10**6);
  * memory_usage()['total'].
The strided kernels are timed alone with CUDA events over many launches on the shapes of this workload (a q/k/v column
block of the packed (128, 8, 2304) gradient), against the bytes floor (input read once at the data-sheet 3.35 TB/s of
the H100 SXM) and, for the factor SYRK, the fp32 flop floor.  The card's name, power limit and maximum SM clock are
printed with the numbers (and written to DIR/attention_overhead.json).
"""
import argparse
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

from embedding_overhead import card  # noqa: E402
from kfac_b200 import _cabi, attention  # noqa: E402
from kfac_b200.preconditioner import KFACPreconditioner  # noqa: E402

HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet
FP32_FLOPS = 67e12                 # H100 SXM data sheet, dense fp32 (the SIMT factor path)
E, HEADS, LAYERS, B, T = 768, 12, 12, 8, 128


def event_ms(fn, launches):
    fn()
    torch.cuda.synchronize()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(launches):
        fn()
    stop.record()
    stop.synchronize()
    return start.elapsed_time(stop) / launches


def kernels(dev):
    lib = _cabi.load()
    stream = _cabi.stream_ptr()
    rows = T * B
    out = {}
    for dtype in (torch.float32, torch.float16):
        code = _cabi.DTYPE_CODE[dtype]
        g = torch.randn(T, B, 3 * E, device=dev).to(dtype)
        blk = g[..., E:2 * E]
        es = g.element_size()
        acc = torch.zeros(E, E, device=dev)
        need = lib.kfac_factor_linear_strided_workspace_bytes(rows, E, 3 * E, 0)
        ws = torch.empty(max(need, 1), dtype=torch.uint8, device=dev)
        rows_out = torch.empty(rows, _cabi.ld4(E), device=dev)
        red_out = torch.empty(B, E, device=dev)
        cases = {
            'factor_linear_strided': (lambda: _cabi.check(lib.kfac_factor_linear_strided(
                blk.data_ptr(), code, rows, E, 3 * E, 0, 1.0 / rows, acc.data_ptr(), ws.data_ptr(), need, stream)),
                rows * E * es, 2.0 * rows * E * E / 2),
            'rows_linear_strided': (lambda: _cabi.check(lib.kfac_rows_linear_strided(
                blk.data_ptr(), code, rows, E, 3 * E, 0, 1.0, None, rows_out.data_ptr(), _cabi.ld4(E), stream)),
                rows * E * es + rows * _cabi.ld4(E) * 4, 0.0),
            'reduce_rows_linear_strided': (lambda: _cabi.check(lib.kfac_reduce_rows_linear_strided(
                blk.data_ptr(), code, B, T, E, 3 * E, B * 3 * E, 0, 1.0, None, red_out.data_ptr(), E, stream)),
                rows * E * es, 0.0),
        }
        for name, (fn, nbytes, flops) in cases.items():
            ms = event_ms(fn, 200)
            floor = max(nbytes / HBM_BYTES_PER_S, flops / FP32_FLOPS) * 1e3
            out[f'{name} {str(dtype).split(".")[-1]}'] = {'ms': ms, 'floor_ms': floor, 'share': floor / ms,
                                                          'bound': 'flops' if flops / FP32_FLOPS > nbytes / HBM_BYTES_PER_S
                                                          else 'bytes'}
    return out


def make_model(dev):
    torch.manual_seed(0)
    layer = nn.TransformerEncoderLayer(E, HEADS, 4 * E, dropout=0.0, batch_first=True)
    return nn.TransformerEncoder(layer, LAYERS, enable_nested_tensor=False).to(dev)


class _NoTaps:
    """Stands in for the preconditioner inside the attention modules: the restated forward with no-op taps."""

    def __init__(self, keys):
        self.keys = keys

    def _active_attention_taps(self, module):
        return self.keys

    def _attention_input(self, key, x):
        pass

    def _attention_grad_output(self, key, g):
        pass


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    info = card()
    print(info, flush=True)
    result = {'card': info, 'kernels': kernels(dev)}

    x = torch.randn(B, T, E, device=dev)

    def fwd_bwd(model):
        model.zero_grad(set_to_none=False)
        model(x).pow(2).mean().backward()

    # one model per configuration: a preconditioner owns the hooks and the taps of its model
    models = {cfg: make_model(dev) for cfg in ('bare', 'restated')}
    pres = {}
    for inv in ('inverse', 'no_inverse'):
        ius = 1 if inv == 'inverse' else 10 ** 6
        for cfg, kw in (('skipped', dict(skip_layers=['self_attn'])), ('attention', dict(precondition_attention=True))):
            models[(cfg, inv)] = make_model(dev)
            pres[(cfg, inv)] = KFACPreconditioner(models[(cfg, inv)], inv_update_steps=ius, damping=0.003, **kw)
    # the restated forward with no-op taps (no preconditioner, no statistics); the stand-in is referenced weakly by the
    # modules, so it is kept here
    no_taps = _NoTaps({w: w for w in 'qkvo'})
    for m in models['restated'].modules():
        if isinstance(m, nn.MultiheadAttention):
            attention.bind(m, no_taps)

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3

    samples = {}
    for _ in range(2 + args.iters):
        for key, model in models.items():
            name = key if isinstance(key, str) else f'{key[0]} {key[1]}'
            samples.setdefault(f'{name} fwd+bwd', []).append(timed(lambda: fwd_bwd(model)))
            if key in pres:
                samples.setdefault(f'{name} step', []).append(timed(pres[key].step))
    med = {k: statistics.median(v[2:]) for k, v in samples.items()}
    result['ms'] = med
    result['spread_ms'] = {k: (min(v[2:]), max(v[2:])) for k, v in samples.items()}
    result['memory_usage_total_bytes'] = {f'{cfg} {inv}': pres[(cfg, inv)].memory_usage()['total']
                                          for cfg, inv in pres}
    result['layers'] = {cfg: len(pres[(cfg, 'inverse')]._layers) for cfg in ('skipped', 'attention')}
    print(json.dumps(result, indent=1), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'attention_overhead.json'), 'w') as f:
            json.dump(result, f, indent=1)


if __name__ == '__main__':
    main()
