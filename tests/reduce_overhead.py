"""Cost of K-FAC-expand and K-FAC-reduce (`kfac_approx`), one GPU.

    python tests/reduce_overhead.py [--iters N] [--out DIR]

Workloads, fp32, factor_update_steps=1:
  * ResNet-50, batch 32 x 3 x 224 x 224;
  * the GPT-2-small-shaped model of tests/embedding_overhead.py (embedding skipped, head skipped: the two NeoX blocks'
    Linear layers), batch 8 x 128 tokens.
For the eigen and EKFAC methods, with inv_update_steps = 1 (every step inverts) and 10**6 (no inverse step in the
window), expand and reduce are alternated in one process with a model without a preconditioner: medians of forward +
backward + step() and of forward + backward alone (wall clock around work that ends in a device synchronise).  The
factor-hook time is the forward + backward time over that of the bare model.  memory_usage() and the native launches
per step are reported too.  The three reduce-row kernels are timed first, alone, with CUDA events over many launches on the
largest inputs of the two workloads, against their bytes floor (the input read once at the data-sheet 3.35 TB/s of
the H100 SXM).  The card's name, power limit and maximum SM clock are printed with the numbers (and written to
DIR/reduce_overhead.json).
"""
import argparse
import gc
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

from embedding_overhead import GPT2Shaped, card  # noqa: E402
from kfac_b200 import _cabi  # noqa: E402
from kfac_b200.preconditioner import KFACPreconditioner  # noqa: E402
from workloads import resnet50  # noqa: E402

HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet


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
    cases = {
        # name: (entry, shape, call)
        'linear_8x128x3072': ('linear', (8, 128, 3072)),
        'linear_8x128x768': ('linear', (8, 128, 768)),
        'conv_input_stem_32x3x224x224_k7s2p3': ('conv_input', (32, 3, 224, 224, 7, 7, 2, 2, 3, 3)),
        'conv_input_32x64x56x56_k3s1p1': ('conv_input', (32, 64, 56, 56, 3, 3, 1, 1, 1, 1)),
        'conv_input_32x256x56x56_k1s1p0': ('conv_input', (32, 256, 56, 56, 1, 1, 1, 1, 0, 0)),
        'conv_input_32x512x7x7_k3s1p1': ('conv_input', (32, 512, 7, 7, 3, 3, 1, 1, 1, 1)),
        'conv_gradout_32x64x112x112': ('gradout', (32, 64, 112, 112)),
        'conv_gradout_32x256x56x56': ('gradout', (32, 256, 56, 56)),
        'conv_gradout_32x2048x7x7': ('gradout', (32, 2048, 7, 7)),
    }
    out = {}
    for name, (kind, geo) in cases.items():
        for dtype in (torch.float32, torch.float16):
            code = _cabi.DTYPE_CODE[dtype]
            if kind == 'linear':
                x = torch.randn(geo, device=dev).to(dtype)
                B, R, F = geo
                o = torch.empty(B, _cabi.ld4(F + 1), device=dev)

                def run():
                    _cabi.check(lib.kfac_reduce_rows_linear(x.data_ptr(), code, B, R, F, 1, 1.0 / R, None, o.data_ptr(),
                                                            _cabi.ld4(F + 1), stream))
            elif kind == 'conv_input':
                B, C, H, W = geo[:4]
                x = torch.randn(B, C, H, W, device=dev).to(dtype)
                d = C * geo[4] * geo[5] + 1
                o = torch.empty(B, _cabi.ld4(d), device=dev)

                def run():
                    _cabi.check(lib.kfac_reduce_rows_conv2d_input(x.data_ptr(), code, *geo, 1, 1.0, o.data_ptr(),
                                                                  _cabi.ld4(d), stream))
            else:
                B, C, Ho, Wo = geo
                x = torch.randn(geo, device=dev).to(dtype)
                o = torch.empty(B, _cabi.ld4(C), device=dev)

                def run():
                    _cabi.check(lib.kfac_reduce_rows_conv2d_gradout(x.data_ptr(), code, B, C, Ho, Wo, 1.0, None,
                                                                    o.data_ptr(), _cabi.ld4(C), stream))
            ms = event_ms(run, 200)
            nbytes = x.numel() * x.element_size()
            out[f'{name}_{str(dtype).split(".")[1]}'] = {
                'ms': ms, 'input_bytes': nbytes, 'floor_ms': nbytes / HBM_BYTES_PER_S * 1e3,
                'share_of_3.35TBps': nbytes / (ms * 1e-3) / HBM_BYTES_PER_S}
            del x, o
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    gen = torch.Generator().manual_seed(0)
    data = {'resnet50': (torch.randn(32, 3, 224, 224, generator=gen).to(dev),
                         torch.randint(0, 1000, (32,), generator=gen).to(dev)),
            'gpt2': (torch.randint(0, 50257, (8, 128), generator=gen).to(dev),
                     torch.randint(0, 50257, (8, 128), generator=gen).to(dev))}
    res = {'card': card(), 'iters': args.iters}
    lib = _cabi.load()
    res['reduce_kernels'] = kernels(dev)
    print(json.dumps(res['reduce_kernels']), flush=True)
    for wname in ('resnet50', 'gpt2'):
        x, y = data[wname]

        def make():
            torch.manual_seed(0)
            return (resnet50() if wname == 'resnet50' else GPT2Shaped()).to(dev)

        def fwd_bwd(model):
            model.zero_grad()
            out = model(x)
            if wname == 'resnet50':
                nn.functional.cross_entropy(out, y).backward()
            else:
                nn.functional.cross_entropy(out.flatten(0, 1), y.flatten()).backward()

        bare = make()
        for method in ('eigen', 'ekfac'):
            for ius in (1, 10 ** 6):
                runs = {}
                for approx in ('expand', 'reduce'):
                    model = make()
                    pre = KFACPreconditioner(model, factor_update_steps=1, inv_update_steps=ius, damping=1e-3,
                                             compute_method=method, kfac_approx=approx,
                                             skip_layers=['emb', 'head'] if wname == 'gpt2' else None)
                    runs[approx] = (model, pre)
                runs['bare'] = (bare, None)
                fb = {k: [] for k in runs}
                tot = {k: [] for k in runs}
                launches = {k: [] for k in runs}
                for it in range(args.iters + 2):        # two warm-up rounds
                    for key, (model, pre) in runs.items():
                        torch.cuda.synchronize()
                        n0 = lib.kfac_launch_count()
                        t0 = time.perf_counter()
                        fwd_bwd(model)
                        torch.cuda.synchronize()
                        t1 = time.perf_counter()
                        if pre is not None:
                            pre.step()
                        torch.cuda.synchronize()
                        t2 = time.perf_counter()
                        if it >= 2:
                            fb[key].append((t1 - t0) * 1e3)
                            tot[key].append((t2 - t0) * 1e3)
                            launches[key].append(lib.kfac_launch_count() - n0)
                bare_fb = statistics.median(fb['bare'])
                r = {'bare_fwd_bwd_ms_median': bare_fb}
                for approx in ('expand', 'reduce'):
                    pre = runs[approx][1]
                    mem = pre.memory_usage()
                    r[approx] = {'fwd_bwd_step_ms_median': statistics.median(tot[approx]),
                                 'fwd_bwd_ms_median': statistics.median(fb[approx]),
                                 'factor_hooks_ms': statistics.median(fb[approx]) - bare_fb,
                                 'step_ms_median': statistics.median(tot[approx]) - statistics.median(fb[approx]),
                                 'native_launches_per_step': statistics.median(launches[approx]),
                                 'memory_usage_bytes': {k: int(v) for k, v in mem.items()}}
                res[f'{wname}_{method}' + ('' if ius == 1 else '_no_inverse_step')] = r
                print(json.dumps({f'{wname}_{method}_{ius}': r}), flush=True)
                del runs, pre, model
                gc.collect()            # the hooks keep a preconditioner and its model in a reference cycle
                torch.cuda.empty_cache()
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'reduce_overhead.json'), 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
