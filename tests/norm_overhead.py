"""Cost of preconditioning the normalization layers (`precondition_norms=True`), one GPU.

    python tests/norm_overhead.py [--iters N] [--out DIR]

Workloads, each with the keyword off and on, all runs alternated in one process:
  * ResNet-50 (53 BatchNorm2d), batch 32 x 3 x 224 x 224, fp32 and fp16 autocast;
  * a GPT-2-small-shaped LayerNorm model: four pre-LN blocks of width 768 (ln_1, ln_2) and a final LayerNorm, batch
    8 x 128 tokens, fp32.
For inv_update_steps = 1 (every step is a factor and an inverse step) and 10**6 (factor steps without an
eigendecomposition), the medians of forward + backward + step() (wall clock around work that ends in a device
synchronise) and the growth of memory_usage()['total'].  Then kfac_factor_norm alone, timed with CUDA events over
many launches, on the largest BatchNorm2d input of ResNet-50 at bs32 (64 x 112 x 112), a late one (2048 x 7 x 7) and
the LayerNorm input of the GPT-2-shaped model (1024 x 768), against its bytes floor: x and g read once each at the
data-sheet 3.35 TB/s of the H100 SXM.  The card's name, power limit and maximum SM clock are printed with the numbers
(and written to DIR/norm_overhead.json).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from kfac_b200 import _cabi  # noqa: E402
from kfac_b200.preconditioner import KFACPreconditioner  # noqa: E402
from workloads import resnet50  # noqa: E402

HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet
D, B_LM, T = 768, 8, 128


class GPT2Block(nn.Module):
    def __init__(self):
        super().__init__()
        self.ln_1 = nn.LayerNorm(D)
        self.c_attn = nn.Linear(D, 3 * D)
        self.c_proj = nn.Linear(D, D)
        self.ln_2 = nn.LayerNorm(D)
        self.c_fc = nn.Linear(D, 4 * D)
        self.mlp_proj = nn.Linear(4 * D, D)

    def forward(self, x):
        q, k, v = self.c_attn(self.ln_1(x)).chunk(3, dim=-1)
        x = x + self.c_proj(torch.tanh(q * k) * v)
        return x + self.mlp_proj(nn.functional.gelu(self.c_fc(self.ln_2(x))))


class GPT2Shaped(nn.Module):
    def __init__(self):
        super().__init__()
        self.blocks = nn.Sequential(*[GPT2Block() for _ in range(4)])
        self.ln_f = nn.LayerNorm(D)

    def forward(self, x):
        return self.ln_f(self.blocks(x))


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        q = torch.cuda.get_device_name() + ', power limit unknown'
    return q


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


def stats_kernel(dev):
    lib = _cabi.load()
    out = {}
    cases = [('bn2d_64x112x112', _cabi.KFAC_NORM_BATCH, (32, 64, 112, 112), 3),
             ('bn2d_2048x7x7', _cabi.KFAC_NORM_BATCH, (32, 2048, 7, 7), 3),
             ('ln_1024x768', _cabi.KFAC_NORM_LAYER, (B_LM * T, D), 3)]
    for name, kind, shape, k in cases:
        for dtype in (torch.float32, torch.float16):
            x = torch.randn(shape, device=dev).to(dtype)
            g = torch.randn(shape, device=dev).to(dtype)
            C = shape[1]
            rows, S = (shape[0], x.numel() // (shape[0] * C)) if kind == _cabi.KFAC_NORM_BATCH else (shape[0], 1)
            acc = torch.zeros(C, k, device=dev)
            need = lib.kfac_factor_norm_workspace_bytes(kind, rows, C, S)
            ws = torch.empty(need, dtype=torch.uint8, device=dev)
            stream = _cabi.stream_ptr()
            code = _cabi.DTYPE_CODE[dtype]

            def run():
                _cabi.check(lib.kfac_factor_norm(x.data_ptr(), code, g.data_ptr(), code, kind, rows, C, S, k, 1e-5,
                                                 1.0, acc.data_ptr(), ws.data_ptr(), need, stream))
            ms = event_ms(run, 100)
            nbytes = 2 * x.numel() * x.element_size()
            out[f'{name}_{str(dtype).split(".")[1]}'] = {
                'ms': ms, 'input_bytes': nbytes, 'floor_ms': nbytes / HBM_BYTES_PER_S * 1e3,
                'share_of_3.35TBps': nbytes / (ms * 1e-3) / HBM_BYTES_PER_S}
            del x, g, ws
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    gen = torch.Generator().manual_seed(0)
    data = {'resnet50': (torch.randn(32, 3, 224, 224, generator=gen).to(dev), torch.randint(0, 1000, (32,)).to(dev)),
            'gpt2': (torch.randn(B_LM, T, D, generator=gen).to(dev), torch.randn(B_LM, T, D, generator=gen).to(dev))}
    workloads = [('resnet50_fp32', 'resnet50', None), ('resnet50_fp16', 'resnet50', torch.float16),
                 ('gpt2_ln_fp32', 'gpt2', None)]
    res = {'card': card(), 'iters': args.iters}
    for wname, mname, amp in workloads:
        runs = {}
        for ius in (1, 10 ** 6):
            for on in (False, True):
                torch.manual_seed(0)
                model = (resnet50() if mname == 'resnet50' else GPT2Shaped()).to(dev)
                pre = KFACPreconditioner(model, factor_update_steps=1, inv_update_steps=ius, damping=1e-3,
                                         precondition_norms=on)
                runs[(ius, on)] = (model, pre)
        x, y = data[mname]

        def fwd_bwd(model):
            model.zero_grad()
            with torch.autocast('cuda', dtype=amp, enabled=amp is not None):
                out = model(x)
            if mname == 'resnet50':
                nn.functional.cross_entropy(out.float(), y).backward()
            else:
                nn.functional.mse_loss(out.float(), y).backward()

        times = {key: [] for key in runs}
        for it in range(args.iters + 2):          # two warm-up rounds
            for key, (model, pre) in runs.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fwd_bwd(model)
                pre.step()
                torch.cuda.synchronize()
                if it >= 2:
                    times[key].append((time.perf_counter() - t0) * 1e3)
        r = {'norm_layers': len(runs[(1, True)][1]._norm_layers)}
        for (ius, on), (model, pre) in runs.items():
            key = ('on' if on else 'off') + ('' if ius == 1 else '_no_inverse_step')
            r[key] = {'fwd_bwd_step_ms_median': statistics.median(times[(ius, on)]),
                      'memory_usage_total_bytes': int(pre.memory_usage()['total'])}
        for suffix in ('', '_no_inverse_step'):
            r['extra_ms' + suffix] = (r['on' + suffix]['fwd_bwd_step_ms_median']
                                      - r['off' + suffix]['fwd_bwd_step_ms_median'])
        r['extra_memory_usage_bytes'] = r['on']['memory_usage_total_bytes'] - r['off']['memory_usage_total_bytes']
        res[wname] = r
        del runs
        torch.cuda.empty_cache()
    res['kfac_factor_norm'] = stats_kernel(dev)
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'norm_overhead.json'), 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
