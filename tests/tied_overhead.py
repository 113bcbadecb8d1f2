"""Cost of preconditioning a tied embedding / LM head as a pair (one GPU, fp32).

    python tests/tied_overhead.py [--iters N] [--out DIR]

Model: nn.Embedding(50257, 768) -> two GPT-NeoX blocks of width 768 -> Linear head 768 -> 50257 (no bias) whose weight
is the embedding's, batch 8 x 128 tokens.  With precondition_embeddings and the head in diagonal_g_layers, the head is
in skip_layers in one run ("head skipped": the embedding alone preconditions the weight) and the two form a pair in
the other (precondition_tied_embeddings).  With factor_update_steps = 1 and inv_update_steps = 1 (every step decomposes
the factors) and 10**6 (no decomposition in the timed window), all four measured alternately in one process, wall
clock around work that ends in a device synchronise:
  * forward + backward (the factor hooks included) and step();
  * memory_usage()['total'].
The card's name, power limit and maximum SM clock are printed with the numbers (and written to
DIR/tied_overhead.json).
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

from kfac_b200.preconditioner import KFACPreconditioner  # noqa: E402
from workloads import NeoXBlock  # noqa: E402

V, D, B, T = 50257, 768, 8, 128


class TiedGPT2Shaped(nn.Module):
    def __init__(self):
        super().__init__()
        self.emb = nn.Embedding(V, D)
        self.blocks = nn.Sequential(NeoXBlock(D), NeoXBlock(D))
        self.head = nn.Linear(D, V, bias=False)
        self.head.weight = self.emb.weight

    def forward(self, idx):
        return self.head(self.blocks(self.emb(idx)))


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
    if not torch.cuda.is_available():
        raise SystemExit('tied_overhead.py measures on a CUDA device; none is available')
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(0)
    idx = torch.randint(0, V, (B, T), generator=g).to(dev)
    y = torch.randint(0, V, (B, T), generator=g).to(dev)
    runs = {}
    for ius in (1, 10 ** 6):
        for tied in (False, True):
            torch.manual_seed(0)
            model = TiedGPT2Shaped().to(dev)
            kw = dict(precondition_tied_embeddings=True) if tied else dict(skip_layers=['head'])
            pre = KFACPreconditioner(model, factor_update_steps=1, inv_update_steps=ius, damping=0.003,
                                     precondition_embeddings=True, diagonal_g_layers=['head'], **kw)
            runs[(ius, tied)] = (model, pre)

    times = {key: {'fwd_bwd': [], 'step': []} for key in runs}
    for it in range(args.iters + 2):            # two warm-up rounds
        for key, (model, pre) in runs.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            model.zero_grad()
            nn.functional.cross_entropy(model(idx).flatten(0, 1), y.flatten()).backward()
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            pre.step()
            torch.cuda.synchronize()
            t2 = time.perf_counter()
            if it >= 2:
                times[key]['fwd_bwd'].append((t1 - t0) * 1e3)
                times[key]['step'].append((t2 - t1) * 1e3)
    res = {'card': card(), 'model': f'tied Embedding({V}, {D}) / head {D}->{V} + 2 NeoX blocks, batch {B}x{T}, fp32',
           'iters': args.iters}
    for (ius, tied), (model, pre) in runs.items():
        key = ('tied' if tied else 'head_skipped') + ('' if ius == 1 else '_no_inverse_step')
        t = times[(ius, tied)]
        res[key] = {'fwd_bwd_ms_median': statistics.median(t['fwd_bwd']),
                    'step_ms_median': statistics.median(t['step']),
                    'step_ms_min_max': [min(t['step']), max(t['step'])],
                    'memory_usage_total_bytes': int(pre.memory_usage()['total'])}
    for suffix in ('', '_no_inverse_step'):
        res['extra_step_ms' + suffix] = (res['tied' + suffix]['step_ms_median']
                                         - res['head_skipped' + suffix]['step_ms_median'])
        res['extra_fwd_bwd_ms' + suffix] = (res['tied' + suffix]['fwd_bwd_ms_median']
                                            - res['head_skipped' + suffix]['fwd_bwd_ms_median'])
    res['extra_memory_usage_bytes'] = (res['tied']['memory_usage_total_bytes']
                                       - res['head_skipped']['memory_usage_total_bytes'])
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'tied_overhead.json'), 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
