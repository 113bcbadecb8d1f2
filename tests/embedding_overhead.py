"""Cost of preconditioning the token embedding of a GPT-2-small-shaped model (one GPU, fp32).

    python tests/embedding_overhead.py [--iters N] [--out DIR]

Model: nn.Embedding(50257, 768) -> two GPT-NeoX blocks of width 768 -> Linear head 768 -> 50257, batch 8 x 128
tokens.  The head is in skip_layers in both runs (its G, 50257 x 50257, is beyond the eigensolver).  With
factor_update_steps = 1, inv_update_steps = 1 (every step decomposes the factors) and 10**6 (no
eigendecomposition in the timed window), and precondition_embeddings off and on, all four measured alternately in one
process:
  * step() alone and forward + backward + step(), wall clock around work that ends in a device synchronise;
  * memory_usage()['total'] and the precondition workspace.
The card's name, power limit and maximum SM clock are printed with the numbers (and written to
DIR/embedding_overhead.json).
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


class GPT2Shaped(nn.Module):
    def __init__(self):
        super().__init__()
        self.emb = nn.Embedding(V, D)
        self.blocks = nn.Sequential(NeoXBlock(D), NeoXBlock(D))
        self.head = nn.Linear(D, V, bias=False)

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
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(0)
    idx = torch.randint(0, V, (B, T), generator=g).to(dev)
    y = torch.randint(0, V, (B, T), generator=g).to(dev)
    runs = {}
    for ius in (1, 10 ** 6):
        for flag in (False, True):
            torch.manual_seed(0)
            model = GPT2Shaped().to(dev)
            pre = KFACPreconditioner(model, precondition_embeddings=flag, skip_layers=['head'], factor_update_steps=1,
                                     inv_update_steps=ius, damping=0.003)
            runs[(ius, flag)] = (model, pre)

    def fwd_bwd(model):
        model.zero_grad()
        nn.functional.cross_entropy(model(idx).flatten(0, 1), y.flatten()).backward()

    times = {key: {'step': [], 'total': []} for key in runs}
    for it in range(args.iters + 2):            # two warm-up rounds
        for key, (model, pre) in runs.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fwd_bwd(model)
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            pre.step()
            torch.cuda.synchronize()
            t2 = time.perf_counter()
            if it >= 2:
                times[key]['step'].append((t2 - t1) * 1e3)
                times[key]['total'].append((t2 - t0) * 1e3)
    res = {'card': card(), 'model': f'Embedding({V}, {D}) + 2 NeoX blocks + head (skipped), batch {B}x{T}, fp32',
           'iters': args.iters}
    for (ius, flag), (model, pre) in runs.items():
        key = ('on' if flag else 'off') + ('' if ius == 1 else '_no_inverse_step')
        res[key] = {'step_ms_median': statistics.median(times[(ius, flag)]['step']),
                    'fwd_bwd_step_ms_median': statistics.median(times[(ius, flag)]['total']),
                    'memory_usage_total_bytes': int(pre.memory_usage()['total']),
                    'precondition_workspace_bytes': int(pre._gemm_scratch.buf.numel())}
    for suffix in ('', '_no_inverse_step'):
        res['extra_step_ms' + suffix] = res['on' + suffix]['step_ms_median'] - res['off' + suffix]['step_ms_median']
    res['extra_memory_usage_bytes'] = res['on']['memory_usage_total_bytes'] - res['off']['memory_usage_total_bytes']
    res['extra_workspace_bytes'] = res['on']['precondition_workspace_bytes'] - res['off']['precondition_workspace_bytes']
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'embedding_overhead.json'), 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
