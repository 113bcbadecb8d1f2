"""Cost of preconditioning nn.EmbeddingBag layers (`precondition_embedding_bags`) on two seeded models (one GPU, fp32).

    python tests/embedding_bag_overhead.py [--iters N] [--out DIR]

Models:
  * the text classifier of PyTorch's text-classification tutorial: EmbeddingBag(95811, 64, mode='mean') +
    Linear(64, 4), 64 bags of 20-200 tokens drawn log-uniformly over the vocabulary (a heavy head of frequent tokens);
  * a DLRM-shaped recommender: bottom MLP 13-512-256-64, 8 x EmbeddingBag(10**6, 64, mode='sum') with bags of 1-64
    uniform indices, top MLP 576-512-256-1 on the concatenation, batch 2048.
For each model, with inv_update_steps = 1 (every step decomposes the factors) and 10**6 (no eigendecomposition in the
timed window) and the keyword off and on, all four measured alternately in one process:
  * step() alone, wall clock around work that ends in a device synchronise;
  * memory_usage()['total'];
and the A kernel's time per call (kfac_factor_embedding_bag on the model's batch, CUDA events over 200 calls; for the
DLRM one table).  The card's name, power limit and maximum SM clock are printed with the numbers (and written to
DIR/embedding_bag_overhead.json).
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


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        q = torch.cuda.get_device_name() + ', power limit unknown'
    return q


class TextClassifier(nn.Module):
    def __init__(self):
        super().__init__()
        self.bag = nn.EmbeddingBag(95811, 64, mode='mean')
        self.fc = nn.Linear(64, 4)

    def forward(self, batch):
        idx, offsets, _ = batch
        return self.fc(self.bag(idx, offsets))

    def loss(self, batch):
        return nn.functional.cross_entropy(self(batch), batch[2])


def mlp(sizes, last_relu):
    layers = []
    for i in range(len(sizes) - 1):
        layers.append(nn.Linear(sizes[i], sizes[i + 1]))
        if i < len(sizes) - 2 or last_relu:
            layers.append(nn.ReLU())
    return nn.Sequential(*layers)


class DLRM(nn.Module):
    def __init__(self):
        super().__init__()
        self.bottom = mlp((13, 512, 256, 64), True)
        self.tables = nn.ModuleList(nn.EmbeddingBag(10 ** 6, 64, mode='sum') for _ in range(8))
        self.top = mlp((576, 512, 256, 1), False)

    def forward(self, batch):
        dense, sparse, _ = batch
        z = [self.bottom(dense)] + [t(i, o) for t, (i, o) in zip(self.tables, sparse)]
        return self.top(torch.cat(z, 1)).squeeze(1)

    def loss(self, batch):
        return nn.functional.binary_cross_entropy_with_logits(self(batch), batch[2])


def bags(g, B, lo, hi, draw):
    lens = torch.randint(lo, hi + 1, (B,), generator=g)
    offsets = torch.cat([torch.zeros(1, dtype=torch.long), lens.cumsum(0)[:-1]])
    return draw(int(lens.sum())), offsets


def batches(dev):
    g = torch.Generator().manual_seed(0)
    V = 95811
    idx, off = bags(g, 64, 20, 200, lambda n: (V ** torch.rand(n, generator=g)).long().clamp(max=V) - 1)
    tc = (idx.to(dev), off.to(dev), torch.randint(0, 4, (64,), generator=g).to(dev))
    sparse = [tuple(t.to(dev) for t in bags(g, 2048, 1, 64, lambda n: torch.randint(0, 10 ** 6, (n,), generator=g)))
              for _ in range(8)]
    dlrm = (torch.randn(2048, 13, generator=g).to(dev), sparse,
            torch.randint(0, 2, (2048,), generator=g).float().to(dev))
    return tc, dlrm


def kernel_ms(module, idx, offsets, calls=200):
    """Time per call of kfac_factor_embedding_bag on one bag module's input (CUDA events)."""
    lib = _cabi.load()
    V, B, n = module.num_embeddings, offsets.numel(), idx.numel()
    need = lib.kfac_factor_embedding_bag_workspace_bytes(n, B, V)
    ws = torch.empty(need, dtype=torch.uint8, device=idx.device)
    acc = torch.zeros(V, device=idx.device)
    mode = {'sum': _cabi.KFAC_BAG_SUM, 'mean': _cabi.KFAC_BAG_MEAN}[module.mode]
    stream = torch.cuda.current_stream().cuda_stream

    def call():
        _cabi.check(lib.kfac_factor_embedding_bag(idx.data_ptr(), offsets.data_ptr(), _cabi.INDEX_DTYPE_CODE[idx.dtype],
                                                  n, B, -1, mode, None, 0, V, 1.0 / B, acc.data_ptr(),
                                                  ws.data_ptr(), need, stream), 'kfac_factor_embedding_bag')
    for _ in range(10):
        call()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(calls):
        call()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / calls


def measure(model_cls, batch, iters, dev):
    runs = {}
    for ius in (1, 10 ** 6):
        for flag in (False, True):
            torch.manual_seed(0)
            model = model_cls().to(dev)
            pre = KFACPreconditioner(model, precondition_embedding_bags=flag, factor_update_steps=1,
                                     inv_update_steps=ius, damping=0.003)
            runs[(ius, flag)] = (model, pre)
    times = {key: [] for key in runs}
    for it in range(iters + 2):                 # two warm-up rounds
        for key, (model, pre) in runs.items():
            model.zero_grad()
            model.loss(batch).backward()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            pre.step()
            torch.cuda.synchronize()
            if it >= 2:
                times[key].append((time.perf_counter() - t0) * 1e3)
    res = {}
    for (ius, flag), (model, pre) in runs.items():
        key = ('on' if flag else 'off') + ('' if ius == 1 else '_no_inverse_step')
        res[key] = {'step_ms_median': statistics.median(times[(ius, flag)]),
                    'memory_usage_total_bytes': int(pre.memory_usage()['total'])}
    for suffix in ('', '_no_inverse_step'):
        res['extra_step_ms' + suffix] = res['on' + suffix]['step_ms_median'] - res['off' + suffix]['step_ms_median']
    res['extra_memory_usage_bytes'] = res['on']['memory_usage_total_bytes'] - res['off']['memory_usage_total_bytes']
    del runs
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    tc, dlrm = batches(dev)
    res = {'card': card(), 'iters': args.iters}
    probe = TextClassifier().to(dev)
    res['text_classifier'] = {'model': 'EmbeddingBag(95811, 64, mean) + Linear(64, 4), 64 bags of 20-200 tokens',
                              'indices': int(tc[0].numel()),
                              'a_kernel_ms_per_call': kernel_ms(probe.bag, tc[0], tc[1])}
    del probe
    res['text_classifier'].update(measure(TextClassifier, tc, args.iters, dev))
    table = nn.EmbeddingBag(10 ** 6, 64, mode='sum')
    res['dlrm'] = {'model': 'MLP 13-512-256-64, 8 x EmbeddingBag(10**6, 64, sum), bags of 1-64, MLP 576-512-256-1, '
                            'batch 2048',
                   'indices_per_table': int(dlrm[1][0][0].numel()),
                   'a_kernel_ms_per_call': kernel_ms(table, *dlrm[1][0])}
    res['dlrm'].update(measure(DLRM, dlrm, args.iters, dev))
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'embedding_bag_overhead.json'), 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
