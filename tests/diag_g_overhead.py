"""Cost of preconditioning the LM head of a GPT-2-small-shaped model with a diagonal G (one GPU, fp32).

    python tests/diag_g_overhead.py [--iters N] [--out DIR]

Model: nn.Embedding(50257, 768) -> two GPT-NeoX blocks of width 768 -> Linear head 768 -> 50257 (no bias), batch
8 x 128 tokens.  The head is in skip_layers in one run and in diagonal_g_layers in the other.  With
factor_update_steps = 1, inv_update_steps = 1 (every step decomposes the factors) and 10**6 (no eigendecomposition in
the timed window), all four measured alternately in one process:
  * step() alone and forward + backward + step(), wall clock around work that ends in a device synchronise;
  * memory_usage()['total'] and the precondition workspace.
Then, timed with CUDA events over many launches:
  * kfac_factor_linear_diag alone at N in {1024, 16384} rows x V = 50257, fp32 and bf16, with the bytes it must read
    (N * V * element size) over its time against the data-sheet 3.35 TB/s of the H100 SXM;
  * the head's precondition products alone (one diagonal-G item, V = 50257, a = 768), eigen and inverse.
The card's name, power limit and maximum SM clock are printed with the numbers (and written to
DIR/diag_g_overhead.json).
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
from workloads import NeoXBlock  # noqa: E402

V, D, B, T = 50257, 768, 8, 128
HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet


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


def factor_kernel(dev):
    lib = _cabi.load()
    out = {}
    for rows in (1024, 16384):
        for dtype in (torch.float32, torch.bfloat16):
            x = torch.randn(rows, V, device=dev).to(dtype)
            acc = torch.zeros(V, device=dev)
            need = lib.kfac_factor_linear_diag_workspace_bytes(rows, V)
            ws = torch.empty(need, dtype=torch.uint8, device=dev)
            stream = _cabi.stream_ptr()

            def run():
                _cabi.check(lib.kfac_factor_linear_diag(x.data_ptr(), _cabi.DTYPE_CODE[dtype], rows, V, 1.0 / rows,
                                                        acc.data_ptr(), ws.data_ptr(), need, stream))
            ms = event_ms(run, 200)
            nbytes = rows * V * x.element_size()
            out[f'N{rows}_{str(dtype).split(".")[1]}'] = {
                'ms': ms, 'input_bytes': nbytes, 'floor_ms': nbytes / HBM_BYTES_PER_S * 1e3,
                'bytes_per_s': nbytes / (ms * 1e-3), 'share_of_3.35TBps': nbytes / (ms * 1e-3) / HBM_BYTES_PER_S}
            del x, ws
    return out


def head_precondition(dev):
    """The head's products alone: one diagonal-G item of V x a = 50257 x 768."""
    lib = _cabi.load()
    a = D
    q, _ = torch.linalg.qr(torch.randn(a, a, device=dev))
    da = torch.rand(a, device=dev)
    dg = torch.rand(V, device=dev)
    a_inv = (q / (da + 0.003)) @ q.t()
    w = torch.randn(V, a, device=dev)
    P = torch.empty(V, a, device=dev)
    qT = q.t().contiguous()
    out = {}
    for name, method in (('eigen', _cabi.KFAC_EIGEN), ('inverse', _cabi.KFAC_INVERSE)):
        e = method == _cabi.KFAC_EIGEN
        items = (_cabi.PrecondItem * 1)()
        items[0] = _cabi.PrecondItem(w.data_ptr(), None, 0, V, a, q.data_ptr() if e else None,
                                     qT.data_ptr() if e else None, None, None, None, da.data_ptr() if e else None,
                                     dg.data_ptr(), None if e else a_inv.data_ptr(), None, a, 0, 0, P.data_ptr(), a,
                                     None, 0, _cabi.KFAC_ITEM_DIAG_G)
        need = lib.kfac_precondition_workspace_bytes(items, 1)
        ws = torch.empty(need, dtype=torch.uint8, device=dev)
        stream = _cabi.stream_ptr()

        def run():
            _cabi.check(lib.kfac_precondition(items, 1, method, 0.003, ws.data_ptr(), need, stream))
        ms = event_ms(run, 50)
        flop = (4 if e else 2) * V * a * a
        out[name] = {'ms': ms, 'flop': flop, 'tflop_per_s': flop / (ms * 1e-3) / 1e12, 'workspace_bytes': need}
    return out


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
        for diag in (False, True):
            torch.manual_seed(0)
            model = GPT2Shaped().to(dev)
            kw = dict(diagonal_g_layers=['head']) if diag else dict(skip_layers=['head'])
            pre = KFACPreconditioner(model, factor_update_steps=1, inv_update_steps=ius, damping=0.003, **kw)
            runs[(ius, diag)] = (model, pre)

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
    res = {'card': card(), 'model': f'Embedding({V}, {D}) + 2 NeoX blocks + head {D}->{V}, batch {B}x{T}, fp32',
           'iters': args.iters}
    for (ius, diag), (model, pre) in runs.items():
        key = ('diag' if diag else 'skip') + ('' if ius == 1 else '_no_inverse_step')
        res[key] = {'step_ms_median': statistics.median(times[(ius, diag)]['step']),
                    'fwd_bwd_step_ms_median': statistics.median(times[(ius, diag)]['total']),
                    'memory_usage_total_bytes': int(pre.memory_usage()['total']),
                    'precondition_workspace_bytes': int(pre._gemm_scratch.buf.numel())}
    for suffix in ('', '_no_inverse_step'):
        res['extra_step_ms' + suffix] = res['diag' + suffix]['step_ms_median'] - res['skip' + suffix]['step_ms_median']
    res['extra_memory_usage_bytes'] = (res['diag']['memory_usage_total_bytes']
                                       - res['skip']['memory_usage_total_bytes'])
    res['extra_workspace_bytes'] = (res['diag']['precondition_workspace_bytes']
                                    - res['skip']['precondition_workspace_bytes'])
    del runs
    torch.cuda.empty_cache()
    res['kfac_factor_linear_diag'] = factor_kernel(dev)
    res['head_precondition'] = head_precondition(dev)
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'diag_g_overhead.json'), 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
