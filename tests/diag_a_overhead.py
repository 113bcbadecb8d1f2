"""Cost of diagonal-A layers on one GPU (not a test; run by hand, writes JSON lines to stdout).

1. A LLaMA-7B-shaped MLP block (d = 4096, hidden = 11008, SwiGLU, no biases) on 8 x 128 tokens: gate_proj and up_proj
   keep a diagonal G (11008 outputs), down_proj (11008 inputs) is either skipped or in diagonal_a_layers.  Reported:
   the time of step() alone and of the whole training step (forward, backward, step()), with and without an inverse
   step (inv_update_steps=10), the two configurations alternated in one process, medians over the steps.
2. kfac_factor_conv_input_diag on a 3 x 3 convolution with 1280 channels (a diffusion U-Net's widest), fp32 and bf16:
   its time, its achieved bandwidth against the read-once floor (B * C * H * W elements at the 3.35 TB/s of the H100
   SXM data sheet), and the im2col route on the same input (kfac_rows_conv_input writing the fp32 im2col rows, then
   kfac_factor_linear_diag on them, rows padded to ld4(d) columns).

    python tests/diag_a_overhead.py [--repeats 2]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import torch
from torch import nn
from torch.nn import functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from kfac_b200 import _cabi  # noqa: E402
from kfac_b200.preconditioner import KFACPreconditioner  # noqa: E402

HBM_BYTES_PER_S = 3.35e12      # H100 SXM data sheet


class MLP(nn.Module):
    def __init__(self, d=4096, hidden=11008):
        super().__init__()
        self.gate_proj = nn.Linear(d, hidden, bias=False)
        self.up_proj = nn.Linear(d, hidden, bias=False)
        self.down_proj = nn.Linear(hidden, d, bias=False)

    def forward(self, x):
        return self.down_proj(F.silu(self.gate_proj(x)) * self.up_proj(x))


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def timed(fn, n):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(n):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / n


def mlp_block(steps):
    dev = torch.device('cuda')
    torch.manual_seed(0)
    x = torch.randn(8, 128, 4096, device=dev)
    target = torch.randn(8, 128, 4096, device=dev)
    runs = {}
    for cfg, kw in (('skip', dict(skip_layers=['down_proj'])), ('diag', dict(diagonal_a_layers=['down_proj']))):
        torch.manual_seed(0)
        model = MLP().to(dev)
        pre = KFACPreconditioner(model, diagonal_g_layers=['gate_proj', 'up_proj'], inv_update_steps=10, **kw)
        runs[cfg] = (model, pre)
    res = {k: {'step_ms': [], 'step_inv_ms': [], 'train_ms': [], 'train_inv_ms': []} for k in runs}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    for cfg, (model, pre) in runs.items():     # warm-up: shapes, workspaces, the first inverse step
        for _ in range(3):
            model.zero_grad(set_to_none=False)
            F.mse_loss(model(x), target).backward()
            pre.step()
    for _ in range(steps):
        for cfg, (model, pre) in runs.items():
            inv = pre.steps % pre.inv_update_steps == 0
            torch.cuda.synchronize()
            ev[0].record()
            model.zero_grad(set_to_none=False)
            F.mse_loss(model(x), target).backward()
            ev[1].record()
            pre.step()
            ev[2].record()
            torch.cuda.synchronize()
            res[cfg]['step_inv_ms' if inv else 'step_ms'].append(ev[1].elapsed_time(ev[2]))
            res[cfg]['train_inv_ms' if inv else 'train_ms'].append(ev[0].elapsed_time(ev[2]))
    out = {}
    for cfg, r in res.items():
        out[cfg] = {k: (sorted(v)[len(v) // 2] if v else None) for k, v in r.items()}
    out['diag_minus_skip_ms'] = {k: out['diag'][k] - out['skip'][k] for k in out['diag'] if out['diag'][k] is not None
                                 and out['skip'][k] is not None}
    return out


def conv_kernel(dtype, B=8, Cc=1280, H=32, W=32, reps=50):
    lib = _cabi.load()
    dev = torch.device('cuda')
    x = torch.randn(B, Cc, H, W, device=dev).to(dtype)
    arr = lambda v: (C.c_int * 3)(*v)  # noqa: E731
    geo = _cabi.ConvGeometry(B, Cc, arr((1, H, W)), arr((1, 3, 3)), arr((1, 1, 1)), arr((1, 1, 1)), arr((0, 1, 1)),
                             arr((0, 1, 1)))
    d = Cc * 9 + 1
    acc = torch.zeros(_cabi.ld4(d), device=dev)
    stream = torch.cuda.current_stream().cuda_stream
    code = _cabi.DTYPE_CODE[dtype]
    need = lib.kfac_factor_conv_input_diag_workspace_bytes(C.byref(geo))
    ws = torch.empty(need, dtype=torch.uint8, device=dev)

    def diag():
        _cabi.check(lib.kfac_factor_conv_input_diag(x.data_ptr(), code, C.byref(geo), 1, 1.0, acc.data_ptr(),
                                                    ws.data_ptr(), need, stream), 'kfac_factor_conv_input_diag')
    rows, ld = B * H * W, _cabi.ld4(d)
    im = torch.empty(rows, ld, device=dev)
    need2 = lib.kfac_factor_linear_diag_workspace_bytes(rows, ld)
    ws2 = torch.empty(need2, dtype=torch.uint8, device=dev)

    def im2col():
        _cabi.check(lib.kfac_rows_conv_input(x.data_ptr(), code, C.byref(geo), 1, 1.0, im.data_ptr(), ld, stream),
                    'kfac_rows_conv_input')
        _cabi.check(lib.kfac_factor_linear_diag(im.data_ptr(), 0, rows, ld, 1.0, acc.data_ptr(), ws2.data_ptr(), need2,
                                                stream), 'kfac_factor_linear_diag')
    for fn in (diag, im2col):
        fn()
    t_diag = timed(diag, reps)
    t_im = timed(im2col, reps)
    floor_s = x.numel() * x.element_size() / HBM_BYTES_PER_S
    return {'dtype': str(dtype).split('.')[-1], 'shape': [B, Cc, H, W], 'diag_ms': t_diag, 'im2col_route_ms': t_im,
            'read_once_floor_ms': floor_s * 1e3, 'diag_share_of_floor': floor_s * 1e3 / t_diag,
            'diag_GBps': x.numel() * x.element_size() / (t_diag * 1e-3) / 1e9, 'speedup_vs_im2col': t_im / t_diag}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeats', type=int, default=2)
    ap.add_argument('--steps', type=int, default=20)
    args = ap.parse_args()
    print(json.dumps({'card': card()}), flush=True)
    for r in range(args.repeats):
        print(json.dumps({'repeat': r, 'mlp_block': mlp_block(args.steps)}), flush=True)
        for dtype in (torch.float32, torch.bfloat16):
            print(json.dumps({'repeat': r, 'conv_diag': conv_kernel(dtype)}), flush=True)


if __name__ == '__main__':
    main()
