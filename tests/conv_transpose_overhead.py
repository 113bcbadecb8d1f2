"""Cost of preconditioning ConvTranspose layers (`precondition_conv_transpose=True`) on one GPU.

    python tests/conv_transpose_overhead.py [--reps 5] [--out DIR]

Models:
  * the DCGAN 64 x 64 generator (z of 100, widths 512-256-128-64, bias-less ConvTranspose2d layers with BatchNorm2d and
    ReLU) at batch 128: the first stride-2 layer has A = 512 * 16 = 8192, the eigensolver's limit;
  * a U-Net decoder at batch 8 on a 1024 x 16^2 bottleneck: four ConvTranspose2d(k = 2, s = 2) steps called with
    output_size=..., each followed by a 3 x 3 Conv2d, up to 64 x 256^2.
Per model, keyword off vs on, alternating in one process, for expand and reduce (eigen): forward + backward at a factor
step, step() with and without an inverse step.  Then each transposed layer's factor kernel alone, with CUDA events, and
the SYRK's rate counting every row and feature, the inserted zeros included (2 rows d^2 flop).  Prints one JSON line per
measurement, the first with the card's name and power limit.
"""
import argparse
import ctypes
import gc
import json
import os
import statistics
import subprocess
import sys

import torch
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from kfac_b200 import _cabi  # noqa: E402
from kfac_b200.layers import CONV_ND_WORKSPACE_BYTES, ConvTransposeModuleHelper  # noqa: E402
from kfac_b200.preconditioner import KFACPreconditioner  # noqa: E402

DEV = torch.device('cuda')


class DCGANGenerator(nn.Module):
    def __init__(self, nz=100, ngf=64):
        super().__init__()
        w = [ngf * 8, ngf * 4, ngf * 2, ngf]
        layers = [nn.ConvTranspose2d(nz, w[0], 4, 1, 0, bias=False), nn.BatchNorm2d(w[0]), nn.ReLU(True)]
        for a, b in zip(w, w[1:]):
            layers += [nn.ConvTranspose2d(a, b, 4, 2, 1, bias=False), nn.BatchNorm2d(b), nn.ReLU(True)]
        layers += [nn.ConvTranspose2d(ngf, 3, 4, 2, 1, bias=False), nn.Tanh()]
        self.main = nn.Sequential(*layers)

    def forward(self, z):
        return self.main(z)


class UNetDecoder(nn.Module):
    def __init__(self, widths=(1024, 512, 256, 128, 64)):
        super().__init__()
        self.ups = nn.ModuleList(nn.ConvTranspose2d(a, b, 2, stride=2) for a, b in zip(widths, widths[1:]))
        self.convs = nn.ModuleList(nn.Conv2d(b, b, 3, padding=1) for b in widths[1:])
        self.head = nn.Conv2d(widths[-1], 2, 1)

    def forward(self, x):
        for up, conv in zip(self.ups, self.convs):
            B, _, H, W = x.shape
            x = torch.relu(conv(up(x, output_size=(B, up.out_channels, 2 * H, 2 * W))))
        return self.head(x)


MODELS = {
    'dcgan64': (DCGANGenerator, (128, 100, 1, 1)),
    'unet_decoder': (UNetDecoder, (8, 1024, 16, 16)),
}


def timed(fn, reps, after=None):
    """(median, max - min) ms of `reps` calls of fn, each between CUDA events, after one warm-up call; `after` runs
    untimed after every call."""
    out = []
    for r in range(reps + 1):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        if r:
            out.append(e0.elapsed_time(e1))
        if after is not None:
            after()
            torch.cuda.synchronize()
    return statistics.median(out), (max(out) - min(out))


def model_costs(name, make, shape, approx, reps, emit):
    torch.manual_seed(0)
    gen = torch.Generator(device=DEV).manual_seed(1)
    base = make().to(DEV)
    with torch.no_grad():
        out_shape = base(torch.zeros(*shape, device=DEV)).shape
    data = [(torch.randn(*shape, device=DEV, generator=gen), torch.randn(*out_shape, device=DEV, generator=gen))
            for _ in range(4)]
    rows = {}
    for _ in range(2):                        # alternate off / on twice
        for on in (False, True):
            rows.setdefault(on, []).append(_one_config(make, base, data, on, approx, reps))
    for on, rs in rows.items():
        emit(dict(kind='model', model=name, approx=approx, method='eigen', conv_transpose=on,
                  **{k: statistics.median(r[k] for r in rs) for k in rs[0]}))


def _one_config(make, base, data, on, approx, reps):
    m = make().to(DEV)
    m.load_state_dict(base.state_dict())
    pre = None
    try:
        pre = KFACPreconditioner(m, precondition_conv_transpose=on, kfac_approx=approx, factor_update_steps=1,
                                 inv_update_steps=1, damping=0.003)

        def fwd_bwd():
            x, y = data[pre.steps % len(data)]
            m.zero_grad(set_to_none=True)
            nn.functional.mse_loss(m(x), y).backward()

        pre._inv_update_steps = 10 ** 9        # only step 0 decomposes; the factor hooks run at every step
        fb, fb_spread = timed(fwd_bwd, reps, after=pre.step)
        pre._inv_update_steps = 1
        inv, inv_spread = timed(lambda: (fwd_bwd(), pre.step()), max(2, reps // 2))
        pre._inv_update_steps = 10 ** 9
        noinv, noinv_spread = timed(lambda: (fwd_bwd(), pre.step()), reps)
        return dict(fwd_bwd_ms=fb, step_inv_ms=inv - fb, step_noinv_ms=noinv - fb,
                    spread_ms=max(fb_spread, inv_spread, noinv_spread), layers=len(pre._layers),
                    largest_a=max((l.a_dim for _, l in pre._layers.values()), default=0))
    finally:
        if pre is not None:
            pre.close()
        del pre, m
        gc.collect()
        torch.cuda.empty_cache()


def kernel_costs(name, make, shape, reps, emit):
    """The factor kernel of each transposed layer alone, on the model's shapes."""
    lib = _cabi.load()
    m = make().to(DEV)
    calls = []
    for mod in m.modules():
        if isinstance(mod, nn.ConvTranspose2d):
            mod.register_forward_pre_hook(lambda mm, a, kw: calls.append((mm, a, kw)), with_kwargs=True)
    with torch.no_grad():
        m(torch.randn(*shape, device=DEV))
    st = _cabi.stream_ptr()
    for mod, args, kwargs in calls:
        h = ConvTransposeModuleHelper(mod)
        h.bind_call(args, kwargs)
        x = h.prepare_input(args[0])
        geo, out = h._geometry(x.shape)
        d = h.a_factor_shape[0]
        ones = int(h.has_bias())
        rows = geo.batch * out[0] * out[1]
        acc = torch.zeros(d, d, device=DEV)
        need = lib.kfac_factor_conv_transpose_input_workspace_bytes(ctypes.byref(geo), ones, CONV_ND_WORKSPACE_BYTES)
        ws = torch.empty(max(need, 1), dtype=torch.uint8, device=DEV)
        red = torch.empty(geo.batch, d, device=DEV)
        fac = lambda: lib.kfac_factor_conv_transpose_input(x.data_ptr(), 0, ctypes.byref(geo), ones, 1.0,  # noqa
                                                           acc.data_ptr(), ws.data_ptr(), need, st)
        rdc = lambda: lib.kfac_reduce_rows_conv_transpose_input(x.data_ptr(), 0, ctypes.byref(geo), ones, 1.0,  # noqa
                                                                red.data_ptr(), d, st)
        t_f, s_f = timed(fac, reps)
        t_r, s_r = timed(rdc, reps)
        phases = 1
        for s in mod.stride:
            phases *= s * s
        emit(dict(kind='kernel', model=name, layer=repr(mod), rows=rows, features=d, workspace_bytes=need,
                  factor_ms=t_f, factor_spread_ms=s_f, syrk_tflops=2.0 * rows * d * d / (t_f * 1e-3) / 1e12,
                  phase_blocks_flop_ratio=phases if mod.dilation == (1, 1) else 1,
                  reduce_ms=t_r, reduce_spread_ms=s_r))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'conv_transpose_overhead.py measures on a CUDA device'
    torch.backends.cudnn.benchmark = True
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    lines = []

    def emit(d):
        lines.append(d)
        print(json.dumps(d), flush=True)

    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader',
                          '-i', str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    emit(dict(kind='device', name=torch.cuda.get_device_name(), nvidia_smi=smi))
    for name, (make, shape) in MODELS.items():
        kernel_costs(name, make, shape, args.reps, emit)
        for approx in ('expand', 'reduce'):
            model_costs(name, make, shape, approx, args.reps, emit)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'conv_transpose_overhead.jsonl'), 'w') as f:
            f.writelines(json.dumps(d) + '\n' for d in lines)


if __name__ == '__main__':
    main()
