"""Cost of preconditioning GroupNorm / InstanceNorm layers (`precondition_group_norms=True`), one GPU.

    python tests/group_norm_overhead.py [--iters N] [--out DIR]

Workloads, each with the keyword off and on (and `precondition_conv_transpose=True` in both), all runs alternated in
one process:
  * a DDPM-CIFAR-shaped U-Net: GroupNorm(32, .) ResBlocks with a time embedding at 128 channels on 32 x 32 and 256
    channels on 16 x 16, a strided-conv down and a ConvTranspose2d up, batch 64 x 3 x 32 x 32, fp32 and bf16 autocast;
  * a CycleGAN / pix2pix-shaped ResNet generator with InstanceNorm2d(affine=True): c7s1-64, two stride-2 convs, nine
    residual blocks at 256 channels on 64 x 64, two ConvTranspose2d ups, c7s1-3; batch 4 x 3 x 256 x 256, fp32.
For inv_update_steps = 1 (every step is a factor and an inverse step) and 10**6 (factor steps without an
eigendecomposition), the medians of forward + backward + step() (wall clock around work that ends in a device
synchronise) and the growth of memory_usage()['total'].  Then kfac_factor_group_norm alone, timed with CUDA events
over many launches, on the U-Net's largest (64 x 128 x 32 x 32) and smallest (64 x 256 x 16 x 16) GroupNorm inputs
and the generator's largest InstanceNorm2d input (4 x 64 x 256 x 256), against its bytes floor: x and g read once each
at the data-sheet 3.35 TB/s of the H100 SXM; and the one copy a channels_last input costs (x.contiguous()).  The
card's name, power limit and maximum SM clock are printed with the numbers (and written to
DIR/group_norm_overhead.json).
"""
import argparse
import json
import math
import os
import statistics
import sys
import time

import torch
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from kfac_b200 import _cabi  # noqa: E402
from kfac_b200.preconditioner import KFACPreconditioner  # noqa: E402
from norm_overhead import HBM_BYTES_PER_S, card, event_ms  # noqa: E402

TEMB = 512


class ResBlock(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.norm1 = nn.GroupNorm(32, c)
        self.conv1 = nn.Conv2d(c, c, 3, padding=1)
        self.temb = nn.Linear(TEMB, c)
        self.norm2 = nn.GroupNorm(32, c)
        self.conv2 = nn.Conv2d(c, c, 3, padding=1)

    def forward(self, x, t):
        h = self.conv1(nn.functional.silu(self.norm1(x))) + self.temb(t)[:, :, None, None]
        return x + self.conv2(nn.functional.silu(self.norm2(h)))


class DDPMUNet(nn.Module):
    def __init__(self):
        super().__init__()
        self.t1, self.t2 = nn.Linear(128, TEMB), nn.Linear(TEMB, TEMB)
        self.conv_in = nn.Conv2d(3, 128, 3, padding=1)
        self.enc = nn.ModuleList([ResBlock(128), ResBlock(128)])
        self.down = nn.Conv2d(128, 256, 3, stride=2, padding=1)
        self.mid = nn.ModuleList([ResBlock(256), ResBlock(256)])
        self.up = nn.ConvTranspose2d(256, 128, 4, stride=2, padding=1)
        self.dec = nn.ModuleList([ResBlock(128), ResBlock(128)])
        self.norm_out = nn.GroupNorm(32, 128)
        self.conv_out = nn.Conv2d(128, 3, 3, padding=1)

    def forward(self, x, t):
        freqs = torch.exp(-math.log(10000.0) * torch.arange(64, device=x.device) / 64)
        t = self.t2(nn.functional.silu(self.t1(torch.cat([torch.sin(t[:, None] * freqs),
                                                           torch.cos(t[:, None] * freqs)], 1))))
        t = nn.functional.silu(t)
        h = self.conv_in(x)
        for b in self.enc:
            h = b(h, t)
        skip = h
        h = self.down(h)
        for b in self.mid:
            h = b(h, t)
        h = self.up(h) + skip
        for b in self.dec:
            h = b(h, t)
        return self.conv_out(nn.functional.silu(self.norm_out(h)))


def _cna(cin, cout, k, stride=1, pad=0, transpose=False):
    conv = (nn.ConvTranspose2d(cin, cout, k, stride, pad, output_padding=1) if transpose
            else nn.Conv2d(cin, cout, k, stride, pad))
    return [conv, nn.InstanceNorm2d(cout, affine=True), nn.ReLU()]


class GenResBlock(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.body = nn.Sequential(nn.ReflectionPad2d(1), *_cna(c, c, 3), nn.ReflectionPad2d(1), nn.Conv2d(c, c, 3),
                                  nn.InstanceNorm2d(c, affine=True))

    def forward(self, x):
        return x + self.body(x)


class ResnetGenerator(nn.Module):
    def __init__(self):
        super().__init__()
        self.net = nn.Sequential(
            nn.ReflectionPad2d(3), *_cna(3, 64, 7), *_cna(64, 128, 3, 2, 1), *_cna(128, 256, 3, 2, 1),
            *[GenResBlock(256) for _ in range(9)],
            *_cna(256, 128, 3, 2, 1, transpose=True), *_cna(128, 64, 3, 2, 1, transpose=True),
            nn.ReflectionPad2d(3), nn.Conv2d(64, 3, 7), nn.Tanh())

    def forward(self, x, t=None):
        return self.net(x)


def stats_kernel(dev):
    lib = _cabi.load()
    out = {}
    cases = [('unet_gn32_128x32x32', (64, 128, 32, 32), 32), ('unet_gn32_256x16x16', (64, 256, 16, 16), 32),
             ('gen_in2d_64x256x256', (4, 64, 256, 256), 64)]
    for name, shape, groups in cases:
        for x_dtype, g_dtype in ((torch.float32, torch.float32), (torch.bfloat16, torch.float32)):
            x = torch.randn(shape, device=dev).to(x_dtype)
            g = torch.randn(shape, device=dev).to(g_dtype)
            B, C = shape[:2]
            S = x.numel() // (B * C)
            acc = torch.zeros(C, 3, device=dev)
            need = lib.kfac_factor_group_norm_workspace_bytes(B, C, S, groups)
            ws = torch.empty(need, dtype=torch.uint8, device=dev)
            stream = _cabi.stream_ptr()
            xc, gc = _cabi.DTYPE_CODE[x_dtype], _cabi.DTYPE_CODE[g_dtype]

            def run():
                _cabi.check(lib.kfac_factor_group_norm(x.data_ptr(), xc, g.data_ptr(), gc, B, C, S, groups, 3, 1e-5,
                                                       1.0, acc.data_ptr(), ws.data_ptr(), need, stream))
            ms = event_ms(run, 200)
            nbytes = x.numel() * x.element_size() + g.numel() * g.element_size()
            key = f'{name}_x{str(x_dtype).split(".")[1]}_g{str(g_dtype).split(".")[1]}'
            out[key] = {'ms': ms, 'input_bytes': nbytes, 'floor_ms': nbytes / HBM_BYTES_PER_S * 1e3,
                        'share_of_3.35TBps': nbytes / (ms * 1e-3) / HBM_BYTES_PER_S}
            if x_dtype == torch.float32:
                # the one copy an input in channels_last strides costs before the statistics
                xl = x.to(memory_format=torch.channels_last)
                out[key]['channels_last_contiguous_ms'] = event_ms(lambda: xl.contiguous(), 200)
                del xl
            del x, g, ws
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    gen = torch.Generator().manual_seed(0)
    data = {'unet': (torch.randn(64, 3, 32, 32, generator=gen).to(dev), (torch.rand(64, generator=gen) * 1000).to(dev),
                     torch.randn(64, 3, 32, 32, generator=gen).to(dev)),
            'gen': (torch.randn(4, 3, 256, 256, generator=gen).to(dev), None,
                    torch.randn(4, 3, 256, 256, generator=gen).to(dev))}
    workloads = [('ddpm_unet_fp32', 'unet', None), ('ddpm_unet_bf16', 'unet', torch.bfloat16),
                 ('resnet_generator_in2d_fp32', 'gen', None)]
    res = {'card': card(), 'iters': args.iters}
    for wname, mname, amp in workloads:
        runs = {}
        for ius in (1, 10 ** 6):
            for on in (False, True):
                torch.manual_seed(0)
                model = (DDPMUNet() if mname == 'unet' else ResnetGenerator()).to(dev)
                pre = KFACPreconditioner(model, factor_update_steps=1, inv_update_steps=ius, damping=1e-3,
                                         precondition_conv_transpose=True, precondition_group_norms=on)
                runs[(ius, on)] = (model, pre)
        x, t, y = data[mname]

        def fwd_bwd(model):
            model.zero_grad()
            with torch.autocast('cuda', dtype=amp, enabled=amp is not None):
                out = model(x, t)
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
        r = {'norm_layers': len(runs[(1, True)][1]._norm_layers), 'kfac_layers': len(runs[(1, True)][1]._layers)}
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
    res['kfac_factor_group_norm'] = stats_kernel(dev)
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'group_norm_overhead.json'), 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
