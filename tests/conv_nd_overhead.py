"""Cost of preconditioning Conv1d / Conv3d layers (`precondition_conv_nd=True`) on one GPU.

    python tests/conv_nd_overhead.py [--reps 3] [--out DIR]

Models:
  * torchvision r2plus1d_18, randomly initialised (no weights are downloaded), on 8 x 3 x 16 x 112^2 clips, in fp32 and
    under fp16 autocast: every conv is a Conv3d below 8192 features; its BatchNorm3d layers stay unregistered;
  * a wav2vec2-shaped feature encoder: seven bias-less Conv1d layers (512 channels, kernels 10, 3 x 4, 2 x 2, strides
    5, 2 x 6) with GELU, on 8 x 16000 samples, and a Linear head.
Per model, keyword off vs on, alternating in one process, for expand and reduce and for eigen and EKFAC: forward +
backward at a factor step, step() with and without an inverse step, memory_usage() and the peak im2col workspace.  Then
each N-d input kernel alone, with CUDA events, on the models' shapes against its HBM floor (bytes it must move at
3.35 TB/s) and, for the expand factor, the SYRK's 2 rows F^2 flop.  Prints one JSON line per measurement.
"""
import argparse
import ctypes
import gc
import json
import os
import statistics
import sys

import torch
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from kfac_b200 import _cabi  # noqa: E402
from kfac_b200.layers import CONV_ND_WORKSPACE_BYTES, ConvNdModuleHelper  # noqa: E402
from kfac_b200.preconditioner import KFACPreconditioner  # noqa: E402

DEV = torch.device('cuda')
HBM = 3.35e12


class Wav2Vec2Encoder(nn.Module):
    def __init__(self):
        super().__init__()
        spec = [(1, 10, 5)] + [(512, 3, 2)] * 4 + [(512, 2, 2)] * 2
        self.convs = nn.ModuleList(nn.Conv1d(c, 512, k, stride=s, bias=False) for c, k, s in spec)
        self.head = nn.Linear(512, 32)

    def forward(self, x):
        x = x.unsqueeze(1)
        for c in self.convs:
            x = nn.functional.gelu(c(x))
        return self.head(x.mean(-1))


def models():
    from torchvision.models.video import r2plus1d_18
    return {
        'r2plus1d_18': (lambda: r2plus1d_18(num_classes=400), (8, 3, 16, 112, 112), 400),
        'wav2vec2_encoder': (Wav2Vec2Encoder, (8, 16000), 32),
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


def model_costs(name, make, shape, classes, amp, approx, method, reps, emit):
    torch.manual_seed(0)
    gen = torch.Generator(device=DEV).manual_seed(1)
    # four distinct batches, cycled, as a training run sees
    data = [(torch.randn(*shape, device=DEV, generator=gen), torch.randint(0, classes, (shape[0],), device=DEV,
                                                                          generator=gen)) for _ in range(4)]
    base = make().to(DEV)
    rows = {}
    for rnd in range(2):                      # alternate off / on twice
        for on in (False, True):
            oom = None
            try:
                rows.setdefault(on, []).append(_one_config(make, base, data, on, amp, approx, method, reps))
            except torch.OutOfMemoryError as e:
                oom = str(e).split('.')[0]
            if oom is not None:                # outside the handler: the traceback no longer holds the model
                gc.collect()
                torch.cuda.empty_cache()
                emit(dict(kind='model', model=name, amp=amp, approx=approx, method=method, conv_nd=on,
                          out_of_memory=oom))
                return
    for on, rs in rows.items():
        emit(dict(kind='model', model=name, amp=amp, approx=approx, method=method, conv_nd=on,
                  **{k: statistics.median(r[k] for r in rs) for k in rs[0]}))


def _one_config(make, base, data, on, amp, approx, method, reps):
    """The timings of one model / keyword setting (a fresh model and preconditioner, released on return)."""
    m = make().to(DEV)
    m.load_state_dict(base.state_dict())
    pre = None
    try:
        pre = KFACPreconditioner(m, precondition_conv_nd=on, kfac_approx=approx, compute_method=method,
                                 factor_update_steps=1, inv_update_steps=1, damping=0.003)

        def fwd_bwd():
            x, y = data[pre.steps % len(data)]
            m.zero_grad(set_to_none=True)
            with torch.autocast('cuda', dtype=torch.float16, enabled=amp):
                loss = nn.functional.cross_entropy(m(x), y)
            loss.backward()

        pre._inv_update_steps = 10 ** 9        # only step 0 decomposes; the factor hooks run at every step
        fb, fb_spread = timed(fwd_bwd, reps, after=pre.step)
        pre._inv_update_steps = 1
        inv, inv_spread = timed(lambda: (fwd_bwd(), pre.step()), max(2, reps // 2))
        pre._inv_update_steps = 10 ** 9
        noinv, noinv_spread = timed(lambda: (fwd_bwd(), pre.step()), reps)
        mem = sum(v for v in pre.memory_usage().values() if isinstance(v, int))
        ws = pre._scratch.buf.numel() if pre._scratch.buf is not None else 0
        return dict(fwd_bwd_ms=fb, step_inv_ms=inv - fb, step_noinv_ms=noinv - fb,
                    spread_ms=max(fb_spread, inv_spread, noinv_spread), memory_usage_bytes=mem, scratch_bytes=ws,
                    layers=len(pre._layers))
    finally:
        if pre is not None:
            pre.close()
        del pre, m
        gc.collect()                           # the model's hooks and the preconditioner reference each other
        torch.cuda.empty_cache()


def kernel_costs(name, make, shape, reps, emit):
    """Each N-d input kernel alone on the shapes of the model's Conv1d / Conv3d layers."""
    lib = _cabi.load()
    m = make().to(DEV)
    calls = []
    for mod in m.modules():
        if isinstance(mod, (nn.Conv1d, nn.Conv3d)):
            mod.register_forward_pre_hook(lambda mm, i: calls.append((mm, i[0].detach())))
    with torch.no_grad():
        m(torch.randn(*shape, device=DEV))
    for mod, x in calls:
        h = ConvNdModuleHelper(mod)
        geo, Sp, _ = h._input_geometry(x.shape)
        d = h.a_factor_shape[0]
        ones = int(h.has_bias())
        B = geo.batch
        acc = torch.zeros(d, d, device=DEV)
        need = lib.kfac_factor_conv_input_workspace_bytes(ctypes.byref(geo), ones, CONV_ND_WORKSPACE_BYTES)
        ws = torch.empty(max(need, 1), dtype=torch.uint8, device=DEV)
        st = _cabi.stream_ptr()
        xb = x.numel() * x.element_size()
        rows = B * Sp
        red = torch.empty(B, d, device=DEV)
        fac = lambda: lib.kfac_factor_conv_input(x.data_ptr(), 0, ctypes.byref(geo), ones, 1.0, acc.data_ptr(),  # noqa
                                                 ws.data_ptr(), need, st)
        rdc = lambda: lib.kfac_reduce_rows_conv_input(x.data_ptr(), 0, ctypes.byref(geo), ones, 1.0,  # noqa
                                                      red.data_ptr(), d, st)
        t_f, s_f = timed(fac, reps)
        t_r, s_r = timed(rdc, reps)
        general = {}
        if isinstance(mod, nn.Conv1d) and mod.padding_mode == 'zeros':
            # the general kernel on the same row: a two-row input whose second row no window touches (kh = 1, sh = 2)
            x2 = torch.zeros(B, x.shape[-2] if x.dim() == 3 else 1, 2, x.shape[-1], device=DEV)
            x2[:, :, 0] = x
            g2 = _cabi.ConvGeometry.from_buffer_copy(geo)
            g2.input[1], g2.stride[1] = 2, 2
            red2 = torch.empty_like(red)
            gen_fn = lambda: lib.kfac_reduce_rows_conv_input(x2.data_ptr(), 0, ctypes.byref(g2), ones, 1.0,  # noqa
                                                             red2.data_ptr(), d, st)
            t_g, s_g = timed(gen_fn, reps)
            torch.cuda.synchronize()
            general = dict(reduce_general_kernel_ms=t_g, reduce_general_spread_ms=s_g,
                           reduce_bitwise_equal=bool(torch.equal(red, red2)))
        # expand: read x, write and read back the fp32 im2col (unless read in place); reduce: read x once
        im2col = 0 if need < rows * d * 4 else rows * d * 4
        floor_f = max((xb + 2 * im2col) / HBM, 2.0 * rows * d * d / 495e12) * 1e3
        emit(dict(kind='kernel', model=name, layer=repr(mod), rows=rows, features=d, workspace_bytes=need,
                  factor_ms=t_f, factor_spread_ms=s_f, factor_floor_ms=floor_f,
                  syrk_tflops=2.0 * rows * d * d / (t_f * 1e-3) / 1e12,
                  reduce_ms=t_r, reduce_spread_ms=s_r, reduce_floor_ms=xb / HBM * 1e3, **general))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--out', default=None)
    ap.add_argument('--no-kernels', action='store_true', help='skip the kernels-alone timings')
    ap.add_argument('--models', nargs='*', default=None, help='a subset of the models (default: all)')
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'conv_nd_overhead.py measures on a CUDA device'
    torch.backends.cudnn.benchmark = True
    lines = []

    def emit(d):
        lines.append(d)
        print(json.dumps(d), flush=True)

    emit(dict(kind='device', name=torch.cuda.get_device_name()))
    for name, (make, shape, classes) in models().items():
        if args.models and name not in args.models:
            continue
        if not args.no_kernels:
            kernel_costs(name, make, shape, args.reps, emit)
        for amp in ((False, True) if name == 'r2plus1d_18' else (False,)):
            for approx in ('expand', 'reduce'):
                for method in ('eigen', 'ekfac'):
                    model_costs(name, make, shape, classes, amp, approx, method, args.reps, emit)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'conv_nd_overhead.jsonl'), 'w') as f:
            f.writelines(json.dumps(d) + '\n' for d in lines)


if __name__ == '__main__':
    main()
