#!/usr/bin/env python
"""bench.py -- K-FAC hot path on ResNet-50 (ImageNet-shaped synthetic data).

    python bench.py --gpus N --steps K --warmup W            (own arm, H100)
    python bench.py ... --dump-outputs DIR                    (also write the last timed step's outputs as .npy)
    python bench.py --impl reference --gpus N --steps K ...   (CPU reference arm)

A "step" is one full training iteration of the data-parallel K-FAC hot path:
forward + backward with the factor hooks (K1-K4), `preconditioner.step()`
(factor EMA/all-reduce, eigendecompositions, precondition, kl-clip, write-back)
and the SGD update, with `factor_update_steps = inv_update_steps = 1`, i.e.
EVERY step runs every stage of the path (SURVEY.md 8(d) "stress 1/1").
Metric: images/s (whole job, all ranks).  One JSON line on rank 0.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import warnings  # noqa: E402

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

warnings.filterwarnings('ignore', message='Full backward hook is firing')

EIGH_KERNEL_NOTE = '(see DESIGN.md 3)'
METRIC = 'images/sec ResNet-50 K-FAC training step (fwd+bwd+factor hooks+preconditioner.step()+SGD), factor=inv=1'


def metric_name(model):
    return METRIC if model == 'resnet50' else METRIC.replace('ResNet-50', 'ResNet-32')


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument('--gpus', type=int, default=1)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--impl', default='b200', choices=['b200', 'reference'])
    ap.add_argument('--model', default='resnet50', choices=['resnet50', 'resnet32'])
    ap.add_argument('--batch', type=int, default=0, help='per-GPU batch (default 32 / 128)')
    ap.add_argument('--grad-worker-fraction', type=float, default=-1.0)
    ap.add_argument('--no-cpu-baseline', action='store_true')
    ap.add_argument('--batches', type=int, default=8, help='distinct pre-generated batches cycled through (>= 8: every '
                    'step sees new statistics; 1 = the stationary-input number of round 1)')
    ap.add_argument('--no-parity', action='store_true', help='skip the untimed parity step after the timed region')
    ap.add_argument('--no-stationary', action='store_true', help='skip the extra stationary-input timing')
    ap.add_argument('--budget-s', type=float, default=240.0, help='reference arm wall-clock budget')
    ap.add_argument('--dump-outputs', default=None, metavar='DIR',
                    help='write what the last timed step computed (loss, a seeded sample of the preconditioned '
                         'gradients and of the updated parameters) as DIR/<name>.npy')
    return ap.parse_args()


def make_workload(name, batch):
    from workloads import resnet32, resnet50
    if name == 'resnet50':
        b = batch or 32
        return resnet50, (b, 3, 224, 224), 1000, dict(damping=0.001, factor_decay=0.95, kl_clip=0.001, lr=0.1), \
            f'ResNet-50 ImageNet-shape synthetic, bs{b}/GPU, factor_update_steps=1, inv_update_steps=1, damping 1e-3'
    b = batch or 128
    return resnet32, (b, 3, 32, 32), 10, dict(damping=0.003, factor_decay=0.95, kl_clip=0.001, lr=0.1), \
        f'ResNet-32 CIFAR-shape synthetic, bs{b}/GPU, factor_update_steps=1, inv_update_steps=1, damping 3e-3'


# ------------------------------------------------------------------ clocks
class ClockSampler(threading.Thread):
    """Samples SM clock + throttle reasons of one GPU during the timed region."""

    def __init__(self, index):
        super().__init__(daemon=True)
        self.index = index
        self.samples, self.reasons = [], set()
        self.max_mhz = None
        self._stop_evt = threading.Event()
        self.ok = False
        try:
            import pynvml
            pynvml.nvmlInit()
            self.nv = pynvml
            self.h = pynvml.nvmlDeviceGetHandleByIndex(index)
            self.max_mhz = pynvml.nvmlDeviceGetMaxClockInfo(self.h, pynvml.NVML_CLOCK_SM)
            self.ok = True
        except Exception:  # noqa: BLE001
            self.ok = False

    def run(self):
        if not self.ok:
            return
        nv = self.nv
        names = {
            getattr(nv, 'nvmlClocksThrottleReasonHwSlowdown', 0x8): 'hw_slowdown',
            getattr(nv, 'nvmlClocksThrottleReasonHwThermalSlowdown', 0x40): 'hw_thermal_slowdown',
            getattr(nv, 'nvmlClocksThrottleReasonSwThermalSlowdown', 0x20): 'sw_thermal_slowdown',
            getattr(nv, 'nvmlClocksThrottleReasonSwPowerCap', 0x4): 'sw_power_cap',
        }
        while not self._stop_evt.is_set():
            try:
                self.samples.append(nv.nvmlDeviceGetClockInfo(self.h, nv.NVML_CLOCK_SM))
                r = nv.nvmlDeviceGetCurrentClocksThrottleReasons(self.h)
                for bit, name in names.items():
                    if r & bit:
                        self.reasons.add(name)
            except Exception:  # noqa: BLE001
                pass
            time.sleep(0.1)

    def stop(self):
        self._stop_evt.set()
        if self.ok:
            self.join(timeout=2)
        s = sorted(self.samples)
        return {'sm_mhz': s[len(s) // 2] if s else None, 'sm_max_mhz': self.max_mhz,
                'reasons': sorted(self.reasons), 'samples': len(s)}


# ------------------------------------------------------------------ phases
class PhaseTimer:
    """CUDA-event timing of the native phases inside step() (current stream)."""

    def __init__(self, pre):
        self.pre = pre
        self.events = {}
        self.enabled = False
        for name in ('_flush_factor_updates', '_compute_inverses', '_precondition', '_scale_and_write_back'):
            self._wrap(pre, name)
        # C1 runs inside the flush (flush_factor_updates includes it); the A block is reduced under backward
        self._wrap(pre, '_reduce_batches', 'reduce_factors')
        for _, layer in pre._layers.values():
            self._wrap(layer.module, 'accumulate_a', 'factor_a')
            self._wrap(layer.module, 'accumulate_g', 'factor_g')

    def _wrap(self, obj, name, key=None):
        key = key or name.strip('_')
        fn = getattr(obj, name)

        def timed(*a, **k):
            if not self.enabled:
                return fn(*a, **k)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = fn(*a, **k)
            e1.record()
            self.events.setdefault(key, []).append((e0, e1))
            return out
        setattr(obj, name, timed)

    def totals_ms(self):
        return {k: sum(a.elapsed_time(b) for a, b in v) for k, v in self.events.items()}


def algorithmic_work(pre):
    """SURVEY.md 8(d) conventions: eigh 9n^3, precondition 4ga(g+a)."""
    eig = prec = 0.0
    for _, l in pre._layers.values():
        a, g = l.a_dim, l.g_dim
        eig += 9.0 * (a ** 3 + g ** 3)
        prec += 4.0 * g * a * (g + a)
    return eig, prec


def tc_gemm_microbench(lib, dev, n=4096, iters=10):
    """Isolated timing of the wgmma GEMM engine (the kernel under K3/K5/K8):
    D = A B^T, n^3 problem, fp32 operands (3 x 64 MB > 50 MB L2), CUDA events."""
    A = torch.randn(n, n, device=dev)
    B = torch.randn(n, n, device=dev)
    D = torch.empty(n, n, device=dev)
    s = torch.cuda.current_stream().cuda_stream

    def run():
        rc = lib.kfac_gemm_tn_tc(A.data_ptr(), n, B.data_ptr(), n, D.data_ptr(), n, n, n, n, 1.0, 0, 1, s)
        assert rc == 0, lib.kfac_last_error()
    for _ in range(3):
        run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        run()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    return 2.0 * n ** 3 / (ms / 1e3) / 1e12, ms


# ------------------------------------------------------------------ own arm
DUMP_SAMPLE = 1 << 22      # entries kept of each long output vector (16 MB as float32)


def snapshot_outputs(model, loss):
    """What a caller of the timed path holds after its last step: the loss, the preconditioned gradients and the
    parameters after the SGD update.  The two vectors (25.6 M entries each for ResNet-50) are sampled at DUMP_SAMPLE
    fixed positions drawn from a seeded generator, so that two runs can be compared entry for entry."""
    params = list(model.parameters())
    g = torch.cat([(p.grad if p.grad is not None else torch.zeros_like(p)).detach().reshape(-1) for p in params])
    w = torch.cat([p.detach().reshape(-1) for p in params])
    if g.numel() > DUMP_SAMPLE:
        idx = torch.randperm(g.numel(), generator=torch.Generator().manual_seed(1234))[:DUMP_SAMPLE].sort().values
        idx = idx.to(g.device)
        g, w = g[idx], w[idx]
    return {'loss': loss.detach().double().reshape(1).cpu(), 'precond_grads': g.float().cpu(), 'params': w.float().cpu()}


def write_outputs(outputs, out_dir):
    import numpy as np
    os.makedirs(out_dir, exist_ok=True)
    for name, t in outputs.items():
        np.save(os.path.join(out_dir, name + '.npy'), t.numpy())


def parity_step(pre, model, world, rank, dev, hp):
    """One UNTIMED step after the timed region, checked against the CPU oracle (test infrastructure used as
    the checker only; nothing here is timed or shipped).  ResNets hold BatchNorm, so the concatenated-batch
    equivalence of tests/dist_parity.py does not apply; instead:
      C1   the library's reduction of the batch-statistics arena must equal the mean over ranks of the local arenas;
      K5-K12 + C2 + C3   rank 0 recomputes, on the host with the oracle's operators, the preconditioned gradient
           of EVERY layer from the all-reduced factors and the DDP-averaged raw gradients, and compares it with
           the P this rank holds after step() (computed here or received from its KAISA source);
      all ranks must end the step with identical final gradients."""
    from oracle import kfac_oracle as O
    out = {}
    layers = [l for _, l in pre._layers.values()]
    raw = [O.grad_matrix(l.module.get_weight_grad().detach().float().cpu(),
                         l.module.get_bias_grad().detach().float().cpu() if l.module.has_bias() else None)
           for l in layers] if rank == 0 else None
    if world > 1:
        # the caller ran this step's forward/backward with pre.overlap_factor_allreduce = False: the batch statistics
        # are still local here
        local = pre._batch_arena.clone()
        dist.all_reduce(local)
        local /= world
        pre._reduce_batches()
        err = float((pre._batch_arena - local).norm() / local.norm())
        out['factor_allreduce_rel_err'] = err
        del local
    pre.step()
    torch.cuda.synchronize()
    if world > 1:
        worst = torch.zeros(1, device=dev)
        for p in model.parameters():
            ref = p.grad.clone()
            dist.broadcast(ref, src=0)
            worst = torch.maximum(worst, (p.grad - ref).norm() / ref.norm().clamp_min(1e-30))
        dist.all_reduce(worst, op=dist.ReduceOp.MAX)
        out['final_grad_rank_spread'] = float(worst.item())
    if rank == 0:
        torch.set_num_threads(usable_cores())
        damping = float(hp['damping'])
        worst, worst_layer, worst_gold = 0.0, None, None
        for l, g in zip(layers, raw):
            Af, Gf = l.a_factor.detach().float().cpu(), l.g_factor.detach().float().cpu()
            da, qa = O.eigen_decompose(Af)
            dg, qg = O.eigen_decompose(Gf)
            want = O.precondition_eigen(g, qa, qg, dgda=O.eigen_dgda(dg, da, damping)).double()
            got = l._p_view.detach().double().cpu()
            e = float((got - want).norm() / want.norm())
            if e > worst:
                worst, worst_layer = e, (l.a_dim, l.g_dim)
            if e > 3e-4:
                # how far is the fp32 oracle itself from exact arithmetic on this layer?  (fp64 restatement of the
                # same operator; a layer whose fp32 reference is ~1e-3 from fp64 cannot be matched more closely)
                da64, qa64 = torch.linalg.eigh(Af.double())
                dg64, qg64 = torch.linalg.eigh(Gf.double())
                gold = qg64 @ ((qg64.t() @ g.double() @ qa64) /
                               (torch.outer(dg64.clamp(min=0), da64.clamp(min=0)) + damping)) @ qa64.t()
                rec = {'dims_a_g': (l.a_dim, l.g_dim), 'b200_vs_oracle_fp32': e,
                       'b200_vs_fp64': float((got - gold).norm() / gold.norm()),
                       'oracle_fp32_vs_fp64': float((want - gold).norm() / gold.norm())}
                if worst_gold is None or e >= worst_gold['b200_vs_oracle_fp32']:
                    worst_gold = rec
        # bar: 1e-3 against the fp32 oracle; a layer on which the fp32 oracle ITSELF is further than that from exact
        # arithmetic (ill-conditioned factors of the synthetic random-label run) passes when this implementation is
        # no further from fp64 than 1.5 x the oracle's own distance (both are fp32 roundings of the same operator)
        ok = worst < 1e-3 or (worst_gold is not None and worst_gold['oracle_fp32_vs_fp64'] > 1e-3 and
                              worst_gold['b200_vs_fp64'] <= 1.5 * worst_gold['oracle_fp32_vs_fp64'])
        out.update({'worst_layer_P_rel_fro_vs_oracle': worst, 'worst_layer_dims_a_g': worst_layer,
                    'layers_checked': len(layers), 'bar': 1e-3, 'ok': bool(ok),
                    'ill_conditioned_layer_vs_fp64': worst_gold})
    return out


def run_b200(args):
    world = int(os.environ.get('WORLD_SIZE', '1'))
    rank = int(os.environ.get('RANK', '0'))
    local = int(os.environ.get('LOCAL_RANK', '0'))
    assert torch.cuda.is_available(), 'bench.py (own arm) needs a CUDA device'
    torch.cuda.set_device(local)
    dev = torch.device('cuda', local)
    if world > 1:
        dist.init_process_group('nccl', device_id=dev)
    from kfac_b200 import _cabi
    from kfac_b200.preconditioner import KFACPreconditioner
    lib = _cabi.load()

    make_model, shape, classes, hp, wl = make_workload(args.model, args.batch)
    torch.manual_seed(0)
    model = make_model().to(dev)
    if world > 1:
        model = torch.nn.parallel.DistributedDataParallel(model, device_ids=[local])
    frac = args.grad_worker_fraction
    if frac < 0:
        frac = 1.0 if world == 1 else 0.5
    pre = KFACPreconditioner(model, factor_update_steps=1, inv_update_steps=1, grad_worker_fraction=frac, **hp)
    opt = torch.optim.SGD(model.parameters(), lr=hp['lr'], momentum=0.9)
    crit = torch.nn.CrossEntropyLoss()
    timer = PhaseTimer(pre)

    # NB distinct pre-generated batches, cycled: every step sees new statistics (round 1 fed a single repeated batch,
    # which flattered its warm-started iterative eigensolver; the direct solver's cost does not depend on the data)
    torch.manual_seed(1 + rank)
    B = shape[0]
    NB = max(1, args.batches)
    host = [(torch.randn(*shape).pin_memory(), torch.randint(0, classes, (B,)).pin_memory()) for _ in range(NB)]
    devb = [(x.to(dev), y.to(dev)) for x, y in host]
    loss_host = torch.zeros(1).pin_memory()
    copy_stream = torch.cuda.Stream(device=dev)
    h2d_bytes = host[0][0].numel() * 4 + host[0][1].numel() * 8
    counter = {'i': 0}
    last = {}

    def stage(i):
        """Issue the H2D copy of batch i on the copy stream (double-buffered prefetch, like a data loader
        worker): returns (x, y, event)."""
        hx, hy = host[i % NB]
        with torch.cuda.stream(copy_stream):
            x = hx.to(dev, non_blocking=True)
            y = hy.to(dev, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(copy_stream)
        return x, y, ev

    def one_step(e2e, staged=None, prefetch=False, stationary=False):
        i = counter['i']
        counter['i'] += 1
        nxt = None
        if e2e:
            x, y, ev = staged if staged is not None else stage(i)
            torch.cuda.current_stream().wait_event(ev)
            x.record_stream(torch.cuda.current_stream())
            y.record_stream(torch.cuda.current_stream())
            if prefetch:
                nxt = stage(i + 1)        # overlaps with this step's compute
        else:
            x, y = devb[0] if stationary else devb[i % NB]
        opt.zero_grad(set_to_none=True)
        loss = crit(model(x), y)
        loss.backward()
        pre.step()
        opt.step()
        last['loss'] = loss
        if e2e:
            loss_host.copy_(loss.detach().reshape(1), non_blocking=True)
        return nxt

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def timed_loop(n, e2e, stationary=False):
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        l0 = lib.kfac_launch_count()
        e0.record()
        staged = None
        for k in range(n):
            # exactly n H2D copies inside the region: step k waits for its own batch and prefetches batch k+1
            staged = one_step(e2e, staged=staged, prefetch=(k + 1 < n), stationary=stationary)
        e1.record()
        barrier()
        ms = torch.tensor([e0.elapsed_time(e1)], device=dev)
        if world > 1:
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return float(ms.item()), lib.kfac_launch_count() - l0

    W = max(args.warmup, 3)
    for _ in range(W):
        one_step(False)
    barrier()
    sampler = ClockSampler(local)
    sampler.start()
    timer.enabled = True
    ms_dev, launches = timed_loop(args.steps, False)
    timer.enabled = False
    # outputs of the last timed step, taken before any later (extra) step changes the model
    outputs = snapshot_outputs(model, last['loss']) if args.dump_outputs and rank == 0 else None
    phase_ms = timer.totals_ms()
    ms_e2e, _ = timed_loop(args.steps, True)
    clocks = sampler.stop()
    # extra keys (not the headline): the stationary-input number of round 1 (same batch every step) and the raw
    # host->device bandwidth of this box (explains value vs e2e when the PCIe path is slow)
    ms_stat = None
    if not args.no_stationary:
        for _ in range(2):
            one_step(False, stationary=True)
        ms_stat, _ = timed_loop(max(3, args.steps // 2), False, stationary=True)
        ms_stat /= max(3, args.steps // 2)
    # second configuration: the reference's default ImageNet schedule (factor_update_steps 10, inv_update_steps 100,
    # examples/torch_imagenet_resnet.py:158-198): 20 steps without an eigendecomposition, 2 of them with factor updates
    sched = None
    if not args.no_stationary:
        fu, iu, st = pre._factor_update_steps, pre._inv_update_steps, pre._steps
        pre._factor_update_steps, pre._inv_update_steps, pre._steps = 10, 100, 1
        for _ in range(2):
            one_step(False)
        pre._steps = 1
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        l0 = lib.kfac_launch_count()
        t_step = []
        e0.record()
        for k in range(20):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            opt.zero_grad(set_to_none=True)
            x, y = devb[k % NB]
            crit(model(x), y).backward()
            a.record()
            pre.step()
            b.record()
            opt.step()
            t_step.append((a, b))
        e1.record()
        barrier()
        ms20 = torch.tensor([e0.elapsed_time(e1)], device=dev)
        if world > 1:
            dist.all_reduce(ms20, op=dist.ReduceOp.MAX)
        plain = sorted(a.elapsed_time(b) for a, b in t_step)
        sched = {'factor_update_steps': 10, 'inv_update_steps': 100, 'steps': 20, 'ms_per_step': float(ms20.item()) / 20,
                 'value': B * world * 20 / (float(ms20.item()) / 1e3), 'unit': 'images/s',
                 'kfac_step_ms_median': plain[len(plain) // 2], 'kfac_step_ms_max': plain[-1],
                 'gpu_launches_per_step': (lib.kfac_launch_count() - l0) / 20.0,
                 'note': 'steps 1..20 of the schedule: no eigendecomposition, factor statistics at steps 10 and 20; '
                         'kfac_step_ms = preconditioner.step() alone (precondition + kl-clip + write-back)'}
        pre._factor_update_steps, pre._inv_update_steps, pre._steps = fu, iu, st
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(4):
        host[0][0].to(dev, non_blocking=True)
    torch.cuda.synchronize()
    h2d_gbs = 4 * host[0][0].numel() * 4 / (time.perf_counter() - t0) / 1e9

    K = args.steps
    imgs = B * world * K
    value = imgs / (ms_dev / 1e3)
    e2e_value = imgs / (ms_e2e / 1e3)
    eig_flops, prec_flops = algorithmic_work(pre)
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(ROOT, 'MEASURED_PEAKS.json')))
    except Exception:  # noqa: BLE001
        pass
    # without a measured peak of this card: the H100 SXM data sheet (dense BF16, 700 W); the card may be set lower
    tensor_peak = float(peaks.get('bf16_tflops_sustained', 989.0))
    peak_src = 'measured (MEASURED_PEAKS.json bf16_tflops_sustained)' if peaks else 'H100 SXM data sheet, dense bf16'
    # dominant phase: the batched eigensolver; at N>1 each rank solves only its
    # KAISA share, the roofline line is reported for rank 0's local phase time.
    inv_ms = phase_ms.get('compute_inverses', 0.0) / K
    my_eig = 0.0
    my_bytes = 0.0
    r = rank
    for name, l in pre._layers.values():
        if pre._assignment.inv_worker(name, 'A') == r:
            my_eig += 9.0 * l.a_dim ** 3
            my_bytes += 12.0 * l.a_dim ** 2
        if pre._assignment.inv_worker(name, 'G') == r:
            my_eig += 9.0 * l.g_dim ** 3
            my_bytes += 12.0 * l.g_dim ** 2
    achieved = (my_eig / (inv_ms / 1e3) / 1e12) if inv_ms > 0 else 0.0
    gemm_tf, gemm_ms = tc_gemm_microbench(lib, dev) if rank == 0 else (0.0, 0.0)
    burst_peak = float(peaks.get('bf16_tflops', 989.0))
    out = {
        'metric': metric_name(args.model), 'value': value, 'unit': 'images/s', 'n_gpus': world, 'steps': K,
        'warmup': W, 'ms_per_step': ms_dev / K, 'higher_is_better': True,
        'scaling': 'weak', 'vs_baseline': None, 'dtype': 'f32 (model fwd/bwd fp32; K-FAC path fp32)',
        'data': 'synthetic',
        'config': {'workload': wl, 'global_batch': B * world, 'grad_worker_fraction': frac,
                   'parallelism': f'dp{world}', 'distinct_batches': NB,
                   'l2': 'inputs+factors >> 50 MB L2 (activations 1.4 GB, factors 615 MB)'},
        'clocks': clocks,
        'e2e': {'value': e2e_value, 'unit': 'images/s', 'ms_per_step': ms_e2e / K,
                'h2d_bytes_per_step': h2d_bytes, 'd2h_bytes_per_step': 4,
                'how': 'pinned-host batch -> device every step on a copy stream (batch k+1 prefetched under the compute '
                       'of step k, every copy inside the timed region), loss read back to pinned host memory',
                'h2d_gb_per_s_this_box': h2d_gbs},
        'gpu_launches': int(launches),
        'kfac_phase_ms_per_step': {k: v / K for k, v in sorted(phase_ms.items())},
        # preconditioner.step() itself (BASELINE.json: "K-FAC step() ms"): the phases step() runs, without the
        # factor hooks that run inside forward/backward
        'kfac_step_ms': sum(v for k, v in phase_ms.items() if k not in ('factor_a', 'factor_g')) / K,
        'kfac_hooks_ms': sum(v for k, v in phase_ms.items() if k in ('factor_a', 'factor_g')) / K,
        'default_schedule': sched,
        'stationary_input': ({'ms_per_step': ms_stat, 'value': B * world / (ms_stat / 1e3),
                              'note': 'same batch every step (round-1 protocol); not the headline'}
                             if ms_stat else None),
        # dominant launch of the step: ONE kfac_eigh_batched call (all factors this rank owns), timed
        # live in the timed region with CUDA events on the launching stream
        'roofline': {'kernel': 'kfac_eigh_batched: one call per step over all factors of this rank '
                               + EIGH_KERNEL_NOTE,
                     'bound': 'tensor', 'achieved': achieved, 'peak': tensor_peak, 'unit': 'TFLOP/s',
                     'frac': achieved / tensor_peak if tensor_peak else None, 'traffic': None,
                     'algorithmic_bytes': my_bytes,
                     'ms_per_launch': inv_ms,
                     'convention': 'algorithmic 9 n^3 flop per eigendecomposition (SURVEY.md 8d) summed over the '
                                   "rank's factors / CUDA-event time of the call; algorithmic bytes 3*4*n^2 per factor",
                     'peak_source': peak_src},
        # the GEMM engine all tensor-core kernels instantiate, timed alone on a 4096^3 problem
        'roofline_engine': {'kernel': 'tc::pipeline_kernel<GemmPolicy> (wgmma 3xTF32 GEMM engine), 4096^3, isolated',
                            'bound': 'tensor', 'achieved': gemm_tf, 'peak': burst_peak, 'unit': 'TFLOP/s',
                            'frac': gemm_tf / burst_peak if burst_peak else None, 'traffic': None,
                            'ms_per_launch': gemm_ms,
                            'convention': 'algorithmic fp32 flops 2*M*N*K per launch / CUDA-event time; every product is '
                                          'issued as 3 TF32 MMAs, so the tensor pipe executes 3x these flops at the TF32 '
                                          'rate (= half the bf16 rate the peak was measured with)',
                            'peak_source': 'measured (MEASURED_PEAKS.json bf16_tflops, burst)' if peaks else
                                           'H100 SXM data sheet, dense bf16'},
        'algorithmic_flops_per_step': {'eigh_9n3': eig_flops, 'precondition_4ga(g+a)': prec_flops},
    }
    if not args.no_parity:
        # one more (untimed) step on a fresh batch, checked against the CPU oracle
        x, y = devb[counter['i'] % NB]
        opt.zero_grad(set_to_none=True)
        pre.overlap_factor_allreduce = False      # keep this step's statistics local until parity_step has cloned them
        crit(model(x), y).backward()
        out['parity'] = parity_step(pre, model, world, rank, dev, hp)
        pre.overlap_factor_allreduce = True
    if rank == 0 and world == 1 and not args.no_cpu_baseline:
        out['cpu_baseline'] = cpu_baseline(args, steps=2, warmup=1, budget=150.0)
    if outputs is not None:
        write_outputs(outputs, args.dump_outputs)
    if rank == 0:
        print(json.dumps(out))
    if world > 1:
        dist.destroy_process_group()


# ------------------------------------------------------------------ CPU arm
def usable_cores():
    """Host threads this process may really use: CPU affinity capped by the cgroup quota (a
    container that sees 128 logical CPUs but owns a fraction of them would otherwise
    oversubscribe MKL/OpenMP catastrophically) and by 32 (LAPACK eigh does not scale further)."""
    try:
        n = len(os.sched_getaffinity(0))
    except Exception:  # noqa: BLE001
        n = os.cpu_count() or 1
    try:
        q, p = open('/sys/fs/cgroup/cpu.max').read().split()[:2]
        if q != 'max':
            n = min(n, max(1, int(float(q) / float(p))))
    except Exception:  # noqa: BLE001
        try:
            q = int(open('/sys/fs/cgroup/cpu/cpu.cfs_quota_us').read())
            p = int(open('/sys/fs/cgroup/cpu/cpu.cfs_period_us').read())
            if q > 0:
                n = min(n, max(1, q // p))
        except Exception:  # noqa: BLE001
            pass
    env = os.environ.get('KFAC_BENCH_CPU_THREADS')
    if env:
        return max(1, int(env))
    return max(1, min(n, 32))


REF_DIR = os.path.join(ROOT, 'oracle', '_ref')


def reference_kind():
    """'reference' when the unmodified reference package was installed into oracle/_ref by
    oracle/build_ref.sh, else 'port' (the oracle)."""
    return 'reference' if os.path.isdir(os.path.join(REF_DIR, 'kfac')) else 'port'


def cpu_reference_loop(args, steps, warmup, budget):
    """The reference's own CPU implementation of the path on the host cores: the UNMODIFIED
    kfac.preconditioner.KFACPreconditioner from oracle/_ref (kind 'reference'), or -- when that install is
    absent -- the oracle port (same torch CPU ops).  World size 1 (kfac/distributed.py:221-222)."""
    make_model, shape, classes, hp, wl = make_workload(args.model, args.batch)
    cores = usable_cores()
    torch.set_num_threads(cores)
    torch.manual_seed(0)
    model = make_model()
    kind = reference_kind()
    if kind == 'reference':
        if REF_DIR not in sys.path:
            sys.path.insert(0, REF_DIR)
        warnings.filterwarnings('ignore', message='NVIDIA Apex')
        import logging
        from kfac.preconditioner import KFACPreconditioner as RefPreconditioner
        pre = RefPreconditioner(model, factor_update_steps=1, inv_update_steps=1, loglevel=logging.DEBUG, **hp)
    else:
        from oracle.kfac_oracle import OraclePreconditioner
        pre = OraclePreconditioner(model, factor_update_steps=1, inv_update_steps=1, **hp)
    opt = torch.optim.SGD(model.parameters(), lr=hp['lr'], momentum=0.9)
    crit = torch.nn.CrossEntropyLoss()
    NB = max(1, args.batches)
    torch.manual_seed(1)
    data = [(torch.randn(*shape), torch.randint(0, classes, (shape[0],))) for _ in range(NB)]

    def one(i):
        x, y = data[i % NB]
        opt.zero_grad(set_to_none=True)
        crit(model(x), y).backward()
        t0 = time.perf_counter()
        pre.step()
        t1 = time.perf_counter()
        opt.step()
        return t1 - t0
    # every step is checked against the wall-clock budget; if not even the warm-up fits, the
    # last completed step is the sample
    t_start = time.perf_counter()
    walls, kfacs = [], []
    for i in range(warmup + steps):
        t0 = time.perf_counter()
        k = one(i)
        walls.append(time.perf_counter() - t0)
        kfacs.append(k)
        if time.perf_counter() - t_start + walls[-1] > budget:
            break
    warm_done = min(warmup, max(0, len(walls) - 1))
    walls, kfacs = walls[warm_done:], kfacs[warm_done:]
    done, total, step_s = len(walls), sum(walls), sum(kfacs)
    return {'images_per_s': shape[0] * done / total, 'ms_per_step': total / done * 1e3,
            'kfac_step_ms': step_s / done * 1e3, 'steps_done': done, 'warmup_done': warm_done, 'cores': cores,
            'workload': wl, 'batch': int(shape[0]), 'kind': kind, 'distinct_batches': NB}


def cpu_baseline(args, steps, warmup, budget):
    """Runs the CPU arm in a child process under a hard wall-clock limit so that the default
    bench run always ends within minutes, whatever the host does."""
    import subprocess
    cmd = [sys.executable, os.path.abspath(__file__), '--impl', 'reference', '--model', args.model,
           '--steps', str(steps), '--warmup', str(warmup), '--budget-s', str(budget), '--batches', str(args.batches)]
    if args.batch:
        cmd += ['--batch', str(args.batch)]
    env = dict(os.environ)
    for k in ('RANK', 'WORLD_SIZE', 'LOCAL_RANK', 'OMP_NUM_THREADS'):
        env.pop(k, None)
    try:
        out = subprocess.run(cmd, capture_output=True, text=True, timeout=budget + 90, env=env)
        line = [l for l in out.stdout.splitlines() if l.startswith('{')][-1]
        d = json.loads(line)
        cb = d['cpu_baseline']
        cb['kfac_step_ms'] = d.get('kfac_step_ms')
        cb['ms_per_step'] = d.get('ms_per_step')
        return cb
    except Exception as e:  # noqa: BLE001
        return {'value': None, 'unit': 'images/s', 'cores': usable_cores(), 'kind': reference_kind(),
                'sample': f'CPU arm did not finish one step within {budget + 90:.0f} s ({type(e).__name__})'}


def run_reference(args):
    """`--impl reference`: under torchrun only rank 0 works (the reference's single-process CPU path); the line
    reports n_gpus = 1 and a world_size-1 global batch so that no N-GPU / 1-process ratio is formed from it."""
    rank = int(os.environ.get('RANK', '0'))
    if rank != 0:
        return
    W = max(args.warmup, 1)
    r = cpu_reference_loop(args, args.steps, W, args.budget_s)
    kind = r['kind']
    what = ('unmodified kfac.preconditioner.KFACPreconditioner (gpauloski/kfac-pytorch v0.4.2 installed into oracle/_ref)'
            if kind == 'reference' else "oracle port (the reference's torch CPU ops)")
    out = {
        'impl': 'reference', 'metric': metric_name(args.model), 'value': r['images_per_s'], 'unit': 'images/s',
        'n_gpus': 1, 'requested_gpus': args.gpus, 'steps': r['steps_done'], 'warmup': r['warmup_done'],
        'ms_per_step': r['ms_per_step'], 'higher_is_better': True, 'scaling': 'weak', 'vs_baseline': None,
        'dtype': 'f32 (model fwd/bwd fp32; K-FAC path fp32)', 'data': 'synthetic',
        'config': {'workload': r['workload'], 'global_batch': r['batch'], 'grad_worker_fraction': 1.0,
                   'parallelism': 'cpu, world_size 1 (one process on the host cores, at every requested N)',
                   'distinct_batches': r['distinct_batches'], 'l2': 'n/a (host)'},
        'cpu_baseline': {'value': r['images_per_s'], 'unit': 'images/s', 'cores': r['cores'], 'kind': kind,
                         'sample': f"{r['steps_done']} of {args.steps} requested full steps (after {r['warmup_done']} warm-up) "
                                   f"within a {args.budget_s:.0f} s budget, {what}; kfac step() {r['kfac_step_ms']:.0f} ms"},
        'e2e': {'value': r['images_per_s'], 'unit': 'images/s', 'h2d_bytes_per_step': 0, 'd2h_bytes_per_step': 0},
        'kfac_step_ms': r['kfac_step_ms'],
    }
    print(json.dumps(out))


if __name__ == '__main__':
    a = parse()
    if a.impl == 'reference':
        run_reference(a)
    else:
        run_b200(a)
