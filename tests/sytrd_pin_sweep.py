"""Diagnostic (not a pytest): L2 residency sweep of the batched tridiagonalisation.  Needs one H100.

One kfac_eigh_batched call over the ResNet-50 factor dimensions (the inputs of the `eigh_r50` case of
tests/gen_engine_bits.py) is timed with CUDA events at several residency budgets, alternating the budgets round by
round; sytrd_kernel alone is timed with torch.profiler in a run of its own.  Every budget must give the same output
bits.  Also prints the bytes model of phase A (tile bytes read per call, those a pinned tile serves, implied HBM
rate) and the per-job timeline of the kernel (%globaltimer on each job's first CTA) against the schedule's time model.

    python tests/sytrd_pin_sweep.py [--rounds 5] [--budgets 0,16,24,32,40] [--timeline 0,32] [--json OUT]

Budgets are in MiB; the budget is set through a test-only entry of the library (kfac_stage_sytrd_pin_budget).
"""
from __future__ import annotations

import argparse
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

from kfac_b200 import _cabi  # noqa: E402
from gen_engine_bits import R50, _kfac_like  # noqa: E402

TILE = 64
TILE_BYTES = TILE * TILE * 4


def load_lib():
    lib = _cabi.load()
    lib.kfac_stage_pin_plan.restype = C.c_int
    lib.kfac_stage_pin_plan.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_longlong, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.kfac_stage_schedule.restype = C.c_int
    lib.kfac_stage_schedule.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.kfac_stage_sytrd_pin_budget.restype = None
    lib.kfac_stage_sytrd_pin_budget.argtypes = [C.c_longlong]
    lib.kfac_stage_sytrd_profile.restype = C.c_int
    lib.kfac_stage_sytrd_profile.argtypes = [C.c_int, C.c_void_p]
    lib.kfac_stage_sytrd_job_times.restype = C.c_int
    lib.kfac_stage_sytrd_job_times.argtypes = [C.c_void_p, C.c_int]
    return lib


def pin_plan(lib, dims, grid, budget_bytes):
    """Per matrix: first pinned block column, predicted start and end (s) of its job."""
    cnt = len(dims)
    n = (C.c_int * cnt)(*dims)
    pin, t0, t1 = (C.c_int * cnt)(), (C.c_double * cnt)(), (C.c_double * cnt)()
    assert lib.kfac_stage_pin_plan(n, cnt, grid, budget_bytes, pin, t0, t1) == cnt
    return list(pin), list(t0), list(t1)


def schedule(lib, dims, grid):
    cnt = len(dims)
    n = (C.c_int * cnt)(*dims)
    mat, cta0, ncta = ((C.c_int * cnt)() for _ in range(3))
    jobs = lib.kfac_stage_schedule(n, cnt, grid, mat, cta0, ncta)
    return [(mat[j], cta0[j], ncta[j]) for j in range(jobs)]


def phase_a_bytes(dims, pin):
    """Lower-tile bytes phase A reads over the call (with tile padding), and those that pinned tiles serve."""
    total = served = 0
    for n, j0 in zip(dims, pin):
        nblk = (n + TILE - 1) // TILE
        for s in range(n - 1):
            b0 = (s + 1) // TILE
            total += (nblk - b0) * (nblk - b0 + 1) // 2
            j = max(b0, j0)
            served += (nblk - j) * (nblk - j + 1) // 2
    return total * TILE_BYTES, served * TILE_BYTES


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        out = torch.cuda.get_device_name(0) + ', power limit unknown'
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--budgets', default='0,16,24,32,40')
    ap.add_argument('--timeline', default='0,32', help='budgets (MiB) whose per-job timeline is printed')
    ap.add_argument('--json', default=None)
    args = ap.parse_args()
    budgets = [int(b) for b in args.budgets.split(',')]
    tl_budgets = [int(b) for b in args.timeline.split(',') if b != '']

    assert torch.cuda.is_available(), 'the sweep needs a CUDA device'
    dev = torch.device('cuda:0')
    lib = load_lib()
    grid = torch.cuda.get_device_properties(0).multi_processor_count
    res = {'card': card(), 'grid': grid, 'budgets_mib': budgets}
    print('card:', res['card'], '| SMs:', grid, flush=True)

    dims = [d for a, g, c in R50 for d in [a, g] * c]
    big = [d for d in dims if d > 128]                  # the direct solver's matrices, in call order
    gen = torch.Generator().manual_seed(0)
    items = (_cabi.EighItem * len(dims))()
    keep, outs = [], []
    for i, n in enumerate(dims):
        F = _kfac_like(gen, n)
        ld = _cabi.ld4(n)
        Q, QT, d = torch.zeros(n, ld, device=dev), torch.zeros(n, ld, device=dev), torch.zeros(n, device=dev)
        keep.append(F)
        outs.extend([Q, QT, d])
        items[i] = _cabi.EighItem(F.data_ptr(), Q.data_ptr(), QT.data_ptr(), d.data_ptr(), n, ld, None)
    ns = (C.c_int * len(dims))(*dims)
    need = lib.kfac_eigh_workspace_bytes(ns, len(dims))
    ws = torch.empty(need, dtype=torch.uint8, device=dev)
    stream = torch.cuda.current_stream().cuda_stream

    def call(mib):
        lib.kfac_stage_sytrd_pin_budget(mib << 20)
        rc = lib.kfac_eigh_batched(items, len(dims), ws.data_ptr(), need, 0, 0.0, stream)
        assert rc == 0, lib.kfac_last_error()

    def digest():
        torch.cuda.synchronize()
        h = hashlib.sha256()
        for t in outs:
            h.update(t.detach().float().contiguous().cpu().numpy().tobytes())
        return h.hexdigest()

    # bytes model and plan per budget
    res['model'] = {}
    for b in budgets:
        pin, t0, t1 = pin_plan(lib, big, grid, b << 20)
        total, served = phase_a_bytes(big, pin)
        pinned = [(n, (n + TILE - 1) // TILE - j) for n, j in zip(big, pin) if j < (n + TILE - 1) // TILE]
        res['model'][b] = {'phase_a_bytes': total, 'pinned_served_bytes': served, 'pinned': pinned,
                           'predicted_makespan_ms': 1e3 * max(t1)}
        print(f'budget {b:3d} MiB: phase-A tile bytes {total / 1e9:.1f} GB, served by pinned tiles {served / 1e9:.1f} GB '
              f'({100.0 * served / total:.1f} %); pinned (n, block columns): {pinned}', flush=True)

    # warm-up and output bits per budget
    res['digest'] = {}
    for b in budgets:
        call(b)
        res['digest'][b] = digest()
    same = len(set(res['digest'].values())) == 1
    print('output bits identical across budgets:', same, flush=True)
    res['bits_identical'] = same

    # call time, budgets alternating (order reversed every other round)
    times = {b: [] for b in budgets}
    for r in range(args.rounds):
        for b in (budgets if r % 2 == 0 else budgets[::-1]):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            call(b)
            e1.record()
            torch.cuda.synchronize()
            times[b].append(e0.elapsed_time(e1))
    res['call_ms'] = times

    # sytrd_kernel alone (device time from the profiler, a run of its own)
    kern = {b: [] for b in budgets}
    from torch.profiler import ProfilerActivity, profile
    for r in range(2):
        for b in (budgets if r % 2 == 0 else budgets[::-1]):
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                call(b)
                torch.cuda.synchronize()
            for ev in prof.events():
                if 'sytrd_kernel' in ev.name:
                    kern[b].append(ev.device_time_total / 1e3)
    res['sytrd_ms'] = kern

    print(f'\n{"budget MiB":>10} {"call ms (min / median / max)":>32} {"sytrd_kernel ms":>16} {"HBM GB/s implied":>17}')
    for b in budgets:
        ts = sorted(times[b])
        k = min(kern[b]) if kern[b] else float('nan')
        m = res['model'][b]
        hbm = (m['phase_a_bytes'] - m['pinned_served_bytes']) / (k * 1e-3) / 1e9 if kern[b] else float('nan')
        res['model'][b]['implied_hbm_gbs'] = hbm
        print(f'{b:>10} {ts[0]:10.2f} / {ts[len(ts) // 2]:7.2f} / {ts[-1]:7.2f} {k:16.2f} {hbm:17.0f}')

    # per-job timeline (first CTA of each job), against the schedule's time model
    jobs = schedule(lib, big, grid)
    res['timeline'] = {}
    for b in tl_budgets:
        pin, t0, t1 = pin_plan(lib, big, grid, b << 20)
        lib.kfac_stage_sytrd_profile(1, None)
        call(b)
        torch.cuda.synchronize()
        raw = (C.c_ulonglong * (2 * len(jobs)))()
        lib.kfac_stage_sytrd_job_times(raw, len(jobs))
        lib.kfac_stage_sytrd_profile(0, (C.c_ulonglong * 16)())
        base = min(raw[2 * j] for j in range(len(jobs)))
        rows = []
        print(f'\ntimeline at budget {b} MiB (ms from the first job start; predicted by the time model)')
        print(f'{"job":>4} {"n":>5} {"C":>3} {"cta0":>4} {"pinned":>6} {"start":>8} {"end":>8} {"pred start":>10} {"pred end":>9}')
        for j, (mi, c0, nc) in enumerate(jobs):
            n = big[mi]
            st, en = (raw[2 * j] - base) / 1e6, (raw[2 * j + 1] - base) / 1e6
            pinned = (n + TILE - 1) // TILE - pin[mi]
            rows.append({'job': j, 'n': n, 'ncta': nc, 'cta0': c0, 'pinned_cols': pinned, 'start_ms': st, 'end_ms': en,
                         'pred_start_ms': 1e3 * t0[mi], 'pred_end_ms': 1e3 * t1[mi]})
            print(f'{j:>4} {n:>5} {nc:>3} {c0:>4} {pinned:>6} {st:8.2f} {en:8.2f} {1e3 * t0[mi]:10.2f} {1e3 * t1[mi]:9.2f}')
        print(f'makespan {max(r["end_ms"] for r in rows):.2f} ms (model {1e3 * max(t1):.2f} ms)')
        res['timeline'][b] = rows
    lib.kfac_stage_sytrd_pin_budget(-1)

    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, 'w') as f:
            json.dump(res, f, indent=1)
        print('wrote', args.json)


if __name__ == '__main__':
    main()
