"""Timeline of one ResNet-50 kfac_eigh_batched call with its schedule run as waves, against one wave.

  python tests/eigh_waves_timeline.py [--rounds R] [--json OUT] [--trace OUT]

Prints the call time (CUDA events, both settings alternating), the %globaltimer stamps of every tridiagonalisation job
with its wave, and from a torch.profiler run of its own the span of each wave's cooperative launch and of the
later-stage kernels on each stream.  The inputs are the seeded K-FAC-like factors of the eigh_r50 case of
gen_engine_bits.py; the outputs of both settings are compared bit for bit."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from gen_engine_bits import R50, _kfac_like  # noqa: E402
from kfac_b200 import _cabi  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=6)
    ap.add_argument('--json', default=None)
    ap.add_argument('--trace', default=None, help='write the chrome trace of the profiled waves call here')
    args = ap.parse_args()
    lib = _cabi.load()
    v = C.c_void_p
    lib.kfac_stage_schedule.argtypes = [v, C.c_int, C.c_int, v, v, v]
    lib.kfac_stage_waves.argtypes = [v, C.c_int, C.c_int, v, v, v]
    lib.kfac_stage_eigh_max_waves.argtypes = [C.c_int]
    lib.kfac_stage_sytrd_profile.argtypes = [C.c_int, v]
    lib.kfac_stage_sytrd_job_times.argtypes = [v, C.c_int]
    dev = torch.device('cuda:0')
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                          capture_output=True, text=True).stdout.strip()
    print('card:', card)

    gen = torch.Generator().manual_seed(0)
    dims = [d for a, g, c in R50 for d in [a, g] * c]
    mats = [_kfac_like(gen, n) for n in dims]
    items = (_cabi.EighItem * len(dims))()
    outs = []
    for i, (n, F) in enumerate(zip(dims, mats)):
        ld = _cabi.ld4(n)
        Q, QT, d = torch.zeros(n, ld, device=dev), torch.zeros(n, ld, device=dev), torch.zeros(n, device=dev)
        outs.append((Q, QT, d))
        items[i] = _cabi.EighItem(F.data_ptr(), Q.data_ptr(), QT.data_ptr(), d.data_ptr(), n, ld, None)
    ns = (C.c_int * len(dims))(*dims)
    ws = {}
    for w in (1, -1):
        lib.kfac_stage_eigh_max_waves(w)
        need = lib.kfac_eigh_workspace_bytes(ns, len(dims))
        ws[w] = (torch.empty(need, dtype=torch.uint8, device=dev), need)
    lib.kfac_stage_eigh_max_waves(-1)
    stream = torch.cuda.current_stream().cuda_stream

    def call(w):
        lib.kfac_stage_eigh_max_waves(w)
        buf, need = ws[w]
        rc = lib.kfac_eigh_batched(items, len(dims), buf.data_ptr(), need, 0, 0.0, stream)
        lib.kfac_stage_eigh_max_waves(-1)
        assert rc == 0, lib.kfac_last_error()

    def snapshot():
        torch.cuda.synchronize()
        return [t.clone() for o in outs for t in o]

    res = {'card': card}
    call(1)
    ref = snapshot()
    call(-1)
    same = all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(snapshot(), ref))
    print('waves vs one wave: bitwise identical =', same)
    res['bitwise_identical'] = same

    times = {1: [], -1: []}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for r in range(args.rounds):
        for w in ((1, -1) if r % 2 == 0 else (-1, 1)):
            torch.cuda.synchronize()
            e0.record()
            call(w)
            e1.record()
            torch.cuda.synchronize()
            times[w].append(e0.elapsed_time(e1))
    for w, name in ((1, 'one wave'), (-1, 'waves')):
        ts = sorted(times[w])
        print(f'call ms, {name:9s}: min {ts[0]:7.2f}  median {ts[len(ts) // 2]:7.2f}  max {ts[-1]:7.2f}')
    res['call_ms'] = {'one_wave': times[1], 'waves': times[-1]}

    # job stamps
    big = [n for n in dims if n > 128]
    cnt = len(big)
    nb = (C.c_int * cnt)(*big)
    grid = torch.cuda.get_device_properties(0).multi_processor_count
    mat, cta0, ncta = (C.c_int * cnt)(), (C.c_int * cnt)(), (C.c_int * cnt)()
    k = lib.kfac_stage_schedule(nb, cnt, grid, mat, cta0, ncta)
    wave, wc, wp = (C.c_int * cnt)(), (C.c_int * cnt)(), (C.c_int * cnt)()
    nw = lib.kfac_stage_waves(nb, cnt, grid, wave, wc, wp)
    lib.kfac_stage_sytrd_profile(1, None)
    call(-1)
    torch.cuda.synchronize()
    raw = (C.c_ulonglong * (2 * k))()
    lib.kfac_stage_sytrd_job_times(raw, k)
    lib.kfac_stage_sytrd_profile(0, (C.c_ulonglong * 16)())
    base = min(raw[2 * j] for j in range(k))
    rows = [{'job': j, 'n': big[mat[j]], 'ncta': ncta[j], 'cta0': cta0[j], 'wave': wave[j],
             'start_ms': (raw[2 * j] - base) / 1e6, 'end_ms': (raw[2 * j + 1] - base) / 1e6} for j in range(k)]
    print(f'\n{nw} waves; tridiagonalisation jobs (ms from the first job start)')
    for w in range(nw):
        rw = [r for r in rows if r['wave'] == w]
        sizes = sorted({r['n'] for r in rw})
        nc = len({c for r in rw for c in range(r['cta0'], r['cta0'] + r['ncta'])})
        print(f' wave {w}: {len(rw):3d} jobs on {nc:3d} CTAs, '
              f'first start {min(r["start_ms"] for r in rw):7.2f}, last end {max(r["end_ms"] for r in rw):7.2f}, n {sizes}')
    res['jobs'] = rows

    # kernel spans per stream from a profiled call of its own
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call(-1)
        torch.cuda.synchronize()
    path = args.trace or os.path.join(tempfile.mkdtemp(), 'eigh_waves_trace.json')
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    prof.export_chrome_trace(path)
    with open(path) as f:
        ev = [e for e in json.load(f)['traceEvents'] if e.get('cat') == 'kernel']
    t0 = min(e['ts'] for e in ev)
    spans = {}
    for e in ev:
        st = e['args'].get('stream')
        kind = 'sytrd_kernel' if 'sytrd_kernel' in e['name'] else 'later stages'
        s = spans.setdefault((st, kind), [1e30, 0.0, 0])
        s[0] = min(s[0], (e['ts'] - t0) / 1e3)
        s[1] = max(s[1], (e['ts'] + e['dur'] - t0) / 1e3)
        s[2] += 1
    print('\nkernel spans per stream (ms from the first kernel; torch.profiler)')
    for (st, kind), (a, b, c) in sorted(spans.items(), key=lambda kv: kv[1][0]):
        print(f' stream {st:>4} {kind:13s} {a:8.2f} .. {b:8.2f}  ({c} kernels)')
    res['spans'] = [{'stream': st, 'kind': kind, 'start_ms': a, 'end_ms': b, 'kernels': c}
                    for (st, kind), (a, b, c) in spans.items()]
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
