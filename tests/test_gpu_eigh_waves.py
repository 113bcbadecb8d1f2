"""kfac_eigh_batched gives the same bits whether its schedule runs as several waves (a cooperative launch and the later
stages of its matrices per wave, each on its own stream) or as one wave on the caller's stream, and a non-finite factor
that is alone in its wave is still reported in the status word."""
import ctypes as C

import pytest
import torch

from test_eigh_waves_host import R50

pytestmark = pytest.mark.gpu

R50_ALL = [d for a, g, c in R50 for d in [a, g] * c]
CASES = {
    'r50': R50_ALL,
    'mixed': [8192, 4608, 2304, 2304, 1024, 1000, 512, 300, 130, 64],
    'lone': [2304],
    'many_small': [300] * 60 + [200] * 30 + [100] * 10,
}


@pytest.fixture(scope='module')
def lib():
    from kfac_b200 import _cabi
    lib = _cabi.load()
    i = C.c_void_p
    lib.kfac_stage_schedule.restype = C.c_int
    lib.kfac_stage_schedule.argtypes = [i, C.c_int, C.c_int, i, i, i]
    lib.kfac_stage_waves.restype = C.c_int
    lib.kfac_stage_waves.argtypes = [i, C.c_int, C.c_int, i, i, i]
    lib.kfac_stage_eigh_max_waves.restype = None
    lib.kfac_stage_eigh_max_waves.argtypes = [C.c_int]
    yield lib
    lib.kfac_stage_eigh_max_waves(-1)


def S():
    return torch.cuda.current_stream().cuda_stream


def kfac_like(gen, n):
    m = max(8, n // 3)
    x = torch.relu(torch.randn(m, n, generator=gen) + 0.3) * torch.logspace(0, -2, n)
    x = x.to('cuda:0', torch.float64)
    F = 0.5 * torch.eye(n, device='cuda:0', dtype=torch.float64) + 0.5 * (x.t() @ x) / m
    return ((F + F.t()) / 2).float().contiguous()


def waves(lib, dims):
    """Wave of every direct-solver matrix (n > 128) of `dims`, by its index in `dims`, and the number of waves."""
    big = [i for i, n in enumerate(dims) if n > 128]
    cnt = len(big)
    n = (C.c_int * cnt)(*[dims[i] for i in big])
    mat, cta0, ncta = (C.c_int * cnt)(), (C.c_int * cnt)(), (C.c_int * cnt)()
    grid = torch.cuda.get_device_properties(0).multi_processor_count
    assert lib.kfac_stage_schedule(n, cnt, grid, mat, cta0, ncta) == cnt
    wave, wc, wp = (C.c_int * cnt)(), (C.c_int * cnt)(), (C.c_int * cnt)()
    nw = lib.kfac_stage_waves(n, cnt, grid, wave, wc, wp)
    return {big[mat[j]]: wave[j] for j in range(cnt)}, nw


def solve(lib, mats, max_waves):
    from kfac_b200 import _cabi
    lib.kfac_stage_eigh_max_waves(max_waves)
    try:
        items = (_cabi.EighItem * len(mats))()
        ns = (C.c_int * len(mats))(*[F.shape[0] for F in mats])
        outs = []
        for i, F in enumerate(mats):
            n = F.shape[0]
            ld = _cabi.ld4(n)
            Q, QT = torch.full((n, ld), float('nan'), device='cuda:0'), torch.full((n, ld), float('nan'), device='cuda:0')
            d = torch.full((n,), float('nan'), device='cuda:0')
            items[i] = _cabi.EighItem(F.data_ptr(), Q.data_ptr(), QT.data_ptr(), d.data_ptr(), n, ld, None)
            outs.append((Q[:, :n], QT[:, :n], d))
        need = lib.kfac_eigh_workspace_bytes(ns, len(mats))
        ws = torch.empty(need, dtype=torch.uint8, device='cuda:0')
        assert lib.kfac_eigh_batched(items, len(mats), ws.data_ptr(), need, 0, 0.0, S()) == 0, lib.kfac_last_error()
        host = torch.zeros(1, dtype=torch.int32).pin_memory()
        assert lib.kfac_eigh_status(ws.data_ptr(), host.data_ptr(), S()) == 0
        torch.cuda.synchronize()
        return outs, int(host.item())
    finally:
        lib.kfac_stage_eigh_max_waves(-1)


def assert_same_bits(a, b, what):
    for i, (x, y) in enumerate(zip(a, b)):
        for u, v, name in zip(x, y, ('Q', 'QT', 'd')):
            assert torch.equal(u.view(torch.int32), v.view(torch.int32)), (what, i, name)


@pytest.mark.parametrize('case', sorted(CASES))
def test_waves_same_bits_as_one_wave(lib, case):
    dims = CASES[case]
    _, nw = waves(lib, dims)
    if case == 'lone':
        assert nw == 1
    else:
        assert nw > 1, case       # the case must exercise several waves
    gen = torch.Generator().manual_seed(7)
    mats = [kfac_like(gen, n) for n in dims]
    one, st1 = solve(lib, mats, 1)
    many, st = solve(lib, mats, -1)
    assert st1 == 0 and st == 0
    assert_same_bits(many, one, case)
    # the outputs of a repeat call are the same bits too (per-wave tables and workspaces are rebuilt every call)
    again, st = solve(lib, mats, -1)
    assert st == 0
    assert_same_bits(again, one, case)


def test_non_finite_factor_alone_in_its_wave(lib):
    dims = CASES['mixed']
    wave_of, nw = waves(lib, dims)
    assert nw > 1
    alone = [i for i, w in wave_of.items() if list(wave_of.values()).count(w) == 1]
    assert alone, wave_of
    bad = alone[0]
    gen = torch.Generator().manual_seed(3)
    mats = [kfac_like(gen, n) for n in dims]
    mats[bad][5, 7] = float('nan')
    mats[bad][7, 5] = float('nan')
    many, st = solve(lib, mats, -1)
    one, st1 = solve(lib, mats, 1)
    assert st & 2 and st1 & 2, (st, st1)
    assert_same_bits(many, one, 'non-finite')
    for i, (Q, QT, d) in enumerate(many):
        if i != bad:
            assert torch.isfinite(Q).all() and torch.isfinite(d).all(), i
