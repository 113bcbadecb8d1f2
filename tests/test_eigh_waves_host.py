"""Host-only checks of the waves of the batched tridiagonalisation (kfac_stage_waves; no GPU).

The schedule's jobs are split into at most 4 waves.  Each wave is a cooperative launch of its own, on a grid of the CTAs
its jobs use, followed by the divide and conquer and back-transformation of its matrices on its own stream.  So a CTA
must belong to one wave only (a group barrier never waits on another launch), every job must run exactly once, on the
same CTAs relative to its group, and each wave must keep its jobs in the schedule's order (the order every CTA walks,
which keeps the group barriers deadlock free)."""
import ctypes

import pytest

R50 = [(147, 64, 1), (64, 64, 1), (64, 256, 4), (256, 64, 2), (576, 64, 3), (128, 512, 4), (256, 128, 1), (256, 512, 1),
       (512, 128, 3), (1152, 128, 4), (256, 1024, 6), (512, 256, 1), (512, 1024, 1), (1024, 256, 5), (2304, 256, 6),
       (512, 2048, 3), (1024, 512, 1), (1024, 2048, 1), (2048, 512, 2), (4608, 512, 3), (2049, 1000, 1)]
R50_DIRECT = [d for a, g, c in R50 for d in [a, g] * c if d > 128]
MAX_WAVES = 4

CASES = {
    'r50': R50_DIRECT,
    'mixed': [8192, 4608, 2304, 2304, 1024, 1000, 512, 300, 130],
    'mixed_small_first': [130, 700, 2049, 6000, 3000, 3000, 8192],
    'lone': [4608],
    'lone_small': [200],
    'many_small': [300] * 200,
    'many_tiny': [129, 140, 256] * 40,
}


@pytest.fixture(scope='module')
def lib():
    from kfac_b200 import _cabi
    lib = _cabi.load()
    i = ctypes.c_void_p
    lib.kfac_stage_schedule.restype = ctypes.c_int
    lib.kfac_stage_schedule.argtypes = [i, ctypes.c_int, ctypes.c_int, i, i, i]
    lib.kfac_stage_waves.restype = ctypes.c_int
    lib.kfac_stage_waves.argtypes = [i, ctypes.c_int, ctypes.c_int, i, i, i]
    lib.kfac_stage_pin_plan.restype = ctypes.c_int
    lib.kfac_stage_pin_plan.argtypes = [i, ctypes.c_int, ctypes.c_int, ctypes.c_longlong, i, i, i]
    lib.kfac_stage_eigh_max_waves.restype = None
    lib.kfac_stage_eigh_max_waves.argtypes = [ctypes.c_int]
    yield lib
    lib.kfac_stage_eigh_max_waves(-1)


def schedule_and_waves(lib, dims, grid):
    cnt = len(dims)
    n = (ctypes.c_int * cnt)(*dims)
    mat, cta0, ncta = (ctypes.c_int * cnt)(), (ctypes.c_int * cnt)(), (ctypes.c_int * cnt)()
    k = lib.kfac_stage_schedule(n, cnt, grid, mat, cta0, ncta)
    assert k == cnt
    wave, wcta0, wpos = (ctypes.c_int * cnt)(*[-1] * cnt), (ctypes.c_int * cnt)(), (ctypes.c_int * cnt)()
    nw = lib.kfac_stage_waves(n, cnt, grid, wave, wcta0, wpos)
    jobs = [(mat[j], cta0[j], ncta[j]) for j in range(k)]
    return jobs, nw, list(wave), list(wcta0), list(wpos)


def check_waves(jobs, nw, wave, wcta0, wpos, grid):
    assert 1 <= nw <= MAX_WAVES
    # every job in exactly one wave, every wave used
    assert all(0 <= w < nw for w in wave)
    assert set(wave) == set(range(nw))
    # no CTA in two waves
    owner = {}
    for (m, c0, nc), w in zip(jobs, wave):
        for c in range(c0, c0 + nc):
            assert owner.setdefault(c, w) == w, (c, owner[c], w)
            assert 0 <= c < grid
    for w in range(nw):
        js = [j for j in range(len(jobs)) if wave[j] == w]
        # the wave's job list is a subsequence of the schedule's order
        assert [wpos[j] for j in js] == list(range(len(js)))
        # rebased onto the wave's grid: a CTA's place is its rank among the wave's CTAs, so every group keeps its
        # CTAs, contiguous and in the same order
        ctas = sorted(c for c, o in owner.items() if o == w)
        rank = {c: r for r, c in enumerate(ctas)}
        for j in js:
            m, c0, nc = jobs[j]
            assert wcta0[j] == rank[c0]
            assert [rank[c] for c in range(c0, c0 + nc)] == list(range(wcta0[j], wcta0[j] + nc))


@pytest.mark.parametrize('grid', [132, 64])
@pytest.mark.parametrize('case', sorted(CASES))
def test_wave_partition(lib, case, grid):
    dims = CASES[case]
    if grid < 132 and max(dims) > 4608:
        pytest.skip('an 8192 or 6000 factor needs more CTAs than the smaller grid has')
    jobs, nw, wave, wcta0, wpos = schedule_and_waves(lib, dims, grid)
    check_waves(jobs, nw, wave, wcta0, wpos, grid)
    if len(dims) == 1:
        assert nw == 1


def test_r50_big_factors_leave_the_last_wave(lib):
    """The three 4608 factors carry most of the later-stage work: they must not wait for the job predicted to end
    last."""
    dims = R50_DIRECT
    cnt = len(dims)
    jobs, nw, wave, _, _ = schedule_and_waves(lib, dims, 132)
    assert nw > 1
    pin, t0, t1 = (ctypes.c_int * cnt)(), (ctypes.c_double * cnt)(), (ctypes.c_double * cnt)()
    n = (ctypes.c_int * cnt)(*dims)
    assert lib.kfac_stage_pin_plan(n, cnt, 132, -1, pin, t0, t1) == cnt
    last = max(range(len(jobs)), key=lambda j: t1[jobs[j][0]])
    big = [j for j, (m, _, _) in enumerate(jobs) if dims[m] == 4608]
    assert len(big) == 3
    assert all(wave[j] != wave[last] for j in big)


def test_max_waves_switch(lib):
    try:
        for limit in (1, 2):
            lib.kfac_stage_eigh_max_waves(limit)
            for case in sorted(CASES):
                jobs, nw, wave, wcta0, wpos = schedule_and_waves(lib, CASES[case], 132)
                assert nw <= limit
                check_waves(jobs, nw, wave, wcta0, wpos, 132)
                if limit == 1:
                    assert wpos == list(range(len(jobs)))
    finally:
        lib.kfac_stage_eigh_max_waves(-1)
