"""Host-only checks of the L2 residency plan of the batched tridiagonalisation (kfac_stage_pin_plan; no GPU).

The plan keeps a trailing triangle of lower tiles (block columns J >= pin_j0) of selected matrices in L2 with
evict_last hints.  It must never promise more L2 than its budget to the jobs that the schedule's time model runs at
the same time, and each matrix's pinned set must be one contiguous trailing triangle: the kernel pins and unpins block
columns by comparing J with pin_j0."""
import ctypes

import pytest

R50 = [(147, 64, 1), (64, 64, 1), (64, 256, 4), (256, 64, 2), (576, 64, 3), (128, 512, 4), (256, 128, 1), (256, 512, 1),
       (512, 128, 3), (1152, 128, 4), (256, 1024, 6), (512, 256, 1), (512, 1024, 1), (1024, 256, 5), (2304, 256, 6),
       (512, 2048, 3), (1024, 512, 1), (1024, 2048, 1), (2048, 512, 2), (4608, 512, 3), (2049, 1000, 1)]
R50_DIRECT = [d for a, g, c in R50 for d in [a, g] * c if d > 128]
TILE_BYTES = 64 * 64 * 4
MIB = 1 << 20


@pytest.fixture(scope='module')
def lib():
    from kfac_b200 import _cabi
    lib = _cabi.load()
    lib.kfac_stage_pin_plan.restype = ctypes.c_int
    lib.kfac_stage_pin_plan.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_longlong,
                                        ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    return lib


def plan(lib, dims, grid, budget):
    cnt = len(dims)
    n = (ctypes.c_int * cnt)(*dims)
    pin, t0, t1 = (ctypes.c_int * cnt)(), (ctypes.c_double * cnt)(), (ctypes.c_double * cnt)()
    assert lib.kfac_stage_pin_plan(n, cnt, grid, budget, pin, t0, t1) == cnt
    return list(pin), list(t0), list(t1)


def pinned_bytes(n, j0):
    nblk = (n + 63) // 64
    return sum(nblk - J for J in range(j0, nblk)) * TILE_BYTES


CASES = [R50_DIRECT, [4608], [4608, 4608, 2304, 2304, 512], [300] * 200, [2304, 2304, 129], [8192, 130]]


@pytest.mark.parametrize('budget_mib', [1, 16, 24, 32, 40])
@pytest.mark.parametrize('case', range(len(CASES)))
def test_budget_holds_at_every_instant(lib, case, budget_mib):
    dims = CASES[case]
    for grid in (132, 16):
        pin, t0, t1 = plan(lib, dims, grid, budget_mib * MIB)
        for i, n in enumerate(dims):
            assert 0 <= pin[i] <= (n + 63) // 64 and t1[i] > t0[i] >= 0.0
        # the running set only grows at job starts: checking every start checks every instant
        for t in sorted(set(t0)):
            load = sum(pinned_bytes(n, j0) for n, j0, a, b in zip(dims, pin, t0, t1) if a <= t < b)
            assert load <= budget_mib * MIB, (grid, t, load)


def test_budget_zero_pins_nothing(lib):
    for dims in CASES:
        pin, _, _ = plan(lib, dims, 132, 0)
        assert pin == [(n + 63) // 64 for n in dims]


@pytest.mark.parametrize('n', [4608, 2304, 1000, 257])
def test_lone_matrix_pins_the_largest_trailing_triangle_that_fits(lib, n):
    """The plan's only output per matrix is pin_j0, the first pinned block column, so a pinned set is a trailing
    triangle by construction.  Block columns are added from the bottom right (longest-lived tiles) outwards, so a lone
    matrix stops exactly where the next block column would overflow the budget."""
    nblk = (n + 63) // 64
    for budget in (TILE_BYTES - 1, TILE_BYTES, 3 * TILE_BYTES, 5 * MIB, 16 * MIB, 64 * MIB):
        (j0,), _, _ = plan(lib, [n], 132, budget)
        assert pinned_bytes(n, j0) <= budget
        assert j0 == 0 or pinned_bytes(n, j0 - 1) > budget, (n, budget, j0)
        assert j0 <= nblk


def test_deterministic(lib):
    for dims in CASES:
        for b in (0, 16 * MIB, 32 * MIB):
            assert plan(lib, dims, 132, b) == plan(lib, dims, 132, b)


def test_resnet50_pins_the_4608s(lib):
    """On the ResNet-50 list most of the budget goes to the three 4608 factors: their bottom-right tiles are read in
    every one of 4607 columns, more reads per pinned byte than any other matrix offers."""
    for budget_mib in (16, 32):
        pin, _, _ = plan(lib, R50_DIRECT, 132, budget_mib * MIB)
        big = [i for i, n in enumerate(R50_DIRECT) if n == 4608]
        assert len(big) == 3
        on_big = sum(pinned_bytes(4608, pin[i]) for i in big)
        total = sum(pinned_bytes(n, j0) for n, j0 in zip(R50_DIRECT, pin))
        assert all(pin[i] < 72 for i in big) and on_big >= 0.75 * total, (budget_mib, on_big, total)


def test_default_budget(lib):
    """A negative budget selects the built-in default, which pins something on the ResNet-50 list."""
    pin, _, _ = plan(lib, R50_DIRECT, 132, -1)
    assert any(j0 < (n + 63) // 64 for n, j0 in zip(R50_DIRECT, pin))
