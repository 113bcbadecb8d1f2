"""Grouped wgmma GEMM engine (csrc/gemm_grouped.cu) through its test-only C entry, every feature against fp64:
tile and k-block edges, split-K through slabs, the SIMT fallback in the same launch, both epilogues and alpha,
read-modify-write and atomic modes, device-side k ranges, one long mixed launch, determinism, canaries around
every output, and rejected lists that must leave every output untouched."""
import ctypes as C
import random

import pytest
import torch

from conftest import rel_fro

pytestmark = pytest.mark.gpu

EPI_NONE, EPI_MUL, EPI_DIV_OUTER = 0, 1, 2
GBK = 32                                   # k-block of the tensor-core engine; a device k range counts in these
DAMPING = float(torch.tensor(3e-3, dtype=torch.float32))
NAN = float('nan')


class StageGemm(C.Structure):
    _fields_ = [('A', C.c_void_p), ('lda', C.c_int64), ('B', C.c_void_p), ('ldb', C.c_int64),
                ('D', C.c_void_p), ('ldd', C.c_int64), ('M', C.c_int), ('N', C.c_int), ('K', C.c_int),
                ('alpha', C.c_float), ('epi', C.c_int), ('E', C.c_void_p), ('lde', C.c_int64),
                ('dg', C.c_void_p), ('da', C.c_void_p), ('damping', C.c_float),
                ('splits', C.c_int), ('slab', C.c_void_p), ('slab_stride', C.c_int64),
                ('mode', C.c_int), ('krange', C.c_void_p)]


@pytest.fixture(scope='module')
def lib():
    from kfac_b200 import _cabi
    lib = _cabi.load()
    lib.kfac_stage_grouped_gemm.restype = C.c_int
    lib.kfac_stage_grouped_gemm.argtypes = [C.POINTER(StageGemm), C.c_int, C.c_void_p, C.c_size_t, C.c_void_p]
    lib.kfac_stage_grouped_gemm_ws_bytes.restype = C.c_size_t
    lib.kfac_stage_grouped_gemm_ws_bytes.argtypes = [C.c_int]
    return lib


def S():
    return torch.cuda.current_stream().cuda_stream


def ld4(n):
    return (n + 3) // 4 * 4


def kblocks(K):
    return (K + GBK - 1) // GBK


def normalised_splits(splits, K):
    kb = kblocks(K)
    per = (kb + max(1, splits) - 1) // max(1, splits)
    return (kb + per - 1) // per


class Prob:
    """One problem D = epi(alpha * A B^T) (+ D0 in modes 1 and 2) with its operands and its fp64 reference.

    D is the top-left M x N block of an (M + 1) x ldd buffer, ldd > N: the extra row and the columns [N, ldd)
    start as NaN and are checked after the call.  Operand padding columns [K, ld) are NaN too, so a read past K
    poisons the result."""

    def __init__(self, M, N, K, seed, alpha=1.0, epi=EPI_NONE, mode=0, splits=1, krange=None, a_offset=0,
                 lda=None, ldd=None, slab=True):
        dev = torch.device('cuda:0')
        gen = torch.Generator(device=dev).manual_seed(seed)
        self.M, self.N, self.K, self.alpha, self.epi, self.mode, self.splits = M, N, K, alpha, epi, mode, splits
        self.krange = krange
        self.lda = lda if lda is not None else ld4(K)
        self.ldb = ld4(K)
        self.ldd = ldd if ldd is not None else N + 5
        abuf = torch.full((a_offset + M * self.lda,), NAN, device=dev)
        self.A = abuf[a_offset:].view(M, self.lda)
        self.A[:, :K] = torch.randn(M, K, device=dev, generator=gen)
        self.B = torch.full((N, self.ldb), NAN, device=dev)
        self.B[:, :K] = torch.randn(N, K, device=dev, generator=gen)
        self.D = torch.full((M + 1, self.ldd), NAN, device=dev)
        self.D0 = None
        if mode != 0:   # accumulate into a D0 of the size of the product
            self.D0 = torch.randn(M, N, device=dev, generator=gen) * K ** 0.5
            self.D[:M, :N] = self.D0
        self.lde = self.ldd + 3          # != ldd: the epilogue must index E with its own leading dimension
        self.E = self.dg = self.da = None
        if epi == EPI_MUL:
            self.E = torch.full((M, self.lde), NAN, device=dev)
            self.E[:, :N] = 0.5 + torch.rand(M, N, device=dev, generator=gen)
        elif epi == EPI_DIV_OUTER:
            self.dg = 0.05 + torch.rand(M, device=dev, generator=gen)
            self.da = 0.05 + torch.rand(N, device=dev, generator=gen)
        self.slab = None
        self.slab_stride = M * self.ldd
        if splits > 1 and slab and mode != 2:
            self.slab = torch.full((splits * self.slab_stride,), NAN, device=dev)
        self.kr = torch.tensor(krange, dtype=torch.int32, device=dev) if krange is not None else None
        self.D_init = self.D.clone()

    @property
    def tc(self):
        """Whether the engine runs this problem on the tensor-core path (grouped_gemm_tc_ok)."""
        return (self.M >= 64 and self.N >= 64 and self.K >= 32 and self.A.data_ptr() % 16 == 0
                and self.B.data_ptr() % 16 == 0 and self.lda % 4 == 0 and self.ldb % 4 == 0)

    @property
    def nsplit(self):
        return normalised_splits(self.splits, self.K) if self.tc else 1

    @property
    def reduced(self):
        """Split through slabs: grouped_reduce_kernel writes D."""
        return self.tc and self.mode != 2 and self.nsplit > 1

    @property
    def atomic_split(self):
        return self.tc and self.mode == 2 and self.nsplit > 1

    def desc(self):
        return (f'M={self.M} N={self.N} K={self.K} alpha={self.alpha} epi={self.epi} mode={self.mode} '
                f'splits={self.splits}->{self.nsplit} krange={self.krange} lda={self.lda} tc={self.tc}')

    def struct(self):
        p = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
        return StageGemm(self.A.data_ptr(), self.lda, self.B.data_ptr(), self.ldb, self.D.data_ptr(), self.ldd,
                         self.M, self.N, self.K, self.alpha, self.epi, p(self.E), self.lde, p(self.dg), p(self.da),
                         DAMPING, self.splits, p(self.slab), self.slab_stride, self.mode, p(self.kr))

    def reset(self):
        self.D.copy_(self.D_init)
        if self.slab is not None:
            self.slab.fill_(NAN)

    def reference(self):
        K = self.K
        A64, B64 = self.A[:, :K].double(), self.B[:, :K].double()
        if self.krange is not None:      # exactly the k columns of the clamped k-block range
            lo, hi = max(0, self.krange[0]), min(kblocks(K), self.krange[1])
            c0, c1 = GBK * lo, min(K, GBK * max(lo, hi))
            A64, B64 = A64[:, c0:c1], B64[:, c0:c1]
        ref = self.alpha * (A64 @ B64.t())
        if self.epi == EPI_MUL:
            ref = ref * self.E[:, :self.N].double()
        elif self.epi == EPI_DIV_OUTER:
            ref = ref / (torch.outer(self.dg.double(), self.da.double()) + DAMPING)
        if self.D0 is not None:
            ref = ref + self.D0.double()
        return ref

    def check(self):
        M, N, K = self.M, self.N, self.K
        out = self.D[:M, :N]
        ref = self.reference()
        assert bool(torch.isfinite(out).all()), self.desc()
        fro = rel_fro(out, ref)
        if self.tc:
            mx = float((out.double() - ref).abs().max() / ref.abs().max())
            assert fro < 3e-6 + 4e-9 * K, (self.desc(), fro)
            assert mx < 2e-5 + 1e-8 * K, (self.desc(), mx)
        else:
            assert fro < 1e-5, (self.desc(), fro)
        assert bool(torch.isnan(self.D[M]).all()), ('row M written', self.desc())
        pad = self.D[:M, N:]
        if self.reduced:                 # the slab reduction stores zeros into the padding columns
            assert bool((pad == 0).all()), ('padding columns of a split problem', self.desc())
        else:
            assert bool(torch.isnan(pad).all()), ('padding columns written', self.desc())
        if self.slab is not None:        # slabs past the normalised split count are never touched
            assert bool(torch.isnan(self.slab[self.nsplit * self.slab_stride:]).all()), self.desc()


def run(lib, probs, ws_bytes=None):
    """One grouped launch over `probs` with a NaN-filled workspace; returns the status."""
    arr = (StageGemm * len(probs))(*[p.struct() for p in probs])
    need = lib.kfac_stage_grouped_gemm_ws_bytes(len(probs))
    ws = torch.full((need,), 255, dtype=torch.uint8, device='cuda:0')   # all-ones bytes: NaN floats
    rc = lib.kfac_stage_grouped_gemm(arr, len(probs), ws.data_ptr(), need if ws_bytes is None else ws_bytes, S())
    torch.cuda.synchronize()
    return rc


def run_and_check(lib, probs):
    rc = run(lib, probs)
    assert rc == 0, lib.kfac_last_error()
    for p in probs:
        p.check()


@pytest.mark.parametrize('M,N,K', [(128, 128, 32), (129, 127, 33), (64, 64, 32), (200, 577, 1000), (4608, 64, 300),
                                   (64, 4608, 64)])
def test_tile_and_kblock_edges(lib, M, N, K):
    p = Prob(M, N, K, seed=M + N + K, alpha=0.5)
    assert p.tc
    run_and_check(lib, [p])


def test_split_k_through_slabs(lib):
    probs = [Prob(256, 200, 1025, seed=1, splits=3),
             Prob(130, 129, 2049, seed=2, splits=5),
             Prob(100, 100, 300, seed=3),                       # an unsplit problem between split ones
             Prob(256, 256, 4608, seed=4, splits=9),
             Prob(128, 192, 64, seed=5, splits=5)]              # more splits than k-blocks: runs as 2
    assert [p.nsplit for p in probs] == [3, 5, 1, 9, 2]
    run_and_check(lib, probs)


def test_simt_fallback_in_a_tensor_core_launch(lib):
    probs = [Prob(128, 128, 64, seed=10),
             Prob(63, 200, 100, seed=11),
             Prob(200, 63, 100, seed=12),
             Prob(256, 300, 160, seed=13, alpha=0.5),
             Prob(100, 100, 31, seed=14),
             Prob(1, 1, 1, seed=15),
             Prob(128, 128, 101, seed=16, a_offset=1, lda=101),  # A is not 16-byte aligned
             Prob(200, 130, 96, seed=17)]
    assert [p.tc for p in probs] == [True, False, False, True, False, False, False, True]
    run_and_check(lib, probs)


def test_epilogues_and_alpha(lib):
    probs = []
    for shape in ((200, 300, 130), (50, 70, 45)):      # tensor-core path, SIMT path
        probs += [Prob(*shape, seed=20, alpha=0.5, epi=EPI_MUL),
                  Prob(*shape, seed=21, alpha=-1.0, epi=EPI_DIV_OUTER),
                  Prob(*shape, seed=22, alpha=0.5, epi=EPI_DIV_OUTER),
                  Prob(*shape, seed=23, alpha=-1.0, epi=EPI_MUL),
                  Prob(*shape, seed=24, alpha=-1.0)]
    assert [p.tc for p in probs] == [True] * 5 + [False] * 5
    run_and_check(lib, probs)


def test_accumulate_modes(lib):
    probs = [Prob(200, 300, 100, seed=30, mode=1, alpha=-1.0),        # D += alpha A B^T, read-modify-write
             Prob(40, 50, 70, seed=31, mode=1, alpha=0.5),
             Prob(129, 130, 200, seed=32, mode=1, ldd=133),           # odd ldd: the scalar store path
             Prob(200, 300, 100, seed=33, mode=2),                    # atomic, one split: every element once
             Prob(256, 192, 1500, seed=34, mode=2, splits=3),         # atomic split-K
             Prob(40, 50, 70, seed=35, mode=2, alpha=-1.0)]
    assert [p.tc for p in probs] == [True, False, True, True, True, False]
    run_and_check(lib, probs)


def test_device_k_range(lib):
    K = 300                                  # 10 k-blocks, the last one partial
    kb = kblocks(K)
    ranges = [(0, kb), (2, 7), (5, 5), (3, 1000), (-4, 3)]
    probs = [Prob(200, 150, K, seed=40 + i, mode=2, krange=r) for i, r in enumerate(ranges)]
    # a range across split boundaries: the third split lies past the range and is skipped
    probs.append(Prob(256, 130, 1100, seed=46, mode=2, splits=3, krange=(5, 20)))
    run_and_check(lib, probs)
    # the empty range leaves D0 (and its NaN walls) bit for bit as it was
    assert torch.equal(probs[2].D.view(torch.int32), probs[2].D_init.view(torch.int32))


def mixed_problems(seed=0, count=60):
    rnd = random.Random(seed)
    probs = []
    for i in range(count):
        kind = rnd.random()
        if kind < 0.15:      # SIMT-sized
            M, N, K = rnd.randint(1, 63), rnd.randint(1, 200), rnd.randint(1, 150)
        else:
            M, N, K = rnd.randint(64, 520), rnd.randint(64, 520), rnd.randint(32, 700)
        mode = rnd.choice([0, 0, 0, 1, 2])
        epi = rnd.choice([EPI_NONE, EPI_MUL, EPI_DIV_OUTER]) if mode == 0 else EPI_NONE
        alpha = rnd.choice([1.0, 0.5, -1.0])
        splits, krange = 1, None
        if mode != 1 and epi == EPI_NONE and kind >= 0.15 and rnd.random() < 0.4:
            K = rnd.randint(1025, 2100)
            splits = (K + 511) // 512
        if mode == 2 and kind >= 0.15 and rnd.random() < 0.5:
            kb = kblocks(K)
            lo = rnd.randint(-2, kb)
            krange = (lo, lo + rnd.randint(0, kb))
        probs.append(Prob(M, N, K, seed=1000 + i, alpha=alpha, epi=epi, mode=mode, splits=splits, krange=krange))
    return probs


def test_mixed_launch_and_determinism(lib):
    probs = mixed_problems()
    tc = [p for p in probs if p.tc]
    work = sum(((p.M + 127) // 128) * ((p.N + 127) // 128) * p.nsplit for p in tc)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    # every CTA of the persistent kernel walks items of several problems
    assert work > 2 * sms and len(tc) < len(probs)
    assert any(p.reduced for p in probs) and any(p.atomic_split for p in probs) and any(p.krange for p in probs)
    run_and_check(lib, probs)
    first = [p.D.clone() for p in probs]
    for p in probs:
        p.reset()
    assert run(lib, probs) == 0, lib.kfac_last_error()
    for p, d in zip(probs, first):
        if not p.atomic_split:          # atomic split-K adds its partials in arrival order
            assert torch.equal(p.D.view(torch.int32), d.view(torch.int32)), p.desc()


@pytest.mark.parametrize('bad', ['split_without_slab', 'krange_without_atomic', 'krange_on_simt', 'workspace'])
def test_rejected_list_has_no_side_effects(lib, bad):
    from kfac_b200 import _cabi
    probs = [Prob(40, 40, 40, seed=50), Prob(128, 128, 64, seed=51)]
    if bad == 'split_without_slab':
        probs.append(Prob(128, 128, 1024, seed=52, splits=2, slab=False))
    elif bad == 'krange_without_atomic':
        probs.append(Prob(128, 128, 256, seed=53, krange=(0, 4)))
    elif bad == 'krange_on_simt':
        probs.append(Prob(32, 128, 256, seed=54, mode=2, krange=(0, 4)))
    assert not probs[0].tc and probs[1].tc
    ws_bytes = lib.kfac_stage_grouped_gemm_ws_bytes(len(probs)) - 1 if bad == 'workspace' else None
    rc = run(lib, probs, ws_bytes)
    assert rc == (_cabi.KFAC_ERR_WORKSPACE if bad == 'workspace' else _cabi.KFAC_ERR_BAD_ARG), rc
    assert lib.kfac_last_error()
    for p in probs:
        assert torch.equal(p.D.view(torch.int32), p.D_init.view(torch.int32)), (bad, p.desc())
