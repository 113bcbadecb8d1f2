"""Reference digests of the wgmma GEMM engine's outputs (tests/golden/engine_bits.json).

Needs one H100.  Every case runs a seeded set of engine calls and hashes the exact output bits (SHA-256 of the
float32 arrays), so a change to the engine's schedule, staging or register use can be checked to leave every bit
of every output where it was.  Each case's kernel launches (kfac_launch_count) are recorded beside its digest:

    python tests/gen_engine_bits.py [OUT.json]        # default: tests/golden/engine_bits.json

tests/test_gpu_engine_bits.py recomputes the same cases and compares.  The benchmark's training dynamics turn any
last-bit change into different outputs within a few steps, so the check is equality, not a tolerance.
"""
from __future__ import annotations

import ctypes as C
import hashlib
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from kfac_b200 import _cabi  # noqa: E402

GOLDEN = os.path.join(HERE, 'golden', 'engine_bits.json')
EPI_NONE, EPI_MUL, EPI_DIV_OUTER, EPI_SQUARE = 0, 1, 2, 3

# ResNet-50 factor dimensions (a, g, count), as in tests/eigh_batch_probe.py
R50 = [(147, 64, 1), (64, 64, 1), (64, 256, 4), (256, 64, 2), (576, 64, 3), (128, 512, 4), (256, 128, 1), (256, 512, 1),
       (512, 128, 3), (1152, 128, 4), (256, 1024, 6), (512, 256, 1), (512, 1024, 1), (1024, 256, 5), (2304, 256, 6),
       (512, 2048, 3), (1024, 512, 1), (1024, 2048, 1), (2048, 512, 2), (4608, 512, 3), (2049, 1000, 1)]


class StageGemm(C.Structure):
    _fields_ = [('A', C.c_void_p), ('lda', C.c_int64), ('B', C.c_void_p), ('ldb', C.c_int64),
                ('D', C.c_void_p), ('ldd', C.c_int64), ('M', C.c_int), ('N', C.c_int), ('K', C.c_int),
                ('alpha', C.c_float), ('epi', C.c_int), ('E', C.c_void_p), ('lde', C.c_int64),
                ('dg', C.c_void_p), ('da', C.c_void_p), ('damping', C.c_float),
                ('splits', C.c_int), ('slab', C.c_void_p), ('slab_stride', C.c_int64),
                ('mode', C.c_int), ('krange', C.c_void_p)]


def _lib():
    lib = _cabi.load()
    lib.kfac_stage_grouped_gemm.restype = C.c_int
    lib.kfac_stage_grouped_gemm.argtypes = [C.POINTER(StageGemm), C.c_int, C.c_void_p, C.c_size_t, C.c_void_p]
    lib.kfac_stage_grouped_gemm_ws_bytes.restype = C.c_size_t
    lib.kfac_stage_grouped_gemm_ws_bytes.argtypes = [C.c_int]
    return lib


def _dev():
    return torch.device('cuda:0')


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _randn(gen, *shape):
    """Seeded on the CPU, so the inputs do not depend on the device's generator."""
    return torch.randn(*shape, generator=gen).to(_dev())


def _digest(*tensors):
    torch.cuda.synchronize()
    h = hashlib.sha256()
    for t in tensors:
        h.update(t.detach().float().contiguous().cpu().numpy().tobytes())
    return h.hexdigest()


def _ld4(n):
    return (n + 3) // 4 * 4


def case_gemm_tn_tc(M, N, K):
    lib = _lib()
    gen = torch.Generator().manual_seed(M * 7 + N * 3 + K)
    lda = _ld4(K)
    A = torch.zeros(M, lda, device=_dev())
    B = torch.zeros(N, lda, device=_dev())
    A[:, :K] = _randn(gen, M, K)
    B[:, :K] = _randn(gen, N, K)
    D = torch.zeros(M, N, device=_dev())
    # one split per tile: split K on this entry point is the atomic path, whose bits depend on the order of the adds
    rc = lib.kfac_gemm_tn_tc(A.data_ptr(), lda, B.data_ptr(), lda, D.data_ptr(), N, M, N, K, 0.75, 0, 1, _stream())
    assert rc == 0, lib.kfac_last_error()
    return _digest(D)


def case_grouped():
    """One grouped launch: split-K through slabs, read-modify-write, a device k range, every epilogue kind, and
    a problem small enough for the SIMT fallback."""
    lib = _lib()
    gen = torch.Generator().manual_seed(2024)
    probs, keep, outs = [], [], []

    def prob(M, N, K, alpha=1.0, epi=EPI_NONE, mode=0, splits=1, krange=None):
        lda = _ld4(K)
        A = torch.zeros(M, lda, device=_dev())
        B = torch.zeros(N, lda, device=_dev())
        A[:, :K] = _randn(gen, M, K)
        B[:, :K] = _randn(gen, N, K)
        ldd = N + 3
        D = _randn(gen, M, ldd) if mode else torch.zeros(M, ldd, device=_dev())
        E = _randn(gen, M, N) if epi == EPI_MUL else None
        dg = _randn(gen, M).abs() if epi == EPI_DIV_OUTER else None
        da = _randn(gen, N).abs() if epi == EPI_DIV_OUTER else None
        slab = torch.zeros(splits, M, ldd, device=_dev()) if splits > 1 else None
        kr = torch.tensor(krange, dtype=torch.int32, device=_dev()) if krange else None
        keep.extend([A, B, D, E, dg, da, slab, kr])
        outs.append(D)
        probs.append(StageGemm(A.data_ptr(), lda, B.data_ptr(), lda, D.data_ptr(), ldd, M, N, K, alpha, epi,
                               E.data_ptr() if E is not None else None, N,
                               dg.data_ptr() if dg is not None else None, da.data_ptr() if da is not None else None,
                               3e-3, splits, slab.data_ptr() if slab is not None else None,
                               M * ldd if splits > 1 else 0, mode, kr.data_ptr() if kr is not None else None))

    prob(512, 384, 2048, splits=4)                          # split-K slabs + fixed-order reduce
    prob(300, 260, 1000, splits=3)                          # ragged tiles, ragged last split
    prob(256, 256, 256, alpha=0.5, mode=1)                  # read-modify-write accumulate
    prob(200, 136, 700, mode=2, krange=(3, 17))             # device-side k range, one split: one add per element
    prob(384, 200, 96, epi=EPI_MUL)
    prob(130, 257, 512, epi=EPI_DIV_OUTER, alpha=-1.25)
    prob(256, 128, 333, epi=EPI_SQUARE)
    prob(40, 30, 20)                                        # SIMT fallback in the same call
    arr = (StageGemm * len(probs))(*probs)
    need = lib.kfac_stage_grouped_gemm_ws_bytes(len(probs))
    ws = torch.empty(need, dtype=torch.uint8, device=_dev())
    rc = lib.kfac_stage_grouped_gemm(arr, len(probs), ws.data_ptr(), need, _stream())
    assert rc == 0, lib.kfac_last_error()
    return _digest(*outs)


def case_factor_syrk(with_slab):
    """The tensor-core SYRK of a tall Linear input: split partials + fixed-order reduce with the full workspace,
    one split accumulating into the factor with only the packing space."""
    lib = _lib()
    gen = torch.Generator().manual_seed(31)
    rows, feat = 6000, 768
    x = _randn(gen, rows, feat)
    acc = _randn(gen, feat + 1, feat + 1)
    full = lib.kfac_factor_linear_workspace_bytes(rows, feat, 1)
    pack = _ld4(rows) * (feat + 1) * 4
    need = full if with_slab else pack
    assert full > pack
    ws = torch.empty(need, dtype=torch.uint8, device=_dev())
    rc = lib.kfac_factor_linear(x.data_ptr(), 0, rows, feat, 1, 1.0 / rows, acc.data_ptr(), ws.data_ptr(), need,
                                _stream())
    assert rc == 0, lib.kfac_last_error()
    return _digest(acc)


def _kfac_like(gen, n):
    m = max(8, n // 3)
    x = torch.relu(torch.randn(m, n, generator=gen) + 0.3) * torch.logspace(0, -2, n)
    x = x.to(_dev(), torch.float64)
    F = 0.5 * torch.eye(n, device=_dev(), dtype=torch.float64) + 0.5 * (x.t() @ x) / m
    return ((F + F.t()) / 2).float().contiguous()


def case_eigh_r50():
    """One kfac_eigh_batched call over all 108 ResNet-50 factors: D&C merges and back-transformation."""
    lib = _cabi.load()
    gen = torch.Generator().manual_seed(0)
    dims = [d for a, g, c in R50 for d in [a, g] * c]
    items = (_cabi.EighItem * len(dims))()
    keep, outs = [], []
    for i, n in enumerate(dims):
        F = _kfac_like(gen, n)
        ld = _cabi.ld4(n)
        Q, QT, d = torch.zeros(n, ld, device=_dev()), torch.zeros(n, ld, device=_dev()), torch.zeros(n, device=_dev())
        keep.append(F)
        outs.extend([Q, QT, d])
        items[i] = _cabi.EighItem(F.data_ptr(), Q.data_ptr(), QT.data_ptr(), d.data_ptr(), n, ld, None)
    ns = (C.c_int * len(dims))(*dims)
    need = lib.kfac_eigh_workspace_bytes(ns, len(dims))
    ws = torch.empty(need, dtype=torch.uint8, device=_dev())
    rc = lib.kfac_eigh_batched(items, len(dims), ws.data_ptr(), need, 0, 0.0, _stream())
    assert rc == 0, lib.kfac_last_error()
    return _digest(*outs)


def case_precondition():
    """One kfac_precondition call (eigen method) over two dense layers: the grouped precondition stages with the
    fused epilogues."""
    lib = _cabi.load()
    gen = torch.Generator().manual_seed(7)
    layers = [(1000, 2049), (512, 4608)]
    items = (_cabi.PrecondItem * len(layers))()
    keep, outs = [], []
    for i, (g, a) in enumerate(layers):
        qa = torch.linalg.qr(torch.randn(a, a, generator=gen, dtype=torch.float64))[0].float()
        qg = torch.linalg.qr(torch.randn(g, g, generator=gen, dtype=torch.float64))[0].float()
        ta = torch.zeros(a, _cabi.ld4(a), device=_dev())
        tg = torch.zeros(g, _cabi.ld4(g), device=_dev())
        ta[:, :a] = qa.to(_dev())
        tg[:, :g] = qg.to(_dev())
        taT = torch.zeros_like(ta)
        tgT = torch.zeros_like(tg)
        taT[:, :a] = qa.t().to(_dev())
        tgT[:, :g] = qg.t().to(_dev())
        da = _randn(gen, a).abs()
        dg = _randn(gen, g).abs()
        w = _randn(gen, g, a - 1)
        b = _randn(gen, g)
        P = torch.zeros(g, _cabi.ld4(a), device=_dev())
        keep.extend([ta, tg, taT, tgT, da, dg, w, b])
        outs.append(P)
        items[i] = _cabi.PrecondItem(w.data_ptr(), b.data_ptr(), 0, g, a, ta.data_ptr(), taT.data_ptr(),
                                     tg.data_ptr(), tgT.data_ptr(), None, da.data_ptr(), dg.data_ptr(), None, None,
                                     _cabi.ld4(a), _cabi.ld4(g), _cabi.ld4(a), P.data_ptr(), _cabi.ld4(a))
    need = lib.kfac_precondition_workspace_bytes(items, len(layers))
    ws = torch.empty(need, dtype=torch.uint8, device=_dev())
    rc = lib.kfac_precondition(items, len(layers), _cabi.KFAC_EIGEN, 3e-3, ws.data_ptr(), need, _stream())
    assert rc == 0, lib.kfac_last_error()
    return _digest(*outs)


def _precond_item(gen, keep, kind, g, a, bias=False, epi='dadg', taps=0, ldp_pad=0):
    """One kfac_precondition item of any kind, with every second-order operand filled (seeded), so that both methods
    can run on it.  g and a are the item's fields: for an embedding or tied item g = d and a = V.  Returns the item
    and its P (rows x ldp, ldp = ld4 of P's columns + ldp_pad)."""
    ld4 = _cabi.ld4

    def mat(n):                                       # n x ld4(n), zero padding columns
        m = torch.zeros(n, ld4(n), device=_dev())
        m[:, :n] = _randn(gen, n, n) / n ** 0.5
        return m

    def vec(n):
        return _randn(gen, n).abs() + 0.1

    it = _cabi.PrecondItem()
    it.kind, it.g, it.a, it.grad_dtype, it.wgrad_taps = kind, g, a, 0, taps
    transposed_rows = kind in (_cabi.KFAC_ITEM_EMBEDDING, _cabi.KFAC_ITEM_TIED)   # wgrad is (a, g) = (V, d)
    rows, cols = (a, g) if transposed_rows else (g, a)
    hb = 1 if bias else 0
    w = _randn(gen, (cols - hb) // taps, rows, taps) if taps else _randn(gen, rows, cols - hb)
    b = _randn(gen, rows) if bias else None
    it.wgrad, it.bgrad = w.data_ptr(), (b.data_ptr() if bias else None)
    keep.extend([w, b])
    fields = {}
    if kind in (_cabi.KFAC_ITEM_DENSE, _cabi.KFAC_ITEM_DIAG_G):
        fields.update(qa=mat(a), qaT=mat(a), a_inv=mat(a), da=vec(a))
        it.ldqa = ld4(a)
    if kind in (_cabi.KFAC_ITEM_DENSE, _cabi.KFAC_ITEM_EMBEDDING, _cabi.KFAC_ITEM_TIED, _cabi.KFAC_ITEM_DIAG_A):
        fields.update(qg=mat(g), qgT=mat(g), g_inv=mat(g), dg=vec(g))
        it.ldqg = ld4(g)
    if kind != _cabi.KFAC_ITEM_DENSE and 'da' not in fields:
        fields['da'] = vec(a)
    if kind == _cabi.KFAC_ITEM_DIAG_G:
        fields['dg'] = vec(g)
    if kind == _cabi.KFAC_ITEM_DENSE and epi == 'dgda':
        fields['dgda'] = _randn(gen, g, ld4(a)).abs() + 0.1
        it.ld_dgda = ld4(a)
    if kind == _cabi.KFAC_ITEM_TIED:
        fields['dh'] = vec(a)
        it.tied_damping = 0.25
    for name, t in fields.items():
        setattr(it, name, t.data_ptr())
        keep.append(t)
    it.ldp = ld4(cols) + ldp_pad
    P = torch.zeros(rows, it.ldp, device=_dev())
    it.P = P.data_ptr()
    return it, P


def case_precondition_kinds(method, specs):
    """One kfac_precondition call over the items of `specs` ((kind, g, a, options) each) with the given method."""
    lib = _cabi.load()
    gen = torch.Generator().manual_seed(11)
    keep, outs = [], []
    items = (_cabi.PrecondItem * len(specs))()
    for i, (kind, g, a, opts) in enumerate(specs):
        items[i], P = _precond_item(gen, keep, kind, g, a, **opts)
        outs.append(P)
    need = lib.kfac_precondition_workspace_bytes(items, len(specs))
    ws = torch.zeros(need, dtype=torch.uint8, device=_dev())
    rc = lib.kfac_precondition(items, len(specs), method, 3e-3, ws.data_ptr(), need, _stream())
    assert rc == 0, lib.kfac_last_error()
    return _digest(*outs)


DENSE, EMB, DIAG_G, TIED, DIAG_A = (_cabi.KFAC_ITEM_DENSE, _cabi.KFAC_ITEM_EMBEDDING, _cabi.KFAC_ITEM_DIAG_G,
                                    _cabi.KFAC_ITEM_TIED, _cabi.KFAC_ITEM_DIAG_A)
EIGEN, INVERSE = _cabi.KFAC_EIGEN, _cabi.KFAC_INVERSE
# every item kind and method; a > 1024 splits stages (1) and (3), g > 1024 (n > 1024 for a diagonal item) stage (4)
PRECOND_CASES = {
    'dense_dgda': (EIGEN, [(DENSE, 300, 1501, dict(bias=True, epi='dgda')), (DENSE, 1500, 300, dict(epi='dgda')),
                           (DENSE, 96, 130, dict(bias=True, epi='dgda'))]),
    'dense_dadg': (EIGEN, [(DENSE, 300, 1501, dict(bias=True)), (DENSE, 1500, 300, {}), (DENSE, 96, 130, {})]),
    'dense_inverse': (INVERSE, [(DENSE, 300, 1501, dict(bias=True)), (DENSE, 1500, 300, {}), (DENSE, 96, 130, {})]),
    'conv_transpose_eigen': (EIGEN, [(DENSE, 96, 40 * 9 + 1, dict(bias=True, taps=9))]),
    'conv_transpose_inverse': (INVERSE, [(DENSE, 1100, 24 * 27, dict(taps=27))]),
    'embedding_eigen': (EIGEN, [(EMB, 1000, 3000, {}), (EMB, 1100, 2000, {})]),
    'embedding_inverse': (INVERSE, [(EMB, 1000, 3000, {}), (EMB, 1100, 2000, {})]),
    'diag_g_eigen': (EIGEN, [(DIAG_G, 3000, 1000, dict(bias=True)), (DIAG_G, 2000, 1101, dict(bias=True))]),
    'diag_g_inverse': (INVERSE, [(DIAG_G, 3000, 1000, dict(bias=True)), (DIAG_G, 2000, 1101, dict(bias=True))]),
    'diag_a_eigen': (EIGEN, [(DIAG_A, 1100, 3001, dict(bias=True)), (DIAG_A, 500, 2000, {})]),
    'diag_a_inverse': (INVERSE, [(DIAG_A, 1100, 3001, dict(bias=True)), (DIAG_A, 500, 2000, {})]),
    'tied_eigen': (EIGEN, [(TIED, 1100, 3000, {}), (TIED, 200, 1500, {})]),
    'mixed_eigen': (EIGEN, [(DENSE, 1100, 1200, dict(bias=True)), (EMB, 1100, 2000, {}),
                            (DIAG_G, 1500, 1030, dict(bias=True)), (TIED, 300, 1000, {}), (DIAG_A, 1050, 2001, dict(bias=True)),
                            (DENSE, 64, 40 * 4, dict(taps=4))]),
    'mixed_inverse': (INVERSE, [(DENSE, 1100, 1200, dict(bias=True)), (EMB, 1100, 2000, {}),
                                (DIAG_G, 1500, 1030, dict(bias=True)), (TIED, 300, 1000, {}),
                                (DIAG_A, 1050, 2001, dict(bias=True)), (DENSE, 64, 40 * 4, dict(taps=4))]),
    'ldp_padded': (EIGEN, [(DENSE, 1500, 300, dict(ldp_pad=8)), (EMB, 1100, 2000, dict(ldp_pad=4))]),
}


CASES = {
    'gemm_tn_tc_4096': lambda: case_gemm_tn_tc(4096, 4096, 4096),
    'gemm_tn_tc_odd_1000x777x1234': lambda: case_gemm_tn_tc(1000, 777, 1234),
    'gemm_tn_tc_odd_129x65x33': lambda: case_gemm_tn_tc(129, 65, 33),
    'gemm_tn_tc_odd_4099x131x517': lambda: case_gemm_tn_tc(4099, 131, 517),
    'grouped_mixed': case_grouped,
    'factor_syrk_split': lambda: case_factor_syrk(True),
    'factor_syrk_one_split': lambda: case_factor_syrk(False),
    'eigh_r50': case_eigh_r50,
    'precondition_eigen': case_precondition,
    **{f'precondition_{name}': (lambda m=m, s=s: case_precondition_kinds(m, s)) for name, (m, s) in PRECOND_CASES.items()},
}


def run(name):
    """(digest, native kernel launches) of one case"""
    lib = _cabi.load()
    before = lib.kfac_launch_count()
    digest = CASES[name]()
    return digest, lib.kfac_launch_count() - before


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else GOLDEN
    res, launches = {}, {}
    for name in CASES:
        res[name], launches[name] = run(name)
        print(name, res[name], launches[name], flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
    with open(out, 'w') as f:
        json.dump({'device': torch.cuda.get_device_name(0), 'digests': res, 'launches': launches}, f, indent=1,
                  sort_keys=True)
        f.write('\n')
    print('wrote', out)


if __name__ == '__main__':
    main()
