"""The fused precondition broadcast (`peer_P` / `n_peers` of kfac_precond_item) on one GPU, against fp64.

With gradient broadcasts over NCCL (KAISA HYBRID-OPT and MEM-OPT), the last precondition GEMM stores P into the local
P arena and into the arena of every receiver of the layer, mapped into this process with CUDA IPC.  The peers are
plain device pointers, so other buffers on the same device exercise every store path: the tile epilogue (float2 and
scalar stores), the reduce pass of a split product (g > 1024, or n > 1024 for the diagonal kinds) and the copies
after the SIMT engine.  The arenas are laid out as the product lays them out: one entry of rows x ld4(n) floats per
layer, one after another, NaN-filled, with guard regions around every arena and entries of layers that are not in
the call.  Eigenbases and inverses are fp32 as stored; the references are fp64 products of those fp32 values.

  * P against fp64 (1e-4 rel-Frobenius), every peer entry equal to P bit for bit, guards and foreign entries untouched;
  * P does not depend on the number of peers (0, 1, 3, 7), nor does the workspace size;
  * a repeat call gives the same bits in P and in every peer;
  * kl-clip scale and write-back of a receiver (reading a peer arena) equal those of the worker (reading P);
  * rejected peer arguments leave P and every peer untouched;
  * a second process on the same GPU exports its arena (kfac_peer_alloc), this one maps it (kfac_peer_open) and
    preconditions into it: the child finds the bytes of P.
"""
import ctypes as C
import multiprocessing as mp

import pytest
import torch

from conftest import rel_fro

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda')
GUARD = 1024                 # floats before and after every arena
MAX_PEERS = 7                # receivers of an 8-GPU node
NAN = float('nan')


@pytest.fixture(scope='module')
def lib():
    from kfac_b200 import _cabi
    return _cabi.load()


def S():
    return torch.cuda.current_stream().cuda_stream


def bits(x):
    return x.contiguous().view(torch.int32 if x.element_size() == 4 else torch.int16)


def ld4(n):
    return (n + 3) & ~3


def _stored(x):
    """fp32 (rows, cols) in storage with ld4(cols) and NaN padding columns."""
    out = torch.full((x.shape[0], ld4(x.shape[1])), NAN, device=DEV)
    out[:, :x.shape[1]] = x
    return out


# ---------------------------------------------------------------------------------------------- items
# dense: name, g, a (with the bias column), bias, gradient dtype, eigen epilogue, transposed-convolution taps
DENSE = [('resnet50_layer4_1x1', 2048, 512, 0, torch.bfloat16, 'dgda', 0),   # g > 1024: stage (4) is split
         ('neox_qkv', 2304, 769, 1, torch.float16, 'dgda', 0),               # split, odd a
         ('dense_dgda', 300, 577, 0, torch.float32, 'dgda', 0),              # unsplit, odd a: scalar last column
         ('dense_dadg', 300, 577, 0, torch.float32, 'dadg', 0),
         ('simt', 10, 21, 1, torch.bfloat16, 'dgda', 0),                     # SIMT engine + cudaMemcpy2DAsync
         ('conv_transpose', 96, 145, 1, torch.float16, 'dadg', 9)]           # (C_in = 16, g, 3 x 3) weight gradient
# diagonal kinds, all with n > 1024 (the plain product with Q^T is split): name, rows (V), n, bias, dtype
DIAG = [('embedding', 300, 1100, 0, torch.float32),
        ('diag_g', 400, 1030, 1, torch.bfloat16),
        ('tied', 300, 1100, 0, torch.float16)]
# entries of layers that other ranks write while this one preconditions: (rows, n), never in a call
FOREIGN = [(64, 100), (33, 7)]


def _build_items():
    from kfac_b200 import _cabi
    damping = float(torch.tensor(0.003, dtype=torch.float32))
    gen = torch.Generator(device=DEV).manual_seed(17)

    def randn(*shape):
        return torch.randn(*shape, device=DEV, generator=gen)

    def rand(*shape):
        return torch.rand(*shape, device=DEV, generator=gen)

    def basis(n):    # orthogonal eigenbasis and a spread of non-negative eigenvalues, fp32 as stored
        q, _ = torch.linalg.qr(torch.randn(n, n, dtype=torch.float64, device=DEV, generator=gen))
        return q.float(), (torch.rand(n, dtype=torch.float64, device=DEV, generator=gen) ** 4).float()

    def inverse(q, d):   # exactly symmetric fp32 damped inverse
        x = (q.double() / (d.double() + damping)) @ q.double().t()
        return ((x + x.t()) / 2).float()

    items = []
    for name, g, a, bias, dtype, epi, taps in DENSE:
        qa, da = basis(a)
        qg, dg = basis(g)
        aw = a - bias
        w = (randn(aw // taps, g, taps) if taps else randn(g, aw)).to(dtype)
        b = randn(g).to(dtype) if bias else None
        wm = w.double().permute(1, 0, 2).reshape(g, aw) if taps else w.double()
        grad = torch.cat([wm, b.double()[:, None]], 1) if bias else wm
        dgda = (1.0 / (dg.double()[:, None] * da.double()[None, :] + damping)).float()
        a_inv, g_inv = inverse(qa, da), inverse(qg, dg)
        qa64, qg64 = qa.double(), qg.double()
        mid = qg64.t() @ grad @ qa64
        mid = mid * dgda.double() if epi == 'dgda' else mid / (dg.double()[:, None] * da.double()[None, :] + damping)
        items.append(dict(name=name, kind=_cabi.KFAC_ITEM_DENSE, rows=g, n=a, g=g, a=a, dtype=dtype, w=w, b=b, taps=taps,
                          epi=epi, qa=_stored(qa), qaT=_stored(qa.t()), qg=_stored(qg), qgT=_stored(qg.t()),
                          dgda=_stored(dgda), da=da, dg=dg, a_inv=_stored(a_inv), g_inv=_stored(g_inv),
                          ref_e=qg64 @ mid @ qa64.t(), ref_i=g_inv.double() @ grad @ a_inv.double()))
    for name, V, n, bias, dtype in DIAG:
        q, ev = basis(n)
        w = randn(V, n - bias).to(dtype)
        b = randn(V).to(dtype) if bias else None
        grad = torch.cat([w.double(), b.double()[:, None]], 1) if bias else w.double()
        q64 = q.double()
        if name == 'tied':
            # M = Q diag(s) is not orthogonal, like the simultaneous diagonaliser; mu > 0, f with absent tokens
            s = 0.5 + 1.5 * rand(n)
            M = (q64 * s.double()).float()
            f = rand(V) ** 4
            f[::7] = 0
            h = rand(V) * 1e-2
            t = float(torch.tensor(3e-3, dtype=torch.float32))
            mu = 0.1 + rand(n)
            M64 = M.double()
            den = (f.double()[:, None] + t) + (h.double()[:, None] + t) * mu.double()[None, :]
            ref = ((grad @ M64) / den) @ M64.t()
            items.append(dict(name=name, kind=_cabi.KFAC_ITEM_TIED, rows=V, n=n, g=n, a=V, dtype=dtype, w=w, b=None,
                              taps=0, qg=_stored(M), qgT=_stored(M.t()), da=f, dg=mu, dh=h, t=t, ref_e=ref, ref_i=ref))
            continue
        vrow = rand(V) * 1e-3 if name == 'embedding' else rand(V) ** 2 * 1e-2
        vrow[::7] = 0
        inv = inverse(q, ev)
        ref_e = ((grad @ q64) / (vrow.double()[:, None] * ev.double()[None, :] + damping)) @ q64.t()
        ref_i = (grad / (vrow.double()[:, None] + damping)) @ inv.double()
        if name == 'embedding':      # g = d, a = V; da is the diagonal A factor, dg the eigenvalues of G
            items.append(dict(name=name, kind=_cabi.KFAC_ITEM_EMBEDDING, rows=V, n=n, g=n, a=V, dtype=dtype, w=w,
                              b=None, taps=0, qg=_stored(q), qgT=_stored(q.t()), da=vrow, dg=ev, g_inv=_stored(inv),
                              ref_e=ref_e, ref_i=ref_i))
        else:                        # g = V, a = n; dg is the diagonal G factor, da the eigenvalues of A
            items.append(dict(name=name, kind=_cabi.KFAC_ITEM_DIAG_G, rows=V, n=n, g=V, a=n, dtype=dtype, w=w, b=b,
                              taps=0, qa=_stored(q), qaT=_stored(q.t()), da=ev, dg=vrow, a_inv=_stored(inv),
                              ref_e=ref_e, ref_i=ref_i))
    return damping, items


@pytest.fixture(scope='module')
def data():
    return _build_items()


def _layout(shapes):
    """Float offsets of entries of (rows, n) laid out one after another at rows x ld4(n) floats, and the total."""
    offs, off = [], 0
    for rows, n in shapes:
        offs.append(off)
        off += rows * ld4(n)
    return offs, off


class Arenas:
    """Arena 0 is the local P arena, arenas 1..7 the receivers'.  The layers of `items` in order with the foreign
    entries in between and at the end; GUARD floats before and after every arena; everything NaN."""

    def __init__(self, items, count=1 + MAX_PEERS):
        shapes = [(l['rows'], l['n']) for l in items]
        self.shapes = shapes[:3] + [FOREIGN[0]] + shapes[3:] + [FOREIGN[1]]
        self.slot = list(range(3)) + list(range(4, len(items) + 1))      # arena entry of item i
        self.foreign = [3, len(self.shapes) - 1]
        self.offs, self.total = _layout(self.shapes)
        self.bufs = [torch.full((GUARD + self.total + GUARD,), NAN, device=DEV) for _ in range(count)]

    def entry(self, k, i):
        """(rows, ld4(n)) view of arena k's entry of item i."""
        return self.raw(k, self.slot[i])

    def raw(self, k, j):
        rows, n = self.shapes[j]
        o = GUARD + self.offs[j]
        return self.bufs[k][o:o + rows * ld4(n)].view(rows, ld4(n))

    def guards(self, k):
        return torch.cat([self.bufs[k][:GUARD], self.bufs[k][GUARD + self.total:]])

    def snapshot(self):
        return [bits(b).clone() for b in self.bufs]


def _precond_item(l, method, P, peers):
    """kfac_precond_item of layer l into P (a device pointer) and the peer pointers (a ctypes array or None)."""
    from kfac_b200 import _cabi
    e = method == _cabi.KFAC_EIGEN
    p = lambda k, use=True: l[k].data_ptr() if use else None  # noqa: E731
    it = _cabi.PrecondItem()
    it.wgrad, it.bgrad, it.grad_dtype = l['w'].data_ptr(), p('b') if l['b'] is not None else None, _cabi.DTYPE_CODE[l['dtype']]
    it.g, it.a, it.kind, it.wgrad_taps = l['g'], l['a'], l['kind'], l['taps']
    it.P, it.ldp = P, ld4(l['n'])
    if l['kind'] == _cabi.KFAC_ITEM_DENSE:
        it.qa, it.qaT, it.qg, it.qgT = p('qa', e), p('qaT', e), p('qg', e), p('qgT', e)
        it.dgda = p('dgda', e and l['epi'] == 'dgda')
        it.da, it.dg = p('da', e and l['epi'] == 'dadg'), p('dg', e and l['epi'] == 'dadg')
        it.a_inv, it.g_inv = p('a_inv', not e), p('g_inv', not e)
        it.ldqa, it.ldqg, it.ld_dgda = ld4(l['a']), ld4(l['g']), ld4(l['a'])
    elif l['kind'] == _cabi.KFAC_ITEM_EMBEDDING:
        it.qg, it.qgT, it.dg, it.g_inv = p('qg', e), p('qgT', e), p('dg', e), p('g_inv', not e)
        it.da, it.ldqg = p('da'), ld4(l['n'])
    elif l['kind'] == _cabi.KFAC_ITEM_DIAG_G:
        it.qa, it.qaT, it.da, it.a_inv = p('qa', e), p('qaT', e), p('da', e), p('a_inv', not e)
        it.dg, it.ldqa = p('dg'), ld4(l['n'])
    else:
        it.qg, it.qgT, it.da, it.dg, it.dh = p('qg'), p('qgT'), p('da'), p('dg'), p('dh')
        it.ldqg, it.tied_damping = ld4(l['n']), l['t']
    if peers is not None:
        it.peer_P = C.cast(peers, C.POINTER(C.c_void_p))
    it.n_peers = len(peers) if peers is not None else 0
    return it


def _precondition(lib, damping, items, arenas, method, n_peers, override=None):
    """One kfac_precondition over `items` into arena 0 with arenas 1..n_peers as the peers, the workspace all-ones
    bytes.  override(arr, keep) may change the item table before the call.  Returns (status, workspace bytes)."""
    from kfac_b200 import _cabi
    arr = (_cabi.PrecondItem * len(items))()
    keep = []
    for i, l in enumerate(items):
        peers = None
        if n_peers:
            peers = (C.c_void_p * n_peers)(*[arenas.entry(q, i).data_ptr() for q in range(1, n_peers + 1)])
            keep.append(peers)
        arr[i] = _precond_item(l, method, arenas.entry(0, i).data_ptr(), peers)
    if override is not None:
        override(arr, keep)
    need = lib.kfac_precondition_workspace_bytes(arr, len(items))
    ws = torch.full((need,), 255, dtype=torch.uint8, device=DEV)
    rc = lib.kfac_precondition(arr, len(items), method, damping, ws.data_ptr(), need, S())
    torch.cuda.synchronize()
    return rc, need


METHODS = [1, 2]      # KFAC_EIGEN, KFAC_INVERSE


def _nan_bits():
    """Bit pattern of the NaN the arenas are filled with: an untouched float."""
    return int(torch.tensor([NAN]).view(torch.int32).item())


# ---------------------------------------------------------------------------------------------- tests
@pytest.mark.parametrize('method', METHODS, ids=['eigen', 'inverse'])
def test_fused_p_matches_fp64_and_peers(lib, data, method):
    damping, items = data
    key = 'ref_e' if method == 1 else 'ref_i'
    nan_bits = _nan_bits()
    for n_peers in (1, 3, MAX_PEERS):
        ar = Arenas(items)
        rc, _ = _precondition(lib, damping, items, ar, method, n_peers)
        assert rc == 0, lib.kfac_last_error()
        for i, l in enumerate(items):
            n = l['n']
            P = ar.entry(0, i)
            err = rel_fro(P[:, :n], l[key])
            print(f"{l['name']} method={method} peers={n_peers}: rel-fro {err:.2e}")
            assert err < 1e-4, (l['name'], method, n_peers, err)
            for q in range(1, n_peers + 1):
                peer = ar.entry(q, i)
                assert torch.equal(bits(peer[:, :n]), bits(P[:, :n])), (l['name'], method, n_peers, q)
                pad_p, pad_q = bits(P[:, n:]), bits(peer[:, n:])
                assert bool(((pad_q == pad_p) | (pad_q == nan_bits)).all()), (l['name'], method, n_peers, q)
        for q in range(1 + MAX_PEERS):       # the arenas of receivers that are not in the call are not touched
            assert bool((bits(ar.guards(q)) == nan_bits).all()), (method, n_peers, q)
            for j in ar.foreign:
                assert bool((bits(ar.raw(q, j)) == nan_bits).all()), (method, n_peers, q, j)
            if q > n_peers:
                assert bool((bits(ar.bufs[q]) == nan_bits).all()), (method, n_peers, q)


@pytest.mark.parametrize('method', METHODS, ids=['eigen', 'inverse'])
def test_p_does_not_depend_on_peers(lib, data, method):
    """The split of the long products (g > 1024, n > 1024) is the same with and without peers, so a layer's P has the
    same bits on every gradient worker, whether its receiver group broadcasts by peer stores or by NCCL."""
    damping, items = data
    base, need0 = None, None
    differ, sizes = [], []
    for n_peers in (0, 1, 3, MAX_PEERS):
        ar = Arenas(items, count=1 + n_peers)
        rc, need = _precondition(lib, damping, items, ar, method, n_peers)
        assert rc == 0, lib.kfac_last_error()
        Ps = [ar.entry(0, i)[:, :l['n']] for i, l in enumerate(items)]
        sizes.append((n_peers, need))
        if base is None:
            base, need0 = Ps, need
            continue
        differ += [(l['name'], n_peers) for l, p, b in zip(items, Ps, base) if not torch.equal(bits(p), bits(b))]
    assert not differ and all(need == need0 for _, need in sizes), \
        f'P differs from the call without peers: {differ}; workspace bytes per n_peers: {sizes}'


def test_fused_repeat_calls(lib, data):
    damping, items = data
    for method in METHODS:
        ar = Arenas(items)
        assert _precondition(lib, damping, items, ar, method, MAX_PEERS)[0] == 0, lib.kfac_last_error()
        first = ar.snapshot()
        assert _precondition(lib, damping, items, ar, method, MAX_PEERS)[0] == 0, lib.kfac_last_error()
        for q, (a, b) in enumerate(zip(first, ar.snapshot())):
            assert torch.equal(a, b), (method, q)


def test_receiver_grad_scale_and_update(lib, data):
    """A receiver runs the kl-clip scale and the write-back on its own arena, which the worker's peer stores filled:
    it must get the scale and the gradients the worker gets from its local P, bit for bit."""
    from kfac_b200 import _cabi
    damping, items = data
    ar = Arenas(items, count=4)
    assert _precondition(lib, damping, items, ar, _cabi.KFAC_EIGEN, 3)[0] == 0, lib.kfac_last_error()

    def scale_and_update(k):
        grads = [(l['w'].clone(), l['b'].clone() if l['b'] is not None else None) for l in items]
        gi = (_cabi.GradItem * len(items))()
        for i, (l, (w, b)) in enumerate(zip(items, grads)):
            gi[i] = _cabi.GradItem(ar.entry(k, i).data_ptr(), w.data_ptr(), b.data_ptr() if b is not None else None,
                                   _cabi.DTYPE_CODE[l['dtype']], l['rows'], l['n'], ld4(l['n']), l['taps'])
        need = lib.kfac_grad_workspace_bytes(len(items))
        ws = torch.full((need,), 255, dtype=torch.uint8, device=DEV)
        nu = torch.zeros(1, device=DEV)
        assert lib.kfac_grad_scale(gi, len(items), 1e-6, 0.1, ws.data_ptr(), need, nu.data_ptr(), S()) == 0
        assert lib.kfac_grad_update(gi, len(items), nu.data_ptr(), ws.data_ptr(), need, S()) == 0
        torch.cuda.synchronize()
        return nu, grads

    nu0, g0 = scale_and_update(0)
    assert 0.0 < float(nu0) < 1.0, float(nu0)
    for k in (1, 3):
        nu, g = scale_and_update(k)
        assert torch.equal(bits(nu), bits(nu0)), k
        for l, (w, b), (w0, b0) in zip(items, g, g0):
            assert torch.equal(bits(w), bits(w0)), (l['name'], k)
            if b is not None:
                assert torch.equal(bits(b), bits(b0)), (l['name'], k)


def test_bad_peer_args_have_no_side_effects(lib, data):
    """More than 7 peers, a negative count and a missing peer array are refused before anything runs: P and every
    peer arena keep their bits, also for the valid items before the bad one."""
    from kfac_b200 import _cabi
    damping, items = data
    ar = Arenas(items)
    assert _precondition(lib, damping, items, ar, _cabi.KFAC_EIGEN, MAX_PEERS)[0] == 0, lib.kfac_last_error()
    before = ar.snapshot()
    last = len(items) - 1

    def eight(arr, keep):      # eight valid pointers: the seven peers' entries and the local one
        p = (C.c_void_p * 8)(*[ar.entry(q, last).data_ptr() for q in range(1, 1 + MAX_PEERS)],
                             ar.entry(0, last).data_ptr())
        keep.append(p)
        arr[last].peer_P, arr[last].n_peers = C.cast(p, C.POINTER(C.c_void_p)), 8

    def negative(arr, keep):
        arr[last].n_peers = -1

    def null(arr, keep):
        arr[last].peer_P, arr[last].n_peers = None, 1

    for case in (eight, negative, null):
        for method in METHODS:
            rc, _ = _precondition(lib, damping, items, ar, method, MAX_PEERS, override=case)
            assert rc == _cabi.KFAC_ERR_BAD_ARG, (case.__name__, method, rc)
            for q, (a, b) in enumerate(zip(before, ar.snapshot())):
                assert torch.equal(a, b), (case.__name__, method, q)


# ---------------------------------------------------------------------------------------------- CUDA IPC
IPC_ITEMS = ('resnet50_layer4_1x1', 'dense_dgda', 'simt')     # split, unsplit with a scalar column, SIMT copies


def _ipc_child(conn, nbytes):
    """The receiver: exports a zeroed arena, then compares it with the bytes the worker stored into it."""
    from kfac_b200 import _cabi
    lib = _cabi.load()
    ptr, handle = C.c_void_p(), (C.c_ubyte * 64)()
    try:
        if lib.kfac_peer_alloc(nbytes, C.byref(ptr), handle) != 0:
            conn.send(('error', 'kfac_peer_alloc: ' + _cabi.last_error()))
            return

        class _Raw:
            pass
        raw = _Raw()
        raw.__cuda_array_interface__ = {'shape': (nbytes,), 'typestr': '|u1', 'data': (ptr.value, False),
                                        'version': 3, 'strides': None}
        arena = torch.as_tensor(raw, device='cuda')
        torch.cuda.synchronize()
        zero = not bool(arena.any())
        conn.send(('handle', bytes(handle), zero))
        want = conn.recv_bytes()
        torch.cuda.synchronize()
        got = arena.cpu().numpy().tobytes()
        ok = zero and got == want
        bad = sum(1 for x, y in zip(got, want) if x != y) if got != want else 0
        conn.send(('result', ok, bad))
    finally:
        if ptr.value:
            lib.kfac_peer_free(ptr)
        conn.close()


def _compute_mode_is_default():
    """Reads (never changes) the compute mode of the current device: a second process needs the default mode."""
    try:
        cu = C.CDLL('libcuda.so.1')
    except OSError:
        return False
    dev, mode = C.c_int(), C.c_int()
    if cu.cuDeviceGet(C.byref(dev), torch.cuda.current_device()) != 0:
        return False
    if cu.cuDeviceGetAttribute(C.byref(mode), 20, dev) != 0:      # CU_DEVICE_ATTRIBUTE_COMPUTE_MODE
        return False
    return mode.value == 0                                        # CU_COMPUTEMODE_DEFAULT


def test_peer_memory_across_processes(lib, data):
    from kfac_b200 import _cabi
    torch.cuda.init()
    if not _compute_mode_is_default():
        pytest.skip('the device is not in the default compute mode: a second process cannot share it')
    damping, all_items = data
    items = [l for l in all_items if l['name'] in IPC_ITEMS]
    ar = Arenas(items, count=1)
    nbytes = ar.total * 4
    ctx = mp.get_context('spawn')
    parent, child = ctx.Pipe()
    proc = ctx.Process(target=_ipc_child, args=(child, nbytes), daemon=True)
    proc.start()
    child.close()
    mapped = C.c_void_p()
    try:
        assert parent.poll(120), 'the child did not export its arena'
        msg = parent.recv()
        assert msg[0] == 'handle', msg
        assert msg[2], 'kfac_peer_alloc did not zero the arena'
        h = (C.c_ubyte * 64).from_buffer_copy(msg[1])
        assert lib.kfac_peer_open(h, C.byref(mapped)) == 0, lib.kfac_last_error()

        def into_child(arr, keep):
            for i in range(len(items)):
                p = (C.c_void_p * 1)(mapped.value + ar.offs[ar.slot[i]] * 4)
                keep.append(p)
                arr[i].peer_P, arr[i].n_peers = C.cast(p, C.POINTER(C.c_void_p)), 1

        rc, _ = _precondition(lib, damping, items, ar, _cabi.KFAC_EIGEN, 0, override=into_child)
        assert rc == 0, lib.kfac_last_error()
        assert lib.kfac_peer_close(mapped) == 0, lib.kfac_last_error()
        mapped = C.c_void_p()
        # the child's arena: P in columns [0, n) of the call's entries, zeros everywhere else (a split product stores
        # its zero padding to the peers, an unsplit one leaves the padding as it was)
        want = torch.zeros(ar.total, device=DEV)
        for i, l in enumerate(items):
            n, (rows, _), o = l['n'], ar.shapes[ar.slot[i]], ar.offs[ar.slot[i]]
            want[o:o + rows * ld4(n)].view(rows, ld4(n))[:, :n] = ar.entry(0, i)[:, :n]
            assert rel_fro(ar.entry(0, i)[:, :n], l['ref_e']) < 1e-4, l['name']
        parent.send_bytes(want.cpu().numpy().tobytes())
        assert parent.poll(120), 'the child did not answer'
        msg = parent.recv()
        assert msg[0] == 'result' and msg[1], f'the child found {msg[2]} bytes that differ from P'
    finally:
        if mapped.value:
            lib.kfac_peer_close(mapped)
        proc.join(60)
        if proc.is_alive():
            proc.kill()
            proc.join()
    assert proc.exitcode == 0, proc.exitcode
