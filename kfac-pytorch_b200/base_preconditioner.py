"""Step orchestrator of the H100-native K-FAC preconditioner.

Mirrors `BaseKFACPreconditioner` (kfac/base_preconditioner.py:22-479): same
constructor keywords, properties, hooks, `step()`, `state_dict()`,
`load_state_dict()`, `reset_batch()`, `memory_usage()` and `__repr__`, and the
same externally visible schedule (`steps % factor_update_steps`,
`steps % inv_update_steps`, micro-batch accumulation).

What is different underneath (H100-first):
  * all per-layer tensors are views into a few contiguous HBM arenas
    (factors | micro-batch sums | second-order data | preconditioned grads);
  * every phase of `step()` is ONE call into libkfac_b200.so over all layers
    (no per-layer Python arithmetic, no `.item()` host syncs: the kl-clip
    scale stays on the device);
  * each communication phase is one collective per (source, group) on an
    arena slice instead of 1-3 collectives per layer.

Mixed precision with a loss scale (`grad_scaler=`): every factor update then
runs through the guarded EMA, which drops a window whose statistics are not
finite (an fp16 overflow step) instead of carrying it into the running factor.
With a `torch.amp.GradScaler` the scale is never read on the host: each G hook
copies the scaler's current scale into a per-layer device slot, the G
statistics are formed unscaled, and the EMA multiplies the window by 1/s^2
from that slot.  This relies on the order of the usual AMP loop:

    scaler.scale(loss).backward()   # G hooks snapshot the scale
    scaler.unscale_(optimizer)
    preconditioner.step()           # every closed window is consumed here
    scaler.step(optimizer)
    scaler.update()                 # the scale changes only here

so all micro-batches of a window share one scale.  A window that stays open
across step() (step() called before `accumulation_steps` micro-batches have
run) can span an update() and so two scales; the last snapshot is applied to
the whole window.  Under data parallelism every rank must use the same scale,
as GradScaler does when it unscales gradients that DDP has already averaged.

EKFAC (`compute_method='ekfac'`): the hooks also keep the rows of the window
(sample-major fp32 row buffers, one forward and one backward per window), and
step() measures their second moments S_batch in the eigenbasis, after the
factor EMA and after the eigendecompositions of an inverse step:
    factor step, no new basis     S <- factor_decay * S + (1 - factor_decay) * S_batch
    factor step, new basis        S <- S_batch
    new basis without a window    S <- dg x da       (also after load_state_dict)
    every step                    dgda <- 1 / (S + damping)
and the eigen precondition runs with that dgda.  S is not part of state_dict().

Normalization layers (`norm_layers`, precondition_norms): their C x k Fisher blocks live at the end of the G block
of the factor and batch arenas (they are complete only after backward; the A block and its overlapped all-reduce are
those of the other layers) and take the vector EMA, guarded under a loss scale.  A tensor hook on each call's output,
registered by a forward hook at factor steps, pairs the gradient with that call's input.  The blocks are snapshotted
at inverse steps and every rank preconditions its normalization layers locally at every step, outside the work
assignment and its broadcasts; kl-clip and the write-back run over all layers.
"""
from __future__ import annotations

import ctypes as C
import logging
import math
import warnings
from collections import defaultdict
from typing import Any, Callable, NamedTuple

import torch

from kfac_b200 import _cabi
from kfac_b200.assignment import WorkAssignment
from kfac_b200.distributed import ArenaCommunicator, get_rank
from kfac_b200.enums import ComputeMethod
from kfac_b200.layers import AttentionProjectionHelper, KFACLayer, RecurrentSubLayerHelper, cast_for_factor

logger = logging.getLogger(__name__)


class _Scratch:
    """Grow-only device scratch buffer (im2col / eigensolver / GEMM workspaces)."""

    def __init__(self) -> None:
        self.buf: torch.Tensor | None = None

    def get(self, nbytes: int, device: torch.device) -> torch.Tensor | None:
        if nbytes <= 0:
            return None
        if self.buf is None or self.buf.numel() < nbytes or self.buf.device != device:
            self.buf = torch.empty(int(nbytes), dtype=torch.uint8, device=device)
        return self.buf


def _storage_numel(shape: tuple[int, ...]) -> int:
    """Floats reserved for one arena entry; always a multiple of 4 so that every
    entry starts 16-byte aligned (TMA / wgmma GEMM operands)."""
    if len(shape) == 2:
        return shape[0] * _cabi.ld4(shape[1])
    return _cabi.ld4(shape[0])


def _bind(arena: torch.Tensor, off: int, shape: tuple[int, ...]) -> torch.Tensor:
    """Storage tensor of one arena entry: (rows, ld4(cols)) or (n,)."""
    n = _storage_numel(shape)
    t = arena.narrow(0, off, n)
    return t.view(shape[0], _cabi.ld4(shape[1])) if len(shape) == 2 else t.narrow(0, 0, shape[0])


class _Segment:
    """Contiguous arena slice moved by one broadcast: (group, src) -> tensors."""

    def __init__(self, src: int, group: Any) -> None:
        self.src = src
        self.group = group
        self.entries: list[tuple[KFACLayer, str, tuple[int, ...]]] = []
        self.offset = 0
        self.numel = 0

    def add(self, layer: KFACLayer, key: str, shape: tuple[int, ...]) -> None:
        """shape = logical shape; matrices are stored with a leading dimension
        padded to a multiple of 4 floats (TMA-addressable rows)."""
        self.entries.append((layer, key, shape))
        self.numel += _storage_numel(shape)


class Entry(NamedTuple):
    """One second-order tensor of a layer, `layer._inv[key]`.  holder: 'A' / 'G' (that factor's inverse worker),
    'grad' (every gradient worker of the layer) or 'all' (every rank).  A shipped entry is broadcast from its holder
    to the layer's gradient-worker group; a receiver builds the K-major copy `kmajor` of it, if any."""
    key: str
    shape: tuple[int, ...]
    holder: str
    shipped: bool = False
    kmajor: str | None = None


class Layout(NamedTuple):
    """What the preconditioner stores, computes and reads for one layer's second-order data (second_order_layout).
    A holder is 'A' or 'G', a side 'a' or 'g'."""
    entries: tuple[Entry, ...]
    factors: tuple[tuple[str, tuple[tuple[KFACLayer, str], ...], str], ...]  # holder, (layer, side) read, error if unset
    snapshots: tuple[tuple[str, KFACLayer, str, str], ...]     # holder, layer and side of a vector factor, key
    decompositions: tuple[tuple[str, int, str, str | None, str], ...]  # side, eigensolver call, keys of Q, Q^T, eigenvalues
    post: tuple[tuple[str, str, tuple[str, ...]], ...]         # holder, op ('dgda', 'inverse', 'tied'), keys it uses
    needs: frozenset[str]            # keys the precondition checks are ready
    unready: str                     # ... and its error when one is not
    fields: tuple[tuple[str, str], ...]  # PrecondItem pointer field, key
    item: dict[str, int]             # the item's kind and leading dimensions
    eigen: bool                      # the item takes the eigen path of kfac_precondition
    damped: bool = False             # the item carries the damping its data was formed with


def second_order_layout(layer: KFACLayer) -> Layout:
    """The one declaration of a layer's second-order data; the comm plan, the local arena, the inverse step and the
    precondition items all follow from it.  Not defined for the head of a tied pair: its embedding carries the pair.

    Eigensolver call 0 takes the dense layers' factors, call 1 the dense factors of diagonal layers and tied pairs,
    so that the dense layers get the same schedule (and bits) with or without those.  The precondition runs on every
    gradient worker and reads what they all hold: the shipped entries and those held by 'grad' or 'all'."""
    a, g = layer.a_dim, layer.g_dim
    E, ld4 = Entry, _cabi.ld4
    head = layer.tied_head
    if head is not None:
        # M (built K-major by every receiver), mu and the snapshots f and h, formed on the rank that holds all four
        # factors with Q_E, e, C (dense, ld = d, the layout the eigensolver reads) and the eigenvectors U of C
        needs = ('tq', '_tqT', 'tmu', 'da', 'dh')
        return Layout(
            (E('tq', (g, g), 'G', True, '_tqT'), E('tmu', (g,), 'G', True), E('da', (a,), 'G', True),
             E('dh', (a,), 'G', True), E('_tqT', (g, g), 'grad'), E('_qg', (g, g), 'G'), E('_qgT', (g, g), 'G'),
             E('_dg', (g,), 'G'), E('_C', (g * g,), 'G'), E('_U', (g, g), 'G'), E('_UT', (g, g), 'G')),
            (('G', ((layer, 'a'), (layer, 'g'), (head, 'a'), (head, 'g')),
              'Cannot decompose the factors of a tied embedding / head pair before they have been computed'),),
            (('G', layer, 'a', 'da'), ('G', head, 'g', 'dh')),
            (('g', 1, '_qg', '_qgT', '_dg'),),
            (('G', 'tied', ('_qg', '_qgT', '_dg', '_C', '_U', '_UT', 'tq', '_tqT', 'tmu')),),
            frozenset(needs), 'The second-order data of the tied embedding / head pair has not been computed',
            tuple(zip(('qg', 'qgT', 'dg', 'da', 'dh'), needs)),
            dict(kind=_cabi.KFAC_ITEM_TIED, ldqa=0, ldqg=ld4(g), ld_dgda=0), eigen=False, damped=True)
    factors = tuple((s.upper(), ((layer, s),), f'Cannot eigendecompose {s.upper()} before {s.upper()} has been computed')
                    for s in 'ag')
    snapshots, post = (), ()
    if layer.diag_side:
        # embedding or diagonal-A layer (d = 'a') or diagonal-G layer (d = 'g'): the diagonal factor is its own
        # eigendecomposition and ships as a snapshot; only the dense factor f is decomposed, and there is never a
        # V x d dgda
        d, f = layer.diag_side, layer.dense_side
        D, F, n, nd = d.upper(), f.upper(), (a if f == 'a' else g), (a if d == 'a' else g)
        snapshots = ((D, layer, d, 'd' + d),)
        if layer.method == ComputeMethod.EIGEN:
            entries = (E('d' + d, (nd,), D, True), E('q' + f, (n, n), F, True, f'_q{f}T'), E('d' + f, (n,), F, True),
                       E(f'_q{f}T', (n, n), 'grad'))
            decompositions = ((f, 1, 'q' + f, f'_q{f}T', 'd' + f),)
            needs = {'d' + d, 'q' + f, 'd' + f}
        else:
            entries = (E('d' + d, (nd,), D, True), E(f + '_inv', (n, n), F, True), E('_q' + f, (n, n), F),
                       E('_d' + f, (n,), F))
            decompositions = ((f, 1, '_q' + f, None, '_d' + f),)
            post = ((F, 'inverse', ('_q' + f, '_d' + f, f + '_inv')),)
            needs = {'d' + d, f + '_inv'}
        kind, what = ((_cabi.KFAC_ITEM_EMBEDDING, 'embedding') if layer.embedding
                      else (_cabi.KFAC_ITEM_DIAG_A, 'diagonal-A layer') if d == 'a'
                      else (_cabi.KFAC_ITEM_DIAG_G, 'diagonal-G layer'))
        unready = f'The second-order data of the {what} has not been computed'
        item = dict(kind=kind,
                    ldqa=ld4(n) if f == 'a' else 0, ldqg=ld4(n) if f == 'g' else 0, ld_dgda=0)
        eigen = layer.method == ComputeMethod.EIGEN
    else:
        eigen = layer.method in (ComputeMethod.EIGEN, ComputeMethod.EKFAC)
        unready = 'Eigendecompositions for both A and G have not been computed'
        if layer.method == ComputeMethod.EIGEN and layer.prediv_eigenvalues:
            # A and G are colocated: their holder divides by the eigenvalue outer product before shipping
            entries = (E('qa', (a, a), 'G', True, '_qaT'), E('qg', (g, g), 'G', True, '_qgT'),
                       E('dgda', (g, a), 'G', True), E('_qaT', (a, a), 'grad'), E('_qgT', (g, g), 'grad'),
                       E('_da', (a,), 'A'), E('_dg', (g,), 'G'))
            decompositions = (('a', 0, 'qa', '_qaT', '_da'), ('g', 0, 'qg', '_qgT', '_dg'))
            post = (('G', 'dgda', ('_dg', '_da', 'dgda')),)
            needs = {'qa', 'qg', 'dgda'}
        elif eigen:
            # EKFAC ships the eigenvalues too: every rank seeds S with dg x da for a basis no window has been measured
            # in, and forms its own dgda from S (_ekfac_update)
            ekfac = layer.method == ComputeMethod.EKFAC
            kT = 'all' if ekfac else 'grad'
            entries = (E('qa', (a, a), 'A', True, '_qaT'), E('da', (a,), 'A', True),
                       E('qg', (g, g), 'G', True, '_qgT'), E('dg', (g,), 'G', True),
                       E('_qaT', (a, a), kT), E('_qgT', (g, g), kT)) + ((E('dgda', (g, a), 'all'),) if ekfac else ())
            decompositions = (('a', 0, 'qa', '_qaT', 'da'), ('g', 0, 'qg', '_qgT', 'dg'))
            needs = {'qa', 'qg', 'dgda'} if ekfac else {'qa', 'qg', 'da', 'dg'}
        else:
            entries = (E('a_inv', (a, a), 'A', True), E('g_inv', (g, g), 'G', True), E('_qa', (a, a), 'A'),
                       E('_da', (a,), 'A'), E('_qg', (g, g), 'G'), E('_dg', (g,), 'G'))
            decompositions = (('a', 0, '_qa', None, '_da'), ('g', 0, '_qg', None, '_dg'))
            post = (('A', 'inverse', ('_qa', '_da', 'a_inv')), ('G', 'inverse', ('_qg', '_dg', 'g_inv')))
            needs = {'a_inv', 'g_inv'}
            unready = 'Cannot precondition gradient before A and G have been inverted'
        item = dict(kind=_cabi.KFAC_ITEM_DENSE, ldqa=ld4(a), ldqg=ld4(g), ld_dgda=ld4(a))
        if layer.module.wgrad_taps:     # a transposed convolution's (C_in, g, T) weight gradient
            item['wgrad_taps'] = layer.module.wgrad_taps
    if layer.pi_damping:
        # pi-adjusted damping: every rank forms pi of every layer from the all-reduced factors at each inverse step;
        # the damped dgda and inverses read it, and so does the precondition
        entries += (E('pi', (1,), 'all'),)
        needs = set(needs) | {'pi'}
        post = tuple((holder, op, keys + ('pi',)) for holder, op, keys in post)
    fields = tuple((e.key.lstrip('_'), e.key) for e in entries if e.shipped or e.holder in ('grad', 'all'))
    return Layout(entries, factors, snapshots, decompositions, post, frozenset(needs), unready, fields, item, eigen)


def pi_s(damping: float) -> float:
    """s = sqrt(damping) of pi-adjusted damping, as kfac_precondition forms it: the fp32 square root of the fp32 damping
    (the square root in fp64 of a float, rounded to a float, is the correctly rounded fp32 square root)."""
    return C.c_float(math.sqrt(C.c_float(damping).value)).value


def _holds(holder: str, name: str, assignment: WorkAssignment, rank: int) -> bool:
    if holder == 'all':
        return True
    if holder == 'grad':
        return assignment.is_grad_worker(name)
    return rank == assignment.inv_worker(name, holder)


def build_comm_plan(layers: list[tuple[str, KFACLayer]], assignment: WorkAssignment):
    """Decide which second-order tensors this rank stores and how they are
    grouped into broadcast segments.  Pure host logic (unit-tested on CPU for
    cross-rank consistency).

    Returns (inv_segments, grad_segments): ordered lists of _Segment.
    """
    inv: dict[tuple[int, int], _Segment] = {}
    # the head of a tied pair has no placement of its own: the embedding carries the pair
    layers = [(name, layer) for name, layer in layers if layer.tied_embedding is None]
    for name, layer in layers:
        if not assignment.is_grad_worker(name):
            continue
        group = assignment.grad_worker_group(name)
        for e in second_order_layout(layer).entries:
            if e.shipped:
                src = assignment.inv_worker(name, e.holder)
                key = (id(group) if group is not None else 0, src)
                if key not in inv:
                    inv[key] = _Segment(src, group)
                inv[key].add(layer, e.key, e.shape)
    grad: dict[int, _Segment] = {}
    for name, layer in layers:
        src = assignment.src_grad_worker(name)
        if src not in grad:
            grad[src] = _Segment(src, assignment.grad_receiver_group(name))
        grad[src].add(layer, 'P', layer.p_shape)
    inv_segments = list(inv.values())
    grad_segments = [grad[k] for k in sorted(grad)]
    for segs in (inv_segments, grad_segments):
        off = 0
        for s in segs:
            s.offset = off
            off += s.numel
    return inv_segments, grad_segments


def build_local_plan(layers: list[tuple[str, KFACLayer]], assignment: WorkAssignment, rank: int):
    """The second-order tensors `rank` keeps for itself (never communicated), in registration order: a list of
    (layer, key, shape)."""
    return [(layer, e.key, e.shape) for name, layer in layers if layer.tied_embedding is None
            for e in second_order_layout(layer).entries if not e.shipped and _holds(e.holder, name, assignment, rank)]


def build_inverse_plan(layers: list[tuple[str, KFACLayer]], assignment: WorkAssignment, rank: int):
    """The work of `rank` at an inverse step, in launch order, in reverse registration order and A before G within a
    layer: the snapshots of vector factors (layer, owner of the factor, its side, key), the matrices of the two
    eigensolver calls (layer, side, Q, Q^T, eigenvalues) and the post-ops (layer, op, keys).  Raises if a factor it
    reads has not been computed yet."""
    snapshots, calls, post = [], ([], []), []
    for name, layer in reversed(layers):
        if layer.tied_embedding is not None:
            continue
        lay = second_order_layout(layer)
        # the holders this rank is (a tied pair is placed by its G alone)
        mine = {h for h, _, _ in lay.factors if rank == assignment.inv_worker(name, h)}
        for holder, factors, error in lay.factors:
            if holder in mine and not all(src._has_a if side == 'a' else src._has_g for src, side in factors):
                raise RuntimeError(error)
        snapshots += [(layer, src, side, key) for holder, src, side, key in lay.snapshots if holder in mine]
        for side, call, q, qT, d in lay.decompositions:
            if side.upper() in mine:
                calls[call].append((layer, side, q, qT, d))
        post += [(layer, op, keys) for holder, op, keys in lay.post if holder in mine]
    return snapshots, calls, post


def _release_peer_memory(peer_bases: list[int], own_ptr: int) -> None:
    """Finalizer of the fused-broadcast arena: unmap the peers' arenas, free our own."""
    try:
        lib = _cabi.load()
        for b in peer_bases:
            lib.kfac_peer_close(C.c_void_p(b))
        lib.kfac_peer_free(C.c_void_p(own_ptr))
    except Exception:  # noqa: BLE001  (interpreter shutdown)
        pass


class BaseKFACPreconditioner:
    """K-FAC distributed gradient preconditioner (native sm_90a hot path)."""

    def __init__(
        self,
        layers: dict[torch.nn.Module, tuple[str, KFACLayer]],
        *,
        norm_layers: dict[torch.nn.Module, tuple[str, KFACLayer]] | None = None,
        assignment: WorkAssignment,
        tdc: ArenaCommunicator,
        factor_update_steps: Callable[[int], int] | int = 1,
        inv_update_steps: Callable[[int], int] | int = 1,
        damping: Callable[[int], float] | float = 0.001,
        factor_decay: Callable[[int], float] | float = 0.95,
        kl_clip: Callable[[int], float] | float = 0.001,
        lr: Callable[[int], float] | float = 0.1,
        accumulation_steps: int = 1,
        update_factors_in_hook: bool = True,
        defaults: dict[str, Any] | None = None,
        loglevel: int = logging.DEBUG,
    ) -> None:
        # validation: same messages / order as base_preconditioner.py:87-110
        if not callable(factor_update_steps) and not 0 < factor_update_steps:
            raise ValueError('factor_update_steps must be > 0')
        if not callable(inv_update_steps) and not 0 < inv_update_steps:
            raise ValueError('inv_update_steps must be > 0')
        if not callable(damping) and not 0.0 < damping:
            raise ValueError('damping must be > 0')
        if not callable(factor_decay) and not 0.0 < factor_decay <= 1:
            raise ValueError('factor_decay must be in (0, 1]')
        if not callable(kl_clip) and kl_clip is not None and not 0.0 < kl_clip:
            raise ValueError('kl_clip must be > 0')
        if not callable(lr) and not 0.0 <= lr:
            raise ValueError('lr be > 0')
        if not 0 < accumulation_steps:
            raise ValueError('accumulation_steps must be > 0')
        if (not callable(inv_update_steps) and not callable(factor_update_steps)
                and not 0 == inv_update_steps % factor_update_steps):
            warnings.warn('It is suggested that inv_update_steps be an integer multiple '
                          'of factor_update_steps', stacklevel=2)

        self._accumulation_steps = accumulation_steps
        self._assignment = assignment
        self._damping = damping
        self._defaults = defaults
        self._factor_decay = factor_decay
        self._factor_update_steps = factor_update_steps
        self._inv_update_steps = inv_update_steps
        self._kl_clip = kl_clip
        self._layers = layers
        # normalization layers (layer.norm): outside the work assignment, preconditioned locally on every rank
        self._norm_layers = norm_layers or {}
        self._loglevel = loglevel
        self._lr = lr
        self._tdc = tdc
        self._update_factors_in_hook = update_factors_in_hook
        self._steps = 0
        self._mini_steps: dict[str, int] = defaultdict(int)

        # native-side state
        self._arenas_ready = False
        self._device: torch.device | None = None
        self._scratch = _Scratch()          # im2col / transposes (forward hooks)
        self._scratch_bwd = _Scratch()      # transposes (backward hooks, autograd thread)
        self._eig_scratch = _Scratch()      # eigensolver workspace
        self._gemm_scratch = _Scratch()     # precondition / inverse temporaries
        self._grad_scratch = _Scratch()     # kl-clip / write-back item table + partial sums
        self._pending_alpha: dict[float, list[tuple[KFACLayer, str]]] = {}
        # with a loss scale every factor goes through the guarded EMA (non-finite windows are dropped and counted)
        self._guard_factors = any(l.grad_scaler is not None for _, l in self._all_layer_list())
        self._ema_scratch = _Scratch()        # drop flags of the guarded EMA
        self._skipped: torch.Tensor | None = None   # device counter of dropped windows
        self._ekfac_scratch = _Scratch()      # EKFAC projections + split partials, and the update's item table
        # C1: the batch statistics (not the factors) are averaged over the ranks BEFORE the EMA -- the same factors by
        # linearity -- so that the A block can be reduced while backward still runs (base_preconditioner.py:452-457)
        self.overlap_factor_allreduce = True
        self._a_reduce_work: Any = None        # in-flight asynchronous all-reduce of the A block
        self._a_block_reduced = False
        self._comm_stream: torch.cuda.Stream | None = None
        self.last_grad_scale: torch.Tensor | None = None   # device scalar nu of the last step
        # store preconditioned gradients straight into the receivers' arenas (P2P) instead of broadcasting
        self.fused_grad_broadcast = True
        self._eig_status: torch.Tensor | None = None     # pinned host int: status word of the last eigensolver call
        self._diag_status: torch.Tensor | None = None    # device int: status of the diagonal-factor snapshots
        self._norm_scratch = _Scratch()       # statistics of the normalization layers (autograd thread)
        self._norm_p_scratch = _Scratch()     # item table of their precondition

        # attention projections (precondition_attention): attention module -> {'q', 'k', 'v', 'o'} -> the helper that
        # keys the projection's layer; their statistics arrive through taps inside the attention's forward
        self._attention_taps: dict[torch.nn.Module, dict[str, AttentionProjectionHelper]] = {}
        # recurrent sub-layers (precondition_recurrent): RNN / LSTM / GRU module -> {'ih_l0', 'hh_l0_reverse', ...} ->
        # the helper that keys the sub-layer's layer; their statistics arrive through taps inside the module's forward
        self._recurrent_taps: dict[torch.nn.Module, dict[str, RecurrentSubLayerHelper]] = {}
        for module in self._norm_layers:
            module.register_forward_hook(self._hook_norm_output)
        for module, (_, layer) in self._layers.items():
            if isinstance(module, AttentionProjectionHelper):
                self._attention_taps.setdefault(module.attn, {})[module.which[0]] = module
                continue
            if isinstance(module, RecurrentSubLayerHelper):
                self._recurrent_taps.setdefault(module.rnn, {})[module.suffix] = module
                continue
            if layer.module.call_kwargs:
                module.register_forward_pre_hook(self._save_input_with_kwargs, with_kwargs=True)
            else:
                module.register_forward_pre_hook(self._save_input)
            if layer.embedding:
                # the input of an embedding (the indices) never requires grad: a full backward hook would fire through
                # the output with a warning on every backward pass, so the output tensor is hooked directly
                module.register_forward_hook(self._hook_output)
            else:
                module.register_full_backward_hook(self._save_grad_output)

    # ------------------------------------------------------------ properties
    def __repr__(self) -> str:
        params = [
            ('accumulation_steps', self._accumulation_steps),
            ('assignment', self._assignment.__class__.__name__),
            ('damping', self._damping),
            ('factor_decay', self._factor_decay),
            ('factor_update_steps', self._factor_update_steps),
            ('inv_update_steps', self._inv_update_steps),
            ('kl_clip', self._kl_clip),
            ('layers', len(self._layers)),
            ('loglevel', self._loglevel),
            ('lr', self._lr),
            ('steps', self.steps),
            ('update_factors_in_hook', self._update_factors_in_hook),
        ]
        if self._defaults is not None:
            params.extend(list(self._defaults.items()))
        body = '\n'.join(f'  {k}={v},' for k, v in sorted(params, key=lambda kv: kv[0]))
        return f'{self.__class__.__name__}(\n{body}\n)'

    def _value(self, v):
        return v(self.steps) if callable(v) else v

    damping = property(lambda self: self._value(self._damping))
    factor_decay = property(lambda self: self._value(self._factor_decay))
    kl_clip = property(lambda self: self._value(self._kl_clip))
    lr = property(lambda self: self._value(self._lr))
    factor_update_steps = property(lambda self: self._value(self._factor_update_steps))
    inv_update_steps = property(lambda self: self._value(self._inv_update_steps))

    @property
    def steps(self) -> int:
        return self._steps

    @property
    def skipped_factor_updates(self) -> int:
        """Number of factor windows dropped because their statistics were not finite (or exceeded 1e15 in
        magnitude): by the guarded EMA, only with a `grad_scaler`; with EKFAC also the windows whose factors were kept
        but whose S_batch was dropped (with or without a `grad_scaler`).  Reading it synchronises the device."""
        return int(self._skipped.item()) if self._skipped is not None else 0

    # ------------------------------------------------------------ arenas
    def _layer_list(self) -> list[tuple[str, KFACLayer]]:
        return list(self._layers.values())

    def _norm_list(self) -> list[tuple[str, KFACLayer]]:
        return list(self._norm_layers.values())

    def _all_layer_list(self) -> list[tuple[str, KFACLayer]]:
        """The layers of the work assignment, then the normalization layers."""
        return self._layer_list() + self._norm_list()

    def _ensure_arenas(self, device: torch.device | None = None) -> None:
        if self._arenas_ready:
            return
        if device is None:
            al = self._all_layer_list()
            device = al[0][1].module.device if al else torch.device('cuda')
        if device.type != 'cuda':
            raise _cabi.KFACNativeError(
                f'kfac_b200 needs the model on a CUDA (sm_90a) device, found {device}; '
                'there is no CPU fallback')
        _cabi.load()
        self._device = device
        ll = self._layer_list()
        # dense d x d factors (a vector of V floats for the diagonal A of an embedding or the diagonal G of a
        # diagonal-G layer), each starting 16-byte aligned
        nl = self._norm_list()
        total = sum(_cabi.ld4(math.prod(l.a_factor_shape)) + _cabi.ld4(math.prod(l.g_factor_shape)) for _, l in ll)
        total += sum(_cabi.ld4(math.prod(l.g_factor_shape)) for _, l in nl)
        self._factor_arena = torch.zeros(total, dtype=torch.float32, device=device)
        self._batch_arena = torch.zeros(total, dtype=torch.float32, device=device)
        # layout: all A factors, then all G factors -- the A block is complete after the forward pass and is
        # all-reduced on its own while backward produces the G statistics.  The blocks of the normalization layers
        # (no A factor) close the G block
        off = 0
        for which in ('a', 'g'):
            for _, l in ll + (nl if which == 'g' else []):
                shape = l.a_factor_shape if which == 'a' else l.g_factor_shape
                n = math.prod(shape)
                setattr(l, f'_{which}_view', self._factor_arena.narrow(0, off, n).view(shape))
                setattr(l, f'_{which}_batch_view', self._batch_arena.narrow(0, off, n).view(shape))
                off += _cabi.ld4(n)
            if which == 'a':
                self._a_block_numel = off
        # a normalization block is seeded with the identity (F_ss, F_sb, F_bb) = (1, 0, 1): its EMA runs with
        # first = 0 on this seed, which gives the bits of a first window on the identity, dropped windows included
        for _, l in nl:
            l._g_view[:, 0] = 1.0
            l._g_view[:, -1] = 1.0
        # snapshots (C x k, in layer._inv['dg']) and P (C x a_dim) of the normalization layers: local to every rank
        self._norm_arena = torch.zeros(max(1, sum(l.g_dim * (l.module.k + l.a_dim) for _, l in nl)),
                                       dtype=torch.float32, device=device)
        off = 0
        for _, l in nl:
            k, C = l.module.k, l.g_dim
            l._inv['dg'] = self._norm_arena.narrow(0, off, C * k).view(C, k)
            l._inv_cols['dg'] = k
            off += C * k
            l._p_store = l._p_view = self._norm_arena.narrow(0, off, C * l.a_dim).view(C, l.a_dim)
            off += C * l.a_dim
        # second-order data + preconditioned gradients
        self._inv_segments, self._grad_segments = build_comm_plan(ll, self._assignment)
        inv_total = sum(s.numel for s in self._inv_segments)
        p_total = sum(s.numel for s in self._grad_segments)
        self._inv_arena = torch.zeros(max(inv_total, 1), dtype=torch.float32, device=device)
        self._peer_p_bases = None      # rank -> device pointer of that rank's P arena (fused broadcast)
        self._p_arena = self._alloc_p_arena(max(p_total, 1), device)
        for segs, arena in ((self._inv_segments, self._inv_arena), (self._grad_segments, self._p_arena)):
            for s in segs:
                off = s.offset
                for layer, key, shape in s.entries:
                    store = _bind(arena, off, shape)
                    if key == 'P':
                        layer._p_store = store
                        layer._p_view = store[:, :shape[1]]
                    else:
                        layer._inv[key] = store
                        layer._inv_cols[key] = shape[-1]
                    off += _storage_numel(shape)
        self._layouts = {l: second_order_layout(l) for _, l in ll if l.tied_embedding is None}
        # local (never communicated) second-order data: K-major bases for the GEMM engine, eigen scratch
        plan = build_local_plan(ll, self._assignment, get_rank())
        local = sum(_storage_numel(shape) for _, _, shape in plan)
        self._local_arena = torch.zeros(max(local, 1), dtype=torch.float32, device=device)
        off = 0
        for l, key, shape in plan:
            l._inv[key] = _bind(self._local_arena, off, shape)
            l._inv_cols[key] = shape[-1]
            off += _storage_numel(shape)
        ek = [l for _, l in ll if l.method == ComputeMethod.EKFAC]
        if ek:
            total = sum(l.g_dim * _cabi.ld4(l.a_dim) for l in ek)
            self._s_arena = torch.zeros(total, dtype=torch.float32, device=device)
            self._s_batch_arena = torch.zeros(total, dtype=torch.float32, device=device)
            off = 0
            for l in ek:
                l._S = _bind(self._s_arena, off, (l.g_dim, l.a_dim))
                l._S_batch = _bind(self._s_batch_arena, off, (l.g_dim, l.a_dim))
                off += _storage_numel((l.g_dim, l.a_dim))
        if self._guard_factors or ek:
            self._skipped = torch.zeros(1, dtype=torch.int64, device=device)
        if self._guard_factors:
            self._g_scales = torch.ones(len(ll) + len(nl), dtype=torch.float32, device=device)
            for i, (_, l) in enumerate(ll + nl):
                l._g_scale_slot = self._g_scales.narrow(0, i, 1)
        self._vg = torch.zeros(1, dtype=torch.float64, device=device)
        self._nu = torch.ones(1, dtype=torch.float32, device=device)
        self._arenas_ready = True

    def _alloc_p_arena(self, numel: int, device: torch.device) -> torch.Tensor:
        """P arena.  With gradient broadcasts (KAISA HYBRID/MEM-OPT) it is allocated as CUDA-IPC
        peer memory and mapped into the other ranks of the gradient-receiver group, so the last
        precondition GEMM can store its tiles straight into every receiver (fused compute +
        broadcast over NVLink) instead of a broadcast per source afterwards.

        Every rank of the group takes the same sequence of collectives whatever happens locally:
        the local attempts (allocation, opening the peers' handles) are wrapped individually and the
        group agrees on the outcome with a MIN all-reduce of a success flag after each of them; the
        fused path is enabled only if EVERY rank succeeded, otherwise all ranks release what they hold
        and fall back to NCCL broadcasts together."""
        import torch.distributed as dist
        want = (self.fused_grad_broadcast and dist.is_available() and dist.is_initialized()
                and self._assignment.broadcast_gradients() and self._layers)
        group = None
        if want:
            name0 = next(n for n, l in self._layers.values() if l.tied_embedding is None)
            group = self._assignment.grad_receiver_group(name0)
            # pure functions of (group, backend): identical on every rank, no collective involved
            want = (dist.get_backend(group) == 'nccl' and 2 <= dist.get_world_size(group) <= 8)
        if not want:
            return torch.zeros(numel, dtype=torch.float32, device=device)

        def agree(ok: bool) -> bool:
            flag = torch.tensor([1 if ok else 0], dtype=torch.int32, device=device)
            dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=group)
            return bool(flag.item())

        lib = _cabi.load()
        ptr = C.c_void_p()
        handle = (C.c_ubyte * 64)()
        why = ''
        try:
            _cabi.check(lib.kfac_peer_alloc(numel * 4, C.byref(ptr), handle), 'kfac_peer_alloc')
            ok = True
        except Exception as e:  # noqa: BLE001
            ok, why = False, str(e)
        if not agree(ok):
            if ok:
                lib.kfac_peer_free(ptr)
            logger.warning('fused gradient broadcast unavailable (%s); using NCCL broadcasts', why or 'a peer failed')
            return torch.zeros(numel, dtype=torch.float32, device=device)
        me = get_rank()
        gathered = [None] * dist.get_world_size(group)
        dist.all_gather_object(gathered, (me, bytes(handle)), group=group)
        bases: dict[int, int] = {}
        try:
            for r, h in gathered:
                if r == me:
                    continue
                out = C.c_void_p()
                buf = (C.c_ubyte * 64).from_buffer_copy(h)
                _cabi.check(lib.kfac_peer_open(buf, C.byref(out)), 'kfac_peer_open')
                bases[r] = out.value
            ok = True
        except Exception as e:  # noqa: BLE001
            ok, why = False, str(e)
        if not agree(ok):
            for b in bases.values():
                lib.kfac_peer_close(C.c_void_p(b))
            dist.barrier(group=group)       # nobody frees an allocation a peer may still have mapped
            lib.kfac_peer_free(ptr)
            logger.warning('fused gradient broadcast unavailable (%s); using NCCL broadcasts', why or 'a peer failed')
            return torch.zeros(numel, dtype=torch.float32, device=device)

        class _Raw:   # zero-copy torch view of the cudaMalloc'ed buffer
            pass
        raw = _Raw()
        raw.__cuda_array_interface__ = {'shape': (numel,), 'typestr': '<f4', 'data': (ptr.value, False),
                                        'version': 3, 'strides': None}
        arena = torch.as_tensor(raw, device=device)
        self._peer_p_bases = bases
        self._p_raw = raw
        self._p_ptr = ptr.value
        self._row_group = group
        self._row_token = torch.zeros(1, dtype=torch.float32, device=device)
        import weakref
        self._peer_finalizer = weakref.finalize(self, _release_peer_memory, list(bases.values()), ptr.value)
        return arena

    def close(self) -> None:
        """Release the CUDA-IPC mappings and the peer-visible P arena (also runs when the
        preconditioner is garbage collected)."""
        fin = getattr(self, '_peer_finalizer', None)
        if fin is not None and fin.alive:
            fin()
        self._peer_p_bases = None

    # ------------------------------------------------------------ state dict
    def state_dict(self, include_factors: bool = True) -> dict[str, Any]:
        sd: dict[str, Any] = {'steps': self.steps}
        for key in ('factor_update_steps', 'inv_update_steps', 'damping', 'factor_decay', 'kl_clip', 'lr'):
            v = getattr(self, '_' + key)
            if not callable(v):
                sd[key] = v
        if include_factors:
            # the reference's factors are already EMA-updated and all-reduced when a state dict is taken
            # (both happen in the hooks, base_preconditioner.py:452-457): flush + reduce, and hand out
            # snapshots (the arena views keep changing in place)
            if self._arenas_ready:
                self._flush_factor_updates()
            sd['layers'] = {name: layer.state_dict() for name, layer in self._all_layer_list()}
        return sd

    def load_state_dict(self, state_dict: dict[str, Any], compute_inverses: bool = True) -> None:
        self._steps = state_dict['steps']
        for key in ('factor_update_steps', 'inv_update_steps', 'damping', 'factor_decay', 'kl_clip', 'lr'):
            if key in state_dict:
                setattr(self, '_' + key, state_dict[key])
        if 'layers' in state_dict:
            if len(state_dict['layers']) != len(self._layers) + len(self._norm_layers):
                raise ValueError('loaded state dict contains a different number of layers')
            self._ensure_arenas()
            by_name = {name: layer for name, layer in self._all_layer_list()}
            for found_name, layer_state in state_dict['layers'].items():
                if found_name in by_name:
                    by_name[found_name].load_state_dict(layer_state)
        elif compute_inverses:
            warnings.warn('Layer factors are not included in the state_dict so inverses cannot be '
                          'computed. Skipping inverse computation.', stacklevel=2)
            compute_inverses = False
        if compute_inverses:
            self._compute_inverses()
            # S <- dg x da: no window has been measured in these bases; rows kept before the load are discarded
            for _, layer in self._layers.values():
                if layer.method == ComputeMethod.EKFAC:
                    layer._rows_n_a = layer._rows_n_g = 0
            self._ekfac_update(new_basis=True)

    # ------------------------------------------------------------ hooks
    def _grad_scale_value(self, layer: KFACLayer) -> float:
        """Loss scale folded into the G statistics on the host (1 when the guarded EMA applies it on the device)."""
        if layer.grad_scaler is None or layer.device_grad_scaler:
            return 1.0
        return float(layer.grad_scaler())

    @staticmethod
    def _snapshot_loss_scale(layer: KFACLayer) -> None:
        """Stream-ordered copy of the GradScaler's current scale into the layer's device slot (no host sync)."""
        scaler = layer.grad_scaler
        scale = scaler._get_scale_async() if scaler.is_enabled() else None
        if scale is not None:
            layer._g_scale_slot.copy_(scale)
        else:
            layer._g_scale_slot.fill_(scaler._init_scale if scaler.is_enabled() else 1.0)

    def _save_input(self, module: torch.nn.Module, input_: tuple[torch.Tensor, ...]) -> None:
        """Forward pre-hook: accumulate A statistics (base_preconditioner.py:437-457)."""
        if not module.training:
            return
        if self.steps % self.factor_update_steps != 0:
            return
        self._accumulate_input(*self._layers[module], input_[0])

    def _save_input_with_kwargs(self, module: torch.nn.Module, args: tuple, kwargs: dict) -> None:
        """Forward pre-hook of a layer whose statistics depend on more of the call than its input: the output_size a
        transposed convolution takes positionally or as a keyword."""
        if not module.training:
            return
        if self.steps % self.factor_update_steps != 0:
            return
        name, layer = self._layers[module]
        layer.module.bind_call(args, kwargs)
        self._accumulate_input(name, layer, args[0])

    def _active_attention_taps(self, module: torch.nn.Module) -> dict[str, AttentionProjectionHelper] | None:
        """The registered projections of an attention module at a factor step (its forward taps them), else None."""
        if self.steps % self.factor_update_steps != 0:
            return None
        return self._attention_taps.get(module)

    def _attention_input(self, key: AttentionProjectionHelper, x: torch.Tensor) -> None:
        """A tap of an attention projection: x is its input, (L, B, features)."""
        self._accumulate_input(*self._layers[key], x)

    def _attention_grad_output(self, key: AttentionProjectionHelper, g: torch.Tensor) -> None:
        """G tap of an attention projection: g is the gradient of its output, (L, B, E), possibly a column block."""
        self._accumulate_grad_output(*self._layers[key], g)

    def _active_recurrent_taps(self, module: torch.nn.Module) -> dict[str, RecurrentSubLayerHelper] | None:
        """The registered sub-layers of a recurrent module at a factor step (its forward taps them), else None."""
        if self.steps % self.factor_update_steps != 0:
            return None
        return self._recurrent_taps.get(module)

    def _recurrent_input(self, key: RecurrentSubLayerHelper, x: torch.Tensor, tap) -> None:
        """A tap of a recurrent sub-layer: x is the layer input (ih) or output (hh), `tap` where its rows lie."""
        key.tap_a = tap
        self._accumulate_input(*self._layers[key], x)

    def _recurrent_grad_output(self, key: RecurrentSubLayerHelper, g: torch.Tensor, tap) -> None:
        """G tap of a recurrent sub-layer: g is the gradient of the input projection z_x, `tap` where its rows lie."""
        key.tap_g = tap
        self._accumulate_grad_output(*self._layers[key], g)

    @torch.no_grad()
    def _accumulate_input(self, name: str, layer: KFACLayer, x: torch.Tensor) -> None:
        self._ensure_arenas(x.device)
        if layer.method == ComputeMethod.EKFAC and layer._rows_n_a:
            raise RuntimeError(f'EKFAC: {name} was called a second time in one factor window (one forward and one '
                               'backward pass per layer between step() calls; weight-shared modules are not supported)')
        if layer._a_pending:       # a completed accumulation window is still queued
            self._flush_factor_updates()
        if self._a_reduce_work is not None:
            # another forward pass before step(): the overlapped reduction must not race with new statistics.
            # What it averaged stays averaged; the flush reduces the block again (idempotent on the averaged part)
            self._a_reduce_work.wait()
            self._a_reduce_work = None
            self._a_block_reduced = False
        if not layer.embedding:     # integer indices are counted as they are
            x = cast_for_factor(x, layer.factor_dtype)
        x = layer.module.prepare_input(x)
        layer.module.accumulate_a(x, layer._a_batch_view, self._scratch)
        if layer.method == ComputeMethod.EKFAC:
            n = layer.module.num_rows_a(x)
            layer._rows_x = self._row_buffer(layer._rows_x, n * _cabi.ld4(layer.a_dim))
            layer.module.write_rows_a(x, layer._rows_x)
            layer._rows_n_a = n
        layer._a_count += 1
        self._mini_steps[name] += 1
        if self._update_factors_in_hook and self._mini_steps[name] % self._accumulation_steps == 0:
            self._mark_pending(layer, 'a')

    def _hook_output(self, module: torch.nn.Module, input_, output: torch.Tensor) -> None:
        """Forward hook of an embedding: the gradient of its output reaches _save_grad_output through a tensor hook."""
        if module.training and output.requires_grad:
            output.register_hook(lambda g: self._save_grad_output(module, None, g))

    def _save_grad_output(self, module: torch.nn.Module, grad_input, grad_output) -> None:
        """Full backward hook: accumulate G statistics (base_preconditioner.py:459-479)."""
        if not module.training:
            return
        if self.steps % self.factor_update_steps != 0:
            return
        g = grad_output if isinstance(grad_output, torch.Tensor) else grad_output[0]
        self._accumulate_grad_output(*self._layers[module], g)

    @torch.no_grad()
    def _accumulate_grad_output(self, name: str, layer: KFACLayer, g: torch.Tensor) -> None:
        self._ensure_arenas(g.device)
        if layer.method == ComputeMethod.EKFAC and layer._rows_n_g:
            raise RuntimeError(f'EKFAC: {name} was called a second time in one factor window (one forward and one '
                               'backward pass per layer between step() calls; weight-shared modules are not supported)')
        if layer._g_pending:
            self._flush_factor_updates()
        if self._update_factors_in_hook and self._mini_steps[name] % self._accumulation_steps == 0:
            self._launch_a_block_reduction()     # first backward hook of the window: every A statistic is complete
        if layer.device_grad_scaler:
            self._snapshot_loss_scale(layer)
        # the backward hook runs on the autograd thread: it gets its own scratch buffer
        g = cast_for_factor(g, layer.factor_dtype)
        grad_scale = self._grad_scale_value(layer)
        layer.module.accumulate_g(g, layer._g_batch_view, grad_scale, self._scratch_bwd)
        if layer.method == ComputeMethod.EKFAC:
            n = layer.module.num_rows_g(g)
            layer._rows_g = self._row_buffer(layer._rows_g, n * _cabi.ld4(layer.g_dim))
            layer.module.write_rows_g(g, layer._rows_g, grad_scale,
                                      layer._g_scale_slot.data_ptr() if layer.device_grad_scaler else None)
            layer._rows_n_g = n
        layer._g_count += 1
        if self._update_factors_in_hook and self._mini_steps[name] % self._accumulation_steps == 0:
            self._mark_pending(layer, 'g')

    def _hook_norm_output(self, module: torch.nn.Module, input_, output) -> None:
        """Forward hook of a normalization layer.  Its statistic needs each call's input together with the gradient of
        that call's output, so at factor steps a tensor hook on the output closes over the input; at other steps
        nothing is registered and no reference to the input is kept.  A module called twice contributes both calls;
        under torch.utils.checkpoint the call whose output receives a gradient is the one paired.

        Memory: the input is held until the output's gradient arrives.  Outside checkpointing that costs nothing, since
        autograd already saves the same storage for the norm's own backward.  Inside a non-reentrant checkpoint region
        it keeps, at factor steps, inputs that checkpointing would have dropped, about one activation per norm call in
        the region.  The recomputed call also registers a hook; it never fires and is released with the recomputed
        graph.  With use_reentrant=True the first forward runs without grad, so nothing is held."""
        if not module.training or not isinstance(output, torch.Tensor) or not output.requires_grad:
            return
        if self.steps % self.factor_update_steps != 0:
            return
        x = input_[0].detach()
        output.register_hook(lambda g: self._save_norm_grad(module, x, g))

    @torch.no_grad()
    def _save_norm_grad(self, module: torch.nn.Module, x: torch.Tensor, g: torch.Tensor) -> None:
        """Tensor hook on a normalization layer's output: accumulate the blocks of one call into the batch arena."""
        _, layer = self._norm_layers[module]
        self._ensure_arenas(g.device)
        if layer.device_grad_scaler:
            self._snapshot_loss_scale(layer)
        eps = layer.module.eps_for(x)
        x = cast_for_factor(x, layer.factor_dtype)
        g = cast_for_factor(g, layer.factor_dtype)
        layer.module.accumulate_norm(x, g, layer._g_batch_view, self._grad_scale_value(layer), eps, self._norm_scratch)
        layer._g_count += 1
        # a pending window stays open until it is consumed, so that every call of a module used more than once in
        # a pass lands in the same window (the mean of its calls)
        if (self._update_factors_in_hook and not layer._g_pending
                and layer._g_count % self._accumulation_steps == 0):
            self._mark_pending(layer, 'g')

    def _row_buffer(self, buf: torch.Tensor | None, numel: int) -> torch.Tensor:
        """Grow-only fp32 row buffer of one layer and side (EKFAC)."""
        if buf is None or buf.numel() < numel:
            buf = torch.empty(numel, dtype=torch.float32, device=self._device)
        return buf

    def _mark_pending(self, layer: KFACLayer, which: str) -> None:
        """Queue the EMA update of one factor (layers/base.py:375-405); it is
        applied -- batched over all layers -- before the factors are next used."""
        count = layer._a_count if which == 'a' else layer._g_count
        if count == 0:
            return
        if which == 'a':
            layer._a_pending = True
        else:
            layer._g_pending = True
        self._pending_alpha.setdefault(float(self.factor_decay), []).append((layer, which))

    def _launch_a_block_reduction(self) -> None:
        """Asynchronous all-reduce (average) of the A block of the batch statistics on a side stream, launched from the
        backward hook that fires first: it overlaps with the rest of backward (the reference launches its factor
        all-reduces from the hooks for the same reason, base_preconditioner.py:452-457, layers/base.py:282-336)."""
        import torch.distributed as dist
        from kfac_b200.distributed import get_world_size
        if (not self.overlap_factor_allreduce or self._a_reduce_work is not None or self._a_block_reduced
                or get_world_size() == 1 or dist.get_backend() != 'nccl'):
            return
        ll = self._layer_list()
        if not ll or ll[0][1].symmetry_aware:       # packed triangles are reduced in one piece at the flush
            return
        if self._comm_stream is None:
            self._comm_stream = torch.cuda.Stream(device=self._device)
        done = torch.cuda.current_stream(self._device).record_event()
        with torch.cuda.stream(self._comm_stream):
            self._comm_stream.wait_event(done)
            self._a_reduce_work = dist.all_reduce(self._batch_arena.narrow(0, 0, self._a_block_numel),
                                                  op=dist.ReduceOp.AVG, async_op=True)
        self._tdc.calls['allreduce'] += 1

    def _reduce_batches(self) -> None:
        """C1: average the pending batch statistics over all ranks (whatever the hooks have not reduced yet).
        Averaging a block twice is harmless (the second average of identical values is the identity)."""
        from kfac_b200.distributed import get_world_size
        if get_world_size() == 1:
            return
        if self._a_reduce_work is not None:
            self._a_reduce_work.wait()            # the current stream waits for the collective; the host does not
            self._a_reduce_work = None
            self._a_block_reduced = True
        ll = self._layer_list()
        al = self._all_layer_list()
        if al and al[0][1].symmetry_aware:
            # communicate only the upper triangles (kfac/distributed.py:422-465):
            # pack -> one all-reduce of the packed arena -> mirror back
            lib = _cabi.load()
            stream = _cabi.stream_ptr()
            # (a diagonal factor -- a vector -- and the blocks of a normalization layer are passed through as they are)
            def packed_numel(view, d):
                return d if view.dim() == 1 else d * (d + 1) // 2
            views = [v for _, l in ll for v in ((l._a_batch_view, l.a_dim), (l._g_batch_view, l.g_dim))]
            views += [(l._g_batch_view.view(-1), l._g_batch_view.numel()) for _, l in self._norm_list()]
            if getattr(self, '_packed_arena', None) is None:
                total = sum(packed_numel(view, d) for view, d in views)
                self._packed_arena = torch.empty(total, dtype=torch.float32, device=self._device)
            off = 0
            todo = []
            for view, d in views:
                n = packed_numel(view, d)
                todo.append((view, d, self._packed_arena.narrow(0, off, n)))
                off += n
            for view, d, packed in todo:
                if view.dim() == 1:
                    packed.copy_(view)
                else:
                    _cabi.check(lib.kfac_triu_pack(view.data_ptr(), d, packed.data_ptr(), stream), 'kfac_triu_pack')
            self._tdc.allreduce_average(self._packed_arena, group=None)
            for view, d, packed in todo:
                if view.dim() == 1:
                    view.copy_(packed)
                else:
                    _cabi.check(lib.kfac_triu_unpack(packed.data_ptr(), d, view.data_ptr(), stream), 'kfac_triu_unpack')
        elif self._a_block_reduced:
            total = self._batch_arena.numel()
            self._tdc.allreduce_average(self._batch_arena.narrow(0, self._a_block_numel, total - self._a_block_numel),
                                        group=None)
        else:
            self._tdc.allreduce_average(self._batch_arena, group=None)
        self._a_block_reduced = False

    def _flush_factor_updates(self) -> None:
        if not self._pending_alpha:
            return
        self._reduce_batches()
        lib = _cabi.load()
        stream = _cabi.stream_ptr()
        flags = None
        # diagonal factors (an embedding's or a diagonal-A layer's A, a diagonal-G layer's G) take the EMA of vectors.
        # A window of token counts is finite whatever the loss scale and is never guarded; a diagonal A of activations
        # or of an embedding bag's pooled rows (per-sample weights are forward values) and a diagonal G are guarded like
        # every dense A and G.  The blocks of a normalization layer (G side) are
        # element-wise too and take the same path
        def vec(l, w):
            return l.diag_side == w or l.norm

        def guard(l, w):
            return self._guard_factors and (w == 'g' or not l.module.counts_a)
        split = {alpha: ([(l, w) for l, w in todo if vec(l, w) and not guard(l, w)],
                         [(l, w) for l, w in todo if vec(l, w) and guard(l, w)],
                         [(l, w) for l, w in todo if not vec(l, w)])
                 for alpha, todo in self._pending_alpha.items()}
        if self._guard_factors:
            # one drop-flag region per call, kept until step() has read the flags of its EKFAC layers
            sizes = [lib.kfac_factor_ema_diag_guarded_workspace_bytes(len(guarded)) +
                     lib.kfac_factor_ema_guarded_workspace_bytes(len(todo)) for _, guarded, todo in split.values()]
            flags = self._ema_scratch.get(sum(sizes), self._device)
            flag_off = 0
        for alpha, (diag, guarded, todo) in split.items():
            if diag:
                items = (_cabi.EmaItem * len(diag))()
                for i, (layer, which) in enumerate(diag):
                    items[i] = self._take_window(layer, which)
                _cabi.check(lib.kfac_factor_ema_diag(items, len(diag), alpha, stream), 'kfac_factor_ema_diag')
            if guarded:
                items = (_cabi.EmaItem * len(guarded))()
                scales = (C.c_void_p * len(guarded))()
                for i, (layer, which) in enumerate(guarded):
                    items[i] = self._take_window(layer, which)
                    if which == 'g' and layer.device_grad_scaler:
                        scales[i] = layer._g_scale_slot.data_ptr()
                need = lib.kfac_factor_ema_diag_guarded_workspace_bytes(len(guarded))
                ws = flags.data_ptr() + flag_off
                flag_off += need
                _cabi.check(lib.kfac_factor_ema_diag_guarded(items, len(guarded), alpha, scales,
                                                             self._skipped.data_ptr(), ws, need, stream),
                            'kfac_factor_ema_diag_guarded')
            if not todo:
                continue
            items = (_cabi.EmaItem * len(todo))()
            scales = (C.c_void_p * len(todo))()      # guarded EMA: loss-scale slot of a G item, NULL otherwise
            for i, (layer, which) in enumerate(todo):
                items[i] = self._take_window(layer, which)
                if which == 'g' and layer.device_grad_scaler:
                    scales[i] = layer._g_scale_slot.data_ptr()
            if not self._guard_factors:
                _cabi.check(lib.kfac_factor_ema(items, len(todo), alpha, stream), 'kfac_factor_ema')
                continue
            # decided after C1, so every rank drops the same windows
            need = lib.kfac_factor_ema_guarded_workspace_bytes(len(todo))
            ws = flags.data_ptr() + flag_off
            flag_off += need
            _cabi.check(lib.kfac_factor_ema_guarded(items, len(todo), alpha, scales, self._skipped.data_ptr(),
                                                    ws, need, stream), 'kfac_factor_ema_guarded')
            for i, (layer, which) in enumerate(todo):
                setattr(layer, '_drop_' + which, ws + 4 * i)
        self._pending_alpha = {}

    @staticmethod
    def _take_window(layer: KFACLayer, which: str) -> _cabi.EmaItem:
        """EMA item of the closed window of one factor; the window is consumed."""
        if which == 'a':
            item = _cabi.EmaItem(layer._a_view.data_ptr(), layer._a_batch_view.data_ptr(), layer.a_dim,
                                 int(not layer._has_a), 1.0 / layer._a_count)
            layer._has_a, layer._a_count, layer._a_pending = True, 0, False
        elif layer.norm:
            # C x k blocks as one vector; first = 0 on the identity seed the arena was given
            item = _cabi.EmaItem(layer._g_view.data_ptr(), layer._g_batch_view.data_ptr(), layer._g_view.numel(),
                                 0, 1.0 / layer._g_count)
            layer._has_g, layer._g_count, layer._g_pending = True, 0, False
        else:
            item = _cabi.EmaItem(layer._g_view.data_ptr(), layer._g_batch_view.data_ptr(), layer.g_dim,
                                 int(not layer._has_g), 1.0 / layer._g_count)
            layer._has_g, layer._g_count, layer._g_pending = True, 0, False
        return item

    # ------------------------------------------------------------ step
    @torch.no_grad()
    def step(self) -> None:
        """One K-FAC step: rewrites weight.grad / bias.grad of every registered
        layer with the (kl-clipped) preconditioned gradient.  Call between
        `loss.backward()` and `optimizer.step()`; gradients must already be
        averaged across ranks (base_preconditioner.py:310-382)."""
        self._ensure_arenas()
        self._check_eigh_status(wait=False)
        if not self._update_factors_in_hook and self.steps % self.factor_update_steps == 0:
            for name, layer in reversed(self._layer_list()):
                self._mini_steps[name] = 0
                self._mark_pending(layer, 'a')
                self._mark_pending(layer, 'g')
            for _, layer in self._norm_list():
                self._mark_pending(layer, 'g')
        self._flush_factor_updates()      # C1 (average of the batch statistics) + EMA

        new_basis = self.steps % self.inv_update_steps == 0
        if new_basis:
            self._compute_inverses()
        self._ekfac_update(new_basis)

        self._precondition()
        self._scale_and_write_back()

        self._steps += 1
        self._mini_steps = defaultdict(int)

    def _check_eigh_status(self, wait: bool) -> None:
        """Raise if the last eigendecomposition reported non-convergence or non-finite eigenvalues
        (KFAC_ERR_NO_CONVERGE).  wait=False: only if the status word has already arrived."""
        if not getattr(self, '_eig_pending', False):
            return
        if not wait and not self._eig_event.query():
            return
        self._eig_event.synchronize()
        self._eig_pending = False
        word = 0
        for slot in self._eig_slots:
            word |= int(self._eig_status[slot])
        if word:
            why = ' and '.join(w for b, w in ((1, 'an iteration did not converge'), (2, 'non-finite eigenvalues')) if word & b)
            raise _cabi.KFACNativeError(f'eigendecomposition of the K-FAC factors failed: {why} '
                                        f'(status {_cabi.KFAC_ERR_NO_CONVERGE}); were the factors finite?')

    # K5/K6/K7 + C2 -------------------------------------------------------
    def _compute_inverses(self) -> None:
        self._ensure_arenas()
        self._flush_factor_updates()
        lib = _cabi.load()
        rank = get_rank()
        damping = float(self.damping)
        stream = _cabi.stream_ptr()
        snapshots, calls, post = build_inverse_plan(self._layer_list(), self._assignment, rank)
        # every rank keeps the damping a tied pair's data is formed with
        for layer, lay in self._layouts.items():
            if lay.damped:
                layer._tied_damping = damping
        # a vector factor (an embedding's A, a diagonal-G layer's G, a tied pair's f and h) is its own
        # eigendecomposition: its snapshot is the one the precondition uses until the next inverse step, like the
        # eigenvalues of a dense factor
        snapshots = [(src._a_view if side == 'a' else src._g_view, layer._inv[key]) for layer, src, side, key in snapshots]
        # normalization layers: every rank snapshots its (all-reduced) blocks, which are their own decomposition
        for name, layer in self._norm_list():
            if not layer._has_g:
                raise RuntimeError(f'Cannot snapshot the blocks of the normalization layer "{name}" before they have '
                                   'been computed')
            snapshots.append((layer._g_view, layer._inv['dg']))
            layer._inv_ready.add('dg')
        if snapshots:
            # an entry that is not finite (or exceeds 1e15) is reported through the eigensolver's status path
            if self._diag_status is None:
                self._diag_status = torch.zeros(1, dtype=torch.int32, device=self._device)
            self._diag_status.zero_()
            for view, out in snapshots:
                _cabi.check(lib.kfac_diag_snapshot(view.data_ptr(), out.data_ptr(), view.numel(),
                                                   self._diag_status.data_ptr(), stream), 'kfac_diag_snapshot')
        # a tied pair's whitened H is decomposed in a call of its own after the one of its E (_tied_inverses)
        tied = [layer for layer, op, _ in post if op == 'tied']
        batches = [b for b in calls if b]
        if (batches or snapshots) and self._eig_status is None:
            self._eig_status = torch.zeros(4, dtype=torch.int32).pin_memory()
            self._eig_event = torch.cuda.Event()
        for slot, batch in enumerate(batches):
            items = (_cabi.EighItem * len(batch))()
            ns = (C.c_int * len(batch))()
            for i, (layer, side, q, qT, d) in enumerate(batch):
                F, n = (layer._a_view, layer.a_dim) if side == 'a' else (layer._g_view, layer.g_dim)
                I = layer._inv
                items[i] = _cabi.EighItem(F.data_ptr(), I[q].data_ptr(), I[qT].data_ptr() if qT else None,
                                          I[d].data_ptr(), n, _cabi.ld4(n), None)
                ns[i] = n
            need = lib.kfac_eigh_workspace_bytes(ns, len(batch))
            ws = self._eig_scratch.get(need, self._device)
            _cabi.check(lib.kfac_eigh_batched(items, len(batch), ws.data_ptr(), need, 0, 0.0, stream),
                        'kfac_eigh_batched')
            # status word (non-convergence / non-finite eigenvalues): copied to pinned memory without a sync and
            # inspected before the NEXT use of the second-order data (torch.linalg.eigh raises immediately,
            # kfac/layers/eigen.py:310; here the error surfaces one call later instead of stalling the stream)
            _cabi.check(lib.kfac_eigh_status(ws.data_ptr(), self._eig_status[slot:].data_ptr(), stream),
                        'kfac_eigh_status')
        if tied:
            self._tied_inverses(tied, damping)
        if snapshots:
            # status word of the diagonal snapshots: same pinned path, no host sync
            self._eig_status[2:3].copy_(self._diag_status, non_blocking=True)
        if batches or snapshots:
            self._eig_slots = list(range(len(batches))) + ([2] if snapshots else []) + ([3] if tied else [])
            self._eig_event.record()
            self._eig_pending = True
        # pi of the layers with pi-adjusted damping, from the factors just decomposed: every rank forms it for every
        # such layer from its copy of the all-reduced factors, in one launch and with the same bits, so it needs no
        # collective; it is kept until the next inverse step
        pi_layers = [l for l in self._layouts if l.pi_damping]
        if pi_layers:
            items = (_cabi.PiItem * len(pi_layers))()
            for i, l in enumerate(pi_layers):
                items[i] = _cabi.PiItem(l._a_view.data_ptr(), l._g_view.data_ptr(), l._inv['pi'].data_ptr(), l.a_dim,
                                        l.g_dim, 0 if l.diag_a else l.a_dim, 0 if l.diag_g else l.g_dim)
                l._inv_ready.add('pi')
            _cabi.check(lib.kfac_pi(items, len(pi_layers), stream), 'kfac_pi')
        s = pi_s(damping)
        for layer, op, keys in post:
            I = layer._inv
            if op == 'dgda':
                dg, da, dgda, *pi = keys
                if pi:
                    _cabi.check(lib.kfac_dgda_pi(I[dg].data_ptr(), I[da].data_ptr(), layer.g_dim, layer.a_dim, s,
                                                 I[pi[0]].data_ptr(), I[dgda].data_ptr(), _cabi.ld4(layer.a_dim),
                                                 stream), 'kfac_dgda_pi')
                else:
                    _cabi.check(lib.kfac_dgda(I[dg].data_ptr(), I[da].data_ptr(), layer.g_dim, layer.a_dim, damping,
                                              I[dgda].data_ptr(), _cabi.ld4(layer.a_dim), stream), 'kfac_dgda')
            elif op == 'inverse':
                q, d, inv, *pi = keys
                n = I[q].shape[0]
                ld = _cabi.ld4(n)
                need = n * ld * 4
                ws = self._gemm_scratch.get(need, self._device)
                if pi:
                    # gamma_A = s pi for A's inverse, gamma_G = s / pi for G's
                    _cabi.check(lib.kfac_inverse_from_eigh_pi(I[q].data_ptr(), ld, I[d].data_ptr(), n, s,
                                                              I[pi[0]].data_ptr(), 1 if inv == 'a_inv' else -1,
                                                              I[inv].data_ptr(), ld, ws.data_ptr(), need, stream),
                                'kfac_inverse_from_eigh_pi')
                else:
                    _cabi.check(lib.kfac_inverse_from_eigh(I[q].data_ptr(), ld, I[d].data_ptr(), n, damping,
                                                           I[inv].data_ptr(), ld, ws.data_ptr(), need, stream),
                                'kfac_inverse_from_eigh')
        # C2: one broadcast per (source, gradient-worker group)
        bcast = self._assignment.broadcast_inverses()
        for seg in self._inv_segments:
            if bcast:
                self._tdc.broadcast(self._inv_arena.narrow(0, seg.offset, seg.numel), src=seg.src,
                                    group=seg.group)
            for layer, key, shape in seg.entries:
                lay = self._layouts[layer]
                kmajor = next(e.kmajor for e in lay.entries if e.key == key)
                layer._inv_ready.add(key)
                if kmajor in lay.needs:
                    layer._inv_ready.add(kmajor)
                # a rank that RECEIVED an eigenbasis (or a tied pair's M) builds its K-major copy locally
                if bcast and seg.src != rank and kmajor:
                    n, ld = shape[0], _cabi.ld4(shape[0])
                    _cabi.check(lib.kfac_transpose(layer._inv[key].data_ptr(), ld, layer._inv[kmajor].data_ptr(), ld,
                                                   n, n, stream), 'kfac_transpose')

    def _tied_inverses(self, tied: list[KFACLayer], damping: float) -> None:
        """M and mu of the tied pairs this rank forms, after the call that decomposed their E: C (whitened H), then
        its eigendecomposition in a third call shared by all pairs (status slot 3), then M and M^T."""
        lib = _cabi.load()
        stream = _cabi.stream_ptr()
        items = (_cabi.TiedItem * len(tied))()
        eigs = (_cabi.EighItem * len(tied))()
        ns = (C.c_int * len(tied))()
        for i, layer in enumerate(tied):
            I, d = layer._inv, layer.g_dim
            items[i] = _cabi.TiedItem(I['_qg'].data_ptr(), I['_qgT'].data_ptr(), I['_dg'].data_ptr(),
                                      layer.tied_head._a_view.data_ptr(), I['_C'].data_ptr(), I['_UT'].data_ptr(),
                                      I['tq'].data_ptr(), I['_tqT'].data_ptr(), d, _cabi.ld4(d))
            eigs[i] = _cabi.EighItem(I['_C'].data_ptr(), I['_U'].data_ptr(), I['_UT'].data_ptr(), I['tmu'].data_ptr(),
                                     d, _cabi.ld4(d), None)
            ns[i] = d
        need = lib.kfac_tied_workspace_bytes(items, len(tied))
        ws = self._gemm_scratch.get(need, self._device)
        _cabi.check(lib.kfac_tied_whiten(items, len(tied), damping, ws.data_ptr(), need, stream), 'kfac_tied_whiten')
        need_e = lib.kfac_eigh_workspace_bytes(ns, len(tied))
        ws_e = self._eig_scratch.get(need_e, self._device)
        _cabi.check(lib.kfac_eigh_batched(eigs, len(tied), ws_e.data_ptr(), need_e, 0, 0.0, stream), 'kfac_eigh_batched')
        _cabi.check(lib.kfac_eigh_status(ws_e.data_ptr(), self._eig_status[3:].data_ptr(), stream), 'kfac_eigh_status')
        ws = self._gemm_scratch.get(need, self._device)
        _cabi.check(lib.kfac_tied_basis(items, len(tied), damping, ws.data_ptr(), need, stream), 'kfac_tied_basis')

    # EKFAC ----------------------------------------------------------------
    def _ekfac_update(self, new_basis: bool) -> None:
        """S and dgda of every EKFAC layer (the schedule of the module docstring).  A layer takes part once its bases
        and eigenvalues are available; its window (the rows of this step's forward and backward) is consumed."""
        ek = [l for _, l in reversed(self._layer_list()) if l.method == ComputeMethod.EKFAC]
        if not ek:
            return
        lib = _cabi.load()
        stream = _cabi.stream_ptr()
        ready = [l for l in ek if {'qa', 'qg', 'da', 'dg'} <= l._inv_ready]
        windows = [l for l in ready if l._rows_n_a and l._rows_n_g]
        for l in windows:
            if l._rows_n_a != l._rows_n_g:
                raise RuntimeError(f'EKFAC: {l._rows_n_a} rows on the A side and {l._rows_n_g} on the G side')
        if windows:
            items = (_cabi.EkfacStatItem * len(windows))()
            for i, l in enumerate(windows):
                a, g = l.a_dim, l.g_dim
                items[i] = _cabi.EkfacStatItem(l._rows_x.data_ptr(), l._rows_g.data_ptr(), l._inv['_qaT'].data_ptr(),
                                               l._inv['_qgT'].data_ptr(), l._S_batch.data_ptr(), l._rows_n_a, a, g,
                                               _cabi.ld4(a), _cabi.ld4(g), _cabi.ld4(a), _cabi.ld4(g), _cabi.ld4(a))
            need = lib.kfac_ekfac_statistics_workspace_bytes(items, len(windows))
            ws = self._ekfac_scratch.get(need, self._device)
            _cabi.check(lib.kfac_ekfac_statistics(items, len(windows), ws.data_ptr(), need, stream),
                        'kfac_ekfac_statistics')
            # C1 for S_batch: one average over the world (linear in the rows, like the factors)
            self._tdc.allreduce_average(self._s_batch_arena, group=None)
        in_window = set(map(id, windows))
        rest = [l for l in ready if id(l) not in in_window]
        damping = float(self.damping)
        alpha = float(self.factor_decay)
        for todo, mode in ((windows, _cabi.KFAC_EKFAC_RESET if new_basis else _cabi.KFAC_EKFAC_EMA),
                           (rest, _cabi.KFAC_EKFAC_SEED if new_basis else _cabi.KFAC_EKFAC_KEEP)):
            if not todo:
                continue
            items = (_cabi.EkfacUpdateItem * len(todo))()
            for i, l in enumerate(todo):
                I = l._inv
                items[i] = _cabi.EkfacUpdateItem(l._S.data_ptr(), l._S_batch.data_ptr(), I['dg'].data_ptr(),
                                                 I['da'].data_ptr(), I['dgda'].data_ptr(), l.g_dim, l.a_dim,
                                                 _cabi.ld4(l.a_dim), l._drop_a, l._drop_g)
            need = lib.kfac_ekfac_update_workspace_bytes(len(todo))
            ws = self._ekfac_scratch.get(need, self._device)
            _cabi.check(lib.kfac_ekfac_update(items, len(todo), alpha, mode, damping, self._skipped.data_ptr(),
                                              ws.data_ptr(), need, stream), 'kfac_ekfac_update')
            for l in todo:
                l._inv_ready.add('dgda')
        for l in ek:
            l._rows_n_a = l._rows_n_g = 0
            l._drop_a = l._drop_g = None

    # K8/K9/K10 + C3 -------------------------------------------------------
    def _grad_ptrs(self, layer: KFACLayer):
        m = layer.module
        w = m.get_weight_grad()
        if w is None:
            raise RuntimeError('module gradient is None: call loss.backward() before step()')
        b = m.get_bias_grad() if m.has_bias() else None
        if not w.is_contiguous() or (b is not None and not b.is_contiguous()):
            raise ValueError('K-FAC requires contiguous weight/bias gradients')
        return w, b

    def _precondition(self) -> None:
        lib = _cabi.load()
        todo = [(n, l) for n, l in reversed(self._layer_list())
                if l.tied_embedding is None and self._assignment.is_grad_worker(n)]
        eigen = False
        items = (_cabi.PrecondItem * max(1, len(todo)))()
        fused = self._peer_p_bases is not None
        peer_arrays = []   # keep the ctypes pointer arrays alive during the call
        p_base = self._p_arena.data_ptr()
        for i, (name, layer) in enumerate(todo):
            w, b = self._grad_ptrs(layer)
            lay = self._layouts[layer]
            if not lay.needs <= layer._inv_ready:
                raise RuntimeError(lay.unready)
            I = layer._inv
            items[i] = _cabi.PrecondItem(
                w.data_ptr(), b.data_ptr() if b is not None else None, _cabi.DTYPE_CODE[w.dtype], layer.g_dim,
                layer.a_dim, P=layer._p_store.data_ptr(), ldp=_cabi.ld4(layer.p_shape[1]),
                tied_damping=layer._tied_damping if lay.damped else 0.0, **lay.item,
                **{field: I[key].data_ptr() for field, key in lay.fields})
            eigen = eigen or lay.eigen
            if fused:
                off = layer._p_store.data_ptr() - p_base
                arr = (C.c_void_p * len(self._peer_p_bases))(*[b + off for b in self._peer_p_bases.values()])
                peer_arrays.append(arr)
                items[i].peer_P = arr
                items[i].n_peers = len(self._peer_p_bases)
        if fused:
            # nobody may still be reading the previous step's P when the peers start storing
            self._tdc.fence(self._row_token, group=self._row_group)
        if todo:
            need = lib.kfac_precondition_workspace_bytes(items, len(todo))
            ws = self._gemm_scratch.get(need, self._device)
            _cabi.check(lib.kfac_precondition(items, len(todo), _cabi.KFAC_EIGEN if eigen else _cabi.KFAC_INVERSE,
                                              float(self.damping), ws.data_ptr(), need, _cabi.stream_ptr()),
                        'kfac_precondition')
        if self._assignment.broadcast_gradients():
            if fused:
                # the tiles are already in every receiver's arena; one tiny collective in the
                # receiver group orders "all sources have stored" before anyone reads P
                self._tdc.fence(self._row_token, group=self._row_group)
            else:
                for seg in self._grad_segments:
                    self._tdc.broadcast(self._p_arena.narrow(0, seg.offset, seg.numel), src=seg.src,
                                        group=seg.group)
        self._precondition_norms()
        for _, layer in self._all_layer_list():
            layer._grad_ready = True

    def _precondition_norms(self) -> None:
        """P_c = (F_c + damping I)^-1 grad_c of every normalization layer, on every rank, in one launch."""
        nl = self._norm_list()
        if not nl:
            return
        lib = _cabi.load()
        items = (_cabi.NormItem * len(nl))()
        for i, (name, layer) in enumerate(nl):
            if 'dg' not in layer._inv_ready:
                raise RuntimeError(f'The blocks of the normalization layer "{name}" have not been snapshotted')
            w, b = self._grad_ptrs(layer)
            items[i] = _cabi.NormItem(layer._inv['dg'].data_ptr(), w.data_ptr(), b.data_ptr() if b is not None else None,
                                      _cabi.DTYPE_CODE[w.dtype], layer.g_dim, layer.module.k, layer._p_store.data_ptr())
        need = lib.kfac_norm_precondition_workspace_bytes(len(nl))
        ws = self._norm_p_scratch.get(need, self._device)
        _cabi.check(lib.kfac_norm_precondition(items, len(nl), float(self.damping), ws.data_ptr(), need,
                                               _cabi.stream_ptr()), 'kfac_norm_precondition')

    # K11/K12 --------------------------------------------------------------
    def _scale_and_write_back(self) -> None:
        lib = _cabi.load()
        # nu over all layers; the weight of a tied pair counts once (through its embedding)
        ll = [(n, l) for n, l in reversed(self._layer_list()) if l.tied_embedding is None] + self._norm_list()
        items = (_cabi.GradItem * max(1, len(ll)))()
        for i, (_, layer) in enumerate(ll):
            w, b = self._grad_ptrs(layer)
            rows, cols = layer.p_shape          # an embedding is a bias-less (V, d) layer here
            lay = self._layouts.get(layer)      # (normalization layers have none)
            # ld4(cols) in the P arena, cols for a normalization layer's P
            items[i] = _cabi.GradItem(layer._p_store.data_ptr(), w.data_ptr(),
                                      b.data_ptr() if b is not None else None,
                                      _cabi.DTYPE_CODE[w.dtype], rows, cols, layer._p_store.stride(0),
                                      lay.item.get('wgrad_taps', 0) if lay is not None else 0)
        stream = _cabi.stream_ptr()
        kl_clip = self.kl_clip
        scale_ptr = None
        need = lib.kfac_grad_workspace_bytes(len(ll))
        ws = self._grad_scratch.get(need, self._device)
        if kl_clip is not None and ll:
            _cabi.check(lib.kfac_grad_scale(items, len(ll), float(kl_clip), float(self.lr), ws.data_ptr(), need,
                                            self._nu.data_ptr(), stream), 'kfac_grad_scale')
            scale_ptr = self._nu.data_ptr()
            self.last_grad_scale = self._nu
        if ll:
            _cabi.check(lib.kfac_grad_update(items, len(ll), scale_ptr, ws.data_ptr(), need, stream), 'kfac_grad_update')
        for _, layer in ll:
            layer._grad_ready = False

    # ------------------------------------------------------------ misc API
    def reset_batch(self) -> None:
        if self._a_reduce_work is not None:      # an overlapped all-reduce of the A block must not race with the zeroing
            self._a_reduce_work.wait()
            self._a_reduce_work = None
        self._a_block_reduced = False
        for _, layer in self._all_layer_list():
            layer.reset_batch()
        self._pending_alpha = {}

    def memory_usage(self) -> dict[str, int]:
        sizes: dict[str, int] = defaultdict(int)
        for _, layer in self._all_layer_list():
            for key, size in layer.memory_usage().items():
                sizes[key] += size
        if 'ekfac' in sizes and self._ekfac_scratch.buf is not None:
            sizes['ekfac'] += self._ekfac_scratch.buf.numel()   # squared projections + split partials of S_batch
        sizes['total'] = sum(sizes.values())
        return sizes

    def _compute_grad_scale(self) -> float:
        """Host-visible kl-clip scale of the last step (debug / tests; syncs)."""
        if not self._layers or self.last_grad_scale is None:
            return 1.0
        return float(self.last_grad_scale.item())
