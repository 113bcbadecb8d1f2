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
"""
from __future__ import annotations

import ctypes as C
import logging
import warnings
from collections import defaultdict
from typing import Any, Callable

import torch

from kfac_b200 import _cabi
from kfac_b200.assignment import WorkAssignment
from kfac_b200.distributed import ArenaCommunicator, get_rank
from kfac_b200.enums import ComputeMethod
from kfac_b200.layers import KFACLayer, cast_for_factor

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


def build_comm_plan(layers: list[tuple[str, KFACLayer]], assignment: WorkAssignment):
    """Decide which second-order tensors this rank stores and how they are
    grouped into broadcast segments.  Pure host logic (unit-tested on CPU for
    cross-rank consistency).

    Returns (inv_segments, grad_segments): ordered lists of _Segment.
    """
    inv: dict[tuple[int, int], _Segment] = {}
    for name, layer in layers:
        if not assignment.is_grad_worker(name):
            continue
        group = assignment.grad_worker_group(name)
        src_a = assignment.inv_worker(name, 'A')
        src_g = assignment.inv_worker(name, 'G')
        a, g = layer.a_dim, layer.g_dim

        def seg(src):
            key = (id(group) if group is not None else 0, src)
            if key not in inv:
                inv[key] = _Segment(src, group)
            return inv[key]

        if layer.method == ComputeMethod.EIGEN:
            if layer.prediv_eigenvalues:
                s = seg(src_g)
                s.add(layer, 'qa', (a, a))
                s.add(layer, 'qg', (g, g))
                s.add(layer, 'dgda', (g, a))
            else:
                sa, sg = seg(src_a), seg(src_g)
                sa.add(layer, 'qa', (a, a))
                sa.add(layer, 'da', (a,))
                sg.add(layer, 'qg', (g, g))
                sg.add(layer, 'dg', (g,))
        else:
            seg(src_a).add(layer, 'a_inv', (a, a))
            seg(src_g).add(layer, 'g_inv', (g, g))
    grad: dict[int, _Segment] = {}
    for name, layer in layers:
        src = assignment.src_grad_worker(name)
        if src not in grad:
            grad[src] = _Segment(src, assignment.grad_receiver_group(name))
        grad[src].add(layer, 'P', (layer.g_dim, layer.a_dim))
    inv_segments = list(inv.values())
    grad_segments = [grad[k] for k in sorted(grad)]
    for segs in (inv_segments, grad_segments):
        off = 0
        for s in segs:
            s.offset = off
            off += s.numel
    return inv_segments, grad_segments


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

        for module in self._layers:
            module.register_forward_pre_hook(self._save_input)
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

    # ------------------------------------------------------------ arenas
    def _layer_list(self) -> list[tuple[str, KFACLayer]]:
        return list(self._layers.values())

    def _ensure_arenas(self, device: torch.device | None = None) -> None:
        if self._arenas_ready:
            return
        if device is None:
            device = next(iter(self._layers.values()))[1].module.device if self._layers else torch.device('cuda')
        if device.type != 'cuda':
            raise _cabi.KFACNativeError(
                f'kfac_b200 needs the model on a CUDA (sm_90a) device, found {device}; '
                'there is no CPU fallback')
        _cabi.load()
        self._device = device
        ll = self._layer_list()
        # dense d x d factors, each starting 16-byte aligned
        total = sum(_cabi.ld4(l.a_dim ** 2) + _cabi.ld4(l.g_dim ** 2) for _, l in ll)
        self._factor_arena = torch.zeros(total, dtype=torch.float32, device=device)
        self._batch_arena = torch.zeros(total, dtype=torch.float32, device=device)
        # layout: all A factors, then all G factors -- the A block is complete after the forward pass and is
        # all-reduced on its own while backward produces the G statistics
        off = 0
        for which in ('a', 'g'):
            for _, l in ll:
                dim = l.a_dim if which == 'a' else l.g_dim
                n = dim * dim
                setattr(l, f'_{which}_view', self._factor_arena.narrow(0, off, n).view(dim, dim))
                setattr(l, f'_{which}_batch_view', self._batch_arena.narrow(0, off, n).view(dim, dim))
                off += _cabi.ld4(n)
            if which == 'a':
                self._a_block_numel = off
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
        # local (never communicated) eigen scratch of the inverse worker
        rank = get_rank()
        local = 0
        plan = []
        for name, l in ll:
            mine_a = rank == self._assignment.inv_worker(name, 'A')
            mine_g = rank == self._assignment.inv_worker(name, 'G')
            if l.method == ComputeMethod.EIGEN:
                if self._assignment.is_grad_worker(name):
                    # K-major (transposed) copies of the eigenbases for the GEMM engine
                    plan += [(l, '_qaT', (l.a_dim, l.a_dim)), (l, '_qgT', (l.g_dim, l.g_dim))]
                if l.prediv_eigenvalues:
                    if mine_a:
                        plan.append((l, '_da', (l.a_dim,)))
                    if mine_g:
                        plan.append((l, '_dg', (l.g_dim,)))
            else:
                if mine_a:
                    plan += [(l, '_qa', (l.a_dim, l.a_dim)), (l, '_da', (l.a_dim,))]
                if mine_g:
                    plan += [(l, '_qg', (l.g_dim, l.g_dim)), (l, '_dg', (l.g_dim,))]
        for _, _, shape in plan:
            local += _storage_numel(shape)
        self._local_arena = torch.zeros(max(local, 1), dtype=torch.float32, device=device)
        off = 0
        for l, key, shape in plan:
            l._inv[key] = _bind(self._local_arena, off, shape)
            l._inv_cols[key] = shape[-1]
            off += _storage_numel(shape)
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
            name0 = next(iter(self._layers.values()))[0]
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
            sd['layers'] = {name: layer.state_dict() for name, layer in self._layers.values()}
        return sd

    def load_state_dict(self, state_dict: dict[str, Any], compute_inverses: bool = True) -> None:
        self._steps = state_dict['steps']
        for key in ('factor_update_steps', 'inv_update_steps', 'damping', 'factor_decay', 'kl_clip', 'lr'):
            if key in state_dict:
                setattr(self, '_' + key, state_dict[key])
        if 'layers' in state_dict:
            if len(state_dict['layers']) != len(self._layers):
                raise ValueError('loaded state dict contains a different number of layers')
            self._ensure_arenas()
            by_name = {name: layer for name, layer in self._layers.values()}
            for found_name, layer_state in state_dict['layers'].items():
                if found_name in by_name:
                    by_name[found_name].load_state_dict(layer_state)
        elif compute_inverses:
            warnings.warn('Layer factors are not included in the state_dict so inverses cannot be '
                          'computed. Skipping inverse computation.', stacklevel=2)
            compute_inverses = False
        if compute_inverses:
            self._compute_inverses()

    # ------------------------------------------------------------ hooks
    def _grad_scale_value(self, layer: KFACLayer) -> float:
        return float(layer.grad_scaler()) if layer.grad_scaler is not None else 1.0

    @torch.no_grad()
    def _save_input(self, module: torch.nn.Module, input_: tuple[torch.Tensor, ...]) -> None:
        """Forward pre-hook: accumulate A statistics (base_preconditioner.py:437-457)."""
        if not module.training:
            return
        if self.steps % self.factor_update_steps != 0:
            return
        name, layer = self._layers[module]
        x = input_[0]
        self._ensure_arenas(x.device)
        if layer._a_pending:       # a completed accumulation window is still queued
            self._flush_factor_updates()
        if self._a_reduce_work is not None:
            # another forward pass before step(): the overlapped reduction must not race with new statistics.
            # What it averaged stays averaged; the flush reduces the block again (idempotent on the averaged part)
            self._a_reduce_work.wait()
            self._a_reduce_work = None
            self._a_block_reduced = False
        layer.module.accumulate_a(cast_for_factor(x, layer.factor_dtype), layer._a_batch_view, self._scratch)
        layer._a_count += 1
        self._mini_steps[name] += 1
        if self._update_factors_in_hook and self._mini_steps[name] % self._accumulation_steps == 0:
            self._mark_pending(layer, 'a')

    @torch.no_grad()
    def _save_grad_output(self, module: torch.nn.Module, grad_input, grad_output) -> None:
        """Full backward hook: accumulate G statistics (base_preconditioner.py:459-479)."""
        if not module.training:
            return
        if self.steps % self.factor_update_steps != 0:
            return
        name, layer = self._layers[module]
        g = grad_output if isinstance(grad_output, torch.Tensor) else grad_output[0]
        self._ensure_arenas(g.device)
        if layer._g_pending:
            self._flush_factor_updates()
        if self._update_factors_in_hook and self._mini_steps[name] % self._accumulation_steps == 0:
            self._launch_a_block_reduction()     # first backward hook of the window: every A statistic is complete
        # the backward hook runs on the autograd thread: it gets its own scratch buffer
        layer.module.accumulate_g(cast_for_factor(g, layer.factor_dtype), layer._g_batch_view,
                                  self._grad_scale_value(layer), self._scratch_bwd)
        layer._g_count += 1
        if self._update_factors_in_hook and self._mini_steps[name] % self._accumulation_steps == 0:
            self._mark_pending(layer, 'g')

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
        if ll and ll[0][1].symmetry_aware:
            # communicate only the upper triangles (kfac/distributed.py:422-465):
            # pack -> one all-reduce of the packed arena -> mirror back
            lib = _cabi.load()
            stream = _cabi.stream_ptr()
            if getattr(self, '_packed_arena', None) is None:
                total = sum(l.a_dim * (l.a_dim + 1) // 2 + l.g_dim * (l.g_dim + 1) // 2 for _, l in ll)
                self._packed_arena = torch.empty(total, dtype=torch.float32, device=self._device)
            off = 0
            todo = []
            for _, l in ll:
                for view, d in ((l._a_batch_view, l.a_dim), (l._g_batch_view, l.g_dim)):
                    n = d * (d + 1) // 2
                    todo.append((view, d, self._packed_arena.narrow(0, off, n)))
                    off += n
            for view, d, packed in todo:
                _cabi.check(lib.kfac_triu_pack(view.data_ptr(), d, packed.data_ptr(), stream), 'kfac_triu_pack')
            self._tdc.allreduce_average(self._packed_arena, group=None)
            for view, d, packed in todo:
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
        for alpha, todo in self._pending_alpha.items():
            items = (_cabi.EmaItem * len(todo))()
            for i, (layer, which) in enumerate(todo):
                if which == 'a':
                    items[i] = _cabi.EmaItem(layer._a_view.data_ptr(), layer._a_batch_view.data_ptr(),
                                             layer.a_dim, int(not layer._has_a), 1.0 / layer._a_count)
                    layer._has_a, layer._a_count, layer._a_pending = True, 0, False
                else:
                    items[i] = _cabi.EmaItem(layer._g_view.data_ptr(), layer._g_batch_view.data_ptr(),
                                             layer.g_dim, int(not layer._has_g), 1.0 / layer._g_count)
                    layer._has_g, layer._g_count, layer._g_pending = True, 0, False
            _cabi.check(lib.kfac_factor_ema(items, len(todo), alpha, _cabi.stream_ptr()), 'kfac_factor_ema')
        self._pending_alpha = {}

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
        self._flush_factor_updates()      # C1 (average of the batch statistics) + EMA

        if self.steps % self.inv_update_steps == 0:
            self._compute_inverses()

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
        word = int(self._eig_status.item())
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
        eig: list[tuple[torch.Tensor, torch.Tensor, torch.Tensor | None, torch.Tensor, int]] = []
        post: list[tuple[KFACLayer, str]] = []
        for name, layer in reversed(self._layer_list()):
            mine_a = rank == self._assignment.inv_worker(name, 'A')
            mine_g = rank == self._assignment.inv_worker(name, 'G')
            if mine_a and not layer._has_a:
                raise RuntimeError('Cannot eigendecompose A before A has been computed')
            if mine_g and not layer._has_g:
                raise RuntimeError('Cannot eigendecompose G before G has been computed')
            I = layer._inv
            if layer.method == ComputeMethod.EIGEN:
                if layer.prediv_eigenvalues:
                    if mine_a:
                        eig.append((layer._a_view, I['qa'], I['_qaT'], I['_da'], layer.a_dim))
                    if mine_g:
                        eig.append((layer._g_view, I['qg'], I['_qgT'], I['_dg'], layer.g_dim))
                        post.append((layer, 'dgda'))
                else:
                    if mine_a:
                        eig.append((layer._a_view, I['qa'], I['_qaT'], I['da'], layer.a_dim))
                    if mine_g:
                        eig.append((layer._g_view, I['qg'], I['_qgT'], I['dg'], layer.g_dim))
            else:
                if mine_a:
                    eig.append((layer._a_view, I['_qa'], None, I['_da'], layer.a_dim))
                    post.append((layer, 'a_inv'))
                if mine_g:
                    eig.append((layer._g_view, I['_qg'], None, I['_dg'], layer.g_dim))
                    post.append((layer, 'g_inv'))
        if eig:
            items = (_cabi.EighItem * len(eig))()
            ns = (C.c_int * len(eig))()
            for i, (F, Q, QT, d, n) in enumerate(eig):
                items[i] = _cabi.EighItem(F.data_ptr(), Q.data_ptr(), QT.data_ptr() if QT is not None else None,
                                          d.data_ptr(), n, _cabi.ld4(n), None)
                ns[i] = n
            need = lib.kfac_eigh_workspace_bytes(ns, len(eig))
            ws = self._eig_scratch.get(need, self._device)
            _cabi.check(lib.kfac_eigh_batched(items, len(eig), ws.data_ptr(), need, 0, 0.0, stream),
                        'kfac_eigh_batched')
            # status word (non-convergence / non-finite eigenvalues): copied to pinned memory without a sync and
            # inspected before the NEXT use of the second-order data (torch.linalg.eigh raises immediately,
            # kfac/layers/eigen.py:310; here the error surfaces one call later instead of stalling the stream)
            if self._eig_status is None:
                self._eig_status = torch.zeros(1, dtype=torch.int32).pin_memory()
                self._eig_event = torch.cuda.Event()
            _cabi.check(lib.kfac_eigh_status(ws.data_ptr(), self._eig_status.data_ptr(), stream), 'kfac_eigh_status')
            self._eig_event.record()
            self._eig_pending = True
        for layer, what in post:
            I = layer._inv
            if what == 'dgda':
                _cabi.check(lib.kfac_dgda(I['_dg'].data_ptr(), I['_da'].data_ptr(), layer.g_dim,
                                          layer.a_dim, damping, I['dgda'].data_ptr(),
                                          _cabi.ld4(layer.a_dim), stream), 'kfac_dgda')
            else:
                q, d, n = (I['_qa'], I['_da'], layer.a_dim) if what == 'a_inv' else (I['_qg'], I['_dg'], layer.g_dim)
                ld = _cabi.ld4(n)
                need = n * ld * 4
                ws = self._gemm_scratch.get(need, self._device)
                _cabi.check(lib.kfac_inverse_from_eigh(q.data_ptr(), ld, d.data_ptr(), n, damping,
                                                       I[what].data_ptr(), ld, ws.data_ptr(), need, stream),
                            'kfac_inverse_from_eigh')
        # C2: one broadcast per (source, gradient-worker group)
        bcast = self._assignment.broadcast_inverses()
        for seg in self._inv_segments:
            if bcast:
                self._tdc.broadcast(self._inv_arena.narrow(0, seg.offset, seg.numel), src=seg.src,
                                    group=seg.group)
            for layer, key, shape in seg.entries:
                layer._inv_ready.add(key)
                # a rank that RECEIVED an eigenbasis builds its K-major copy locally
                if bcast and seg.src != rank and key in ('qa', 'qg'):
                    n, ld = shape[0], _cabi.ld4(shape[0])
                    _cabi.check(lib.kfac_transpose(layer._inv[key].data_ptr(), ld,
                                                   layer._inv['_' + key + 'T'].data_ptr(), ld, n, n, stream),
                                'kfac_transpose')

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
        todo = [(n, l) for n, l in reversed(self._layer_list()) if self._assignment.is_grad_worker(n)]
        eigen = None
        items = (_cabi.PrecondItem * max(1, len(todo)))()
        fused = self._peer_p_bases is not None
        peer_arrays = []   # keep the ctypes pointer arrays alive during the call
        p_base = self._p_arena.data_ptr()
        for i, (name, layer) in enumerate(todo):
            w, b = self._grad_ptrs(layer)
            I = layer._inv
            ready = layer._inv_ready
            if layer.method == ComputeMethod.EIGEN:
                ok = ('qa' in ready and 'qg' in ready and
                      ('dgda' in ready if layer.prediv_eigenvalues else ('da' in ready and 'dg' in ready)))
                if not ok:
                    raise RuntimeError('Eigendecompositions for both A and G have not been computed')
                eigen = True
            else:
                if not ('a_inv' in ready and 'g_inv' in ready):
                    raise RuntimeError('Cannot precondition gradient before A and G have been inverted')
                eigen = False

            def p(key):
                return I[key].data_ptr() if key in ready else None

            eig_ok = 'qa' in ready and 'qg' in ready
            items[i] = _cabi.PrecondItem(
                w.data_ptr(), b.data_ptr() if b is not None else None, _cabi.DTYPE_CODE[w.dtype],
                layer.g_dim, layer.a_dim,
                p('qa'), I['_qaT'].data_ptr() if eig_ok else None,
                p('qg'), I['_qgT'].data_ptr() if eig_ok else None,
                p('dgda'), p('da'), p('dg'), p('a_inv'), p('g_inv'),
                _cabi.ld4(layer.a_dim), _cabi.ld4(layer.g_dim), _cabi.ld4(layer.a_dim),
                layer._p_store.data_ptr(), _cabi.ld4(layer.a_dim), None, 0)
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
        for _, layer in self._layer_list():
            layer._grad_ready = True

    # K11/K12 --------------------------------------------------------------
    def _scale_and_write_back(self) -> None:
        lib = _cabi.load()
        ll = list(reversed(self._layer_list()))
        items = (_cabi.GradItem * max(1, len(ll)))()
        for i, (_, layer) in enumerate(ll):
            w, b = self._grad_ptrs(layer)
            items[i] = _cabi.GradItem(layer._p_store.data_ptr(), w.data_ptr(),
                                      b.data_ptr() if b is not None else None,
                                      _cabi.DTYPE_CODE[w.dtype], layer.g_dim, layer.a_dim,
                                      _cabi.ld4(layer.a_dim))
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
        for _, layer in self._layers.values():
            layer.reset_batch()
        self._pending_alpha = {}

    def memory_usage(self) -> dict[str, int]:
        sizes: dict[str, int] = defaultdict(int)
        for _, layer in self._layers.values():
            for key, size in layer.memory_usage().items():
                sizes[key] += size
        sizes['total'] = sum(sizes.values())
        return sizes

    def _compute_grad_scale(self) -> float:
        """Host-visible kl-clip scale of the last step (debug / tests; syncs)."""
        if not self._layers or self.last_grad_scale is None:
            return 1.0
        return float(self.last_grad_scale.item())
