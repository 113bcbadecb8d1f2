"""K-FAC taps inside `torch.nn.RNN`, `torch.nn.LSTM` and `torch.nn.GRU` (opt-in through `precondition_recurrent`).

A recurrent module runs its whole stack in one fused op (cuDNN on the GPU), so no module hook sees the input and
hidden projections of a layer.  With `precondition_recurrent=True` the preconditioner sets the class of each
registered module to `KFACRNN`, `KFACLSTM` or `KFACGRU`: a subclass that adds no parameters, buffers or state and
overrides only `forward` (as `kfac_b200.attention` does).  `isinstance`, the parameters, `state_dict()`, `deepcopy` and
pickling are unaffected.

Outside the preconditioner's factor steps (eval, no grad, a step that is not a factor step, or once the preconditioner
has been garbage-collected) `forward` is the stock `forward`.  At factor steps in training it runs `_tapped_forward`, a
restatement of torch's `RNNBase` / `LSTM` / `GRU` forward.  Per layer and direction it computes the input projection
`z_x = F.linear(x, W_ih, b_ih)` over all positions at once and then loops over time with `F.linear(h, W_hh, b_hh)` and
the cell (on CUDA the fused cell ops torch's own non-cuDNN path uses, `_thnn_fused_lstm_cell` / `_thnn_fused_gru_cell`).
The taps:
  * the A tap of `ih_l{k}{sfx}` receives x, the layer input (time-major (T, B, I) or the packed data (N, I));
  * the A tap of `hh_l{k}{sfx}` receives the layer output together with h0 of that direction: the native gather forms
    the rows h_{t-1} (forward) or h_{t+1} (reverse), h0 where a sequence starts, without a copy;
  * a hook on z_x gives the G rows of every position of both sub-layers.  For RNN and LSTM the hidden projection has
    the same gradient; for GRU it is [dr, dz, r * dn], with r recomputed after the loop from z_x and the hidden gates.
Every A tap fires during the forward, so the A statistics are complete when the first backward hook starts their
all-reduce.  The inter-layer dropout is `F.dropout` on the layer output, so at factor steps its mask is drawn
differently from cuDNN's.

Restated from torch 2.11 (torch/nn/modules/rnn.py and aten/src/ATen/native/RNN.cpp).  Nothing compares it with the
stock forward at run time: after a torch upgrade, tests/test_recurrent_host.py (against stock) must pass before this is
trusted, and a change of torch's recurrent path has to be carried over here.
"""
from __future__ import annotations

import contextlib
import weakref
from typing import Any, NamedTuple

import torch
import torch.nn.functional as F
from torch.nn.utils.rnn import PackedSequence

# recurrent module -> weakref to the preconditioner that taps it (no reference cycle model <-> preconditioner)
_BOUND: 'weakref.WeakKeyDictionary[torch.nn.Module, weakref.ref]' = weakref.WeakKeyDictionary()


class _Tapped:
    """The `forward` of the swapped classes: the stock one, or the restatement with the taps at factor steps."""

    def forward(self, input, hx=None):
        ref = _BOUND.get(self)
        pre = ref() if ref is not None else None
        taps = (pre._active_recurrent_taps(self) if pre is not None and self.training and torch.is_grad_enabled()
                else None)
        if not taps:
            return super().forward(input, hx)
        return _tapped_forward(self, _Taps(pre, taps), input, hx)


class KFACRNN(_Tapped, torch.nn.RNN):
    """`torch.nn.RNN` whose projections are visible to a K-FAC preconditioner; see the module docstring."""


class KFACLSTM(_Tapped, torch.nn.LSTM):
    """`torch.nn.LSTM` whose projections are visible to a K-FAC preconditioner; see the module docstring."""


class KFACGRU(_Tapped, torch.nn.GRU):
    """`torch.nn.GRU` whose projections are visible to a K-FAC preconditioner; see the module docstring."""


SWAPPED = {torch.nn.RNN: KFACRNN, torch.nn.LSTM: KFACLSTM, torch.nn.GRU: KFACGRU}


def bind(module: torch.nn.Module, preconditioner: Any) -> None:
    """Swap the class of `module` (a torch.nn.RNN, LSTM or GRU, not a subclass) and let it reach `preconditioner`
    through a weak reference."""
    if type(module) in SWAPPED:
        module.__class__ = SWAPPED[type(module)]
    _BOUND[module] = weakref.ref(preconditioner)


class SequenceTap(NamedTuple):
    """Where the rows of one recurrent tap lie.  Positions (t, b) are time-major (T, B) or packed: `offsets` is then
    the device int32 tensor [0, cumsum(batch_sizes)].  `h0` (B, H) with `shift` +1 / -1: the rows are the previous
    hidden state of a forward / reverse direction, gathered from columns [col0, col0 + H) of the layer output.  `mul`
    (rows, H): the columns from `mul_col0` on are multiplied by it (the GRU's r)."""
    T: int
    B: int
    offsets: torch.Tensor | None = None
    h0: torch.Tensor | None = None
    shift: int = 0
    col0: int = 0
    mul: torch.Tensor | None = None
    mul_col0: int = 0


class _Taps:
    """The registered sub-layers of one call, keyed 'ih_l0', 'hh_l1_reverse', ..."""

    def __init__(self, pre: Any, keys: dict[str, Any]) -> None:
        self.pre, self.keys = pre, keys

    def a(self, which: str, x: torch.Tensor, seq: SequenceTap) -> None:
        key = self.keys.get(which)
        if key is not None:
            self.pre._recurrent_input(key, x, seq)

    def wants(self, which: str) -> bool:
        return which in self.keys

    def g(self, sfx: str, zx: torch.Tensor, seq: SequenceTap, r: torch.Tensor | None) -> None:
        ih, hh = self.keys.get('ih' + sfx), self.keys.get('hh' + sfx)
        if (ih is None and hh is None) or not zx.requires_grad:
            return
        pre = self.pre
        hh_seq = seq if r is None else seq._replace(mul=r, mul_col0=2 * r.size(-1))

        def hook(grad):
            if ih is not None:
                pre._recurrent_grad_output(ih, grad, seq)
            if hh is not None:
                pre._recurrent_grad_output(hh, grad, hh_seq)
        zx.register_hook(hook)


def _rnn_cell(act):
    def cell(gx, gh, h, c, fused):
        return act(gh + gx), None
    return cell


def _lstm_cell(gx, gh, h, c, fused):
    if fused:
        hy, cy, _ = torch.ops.aten._thnn_fused_lstm_cell(gx, gh, c)
        return hy, cy
    i, f, g, o = (gh + gx).chunk(4, 1)
    cy = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(g)
    return torch.sigmoid(o) * torch.tanh(cy), cy


def _gru_cell(gx, gh, h, c, fused):
    if fused:
        hy, _ = torch.ops.aten._thnn_fused_gru_cell(gx, gh, h)
        return hy, None
    xr, xz, xn = gx.chunk(3, 1)
    hr, hz, hn = gh.chunk(3, 1)
    r = torch.sigmoid(hr + xr)
    z = torch.sigmoid(hz + xz)
    n = torch.tanh(xn + r * hn)
    return (h - n) * z + n, None


def _direction(cell, zx, w_hh, b_hh, h0, c0, T, bs, offs, reverse, fused, keep_gh):
    """One direction of one layer: (outputs in the order of zx's rows, final h, final c, the hidden gates or None)."""
    hs: list = [None] * T
    ghs: list = [None] * T
    if bs is None:
        h, c = h0, c0
        for t in (range(T - 1, -1, -1) if reverse else range(T)):
            gh = F.linear(h, w_hh, b_hh)
            h, c = cell(zx[t], gh, h, c, fused)
            hs[t] = h
            if keep_gh:
                ghs[t] = gh
        return torch.stack(hs), h, c, (torch.stack(ghs) if keep_gh else None)
    if not reverse:
        # a sequence that ends leaves the batch (the batch sizes do not increase): its state is final
        h, c = h0, c0
        fin_h, fin_c = [], []
        for t in range(T):
            n = bs[t]
            if n < h.size(0):
                fin_h.append(h[n:])
                h = h[:n]
                if c is not None:
                    fin_c.append(c[n:])
                    c = c[:n]
            gh = F.linear(h, w_hh, b_hh)
            h, c = cell(zx[offs[t]:offs[t + 1]], gh, h, c, fused)
            hs[t] = h
            if keep_gh:
                ghs[t] = gh
        fin_h.append(h)
        hT = torch.cat(fin_h[::-1])
        cT = None
        if c is not None:
            fin_c.append(c)
            cT = torch.cat(fin_c[::-1])
    else:
        # a sequence joins the batch at its last step, from h0
        n = bs[T - 1]
        h = h0[:n]
        c = c0[:n] if c0 is not None else None
        for t in range(T - 1, -1, -1):
            n = bs[t]
            if n > h.size(0):
                h = torch.cat((h, h0[h.size(0):n]))
                if c is not None:
                    c = torch.cat((c, c0[c.size(0):n]))
            gh = F.linear(h, w_hh, b_hh)
            h, c = cell(zx[offs[t]:offs[t + 1]], gh, h, c, fused)
            hs[t] = h
            if keep_gh:
                ghs[t] = gh
        hT, cT = h, c
    return torch.cat(hs), hT, cT, (torch.cat(ghs) if keep_gh else None)


def _tapped_forward(self: torch.nn.RNNBase, taps: _Taps, input, hx):
    """RNNBase.forward / LSTM.forward / GRU.forward with the taps (proj_size = 0)."""
    self._update_flat_weights()
    mode = self.mode
    lstm = mode == 'LSTM'
    D = 2 if self.bidirectional else 1
    H = self.hidden_size
    L = self.num_layers
    kind = {'LSTM': 'LSTM', 'GRU': 'GRU'}.get(mode, 'RNN')

    # ---- the preamble of the stock forward
    orig_input = input
    batch_sizes = sorted_indices = unsorted_indices = None
    is_batched = True
    if isinstance(orig_input, PackedSequence):
        input, batch_sizes, sorted_indices, unsorted_indices = orig_input
        max_batch_size = int(batch_sizes[0])
        if hx is not None:
            hx = self.permute_hidden(hx, sorted_indices)
    else:
        if input.dim() not in (2, 3):
            raise ValueError(f'{kind}: Expected input to be 2D or 3D, got {input.dim()}D tensor instead')
        is_batched = input.dim() == 3
        batch_dim = 0 if self.batch_first else 1
        if not is_batched:
            input = input.unsqueeze(batch_dim)
        if hx is not None:
            want = 3 if is_batched else 2
            hs_ = hx if lstm else (hx,)
            if any(h.dim() != want for h in hs_):
                raise RuntimeError(f'For {"batched 3-D" if is_batched else "unbatched 2-D"} input, hx should also be '
                                   f'{want}-D but got {tuple(h.dim() for h in hs_)}-D tensor')
            if not is_batched:
                hx = tuple(h.unsqueeze(1) for h in hx) if lstm else hx.unsqueeze(1)
        max_batch_size = input.size(0) if self.batch_first else input.size(1)
    if hx is None:
        zeros = torch.zeros(L * D, max_batch_size, H, dtype=input.dtype, device=input.device)
        hx = (zeros, torch.zeros_like(zeros)) if lstm else zeros
    self.check_forward_args(input, hx, batch_sizes)

    # ---- the stack (aten/src/ATen/native/RNN.cpp: _rnn_impl over full / packed layers)
    weights = {n: getattr(self, n) for n in self._flat_weights_names}
    h0_all, c0_all = hx if lstm else (hx, None)
    x = input
    autocast = x.is_cuda and torch.is_autocast_enabled('cuda')
    if autocast:
        # the fused op is cast as a whole to the autocast dtype; here every operand is, and the ops run uncast
        dt = torch.get_autocast_dtype('cuda')
        x, h0_all = x.to(dt), h0_all.to(dt)
        c0_all = c0_all.to(dt) if c0_all is not None else None
        weights = {n: w.to(dt) for n, w in weights.items()}
    with torch.autocast('cuda', enabled=False) if autocast else contextlib.nullcontext():
        fused = x.is_cuda and mode in ('LSTM', 'GRU')
        cell = {'LSTM': _lstm_cell, 'GRU': _gru_cell, 'RNN_TANH': _rnn_cell(torch.tanh),
                'RNN_RELU': _rnn_cell(torch.relu)}[mode]
        if batch_sizes is None:
            if self.batch_first:
                x = x.transpose(0, 1)
            T, B = x.size(0), x.size(1)
            bs = offs = None
            seq = SequenceTap(T, B)
        else:
            bs = batch_sizes.tolist()
            T, B = len(bs), bs[0]
            offs = [0]
            for n in bs:
                offs.append(offs[-1] + n)
            offsets = torch.tensor(offs, dtype=torch.int32)
            if x.is_cuda:     # from pinned memory: the copy is ordered on the stream, the host does not wait
                offsets = offsets.pin_memory().to(x.device, non_blocking=True)
            seq = SequenceTap(T, B, offsets)
        h_n, c_n = [], []
        for k in range(L):
            outs = []
            for d in range(D):
                sfx = f'_l{k}' + ('_reverse' if d else '')
                i = k * D + d
                w_ih, w_hh = weights['weight_ih' + sfx], weights['weight_hh' + sfx]
                b_ih, b_hh = (weights['bias_ih' + sfx], weights['bias_hh' + sfx]) if self.bias else (None, None)
                taps.a('ih' + sfx, x, seq)
                zx = F.linear(x, w_ih, b_ih)
                gru_hh = mode == 'GRU' and taps.wants('hh' + sfx)
                out, hT, cT, gh = _direction(cell, zx, w_hh, b_hh, h0_all[i], c0_all[i] if lstm else None, T, bs,
                                             offs, bool(d), fused, gru_hh)
                r = None
                if gru_hh:
                    with torch.no_grad():
                        r = torch.sigmoid(zx[..., :H] + gh[..., :H])
                taps.g(sfx, zx, seq, r)
                outs.append(out)
                h_n.append(hT)
                c_n.append(cT)
            y = torch.cat(outs, -1) if D == 2 else outs[0]
            for d in range(D):
                sfx = f'_l{k}' + ('_reverse' if d else '')
                taps.a('hh' + sfx, y, seq._replace(h0=h0_all[k * D + d], shift=-1 if d else 1, col0=d * H))
            if self.dropout != 0 and self.training and k < L - 1:
                y = F.dropout(y, p=self.dropout, training=True)
            x = y
        output = x
        hidden = torch.stack(h_n)
        if lstm:
            hidden = (hidden, torch.stack(c_n))

    # ---- the epilogue of the stock forward
    if batch_sizes is not None:
        return (PackedSequence(output, batch_sizes, sorted_indices, unsorted_indices),
                self.permute_hidden(hidden, unsorted_indices))
    if self.batch_first:
        output = output.transpose(0, 1).contiguous()
    if not is_batched:
        output = output.squeeze(0 if self.batch_first else 1)
        hidden = tuple(h.squeeze(1) for h in hidden) if lstm else hidden.squeeze(1)
    return output, hidden

