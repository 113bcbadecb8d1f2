"""K-FAC taps inside `torch.nn.MultiheadAttention` (opt-in through `precondition_attention`).

`F.multi_head_attention_forward` reads the projection weights directly, so neither module hooks nor a
TorchFunctionMode see the four projections.  With `precondition_attention=True` the preconditioner sets the class of
each registered attention to `KFACMultiheadAttention`: a subclass that adds no parameters, buffers or state and
overrides only `forward` (the way torch's FSDP2 `fully_shard` swaps classes).  `isinstance`, the parameters,
`state_dict()`, `deepcopy` and pickling are unaffected.

Outside the preconditioner's factor steps (eval, no grad, a step that is not a factor step, or once the preconditioner
has been garbage-collected) `forward` is the stock `forward`.  At factor steps in training it runs `_tapped_forward`,
a restatement of torch's training path with the same torch ops, in the same order and with the same shapes, which
calls the preconditioner's A tap with the input of every projection and registers a tensor hook (G side) on its
output.  The taps see every tensor in the sequence-first (L, B, features) layout of that path; q/k/v of a packed
linear are column blocks of one output gradient, read in place by the strided native entry points.
"""
from __future__ import annotations

import math
import weakref
from typing import Any

import torch
import torch.nn.functional as F

# attention module -> weakref to the preconditioner that taps it (no reference cycle model <-> preconditioner)
_BOUND: 'weakref.WeakKeyDictionary[torch.nn.MultiheadAttention, weakref.ref]' = weakref.WeakKeyDictionary()


class KFACMultiheadAttention(torch.nn.MultiheadAttention):
    """`torch.nn.MultiheadAttention` whose projections are visible to a K-FAC preconditioner; see the module
    docstring.  Only `forward` differs, and only at the preconditioner's factor steps in training."""

    def forward(self, query, key, value, key_padding_mask=None, need_weights=True, attn_mask=None,
                average_attn_weights=True, is_causal=False):
        ref = _BOUND.get(self)
        pre = ref() if ref is not None else None
        taps = (pre._active_attention_taps(self) if pre is not None and self.training and torch.is_grad_enabled()
                else None)
        if not taps or query.is_nested or key.is_nested or value.is_nested:
            return super().forward(query, key, value, key_padding_mask=key_padding_mask, need_weights=need_weights,
                                   attn_mask=attn_mask, average_attn_weights=average_attn_weights,
                                   is_causal=is_causal)
        return _tapped_forward(self, _Taps(pre, taps), query, key, value, key_padding_mask, need_weights, attn_mask,
                               average_attn_weights, is_causal)


def bind(module: torch.nn.MultiheadAttention, preconditioner: Any) -> None:
    """Swap the class of `module` (a torch.nn.MultiheadAttention, not a subclass) and let it reach `preconditioner`
    through a weak reference."""
    module.__class__ = KFACMultiheadAttention
    _BOUND[module] = weakref.ref(preconditioner)


class _Taps:
    """The registered projections of one attention call: `a(which, x)` feeds the A statistics, `g(which, t)` hooks
    the projection output `t` (columns [i E, (i + 1) E) of t belong to the i-th name of `which`)."""

    def __init__(self, pre: Any, keys: dict[str, Any]) -> None:
        self.pre, self.keys = pre, keys

    def a(self, which: str, x: torch.Tensor) -> None:
        for w in which:
            if w in self.keys:
                self.pre._attention_input(self.keys[w], x)

    def g(self, which: str, t: torch.Tensor, L: int, B: int) -> None:
        keys = [(i, self.keys[w]) for i, w in enumerate(which) if w in self.keys]
        if not keys or not t.requires_grad:
            return
        pre = self.pre

        def hook(grad):
            g = grad.reshape(L, B, grad.size(-1)) if grad.dim() == 2 else grad
            E = g.size(-1) // len(which)
            for i, k in keys:
                pre._attention_grad_output(k, g[..., i * E:(i + 1) * E] if len(which) > 1 else g)
        t.register_hook(hook)


def _tapped_forward(self: torch.nn.MultiheadAttention, taps: _Taps, query, key, value, key_padding_mask,
                    need_weights, attn_mask, average_attn_weights, is_causal):
    """nn.MultiheadAttention.forward -> F.multi_head_attention_forward on their training path (no fast path, no
    bias_k / bias_v, no add_zero_attn, no static k / v), with the projection taps ('q', 'k', 'v', 'o').

    Restated from torch 2.11 (torch/nn/modules/activation.py and torch/nn/functional.py), including its private mask
    helpers F._canonical_mask, F._none_or_dtype, F._mha_shape_check and F._check_key_padding_mask.  Nothing compares it
    with the stock forward at run time: after a torch upgrade, tests/test_attention_host.py (bitwise against stock)
    must pass before this is trusted, and a change of torch's attention path has to be carried over here."""
    # ---- nn.MultiheadAttention.forward
    is_batched = query.dim() == 3
    key_padding_mask = F._canonical_mask(mask=key_padding_mask, mask_name='key_padding_mask',
                                         other_type=F._none_or_dtype(attn_mask), other_name='attn_mask',
                                         target_type=query.dtype)
    attn_mask = F._canonical_mask(mask=attn_mask, mask_name='attn_mask', other_type=None, other_name='',
                                  target_type=query.dtype, check_other=False)
    if self.batch_first and is_batched:
        if key is value:
            if query is key:
                query = key = value = query.transpose(1, 0)
            else:
                query, key = (x.transpose(1, 0) for x in (query, key))
                value = key
        else:
            query, key, value = (x.transpose(1, 0) for x in (query, key, value))
    separate = not self._qkv_same_embed_dim
    num_heads = self.num_heads

    # ---- F.multi_head_attention_forward
    is_batched = F._mha_shape_check(query, key, value, key_padding_mask, attn_mask, num_heads)
    if not is_batched:
        query = query.unsqueeze(1)
        key = key.unsqueeze(1)
        value = value.unsqueeze(1)
        if key_padding_mask is not None:
            key_padding_mask = key_padding_mask.unsqueeze(0)
    tgt_len, bsz, embed_dim = query.shape
    src_len, _, _ = key.shape
    key_padding_mask = F._canonical_mask(mask=key_padding_mask, mask_name='key_padding_mask',
                                         other_type=F._none_or_dtype(attn_mask), other_name='attn_mask',
                                         target_type=query.dtype)
    if is_causal and attn_mask is None:
        raise RuntimeError('Need attn_mask if specifying the is_causal hint. You may use the Transformer module '
                           'method `generate_square_subsequent_mask` to create this mask.')
    if is_causal and key_padding_mask is None and not need_weights:
        attn_mask = None
    else:
        attn_mask = F._canonical_mask(mask=attn_mask, mask_name='attn_mask', other_type=None, other_name='',
                                      target_type=query.dtype, check_other=False)
        if key_padding_mask is not None:
            is_causal = False
    if embed_dim != self.embed_dim:
        raise AssertionError(f'was expecting embedding dimension of {self.embed_dim}, but got {embed_dim}')
    head_dim = embed_dim // num_heads
    if separate:
        if key.shape[:2] != value.shape[:2]:
            raise AssertionError(f"key's sequence and batch dims {key.shape[:2]} do not match value's "
                                 f'{value.shape[:2]}')
    elif key.shape != value.shape:
        raise AssertionError(f'key shape {key.shape} does not match value shape {value.shape}')

    # in-projection (F._in_projection_packed / F._in_projection), tapped
    w, b = self.in_proj_weight, self.in_proj_bias
    E = query.size(-1)
    if not separate:
        if key is value:
            if query is key:
                taps.a('qkv', query)
                proj = F.linear(query, w, b)
                taps.g('qkv', proj, tgt_len, bsz)
                proj = proj.unflatten(-1, (3, E)).unsqueeze(0).transpose(0, -2).squeeze(-2).contiguous()
                q, k, v = proj[0], proj[1], proj[2]
            else:
                w_q, w_kv = w.split([E, E * 2])
                b_q, b_kv = (None, None) if b is None else b.split([E, E * 2])
                taps.a('q', query)
                q = F.linear(query, w_q, b_q)
                taps.g('q', q, tgt_len, bsz)
                taps.a('kv', key)
                kv_proj = F.linear(key, w_kv, b_kv)
                taps.g('kv', kv_proj, src_len, bsz)
                kv_proj = kv_proj.unflatten(-1, (2, E)).unsqueeze(0).transpose(0, -2).squeeze(-2).contiguous()
                k, v = kv_proj[0], kv_proj[1]
        else:
            w_q, w_k, w_v = w.chunk(3)
            b_q, b_k, b_v = (None, None, None) if b is None else b.chunk(3)
            q, k, v = _three_linears(taps, query, key, value, w_q, w_k, w_v, b_q, b_k, b_v, tgt_len, src_len, bsz)
    else:
        b_q, b_k, b_v = (None, None, None) if b is None else b.chunk(3)
        q, k, v = _three_linears(taps, query, key, value, self.q_proj_weight, self.k_proj_weight, self.v_proj_weight,
                                 b_q, b_k, b_v, tgt_len, src_len, bsz)

    if attn_mask is not None:
        if attn_mask.dim() == 2:
            if attn_mask.shape != (tgt_len, src_len):
                raise RuntimeError(f'The shape of the 2D attn_mask is {attn_mask.shape}, but should be '
                                   f'{(tgt_len, src_len)}.')
            attn_mask = attn_mask.unsqueeze(0)
        elif attn_mask.dim() == 3:
            if attn_mask.shape != (bsz * num_heads, tgt_len, src_len):
                raise RuntimeError(f'The shape of the 3D attn_mask is {attn_mask.shape}, but should be '
                                   f'{(bsz * num_heads, tgt_len, src_len)}.')
        else:
            raise RuntimeError(f"attn_mask's dimension {attn_mask.dim()} is not supported")

    q = q.view(tgt_len, bsz * num_heads, head_dim).transpose(0, 1)
    k = k.view(k.shape[0], bsz * num_heads, head_dim).transpose(0, 1)
    v = v.view(v.shape[0], bsz * num_heads, head_dim).transpose(0, 1)
    src_len = k.size(1)
    if key_padding_mask is not None:
        F._check_key_padding_mask(key_padding_mask, src_len, bsz)
        key_padding_mask = (key_padding_mask.view(bsz, 1, 1, src_len).expand(-1, num_heads, -1, -1)
                            .reshape(bsz * num_heads, 1, src_len))
        attn_mask = key_padding_mask if attn_mask is None else attn_mask + key_padding_mask
    dropout_p = self.dropout

    out_w, out_b = self.out_proj.weight, self.out_proj.bias
    if need_weights:
        _B, _Nt, E_h = q.shape
        q_scaled = q * math.sqrt(1.0 / float(E_h))
        if is_causal and attn_mask is None:
            raise AssertionError('FIXME: is_causal not implemented for need_weights')
        if attn_mask is not None:
            attn_output_weights = torch.baddbmm(attn_mask, q_scaled, k.transpose(-2, -1))
        else:
            attn_output_weights = torch.bmm(q_scaled, k.transpose(-2, -1))
        attn_output_weights = F.softmax(attn_output_weights, dim=-1)
        if dropout_p > 0.0:
            attn_output_weights = F.dropout(attn_output_weights, p=dropout_p)
        attn_output = torch.bmm(attn_output_weights, v)
        attn_output = attn_output.transpose(0, 1).contiguous().view(tgt_len * bsz, embed_dim)
        attn_output = _out_linear(taps, attn_output, out_w, out_b, tgt_len, bsz)
        attn_output = attn_output.view(tgt_len, bsz, attn_output.size(1))
        attn_output_weights = attn_output_weights.view(bsz, num_heads, tgt_len, src_len)
        if average_attn_weights:
            attn_output_weights = attn_output_weights.mean(dim=1)
        if not is_batched:
            attn_output = attn_output.squeeze(1)
            attn_output_weights = attn_output_weights.squeeze(0)
    else:
        if attn_mask is not None:
            if attn_mask.size(0) == 1 and attn_mask.dim() == 3:
                attn_mask = attn_mask.unsqueeze(0)
            else:
                attn_mask = attn_mask.view(bsz, num_heads, -1, src_len)
        q = q.view(bsz, num_heads, tgt_len, head_dim)
        k = k.view(bsz, num_heads, src_len, head_dim)
        v = v.view(bsz, num_heads, src_len, head_dim)
        attn_output = F.scaled_dot_product_attention(q, k, v, attn_mask, dropout_p, is_causal)
        attn_output = attn_output.permute(2, 0, 1, 3).contiguous().view(bsz * tgt_len, embed_dim)
        attn_output = _out_linear(taps, attn_output, out_w, out_b, tgt_len, bsz)
        attn_output = attn_output.view(tgt_len, bsz, attn_output.size(1))
        if not is_batched:
            attn_output = attn_output.squeeze(1)
        attn_output_weights = None

    # ---- nn.MultiheadAttention.forward
    if self.batch_first and is_batched:
        return attn_output.transpose(1, 0), attn_output_weights
    return attn_output, attn_output_weights


def _three_linears(taps, query, key, value, w_q, w_k, w_v, b_q, b_k, b_v, tgt_len, src_len, bsz):
    """F._in_projection, or the chunked branch of F._in_projection_packed: one linear per projection."""
    Eq, Ek, Ev = query.size(-1), key.size(-1), value.size(-1)
    if w_q.shape != (Eq, Eq) or w_k.shape != (Eq, Ek) or w_v.shape != (Eq, Ev):
        raise AssertionError(f'projection weights of shapes {tuple(w_q.shape)}, {tuple(w_k.shape)}, '
                             f'{tuple(w_v.shape)} for inputs of {Eq}, {Ek}, {Ev} features')
    out = []
    for which, x, w, b, L in (('q', query, w_q, b_q, tgt_len), ('k', key, w_k, b_k, src_len),
                              ('v', value, w_v, b_v, src_len)):
        taps.a(which, x)
        y = F.linear(x, w, b)
        taps.g(which, y, L, bsz)
        out.append(y)
    return out


def _out_linear(taps, attn_output, w, b, tgt_len, bsz):
    """The out-projection on the (tgt_len * bsz, E) head outputs, tapped as (tgt_len, bsz, E)."""
    taps.a('o', attn_output.view(tgt_len, bsz, attn_output.size(-1)))
    y = F.linear(attn_output, w, b)
    taps.g('o', y, tgt_len, bsz)
    return y
