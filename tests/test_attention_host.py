"""CPU tests of `precondition_attention`: the restated training forward of `KFACMultiheadAttention` is bitwise equal
to stock `nn.MultiheadAttention` (outputs, attention weights, every parameter gradient), the class swap keeps the
module's identity, and the registration (names, skipping, refusals, the out_proj leaf)."""
import copy
import itertools
import pickle

import pytest
import torch
from torch import nn

from conftest import ROOT  # noqa: F401  (puts the repository on sys.path)


class _Recorder:
    """Stands in for the preconditioner: every projection is tapped, the taps record (which, side, shape, stride)."""

    def __init__(self, keys):
        self.keys, self.calls = keys, []

    def _active_attention_taps(self, module):
        return self.keys

    def _attention_input(self, key, x):
        self.calls.append((key, 'a', tuple(x.shape)))

    def _attention_grad_output(self, key, g):
        self.calls.append((key, 'g', tuple(g.shape)))


def _bound(mha, keys='qkvo'):
    from kfac_b200 import attention
    twin = copy.deepcopy(mha)
    rec = _Recorder({k: k for k in keys})
    attention.bind(twin, rec)
    return twin, rec


def _run(m, q, k, v, kw, seed):
    torch.manual_seed(seed)
    out, w = m(q, k, v, **kw)
    loss = out.pow(2).sum() + (w.sum() * 0.5 if w is not None else 0.0)
    loss.backward()
    return out, w, {n: p.grad.clone() for n, p in m.named_parameters()}


def _inputs(mode, batch_first, unbatched, E, kdim, vdim, L=5, S=7, B=3):
    shape = (lambda n, d: (n, d)) if unbatched else ((lambda n, d: (B, n, d)) if batch_first else (lambda n, d: (n, B, d)))
    q = torch.randn(*shape(L, E), requires_grad=True)
    if mode == 'self':
        return q, q, q, L
    k = torch.randn(*shape(S, kdim), requires_grad=True)
    if mode == 'kv':
        return q, k, k, S
    return q, k, torch.randn(*shape(S, vdim), requires_grad=True), S


CASES = [c for c in itertools.product(
    [False, True],                         # batch_first
    ['self', 'kv', 'qkv'],                 # which inputs are the same tensor
    [(True, True), (True, False), (False, True)],   # need_weights, average_attn_weights
    ['none', 'attn2d', 'attn3d_float', 'kpm', 'causal'],
    [True, False],                         # bias
)]


@pytest.mark.parametrize('batch_first,mode,weights,mask,bias', CASES)
def test_restated_forward_is_bitwise(batch_first, mode, weights, mask, bias):
    E, H, B, L = 8, 2, 3, 5
    torch.manual_seed(0)
    mha = nn.MultiheadAttention(E, H, bias=bias, batch_first=batch_first)
    q, k, v, S = _inputs(mode, batch_first, False, E, E, E, L=L, B=B)
    if mode == 'self':
        S = L
    kw = {'need_weights': weights[0], 'average_attn_weights': weights[1]}
    if mask == 'attn2d':
        kw['attn_mask'] = torch.rand(L, S) > 0.7
    elif mask == 'attn3d_float':
        kw['attn_mask'] = torch.randn(B * H, L, S)
    elif mask == 'kpm':
        kpm = torch.zeros(B, S, dtype=torch.bool)
        kpm[:, -1] = True
        kw['key_padding_mask'] = kpm
    elif mask == 'causal':
        kw['attn_mask'] = nn.Transformer.generate_square_subsequent_mask(L)[:, :S] if S == L else torch.zeros(L, S)
        kw['is_causal'] = S == L
    tapped, rec = _bound(mha)
    ref = _run(mha, q, k, v, kw, 1)
    for t in (q, k, v):
        t.grad = None
    got = _run(tapped, q, k, v, kw, 1)
    assert torch.equal(ref[0], got[0])
    assert (ref[1] is None and got[1] is None) or torch.equal(ref[1], got[1])
    for n in ref[2]:
        assert torch.equal(ref[2][n], got[2][n]), n
    # every projection tapped once on each side, in the sequence-first (L, B, features) layout
    seen = {(key, side): shape for key, side, shape in rec.calls}
    assert len(rec.calls) == 8
    assert seen[('q', 'a')] == (L, B, E) and seen[('q', 'g')] == (L, B, E)
    assert seen[('k', 'a')] == (S, B, E) and seen[('v', 'g')] == (S, B, E)
    assert seen[('o', 'a')] == (L, B, E) and seen[('o', 'g')] == (L, B, E)


@pytest.mark.parametrize('batch_first,unbatched,mode,need_weights,dropout', [
    (False, False, 'qkv', True, 0.0), (True, False, 'kv', False, 0.0), (True, False, 'qkv', True, 0.0),
    (False, True, 'self', True, 0.0), (True, True, 'qkv', False, 0.0), (False, True, 'kv', False, 0.0),
    (True, False, 'self', True, 0.3), (False, False, 'qkv', False, 0.3), (True, False, 'kv', True, 0.3)])
def test_restated_forward_kdim_vdim_unbatched_dropout(batch_first, unbatched, mode, need_weights, dropout):
    E, H = 8, 2
    kdim, vdim = (E, E) if mode == 'self' else (6, 6 if mode == 'kv' else 5)
    torch.manual_seed(0)
    mha = nn.MultiheadAttention(E, H, dropout=dropout, batch_first=batch_first, kdim=kdim, vdim=vdim)
    q, k, v, S = _inputs(mode, batch_first, unbatched, E, kdim, vdim)
    tapped, rec = _bound(mha)
    kw = {'need_weights': need_weights}
    ref = _run(mha, q, k, v, kw, 5)
    for t in (q, k, v):
        t.grad = None
    got = _run(tapped, q, k, v, kw, 5)
    assert torch.equal(ref[0], got[0])
    assert (ref[1] is None and got[1] is None) or torch.equal(ref[1], got[1])
    for n in ref[2]:
        assert torch.equal(ref[2][n], got[2][n]), n
    assert len(rec.calls) == 8


def test_partial_taps_and_stock_path():
    from kfac_b200.attention import KFACMultiheadAttention
    torch.manual_seed(0)
    mha = nn.MultiheadAttention(8, 2)
    tapped, rec = _bound(mha, keys='qv')
    x = torch.randn(4, 2, 8)
    tapped(x, x, x)[0].sum().backward()
    assert sorted((k, s) for k, s, _ in rec.calls) == [('q', 'a'), ('q', 'g'), ('v', 'a'), ('v', 'g')]
    rec.calls.clear()
    tapped.eval()
    tapped(x, x, x)
    tapped.train()
    with torch.no_grad():
        tapped(x, x, x)
    assert rec.calls == []
    # a module whose preconditioner is gone (or a copy that was never bound) runs the stock forward
    plain = copy.deepcopy(tapped)
    assert type(plain) is KFACMultiheadAttention
    plain(x, x, x)[0].sum().backward()
    assert rec.calls == []


def test_class_swap_keeps_identity():
    from kfac_b200.preconditioner import KFACPreconditioner
    from kfac_b200.attention import KFACMultiheadAttention
    torch.manual_seed(0)
    model = nn.TransformerEncoderLayer(16, 4, 32, batch_first=True)
    params = dict(model.named_parameters())
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    pre = KFACPreconditioner(model, precondition_attention=True)
    attn = model.self_attn
    assert type(attn) is KFACMultiheadAttention and isinstance(attn, nn.MultiheadAttention)
    assert dict(model.named_parameters()) == params
    assert model.state_dict().keys() == sd.keys()
    assert all(torch.equal(model.state_dict()[k], sd[k]) for k in sd)
    assert set(vars(attn)) == set(vars(nn.MultiheadAttention(16, 4, batch_first=True)))
    for clone in (copy.deepcopy(model), pickle.loads(pickle.dumps(model))):
        assert type(clone.self_attn) is KFACMultiheadAttention
        assert all(torch.equal(clone.state_dict()[k], sd[k]) for k in sd)
    # eval: the stock forward (no tap, so no device is needed)
    model.eval()
    x = torch.randn(2, 5, 16)
    assert torch.equal(model(x), pickle.loads(pickle.dumps(model))(x))
    del pre
    # the attention refers to its preconditioner weakly (the hooks of the other layers hold it strongly)
    import gc
    import weakref
    solo = nn.MultiheadAttention(16, 4)
    ref = weakref.ref(KFACPreconditioner(solo, precondition_attention=True))
    gc.collect()
    assert ref() is None and type(solo) is KFACMultiheadAttention
    solo(x, x, x)[0].sum().backward()       # stock forward once the preconditioner is gone


class _Block(nn.Module):
    def __init__(self, **kw):
        super().__init__()
        self.attn = nn.MultiheadAttention(16, 4, **kw)
        self.fc = nn.Linear(16, 16)

    def forward(self, x):
        return self.fc(self.attn(x, x, x)[0])


def _names(pre):
    return [n for n, _ in pre._layers.values()]


def test_registration():
    from kfac_b200.layers import AttentionProjectionHelper
    from kfac_b200.preconditioner import KFACPreconditioner
    off = KFACPreconditioner(_Block())
    assert _names(off) == ['attn.out_proj', 'fc']           # unchanged: the out_proj leaf as a Linear
    on = KFACPreconditioner(_Block(), precondition_attention=True)
    assert _names(on) == ['attn.q_proj', 'attn.k_proj', 'attn.v_proj', 'attn.out_proj', 'fc']
    assert [l.index for _, l in on._layers.values()] == [0, 1, 2, 3, 4]
    assert all(isinstance(k, AttentionProjectionHelper) for k in list(on._layers)[:4])
    assert [(l.a_factor_shape, l.g_factor_shape) for _, l in on._layers.values()][:4] == [((17, 17), (16, 16))] * 4
    assert on._defaults['precondition_attention'] is True and 'precondition_attention=True,' in repr(on)
    assert off._defaults['precondition_attention'] is False
    sep = KFACPreconditioner(_Block(kdim=6, vdim=5, bias=False), precondition_attention=True)
    assert [l.a_factor_shape[0] for _, l in sep._layers.values()] == [16, 6, 5, 16, 17]
    # skipping: the attention by name or class (out_proj is still never a leaf), one projection by name
    assert _names(KFACPreconditioner(_Block(), precondition_attention=True, skip_layers=['attn'])) == ['fc']
    assert _names(KFACPreconditioner(_Block(), precondition_attention=True,
                                     skip_layers=['MultiheadAttention'])) == ['fc']
    assert _names(KFACPreconditioner(_Block(), precondition_attention=True, skip_layers=[r'attn\.k_proj'])) == [
        'attn.q_proj', 'attn.v_proj', 'attn.out_proj', 'fc']
    frozen = _Block()
    frozen.attn.in_proj_bias.requires_grad_(False)
    assert _names(KFACPreconditioner(frozen, precondition_attention=True)) == ['fc']


def test_gradient_views():
    from kfac_b200.layers import AttentionProjectionHelper
    m = nn.MultiheadAttention(8, 2)
    m.in_proj_weight.grad = torch.arange(24 * 8.).view(24, 8)
    m.in_proj_bias.grad = torch.arange(24.)
    k = AttentionProjectionHelper(m, 'k')
    w = k.get_weight_grad()
    assert w.is_contiguous() and w.data_ptr() == m.in_proj_weight.grad[8].data_ptr() and w.shape == (8, 8)
    assert torch.equal(k.get_bias_grad(), torch.arange(8., 16.))
    sep = nn.MultiheadAttention(8, 2, kdim=3, vdim=3)
    sep.v_proj_weight.grad = torch.ones(8, 3)
    sep.in_proj_bias.grad = torch.arange(24.)
    v = AttentionProjectionHelper(sep, 'v')
    assert v.get_weight_grad() is sep.v_proj_weight.grad and torch.equal(v.get_bias_grad(), torch.arange(16., 24.))
    assert v.get_grad().shape == (8, 4)


def test_reduce_rows():
    from kfac_b200.layers import AttentionProjectionHelper, _strided_rows
    h = AttentionProjectionHelper(nn.MultiheadAttention(8, 2), 'q', reduce=True)
    assert h._positions(torch.zeros(5, 3, 8)) == (3, 5) and h.num_rows_a(torch.zeros(5, 3, 8)) == 3
    assert h._positions(torch.zeros(1, 3, 8)) is None            # one position: the expand rows
    assert h.num_rows_a(torch.zeros(5, 1, 8)) == 1                # unbatched: one example
    assert AttentionProjectionHelper(nn.MultiheadAttention(8, 2), 'q').num_rows_a(torch.zeros(5, 3, 8)) == 15
    packed = torch.zeros(5, 3, 24)
    r, ld = _strided_rows(packed[..., 8:16], ordered=True)
    assert r.shape == (15, 8) and ld == 24 and r.data_ptr() == packed[..., 8:16].data_ptr()
    bf = torch.zeros(3, 5, 8)
    r, ld = _strided_rows(bf.transpose(0, 1), ordered=False)
    assert ld == 8 and r.data_ptr() == bf.data_ptr()
    r, ld = _strided_rows(bf.transpose(0, 1), ordered=True)        # EKFAC rows keep the (L, B) order: a copy
    assert ld == 8 and r.data_ptr() != bf.data_ptr()


@pytest.mark.parametrize('kw,match', [
    (dict(model_kw=dict(add_bias_kv=True)), 'add_bias_kv'),
    (dict(model_kw=dict(add_zero_attn=True)), 'add_zero_attn'),
    (dict(diagonal_g_layers=['attn']), 'diagonal_g_layers'),
    (dict(diagonal_g_layers=['MultiheadAttention']), 'diagonal_g_layers'),
    (dict(diagonal_g_layers=[r'v_proj']), 'diagonal_g_layers'),
    (dict(tie=True), 'shares a weight'),
])
def test_refusals(kw, match):
    from kfac_b200.preconditioner import KFACPreconditioner
    model = _Block(**kw.pop('model_kw', {}))
    if kw.pop('tie', False):
        model.fc.weight = model.attn.out_proj.weight
    with pytest.raises(ValueError, match=match) as e:
        KFACPreconditioner(model, precondition_attention=True, **kw)
    assert 'skip_layers' in str(e.value)
    # skipping the attention is the way out
    KFACPreconditioner(_Block(**({} if 'bias' in match or 'zero' in match else {})), precondition_attention=True,
                       skip_layers=['attn'], **kw)


def test_subclass_refused():
    from kfac_b200.preconditioner import KFACPreconditioner

    class MyAttention(nn.MultiheadAttention):
        pass

    model = _Block()
    model.attn = MyAttention(16, 4)
    with pytest.raises(ValueError, match='skip_layers'):
        KFACPreconditioner(model, precondition_attention=True)
