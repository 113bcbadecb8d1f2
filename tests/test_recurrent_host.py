"""CPU tests of `precondition_recurrent`: the restated forward of `KFACRNN` / `KFACLSTM` / `KFACGRU` matches stock
`nn.RNN` / `nn.LSTM` / `nn.GRU` (outputs, final states, every parameter gradient), the taps give exactly the rows whose
outer products sum to each sub-layer's `[weight.grad | bias.grad]`, and the module plumbing (class swap, registration
names and factor shapes, skipping, refusals, state_dict).

`ref_rows` / `ref_reduce` are the fp64 restatement of the native row writers that the GPU tests compare against."""
import copy
import itertools
import pickle
import types

import pytest
import torch
from torch import nn
from torch.nn.utils.rnn import pack_padded_sequence

from conftest import ROOT  # noqa: F401  (puts the repository on sys.path)

MODES = ['RNN_TANH', 'RNN_RELU', 'LSTM', 'GRU']


def make(mode, *args, **kw):
    if mode.startswith('RNN'):
        return nn.RNN(*args, nonlinearity=mode[4:].lower(), **kw)
    return {'LSTM': nn.LSTM, 'GRU': nn.GRU}[mode](*args, **kw)


def _positions(tap):
    """[(t, b, row)] in row order, and the batch size of every step."""
    T, B = tap.T, tap.B
    if tap.offsets is None:
        offs = [t * B for t in range(T + 1)]
    else:
        offs = [int(v) for v in tap.offsets.cpu().tolist()]
    bs = [offs[t + 1] - offs[t] for t in range(T)]
    return [(t, b, offs[t] + b) for t in range(T) for b in range(bs[t])], offs, bs


def ref_rows(x, tap, feat, ones):
    """The rows of one tap (fp64, N x (feat + ones)): kfac_rows_sequence's rows for the row source `tap`."""
    X = x.detach().double().reshape(-1, x.size(-1))[:, tap.col0:tap.col0 + feat]
    pos, offs, bs = _positions(tap)
    src = X
    if tap.shift:
        src = torch.cat([X, tap.h0.detach().double()])       # row N + b: h0[b]
    N = X.shape[0]
    idx = []
    for t, b, r in pos:
        if tap.shift == 1:
            idx.append(N + b if t == 0 else offs[t - 1] + b)
        elif tap.shift == -1:
            idx.append(offs[t + 1] + b if t + 1 < tap.T and b < bs[t + 1] else N + b)
        else:
            idx.append(r)
    rows = src[torch.tensor(idx, device=src.device)]
    if tap.mul is not None:
        mul = tap.mul.detach().double().reshape(-1, tap.mul.size(-1))
        rows = torch.cat([rows[:, :tap.mul_col0], rows[:, tap.mul_col0:] * mul[[r for _, _, r in pos]]], 1)
    return torch.cat([rows, rows.new_ones(rows.shape[0], ones)], 1)


def ref_reduce(x, tap, feat, ones, power):
    """kfac_reduce_rows_sequence's rows (fp64, B x (feat + ones)): the sum of each sequence's rows times R_b^-power."""
    rows = ref_rows(x, tap, feat, ones)
    pos, _, _ = _positions(tap)
    out = rows.new_zeros(tap.B, feat + ones)
    count = [0] * tap.B
    for (t, b, r) in pos:
        out[b] += rows[r]
        count[b] += 1
    return out * torch.tensor(count, dtype=torch.float64, device=rows.device).pow(-power)[:, None]


class _Recorder:
    """Stands in for the preconditioner: every sub-layer is tapped, the taps keep (tensor, SequenceTap)."""

    def __init__(self, names):
        self.keys = {n: types.SimpleNamespace(suffix=n) for n in names}
        self.a, self.g = {}, {}

    def _active_recurrent_taps(self, module):
        return self.keys

    def _recurrent_input(self, key, x, tap):
        self.a[key.suffix] = (x.detach().clone(), tap)

    def _recurrent_grad_output(self, key, g, tap):
        self.g[key.suffix] = (g.detach().clone(), tap)


def sublayers(m):
    return [f'{s}_l{k}' + ('_reverse' if d else '') for k in range(m.num_layers)
            for d in range(2 if m.bidirectional else 1) for s in ('ih', 'hh')]


def bound(m, names=None):
    from kfac_b200 import recurrent
    twin = copy.deepcopy(m)
    rec = _Recorder(sublayers(m) if names is None else names)
    recurrent.bind(twin, rec)
    return twin, rec


def inputs(kind, batch_first, I, dtype, seed=0):
    """(module input, the tensor the loss weights come from): 'batched', 'unbatched', 'sorted' / 'unsorted' packed."""
    g = torch.Generator().manual_seed(seed)
    T, B = 5, 4
    if kind == 'unbatched':
        return torch.randn(T, I, generator=g, dtype=dtype), None
    x = torch.randn(B, T, I, generator=g, dtype=dtype) if batch_first else torch.randn(T, B, I, generator=g, dtype=dtype)
    if kind == 'batched':
        return x, None
    lengths = torch.tensor([5, 3, 3, 1]) if kind == 'sorted' else torch.tensor([2, 5, 1, 4])
    return pack_padded_sequence(x, lengths, batch_first=batch_first, enforce_sorted=kind == 'sorted'), lengths


def hidden(m, kind, dtype, seed=1):
    g = torch.Generator().manual_seed(seed)
    D = 2 if m.bidirectional else 1
    shape = (m.num_layers * D, m.hidden_size) if kind == 'unbatched' else (m.num_layers * D, 4, m.hidden_size)
    h = torch.randn(*shape, generator=g, dtype=dtype, requires_grad=True)
    if isinstance(m, nn.LSTM):
        return (h, torch.randn(*shape, generator=g, dtype=dtype, requires_grad=True))
    return h


def _loss(out, hid, seed=2):
    """A fixed random linear functional of every output."""
    g = torch.Generator().manual_seed(seed)
    data = out.data if hasattr(out, 'batch_sizes') else out
    parts = [data] + (list(hid) if isinstance(hid, tuple) else [hid])
    return sum((p * torch.randn(p.shape, generator=g, dtype=p.dtype)).sum() for p in parts)


def _run(m, x, hx):
    hx_ = None if hx is None else (tuple(h.detach().clone().requires_grad_() for h in hx) if isinstance(hx, tuple)
                                   else hx.detach().clone().requires_grad_())
    out, hid = m(x) if hx_ is None else m(x, hx_)
    _loss(out, hid).backward()
    grads = {n: p.grad.clone() for n, p in m.named_parameters()}
    hgrads = [] if hx_ is None else [h.grad for h in (hx_ if isinstance(hx_, tuple) else (hx_,))]
    data = out.data if hasattr(out, 'batch_sizes') else out
    return data, (hid if isinstance(hid, tuple) else (hid,)), grads, hgrads


def _close(a, b, tol):
    a, b = a.double(), b.double()
    den = max(b.abs().max().item(), 1e-30)
    return (a - b).abs().max().item() / den <= tol


CASES = list(itertools.product(MODES, [1, 2], [False, True], [True, False], [False, True],
                               ['batched', 'unbatched', 'sorted', 'unsorted'], [False, True]))


@pytest.mark.parametrize('dtype,tol', [(torch.float64, 1e-12), (torch.float32, 1e-6)])
@pytest.mark.parametrize('mode', MODES)
def test_restated_forward_matches_stock(dtype, tol, mode):
    """Outputs, h_n / c_n, every parameter gradient and the hx gradients against the stock module, over layers x
    bidirectional x bias x batch_first x (batched, unbatched, packed sorted / unsorted) x hx given or absent."""
    for _, L, bidir, bias, bf, kind, with_hx in (c for c in CASES if c[0] == mode):
        torch.manual_seed(0)
        m = make(mode, 3, 6, num_layers=L, bidirectional=bidir, bias=bias, batch_first=bf).to(dtype)
        x, _ = inputs(kind, bf, 3, dtype)
        hx = hidden(m, kind, dtype) if with_hx else None
        twin, rec = bound(m)
        ref = _run(m, x, hx)
        got = _run(twin, x, hx)
        case = (mode, L, bidir, bias, bf, kind, with_hx)
        assert rec.a and len(rec.g) == len(rec.a), case         # the restated forward ran
        assert got[0].shape == ref[0].shape and _close(got[0], ref[0], tol), case
        for a, b in zip(got[1], ref[1]):
            assert a.shape == b.shape and _close(a, b, tol), case
        for n in ref[2]:
            assert _close(got[2][n], ref[2][n], tol), (case, n)
        for a, b in zip(got[3], ref[3]):
            assert _close(a, b, tol), case


@pytest.mark.parametrize('mode', MODES)
def test_tap_rows_give_the_weight_gradients(mode):
    """For every sub-layer, sum_rows g a^T over the tapped tensors (rows reassembled by the fp64 restatement of the
    gather and the GRU rule) equals [weight.grad | bias.grad] (fp64)."""
    for _, L, bidir, bias, bf, kind, with_hx in (c for c in CASES if c[0] == mode):
        torch.manual_seed(0)
        m = make(mode, 3, 6, num_layers=L, bidirectional=bidir, bias=bias, batch_first=bf).double()
        x, _ = inputs(kind, bf, 3, torch.float64)
        hx = hidden(m, kind, torch.float64) if with_hx else None
        twin, rec = bound(m)
        _, _, grads, _ = _run(twin, x, hx)
        for name in sublayers(m):
            xa, ta = rec.a[name]
            gg, tg = rec.g[name]
            w = grads['weight_' + name]
            A = ref_rows(xa, ta, w.size(1), int(bias))
            G = ref_rows(gg, tg, w.size(0), 0)
            want = torch.cat([w, grads['bias_' + name][:, None]], 1) if bias else w
            assert A.shape[0] == G.shape[0]
            assert _close(G.t() @ A, want, 1e-12), (mode, L, bidir, bias, bf, kind, with_hx, name)


def test_reduce_reference_counts_sequence_lengths():
    """ref_reduce: packed sequences are reduced over their own lengths, in sorted order."""
    from kfac_b200.recurrent import SequenceTap
    x = torch.arange(8.).view(8, 1)          # batch sizes 3, 3, 1, 1
    tap = SequenceTap(4, 3, torch.tensor([0, 3, 6, 7, 8], dtype=torch.int32))
    r = ref_reduce(x, tap, 1, 1, 1.0)
    assert torch.equal(r, torch.tensor([[(0 + 3 + 6 + 7) / 4, 1.], [(1 + 4) / 2, 1.], [(2 + 5) / 2, 1.]],
                                       dtype=torch.float64))


def test_partial_taps_and_stock_path():
    """Only the registered sub-layers are tapped; eval and no-grad calls run the stock forward."""
    m = nn.LSTM(3, 4, num_layers=2, bidirectional=True)
    twin, rec = bound(m, ['hh_l1_reverse', 'ih_l0'])
    x = torch.randn(5, 2, 3)
    out, _ = twin(x)
    out.sum().backward()
    assert set(rec.a) == set(rec.g) == {'hh_l1_reverse', 'ih_l0'}
    twin.eval()
    rec.a.clear()
    assert torch.equal(twin(x)[0], m.eval()(x)[0]) and not rec.a
    twin.train()
    with torch.no_grad():
        twin(x)
    assert not rec.a


def test_dropout_runs_between_layers():
    torch.manual_seed(0)
    m = nn.GRU(3, 4, num_layers=3, dropout=0.5)
    twin, rec = bound(m)
    out, _ = twin(torch.randn(6, 2, 3))
    out.sum().backward()
    assert all(p.grad is not None for p in twin.parameters())


# ---------------------------------------------------------------------------------------------- module plumbing
class _Model(nn.Module):
    def __init__(self, mode='LSTM', **kw):
        super().__init__()
        self.emb = nn.Linear(4, 8)
        self.rnn = make(mode, 8, 16, **kw)
        self.head = nn.Linear(16 * (2 if kw.get('bidirectional') else 1), 3)

    def forward(self, x):
        return self.head(self.rnn(self.emb(x))[0])


def _names(pre):
    return [n for n, _ in pre._layer_list()]


def test_off_switch_keeps_todays_registered_set():
    from kfac_b200.preconditioner import KFACPreconditioner
    model = _Model(num_layers=2, bidirectional=True)
    pre = KFACPreconditioner(model)
    assert _names(pre) == ['emb', 'head'] and type(model.rnn) is nn.LSTM
    assert pre._defaults['precondition_recurrent'] is False


def test_registration_names_and_shapes():
    from kfac_b200.preconditioner import KFACPreconditioner
    for mode, gates in (('RNN_TANH', 1), ('LSTM', 4), ('GRU', 3)):
        model = _Model(mode, num_layers=2, bidirectional=True)
        pre = KFACPreconditioner(model, precondition_recurrent=True)
        names = _names(pre)
        subs = [f'rnn.{s}_l{k}{sfx}' for k in range(2) for sfx in ('', '_reverse') for s in ('ih', 'hh')]
        assert sorted(names) == sorted(['emb', 'head'] + subs), mode
        layers = dict(pre._layer_list())
        assert layers['rnn.ih_l0'].a_factor_shape == (9, 9)
        assert layers['rnn.ih_l1_reverse'].a_factor_shape == (33, 33)     # 2H + 1: bidirectional layer input
        assert layers['rnn.hh_l1'].a_factor_shape == (17, 17)
        assert layers['rnn.ih_l0'].g_factor_shape == layers['rnn.hh_l0'].g_factor_shape == (16 * gates,) * 2
        assert pre._defaults['precondition_recurrent'] is True
    nob = KFACPreconditioner(_Model('GRU', bias=False), precondition_recurrent=True)
    assert dict(nob._layer_list())['rnn.hh_l0'].a_factor_shape == (16, 16)


def test_skip_layers():
    from kfac_b200.preconditioner import KFACPreconditioner
    assert _names(KFACPreconditioner(_Model(), precondition_recurrent=True, skip_layers=['rnn'])) == ['emb', 'head']
    assert _names(KFACPreconditioner(_Model(), precondition_recurrent=True, skip_layers=['LSTM'])) == ['emb', 'head']
    model = _Model(num_layers=2, bidirectional=True)
    pre = KFACPreconditioner(model, precondition_recurrent=True, skip_layers=[r'rnn\.hh_l1_reverse'])
    assert 'rnn.hh_l1_reverse' not in _names(pre) and 'rnn.ih_l1_reverse' in _names(pre)
    assert type(model.rnn).__name__ == 'KFACLSTM'
    every = '|'.join(rf'rnn\.{s}_l0' for s in ('ih', 'hh'))
    model = _Model()
    KFACPreconditioner(model, precondition_recurrent=True, skip_layers=[every])
    assert type(model.rnn) is nn.LSTM            # nothing registered: no class swap
    frozen = _Model()
    frozen.rnn.weight_hh_l0.requires_grad_(False)
    assert _names(KFACPreconditioner(frozen, precondition_recurrent=True)) == ['emb', 'head']


class _SubLSTM(nn.LSTM):
    pass


class _Shared(nn.Module):
    def __init__(self):
        super().__init__()
        self.rnn = nn.GRU(8, 8)
        self.fc = nn.Linear(8, 24)
        self.fc.weight = self.rnn.weight_ih_l0

    def forward(self, x):
        return self.fc(self.rnn(x)[0])


@pytest.mark.parametrize('build,kw,match', [
    (lambda: _Model(proj_size=4), {}, 'proj_size'),
    (lambda: nn.LSTM(8, 2049), {}, 'KFAC_EIGH_MAX_N'),
    (lambda: nn.GRU(8, 2731), {}, 'KFAC_EIGH_MAX_N'),
    (lambda: _Model(), {'diagonal_g_layers': [r'rnn\.hh_l0']}, 'diagonal_g_layers'),
    (lambda: _Model(), {'diagonal_g_layers': ['LSTM']}, 'diagonal_g_layers'),
    (_Shared, {}, 'shares a weight'),
    (lambda: _SubLSTM(4, 4), {}, 'subclass'),
])
def test_refusals(build, kw, match):
    from kfac_b200.preconditioner import KFACPreconditioner
    with pytest.raises(ValueError, match=match) as e:
        KFACPreconditioner(build(), precondition_recurrent=True, **kw)
    assert 'skip_layers' in str(e.value)


def test_largest_accepted_widths():
    from kfac_b200.layers import register_modules
    from kfac_b200.enums import ComputeMethod
    for m in (nn.LSTM(8, 2048), nn.GRU(8, 2730)):
        assert len(register_modules(m, [], precondition_recurrent=True, method=ComputeMethod.EIGEN)) == 2


def test_class_swap_keeps_identity():
    from kfac_b200.preconditioner import KFACPreconditioner
    from kfac_b200.recurrent import KFACGRU, KFACLSTM, KFACRNN
    for mode, cls in (('RNN_RELU', KFACRNN), ('LSTM', KFACLSTM), ('GRU', KFACGRU)):
        torch.manual_seed(0)
        model = _Model(mode, num_layers=2)
        params = dict(model.named_parameters())
        sd = {k: v.clone() for k, v in model.state_dict().items()}
        pre = KFACPreconditioner(model, precondition_recurrent=True)
        rnn = model.rnn
        assert type(rnn) is cls and isinstance(rnn, type(make(mode, 1, 1)))
        assert rnn.mode == mode and dict(model.named_parameters()) == params
        assert model.state_dict().keys() == sd.keys()
        assert set(vars(rnn)) == set(vars(make(mode, 8, 16, num_layers=2)))
        for clone in (copy.deepcopy(model), pickle.loads(pickle.dumps(model))):
            assert type(clone.rnn) is cls
            assert all(torch.equal(clone.state_dict()[k], sd[k]) for k in sd)
        model.eval()
        x = torch.randn(5, 2, 4)
        assert torch.equal(model(x), pickle.loads(pickle.dumps(model))(x))
        fresh = _Model(mode, num_layers=2)
        fresh.load_state_dict(model.state_dict())
        assert all(torch.equal(fresh.state_dict()[k], model.state_dict()[k]) for k in sd)
        del pre


def test_preconditioner_state_dict_names():
    """The state_dict keys are the sub-layer names; a preconditioner without the keyword refuses it (the GPU test
    loads the factors back)."""
    from kfac_b200.preconditioner import KFACPreconditioner
    sd = KFACPreconditioner(_Model('GRU', bidirectional=True), precondition_recurrent=True).state_dict()
    names = sorted(sd['layers'])
    assert names == sorted(['emb', 'head'] + [f'rnn.{s}_l0{sfx}' for sfx in ('', '_reverse') for s in ('ih', 'hh')])
    with pytest.raises(ValueError):
        KFACPreconditioner(_Model('GRU', bidirectional=True)).load_state_dict(sd, compute_inverses=False)
