"""`precondition_recurrent` on the GPU:

  * the sequence row writers (kfac_rows_sequence, kfac_reduce_rows_sequence) against the fp64 restatement of
    tests/test_recurrent_host.py for f32 / f16 / bf16, time-major and packed, the row itself and the forward / reverse
    hidden-state gather, the GRU multiplier and ones in {0, 1}; the gather of a forward direction gives the bits of
    kfac_rows_linear on torch.cat((h0, out[:-1])), and the factor from its rows those of kfac_factor_linear on it;
  * RNN, LSTM and GRU models under EIGEN / INVERSE / EKFAC x expand / reduce, packed and unpacked: A, G (and S) and
    every preconditioned gradient against an fp64 restatement from the tapped tensors;
  * stock nn.LSTM against its unrolled twin written with nn.Linear modules (an ih Linear over the sequence, an hh
    Linear called per step): P of every sub-layer agrees under expand EIGEN and INVERSE;
  * the restated forward against cuDNN, non-factor steps bit for bit cuDNN;
  * fp16 autocast with a GradScaler, accumulation_steps=2, a factor / inverse schedule and factor_dtype=bf16;
  * skipped sub-layers keep their gradients bit for bit, and the keyword leaves other layers' factors bit for bit;
  * two ranks (tests/dist_recurrent.py).
"""
import copy
import ctypes as C

import pytest
import torch
from torch import nn
from torch.nn.utils.rnn import pack_padded_sequence

from conftest import rel_fro
from test_recurrent_host import make, ref_reduce, ref_rows

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda')
DTYPES = [torch.float32, torch.float16, torch.bfloat16]


@pytest.fixture(scope='module')
def lib():
    from kfac_b200 import _cabi
    return _cabi.load()


def S():
    return torch.cuda.current_stream().cuda_stream


def _code(dtype):
    from kfac_b200 import _cabi
    return _cabi.DTYPE_CODE[dtype]


def _src(x, tap, keep):
    from kfac_b200 import _cabi
    keep += [x, tap.h0, tap.mul, tap.offsets]
    return _cabi.SequenceRows(x.data_ptr(), x.size(-1), tap.col0,
                              tap.h0.data_ptr() if tap.h0 is not None else None,
                              tap.h0.size(-1) if tap.h0 is not None else 0, tap.shift,
                              tap.mul.data_ptr() if tap.mul is not None else None,
                              tap.mul.size(-1) if tap.mul is not None else 0, tap.mul_col0, tap.T, tap.B,
                              tap.offsets.data_ptr() if tap.offsets is not None else None)


def _tap(T, B, packed, shift, D, H, dtype, mul, seed=0):
    """(x, tap, feat): a layer output (or gradient) of D directions of H columns and the tap of direction D - 1."""
    from kfac_b200.recurrent import SequenceTap
    g = torch.Generator().manual_seed(seed)
    offsets, N = None, T * B
    if packed:
        lengths = sorted([T] + [int(v) for v in torch.randint(1, T + 1, (B - 1,), generator=g)], reverse=True)
        bs = [sum(1 for n in lengths if n > t) for t in range(T)]
        offs = [0]
        for n in bs:
            offs.append(offs[-1] + n)
        offsets, N = torch.tensor(offs, dtype=torch.int32, device=DEV), offs[-1]
    x = (torch.randn(N, D * H, generator=g) * 3).to(DEV, dtype)
    h0 = (torch.randn(B, H, generator=g)).to(DEV, dtype) if shift else None
    m = torch.rand(N, H // 3, generator=g).to(DEV, dtype) if mul else None
    tap = SequenceTap(T, B, offsets, h0, shift, (D - 1) * H, m, H - H // 3 if mul else 0)
    return (x if packed else x.view(T, B, D * H)), tap, H


@pytest.mark.parametrize('mul', [False, True])
@pytest.mark.parametrize('shift', [0, 1, -1])
@pytest.mark.parametrize('packed', [False, True])
@pytest.mark.parametrize('dtype', DTYPES)
def test_row_writers_against_fp64(lib, dtype, packed, shift, mul):
    for ones in (0, 1):
        for T, B, D, H in ((7, 5, 2, 48), (40, 9, 1, 96)):
            x, tap, feat = _tap(T, B, packed, shift, D, H, dtype, mul)
            keep = []
            src = _src(x, tap, keep)
            d = feat + ones
            ld = (d + 3) // 4 * 4
            N = x.numel() // x.size(-1)
            out = torch.full((N, ld), float('nan'), device=DEV)
            loss = torch.tensor([4.0], device=DEV)
            assert lib.kfac_rows_sequence(C.byref(src), _code(dtype), feat, ones, 0.5, loss.data_ptr(),
                                          out.data_ptr(), ld, S()) == 0
            want = ref_rows(x, tap, feat, ones) * (0.5 / 4.0)
            assert torch.equal(out[:, d:], torch.zeros_like(out[:, d:]))
            assert rel_fro(out[:, :d], want) <= 1e-6, (T, B, ones)
            for power in (1.0, 0.5):
                red = torch.full((B, ld), float('nan'), device=DEV)
                assert lib.kfac_reduce_rows_sequence(C.byref(src), _code(dtype), feat, ones, 0.5, power, None,
                                                     red.data_ptr(), ld, S()) == 0
                want = ref_reduce(x, tap, feat, ones, power) * 0.5
                assert rel_fro(red[:, :d], want) <= 1e-6, (T, B, ones, power)
                assert torch.equal(red[:, d:], torch.zeros_like(red[:, d:]))


def test_row_writers_reject_bad_arguments(lib):
    x, tap, feat = _tap(4, 3, False, 1, 1, 8, torch.float32, False)
    keep = []
    out = torch.empty(12, 12, device=DEV)
    bad = [tap._replace(h0=None), tap._replace(shift=2), tap._replace(col0=4)]
    for t in bad:
        assert lib.kfac_rows_sequence(C.byref(_src(x, t, keep)), 0, feat, 1, 1.0, None, out.data_ptr(), 12, S()) == -1
    assert lib.kfac_rows_sequence(C.byref(_src(x, tap, keep)), 0, feat, 1, 1.0, None, out.data_ptr(), 8, S()) == -1
    assert lib.kfac_rows_sequence(C.byref(_src(x, tap, keep)), 7, feat, 1, 1.0, None, out.data_ptr(), 12, S()) == -1


@pytest.mark.parametrize('T,B,H', [(6, 5, 40), (64, 16, 256)])
def test_forward_gather_is_bitwise_rows_linear(lib, T, B, H):
    """The unpacked forward gather is kfac_rows_linear of cat((h0, out[:-1])), bit for bit, and the factor from its rows
    is kfac_factor_linear of that tensor (SIMT and tensor-core paths)."""
    from kfac_b200.recurrent import SequenceTap
    g = torch.Generator().manual_seed(1)
    out = torch.randn(T, B, H, generator=g).to(DEV)
    h0 = torch.randn(B, H, generator=g).to(DEV)
    cat = torch.cat((h0[None], out[:-1])).contiguous()
    keep = []
    src = _src(out, SequenceTap(T, B, None, h0, 1, 0), keep)
    d, N = H + 1, T * B
    ld = (d + 3) // 4 * 4
    mine = torch.empty(N, ld, device=DEV)
    theirs = torch.empty(N, ld, device=DEV)
    assert lib.kfac_rows_sequence(C.byref(src), 0, H, 1, 0.75, None, mine.data_ptr(), ld, S()) == 0
    assert lib.kfac_rows_linear(cat.data_ptr(), 0, N, H, 1, 0.75, None, theirs.data_ptr(), ld, S()) == 0
    assert torch.equal(mine, theirs)
    rows = torch.empty(N, d, device=DEV)
    assert lib.kfac_rows_sequence(C.byref(src), 0, H, 1, 1.0, None, rows.data_ptr(), d, S()) == 0
    fa, fb = torch.zeros(d, d, device=DEV), torch.zeros(d, d, device=DEV)
    for x, feat, ones, acc in ((rows, d, 0, fa), (cat, H, 1, fb)):
        need = lib.kfac_factor_linear_workspace_bytes(N, feat, ones)
        ws = torch.empty(max(need, 1), dtype=torch.uint8, device=DEV)
        assert lib.kfac_factor_linear(x.data_ptr(), 0, N, feat, ones, 1.0 / N, acc.data_ptr(), ws.data_ptr(), need,
                                      S()) == 0
    assert torch.equal(fa, fb)


# ---------------------------------------------------------------------------------------------- module level
class Net(nn.Module):
    def __init__(self, mode, L=2, bidir=True, bias=True, I=24, H=32, batch_first=False):
        super().__init__()
        self.rnn = make(mode, I, H, num_layers=L, bidirectional=bidir, bias=bias, batch_first=batch_first)

    def forward(self, x):
        out = self.rnn(x)[0]
        return out.data if hasattr(out, 'batch_sizes') else out


def _batches(packed, T=9, B=6, I=24, batch_first=False):
    def get(s):
        g = torch.Generator().manual_seed(100 + s)
        x = torch.randn(B, T, I, generator=g) if batch_first else torch.randn(T, B, I, generator=g)
        x = x.to(DEV)
        if packed:
            lengths = torch.randint(1, T + 1, (B,), generator=g)
            lengths[0] = T
            x = pack_padded_sequence(x, lengths, batch_first=batch_first, enforce_sorted=False)
        return x, g
    return get


def _record(pre):
    """Wrap the preconditioner's recurrent taps: suffix -> side -> [(tensor, tap)] of the open window."""
    calls = {}

    def a(key, x, tap, orig=pre._recurrent_input):
        calls.setdefault(key.suffix, {'a': [], 'g': []})['a'].append((x.detach().clone(), tap))
        orig(key, x, tap)

    def g(key, gr, tap, orig=pre._recurrent_grad_output):
        calls.setdefault(key.suffix, {'a': [], 'g': []})['g'].append((gr.detach().clone(), tap))
        orig(key, gr, tap)
    pre._recurrent_input, pre._recurrent_grad_output = a, g
    return calls


def _rows64(helper, x, tap, side, reduce, cast=None):
    ones = int(helper.has_bias()) if side == 'a' else 0
    feat = (helper.a_factor_shape[0] - ones) if side == 'a' else helper.g_factor_shape[0]
    if cast is not None:
        x = x.to(cast)
        tap = tap._replace(h0=tap.h0.to(cast) if tap.h0 is not None else None,
                           mul=tap.mul.to(cast) if tap.mul is not None else None)
    if reduce and tap.T > 1:
        return ref_reduce(x, tap, feat, ones, 1.0 if side == 'a' else 0.5)
    return ref_rows(x, tap, feat, ones)


def _run(model, batches, method, approx, steps, ius=1, acc=1, damping=0.003, alpha=0.9, tol=1e-3, fus=1, kw=None,
         cast=None, ftol=1e-5):
    """Train `steps` steps of sum(model(x) * y) and check every sub-layer's A, G (S under EKFAC) and preconditioned
    gradient against fp64 from the tapped tensors after each."""
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    pre = KFACPreconditioner(model, compute_method=method, kfac_approx=approx, factor_update_steps=fus,
                             inv_update_steps=ius, damping=damping, factor_decay=alpha, kl_clip=None,
                             accumulation_steps=acc, precondition_recurrent=True, **(kw or {}))
    calls = _record(pre)
    A, G, Sm, snap = {}, {}, {}, {}
    reduce = approx == 'reduce'
    eye = lambda n: torch.eye(n, dtype=torch.float64, device=DEV)  # noqa: E731
    opt = torch.optim.SGD(model.parameters(), lr=0.01)
    for s in range(steps):
        opt.zero_grad()
        calls.clear()
        for k in range(acc):
            x, g = batches(s * acc + k)
            out = model(x)
            (out * torch.randn(out.shape, generator=g).to(DEV)).sum().backward()
        grads = {name: l.module.get_grad().detach().double() for name, l in pre._layers.values()}
        pre.step()
        torch.cuda.synchronize()
        for key, (name, layer) in pre._layers.items():
            if s % fus == 0:
                wa = wg = 0.0
                for (xa, ta), (gg, tg) in zip(calls[key.suffix]['a'], calls[key.suffix]['g']):
                    X, Gr = _rows64(key, xa, ta, 'a', reduce, cast), _rows64(key, gg, tg, 'g', reduce, cast)
                    wa = wa + X.T @ X / X.shape[0] / acc
                    wg = wg + Gr.T @ Gr / Gr.shape[0] / acc
                A[name] = alpha * A.get(name, eye(wa.shape[0])) + (1 - alpha) * wa
                G[name] = alpha * G.get(name, eye(wg.shape[0])) + (1 - alpha) * wg
            assert rel_fro(layer._a_view, A[name]) <= ftol, (s, name, 'A', rel_fro(layer._a_view, A[name]))
            assert rel_fro(layer._g_view, G[name]) <= ftol, (s, name, 'G', rel_fro(layer._g_view, G[name]))
            if s % ius == 0:
                da, qa = torch.linalg.eigh(A[name])
                dg, qg = torch.linalg.eigh(G[name])
                snap[name] = (A[name], G[name], da.clamp(min=0), qa, dg.clamp(min=0), qg)
            An, Gn, da, qa, dg, qg = snap[name]
            grad = grads[name]
            if method == 'inverse':
                want = (torch.linalg.inv(Gn + damping * eye(Gn.shape[0])) @ grad
                        @ torch.linalg.inv(An + damping * eye(An.shape[0])))
            elif method == 'eigen':
                want = qg @ ((qg.T @ grad @ qa) / (torch.outer(dg, da) + damping)) @ qa.T
            else:
                Qa, Qg = layer.qa.double(), layer.qg.double()
                if s % fus == 0:
                    (xa, ta), (gg, tg) = calls[key.suffix]['a'][0], calls[key.suffix]['g'][0]
                    X, Gr = _rows64(key, xa, ta, 'a', reduce), _rows64(key, gg, tg, 'g', reduce)
                    Sb = ((Gr @ Qg) ** 2).T @ ((X @ Qa) ** 2) / X.shape[0]
                    Sm[name] = Sb if s % ius == 0 else alpha * Sm[name] + (1 - alpha) * Sb
                assert rel_fro(layer._S[:, :layer.a_dim], Sm[name]) < 1e-4, (s, name, 'S')
                want = Qg @ ((Qg.T @ grad @ Qa) / (Sm[name] + damping)) @ Qa.T
            e = rel_fro(key.get_grad(), want)
            assert e < tol, (s, name, 'P', e)
        opt.step()
    return pre


@pytest.mark.parametrize('packed', [False, True])
@pytest.mark.parametrize('approx', ['expand', 'reduce'])
@pytest.mark.parametrize('method', ['eigen', 'inverse', 'ekfac'])
@pytest.mark.parametrize('mode', ['LSTM', 'GRU', 'RNN_TANH'])
def test_module_against_fp64(mode, method, approx, packed):
    torch.manual_seed(0)
    _run(Net(mode).to(DEV), _batches(packed), method, approx, steps=2)


def test_batch_first_unbiased_relu():
    torch.manual_seed(0)
    _run(Net('RNN_RELU', L=1, bidir=False, bias=False, batch_first=True).to(DEV),
         _batches(False, batch_first=True), 'eigen', 'expand', steps=2)


class UnrolledLSTM(nn.Module):
    """nn.LSTM (unidirectional) written with nn.Linear modules: an ih Linear over the sequence and an hh Linear called
    once per step, registered in the order ih_l0, hh_l0, ih_l1, ... of the LSTM's sub-layers."""

    def __init__(self, lstm):
        super().__init__()
        self.H, self.L = lstm.hidden_size, lstm.num_layers
        self.lin = nn.ModuleList()
        for k in range(lstm.num_layers):
            for side in ('ih', 'hh'):
                w = getattr(lstm, f'weight_{side}_l{k}')
                lin = nn.Linear(w.size(1), w.size(0)).to(w.device, w.dtype)
                with torch.no_grad():
                    lin.weight.copy_(w)
                    lin.bias.copy_(getattr(lstm, f'bias_{side}_l{k}'))
                self.lin.append(lin)

    def forward(self, x):
        for k in range(self.L):
            ih, hh = self.lin[2 * k], self.lin[2 * k + 1]
            zx = ih(x)
            h = c = x.new_zeros(x.size(1), self.H)
            outs = []
            for t in range(x.size(0)):
                i, f, g, o = (zx[t] + hh(h)).chunk(4, 1)
                c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(g)
                h = torch.sigmoid(o) * torch.tanh(c)
                outs.append(h)
            x = torch.stack(outs)
        return x

    def sublayer(self, name):
        """The Linear of the LSTM sub-layer `name` ('ih_l0', 'hh_l1', ...)."""
        side, k = name.split('_l')
        return self.lin[2 * int(k) + (side == 'hh')]


@pytest.mark.parametrize('method', ['eigen', 'inverse'])
def test_twin_of_linear_layers(method):
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.manual_seed(0)
    model = Net('LSTM', bidir=False).to(DEV)
    twin = UnrolledLSTM(model.rnn)
    # the twin's hh Linear is called once per step: its statistics are averaged over the calls at step()
    kw = dict(compute_method=method, damping=0.003, factor_decay=0.9, kl_clip=None, update_factors_in_hook=False)
    pre = KFACPreconditioner(model, precondition_recurrent=True, **kw)
    pre_t = KFACPreconditioner(twin, **kw)
    batches = _batches(False)
    for s in range(2):
        x, g = batches(s)
        y = torch.randn(9, 6, 32, generator=g).to(DEV)
        for m, p in ((model, pre), (twin, pre_t)):
            m.zero_grad()
            (m(x) * y).sum().backward()
            p.step()
        for name in ('ih_l0', 'hh_l0', 'ih_l1', 'hh_l1'):
            for what in ('weight', 'bias'):
                e = rel_fro(getattr(model.rnn, f'{what}_{name}').grad, getattr(twin.sublayer(name), what).grad)
                assert e <= 1e-4, (s, name, what, e)


def test_restated_forward_against_cudnn_and_stock_bits_off_factor_steps():
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    for mode in ('LSTM', 'GRU', 'RNN_TANH'):
        for packed in (False, True):
            torch.manual_seed(0)
            model = Net(mode).to(DEV)
            stock = copy.deepcopy(model)
            pre = KFACPreconditioner(model, precondition_recurrent=True, factor_update_steps=2)
            batches = _batches(packed)
            for s in range(2):                # step 0 is a factor step (restated), step 1 is not (cuDNN)
                x, g = batches(s)
                outs = []
                for m in (model, stock):
                    m.zero_grad()
                    out = m(x)
                    (out * torch.randn(out.shape, generator=torch.Generator().manual_seed(s)).to(DEV)).sum().backward()
                    outs.append((out, {n: p.grad.clone() for n, p in m.named_parameters()}))
                (o1, g1), (o2, g2) = outs
                if s == 0:
                    assert rel_fro(o1, o2) <= 1e-5, (mode, packed)
                    for n in g2:
                        assert rel_fro(g1[n], g2[n]) <= 1e-5, (mode, packed, n, rel_fro(g1[n], g2[n]))
                else:
                    assert torch.equal(o1, o2) and all(torch.equal(g1[n], g2[n]) for n in g2), (mode, packed)
                pre.step()
                with torch.no_grad():
                    for p, q in zip(stock.parameters(), model.parameters()):
                        p.copy_(q)


@pytest.mark.parametrize('approx', ['expand', 'reduce'])
def test_accumulation_steps(approx):
    torch.manual_seed(0)
    _run(Net('GRU').to(DEV), _batches(True), 'eigen', approx, steps=2, acc=2)


@pytest.mark.parametrize('method', ['eigen', 'inverse', 'ekfac'])
def test_factor_and_inverse_schedule(method):
    torch.manual_seed(0)
    _run(Net('LSTM').to(DEV), _batches(False), method, 'expand', steps=4, fus=2, ius=2)


def test_factor_dtype_bf16():
    torch.manual_seed(0)
    _run(Net('GRU').to(DEV), _batches(True), 'eigen', 'expand', steps=2, kw={'factor_dtype': torch.bfloat16},
         cast=torch.bfloat16)


@pytest.mark.parametrize('mode', ['LSTM', 'GRU'])
def test_amp_grad_scaler(mode):
    """fp16 autocast with a GradScaler: the taps see fp16 tensors, G is formed from the scaled gradient and unscaled on
    the device; the factors match fp64 from the taps and the step keeps every parameter finite."""
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(0)
    model = Net(mode).to(DEV)
    scaler = torch.amp.GradScaler('cuda', init_scale=2.0 ** 10)
    pre = KFACPreconditioner(model, precondition_recurrent=True, grad_scaler=scaler, damping=0.003, factor_decay=0.9,
                             kl_clip=None)
    calls = _record(pre)
    opt = torch.optim.SGD(model.parameters(), lr=0.01)
    eye = lambda n: torch.eye(n, dtype=torch.float64, device=DEV)  # noqa: E731
    batches = _batches(True)
    A, G = {}, {}
    for s in range(2):
        opt.zero_grad()
        calls.clear()
        x, g = batches(s)
        with torch.autocast('cuda', dtype=torch.float16):
            out = model(x)
        scale = scaler.get_scale()
        scaler.scale((out.float() * torch.randn(out.shape, generator=g).to(DEV)).sum()).backward()
        scaler.unscale_(opt)
        pre.step()
        scaler.step(opt)
        scaler.update()
        torch.cuda.synchronize()
        for key, (name, layer) in pre._layers.items():
            (xa, ta), (gg, tg) = calls[key.suffix]['a'][0], calls[key.suffix]['g'][0]
            assert xa.dtype == torch.float16 and gg.dtype == torch.float16
            X, Gr = _rows64(key, xa, ta, 'a', False), _rows64(key, gg, tg, 'g', False) / scale
            A[name] = 0.9 * A.get(name, eye(X.shape[1])) + 0.1 * X.T @ X / X.shape[0]
            G[name] = 0.9 * G.get(name, eye(Gr.shape[1])) + 0.1 * Gr.T @ Gr / Gr.shape[0]
            assert rel_fro(layer.a_factor, A[name]) <= 1e-5, (s, name)
            assert rel_fro(layer.g_factor, G[name]) <= 1e-5, (s, name)
    assert all(torch.isfinite(p).all() for p in model.parameters())


def test_skipped_sublayers_are_untouched():
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(0)
    model = Net('LSTM').to(DEV)
    pre = KFACPreconditioner(model, precondition_recurrent=True, skip_layers=[r'rnn\.hh_l1_reverse', r'rnn\.ih_l0$'])
    x, g = _batches(True)(0)
    out = model(x)
    (out * torch.randn(out.shape, generator=g).to(DEV)).sum().backward()
    raw = {n: p.grad.clone() for n, p in model.rnn.named_parameters()}
    pre.step()
    for n, p in model.rnn.named_parameters():
        untouched = n.endswith('hh_l1_reverse') or n.endswith('ih_l0')
        assert torch.equal(p.grad, raw[n]) == untouched, n


def test_state_dict_round_trip():
    """Factors saved after two steps load into a fresh preconditioner of a fresh model under the same names, and both
    then precondition a gradient to the same bits."""
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(0)
    model = Net('GRU').to(DEV)
    pre = _run(model, _batches(True), 'eigen', 'expand', steps=2)
    sd = pre.state_dict()
    fresh = copy.deepcopy(model)
    again = KFACPreconditioner(fresh, precondition_recurrent=True, damping=0.003, factor_decay=0.9, kl_clip=None)
    again.load_state_dict(sd)
    for (n, a), (m, b) in zip(pre._layer_list(), again._layer_list()):
        assert n == m and torch.equal(a.a_factor, b.a_factor) and torch.equal(a.g_factor, b.g_factor), n
    for p in (pre, again):
        p._factor_update_steps = p._inv_update_steps = 10 ** 6      # keep the loaded factors and decompositions
    x, g = _batches(True)(5)
    model.zero_grad()
    out = model(x)
    (out * torch.randn(out.shape, generator=g).to(DEV)).sum().backward()
    for p, q in zip(model.parameters(), fresh.parameters()):
        q.grad = p.grad.clone()
    pre.step()
    again.step()
    assert all(torch.equal(p.grad, q.grad) for p, q in zip(model.parameters(), fresh.parameters()))


class _TwoBranch(nn.Module):
    def __init__(self):
        super().__init__()
        self.fc = nn.Sequential(nn.Linear(12, 20), nn.Tanh(), nn.Linear(20, 5))
        self.rnn = nn.LSTM(24, 16)

    def forward(self, x, z):
        return self.fc(z).sum() + self.rnn(x)[0].pow(2).sum()


def test_keyword_leaves_other_layers_bitwise():
    from kfac_b200.preconditioner import KFACPreconditioner
    factors = []
    for on in (False, True):
        torch.manual_seed(0)
        model = _TwoBranch().to(DEV)
        pre = KFACPreconditioner(model, precondition_recurrent=on, damping=0.003)
        for s in range(2):
            g = torch.Generator().manual_seed(s)
            x, z = torch.randn(9, 6, 24, generator=g).to(DEV), torch.randn(8, 12, generator=g).to(DEV)
            model.zero_grad()
            model(x, z).backward()
            pre.step()
        layers = dict(pre._layer_list())
        factors.append({n: (layers[n].a_factor.clone(), layers[n].g_factor.clone()) for n in ('fc.0', 'fc.2')})
    for n in factors[0]:
        assert all(torch.equal(a, b) for a, b in zip(factors[0][n], factors[1][n])), n


def _run_dist(backend):
    import os
    import socket
    import subprocess
    import sys
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    script = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'dist_recurrent.py')
    out = subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node=2',
                          '--master-addr', '127.0.0.1', '--master-port', str(port), script, '--backend', backend],
                         capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, (out.stdout[-3000:], out.stderr[-3000:])
    assert out.stdout.count('dist_recurrent ok') == 2, out.stdout[-2000:]


def test_two_ranks_gloo():
    _run_dist('gloo')


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='NCCL needs one GPU per rank')
def test_two_ranks_nccl():
    _run_dist('nccl')
