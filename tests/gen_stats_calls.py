"""Digests of the exact record of every native call the layer helpers make for the factor statistics
(tests/golden/stats_calls.json).

Runs on the CPU without libkfac_b200.so.  A fake library stands in for `_cabi.load()` and records each call as the
library would receive it, argument by argument, typed by `_cabi.SIGNATURES`: a c_float as its float32 bit pattern, a
c_double as a double, integers as they are, a struct passed by reference as its field values, and every pointer as
[buffer, byte offset], the buffer being the tensor handed to the helper ('x' or 'g', offsets from the start of its
storage), 'acc', 'out', 'scratch', 'loss_scale', a recurrent tap's 'h0' / 'mul' / 'offsets', 'stream', or
'temporary' for a copy the helper made itself.  The `*_workspace_bytes` queries answer by `workspace_bytes`.

Each case makes the calls the preconditioner's hooks make, in their order: on the A side prepare_input, accumulate_a,
num_rows_a and write_rows_a, on the G side accumulate_g, num_rows_g and write_rows_g at grad_scale 3.0 with a
loss-scale slot (the row writers only for the kinds EKFAC takes).  An exception ends its side and is recorded.  A
case runs its layer in fp32, fp16 and bf16, in expand and (where the kind has it) K-FAC-reduce mode, and the golden
keeps the SHA-256 of its whole record; `record(name)` gives the record itself, to see where two versions differ.

    python tests/gen_stats_calls.py [OUT.json]        # default: tests/golden/stats_calls.json

tests/test_stats_calls_host.py replays the same cases and compares.  The scale arguments are compared bit for bit:
the benchmark's training dynamics turn a last-bit change of a factor into different outputs within a few steps, so
two mathematically equal ways of writing a scale are not interchangeable.
"""
from __future__ import annotations

import contextlib
import ctypes as C
import hashlib
import json
import os
import struct
import sys
import types

import torch
from torch import nn
from torch.nn.utils.rnn import pack_padded_sequence

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from kfac_b200 import _cabi, attention, recurrent  # noqa: E402
from kfac_b200 import layers as L  # noqa: E402
from kfac_b200.base_preconditioner import _Scratch  # noqa: E402

GOLDEN = os.path.join(HERE, 'golden', 'stats_calls.json')
GRAD_SCALE = 3.0                # not a power of two, so that a rewritten scale expression shows
STREAM = 0x5EED0000             # what the patched _cabi.stream_ptr() returns
DTYPES = {'f32': torch.float32, 'f16': torch.float16, 'bf16': torch.bfloat16}
MODES = {'expand': False, 'reduce': True}
_INTS = (C.c_int, C.c_int64, C.c_size_t, C.c_longlong)
# the workspace queries answered 0 for an even row count (first argument)
ZERO_WORKSPACE = ('kfac_factor_linear_workspace_bytes', 'kfac_factor_linear_strided_workspace_bytes')


def workspace_bytes(name: str, args: list) -> int:
    """The fake library's answer to a workspace query: 0 for the Linear statistics (dense and strided) of an even
    number of rows (their callers then pass no workspace), else a multiple of 256 that depends on the integer
    arguments."""
    if name in ZERO_WORKSPACE and args[0] % 2 == 0:
        return 0
    return 256 * (1 + sum(a for a in args if isinstance(a, int)) % 7)


class FakeLib:
    """Records every call; `buffers` maps a label to the tensor (or zero-argument callable giving it) whose storage a
    pointer may lie in."""

    def __init__(self):
        self.events: list = []
        self.buffers: dict = {}

    def pointer(self, p):
        if p is None or p == 0:
            return None
        if p == STREAM:
            return 'stream'
        for label, t in self.buffers.items():
            t = t() if callable(t) else t
            if t is None:
                continue
            st = t.untyped_storage()
            base = st.data_ptr()
            if base <= p < base + max(st.nbytes(), 1):
                return [label, p - base]
        return 'temporary'

    def convert(self, ctype, a):
        if ctype is C.c_float:
            return '%08x' % struct.unpack('<I', struct.pack('<f', a))[0]
        if ctype is C.c_double:
            return float(a)
        if ctype is C.c_void_p:
            if a is not None and not isinstance(a, int):
                raise TypeError(f'pointer argument {a!r}')
            return self.pointer(a)
        if ctype in _INTS:
            if not isinstance(a, int):
                raise TypeError(f'integer argument {a!r}')
            return int(a)
        if isinstance(ctype, type) and issubclass(ctype, C._Pointer):
            s = a._obj
            if not isinstance(s, ctype._type_):
                raise TypeError(f'{type(s).__name__} passed for {ctype._type_.__name__}')
            return {f: self.convert(t, getattr(s, f)) if t in (C.c_void_p, C.c_float) or t in _INTS
                    else list(getattr(s, f)) for f, t in s._fields_}
        raise TypeError(f'argument type {ctype}')

    def __getattr__(self, name):
        if name not in _cabi.SIGNATURES:
            raise AttributeError(name)
        argtypes = _cabi.SIGNATURES[name][1]

        def call(*args):
            if len(args) != len(argtypes):
                raise TypeError(f'{name}: {len(args)} arguments, expected {len(argtypes)}')
            rec = [self.convert(t, a) for t, a in zip(argtypes, args)]
            self.events.append([name] + rec)
            return workspace_bytes(name, rec) if name.endswith('_workspace_bytes') else _cabi.KFAC_OK
        return call


@contextlib.contextmanager
def fake_native(lib: FakeLib):
    saved = _cabi.load, _cabi.require_device, _cabi.stream_ptr
    _cabi.load, _cabi.require_device, _cabi.stream_ptr = (lambda: lib), (lambda t: None), (lambda: STREAM)
    try:
        yield
    finally:
        _cabi.load, _cabi.require_device, _cabi.stream_ptr = saved


def drive(helper, x, g, rows: bool = True, call=None, tap_a=None, tap_g=None) -> list:
    """The calls of the preconditioner's _accumulate_input and _accumulate_grad_output for one forward and backward
    call of `helper`'s layer: x its input, g the gradient of its output."""
    lib = FakeLib()
    scratch, scratch_bwd = _Scratch(), _Scratch()
    loss_scale = torch.ones(1)
    with fake_native(lib):
        for side, t, tap in (('a', x, tap_a), ('g', g, tap_g)):
            d = (helper.a_factor_shape if side == 'a' else helper.g_factor_shape)
            acc = torch.zeros(d)
            lib.buffers = {'acc': acc, 'scratch': (lambda s=(scratch if side == 'a' else scratch_bwd): s.buf),
                           'loss_scale': loss_scale}
            if tap is not None:
                setattr(helper, 'tap_' + side, tap)
                lib.buffers.update(h0=tap.h0, mul=tap.mul, offsets=tap.offsets)
            try:
                if side == 'a':
                    if call is not None:
                        helper.bind_call(*call)
                    t = helper.prepare_input(t)
                    lib.buffers['x'] = t
                    helper.accumulate_a(t, acc, scratch)
                else:
                    lib.buffers['g'] = t
                    helper.accumulate_g(t, acc, GRAD_SCALE, scratch_bwd)
                if rows:
                    n = getattr(helper, 'num_rows_' + side)(t)
                    lib.events.append(['num_rows_' + side, n])
                    out = torch.empty(max(n, 1) * _cabi.ld4(d[0]))
                    lib.buffers['out'] = out
                    if side == 'a':
                        helper.write_rows_a(t, out)
                    else:
                        helper.write_rows_g(t, out, GRAD_SCALE, loss_scale.data_ptr())
            except (ValueError, ZeroDivisionError) as e:
                lib.events.append([type(e).__name__, str(e)])
    return lib.events


def _randn(seed, *shape, dtype=torch.float32):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)).to(dtype)


def _out_shape(m, x, *args, **kwargs):
    with torch.no_grad():
        return m(x.float(), *args, **kwargs).shape


CASES: dict = {}        # name -> zero-argument function giving the case's record


def case(name):
    def put(fn):
        CASES[name] = fn
        return fn
    return put


def _variants(run, modes=MODES):
    """A case that runs `run(dtype, reduce)` for every dtype and mode, each record preceded by the variant's name."""
    def each():
        return [e for dname, dt in DTYPES.items() for mname, red in modes.items()
                for e in [['variant', dname, mname]] + run(dt, red)]
    return each


def _module_cases(prefix, make, inputs, rows=True, helper=None):
    """One case per input and bias: `make(bias)` the module, `inputs` {name: (x fn, forward args, forward kwargs)}."""
    for bias in (True, False):
        for iname, (xf, args, kwargs) in inputs.items():
            def run(dt, red, bias=bias, xf=xf, args=args, kwargs=kwargs):
                torch.manual_seed(0)
                m = make(bias)
                x = xf(dt)
                g = _randn(2, *_out_shape(m, x, *args, **kwargs), dtype=dt)
                h = helper(m, red)
                call = (((x,) + tuple(args), dict(kwargs)) if h.call_kwargs else None)
                return drive(h, x, g, rows=rows, call=call)
            CASES[f'{prefix}-{iname}-bias{int(bias)}'] = _variants(run)


def _helper(cls):
    return lambda m, red: cls(m, reduce=red)


# ---- Linear
_module_cases('linear', lambda b: nn.Linear(6, 5, bias=b), {
    '1d': (lambda dt: _randn(1, 6, dtype=dt), (), {}),
    '2d': (lambda dt: _randn(1, 4, 6, dtype=dt), (), {}),
    '3d': (lambda dt: _randn(1, 3, 4, 6, dtype=dt), (), {}),
    'strided': (lambda dt: _randn(1, 4, 3, 6, dtype=dt).transpose(0, 1), (), {}),
}, helper=_helper(L.LinearModuleHelper))

# ---- diagonal-G Linear (no EKFAC)
_module_cases('diag_g', lambda b: nn.Linear(6, 5, bias=b), {
    '2d': (lambda dt: _randn(1, 4, 6, dtype=dt), (), {}),
    '3d': (lambda dt: _randn(1, 3, 4, 6, dtype=dt), (), {}),
    'zero_rows': (lambda dt: _randn(1, 0, 6, dtype=dt), (), {}),
    'zero_positions': (lambda dt: _randn(1, 2, 0, 6, dtype=dt), (), {}),
}, rows=False, helper=_helper(L.DiagonalGLinearModuleHelper))

# ---- Conv2d: padding and stride; a 1x1 output (reduce takes the expand path)
_module_cases('conv2d', lambda b: nn.Conv2d(3, 4, 3, stride=2, padding=1, bias=b), {
    'pad_stride': (lambda dt: _randn(1, 2, 3, 7, 6, dtype=dt), (), {}),
}, helper=_helper(L.Conv2dModuleHelper))
_module_cases('conv2d', lambda b: nn.Conv2d(3, 4, (3, 2), bias=b), {
    'out1x1': (lambda dt: _randn(1, 2, 3, 3, 2, dtype=dt), (), {}),
}, helper=_helper(L.Conv2dModuleHelper))

# ---- Conv1d / Conv3d
_CONV_ND = {
    'conv1d-dilation': (lambda b: nn.Conv1d(3, 4, 3, dilation=2, padding=1, bias=b), (2, 3, 9)),
    'conv1d-same': (lambda b: nn.Conv1d(3, 4, 4, padding='same', bias=b), (2, 3, 8)),
    'conv1d-reflect': (lambda b: nn.Conv1d(3, 4, 3, stride=2, padding=2, padding_mode='reflect', bias=b), (2, 3, 9)),
    'conv1d-unbatched': (lambda b: nn.Conv1d(3, 4, 3, bias=b), (3, 7)),
    'conv3d-circular': (lambda b: nn.Conv3d(2, 3, (2, 3, 3), stride=(1, 2, 2), dilation=(1, 1, 2), padding=1,
                                            padding_mode='circular', bias=b), (2, 2, 4, 6, 7)),
    'conv3d-same': (lambda b: nn.Conv3d(2, 3, (1, 2, 3), padding='same', dilation=(1, 2, 1), bias=b), (2, 2, 3, 5, 4)),
    'conv3d-unbatched': (lambda b: nn.Conv3d(2, 3, 2, padding=(0, 1, 0), bias=b), (2, 3, 4, 5)),
}
for _name, (_make, _shape) in _CONV_ND.items():
    _module_cases(_name, _make, {'x': (lambda dt, s=_shape: _randn(1, *s, dtype=dt), (), {})},
                  helper=_helper(L.ConvNdModuleHelper))

# ---- ConvTranspose1d / 2d / 3d: output_size positionally and as a keyword
_CONV_T = {
    'convt1d-output_size_arg': (lambda b: nn.ConvTranspose1d(3, 4, 3, stride=2, padding=1, bias=b), (2, 3, 5),
                                ([10],), {}),
    'convt1d-unbatched': (lambda b: nn.ConvTranspose1d(3, 4, 3, stride=2, bias=b), (3, 5), (), {}),
    'convt2d-plain': (lambda b: nn.ConvTranspose2d(3, 4, 3, stride=2, padding=1, dilation=(1, 2), bias=b),
                      (2, 3, 4, 5), (), {}),
    'convt2d-output_size_kw': (lambda b: nn.ConvTranspose2d(3, 4, 3, stride=2, padding=1, bias=b), (2, 3, 4, 5), (),
                               {'output_size': (8, 10)}),
    'convt2d-unbatched': (lambda b: nn.ConvTranspose2d(3, 4, 2, stride=(1, 2), bias=b), (3, 4, 5), (),
                          {'output_size': [5, 11]}),
    'convt3d-output_size_arg': (lambda b: nn.ConvTranspose3d(2, 3, (1, 3, 2), stride=(1, 2, 2), padding=(0, 1, 0),
                                                             bias=b), (2, 2, 2, 3, 4), ((2, 6, 9),), {}),
}
for _name, (_make, _shape, _args, _kwargs) in _CONV_T.items():
    _module_cases(_name, _make, {'x': (lambda dt, s=_shape: _randn(1, *s, dtype=dt), _args, _kwargs)},
                  helper=_helper(L.ConvTransposeModuleHelper))


# ---- Embedding (A: the index histogram; no EKFAC, no K-FAC-reduce)
for _iname, _shape in (('2d', (4, 3)), ('1d', (5,)), ('empty', (0,))):
    for _idt in (torch.int32, torch.int64):
        def _run(dt, red, shape=_shape, idt=_idt):
            m = nn.Embedding(10, 5)
            x = torch.randint(0, 10, shape, generator=torch.Generator().manual_seed(1)).to(idt)
            return drive(L.EmbeddingModuleHelper(m), x, _randn(2, *shape, 5, dtype=dt), rows=False)
        CASES[f'embedding-{_iname}-{str(_idt)[6:]}'] = _variants(_run, {'expand': False})


# ---- errors the helpers raise
@case('error-conv2d-string_padding')
def _():
    m = nn.Conv2d(3, 4, 3, padding='same')
    return drive(L.Conv2dModuleHelper(m), _randn(1, 2, 3, 5, 5), _randn(2, 2, 4, 5, 5))


@case('error-conv1d-empty_output')
def _():
    m = nn.Conv1d(3, 4, 5)
    return drive(L.ConvNdModuleHelper(m), _randn(1, 2, 3, 4), _randn(2, 2, 4, 1))


@case('error-conv1d-gradout_extent')
def _():
    m = nn.Conv1d(3, 4, 3)
    return drive(L.ConvNdModuleHelper(m), _randn(1, 2, 3, 8), _randn(2, 2, 4, 7))


@case('error-convt1d-empty_output')
def _():
    m = nn.ConvTranspose1d(3, 4, 1, padding=1)
    return drive(L.ConvTransposeModuleHelper(m), _randn(1, 2, 3, 1), _randn(2, 2, 4, 1), call=((None,), {}))


@case('error-linear-int_input')
def _():
    return drive(L.LinearModuleHelper(nn.Linear(6, 5)), torch.ones(4, 6, dtype=torch.int32), _randn(2, 4, 5))


@case('error-embedding-float_index')
def _():
    return drive(L.EmbeddingModuleHelper(nn.Embedding(10, 5)), torch.ones(4), _randn(2, 4, 5), rows=False)


# ---- attention projections: taps captured from KFACMultiheadAttention's forward on the CPU
class _Recorder:
    """Stands in for the preconditioner: every projection is tapped, each tap keeps the tensor it was handed."""

    def __init__(self, keys):
        self.keys, self.a, self.g = keys, {}, {}

    def _active_attention_taps(self, module):
        return self.keys

    def _attention_input(self, key, x):
        self.a[key] = x

    def _attention_grad_output(self, key, g):
        self.g[key] = g

    def _active_recurrent_taps(self, module):
        return self.keys

    def _recurrent_input(self, key, x, tap):
        self.a[key.suffix] = (x, tap)

    def _recurrent_grad_output(self, key, g, tap):
        self.g[key.suffix] = (g, tap)


_ATTN = {
    # name: (module kwargs, query shape, key/value shapes or None for self-attention)
    'packed': (dict(embed_dim=8, num_heads=2), (5, 3, 8), None),
    'separate': (dict(embed_dim=8, num_heads=2, kdim=6, vdim=4, bias=False), (5, 3, 8), ((7, 3, 6), (7, 3, 4))),
    'batch_first': (dict(embed_dim=8, num_heads=2, batch_first=True), (3, 5, 8), None),
    'batch_first_cross': (dict(embed_dim=8, num_heads=2, batch_first=True), (3, 5, 8), ((3, 4, 8), (3, 4, 8))),
    'L1': (dict(embed_dim=8, num_heads=2), (1, 3, 8), None),
    'unbatched': (dict(embed_dim=8, num_heads=2), (5, 8), None),
}


def _attention_taps(kwargs, qshape, kv):
    torch.manual_seed(0)
    m = nn.MultiheadAttention(**kwargs)
    rec = _Recorder({w: w for w in 'qkvo'})
    attention.bind(m, rec)
    q = _randn(1, *qshape).requires_grad_()
    k, v = (q, q) if kv is None else (_randn(3, *kv[0]).requires_grad_(), _randn(4, *kv[1]).requires_grad_())
    out, _ = m(q, k, v, need_weights=False)
    (out * _randn(5, *out.shape)).sum().backward()
    return m, rec


for _aname, _spec in _ATTN.items():
    for _which in ('q', 'k', 'v', 'out'):
        def _run(dt, red, spec=_spec, which=_which):
            m, rec = _attention_taps(*spec)
            h = L.AttentionProjectionHelper(m, which, reduce=red)
            w = which[0]
            return drive(h, L.cast_for_factor(rec.a[w], dt), L.cast_for_factor(rec.g[w], dt))
        CASES[f'attention-{_aname}-{_which}'] = _variants(_run)


# ---- RNN / LSTM / GRU sub-layers: taps captured from the KFAC* forward on the CPU
_RNN = {
    # name: (module, input kind, h0 given)
    'rnn-batched': (lambda: nn.RNN(3, 4, num_layers=2), 'batched', False),
    'rnn-bidir-h0': (lambda: nn.RNN(3, 4, bidirectional=True, batch_first=True), 'batched', True),
    'rnn-unsorted': (lambda: nn.RNN(3, 4), 'unsorted', True),
    'lstm-batched-h0': (lambda: nn.LSTM(3, 4), 'batched', True),
    'lstm-bidir-sorted': (lambda: nn.LSTM(3, 4, bidirectional=True), 'sorted', False),
    'lstm-unbatched': (lambda: nn.LSTM(3, 4, bias=False), 'unbatched', True),
    'gru-batched': (lambda: nn.GRU(3, 4), 'batched', False),
    'gru-bidir-unsorted-h0': (lambda: nn.GRU(3, 4, bidirectional=True, batch_first=True), 'unsorted', True),
    'gru-sorted-h0': (lambda: nn.GRU(3, 4, num_layers=2), 'sorted', True),
}


def _sublayers(m):
    return [(k, d, s) for k in range(m.num_layers) for d in range(2 if m.bidirectional else 1) for s in ('ih', 'hh')]


def _recurrent_taps(make, kind, with_h0):
    torch.manual_seed(0)
    m = make()
    keys = {f'{s}_l{k}' + ('_reverse' if d else ''): types.SimpleNamespace(suffix=f'{s}_l{k}' + ('_reverse' if d
                                                                                                  else ''))
            for k, d, s in _sublayers(m)}
    rec = _Recorder(keys)
    recurrent.bind(m, rec)
    T, B, D = 5, 4, 2 if m.bidirectional else 1
    if kind == 'unbatched':
        x = _randn(1, T, 3)
    else:
        x = _randn(1, B, T, 3) if m.batch_first else _randn(1, T, B, 3)
        if kind != 'batched':
            lengths = torch.tensor([5, 3, 3, 1]) if kind == 'sorted' else torch.tensor([2, 5, 1, 4])
            x = pack_padded_sequence(x, lengths, batch_first=m.batch_first, enforce_sorted=kind == 'sorted')
    hx = None
    if with_h0:
        shape = (m.num_layers * D, 4) if kind == 'unbatched' else (m.num_layers * D, B, 4)
        hx = _randn(6, *shape).requires_grad_()
        if isinstance(m, nn.LSTM):
            hx = (hx, _randn(7, *shape).requires_grad_())
    out, hid = m(x, hx) if hx is not None else m(x)
    data = out.data if hasattr(out, 'batch_sizes') else out
    parts = [data] + (list(hid) if isinstance(hid, tuple) else [hid])
    sum((p * _randn(8 + i, *p.shape)).sum() for i, p in enumerate(parts)).backward()
    return m, rec


for _rname, _spec in _RNN.items():
    def _run(dt, red, spec=_spec):
        m, rec = _recurrent_taps(*spec)
        events = []
        for k, d, s in _sublayers(m):
            h = L.RecurrentSubLayerHelper(m, k, d, s, reduce=red)
            (x, tap_a), (g, tap_g) = rec.a[h.suffix], rec.g[h.suffix]
            events += [[h.suffix]] + drive(h, L.cast_for_factor(x, dt), L.cast_for_factor(g, dt), tap_a=tap_a,
                                           tap_g=tap_g)
        return events
    CASES[f'recurrent-{_rname}'] = _variants(_run)


def record(name: str) -> list:
    """The record of one case: its events, as JSON values."""
    return json.loads(json.dumps(CASES[name]()))


def digest(name: str) -> str:
    return hashlib.sha256(json.dumps(record(name), separators=(',', ':')).encode()).hexdigest()


def main(argv) -> None:
    path = argv[1] if len(argv) > 1 else GOLDEN
    lines = ',\n'.join(f'  {json.dumps(name)}: "{digest(name)}"' for name in sorted(CASES))
    with open(path, 'w') as f:
        f.write('{"digests": {\n' + lines + '\n}}\n')
    print(f'{len(CASES)} cases -> {path}')


if __name__ == '__main__':
    main(sys.argv)
