"""CPU tests of Conv1d / Conv3d layers (`precondition_conv_nd=True`): the keyword off changes nothing, registration,
factor shapes, placement cost and repr with it on, the refusals, the resolution of padding and output extents against
real torch convolutions, and a state_dict round trip."""
import itertools

import pytest
import torch
from torch import nn
from torch.nn import functional as F

from conftest import ROOT  # noqa: F401  (puts the repository on sys.path)


class _AV(nn.Module):
    """An audio stem, a video stem and a head: Conv1d, Conv3d, Conv2d and Linear layers."""

    def __init__(self):
        super().__init__()
        self.audio = nn.Conv1d(1, 16, 10, stride=5, bias=False)
        self.tcn = nn.Conv1d(16, 24, 3, dilation=2, padding='same')
        self.video = nn.Conv3d(3, 8, (3, 7, 7), stride=(1, 2, 2), padding=(1, 3, 3))
        self.image = nn.Conv2d(3, 6, 3)
        self.head = nn.Linear(24, 5)


def _names(pre):
    return {n: l for n, l in pre._layers.values()}


def test_keyword_off_registers_todays_set():
    from kfac_b200.preconditioner import KFACPreconditioner
    pre = KFACPreconditioner(_AV())
    assert list(_names(pre)) == ['image', 'head']
    assert 'precondition_conv_nd=False' in repr(pre)


def test_registration_shapes_cost_and_repr():
    from kfac_b200.enums import AssignmentStrategy
    from kfac_b200.layers import ConvNdModuleHelper, register_modules
    from kfac_b200.preconditioner import KFACPreconditioner, layer_work
    pre = KFACPreconditioner(_AV(), precondition_conv_nd=True)
    names = _names(pre)
    assert list(names) == ['audio', 'tcn', 'video', 'image', 'head']
    assert names['audio'].a_factor_shape == (10, 10) and names['audio'].g_factor_shape == (16, 16)
    assert names['tcn'].a_factor_shape == (16 * 3 + 1,) * 2 and names['tcn'].g_factor_shape == (24, 24)
    assert names['video'].a_factor_shape == (3 * 3 * 7 * 7 + 1,) * 2 and names['video'].g_factor_shape == (8, 8)
    assert isinstance(names['video'].module, ConvNdModuleHelper) and names['video'].module.nd == 3
    assert 'precondition_conv_nd=True' in repr(pre)
    layers = register_modules(_AV(), [], precondition_conv_nd=True, method=None)
    for strategy, cost in ((AssignmentStrategy.COMPUTE, lambda n: n ** 3), (AssignmentStrategy.MEMORY, lambda n: n ** 2)):
        work = layer_work(layers, strategy)
        assert work['video'] == {'A': cost(442), 'G': cost(8)}
        assert work['audio'] == {'A': cost(10), 'G': cost(16)}
    # skip_layers by name and by class, and frozen parameters
    assert list(_names(KFACPreconditioner(_AV(), precondition_conv_nd=True, skip_layers=['Conv3d', 'tcn']))) == \
        ['audio', 'image', 'head']
    m = _AV()
    m.audio.weight.requires_grad_(False)
    assert 'audio' not in _names(KFACPreconditioner(m, precondition_conv_nd=True))


def test_refusals():
    from kfac_b200.preconditioner import KFACPreconditioner
    grouped = nn.Sequential(nn.Conv1d(8, 8, 3, groups=2))
    with pytest.raises(ValueError, match=r'"0" \(Conv1d\) has groups=2.*add it to `?skip_layers'):
        KFACPreconditioner(grouped, precondition_conv_nd=True)
    depthwise = nn.Sequential(nn.Conv3d(4, 4, 3, groups=4))
    with pytest.raises(ValueError, match=r'"0" \(Conv3d\) has groups=4.*skip_layers'):
        KFACPreconditioner(depthwise, precondition_conv_nd=True)
    # r3d_18's layer4: 512 * 27 = 13824 > 8192
    wide = nn.Sequential(nn.Conv3d(512, 512, 3, bias=False))
    with pytest.raises(ValueError, match=r'"0" \(Conv3d\) has factors of 13824 \(A\).*skip_layers'):
        KFACPreconditioner(wide, precondition_conv_nd=True)
    with pytest.raises(ValueError, match=r'"0" \(Conv1d\).*9000 \(G\).*skip_layers'):
        KFACPreconditioner(nn.Sequential(nn.Conv1d(4, 9000, 1)), precondition_conv_nd=True)
    # K-FAC-reduce forms window sums of at most 2048 taps: 13^3 = 2197 is refused under reduce only
    big = nn.Sequential(nn.Conv3d(1, 2, 13))
    with pytest.raises(ValueError, match=r'"0" \(Conv3d\) has a kernel of 2197 taps.*skip_layers'):
        KFACPreconditioner(big, precondition_conv_nd=True, kfac_approx='reduce')
    KFACPreconditioner(big, precondition_conv_nd=True)
    # A = 8191 + bias = 8192 is the largest accepted
    KFACPreconditioner(nn.Sequential(nn.Conv1d(8191, 4, 1)), precondition_conv_nd=True)
    with pytest.raises(ValueError, match='"tcn" \\(Conv1d\\): only torch.nn.Linear layers can keep a diagonal G'):
        KFACPreconditioner(_AV(), precondition_conv_nd=True, diagonal_g_layers=['tcn'])
    # skipped or not registered: no refusal
    KFACPreconditioner(grouped, precondition_conv_nd=True, skip_layers=['0'])
    KFACPreconditioner(grouped)
    KFACPreconditioner(_AV(), diagonal_g_layers=['tcn'])


def _conv(nd, kernel, stride, dilation, padding, mode):
    cls = nn.Conv1d if nd == 1 else nn.Conv3d
    return cls(2, 3, kernel, stride=stride, dilation=dilation, padding=padding, padding_mode=mode)


PAD_CASES_1D = [
    # kernel, stride, dilation, padding
    (4, 1, 1, 'same'), (4, 1, 3, 'same'), (5, 1, 2, 'same'), (2, 1, 1, 'same'), (6, 1, 1, 'same'),
    (3, 2, 1, 'valid'), (10, 5, 1, 0), (3, 3, 2, 4), (7, 2, 3, 5), (1, 1, 1, 0), (1, 4, 1, 2),
]
PAD_CASES_3D = [
    ((2, 4, 3), 1, (1, 2, 3), 'same'), ((3, 3, 3), 1, 1, 'same'), ((2, 2, 2), 2, 2, (1, 0, 2)),
    ((1, 3, 3), (1, 2, 2), 1, (0, 1, 1)), ((3, 1, 1), 1, (2, 1, 1), 'valid'), ((4, 2, 6), (2, 1, 3), (1, 3, 1), (3, 0, 2)),
]


@pytest.mark.parametrize('mode', ['zeros', 'reflect', 'replicate', 'circular'])
@pytest.mark.parametrize('nd,case', [(1, c) for c in PAD_CASES_1D] + [(3, c) for c in PAD_CASES_3D])
def test_padding_and_output_extent(nd, case, mode):
    """The helper's per-axis padding, applied as zero padding (or by F.pad for another padding_mode) to a convolution
    without padding, gives the module's output; its output extent is the output's shape, batched and unbatched."""
    from kfac_b200.layers import ConvNdModuleHelper
    kernel, stride, dilation, padding = case
    if padding == 'same' and (stride != 1 if isinstance(stride, int) else any(s != 1 for s in stride)):
        pytest.skip("torch refuses padding='same' with strides")
    torch.manual_seed(0)
    m = _conv(nd, kernel, stride, dilation, padding, mode).double()
    h = ConvNdModuleHelper(m)
    shape = (2, 2, 23) if nd == 1 else (2, 2, 7, 9, 11)
    x = torch.randn(*shape, dtype=torch.float64)
    y = m(x)
    geo, S, out = h._input_geometry(x.shape)
    assert out == tuple(y.shape[2:]) and S == y[0, 0].numel()
    assert (geo.batch, geo.C) == (2, 2)
    before, after = h._pads()
    conv = F.conv1d if nd == 1 else F.conv3d
    if mode == 'zeros':
        pads = list(itertools.chain.from_iterable((before[a], after[a]) for a in reversed(range(3 - nd, 3))))
        xp = F.pad(x, pads)
        assert list(geo.input) == [1] * (3 - nd) + list(shape[2:])
    else:
        assert before == [0, 0, 0] and after == [0, 0, 0]
        xp = F.pad(x, m._reversed_padding_repeated_twice, mode=mode)
        assert list(geo.input) == [1] * (3 - nd) + list(xp.shape[2:])
    assert torch.allclose(conv(xp, m.weight, m.bias, m.stride, 0, m.dilation), y, rtol=0, atol=1e-12)
    assert list(geo.kernel)[3 - nd:] == list(m.kernel_size) and list(geo.dilation)[3 - nd:] == list(m.dilation)
    # an unbatched input is one example of the same extent
    geo1, S1, out1 = h._input_geometry(x[0].shape)
    assert geo1.batch == 1 and out1 == out and S1 == S and tuple(m(x[0]).shape[1:]) == out


def test_empty_output_is_refused():
    from kfac_b200.layers import ConvNdModuleHelper
    h = ConvNdModuleHelper(nn.Conv1d(2, 3, 5))
    with pytest.raises(ValueError, match='empty output'):
        h._input_geometry((2, 2, 3))


def test_state_dict_round_trip():
    from kfac_b200.preconditioner import KFACPreconditioner
    pre = KFACPreconditioner(_AV(), precondition_conv_nd=True)
    names = _names(pre)
    for n in ('audio', 'video'):
        l = names[n]
        l._a_view = torch.zeros(l.a_dim, l.a_dim)        # stand-ins for the arena views (no device here)
        l._g_view = torch.zeros(l.g_dim, l.g_dim)
        A = torch.rand(l.a_dim, l.a_dim)
        G = torch.rand(l.g_dim, l.g_dim)
        l.load_state_dict({'A': A, 'G': G})
        sd = l.state_dict()
        assert torch.equal(sd['A'], A) and torch.equal(sd['G'], G)
        assert l.memory_usage()['a_factors'] == l.a_dim * l.a_dim * 4
    # a checkpoint of a run with the keyword off has no entries for the new layers
    sd = KFACPreconditioner(_AV()).state_dict(include_factors=False)
    assert 'audio' not in str(sd.get('layers', {}))
