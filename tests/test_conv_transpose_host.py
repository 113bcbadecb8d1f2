"""CPU tests of ConvTranspose1d / 2d / 3d layers (`precondition_conv_transpose=True`): the keyword off changes nothing,
registration, factor shapes, the weight-gradient layout and repr with it on, the refusals, the output extent against
real torch transposed convolutions (output padding, output_size positional and keyword, unbatched inputs), and a
state_dict round trip."""
import itertools

import pytest
import torch
from torch import nn

from conftest import ROOT  # noqa: F401  (puts the repository on sys.path)


class _Gen(nn.Module):
    """A DCGAN-style generator stage, a 1-D upsampler, a 3-D decoder stage, a Conv2d and a Linear."""

    def __init__(self):
        super().__init__()
        self.up1 = nn.ConvTranspose2d(16, 8, 4, stride=2, padding=1, bias=False)
        self.up2 = nn.ConvTranspose1d(8, 4, 16, stride=8, padding=4)
        self.up3 = nn.ConvTranspose3d(4, 2, (1, 2, 2), stride=(1, 2, 2))
        self.conv = nn.Conv2d(8, 6, 3)
        self.head = nn.Linear(6, 5)


def _names(pre):
    return {n: l for n, l in pre._layers.values()}


def test_keyword_off_registers_todays_set():
    from kfac_b200.preconditioner import KFACPreconditioner
    pre = KFACPreconditioner(_Gen())
    assert list(_names(pre)) == ['conv', 'head']
    assert 'precondition_conv_transpose=False' in repr(pre)
    # the N-d keyword does not register transposed convolutions either
    assert list(_names(KFACPreconditioner(_Gen(), precondition_conv_nd=True))) == ['conv', 'head']


def test_registration_shapes_layout_and_repr():
    from kfac_b200.base_preconditioner import second_order_layout
    from kfac_b200.layers import ConvTransposeModuleHelper
    from kfac_b200.preconditioner import KFACPreconditioner
    pre = KFACPreconditioner(_Gen(), precondition_conv_transpose=True)
    names = _names(pre)
    assert list(names) == ['up1', 'up2', 'up3', 'conv', 'head']
    assert names['up1'].a_factor_shape == (16 * 16,) * 2 and names['up1'].g_factor_shape == (8, 8)
    assert names['up2'].a_factor_shape == (8 * 16 + 1,) * 2 and names['up2'].g_factor_shape == (4, 4)
    assert names['up3'].a_factor_shape == (4 * 4 + 1,) * 2 and names['up3'].g_factor_shape == (2, 2)
    assert isinstance(names['up3'].module, ConvTransposeModuleHelper) and names['up3'].module.nd == 3
    assert [names[n].module.wgrad_taps for n in ('up1', 'up2', 'up3', 'conv', 'head')] == [16, 16, 4, 0, 0]
    # the precondition items carry the layout; every other layer's item is as before
    assert second_order_layout(names['up2']).item['wgrad_taps'] == 16
    assert 'wgrad_taps' not in second_order_layout(names['conv']).item
    assert 'precondition_conv_transpose=True' in repr(pre)
    assert list(_names(KFACPreconditioner(_Gen(), precondition_conv_transpose=True,
                                          skip_layers=['ConvTranspose3d', 'up1']))) == ['up2', 'conv', 'head']
    m = _Gen()
    m.up2.bias.requires_grad_(False)
    assert 'up2' not in _names(KFACPreconditioner(m, precondition_conv_transpose=True))


def test_gradient_matrix_is_the_permuted_weight_gradient():
    """get_grad is Wmat's gradient, Wmat[co, ci * K + k] = W[ci, co, k], with the bias column last."""
    from kfac_b200.layers import ConvTransposeModuleHelper
    m = nn.ConvTranspose2d(3, 5, (2, 3))
    m.weight.grad = torch.randn_like(m.weight)
    m.bias.grad = torch.randn_like(m.bias)
    g = ConvTransposeModuleHelper(m).get_grad()
    assert g.shape == (5, 3 * 6 + 1)
    for ci, co, kh, kw in itertools.product(range(3), range(5), range(2), range(3)):
        assert g[co, ci * 6 + kh * 3 + kw] == m.weight.grad[ci, co, kh, kw]
    assert torch.equal(g[:, -1], m.bias.grad)


def test_refusals():
    from kfac_b200.preconditioner import KFACPreconditioner
    kw = dict(precondition_conv_transpose=True)
    with pytest.raises(ValueError, match=r'precondition_conv_transpose: "0" \(ConvTranspose2d\) has groups=2.*skip_layers'):
        KFACPreconditioner(nn.Sequential(nn.ConvTranspose2d(8, 8, 3, groups=2)), **kw)
    with pytest.raises(ValueError, match=r'"0" \(ConvTranspose1d\) has groups=4.*skip_layers'):
        KFACPreconditioner(nn.Sequential(nn.ConvTranspose1d(4, 4, 3, groups=4)), **kw)
    # a HiFi-GAN first upsampler: 512 * 16 + 1 = 8193 > 8192
    with pytest.raises(ValueError, match=r'"0" \(ConvTranspose1d\) has factors of 8193 \(A\).*skip_layers'):
        KFACPreconditioner(nn.Sequential(nn.ConvTranspose1d(512, 256, 16, stride=8, padding=4)), **kw)
    with pytest.raises(ValueError, match=r'"0" \(ConvTranspose3d\).*9000 \(G\).*skip_layers'):
        KFACPreconditioner(nn.Sequential(nn.ConvTranspose3d(2, 9000, 1)), **kw)
    big = nn.Sequential(nn.ConvTranspose3d(1, 2, 13))
    with pytest.raises(ValueError, match=r'"0" \(ConvTranspose3d\) has a kernel of 2197 taps.*skip_layers'):
        KFACPreconditioner(big, kfac_approx='reduce', **kw)
    KFACPreconditioner(big, **kw)
    # the largest accepted A: 512 * 16 without a bias
    KFACPreconditioner(nn.Sequential(nn.ConvTranspose1d(512, 256, 16, stride=8, padding=4, bias=False)), **kw)
    with pytest.raises(ValueError, match='"up1" \\(ConvTranspose2d\\): only torch.nn.Linear layers can keep a diagonal G'
                                         '.*skip_layers'):
        KFACPreconditioner(_Gen(), diagonal_g_layers=['up1'], **kw)
    # skipped or not registered: no refusal
    KFACPreconditioner(nn.Sequential(nn.ConvTranspose2d(8, 8, 3, groups=2)), skip_layers=['0'], **kw)
    KFACPreconditioner(nn.Sequential(nn.ConvTranspose2d(8, 8, 3, groups=2)))
    KFACPreconditioner(_Gen(), diagonal_g_layers=['up1'])


# (kernel, stride, dilation, padding, output_padding) per case; a case lists one value or one per axis
CASES_1D = [(4, 2, 1, 1, 0), (16, 8, 1, 4, 0), (3, 3, 2, 1, 2), (2, 3, 1, 0, 1), (3, 1, 1, 5, 0), (5, 2, 2, 9, 1),
            (1, 4, 1, 0, 3), (7, 3, 1, 3, 2)]
CASES_2D = [(4, 2, 1, 1, 0), (3, 2, 1, 1, 1), ((2, 3), (3, 1), (1, 2), (0, 5), (2, 0)), ((1, 5), (4, 2), 1, (1, 7), (3, 1))]
CASES_3D = [(2, 2, 1, 0, 0), ((3, 1, 2), (2, 1, 3), (2, 1, 1), (4, 0, 1), (1, 0, 2)), ((1, 4, 4), (1, 2, 2), 1, (0, 1, 1),
                                                                                       (0, 1, 0))]


def _module(nd, case):
    k, s, d, p, op = case
    cls = {1: nn.ConvTranspose1d, 2: nn.ConvTranspose2d, 3: nn.ConvTranspose3d}[nd]
    return cls(2, 3, k, stride=s, dilation=d, padding=p, output_padding=op).double()


@pytest.mark.parametrize('nd,case', [(1, c) for c in CASES_1D] + [(2, c) for c in CASES_2D] + [(3, c) for c in CASES_3D])
def test_output_extent_matches_torch(nd, case):
    """The helper's output extent is the module's output shape for the module's own output padding and for every
    output_size it accepts, passed positionally or as a keyword, batched and unbatched; the native geometry states the
    module's parameters."""
    from kfac_b200.layers import ConvTransposeModuleHelper
    m = _module(nd, case)
    h = ConvTransposeModuleHelper(m)
    ins = {1: (11,), 2: (4, 9), 3: (3, 4, 5)}[nd]
    x = torch.randn(2, 2, *ins, dtype=torch.float64)
    h.bind_call((x,), {})
    assert h.output_extent(x.shape) == tuple(m(x).shape[2:])
    assert h.output_extent(x[0].shape) == tuple(m(x[0]).shape[1:])
    # every output size torch accepts: the least (output padding 0) up to stride - 1 more on each axis
    least = [(ins[a] - 1) * m.stride[a] - 2 * m.padding[a] + m.dilation[a] * (m.kernel_size[a] - 1) + 1
             for a in range(nd)]
    for extra in itertools.product(*(range(min(s, 3)) for s in m.stride)):
        size = [least[a] + extra[a] for a in range(nd)]
        for args, kwargs in (((x, size), {}), ((x,), {'output_size': size}), ((x,), {'output_size': [2, 3] + size}),
                             ((x[0],), {'output_size': size})):
            y = m(*args, **kwargs)
            h.bind_call(args, kwargs)
            assert h.output_extent(args[0].shape) == tuple(y.shape[-nd:]) == tuple(size)
    h.bind_call((x,), {})
    geo, out = h._geometry(x.shape)
    ones, zeros = [1] * (3 - nd), [0] * (3 - nd)     # the leading axes of a 1-D or 2-D layer: extent 1, no padding
    assert (geo.batch, geo.C) == (2, 2) and list(geo.input) == ones + list(ins)
    for field, v, lead in (('kernel', m.kernel_size, ones), ('stride', m.stride, ones), ('dilation', m.dilation, ones),
                           ('padding', m.padding, zeros), ('output_padding', m.output_padding, zeros)):
        assert list(getattr(geo, field)) == lead + list(v), field
    assert out == tuple(m(x).shape[2:])


def test_kwargs_hook_only_on_transposed_layers():
    """Only the transposed convolutions get the keyword-aware input hook; every other layer keeps its hook."""
    from kfac_b200.preconditioner import KFACPreconditioner
    m = _Gen()
    pre = KFACPreconditioner(m, precondition_conv_transpose=True)
    for name in ('up1', 'up2', 'up3'):
        mod = getattr(m, name)
        assert list(mod._forward_pre_hooks_with_kwargs) == list(mod._forward_pre_hooks)
        assert [h.__func__ for h in mod._forward_pre_hooks.values()] == [type(pre)._save_input_with_kwargs]
    for name in ('conv', 'head'):
        mod = getattr(m, name)
        assert not mod._forward_pre_hooks_with_kwargs
        assert [h.__func__ for h in mod._forward_pre_hooks.values()] == [type(pre)._save_input]


def test_state_dict_round_trip():
    from kfac_b200.preconditioner import KFACPreconditioner
    pre = KFACPreconditioner(_Gen(), precondition_conv_transpose=True)
    names = _names(pre)
    for n in ('up1', 'up2', 'up3'):
        l = names[n]
        l._a_view = torch.zeros(l.a_dim, l.a_dim)        # stand-ins for the arena views (no device here)
        l._g_view = torch.zeros(l.g_dim, l.g_dim)
        A = torch.rand(l.a_dim, l.a_dim)
        G = torch.rand(l.g_dim, l.g_dim)
        l.load_state_dict({'A': A, 'G': G})
        sd = l.state_dict()
        assert torch.equal(sd['A'], A) and torch.equal(sd['G'], G)
        assert l.memory_usage()['a_factors'] == l.a_dim * l.a_dim * 4
