"""CPU tests of K-FAC-reduce (`kfac_approx='reduce'`): keyword validation, the config / repr entry, which helpers take
the reduced path and how many rows a call gives, and a state_dict round trip between an expand and a reduce
preconditioner (the factor shapes are the same)."""
import pytest
import torch
from torch import nn

from conftest import ROOT  # noqa: F401  (puts the repository on sys.path)


class _Net(nn.Module):
    def __init__(self):
        super().__init__()
        self.emb = nn.Embedding(50, 16)
        self.conv = nn.Conv2d(3, 8, 3, padding=1)
        self.fc = nn.Linear(16, 16)
        self.ln = nn.LayerNorm(16)
        self.head = nn.Linear(16, 40)

    def forward(self, idx, img):
        h = self.fc(self.emb(idx)) + self.conv(img).mean((2, 3))[:, None, :].repeat(1, 1, 2)
        return self.head(self.ln(h))


@pytest.mark.parametrize('bad', ['Reduce', 'none', '', None, 1])
def test_keyword_validation(bad):
    from kfac_b200.preconditioner import KFACPreconditioner
    with pytest.raises(ValueError, match='kfac_approx'):
        KFACPreconditioner(_Net(), kfac_approx=bad)


def test_config_and_repr():
    from kfac_b200.preconditioner import KFACPreconditioner
    off = KFACPreconditioner(_Net())
    assert off._defaults['kfac_approx'] == 'expand' and "kfac_approx=expand," in repr(off)
    on = KFACPreconditioner(_Net(), kfac_approx='reduce')
    assert on._defaults['kfac_approx'] == 'reduce' and "kfac_approx=reduce," in repr(on)
    # the same layers, in the same order, with the same shapes
    assert ([(n, l.a_factor_shape, l.g_factor_shape) for n, l in off._layers.values()]
            == [(n, l.a_factor_shape, l.g_factor_shape) for n, l in on._layers.values()])


def test_which_helpers_reduce():
    from kfac_b200.preconditioner import KFACPreconditioner
    pre = KFACPreconditioner(_Net(), kfac_approx='reduce', precondition_embeddings=True, precondition_norms=True,
                             diagonal_g_layers=['head'])
    helpers = {n: l.module for n, l in list(pre._layers.values()) + list(pre._norm_layers.values())}
    assert {n: h.reduce for n, h in helpers.items()} == {'emb': False, 'conv': True, 'fc': True, 'ln': False,
                                                         'head': True}
    assert helpers['head'].diagonal_g
    off = KFACPreconditioner(_Net(), precondition_embeddings=True, precondition_norms=True)
    assert not any(l.module.reduce for _, l in list(off._layers.values()) + list(off._norm_layers.values()))


def test_rows_per_call():
    """Dimension 0 is the example dimension; R = 1 keeps the expand rows."""
    from kfac_b200.layers import Conv2dModuleHelper, LinearModuleHelper
    lin = nn.Linear(5, 3)
    expand, reduce = LinearModuleHelper(lin), LinearModuleHelper(lin, reduce=True)
    for shape, want_reduce in (((4, 7, 5), 4), ((2, 3, 4, 5), 2), ((4, 5), 4), ((5,), 1), ((1, 9, 5), 1)):
        x = torch.zeros(shape)
        assert reduce.num_rows_a(x) == reduce.num_rows_g(x) == want_reduce, shape
        assert expand.num_rows_a(x) == x.numel() // 5
    assert reduce._positions(torch.zeros(4, 5)) is None and reduce._positions(torch.zeros(5)) is None
    assert reduce._positions(torch.zeros(4, 7, 5)) == (4, 7)
    assert expand._positions(torch.zeros(4, 7, 5)) is None
    for conv, hw, want_expand in ((nn.Conv2d(3, 8, 3, padding=1), 6, 2 * 36), (nn.Conv2d(3, 8, 7, stride=2, padding=3),
                                                                               224, 2 * 112 * 112),
                                  (nn.Conv2d(3, 8, 3), 3, 2)):
        x = torch.zeros(2, 3, hw, hw)
        e, r = Conv2dModuleHelper(conv), Conv2dModuleHelper(conv, reduce=True)
        assert e.num_rows_a(x) == want_expand
        assert r.num_rows_a(x) == 2
        g = torch.zeros(2, 8, *conv(torch.zeros(1, 3, hw, hw)).shape[2:])
        assert e.num_rows_g(g) == want_expand and r.num_rows_g(g) == 2


def _bind_standins(pre):
    for _, l in pre._layers.values():
        l._a_view = torch.zeros(l.a_factor_shape)
        l._g_view = torch.zeros(l.g_factor_shape)


@pytest.mark.parametrize('src,dst', [('expand', 'reduce'), ('reduce', 'expand')])
def test_state_dict_round_trip(src, dst):
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(0)
    kw = dict(precondition_embeddings=True, diagonal_g_layers=['head'])
    a = KFACPreconditioner(_Net(), kfac_approx=src, **kw)
    b = KFACPreconditioner(_Net(), kfac_approx=dst, **kw)
    _bind_standins(a)
    _bind_standins(b)
    for _, l in a._layers.values():
        l._a_view.copy_(torch.rand(l.a_factor_shape))
        l._g_view.copy_(torch.rand(l.g_factor_shape))
        l._has_a = l._has_g = True
    sd = a.state_dict()
    by_name = {n: l for n, l in b._layers.values()}
    for name, layer_state in sd['layers'].items():
        by_name[name].load_state_dict(layer_state)
    for (n, la), (_, lb) in zip(a._layers.values(), b._layers.values()):
        assert torch.equal(la.a_factor, lb.a_factor) and torch.equal(la.g_factor, lb.g_factor), n
    assert b.state_dict()['layers'].keys() == sd['layers'].keys()
