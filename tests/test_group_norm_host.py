"""CPU tests of GroupNorm / InstanceNorm layers (`precondition_group_norms=True`): registration only with the keyword,
the modules that stay unregistered, skip_layers and diagonal_g_layers, the other layers' indices and the KAISA
placement (identical with the keyword off and on), independence from `precondition_norms`, and the shapes, kind and
groups of the blocks."""
import pytest
import torch
from torch import nn

from conftest import ROOT  # noqa: F401  (puts the repository on sys.path)


class _Net(nn.Module):
    def __init__(self):
        super().__init__()
        self.conv = nn.Conv2d(3, 64, 3)
        self.gn = nn.GroupNorm(32, 64)
        self.gn1 = nn.GroupNorm(1, 64)
        self.in2 = nn.InstanceNorm2d(64, affine=True)
        self.bn = nn.BatchNorm2d(64)
        self.fc = nn.Linear(64, 16)
        self.gn_flat = nn.GroupNorm(8, 16)
        self.in1 = nn.InstanceNorm1d(4, affine=True)
        self.in3 = nn.InstanceNorm3d(2, affine=True)
        self.head = nn.Linear(16, 5)

    def forward(self, x):
        h = self.bn(self.in2(self.gn1(self.gn(self.conv(x))))).mean((2, 3))
        h = self.gn_flat(self.fc(h))
        h = self.in1(h.view(-1, 4, 4)).view(-1, 2, 2, 2, 2)
        return self.head(self.in3(h).flatten(1))


DENSE = ['conv', 'fc', 'head']
GROUP_NORMS = ['gn', 'gn1', 'in2', 'gn_flat', 'in1', 'in3']


def test_registration_only_with_the_keyword():
    from kfac_b200 import _cabi
    from kfac_b200.preconditioner import KFACPreconditioner
    off = KFACPreconditioner(_Net())
    assert [n for n, _ in off._layers.values()] == DENSE and off._norm_layers == {}
    assert 'precondition_group_norms=False' in repr(off)
    # precondition_norms alone keeps registering BatchNorm only
    norms = KFACPreconditioner(_Net(), precondition_norms=True)
    assert [n for n, _ in norms._norm_layers.values()] == ['bn']
    on = KFACPreconditioner(_Net(), precondition_group_norms=True)
    assert 'precondition_group_norms=True' in repr(on)
    assert on._defaults['precondition_group_norms'] is True
    assert [n for n, _ in on._layers.values()] == DENSE
    assert [n for n, _ in on._norm_layers.values()] == GROUP_NORMS
    layers = {n: l for n, l in on._norm_layers.values()}
    want = {'gn': (64, 32), 'gn1': (64, 1), 'in2': (64, 64), 'gn_flat': (16, 8), 'in1': (4, 4), 'in3': (2, 2)}
    for name, (C, groups) in want.items():
        l = layers[name]
        assert l.norm and l.diag_side is None
        assert l.module.kind == _cabi.KFAC_NORM_GROUP and l.module.groups == groups
        assert l.g_dim == C and l.module.k == 3 and l.a_dim == 2
        assert l.g_factor_shape == (C, 3) and l.p_shape == (C, 2) and l.a_factor_shape == ()
    # both keywords: the union, in module order
    both = KFACPreconditioner(_Net(), precondition_norms=True, precondition_group_norms=True)
    assert [n for n, _ in both._norm_layers.values()] == ['gn', 'gn1', 'in2', 'bn', 'gn_flat', 'in1', 'in3']
    assert {n: l.module.kind for n, l in both._norm_layers.values()}['bn'] == _cabi.KFAC_NORM_BATCH
    # the other layers' indices do not move
    for p in (on, both):
        assert [l.index for _, l in p._layers.values()] == [l.index for _, l in off._layers.values()] == [0, 1, 2]
        assert [l.index for _, l in p._norm_layers.values()] == list(range(len(p._norm_layers)))


@pytest.mark.parametrize('module', [
    nn.GroupNorm(2, 4, affine=False), nn.InstanceNorm1d(4), nn.InstanceNorm2d(4), nn.InstanceNorm3d(4),
    nn.InstanceNorm2d(4, affine=False, track_running_stats=True), nn.BatchNorm2d(4), nn.LayerNorm(4),
    nn.SyncBatchNorm(4), nn.BatchNorm3d(4)], ids=lambda m: repr(m))
def test_unsupported_modules_are_not_registered(module):
    from kfac_b200.preconditioner import KFACPreconditioner
    pre = KFACPreconditioner(nn.Sequential(nn.Linear(4, 4), module), precondition_group_norms=True)
    assert pre._norm_layers == {} and [n for n, _ in pre._layers.values()] == ['0']


@pytest.mark.parametrize('module', [nn.GroupNorm(2, 4), nn.InstanceNorm2d(4, affine=True)], ids=lambda m: repr(m))
@pytest.mark.parametrize('frozen', ['weight', 'bias'])
def test_frozen_affine_parameters_are_not_registered(module, frozen):
    from kfac_b200.preconditioner import KFACPreconditioner
    model = nn.Sequential(nn.Linear(4, 4), module)
    getattr(model[1], frozen).requires_grad_(False)
    assert KFACPreconditioner(model, precondition_group_norms=True)._norm_layers == {}


def test_skip_layers_and_diagonal_g_layers():
    from kfac_b200.preconditioner import KFACPreconditioner
    pre = KFACPreconditioner(_Net(), precondition_group_norms=True, skip_layers=['gn1', 'InstanceNorm3d'])
    assert [n for n, _ in pre._norm_layers.values()] == ['gn', 'in2', 'gn_flat', 'in1']
    with pytest.raises(ValueError, match='"gn".*GroupNorm.*only torch.nn.Linear'):
        KFACPreconditioner(_Net(), precondition_group_norms=True, diagonal_g_layers=['^gn$'])
    with pytest.raises(ValueError, match='"in2".*InstanceNorm2d.*only torch.nn.Linear'):
        KFACPreconditioner(_Net(), precondition_group_norms=True, diagonal_g_layers=['InstanceNorm2d'])
    # unregistered (keyword off, or skipped): no error
    KFACPreconditioner(_Net(), diagonal_g_layers=['^gn$'])
    KFACPreconditioner(_Net(), precondition_norms=True, diagonal_g_layers=['^gn$'])
    KFACPreconditioner(_Net(), precondition_group_norms=True, diagonal_g_layers=['^gn$'], skip_layers=['^gn$'])
    # EKFAC: the norm blocks take the same P, so no error
    KFACPreconditioner(_Net(), precondition_group_norms=True, compute_method='ekfac')


@pytest.mark.parametrize('world,frac', [(1, 1.0), (2, 1.0), (2, 0.5), (4, 0.5), (4, 0.25), (8, 0.125)])
def test_placement_identical_with_the_keyword_off_and_on(world, frac):
    from kfac_b200.assignment import KAISAAssignment
    from kfac_b200.base_preconditioner import build_comm_plan
    from kfac_b200.enums import AssignmentStrategy, ComputeMethod
    from kfac_b200.layers import register_modules
    from kfac_b200.preconditioner import layer_work
    model = _Net()

    def placement(group_norms, rank):
        layers = register_modules(model, [], precondition_group_norms=group_norms, method=ComputeMethod.EIGEN)
        dense = {m: v for m, v in layers.items() if not v[1].norm}
        assert len(dense) < len(layers) if group_norms else len(dense) == len(layers)
        work = layer_work(dense, AssignmentStrategy.COMPUTE)
        handles = {}
        a = KAISAAssignment(work, local_rank=rank, world_size=world, grad_worker_fraction=frac,
                            group_func=lambda r: handles.setdefault(tuple(sorted(r)), tuple(sorted(r))),
                            colocate_factors=True)
        inv, grad = build_comm_plan(list(dense.values()), a)
        segs = [(s.group, s.src, s.numel, [(l.index, k, sh) for l, k, sh in s.entries]) for s in inv + grad]
        return list(work.items()), repr(a), segs

    for rank in range(world):
        assert placement(False, rank) == placement(True, rank)


def test_state_dict_shapes():
    from kfac_b200.preconditioner import KFACPreconditioner
    pre = KFACPreconditioner(_Net(), precondition_group_norms=True)
    l = {n: l for n, l in pre._norm_layers.values()}['gn']
    l._g_view = torch.zeros(64, 3)          # a stand-in for the arena view (no device here)
    blocks = torch.rand(64, 3)
    l.load_state_dict({'A': None, 'G': blocks})
    sd = l.state_dict()
    assert sd['A'] is None and torch.equal(sd['G'], blocks)
    for bad in ({'A': None, 'G': torch.ones(64, 2)}, {'A': torch.ones(2, 2), 'G': blocks}):
        with pytest.raises(ValueError):
            l.load_state_dict(bad)
    use = l.memory_usage()
    assert use['g_factors'] == 64 * 3 * 4 and use['a_factors'] == 0
