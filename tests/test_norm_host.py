"""CPU tests of normalization layers (`precondition_norms=True`): registration of BatchNorm1d/2d, LayerNorm and
RMSNorm, the modules that stay unregistered, skip_layers and diagonal_g_layers, the KAISA placement (identical with
the keyword off and on), and the state_dict shapes of the blocks."""
import pytest
import torch
from torch import nn

from conftest import ROOT  # noqa: F401  (puts the repository on sys.path)


class _Net(nn.Module):
    def __init__(self):
        super().__init__()
        self.conv = nn.Conv2d(3, 8, 3)
        self.bn2 = nn.BatchNorm2d(8)
        self.fc = nn.Linear(8, 16)
        self.bn1 = nn.BatchNorm1d(16)
        self.ln = nn.LayerNorm(16)
        self.ln_nobias = nn.LayerNorm((4, 4), bias=False)
        self.rms = nn.RMSNorm(16)
        self.head = nn.Linear(16, 5)

    def forward(self, x):
        h = self.bn2(self.conv(x)).mean((2, 3))
        h = self.ln(self.bn1(self.fc(h)))
        h = self.rms(self.ln_nobias(h.view(-1, 4, 4)).flatten(1))
        return self.head(h)


DENSE = ['conv', 'fc', 'head']
NORMS = ['bn2', 'bn1', 'ln', 'ln_nobias', 'rms']


def test_registration_only_with_the_keyword():
    from kfac_b200.preconditioner import KFACPreconditioner
    off = KFACPreconditioner(_Net())
    assert [n for n, _ in off._layers.values()] == DENSE and off._norm_layers == {}
    assert 'precondition_norms=False' in repr(off)
    on = KFACPreconditioner(_Net(), precondition_norms=True)
    assert [n for n, _ in on._layers.values()] == DENSE
    assert [n for n, _ in on._norm_layers.values()] == NORMS
    assert 'precondition_norms=True' in repr(on)
    layers = {n: l for n, l in on._norm_layers.values()}
    for name, (C, k, np_) in {'bn2': (8, 3, 2), 'bn1': (16, 3, 2), 'ln': (16, 3, 2), 'ln_nobias': (16, 1, 1),
                              'rms': (16, 1, 1)}.items():
        l = layers[name]
        assert l.norm and l.diag_side is None
        assert l.g_dim == C and l.module.k == k and l.a_dim == np_
        assert l.g_factor_shape == (C, k) and l.p_shape == (C, np_) and l.a_factor_shape == ()
    kinds = {n: l.module.kind for n, l in layers.items()}
    assert kinds == {'bn2': 0, 'bn1': 0, 'ln': 1, 'ln_nobias': 1, 'rms': 2}
    # the other layers' indices do not move
    assert [l.index for _, l in on._layers.values()] == [l.index for _, l in off._layers.values()] == [0, 1, 2]
    assert [l.index for _, l in on._norm_layers.values()] == list(range(len(NORMS)))


def test_rmsnorm_default_eps_is_that_of_the_computation_type():
    """RMSNorm(eps=None) adds torch's opmath epsilon: float32's for fp16 / bf16 / fp32 inputs, float64's for fp64 -- the
    statistics use it, and it is what the module's own forward uses."""
    from kfac_b200.layers import NormModuleHelper
    m = nn.RMSNorm(8)
    h = NormModuleHelper(m)
    f32, f64 = torch.finfo(torch.float32).eps, torch.finfo(torch.float64).eps
    for dtype, want in ((torch.float16, f32), (torch.bfloat16, f32), (torch.float32, f32), (torch.float64, f64)):
        assert h.eps_for(torch.zeros(1, 8, dtype=dtype)) == want, dtype
        # small activations make the eps visible; the module's forward agrees with the restatement with `want`
        x = (torch.randn(64, 8, generator=torch.Generator().manual_seed(0), dtype=torch.float64) * 0.02).to(dtype)
        with torch.no_grad():
            y = m.to(dtype)(x).double()
        xd = x.double()
        ref = xd / torch.sqrt((xd * xd).mean(1, keepdim=True) + want)
        assert float((y - ref).abs().max()) <= 2 ** -7 * float(ref.abs().max()), dtype
    assert NormModuleHelper(nn.RMSNorm(8, eps=1e-3)).eps_for(torch.zeros(1, 8, dtype=torch.bfloat16)) == 1e-3


@pytest.mark.parametrize('module', [
    nn.BatchNorm2d(4, affine=False), nn.BatchNorm1d(4, affine=False), nn.LayerNorm(4, elementwise_affine=False),
    nn.RMSNorm(4, elementwise_affine=False), nn.SyncBatchNorm(4), nn.GroupNorm(2, 4), nn.InstanceNorm2d(4, affine=True),
    nn.BatchNorm3d(4)], ids=lambda m: repr(m))
def test_unsupported_modules_are_not_registered(module):
    from kfac_b200.preconditioner import KFACPreconditioner
    pre = KFACPreconditioner(nn.Sequential(nn.Linear(4, 4), module), precondition_norms=True)
    assert pre._norm_layers == {} and [n for n, _ in pre._layers.values()] == ['0']


def test_frozen_affine_parameters_are_not_registered():
    from kfac_b200.preconditioner import KFACPreconditioner
    model = nn.Sequential(nn.Linear(4, 4), nn.LayerNorm(4))
    model[1].weight.requires_grad_(False)
    assert KFACPreconditioner(model, precondition_norms=True)._norm_layers == {}


def test_skip_layers_and_diagonal_g_layers():
    from kfac_b200.preconditioner import KFACPreconditioner
    pre = KFACPreconditioner(_Net(), precondition_norms=True, skip_layers=['bn1', 'RMSNorm'])
    assert [n for n, _ in pre._norm_layers.values()] == ['bn2', 'ln', 'ln_nobias']
    with pytest.raises(ValueError, match='"ln".*LayerNorm.*only torch.nn.Linear'):
        KFACPreconditioner(_Net(), precondition_norms=True, diagonal_g_layers=['^ln$'])
    # unregistered (keyword off, or skipped): no error
    KFACPreconditioner(_Net(), diagonal_g_layers=['^ln$'])
    KFACPreconditioner(_Net(), precondition_norms=True, diagonal_g_layers=['^ln$'], skip_layers=['^ln$'])
    # EKFAC: the norm blocks take the same P, so no error
    KFACPreconditioner(_Net(), precondition_norms=True, compute_method='ekfac')


@pytest.mark.parametrize('world,frac', [(1, 1.0), (2, 1.0), (2, 0.5), (4, 0.5), (4, 0.25), (8, 0.125)])
def test_placement_identical_with_the_keyword_off_and_on(world, frac):
    from kfac_b200.assignment import KAISAAssignment
    from kfac_b200.base_preconditioner import build_comm_plan
    from kfac_b200.enums import AssignmentStrategy, ComputeMethod
    from kfac_b200.layers import register_modules
    from kfac_b200.preconditioner import layer_work
    model = _Net()

    def placement(norms, rank):
        layers = register_modules(model, [], precondition_norms=norms, method=ComputeMethod.EIGEN)
        dense = {m: v for m, v in layers.items() if not v[1].norm}
        assert len(dense) < len(layers) if norms else len(dense) == len(layers)
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
    pre = KFACPreconditioner(_Net(), precondition_norms=True)
    layers = {n: l for n, l in pre._norm_layers.values()}
    bn, rms = layers['bn2'], layers['rms']
    bn._g_view = torch.zeros(8, 3)        # stand-ins for the arena views (no device here)
    rms._g_view = torch.zeros(16, 1)
    assert bn.state_dict() == {'A': None, 'G': None}
    blocks = torch.rand(8, 3)
    bn.load_state_dict({'A': None, 'G': blocks})
    sd = bn.state_dict()
    assert sd['A'] is None and torch.equal(sd['G'], blocks) and sd['G'].data_ptr() != bn._g_view.data_ptr()
    rms.load_state_dict({'A': None, 'G': torch.ones(16, 1)})
    assert rms.state_dict()['G'].shape == (16, 1)
    for bad in ({'A': None, 'G': torch.ones(8, 2)}, {'A': None, 'G': torch.ones(24)},
                {'A': torch.ones(2, 2), 'G': blocks}):
        with pytest.raises(ValueError):
            bn.load_state_dict(bad)
    with pytest.raises(ValueError, match='shape'):
        rms.load_state_dict({'A': None, 'G': torch.ones(16)})
    use = bn.memory_usage()
    assert use['g_factors'] == 8 * 3 * 4 and use['a_factors'] == 0 and use['a_batch'] == 0
    assert set(use) == {'a_factors', 'g_factors', 'a_batch', 'g_batch', 'a_inverses', 'g_inverses'}
