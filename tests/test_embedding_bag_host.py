"""CPU tests of embedding-bag preconditioning (`precondition_embedding_bags=True`): registration, every refusal,
skip_layers and frozen weights, the linear A cost in the KAISA placement, comm-plan consistency across ranks and the
state_dict shape checks."""
import pytest
import torch
from torch import nn

from conftest import ROOT  # noqa: F401  (puts the repository on sys.path)


class _Classifier(nn.Module):
    """The text classifier of PyTorch's tutorial: a mean bag over the vocabulary and a Linear head."""

    def __init__(self, V=1000, d=64, classes=4, head_weight=False, **bag_kw):
        super().__init__()
        self.bag = nn.EmbeddingBag(V, d, **bag_kw)
        self.fc = nn.Linear(d, classes)
        if head_weight:                     # a head that uses the bag's weight (V, d) as its own
            self.fc = nn.Linear(d, V, bias=False)
            self.fc.weight = self.bag.weight

    def forward(self, idx, offsets=None):
        return self.fc(self.bag(idx, offsets))


def _names(pre):
    return [n for n, _ in pre._layers.values()]


def test_registration_on_and_off():
    from kfac_b200.preconditioner import KFACPreconditioner
    off = KFACPreconditioner(_Classifier())
    assert _names(off) == ['fc']
    assert 'precondition_embedding_bags=False' in repr(off)
    on = KFACPreconditioner(_Classifier(), precondition_embedding_bags=True)
    layers = {n: l for n, l in on._layers.values()}
    assert list(layers) == ['bag', 'fc']
    bag = layers['bag']
    assert bag.diag_a and bag.embedding and not bag.diag_g
    assert bag.a_dim == 1000 and bag.g_dim == 64 and bag.p_shape == (1000, 64)
    assert bag.a_factor_shape == (1000,) and bag.g_factor_shape == (64, 64)
    assert 'precondition_embedding_bags=True' in repr(on)
    # independent of precondition_embeddings, in both directions
    mixed = nn.ModuleDict({'emb': nn.Embedding(50, 8), 'bag': nn.EmbeddingBag(60, 8), 'fc': nn.Linear(8, 2)})
    assert _names(KFACPreconditioner(mixed, precondition_embeddings=True)) == ['emb', 'fc']
    assert _names(KFACPreconditioner(mixed, precondition_embedding_bags=True)) == ['bag', 'fc']
    assert _names(KFACPreconditioner(mixed, precondition_embeddings=True, precondition_embedding_bags=True)) == [
        'emb', 'bag', 'fc']
    # K-FAC-reduce leaves the bag's statistics alone: every bag is already one row
    reduce = KFACPreconditioner(_Classifier(), precondition_embedding_bags=True, kfac_approx='reduce')
    assert not next(l for n, l in reduce._layers.values() if n == 'bag').module.reduce


def test_skip_layers_and_frozen_weights():
    from kfac_b200.preconditioner import KFACPreconditioner
    assert _names(KFACPreconditioner(_Classifier(), precondition_embedding_bags=True, skip_layers=['bag'])) == ['fc']
    assert _names(KFACPreconditioner(_Classifier(), precondition_embedding_bags=True,
                                     skip_layers=['EmbeddingBag'])) == ['fc']
    frozen = _Classifier()
    frozen.bag.weight.requires_grad_(False)
    assert _names(KFACPreconditioner(frozen, precondition_embedding_bags=True)) == ['fc']


@pytest.mark.parametrize('model_kw,kw,match', [
    ({'mode': 'max'}, {}, '"bag".*mode=\'max\'.*Kronecker.*skip_layers'),
    ({'sparse': True}, {}, 'embedding bag "bag" has sparse=True.*skip_layers'),
    ({'scale_grad_by_freq': True}, {}, 'embedding bag "bag" has scale_grad_by_freq=True.*skip_layers'),
    ({}, {'compute_method': 'ekfac'}, 'precondition_embedding_bags.*EKFAC.*"bag".*skip_layers'),
    ({}, {'diagonal_g_layers': ['bag']}, 'diagonal_g_layers matches "bag".*skip_layers'),
    ({}, {'diagonal_a_layers': ['bag']}, 'diagonal_a_layers matches "bag".*skip_layers'),
    ({'head_weight': True}, {}, 'embedding bag "bag" shares its weight with "fc".*skip_layers'),
    # a bag never forms a tied pair: the shared weight stays refused with precondition_tied_embeddings as well
    ({'head_weight': True}, {'precondition_tied_embeddings': True, 'diagonal_g_layers': ['fc']},
     'embedding bag "bag" shares its weight with "fc".*skip_layers'),
])
def test_refusals(model_kw, kw, match):
    from kfac_b200.preconditioner import KFACPreconditioner
    with pytest.raises(ValueError, match=match):
        KFACPreconditioner(_Classifier(**model_kw), precondition_embedding_bags=True, **kw)
    # fine once the bag is not registered (keyword off or skipped)
    KFACPreconditioner(_Classifier(**model_kw), **kw)
    KFACPreconditioner(_Classifier(**model_kw), precondition_embedding_bags=True, skip_layers=['bag'], **kw)


def test_tied_pairs_skip_bags():
    from kfac_b200.enums import ComputeMethod
    from kfac_b200.layers import register_modules
    from kfac_b200.preconditioner import _tie_pairs
    layers = register_modules(_Classifier(head_weight=True), [], precondition_embedding_bags=True,
                              diagonal_g_layers=['fc'], method=ComputeMethod.EIGEN)
    _tie_pairs(layers, ComputeMethod.EIGEN)
    assert all(l.tied_head is None and l.tied_embedding is None for _, l in layers.values())


def test_kaisa_cost_of_the_bag_is_linear():
    from kfac_b200.enums import AssignmentStrategy
    from kfac_b200.layers import register_modules
    from kfac_b200.preconditioner import layer_work
    layers = register_modules(_Classifier(V=95811, d=64), [], precondition_embedding_bags=True, method=None)
    for strategy, cost in ((AssignmentStrategy.COMPUTE, lambda n: n ** 3), (AssignmentStrategy.MEMORY, lambda n: n ** 2)):
        work = layer_work(layers, strategy)
        assert work['bag'] == {'A': 95811, 'G': cost(64)}
        assert work['fc'] == {'A': cost(65), 'G': cost(4)}


def _plans(world, frac, method, prediv, colocate):
    from kfac_b200.assignment import KAISAAssignment
    from kfac_b200.base_preconditioner import build_comm_plan
    from kfac_b200.enums import AssignmentStrategy
    from kfac_b200.layers import register_modules
    from kfac_b200.preconditioner import layer_work
    torch.manual_seed(0)
    model = nn.Sequential(nn.EmbeddingBag(1000, 48), nn.Linear(48, 64), nn.EmbeddingBag(30, 8, mode='sum'),
                          nn.Embedding(40, 8), nn.Conv2d(3, 8, 3), nn.Linear(64, 10))
    out = []
    handles = {}
    for rank in range(world):
        layers = register_modules(model, [], precondition_embeddings=True, precondition_embedding_bags=True,
                                  method=method, prediv_eigenvalues=prediv)
        ll = list(layers.values())
        a = KAISAAssignment(layer_work(layers, AssignmentStrategy.COMPUTE), local_rank=rank, world_size=world,
                            grad_worker_fraction=frac,
                            group_func=lambda r: handles.setdefault(tuple(sorted(r)), tuple(sorted(r))),
                            colocate_factors=colocate)
        out.append((a, ll, build_comm_plan(ll, a)))
    return out


@pytest.mark.parametrize('world,frac', [(1, 1.0), (2, 1.0), (2, 0.5), (3, 1.0), (4, 1.0), (4, 0.5), (4, 0.25),
                                        (5, 0.2), (6, 0.5), (7, 1.0), (8, 1.0), (8, 0.5), (8, 0.125)])
@pytest.mark.parametrize('method,prediv,colocate', [('EIGEN', True, True), ('EIGEN', False, False),
                                                    ('INVERSE', False, True)])
def test_comm_plan_with_embedding_bags_consistent_across_ranks(world, frac, method, prediv, colocate):
    """COMM_OPT (frac 1), HYBRID_OPT and MEM_OPT (frac 1/world) for world sizes 1-8: every (group, src) broadcast
    looks the same on every member, a bag ships qg, dg, da (eigen) or g_inv and da (inverse) and never a dgda, and
    its P is stored in the weight's layout."""
    from kfac_b200.base_preconditioner import _storage_numel
    from kfac_b200.enums import ComputeMethod
    if colocate is False and frac * world <= 1:
        colocate = True
    plans = _plans(world, frac, ComputeMethod[method], prediv, colocate)
    for kind in (0, 1):
        per_rank = [[(s.group, s.src, s.numel, [(l.index, k, sh) for l, k, sh in s.entries]) for s in plan[kind]]
                    for _, _, plan in plans]
        for rank, segs in enumerate(per_rank):
            for grp, src, numel, entries in segs:
                assert rank in grp and src in grp
                for other in grp:
                    assert [s for s in per_rank[other] if s[0] == grp] == [s for s in segs if s[0] == grp]
    for a, ll, (inv, grad) in plans:
        assert sorted(l.index for s in grad for l, _, _ in s.entries) == list(range(len(ll)))
        for s in inv + grad:
            assert s.offset % 4 == 0 and s.numel == sum(_storage_numel(sh) for _, _, sh in s.entries)
        bags = [(name, l) for name, l in ll if isinstance(l.module.module, nn.EmbeddingBag)]
        assert len(bags) == 2
        for name, l in bags:
            keys = {k: sh for s in inv for ll_, k, sh in s.entries if ll_ is l}
            if a.is_grad_worker(name):
                want = ({'da': (l.a_dim,), 'qg': (l.g_dim, l.g_dim), 'dg': (l.g_dim,)} if method == 'EIGEN'
                        else {'da': (l.a_dim,), 'g_inv': (l.g_dim, l.g_dim)})
                assert keys == want
            else:
                assert keys == {}
            assert [sh for s in grad for ll_, k, sh in s.entries if ll_ is l] == [(l.a_dim, l.g_dim)]


def test_state_dict_shape_check():
    from kfac_b200.preconditioner import KFACPreconditioner
    pre = KFACPreconditioner(_Classifier(V=10, d=4), precondition_embedding_bags=True)
    bag = next(l for _, l in pre._layers.values() if l.diag_a)
    bag._a_view = torch.zeros(10)          # stand-ins for the arena views (no device here)
    bag._g_view = torch.zeros(4, 4)
    bag.load_state_dict({'A': torch.ones(10), 'G': torch.eye(4)})
    assert torch.equal(bag.a_factor, torch.ones(10)) and bag.qa is None and bag.a_inv is None
    assert torch.equal(bag.state_dict()['A'], torch.ones(10))
    with pytest.raises(ValueError, match='shape'):
        bag.load_state_dict({'A': torch.eye(10), 'G': torch.eye(4)})
    with pytest.raises(ValueError, match='shape'):
        bag.load_state_dict({'A': torch.ones(11), 'G': torch.eye(4)})
    with pytest.raises(ValueError, match='shape'):
        bag.load_state_dict({'A': torch.ones(10), 'G': torch.eye(5)})
    assert bag.memory_usage()['a_factors'] == 10 * 4
