"""CPU tests of embedding preconditioning (`precondition_embeddings=True`): registration, constructor validation,
comm-plan consistency across ranks with an embedding layer present, and the linear A cost in the KAISA placement."""
import pytest
import torch
from torch import nn

from conftest import ROOT  # noqa: F401  (puts the repository on sys.path)


class _LM(nn.Module):
    def __init__(self, V=1000, d=64, tie=False, **emb_kw):
        super().__init__()
        self.emb = nn.Embedding(V, d, **emb_kw)
        self.hidden = nn.Linear(d, d)
        self.head = nn.Linear(d, V, bias=False)
        if tie:
            self.head.weight = self.emb.weight

    def forward(self, idx):
        return self.head(torch.tanh(self.hidden(self.emb(idx))))


def test_registration_on_and_off():
    from kfac_b200.preconditioner import KFACPreconditioner
    off = KFACPreconditioner(_LM())
    assert [n for n, _ in off._layers.values()] == ['hidden', 'head']
    assert 'precondition_embeddings=False' in repr(off)
    on = KFACPreconditioner(_LM(), precondition_embeddings=True)
    names = {n: l for n, l in on._layers.values()}
    assert list(names) == ['emb', 'hidden', 'head']
    emb = names['emb']
    assert emb.diag_a and emb.a_dim == 1000 and emb.g_dim == 64 and emb.p_shape == (1000, 64)
    assert not names['hidden'].diag_a and names['hidden'].p_shape == (64, 65)
    assert 'precondition_embeddings=True' in repr(on)
    # skip_layers and requires_grad apply as for any layer; EmbeddingBag is not covered
    assert 'emb' not in {n for n, _ in KFACPreconditioner(_LM(), precondition_embeddings=True,
                                                          skip_layers=['emb'])._layers.values()}
    frozen = _LM()
    frozen.emb.weight.requires_grad_(False)
    assert 'emb' not in {n for n, _ in KFACPreconditioner(frozen, precondition_embeddings=True)._layers.values()}
    bag = nn.Sequential(nn.EmbeddingBag(100, 8), nn.Linear(8, 2))
    assert len(KFACPreconditioner(bag, precondition_embeddings=True)._layers) == 1


def test_constructor_rejects_unsupported_embeddings():
    from kfac_b200.preconditioner import KFACPreconditioner
    with pytest.raises(ValueError, match='"emb".*sparse'):
        KFACPreconditioner(_LM(sparse=True), precondition_embeddings=True)
    with pytest.raises(ValueError, match='"emb".*scale_grad_by_freq'):
        KFACPreconditioner(_LM(scale_grad_by_freq=True), precondition_embeddings=True)
    with pytest.raises(ValueError, match='EKFAC'):
        KFACPreconditioner(_LM(), precondition_embeddings=True, compute_method='ekfac')
    with pytest.raises(ValueError, match='"emb" shares its weight with "head".*skip_layers'):
        KFACPreconditioner(_LM(tie=True), precondition_embeddings=True)
    # each of them is fine once the embedding is not registered (keyword off or skipped), and a tied head is
    # fine once one of the two layers is skipped
    KFACPreconditioner(_LM(sparse=True))
    KFACPreconditioner(_LM(sparse=True), precondition_embeddings=True, skip_layers=['emb'])
    KFACPreconditioner(_LM(), compute_method='ekfac')
    KFACPreconditioner(_LM(tie=True), precondition_embeddings=True, skip_layers=['head'])


def test_state_dict_shape_check():
    from kfac_b200.preconditioner import KFACPreconditioner
    pre = KFACPreconditioner(_LM(V=10, d=4), precondition_embeddings=True)
    emb = next(l for _, l in pre._layers.values() if l.diag_a)
    emb._a_view = torch.zeros(10)          # stand-ins for the arena views (no device here)
    emb._g_view = torch.zeros(4, 4)
    emb.load_state_dict({'A': torch.ones(10), 'G': torch.eye(4)})
    assert torch.equal(emb.a_factor, torch.ones(10)) and emb.qa is None and emb.a_inv is None
    with pytest.raises(ValueError, match='shape'):
        emb.load_state_dict({'A': torch.eye(10), 'G': torch.eye(4)})
    with pytest.raises(ValueError, match='shape'):
        emb.load_state_dict({'A': torch.ones(10), 'G': torch.eye(5)})
    assert emb.memory_usage()['a_factors'] == 10 * 4


def test_kaisa_cost_of_a_diagonal_factor_is_linear():
    from kfac_b200.assignment import KAISAAssignment
    from kfac_b200.enums import AssignmentStrategy
    from kfac_b200.layers import register_modules
    from kfac_b200.preconditioner import layer_work
    layers = register_modules(_LM(V=50257, d=64), [], precondition_embeddings=True, method=None)
    for strategy, cost in ((AssignmentStrategy.COMPUTE, lambda n: n ** 3), (AssignmentStrategy.MEMORY, lambda n: n ** 2)):
        work = layer_work(layers, strategy)
        assert work['emb'] == {'A': 50257, 'G': cost(64)}
        assert work['hidden'] == {'A': cost(65), 'G': cost(64)}
        assert work['head'] == {'A': cost(64), 'G': cost(50257)}
    # the keyword off: the same table as before for the registered layers
    assert layer_work(register_modules(_LM(), [], method=None), AssignmentStrategy.COMPUTE) == {
        'hidden': {'A': 65 ** 3, 'G': 64 ** 3}, 'head': {'A': 64 ** 3, 'G': 1000 ** 3}}
    # four ranks, one grad worker each: the embedding weighs what its G weighs plus V, and is not the heaviest layer
    many = nn.Sequential(nn.Embedding(50257, 256), *[nn.Linear(256, 256) for _ in range(6)])
    layers = register_modules(many, [], precondition_embeddings=True, method=None)
    work = layer_work(layers, AssignmentStrategy.COMPUTE)
    assert work['0']['A'] + work['0']['G'] < work['1']['A'] + work['1']['G']
    a = KAISAAssignment(work, local_rank=0, world_size=4, grad_worker_fraction=1.0, group_func=lambda r: None)
    ranks = [a.inv_worker(n, 'A') for n in work]
    assert sorted(set(ranks)) == [0, 1, 2, 3]


def _plans(world, frac, method, prediv, colocate):
    from kfac_b200.assignment import KAISAAssignment
    from kfac_b200.base_preconditioner import build_comm_plan
    from kfac_b200.enums import AssignmentStrategy
    from kfac_b200.layers import register_modules
    from kfac_b200.preconditioner import layer_work
    torch.manual_seed(0)
    model = nn.Sequential(nn.Embedding(1000, 48), nn.Linear(48, 64), nn.Embedding(30, 8),
                          nn.Conv2d(3, 8, 3), nn.Linear(64, 10))
    out = []
    handles = {}
    for rank in range(world):
        layers = register_modules(model, [], precondition_embeddings=True, method=method, prediv_eigenvalues=prediv)
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
def test_comm_plan_with_embeddings_consistent_across_ranks(world, frac, method, prediv, colocate):
    """COMM_OPT (frac 1), HYBRID_OPT and MEM_OPT (frac 1/world) for world sizes 1-8: every (group, src) broadcast
    looks the same on every member, an embedding ships qg, dg, da (eigen) or g_inv and da (inverse) and never a
    dgda, and its P is stored in the weight's layout."""
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
        for name, l in ll:
            if not l.diag_a:
                continue
            keys = {k: sh for s in inv for ll_, k, sh in s.entries if ll_ is l}
            if a.is_grad_worker(name):
                want = ({'da': (l.a_dim,), 'qg': (l.g_dim, l.g_dim), 'dg': (l.g_dim,)} if method == 'EIGEN'
                        else {'da': (l.a_dim,), 'g_inv': (l.g_dim, l.g_dim)})
                assert keys == want
            else:
                assert keys == {}
            assert [sh for s in grad for ll_, k, sh in s.entries if ll_ is l] == [(l.a_dim, l.g_dim)]
