"""CPU tests of tied embedding / LM-head pairs (`precondition_tied_embeddings=True`): registration and repr, the
refusals, `skip_layers` precedence, the placement cost of a pair, and comm-plan consistency across ranks."""
import pytest
import torch
from torch import nn

from conftest import ROOT  # noqa: F401  (puts the repository on sys.path)

KW = dict(precondition_embeddings=True, diagonal_g_layers=['head'], precondition_tied_embeddings=True)


class _LM(nn.Module):
    def __init__(self, V=1000, d=64, tie=True, bias=False):
        super().__init__()
        self.emb = nn.Embedding(V, d)
        self.hidden = nn.Linear(d, d)
        self.head = nn.Linear(d, V, bias=bias)
        if tie:
            self.head.weight = self.emb.weight

    def forward(self, idx):
        return self.head(torch.tanh(self.hidden(self.emb(idx))))


def _names(pre):
    return {n: l for n, l in pre._layers.values()}


def test_registration_and_repr():
    from kfac_b200.preconditioner import KFACPreconditioner
    pre = KFACPreconditioner(_LM(), **KW)
    names = _names(pre)
    emb, head = names['emb'], names['head']
    assert emb.tied_head is head and head.tied_embedding is emb
    assert emb.tied_embedding is None and head.tied_head is None and names['hidden'].tied_head is None
    assert emb.p_shape == (1000, 64) and head.diag_g and emb.diag_a
    assert 'precondition_tied_embeddings=True' in repr(pre)
    assert 'precondition_tied_embeddings=False' in repr(KFACPreconditioner(_LM(tie=False)))
    # the keyword on without a tied weight: the same layers, no pair
    untied = _names(KFACPreconditioner(_LM(tie=False), **KW))
    assert list(untied) == ['emb', 'hidden', 'head']
    assert all(l.tied_head is None and l.tied_embedding is None for l in untied.values())
    # the head alone (embeddings not registered) is a diagonal-G layer as before
    alone = _names(KFACPreconditioner(_LM(), diagonal_g_layers=['head'], precondition_tied_embeddings=True))
    assert list(alone) == ['hidden', 'head'] and alone['head'].tied_embedding is None


def test_existing_refusals_with_the_keyword_off():
    from kfac_b200.preconditioner import KFACPreconditioner
    with pytest.raises(ValueError, match='"emb" shares its weight with "head".*skip_layers'):
        KFACPreconditioner(_LM(), precondition_embeddings=True, diagonal_g_layers=['head'])
    with pytest.raises(ValueError, match='"emb" shares its weight with "head".*skip_layers'):
        KFACPreconditioner(_LM(), precondition_embeddings=True)
    tied = nn.Sequential(nn.Linear(8, 8), nn.Linear(8, 8))
    tied[1].weight = tied[0].weight
    with pytest.raises(ValueError, match='"1" shares its weight with "0".*skip_layers'):
        KFACPreconditioner(tied, diagonal_g_layers=['1'])


def test_refusals_with_the_keyword_on():
    from kfac_b200.preconditioner import KFACPreconditioner
    with pytest.raises(ValueError, match='"head", which is not in diagonal_g_layers.*add "head" to diagonal_g_layers'):
        KFACPreconditioner(_LM(), precondition_embeddings=True, precondition_tied_embeddings=True)
    with pytest.raises(ValueError, match='"head", which has a bias.*skip_layers'):
        KFACPreconditioner(_LM(bias=True), **KW)
    three = _LM()
    three.head2 = nn.Linear(64, 1000, bias=False)
    three.head2.weight = three.emb.weight
    with pytest.raises(ValueError, match='"emb" shares its weight with "head", "head2".*skip_layers'):
        KFACPreconditioner(three, precondition_embeddings=True, diagonal_g_layers=['head'],
                           precondition_tied_embeddings=True)
    two = nn.Sequential(nn.Linear(8, 8), nn.Linear(8, 8))
    two[1].weight = two[0].weight
    with pytest.raises(ValueError, match='"1" shares its weight with "0".*skip_layers'):
        KFACPreconditioner(two, diagonal_g_layers=['1'], precondition_embeddings=True, precondition_tied_embeddings=True)
    with pytest.raises(ValueError, match='EKFAC'):
        KFACPreconditioner(_LM(), compute_method='ekfac', **KW)
    # each refusal goes away once one of the members is skipped
    KFACPreconditioner(three, precondition_embeddings=True, diagonal_g_layers=['head'],
                       precondition_tied_embeddings=True, skip_layers=['head2'])
    KFACPreconditioner(_LM(bias=True), skip_layers=['head'], **KW)
    KFACPreconditioner(_LM(), compute_method='ekfac', skip_layers=['emb', 'head'], **KW)


def test_skip_layers_wins():
    from kfac_b200.preconditioner import KFACPreconditioner
    no_head = _names(KFACPreconditioner(_LM(), skip_layers=['head'], **KW))
    assert list(no_head) == ['emb', 'hidden'] and no_head['emb'].tied_head is None
    no_emb = _names(KFACPreconditioner(_LM(), skip_layers=['emb'], **KW))
    assert list(no_emb) == ['hidden', 'head'] and no_emb['head'].tied_embedding is None and no_emb['head'].diag_g


def test_pair_is_one_unit_of_the_placement():
    from kfac_b200.enums import AssignmentStrategy
    from kfac_b200.preconditioner import KFACPreconditioner, layer_work
    pre = KFACPreconditioner(_LM(V=50257, d=64), **KW)
    for strategy, cost in ((AssignmentStrategy.COMPUTE, lambda n: n ** 3), (AssignmentStrategy.MEMORY, lambda n: n ** 2)):
        work = layer_work(pre._layers, strategy)
        assert work == {'emb': {'G': 2 * cost(64) + 2 * 50257}, 'hidden': {'A': cost(65), 'G': cost(64)}}
    assert pre._assignment.get_factors('emb') == ('G',)
    assert 'head' not in pre._assignment.get_layers()


def _plans(world, frac, method, colocate):
    from kfac_b200.assignment import KAISAAssignment
    from kfac_b200.base_preconditioner import build_comm_plan
    from kfac_b200.enums import AssignmentStrategy
    from kfac_b200.layers import register_modules
    from kfac_b200.preconditioner import _check_diagonal_layers, layer_work

    class Net(nn.Module):
        def __init__(self):
            super().__init__()
            self.emb = nn.Embedding(1000, 48)
            self.body = nn.Sequential(nn.Linear(48, 64), nn.Linear(64, 48))
            self.other = nn.Embedding(30, 8)
            self.head = nn.Linear(48, 1000, bias=False)
            self.head.weight = self.emb.weight
            self.lm2 = nn.Linear(48, 300)

    model = Net()
    out = []
    handles = {}
    for rank in range(world):
        layers = register_modules(model, [], precondition_embeddings=True, diagonal_g_layers=['head', 'lm2'],
                                  method=method, prediv_eigenvalues=True)
        _check_diagonal_layers(layers, method, tied_embeddings=True)
        ll = list(layers.values())
        a = KAISAAssignment(layer_work(layers, AssignmentStrategy.COMPUTE), local_rank=rank, world_size=world,
                            grad_worker_fraction=frac,
                            group_func=lambda r: handles.setdefault(tuple(sorted(r)), tuple(sorted(r))),
                            colocate_factors=colocate)
        out.append((a, ll, build_comm_plan(ll, a)))
    return out


@pytest.mark.parametrize('world,frac', [(1, 1.0), (2, 1.0), (2, 0.5), (4, 1.0), (4, 0.5), (4, 0.25)])
@pytest.mark.parametrize('method', ['EIGEN', 'INVERSE'])
@pytest.mark.parametrize('colocate', [True, False])
def test_comm_plan_with_a_tied_pair_consistent_across_ranks(world, frac, method, colocate):
    """Every (group, src) broadcast looks the same on every member; the pair ships M, mu, f and h from the one rank
    that holds its four factors, the head has no entry of its own, and P is stored once in the weight's layout."""
    from kfac_b200.base_preconditioner import _storage_numel
    from kfac_b200.enums import ComputeMethod
    if colocate is False and frac * world <= 1:
        colocate = True
    plans = _plans(world, frac, ComputeMethod[method], colocate)
    for kind in (0, 1):
        per_rank = [[(s.group, s.src, s.numel, [(l.index, k, sh) for l, k, sh in s.entries]) for s in plan[kind]]
                    for _, _, plan in plans]
        for rank, segs in enumerate(per_rank):
            for grp, src, numel, entries in segs:
                assert rank in grp and src in grp
                for other in grp:
                    assert [s for s in per_rank[other] if s[0] == grp] == [s for s in segs if s[0] == grp]
    for a, ll, (inv, grad) in plans:
        names = dict(ll)
        emb, head = names['emb'], names['head']
        assert emb.tied_head is head
        src = a.inv_worker('emb', 'G')
        entries = [(s.src, k, sh) for s in inv for l, k, sh in s.entries if l is emb]
        if a.is_grad_worker('emb'):
            assert sorted(entries) == sorted([(src, 'tq', (48, 48)), (src, 'tmu', (48,)), (src, 'da', (1000,)),
                                              (src, 'dh', (1000,))])
            assert src in a.grad_worker_ranks('emb')
        else:
            assert entries == []
        assert not any(l is head for s in inv + grad for l, _, _ in s.entries)
        assert [sh for s in grad for l, k, sh in s.entries if l is emb] == [(1000, 48)]
        assert len([1 for s in grad for _ in s.entries]) == len(ll) - 1
        for s in inv + grad:
            assert s.offset % 4 == 0 and s.numel == sum(_storage_numel(sh) for _, _, sh in s.entries)
