"""CPU tests of diagonal-G Linear layers (`diagonal_g_layers=[...]`): registration, constructor validation,
comm-plan consistency across ranks with a diagonal-G layer present, and the linear G cost in the KAISA placement."""
import pytest
import torch
from torch import nn

from conftest import ROOT  # noqa: F401  (puts the repository on sys.path)


class _LM(nn.Module):
    def __init__(self, V=1000, d=64, tie=False):
        super().__init__()
        self.emb = nn.Embedding(V, d)
        self.hidden = nn.Linear(d, d)
        self.head = nn.Linear(d, V)
        if tie:
            self.head.weight = self.emb.weight

    def forward(self, idx):
        return self.head(torch.tanh(self.hidden(self.emb(idx))))


def test_registration_and_repr():
    from kfac_b200.preconditioner import KFACPreconditioner
    off = KFACPreconditioner(_LM())
    assert not any(l.diag_g for _, l in off._layers.values())
    assert 'diagonal_g_layers=None' in repr(off)
    on = KFACPreconditioner(_LM(), diagonal_g_layers=['head'])
    names = {n: l for n, l in on._layers.values()}
    head = names['head']
    assert head.diag_g and not head.diag_a and head.diag_side == 'g' and head.dense_side == 'a'
    assert head.g_dim == 1000 and head.a_dim == 65 and head.p_shape == (1000, 65)
    assert not names['hidden'].diag_g and names['hidden'].diag_side is None
    assert "diagonal_g_layers=['head']" in repr(on)
    # a class-name pattern matches every Linear; a pattern that matches nothing is not an error
    assert all(l.diag_g for _, l in KFACPreconditioner(_LM(), diagonal_g_layers=['Linear'])._layers.values())
    assert not any(l.diag_g for _, l in KFACPreconditioner(_LM(), diagonal_g_layers=['nothing'])._layers.values())
    # skip_layers wins
    skipped = KFACPreconditioner(_LM(), diagonal_g_layers=['head'], skip_layers=['head'])
    assert 'head' not in {n for n, _ in skipped._layers.values()}
    # with precondition_embeddings: the embedding keeps a diagonal A, the head a diagonal G
    both = {n: l for n, l in KFACPreconditioner(_LM(), precondition_embeddings=True,
                                                diagonal_g_layers=['head'])._layers.values()}
    assert both['emb'].diag_side == 'a' and both['head'].diag_side == 'g'


def test_constructor_rejects_unsupported_layers():
    from kfac_b200.preconditioner import KFACPreconditioner
    conv = nn.Sequential(nn.Conv2d(3, 8, 3), nn.Flatten(), nn.Linear(8, 2))
    with pytest.raises(ValueError, match='"0".*Conv2d.*Linear'):
        KFACPreconditioner(conv, diagonal_g_layers=['0'])
    with pytest.raises(ValueError, match='"emb".*Embedding'):
        KFACPreconditioner(_LM(), precondition_embeddings=True, diagonal_g_layers=['emb'])
    with pytest.raises(ValueError, match='diagonal_g_layers.*EKFAC'):
        KFACPreconditioner(_LM(), diagonal_g_layers=['head'], compute_method='ekfac')
    tied = nn.Sequential(nn.Linear(8, 8), nn.Linear(8, 8))
    tied[1].weight = tied[0].weight
    with pytest.raises(ValueError, match='"1" shares its weight with "0".*skip_layers'):
        KFACPreconditioner(tied, diagonal_g_layers=['1'])
    # an unregistered Embedding that matches is no error (nothing is registered for it)
    KFACPreconditioner(_LM(), diagonal_g_layers=['emb'])
    KFACPreconditioner(conv, diagonal_g_layers=['0'], skip_layers=['0'])
    KFACPreconditioner(tied, diagonal_g_layers=['1'], skip_layers=['0'])


def test_state_dict_shape_check():
    from kfac_b200.preconditioner import KFACPreconditioner
    pre = KFACPreconditioner(_LM(V=10, d=4), diagonal_g_layers=['head'])
    head = next(l for _, l in pre._layers.values() if l.diag_g)
    head._a_view = torch.zeros(5, 5)       # stand-ins for the arena views (no device here)
    head._g_view = torch.zeros(10)
    head.load_state_dict({'A': torch.eye(5), 'G': torch.ones(10)})
    assert torch.equal(head.g_factor, torch.ones(10)) and head.qg is None and head.g_inv is None
    with pytest.raises(ValueError, match='shape'):
        head.load_state_dict({'A': torch.eye(5), 'G': torch.eye(10)})
    with pytest.raises(ValueError, match='shape'):
        head.load_state_dict({'A': torch.ones(5), 'G': torch.ones(10)})
    assert head.memory_usage()['g_factors'] == 10 * 4


def test_kaisa_cost_of_a_diagonal_g_is_linear():
    from kfac_b200.enums import AssignmentStrategy
    from kfac_b200.layers import register_modules
    from kfac_b200.preconditioner import layer_work
    layers = register_modules(_LM(V=50257, d=64), [], diagonal_g_layers=['head'], method=None)
    for strategy, cost in ((AssignmentStrategy.COMPUTE, lambda n: n ** 3), (AssignmentStrategy.MEMORY, lambda n: n ** 2)):
        work = layer_work(layers, strategy)
        assert work['head'] == {'A': cost(65), 'G': 50257}
        assert work['hidden'] == {'A': cost(65), 'G': cost(64)}


def _plans(world, frac, method, prediv, colocate):
    from kfac_b200.assignment import KAISAAssignment
    from kfac_b200.base_preconditioner import build_comm_plan
    from kfac_b200.enums import AssignmentStrategy
    from kfac_b200.layers import register_modules
    from kfac_b200.preconditioner import layer_work
    model = nn.Sequential(nn.Embedding(1000, 48), nn.Linear(48, 64), nn.Linear(64, 9000), nn.Conv2d(3, 8, 3),
                          nn.Linear(64, 10007, bias=False), nn.Linear(64, 10))
    out = []
    handles = {}
    for rank in range(world):
        layers = register_modules(model, [], precondition_embeddings=True, diagonal_g_layers=['^2$', '^4$'],
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
def test_comm_plan_with_diag_g_consistent_across_ranks(world, frac, method, prediv, colocate):
    """COMM_OPT, HYBRID_OPT and MEM_OPT for world sizes 1-8: every (group, src) broadcast looks the same on every
    member; a diagonal-G layer ships dg plus qa, da (eigen) or a_inv (inverse) and never a dgda, and its P keeps the
    dense layout."""
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
    n_diag = 0
    for a, ll, (inv, grad) in plans:
        assert sorted(l.index for s in grad for l, _, _ in s.entries) == list(range(len(ll)))
        for s in inv + grad:
            assert s.offset % 4 == 0 and s.numel == sum(_storage_numel(sh) for _, _, sh in s.entries)
        for name, l in ll:
            if not l.diag_g:
                continue
            n_diag += 1
            keys = {k: sh for s in inv for ll_, k, sh in s.entries if ll_ is l}
            if a.is_grad_worker(name):
                want = ({'dg': (l.g_dim,), 'qa': (l.a_dim, l.a_dim), 'da': (l.a_dim,)} if method == 'EIGEN'
                        else {'dg': (l.g_dim,), 'a_inv': (l.a_dim, l.a_dim)})
                assert keys == want
            else:
                assert keys == {}
            assert [sh for s in grad for ll_, k, sh in s.entries if ll_ is l] == [(l.g_dim, l.a_dim)]
    assert n_diag == 2 * world
