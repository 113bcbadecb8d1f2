"""CPU tests of diagonal-A Linear and convolution layers (`diagonal_a_layers=[...]`): matching, every refusal, the comm,
local and inverse plans across ranks for COMM_OPT, HYBRID_OPT and MEM_OPT, the KAISA cost, the state_dict shape checks,
and that without the keyword the layouts and plans are those of today."""
import pytest
import torch
from torch import nn

from conftest import ROOT  # noqa: F401  (puts the repository on sys.path)


class _Net(nn.Module):
    """A LLaMA-shaped MLP (down_proj with 11008 inputs) next to a wide 3 x 3 convolution (A = 9217)."""

    def __init__(self):
        super().__init__()
        self.inp = nn.Linear(16, 64)
        self.down_proj = nn.Linear(11008, 64, bias=False)
        self.wide = nn.Conv2d(1024, 32, 3)
        self.head = nn.Linear(64, 10)


def _names(pre):
    return {n: l for n, l in pre._layers.values()}


def test_matching_by_name_and_class():
    from kfac_b200.preconditioner import KFACPreconditioner
    off = _names(KFACPreconditioner(_Net()))
    assert not any(l.diag_a for l in off.values())
    on = KFACPreconditioner(_Net(), diagonal_a_layers=['down_proj', 'wide'])
    names = _names(on)
    d = names['down_proj']
    assert d.diag_a and not d.embedding and d.diag_side == 'a' and d.dense_side == 'g'
    assert d.a_dim == 11008 and d.a_factor_shape == (11008,) and d.g_factor_shape == (64, 64)
    assert d.p_shape == (64, 11008)            # the dense layout, not an embedding's (a, g)
    w = names['wide']
    assert w.diag_a and w.a_dim == 1024 * 9 + 1 and w.p_shape == (32, 9217)
    assert not names['inp'].diag_a and not names['head'].diag_a
    assert "diagonal_a_layers=['down_proj', 'wide']" in repr(on)
    # a class pattern matches every Conv2d; a pattern that matches nothing is no error; skip_layers wins
    assert [n for n, l in _names(KFACPreconditioner(_Net(), diagonal_a_layers=['Conv2d'])).items()
            if l.diag_a] == ['wide']
    assert not any(l.diag_a for l in _names(KFACPreconditioner(nn.Linear(4, 4), diagonal_a_layers=['x'])).values())
    assert 'wide' not in _names(KFACPreconditioner(_Net(), diagonal_a_layers=['wide'], skip_layers=['wide']))
    # Conv1d / Conv3d with precondition_conv_nd, with A above the eigensolver's limit
    nd = nn.Sequential(nn.Conv1d(4096, 8, 3), nn.Conv3d(512, 8, 3))
    got = _names(KFACPreconditioner(nd, precondition_conv_nd=True, diagonal_a_layers=['0', '1']))
    assert got['0'].a_factor_shape == (4096 * 3 + 1,) and got['1'].a_factor_shape == (512 * 27 + 1,)
    # an embedding keeps its own notion
    emb = _names(KFACPreconditioner(nn.Sequential(nn.Embedding(100, 8), nn.Linear(8, 4)), precondition_embeddings=True))
    assert emb['0'].diag_a and emb['0'].embedding and emb['0'].p_shape == (100, 8)


def test_refusals():
    from kfac_b200.preconditioner import KFACPreconditioner
    with pytest.raises(ValueError, match='diagonal_a_layers.*EKFAC.*skip_layers'):
        KFACPreconditioner(_Net(), diagonal_a_layers=['down_proj'], compute_method='ekfac')
    emb = nn.Sequential(nn.Embedding(100, 8), nn.Linear(8, 4))
    with pytest.raises(ValueError, match='diagonal_a_layers matches "0" \\(Embedding\\).*skip_layers'):
        KFACPreconditioner(emb, precondition_embeddings=True, diagonal_a_layers=['0'])
    norm = nn.Sequential(nn.Linear(8, 8), nn.LayerNorm(8))
    with pytest.raises(ValueError, match='diagonal_a_layers matches "1" \\(LayerNorm\\).*skip_layers'):
        KFACPreconditioner(norm, precondition_norms=True, diagonal_a_layers=['1'])
    gn = nn.Sequential(nn.Conv2d(4, 8, 1), nn.GroupNorm(2, 8))
    with pytest.raises(ValueError, match='diagonal_a_layers matches "1" \\(GroupNorm\\)'):
        KFACPreconditioner(gn, precondition_group_norms=True, diagonal_a_layers=['1'])
    tr = nn.Sequential(nn.ConvTranspose2d(4, 8, 3))
    with pytest.raises(ValueError, match='diagonal_a_layers matches "0" \\(ConvTranspose2d\\).*skip_layers'):
        KFACPreconditioner(tr, precondition_conv_transpose=True, diagonal_a_layers=['0'])
    att = nn.Sequential(nn.MultiheadAttention(16, 2))
    with pytest.raises(ValueError, match='diagonal_a_layers matches the attention projection "0.q_proj"'):
        KFACPreconditioner(att, precondition_attention=True, diagonal_a_layers=['0'])
    rnn = nn.Sequential(nn.LSTM(8, 8))
    with pytest.raises(ValueError, match='diagonal_a_layers matches the recurrent sub-layer "0.ih_l0"'):
        KFACPreconditioner(rnn, precondition_recurrent=True, diagonal_a_layers=['0'])
    with pytest.raises(ValueError, match='diagonal_a_layers and diagonal_g_layers both match "head"'):
        KFACPreconditioner(_Net(), diagonal_a_layers=['head'], diagonal_g_layers=['head'])
    with pytest.raises(ValueError, match='"big".*G factor of 9000 exceeds.*skip_layers'):
        KFACPreconditioner(nn.ModuleDict({'big': nn.Linear(10000, 9000)}), diagonal_a_layers=['big'])
    with pytest.raises(ValueError, match='G factor of 9000 exceeds'):
        KFACPreconditioner(nn.Sequential(nn.Conv1d(4, 9000, 3)), precondition_conv_nd=True, diagonal_a_layers=['0'])
    with pytest.raises(ValueError, match='kernel of 2197 taps.*skip_layers'):
        KFACPreconditioner(nn.Sequential(nn.Conv3d(2, 4, 13)), precondition_conv_nd=True, diagonal_a_layers=['0'])
    shared = nn.Sequential(nn.Linear(8, 8), nn.Linear(8, 8))
    shared[1].weight = shared[0].weight
    with pytest.raises(ValueError, match='"1" shares its weight with "0".*skip_layers'):
        KFACPreconditioner(shared, diagonal_a_layers=['1'])
    # without the keyword, a dense N-d layer beyond the eigensolver is still refused at construction
    with pytest.raises(ValueError, match='beyond the eigensolver'):
        KFACPreconditioner(nn.Sequential(nn.Conv1d(4096, 8, 3)), precondition_conv_nd=True)
    # patterns matching modules that are not registered are no error
    KFACPreconditioner(emb, diagonal_a_layers=['0'])
    KFACPreconditioner(tr, diagonal_a_layers=['0'])


def test_state_dict_shape_check():
    from kfac_b200.preconditioner import KFACPreconditioner
    pre = KFACPreconditioner(nn.Sequential(nn.Linear(9, 4), nn.Linear(4, 3)), diagonal_a_layers=['0'])
    names = _names(pre)
    d, dense = names['0'], names['1']
    d._a_view, d._g_view = torch.zeros(10), torch.zeros(4, 4)        # stand-ins for the arena views (no device)
    dense._a_view, dense._g_view = torch.zeros(5, 5), torch.zeros(3, 3)
    d.load_state_dict({'A': torch.ones(10), 'G': torch.eye(4)})
    assert torch.equal(d.a_factor, torch.ones(10)) and d.qa is None and d.a_inv is None
    with pytest.raises(ValueError, match=r'diagonal-A layer factor A has shape \(10, 10\), expected \(10,\)'):
        d.load_state_dict({'A': torch.eye(10), 'G': torch.eye(4)})
    with pytest.raises(ValueError, match=r'factor A has shape \(5,\), expected \(5, 5\)'):
        dense.load_state_dict({'A': torch.ones(5), 'G': None})
    assert d.memory_usage()['a_factors'] == 10 * 4 and d.memory_usage()['g_factors'] == 16 * 4


def test_kaisa_cost_of_a_diagonal_a_is_linear():
    from kfac_b200.enums import AssignmentStrategy
    from kfac_b200.layers import register_modules
    from kfac_b200.preconditioner import layer_work
    layers = register_modules(_Net(), [], diagonal_a_layers=['down_proj', 'wide'], method=None)
    for strategy, cost in ((AssignmentStrategy.COMPUTE, lambda n: n ** 3), (AssignmentStrategy.MEMORY, lambda n: n ** 2)):
        work = layer_work(layers, strategy)
        assert work['down_proj'] == {'A': 11008, 'G': cost(64)}
        assert work['wide'] == {'A': 9217, 'G': cost(32)}
        assert work['inp'] == {'A': cost(17), 'G': cost(64)}


def _plans(world, frac, method, prediv, colocate, diagonal_a_layers):
    from kfac_b200.assignment import KAISAAssignment
    from kfac_b200.base_preconditioner import build_comm_plan, build_inverse_plan, build_local_plan
    from kfac_b200.enums import AssignmentStrategy
    from kfac_b200.layers import register_modules
    from kfac_b200.preconditioner import layer_work
    model = nn.Sequential(nn.Embedding(1000, 48), nn.Linear(48, 64), nn.Linear(11008, 64), nn.Conv2d(1024, 8, 3),
                          nn.Linear(64, 10007, bias=False), nn.Conv2d(3, 8, 3), nn.Linear(64, 10))
    out = []
    handles = {}
    for rank in range(world):
        layers = register_modules(model, [], precondition_embeddings=True, diagonal_g_layers=['^4$'],
                                  diagonal_a_layers=diagonal_a_layers, method=method, prediv_eigenvalues=prediv)
        ll = list(layers.values())
        for _, l in ll:                 # every factor computed: the inverse plan reads them
            l._has_a = l._has_g = True
        a = KAISAAssignment(layer_work(layers, AssignmentStrategy.COMPUTE), local_rank=rank, world_size=world,
                            grad_worker_fraction=frac,
                            group_func=lambda r: handles.setdefault(tuple(sorted(r)), tuple(sorted(r))),
                            colocate_factors=colocate)
        out.append((a, ll, build_comm_plan(ll, a), build_local_plan(ll, a, rank), build_inverse_plan(ll, a, rank)))
    return out


@pytest.mark.parametrize('world,frac', [(1, 1.0), (2, 1.0), (2, 0.5), (4, 1.0), (4, 0.5), (4, 0.25), (6, 0.5),
                                        (8, 1.0), (8, 0.5), (8, 0.125)])
@pytest.mark.parametrize('method,prediv,colocate', [('EIGEN', True, True), ('EIGEN', False, False),
                                                    ('INVERSE', False, True)])
def test_plans_with_diag_a_consistent_across_ranks(world, frac, method, prediv, colocate):
    """COMM_OPT, HYBRID_OPT and MEM_OPT for world sizes 1-8: every (group, src) broadcast looks the same on every
    member; a diagonal-A layer ships da plus qg, dg (eigen) or g_inv (inverse) and never a dgda, keeps a K-major Qg
    locally on its gradient workers (eigen), decomposes only G in the second eigensolver call and snapshots its A,
    and its P keeps the dense (g, a) layout."""
    from kfac_b200.base_preconditioner import _storage_numel
    from kfac_b200.enums import ComputeMethod
    if colocate is False and frac * world <= 1:
        colocate = True
    plans = _plans(world, frac, ComputeMethod[method], prediv, colocate, ['^2$', '^3$'])
    for kind in (0, 1):
        per_rank = [[(s.group, s.src, s.numel, [(l.index, k, sh) for l, k, sh in s.entries]) for s in plan[kind]]
                    for _, _, plan, _, _ in plans]
        for rank, segs in enumerate(per_rank):
            for grp, src, numel, entries in segs:
                assert rank in grp and src in grp
                for other in grp:
                    assert [s for s in per_rank[other] if s[0] == grp] == [s for s in segs if s[0] == grp]
    n_diag = 0
    for rank, (a, ll, (inv, grad), local, (snaps, calls, post)) in enumerate(plans):
        assert sorted(l.index for s in grad for l, _, _ in s.entries) == list(range(len(ll)))
        for s in inv + grad:
            assert s.offset % 4 == 0 and s.numel == sum(_storage_numel(sh) for _, _, sh in s.entries)
        for name, l in ll:
            if not l.diag_a or l.embedding:
                continue
            n_diag += 1
            keys = {k: sh for s in inv for ll_, k, sh in s.entries if ll_ is l}
            mine = {k: sh for ll_, k, sh in local if ll_ is l}
            if a.is_grad_worker(name):
                want = ({'da': (l.a_dim,), 'qg': (l.g_dim, l.g_dim), 'dg': (l.g_dim,)} if method == 'EIGEN'
                        else {'da': (l.a_dim,), 'g_inv': (l.g_dim, l.g_dim)})
                assert keys == want
                if method == 'EIGEN':
                    assert mine['_qgT'] == (l.g_dim, l.g_dim)
            else:
                assert keys == {}
            assert [sh for s in grad for ll_, k, sh in s.entries if ll_ is l] == [(l.g_dim, l.a_dim)]
            holder = rank == a.inv_worker(name, 'A')
            assert [k for ll_, src, side, k in snaps if ll_ is l] == (['da'] if holder else [])
            assert not any(ll_ is l for ll_, *_ in calls[0])
            g_mine = rank == a.inv_worker(name, 'G')
            assert [side for ll_, side, *_ in calls[1] if ll_ is l] == (['g'] if g_mine else [])
            assert all(op == 'inverse' for ll_, op, _ in post if ll_ is l)
    assert n_diag == 2 * world


@pytest.mark.parametrize('world,frac', [(1, 1.0), (4, 0.5), (8, 0.125)])
@pytest.mark.parametrize('method,prediv', [('EIGEN', True), ('EIGEN', False), ('INVERSE', False)])
def test_unset_keyword_changes_nothing(world, frac, method, prediv):
    """Without diagonal_a_layers (None, or a pattern that matches nothing) the layouts and the comm, local and inverse
    plans are those of a registration that never heard of the keyword."""
    from kfac_b200.base_preconditioner import second_order_layout
    from kfac_b200.enums import ComputeMethod

    def view(plans):
        out = []
        for a, ll, (inv, grad), local, (snaps, calls, post) in plans:
            out.append(([(s.src, s.numel, [(l.index, k, sh) for l, k, sh in s.entries]) for s in inv + grad],
                        [(l.index, k, sh) for l, k, sh in local],
                        [(l.index, src.index, side, k) for l, src, side, k in snaps],
                        [[(l.index, side, q, qT, d) for l, side, q, qT, d in c] for c in calls],
                        [(l.index, op, keys) for l, op, keys in post],
                        [second_order_layout(l)._replace(factors=None, snapshots=None) for _, l in ll
                         if l.tied_embedding is None]))
        return out
    m = ComputeMethod[method]
    base = view(_plans(world, frac, m, prediv, True, None))
    assert view(_plans(world, frac, m, prediv, True, ['nothing'])) == base
    assert view(_plans(world, frac, m, prediv, True, [])) == base
