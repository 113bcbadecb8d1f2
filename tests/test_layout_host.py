"""CPU tests of the declaration of each layer kind's second-order data (`second_order_layout`) and of what follows from
it: every key a rank's inverse step and precondition read is allocated on that rank exactly once, and the
eigensolver calls list their matrices in the order the batched solver's schedule depends on."""
import pytest
import torch
from torch import nn

from conftest import ROOT  # noqa: F401  (puts the repository on sys.path)

WORLDS = [(1, 1.0), (2, 1.0), (2, 0.5), (3, 1.0), (4, 1.0), (4, 0.5), (4, 0.25), (5, 0.2), (6, 0.5), (7, 1.0),
          (8, 1.0), (8, 0.5), (8, 0.125)]


class _Net(nn.Module):
    """Dense Linear and Conv2d layers, an embedding, a diagonal-G head and a tied embedding / head pair."""

    def __init__(self):
        super().__init__()
        self.emb = nn.Embedding(10, 4)
        self.emb2 = nn.Embedding(30, 8)
        self.lin = nn.Linear(4, 6)
        self.conv = nn.Conv2d(3, 8, 3)
        self.lm = nn.Linear(6, 12)
        self.down = nn.Linear(6, 4)
        self.head = nn.Linear(4, 10, bias=False)
        self.head.weight = self.emb.weight


def _layers(method, prediv=True, model=None):
    from kfac_b200.enums import ComputeMethod
    from kfac_b200.layers import register_modules
    from kfac_b200.preconditioner import _check_diagonal_layers
    method = ComputeMethod[method]
    if model is None:
        model = _Net() if method != ComputeMethod.EKFAC else nn.Sequential(nn.Linear(4, 6), nn.Conv2d(3, 8, 3))
    kw = (dict(precondition_embeddings=True, diagonal_g_layers=['lm', 'head'])
          if method != ComputeMethod.EKFAC else {})
    layers = register_modules(model, [], method=method, prediv_eigenvalues=prediv, **kw)
    _check_diagonal_layers(layers, method, tied_embeddings=True)
    return layers


def _named(method, prediv=True):
    return dict(_layers(method, prediv).values())


def _view(lay, names):
    """The layout with layers replaced by their names."""
    return dict(
        entries=[tuple(e) for e in lay.entries],
        factors=[(h, [(names[id(l)], s) for l, s in fs], err) for h, fs, err in lay.factors],
        snapshots=[(h, names[id(l)], s, k) for h, l, s, k in lay.snapshots],
        decompositions=list(lay.decompositions), post=list(lay.post), needs=set(lay.needs), unready=lay.unready,
        fields=dict(lay.fields), item=lay.item, eigen=lay.eigen, damped=lay.damped)


def _dense_factors(name):
    return [('A', [(name, 'a')], 'Cannot eigendecompose A before A has been computed'),
            ('G', [(name, 'g')], 'Cannot eigendecompose G before G has been computed')]


EIG_UNREADY = 'Eigendecompositions for both A and G have not been computed'
# lin: a = 5 (weight and bias), g = 6; emb2: a = V = 30, g = 8; lm: a = 7, g = V = 12; emb: V = 10, d = 4
EXPECTED = {
    ('EIGEN', True, 'lin'): dict(
        entries=[('qa', (5, 5), 'G', True, '_qaT'), ('qg', (6, 6), 'G', True, '_qgT'), ('dgda', (6, 5), 'G', True, None),
                 ('_qaT', (5, 5), 'grad', False, None), ('_qgT', (6, 6), 'grad', False, None),
                 ('_da', (5,), 'A', False, None), ('_dg', (6,), 'G', False, None)],
        factors=_dense_factors('lin'), snapshots=[],
        decompositions=[('a', 0, 'qa', '_qaT', '_da'), ('g', 0, 'qg', '_qgT', '_dg')],
        post=[('G', 'dgda', ('_dg', '_da', 'dgda'))], needs={'qa', 'qg', 'dgda'}, unready=EIG_UNREADY,
        fields={'qa': 'qa', 'qg': 'qg', 'dgda': 'dgda', 'qaT': '_qaT', 'qgT': '_qgT'},
        item=dict(kind=0, ldqa=8, ldqg=8, ld_dgda=8), eigen=True, damped=False),
    ('EIGEN', False, 'lin'): dict(
        entries=[('qa', (5, 5), 'A', True, '_qaT'), ('da', (5,), 'A', True, None), ('qg', (6, 6), 'G', True, '_qgT'),
                 ('dg', (6,), 'G', True, None), ('_qaT', (5, 5), 'grad', False, None),
                 ('_qgT', (6, 6), 'grad', False, None)],
        factors=_dense_factors('lin'), snapshots=[],
        decompositions=[('a', 0, 'qa', '_qaT', 'da'), ('g', 0, 'qg', '_qgT', 'dg')],
        post=[], needs={'qa', 'qg', 'da', 'dg'}, unready=EIG_UNREADY,
        fields={'qa': 'qa', 'da': 'da', 'qg': 'qg', 'dg': 'dg', 'qaT': '_qaT', 'qgT': '_qgT'},
        item=dict(kind=0, ldqa=8, ldqg=8, ld_dgda=8), eigen=True, damped=False),
    ('EKFAC', True, '0'): dict(
        entries=[('qa', (5, 5), 'A', True, '_qaT'), ('da', (5,), 'A', True, None), ('qg', (6, 6), 'G', True, '_qgT'),
                 ('dg', (6,), 'G', True, None), ('_qaT', (5, 5), 'all', False, None),
                 ('_qgT', (6, 6), 'all', False, None), ('dgda', (6, 5), 'all', False, None)],
        factors=_dense_factors('0'), snapshots=[],
        decompositions=[('a', 0, 'qa', '_qaT', 'da'), ('g', 0, 'qg', '_qgT', 'dg')],
        post=[], needs={'qa', 'qg', 'dgda'}, unready=EIG_UNREADY,
        fields={'qa': 'qa', 'da': 'da', 'qg': 'qg', 'dg': 'dg', 'qaT': '_qaT', 'qgT': '_qgT', 'dgda': 'dgda'},
        item=dict(kind=0, ldqa=8, ldqg=8, ld_dgda=8), eigen=True, damped=False),
    ('INVERSE', True, 'lin'): dict(
        entries=[('a_inv', (5, 5), 'A', True, None), ('g_inv', (6, 6), 'G', True, None),
                 ('_qa', (5, 5), 'A', False, None), ('_da', (5,), 'A', False, None),
                 ('_qg', (6, 6), 'G', False, None), ('_dg', (6,), 'G', False, None)],
        factors=_dense_factors('lin'), snapshots=[],
        decompositions=[('a', 0, '_qa', None, '_da'), ('g', 0, '_qg', None, '_dg')],
        post=[('A', 'inverse', ('_qa', '_da', 'a_inv')), ('G', 'inverse', ('_qg', '_dg', 'g_inv'))],
        needs={'a_inv', 'g_inv'}, unready='Cannot precondition gradient before A and G have been inverted',
        fields={'a_inv': 'a_inv', 'g_inv': 'g_inv'}, item=dict(kind=0, ldqa=8, ldqg=8, ld_dgda=8), eigen=False,
        damped=False),
    ('EIGEN', True, 'emb2'): dict(
        entries=[('da', (30,), 'A', True, None), ('qg', (8, 8), 'G', True, '_qgT'), ('dg', (8,), 'G', True, None),
                 ('_qgT', (8, 8), 'grad', False, None)],
        factors=_dense_factors('emb2'), snapshots=[('A', 'emb2', 'a', 'da')],
        decompositions=[('g', 1, 'qg', '_qgT', 'dg')], post=[], needs={'da', 'qg', 'dg'},
        unready='The second-order data of the embedding has not been computed',
        fields={'da': 'da', 'qg': 'qg', 'dg': 'dg', 'qgT': '_qgT'}, item=dict(kind=1, ldqa=0, ldqg=8, ld_dgda=0),
        eigen=True, damped=False),
    ('INVERSE', True, 'emb2'): dict(
        entries=[('da', (30,), 'A', True, None), ('g_inv', (8, 8), 'G', True, None),
                 ('_qg', (8, 8), 'G', False, None), ('_dg', (8,), 'G', False, None)],
        factors=_dense_factors('emb2'), snapshots=[('A', 'emb2', 'a', 'da')],
        decompositions=[('g', 1, '_qg', None, '_dg')], post=[('G', 'inverse', ('_qg', '_dg', 'g_inv'))],
        needs={'da', 'g_inv'}, unready='The second-order data of the embedding has not been computed',
        fields={'da': 'da', 'g_inv': 'g_inv'}, item=dict(kind=1, ldqa=0, ldqg=8, ld_dgda=0), eigen=False,
        damped=False),
    ('EIGEN', True, 'lm'): dict(
        entries=[('dg', (12,), 'G', True, None), ('qa', (7, 7), 'A', True, '_qaT'), ('da', (7,), 'A', True, None),
                 ('_qaT', (7, 7), 'grad', False, None)],
        factors=_dense_factors('lm'), snapshots=[('G', 'lm', 'g', 'dg')],
        decompositions=[('a', 1, 'qa', '_qaT', 'da')], post=[], needs={'dg', 'qa', 'da'},
        unready='The second-order data of the diagonal-G layer has not been computed',
        fields={'dg': 'dg', 'qa': 'qa', 'da': 'da', 'qaT': '_qaT'}, item=dict(kind=2, ldqa=8, ldqg=0, ld_dgda=0),
        eigen=True, damped=False),
    ('INVERSE', True, 'lm'): dict(
        entries=[('dg', (12,), 'G', True, None), ('a_inv', (7, 7), 'A', True, None),
                 ('_qa', (7, 7), 'A', False, None), ('_da', (7,), 'A', False, None)],
        factors=_dense_factors('lm'), snapshots=[('G', 'lm', 'g', 'dg')],
        decompositions=[('a', 1, '_qa', None, '_da')], post=[('A', 'inverse', ('_qa', '_da', 'a_inv'))],
        needs={'dg', 'a_inv'}, unready='The second-order data of the diagonal-G layer has not been computed',
        fields={'dg': 'dg', 'a_inv': 'a_inv'}, item=dict(kind=2, ldqa=8, ldqg=0, ld_dgda=0), eigen=False,
        damped=False),
}
TIED = dict(
    entries=[('tq', (4, 4), 'G', True, '_tqT'), ('tmu', (4,), 'G', True, None), ('da', (10,), 'G', True, None),
             ('dh', (10,), 'G', True, None), ('_tqT', (4, 4), 'grad', False, None), ('_qg', (4, 4), 'G', False, None),
             ('_qgT', (4, 4), 'G', False, None), ('_dg', (4,), 'G', False, None), ('_C', (16,), 'G', False, None),
             ('_U', (4, 4), 'G', False, None), ('_UT', (4, 4), 'G', False, None)],
    factors=[('G', [('emb', 'a'), ('emb', 'g'), ('head', 'a'), ('head', 'g')],
              'Cannot decompose the factors of a tied embedding / head pair before they have been computed')],
    snapshots=[('G', 'emb', 'a', 'da'), ('G', 'head', 'g', 'dh')],
    decompositions=[('g', 1, '_qg', '_qgT', '_dg')],
    post=[('G', 'tied', ('_qg', '_qgT', '_dg', '_C', '_U', '_UT', 'tq', '_tqT', 'tmu'))],
    needs={'tq', '_tqT', 'tmu', 'da', 'dh'},
    unready='The second-order data of the tied embedding / head pair has not been computed',
    fields={'qg': 'tq', 'qgT': '_tqT', 'dg': 'tmu', 'da': 'da', 'dh': 'dh'},
    item=dict(kind=3, ldqa=0, ldqg=4, ld_dgda=0), eigen=False, damped=True)
EXPECTED.update({('EIGEN', True, 'emb'): TIED, ('INVERSE', True, 'emb'): TIED})


@pytest.mark.parametrize('method,prediv,name', list(EXPECTED))
def test_declared_layout(method, prediv, name):
    from kfac_b200.base_preconditioner import second_order_layout
    layers = _named(method, prediv)
    names = {id(l): n for n, l in layers.items()}
    assert _view(second_order_layout(layers[name]), names) == EXPECTED[(method, prediv, name)]


def _plans(method, prediv, colocate, world, frac):
    from kfac_b200.assignment import KAISAAssignment
    from kfac_b200.base_preconditioner import build_comm_plan, build_inverse_plan, build_local_plan
    from kfac_b200.enums import AssignmentStrategy
    from kfac_b200.preconditioner import layer_work
    handles = {}
    for rank in range(world):
        layers = _layers(method, prediv)
        ll = list(layers.values())
        for _, l in ll:
            l._has_a = l._has_g = True
        a = KAISAAssignment(layer_work(layers, AssignmentStrategy.COMPUTE), local_rank=rank, world_size=world,
                            grad_worker_fraction=frac,
                            group_func=lambda r: handles.setdefault(tuple(sorted(r)), tuple(sorted(r))),
                            colocate_factors=colocate)
        yield (rank, a, ll, build_comm_plan(ll, a)[0], build_local_plan(ll, a, rank),
               build_inverse_plan(ll, a, rank))


@pytest.mark.parametrize('method,prediv,colocate', [('EIGEN', True, True), ('EIGEN', False, False),
                                                    ('INVERSE', False, True), ('INVERSE', False, False),
                                                    ('EKFAC', False, True)])
def test_every_key_read_is_allocated_on_its_rank(method, prediv, colocate):
    """On every rank of every placement: each key its inverse step (snapshots, eigensolver calls, post-ops, the K-major
    copy of what it receives) and its precondition read is allocated there, as a shipped entry of one of its segments
    or as a local entry, and no key is allocated twice."""
    from kfac_b200.base_preconditioner import second_order_layout
    n_ranks = 0
    for world, frac in WORLDS:
        for rank, a, ll, inv, local, (snapshots, calls, post) in _plans(
                method, prediv, colocate or frac * world <= 1, world, frac):
            held = [(id(l), k) for s in inv for l, k, _ in s.entries] + [(id(l), k) for l, k, _ in local]
            assert len(held) == len(set(held)), (world, frac, rank)
            held = set(held)
            reads = [(l, k) for l, _, _, k in snapshots]
            reads += [(l, k) for call in calls for l, _, q, qT, d in call for k in (q, qT, d) if k]
            reads += [(l, k) for l, _, keys in post for k in keys]
            for name, l in ll:
                if l.tied_embedding is None and a.is_grad_worker(name):
                    lay = second_order_layout(l)
                    reads += [(l, k) for k in lay.needs] + [(l, k) for _, k in lay.fields]
            for s in inv:
                if s.src != rank:
                    for l, key, _ in s.entries:
                        kmajor = next(e.kmajor for e in second_order_layout(l).entries if e.key == key)
                        reads += [(l, kmajor)] if kmajor else []
            names = {id(l): n for n, l in ll}
            missing = {(names[id(l)], k) for l, k in reads if (id(l), k) not in held}
            assert not missing, (world, frac, rank, missing)
            n_ranks += 1
    assert n_ranks == sum(w for w, _ in WORLDS)


def test_eigensolver_calls_and_snapshots_in_order():
    """Reverse registration order, A before G within a layer; the dense factors of diagonal layers and the tied pair
    in a call of their own."""
    from kfac_b200.assignment import KAISAAssignment
    from kfac_b200.base_preconditioner import build_inverse_plan
    from kfac_b200.enums import AssignmentStrategy
    from kfac_b200.preconditioner import layer_work
    for method, prediv in (('EIGEN', True), ('EIGEN', False), ('INVERSE', False)):
        layers = _layers(method, prediv)
        ll = list(layers.values())
        assert [n for n, _ in ll] == ['emb', 'emb2', 'lin', 'conv', 'lm', 'down', 'head']
        for _, l in ll:
            l._has_a = l._has_g = True
        a = KAISAAssignment(layer_work(layers, AssignmentStrategy.COMPUTE), local_rank=0, world_size=1,
                            grad_worker_fraction=1.0, group_func=lambda r: None, colocate_factors=True)
        snapshots, calls, post = build_inverse_plan(ll, a, 0)
        names = {id(l): n for n, l in ll}
        assert [(names[id(l)], side) for l, side, *_ in calls[0]] == [
            ('down', 'a'), ('down', 'g'), ('conv', 'a'), ('conv', 'g'), ('lin', 'a'), ('lin', 'g')]
        assert [(names[id(l)], side) for l, side, *_ in calls[1]] == [('lm', 'a'), ('emb2', 'g'), ('emb', 'g')]
        assert [(names[id(l)], names[id(src)], key) for l, src, _, key in snapshots] == [
            ('lm', 'lm', 'dg'), ('emb2', 'emb2', 'da'), ('emb', 'emb', 'da'), ('emb', 'head', 'dh')]
        want = {'EIGEN': [('down', 'dgda'), ('conv', 'dgda'), ('lin', 'dgda')] if prediv else [],
                'INVERSE': [('down', 'inverse'), ('down', 'inverse'), ('lm', 'inverse'), ('conv', 'inverse'),
                            ('conv', 'inverse'), ('lin', 'inverse'), ('lin', 'inverse'), ('emb2', 'inverse')]}[method]
        assert [(names[id(l)], op) for l, op, _ in post] == want + [('emb', 'tied')]


def test_inverse_plan_refuses_uncomputed_factors():
    from kfac_b200.assignment import KAISAAssignment
    from kfac_b200.base_preconditioner import build_inverse_plan
    from kfac_b200.enums import AssignmentStrategy
    from kfac_b200.preconditioner import layer_work
    layers = _layers('EIGEN')
    ll = list(layers.values())
    a = KAISAAssignment(layer_work(layers, AssignmentStrategy.COMPUTE), local_rank=0, world_size=1,
                        grad_worker_fraction=1.0, group_func=lambda r: None, colocate_factors=True)
    named = dict(ll)
    for _, l in ll:
        l._has_a = l._has_g = True
    named['head']._has_g = False
    with pytest.raises(RuntimeError, match='tied embedding / head pair before'):
        build_inverse_plan(ll, a, 0)
    named['head']._has_g = True
    named['lin']._has_g = False
    with pytest.raises(RuntimeError, match='Cannot eigendecompose G before G'):
        build_inverse_plan(ll, a, 0)
    named['lin']._has_g = True
    assert build_inverse_plan(ll, a, 0)[1][0]
