"""CPU tests of pi-adjusted damping (`pi_damping=True`): validation and refusals, `repr` and `defaults`, unchanged
state_dict entries, every layer kind's layout (a `pi` field with the keyword, none without), the comm plan unchanged
for world sizes 1-8 under every strategy, and an fp64 restatement of pi and of every kind's damped operator, which
tests/test_gpu_pi_damping.py imports."""
import math

import numpy as np
import pytest
import torch
from torch import nn

from conftest import ROOT  # noqa: F401  (puts the repository on sys.path)


# ------------------------------------------------------------------------------------------- fp64 restatement
def f32(x: float) -> float:
    return float(np.float32(x))


def trace64(F: torch.Tensor) -> float:
    """The trace of a dense factor, or the sum of a diagonal factor's vector, in fp64."""
    F = F.double()
    return float(F.sum() if F.dim() == 1 else F.diagonal().sum())


def pi_ref(A: torch.Tensor, G: torch.Tensor) -> float:
    """pi = sqrt((tr A / a) / (tr G / g)) rounded once to fp32; 1 where a mean (or pi) is not a positive finite number."""
    ma, mg = trace64(A) / A.shape[0], trace64(G) / G.shape[0]
    if not (0 < ma < math.inf and 0 < mg < math.inf):
        return 1.0
    p = f32(math.sqrt(ma / mg))
    return p if 0 < p < math.inf else 1.0


def gammas(pi: float, damping: float) -> tuple[float, float]:
    """(gamma_A, gamma_G) in fp32: s = sqrt(damping), gamma_A = s pi, gamma_G = s / pi."""
    s = f32(math.sqrt(f32(damping)))
    return f32(s * pi), f32(s / pi)


def damped_inverse64(F: torch.Tensor, gamma: float) -> torch.Tensor:
    """(F + gamma I)^-1 in fp64; a diagonal factor (a vector) gives the vector 1 / (F + gamma)."""
    F = F.double()
    if F.dim() == 1:
        return 1.0 / (F + gamma)
    return torch.linalg.inv(F + gamma * torch.eye(F.shape[0], dtype=torch.float64, device=F.device))


def apply_left(M: torch.Tensor, X: torch.Tensor) -> torch.Tensor:
    return M[:, None] * X if M.dim() == 1 else M @ X


def apply_right(X: torch.Tensor, M: torch.Tensor) -> torch.Tensor:
    return X * M[None, :] if M.dim() == 1 else X @ M


def precondition_ref(grad: torch.Tensor, A: torch.Tensor, G: torch.Tensor, pi: float, damping_a: float,
                     damping_g: float) -> torch.Tensor:
    """P = (G + gamma_G I)^-1 grad (A + gamma_A I)^-1 in fp64 for the (g, a) gradient matrix [wgrad | bgrad], with
    gamma_A from damping_a and gamma_G from damping_g (the eigen and inverse methods agree on this operator; which
    step's damping each factor takes is the caller's choice).  A diagonal factor is a vector.  An embedding's P is the
    transpose of this, in its weight's (V, d) layout."""
    g_a, _ = gammas(pi, damping_a)
    _, g_g = gammas(pi, damping_g)
    return apply_right(apply_left(damped_inverse64(G, g_g), grad.double()), damped_inverse64(A, g_a))


def test_restatement_is_scale_invariant():
    gen = torch.Generator().manual_seed(0)
    x = torch.randn(40, 7, dtype=torch.float64, generator=gen)
    A, G = x.t() @ x / 40, torch.rand(5, dtype=torch.float64, generator=gen)
    grad = torch.randn(5, 7, dtype=torch.float64, generator=gen)
    p = precondition_ref(grad, A, G, pi_ref(A, G), 1e-2, 1e-2)
    for k in (-3, 2):
        c = 4.0 ** k
        q = precondition_ref(grad, c * A, G / c, pi_ref(c * A, G / c), 1e-2, 1e-2)
        assert torch.allclose(p, q, rtol=1e-12, atol=0)
        assert pi_ref(c * A, G / c) == c * pi_ref(A, G)
    # the Kronecker product of the damped factors is the product damped by sqrt(damping) on each side
    pi = pi_ref(A, G)
    ga, gg = gammas(pi, 1e-2)
    assert math.isclose(ga * gg, 1e-2, rel_tol=1e-6)
    assert pi_ref(torch.zeros(3, 3), G) == 1.0 and pi_ref(A, -torch.ones(4)) == 1.0
    assert pi_ref(A, torch.tensor([1.0, math.inf])) == 1.0 and pi_ref(torch.tensor([math.nan]), G) == 1.0


# ------------------------------------------------------------------------------------------- the keyword
class _Net(nn.Module):
    def __init__(self):
        super().__init__()
        self.emb = nn.Embedding(100, 16)
        self.conv = nn.Conv2d(3, 8, 3)
        self.bn = nn.BatchNorm2d(8)
        self.up = nn.ConvTranspose2d(8, 4, 2, stride=2)
        self.fc = nn.Linear(16, 32)
        self.wide = nn.Linear(32, 8)
        self.head = nn.Linear(8, 200, bias=False)


KW = dict(precondition_embeddings=True, precondition_norms=True, precondition_conv_transpose=True,
          diagonal_g_layers=['head'], diagonal_a_layers=['wide'])


def _names(pre):
    return {n: l for n, l in pre._layers.values()}


def test_keyword_repr_and_defaults():
    from kfac_b200.preconditioner import KFACPreconditioner
    off = KFACPreconditioner(_Net(), **KW)
    assert off._defaults['pi_damping'] is False and 'pi_damping=False' in repr(off)
    assert not any(l.pi_damping for l in _names(off).values())
    on = KFACPreconditioner(_Net(), pi_damping=True, **KW)
    assert on._defaults['pi_damping'] is True and 'pi_damping=True' in repr(on)
    assert all(l.pi_damping for l in _names(on).values())
    assert not any(l.pi_damping for _, l in on._norm_layers.values())
    for method in ('eigen', 'inverse'):
        KFACPreconditioner(_Net(), pi_damping=True, compute_method=method, **KW)
    for bad in (1, 'yes', None):
        with pytest.raises(ValueError, match='pi_damping must be a bool'):
            KFACPreconditioner(_Net(), pi_damping=bad)


def test_refusals_name_the_layer():
    from kfac_b200.preconditioner import KFACPreconditioner
    with pytest.raises(ValueError, match='pi_damping.*EKFAC.*"fc".*skip_layers'):
        KFACPreconditioner(nn.ModuleDict({'fc': nn.Linear(4, 4)}), compute_method='ekfac', pi_damping=True)
    KFACPreconditioner(nn.ModuleDict({'fc': nn.Linear(4, 4)}), compute_method='ekfac')

    class Tied(nn.Module):
        def __init__(self):
            super().__init__()
            self.wte = nn.Embedding(50, 8)
            self.lm_head = nn.Linear(8, 50, bias=False)
            self.lm_head.weight = self.wte.weight

    kw = dict(precondition_embeddings=True, diagonal_g_layers=['lm_head'], precondition_tied_embeddings=True)
    with pytest.raises(ValueError, match='pi_damping.*tied.*"wte" / "lm_head".*skip_layers'):
        KFACPreconditioner(Tied(), pi_damping=True, **kw)
    KFACPreconditioner(Tied(), **kw)
    KFACPreconditioner(Tied(), pi_damping=True, skip_layers=['lm_head'], precondition_embeddings=True)


def test_state_dict_unchanged():
    from kfac_b200.preconditioner import KFACPreconditioner
    sds = []
    for on in (False, True):
        pre = KFACPreconditioner(_Net(), pi_damping=on, **KW)
        for _, l in list(pre._layers.values()) + list(pre._norm_layers.values()):   # stand-ins for the arena views
            l._a_view = None if l.norm else torch.ones(l.a_factor_shape)
            l._g_view = torch.ones(l.g_factor_shape)
            l._has_a, l._has_g = not l.norm, True
        sd = pre.state_dict()
        sds.append({k: (v if k != 'layers' else {n: {f: (None if t is None else tuple(t.shape)) for f, t in e.items()}
                                                 for n, e in v.items()})
                    for k, v in sd.items()})
    assert sds[0] == sds[1]


def _layouts(on, method, prediv=True):
    from kfac_b200.base_preconditioner import second_order_layout
    from kfac_b200.preconditioner import KFACPreconditioner
    pre = KFACPreconditioner(_Net(), pi_damping=on, compute_method=method, compute_eigenvalue_outer_product=prediv,
                             **KW)
    return {n: second_order_layout(l) for n, l in pre._layers.values()}


@pytest.mark.parametrize('method,prediv', [('eigen', True), ('eigen', False), ('inverse', False)])
def test_every_kind_carries_a_pi_field(method, prediv):
    from kfac_b200 import _cabi
    off, on = _layouts(False, method, prediv), _layouts(True, method, prediv)
    kinds = {lay.item['kind'] for lay in on.values()}
    assert kinds == {_cabi.KFAC_ITEM_DENSE, _cabi.KFAC_ITEM_EMBEDDING, _cabi.KFAC_ITEM_DIAG_G, _cabi.KFAC_ITEM_DIAG_A}
    assert 'wgrad_taps' in on['up'].item
    assert 'pi' in dict(_cabi.PrecondItem._fields_)
    for name in off:
        a, b = off[name], on[name]
        assert 'pi' not in dict(a.fields) and dict(b.fields)['pi'] == 'pi'
        assert 'pi' not in a.needs and b.needs == a.needs | {'pi'}
        assert [e for e in b.entries if e.key == 'pi'] == [('pi', (1,), 'all', False, None)]
        assert [e for e in b.entries if e.key != 'pi'] == list(a.entries)
        assert b.decompositions == a.decompositions and b.item == a.item and b.eigen == a.eigen
        # the damped dgda and inverses read pi
        assert [(h, op, keys) for h, op, keys in a.post] == [(h, op, keys[:-1]) for h, op, keys in b.post]
        assert all(keys[-1] == 'pi' for _, _, keys in b.post)


def _plans(world, frac, method, prediv, colocate, pi):
    from kfac_b200.assignment import KAISAAssignment
    from kfac_b200.base_preconditioner import build_comm_plan, build_inverse_plan, build_local_plan
    from kfac_b200.enums import AssignmentStrategy
    from kfac_b200.layers import register_modules
    from kfac_b200.preconditioner import layer_work
    out = []
    handles = {}
    for rank in range(world):
        layers = register_modules(_Net(), [], precondition_embeddings=True, precondition_conv_transpose=True,
                                  diagonal_g_layers=['head'], diagonal_a_layers=['wide'], method=method,
                                  prediv_eigenvalues=prediv)
        ll = list(layers.values())
        for _, l in ll:
            l._has_a = l._has_g = True
            l.pi_damping = pi
        a = KAISAAssignment(layer_work(layers, AssignmentStrategy.COMPUTE), local_rank=rank, world_size=world,
                            grad_worker_fraction=frac,
                            group_func=lambda r: handles.setdefault(tuple(sorted(r)), tuple(sorted(r))),
                            colocate_factors=colocate)
        out.append((ll, build_comm_plan(ll, a), build_local_plan(ll, a, rank), build_inverse_plan(ll, a, rank)))
    return out


@pytest.mark.parametrize('world,frac', [(1, 1.0), (2, 1.0), (2, 0.5), (3, 1.0), (4, 1.0), (4, 0.5), (4, 0.25),
                                        (5, 0.2), (6, 0.5), (7, 1.0), (8, 1.0), (8, 0.5), (8, 0.125)])
@pytest.mark.parametrize('method,prediv,colocate', [('EIGEN', True, True), ('EIGEN', False, False),
                                                    ('INVERSE', False, True), ('INVERSE', False, False)])
def test_comm_plan_unchanged(world, frac, method, prediv, colocate):
    """pi is formed on every rank and never shipped: the broadcast segments of C2 and C3 are those without the keyword,
    and every rank keeps one pi per layer locally."""
    from kfac_b200.enums import ComputeMethod
    if colocate is False and frac * world <= 1:
        colocate = True
    m = ComputeMethod[method]
    off, on = _plans(world, frac, m, prediv, colocate, False), _plans(world, frac, m, prediv, colocate, True)

    def segs(plan):
        return [(s.src, s.group, s.offset, s.numel, [(l.index, k, sh) for l, k, sh in s.entries]) for s in plan]
    for (ll, (inv0, grad0), local0, (sn0, calls0, post0)), (_, (inv1, grad1), local1, (sn1, calls1, post1)) in zip(off,
                                                                                                                on):
        assert segs(inv0) == segs(inv1) and segs(grad0) == segs(grad1)
        assert [(l.index, k, sh) for l, k, sh in local1 if k != 'pi'] == [(l.index, k, sh) for l, k, sh in local0]
        assert sorted(l.index for l, k, sh in local1 if k == 'pi') == sorted(l.index for _, l in ll)
        assert all(sh == (1,) for _, k, sh in local1 if k == 'pi')
        assert [(l.index, s.index, side, k) for l, s, side, k in sn0] == [(l.index, s.index, side, k)
                                                                          for l, s, side, k in sn1]
        assert [[(l.index, *r) for l, *r in c] for c in calls0] == [[(l.index, *r) for l, *r in c] for c in calls1]
        assert [(l.index, op, keys + ('pi',)) for l, op, keys in post0] == [(l.index, op, keys) for l, op, keys in post1]


def test_pi_s_is_the_fp32_square_root():
    from kfac_b200.base_preconditioner import pi_s
    for lam in (1e-3, 0.003, 1.0, 2.0, 1e-7, 123.456):
        assert pi_s(lam) == float(np.sqrt(np.float32(lam)))
