import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, 'tests', 'golden')


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100)')


def rel_fro(a: torch.Tensor, b: torch.Tensor) -> float:
    a = a.detach().double().cpu()
    b = b.detach().double().cpu()
    den = b.norm().item()
    return (a - b).norm().item() / (den if den > 0 else 1.0)


def load_fixture(name):
    return torch.load(os.path.join(GOLDEN, name + '.pt'), weights_only=False)


MODELS = {}


GOLDEN_NAMES = ['tiny_eigen', 'tiny_eigen_noprediv', 'tiny_inverse', 'tiny_sched',
                'conv_eigen', 'conv_inverse', 'conv_accum',
                # widened cases: per-axis conv geometry, (batch, seq, feature) Linear inputs,
                # callable hyper-parameters, skip_layers
                'geom_eigen', 'geom_inverse', 'seq_eigen', 'tiny_callable', 'conv_skip',
                # factors updated in step() with gradient accumulation; conv net on a factor/inverse schedule
                'conv_nohook', 'conv_sched']

GOLDEN_CPU_ONLY = []


def model_for(name, fx=None):
    from oracle.models import MODEL_ZOO, SmallConvNet, TinyModel
    if fx is not None and fx.get('model'):
        return MODEL_ZOO[fx['model']]()
    return TinyModel() if name.startswith('tiny') else SmallConvNet()


def loss_for(name, fx=None):
    if fx is not None and fx.get('loss'):
        from oracle.fixture_util import loss_by_name
        return loss_by_name(fx['loss'])
    if name.startswith('tiny'):
        return torch.nn.MSELoss(reduction='sum')
    return torch.nn.CrossEntropyLoss()


def replay(name, make_precond, device='cpu', get_layers=None):
    """Replay a golden fixture through a preconditioner implementation.

    make_precond(model, **kwargs) -> object with .step(); get_layers(pre) ->
    {layer_name: (A, G)} after each step.  Yields (step_idx, golden_step,
    model, pre) after every step().
    """
    from oracle.fixture_util import materialize_kwargs
    fx = load_fixture(name)
    model = model_for(name, fx)
    model.load_state_dict(fx['init'])
    model.to(device)
    pre = make_precond(model, **materialize_kwargs(fx['kwargs']))
    opt = torch.optim.SGD(model.parameters(), lr=0.05)
    loss_fn = loss_for(name, fx)
    bi = 0
    for s in range(fx['steps']):
        opt.zero_grad()
        for _ in range(fx['micro']):
            x, y = fx['batches'][bi % len(fx['batches'])]
            bi += 1
            loss_fn(model(x.to(device)), y.to(device)).backward()
        pre.step()
        yield s, fx['record'][s], model, pre
        opt.step()


@pytest.fixture
def golden_names():
    return list(GOLDEN_NAMES)
