"""Multi-process pi-adjusted damping (run under torchrun, two ranks).

    torchrun --nnodes=1 --nproc-per-node=2 --master-addr 127.0.0.1 --master-port P tests/dist_pi_damping.py [--backend gloo]

For COMM_OPT (every rank preconditions every layer) and MEM_OPT (one rank per layer, P broadcast) under the eigen and
inverse methods, and for colocate_factors=False under the inverse method (A and G of a layer inverted on different
ranks, each with its own gamma from the same pi), each rank runs one half of a global batch of the conv net of
test_gpu_pi_damping.py (BatchNorm, a diagonal-A head) with pi_damping=True, the gradients are averaged, and after
each of two steps
  * every rank holds the same pi for every layer and writes the same gradients (kl-clip off);
  * every layer's gradient matches fp64 formed from the averaged gradient (the gradient of the concatenated batch),
    the factors the ranks hold and pi from their fp64 traces;
  * the run takes exactly the collectives of a run with pi_damping=False.
`--backend gloo` runs both ranks on shared GPUs; NCCL needs one GPU per rank.
"""
import argparse
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from conftest import rel_fro  # noqa: E402
from kfac_b200.enums import DistributedStrategy  # noqa: E402
from kfac_b200.preconditioner import KFACPreconditioner  # noqa: E402
from test_gpu_pi_damping import MODELS, _close_pi, _data, _grad_matrix, _loss  # noqa: E402
from test_pi_damping_host import pi_ref, precondition_ref  # noqa: E402

DAMPING, STEPS = 0.003, 2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--backend', default='nccl', choices=['nccl', 'gloo'])
    args = ap.parse_args()
    rank, world = int(os.environ['RANK']), int(os.environ['WORLD_SIZE'])
    local = int(os.environ.get('LOCAL_RANK', rank))
    dev = torch.device('cuda', local % torch.cuda.device_count())
    torch.cuda.set_device(dev)
    if args.backend == 'nccl':
        dist.init_process_group('nccl', device_id=dev)
    else:
        dist.init_process_group('gloo')

    def gather(t):
        t = t.contiguous() if args.backend == 'nccl' else t.detach().cpu().contiguous()
        out = [torch.empty_like(t) for _ in range(world)]
        dist.all_gather(out, t)
        return [o.to(dev) for o in out]

    cls, kw = MODELS['conv']

    def run(strategy, method, colocate, pi_damping):
        torch.manual_seed(0)
        model = cls().to(dev)
        pre = KFACPreconditioner(model, kl_clip=None, damping=DAMPING, grad_worker_fraction=strategy,
                                 compute_method=method, colocate_factors=colocate,
                                 compute_eigenvalue_outer_product=colocate, pi_damping=pi_damping, **kw)
        layers = {n: l for n, l in pre._layers.values()}
        opt = torch.optim.SGD(model.parameters(), lr=0.05)
        for s in range(STEPS):
            x_all, y_all = _data('conv', s)
            half = x_all.shape[0] // world
            opt.zero_grad()
            _loss(model, x_all[rank * half:(rank + 1) * half], y_all[rank * half:(rank + 1) * half]).backward()
            for p in model.parameters():          # data parallelism: the gradients are averaged before step()
                dist.all_reduce(p.grad)
                p.grad /= world
            grads = {n: _grad_matrix(l) for n, l in layers.items()}
            pre.step()
            torch.cuda.synchronize()
            if pi_damping:
                for n, l in layers.items():
                    pis = gather(l._inv['pi'][:1].clone())
                    assert all(torch.equal(p, pis[0]) for p in pis), (strategy, method, s, n)
                    A, G = l.a_factor, l.g_factor
                    pi = float(pis[0])
                    assert _close_pi(pi, pi_ref(A, G)), (strategy, method, s, n)
                    got = _grad_matrix(l)
                    others = gather(got)
                    assert all(torch.equal(o, others[0]) for o in others), (strategy, method, s, n)
                    err = rel_fro(got, precondition_ref(grads[n], A, G, pi, DAMPING, DAMPING))
                    assert err < 1e-3, (strategy, method, colocate, s, n, err)
            opt.step()
        calls = dict(pre._tdc.calls)
        pre.close()
        dist.barrier()
        return calls

    cases = [(DistributedStrategy.COMM_OPT, 'eigen', True), (DistributedStrategy.COMM_OPT, 'inverse', True),
             (DistributedStrategy.MEM_OPT, 'eigen', True), (DistributedStrategy.MEM_OPT, 'inverse', True),
             (DistributedStrategy.COMM_OPT, 'inverse', False)]
    for strategy, method, colocate in cases:
        on = run(strategy, method, colocate, True)
        off = run(strategy, method, colocate, False)
        assert on == off, (strategy, method, colocate, on, off)
    print(f'rank {rank}: dist_pi_damping ok', flush=True)
    dist.destroy_process_group()


if __name__ == '__main__':
    main()
