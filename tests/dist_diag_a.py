"""Multi-process diagonal-A preconditioning (run under torchrun, two ranks).

    torchrun --nnodes=1 --nproc-per-node=2 --master-addr 127.0.0.1 --master-port P tests/dist_diag_a.py [--backend gloo]

For COMM_OPT (every rank preconditions every layer) and MEM_OPT (one rank per layer, P broadcast), and for the eigen
and inverse methods, each rank runs one half of a global batch of the SwiGLU block of test_gpu_diag_a.py with its
down_proj (8201 inputs) in `diagonal_a_layers`, the gradients are averaged, and after two steps
  * every rank holds the same down_proj factors and writes the same gradients (P, kl-clip off);
  * down_proj's diagonal A matches fp64 on the concatenated batch (the inputs of both ranks, averaged like the
    preconditioner averages the statistics);
  * every layer's P matches fp64 formed from the factors the ranks hold;
  * the run takes exactly the all-reduces of a run with down_proj skipped.
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
from test_gpu_diag_a import MODELS, SwiGLU, _a_rows64, _data, _grad_matrix, _loss, p_ref  # noqa: E402

ALPHA, DAMPING, STEPS = 0.9, 0.003, 2


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

    def run(strategy, method, check, **kw):
        torch.manual_seed(0)
        model = SwiGLU().to(dev)
        pre = KFACPreconditioner(model, kl_clip=None, damping=DAMPING, factor_decay=ALPHA,
                                 grad_worker_fraction=strategy, compute_method=method, **kw)
        layers = {m: l for m, (_, l) in pre._layers.items()}
        seen = {}
        model.down.register_forward_pre_hook(lambda mod, inp: seen.__setitem__('x', inp[0].detach()))
        opt = torch.optim.SGD(model.parameters(), lr=0.05)
        A_ref = None
        for s in range(STEPS):
            x_all, y_all = _data('swiglu', s)
            half = x_all.shape[0] // world
            x, y = x_all[rank * half:(rank + 1) * half], y_all[rank * half:(rank + 1) * half]
            opt.zero_grad()
            _loss('swiglu', model, x.to(dev), y.to(dev)).backward()
            for p in model.parameters():          # data parallelism: the gradients are averaged before step()
                dist.all_reduce(p.grad)
                p.grad /= world
            grads = {m: _grad_matrix(m) for m in layers}
            pre.step()
            torch.cuda.synchronize()
            if not check:
                continue
            xs = gather(seen['x'])
            win = sum(((r := _a_rows64(model.down, xi, False)) ** 2).sum(0) / r.shape[0] for xi in xs) / world
            A_ref = ALPHA * (torch.ones_like(win) if A_ref is None else A_ref) + (1 - ALPHA) * win
            ld = layers[model.down]
            assert ld.a_factor.shape == (8201,) and rel_fro(ld.a_factor, A_ref) < 1e-5, (strategy, method, s)
            for t in (ld.a_factor, ld.g_factor):
                others = gather(t)
                assert all(torch.equal(o, others[0]) for o in others), (strategy, method, s)
            for m, l in layers.items():
                got = _grad_matrix(m)
                others = gather(got)
                assert all(torch.equal(o, others[0]) for o in others), (strategy, method, s, pre._layers[m][0])
                ref = p_ref(l, method, grads[m], l.a_factor, l.g_factor, DAMPING)
                err = rel_fro(got, ref)
                assert err < 1e-3, (strategy, method, s, pre._layers[m][0], err)
            opt.step()
        calls = dict(pre._tdc.calls)
        pre.close()
        dist.barrier()
        return calls

    kw = MODELS['swiglu'][1]
    skip = dict(diagonal_g_layers=kw['diagonal_g_layers'], skip_layers=['down'])
    for strategy in (DistributedStrategy.COMM_OPT, DistributedStrategy.MEM_OPT):
        for method in ('eigen', 'inverse'):
            diag = run(strategy, method, True, **kw)
            skipped = run(strategy, method, False, **skip)
            assert diag['allreduce'] == skipped['allreduce'], (strategy, method, diag, skipped)
    print(f'rank {rank}: dist_diag_a ok', flush=True)
    dist.destroy_process_group()


if __name__ == '__main__':
    main()
