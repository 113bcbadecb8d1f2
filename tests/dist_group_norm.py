"""Multi-process preconditioning of GroupNorm / InstanceNorm layers (run under torchrun, two ranks).

    torchrun --nnodes=1 --nproc-per-node=2 --master-addr 127.0.0.1 --master-port P tests/dist_group_norm.py [--backend gloo]

For COMM_OPT and MEM_OPT, and for the eigen and inverse methods, each rank runs one half of a global batch of the
U-Net-shaped model (GroupNorm) and of the generator (InstanceNorm2d) of test_gpu_group_norm.py with
`precondition_group_norms=True`; the losses are sums, so the summed gradients are those of the whole batch.  After
every step
  * every rank writes the same norm gradients, bit for bit;
  * the blocks are the mean of the ranks' fp64 blocks (the statistics are per example, so each rank's block is exact
    for its half), and P matches the fp64 solve with them;
  * the run takes exactly the collectives of a run with the keyword off.
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
from test_gpu_group_norm import batch, capture, loss_of, make_model, ref_group_blocks  # noqa: E402
from test_gpu_norm import _norm_grad, ref_solve  # noqa: E402

ALPHA, DAMPING, STEPS = 0.9, 1e-3, 2


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

    def run(kind, strategy, method, group_norms):
        torch.manual_seed(0)
        model = make_model(kind)
        pre = KFACPreconditioner(model, kl_clip=None, damping=DAMPING, factor_decay=ALPHA,
                                 grad_worker_fraction=strategy, compute_method=method,
                                 precondition_conv_transpose=True, precondition_group_norms=group_norms)
        calls = capture(model)
        F = {}
        for s in range(STEPS):
            x_all, t_all, y_all = batch(kind, s, B=8)
            half = x_all.shape[0] // world
            x, t, y = (v[rank * half:(rank + 1) * half] for v in (x_all, t_all, y_all))
            model.zero_grad()
            for c in calls.values():
                c.clear()
            loss_of(model, x, t, y).backward()
            for p in model.parameters():          # data parallelism: sum losses, so the gradients are summed
                dist.all_reduce(p.grad)
            grads = {m: _norm_grad(m).clone() for m in calls}
            pre.step()
            torch.cuda.synchronize()
            if not group_norms:
                continue
            assert len(pre._norm_layers) == len(calls)
            for m, (name, l) in pre._norm_layers.items():
                (c,) = calls[m]
                w = sum(ref_group_blocks(m, xr, gr) for xr, gr in zip(gather(c['x']), gather(c['g']))) / world
                seed = torch.zeros_like(w)
                seed[:, 0] = seed[:, -1] = 1.0
                F[m] = ALPHA * F.get(m, seed) + (1 - ALPHA) * w
                assert rel_fro(l.g_factor, F[m]) <= 1e-5, (kind, strategy, method, s, name)
                got = _norm_grad(m)
                assert all(torch.equal(o, got) for o in gather(got)), (kind, strategy, method, s, name)
                err = rel_fro(got, ref_solve(F[m], grads[m], DAMPING))
                assert err <= 1e-5, (kind, strategy, method, s, name, err)
        calls_made = dict(pre._tdc.calls)
        pre.close()
        dist.barrier()
        return calls_made

    for kind in ('unet', 'gen'):
        for strategy in (DistributedStrategy.COMM_OPT, DistributedStrategy.MEM_OPT):
            for method in ('eigen', 'inverse'):
                on = run(kind, strategy, method, True)
                off = run(kind, strategy, method, False)
                assert on == off, (kind, strategy, method, on, off)
    print(f'rank {rank}: dist_group_norm ok', flush=True)
    dist.destroy_process_group()


if __name__ == '__main__':
    main()
