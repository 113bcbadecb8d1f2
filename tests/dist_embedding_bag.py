"""Multi-process embedding-bag preconditioning (run under torchrun, two ranks).

    torchrun --nnodes=1 --nproc-per-node=2 --master-addr 127.0.0.1 --master-port P tests/dist_embedding_bag.py [--backend gloo]

For COMM_OPT (every rank preconditions every layer) and MEM_OPT (one rank per layer, P is broadcast), and for the
eigen and inverse methods, each rank runs one half of the bags of a global batch of the text classifier of
test_gpu_embedding_bag.py, the gradients are averaged, and after two steps
  * every rank holds the same bag factors and writes the same gradients (P, kl-clip off);
  * the bag's P matches fp64 on the concatenated batch: A from the pooled rows of both ranks' bags, G from the
    output gradients of both ranks (averaged like the preconditioner averages the statistics; equal batches per rank);
  * the Linear layer's P matches fp64 formed from the factors the ranks hold.
`--backend gloo` runs both ranks on shared GPUs; NCCL needs one GPU per rank.
"""
import argparse
import os
import sys

import torch
import torch.distributed as dist
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from conftest import rel_fro  # noqa: E402
from kfac_b200.enums import DistributedStrategy  # noqa: E402
from kfac_b200.preconditioner import KFACPreconditioner  # noqa: E402
from test_gpu_embedding import _grad_matrix, _p_dense, _p_embedding  # noqa: E402
from test_gpu_embedding_bag import D_TC, V_TC, TextClassifier, bag_a, pooled_rows, tc_batch  # noqa: E402

ALPHA, DAMPING, STEPS = 0.9, 0.003, 2


def split(idx, offsets, y, rank, world):
    """Bags [rank * B / world, (rank + 1) * B / world) of a batch, with their offsets rebased."""
    B = offsets.numel()
    half = B // world
    lo, hi = rank * half, (rank + 1) * half
    start = int(offsets[lo])
    end = int(offsets[hi]) if hi < B else idx.numel()
    return idx[start:end], offsets[lo:hi] - start, y[lo:hi]


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

    for strategy in (DistributedStrategy.COMM_OPT, DistributedStrategy.MEM_OPT):
        for method in ('eigen', 'inverse'):
            torch.manual_seed(0)
            model = TextClassifier().to(dev)
            pre = KFACPreconditioner(model, precondition_embedding_bags=True, kl_clip=None, damping=DAMPING,
                                     factor_decay=ALPHA, grad_worker_fraction=strategy, compute_method=method)
            layers = {m: l for m, (_, l) in pre._layers.items()}
            seen = {}

            def keep_grad_output(module, input_, output, seen=seen):   # returns None: the output is left as it is
                output.register_hook(lambda g: seen.__setitem__('g', g.detach()))
            model.bag.register_forward_hook(keep_grad_output)
            opt = torch.optim.SGD(model.parameters(), lr=0.05)
            A_ref = G_ref = None
            for s in range(STEPS):
                idx_all, off_all, y_all = tc_batch(s)
                idx, offsets, y = split(idx_all, off_all, y_all, rank, world)
                opt.zero_grad()
                nn.functional.cross_entropy(model(idx, offsets), y).backward()
                for p in model.parameters():          # data parallelism: the gradients are averaged before step()
                    dist.all_reduce(p.grad)
                    p.grad /= world
                grads = {m: _grad_matrix(m) for m in layers}
                pre.step()
                torch.cuda.synchronize()
                # fp64 statistics of the concatenated batch, averaged over the ranks like the preconditioner does
                B = off_all.numel()
                a_b = bag_a(pooled_rows(idx_all, off_all, B, V_TC, 'mean', padding_idx=model.bag.padding_idx))
                gs = [g.double() for g in gather(seen['g'])]
                g_b = sum(g.t() @ g / g.shape[0] for g in gs) / world
                if A_ref is None:
                    A_ref, G_ref = torch.ones_like(a_b), torch.eye(D_TC, dtype=torch.float64, device=dev)
                A_ref = ALPHA * A_ref + (1 - ALPHA) * a_b
                G_ref = ALPHA * G_ref + (1 - ALPHA) * g_b
                lb = layers[model.bag]
                assert rel_fro(lb.a_factor, A_ref) < 1e-6 and rel_fro(lb.g_factor, G_ref) < 1e-5, (strategy, method, s)
                for t in (lb.a_factor, lb.g_factor):
                    others = gather(t)
                    assert all(torch.equal(o, others[0]) for o in others), (strategy, method, s)
                for m, l in layers.items():
                    got = _grad_matrix(m)
                    others = gather(got)
                    assert all(torch.equal(o, others[0]) for o in others), (strategy, method, s, pre._layers[m][0])
                    if l.diag_a:
                        ref = _p_embedding(method, grads[m], A_ref, G_ref, DAMPING)
                    else:
                        ref = _p_dense(method, grads[m], l.a_factor, l.g_factor, DAMPING)
                    err = rel_fro(got, ref)
                    assert err < 1e-3, (strategy, method, s, pre._layers[m][0], err)
                opt.step()
            pre.close()
            dist.barrier()
    print(f'rank {rank}: dist_embedding_bag ok', flush=True)
    dist.destroy_process_group()


if __name__ == '__main__':
    main()
