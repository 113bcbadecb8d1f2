"""Multi-process embedding preconditioning (run under torchrun, two ranks).

    torchrun --nnodes=1 --nproc-per-node=2 --master-addr 127.0.0.1 --master-port P tests/dist_embedding.py [--backend gloo]

For every placement two ranks allow -- COMM_OPT (grad_worker_fraction 1: every rank preconditions every layer) and
MEM_OPT (1/2: one rank per layer, the second-order data stays on it and P is broadcast) -- and for the eigen and
inverse methods, each rank runs one half of a global batch of the LM of test_gpu_embedding.py, the gradients are
averaged, and after two steps
  * every rank holds the same embedding factors and writes the same gradients (P, kl-clip off);
  * the embedding's P matches fp64 on the concatenated batch: A from the indices of both ranks, G from the
    grad-outputs of both ranks (averaged like the preconditioner averages the statistics);
  * every dense layer's P matches fp64 formed from the factors the ranks hold.
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
from test_gpu_embedding import D_LM, LM, V_LM, _batch, _grad_matrix, _p_dense, _p_embedding  # noqa: E402

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

    for strategy in (DistributedStrategy.COMM_OPT, DistributedStrategy.MEM_OPT):
        for method in ('eigen', 'inverse'):
            torch.manual_seed(0)
            model = LM().to(dev)
            pre = KFACPreconditioner(model, precondition_embeddings=True, kl_clip=None, damping=DAMPING,
                                     factor_decay=ALPHA, grad_worker_fraction=strategy, compute_method=method)
            layers = {m: l for m, (_, l) in pre._layers.items()}
            seen = {}

            def keep_grad_output(module, input_, output, seen=seen):   # returns None: the output is left as it is
                output.register_hook(lambda g: seen.__setitem__('g', g.detach()))
            model.emb.register_forward_hook(keep_grad_output)
            opt = torch.optim.SGD(model.parameters(), lr=0.05)
            A_ref = G_ref = None
            for s in range(STEPS):
                idx_all, y_all = _batch(s)
                half = idx_all.shape[0] // world
                idx, y = idx_all[rank * half:(rank + 1) * half], y_all[rank * half:(rank + 1) * half]
                opt.zero_grad()
                nn.functional.cross_entropy(model(idx).flatten(0, 1), y.flatten()).backward()
                for p in model.parameters():          # data parallelism: the gradients are averaged before step()
                    dist.all_reduce(p.grad)
                    p.grad /= world
                grads = {m: _grad_matrix(m) for m in layers}
                pre.step()
                torch.cuda.synchronize()
                # fp64 statistics of the concatenated batch, averaged over the ranks like the preconditioner does
                n = idx.numel()
                a_b = torch.bincount(idx_all.flatten(), minlength=V_LM).double() / idx_all.numel()
                gs = [g.double().reshape(n, D_LM) for g in gather(seen['g'])]
                g_b = sum(g.t() @ g / n for g in gs) / world
                if A_ref is None:
                    A_ref, G_ref = torch.ones_like(a_b), torch.eye(D_LM, dtype=torch.float64, device=dev)
                A_ref = ALPHA * A_ref + (1 - ALPHA) * a_b
                G_ref = ALPHA * G_ref + (1 - ALPHA) * g_b
                le = layers[model.emb]
                assert rel_fro(le.a_factor, A_ref) < 1e-6 and rel_fro(le.g_factor, G_ref) < 1e-5, (strategy, method, s)
                for t in (le.a_factor, le.g_factor):
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
    print(f'rank {rank}: dist_embedding ok', flush=True)
    dist.destroy_process_group()


if __name__ == '__main__':
    main()
