"""Multi-process preconditioning of a tied embedding / LM head (run under torchrun, two ranks).

    torchrun --nnodes=1 --nproc-per-node=2 --master-addr 127.0.0.1 --master-port P tests/dist_tied.py [--backend gloo]

For COMM_OPT (every rank preconditions every layer) and MEM_OPT (one rank per layer, P broadcast), and for the eigen
and inverse methods, each rank runs one half of a global batch of the nanoGPT-shaped model of test_gpu_tied.py with
`precondition_tied_embeddings`, the gradients are averaged, and after every step
  * every rank writes the same gradients, bit for bit (kl-clip off);
  * the tied weight's gradient matches the fp64 formula built from the pair's snapshots and the factors the ranks
    hold at the inverse step.
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
from test_gpu_tied import KW, NanoGPT, _batch, _loss, _p_ref  # noqa: E402

V, STEPS = 1000, 3


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
            model = NanoGPT(V).to(dev)
            pre = KFACPreconditioner(model, kl_clip=None, damping=0.003, inv_update_steps=2, compute_method=method,
                                     grad_worker_fraction=strategy, **KW)
            emb = pre._layers[model.emb][1]
            E = H = None
            for step in range(STEPS):
                idx_all, y_all = _batch(step, V)
                half = idx_all.shape[0] // world
                idx, y = idx_all[rank * half:(rank + 1) * half], y_all[rank * half:(rank + 1) * half]
                model.zero_grad()
                _loss(model, idx, y).backward()
                for p in model.parameters():          # data parallelism: the gradients are averaged before step()
                    dist.all_reduce(p.grad)
                    p.grad /= world
                g = model.emb.weight.grad.clone()
                new_basis = pre.steps % pre.inv_update_steps == 0
                pre.step()
                torch.cuda.synchronize()
                if new_basis:
                    E, H = emb.g_factor.clone(), emb.tied_head.a_factor.clone()
                for n, p in model.named_parameters():
                    got = gather(p.grad)
                    assert all(torch.equal(got[0], o) for o in got[1:]), (strategy, method, step, n)
                if pre._assignment.is_grad_worker('emb'):
                    err = rel_fro(model.emb.weight.grad, _p_ref(g, emb, E, H, emb._tied_damping))
                    assert err <= 1e-3, (strategy, method, step, err)
                with torch.no_grad():
                    for p in model.parameters():
                        p -= 0.05 * p.grad
            pre.close()
    dist.barrier()
    print(f'dist_tied ok rank {rank}')
    dist.destroy_process_group()


if __name__ == '__main__':
    main()
