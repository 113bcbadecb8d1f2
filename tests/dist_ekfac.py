"""Multi-process EKFAC (run under torchrun; COMM_OPT, the placement EKFAC supports).

    torchrun --nnodes=1 --nproc-per-node=N --master-addr 127.0.0.1 --master-port P tests/dist_ekfac.py [--backend gloo]

Every rank runs a shard of a global batch with factor_update_steps=1 and inv_update_steps=3 over 5 steps, so S is
reset to S_batch on steps 0 and 3 (new bases) and follows the EMA on steps 1, 2 and 4.  After every step
  * all ranks hold the same S and the same preconditioned gradients P;
  * S matches the fp64 per-row restatement of test_gpu_ekfac.py on the concatenated rows of all ranks, with the
    same schedule and the GPU's own eigenbases, and P matches Qg [(Qg^T grad Qa) / (S + damping)] Qa^T in fp64;
  * EKFAC issues exactly one all-reduce more per factor step than the eigen method (the average of S_batch).
NCCL needs one GPU per rank; `--backend gloo` runs the ranks on shared GPUs (gloo all-reduces and broadcasts the CUDA
arenas), which exercises the same collectives of the preconditioner on a single-GPU machine.
"""
import argparse
import copy
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from conftest import rel_fro  # noqa: E402
from kfac_b200.preconditioner import KFACPreconditioner  # noqa: E402
from oracle.models import SmallConvNet  # noqa: E402
from test_gpu_ekfac import _grad_matrix, _layer_rows, _Rec, _s_batch_per_row  # noqa: E402

STEPS, FUS, IUS, ALPHA, DAMPING = 5, 1, 3, 0.9, 0.003


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
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False

    def gather(t):
        """all_gather (gloo gathers host tensors)."""
        t = t.contiguous() if args.backend == 'nccl' else t.detach().cpu().contiguous()
        out = [torch.empty_like(t) for _ in range(world)]
        dist.all_gather(out, t)
        return out

    crit = torch.nn.CrossEntropyLoss()
    per_rank = 4
    torch.manual_seed(0)
    base = SmallConvNet()
    torch.manual_seed(1)
    batches = [(torch.randn(world * per_rank, 3, 12, 12), torch.randint(0, 5, (world * per_rank,)))
               for _ in range(STEPS)]
    calls = {}
    ok = True
    worst_s = worst_p = 0.0
    for method in ('eigen', 'ekfac'):
        model = copy.deepcopy(base).to(dev)
        pre = KFACPreconditioner(model, damping=DAMPING, compute_method=method, factor_decay=ALPHA, kl_clip=None,
                                 factor_update_steps=FUS, inv_update_steps=IUS)
        rec = _Rec(pre) if method == 'ekfac' else None
        S_ref = {}
        for step, (gx, gy) in enumerate(batches):
            x, y = gx[rank * per_rank:(rank + 1) * per_rank].to(dev), gy[rank * per_rank:(rank + 1) * per_rank].to(dev)
            if rec is not None:
                rec.clear()
            model.zero_grad()
            crit(model(x), y).backward()
            for p in model.parameters():          # what DDP does
                dist.all_reduce(p.grad)
                p.grad /= world
            grads = {name: _grad_matrix(m) for m, (name, _) in pre._layers.items()}
            pre.step()
            torch.cuda.synchronize()
            if method != 'ekfac':
                continue
            for m, (name, layer) in pre._layers.items():
                for t in (layer._S, layer._p_view):
                    allt = gather(t)
                    if not all(torch.equal(allt[0], u) for u in allt):
                        print(f'rank {rank}: step {step} {name}: ranks differ', flush=True)
                        ok = False
                # the concatenated rows of all ranks (each rank's rows come from its own mean loss)
                xs, gs = gather(rec.inp[m]), gather(rec.gout[m])
                if rank != 0:
                    continue
                Qa, Qg = layer.qa.double().cpu(), layer.qg.double().cpu()
                parts = [_layer_rows(m, xi, gi) for xi, gi in zip(xs, gs)]
                X = torch.cat([p[0] for p in parts])
                G = torch.cat([p[1] for p in parts])
                Sb = _s_batch_per_row(X, G, Qa, Qg)
                S_ref[name] = Sb if step % IUS == 0 else ALPHA * S_ref[name] + (1 - ALPHA) * Sb
                e = rel_fro(layer._S[:, :layer.a_dim], S_ref[name])
                worst_s = max(worst_s, e)
                if e > 1e-4:
                    print(f'step {step} {name}: S rel-fro vs fp64 = {e:.2e}', flush=True)
                    ok = False
                P = Qg @ ((Qg.T @ grads[name] @ Qa) / (S_ref[name] + DAMPING)) @ Qa.T
                e = rel_fro(_grad_matrix(m), P)      # kl_clip=None: the written gradient is P
                worst_p = max(worst_p, e)
                if e > 1e-3:
                    print(f'step {step} {name}: P rel-fro vs fp64 = {e:.2e}', flush=True)
                    ok = False
            with torch.no_grad():
                for p in model.parameters():
                    p -= 0.05 * p.grad
        calls[method] = pre._tdc.calls['allreduce']
    factor_steps = sum(1 for s in range(STEPS) if s % FUS == 0)
    if calls['ekfac'] - calls['eigen'] != factor_steps:
        print(f'rank {rank}: all-reduces eigen {calls["eigen"]}, ekfac {calls["ekfac"]}: expected {factor_steps} more',
              flush=True)
        ok = False
    t = torch.tensor([0 if ok else 1], device=dev if args.backend == 'nccl' else 'cpu')
    dist.all_reduce(t)
    dist.barrier()
    dist.destroy_process_group()
    if t.item():
        sys.exit(1)
    if rank == 0:
        print(f'world={world} backend={args.backend} all-reduces eigen={calls["eigen"]} ekfac={calls["ekfac"]} '
              f'worst S rel-fro {worst_s:.2e}, worst P rel-fro {worst_p:.2e}', flush=True)
        print('DIST EKFAC OK', flush=True)


if __name__ == '__main__':
    main()
