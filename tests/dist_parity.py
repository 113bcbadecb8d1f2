"""Multi-GPU parity of the KAISA data-parallel path (run under torchrun).

    torchrun --nnodes=1 --nproc-per-node=N --master-addr 127.0.0.1 --master-port P tests/dist_parity.py

Every rank runs kfac_b200 on its own shard of a global batch; the result must
equal the single-process CPU oracle on the CONCATENATED batch (for a model
without BatchNorm, averaging per-rank covariances / gradients is exactly the
covariance / gradient of the concatenated batch once the loss scaling of the
per-rank mean losses is reproduced).  Checks every
grad_worker_fraction the world size admits (COMM-OPT, HYBRID-OPT, MEM-OPT).
"""
import copy
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from kfac_b200.preconditioner import KFACPreconditioner  # noqa: E402
from oracle.kfac_oracle import OraclePreconditioner  # noqa: E402
from oracle.models import SmallConvNet  # noqa: E402


def main():
    rank, world = int(os.environ['RANK']), int(os.environ['WORLD_SIZE'])
    local = int(os.environ.get('LOCAL_RANK', rank))
    torch.cuda.set_device(local)
    dev = torch.device('cuda', local)
    dist.init_process_group('nccl', device_id=dev)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    fracs = sorted({1.0, 1.0 / world, 0.5 if world % 2 == 0 else 1.0})
    crit = torch.nn.CrossEntropyLoss()
    per_rank = 4
    ok = True
    for method, sym in (('eigen', False), ('eigen', True), ('inverse', False)):
        for frac in fracs:
            torch.manual_seed(0)
            ref_model = SmallConvNet()
            model = copy.deepcopy(ref_model).to(dev)
            torch.manual_seed(1)
            gx = torch.randn(world * per_rank, 3, 12, 12)
            gy = torch.randint(0, 5, (world * per_rank,))
            x, y = gx[rank * per_rank:(rank + 1) * per_rank].to(dev), gy[rank * per_rank:(rank + 1) * per_rank].to(dev)
            pre = KFACPreconditioner(model, damping=0.003, grad_worker_fraction=frac, compute_method=method,
                                     symmetry_aware=sym)
            ref = OraclePreconditioner(ref_model, damping=0.003, compute_method=method) if rank == 0 else None
            worst = 0.0
            for step in range(3):
                model.zero_grad()
                crit(model(x), y).backward()
                for p in model.parameters():          # what DDP does
                    dist.all_reduce(p.grad)
                    p.grad /= world
                pre.step()
                torch.cuda.synchronize()
                if rank == 0:
                    # every rank back-propagates the MEAN loss of its own shard, so the
                    # grad-outputs the G hooks see are 1/per_rank-scaled: reproduce that on the
                    # concatenated batch with world * mean-loss, then undo the factor on the
                    # parameter gradients (DDP averages them).
                    ref_model.zero_grad()
                    (crit(ref_model(gx), gy) * world).backward()
                    for q in ref_model.parameters():
                        q.grad /= world
                    ref.step()
                for i, (p, q) in enumerate(zip(model.parameters(), ref_model.parameters())):
                    want = q.grad.to(dev) if rank == 0 else torch.empty_like(p.grad)
                    dist.broadcast(want, src=0)
                    err = ((p.grad.double() - want.double()).norm() / want.double().norm()).item()
                    worst = max(worst, err)
                # lock-step update
                with torch.no_grad():
                    for p, q in zip(model.parameters(), ref_model.parameters()):
                        p -= 0.05 * p.grad
                        if rank == 0:
                            q -= 0.05 * q.grad
            t = torch.tensor([worst], device=dev)
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            if rank == 0:
                print(f'world={world} method={method} symmetry_aware={sym} grad_worker_fraction={frac:.3f} '
                      f'collectives={pre._tdc.calls} worst rel-fro vs oracle = {t.item():.2e}', flush=True)
            ok = ok and t.item() < 1e-3
            # C1: the A block of the batch statistics is all-reduced from the first backward hook (overlapped with
            # backward), the G block at step(); packed triangles (symmetry_aware) go in one piece at step()
            want_calls = 3 * (1 if sym else 2)
            if pre._tdc.calls['allreduce'] != want_calls:
                print(f'rank {rank}: {pre._tdc.calls["allreduce"]} factor all-reduces, expected {want_calls}', flush=True)
                ok = False
    # wide layers (a = 833 / 769, g = 768): the large-matrix eigensolver class, an eigenbasis broadcast
    # segment of several MB (C2) and a multi-tile (6 x 7 tiles of 128 x 128) wgmma precondition epilogue
    # that stores straight into the peers' arenas (fused compute + broadcast, C3)
    class Wide(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.l1 = torch.nn.Linear(832, 768)
            self.l2 = torch.nn.Linear(768, 128)
            self.l3 = torch.nn.Linear(128, 5)

        def forward(self, x):
            return self.l3(torch.tanh(self.l2(torch.tanh(self.l1(x)))))

    for wi, frac in enumerate(sorted({1.0 / world, 0.5 if world % 2 == 0 else 1.0 / world})):
        torch.manual_seed(0)
        ref_model = Wide()
        model = copy.deepcopy(ref_model).to(dev)
        torch.manual_seed(2)
        gx = torch.randn(world * 16, 832)
        gy = torch.randint(0, 5, (world * 16,))
        x, y = gx[rank * 16:(rank + 1) * 16].to(dev), gy[rank * 16:(rank + 1) * 16].to(dev)
        pre = KFACPreconditioner(model, damping=0.003, grad_worker_fraction=frac)
        pre.overlap_factor_allreduce = wi != 0       # the first configuration takes the one-piece reduction at step()
        ref = OraclePreconditioner(ref_model, damping=0.003) if rank == 0 else None
        worst = 0.0
        for step in range(2):
            model.zero_grad()
            crit(model(x), y).backward()
            for p in model.parameters():
                dist.all_reduce(p.grad)
                p.grad /= world
            pre.step()
            torch.cuda.synchronize()
            if rank == 0:
                ref_model.zero_grad()
                (crit(ref_model(gx), gy) * world).backward()
                for q in ref_model.parameters():
                    q.grad /= world
                ref.step()
            for p, q in zip(model.parameters(), ref_model.parameters()):
                want = q.grad.to(dev) if rank == 0 else torch.empty_like(p.grad)
                dist.broadcast(want, src=0)
                worst = max(worst, ((p.grad.double() - want.double()).norm() / want.double().norm()).item())
        t = torch.tensor([worst], device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        if rank == 0:
            print(f'world={world} wide-MLP grad_worker_fraction={frac:.3f} overlap={pre.overlap_factor_allreduce} fused={pre._peer_p_bases is not None} '
                  f'collectives={pre._tdc.calls} worst rel-fro vs oracle = {t.item():.2e}', flush=True)
        ok = ok and t.item() < 1e-3
    dist.barrier()
    dist.destroy_process_group()
    if not ok:
        sys.exit(1)
    if rank == 0:
        print('DIST PARITY OK', flush=True)


if __name__ == '__main__':
    main()
