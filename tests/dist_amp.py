"""Two-rank run of the guarded EMA under a GradScaler (run under torchrun, launched by tests/test_gpu_amp.py).

    torchrun --nnodes=1 --nproc-per-node=2 --master-addr 127.0.0.1 --master-port P tests/dist_amp.py

Rank 0 alone overflows on one step (its loss is scaled by another 2^50).  The batch statistics are averaged over the
ranks before the EMA decides, so both ranks drop the same windows and keep bitwise-equal factors.
"""
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from kfac_b200.preconditioner import KFACPreconditioner  # noqa: E402


class Net(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.conv1 = torch.nn.Conv2d(3, 32, 3, padding=1)
        self.conv2 = torch.nn.Conv2d(32, 64, 3, stride=2, padding=1, bias=False)
        self.fc = torch.nn.Linear(64, 10)

    def forward(self, x):
        x = torch.relu(self.conv2(torch.relu(self.conv1(x))))
        return self.fc(torch.nn.functional.adaptive_avg_pool2d(x, 1).flatten(1))


def same_on_all_ranks(t):
    ref = t.clone()
    dist.broadcast(ref, src=0)
    ok = torch.tensor([1 if torch.equal(ref, t) else 0], device=t.device)
    dist.all_reduce(ok, op=dist.ReduceOp.MIN)
    return bool(ok.item())


def main():
    rank, world = int(os.environ['RANK']), int(os.environ['WORLD_SIZE'])
    local = int(os.environ.get('LOCAL_RANK', rank))
    torch.cuda.set_device(local)
    dev = torch.device('cuda', local)
    dist.init_process_group('nccl', device_id=dev)
    torch.manual_seed(0)
    model = Net().to(dev)
    scaler = torch.amp.GradScaler('cuda', init_scale=2.0 ** 10, growth_interval=10 ** 9)
    pre = KFACPreconditioner(model, grad_scaler=scaler, damping=0.003)
    opt = torch.optim.SGD(model.parameters(), lr=0.01)
    layers = [layer for _, layer in pre._layers.values()]
    ok = True
    for step in range(5):
        g = torch.Generator(device='cpu').manual_seed(100 * step + rank)
        x = torch.randn(8, 3, 12, 12, generator=g).to(dev)
        y = torch.randint(0, 10, (8,), generator=g).to(dev)
        opt.zero_grad()
        if step == 2:
            before = [layer.g_factor.clone() for layer in layers]
        with torch.autocast('cuda', dtype=torch.float16):
            loss = torch.nn.functional.cross_entropy(model(x), y)
        (scaler.scale(loss) * (2.0 ** 50 if step == 2 and rank == 0 else 1.0)).backward()
        for p in model.parameters():          # what DDP does
            dist.all_reduce(p.grad)
            p.grad /= world
        scaler.unscale_(opt)
        pre.step()
        torch.cuda.synchronize()
        for i, layer in enumerate(layers):
            for name, f in (('A', layer.a_factor), ('G', layer.g_factor)):
                if not torch.isfinite(f).all() or not same_on_all_ranks(f):
                    print(f'rank {rank} step {step}: factor {name} of layer {i} is not finite or differs', flush=True)
                    ok = False
        if step == 2:
            for i, (layer, b) in enumerate(zip(layers, before)):
                if not torch.equal(layer.g_factor, b):
                    print(f'rank {rank}: G factor of layer {i} changed on the overflow step', flush=True)
                    ok = False
        if step > 2:
            for p in model.parameters():
                if not torch.isfinite(p.grad).all():
                    print(f'rank {rank} step {step}: non-finite preconditioned gradient', flush=True)
                    ok = False
        scaler.step(opt)
        scaler.update()
    skipped = torch.tensor([pre.skipped_factor_updates], device=dev)
    if skipped.item() != len(layers) or not same_on_all_ranks(skipped):
        print(f'rank {rank}: {skipped.item()} windows dropped, expected {len(layers)} on every rank', flush=True)
        ok = False
    flag = torch.tensor([1 if ok else 0], device=dev)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    dist.barrier()
    dist.destroy_process_group()
    if not flag.item():
        sys.exit(1)
    if rank == 0:
        print(f'world={world} dropped windows per rank = {len(layers)}', flush=True)
        print('DIST AMP OK', flush=True)


if __name__ == '__main__':
    main()
