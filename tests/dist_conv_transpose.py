"""Multi-process ConvTranspose1d / 2d / 3d preconditioning (run under torchrun, two ranks).

    torchrun --nnodes=1 --nproc-per-node=2 --master-addr 127.0.0.1 --master-port P tests/dist_conv_transpose.py \
        [--backend gloo]

Each rank runs its half of a global batch of the DCGAN-style generator, the 1-D upsampler and the 3-D decoder of
test_gpu_conv_transpose.py with `precondition_conv_transpose=True` (gradients averaged over the ranks, as data
parallelism does).  After every step
  * every layer's A and G are the EMA of the mean of the ranks' fp64 factors (restated from the inputs and output
    gradients each rank captured);
  * every rank writes the same gradients, bit for bit,
under COMM_OPT, HYBRID_OPT and MEM_OPT for the eigen method, and under COMM_OPT for EKFAC.
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
from test_gpu_conv_transpose import NETS, _rows64, _Rec  # noqa: E402

ALPHA, DAMPING, STEPS = 0.9, 3e-3, 3


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

    def gather(t):
        t = t.contiguous() if args.backend == 'nccl' else t.detach().cpu().contiguous()
        out = [torch.empty_like(t) for _ in range(world)]
        dist.all_gather(out, t)
        return [o.to(dev) for o in out]

    def run(net, strategy, method):
        cls, shape = NETS[net]
        torch.manual_seed(0)
        model = cls().to(dev)
        with torch.no_grad():       # before the preconditioner hooks the model
            out_shape = model(torch.zeros(2 * shape[0], *shape[1:], device=dev)).shape
        pre = KFACPreconditioner(model, kl_clip=None, damping=DAMPING, factor_decay=ALPHA, grad_worker_fraction=strategy,
                                 compute_method=method, precondition_conv_transpose=True)
        rec = _Rec(pre._layers)
        gen = torch.Generator().manual_seed(1)
        A, G = {}, {}
        for s in range(STEPS):
            x_all = torch.randn(2 * shape[0], *shape[1:], generator=gen).to(dev)
            y_all = torch.randn(out_shape, generator=gen).to(dev)
            half = x_all.shape[0] // world
            x, y = x_all[rank * half:(rank + 1) * half], y_all[rank * half:(rank + 1) * half]
            model.zero_grad()
            rec.clear()
            (model(x) * y).sum().backward()
            for p in model.parameters():
                dist.all_reduce(p.grad)
                p.grad /= world
            pre.step()
            torch.cuda.synchronize()
            for m, (name, l) in pre._layers.items():
                wa, wg = 0.0, 0.0
                for xr, gr in zip(gather(rec.inp[m][0]), gather(rec.gout[m][0])):
                    X, Gr = _rows64(m, xr, gr, False)
                    wa = wa + X.T @ X / X.shape[0] / world
                    wg = wg + Gr.T @ Gr / Gr.shape[0] / world
                eye = lambda n: torch.eye(n, dtype=torch.float64, device=dev)  # noqa: E731
                A[name] = ALPHA * A.get(name, eye(wa.shape[0])) + (1 - ALPHA) * wa
                G[name] = ALPHA * G.get(name, eye(wg.shape[0])) + (1 - ALPHA) * wg
                assert rel_fro(l.a_factor, A[name]) <= 1e-5, (net, strategy, method, s, name, 'A')
                assert rel_fro(l.g_factor, G[name]) <= 1e-5, (net, strategy, method, s, name, 'G')
                got = m.weight.grad
                assert all(torch.equal(o, got) for o in gather(got)), (net, strategy, method, s, name)
                assert torch.isfinite(got).all()
        pre.close()
        dist.barrier()

    for net in ('dcgan', 'audio', 'vol'):
        for strategy in (DistributedStrategy.COMM_OPT, DistributedStrategy.HYBRID_OPT, DistributedStrategy.MEM_OPT):
            run(net, strategy, 'eigen')
        run(net, DistributedStrategy.COMM_OPT, 'ekfac')
    print(f'rank {rank}: dist_conv_transpose ok', flush=True)
    dist.destroy_process_group()


if __name__ == '__main__':
    main()
