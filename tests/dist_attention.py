"""Multi-process preconditioning of attention projections (run under torchrun, two ranks).

    torchrun --nnodes=1 --nproc-per-node=2 --master-addr 127.0.0.1 --master-port P tests/dist_attention.py [--backend gloo]

For COMM_OPT and MEM_OPT, and for the eigen and inverse methods, each rank runs one half of a global batch of the
batch-first nn.TransformerEncoderLayer of test_gpu_attention.py with `precondition_attention=True`; the losses are
sums, so the summed gradients are those of the whole batch.  Under MEM_OPT the q, k and v rows of one
in_proj_weight.grad have different gradient workers and reach the other rank through the gradient broadcast.  After
every step
  * every rank writes the same gradients, bit for bit;
  * every layer's written gradient (kl-clip off, so P) matches an fp64 restatement on the concatenated batch: the
    factors formed in fp64 from the inputs and output gradients of the twin model (four nn.Linear layers, run in fp64
    on the whole batch), their EMA from the identity, and P from fp64 eigendecompositions or inverses;
  * the run takes exactly the collectives of the twin model's run.
`--backend gloo` runs both ranks on shared GPUs; NCCL needs one GPU per rank.
"""
import argparse
import copy
import os
import sys

import torch
import torch.distributed as dist
from torch import nn
from torch.nn.attention import SDPBackend, sdpa_kernel

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from conftest import rel_fro  # noqa: E402
from kfac_b200.enums import DistributedStrategy  # noqa: E402
from kfac_b200.preconditioner import KFACPreconditioner  # noqa: E402
from test_gpu_attention import Enc, _grads, _twin  # noqa: E402

ALPHA, DAMPING, STEPS, B, L = 0.9, 0.01, 2, 8, 12


def batch(s, dev):
    g = torch.Generator().manual_seed(100 + s)
    return torch.randn(B, L, 64, generator=g).to(dev), torch.randn(B, L, 10, generator=g).to(dev)


def fp64_statistics(twin64, x, y):
    """name -> (A, G) of one window, fp64, from the twin's Linear inputs and output gradients on the whole batch."""
    rows = {}
    hooks = []
    for name, m in twin64.named_modules():
        if isinstance(m, nn.Linear):
            def pre(mod, inp, name=name):
                a = inp[0].detach().reshape(-1, mod.in_features)
                rows[name] = [torch.cat([a, torch.ones(a.shape[0], 1, dtype=a.dtype, device=a.device)], 1)]

            def bwd(mod, gin, gout, name=name):
                rows[name].append(gout[0].detach().reshape(-1, mod.out_features))
            hooks += [m.register_forward_pre_hook(pre), m.register_full_backward_hook(bwd)]
    twin64.zero_grad()
    (twin64(x.double()) - y.double()).pow(2).sum().backward()
    for h in hooks:
        h.remove()
    return {n: (a.T @ a / a.shape[0], g.T @ g / g.shape[0]) for n, (a, g) in rows.items()}


def fp64_precondition(A, G, grad, method):
    if method == 'inverse':
        eye = lambda n: torch.eye(n, dtype=torch.float64, device=grad.device)  # noqa: E731
        return torch.linalg.solve(G + DAMPING * eye(G.shape[0]), grad) @ torch.linalg.inv(A + DAMPING * eye(A.shape[0]))
    da, qa = torch.linalg.eigh(A)
    dg, qg = torch.linalg.eigh(G)
    return qg @ ((qg.T @ grad @ qa) / (dg[:, None] * da[None, :] + DAMPING)) @ qa.T


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

    def run(strategy, method, twin):
        torch.manual_seed(0)
        model = Enc(True).to(dev)
        twin64 = _twin(model).double()
        if twin:
            model = _twin(model)
        pre = KFACPreconditioner(model, kl_clip=None, damping=DAMPING, factor_decay=ALPHA, grad_worker_fraction=strategy,
                                 compute_method=method, precondition_attention=not twin)
        names = [n for n, _ in pre._layers.values()]
        A = {n: torch.eye(pre_l.a_dim, dtype=torch.float64, device=dev) for n, pre_l in pre._layers.values()}
        G = {n: torch.eye(pre_l.g_dim, dtype=torch.float64, device=dev) for n, pre_l in pre._layers.values()}
        for s in range(STEPS):
            x_all, y_all = batch(s, dev)
            half = B // world
            x, y = x_all[rank * half:(rank + 1) * half], y_all[rank * half:(rank + 1) * half]
            model.zero_grad()
            (model(x) - y).pow(2).sum().backward()
            for p in model.parameters():          # data parallelism: sum losses, so the gradients are summed
                dist.all_reduce(p.grad)
            raw = {k: v.double().clone() for k, v in _grads(model).items()}
            pre.step()
            torch.cuda.synchronize()
            if twin:
                continue
            stats = fp64_statistics(twin64, x_all, y_all)
            got = _grads(model)
            for n in names:
                A[n] = ALPHA * A[n] + (1 - ALPHA) * stats[n][0]
                G[n] = ALPHA * G[n] + (1 - ALPHA) * stats[n][1]
                assert all(torch.equal(o, got[n]) for o in gather(got[n])), (strategy, method, s, n)
                err = rel_fro(got[n], fp64_precondition(A[n], G[n], raw[n], method))
                assert err <= 1e-3, (strategy, method, s, n, err)
        calls_made = dict(pre._tdc.calls)
        pre.close()
        dist.barrier()
        return calls_made

    with sdpa_kernel(SDPBackend.MATH):
        for strategy in (DistributedStrategy.COMM_OPT, DistributedStrategy.MEM_OPT):
            for method in ('eigen', 'inverse'):
                on = run(strategy, method, False)
                twin = run(strategy, method, True)
                assert on == twin, (strategy, method, on, twin)
    print(f'rank {rank}: dist_attention ok', flush=True)
    dist.destroy_process_group()


if __name__ == '__main__':
    main()
