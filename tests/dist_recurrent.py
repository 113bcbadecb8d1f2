"""Multi-process preconditioning of recurrent layers (run under torchrun, two ranks).

    torchrun --nnodes=1 --nproc-per-node=2 --master-addr 127.0.0.1 --master-port P tests/dist_recurrent.py [--backend gloo]

For COMM_OPT and MEM_OPT, and for the eigen and inverse methods, each rank runs one half of a global batch of a
2-layer nn.LSTM with `precondition_recurrent=True`; the losses are sums, so the summed gradients are those of the whole
batch.  After every step
  * every rank writes the same gradients, bit for bit;
  * every sub-layer's written gradient (kl-clip off, so P) matches an fp64 restatement on the concatenated batch: the
    factors formed in fp64 from the inputs and output gradients of the unrolled twin (nn.Linear layers, run in fp64 on
    the whole batch), their EMA from the identity, and P from fp64 eigendecompositions or inverses;
  * the run takes exactly the collectives of the twin model's run.
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
from test_gpu_recurrent import Net, UnrolledLSTM  # noqa: E402

ALPHA, DAMPING, STEPS, B, T = 0.9, 0.01, 2, 8, 7
SUBS = ('ih_l0', 'hh_l0', 'ih_l1', 'hh_l1')


def batch(s, dev):
    g = torch.Generator().manual_seed(100 + s)
    return torch.randn(T, B, 24, generator=g).to(dev), torch.randn(T, B, 32, generator=g).to(dev)


def fp64_statistics(twin64, x, y):
    """sub-layer -> (A, G) of one window, fp64, from the twin's Linear inputs and output gradients on the whole batch
    (the hh Linear's rows of all its calls)."""
    rows = {n: ([], []) for n in SUBS}
    hooks = []
    for n in SUBS:
        m = twin64.sublayer(n)

        def pre(mod, inp, n=n):
            a = inp[0].detach().reshape(-1, mod.in_features)
            rows[n][0].append(torch.cat([a, a.new_ones(a.shape[0], 1)], 1))

        def bwd(mod, gin, gout, n=n):
            rows[n][1].append(gout[0].detach().reshape(-1, mod.out_features))
        hooks += [m.register_forward_pre_hook(pre), m.register_full_backward_hook(bwd)]
    twin64.zero_grad()
    (twin64(x.double()) * y.double()).sum().backward()
    for h in hooks:
        h.remove()
    out = {}
    for n, (a, g) in rows.items():
        a, g = torch.cat(a), torch.cat(g)
        out[n] = (a.T @ a / a.shape[0], g.T @ g / g.shape[0])
    return out


def fp64_precondition(A, G, grad, method):
    eye = lambda n: torch.eye(n, dtype=torch.float64, device=grad.device)  # noqa: E731
    if method == 'inverse':
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
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False

    def gather(t):
        t = t.contiguous() if args.backend == 'nccl' else t.detach().cpu().contiguous()
        out = [torch.empty_like(t) for _ in range(world)]
        dist.all_gather(out, t)
        return [o.to(dev) for o in out]

    def run(strategy, method, twin):
        torch.manual_seed(0)
        model = Net('LSTM', bidir=False).to(dev)
        twin64 = UnrolledLSTM(model.rnn).double()
        if twin:
            model = UnrolledLSTM(model.rnn)
        pre = KFACPreconditioner(model, kl_clip=None, damping=DAMPING, factor_decay=ALPHA, grad_worker_fraction=strategy,
                                 compute_method=method, precondition_recurrent=not twin, update_factors_in_hook=False)
        A = {n: torch.eye(twin64.sublayer(n).in_features + 1, dtype=torch.float64, device=dev) for n in SUBS}
        G = {n: torch.eye(twin64.sublayer(n).out_features, dtype=torch.float64, device=dev) for n in SUBS}
        for s in range(STEPS):
            x_all, y_all = batch(s, dev)
            half = B // world
            x, y = x_all[:, rank * half:(rank + 1) * half], y_all[:, rank * half:(rank + 1) * half]
            model.zero_grad()
            (model(x) * y).sum().backward()
            for p in model.parameters():          # data parallelism: sum losses, so the gradients are summed
                dist.all_reduce(p.grad)
            if twin:
                pre.step()
                continue
            raw = {n: torch.cat([getattr(model.rnn, f'weight_{n}').grad, getattr(model.rnn, f'bias_{n}').grad[:, None]],
                                1).double() for n in SUBS}
            pre.step()
            torch.cuda.synchronize()
            stats = fp64_statistics(twin64, x_all, y_all)
            for n in SUBS:
                got = torch.cat([getattr(model.rnn, f'weight_{n}').grad, getattr(model.rnn, f'bias_{n}').grad[:, None]], 1)
                A[n] = ALPHA * A[n] + (1 - ALPHA) * stats[n][0]
                G[n] = ALPHA * G[n] + (1 - ALPHA) * stats[n][1]
                assert all(torch.equal(o, got) for o in gather(got)), (strategy, method, s, n)
                err = rel_fro(got, fp64_precondition(A[n], G[n], raw[n], method))
                assert err <= 1e-3, (strategy, method, s, n, err)
        calls_made = dict(pre._tdc.calls)
        pre.close()
        dist.barrier()
        return calls_made

    for strategy in (DistributedStrategy.COMM_OPT, DistributedStrategy.MEM_OPT):
        for method in ('eigen', 'inverse'):
            on = run(strategy, method, False)
            twin = run(strategy, method, True)
            assert on == twin, (strategy, method, on, twin)
    print(f'rank {rank}: dist_recurrent ok', flush=True)
    dist.destroy_process_group()


if __name__ == '__main__':
    main()
