"""Multi-process diagonal-G preconditioning (run under torchrun, two ranks).

    torchrun --nnodes=1 --nproc-per-node=2 --master-addr 127.0.0.1 --master-port P tests/dist_diag_g.py [--backend gloo]

For COMM_OPT (every rank preconditions every layer) and MEM_OPT (one rank per layer, P broadcast), and for the eigen
and inverse methods, each rank runs one half of a global batch of the LM of test_gpu_diag_g.py with the head in
`diagonal_g_layers`, the gradients are averaged, and after two steps
  * every rank holds the same head factors and writes the same gradients (P, kl-clip off);
  * the head's P matches fp64 on the concatenated batch: diag(G) from the logits gradients of both ranks (averaged
    like the preconditioner averages the statistics), A from the factor the ranks hold;
  * every other layer's P matches fp64 formed from the factors the ranks hold;
  * the run takes exactly the all-reduces of a run with the head skipped, and one broadcast per segment of the
    communication plan.
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
from kfac_b200.distributed import get_world_size  # noqa: E402
from kfac_b200.enums import DistributedStrategy  # noqa: E402
from kfac_b200.preconditioner import KFACPreconditioner  # noqa: E402
from test_gpu_diag_g import LM, V_LM, _batch, _grad_matrix, keep_logits_grad, p_ref  # noqa: E402

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

    def run(strategy, method, check, **kw):
        torch.manual_seed(0)
        model = LM().to(dev)
        pre = KFACPreconditioner(model, kl_clip=None, damping=DAMPING, factor_decay=ALPHA,
                                 grad_worker_fraction=strategy, compute_method=method, **kw)
        layers = {m: l for m, (_, l) in pre._layers.items()}
        seen = {}
        keep_logits_grad(model, seen)
        opt = torch.optim.SGD(model.parameters(), lr=0.05)
        G_ref = None
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
            if not check:
                continue
            gs = [g.double().reshape(-1, V_LM) for g in gather(seen['g'])]
            g_b = sum((g * g).sum(0) / g.shape[0] for g in gs) / world
            G_ref = ALPHA * (torch.ones_like(g_b) if G_ref is None else G_ref) + (1 - ALPHA) * g_b
            lh = layers[model.head]
            assert rel_fro(lh.g_factor, G_ref) < 1e-5, (strategy, method, s)
            for t in (lh.a_factor, lh.g_factor):
                others = gather(t)
                assert all(torch.equal(o, others[0]) for o in others), (strategy, method, s)
            for m, l in layers.items():
                got = _grad_matrix(m)
                others = gather(got)
                assert all(torch.equal(o, others[0]) for o in others), (strategy, method, s, pre._layers[m][0])
                ref = p_ref(l, method, grads[m], l.a_factor, G_ref if l.diag_g else l.g_factor, DAMPING)
                err = rel_fro(got, ref)
                assert err < 1e-3, (strategy, method, s, pre._layers[m][0], err)
            opt.step()
        calls = dict(pre._tdc.calls)

        def sent(segs):      # a broadcast in a group of one is skipped
            return sum(get_world_size(seg.group) > 1 for seg in segs) * STEPS
        want_b = sent(pre._inv_segments) if pre._assignment.broadcast_inverses() else 0
        if pre._assignment.broadcast_gradients() and pre._peer_p_bases is None:
            want_b += sent(pre._grad_segments)
        assert calls['broadcast'] == want_b, (strategy, method, calls, want_b)
        pre.close()
        dist.barrier()
        return calls

    for strategy in (DistributedStrategy.COMM_OPT, DistributedStrategy.MEM_OPT):
        for method in ('eigen', 'inverse'):
            diag = run(strategy, method, True, diagonal_g_layers=['head'])
            skip = run(strategy, method, False, skip_layers=['head'])
            assert diag['allreduce'] == skip['allreduce'], (strategy, method, diag, skip)
    print(f'rank {rank}: dist_diag_g ok', flush=True)
    dist.destroy_process_group()


if __name__ == '__main__':
    main()
