"""CPU tests of the host side: C-ABI export table, constructor validation
(kfac/preconditioner.py:155-211, tests/preconditioner_test.py of the
reference), comm-plan consistency across ranks, and a world_size-2 gloo run of
the arena communicator."""
import ctypes
import os
import re

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from conftest import ROOT


def test_cabi_exports_every_header_symbol():
    from kfac_b200 import _cabi
    lib = _cabi.load()
    header = open(os.path.join(ROOT, 'include', 'kfac_b200.h')).read()
    declared = set(re.findall(r'\b(kfac_[a-z0-9_]+)\s*\(', header))
    assert declared, 'no declarations parsed'
    for name in declared:
        assert hasattr(lib, name), f'{name} declared in kfac_b200.h but not exported'
        assert name in _cabi.SIGNATURES, f'{name} has no ctypes prototype'
    assert lib.kfac_version() >= 100
    assert isinstance(lib.kfac_last_error(), bytes)


def test_no_cpu_fallback():
    from kfac_b200 import _cabi
    from kfac_b200.preconditioner import KFACPreconditioner
    from oracle.models import TinyModel
    m = TinyModel()
    p = KFACPreconditioner(m)
    if torch.cuda.is_available():
        pytest.skip('CPU-only check')
    with pytest.raises(_cabi.KFACNativeError):
        m(torch.rand(2, 10)).sum().backward()
    with pytest.raises(_cabi.KFACNativeError):
        p.step()


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, 'kfac-pytorch_b200')
    for fn in os.listdir(pkg):
        if fn.endswith('.py'):
            src = open(os.path.join(pkg, fn)).read()
            assert 'oracle' not in src.replace('no CPU / PyTorch fallback', ''), fn


def test_constructor_validation():
    from kfac_b200.enums import AssignmentStrategy, ComputeMethod, DistributedStrategy
    from kfac_b200.preconditioner import KFACPreconditioner
    from oracle.models import TinyModel
    K = KFACPreconditioner
    with pytest.raises(ValueError):
        K(TinyModel(), allreduce_bucket_cap_mb=-1)
    with pytest.raises(ValueError):
        K(TinyModel(), compute_eigenvalue_outer_product=True, colocate_factors=False)
    with pytest.raises(ValueError):
        K(TinyModel(), grad_worker_fraction=2)
    with pytest.raises(ValueError):
        K(TinyModel(), grad_worker_fraction=-1)
    for kw in (dict(factor_update_steps=0), dict(inv_update_steps=0), dict(damping=0.0),
               dict(factor_decay=0.0), dict(factor_decay=1.5), dict(kl_clip=0.0), dict(lr=-1.0),
               dict(accumulation_steps=0)):
        with pytest.raises(ValueError):
            K(TinyModel(), **kw)
    with pytest.warns(UserWarning):
        K(TinyModel(), factor_update_steps=3, inv_update_steps=4)
    with pytest.warns(UserWarning):   # MEM_OPT forces colocate_factors
        p = K(TinyModel(), grad_worker_fraction=DistributedStrategy.MEM_OPT, colocate_factors=False,
              compute_eigenvalue_outer_product=False)
    assert p.colocate_factors
    p = K(TinyModel(), assignment_strategy='memory', compute_method='inverse')
    assert p.assignment_strategy == AssignmentStrategy.MEMORY and p.compute_method == ComputeMethod.INVERSE
    assert K(TinyModel(), grad_worker_fraction=1).distributed_strategy == DistributedStrategy.COMM_OPT
    # world size 1: fraction 0 -> 1/1 == 1 -> COMM_OPT, exactly like the reference (preconditioner.py:186-197)
    assert K(TinyModel(), grad_worker_fraction=0).distributed_strategy == DistributedStrategy.COMM_OPT
    p = K(TinyModel(), damping=lambda s: 0.1 * (s + 1), lr=lambda s: 0.5)
    assert p.damping == pytest.approx(0.1) and p.lr == 0.5
    assert 'damping' not in p.state_dict(include_factors=False)
    r = repr(K(TinyModel(), skip_layers=['linear1']))
    assert 'layers=1' in r and 'KAISAAssignment' in r
    assert len(K(TinyModel(), skip_layers=['Linear'])._layers) == 0


def _plans(world, frac, method, prediv, colocate=True):
    """Build the comm plan of every rank without any process group."""
    from kfac_b200.assignment import KAISAAssignment
    from kfac_b200.base_preconditioner import build_comm_plan
    from kfac_b200.enums import ComputeMethod
    from kfac_b200.layers import register_modules
    from oracle.models import SmallConvNet
    torch.manual_seed(0)
    model = SmallConvNet()
    out = []
    handles = {}
    for rank in range(world):
        layers = register_modules(model, [], method=method, prediv_eigenvalues=prediv)
        ll = list(layers.values())
        work = {n: {'A': l.a_dim ** 3, 'G': l.g_dim ** 3} for n, l in ll}
        a = KAISAAssignment(work, local_rank=rank, world_size=world, grad_worker_fraction=frac,
                            group_func=lambda r: handles.setdefault(tuple(sorted(r)), tuple(sorted(r))),
                            colocate_factors=colocate)
        out.append((a, build_comm_plan(ll, a)))
    return out


@pytest.mark.parametrize('world,frac', [(1, 1.0), (2, 1.0), (2, 0.5), (4, 1.0), (4, 0.5), (4, 0.25), (8, 1.0), (8, 0.5), (8, 0.125)])
@pytest.mark.parametrize('method,prediv,colocate', [('EIGEN', True, True), ('EIGEN', False, False), ('INVERSE', False, True)])
def test_comm_plan_consistent_across_ranks(world, frac, method, prediv, colocate):
    from kfac_b200.enums import ComputeMethod
    if colocate is False and frac * world <= 1:
        colocate = True
    plans = _plans(world, frac, ComputeMethod[method], prediv, colocate)
    # every broadcast (group, src) must look identical on every member, in the same order
    for kind in (0, 1):
        per_rank = []
        for rank, (a, plan) in enumerate(plans):
            segs = plan[kind]
            per_rank.append([(s.group, s.src, s.numel, [(l.index, k, sh) for l, k, sh in s.entries]) for s in segs])
        for rank, segs in enumerate(per_rank):
            for grp, src, numel, entries in segs:
                assert rank in grp and src in grp
                for other in grp:
                    theirs = [s for s in per_rank[other] if s[0] == grp]
                    mine = [s for s in per_rank[rank] if s[0] == grp]
                    assert theirs == mine, (kind, rank, other)
    # every layer's P is owned by exactly one segment on each rank
    for a, (inv, grad) in plans:
        seen = sorted(l.index for s in grad for l, _, _ in s.entries)
        assert seen == list(range(len(a.get_layers())))


def _gloo_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        from kfac_b200.distributed import ArenaCommunicator
        from kfac_b200.enums import DistributedStrategy
        from kfac_b200.preconditioner import KFACPreconditioner
        from oracle.models import TinyModel
        tdc = ArenaCommunicator()
        arena = torch.full((1000,), float(rank + 1))
        tdc.allreduce_average(arena)
        assert torch.allclose(arena, torch.full((1000,), (1 + world) / 2 * 1.0))
        seg = torch.full((10,), float(rank))
        tdc.broadcast(seg, src=1)
        assert torch.equal(seg, torch.ones(10))
        # constructor builds the KAISA groups collectively on every rank
        for strat in (DistributedStrategy.COMM_OPT, DistributedStrategy.MEM_OPT):
            p = KFACPreconditioner(TinyModel(), grad_worker_fraction=strat)
            a = p._assignment
            assert a.world_size == world and a.local_rank == rank
            names = a.get_layers()
            workers = [a.inv_worker(n, 'A') for n in names]
            gathered = [None] * world
            dist.all_gather_object(gathered, workers)
            assert all(g == gathered[0] for g in gathered)
            # broadcast an arena slice inside a real KAISA group
            grp = a.grad_receiver_group(names[0])
            t = torch.full((4,), float(rank))
            tdc.broadcast(t, src=a.src_grad_worker(names[0]), group=grp)
            assert float(t[0]) == float(a.src_grad_worker(names[0]))
        with pytest.raises(ValueError):
            KFACPreconditioner(TinyModel(), grad_worker_fraction=0.75)
        dist.barrier()
        q.put((rank, 'ok'))
    except BaseException as e:  # noqa: BLE001
        q.put((rank, repr(e)))
    finally:
        dist.destroy_process_group()


def test_gloo_world2():
    import socket
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert sorted(res) == [(0, 'ok'), (1, 'ok')], res


def test_arena_entries_are_16_byte_aligned():
    """Every second-order arena entry must start on a multiple of 4 floats: a vector entry of odd
    length in front of a matrix would break the TMA alignment of everything behind it."""
    from kfac_b200.base_preconditioner import _storage_numel
    from kfac_b200.enums import ComputeMethod
    for method, prediv in ((ComputeMethod.EIGEN, True), (ComputeMethod.EIGEN, False), (ComputeMethod.INVERSE, False)):
        for a, (inv, grad) in _plans(2, 1.0, method, prediv, True):
            for segs in (inv, grad):
                for s in segs:
                    assert s.offset % 4 == 0 and s.numel % 4 == 0
                    off = s.offset
                    for _, _, shape in s.entries:
                        assert off % 4 == 0, (method, shape)
                        off += _storage_numel(shape)
    assert _storage_numel((147,)) == 148 and _storage_numel((10, 21)) == 10 * 24


def test_bench_reference_arm_contract():
    """`bench.py --impl reference` (the CPU arm run beside the GPU arm) prints ONE JSON
    line with the contract keys; exercised on the small workload so it stays in the CPU budget."""
    import json
    import subprocess
    import sys
    out = subprocess.run([sys.executable, os.path.join(ROOT, 'bench.py'), '--impl', 'reference', '--model', 'resnet32',
                          '--steps', '1', '--warmup', '0', '--budget-s', '120'],
                         capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [l for l in out.stdout.splitlines() if l.startswith('{')]
    assert len(lines) == 1, out.stdout[-1000:]
    d = json.loads(lines[0])
    for key in ('impl', 'metric', 'value', 'unit', 'n_gpus', 'steps', 'warmup', 'ms_per_step', 'higher_is_better',
                'scaling', 'vs_baseline', 'dtype', 'data', 'config', 'cpu_baseline', 'e2e'):
        assert key in d, key
    assert d['impl'] == 'reference' and d['unit'] == 'images/s' and d['value'] > 0
    # 'reference' when oracle/_ref (the unmodified reference installed by oracle/build_ref.sh) is present
    want = 'reference' if os.path.isdir(os.path.join(ROOT, 'oracle', '_ref', 'kfac')) else 'port'
    assert d['cpu_baseline']['kind'] == want and d['cpu_baseline']['cores'] >= 1
    assert d['e2e']['h2d_bytes_per_step'] == 0 and d['e2e']['d2h_bytes_per_step'] == 0
    assert d['config']['global_batch'] == 128


def test_bench_cpu_arm_other_ranks_exit_quietly():
    """Under torchrun only rank 0 runs the CPU arm; the other ranks print nothing and exit 0."""
    import subprocess
    import sys
    env = dict(os.environ, RANK='1', WORLD_SIZE='2', LOCAL_RANK='1')
    out = subprocess.run([sys.executable, os.path.join(ROOT, 'bench.py'), '--impl', 'reference', '--gpus', '2'],
                         capture_output=True, text=True, timeout=300, env=env)
    assert out.returncode == 0 and out.stdout.strip() == '', (out.stdout[-500:], out.stderr[-500:])


def test_sytrd_schedule_covers_all_and_cannot_deadlock():
    """The tridiagonalisation kernel is ONE cooperative launch in which every CTA walks the job list front to back
    and spins at group barriers: the host-side schedule must (i) place every matrix exactly once on a CTA range inside
    the grid, at least as wide as the kernel's tile lists need, and (ii) order the jobs so that the walk always makes
    progress.  Checked by simulating the walk (host-only entry of the library, no GPU)."""
    from kfac_b200 import _cabi
    lib = _cabi.load()
    lib.kfac_stage_schedule.restype = ctypes.c_int
    lib.kfac_stage_sytrd_min_ctas.restype = ctypes.c_int
    r50 = [(147, 64, 1), (64, 64, 1), (64, 256, 4), (256, 64, 2), (576, 64, 3), (128, 512, 4), (256, 128, 1),
           (256, 512, 1), (512, 128, 3), (1152, 128, 4), (256, 1024, 6), (512, 256, 1), (512, 1024, 1), (1024, 256, 5),
           (2304, 256, 6), (512, 2048, 3), (1024, 512, 1), (1024, 2048, 1), (2048, 512, 2), (4608, 512, 3), (2049, 1000, 1)]
    cases = [[d for a, g, c in r50 for d in [a, g] * c if d > 128], [4608], [8192, 130], [300] * 200, [2304, 2304, 129]]
    for dims in cases:
        for grid in (148, 132, 16):
            count = len(dims)
            n = (ctypes.c_int * count)(*dims)
            mat, cta0, ncta = ((ctypes.c_int * count)() for _ in range(3))
            jobs = lib.kfac_stage_schedule(n, count, grid, mat, cta0, ncta)
            assert jobs == count
            assert sorted(mat[i] for i in range(jobs)) == list(range(count))
            queues = [[] for _ in range(grid)]
            for j in range(jobs):
                need = min(grid, lib.kfac_stage_sytrd_min_ctas(dims[mat[j]]))
                assert 0 <= cta0[j] and cta0[j] + ncta[j] <= grid and ncta[j] >= need, (dims[mat[j]], cta0[j], ncta[j])
                for c in range(cta0[j], cta0[j] + ncta[j]):
                    queues[c].append(j)
            # a job runs when it is at the head of the queue of every CTA of its group
            head = [0] * grid
            done = 0
            progress = True
            while progress:
                progress = False
                for j in range(jobs):
                    cs = range(cta0[j], cta0[j] + ncta[j])
                    if all(head[c] < len(queues[c]) and queues[c][head[c]] == j for c in cs):
                        for c in cs:
                            head[c] += 1
                        done += 1
                        progress = True
            assert done == jobs, f'schedule deadlocks: {done} of {jobs} jobs can run (grid {grid})'


def test_linear_factor_workspace_of_zero_rows():
    """A Linear layer called on an empty batch: its factor call asks for the workspace of zero rows, which needs none
    (the split plan of an empty reduction is one split; host-only entries of the library, no GPU)."""
    from kfac_b200 import _cabi
    lib = _cabi.load()
    for feat, ones in ((64, 1), (1024, 0), (2048, 1)):
        assert lib.kfac_factor_linear_workspace_bytes(0, feat, ones) == 0
        assert lib.kfac_factor_linear_strided_workspace_bytes(0, feat, feat + 3, ones) == 0
    assert lib.kfac_factor_linear_workspace_bytes(2048, 1024, 1) > 0
