"""Diagnostic: tridiagonalisation time over (n, CTA group size), the data the schedule model of eigh_direct.cu is fitted to.
python tests/sytrd_sweep.py > sytrd_sweep.csv"""
import ctypes as C
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from kfac_b200 import _cabi  # noqa: E402

lib = _cabi.load()
lib.kfac_stage_sytrd.restype = C.c_int
lib.kfac_stage_sytrd.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                        C.c_void_p, C.c_size_t, C.c_int, C.c_void_p]
lib.kfac_stage_direct_workspace_bytes.restype = C.c_size_t
lib.kfac_stage_direct_workspace_bytes.argtypes = [C.c_int]
dev = torch.device('cuda:0')
print('n,ncta,ms')
for n in (256, 512, 576, 1024, 1152, 2048, 2304, 4608):
    torch.manual_seed(0)
    A = torch.randn(n, n, device=dev)
    F = ((A + A.t()) / 2).contiguous()
    d, e, tau = torch.zeros(n, device=dev), torch.zeros(n, device=dev), torch.zeros(n, device=dev)
    need = lib.kfac_stage_direct_workspace_bytes(n)
    ws = torch.empty(need, dtype=torch.uint8, device=dev)
    for ncta in (1, 2, 3, 4, 6, 8, 12, 16, 24, 36, 48, 72, 100, 132):
        best = 1e9
        ok = True
        for it in range(3):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            rc = lib.kfac_stage_sytrd(F.data_ptr(), n, d.data_ptr(), e.data_ptr(), None, n, tau.data_ptr(), ws.data_ptr(),
                                             need, ncta, torch.cuda.current_stream().cuda_stream)
            e1.record()
            torch.cuda.synchronize()
            if rc != 0:
                ok = False
                break
            if it:
                best = min(best, e0.elapsed_time(e1))
        if ok:
            print(f'{n},{ncta},{best:.3f}', flush=True)
