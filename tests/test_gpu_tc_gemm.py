"""wgmma GEMM engine (3xTF32 split, TMA-fed, register accumulators) vs fp64."""
import pytest
import torch

from conftest import rel_fro

pytestmark = pytest.mark.gpu


def S():
    return torch.cuda.current_stream().cuda_stream


@pytest.fixture(scope='module')
def lib():
    from kfac_b200 import _cabi
    return _cabi.load()


@pytest.mark.parametrize('M,N,K', [(128, 128, 32), (128, 128, 256), (256, 384, 512), (100, 130, 260),
                                   (64, 576, 576), (577, 64, 64), (1000, 2048, 2048), (4608, 512, 4608),
                                   (1, 1, 4), (300, 300, 36)])
def test_tc_gemm_matches_fp64(lib, M, N, K):
    dev = torch.device('cuda:0')
    torch.manual_seed(M + N + K)
    lda = (K + 3) // 4 * 4
    A = torch.zeros(M, lda, device=dev)
    B = torch.zeros(N, lda, device=dev)
    A[:, :K] = torch.randn(M, K, device=dev) * torch.logspace(0, -3, K, device=dev)
    B[:, :K] = torch.randn(N, K, device=dev)
    D = torch.full((M, N), float('nan'), device=dev)
    rc = lib.kfac_gemm_tn_tc(A.data_ptr(), lda, B.data_ptr(), lda, D.data_ptr(), N, M, N, K, 0.5, 0, 1, S())
    assert rc == 0, lib.kfac_last_error()
    torch.cuda.synchronize()
    ref = 0.5 * (A[:, :K].double() @ B[:, :K].double().t())
    e = rel_fro(D, ref)
    # single-pass TF32 gives ~5e-4 here; the 3-term split is fp32-class.  The tensor-core
    # accumulator may truncate (one add per k-step of 8): allow ~4e-9 * K.
    assert e < 3e-6 + 4e-9 * K, (M, N, K, e)
    e_max = ((D.double() - ref).abs().max() / ref.abs().max()).item()
    assert e_max < 2e-5 + 1e-8 * K, e_max


def test_tc_gemm_splitk_atomic_accumulates(lib):
    dev = torch.device('cuda:0')
    torch.manual_seed(0)
    M, N, K = 256, 128, 8192
    A = torch.randn(M, K, device=dev)
    B = torch.randn(N, K, device=dev)
    D = torch.ones(M, N, device=dev)
    rc = lib.kfac_gemm_tn_tc(A.data_ptr(), K, B.data_ptr(), K, D.data_ptr(), N, M, N, K, 1.0, 1, 0, S())
    assert rc == 0, lib.kfac_last_error()
    torch.cuda.synchronize()
    ref = 1.0 + A.double() @ B.double().t()
    assert rel_fro(D, ref) < 4e-6


def test_tc_gemm_rejects_misaligned(lib):
    dev = torch.device('cuda:0')
    A = torch.randn(64, 33, device=dev)
    D = torch.empty(64, 64, device=dev)
    from kfac_b200 import _cabi
    rc = lib.kfac_gemm_tn_tc(A.data_ptr(), 33, A.data_ptr(), 33, D.data_ptr(), 64, 64, 64, 33, 1.0, 0, 1, S())
    assert rc == _cabi.KFAC_ERR_UNSUPPORTED
