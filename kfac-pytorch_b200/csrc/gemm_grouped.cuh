// Grouped wgmma GEMM (gemm_grouped.cu): one launch for a list of independent D_i = epi_i(alpha_i A_i B_i^T).
#pragma once
#include "common.cuh"

namespace kfac {

struct GroupedGemm {
  const float* A; int64_t lda;     // M x K row-major
  const float* B; int64_t ldb;     // N x K row-major
  float* D; int64_t ldd;           // M x N row-major
  int M, N, K;
  float alpha;
  int epi; const float* E; int64_t lde; const float* dg; const float* da; float damping;   // GemmEpilogue
  float* peerD[7]; int npeer;      // fused broadcast: tiles are also stored into these peer copies of D
  int splits;                      // > 1: split-K -- deterministic through `slab` (plain epilogue, no peers), or mode 2
  float* slab; int64_t slab_stride;
  int mode;                        // 0: D = ..., 1: D += ... (read-modify-write, splits == 1), 2: atomicAdd into D (caller zeroes D)
  const int* krange;               // optional (mode 2 only): DEVICE pointer to {first, end} k-block (32 columns of K) the product
                                   // runs over, read by the kernel -- for reductions whose extent is only known on the device
};

size_t grouped_gemm_ws_bytes(int count);
bool grouped_gemm_tc_ok(const GroupedGemm& g);
// problems the tensor-core kernel cannot take (tiny / unaligned) run as individual SIMT launches
int launch_grouped_gemm(const GroupedGemm* probs, int count, void* ws, size_t ws_bytes, cudaStream_t s);

}  // namespace kfac
