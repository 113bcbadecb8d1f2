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
  const float* pi; int pi_side_m, pi_side_n;                                                 // EPI_DIV_FACTORED
  float* peerD[7]; int npeer;      // fused broadcast (mode 0, npeer <= 7): D is also stored into these peer copies, by
                                   // the tile epilogue, or by the reduce pass of a slab split (the same bits as D)
  int splits;                      // > 1: split-K -- deterministic through `slab` (plain epilogue), or mode 2
  float* slab; int64_t slab_stride;
  int mode;                        // 0: D = ..., 1: D += ... (read-modify-write, splits == 1), 2: atomicAdd into D (caller zeroes D)
  const int* krange;               // optional (mode 2 only): DEVICE pointer to {first, end} k-block (32 columns of K) the product
                                   // runs over, read by the kernel -- for reductions whose extent is only known on the device
};

size_t grouped_gemm_ws_bytes(int count);
bool grouped_gemm_tc_ok(const GroupedGemm& g);
// problems the tensor-core kernel cannot take (tiny / unaligned) run as individual SIMT launches.
// max_ctas > 0 caps the grid of the tensor-core and reduce launches (default: one CTA per SM).  Work items are dealt
// statically over the grid, so a launch that shares the GPU with a long-running kernel is capped at the SMs it can
// get: CTAs that wait for an SM would hold back the whole launch.  The results do not depend on the grid.
// stage: if given, the problem tables are sent through it (HostStage, common.cuh)
int launch_grouped_gemm(const GroupedGemm* probs, int count, void* ws, size_t ws_bytes, cudaStream_t s, int max_ctas = 0,
                        HostStage* stage = nullptr);

}  // namespace kfac
