// Shared helpers for the K-FAC kernels.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/kfac_b200.h"

namespace kfac {

void set_error(const char* fmt, ...);
void count_launch(int n);

#define KFAC_CHECK_ARG(cond, msg)                         \
  do {                                                    \
    if (!(cond)) {                                        \
      ::kfac::set_error("bad argument: %s (%s)", msg, #cond); \
      return KFAC_ERR_BAD_ARG;                            \
    }                                                     \
  } while (0)

#define KFAC_CUDA(call)                                                        \
  do {                                                                         \
    cudaError_t e__ = (call);                                                  \
    if (e__ != cudaSuccess) {                                                  \
      ::kfac::set_error("CUDA error %s at %s:%d", cudaGetErrorString(e__),     \
                        __FILE__, __LINE__);                                   \
      return KFAC_ERR_CUDA;                                                    \
    }                                                                          \
  } while (0)

#define KFAC_LAUNCH_CHECK()            \
  do {                                 \
    ::kfac::count_launch(1);           \
    KFAC_CUDA(cudaGetLastError());     \
  } while (0)

inline int ceil_div(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }
inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

template <typename T>
__device__ __forceinline__ float to_float(T v);
template <>
__device__ __forceinline__ float to_float<float>(float v) { return v; }
template <>
__device__ __forceinline__ float to_float<__half>(__half v) { return __half2float(v); }
template <>
__device__ __forceinline__ float to_float<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }

template <typename T>
__device__ __forceinline__ T from_float(float v);
template <>
__device__ __forceinline__ float from_float<float>(float v) { return v; }
template <>
__device__ __forceinline__ __half from_float<__half>(float v) { return __float2half(v); }
template <>
__device__ __forceinline__ __nv_bfloat16 from_float<__nv_bfloat16>(float v) { return __float2bfloat16(v); }

__device__ __forceinline__ float load_as_float(const void* p, int dtype, int64_t i) {
  if (dtype == KFAC_F32) return ((const float*)p)[i];
  if (dtype == KFAC_F16) return __half2float(((const __half*)p)[i]);
  return __bfloat162float(((const __nv_bfloat16*)p)[i]);
}
__device__ __forceinline__ void store_from_float(void* p, int dtype, int64_t i, float v) {
  if (dtype == KFAC_F32) ((float*)p)[i] = v;
  else if (dtype == KFAC_F16) ((__half*)p)[i] = __float2half(v);
  else ((__nv_bfloat16*)p)[i] = __float2bfloat16(v);
}

// ---------------------------------------------------------------- SIMT GEMM
enum GemmEpilogue { EPI_NONE = 0, EPI_MUL = 1, EPI_DIV_OUTER = 2 };

struct GemmArgs {
  const float* A; int64_t sa_m, sa_k, sa_b;   // A(m,k) = A[b*sa_b + m*sa_m + k*sa_k]
  const float* B; int64_t sb_k, sb_n, sb_b;
  float* C; int64_t ldc, sc_b;                // C(m,n) = C[b*sc_b + m*ldc + n]
  int M, N, K;
  int batch;        // number of batch entries
  int splitk;       // K split count (>=1)
  int atomic;       // 1: atomicAdd(alpha*acc) into C (used for split-K / batch-reduce)
  float alpha, beta;
  int epi;
  const float* E; int64_t lde;   // EPI_MUL: C *= E[m*lde+n]
  const float* dg; const float* da; float damping;  // EPI_DIV_OUTER
};

int launch_gemm(const GemmArgs& g, cudaStream_t stream);

// wgmma engine (gemm_tc.cu); returns KFAC_ERR_UNSUPPORTED when the shape /
// alignment is outside what the tensor-core kernel handles.
struct TcGemmArgs {
  const float* A; int64_t lda;     // M x K row-major (K-major operand), lda % 4 == 0
  const float* B; int64_t ldb;     // N x K row-major
  float* D; int64_t ldd;           // M x N row-major
  int M, N, K;
  int kbatch;                      // reduction batches: D = sum_b A_b B_b^T
  int64_t a_kb_stride, b_kb_stride;
  int upper_only;                  // SYRK: compute tiles tn >= tm, mirror the rest
  int atomic;                      // epilogue accumulates with atomicAdd (split-K)
  int accumulate;                  // D += alpha * A B^T with a plain read-modify-write (no split-K)
  float* slab; int64_t slab_stride; // deterministic split-K: split sp stores its partial tile to slab + sp * slab_stride (ld = ldd)
  int splits;                      // <= 0: automatic
  float alpha;
  int epi; const float* E; int64_t lde; const float* dg; const float* da; float damping;
  float* peerD[7]; int npeer;      // fused broadcast: the epilogue also stores the tile into these peer copies of D
};
bool tc_gemm_supported(const TcGemmArgs& a);
// the split count launch_tc_gemm runs for a request of `splits` over kb_total k-blocks (every split non-empty)
inline int tc_normalize_splits(int splits, int kb_total) {
  splits = splits < 1 ? 1 : (splits > kb_total ? kb_total : splits);
  const int per = (kb_total + splits - 1) / splits;
  return (kb_total + per - 1) / per;
}
int launch_tc_gemm(const TcGemmArgs& a, cudaStream_t stream);
int tc_num_sms();

}  // namespace kfac
