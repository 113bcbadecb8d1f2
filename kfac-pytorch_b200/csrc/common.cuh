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
// The number of chains a tensor-core reduction of length K runs in: above 1024, chains of at most 512.  The engine's
// accumulator truncates, and short chains keep the 3xTF32 result at fp32 accuracy.
inline int chain_splits(int64_t K) { return K > 1024 ? ceil_div(K, 512) : 1; }

// A kfac_conv_geometry flattened for the kernels, with its output extents.  Only the padding before an axis enters the
// input index; the padding after it only extends the output.
struct ConvGeo {
  int batch, C, D, H, W, kd, kh, kw, sd, sh, sw, dd, dh, dw, pd, ph, pw, Do, Ho, Wo;
  __host__ __device__ int64_t spatial() const { return (int64_t)Do * Ho * Wo; }
  __host__ __device__ int64_t features() const { return (int64_t)C * kd * kh * kw; }
};

// Conv2d's geometry: depth 1, dilation 1, symmetric padding
inline ConvGeo conv2d_geo(int batch, int C, int H, int W, int kh, int kw, int sh, int sw, int ph, int pw) {
  return ConvGeo{batch, C, 1, H, W, 1, kh, kw, 1, sh, sw, 1, 1, 1, 0, ph, pw,
                 1, (H + 2 * ph - kh) / sh + 1, (W + 2 * pw - kw) / sw + 1};
}

// KFAC_OK with *o filled, or KFAC_ERR_BAD_ARG for a malformed geometry or an empty output
inline int resolve_conv_geometry(const kfac_conv_geometry* g, ConvGeo* o) {
  KFAC_CHECK_ARG(g != nullptr, "null geometry");
  KFAC_CHECK_ARG(g->batch > 0 && g->C > 0, "geometry");
  int out[3];
  for (int a = 0; a < 3; ++a) {
    KFAC_CHECK_ARG(g->in[a] > 0 && g->kernel[a] > 0 && g->stride[a] > 0 && g->dilation[a] > 0 &&
                       g->pad_before[a] >= 0 && g->pad_after[a] >= 0, "geometry");
    const int64_t span = (int64_t)g->in[a] + g->pad_before[a] + g->pad_after[a] - (int64_t)g->dilation[a] * (g->kernel[a] - 1) - 1;
    KFAC_CHECK_ARG(span >= 0 && span / g->stride[a] + 1 < (1ll << 31), "empty output");
    out[a] = (int)(span / g->stride[a] + 1);
  }
  *o = ConvGeo{g->batch, g->C, g->in[0], g->in[1], g->in[2], g->kernel[0], g->kernel[1], g->kernel[2],
               g->stride[0], g->stride[1], g->stride[2], g->dilation[0], g->dilation[1], g->dilation[2],
               g->pad_before[0], g->pad_before[1], g->pad_before[2], out[0], out[1], out[2]};
  return KFAC_OK;
}

// A kfac_conv_transpose_geometry as a ConvGeo: (D, H, W) the input extents, (pd, ph, pw) torch's padding, (Do, Ho, Wo)
// the output extents (in - 1) s - 2 p + d (k - 1) + op + 1.  KFAC_ERR_BAD_ARG for a malformed geometry, an empty
// output, an output padding of at least max(s, d) (torch refuses it) or batch x output positions of 2^31 or more.
inline int resolve_conv_transpose_geometry(const kfac_conv_transpose_geometry* g, ConvGeo* o) {
  KFAC_CHECK_ARG(g != nullptr, "null geometry");
  KFAC_CHECK_ARG(g->batch > 0 && g->C > 0, "geometry");
  int out[3];
  int64_t rows = g->batch;
  for (int a = 0; a < 3; ++a) {
    KFAC_CHECK_ARG(g->in[a] > 0 && g->kernel[a] > 0 && g->stride[a] > 0 && g->dilation[a] > 0 && g->padding[a] >= 0 &&
                       g->output_padding[a] >= 0, "geometry");
    KFAC_CHECK_ARG(g->output_padding[a] < (g->stride[a] > g->dilation[a] ? g->stride[a] : g->dilation[a]),
                   "output padding of at least max(stride, dilation)");
    const int64_t n = ((int64_t)g->in[a] - 1) * g->stride[a] - 2 * (int64_t)g->padding[a] +
                      (int64_t)g->dilation[a] * (g->kernel[a] - 1) + g->output_padding[a] + 1;
    KFAC_CHECK_ARG(n > 0, "empty output");
    rows *= n;
    KFAC_CHECK_ARG(rows < (1ll << 31), "rows overflow");
    out[a] = (int)n;
  }
  *o = ConvGeo{g->batch, g->C, g->in[0], g->in[1], g->in[2], g->kernel[0], g->kernel[1], g->kernel[2],
               g->stride[0], g->stride[1], g->stride[2], g->dilation[0], g->dilation[1], g->dilation[2],
               g->padding[0], g->padding[1], g->padding[2], out[0], out[1], out[2]};
  return KFAC_OK;
}

// The tap -> input index map of one axis (stride s, dilation d, padding p; L inputs, n_out outputs).  A convolution
// gathers: output o reads input o s + k d - p through tap k.  A transposed convolution scatters: input i feeds output
// i s - p + k d, so output o reads input (o + p - k d) / s when s divides it.  Both read a tap's inputs in the order of
// their outputs.  The kernels take it as a template parameter; the direct instantiations give the results they gave.
template <bool TRANSPOSED>
struct TapMap;

template <>
struct TapMap<false> {
  // the input that output o reads through tap k, or -1 in the padding
  __device__ __forceinline__ static int input(int o, int k, int s, int d, int p, int L) {
    const int i = o * s + k * d - p;
    return i >= 0 && i < L ? i : -1;
  }
  // input q is read through tap k by an output in [0, n_out)
  __device__ __forceinline__ static bool feeds(int q, int k, int s, int d, int p, int n_out) {
    const int t = q + p - k * d;
    return t >= 0 && t % s == 0 && t / s < n_out;
  }
  // the inputs read through tap k, in output order: first + m step for m in [0, count)
  __device__ __forceinline__ static void span(int L, int k, int s, int d, int p, int n_out, int& first, int& step,
                                              int& count) {
    const int off = k * d - p;   // input of output 0
    const int lo = off < 0 ? (-off + s - 1) / s : 0;
    const int hi = L - 1 - off < 0 ? -1 : min(n_out - 1, (L - 1 - off) / s);
    first = off + lo * s;
    step = s;
    count = hi >= lo ? hi - lo + 1 : 0;
  }
};

template <>
struct TapMap<true> {
  __device__ __forceinline__ static int input(int o, int k, int s, int d, int p, int L) {
    const int t = o + p - k * d;
    if (t < 0) return -1;
    const int i = (int)((unsigned)t / (unsigned)s);
    return i * s == t && i < L ? i : -1;
  }
  __device__ __forceinline__ static bool feeds(int q, int k, int s, int d, int p, int n_out) {
    const int o = q * s - p + k * d;
    return o >= 0 && o < n_out;
  }
  // the box of inputs i in [0, L) whose output i s - p + k d lies in [0, n_out), step 1
  __device__ __forceinline__ static void span(int L, int k, int s, int d, int p, int n_out, int& first, int& step,
                                              int& count) {
    const int off = k * d - p;   // output of input 0
    const int lo = off < 0 ? (-off + s - 1) / s : 0;
    const int hi = n_out - 1 - off < 0 ? -1 : min(L - 1, (n_out - 1 - off) / s);
    first = lo;
    step = 1;
    count = hi >= lo ? hi - lo + 1 : 0;
  }
};

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
// EPI_SQUARE: store x^2.  EPI_DIV_FACTORED: x / ((dg[m] + gamma_m) (da[n] + gamma_n)), the factored (pi-adjusted)
// Tikhonov damping, with damping = s and gamma_m = pi_gamma(s, *pi, pi_side_m), gamma_n likewise
enum GemmEpilogue { EPI_NONE = 0, EPI_MUL = 1, EPI_DIV_OUTER = 2, EPI_SQUARE = 3, EPI_DIV_FACTORED = 4 };

// The damping of one Kronecker factor under pi-adjusted damping: side +1 (the A factor) s * pi, side -1 (the G
// factor) s / pi, side 0 (no factor: a vector of ones) 0.  Rounded on its own (never fused into the add that follows),
// so that it is the fp32 gamma the caller would form.
__device__ __forceinline__ float pi_gamma(float s, float pi, int side) {
  return side > 0 ? __fmul_rn(s, pi) : side < 0 ? __fdiv_rn(s, pi) : 0.f;
}
__device__ __forceinline__ float div_factored(float x, float dm, float dn, float s, const float* pi, int side_m,
                                              int side_n) {
  const float p = *pi;
  return x / (__fmul_rn(__fadd_rn(dm, pi_gamma(s, p, side_m)), __fadd_rn(dn, pi_gamma(s, p, side_n))));
}

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
  const float* dg; const float* da; float damping;  // EPI_DIV_OUTER; EPI_DIV_FACTORED (damping = s)
  const float* pi; int pi_side_m, pi_side_n;        // EPI_DIV_FACTORED
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
  const float* pi; int pi_side_m, pi_side_n;   // EPI_DIV_FACTORED
  float* peerD[7]; int npeer;      // fused broadcast: the epilogue also stores the tile into these peer copies of D
};
bool tc_gemm_supported(const TcGemmArgs& a);
// the split count launch_tc_gemm runs for a request of `splits` over kb_total k-blocks (every split non-empty); one
// when there is nothing to reduce (the split plan of a factor call on zero rows)
inline int tc_normalize_splits(int splits, int kb_total) {
  if (kb_total < 1) return 1;
  splits = splits < 1 ? 1 : (splits > kb_total ? kb_total : splits);
  const int per = (kb_total + splits - 1) / splits;
  return (kb_total + per - 1) / per;
}
int launch_tc_gemm(const TcGemmArgs& a, cudaStream_t stream);
int tc_num_sms();

// Pinned host memory for the small tables a call sends to the device.  A copy from pageable memory may make the host
// wait until the stream reaches it (the driver stages it), which holds back the enqueue of work for other streams; a
// copy from pinned memory is only queued.  The tables of a call must stay until the device has read them: begin()
// waits for the event that the previous call's end() recorded, then reuses the memory (merged into one block).
struct HostStage {
  char* buf[8] = {};
  size_t size[8] = {};
  int nbuf = 0;
  size_t used = 0;               // bytes taken from buf[nbuf - 1]
  cudaEvent_t done = nullptr;
  bool pending = false;
  int begin();
  int send(void* dst, const void* src, size_t bytes, cudaStream_t s);   // cudaMemcpyAsync host -> device through it
  int end(cudaStream_t s);       // the device has read every table sent since begin() once s reaches this point
};
// host -> device copy of a table on s: through `stage` when given, straight from src otherwise
int send_table(HostStage* stage, void* dst, const void* src, size_t bytes, cudaStream_t s);

}  // namespace kfac
