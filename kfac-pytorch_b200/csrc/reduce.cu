// K-FAC-reduce rows (Eschenhagen et al., 2023) of weight-shared layers: one row per example, the sum over the R shared
// positions of the example's expand rows (those the kfac_rows_* writers form), times scale / *loss_scale.
//
//   linear          (B, R, features) -> B x ld_out                              a CTA per (example, 32 columns)
//   conv2d_input    NCHW -> B x ld_out, features (C, kh, kw) [+ ones]          a CTA per (example, channel) plane
//   conv2d_gradout  NCHW -> B x ld_out, features C                             a warp per (example, channel) plane
//
// Every input element is read from HBM once (the conv input's window sums re-read a plane row from L1 only).  Sums run
// in fp32 over runs of at most 16 elements, then in fp64, in an order fixed by the shape: no atomics, the same bits on
// every run.  The output is rounded to fp32 once, after the scaling.
#include "common.cuh"

namespace kfac {
namespace {

constexpr int RUN = 16;   // fp32 run length before a partial sum is added in fp64

__device__ __forceinline__ double out_scale(float scale, const float* loss_scale) {
  return loss_scale ? (double)scale / (double)*loss_scale : (double)scale;
}

// out[b][f] = s * sum_t x[b sb + t st + f] (f < feat), s * R (f == feat, ones), 0 up to ld.  The 8 warps of a CTA take
// the rows t = warp, warp + 8, ...; their fp64 partials are added in warp order.
template <typename T>
__global__ void __launch_bounds__(256) reduce_linear_kernel(const T* __restrict__ x, int64_t R, int feat, int64_t sb,
                                                            int64_t st, int ones, float scale, const float* loss_scale,
                                                            float* out, int64_t ld, int tiles) {
  __shared__ double part[8][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t b = blockIdx.x / tiles;
  const int64_t f = (int64_t)(blockIdx.x % tiles) * 32 + lane;
  double acc = 0.0;
  if (f < feat) {
    const T* __restrict__ p = x + b * sb + f;
    for (int64_t t0 = warp; t0 < R; t0 += 8 * RUN) {
      float s = 0.f;
#pragma unroll
      for (int k = 0; k < RUN; ++k) {
        const int64_t t = t0 + 8 * k;
        if (t < R) s += to_float<T>(p[t * st]);
      }
      acc += (double)s;
    }
  }
  part[warp][lane] = acc;
  __syncthreads();
  if (warp != 0 || f >= ld) return;
  const double sc = out_scale(scale, loss_scale);
  float v = 0.f;
  if (f < feat) {
    double t = part[0][lane];
#pragma unroll
    for (int w = 1; w < 8; ++w) t += part[w][lane];
    v = (float)(t * sc);
  } else if (f == feat && ones) {
    v = (float)((double)R * sc);
  }
  out[b * ld + f] = v;
}

// Window sums of one (b, c) plane: out[b][(c, i, j)] = scale * sum_{ho, wo} xpad[ho sh + i - ph][wo sw + j - pw].
// Separable: rowsum[h][j] = sum_wo x[h][wo sw + j - pw] for a chunk of rows (a thread per (h, j), so a row is read once
// from HBM and re-read from L1 for the other j), then acc[i][j] += sum_ho rowsum[ho sh + i - ph][j] in row order (a
// thread per (i, j), the same thread for every chunk).  Rows no window touches are not read.
constexpr int CONV_SMEM = 2048;   // doubles of rowsum per chunk, and the most (i, j) pairs of a CTA

template <typename T>
__global__ void __launch_bounds__(256) reduce_conv_input_kernel(const T* __restrict__ x, int C, int H, int W, int kh,
                                                                int kw, int sh, int sw, int ph, int pw, int Ho, int Wo,
                                                                int ones, float scale, float* out, int64_t ld) {
  __shared__ double rowsum[CONV_SMEM];
  __shared__ double pacc[CONV_SMEM];
  const int64_t plane = blockIdx.x;
  const int64_t b = plane / C;
  const int c = (int)(plane - b * C);
  const T* __restrict__ xp = x + plane * H * W;
  const int P = kh * kw;
  const int HC = max(1, min(H, CONV_SMEM / kw));
  for (int p = threadIdx.x; p < P; p += blockDim.x) pacc[p] = 0.0;
  for (int h0 = 0; h0 < H; h0 += HC) {
    const int hc = min(HC, H - h0);
    for (int e = threadIdx.x; e < hc * kw; e += blockDim.x) {
      const int r = e / kw, j = e - r * kw, h = h0 + r;
      // the rows of window offset i are h = ho sh + i - ph, 0 <= ho < Ho
      bool used = false;
      for (int i = 0; i < kh && !used; ++i) {
        const int q = h + ph - i;
        used = q >= 0 && q % sh == 0 && q / sh < Ho;
      }
      double acc = 0.0;
      if (used) {
        // wo with 0 <= wo sw + j - pw < W
        const int lo = j < pw ? (pw - j + sw - 1) / sw : 0;
        const int hi = W - 1 + pw - j < 0 ? -1 : min(Wo - 1, (W - 1 + pw - j) / sw);
        const T* __restrict__ row = xp + (int64_t)h * W + j - pw;
        for (int w0 = lo; w0 <= hi; w0 += RUN) {
          float s = 0.f;
          const int w1 = min(hi + 1, w0 + RUN);
          for (int wo = w0; wo < w1; ++wo) s += to_float<T>(row[wo * sw]);
          acc += (double)s;
        }
      }
      rowsum[e] = acc;
    }
    __syncthreads();
    for (int p = threadIdx.x; p < P; p += blockDim.x) {
      const int i = p / kw, j = p - i * kw;
      double acc = pacc[p];
      // first row of the chunk on the lattice of i, then every sh-th row
      int q = h0 + ph - i;
      int r = q <= 0 ? -q : (sh - q % sh) % sh;
      for (; r < hc; r += sh) {
        if ((h0 + r + ph - i) / sh >= Ho) break;
        acc += rowsum[r * kw + j];
      }
      pacc[p] = acc;
    }
    __syncthreads();
  }
  const double sc = (double)scale;
  float* o = out + b * ld;
  for (int p = threadIdx.x; p < P; p += blockDim.x) o[(int64_t)c * P + p] = (float)(pacc[p] * sc);
  if (c == 0) {   // the ones column and the padding of the example's row
    const int64_t d = (int64_t)C * P;
    for (int64_t f = d + threadIdx.x; f < ld; f += blockDim.x)
      o[f] = (f == d && ones) ? (float)((double)Ho * Wo * sc) : 0.f;
  }
}

// out[b][c] = s * sum of the (b, c) plane of S elements (c < C), 0 for c in [C, ld): a warp per (b, c) of B x ld
template <typename T>
__global__ void __launch_bounds__(256) reduce_planes_kernel(const T* __restrict__ g, int64_t B, int C, int64_t S,
                                                            float scale, const float* loss_scale, float* out,
                                                            int64_t ld) {
  const int lane = threadIdx.x & 31;
  const int64_t q = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (q >= B * ld) return;
  const int64_t b = q / ld, c = q - b * ld;
  if (c >= C) {
    if (lane == 0) out[q] = 0.f;
    return;
  }
  const T* __restrict__ p = g + (b * C + c) * S;
  double acc = 0.0;
  for (int64_t s0 = lane; s0 < S; s0 += 32 * RUN) {
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < RUN; ++k) {
      const int64_t s1 = s0 + 32 * k;
      if (s1 < S) s += to_float<T>(p[s1]);
    }
    acc += (double)s;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, o);
  if (lane == 0) out[q] = (float)(acc * out_scale(scale, loss_scale));
}

}  // namespace
}  // namespace kfac

using namespace kfac;

extern "C" int kfac_reduce_rows_linear_strided(const void* x, int dtype, int64_t B, int64_t R, int features,
                                               int64_t example_stride, int64_t position_stride, int append_ones,
                                               float scale, const float* loss_scale, float* out, int ld_out,
                                               void* stream) {
  KFAC_CHECK_ARG(x && out, "null pointer");
  KFAC_CHECK_ARG(B > 0 && R > 0 && features > 0, "dims");
  KFAC_CHECK_ARG(example_stride >= 0 && position_stride >= 0, "strides");
  const int ones = append_ones ? 1 : 0;
  KFAC_CHECK_ARG(ld_out >= features + ones, "ld_out");
  const int tiles = ceil_div(ld_out, 32);
  KFAC_CHECK_ARG(B * tiles < (1ll << 31), "grid");
  cudaStream_t s = (cudaStream_t)stream;
  const unsigned grid = (unsigned)(B * tiles);
  const int64_t sb = example_stride, st = position_stride;
  if (dtype == KFAC_F32)
    reduce_linear_kernel<float><<<grid, 256, 0, s>>>((const float*)x, R, features, sb, st, ones, scale, loss_scale, out,
                                                     ld_out, tiles);
  else if (dtype == KFAC_F16)
    reduce_linear_kernel<__half><<<grid, 256, 0, s>>>((const __half*)x, R, features, sb, st, ones, scale, loss_scale, out,
                                                      ld_out, tiles);
  else if (dtype == KFAC_BF16)
    reduce_linear_kernel<__nv_bfloat16><<<grid, 256, 0, s>>>((const __nv_bfloat16*)x, R, features, sb, st, ones, scale,
                                                             loss_scale, out, ld_out, tiles);
  else { set_error("unknown dtype %d", dtype); return KFAC_ERR_BAD_ARG; }
  KFAC_LAUNCH_CHECK();
  return KFAC_OK;
}

extern "C" int kfac_reduce_rows_linear(const void* x, int dtype, int64_t B, int64_t R, int features, int append_ones,
                                       float scale, const float* loss_scale, float* out, int ld_out, void* stream) {
  return kfac_reduce_rows_linear_strided(x, dtype, B, R, features, R * features, features, append_ones, scale,
                                         loss_scale, out, ld_out, stream);
}

extern "C" int kfac_reduce_rows_conv2d_input(const void* x, int dtype, int batch, int C, int H, int W, int kh, int kw,
                                             int sh, int sw, int ph, int pw, int append_ones, float scale, float* out,
                                             int ld_out, void* stream) {
  KFAC_CHECK_ARG(x && out, "null pointer");
  KFAC_CHECK_ARG(batch > 0 && C > 0 && H > 0 && W > 0 && kh > 0 && kw > 0 && sh > 0 && sw > 0 && ph >= 0 && pw >= 0,
                 "geometry");
  const int Ho = (H + 2 * ph - kh) / sh + 1, Wo = (W + 2 * pw - kw) / sw + 1;
  KFAC_CHECK_ARG(Ho > 0 && Wo > 0, "empty output");
  KFAC_CHECK_ARG(kh * kw <= CONV_SMEM, "kernel window of more than 2048 taps");
  const int ones = append_ones ? 1 : 0;
  KFAC_CHECK_ARG((int64_t)ld_out >= (int64_t)C * kh * kw + ones, "ld_out");
  KFAC_CHECK_ARG((int64_t)batch * C < (1ll << 31), "grid");
  cudaStream_t s = (cudaStream_t)stream;
  const unsigned grid = (unsigned)((int64_t)batch * C);
  if (dtype == KFAC_F32)
    reduce_conv_input_kernel<float><<<grid, 256, 0, s>>>((const float*)x, C, H, W, kh, kw, sh, sw, ph, pw, Ho, Wo, ones,
                                                         scale, out, ld_out);
  else if (dtype == KFAC_F16)
    reduce_conv_input_kernel<__half><<<grid, 256, 0, s>>>((const __half*)x, C, H, W, kh, kw, sh, sw, ph, pw, Ho, Wo, ones,
                                                          scale, out, ld_out);
  else if (dtype == KFAC_BF16)
    reduce_conv_input_kernel<__nv_bfloat16><<<grid, 256, 0, s>>>((const __nv_bfloat16*)x, C, H, W, kh, kw, sh, sw, ph, pw,
                                                                 Ho, Wo, ones, scale, out, ld_out);
  else { set_error("unknown dtype %d", dtype); return KFAC_ERR_BAD_ARG; }
  KFAC_LAUNCH_CHECK();
  return KFAC_OK;
}

extern "C" int kfac_reduce_rows_conv2d_gradout(const void* g, int dtype, int batch, int C, int Ho, int Wo, float scale,
                                               const float* loss_scale, float* out, int ld_out, void* stream) {
  KFAC_CHECK_ARG(g && out, "null pointer");
  KFAC_CHECK_ARG(batch > 0 && C > 0 && Ho > 0 && Wo > 0, "geometry");
  KFAC_CHECK_ARG(ld_out >= C, "ld_out");
  const int64_t warps = (int64_t)batch * ld_out;
  KFAC_CHECK_ARG((warps + 7) / 8 < (1ll << 31), "grid");
  cudaStream_t s = (cudaStream_t)stream;
  const unsigned grid = (unsigned)((warps + 7) / 8);
  const int64_t S = (int64_t)Ho * Wo;
  if (dtype == KFAC_F32)
    reduce_planes_kernel<float><<<grid, 256, 0, s>>>((const float*)g, batch, C, S, scale, loss_scale, out, ld_out);
  else if (dtype == KFAC_F16)
    reduce_planes_kernel<__half><<<grid, 256, 0, s>>>((const __half*)g, batch, C, S, scale, loss_scale, out, ld_out);
  else if (dtype == KFAC_BF16)
    reduce_planes_kernel<__nv_bfloat16><<<grid, 256, 0, s>>>((const __nv_bfloat16*)g, batch, C, S, scale, loss_scale, out,
                                                             ld_out);
  else { set_error("unknown dtype %d", dtype); return KFAC_ERR_BAD_ARG; }
  KFAC_LAUNCH_CHECK();
  return KFAC_OK;
}
