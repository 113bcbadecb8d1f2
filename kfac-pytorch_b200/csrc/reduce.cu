// K-FAC-reduce rows (Eschenhagen et al., 2023) of weight-shared layers: one row per example, the sum over the R shared
// positions of the example's expand rows (those the kfac_rows_* writers form), times scale / *loss_scale.
//
//   linear          (B, R, features) -> B x ld_out                              a CTA per (example, 32 columns)
//   conv_input      NCDHW -> B x ld_out, features (C, kd, kh, kw) [+ ones]     a CTA per (example, channel) volume,
//                                                                              or per (example, channel, tap) of a Conv1d
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

// Window sums of one (b, c) volume:
//   out[b][(c, l, i, j)] = scale * sum over the output positions (do, ho, wo) of the input read through tap (l, i, j)
// (TapMap: a convolution's window, or a transposed convolution's scatter; for the latter the inputs of one tap form a
// box).  Separable: the volume is a sequence of D * H rows (z, h) of W elements.  rowsum[(z, h)][j] = the sum over the
// inputs of row (z, h) that tap j reads (TapMap::span) for a chunk of rows (a thread per (row, j), so a row is read
// once from HBM and re-read from L1 for the other j), then acc[l][i][j] += rowsum[(z, h)][j] over the chunk's rows that
// taps l and i read, in row order (a thread per (l, i, j), the same thread for every chunk).  Rows no tap reads are not
// read.
constexpr int CONV_SMEM = 2048;   // doubles of rowsum per chunk, and the most (l, i, j) taps of a CTA

// fp32 sum of row[m step] (of its squares: SQ) over one run [m0, m1), in order
template <typename T, bool SQ = false>
__device__ __forceinline__ float run_sum(const T* __restrict__ row, int m0, int m1, int step) {
  float acc = 0.f;
  for (int m = m0; m < m1; ++m) {
    const float v = to_float<T>(row[m * step]);
    if constexpr (SQ) acc = fmaf(v, v, acc);
    else acc += v;
  }
  return acc;
}

// the ones column and the zero padding of an example's row, written once per example
__device__ __forceinline__ void ones_and_padding(const ConvGeo& g, int ones, double sc, float* o, int64_t ld) {
  const int64_t d = g.features();
  for (int64_t f = d + threadIdx.x; f < ld; f += blockDim.x)
    o[f] = (f == d && ones) ? (float)((double)g.spatial() * sc) : 0.f;
}

// SQ: the window sums of the squared input (kfac_factor_conv_input_diag), with ones = 0 and ld = features
template <typename T, bool TRANSPOSED, bool SQ = false>
__global__ void __launch_bounds__(256) reduce_conv_input_kernel(const T* __restrict__ x, const ConvGeo g, int ones,
                                                                float scale, float* out, int64_t ld) {
  using Tap = TapMap<TRANSPOSED>;
  __shared__ double rowsum[CONV_SMEM];
  __shared__ double pacc[CONV_SMEM];
  const int64_t plane = blockIdx.x;
  const int64_t b = plane / g.C;
  const int c = (int)(plane - b * g.C);
  const int kw = g.kw;
  const int NR = g.D * g.H;
  const T* __restrict__ xp = x + plane * NR * g.W;
  const int P = g.kd * g.kh * kw;
  const int HC = max(1, min(NR, CONV_SMEM / kw));
  for (int p = threadIdx.x; p < P; p += blockDim.x) pacc[p] = 0.0;
  for (int r0 = 0; r0 < NR; r0 += HC) {
    const int hc = min(HC, NR - r0);
    for (int e = threadIdx.x; e < hc * kw; e += blockDim.x) {
      const int r = e / kw, j = e - r * kw, q = r0 + r, z = q / g.H, h = q - z * g.H;
      bool used_z = false, used_h = false;
      for (int l = 0; l < g.kd && !used_z; ++l) used_z = Tap::feeds(z, l, g.sd, g.dd, g.pd, g.Do);
      for (int i = 0; i < g.kh && !used_h; ++i) used_h = Tap::feeds(h, i, g.sh, g.dh, g.ph, g.Ho);
      double acc = 0.0;
      if (used_z && used_h) {
        int first, step, n;
        Tap::span(g.W, j, g.sw, g.dw, g.pw, g.Wo, first, step, n);
        const T* __restrict__ row = xp + (int64_t)q * g.W + first;
        for (int m0 = 0; m0 < n; m0 += RUN) acc += (double)run_sum<T, SQ>(row, m0, min(n, m0 + RUN), step);
      }
      rowsum[e] = acc;
    }
    __syncthreads();
    for (int p = threadIdx.x; p < P; p += blockDim.x) {
      const int j = p % kw, i = (p / kw) % g.kh, l = p / (kw * g.kh);
      int first, step, n;
      Tap::span(g.H, i, g.sh, g.dh, g.ph, g.Ho, first, step, n);
      double acc = pacc[p];
      for (int z = r0 / g.H; z <= (r0 + hc - 1) / g.H; ++z) {
        if (!Tap::feeds(z, l, g.sd, g.dd, g.pd, g.Do)) continue;
        const int hlo = max(0, r0 - z * g.H), hhi = min(g.H, r0 + hc - z * g.H);
        // the rows of tap i's span inside the chunk
        int m = hlo > first ? (hlo - first + step - 1) / step : 0;
        for (int h = first + m * step; m < n && h < hhi; ++m, h += step) acc += rowsum[(z * g.H + h - r0) * kw + j];
      }
      pacc[p] = acc;
    }
    __syncthreads();
  }
  const double sc = (double)scale;
  float* o = out + b * ld;
  for (int p = threadIdx.x; p < P; p += blockDim.x) o[(int64_t)c * P + p] = (float)(pacc[p] * sc);
  if (c == 0) ones_and_padding(g, ones, sc, o, ld);
}

// A single-row input (D = H = 1, kd = kh = 1, no depth or height padding, Do = Ho = 1: a Conv1d or ConvTranspose1d).
// reduce_conv_input_kernel would give one thread per tap j a whole signal; here a CTA per (b, c, j) forms the fp32 runs
// of the tap's sum in parallel and one thread adds them in fp64 in run order -- the order of reduce_conv_input_kernel,
// so both give the same bits.
template <typename T, bool TRANSPOSED, bool SQ = false>
__global__ void __launch_bounds__(256) reduce_conv_input_1d_kernel(const T* __restrict__ x, const ConvGeo g, int ones,
                                                                   float scale, float* out, int64_t ld) {
  __shared__ double runs[CONV_SMEM];
  const int64_t plane = blockIdx.x;
  const int64_t b = plane / g.C;
  const int c = (int)(plane - b * g.C);
  const int j = blockIdx.y;
  int first, step, cnt;
  TapMap<TRANSPOSED>::span(g.W, j, g.sw, g.dw, g.pw, g.Wo, first, step, cnt);
  const T* __restrict__ row = x + plane * g.W + first;
  const int n = (cnt + RUN - 1) / RUN;
  double acc = 0.0;
  for (int k0 = 0; k0 < n; k0 += CONV_SMEM) {
    const int kn = min(CONV_SMEM, n - k0);
    for (int k = threadIdx.x; k < kn; k += blockDim.x) {
      const int m0 = (k0 + k) * RUN;
      runs[k] = (double)run_sum<T, SQ>(row, m0, min(cnt, m0 + RUN), step);
    }
    __syncthreads();
    if (threadIdx.x == 0)
      for (int k = 0; k < kn; ++k) acc += runs[k];
    __syncthreads();
  }
  const double sc = (double)scale;
  float* o = out + b * ld;
  if (threadIdx.x == 0) {
    double t = 0.0;   // as pacc in reduce_conv_input_kernel: 0 + acc (a signed zero becomes +0 there too)
    t += acc;
    o[(int64_t)c * g.kw + j] = (float)(t * sc);
  }
  if (c == 0 && j == 0) ones_and_padding(g, ones, sc, o, ld);
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

namespace kfac {
// acc[j] += scale * sum_c partial[c][j] (j < V, the chunks added in order in fp64), acc[V] += scale * ones_sum when
// ones: the second launch of the diagonal statistics (factor.cu)
int launch_diag_reduce(const float* partial, int chunks, int V, int ones, double ones_sum, float scale, float* acc,
                       cudaStream_t s);
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

template <bool TRANSPOSED = false, bool SQ = false>
static int reduce_conv_input(const void* x, int dtype, const ConvGeo& g, int append_ones, float scale, float* out,
                             int ld_out, cudaStream_t s) {
  KFAC_CHECK_ARG((int64_t)g.kd * g.kh * g.kw <= CONV_SMEM, "kernel window of more than 2048 taps");
  const int ones = append_ones ? 1 : 0;
  KFAC_CHECK_ARG((int64_t)ld_out >= g.features() + ones, "ld_out");
  KFAC_CHECK_ARG((int64_t)g.batch * g.C < (1ll << 31), "grid");
  const unsigned planes = (unsigned)((int64_t)g.batch * g.C);
  // the single-row kernel sums row 0 only: no depth or height padding may move the one output row off it (for a
  // transposed geometry with these extents the output row is row 0 as well)
  if (g.D == 1 && g.H == 1 && g.kd == 1 && g.kh == 1 && g.pd == 0 && g.ph == 0 && g.Do == 1 && g.Ho == 1) {
    const dim3 grid(planes, (unsigned)g.kw);
    if (dtype == KFAC_F32)
      reduce_conv_input_1d_kernel<float, TRANSPOSED, SQ><<<grid, 256, 0, s>>>((const float*)x, g, ones, scale, out,
                                                                          ld_out);
    else if (dtype == KFAC_F16)
      reduce_conv_input_1d_kernel<__half, TRANSPOSED, SQ><<<grid, 256, 0, s>>>((const __half*)x, g, ones, scale, out,
                                                                           ld_out);
    else if (dtype == KFAC_BF16)
      reduce_conv_input_1d_kernel<__nv_bfloat16, TRANSPOSED, SQ><<<grid, 256, 0, s>>>((const __nv_bfloat16*)x, g, ones,
                                                                                  scale, out, ld_out);
    else { set_error("unknown dtype %d", dtype); return KFAC_ERR_BAD_ARG; }
  } else {
    if (dtype == KFAC_F32)
      reduce_conv_input_kernel<float, TRANSPOSED, SQ><<<planes, 256, 0, s>>>((const float*)x, g, ones, scale, out, ld_out);
    else if (dtype == KFAC_F16)
      reduce_conv_input_kernel<__half, TRANSPOSED, SQ><<<planes, 256, 0, s>>>((const __half*)x, g, ones, scale, out,
                                                                          ld_out);
    else if (dtype == KFAC_BF16)
      reduce_conv_input_kernel<__nv_bfloat16, TRANSPOSED, SQ><<<planes, 256, 0, s>>>((const __nv_bfloat16*)x, g, ones,
                                                                                 scale, out, ld_out);
    else { set_error("unknown dtype %d", dtype); return KFAC_ERR_BAD_ARG; }
  }
  KFAC_LAUNCH_CHECK();
  return KFAC_OK;
}

extern "C" int kfac_reduce_rows_conv2d_input(const void* x, int dtype, int batch, int C, int H, int W, int kh, int kw,
                                             int sh, int sw, int ph, int pw, int append_ones, float scale, float* out,
                                             int ld_out, void* stream) {
  KFAC_CHECK_ARG(x && out, "null pointer");
  KFAC_CHECK_ARG(batch > 0 && C > 0 && H > 0 && W > 0 && kh > 0 && kw > 0 && sh > 0 && sw > 0 && ph >= 0 && pw >= 0,
                 "geometry");
  const ConvGeo g = conv2d_geo(batch, C, H, W, kh, kw, sh, sw, ph, pw);
  KFAC_CHECK_ARG(g.Ho > 0 && g.Wo > 0, "empty output");
  return reduce_conv_input(x, dtype, g, append_ones, scale, out, ld_out, (cudaStream_t)stream);
}

extern "C" int kfac_reduce_rows_conv_input(const void* x, int dtype, const kfac_conv_geometry* geom, int append_ones,
                                           float scale, float* out, int ld_out, void* stream) {
  KFAC_CHECK_ARG(x && out, "null pointer");
  ConvGeo g;
  const int rc = resolve_conv_geometry(geom, &g);
  if (rc) return rc;
  return reduce_conv_input(x, dtype, g, append_ones, scale, out, ld_out, (cudaStream_t)stream);
}

extern "C" int kfac_reduce_rows_conv_transpose_input(const void* x, int dtype, const kfac_conv_transpose_geometry* geom,
                                                     int append_ones, float scale, float* out, int ld_out,
                                                     void* stream) {
  KFAC_CHECK_ARG(x && out, "null pointer");
  ConvGeo g;
  const int rc = resolve_conv_transpose_geometry(geom, &g);
  if (rc) return rc;
  return reduce_conv_input<true>(x, dtype, g, append_ones, scale, out, ld_out, (cudaStream_t)stream);
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

// The diagonal of kfac_factor_conv_input's A without the im2col: each (b, c) volume is read once, and the window sums
// of its squares over the output lattice (reduce_conv_input_kernel with SQ, the re-reads of a row from L1) give the
// example's partial for the C x taps features; the partials (B x features fp32, example-major) are added per feature
// in example order, in fp64, by a second launch.
static size_t conv_diag_ws_bytes(const ConvGeo& g) {
  return align_up((size_t)g.batch * (size_t)g.features() * sizeof(float), 256);
}

extern "C" size_t kfac_factor_conv_input_diag_workspace_bytes(const kfac_conv_geometry* geom) {
  ConvGeo g;
  if (resolve_conv_geometry(geom, &g) != KFAC_OK) return 0;
  return conv_diag_ws_bytes(g);
}

extern "C" int kfac_factor_conv_input_diag(const void* x, int dtype, const kfac_conv_geometry* geom, int append_ones,
                                           float scale, float* acc, void* ws, size_t ws_bytes, void* stream) {
  KFAC_CHECK_ARG(x && acc, "null pointer");
  ConvGeo g;
  const int rc = resolve_conv_geometry(geom, &g);
  if (rc) return rc;
  KFAC_CHECK_ARG(dtype == KFAC_F32 || dtype == KFAC_F16 || dtype == KFAC_BF16, "dtype");
  KFAC_CHECK_ARG(g.features() < (1ll << 31), "features");
  const size_t need = conv_diag_ws_bytes(g);
  if (!ws || ws_bytes < need) {
    set_error("factor_conv_input_diag: workspace too small (%zu < %zu)", ws_bytes, need);
    return KFAC_ERR_WORKSPACE;
  }
  cudaStream_t s = (cudaStream_t)stream;
  const int d = (int)g.features();
  float* partial = (float*)ws;
  const int r = reduce_conv_input<false, true>(x, dtype, g, 0, 1.f, partial, d, s);
  if (r) return r;
  return launch_diag_reduce(partial, g.batch, d, append_ones ? 1 : 0, (double)g.batch * (double)g.spatial(), scale,
                            acc, s);
}
