// Normalization layers (BatchNorm, LayerNorm, RMSNorm, GroupNorm, InstanceNorm; an extension beyond the reference,
// opt-in): the exact per-channel Fisher block of the affine part y = s * xhat + b, and its damped 2 x 2 (or 1 x 1)
// solve.
//
// A channel c is a one-input layer with bias acting on xhat, so its rows are a_r = (xhat_rc, 1) and g_r, and
//   F_c = (1/N) sum_r g_rc^2 a_r a_r^T = (1/N) (sum g^2 xhat^2, sum g^2 xhat, sum g^2)      (k = 3 packed entries)
// or (1/N) sum g^2 xhat^2 alone for a scale-only layer (k = 1).  xhat is recomputed from the layer input: BatchNorm
// with the biased batch statistics of each channel, LayerNorm / RMSNorm with the statistics of each row, GroupNorm /
// InstanceNorm with the statistics of each example and group.
//
// Every sum is accumulated in fp64, every reduction runs in a fixed order and the chunking depends on the shape only:
// the same input gives the same bits.  No floating-point atomics, no host sync.
#include <algorithm>
#include <vector>

#include "common.cuh"

namespace kfac {

static inline int norm_grid_for(int64_t total) {
  const int64_t b = (total + 255) / 256;
  return (int)std::max<int64_t>(1, std::min<int64_t>(b, (int64_t)tc_num_sms() * 8));
}

// ---- fixed-order block reduction of NV doubles (256 threads); the result is valid in thread 0 ------------------
template <int NV>
__device__ __forceinline__ void block_sum(double (&v)[NV]) {
  __shared__ double red[8][NV];
#pragma unroll
  for (int q = 0; q < NV; ++q)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[q] += __shfl_xor_sync(0xffffffffu, v[q], o);
  if ((threadIdx.x & 31) == 0)
#pragma unroll
    for (int q = 0; q < NV; ++q) red[threadIdx.x >> 5][q] = v[q];
  __syncthreads();
  if (threadIdx.x == 0) {
#pragma unroll
    for (int q = 0; q < NV; ++q) {
      double t = 0.0;
      for (int w = 0; w < 8; ++w) t += red[w][q];
      v[q] = t;
    }
  }
}

// ================================================================ BatchNorm: x, g are (B, C, S), S = H*W, L or 1
// One pass over x and g.  For each (chunk, channel) five fp64 sums of y = x - K_c, where the shift K_c = x[0, c, 0]
// keeps the variance free of cancellation when |mean| >> std:
//   s0 = sum y, s1 = sum y^2, s2 = sum g^2, s3 = sum g^2 y, s4 = sum g^2 y^2.
// With m = s0 / N the mean of y and r = 1 / sqrt(s1 / N - m^2 + eps), xhat = (y - m) r and
//   sum g^2 xhat^2 = (s4 - 2 m s3 + m^2 s2) r^2,   sum g^2 xhat = (s3 - m s2) r,   sum g^2 = s2.
constexpr int NC_SUMS = 5;

// chunks of whole batch rows: about 4 blocks per SM of a 132-SM part in total, at least 4096 elements per block
static int64_t nc_chunks(int64_t B, int C, int64_t S) {
  const int64_t want = std::max<int64_t>(1, (528 + C - 1) / C);
  const int64_t by_size = std::max<int64_t>(1, B * S / 4096);
  const int64_t ch = std::max<int64_t>(1, std::min<int64_t>(std::min(want, by_size), B));
  const int64_t rows = (B + ch - 1) / ch;
  return (B + rows - 1) / rows;   // every chunk non-empty
}

// S >= 2: block (c, chunk).  Thread t reads position t % S of batch rows chunk_begin + t / S, stepping by P = 256 / S
// rows (S >= 256: every thread walks the S positions of each row), so no index is divided inside the loop.
template <typename TX, typename TG>
__global__ void __launch_bounds__(256) bn_spatial_kernel(const TX* __restrict__ x, const TG* __restrict__ g, int64_t B,
                                                         int C, int64_t S, int64_t chunk_rows,
                                                         double* __restrict__ partial) {
  const int c = blockIdx.x;
  const int64_t b0 = (int64_t)blockIdx.y * chunk_rows, b1 = min(B, b0 + chunk_rows);
  const double K = (double)to_float<TX>(x[(int64_t)c * S]);
  double v[NC_SUMS] = {0.0, 0.0, 0.0, 0.0, 0.0};
  auto add = [&](int64_t off) {
    const double y = (double)to_float<TX>(x[off]) - K;
    const double gv = (double)to_float<TG>(g[off]);
    const double g2 = gv * gv, g2y = g2 * y;
    v[0] += y;
    v[1] = fma(y, y, v[1]);
    v[2] += g2;
    v[3] += g2y;
    v[4] = fma(g2y, y, v[4]);
  };
  if (S >= 256) {
    for (int64_t b = b0; b < b1; ++b) {
      const int64_t base = (b * C + c) * S;
      for (int64_t i = threadIdx.x; i < S; i += 256) add(base + i);
    }
  } else {
    const int P = 256 / (int)S;
    const int tb = threadIdx.x / (int)S, ti = threadIdx.x - tb * (int)S;
    if (tb < P)
      for (int64_t b = b0 + tb; b < b1; b += P) add((b * C + c) * S + ti);
  }
  block_sum<NC_SUMS>(v);
  if (threadIdx.x == 0) {
    double* out = partial + ((int64_t)blockIdx.y * C + c) * NC_SUMS;
#pragma unroll
    for (int q = 0; q < NC_SUMS; ++q) out[q] = v[q];
  }
}

// S = 1 (BatchNorm1d on (B, C)): the rows are contiguous, one thread per channel, coalesced over the channels
template <typename TX, typename TG>
__global__ void __launch_bounds__(256) bn_flat_kernel(const TX* __restrict__ x, const TG* __restrict__ g, int64_t B,
                                                      int C, int64_t chunk_rows, double* __restrict__ partial) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const int64_t b0 = (int64_t)blockIdx.y * chunk_rows, b1 = min(B, b0 + chunk_rows);
  const double K = (double)to_float<TX>(x[c]);
  double v[NC_SUMS] = {0.0, 0.0, 0.0, 0.0, 0.0};
  for (int64_t b = b0; b < b1; ++b) {
    const double y = (double)to_float<TX>(x[b * C + c]) - K;
    const double gv = (double)to_float<TG>(g[b * C + c]);
    const double g2 = gv * gv, g2y = g2 * y;
    v[0] += y;
    v[1] = fma(y, y, v[1]);
    v[2] += g2;
    v[3] += g2y;
    v[4] = fma(g2y, y, v[4]);
  }
  double* out = partial + ((int64_t)blockIdx.y * C + c) * NC_SUMS;
#pragma unroll
  for (int q = 0; q < NC_SUMS; ++q) out[q] = v[q];
}

// acc[c * k + .] += scale * F_c, the chunks added in order
__global__ void bn_finalize_kernel(const double* __restrict__ partial, int chunks, int C, double n, double eps, int k,
                                   float scale, float* acc) {
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < C; c += gridDim.x * blockDim.x) {
    double v[NC_SUMS] = {0.0, 0.0, 0.0, 0.0, 0.0};
    for (int ch = 0; ch < chunks; ++ch)
#pragma unroll
      for (int q = 0; q < NC_SUMS; ++q) v[q] += partial[((int64_t)ch * C + c) * NC_SUMS + q];
    const double m = v[0] / n;
    const double var = fmax(v[1] / n - m * m, 0.0);
    const double r = 1.0 / sqrt(var + eps);
    const double fss = (v[4] - 2.0 * m * v[3] + m * m * v[2]) * r * r;
    const double s = (double)scale;
    if (k == 1) {
      acc[c] = __fadd_rn(acc[c], (float)(s * fss));
    } else {
      acc[3 * c] = __fadd_rn(acc[3 * c], (float)(s * fss));
      acc[3 * c + 1] = __fadd_rn(acc[3 * c + 1], (float)(s * (v[3] - m * v[2]) * r));
      acc[3 * c + 2] = __fadd_rn(acc[3 * c + 2], (float)(s * v[2]));
    }
  }
}

// ================================================================ LayerNorm / RMSNorm: x, g are (rows, D) row-major
// (1) one warp per row: mean and 1 / sqrt(var + eps) in fp64 (LayerNorm; the row is shifted by its first entry), or
//     mean 0 and 1 / sqrt(mean(x^2) + eps) (RMSNorm), stored as two doubles per row;
// (2) one thread per feature and row chunk: sum g^2 xhat^2, sum g^2 xhat, sum g^2 in fp64 -> fp64 partials;
// (3) the chunks added in order, acc += scale * F.
constexpr int ROW_SUMS = 3;

static int64_t row_chunks(int64_t rows) { return std::max<int64_t>(1, std::min<int64_t>(256, (rows + 15) / 16)); }

template <typename TX>
__global__ void __launch_bounds__(256) row_stats_kernel(const TX* __restrict__ x, int64_t rows, int D, int rms,
                                                        double eps, double2* __restrict__ stats) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < rows; r += warps) {
    const TX* row = x + r * D;
    const double K = rms ? 0.0 : (double)to_float<TX>(row[0]);
    double s0 = 0.0, s1 = 0.0;
    for (int j = lane; j < D; j += 32) {
      const double y = (double)to_float<TX>(row[j]) - K;
      s0 += y;
      s1 = fma(y, y, s1);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      s0 += __shfl_xor_sync(0xffffffffu, s0, o);
      s1 += __shfl_xor_sync(0xffffffffu, s1, o);
    }
    if (lane == 0) {
      const double m = s0 / D;
      const double var = rms ? s1 / D : fmax(s1 / D - m * m, 0.0);
      stats[r] = make_double2(rms ? 0.0 : K + m, 1.0 / sqrt(var + eps));
    }
  }
}

template <typename TX, typename TG>
__global__ void __launch_bounds__(256) row_cols_kernel(const TX* __restrict__ x, const TG* __restrict__ g,
                                                       const double2* __restrict__ stats, int64_t rows, int D,
                                                       int64_t chunk_rows, double* __restrict__ partial) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= D) return;
  const int64_t r0 = (int64_t)blockIdx.y * chunk_rows, r1 = min(rows, r0 + chunk_rows);
  double t0 = 0.0, t1 = 0.0, t2 = 0.0;
  for (int64_t r = r0; r < r1; ++r) {
    const double2 st = __ldg(stats + r);
    const double xh = ((double)to_float<TX>(x[r * D + j]) - st.x) * st.y;
    const double gv = (double)to_float<TG>(g[r * D + j]);
    const double g2 = gv * gv, g2x = g2 * xh;
    t0 += g2;
    t1 += g2x;
    t2 = fma(g2x, xh, t2);
  }
  double* out = partial + ((int64_t)blockIdx.y * D + j) * ROW_SUMS;
  out[0] = t2;
  out[1] = t1;
  out[2] = t0;
}

__global__ void row_finalize_kernel(const double* __restrict__ partial, int chunks, int D, int k, float scale,
                                    float* acc) {
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < D; j += gridDim.x * blockDim.x) {
    double v[ROW_SUMS] = {0.0, 0.0, 0.0};
    for (int ch = 0; ch < chunks; ++ch)
#pragma unroll
      for (int q = 0; q < ROW_SUMS; ++q) v[q] += partial[((int64_t)ch * D + j) * ROW_SUMS + q];
    const double s = (double)scale;
    if (k == 1) {
      acc[j] = __fadd_rn(acc[j], (float)(s * v[0]));
    } else {
#pragma unroll
      for (int q = 0; q < 3; ++q) acc[3 * j + q] = __fadd_rn(acc[3 * j + q], (float)(s * v[q]));
    }
  }
}

// ================================================================ GroupNorm / InstanceNorm: x, g are (B, C, S)
// xhat is normalized per example and group: group gi of example b is the Cg * S contiguous elements of channels
// [gi * Cg, (gi + 1) * Cg).  Three launches:
// (1) one pass over x and g: the five NC_SUMS of each (b, c) plane, of y = x - K_bg with the shift K_bg the group's
//     first element (so a group with |mean| >> std keeps its variance), stored at plane[(b * C + c) * 5 + q];
// (2) one warp per (b, gi): the Cg planes' sum y and sum y^2 in channel order -> (m_bg, r_bg), the mean of y and
//     1 / sqrt(var + eps);
// (3) one thread per channel: for b = 0 .. B-1 in order, the BatchNorm formulas with (m_bg, r_bg), then
//     acc += scale * F_c.
// (2) is its own launch so that (3) reads one (m, r) pair per example instead of all Cg planes of the group, which
// for GroupNorm(1, C) would be B * C serial reads in every thread.
// Planes of up to GN_WARP_MAX_S elements take a warp each, eight per block.  Larger planes take a block each, unless
// there are so many that warps alone fill the device (16 x 16 and 32 x 32 maps of a U-Net at batch 64): a block per
// 256-element plane spends more time in its reduction than in its loads.
constexpr int GN_WARP_MAX_S = 255, GN_WARP_MAX_S_MANY = 4096;
constexpr int64_t GN_MANY_PLANES = 4096;

static bool gn_warp_per_plane(int64_t planes, int64_t S) {
  return S <= GN_WARP_MAX_S || (S <= GN_WARP_MAX_S_MANY && planes >= GN_MANY_PLANES);
}

template <typename TX, typename TG>
__device__ __forceinline__ void gn_add(const TX* __restrict__ x, const TG* __restrict__ g, int64_t off, double K,
                                       double (&v)[NC_SUMS]) {
  const double y = (double)to_float<TX>(x[off]) - K;
  const double gv = (double)to_float<TG>(g[off]);
  const double g2 = gv * gv, g2y = g2 * y;
  v[0] += y;
  v[1] = fma(y, y, v[1]);
  v[2] += g2;
  v[3] += g2y;
  v[4] = fma(g2y, y, v[4]);
}

__device__ __forceinline__ void gn_store(double* __restrict__ plane, int64_t p, const double (&v)[NC_SUMS]) {
#pragma unroll
  for (int q = 0; q < NC_SUMS; ++q) plane[p * NC_SUMS + q] = v[q];
}

// the other planes: block p = b * C + c walks its plane
template <typename TX, typename TG>
__global__ void __launch_bounds__(256) gn_plane_block_kernel(const TX* __restrict__ x, const TG* __restrict__ g,
                                                             int C, int Cg, int64_t S, double* __restrict__ plane) {
  const int64_t p = blockIdx.x;
  const int c = (int)(p % C);
  const double K = (double)to_float<TX>(x[(p - c % Cg) * S]);
  double v[NC_SUMS] = {0.0, 0.0, 0.0, 0.0, 0.0};
  const int64_t base = p * S;
#pragma unroll 4
  for (int64_t i = threadIdx.x; i < S; i += 256) gn_add(x, g, base + i, K, v);
  block_sum<NC_SUMS>(v);
  if (threadIdx.x == 0) gn_store(plane, p, v);
}

// S >= 2 with gn_warp_per_plane (7 x 7, 8 x 8, short sequences, or many mid-sized planes): one warp per plane, eight
// planes per block
template <typename TX, typename TG>
__global__ void __launch_bounds__(256) gn_plane_warp_kernel(const TX* __restrict__ x, const TG* __restrict__ g,
                                                            int64_t planes, int C, int Cg, int S,
                                                            double* __restrict__ plane) {
  const int64_t p = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (p >= planes) return;
  const int c = (int)(p % C);
  const double K = (double)to_float<TX>(x[(p - c % Cg) * S]);
  double v[NC_SUMS] = {0.0, 0.0, 0.0, 0.0, 0.0};
#pragma unroll 4
  for (int i = lane; i < S; i += 32) gn_add(x, g, p * S + i, K, v);
#pragma unroll
  for (int q = 0; q < NC_SUMS; ++q)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[q] += __shfl_xor_sync(0xffffffffu, v[q], o);
  if (lane == 0) gn_store(plane, p, v);
}

// S = 1 (GroupNorm on (B, C)): one thread per (b, c), coalesced over the channels
template <typename TX, typename TG>
__global__ void __launch_bounds__(256) gn_plane_flat_kernel(const TX* __restrict__ x, const TG* __restrict__ g,
                                                            int64_t planes, int C, int Cg,
                                                            double* __restrict__ plane) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= planes) return;
  const int c = (int)(p % C);
  const double K = (double)to_float<TX>(x[p - c % Cg]);
  double v[NC_SUMS] = {0.0, 0.0, 0.0, 0.0, 0.0};
  gn_add(x, g, p, K, v);
  gn_store(plane, p, v);
}

// one warp per (b, gi): (mean of y, 1 / sqrt(var + eps)) over the group's Cg * S elements
__global__ void __launch_bounds__(256) gn_group_stats_kernel(const double* __restrict__ plane, int64_t B, int groups,
                                                             int Cg, double n, double eps,
                                                             double2* __restrict__ stats) {
  const int64_t bg = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (bg >= B * groups) return;
  const double* pl = plane + bg * Cg * NC_SUMS;   // the group's planes are consecutive: (b * G + gi) * Cg + j
  double s0 = 0.0, s1 = 0.0;
  for (int j = lane; j < Cg; j += 32) {
    s0 += pl[(int64_t)j * NC_SUMS];
    s1 += pl[(int64_t)j * NC_SUMS + 1];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s0 += __shfl_xor_sync(0xffffffffu, s0, o);
    s1 += __shfl_xor_sync(0xffffffffu, s1, o);
  }
  if (lane == 0) {
    const double m = s0 / n;
    const double var = fmax(s1 / n - m * m, 0.0);
    stats[bg] = make_double2(m, 1.0 / sqrt(var + eps));
  }
}

// acc[c * k + .] += scale * F_c, the examples added in order
__global__ void gn_finalize_kernel(const double* __restrict__ plane, const double2* __restrict__ stats, int64_t B,
                                   int C, int Cg, int k, float scale, float* acc) {
  const int groups = C / Cg;
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < C; c += gridDim.x * blockDim.x) {
    const int gi = c / Cg;
    double fss = 0.0, fsb = 0.0, fbb = 0.0;
    for (int64_t b = 0; b < B; ++b) {
      const double2 st = stats[b * groups + gi];
      const double* v = plane + (b * C + c) * NC_SUMS;
      const double m = st.x, r = st.y;
      fss += (v[4] - 2.0 * m * v[3] + m * m * v[2]) * r * r;
      fsb += (v[3] - m * v[2]) * r;
      fbb += v[2];
    }
    const double s = (double)scale;
    if (k == 1) {
      acc[c] = __fadd_rn(acc[c], (float)(s * fss));
    } else {
      acc[3 * c] = __fadd_rn(acc[3 * c], (float)(s * fss));
      acc[3 * c + 1] = __fadd_rn(acc[3 * c + 1], (float)(s * fsb));
      acc[3 * c + 2] = __fadd_rn(acc[3 * c + 2], (float)(s * fbb));
    }
  }
}

struct GroupNormArgs {
  const void* x; const void* g;
  int64_t B; int C; int64_t S; int groups; int k; double eps; float scale; float* acc; void* ws;
};

static size_t group_norm_ws_bytes(int64_t B, int C, int groups) {
  return align_up((size_t)B * (size_t)C * NC_SUMS * sizeof(double), 256) +
         align_up((size_t)B * (size_t)groups * sizeof(double2), 256);
}

template <typename TX, typename TG>
static int launch_group_norm(const GroupNormArgs& a, cudaStream_t s) {
  const TX* x = (const TX*)a.x;
  const TG* g = (const TG*)a.g;
  const int Cg = a.C / a.groups;
  const int64_t planes = a.B * a.C;
  double* plane = (double*)a.ws;
  double2* stats = (double2*)((char*)a.ws + align_up((size_t)planes * NC_SUMS * sizeof(double), 256));
  if (a.S == 1) {
    gn_plane_flat_kernel<TX, TG><<<(unsigned)ceil_div(planes, 256), 256, 0, s>>>(x, g, planes, a.C, Cg, plane);
  } else if (gn_warp_per_plane(planes, a.S)) {
    gn_plane_warp_kernel<TX, TG><<<(unsigned)ceil_div(planes, 8), 256, 0, s>>>(x, g, planes, a.C, Cg, (int)a.S,
                                                                                plane);
  } else {
    gn_plane_block_kernel<TX, TG><<<(unsigned)planes, 256, 0, s>>>(x, g, a.C, Cg, a.S, plane);
  }
  KFAC_LAUNCH_CHECK();
  gn_group_stats_kernel<<<(unsigned)ceil_div(a.B * a.groups, 8), 256, 0, s>>>(plane, a.B, a.groups, Cg,
                                                                               (double)Cg * (double)a.S, a.eps, stats);
  KFAC_LAUNCH_CHECK();
  gn_finalize_kernel<<<norm_grid_for(a.C), 256, 0, s>>>(plane, stats, a.B, a.C, Cg, a.k, a.scale, a.acc);
  KFAC_LAUNCH_CHECK();
  return KFAC_OK;
}

template <typename TX>
static int launch_group_norm_g(const GroupNormArgs& a, int g_dtype, cudaStream_t s) {
  if (g_dtype == KFAC_F32) return launch_group_norm<TX, float>(a, s);
  if (g_dtype == KFAC_F16) return launch_group_norm<TX, __half>(a, s);
  return launch_group_norm<TX, __nv_bfloat16>(a, s);
}

// ---------------------------------------------------------------- launch
struct NormArgs {
  const void* x; const void* g;
  int kind; int64_t rows; int C; int64_t S; int k; double eps; float scale; float* acc; void* ws;
};

static size_t norm_ws_bytes(int kind, int64_t rows, int C, int64_t S) {
  if (kind == KFAC_NORM_BATCH)
    return align_up((size_t)nc_chunks(rows, C, S) * (size_t)C * NC_SUMS * sizeof(double), 256);
  return align_up((size_t)rows * sizeof(double2), 256) +
         align_up((size_t)row_chunks(rows) * (size_t)C * ROW_SUMS * sizeof(double), 256);
}

template <typename TX, typename TG>
static int launch_norm(const NormArgs& a, cudaStream_t s) {
  const TX* x = (const TX*)a.x;
  const TG* g = (const TG*)a.g;
  if (a.kind == KFAC_NORM_BATCH) {
    const int64_t chunks = nc_chunks(a.rows, a.C, a.S), chunk_rows = (a.rows + chunks - 1) / chunks;
    double* partial = (double*)a.ws;
    if (a.S == 1) {
      bn_flat_kernel<TX, TG><<<dim3((unsigned)ceil_div(a.C, 256), (unsigned)chunks), 256, 0, s>>>(
          x, g, a.rows, a.C, chunk_rows, partial);
    } else {
      bn_spatial_kernel<TX, TG><<<dim3((unsigned)a.C, (unsigned)chunks), 256, 0, s>>>(x, g, a.rows, a.C, a.S,
                                                                                       chunk_rows, partial);
    }
    KFAC_LAUNCH_CHECK();
    bn_finalize_kernel<<<norm_grid_for(a.C), 256, 0, s>>>(partial, (int)chunks, a.C, (double)(a.rows * a.S), a.eps,
                                                          a.k, a.scale, a.acc);
    KFAC_LAUNCH_CHECK();
    return KFAC_OK;
  }
  const int64_t chunks = row_chunks(a.rows), chunk_rows = (a.rows + chunks - 1) / chunks;
  double2* stats = (double2*)a.ws;
  double* partial = (double*)((char*)a.ws + align_up((size_t)a.rows * sizeof(double2), 256));
  row_stats_kernel<TX><<<norm_grid_for(a.rows * 32), 256, 0, s>>>(x, a.rows, a.C, a.kind == KFAC_NORM_RMS, a.eps,
                                                                   stats);
  KFAC_LAUNCH_CHECK();
  row_cols_kernel<TX, TG><<<dim3((unsigned)ceil_div(a.C, 256), (unsigned)chunks), 256, 0, s>>>(
      x, g, stats, a.rows, a.C, chunk_rows, partial);
  KFAC_LAUNCH_CHECK();
  row_finalize_kernel<<<norm_grid_for(a.C), 256, 0, s>>>(partial, (int)chunks, a.C, a.k, a.scale, a.acc);
  KFAC_LAUNCH_CHECK();
  return KFAC_OK;
}

template <typename TX>
static int launch_norm_g(const NormArgs& a, int g_dtype, cudaStream_t s) {
  if (g_dtype == KFAC_F32) return launch_norm<TX, float>(a, s);
  if (g_dtype == KFAC_F16) return launch_norm<TX, __half>(a, s);
  return launch_norm<TX, __nv_bfloat16>(a, s);
}

// ================================================================ precondition
// P_c = (F_c + damping I)^-1 grad_c for every channel of every item, in fp64: one thread per channel.
struct NormDev { const float* F; const void* w; const void* b; int dtype, C, k; float* P; long long c0; };

__global__ void __launch_bounds__(256) norm_precondition_kernel(const NormDev* items, int count, long long total,
                                                                float damping) {
  const double lam = (double)damping;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total;
       e += (long long)gridDim.x * blockDim.x) {
    int lo = 0, hi = count - 1;
    while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (items[mid].c0 <= e) lo = mid; else hi = mid - 1; }
    const NormDev& it = items[lo];
    const int c = (int)(e - it.c0);
    const double gs = (double)load_as_float(it.w, it.dtype, c);
    if (it.k == 1) {
      it.P[c] = (float)(gs / ((double)it.F[c] + lam));
      continue;
    }
    const double gb = (double)load_as_float(it.b, it.dtype, c);
    const double fss = (double)it.F[3 * c] + lam, fsb = (double)it.F[3 * c + 1], fbb = (double)it.F[3 * c + 2] + lam;
    const double det = fss * fbb - fsb * fsb;
    it.P[2 * c] = (float)((fbb * gs - fsb * gb) / det);
    it.P[2 * c + 1] = (float)((fss * gb - fsb * gs) / det);
  }
}

}  // namespace kfac

using namespace kfac;

extern "C" size_t kfac_factor_norm_workspace_bytes(int kind, int64_t rows, int C, int64_t S) {
  if (rows <= 0 || C <= 0 || S <= 0) return 0;
  if (kind != KFAC_NORM_BATCH && kind != KFAC_NORM_LAYER && kind != KFAC_NORM_RMS) return 0;
  if (kind != KFAC_NORM_BATCH && S != 1) return 0;
  return norm_ws_bytes(kind, rows, C, S);
}

extern "C" int kfac_factor_norm(const void* x, int x_dtype, const void* g, int g_dtype, int kind, int64_t rows, int C,
                                int64_t S, int k, double eps, float scale, float* acc, void* ws, size_t ws_bytes,
                                void* stream) {
  KFAC_CHECK_ARG(acc && C > 0 && rows >= 0 && S > 0 && ((x && g) || rows == 0), "factor_norm args");
  KFAC_CHECK_ARG(kind == KFAC_NORM_BATCH || kind == KFAC_NORM_LAYER || kind == KFAC_NORM_RMS, "norm kind");
  KFAC_CHECK_ARG(kind == KFAC_NORM_BATCH || S == 1, "LayerNorm / RMSNorm take S = 1");
  KFAC_CHECK_ARG(k == 1 || k == 3, "k must be 1 or 3");
  KFAC_CHECK_ARG(kind != KFAC_NORM_RMS || k == 1, "RMSNorm has no bias (k = 1)");
  KFAC_CHECK_ARG(eps >= 0.0, "eps");
  for (int d : {x_dtype, g_dtype}) KFAC_CHECK_ARG(d == KFAC_F32 || d == KFAC_F16 || d == KFAC_BF16, "dtype");
  KFAC_CHECK_ARG(rows * S < (1ll << 31), "more than 2^31 rows per channel");
  if (rows == 0) return KFAC_OK;
  const size_t need = kfac_factor_norm_workspace_bytes(kind, rows, C, S);
  if (!ws || ws_bytes < need) {
    set_error("factor_norm: workspace too small (%zu < %zu)", ws_bytes, need);
    return KFAC_ERR_WORKSPACE;
  }
  const NormArgs a{x, g, kind, rows, C, S, k, eps, scale, acc, ws};
  cudaStream_t s = (cudaStream_t)stream;
  if (x_dtype == KFAC_F32) return launch_norm_g<float>(a, g_dtype, s);
  if (x_dtype == KFAC_F16) return launch_norm_g<__half>(a, g_dtype, s);
  return launch_norm_g<__nv_bfloat16>(a, g_dtype, s);
}

extern "C" size_t kfac_factor_group_norm_workspace_bytes(int64_t B, int C, int64_t S, int groups) {
  if (B <= 0 || C <= 0 || S <= 0 || groups <= 0 || C % groups != 0) return 0;
  return group_norm_ws_bytes(B, C, groups);
}

extern "C" int kfac_factor_group_norm(const void* x, int x_dtype, const void* g, int g_dtype, int64_t B, int C,
                                      int64_t S, int groups, int k, double eps, float scale, float* acc, void* ws,
                                      size_t ws_bytes, void* stream) {
  KFAC_CHECK_ARG(acc && C > 0 && B >= 0 && S > 0 && ((x && g) || B == 0), "factor_group_norm args");
  KFAC_CHECK_ARG(groups > 0 && C % groups == 0, "groups must divide the channels");
  KFAC_CHECK_ARG(k == 1 || k == 3, "k must be 1 or 3");
  KFAC_CHECK_ARG(eps >= 0.0, "eps");
  for (int d : {x_dtype, g_dtype}) KFAC_CHECK_ARG(d == KFAC_F32 || d == KFAC_F16 || d == KFAC_BF16, "dtype");
  KFAC_CHECK_ARG(B * (int64_t)C * S < (1ll << 31), "2^31 or more elements");
  if (B == 0) return KFAC_OK;
  const size_t need = kfac_factor_group_norm_workspace_bytes(B, C, S, groups);
  if (!ws || ws_bytes < need) {
    set_error("factor_group_norm: workspace too small (%zu < %zu)", ws_bytes, need);
    return KFAC_ERR_WORKSPACE;
  }
  const GroupNormArgs a{x, g, B, C, S, groups, k, eps, scale, acc, ws};
  cudaStream_t s = (cudaStream_t)stream;
  if (x_dtype == KFAC_F32) return launch_group_norm_g<float>(a, g_dtype, s);
  if (x_dtype == KFAC_F16) return launch_group_norm_g<__half>(a, g_dtype, s);
  return launch_group_norm_g<__nv_bfloat16>(a, g_dtype, s);
}

extern "C" size_t kfac_norm_precondition_workspace_bytes(int count) {
  return count > 0 ? align_up((size_t)count * sizeof(NormDev), 256) : 0;
}

extern "C" int kfac_norm_precondition(const kfac_norm_item* items, int count, float damping, void* ws,
                                      size_t ws_bytes, void* stream) {
  KFAC_CHECK_ARG(count >= 0 && (items || count == 0), "norm_precondition args");
  if (count == 0) return KFAC_OK;
  const size_t need = kfac_norm_precondition_workspace_bytes(count);
  if (!ws || ws_bytes < need) {
    set_error("norm_precondition: workspace too small (%zu < %zu)", ws_bytes, need);
    return KFAC_ERR_WORKSPACE;
  }
  std::vector<NormDev> dev(count);
  long long total = 0;
  for (int i = 0; i < count; ++i) {   // every item is checked before anything is launched
    const kfac_norm_item& it = items[i];
    KFAC_CHECK_ARG(it.F && it.wgrad && it.P && it.C > 0 && (it.k == 1 || it.k == 3), "norm item");
    KFAC_CHECK_ARG((it.k == 3) == (it.bgrad != nullptr), "norm item: bgrad must be given exactly when k = 3");
    KFAC_CHECK_ARG(it.grad_dtype == KFAC_F32 || it.grad_dtype == KFAC_F16 || it.grad_dtype == KFAC_BF16, "dtype");
    dev[i] = NormDev{it.F, it.wgrad, it.bgrad, it.grad_dtype, it.C, it.k, it.P, total};
    total += it.C;
  }
  cudaStream_t s = (cudaStream_t)stream;
  KFAC_CUDA(cudaMemcpyAsync(ws, dev.data(), sizeof(NormDev) * count, cudaMemcpyHostToDevice, s));   // pageable: staged
  norm_precondition_kernel<<<norm_grid_for(total), 256, 0, s>>>((const NormDev*)ws, count, total, damping);
  KFAC_LAUNCH_CHECK();
  return KFAC_OK;
}
