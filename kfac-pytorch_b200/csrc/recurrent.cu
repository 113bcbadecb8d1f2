// Rows of the recurrent layers (nn.RNN / nn.LSTM / nn.GRU, opt-in through precondition_recurrent), read in place from
// the tensors the taps of the restated forward see.
//
//   rows    one row per position (t, b), in time-major (t * B + b) or packed (offsets[t] + b) order     a CTA per
//           (time step, chunk of that step's rows)
//   reduce  one row per sequence b: the sum over its R_b positions times scale * R_b^-power              a CTA per
//           (sequence, 32 columns)
//
// A position's source row is described by kfac_sequence_rows (include/kfac_b200.h): the row itself, or the previous
// hidden state of a direction -- h_{t-1} forward, h_{t+1} reverse, h0 where the sequence starts -- gathered from the
// layer output and h0, optionally times a per-position multiplier over the trailing columns (GRU: r * dn).  The
// existing writers address a row by one flat index; these rows are addressed by (t, b) with a per-step batch size.
// The reduce sums keep reduce_linear_kernel's order (fp32 runs of 16, then fp64, warps added in order): no atomics, the
// same bits on every run.
#include "common.cuh"

#include <cmath>

namespace kfac {
namespace {

constexpr int RUN = 16;

struct Seq {
  const void* x; int64_t ldx; int col0;
  const void* h0; int64_t ldh; int shift;
  const void* mul; int64_t ldm; int mul_col0;
  int T, B; const int* off;

  __device__ __forceinline__ int64_t row0(int t) const { return off ? (int64_t)off[t] : (int64_t)t * B; }
  __device__ __forceinline__ int bs(int t) const { return off ? off[t + 1] - off[t] : B; }
  // steps of sequence b: the first t whose batch size is <= b (batch sizes do not increase)
  __device__ __forceinline__ int length(int b) const {
    if (!off) return T;
    int lo = 0, hi = T;
    while (lo < hi) {
      const int m = (lo + hi) >> 1;
      if (bs(m) > b) lo = m + 1; else hi = m;
    }
    return lo;
  }
  // element offset of the source row of position (t, b) in x, or -1 - (offset in h0)
  __device__ __forceinline__ int64_t source(int t, int b) const {
    if (shift > 0) return t == 0 ? -1 - (int64_t)b * ldh : (row0(t - 1) + b) * ldx + col0;
    if (shift < 0) return (t + 1 < T && b < bs(t + 1)) ? (row0(t + 1) + b) * ldx + col0 : -1 - (int64_t)b * ldh;
    return (row0(t) + b) * ldx + col0;
  }
  template <typename T_>
  __device__ __forceinline__ float value(int64_t src, int64_t pos, int f) const {
    const T_* __restrict__ p = src >= 0 ? reinterpret_cast<const T_*>(x) + src
                                        : reinterpret_cast<const T_*>(h0) + (-1 - src);
    float v = to_float<T_>(p[f]);
    if (mul && f >= mul_col0) v *= to_float<T_>(reinterpret_cast<const T_*>(mul)[pos * ldm + (f - mul_col0)]);
    return v;
  }
};

__device__ __forceinline__ float row_scale(float scale, const float* loss_scale) {
  return loss_scale ? scale / *loss_scale : scale;
}

// out[row(t, b)][f] = s * value (f < feat), s (f == feat, ones), 0 up to ld: kfac_rows_linear's values
template <typename T>
__global__ void __launch_bounds__(256) seq_rows_kernel(const Seq q, int feat, int ones, float scale,
                                                       const float* loss_scale, float* out, int64_t ld) {
  const int t = blockIdx.x;
  const float s = row_scale(scale, loss_scale);
  const int64_t r0 = q.row0(t), total = (int64_t)q.bs(t) * ld;
  for (int64_t idx = (int64_t)blockIdx.y * blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.y * blockDim.x) {
    const int b = (int)(idx / ld);
    const int f = (int)(idx - (int64_t)b * ld);
    float v = 0.f;
    if (f < feat) v = q.value<T>(q.source(t, b), r0 + b, f) * s;
    else if (f == feat && ones) v = s;
    out[(r0 + b) * ld + f] = v;
  }
}

// out[b][f] = scale * R_b^-power / *loss_scale * sum_{t < R_b} value(t, b, f); the ones column is R_b times that factor
template <typename T>
__global__ void __launch_bounds__(256) seq_reduce_kernel(const Seq q, int feat, int ones, float scale, float power,
                                                         const float* loss_scale, float* out, int64_t ld, int tiles) {
  __shared__ double part[8][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int b = blockIdx.x / tiles;
  const int f = (blockIdx.x % tiles) * 32 + lane;
  const int R = q.length(b);
  double acc = 0.0;
  if (f < feat) {
    for (int t0 = warp; t0 < R; t0 += 8 * RUN) {
      float s = 0.f;
#pragma unroll
      for (int k = 0; k < RUN; ++k) {
        const int t = t0 + 8 * k;
        if (t < R) s += q.value<T>(q.source(t, b), q.row0(t) + b, f);
      }
      acc += (double)s;
    }
  }
  part[warp][lane] = acc;
  __syncthreads();
  if (warp != 0 || f >= ld) return;
  double sc = (double)scale * pow((double)R, -(double)power);
  if (loss_scale) sc /= (double)*loss_scale;
  float v = 0.f;
  if (f < feat) {
    double t = part[0][lane];
#pragma unroll
    for (int w = 1; w < 8; ++w) t += part[w][lane];
    v = (float)(t * sc);
  } else if (f == feat && ones) {
    v = (float)((double)R * sc);
  }
  out[(int64_t)b * ld + f] = v;
}

int check_seq(const kfac_sequence_rows* src, int features, int ones, int64_t ld_out) {
  KFAC_CHECK_ARG(src && src->x, "null pointer");
  KFAC_CHECK_ARG(src->T > 0 && src->B > 0 && features > 0, "dims");
  KFAC_CHECK_ARG(src->col0 >= 0 && src->ldx >= src->col0 + features, "ldx");
  KFAC_CHECK_ARG(src->shift >= -1 && src->shift <= 1, "shift");
  KFAC_CHECK_ARG(src->shift == 0 || (src->h0 && src->ldh >= features), "h0");
  KFAC_CHECK_ARG(!src->mul || (src->mul_col0 >= 0 && src->mul_col0 <= features &&
                               src->ldm >= features - src->mul_col0), "mul");
  KFAC_CHECK_ARG((int64_t)src->T * src->B < (1ll << 31), "rows overflow");
  KFAC_CHECK_ARG(ld_out >= features + ones, "ld_out");
  return KFAC_OK;
}

Seq make_seq(const kfac_sequence_rows* s) {
  return Seq{s->x, s->ldx, s->col0, s->h0, s->ldh, s->shift, s->mul, s->ldm, s->mul_col0, s->T, s->B, s->offsets};
}

}  // namespace
}  // namespace kfac

using namespace kfac;

extern "C" int kfac_rows_sequence(const kfac_sequence_rows* src, int dtype, int features, int append_ones, float scale,
                                  const float* loss_scale, float* out, int ld_out, void* stream) {
  const int ones = append_ones ? 1 : 0;
  if (int rc = check_seq(src, features, ones, ld_out)) return rc;
  KFAC_CHECK_ARG(out, "null pointer");
  const Seq q = make_seq(src);
  // a CTA moves up to 16 elements per thread; the steps of one sequence run side by side in blockIdx.x
  const int64_t per_step = (int64_t)src->B * ld_out;
  const dim3 grid((unsigned)src->T, (unsigned)std::min<int64_t>(65535, std::max<int64_t>(1, ceil_div(per_step, 4096))));
  cudaStream_t s = (cudaStream_t)stream;
  if (dtype == KFAC_F32) seq_rows_kernel<float><<<grid, 256, 0, s>>>(q, features, ones, scale, loss_scale, out, ld_out);
  else if (dtype == KFAC_F16) seq_rows_kernel<__half><<<grid, 256, 0, s>>>(q, features, ones, scale, loss_scale, out, ld_out);
  else if (dtype == KFAC_BF16)
    seq_rows_kernel<__nv_bfloat16><<<grid, 256, 0, s>>>(q, features, ones, scale, loss_scale, out, ld_out);
  else { set_error("unknown dtype %d", dtype); return KFAC_ERR_BAD_ARG; }
  KFAC_LAUNCH_CHECK();
  return KFAC_OK;
}

extern "C" int kfac_reduce_rows_sequence(const kfac_sequence_rows* src, int dtype, int features, int append_ones,
                                         float scale, float power, const float* loss_scale, float* out, int ld_out,
                                         void* stream) {
  const int ones = append_ones ? 1 : 0;
  if (int rc = check_seq(src, features, ones, ld_out)) return rc;
  KFAC_CHECK_ARG(out, "null pointer");
  const int tiles = ceil_div(ld_out, 32);
  KFAC_CHECK_ARG((int64_t)src->B * tiles < (1ll << 31), "grid");
  const Seq q = make_seq(src);
  const unsigned grid = (unsigned)(src->B * tiles);
  cudaStream_t s = (cudaStream_t)stream;
  if (dtype == KFAC_F32)
    seq_reduce_kernel<float><<<grid, 256, 0, s>>>(q, features, ones, scale, power, loss_scale, out, ld_out, tiles);
  else if (dtype == KFAC_F16)
    seq_reduce_kernel<__half><<<grid, 256, 0, s>>>(q, features, ones, scale, power, loss_scale, out, ld_out, tiles);
  else if (dtype == KFAC_BF16)
    seq_reduce_kernel<__nv_bfloat16><<<grid, 256, 0, s>>>(q, features, ones, scale, power, loss_scale, out, ld_out,
                                                          tiles);
  else { set_error("unknown dtype %d", dtype); return KFAC_ERR_BAD_ARG; }
  KFAC_LAUNCH_CHECK();
  return KFAC_OK;
}
