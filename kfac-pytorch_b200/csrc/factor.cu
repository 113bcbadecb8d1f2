// K1-K4: Kronecker-factor statistics (A = a^T a, G = g^T g), EMA, packing.
//
// Data layout in HBM: every factor is a dense d x d fp32 row-major matrix that
// lives inside one contiguous arena owned by the Python side (so the factor
// all-reduce is ONE collective over the arena).  Activations / grad-outputs
// are read in their native NCHW / (rows, features) layout.
#include "common.cuh"

#include <cfloat>
#include <string.h>

#include <algorithm>
#include <type_traits>

namespace kfac {

constexpr int CT = 64;   // covariance output tile
constexpr int CK = 16;   // reduction chunk

struct CovArgs {
  const void* x;
  int64_t ld;          // SAMPLE_MAJOR: row stride ; FEATURE_MAJOR: feature stride
  int64_t batch_stride;
  int rows;            // samples per batch entry
  int batch;
  int feat;            // real features (without the ones column)
  int ones;            // append a constant-one feature
  int splits;          // splits of the sample range (all batch entries, flattened)
  float scale;
  float* acc;          // d x d, d = feat + ones
  float* slab;         // splits x d x d partials (upper tiles), required when splits > 1
};

// acc += scale * X^T X over upper-triangular 64x64 tiles (mirrored).  The reduction over the samples of all batch
// entries is split across CTAs; split sp stores its partial tile into slab sp and cov_reduce_kernel adds the slabs
// in a fixed order (every run gives the same bits).  With one split the CTA is the only writer of its tile.
template <typename T, bool FEATURE_MAJOR>
__global__ void __launch_bounds__(256) cov_kernel(CovArgs a) {
  __shared__ __align__(16) float As[CK][CT + 4];
  __shared__ __align__(16) float Bs[CK][CT + 4];
  const int d = a.feat + a.ones;
  const int nt = (d + CT - 1) / CT;
  // decode upper-triangular tile index
  int t = blockIdx.x, tm = 0;
  while (t >= nt - tm) { t -= nt - tm; ++tm; }
  const int tn = tm + t;
  const int sp = blockIdx.y;
  const int64_t total = (int64_t)a.rows * a.batch;
  int64_t chunk = (total + a.splits - 1) / a.splits;
  chunk = (chunk + CK - 1) / CK * CK;
  const int64_t r_begin = sp * chunk, r_end = min(total, r_begin + chunk);
  const T* __restrict__ xb = reinterpret_cast<const T*>(a.x);
  const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
  const int m0 = tm * CT, n0 = tn * CT;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int64_t r0 = r_begin; r0 < r_end; r0 += CK) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      int f, r;
      if (FEATURE_MAJOR) { r = tid % 16; f = tid / 16 + 16 * i; }
      else               { f = tid % 64; r = tid / 64 + 4 * i; }
      const bool rv = (r0 + r) < r_end;
      float va = 0.f, vb = 0.f;
      const int fa = m0 + f, fb = n0 + f;
      if (rv) {
        // flattened sample index -> (batch entry, row)
        const int64_t q = r0 + r;
        const int b = a.batch > 1 ? (int)(q / a.rows) : 0;
        const int64_t rr = q - (int64_t)b * a.rows;
        const T* __restrict__ x = xb + (int64_t)b * a.batch_stride;
        if (fa < a.feat)
          va = to_float<T>(FEATURE_MAJOR ? x[(int64_t)fa * a.ld + rr]
                                         : x[rr * a.ld + fa]);
        else if (fa < d) va = 1.f;
        if (tn != tm) {
          if (fb < a.feat)
            vb = to_float<T>(FEATURE_MAJOR ? x[(int64_t)fb * a.ld + rr]
                                           : x[rr * a.ld + fb]);
          else if (fb < d) vb = 1.f;
        }
      }
      As[r][f] = va;
      if (tn != tm) Bs[r][f] = vb;
    }
    __syncthreads();
    const float (*Bp)[CT + 4] = (tn != tm) ? Bs : As;
#pragma unroll
    for (int k = 0; k < CK; ++k) {
      const float4 a4 = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      const float4 b4 = *reinterpret_cast<const float4*>(&Bp[k][tx * 4]);
      const float av[4] = {a4.x, a4.y, a4.z, a4.w};
      const float bv[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= d) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= d) continue;
      const float v = a.scale * acc[i][j];
      if (a.splits > 1) {
        a.slab[(int64_t)sp * d * d + (int64_t)m * d + n] = v;
      } else {
        a.acc[(int64_t)m * d + n] += v;
        if (tn != tm) a.acc[(int64_t)n * d + m] += v;
      }
    }
  }
}

// acc[i][j] += sum_sp slab[sp][min(i,j)][max(i,j)], splits added in a fixed order
__global__ void cov_reduce_kernel(const float* __restrict__ slab, int splits, int d, float* acc) {
  const int64_t dd = (int64_t)d * d;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < dd; idx += (int64_t)gridDim.x * blockDim.x) {
    const int i = (int)(idx / d), j = (int)(idx - (int64_t)i * d);
    const int64_t src = i <= j ? idx : (int64_t)j * d + i;
    float t = slab[src];
    for (int sp = 1; sp < splits; ++sp) t += slab[sp * dd + src];
    acc[idx] += t;
  }
}

// split plans of the two covariance paths (shared by the launches and the workspace sizes)
static int cov_tc_splits(int d, int64_t rows, int batch) {
  const int nt = ceil_div(d, 128), ntiles = nt * (nt + 1) / 2;
  const int kb_total = ceil_div(rows, 32) * batch;
  const int num_sms = tc_num_sms();
  int splits = 1;
  if (ntiles < num_sms) splits = std::max(1, std::min(num_sms / ntiles, kb_total / 8));
  return tc_normalize_splits(splits, kb_total);
}
static int cov_simt_splits(int d, int64_t rows, int batch) {
  const int nt = ceil_div(d, CT), tiles = nt * (nt + 1) / 2;
  const int64_t total = rows * batch;
  int splits = ceil_div((int64_t)tc_num_sms() * 3, tiles);
  return (int)std::max<int64_t>(1, std::min<int64_t>(splits, ceil_div(total, 4 * CK)));
}
// bytes of the split partials: the larger of the two paths (the tensor-core path also depends on alignment)
static size_t cov_slab_bytes(int d, int64_t rows, int batch) {
  const int s = std::max(cov_tc_splits(d, rows, batch), cov_simt_splits(d, rows, batch));
  return s > 1 ? (size_t)s * d * d * sizeof(float) : 0;
}

static int cov_reduce(const CovArgs& a, int d, int splits, cudaStream_t s) {
  const int blocks = (int)std::min<int64_t>(ceil_div((int64_t)d * d, 256), (int64_t)tc_num_sms() * 16);
  cov_reduce_kernel<<<blocks, 256, 0, s>>>(a.slab, splits, d, a.acc);
  KFAC_LAUNCH_CHECK();
  return KFAC_OK;
}

// a.slab (cov_slab_bytes) lets long reductions be split over the SMs; without it they run as one split
template <bool FEATURE_MAJOR>
static int launch_cov(CovArgs a, int dtype, cudaStream_t s) {
  const int d = a.feat + a.ones;
  if (d <= 0 || a.rows <= 0 || a.batch <= 0) return KFAC_OK;
  if (FEATURE_MAJOR && dtype == KFAC_F32 && a.ones == 0 && d >= 64 && (int64_t)a.rows * a.batch >= 256) {
    // tensor-core SYRK: X (features x samples) is a K-major operand as it lies in HBM;
    // upper-triangular tiles only, split over the samples into per-split partials.
    TcGemmArgs t{};
    t.A = (const float*)a.x; t.lda = a.ld; t.B = t.A; t.ldb = a.ld;
    t.D = a.acc; t.ldd = d; t.M = d; t.N = d; t.K = a.rows;
    t.kbatch = a.batch; t.a_kb_stride = a.batch_stride; t.b_kb_stride = a.batch_stride;
    t.upper_only = 1; t.alpha = a.scale;
    if (tc_gemm_supported(t)) {
      const int splits = a.slab ? cov_tc_splits(d, a.rows, a.batch) : 1;
      if (splits > 1) { t.slab = a.slab; t.slab_stride = (int64_t)d * d; t.splits = splits; }
      else { t.accumulate = 1; t.splits = 1; }
      const int rc = launch_tc_gemm(t, s);
      if (rc || splits == 1) return rc;
      return cov_reduce(a, d, splits, s);
    }
  }
  const int nt = ceil_div(d, CT);
  const int tiles = nt * (nt + 1) / 2;
  a.splits = a.slab ? cov_simt_splits(d, a.rows, a.batch) : 1;
  dim3 grid(tiles, a.splits);
  if (dtype == KFAC_F32) cov_kernel<float, FEATURE_MAJOR><<<grid, 256, 0, s>>>(a);
  else if (dtype == KFAC_F16) cov_kernel<__half, FEATURE_MAJOR><<<grid, 256, 0, s>>>(a);
  else if (dtype == KFAC_BF16) cov_kernel<__nv_bfloat16, FEATURE_MAJOR><<<grid, 256, 0, s>>>(a);
  else { set_error("unknown dtype %d", dtype); return KFAC_ERR_BAD_ARG; }
  KFAC_LAUNCH_CHECK();
  return a.splits > 1 ? cov_reduce(a, d, a.splits, s) : KFAC_OK;
}

// N-d, dilated im2col into a FEATURE-major fp32 matrix: out[(c,l,i,j)][(n,do,ho,wo)]
struct Im2colArgs {
  const void* x; float* out;
  ConvGeo g;
  int ones;        // append a feature row of ones
  int64_t ld;      // leading dimension of the feature-major output (>= rows, multiple of 4)
};
// grid (ceil(ld / 4 / 256), features [+ 1]): a thread writes 4 consecutive samples of one feature row with one 16-byte
// store; the (image, do, ho, wo) decomposition is done once per thread in 32-bit arithmetic and advanced incrementally
// (the element-wise version spent its time in 64-bit divisions: 480 us for a 231 MB matrix, now bandwidth bound).
// TRANSPOSED: the index map of a transposed convolution (TapMap); a tap between two inputs is an exact zero.
template <typename T, bool TRANSPOSED = false>
__global__ void __launch_bounds__(256) im2col_kernel(Im2colArgs a) {
  using Tap = TapMap<TRANSPOSED>;
  const ConvGeo& g = a.g;
  const int64_t rows = (int64_t)g.batch * g.Do * g.Ho * g.Wo;
  const int nfeat = g.C * g.kd * g.kh * g.kw;
  const int f = blockIdx.y;
  const int64_t r4 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (r4 >= a.ld) return;
  float v[4] = {0.f, 0.f, 0.f, 0.f};
  if (f >= nfeat) {
#pragma unroll
    for (int k = 0; k < 4; ++k) v[k] = (r4 + k < rows) ? 1.f : 0.f;
  } else if (r4 < rows) {
    const T* __restrict__ x = reinterpret_cast<const T*>(a.x);
    const int j = f % g.kw, i = (f / g.kw) % g.kh, fl = f / (g.kw * g.kh);
    const int l = fl % g.kd, c = fl / g.kd;
    const unsigned row = (unsigned)r4;                    // rows < 2^31 (checked by the caller)
    int wo = (int)(row % (unsigned)g.Wo);
    unsigned t = row / (unsigned)g.Wo;
    int ho = (int)(t % (unsigned)g.Ho);
    t /= (unsigned)g.Ho;
    int dz = (int)(t % (unsigned)g.Do), n = (int)(t / (unsigned)g.Do);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (r4 + k < rows) {
        const int z = Tap::input(dz, l, g.sd, g.dd, g.pd, g.D), h = Tap::input(ho, i, g.sh, g.dh, g.ph, g.H),
                  w = Tap::input(wo, j, g.sw, g.dw, g.pw, g.W);
        if ((z | h | w) >= 0) v[k] = to_float<T>(x[((((int64_t)n * g.C + c) * g.D + z) * g.H + h) * g.W + w]);
      }
      if (++wo == g.Wo) { wo = 0; if (++ho == g.Ho) { ho = 0; if (++dz == g.Do) { dz = 0; ++n; } } }
    }
  }
  *reinterpret_cast<float4*>(a.out + (int64_t)f * a.ld + r4) = make_float4(v[0], v[1], v[2], v[3]);
}

// X (rows x feat, sample-major with row stride ldx >= feat, any dtype) -> out (feat [+1 ones row]) x ld, feature-major
// fp32
template <typename T>
__global__ void to_feature_major_kernel(const void* xin, int64_t rows, int feat, int64_t ldx, int ones, float* out,
                                        int64_t ld) {
  __shared__ float tile[32][33];
  const T* __restrict__ x = reinterpret_cast<const T*>(xin);
  const int64_t r0 = (int64_t)blockIdx.x * 32;
  const int f0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int64_t r = r0 + i;
    const int f = f0 + threadIdx.x;
    tile[i][threadIdx.x] = (r < rows && f < feat) ? to_float<T>(x[r * ldx + f]) : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int f = f0 + i;
    const int64_t r = r0 + threadIdx.x;
    if (r < ld) {
      if (f < feat) out[(int64_t)f * ld + r] = tile[threadIdx.x][i];
      else if (f == feat && ones) out[(int64_t)f * ld + r] = (r < rows) ? 1.f : 0.f;
    }
  }
}

// ------------------------------------------------------------------ EMA
// factor = alpha * (first ? I : factor) + (1 - alpha) * inv_count * (batch + batch^T) / 2, batch = 0.
// A CTA owns the pair of 32 x 32 tiles (ti, tj) / (tj, ti): both are read and written row-wise, the
// transposition happens in shared memory (every access is coalesced: 5 x 4 d^2 bytes at HBM speed).
struct EmaBatch {
  kfac_ema_item it[40];
  int first_block[41];   // prefix sums of the number of tile pairs T (T + 1) / 2 per item
  int count;
  float alpha;
  // guarded EMA only: per-item loss scale (NULL = 1), drop flags set by window_scan_kernel, drop counter
  const float* scale[40];
  const int* dropped;
  unsigned long long* skipped;
};

// 1/s^2 of a loss scale, formed as (1/s)^2: exact for the powers of two a GradScaler uses, and still normal for
// scales up to 2^63 (s * s would overflow first).  A non-finite or zero scale gives a non-finite or zero factor,
// which makes every non-zero window entry non-finite, so the window is dropped.
__device__ __forceinline__ float window_unscale(const float* s) {
  if (s == nullptr) return 1.f;
  const float r = 1.f / *s;
  return r * r;
}

// alpha * f + beta * (x + y), rounded as fma(beta, x + y, alpha * f).  Spelled out so that the compiler cannot contract
// it differently in the two instantiations of ema_kernel: the guarded EMA must give the bits of the unguarded one.
__device__ __forceinline__ float ema_update(float alpha, float f, float beta, float x, float y) {
  return __fmaf_rn(beta, __fadd_rn(x, y), __fmul_rn(alpha, f));
}

// GUARD = false: kfac_factor_ema.  GUARD = true: the window is multiplied by window_unscale() as it is read, and a
// window flagged by window_scan_kernel is dropped (factor unchanged, or I when it is the first window; batch = 0).
template <bool GUARD>
__global__ void __launch_bounds__(256) ema_kernel(const __grid_constant__ EmaBatch eb) {
  __shared__ float A[32][33], B[32][33];
  int item = 0;
  while (item + 1 < eb.count && (int)blockIdx.x >= eb.first_block[item + 1]) ++item;
  const kfac_ema_item it = eb.it[item];
  const int p = blockIdx.x - eb.first_block[item];
  // unrank the tile pair (ti <= tj) from p = tj (tj + 1) / 2 + ti
  int tj = (int)((sqrtf(8.f * (float)p + 1.f) - 1.f) * 0.5f);
  while ((tj + 1) * (tj + 2) / 2 <= p) ++tj;
  while (tj * (tj + 1) / 2 > p) --tj;
  const int ti = p - tj * (tj + 1) / 2;
  const int d = it.d, tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const float alpha = eb.alpha, beta = (1.f - eb.alpha) * it.inv_count * 0.5f;
  const int i0 = ti * 32, j0 = tj * 32;
  bool drop = false;
  float u = 1.f;
  if (GUARD) {
    drop = eb.dropped[item] != 0;
    u = window_unscale(eb.scale[item]);
    if (drop && p == 0 && threadIdx.x == 0 && eb.skipped) atomicAdd(eb.skipped, 1ull);
  }
#pragma unroll
  for (int r = ty; r < 32; r += 8) {
    const int iu = i0 + r, ju = j0 + tx;   // upper tile (ti, tj)
    float va = (iu < d && ju < d) ? it.batch[(int64_t)iu * d + ju] : 0.f;
    const int il = j0 + r, jl = i0 + tx;   // mirror tile (tj, ti)
    float vb = (il < d && jl < d) ? it.batch[(int64_t)il * d + jl] : 0.f;
    if (GUARD) { va *= u; vb *= u; }
    A[r][tx] = va;
    B[r][tx] = vb;
  }
  __syncthreads();
#pragma unroll
  for (int r = ty; r < 32; r += 8) {
    {
      const int i = i0 + r, j = j0 + tx;
      if (i < d && j < d) {
        const int64_t idx = (int64_t)i * d + j;
        if (!drop) {
          const float f = it.first ? (i == j ? 1.f : 0.f) : it.factor[idx];
          it.factor[idx] = ema_update(alpha, f, beta, A[r][tx], B[tx][r]);
        } else if (it.first) {
          it.factor[idx] = i == j ? 1.f : 0.f;
        }
        it.batch[idx] = 0.f;
      }
    }
    if (ti != tj) {
      const int i = j0 + r, j = i0 + tx;
      if (i < d && j < d) {
        const int64_t idx = (int64_t)i * d + j;
        if (!drop) {
          const float f = it.first ? 0.f : it.factor[idx];
          it.factor[idx] = ema_update(alpha, f, beta, A[tx][r], B[r][tx]);
        } else if (it.first) {
          it.factor[idx] = 0.f;
        }
        it.batch[idx] = 0.f;
      }
    }
  }
}

// Drop flags of the guarded EMA: dropped[i] = 1 if an entry of window i, unscaled, is not finite or exceeds 1e15 in
// magnitude (the bound the eigensolver rejects).  Every block of an item strides over its d x d window (16-byte
// loads where the window is 16-byte aligned); the flag is raised with an integer atomic, so the result does not
// depend on the order of the blocks.
struct ScanBatch {
  const float* batch[40];
  const float* scale[40];
  int64_t n[40];         // d * d
  int first_block[41];   // prefix sums of the blocks per item
  int count;
  int* dropped;
};

__device__ __forceinline__ bool window_entry_bad(float v, float u) { return !(fabsf(v * u) <= 1e15f); }

__global__ void __launch_bounds__(256) window_scan_kernel(const __grid_constant__ ScanBatch sb) {
  int item = 0;
  while (item + 1 < sb.count && (int)blockIdx.x >= sb.first_block[item + 1]) ++item;
  const float* __restrict__ x = sb.batch[item];
  const int64_t n = sb.n[item];
  const float u = window_unscale(sb.scale[item]);
  const int64_t tid = (int64_t)(blockIdx.x - sb.first_block[item]) * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)(sb.first_block[item + 1] - sb.first_block[item]) * blockDim.x;
  bool bad = false;
  int64_t done = 0;
  if ((reinterpret_cast<uintptr_t>(x) & 15) == 0) {
    const float4* __restrict__ x4 = reinterpret_cast<const float4*>(x);
    for (int64_t i = tid; i < n / 4; i += stride) {
      const float4 v = x4[i];
      bad |= window_entry_bad(v.x, u) | window_entry_bad(v.y, u) | window_entry_bad(v.z, u) | window_entry_bad(v.w, u);
    }
    done = n / 4 * 4;
  }
  for (int64_t i = done + tid; i < n; i += stride) bad |= window_entry_bad(x[i], u);
  if (__syncthreads_or(bad) && threadIdx.x == 0) atomicOr(sb.dropped + item, 1);
}

// ---- embedding layers: diagonal A -------------------------------------------------------------
// counts[idx[r]] += 1 (integer atomics: the histogram does not depend on the order of the rows)
template <typename I>
__global__ void histogram_kernel(const I* __restrict__ idx, int64_t n, unsigned int* counts) {
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x)
    atomicAdd(counts + idx[r], 1u);
}

// acc[v] += alpha * counts[v]: one rounding of the product, one of the sum, in a fixed order per entry
__global__ void scale_add_counts_kernel(const unsigned int* __restrict__ counts, int V, float alpha, float* acc) {
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < V; v += gridDim.x * blockDim.x)
    acc[v] = __fadd_rn(acc[v], __fmul_rn(alpha, (float)counts[v]));
}

// EMA of diagonal factors over up to 40 items: the diagonal of ema_kernel, with its beta and its rounding
struct EmaDiagBatch {
  kfac_ema_item it[40];
  int64_t elem0[41];     // prefix sums of d
  int count;
  float alpha;
  // guarded EMA only: as in EmaBatch
  const float* scale[40];
  const int* dropped;
  unsigned long long* skipped;
};

// GUARD = false: kfac_factor_ema_diag.  GUARD = true: the window is multiplied by window_unscale() as it is read, and a
// window flagged by window_scan_kernel is dropped (factor unchanged, or ones when it is the first window; batch = 0).
template <bool GUARD>
__global__ void __launch_bounds__(256) ema_diag_kernel(const __grid_constant__ EmaDiagBatch eb) {
  const int64_t total = eb.elem0[eb.count];
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    int item = 0;
    while (item + 1 < eb.count && e >= eb.elem0[item + 1]) ++item;
    const kfac_ema_item& it = eb.it[item];
    const int64_t v = e - eb.elem0[item];
    const float beta = (1.f - eb.alpha) * it.inv_count * 0.5f;
    float x = it.batch[v];
    if (GUARD) {
      if (eb.dropped[item]) {
        if (v == 0 && eb.skipped) atomicAdd(eb.skipped, 1ull);
        if (it.first) it.factor[v] = 1.f;
        it.batch[v] = 0.f;
        continue;
      }
      x *= window_unscale(eb.scale[item]);
    }
    const float f = it.first ? 1.f : it.factor[v];
    it.factor[v] = ema_update(eb.alpha, f, beta, x, x);   // (x + x) * 0.5 = x, as batch + batch^T on the diagonal
    it.batch[v] = 0.f;
  }
}

// ---- diagonal-G Linear layers: column sums of squares -----------------------------------------
// The rows are split into linear_diag_chunks(rows) chunks (a function of the shape only); the thread of column group
// j0..j0+VEC-1 and chunk c sums x[r, j]^2 over the chunk's rows -- in fp32 over 16 rows, then in fp64 -- and stores
// the chunk's sums as fp32 partials.  A row of V elements starts at any element offset modulo the 16-byte vector
// (V = 50257 is odd), so each thread loads the aligned vector holding its first column and, when the row is
// misaligned, the next one, and picks its VEC columns out of the pair.  The offset is the same for every thread of
// a row (j0 is a multiple of VEC), so the selection does not diverge.
static int64_t linear_diag_chunks(int64_t rows) { return std::max<int64_t>(1, std::min<int64_t>(128, (rows + 31) / 32)); }

template <typename T>
__device__ __forceinline__ float vec_lane(const uint32_t (&w)[8], int i) {
  if constexpr (sizeof(T) == 4) {
    return __uint_as_float(w[i]);
  } else {
    const unsigned short h = (unsigned short)(w[i >> 1] >> ((i & 1) * 16));
    if constexpr (std::is_same<T, __half>::value) return __half2float(__ushort_as_half(h));
    else return __bfloat162float(__ushort_as_bfloat16(h));
  }
}

template <typename T>
__global__ void __launch_bounds__(256) linear_diag_kernel(const T* __restrict__ x, int64_t rows, int V,
                                                          int64_t chunk_rows, float* __restrict__ partial) {
  constexpr int VEC = 16 / sizeof(T);
  const int j0 = (blockIdx.x * blockDim.x + threadIdx.x) * VEC;
  if (j0 >= V) return;
  const int64_t r_begin = (int64_t)blockIdx.y * chunk_rows, r_end = min(rows, r_begin + chunk_rows);
  double acc[VEC];
#pragma unroll
  for (int k = 0; k < VEC; ++k) acc[k] = 0.0;
  const bool full = j0 + VEC <= V;
  for (int64_t r0 = r_begin; r0 < r_end; r0 += 16) {
    float s[VEC];
#pragma unroll
    for (int k = 0; k < VEC; ++k) s[k] = 0.f;
    const int64_t r1 = min(r_end, r0 + 16);
    if (full) {
#pragma unroll 4
      for (int64_t r = r0; r < r1; ++r) {
        const uintptr_t addr = reinterpret_cast<uintptr_t>(x + r * V + j0);
        const int off = (int)((addr & 15) / sizeof(T));
        const uint4* q = reinterpret_cast<const uint4*>(addr & ~(uintptr_t)15);
        const uint4 lo = __ldg(q);
        const uint4 hi = off ? __ldg(q + 1) : make_uint4(0u, 0u, 0u, 0u);   // both vectors hold a column of this row
        const uint32_t w[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
#pragma unroll
        for (int o = 0; o < VEC; ++o) {
          if (o == off) {
#pragma unroll
            for (int k = 0; k < VEC; ++k) { const float v = vec_lane<T>(w, o + k); s[k] = fmaf(v, v, s[k]); }
          }
        }
      }
    } else {
      for (int64_t r = r0; r < r1; ++r)
#pragma unroll
        for (int k = 0; k < VEC; ++k)
          if (j0 + k < V) { const float v = to_float<T>(x[r * V + j0 + k]); s[k] = fmaf(v, v, s[k]); }
    }
#pragma unroll
    for (int k = 0; k < VEC; ++k) acc[k] += (double)s[k];
  }
  float* out = partial + (int64_t)blockIdx.y * V;
#pragma unroll
  for (int k = 0; k < VEC; ++k)
    if (j0 + k < V) out[j0 + k] = (float)acc[k];
}

// acc[j] += scale * sum_c partial[c][j], the chunks added in order in fp64; acc[V] += scale * ones_sum when ones (the
// bias entry of a diagonal A: the sum of the ones column's squares)
__global__ void linear_diag_reduce_kernel(const float* __restrict__ partial, int chunks, int V, int ones,
                                          double ones_sum, float scale, float* acc) {
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < V + ones; j += gridDim.x * blockDim.x) {
    double t = 0.0;
    if (j < V)
      for (int c = 0; c < chunks; ++c) t += (double)partial[(int64_t)c * V + j];
    else
      t = ones_sum;
    acc[j] = __fadd_rn(acc[j], (float)((double)scale * t));
  }
}

// dst = src; status |= 2 when an entry is not finite or exceeds 1e15 in magnitude
__global__ void __launch_bounds__(256) diag_snapshot_kernel(const float* __restrict__ src, float* dst, int n, int* status) {
  bool bad = false;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float v = src[i];
    dst[i] = v;
    bad |= window_entry_bad(v, 1.f);
  }
  if (__syncthreads_or(bad) && threadIdx.x == 0) atomicOr(status, 2);
}

__global__ void dgda_kernel(const float* dg, const float* da, int g, int a, float damping, float* out, int ldo) {
  const int64_t total = (int64_t)g * ldo;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int j = (int)(idx % ldo);
    out[idx] = j < a ? 1.f / (dg[idx / ldo] * da[j] + damping) : 0.f;
  }
}

// out[i][j] = 1 / ((dg[i] + gamma_G) (da[j] + gamma_A)), gamma_A = s pi, gamma_G = s / pi; zero in the padding columns
__global__ void dgda_pi_kernel(const float* dg, const float* da, int g, int a, float s, const float* pi, float* out,
                               int ldo) {
  const float p = *pi, gam_a = pi_gamma(s, p, 1), gam_g = pi_gamma(s, p, -1);
  const int64_t total = (int64_t)g * ldo;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int j = (int)(idx % ldo);
    out[idx] = j < a ? 1.f / __fmul_rn(__fadd_rn(dg[idx / ldo], gam_g), __fadd_rn(da[j], gam_a)) : 0.f;
  }
}

// pi of up to PI_BATCH items, one block each: the traces of A and G summed in fp64 (a fixed assignment of the diagonal
// entries to the threads and a fixed reduction tree, so the same factors give the same bits), then
// pi = sqrt((tr A / a) / (tr G / g)) rounded once to fp32, or 1 where a mean or pi is not a positive finite number
constexpr int PI_BATCH = 768;
struct PiBatch { kfac_pi_item it[PI_BATCH]; };
static_assert(sizeof(PiBatch) <= 32000, "kernel parameter space");

__device__ double block_sum(double v, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double t = 0.0;
  for (int k = 0; k < (int)(blockDim.x >> 5); ++k) t += red[k];
  __syncthreads();
  return t;
}

__device__ double trace_of(const float* F, int n, int ld, double* red) {
  const int64_t step = (int64_t)ld + 1;   // ld 0: a vector, its own diagonal
  double acc = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) acc += (double)F[i * step];
  return block_sum(acc, red);
}

__global__ void __launch_bounds__(256) pi_kernel(const __grid_constant__ PiBatch b) {
  __shared__ double red[8];
  const kfac_pi_item& it = b.it[blockIdx.x];
  const double ma = trace_of(it.A, it.a, it.lda, red) / it.a;
  const double mg = trace_of(it.G, it.g, it.ldg, red) / it.g;
  if (threadIdx.x != 0) return;
  float pi = 1.f;
  if (ma > 0.0 && ma <= DBL_MAX && mg > 0.0 && mg <= DBL_MAX) {
    const float p = (float)sqrt(ma / mg);
    if (p > 0.f && p <= FLT_MAX) pi = p;
  }
  *it.pi = pi;
}

__global__ void triu_pack_kernel(const float* F, int n, float* packed) {
  const int64_t total = (int64_t)n * n;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = idx / n, j = idx % n;
    if (j < i) continue;
    packed[i * n - i * (i - 1) / 2 + (j - i)] = F[idx];
  }
}
__global__ void triu_unpack_kernel(const float* packed, int n, float* F) {
  const int64_t total = (int64_t)n * n;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    int64_t i = idx / n, j = idx % n;
    if (j < i) { int64_t t = i; i = j; j = t; }
    F[idx] = packed[i * n - i * (i - 1) / 2 + (j - i)];
  }
}
__global__ void scale_kernel(float* buf, int64_t count, float s) {
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < count;
       idx += (int64_t)gridDim.x * blockDim.x)
    buf[idx] *= s;
}

static inline int grid_for(int64_t total, int threads = 256) {
  int64_t b = (total + threads - 1) / threads;
  return (int)max((int64_t)1, min(b, (int64_t)tc_num_sms() * 16));
}

// Workspace of a factor call: [packed feature-major matrix (pack bytes, may be 0)] [split partials of the SYRK].
// Without the partials region the reduction runs as one split (deterministic as well, less parallel).
struct CovWs {
  size_t pack, slab_off, total;
  CovWs(size_t pack_bytes, int d, int64_t rows, int batch) : pack(pack_bytes) {
    slab_off = pack ? align_up(pack, 256) : 0;
    const size_t slab = cov_slab_bytes(d, rows, batch);
    total = slab ? slab_off + slab : pack;
  }
  float* slab(void* ws, size_t ws_bytes) const {
    return (ws && total > slab_off && ws_bytes >= total) ? (float*)((char*)ws + slab_off) : nullptr;
  }
};

}  // namespace kfac

using namespace kfac;

static size_t linear_pack_bytes(int64_t rows, int features, int append_ones) {
  if (rows < 512 || features < 128) return 0;   // small problems stay on the SIMT kernel
  const int64_t ld = (rows + 3) / 4 * 4;
  return (size_t)ld * (size_t)(features + (append_ones ? 1 : 0)) * sizeof(float);
}

extern "C" size_t kfac_factor_linear_workspace_bytes(int64_t rows, int features, int append_ones) {
  return CovWs(linear_pack_bytes(rows, features, append_ones), features + (append_ones ? 1 : 0), rows, 1).total;
}

extern "C" size_t kfac_factor_linear_strided_workspace_bytes(int64_t rows, int features, int64_t ld, int append_ones) {
  (void)ld;   // the packed matrix and the split partials do not depend on the input's row stride
  return kfac_factor_linear_workspace_bytes(rows, features, append_ones);
}

extern "C" int kfac_factor_linear_strided(const void* x, int dtype, int64_t rows, int features, int64_t ldx,
                                          int append_ones, float scale, float* acc, void* ws, size_t ws_bytes,
                                          void* stream) {
  KFAC_CHECK_ARG(x && acc, "null pointer");
  KFAC_CHECK_ARG(rows >= 0 && rows < (1ll << 31) && features > 0, "dims");
  KFAC_CHECK_ARG(ldx >= features, "ld");
  const CovWs w(linear_pack_bytes(rows, features, append_ones), features + (append_ones ? 1 : 0), rows, 1);
  if (w.pack > 0 && ws && ws_bytes >= w.pack) {
    // tall activations (tokens x hidden): transpose once into a feature-major matrix
    // (ones row materialised) and run the tensor-core SYRK on it
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t ld = (rows + 3) / 4 * 4;
    const int ones = append_ones ? 1 : 0;
    dim3 grid(ceil_div(ld, 32), ceil_div(features + ones, 32));
    if (dtype == KFAC_F32) to_feature_major_kernel<float><<<grid, dim3(32, 8), 0, st>>>(x, rows, features, ldx, ones, (float*)ws, ld);
    else if (dtype == KFAC_F16) to_feature_major_kernel<__half><<<grid, dim3(32, 8), 0, st>>>(x, rows, features, ldx, ones, (float*)ws, ld);
    else if (dtype == KFAC_BF16) to_feature_major_kernel<__nv_bfloat16><<<grid, dim3(32, 8), 0, st>>>(x, rows, features, ldx, ones, (float*)ws, ld);
    else { set_error("unknown dtype %d", dtype); return KFAC_ERR_BAD_ARG; }
    KFAC_LAUNCH_CHECK();
    CovArgs a{};
    a.x = ws; a.ld = ld; a.batch_stride = 0; a.rows = (int)rows; a.batch = 1;
    a.feat = features + ones; a.ones = 0; a.scale = scale; a.acc = acc; a.slab = w.slab(ws, ws_bytes);
    return launch_cov<true>(a, KFAC_F32, st);
  }
  CovArgs a{};
  a.x = x; a.ld = ldx; a.batch_stride = 0; a.rows = (int)rows; a.batch = 1;
  a.feat = features; a.ones = append_ones ? 1 : 0; a.scale = scale; a.acc = acc; a.slab = w.slab(ws, ws_bytes);
  return launch_cov<false>(a, dtype, (cudaStream_t)stream);
}

extern "C" int kfac_factor_linear(const void* x, int dtype, int64_t rows, int features,
                                  int append_ones, float scale, float* acc, void* ws, size_t ws_bytes,
                                  void* stream) {
  return kfac_factor_linear_strided(x, dtype, rows, features, features, append_ones, scale, acc, ws, ws_bytes, stream);
}

// A kernel of all ones with unit stride and an output the size of the input reads the NCDHW input in place: it already
// is a feature-major (C x DHW) matrix per example -- unless its rows (DHW floats) are not 16-byte multiples (7 x 7
// maps): TMA cannot address those, so they are packed like an im2col matrix
static bool conv_in_place(const ConvGeo& g) {
  return g.kd == 1 && g.kh == 1 && g.kw == 1 && g.sd == 1 && g.sh == 1 && g.sw == 1 && g.pd == 0 && g.ph == 0 &&
         g.pw == 0 && g.Do == g.D && g.Ho == g.H && g.Wo == g.W &&
         ((int64_t)g.D * g.H * g.W % 4 == 0 || g.C < 64);
}

// workspace of a chunk of n examples: [im2col matrix (none in place)] [SYRK partials]
static CovWs conv_chunk_ws(const ConvGeo& g, int64_t n, int append_ones) {
  const int ones = append_ones ? 1 : 0;
  if (conv_in_place(g)) return CovWs(0, g.C + ones, (int64_t)g.D * g.H * g.W, g.batch);
  const int64_t rows = n * g.spatial(), ld = (rows + 3) / 4 * 4;
  const int64_t d = g.features() + ones;
  return CovWs((size_t)ld * (size_t)d * sizeof(float), (int)d, rows, 1);
}

// the largest chunk n in [1, batch] whose workspace (with its SYRK partials, or the matrix alone) fits in `bytes`, and
// whose rows stay below 2^31; 0 when not even one example fits.  Both sizes grow with n.
static int conv_chunk_for(const ConvGeo& g, int ones, size_t bytes, bool with_slab) {
  auto fits = [&](int64_t n) {
    const CovWs w = conv_chunk_ws(g, n, ones);
    return n * g.spatial() < (1ll << 31) && (with_slab ? w.total : w.pack) <= bytes;
  };
  if (!fits(1)) return 0;
  int64_t lo = 1, hi = g.batch;
  while (lo < hi) {
    const int64_t mid = (lo + hi + 1) / 2;
    if (fits(mid)) lo = mid; else hi = mid - 1;
  }
  return (int)lo;
}

// acc += scale * X^T X of the im2col X, formed `chunk` examples at a time into the workspace (see the header).  A
// kernel of ones with unit stride and no padding has the identity index map in both directions, so conv_in_place
// holds for a transposed geometry as well.
template <bool TRANSPOSED = false>
static int conv_input_factor(const void* x, int dtype, const ConvGeo& g, int append_ones, int chunk, float scale,
                             float* acc, void* ws, size_t ws_bytes, cudaStream_t s) {
  const int ones = append_ones ? 1 : 0;
  CovArgs a{};
  a.ones = ones; a.scale = scale; a.acc = acc;
  if (conv_in_place(g)) {
    const CovWs w = conv_chunk_ws(g, g.batch, ones);
    const int64_t plane = (int64_t)g.D * g.H * g.W;
    KFAC_CHECK_ARG(plane < (1ll << 31), "rows overflow");
    a.x = x; a.ld = plane; a.batch_stride = (int64_t)g.C * plane;
    a.rows = (int)plane; a.batch = g.batch; a.feat = g.C; a.slab = w.slab(ws, ws_bytes);
    return launch_cov<true>(a, dtype, s);
  }
  const CovWs w = conv_chunk_ws(g, chunk, ones);
  if (!ws || ws_bytes < w.pack) {
    set_error("conv_input: workspace too small (%zu < %zu)", ws_bytes, w.pack);
    return KFAC_ERR_WORKSPACE;
  }
  KFAC_CHECK_ARG((int64_t)chunk * g.spatial() < (1ll << 31), "rows overflow");
  KFAC_CHECK_ARG(g.features() + ones <= 65535, "conv_input: more than 65535 features");
  size_t elem;
  if (dtype == KFAC_F32) elem = 4;
  else if (dtype == KFAC_F16 || dtype == KFAC_BF16) elem = 2;
  else { set_error("unknown dtype %d", dtype); return KFAC_ERR_BAD_ARG; }
  const int64_t example = (int64_t)g.C * g.D * g.H * g.W;
  const int d = (int)g.features() + ones;
  for (int b0 = 0; b0 < g.batch; b0 += chunk) {
    Im2colArgs ia{(const char*)x + (size_t)b0 * example * elem, (float*)ws, g, ones, 0};
    ia.g.batch = std::min(chunk, g.batch - b0);
    const int64_t rows = (int64_t)ia.g.batch * g.spatial();
    ia.ld = (rows + 3) / 4 * 4;
    const dim3 grid((unsigned)ceil_div(ia.ld / 4, 256), (unsigned)d);
    if (dtype == KFAC_F32) im2col_kernel<float, TRANSPOSED><<<grid, 256, 0, s>>>(ia);
    else if (dtype == KFAC_F16) im2col_kernel<__half, TRANSPOSED><<<grid, 256, 0, s>>>(ia);
    else im2col_kernel<__nv_bfloat16, TRANSPOSED><<<grid, 256, 0, s>>>(ia);
    KFAC_LAUNCH_CHECK();
    // the ones row is materialised, so the SYRK sees d = C*kd*kh*kw + ones plain features
    CovArgs c = a;
    c.x = ws; c.ld = ia.ld; c.batch_stride = 0; c.rows = (int)rows; c.batch = 1; c.feat = d; c.ones = 0;
    c.slab = w.slab(ws, ws_bytes);
    const int rc = launch_cov<true>(c, KFAC_F32, s);
    if (rc) return rc;
  }
  return KFAC_OK;
}

extern "C" size_t kfac_factor_conv2d_input_workspace_bytes(int batch, int C, int H, int W, int kh,
                                                           int kw, int sh, int sw, int ph, int pw,
                                                           int append_ones) {
  if (batch <= 0 || C <= 0 || H <= 0 || W <= 0 || kh <= 0 || kw <= 0 || sh <= 0 || sw <= 0 || ph < 0 || pw < 0) return 0;
  if ((H + 2 * ph - kh) / sh + 1 <= 0 || (W + 2 * pw - kw) / sw + 1 <= 0) return 0;
  return conv_chunk_ws(conv2d_geo(batch, C, H, W, kh, kw, sh, sw, ph, pw), batch, append_ones).total;
}

extern "C" int kfac_factor_conv2d_input(const void* x, int dtype, int batch, int C, int H, int W,
                                        int kh, int kw, int sh, int sw, int ph, int pw,
                                        int append_ones, float scale, float* acc, void* ws,
                                        size_t ws_bytes, void* stream) {
  KFAC_CHECK_ARG(x && acc, "null pointer");
  KFAC_CHECK_ARG(batch > 0 && C > 0 && H > 0 && W > 0 && kh > 0 && kw > 0 && sh > 0 && sw > 0 &&
                     ph >= 0 && pw >= 0, "geometry");
  const ConvGeo g = conv2d_geo(batch, C, H, W, kh, kw, sh, sw, ph, pw);
  KFAC_CHECK_ARG(g.Ho > 0 && g.Wo > 0, "empty output");
  return conv_input_factor(x, dtype, g, append_ones, batch, scale, acc, ws, ws_bytes, (cudaStream_t)stream);
}

// the workspace query of the chunked factor calls
static size_t conv_chunked_ws_bytes(const ConvGeo& g, int append_ones, size_t max_bytes) {
  const int ones = append_ones ? 1 : 0;
  if (conv_in_place(g)) return conv_chunk_ws(g, g.batch, ones).total;
  // the largest chunk whose matrix and SYRK partials fit; else one example (beyond max_bytes when it alone does not fit)
  const int n = std::max(1, conv_chunk_for(g, ones, max_bytes, true));
  return conv_chunk_ws(g, n, ones).total;
}

// the chunked factor calls: the chunk is the largest that ws_bytes holds
template <bool TRANSPOSED>
static int conv_chunked_factor(const void* x, int dtype, const ConvGeo& g, int append_ones, float scale, float* acc,
                               void* ws, size_t ws_bytes, cudaStream_t s) {
  const int ones = append_ones ? 1 : 0;
  int chunk = g.batch;
  if (!conv_in_place(g)) {
    chunk = conv_chunk_for(g, ones, ws_bytes, true);
    if (chunk == 0) chunk = conv_chunk_for(g, ones, ws_bytes, false);   // one matrix, unsplit SYRK
    if (chunk == 0) {
      set_error("conv_input: workspace too small for one example (%zu < %zu)", ws_bytes, conv_chunk_ws(g, 1, ones).pack);
      return KFAC_ERR_WORKSPACE;
    }
  }
  return conv_input_factor<TRANSPOSED>(x, dtype, g, ones, chunk, scale, acc, ws, ws_bytes, s);
}

extern "C" size_t kfac_factor_conv_input_workspace_bytes(const kfac_conv_geometry* geom, int append_ones,
                                                         size_t max_bytes) {
  ConvGeo g;
  if (resolve_conv_geometry(geom, &g) != KFAC_OK) return 0;
  return conv_chunked_ws_bytes(g, append_ones, max_bytes);
}

extern "C" int kfac_factor_conv_input(const void* x, int dtype, const kfac_conv_geometry* geom, int append_ones,
                                      float scale, float* acc, void* ws, size_t ws_bytes, void* stream) {
  KFAC_CHECK_ARG(x && acc, "null pointer");
  ConvGeo g;
  const int rc = resolve_conv_geometry(geom, &g);
  if (rc) return rc;
  return conv_chunked_factor<false>(x, dtype, g, append_ones, scale, acc, ws, ws_bytes, (cudaStream_t)stream);
}

extern "C" size_t kfac_factor_conv_transpose_input_workspace_bytes(const kfac_conv_transpose_geometry* geom,
                                                                   int append_ones, size_t max_bytes) {
  ConvGeo g;
  if (resolve_conv_transpose_geometry(geom, &g) != KFAC_OK) return 0;
  return conv_chunked_ws_bytes(g, append_ones, max_bytes);
}

extern "C" int kfac_factor_conv_transpose_input(const void* x, int dtype, const kfac_conv_transpose_geometry* geom,
                                                int append_ones, float scale, float* acc, void* ws, size_t ws_bytes,
                                                void* stream) {
  KFAC_CHECK_ARG(x && acc, "null pointer");
  ConvGeo g;
  const int rc = resolve_conv_transpose_geometry(geom, &g);
  if (rc) return rc;
  return conv_chunked_factor<true>(x, dtype, g, append_ones, scale, acc, ws, ws_bytes, (cudaStream_t)stream);
}

static CovWs gradout_ws(int batch, int C, int Ho, int Wo) {
  // maps whose rows (Ho*Wo floats) are not 16-byte multiples (7 x 7) are packed into an aligned feature-major
  // matrix for the tensor-core SYRK; everything else is read in place
  if (((int64_t)Ho * Wo) % 4 == 0 || C < 64) return CovWs(0, C, (int64_t)Ho * Wo, batch);
  const int64_t rows = (int64_t)batch * Ho * Wo, ld = (rows + 3) / 4 * 4;
  return CovWs((size_t)ld * (size_t)C * sizeof(float), C, rows, 1);
}

extern "C" size_t kfac_factor_conv2d_gradout_workspace_bytes(int batch, int C, int Ho, int Wo) {
  if (batch <= 0 || C <= 0 || Ho <= 0 || Wo <= 0) return 0;
  return gradout_ws(batch, C, Ho, Wo).total;
}

extern "C" int kfac_factor_conv2d_gradout(const void* g, int dtype, int batch, int C, int Ho, int Wo,
                                          float scale, float* acc, void* ws, size_t ws_bytes, void* stream) {
  KFAC_CHECK_ARG(g && acc, "null pointer");
  KFAC_CHECK_ARG(batch > 0 && C > 0 && Ho > 0 && Wo > 0, "geometry");
  const CovWs w = gradout_ws(batch, C, Ho, Wo);
  if (w.pack > 0 && ws && ws_bytes >= w.pack) {
    cudaStream_t s = (cudaStream_t)stream;
    const int64_t rows = (int64_t)batch * Ho * Wo;
    KFAC_CHECK_ARG(rows < (1ll << 31), "rows overflow");
    const int64_t ld = (rows + 3) / 4 * 4;
    Im2colArgs ia{g, (float*)ws, conv2d_geo(batch, C, Ho, Wo, 1, 1, 1, 1, 0, 0), 0, ld};
    KFAC_CHECK_ARG(C <= 65535, "conv2d_gradout: more than 65535 channels");
    const dim3 grid((unsigned)ceil_div(ld / 4, 256), (unsigned)C);
    if (dtype == KFAC_F32) im2col_kernel<float><<<grid, 256, 0, s>>>(ia);
    else if (dtype == KFAC_F16) im2col_kernel<__half><<<grid, 256, 0, s>>>(ia);
    else if (dtype == KFAC_BF16) im2col_kernel<__nv_bfloat16><<<grid, 256, 0, s>>>(ia);
    else { set_error("unknown dtype %d", dtype); return KFAC_ERR_BAD_ARG; }
    KFAC_LAUNCH_CHECK();
    CovArgs a{};
    a.x = ws; a.ld = ld; a.batch_stride = 0; a.rows = (int)rows; a.batch = 1; a.feat = C; a.ones = 0;
    a.scale = scale; a.acc = acc; a.slab = w.slab(ws, ws_bytes);
    return launch_cov<true>(a, KFAC_F32, s);
  }
  CovArgs a{};
  a.x = g; a.ld = (int64_t)Ho * Wo; a.batch_stride = (int64_t)C * Ho * Wo;
  a.rows = Ho * Wo; a.batch = batch; a.feat = C; a.ones = 0; a.scale = scale; a.acc = acc; a.slab = w.slab(ws, ws_bytes);
  return launch_cov<true>(a, dtype, (cudaStream_t)stream);
}

// Drop flags of the guarded EMAs for the (up to 40) items it[0, count): windows of d x d floats, or of d (diag).
static int launch_window_scan(const kfac_ema_item* it, int count, const float* const* scale, bool diag, int* dropped,
                              cudaStream_t s) {
  ScanBatch sb{};
  sb.count = count;
  sb.dropped = dropped;
  int scan_blocks = 0;
  for (int i = 0; i < count; ++i) {
    sb.scale[i] = scale[i];
    sb.batch[i] = it[i].batch;
    sb.n[i] = diag ? (int64_t)it[i].d : (int64_t)it[i].d * it[i].d;
    sb.first_block[i] = scan_blocks;
    scan_blocks += (int)std::min<int64_t>(ceil_div(sb.n[i], 256 * 4 * 8), 1024);   // ~32 floats per thread
  }
  sb.first_block[count] = scan_blocks;
  window_scan_kernel<<<scan_blocks, 256, 0, s>>>(sb);
  KFAC_LAUNCH_CHECK();
  return KFAC_OK;
}

// EMA over up to 40 items per launch.  guard: `dropped` (one int per item, zeroed) receives the drop flags of a scan
// launch that precedes each EMA launch.
static int launch_ema(const kfac_ema_item* items, int count, float alpha, const float* const* loss_scale,
                      int* dropped, unsigned long long* skipped, cudaStream_t s) {
  for (int base = 0; base < count; base += 40) {
    EmaBatch eb{};
    eb.count = min(40, count - base);
    eb.alpha = alpha;
    int blocks = 0;
    for (int i = 0; i < eb.count; ++i) {
      eb.it[i] = items[base + i];
      KFAC_CHECK_ARG(eb.it[i].factor && eb.it[i].batch && eb.it[i].d > 0, "ema item");
      eb.first_block[i] = blocks;
      const int T = (eb.it[i].d + 31) / 32;
      blocks += T * (T + 1) / 2;
    }
    eb.first_block[eb.count] = blocks;
    if (!dropped) {
      ema_kernel<false><<<blocks, 256, 0, s>>>(eb);
      KFAC_LAUNCH_CHECK();
      continue;
    }
    for (int i = 0; i < eb.count; ++i) eb.scale[i] = loss_scale ? loss_scale[base + i] : nullptr;
    const int rc = launch_window_scan(eb.it, eb.count, eb.scale, false, dropped + base, s);
    if (rc) return rc;
    eb.dropped = dropped + base;
    eb.skipped = skipped;
    ema_kernel<true><<<blocks, 256, 0, s>>>(eb);
    KFAC_LAUNCH_CHECK();
  }
  return KFAC_OK;
}

extern "C" int kfac_factor_ema(const kfac_ema_item* items, int count, float alpha, void* stream) {
  KFAC_CHECK_ARG(count >= 0 && (items || count == 0), "items");
  return launch_ema(items, count, alpha, nullptr, nullptr, nullptr, (cudaStream_t)stream);
}

extern "C" size_t kfac_factor_ema_guarded_workspace_bytes(int count) {
  return count > 0 ? align_up((size_t)count * sizeof(int), 256) : 0;
}

extern "C" int kfac_factor_ema_guarded(const kfac_ema_item* items, int count, float alpha,
                                       const float* const* loss_scale, unsigned long long* skipped, void* ws,
                                       size_t ws_bytes, void* stream) {
  KFAC_CHECK_ARG(count >= 0 && (items || count == 0), "items");
  if (count == 0) return KFAC_OK;
  for (int i = 0; i < count; ++i)   // every item is checked before anything is launched
    KFAC_CHECK_ARG(items[i].factor && items[i].batch && items[i].d > 0, "ema item");
  const size_t need = kfac_factor_ema_guarded_workspace_bytes(count);
  if (!ws || ws_bytes < need) {
    set_error("factor_ema_guarded: workspace too small (%zu < %zu)", ws_bytes, need);
    return KFAC_ERR_WORKSPACE;
  }
  cudaStream_t s = (cudaStream_t)stream;
  KFAC_CUDA(cudaMemsetAsync(ws, 0, (size_t)count * sizeof(int), s));
  return launch_ema(items, count, alpha, loss_scale, (int*)ws, skipped, s);
}

extern "C" size_t kfac_factor_embedding_workspace_bytes(int V) {
  return V > 0 ? align_up((size_t)V * sizeof(unsigned int), 256) : 0;
}

extern "C" int kfac_factor_embedding(const void* idx, int index_dtype, int64_t N, int V, float alpha, float* acc,
                                     void* ws, size_t ws_bytes, void* stream) {
  KFAC_CHECK_ARG(acc && V > 0 && N >= 0 && N < (1ll << 32) && (idx || N == 0), "embedding factor args");
  KFAC_CHECK_ARG(index_dtype == KFAC_I32 || index_dtype == KFAC_I64, "index dtype");
  const size_t need = kfac_factor_embedding_workspace_bytes(V);
  if (!ws || ws_bytes < need) {
    set_error("factor_embedding: workspace too small (%zu < %zu)", ws_bytes, need);
    return KFAC_ERR_WORKSPACE;
  }
  if (N == 0) return KFAC_OK;
  cudaStream_t s = (cudaStream_t)stream;
  unsigned int* counts = (unsigned int*)ws;
  KFAC_CUDA(cudaMemsetAsync(counts, 0, (size_t)V * sizeof(unsigned int), s));
  if (index_dtype == KFAC_I32) histogram_kernel<int><<<grid_for(N), 256, 0, s>>>((const int*)idx, N, counts);
  else histogram_kernel<long long><<<grid_for(N), 256, 0, s>>>((const long long*)idx, N, counts);
  KFAC_LAUNCH_CHECK();
  scale_add_counts_kernel<<<grid_for(V), 256, 0, s>>>(counts, V, alpha, acc);
  KFAC_LAUNCH_CHECK();
  return KFAC_OK;
}

// The diagonal counterpart of launch_ema (same arguments, same guard).
static int launch_ema_diag(const kfac_ema_item* items, int count, float alpha, const float* const* loss_scale,
                           int* dropped, unsigned long long* skipped, cudaStream_t s) {
  for (int i = 0; i < count; ++i)
    KFAC_CHECK_ARG(items[i].factor && items[i].batch && items[i].d > 0, "ema item");
  for (int base = 0; base < count; base += 40) {
    EmaDiagBatch eb{};
    eb.count = min(40, count - base);
    eb.alpha = alpha;
    int64_t total = 0;
    for (int i = 0; i < eb.count; ++i) {
      eb.it[i] = items[base + i];
      eb.elem0[i] = total;
      total += eb.it[i].d;
    }
    eb.elem0[eb.count] = total;
    if (!dropped) {
      ema_diag_kernel<false><<<grid_for(total), 256, 0, s>>>(eb);
      KFAC_LAUNCH_CHECK();
      continue;
    }
    for (int i = 0; i < eb.count; ++i) eb.scale[i] = loss_scale ? loss_scale[base + i] : nullptr;
    const int rc = launch_window_scan(eb.it, eb.count, eb.scale, true, dropped + base, s);
    if (rc) return rc;
    eb.dropped = dropped + base;
    eb.skipped = skipped;
    ema_diag_kernel<true><<<grid_for(total), 256, 0, s>>>(eb);
    KFAC_LAUNCH_CHECK();
  }
  return KFAC_OK;
}

extern "C" int kfac_factor_ema_diag(const kfac_ema_item* items, int count, float alpha, void* stream) {
  KFAC_CHECK_ARG(count >= 0 && (items || count == 0), "items");
  return launch_ema_diag(items, count, alpha, nullptr, nullptr, nullptr, (cudaStream_t)stream);
}

extern "C" size_t kfac_factor_ema_diag_guarded_workspace_bytes(int count) {
  return kfac_factor_ema_guarded_workspace_bytes(count);
}

extern "C" int kfac_factor_ema_diag_guarded(const kfac_ema_item* items, int count, float alpha,
                                            const float* const* loss_scale, unsigned long long* skipped, void* ws,
                                            size_t ws_bytes, void* stream) {
  KFAC_CHECK_ARG(count >= 0 && (items || count == 0), "items");
  if (count == 0) return KFAC_OK;
  for (int i = 0; i < count; ++i)   // every item is checked before anything is launched
    KFAC_CHECK_ARG(items[i].factor && items[i].batch && items[i].d > 0, "ema item");
  const size_t need = kfac_factor_ema_diag_guarded_workspace_bytes(count);
  if (!ws || ws_bytes < need) {
    set_error("factor_ema_diag_guarded: workspace too small (%zu < %zu)", ws_bytes, need);
    return KFAC_ERR_WORKSPACE;
  }
  cudaStream_t s = (cudaStream_t)stream;
  KFAC_CUDA(cudaMemsetAsync(ws, 0, (size_t)count * sizeof(int), s));
  return launch_ema_diag(items, count, alpha, loss_scale, (int*)ws, skipped, s);
}

namespace kfac {
int launch_diag_reduce(const float* partial, int chunks, int V, int ones, double ones_sum, float scale, float* acc,
                       cudaStream_t s) {
  linear_diag_reduce_kernel<<<grid_for(V + ones), 256, 0, s>>>(partial, chunks, V, ones, ones_sum, scale, acc);
  KFAC_LAUNCH_CHECK();
  return KFAC_OK;
}
}  // namespace kfac

extern "C" size_t kfac_factor_linear_diag_workspace_bytes(int64_t rows, int features) {
  if (rows <= 0 || features <= 0) return 0;
  return align_up((size_t)linear_diag_chunks(rows) * (size_t)features * sizeof(float), 256);
}

extern "C" int kfac_factor_linear_diag(const void* x, int dtype, int64_t rows, int features, float scale, float* acc,
                                       void* ws, size_t ws_bytes, void* stream) {
  return kfac_factor_linear_diag_ones(x, dtype, rows, features, 0, scale, acc, ws, ws_bytes, stream);
}

extern "C" int kfac_factor_linear_diag_ones(const void* x, int dtype, int64_t rows, int features, int append_ones,
                                            float scale, float* acc, void* ws, size_t ws_bytes, void* stream) {
  KFAC_CHECK_ARG(acc && features > 0 && rows >= 0 && (x || rows == 0), "linear_diag args");
  KFAC_CHECK_ARG(dtype == KFAC_F32 || dtype == KFAC_F16 || dtype == KFAC_BF16, "dtype");
  if (rows == 0) return KFAC_OK;
  const size_t need = kfac_factor_linear_diag_workspace_bytes(rows, features);
  if (!ws || ws_bytes < need) {
    set_error("factor_linear_diag: workspace too small (%zu < %zu)", ws_bytes, need);
    return KFAC_ERR_WORKSPACE;
  }
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t chunks = linear_diag_chunks(rows), chunk_rows = (rows + chunks - 1) / chunks;
  const int vec = dtype == KFAC_F32 ? 4 : 8;
  const dim3 grid((unsigned)ceil_div(ceil_div(features, vec), 256), (unsigned)chunks);
  float* partial = (float*)ws;
  if (dtype == KFAC_F32) linear_diag_kernel<float><<<grid, 256, 0, s>>>((const float*)x, rows, features, chunk_rows, partial);
  else if (dtype == KFAC_F16) linear_diag_kernel<__half><<<grid, 256, 0, s>>>((const __half*)x, rows, features, chunk_rows, partial);
  else linear_diag_kernel<__nv_bfloat16><<<grid, 256, 0, s>>>((const __nv_bfloat16*)x, rows, features, chunk_rows, partial);
  KFAC_LAUNCH_CHECK();
  return launch_diag_reduce(partial, (int)chunks, features, append_ones ? 1 : 0, (double)rows, scale, acc, s);
}

extern "C" int kfac_diag_snapshot(const float* src, float* dst, int n, int* status, void* stream) {
  KFAC_CHECK_ARG(src && dst && status && n > 0, "diag_snapshot args");
  diag_snapshot_kernel<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(src, dst, n, status);
  KFAC_LAUNCH_CHECK();
  return KFAC_OK;
}

extern "C" int kfac_dgda(const float* dg, const float* da, int g, int a, float damping, float* out,
                         int ld_out, void* stream) {
  KFAC_CHECK_ARG(dg && da && out && g > 0 && a > 0 && ld_out >= a, "dgda args");
  dgda_kernel<<<grid_for((int64_t)g * ld_out), 256, 0, (cudaStream_t)stream>>>(dg, da, g, a, damping, out, ld_out);
  KFAC_LAUNCH_CHECK();
  return KFAC_OK;
}

extern "C" int kfac_dgda_pi(const float* dg, const float* da, int g, int a, float s, const float* pi, float* out,
                            int ld_out, void* stream) {
  KFAC_CHECK_ARG(dg && da && pi && out && g > 0 && a > 0 && ld_out >= a, "dgda_pi args");
  dgda_pi_kernel<<<grid_for((int64_t)g * ld_out), 256, 0, (cudaStream_t)stream>>>(dg, da, g, a, s, pi, out, ld_out);
  KFAC_LAUNCH_CHECK();
  return KFAC_OK;
}

extern "C" int kfac_pi(const kfac_pi_item* items, int count, void* stream) {
  KFAC_CHECK_ARG(count >= 0 && (items || count == 0), "pi args");
  for (int i = 0; i < count; ++i) {
    const kfac_pi_item& it = items[i];
    KFAC_CHECK_ARG(it.A && it.G && it.pi && it.a > 0 && it.g > 0 && (it.lda == 0 || it.lda >= it.a) &&
                       (it.ldg == 0 || it.ldg >= it.g), "pi item");
  }
  for (int i0 = 0; i0 < count; i0 += PI_BATCH) {
    const int n = std::min(PI_BATCH, count - i0);
    PiBatch b;
    memcpy(b.it, items + i0, sizeof(kfac_pi_item) * n);
    pi_kernel<<<n, 256, 0, (cudaStream_t)stream>>>(b);
    KFAC_LAUNCH_CHECK();
  }
  return KFAC_OK;
}

extern "C" int kfac_triu_pack(const float* F, int n, float* packed, void* stream) {
  KFAC_CHECK_ARG(F && packed && n > 0, "triu_pack args");
  triu_pack_kernel<<<grid_for((int64_t)n * n), 256, 0, (cudaStream_t)stream>>>(F, n, packed);
  KFAC_LAUNCH_CHECK();
  return KFAC_OK;
}
extern "C" int kfac_triu_unpack(const float* packed, int n, float* F, void* stream) {
  KFAC_CHECK_ARG(F && packed && n > 0, "triu_unpack args");
  triu_unpack_kernel<<<grid_for((int64_t)n * n), 256, 0, (cudaStream_t)stream>>>(packed, n, F);
  KFAC_LAUNCH_CHECK();
  return KFAC_OK;
}
extern "C" int kfac_scale_inplace(float* buf, int64_t count, float s, void* stream) {
  KFAC_CHECK_ARG(buf && count >= 0, "scale args");
  if (count == 0) return KFAC_OK;
  scale_kernel<<<grid_for(count), 256, 0, (cudaStream_t)stream>>>(buf, count, s);
  KFAC_LAUNCH_CHECK();
  return KFAC_OK;
}
