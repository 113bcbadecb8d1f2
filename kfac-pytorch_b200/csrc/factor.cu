// K1-K4: Kronecker-factor statistics (A = a^T a, G = g^T g), EMA, packing.
//
// Data layout in HBM: every factor is a dense d x d fp32 row-major matrix that
// lives inside one contiguous arena owned by the Python side (so the factor
// all-reduce is ONE collective over the arena).  Activations / grad-outputs
// are read in their native NCHW / (rows, features) layout.
#include "common.cuh"

#include <algorithm>

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

// im2col into a FEATURE-major fp32 matrix: out[(c,i,j)][(n,ho,wo)]
struct Im2colArgs {
  const void* x; float* out;
  int batch, C, H, W, kh, kw, sh, sw, ph, pw, Ho, Wo;
  int ones;        // append a feature row of ones
  int64_t ld;      // leading dimension of the feature-major output (>= rows, multiple of 4)
};
// grid (ceil(ld / 4 / 256), features [+ 1]): a thread writes 4 consecutive samples of one feature row with one 16-byte
// store; the (image, ho, wo) decomposition is done once per thread in 32-bit arithmetic and advanced incrementally
// (the element-wise version spent its time in 64-bit divisions: 480 us for a 231 MB matrix, now bandwidth bound)
template <typename T>
__global__ void __launch_bounds__(256) im2col_kernel(Im2colArgs a) {
  const int64_t rows = (int64_t)a.batch * a.Ho * a.Wo;
  const int nfeat = a.C * a.kh * a.kw;
  const int f = blockIdx.y;
  const int64_t r4 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (r4 >= a.ld) return;
  float v[4] = {0.f, 0.f, 0.f, 0.f};
  if (f >= nfeat) {
#pragma unroll
    for (int k = 0; k < 4; ++k) v[k] = (r4 + k < rows) ? 1.f : 0.f;
  } else if (r4 < rows) {
    const T* __restrict__ x = reinterpret_cast<const T*>(a.x);
    const int j = f % a.kw, i = (f / a.kw) % a.kh, c = f / (a.kw * a.kh);
    const unsigned row = (unsigned)r4;                    // rows < 2^31 (checked by the caller)
    int wo = (int)(row % (unsigned)a.Wo);
    const unsigned t = row / (unsigned)a.Wo;
    int ho = (int)(t % (unsigned)a.Ho), n = (int)(t / (unsigned)a.Ho);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (r4 + k < rows) {
        const int h = ho * a.sh + i - a.ph, w = wo * a.sw + j - a.pw;
        if (h >= 0 && h < a.H && w >= 0 && w < a.W) v[k] = to_float<T>(x[(((int64_t)n * a.C + c) * a.H + h) * a.W + w]);
      }
      if (++wo == a.Wo) { wo = 0; if (++ho == a.Ho) { ho = 0; ++n; } }
    }
  }
  *reinterpret_cast<float4*>(a.out + (int64_t)f * a.ld + r4) = make_float4(v[0], v[1], v[2], v[3]);
}

// X (rows x feat, sample-major, any dtype) -> out (feat [+1 ones row]) x ld, feature-major fp32
template <typename T>
__global__ void to_feature_major_kernel(const void* xin, int64_t rows, int feat, int ones, float* out, int64_t ld) {
  __shared__ float tile[32][33];
  const T* __restrict__ x = reinterpret_cast<const T*>(xin);
  const int64_t r0 = (int64_t)blockIdx.x * 32;
  const int f0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int64_t r = r0 + i;
    const int f = f0 + threadIdx.x;
    tile[i][threadIdx.x] = (r < rows && f < feat) ? to_float<T>(x[r * feat + f]) : 0.f;
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
};

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
#pragma unroll
  for (int r = ty; r < 32; r += 8) {
    const int iu = i0 + r, ju = j0 + tx;   // upper tile (ti, tj)
    A[r][tx] = (iu < d && ju < d) ? it.batch[(int64_t)iu * d + ju] : 0.f;
    const int il = j0 + r, jl = i0 + tx;   // mirror tile (tj, ti)
    B[r][tx] = (il < d && jl < d) ? it.batch[(int64_t)il * d + jl] : 0.f;
  }
  __syncthreads();
#pragma unroll
  for (int r = ty; r < 32; r += 8) {
    {
      const int i = i0 + r, j = j0 + tx;
      if (i < d && j < d) {
        const int64_t idx = (int64_t)i * d + j;
        const float s = beta * (A[r][tx] + B[tx][r]);
        const float f = it.first ? (i == j ? 1.f : 0.f) : it.factor[idx];
        it.factor[idx] = alpha * f + s;
        it.batch[idx] = 0.f;
      }
    }
    if (ti != tj) {
      const int i = j0 + r, j = i0 + tx;
      if (i < d && j < d) {
        const int64_t idx = (int64_t)i * d + j;
        const float s = beta * (A[tx][r] + B[r][tx]);
        const float f = it.first ? 0.f : it.factor[idx];
        it.factor[idx] = alpha * f + s;
        it.batch[idx] = 0.f;
      }
    }
  }
}

__global__ void dgda_kernel(const float* dg, const float* da, int g, int a, float damping, float* out, int ldo) {
  const int64_t total = (int64_t)g * ldo;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int j = (int)(idx % ldo);
    out[idx] = j < a ? 1.f / (dg[idx / ldo] * da[j] + damping) : 0.f;
  }
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

extern "C" int kfac_factor_linear(const void* x, int dtype, int64_t rows, int features,
                                  int append_ones, float scale, float* acc, void* ws, size_t ws_bytes,
                                  void* stream) {
  KFAC_CHECK_ARG(x && acc, "null pointer");
  KFAC_CHECK_ARG(rows >= 0 && rows < (1ll << 31) && features > 0, "dims");
  const CovWs w(linear_pack_bytes(rows, features, append_ones), features + (append_ones ? 1 : 0), rows, 1);
  if (w.pack > 0 && ws && ws_bytes >= w.pack) {
    // tall activations (tokens x hidden): transpose once into a feature-major matrix
    // (ones row materialised) and run the tensor-core SYRK on it
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t ld = (rows + 3) / 4 * 4;
    const int ones = append_ones ? 1 : 0;
    dim3 grid(ceil_div(ld, 32), ceil_div(features + ones, 32));
    if (dtype == KFAC_F32) to_feature_major_kernel<float><<<grid, dim3(32, 8), 0, st>>>(x, rows, features, ones, (float*)ws, ld);
    else if (dtype == KFAC_F16) to_feature_major_kernel<__half><<<grid, dim3(32, 8), 0, st>>>(x, rows, features, ones, (float*)ws, ld);
    else if (dtype == KFAC_BF16) to_feature_major_kernel<__nv_bfloat16><<<grid, dim3(32, 8), 0, st>>>(x, rows, features, ones, (float*)ws, ld);
    else { set_error("unknown dtype %d", dtype); return KFAC_ERR_BAD_ARG; }
    KFAC_LAUNCH_CHECK();
    CovArgs a{};
    a.x = ws; a.ld = ld; a.batch_stride = 0; a.rows = (int)rows; a.batch = 1;
    a.feat = features + ones; a.ones = 0; a.scale = scale; a.acc = acc; a.slab = w.slab(ws, ws_bytes);
    return launch_cov<true>(a, KFAC_F32, st);
  }
  CovArgs a{};
  a.x = x; a.ld = features; a.batch_stride = 0; a.rows = (int)rows; a.batch = 1;
  a.feat = features; a.ones = append_ones ? 1 : 0; a.scale = scale; a.acc = acc; a.slab = w.slab(ws, ws_bytes);
  return launch_cov<false>(a, dtype, (cudaStream_t)stream);
}

static bool conv_in_place(int C, int H, int W, int kh, int kw, int sh, int sw, int ph, int pw) {
  // 1x1 / stride 1 reads the NCHW input in place -- unless its rows (H*W floats) are not 16-byte multiples
  // (7 x 7 maps): TMA cannot address those, so they are packed like an im2col matrix
  return kh == 1 && kw == 1 && sh == 1 && sw == 1 && ph == 0 && pw == 0 && (((int64_t)H * W) % 4 == 0 || C < 64);
}

static CovWs conv_input_ws(int batch, int C, int H, int W, int kh, int kw, int sh, int sw, int ph, int pw,
                           int append_ones) {
  const int ones = append_ones ? 1 : 0;
  if (conv_in_place(C, H, W, kh, kw, sh, sw, ph, pw)) return CovWs(0, C + ones, (int64_t)H * W, batch);
  const int64_t Ho = (H + 2 * ph - kh) / sh + 1, Wo = (W + 2 * pw - kw) / sw + 1;
  const int64_t rows = (int64_t)batch * Ho * Wo, ld = (rows + 3) / 4 * 4;
  const int d = C * kh * kw + ones;
  return CovWs((size_t)ld * d * sizeof(float), d, rows, 1);
}

extern "C" size_t kfac_factor_conv2d_input_workspace_bytes(int batch, int C, int H, int W, int kh,
                                                           int kw, int sh, int sw, int ph, int pw,
                                                           int append_ones) {
  if (batch <= 0 || C <= 0 || H <= 0 || W <= 0 || kh <= 0 || kw <= 0 || sh <= 0 || sw <= 0 || ph < 0 || pw < 0) return 0;
  if ((H + 2 * ph - kh) / sh + 1 <= 0 || (W + 2 * pw - kw) / sw + 1 <= 0) return 0;
  return conv_input_ws(batch, C, H, W, kh, kw, sh, sw, ph, pw, append_ones).total;
}

extern "C" int kfac_factor_conv2d_input(const void* x, int dtype, int batch, int C, int H, int W,
                                        int kh, int kw, int sh, int sw, int ph, int pw,
                                        int append_ones, float scale, float* acc, void* ws,
                                        size_t ws_bytes, void* stream) {
  KFAC_CHECK_ARG(x && acc, "null pointer");
  KFAC_CHECK_ARG(batch > 0 && C > 0 && H > 0 && W > 0 && kh > 0 && kw > 0 && sh > 0 && sw > 0 &&
                     ph >= 0 && pw >= 0, "geometry");
  cudaStream_t s = (cudaStream_t)stream;
  const int Ho = (H + 2 * ph - kh) / sh + 1, Wo = (W + 2 * pw - kw) / sw + 1;
  KFAC_CHECK_ARG(Ho > 0 && Wo > 0, "empty output");
  const CovWs w = conv_input_ws(batch, C, H, W, kh, kw, sh, sw, ph, pw, append_ones);
  CovArgs a{};
  a.ones = append_ones ? 1 : 0; a.scale = scale; a.acc = acc; a.slab = w.slab(ws, ws_bytes);
  if (conv_in_place(C, H, W, kh, kw, sh, sw, ph, pw)) {
    // 1x1 / stride 1: the NCHW input already is a feature-major (C x HW) matrix per image
    a.x = x; a.ld = (int64_t)H * W; a.batch_stride = (int64_t)C * H * W;
    a.rows = H * W; a.batch = batch; a.feat = C;
    return launch_cov<true>(a, dtype, s);
  }
  if (!ws || ws_bytes < w.pack) {
    set_error("conv2d_input: workspace too small (%zu < %zu)", ws_bytes, w.pack);
    return KFAC_ERR_WORKSPACE;
  }
  const int64_t rows = (int64_t)batch * Ho * Wo;
  KFAC_CHECK_ARG(rows < (1ll << 31), "rows overflow");
  const int64_t ld = (rows + 3) / 4 * 4;
  Im2colArgs ia{x, (float*)ws, batch, C, H, W, kh, kw, sh, sw, ph, pw, Ho, Wo, a.ones, ld};
  KFAC_CHECK_ARG((int64_t)C * kh * kw + a.ones <= 65535, "conv2d_input: more than 65535 features");
  const dim3 grid((unsigned)ceil_div(ld / 4, 256), (unsigned)(C * kh * kw + a.ones));
  if (dtype == KFAC_F32) im2col_kernel<float><<<grid, 256, 0, s>>>(ia);
  else if (dtype == KFAC_F16) im2col_kernel<__half><<<grid, 256, 0, s>>>(ia);
  else if (dtype == KFAC_BF16) im2col_kernel<__nv_bfloat16><<<grid, 256, 0, s>>>(ia);
  else { set_error("unknown dtype %d", dtype); return KFAC_ERR_BAD_ARG; }
  KFAC_LAUNCH_CHECK();
  // the ones row is materialised, so the SYRK sees d = C*kh*kw + ones plain features
  a.x = ws; a.ld = ld; a.batch_stride = 0; a.rows = (int)rows; a.batch = 1; a.feat = C * kh * kw + a.ones;
  a.ones = 0;
  return launch_cov<true>(a, KFAC_F32, s);
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
    Im2colArgs ia{g, (float*)ws, batch, C, Ho, Wo, 1, 1, 1, 1, 0, 0, Ho, Wo, 0, ld};
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

extern "C" int kfac_factor_ema(const kfac_ema_item* items, int count, float alpha, void* stream) {
  KFAC_CHECK_ARG(count >= 0 && (items || count == 0), "items");
  cudaStream_t s = (cudaStream_t)stream;
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
    ema_kernel<<<blocks, 256, 0, s>>>(eb);
    KFAC_LAUNCH_CHECK();
  }
  return KFAC_OK;
}

extern "C" int kfac_dgda(const float* dg, const float* da, int g, int a, float damping, float* out,
                         int ld_out, void* stream) {
  KFAC_CHECK_ARG(dg && da && out && g > 0 && a > 0 && ld_out >= a, "dgda args");
  dgda_kernel<<<grid_for((int64_t)g * ld_out), 256, 0, (cudaStream_t)stream>>>(dg, da, g, a, damping, out, ld_out);
  KFAC_LAUNCH_CHECK();
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
