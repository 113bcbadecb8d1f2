// EKFAC (George et al., 2018): second moments of the layer's rows measured in the Kronecker-factored eigenbasis.
//
//   rows      x_r (A side) and g_r (G side), written SAMPLE-major (N x ld) in fp32 by the kfac_rows_* writers: the
//             projections contract over the features, and the tf32 wgmma engine takes only K-major operands
//   project   Xh^T = (Qa^T X^T)^2, Gh^T = (Qg^T G^T)^2, element-wise squares, written feature-major (d x ld4(N))
//             by the EPI_SQUARE epilogue of the grouped engine -- the K-major operands of the next product
//   S_batch   (1/N) Gh^T Xh                                   (g x a, a reduction over the N rows)
//   update    S <- alpha S + (1 - alpha) S_batch | S_batch | dg x da ;  dgda <- 1 / (S + damping)
//
// No floating-point atomics: the long reduction over the rows is split into chains of <= 512 rows whose partial tiles
// are added in a fixed order, and projections with K = a or g > 1024 run as chained launches over chunks of <= 512
// columns that accumulate in place (then one squaring pass), so every run gives the same bits.
#include "common.cuh"
#include "gemm_grouped.cuh"

#include <algorithm>
#include <vector>

namespace kfac {
namespace {

// ------------------------------------------------------------------ row writers
struct RowsArgs {
  const void* x; float* out;
  ConvGeo g;
  int ones;                  // append a constant feature (scaled like the others)
  int64_t ld;                // row stride of `out` (>= d, multiple of 4); columns [d, ld) are written as 0
  float scale; const float* loss_scale;   // every value is multiplied by scale / *loss_scale (loss_scale may be null)
};

__device__ __forceinline__ float row_scale(float scale, const float* loss_scale) {
  return loss_scale ? scale / *loss_scale : scale;
}

// out[(n, do, ho, wo)][(c, l, i, j) | ones] of an NCDHW input.  A CTA moves a 32 rows x 32 features tile through shared
// memory: it reads along the rows (neighbouring output positions) and writes along the features, both coalesced.  The
// 1 x 1 / stride-1 case is the gather of an NCHW tensor into rows (the conv G side uses it with kh = kw = 1).
// TRANSPOSED: the index map of a transposed convolution (TapMap).
template <typename T, bool TRANSPOSED>
__global__ void __launch_bounds__(256) rows_im2col_kernel(RowsArgs a) {
  using Tap = TapMap<TRANSPOSED>;
  __shared__ float tile[32][33];
  const ConvGeo& g = a.g;
  const int64_t rows = (int64_t)g.batch * g.Do * g.Ho * g.Wo;
  const int nfeat = g.C * g.kd * g.kh * g.kw;
  const int64_t r0 = (int64_t)blockIdx.x * 32;
  const int f0 = blockIdx.y * 32;
  const float s = row_scale(a.scale, a.loss_scale);
  const T* __restrict__ x = reinterpret_cast<const T*>(a.x);
  {
    const int64_t r = r0 + threadIdx.x;
    int wo = 0, ho = 0, dz = 0, n = 0;
    if (r < rows) {
      const unsigned ur = (unsigned)r;                     // rows < 2^31 (checked by the caller)
      wo = (int)(ur % (unsigned)g.Wo);
      unsigned t = ur / (unsigned)g.Wo;
      ho = (int)(t % (unsigned)g.Ho);
      t /= (unsigned)g.Ho;
      dz = (int)(t % (unsigned)g.Do);
      n = (int)(t / (unsigned)g.Do);
    }
    for (int i = threadIdx.y; i < 32; i += 8) {
      const int f = f0 + i;
      float v = 0.f;
      if (r < rows) {
        if (f < nfeat) {
          const int j = f % g.kw, ki = (f / g.kw) % g.kh, fl = f / (g.kw * g.kh);
          const int l = fl % g.kd, c = fl / g.kd;
          const int z = Tap::input(dz, l, g.sd, g.dd, g.pd, g.D), h = Tap::input(ho, ki, g.sh, g.dh, g.ph, g.H),
                    w = Tap::input(wo, j, g.sw, g.dw, g.pw, g.W);
          if ((z | h | w) >= 0) v = to_float<T>(x[((((int64_t)n * g.C + c) * g.D + z) * g.H + h) * g.W + w]) * s;
        } else if (f == nfeat && a.ones) {
          v = s;
        }
      }
      tile[threadIdx.x][i] = v;
    }
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int64_t r = r0 + i;
    const int f = f0 + threadIdx.x;
    if (r < rows && f < a.ld) a.out[r * a.ld + f] = tile[i][threadIdx.x];
  }
}

// out[r][f] = s * x[r][f] (f < feat), s (f == feat, ones), 0 up to ld: a (rows, feat) input with row stride ldx is
// already sample-major
template <typename T>
__global__ void __launch_bounds__(256) rows_linear_kernel(const void* xin, int64_t rows, int feat, int64_t ldx, int ones,
                                                          float scale, const float* loss_scale, float* out, int64_t ld) {
  const T* __restrict__ x = reinterpret_cast<const T*>(xin);
  const float s = row_scale(scale, loss_scale);
  const int64_t total = rows * ld;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = idx / ld;
    const int f = (int)(idx - r * ld);
    out[idx] = f < feat ? to_float<T>(x[r * ldx + f]) * s : (f == feat && ones ? s : 0.f);
  }
}

template <bool TRANSPOSED = false>
static int launch_rows_im2col(const RowsArgs& a, int dtype, cudaStream_t s) {
  const int64_t rows = (int64_t)a.g.batch * a.g.spatial();
  KFAC_CHECK_ARG(rows < (1ll << 31), "rows overflow");
  const dim3 grid((unsigned)ceil_div(rows, 32), (unsigned)ceil_div(a.ld, 32)), block(32, 8);
  KFAC_CHECK_ARG(grid.y <= 65535, "more than 2^21 features");
  if (dtype == KFAC_F32) rows_im2col_kernel<float, TRANSPOSED><<<grid, block, 0, s>>>(a);
  else if (dtype == KFAC_F16) rows_im2col_kernel<__half, TRANSPOSED><<<grid, block, 0, s>>>(a);
  else if (dtype == KFAC_BF16) rows_im2col_kernel<__nv_bfloat16, TRANSPOSED><<<grid, block, 0, s>>>(a);
  else { set_error("unknown dtype %d", dtype); return KFAC_ERR_BAD_ARG; }
  KFAC_LAUNCH_CHECK();
  return KFAC_OK;
}

static inline int grid_for(int64_t total, int threads = 256) {
  const int64_t b = (total + threads - 1) / threads;
  return (int)std::max<int64_t>(1, std::min<int64_t>(b, (int64_t)tc_num_sms() * 16));
}

static inline int64_t ld4(int64_t n) { return (n + 3) & ~int64_t(3); }

// ------------------------------------------------------------------ statistics
struct SqDev { float* p; long long elem0; };

constexpr int CHAIN = 512;          // longest reduction chain of the tensor-core engine that stays at fp32 accuracy
constexpr int SIMT_CHAIN = 4096;    // longest sequential fp32 chain of the SIMT engine

// workspace: [grouped-GEMM tables][squaring table][per item: Xh (a x ld4 N), Gh (g x ld4 N)][split partials of S_batch]
struct StatLayout {
  size_t off_gemm, gemm_bytes, off_sq, total;
  std::vector<size_t> xh, gh, slab_s;
  std::vector<int> ch_x, ch_g, sp_s;     // ch_*: column chunks of a projection (1: one launch with EPI_SQUARE)
  std::vector<bool> simt_s;          // S_batch on the SIMT engine, chunked by the caller into SIMT_CHAIN rows
};

static GroupedGemm gemm(const float* A, int64_t lda, const float* B, int64_t ldb, float* D, int64_t ldd, int M, int N,
                        int K, float alpha, int epi) {
  GroupedGemm g{};
  g.A = A; g.lda = lda; g.B = B; g.ldb = ldb; g.D = D; g.ldd = ldd; g.M = M; g.N = N; g.K = K;
  g.alpha = alpha; g.epi = epi; g.splits = 1;
  return g;
}

static void stat_layout(const kfac_ekfac_stat_item* items, int count, StatLayout& L) {
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t o = off; off = align_up(off + bytes, 256); return o; };
  L.off_gemm = 0;
  L.xh.resize(count); L.gh.resize(count);
  L.slab_s.assign(count, 0);
  L.ch_x.assign(count, 1); L.ch_g.assign(count, 1); L.sp_s.assign(count, 1); L.simt_s.assign(count, false);
  // the tables of the larger of the two grouped launches: 2 projections per item, or the S_batch problems (a
  // chunked SIMT-class item contributes one problem per chunk)
  int probs = 2 * count;
  {
    const float* al = reinterpret_cast<const float*>(256);
    int n_s = 0;
    for (int i = 0; i < count; ++i) {
      const kfac_ekfac_stat_item& it = items[i];
      const int64_t ldN = ld4(it.N);
      const bool tc = grouped_gemm_tc_ok(gemm(al, ldN, al, ldN, nullptr, it.lds, it.g, it.a, (int)it.N, 1.f, EPI_NONE));
      n_s += (!tc && it.N > 2 * SIMT_CHAIN) ? ceil_div(it.N, SIMT_CHAIN) : 1;
    }
    probs = std::max(probs, n_s);
  }
  L.gemm_bytes = grouped_gemm_ws_bytes(probs);
  take(L.gemm_bytes);
  L.off_sq = take(sizeof(SqDev) * (size_t)(2 * count));
  for (int i = 0; i < count; ++i) {
    const kfac_ekfac_stat_item& it = items[i];
    L.xh[i] = take((size_t)it.a * ld4(it.N) * sizeof(float));
    L.gh[i] = take((size_t)it.g * ld4(it.N) * sizeof(float));
  }
  // tensor-core problems with K > 1024 are reduced in chains of <= CHAIN (as in kfac_precondition): here as chained
  // launches that accumulate into the projection, which needs no partials.  Operands are 256-byte aligned workspace
  // regions or arena entries, so whether a problem takes the tensor cores depends on its shape only
  const float* al = reinterpret_cast<const float*>(256);
  for (int i = 0; i < count; ++i) {
    const kfac_ekfac_stat_item& it = items[i];
    const int N = (int)it.N, ldN = (int)ld4(it.N);
    if (grouped_gemm_tc_ok(gemm(al, it.ldqa, al, it.ldx, nullptr, ldN, it.a, N, it.a, 1.f, EPI_NONE)))
      L.ch_x[i] = chain_splits(it.a);
    if (grouped_gemm_tc_ok(gemm(al, it.ldqg, al, it.ldg, nullptr, ldN, it.g, N, it.g, 1.f, EPI_NONE)))
      L.ch_g[i] = chain_splits(it.g);
    const bool tc = grouped_gemm_tc_ok(gemm(al, ldN, al, ldN, nullptr, it.lds, it.g, it.a, N, 1.f, EPI_NONE));
    const int chain = tc ? CHAIN : SIMT_CHAIN;
    if (N > 2 * chain) {
      L.sp_s[i] = ceil_div(N, chain);
      L.simt_s[i] = !tc;
      L.slab_s[i] = take((size_t)L.sp_s[i] * it.g * it.lds * sizeof(float));
    }
  }
  L.total = off;
}

// S_batch[i][j] = sum_c slab[c][i][j] for the chunks of a SIMT-class problem, in a fixed order (padding columns 0)
__global__ void chunk_sum_kernel(const float* __restrict__ slab, int chunks, int64_t stride, int a, int64_t ld,
                                 int64_t total, float* __restrict__ out) {
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    float t = 0.f;
    if (idx % ld < a) {
      t = slab[idx];
      for (int c = 1; c < chunks; ++c) t += slab[c * stride + idx];
    }
    out[idx] = t;
  }
}

// x <- x^2 over the projections that were accumulated in column chunks (one launch for all of them)
__global__ void __launch_bounds__(256) square_all_kernel(const SqDev* t, int count, long long total) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    int lo = 0, hi = count - 1;
    while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (t[mid].elem0 <= e) lo = mid; else hi = mid - 1; }
    float* p = t[lo].p + (e - t[lo].elem0);
    const float v = *p;
    *p = v * v;
  }
}

// chunk c of n over K columns: [k0, k0 + k); chunks are multiples of 32 columns (whole k-blocks of the engine)
static void column_chunk(int K, int n, int c, int* k0, int* k) {
  const int cs = (ceil_div(K, n) + 31) / 32 * 32;
  *k0 = std::min(K, c * cs);
  *k = std::max(0, std::min(K, *k0 + cs) - *k0);
}

// ------------------------------------------------------------------ update
struct UpdDev {
  float* S; const float* Sb; const float* dg; const float* da; float* dgda;
  const int* drop_a; const int* drop_g;
  int g, a; int64_t ld; long long elem0;
};

__device__ __forceinline__ int upd_find(const UpdDev* t, int count, long long e) {
  int lo = 0, hi = count - 1;
  while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (t[mid].elem0 <= e) lo = mid; else hi = mid - 1; }
  return lo;
}

// bad[i] = 1 if S_batch of item i holds an entry that is not finite or exceeds 1e15 in magnitude (the bound of the
// guarded factor EMA); an integer flag, so the result does not depend on the order of the threads
__global__ void __launch_bounds__(256) sbatch_scan_kernel(const UpdDev* t, int count, long long total, int* bad) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int lo = upd_find(t, count, e);
    const UpdDev& p = t[lo];
    const long long idx = e - p.elem0;
    if (idx % p.ld < p.a && !(fabsf(p.Sb[idx]) <= 1e15f)) atomicOr(bad + lo, 1);
  }
}

__global__ void __launch_bounds__(256) ekfac_update_kernel(const UpdDev* t, int count, long long total, float alpha,
                                                           int mode, float damping, const int* bad,
                                                           unsigned long long* skipped) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int lo = upd_find(t, count, e);
    const UpdDev& p = t[lo];
    const long long idx = e - p.elem0;
    const int i = (int)(idx / p.ld), j = (int)(idx - (long long)i * p.ld);
    if (j >= p.a) { p.dgda[idx] = 0.f; continue; }      // padding columns feed the K dimension of the next GEMM
    const bool reads = mode == KFAC_EKFAC_EMA || mode == KFAC_EKFAC_RESET;
    const bool factor_drop = (p.drop_a && *p.drop_a) || (p.drop_g && *p.drop_g);
    const bool drop = reads && (bad[lo] || factor_drop);
    // a window dropped for its S_batch alone is counted here (the guarded EMA has counted the others)
    if (idx == 0 && reads && bad[lo] && !factor_drop && skipped) atomicAdd(skipped, 1ull);
    if (mode == KFAC_EKFAC_SEED || (mode == KFAC_EKFAC_RESET && drop)) {   // a new basis without (a usable) window
      p.S[idx] = __fmul_rn(p.dg[i], p.da[j]);
      p.dgda[idx] = 1.f / __fmaf_rn(p.dg[i], p.da[j], damping);   // the bits of kfac_dgda (the eigen method)
      continue;
    }
    float s;
    if (mode == KFAC_EKFAC_KEEP || drop) s = p.S[idx];
    else if (mode == KFAC_EKFAC_EMA) s = __fmaf_rn(alpha, p.S[idx], __fmul_rn(1.f - alpha, p.Sb[idx]));
    else s = p.Sb[idx];
    if (mode != KFAC_EKFAC_KEEP) p.S[idx] = s;
    p.dgda[idx] = 1.f / __fadd_rn(s, damping);
  }
}

static size_t upd_table_bytes(int count) { return align_up(sizeof(UpdDev) * (size_t)std::max(1, count), 256); }

}  // namespace
}  // namespace kfac

using namespace kfac;

// ---------------------------------------------------------------------------------------------------- row writers
extern "C" int kfac_rows_linear_strided(const void* x, int dtype, int64_t rows, int features, int64_t ldx,
                                        int append_ones, float scale, const float* loss_scale, float* out, int ld_out,
                                        void* stream) {
  KFAC_CHECK_ARG(x && out, "null pointer");
  KFAC_CHECK_ARG(rows > 0 && rows < (1ll << 31) && features > 0, "dims");
  KFAC_CHECK_ARG(ldx >= features, "ld");
  KFAC_CHECK_ARG(ld_out >= features + (append_ones ? 1 : 0) && ld_out % 4 == 0, "ld_out");
  cudaStream_t s = (cudaStream_t)stream;
  const int ones = append_ones ? 1 : 0;
  const int grid = grid_for(rows * ld_out);
  if (dtype == KFAC_F32)
    rows_linear_kernel<float><<<grid, 256, 0, s>>>(x, rows, features, ldx, ones, scale, loss_scale, out, ld_out);
  else if (dtype == KFAC_F16)
    rows_linear_kernel<__half><<<grid, 256, 0, s>>>(x, rows, features, ldx, ones, scale, loss_scale, out, ld_out);
  else if (dtype == KFAC_BF16)
    rows_linear_kernel<__nv_bfloat16><<<grid, 256, 0, s>>>(x, rows, features, ldx, ones, scale, loss_scale, out, ld_out);
  else { set_error("unknown dtype %d", dtype); return KFAC_ERR_BAD_ARG; }
  KFAC_LAUNCH_CHECK();
  return KFAC_OK;
}

extern "C" int kfac_rows_linear(const void* x, int dtype, int64_t rows, int features, int append_ones, float scale,
                                const float* loss_scale, float* out, int ld_out, void* stream) {
  return kfac_rows_linear_strided(x, dtype, rows, features, features, append_ones, scale, loss_scale, out, ld_out,
                                  stream);
}

extern "C" int kfac_rows_conv2d_input(const void* x, int dtype, int batch, int C, int H, int W, int kh, int kw, int sh,
                                      int sw, int ph, int pw, int append_ones, float scale, float* out, int ld_out,
                                      void* stream) {
  KFAC_CHECK_ARG(x && out, "null pointer");
  KFAC_CHECK_ARG(batch > 0 && C > 0 && H > 0 && W > 0 && kh > 0 && kw > 0 && sh > 0 && sw > 0 && ph >= 0 && pw >= 0,
                 "geometry");
  const ConvGeo g = conv2d_geo(batch, C, H, W, kh, kw, sh, sw, ph, pw);
  KFAC_CHECK_ARG(g.Ho > 0 && g.Wo > 0, "empty output");
  const int ones = append_ones ? 1 : 0;
  KFAC_CHECK_ARG((int64_t)ld_out >= g.features() + ones && ld_out % 4 == 0, "ld_out");
  RowsArgs a{x, out, g, ones, ld_out, scale, nullptr};
  return launch_rows_im2col(a, dtype, (cudaStream_t)stream);
}

extern "C" int kfac_rows_conv_input(const void* x, int dtype, const kfac_conv_geometry* geom, int append_ones,
                                    float scale, float* out, int ld_out, void* stream) {
  KFAC_CHECK_ARG(x && out, "null pointer");
  ConvGeo g;
  const int rc = resolve_conv_geometry(geom, &g);
  if (rc) return rc;
  const int ones = append_ones ? 1 : 0;
  KFAC_CHECK_ARG((int64_t)ld_out >= g.features() + ones && ld_out % 4 == 0, "ld_out");
  RowsArgs a{x, out, g, ones, ld_out, scale, nullptr};
  return launch_rows_im2col(a, dtype, (cudaStream_t)stream);
}

extern "C" int kfac_rows_conv_transpose_input(const void* x, int dtype, const kfac_conv_transpose_geometry* geom,
                                              int append_ones, float scale, float* out, int ld_out, void* stream) {
  KFAC_CHECK_ARG(x && out, "null pointer");
  ConvGeo g;
  const int rc = resolve_conv_transpose_geometry(geom, &g);
  if (rc) return rc;
  const int ones = append_ones ? 1 : 0;
  KFAC_CHECK_ARG((int64_t)ld_out >= g.features() + ones && ld_out % 4 == 0, "ld_out");
  RowsArgs a{x, out, g, ones, ld_out, scale, nullptr};
  return launch_rows_im2col<true>(a, dtype, (cudaStream_t)stream);
}

extern "C" int kfac_rows_conv2d_gradout(const void* g, int dtype, int batch, int C, int Ho, int Wo, float scale,
                                        const float* loss_scale, float* out, int ld_out, void* stream) {
  KFAC_CHECK_ARG(g && out, "null pointer");
  KFAC_CHECK_ARG(batch > 0 && C > 0 && Ho > 0 && Wo > 0, "geometry");
  KFAC_CHECK_ARG(ld_out >= C && ld_out % 4 == 0, "ld_out");
  RowsArgs a{g, out, conv2d_geo(batch, C, Ho, Wo, 1, 1, 1, 1, 0, 0), 0, ld_out, scale, loss_scale};
  return launch_rows_im2col(a, dtype, (cudaStream_t)stream);
}

// ---------------------------------------------------------------------------------------------------- statistics
extern "C" size_t kfac_ekfac_statistics_workspace_bytes(const kfac_ekfac_stat_item* items, int count) {
  if (count <= 0 || !items) return 0;
  StatLayout L;
  stat_layout(items, count, L);
  return L.total;
}

extern "C" int kfac_ekfac_statistics(const kfac_ekfac_stat_item* items, int count, void* ws, size_t ws_bytes,
                                     void* stream) {
  KFAC_CHECK_ARG(count >= 0 && (items || count == 0), "items");
  if (count == 0) return KFAC_OK;
  for (int i = 0; i < count; ++i) {
    const kfac_ekfac_stat_item& it = items[i];
    KFAC_CHECK_ARG(it.X && it.G && it.qaT && it.qgT && it.S_batch, "ekfac statistics item");
    KFAC_CHECK_ARG(it.N > 0 && it.N < (1ll << 31) && it.a > 0 && it.g > 0, "ekfac statistics dims");
    KFAC_CHECK_ARG(it.ldx >= it.a && it.ldg >= it.g && it.ldqa >= it.a && it.ldqg >= it.g && it.lds >= it.a,
                   "ekfac statistics leading dims");
    KFAC_CHECK_ARG(it.ldx % 4 == 0 && it.ldg % 4 == 0 && it.lds % 4 == 0, "ekfac statistics leading dims (multiples of 4)");
  }
  StatLayout L;
  stat_layout(items, count, L);
  if (!ws || ws_bytes < L.total) {
    set_error("ekfac_statistics: workspace too small (%zu < %zu)", ws_bytes, L.total);
    return KFAC_ERR_WORKSPACE;
  }
  cudaStream_t s = (cudaStream_t)stream;
  char* base = (char*)ws;
  auto F = [&](size_t off) { return (float*)(base + off); };
  void* gws = base + L.off_gemm;
  const size_t gws_bytes = L.gemm_bytes;
  // (1) Xh^T[f, r] = (sum_k QaT[f, k] X[r, k])^2  and  Gh^T[f, r] = (sum_k QgT[f, k] G[r, k])^2      (K = a | g)
  // round 0 holds every projection (squared in the epilogue unless it is chunked); round c >= 1 adds chunk c of the
  // chunked ones in place (read-modify-write, a fixed order); then the chunked outputs are squared
  int rounds = 1;
  for (int i = 0; i < count; ++i) rounds = std::max(rounds, std::max(L.ch_x[i], L.ch_g[i]));
  std::vector<GroupedGemm> pr;
  pr.reserve(2 * count);
  int rc;
  for (int c = 0; c < rounds; ++c) {
    pr.clear();
    for (int i = 0; i < count; ++i) {
      const kfac_ekfac_stat_item& it = items[i];
      const int N = (int)it.N;
      const int64_t ldN = ld4(it.N);
      const struct { const float* Q; int ldq; const float* R; int ldr; float* out; int d; int ch; } side[2] = {
          {it.qaT, it.ldqa, it.X, it.ldx, F(L.xh[i]), it.a, L.ch_x[i]},
          {it.qgT, it.ldqg, it.G, it.ldg, F(L.gh[i]), it.g, L.ch_g[i]}};
      for (const auto& sd : side) {
        if (c >= sd.ch) continue;
        if (sd.ch == 1) { pr.push_back(gemm(sd.Q, sd.ldq, sd.R, sd.ldr, sd.out, ldN, sd.d, N, sd.d, 1.f, EPI_SQUARE)); continue; }
        int k0, k;
        column_chunk(sd.d, sd.ch, c, &k0, &k);
        if (k == 0) continue;
        GroupedGemm g = gemm(sd.Q + k0, sd.ldq, sd.R + k0, sd.ldr, sd.out, ldN, sd.d, N, k, 1.f, EPI_NONE);
        g.mode = c == 0 ? 0 : 1;
        pr.push_back(g);
      }
    }
    if ((rc = launch_grouped_gemm(pr.data(), (int)pr.size(), gws, gws_bytes, s))) return rc;
  }
  if (rounds > 1) {
    std::vector<SqDev> sq;
    long long total = 0;
    for (int i = 0; i < count; ++i) {
      const int64_t ldN = ld4(items[i].N);
      if (L.ch_x[i] > 1) { sq.push_back(SqDev{F(L.xh[i]), total}); total += (long long)items[i].a * ldN; }
      if (L.ch_g[i] > 1) { sq.push_back(SqDev{F(L.gh[i]), total}); total += (long long)items[i].g * ldN; }
    }
    KFAC_CUDA(cudaMemcpyAsync(base + L.off_sq, sq.data(), sizeof(SqDev) * sq.size(), cudaMemcpyHostToDevice, s));
    square_all_kernel<<<grid_for(total), 256, 0, s>>>((const SqDev*)(base + L.off_sq), (int)sq.size(), total);
    KFAC_LAUNCH_CHECK();
  }
  // (2) S_batch[i, j] = (1/N) sum_r Gh^T[i, r] Xh^T[j, r]                                              (K = N)
  std::vector<GroupedGemm> st;
  std::vector<int> chunked;
  for (int i = 0; i < count; ++i) {
    const kfac_ekfac_stat_item& it = items[i];
    const int N = (int)it.N;
    const int64_t ldN = ld4(it.N);
    const float alpha = (float)(1.0 / (double)it.N);
    if (!L.simt_s[i]) {
      GroupedGemm g = gemm(F(L.gh[i]), ldN, F(L.xh[i]), ldN, it.S_batch, it.lds, it.g, it.a, N, alpha, EPI_NONE);
      if (L.sp_s[i] > 1) { g.splits = L.sp_s[i]; g.slab = F(L.slab_s[i]); g.slab_stride = (int64_t)it.g * it.lds; }
      st.push_back(g);
      continue;
    }
    // SIMT-class (g or a < 64) with a long reduction: chunks of SIMT_CHAIN rows into the partials, summed below
    for (int c = 0; c < L.sp_s[i]; ++c) {
      const int k0 = c * SIMT_CHAIN, k = std::min(N - k0, SIMT_CHAIN);
      st.push_back(gemm(F(L.gh[i]) + k0, ldN, F(L.xh[i]) + k0, ldN, F(L.slab_s[i]) + (int64_t)c * it.g * it.lds, it.lds,
                        it.g, it.a, k, alpha, EPI_NONE));
    }
    chunked.push_back(i);
  }
  if ((rc = launch_grouped_gemm(st.data(), (int)st.size(), gws, gws_bytes, s))) return rc;
  for (const int i : chunked) {
    const kfac_ekfac_stat_item& it = items[i];
    const int64_t total = (int64_t)it.g * it.lds;
    chunk_sum_kernel<<<grid_for(total), 256, 0, s>>>(F(L.slab_s[i]), L.sp_s[i], total, it.a, it.lds, total, it.S_batch);
    KFAC_LAUNCH_CHECK();
  }
  return KFAC_OK;
}

// ---------------------------------------------------------------------------------------------------- update
extern "C" size_t kfac_ekfac_update_workspace_bytes(int count) {
  return count > 0 ? upd_table_bytes(count) + align_up((size_t)count * sizeof(int), 256) : 0;
}

extern "C" int kfac_ekfac_update(const kfac_ekfac_update_item* items, int count, float alpha, int mode, float damping,
                                 unsigned long long* skipped, void* ws, size_t ws_bytes, void* stream) {
  KFAC_CHECK_ARG(count >= 0 && (items || count == 0), "items");
  KFAC_CHECK_ARG(mode >= KFAC_EKFAC_KEEP && mode <= KFAC_EKFAC_SEED, "mode");
  if (count == 0) return KFAC_OK;
  const bool reads = mode == KFAC_EKFAC_EMA || mode == KFAC_EKFAC_RESET;
  std::vector<UpdDev> dev(count);
  long long total = 0;
  for (int i = 0; i < count; ++i) {
    const kfac_ekfac_update_item& it = items[i];
    KFAC_CHECK_ARG(it.S && it.dgda && it.g > 0 && it.a > 0 && it.ld >= it.a, "ekfac update item");
    KFAC_CHECK_ARG(!reads || it.S_batch, "ekfac update: S_batch is needed by the EMA and reset modes");
    KFAC_CHECK_ARG((mode != KFAC_EKFAC_SEED && mode != KFAC_EKFAC_RESET) || (it.dg && it.da),
                   "ekfac update: the seed (and the reset fallback) need dg and da");
    dev[i] = UpdDev{it.S, it.S_batch, it.dg, it.da, it.dgda, it.drop_a, it.drop_g, it.g, it.a, it.ld, total};
    total += (long long)it.g * it.ld;
  }
  const size_t need = kfac_ekfac_update_workspace_bytes(count);
  if (!ws || ws_bytes < need) {
    set_error("ekfac_update: workspace too small (%zu < %zu)", ws_bytes, need);
    return KFAC_ERR_WORKSPACE;
  }
  cudaStream_t s = (cudaStream_t)stream;
  const UpdDev* table = (const UpdDev*)ws;
  int* bad = (int*)((char*)ws + upd_table_bytes(count));
  KFAC_CUDA(cudaMemcpyAsync(ws, dev.data(), sizeof(UpdDev) * count, cudaMemcpyHostToDevice, s));   // pageable: staged
  KFAC_CUDA(cudaMemsetAsync(bad, 0, (size_t)count * sizeof(int), s));
  if (reads) {
    sbatch_scan_kernel<<<grid_for(total), 256, 0, s>>>(table, count, total, bad);
    KFAC_LAUNCH_CHECK();
  }
  ekfac_update_kernel<<<grid_for(total), 256, 0, s>>>(table, count, total, alpha, mode, damping, bad, skipped);
  KFAC_LAUNCH_CHECK();
  return KFAC_OK;
}
