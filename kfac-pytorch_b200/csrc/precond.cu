// K7-K12: damped inverse from the eigendecomposition, two-sided Kronecker
// precondition, kl-clip scale and in-place gradient write-back.
#include <string.h>

#include <algorithm>
#include <array>
#include <cmath>
#include <vector>

#include "common.cuh"
#include "gemm_grouped.cuh"

namespace kfac {

// grad matrix (g x a) fp32 = [wgrad (g x a-hb) | bgrad]   (modules.py:56-69)
__global__ void gather_grad_kernel(const void* w, const void* b, int dtype, int g, int a, float* out,
                                   int ldo) {
  const int aw = b ? a - 1 : a;
  const int64_t total = (int64_t)g * ldo;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = idx / ldo;
    const int j = (int)(idx % ldo);
    float v = 0.f;   // padding columns are zero (they feed the K dimension of the next GEMM)
    if (j < aw) v = load_as_float(w, dtype, i * aw + j);
    else if (j < a) v = load_as_float(b, dtype, i);
    out[idx] = v;
  }
}

// Offset in wgrad of element (r, c) of the (g, aw) weight-gradient matrix: row-major (taps = 0), or a transposed
// convolution's (C_in, g, taps) weight with c = ci * taps + t (kfac_precond_item.wgrad_taps)
__device__ __forceinline__ long long wgrad_offset(long long r, int c, int g, int aw, int taps) {
  if (taps == 0) return r * aw + c;
  const int ci = c / taps;
  return ((long long)ci * g + r) * taps + (c - ci * taps);
}

// all layers in one launch: item i owns the elements [elem0, elem0 + g * ldo) of the concatenated space
struct GatherDev { const void* w; const void* b; int dtype, g, a, ldo; float* out; long long elem0; int taps; };
__global__ void __launch_bounds__(256) gather_all_kernel(const GatherDev* items, int count, long long total) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    int lo = 0, hi = count - 1;
    while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (items[mid].elem0 <= e) lo = mid; else hi = mid - 1; }
    const GatherDev& it = items[lo];
    const long long idx = e - it.elem0;
    const long long i = idx / it.ldo;
    const int j = (int)(idx % it.ldo);
    const int aw = it.b ? it.a - 1 : it.a;
    float v = 0.f;
    if (j < aw) v = load_as_float(it.w, it.dtype, wgrad_offset(i, j, it.g, aw, it.taps));
    else if (j < it.a) v = load_as_float(it.b, it.dtype, i);
    it.out[idx] = v;
  }
}

// out (a x ldo) = grad^T for the (g, a) grad matrix [wgrad | bgrad], zero in the columns [g, ldo): the K-major operand of a
// diagonal-A item's products.  32 x 32 tiles through shared memory, so that both the reads of grad and the writes of
// out are coalesced
__global__ void __launch_bounds__(256) gather_t_kernel(const void* w, const void* b, int dtype, int g, int a, float* out,
                                                       int ldo) {
  __shared__ float tile[32][33];
  const int j0 = blockIdx.x * 32, i0 = blockIdx.y * 32;   // j: row of grad (column of out), i: column of grad
  const int aw = b ? a - 1 : a;
  for (int r = threadIdx.y; r < 32; r += 8) {
    const int j = j0 + r, i = i0 + threadIdx.x;
    float v = 0.f;
    if (j < g && i < aw) v = load_as_float(w, dtype, (long long)j * aw + i);
    else if (j < g && i < a) v = load_as_float(b, dtype, j);
    tile[r][threadIdx.x] = v;
  }
  __syncthreads();
  for (int r = threadIdx.y; r < 32; r += 8) {
    const int i = i0 + r, j = j0 + threadIdx.x;
    if (i < a && j < ldo) out[(long long)i * ldo + j] = tile[threadIdx.x][r];
  }
}

// ---- kl-clip scale and write-back: ONE launch each over all layers, deterministic ---------------
// device copy of a kfac_grad_item + the offset of its g*a elements in the concatenated element space
struct GradDev { const float* P; void* w; void* b; int dtype, g, a, ldp; long long elem0; int taps; };
constexpr int VG_BLOCKS = 592;          // 4 per SM; partial sums are combined in a fixed order

__device__ __forceinline__ int find_item(const GradDev* items, int count, long long e) {
  int lo = 0, hi = count - 1;
  while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (items[mid].elem0 <= e) lo = mid; else hi = mid - 1; }
  return lo;
}

// partials[block] = sum over the block's contiguous element range of P * grad (double accumulation);
// the assignment of elements to threads and the reduction tree are fixed -> bitwise reproducible
__global__ void __launch_bounds__(256) vg_all_kernel(const GradDev* items, int count, long long total, double* partials) {
  const long long per = (total + gridDim.x - 1) / gridDim.x;
  const long long e0 = (long long)blockIdx.x * per, e1 = min(total, e0 + per);
  double acc = 0.0;
  for (long long e = e0 + threadIdx.x; e < e1; e += blockDim.x) {
    const GradDev& it = items[find_item(items, count, e)];
    const long long loc = e - it.elem0;
    const long long i = loc / it.a;
    const int j = (int)(loc % it.a);
    const int aw = it.b ? it.a - 1 : it.a;
    const float gr = (j < aw) ? load_as_float(it.w, it.dtype, wgrad_offset(i, j, it.g, aw, it.taps))
                              : load_as_float(it.b, it.dtype, i);
    acc += (double)it.P[i * it.ldp + j] * (double)gr;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  __shared__ double red[8];
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int k = 0; k < 8; ++k) t += red[k];
    partials[blockIdx.x] = t;
  }
}

__global__ void nu_kernel(const double* partials, int n, float kl_clip, float lr, double* vg_out, float* out) {
  double vg = 0.0;
  for (int i = 0; i < n; ++i) vg += partials[i];
  *vg_out = vg;
  const double v = vg * (double)lr * (double)lr;
  float nu = 1.f;
  if (v != 0.0) nu = (float)fmin(1.0, sqrt((double)kl_clip / fabs(v)));
  *out = nu;
}

__global__ void __launch_bounds__(256) update_all_kernel(const GradDev* items, int count, long long total, const float* scale) {
  const float s = scale ? *scale : 1.f;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const GradDev& it = items[find_item(items, count, e)];
    const long long loc = e - it.elem0;
    const long long i = loc / it.a;
    const int j = (int)(loc % it.a);
    const int aw = it.b ? it.a - 1 : it.a;
    const float v = s * it.P[i * it.ldp + j];
    if (j < aw) store_from_float(it.w, it.dtype, wgrad_offset(i, j, it.g, aw, it.taps), v);
    else store_from_float(it.b, it.dtype, i, v);
  }
}

// out[i][j] = Q[i][j] / (d[j] + damping), zero in the padding columns; with pi, damping is pi_gamma(damping, *pi, side)
__global__ void scale_cols_kernel(const float* Q, int ldq, const float* d, int n, float damping, const float* pi,
                                  int side, float* out) {
  if (pi) damping = pi_gamma(damping, *pi, side);
  const int64_t total = (int64_t)n * ldq;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int j = (int)(idx % ldq);
    out[idx] = j < n ? Q[idx] / (d[j] + damping) : 0.f;
  }
}

__global__ void transpose_kernel(const float* src, int lds, float* dst, int ldd, int rows, int cols) {
  __shared__ float tile[32][33];
  const int bx = blockIdx.x * 32, by = blockIdx.y * 32;
  for (int r = threadIdx.y; r < 32; r += 8) {
    const int i = by + r, j = bx + threadIdx.x;
    tile[r][threadIdx.x] = (i < rows && j < cols) ? src[(int64_t)i * lds + j] : 0.f;
  }
  __syncthreads();
  for (int r = threadIdx.y; r < 32; r += 8) {
    const int j = bx + r, i = by + threadIdx.x;    // dst[j][i] = src[i][j]
    if (j < cols && i < rows) dst[(int64_t)j * ldd + i] = tile[threadIdx.x][r];
  }
}

static inline int grid_for(int64_t total) {
  int64_t b = (total + 255) / 256;
  return (int)max((int64_t)1, min(b, (int64_t)tc_num_sms() * 8));
}

struct Epi { int kind = EPI_NONE; const float* E = nullptr; int64_t lde = 0;
             const float* dg = nullptr; const float* da = nullptr; float damping = 0.f; };

// D (M x N, ldd) = epi(A B^T), A (M x K, lda), B (N x K, ldb): tensor-core engine for
// aligned operands with at least one full tile worth of work, SIMT engine otherwise.
// Deterministic: no floating-point atomics on any path.
int gemm_tn(const float* A, int64_t lda, const float* B, int64_t ldb, float* D, int64_t ldd, int M, int N,
            int K, const Epi& e, cudaStream_t s) {
  TcGemmArgs t{};
  t.npeer = 0;
  t.A = A; t.lda = lda; t.B = B; t.ldb = ldb; t.D = D; t.ldd = ldd; t.M = M; t.N = N; t.K = K;
  t.kbatch = 1; t.alpha = 1.f; t.splits = 1;
  t.epi = e.kind; t.E = e.E; t.lde = e.lde; t.dg = e.dg; t.da = e.da; t.damping = e.damping;
  if (M >= 64 && N >= 64 && K >= 32 && tc_gemm_supported(t)) {
    if (e.kind == EPI_NONE && chain_splits(K) > 1) {
      // long reductions run as chains of <= 512, split the way the engine splits k-blocks for ceil(K / 512)
      // splits: the tensor-core accumulator truncates, so short chains keep the 3xTF32 result at fp32 accuracy.
      // The chains run in order on the stream, the first storing D and each later one adding its product to D
      // (plain read-modify-write epilogue), so the sum has one fixed order; the TMA maps zero-fill past a chain.
      constexpr int KB = 32;                    // the engine's k-block
      const int kb_total = ceil_div(K, KB);
      const int chain = ceil_div(kb_total, tc_normalize_splits(chain_splits(K), kb_total)) * KB;
      for (int k0 = 0; k0 < K; k0 += chain) {
        TcGemmArgs c = t;
        c.A = A + k0; c.B = B + k0; c.K = std::min(chain, K - k0); c.accumulate = k0 > 0;
        const int rc = launch_tc_gemm(c, s);
        if (rc) return rc;
      }
      return KFAC_OK;
    }
    return launch_tc_gemm(t, s);
  }
  GemmArgs g{};
  g.A = A; g.sa_m = lda; g.sa_k = 1; g.B = B; g.sb_k = 1; g.sb_n = ldb;
  g.C = D; g.ldc = ldd; g.M = M; g.N = N; g.K = K; g.batch = 1; g.splitk = 1;
  g.alpha = 1.f; g.beta = 0.f;
  g.epi = e.kind; g.E = e.E; g.lde = e.lde; g.dg = e.dg; g.da = e.da; g.damping = e.damping;
  return launch_gemm(g, s);
}

int gemm_tn_plain(const float* A, int64_t lda, const float* B, int64_t ldb, float* D, int64_t ldd, int M, int N,
                  int K, cudaStream_t s) {
  return gemm_tn(A, lda, B, ldb, D, ldd, M, N, K, Epi{}, s);
}

}  // namespace kfac

using namespace kfac;

static inline int ld4(int x) { return (x + 3) & ~3; }

// inv = Q diag(1 / (d + gamma)) Q^T with gamma = damping, or pi_gamma(damping, *pi, side) with pi
static int inverse_from_eigh(const float* Q, int ldq, const float* d, int n, float damping, const float* pi, int side,
                             float* inv, int ld_inv, void* ws, size_t ws_bytes, void* stream) {
  KFAC_CHECK_ARG(Q && d && inv && n > 0 && ldq >= n && ld_inv >= n, "inverse args");
  const size_t need = (size_t)n * ldq * sizeof(float);
  if (!ws || ws_bytes < need) {
    set_error("inverse_from_eigh: workspace too small (%zu < %zu)", ws_bytes, need);
    return KFAC_ERR_WORKSPACE;
  }
  cudaStream_t s = (cudaStream_t)stream;
  float* T = (float*)ws;
  scale_cols_kernel<<<grid_for((int64_t)n * ldq), 256, 0, s>>>(Q, ldq, d, n, damping, pi, side, T);
  KFAC_LAUNCH_CHECK();
  // inv[i][j] = sum_k T[i][k] Q[j][k]; the same bits in every call (for n > 1024 the chains of gemm_tn)
  return gemm_tn(T, ldq, Q, ldq, inv, ld_inv, n, n, n, Epi{}, s);
}

extern "C" int kfac_inverse_from_eigh(const float* Q, int ldq, const float* d, int n, float damping,
                                      float* inv, int ld_inv, void* ws, size_t ws_bytes, void* stream) {
  return inverse_from_eigh(Q, ldq, d, n, damping, nullptr, 0, inv, ld_inv, ws, ws_bytes, stream);
}

extern "C" int kfac_inverse_from_eigh_pi(const float* Q, int ldq, const float* d, int n, float s, const float* pi,
                                         int side, float* inv, int ld_inv, void* ws, size_t ws_bytes, void* stream) {
  KFAC_CHECK_ARG(pi && (side == 1 || side == -1), "inverse_pi args");
  return inverse_from_eigh(Q, ldq, d, n, s, pi, side, inv, ld_inv, ws, ws_bytes, stream);
}

extern "C" int kfac_transpose(const float* src, int ld_src, float* dst, int ld_dst, int rows, int cols,
                              void* stream) {
  KFAC_CHECK_ARG(src && dst && rows > 0 && cols > 0 && ld_src >= cols && ld_dst >= rows, "transpose args");
  dim3 grid(ceil_div(cols, 32), ceil_div(rows, 32));
  transpose_kernel<<<grid, dim3(32, 8), 0, (cudaStream_t)stream>>>(src, ld_src, dst, ld_dst, rows, cols);
  KFAC_LAUNCH_CHECK();
  return KFAC_OK;
}

struct TiedScaleDev { float* T; const float* f; const float* h; const float* mu; float t; int n, ld; long long elem0; };

// ---- precondition: stage-wise over ALL items -------------------------------------------------------
// Every item is a chain of up to four products, and stage k of all items is one grouped launch.  An item's plan
// (plan_item) says how its gradient is gathered, which scratch matrices it needs and which product it runs in each
// stage; the workspace and the launches are derived from the plans.
//
// An embedding item and a diagonal-G item are the same problem with the sides swapped: a gradient of `rows` x n
// (V x d for an embedding, V x a for a diagonal-G layer), one dense factor of size n on its columns (G, resp. A:
// basis q, its transpose qT, inverse inv, eigenvalues vcol) and one diagonal factor vrow on its rows.  P has the
// gradient's layout, rows x n.  A tied item is an embedding item whose basis q = M is not orthogonal and whose
// epilogue reads a second row vector vrow2 = h and its own damping (KFAC_ITEM_TIED in the header).  A diagonal-A item
// is the embedding problem on grad^T (rows = a, n = g), gathered transposed; its last product is formed transposed,
// so that P keeps the dense layout n x rows (g x a).
struct DiagItem {
  int rows, n;
  const float *q, *qT, *inv, *vrow, *vcol;
  int ldq;
  const float* vrow2;
  float damping;
  int side_row;   // the factor of vrow under pi-adjusted damping: +1 A, -1 G (vcol is the other one)
};

static bool is_diag_a(const kfac_precond_item& it) { return it.kind == KFAC_ITEM_DIAG_A; }

// the workspace regions of one item (null while the workspace is being sized)
struct Scratch { float *gr, *t1, *t2; const float* ones; };

struct ItemPlan {
  int rc = KFAC_OK; const char* err = nullptr;   // the first check the item fails, reported after the workspace check
  // the gradient matrix [wgrad | bgrad], rows x cols (wgrad laid out as wgrad_offset says for taps), goes to GR as
  // rows x ld4(cols), or transposed as cols x ld4(rows) by gather_t_kernel
  int rows = 0, cols = 0, taps = 0;
  bool transposed = false;
  size_t gr = 0, t1 = 0, t2 = 0;   // floats of the scratch matrices GR, T1, T2
  int ones = 0;                    // length of the ones vector its product reads under the inverse method
  Scratch w{};
  // the product of stages (1) to (4) (M = N = K = 0: none); the last one writes P and carries the peer stores.  A
  // product with splits > 1 keeps its partial tiles in the slab of the product of stage slab_of[k] of this item.
  GroupedGemm stage[4] = {};
  int slab_of[4] = {0, 1, 2, 3};
  bool tied = false; TiedScaleDev tied_scale{};   // stage (1)'s product is divided by tied_scale_kernel
};

static GroupedGemm product(const float* A, int64_t lda, const float* B, int64_t ldb, float* D, int64_t ldd, int M,
                           int N, int K, int splits = 1) {
  GroupedGemm g{};
  g.A = A; g.lda = lda; g.B = B; g.ldb = ldb; g.D = D; g.ldd = ldd; g.M = M; g.N = N; g.K = K; g.alpha = 1.f;
  g.epi = EPI_NONE; g.splits = splits;
  return g;
}

// the product divided by (dg[m] * da[n] + damping) in its epilogue
static GroupedGemm div_outer(GroupedGemm g, const float* dg, const float* da, float damping) {
  g.epi = EPI_DIV_OUTER; g.dg = dg; g.da = da; g.damping = damping;
  return g;
}

// the product divided by (dm[m] + gamma_m) (dn[n] + gamma_n) in its epilogue, gamma_m = pi_gamma(s, *pi, side_m)
static GroupedGemm div_factored(GroupedGemm g, const float* dm, const float* dn, const float* pi, float s, int side_m,
                                int side_n) {
  g.epi = EPI_DIV_FACTORED; g.dg = dm; g.da = dn; g.pi = pi; g.damping = s; g.pi_side_m = side_m; g.pi_side_n = side_n;
  return g;
}

#define PLAN_CHECK(cond, what) \
  do { if (!p.err && !(cond)) fail(KFAC_ERR_BAD_ARG, "bad argument: " what " (" #cond ")"); } while (0)

// The plan of one item under `method`.  The sizes and the products do not depend on whether the item passes its
// checks, so that a call is sized the same way before and after they run.
static ItemPlan plan_item(const kfac_precond_item& it, int method, float damping, const Scratch& w) {
  ItemPlan p;
  p.w = w;
  auto fail = [&](int rc, const char* msg) { if (!p.err) { p.rc = rc; p.err = msg; } };
  PLAN_CHECK(it.kind == KFAC_ITEM_DENSE || it.kind == KFAC_ITEM_EMBEDDING || it.kind == KFAC_ITEM_DIAG_G ||
                 it.kind == KFAC_ITEM_TIED || it.kind == KFAC_ITEM_DIAG_A, "precond item kind");
  PLAN_CHECK(it.n_peers >= 0 && it.n_peers <= 7 && (it.n_peers == 0 || it.peer_P), "precond peers");
  PLAN_CHECK(!it.pi || it.kind != KFAC_ITEM_TIED, "precond tied item pi");
  const bool eigen = method == KFAC_EIGEN;
  // the division of an item's eigenvalues (or diagonal factor): by (u v + damping), or with pi by the factored
  // (u + gamma_u)(v + gamma_v) with s = sqrt(damping); side 0 is a vector of ones, which takes no damping
  const float s = std::sqrt(damping);
  auto divide = [&](GroupedGemm g, const float* u, const float* v, int side_u, int side_v) {
    return it.pi ? div_factored(g, u, v, it.pi, s, side_u, side_v) : div_outer(g, u, v, damping);
  };
  GroupedGemm* st = p.stage;
  if (it.kind == KFAC_ITEM_DENSE) {
    PLAN_CHECK(it.wgrad && it.P && it.g > 0 && it.a > 0 && it.ldp >= it.a, "precond item");
    if (eigen ? !(it.qa && it.qg && it.qaT && it.qgT && (it.dgda || (it.da && it.dg))) : !(it.a_inv && it.g_inv))
      fail(KFAC_ERR_NOT_READY, eigen ? "precondition: eigendecompositions for both A and G have not been computed"
                                     : "precondition: A and G have not been inverted");
    PLAN_CHECK(it.ldqa >= it.a && it.ldqg >= it.g, "second-order leading dims");
    PLAN_CHECK(it.wgrad_taps >= 0 && (it.wgrad_taps == 0 || (it.a - (it.bgrad ? 1 : 0)) % it.wgrad_taps == 0),
               "precond item wgrad_taps");
    const int g = it.g, a = it.a;
    p.rows = g; p.cols = a; p.taps = it.wgrad_taps;
    p.gr = (size_t)g * ld4(a); p.t1 = (size_t)a * ld4(g); p.t2 = (size_t)g * ld4(a);
    // (1) T^T[a', r] = sum_k (QaT | Ainv)[a', k] grad[r, k]                                  (a x g, K = a)
    st[0] = product(eigen ? it.qaT : it.a_inv, it.ldqa, w.gr, ld4(a), w.t1, ld4(g), a, g, a, chain_splits(a));
    if (eigen) {
      // (2) V2[g', a'] = (sum_k QgT[g', k] T^T[a', k]) * dgda[g', a'], or / (dg[g'] da[a'] + damping)   (g x a, K = g)
      st[1] = product(it.qgT, it.ldqg, w.t1, ld4(g), w.t2, ld4(a), g, a, g);
      if (it.dgda) { st[1].epi = EPI_MUL; st[1].E = it.dgda; st[1].lde = it.ld_dgda; }
      else st[1] = divide(st[1], it.dg, it.da, -1, 1);
      // (3) U^T[c, g'] = sum_k Qa[c, k] V2[g', k]                                  (a x g, K = a, stage (1)'s slab)
      st[2] = product(it.qa, it.ldqa, w.t2, ld4(a), w.t1, ld4(g), a, g, a, chain_splits(a));
      p.slab_of[2] = 0;
    }
    // (4) P[r, c] = sum_k (Qg | Ginv)[r, k] U^T[c, k]                                       (g x a, K = g)
    st[3] = product(eigen ? it.qg : it.g_inv, it.ldqg, w.t1, ld4(g), it.P, it.ldp, g, a, g);
  } else {
    DiagItem D;
    const char* not_ready;
    switch (it.kind) {
      case KFAC_ITEM_EMBEDDING:
      case KFAC_ITEM_DIAG_A:
        D = DiagItem{it.a, it.g, it.qg, it.qgT, it.g_inv, it.da, it.dg, it.ldqg, nullptr, 0.f, 1};
        not_ready = is_diag_a(it) ? "precondition: the second-order data of a diagonal-A layer has not been computed"
                                  : "precondition: the second-order data of an embedding layer has not been computed";
        break;
      case KFAC_ITEM_TIED:
        D = DiagItem{it.a, it.g, it.qg, it.qgT, nullptr, it.da, it.dg, it.ldqg, it.dh, it.tied_damping, 1};
        not_ready = "precondition: the second-order data of a tied embedding / head pair has not been computed";
        break;
      default:                          // KFAC_ITEM_DIAG_G, or a kind the first check rejects
        D = DiagItem{it.g, it.a, it.qa, it.qaT, it.a_inv, it.dg, it.da, it.ldqa, nullptr, 0.f, -1};
        not_ready = "precondition: the second-order data of a diagonal-G layer has not been computed";
    }
    PLAN_CHECK(it.wgrad && it.P && it.g > 0 && it.a > 0 && it.ldp >= (is_diag_a(it) ? D.rows : D.n) &&
                   D.ldq >= D.n && (it.kind == KFAC_ITEM_DIAG_G || is_diag_a(it) || !it.bgrad),
               "precond diagonal item");
    PLAN_CHECK(it.kind != KFAC_ITEM_TIED || it.tied_damping > 0.f, "precond tied item damping");
    const bool tied = it.kind == KFAC_ITEM_TIED;
    if (!(D.vrow && (tied ? (D.q && D.qT && D.vcol && D.vrow2) : eigen ? (D.q && D.qT && D.vcol) : D.inv != nullptr)))
      fail(KFAC_ERR_NOT_READY, not_ready);
    const int ldn = ld4(D.n);
    p.transposed = is_diag_a(it);
    p.rows = p.transposed ? D.n : D.rows; p.cols = p.transposed ? D.rows : D.n;
    p.gr = p.t1 = (size_t)D.rows * ldn;
    p.ones = tied ? 0 : D.n;
    if (tied || eigen) {
      // (1) T[v, j] = (sum_k grad[v, k] Q[k, j]) / (vrow[v] vcol[j] + damping), the division of a tied item by
      // tied_scale_kernel                                                                      (rows x n, K = n)
      st[0] = product(w.gr, ldn, D.qT, D.ldq, w.t1, ldn, D.rows, D.n, D.n);
      if (!tied) st[0] = divide(st[0], D.vrow, D.vcol, D.side_row, -D.side_row);
      else { p.tied = true; p.tied_scale = TiedScaleDev{w.t1, D.vrow, D.vrow2, D.vcol, D.damping, D.n, ldn, 0}; }
    }
    if (is_diag_a(it)) {
      // (4) P[r, c] = sum_k Qg[r, k] T[c, k], or (sum_k Ginv[r, k] grad^T[c, k]) / (a[c] + damping)   (g x a, K = g)
      st[3] = eigen ? product(D.q, D.ldq, w.t1, ldn, it.P, it.ldp, D.n, D.rows, D.n)
                    : divide(product(D.inv, D.ldq, w.gr, ldn, it.P, it.ldp, D.n, D.rows, D.n), w.ones, D.vrow, 0,
                             D.side_row);
    } else {
      // (4) P[v, c] = sum_k T[v, k] Q[c, k], or (sum_k grad[v, k] Inv[c, k]) / (vrow[v] + damping)  (rows x n, K = n)
      st[3] = eigen || tied ? product(w.t1, ldn, D.q, D.ldq, it.P, it.ldp, D.rows, D.n, D.n)
                            : divide(product(w.gr, ldn, D.inv, D.ldq, it.P, it.ldp, D.rows, D.n, D.n), D.vrow,
                                     w.ones, D.side_row, 0);
    }
  }
  // the last product splits where it has the plain epilogue and P is at its padded width
  if (st[3].epi == EPI_NONE && it.ldp == ld4(st[3].N)) st[3].splits = chain_splits(st[3].K);
  if (!p.err) {
    // fused compute + broadcast: the same P goes to the peers, from the tile epilogue or from the split's reduce pass
    st[3].npeer = it.n_peers;
    for (int q = 0; q < it.n_peers; ++q) st[3].peerD[q] = it.peer_P[q];
  }
  return p;
}

#undef PLAN_CHECK

// workspace: [GatherDev table][TiedScaleDev table][grouped-GEMM tables][ones vector][per item: GR, T1, T2][slabs]
struct PrecondLayout { size_t off_gather, off_tied, off_gemm, off_ones, total; int ones_n; };

// Plans every item and lays out the workspace from the plans; with a base, the plans address that workspace.
static PrecondLayout plan_items(const kfac_precond_item* items, int count, int method, float damping, char* base,
                                std::vector<ItemPlan>& plans) {
  PrecondLayout L{};
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off = align_up(off + bytes, 256); return o; };
  auto at = [&](size_t o) { return base ? (float*)(base + o) : nullptr; };
  plans.resize(count);
  for (int i = 0; i < count; ++i) plans[i] = plan_item(items[i], method, damping, Scratch{});
  L.off_gather = take(sizeof(GatherDev) * (size_t)std::max(1, count));
  L.off_tied = take(sizeof(TiedScaleDev) * (size_t)std::max(1, count));
  L.off_gemm = take(grouped_gemm_ws_bytes(count));
  for (const ItemPlan& p : plans) L.ones_n = std::max(L.ones_n, p.ones);
  L.off_ones = L.ones_n ? take((size_t)L.ones_n * sizeof(float)) : off;
  std::vector<Scratch> w(count);
  for (int i = 0; i < count; ++i) {   // a braced list is evaluated in order: GR, T1, T2
    const ItemPlan& p = plans[i];
    w[i] = Scratch{at(take(p.gr * sizeof(float))), at(take(p.t1 * sizeof(float))), at(take(p.t2 * sizeof(float))),
                   at(L.off_ones)};
  }
  // long reductions (K > 1024) are split into chains of <= 512: the tensor-core accumulator truncates, short
  // chains keep the 3xTF32 result at fp32 accuracy; the partial tiles go to slabs and are added in a fixed order
  // (deterministic: every replica that preconditions a layer locally must get the same bits).  The layout does not
  // depend on n_peers: a fused broadcast runs the same split, its peers get the reduced sums.
  std::vector<std::array<float*, 4>> slab(count);
  for (int i = 0; i < count; ++i)
    for (int k = 0; k < 4; ++k) {
      const GroupedGemm& g = plans[i].stage[k];
      if (g.splits > 1 && plans[i].slab_of[k] == k) slab[i][k] = at(take((size_t)g.splits * g.M * g.ldd * sizeof(float)));
    }
  L.total = off;
  if (!base) return L;
  for (int i = 0; i < count; ++i) {
    ItemPlan& p = plans[i] = plan_item(items[i], method, damping, w[i]);
    for (int k = 0; k < 4; ++k) {
      GroupedGemm& g = p.stage[k];
      if (g.splits > 1) { g.slab = slab[i][p.slab_of[k]]; g.slab_stride = (int64_t)g.M * g.ldd; }
    }
  }
  return L;
}

// T[v][j] /= (f[v] + t) + (h[v] + t) mu[j] for every tied item, one launch: the division of a tied item's first product,
// kept out of the GEMM engines so that their epilogues (shared by every layer) stay as they are
__global__ void __launch_bounds__(256) tied_scale_kernel(const TiedScaleDev* items, int count, long long total) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    int lo = 0, hi = count - 1;
    while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (items[mid].elem0 <= e) lo = mid; else hi = mid - 1; }
    const TiedScaleDev& it = items[lo];
    const long long idx = e - it.elem0;
    const long long v = idx / it.ld;
    const int j = (int)(idx % it.ld);
    if (j < it.n) it.T[idx] = it.T[idx] / ((it.f[v] + it.t) + (it.h[v] + it.t) * it.mu[j]);
  }
}

__global__ void fill_ones_kernel(float* out, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) out[i] = 1.f;
}

extern "C" size_t kfac_precondition_workspace_bytes(const kfac_precond_item* items, int count) {
  if (count <= 0) return 0;
  // enough for either method (the eigen method's plans split the most)
  std::vector<ItemPlan> plans;
  return std::max(plan_items(items, count, KFAC_EIGEN, 0.f, nullptr, plans).total,
                  plan_items(items, count, KFAC_INVERSE, 0.f, nullptr, plans).total);
}

extern "C" int kfac_precondition(const kfac_precond_item* items, int count, int method, float damping,
                                 void* ws, size_t ws_bytes, void* stream) {
  KFAC_CHECK_ARG(count >= 0 && (items || count == 0), "items");
  KFAC_CHECK_ARG(method == KFAC_EIGEN || method == KFAC_INVERSE, "method");
  if (count == 0) return KFAC_OK;
  std::vector<ItemPlan> plans;
  char* base = (char*)ws;
  const PrecondLayout L = plan_items(items, count, method, damping, base, plans);
  if (!ws || ws_bytes < L.total) {
    set_error("precondition: workspace too small (%zu < %zu)", ws_bytes, L.total);
    return KFAC_ERR_WORKSPACE;
  }
  for (const ItemPlan& p : plans)
    if (p.rc) { set_error("%s", p.err); return p.rc; }
  cudaStream_t s = (cudaStream_t)stream;
  // stage 0: the gradient matrices of all items, one launch (the transposed ones have no elements in it)
  std::vector<GatherDev> gat(count);
  long long total = 0;
  for (int i = 0; i < count; ++i) {
    const kfac_precond_item& it = items[i];
    const ItemPlan& p = plans[i];
    if (p.transposed) { gat[i] = GatherDev{it.wgrad, it.bgrad, it.grad_dtype, 0, 0, 1, p.w.gr, total, 0}; continue; }
    gat[i] = GatherDev{it.wgrad, it.bgrad, it.grad_dtype, p.rows, p.cols, ld4(p.cols), p.w.gr, total, p.taps};
    total += (long long)p.rows * ld4(p.cols);
  }
  KFAC_CUDA(cudaMemcpyAsync(base + L.off_gather, gat.data(), sizeof(GatherDev) * count, cudaMemcpyHostToDevice, s));
  gather_all_kernel<<<grid_for(total), 256, 0, s>>>((const GatherDev*)(base + L.off_gather), count, total);
  KFAC_LAUNCH_CHECK();
  for (int i = 0; i < count; ++i) {
    const kfac_precond_item& it = items[i];
    if (!plans[i].transposed) continue;
    KFAC_CHECK_ARG(ceil_div(it.a, 32) <= 65535, "precond diagonal-A item: a");
    const dim3 grid((unsigned)ceil_div(ld4(it.g), 32), (unsigned)ceil_div(it.a, 32));
    gather_t_kernel<<<grid, dim3(32, 8), 0, s>>>(it.wgrad, it.bgrad, it.grad_dtype, it.g, it.a, plans[i].w.gr, ld4(it.g));
    KFAC_LAUNCH_CHECK();
  }
  if (L.ones_n && method == KFAC_INVERSE) {
    fill_ones_kernel<<<grid_for(L.ones_n), 256, 0, s>>>((float*)(base + L.off_ones), L.ones_n);
    KFAC_LAUNCH_CHECK();
  }
  // stage k of all items is one grouped launch (none where no item has a product in it)
  std::vector<GroupedGemm> st(count);
  auto run = [&](int k) {
    for (int i = 0; i < count; ++i) st[i] = plans[i].stage[k];
    return launch_grouped_gemm(st.data(), count, base + L.off_gemm, grouped_gemm_ws_bytes(count), s);
  };
  int rc;
  if ((rc = run(0))) return rc;
  // the tied items' division, elementwise over all of them in one launch
  std::vector<TiedScaleDev> tied;
  long long tied_total = 0;
  for (const ItemPlan& p : plans) {
    if (!p.tied) continue;
    tied.push_back(p.tied_scale);
    tied.back().elem0 = tied_total;
    tied_total += (long long)p.stage[0].M * p.stage[0].ldd;
  }
  if (!tied.empty()) {
    KFAC_CUDA(cudaMemcpyAsync(base + L.off_tied, tied.data(), sizeof(TiedScaleDev) * tied.size(), cudaMemcpyHostToDevice, s));
    tied_scale_kernel<<<grid_for(tied_total), 256, 0, s>>>((const TiedScaleDev*)(base + L.off_tied), (int)tied.size(),
                                                           tied_total);
    KFAC_LAUNCH_CHECK();
  }
  for (int k = 1; k < 4; ++k)
    if ((rc = run(k))) return rc;
  return KFAC_OK;
}

extern "C" size_t kfac_grad_workspace_bytes(int count) {
  return align_up(sizeof(GradDev) * (size_t)std::max(1, count), 256) + align_up(sizeof(double) * (VG_BLOCKS + 1), 256);
}

// uploads the item table into the workspace; returns the total number of gradient elements
static int upload_grad_items(const kfac_grad_item* items, int count, void* ws, size_t ws_bytes, cudaStream_t s,
                             long long* total_out) {
  if (!ws || ws_bytes < kfac_grad_workspace_bytes(count)) {
    set_error("grad scale/update: workspace too small (%zu < %zu)", ws_bytes, kfac_grad_workspace_bytes(count));
    return KFAC_ERR_WORKSPACE;
  }
  std::vector<GradDev> dev(count);
  long long total = 0;
  for (int i = 0; i < count; ++i) {
    const kfac_grad_item& it = items[i];
    KFAC_CHECK_ARG(it.P && it.wgrad && it.g > 0 && it.a > 0 && it.ldp >= it.a, "grad item");
    KFAC_CHECK_ARG(it.wgrad_taps >= 0 && (it.wgrad_taps == 0 || (it.a - (it.bgrad ? 1 : 0)) % it.wgrad_taps == 0),
                   "grad item wgrad_taps");
    dev[i] = GradDev{it.P, it.wgrad, it.bgrad, it.grad_dtype, it.g, it.a, it.ldp, total, it.wgrad_taps};
    total += (long long)it.g * it.a;
  }
  KFAC_CUDA(cudaMemcpyAsync(ws, dev.data(), sizeof(GradDev) * count, cudaMemcpyHostToDevice, s));   // pageable: staged
  *total_out = total;
  return KFAC_OK;
}

extern "C" int kfac_grad_scale(const kfac_grad_item* items, int count, float kl_clip, float lr, void* ws,
                               size_t ws_bytes, float* scale_out, void* stream) {
  KFAC_CHECK_ARG(count >= 0 && (items || count == 0) && scale_out, "grad_scale args");
  cudaStream_t s = (cudaStream_t)stream;
  long long total = 0;
  if (count > 0) { const int rc = upload_grad_items(items, count, ws, ws_bytes, s, &total); if (rc) return rc; }
  else if (!ws || ws_bytes < kfac_grad_workspace_bytes(0)) { set_error("grad_scale: workspace"); return KFAC_ERR_WORKSPACE; }
  double* partials = (double*)((char*)ws + align_up(sizeof(GradDev) * (size_t)std::max(1, count), 256));
  const int nblk = (int)std::max<long long>(1, std::min<long long>(VG_BLOCKS, (total + 255) / 256));
  if (count > 0) {
    vg_all_kernel<<<nblk, 256, 0, s>>>((const GradDev*)ws, count, total, partials);
    KFAC_LAUNCH_CHECK();
  }
  nu_kernel<<<1, 1, 0, s>>>(partials, count > 0 ? nblk : 0, kl_clip, lr, partials + VG_BLOCKS, scale_out);
  KFAC_LAUNCH_CHECK();
  return KFAC_OK;
}

extern "C" int kfac_grad_update(const kfac_grad_item* items, int count, const float* scale, void* ws,
                                size_t ws_bytes, void* stream) {
  KFAC_CHECK_ARG(count >= 0 && (items || count == 0), "grad_update args");
  if (count == 0) return KFAC_OK;
  cudaStream_t s = (cudaStream_t)stream;
  long long total = 0;
  { const int rc = upload_grad_items(items, count, ws, ws_bytes, s, &total); if (rc) return rc; }
  update_all_kernel<<<grid_for(total), 256, 0, s>>>((const GradDev*)ws, count, total, scale);
  KFAC_LAUNCH_CHECK();
  return KFAC_OK;
}

// ------------------------------------------------------------ peer memory (CUDA IPC)
extern "C" int kfac_peer_alloc(size_t bytes, void** dev_ptr, void* handle64) {
  KFAC_CHECK_ARG(bytes > 0 && dev_ptr && handle64, "peer_alloc args");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t size");
  void* p = nullptr;
  KFAC_CUDA(cudaMalloc(&p, bytes));
  cudaIpcMemHandle_t h;
  cudaError_t e = cudaIpcGetMemHandle(&h, p);
  if (e != cudaSuccess) { cudaFree(p); set_error("cudaIpcGetMemHandle: %s", cudaGetErrorString(e)); return KFAC_ERR_CUDA; }
  KFAC_CUDA(cudaMemset(p, 0, bytes));
  memcpy(handle64, &h, 64);
  *dev_ptr = p;
  return KFAC_OK;
}
extern "C" int kfac_peer_open(const void* handle64, void** dev_ptr) {
  KFAC_CHECK_ARG(handle64 && dev_ptr, "peer_open args");
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, 64);
  void* p = nullptr;
  KFAC_CUDA(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
  *dev_ptr = p;
  return KFAC_OK;
}
extern "C" int kfac_peer_close(void* dev_ptr) {
  if (dev_ptr) KFAC_CUDA(cudaIpcCloseMemHandle(dev_ptr));
  return KFAC_OK;
}
extern "C" int kfac_peer_free(void* dev_ptr) {
  if (dev_ptr) KFAC_CUDA(cudaFree(dev_ptr));
  return KFAC_OK;
}
