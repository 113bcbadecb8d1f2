// K7-K12: damped inverse from the eigendecomposition, two-sided Kronecker
// precondition, kl-clip scale and in-place gradient write-back.
#include <string.h>

#include <algorithm>
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

// all layers in one launch: item i owns the elements [elem0, elem0 + g * ldo) of the concatenated space
struct GatherDev { const void* w; const void* b; int dtype, g, a, ldo; float* out; long long elem0; };
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
    if (j < aw) v = load_as_float(it.w, it.dtype, i * aw + j);
    else if (j < it.a) v = load_as_float(it.b, it.dtype, i);
    it.out[idx] = v;
  }
}

// ---- kl-clip scale and write-back: ONE launch each over all layers, deterministic ---------------
// device copy of a kfac_grad_item + the offset of its g*a elements in the concatenated element space
struct GradDev { const float* P; void* w; void* b; int dtype, g, a, ldp; long long elem0; };
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
    const float gr = (j < aw) ? load_as_float(it.w, it.dtype, i * aw + j) : load_as_float(it.b, it.dtype, i);
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
    if (j < aw) store_from_float(it.w, it.dtype, i * aw + j, v);
    else store_from_float(it.b, it.dtype, i, v);
  }
}

// out[i][j] = Q[i][j] / (d[j] + damping), zero in the padding columns
__global__ void scale_cols_kernel(const float* Q, int ldq, const float* d, int n, float damping, float* out) {
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
// row-major (rows x ld) copy of D into the peers' buffers (layers that did not go through
// the tensor-core epilogue)
__global__ void peer_scatter_kernel(const float* D, int64_t total, float* p0, float* p1, float* p2, float* p3,
                                    float* p4, float* p5, float* p6, int npeer) {
  float* peers[7] = {p0, p1, p2, p3, p4, p5, p6};
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const float v = D[idx];
    for (int q = 0; q < npeer; ++q) peers[q][idx] = v;
  }
}

// D[m][n] = sum_sp slab[sp][m][n] (fixed order) -- second half of the deterministic split-K
__global__ void reduce_slabs_kernel(const float* slab, int64_t slab_stride, int splits, float* D, int64_t total) {
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    float t = slab[idx];
    for (int sp = 1; sp < splits; ++sp) t += slab[(int64_t)sp * slab_stride + idx];
    D[idx] = t;
  }
}

// slab / slab_floats: optional workspace for a DETERMINISTIC split-K (partial tiles stored per split, then summed
// in a fixed order); without it long reductions use atomic accumulation (order not reproducible).
int gemm_tn(const float* A, int64_t lda, const float* B, int64_t ldb, float* D, int64_t ldd, int M, int N,
            int K, const Epi& e, cudaStream_t s, float* const* peers = nullptr, int npeer = 0, float* slab = nullptr,
            size_t slab_floats = 0) {
  TcGemmArgs t{};
  t.npeer = 0;
  t.A = A; t.lda = lda; t.B = B; t.ldb = ldb; t.D = D; t.ldd = ldd; t.M = M; t.N = N; t.K = K;
  t.kbatch = 1; t.alpha = 1.f; t.splits = 1;
  t.epi = e.kind; t.E = e.E; t.lde = e.lde; t.dg = e.dg; t.da = e.da; t.damping = e.damping;
  if (M >= 64 && N >= 64 && K >= 32 && tc_gemm_supported(t)) {
    if (npeer > 0) {   // fused broadcast: plain-store epilogue, no split-K
      t.npeer = npeer;
      for (int q = 0; q < npeer; ++q) t.peerD[q] = peers[q];
      return launch_tc_gemm(t, s);
    }
    if (e.kind == EPI_NONE && K > 1024) {
      // long reductions are split across CTAs: the tensor-core accumulator truncates, so short chains
      // keep the 3xTF32 result at fp32 accuracy, and small tile counts fill the SMs.
      const int splits = ceil_div(K, 512);
      const int64_t stride = (int64_t)M * ldd;
      if (slab && slab_floats >= (size_t)splits * stride) {
        // deterministic: every split stores its partial tile, a second pass adds them in a fixed order
        t.slab = slab; t.slab_stride = stride; t.splits = splits;
        const int rc = launch_tc_gemm(t, s);
        if (rc) return rc;
        reduce_slabs_kernel<<<grid_for(stride), 256, 0, s>>>(slab, stride, splits, D, stride);
        KFAC_LAUNCH_CHECK();
        return KFAC_OK;
      }
      // no workspace: partial tiles are added with (round-to-nearest) L2 atomics
      KFAC_CUDA(cudaMemset2DAsync(D, (size_t)ldd * 4, 0, (size_t)N * 4, (size_t)M, s));
      t.atomic = 1;
      t.splits = splits;
    }
    return launch_tc_gemm(t, s);
  }
  GemmArgs g{};
  g.A = A; g.sa_m = lda; g.sa_k = 1; g.B = B; g.sb_k = 1; g.sb_n = ldb;
  g.C = D; g.ldc = ldd; g.M = M; g.N = N; g.K = K; g.batch = 1; g.splitk = 1;
  g.alpha = 1.f; g.beta = 0.f;
  g.epi = e.kind; g.E = e.E; g.lde = e.lde; g.dg = e.dg; g.da = e.da; g.damping = e.damping;
  const int rc = launch_gemm(g, s);
  if (rc || npeer == 0) return rc;
  float* pp[7] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  for (int q = 0; q < npeer; ++q) pp[q] = peers[q];
  const int64_t total = (int64_t)M * ldd;
  peer_scatter_kernel<<<grid_for(total), 256, 0, s>>>(D, total, pp[0], pp[1], pp[2], pp[3], pp[4], pp[5], pp[6], npeer);
  KFAC_LAUNCH_CHECK();
  return KFAC_OK;
}

int gemm_tn_plain(const float* A, int64_t lda, const float* B, int64_t ldb, float* D, int64_t ldd, int M, int N,
                  int K, cudaStream_t s) {
  return gemm_tn(A, lda, B, ldb, D, ldd, M, N, K, Epi{}, s);
}

}  // namespace kfac

using namespace kfac;

static inline int ld4(int x) { return (x + 3) & ~3; }

extern "C" int kfac_inverse_from_eigh(const float* Q, int ldq, const float* d, int n, float damping,
                                      float* inv, int ld_inv, void* ws, size_t ws_bytes, void* stream) {
  KFAC_CHECK_ARG(Q && d && inv && n > 0 && ldq >= n && ld_inv >= n, "inverse args");
  const size_t need = (size_t)n * ldq * sizeof(float);
  if (!ws || ws_bytes < need) {
    set_error("inverse_from_eigh: workspace too small (%zu < %zu)", ws_bytes, need);
    return KFAC_ERR_WORKSPACE;
  }
  cudaStream_t s = (cudaStream_t)stream;
  float* T = (float*)ws;
  scale_cols_kernel<<<grid_for((int64_t)n * ldq), 256, 0, s>>>(Q, ldq, d, n, damping, T);
  KFAC_LAUNCH_CHECK();
  // inv[i][j] = sum_k T[i][k] Q[j][k]
  return gemm_tn(T, ldq, Q, ldq, inv, ld_inv, n, n, n, Epi{}, s);
}

extern "C" int kfac_transpose(const float* src, int ld_src, float* dst, int ld_dst, int rows, int cols,
                              void* stream) {
  KFAC_CHECK_ARG(src && dst && rows > 0 && cols > 0 && ld_src >= cols && ld_dst >= rows, "transpose args");
  dim3 grid(ceil_div(cols, 32), ceil_div(rows, 32));
  transpose_kernel<<<grid, dim3(32, 8), 0, (cudaStream_t)stream>>>(src, ld_src, dst, ld_dst, rows, cols);
  KFAC_LAUNCH_CHECK();
  return KFAC_OK;
}

// ---- precondition: stage-wise over ALL layers ------------------------------------------------------
// workspace: [GatherDev table][grouped-GEMM tables][per layer: GR (g x ld4 a), T1 (a x ld4 g), T2 (g x ld4 a)][slabs]
struct PrecondLayout {
  size_t off_gather, off_gemm, off_tiles, off_slab, total;
  std::vector<size_t> gr, t1, t2, slab_a, slab_g;     // byte offsets per layer (slab_*: 0 = no split)
  std::vector<int> splits_a, splits_g;
};

static void precond_layout(const kfac_precond_item* items, int count, PrecondLayout& L) {
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off = align_up(off + bytes, 256); return o; };
  L.off_gather = take(sizeof(GatherDev) * (size_t)std::max(1, count));
  L.off_gemm = take(grouped_gemm_ws_bytes(count));
  L.off_tiles = off;
  L.gr.resize(count); L.t1.resize(count); L.t2.resize(count);
  L.slab_a.assign(count, 0); L.slab_g.assign(count, 0); L.splits_a.assign(count, 1); L.splits_g.assign(count, 1);
  for (int i = 0; i < count; ++i) {
    const size_t a = items[i].a, g = items[i].g;
    L.gr[i] = take(g * ld4((int)a) * sizeof(float));
    L.t1[i] = take(a * ld4((int)g) * sizeof(float));
    L.t2[i] = take(g * ld4((int)a) * sizeof(float));
  }
  L.off_slab = off;
  // long reductions (K > 1024) are split into chains of <= 512: the tensor-core accumulator truncates, short
  // chains keep the 3xTF32 result at fp32 accuracy; the partial tiles go to slabs and are added in a fixed order
  // (deterministic: every replica that preconditions a layer locally must get the same bits)
  for (int i = 0; i < count; ++i) {
    const size_t a = items[i].a, g = items[i].g;
    if (a > 1024) { L.splits_a[i] = ceil_div(a, 512); L.slab_a[i] = take((size_t)L.splits_a[i] * a * ld4((int)g) * sizeof(float)); }
    if (g > 1024 && items[i].n_peers == 0) {
      L.splits_g[i] = ceil_div(g, 512); L.slab_g[i] = take((size_t)L.splits_g[i] * g * ld4((int)a) * sizeof(float));
    }
  }
  L.total = off;
}

extern "C" size_t kfac_precondition_workspace_bytes(const kfac_precond_item* items, int count) {
  if (count <= 0) return 0;
  PrecondLayout L;
  precond_layout(items, count, L);
  return L.total;
}

extern "C" int kfac_precondition(const kfac_precond_item* items, int count, int method, float damping,
                                 void* ws, size_t ws_bytes, void* stream) {
  KFAC_CHECK_ARG(count >= 0 && (items || count == 0), "items");
  KFAC_CHECK_ARG(method == KFAC_EIGEN || method == KFAC_INVERSE, "method");
  if (count == 0) return KFAC_OK;
  PrecondLayout L;
  precond_layout(items, count, L);
  if (!ws || ws_bytes < L.total) {
    set_error("precondition: workspace too small (%zu < %zu)", ws_bytes, L.total);
    return KFAC_ERR_WORKSPACE;
  }
  cudaStream_t s = (cudaStream_t)stream;
  char* base = (char*)ws;
  auto F = [&](size_t off) { return (float*)(base + off); };
  // stage 0: grad matrices [wgrad | bgrad] of all layers, one launch
  std::vector<GatherDev> gat(count);
  long long total = 0;
  for (int i = 0; i < count; ++i) {
    const kfac_precond_item& it = items[i];
    KFAC_CHECK_ARG(it.wgrad && it.P && it.g > 0 && it.a > 0 && it.ldp >= it.a, "precond item");
    KFAC_CHECK_ARG(it.n_peers >= 0 && it.n_peers <= 7 && (it.n_peers == 0 || it.peer_P), "precond peers");
    if (method == KFAC_EIGEN) {
      if (!(it.qa && it.qg && it.qaT && it.qgT && (it.dgda || (it.da && it.dg)))) {
        set_error("precondition: eigendecompositions for both A and G have not been computed");
        return KFAC_ERR_NOT_READY;
      }
    } else if (!(it.a_inv && it.g_inv)) {
      set_error("precondition: A and G have not been inverted");
      return KFAC_ERR_NOT_READY;
    }
    KFAC_CHECK_ARG(it.ldqa >= it.a && it.ldqg >= it.g, "second-order leading dims");
    gat[i] = GatherDev{it.wgrad, it.bgrad, it.grad_dtype, it.g, it.a, ld4(it.a), F(L.gr[i]), total};
    total += (long long)it.g * ld4(it.a);
  }
  KFAC_CUDA(cudaMemcpyAsync(base + L.off_gather, gat.data(), sizeof(GatherDev) * count, cudaMemcpyHostToDevice, s));
  gather_all_kernel<<<grid_for(total), 256, 0, s>>>((const GatherDev*)(base + L.off_gather), count, total);
  KFAC_LAUNCH_CHECK();

  std::vector<GroupedGemm> st(count);
  auto run = [&]() { return launch_grouped_gemm(st.data(), count, base + L.off_gemm, grouped_gemm_ws_bytes(count), s); };
  auto plain = [&](int i, const float* A, int64_t lda, const float* B, int64_t ldb, float* D, int64_t ldd, int M, int N, int K) {
    GroupedGemm g{};
    g.A = A; g.lda = lda; g.B = B; g.ldb = ldb; g.D = D; g.ldd = ldd; g.M = M; g.N = N; g.K = K; g.alpha = 1.f;
    g.epi = EPI_NONE; g.splits = 1;
    st[i] = g;
  };
  int rc;
  // the four (two) GEMMs of every layer form a chain; stage k of all layers is one grouped launch
  for (int i = 0; i < count; ++i) {     // (1) T^T[a', r] = sum_k (QaT | Ainv)[a', k] grad[r, k]          (a x g, K = a)
    const kfac_precond_item& it = items[i];
    const int g = it.g, a = it.a;
    plain(i, method == KFAC_EIGEN ? it.qaT : it.a_inv, it.ldqa, F(L.gr[i]), ld4(a), F(L.t1[i]), ld4(g), a, g, a);
    if (L.splits_a[i] > 1) { st[i].splits = L.splits_a[i]; st[i].slab = F(L.slab_a[i]); st[i].slab_stride = (int64_t)a * ld4(g); }
  }
  if ((rc = run())) return rc;
  if (method == KFAC_EIGEN) {
    for (int i = 0; i < count; ++i) {   // (2) V2[g', a'] = (sum_k QgT[g', k] T^T[a', k]) * dgda[g', a']     (g x a, K = g)
      const kfac_precond_item& it = items[i];
      const int g = it.g, a = it.a;
      plain(i, it.qgT, it.ldqg, F(L.t1[i]), ld4(g), F(L.t2[i]), ld4(a), g, a, g);
      if (it.dgda) { st[i].epi = EPI_MUL; st[i].E = it.dgda; st[i].lde = it.ld_dgda; }
      else { st[i].epi = EPI_DIV_OUTER; st[i].dg = it.dg; st[i].da = it.da; st[i].damping = damping; }
    }
    if ((rc = run())) return rc;
    for (int i = 0; i < count; ++i) {   // (3) U^T[c, g'] = sum_k Qa[c, k] V2[g', k]                         (a x g, K = a)
      const kfac_precond_item& it = items[i];
      const int g = it.g, a = it.a;
      plain(i, it.qa, it.ldqa, F(L.t2[i]), ld4(a), F(L.t1[i]), ld4(g), a, g, a);
      if (L.splits_a[i] > 1) { st[i].splits = L.splits_a[i]; st[i].slab = F(L.slab_a[i]); st[i].slab_stride = (int64_t)a * ld4(g); }
    }
    if ((rc = run())) return rc;
  }
  for (int i = 0; i < count; ++i) {     // (4) P[r, c] = sum_k (Qg | Ginv)[r, k] U^T[c, k]                  (g x a, K = g)
    const kfac_precond_item& it = items[i];
    const int g = it.g, a = it.a;
    plain(i, method == KFAC_EIGEN ? it.qg : it.g_inv, it.ldqg, F(L.t1[i]), ld4(g), it.P, it.ldp, g, a, g);
    if (it.n_peers > 0) {               // fused compute + broadcast: no split (the tiles are final when stored)
      st[i].npeer = it.n_peers;
      for (int q = 0; q < it.n_peers; ++q) st[i].peerD[q] = it.peer_P[q];
    } else if (L.splits_g[i] > 1 && it.ldp == ld4(a)) {
      st[i].splits = L.splits_g[i]; st[i].slab = F(L.slab_g[i]); st[i].slab_stride = (int64_t)g * ld4(a);
    }
  }
  return run();
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
    dev[i] = GradDev{it.P, it.wgrad, it.bgrad, it.grad_dtype, it.g, it.a, it.ldp, total};
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
