// Tied embedding / LM-head pairs: simultaneous diagonalisation of the two d x d factors E and H
// (kfac_tied_whiten, kfac_tied_basis in kfac_b200.h).  With E = Q diag(e) Q^T and s = (e + damping)^-1/2,
//   whiten:  C = diag(s) (Q^T H Q + damping I) diag(s)        (exactly symmetric: the input of the eigensolver)
//   basis:   M = Q diag(s) U,  MT = M^T                        (U: the eigenvectors of C)
// The products run on the grouped engine; a product with K > 1024 is split into chains of <= 512 whose partial
// tiles are added in a fixed order, as in the precondition.
#include <algorithm>
#include <vector>

#include "common.cuh"
#include "gemm_grouped.cuh"

namespace kfac {
namespace {

// per-item device view of the elementwise kernels
struct TiedDev { const float* src; const float* e; float* dst; int d, ld; };

// out (d x ld) = H (d x d, ld = d) with zero padding columns: a TMA-addressable copy of H
__global__ void pad_kernel(const TiedDev* items) {
  const TiedDev t = items[blockIdx.y];
  const int64_t total = (int64_t)t.d * t.ld;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int i = (int)(idx / t.ld), j = (int)(idx % t.ld);
    t.dst[idx] = j < t.d ? t.src[(int64_t)i * t.d + j] : 0.f;
  }
}

__device__ __forceinline__ float inv_sqrt_shift(float e, float damping) {
  return (float)(1.0 / sqrt((double)e + (double)damping));
}

// C[i][j] = ((X[i][j] + X[j][i]) / 2 + damping [i == j]) * (s_i s_j), ld(C) = d.  Every factor of the product is
// symmetric in (i, j), so C[i][j] and C[j][i] get the same bits
__global__ void whiten_kernel(const TiedDev* items, float damping) {
  const TiedDev t = items[blockIdx.y];
  const int64_t total = (int64_t)t.d * t.d;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int i = (int)(idx / t.d), j = (int)(idx % t.d);
    float x = 0.5f * (t.src[(int64_t)i * t.ld + j] + t.src[(int64_t)j * t.ld + i]);
    if (i == j) x += damping;
    t.dst[idx] = x * (inv_sqrt_shift(t.e[i], damping) * inv_sqrt_shift(t.e[j], damping));
  }
}

// dst[j][k] = UT[j][k] * s_k (d x ld, padding columns zero): the operand that folds diag(s) into M = Q (UT diag(s))^T
__global__ void scale_cols_tied_kernel(const TiedDev* items, float damping) {
  const TiedDev t = items[blockIdx.y];
  const int64_t total = (int64_t)t.d * t.ld;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int k = (int)(idx % t.ld);
    t.dst[idx] = k < t.d ? t.src[idx] * inv_sqrt_shift(t.e[k], damping) : 0.f;
  }
}

__global__ void transpose_tied_kernel(const TiedDev* items) {
  const TiedDev t = items[blockIdx.z];
  __shared__ float tile[32][33];
  const int bx = blockIdx.x * 32, by = blockIdx.y * 32;
  if (bx >= t.d || by >= t.d) return;
  for (int r = threadIdx.y; r < 32; r += 8) {
    const int i = by + r, j = bx + threadIdx.x;
    tile[r][threadIdx.x] = (i < t.d && j < t.d) ? t.src[(int64_t)i * t.ld + j] : 0.f;
  }
  __syncthreads();
  for (int r = threadIdx.y; r < 32; r += 8) {
    const int j = bx + r, i = by + threadIdx.x;
    if (j < t.d && i < t.d) t.dst[(int64_t)j * t.ld + i] = tile[threadIdx.x][r];
  }
}

// workspace: [grouped-GEMM tables][TiedDev table][per item: X (d x ld), Y (d x ld), slab (splits x d x ld)]
struct TiedLayout {
  size_t off_gemm, off_dev, total;
  std::vector<size_t> x, y, slab;
};

void tied_layout(const kfac_tied_item* items, int count, TiedLayout& L) {
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off = align_up(off + bytes, 256); return o; };
  L.off_gemm = take(grouped_gemm_ws_bytes(count));
  L.off_dev = take(sizeof(TiedDev) * (size_t)std::max(1, count));
  L.x.resize(count); L.y.resize(count); L.slab.assign(count, 0);
  for (int i = 0; i < count; ++i) {
    const size_t mat = (size_t)items[i].d * items[i].ld * sizeof(float);
    L.x[i] = take(mat);
    L.y[i] = take(mat);
    if (chain_splits(items[i].d) > 1) L.slab[i] = take(chain_splits(items[i].d) * mat);
  }
  L.total = off;
}

GroupedGemm product(const float* A, const float* B, float* D, int d, int ld, float* slab) {
  GroupedGemm g{};
  g.A = A; g.lda = ld; g.B = B; g.ldb = ld; g.D = D; g.ldd = ld; g.M = d; g.N = d; g.K = d; g.alpha = 1.f;
  g.epi = EPI_NONE; g.splits = 1;
  if (chain_splits(d) > 1) { g.splits = chain_splits(d); g.slab = slab; g.slab_stride = (int64_t)d * ld; }
  return g;
}

int grid_x(int max_d, int max_ld) {
  return std::max(1, std::min(ceil_div((int64_t)max_d * max_ld, 256), tc_num_sms() * 2));
}

int check_items(const kfac_tied_item* items, int count, void* ws, size_t ws_bytes, TiedLayout& L, bool whiten) {
  KFAC_CHECK_ARG(count >= 0 && (items || count == 0), "tied items");
  for (int i = 0; i < count; ++i) {
    const kfac_tied_item& t = items[i];
    KFAC_CHECK_ARG(t.d > 0 && t.d <= KFAC_EIGH_MAX_N && t.ld >= t.d && (t.ld & 3) == 0 && t.Q && t.QT && t.e,
                   "tied item");
    if (whiten) KFAC_CHECK_ARG(t.H && t.C, "tied whiten item");
    else KFAC_CHECK_ARG(t.UT && t.M && t.MT, "tied basis item");
  }
  tied_layout(items, count, L);
  if (!ws || ws_bytes < L.total) {
    set_error("tied: workspace too small (%zu < %zu)", ws_bytes, L.total);
    return KFAC_ERR_WORKSPACE;
  }
  return KFAC_OK;
}

}  // namespace
}  // namespace kfac

using namespace kfac;

extern "C" size_t kfac_tied_workspace_bytes(const kfac_tied_item* items, int count) {
  if (count <= 0 || !items) return 0;
  TiedLayout L;
  tied_layout(items, count, L);
  return L.total;
}

extern "C" int kfac_tied_whiten(const kfac_tied_item* items, int count, float damping, void* ws, size_t ws_bytes,
                                void* stream) {
  KFAC_CHECK_ARG(damping > 0.f, "tied damping");
  TiedLayout L;
  int rc = check_items(items, count, ws, ws_bytes, L, true);
  if (rc || count == 0) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  char* base = (char*)ws;
  auto F = [&](size_t off) { return (float*)(base + off); };
  TiedDev* dev = (TiedDev*)(base + L.off_dev);
  std::vector<TiedDev> tab(count);
  std::vector<GroupedGemm> st(count);
  int max_d = 1, max_ld = 1;
  for (int i = 0; i < count; ++i) {
    max_d = std::max(max_d, items[i].d); max_ld = std::max(max_ld, items[i].ld);
  }
  const dim3 grid(grid_x(max_d, max_ld), count);
  // X = H with a padded leading dimension
  for (int i = 0; i < count; ++i) tab[i] = TiedDev{items[i].H, nullptr, F(L.x[i]), items[i].d, items[i].ld};
  KFAC_CUDA(cudaMemcpyAsync(dev, tab.data(), sizeof(TiedDev) * count, cudaMemcpyHostToDevice, s));
  pad_kernel<<<grid, 256, 0, s>>>(dev);
  KFAC_LAUNCH_CHECK();
  // Y[i][j] = sum_k QT[i][k] H[j][k] = (Q^T H)[i][j]   (H symmetric)
  for (int i = 0; i < count; ++i)
    st[i] = product(items[i].QT, F(L.x[i]), F(L.y[i]), items[i].d, items[i].ld, L.slab[i] ? F(L.slab[i]) : nullptr);
  if ((rc = launch_grouped_gemm(st.data(), count, base + L.off_gemm, grouped_gemm_ws_bytes(count), s))) return rc;
  // X[i][j] = sum_k Y[i][k] QT[j][k] = (Q^T H Q)[i][j]
  for (int i = 0; i < count; ++i)
    st[i] = product(F(L.y[i]), items[i].QT, F(L.x[i]), items[i].d, items[i].ld, L.slab[i] ? F(L.slab[i]) : nullptr);
  if ((rc = launch_grouped_gemm(st.data(), count, base + L.off_gemm, grouped_gemm_ws_bytes(count), s))) return rc;
  // the table is rewritten in stream order, after pad_kernel has read it
  for (int i = 0; i < count; ++i) tab[i] = TiedDev{F(L.x[i]), items[i].e, items[i].C, items[i].d, items[i].ld};
  KFAC_CUDA(cudaMemcpyAsync(dev, tab.data(), sizeof(TiedDev) * count, cudaMemcpyHostToDevice, s));
  whiten_kernel<<<grid, 256, 0, s>>>(dev, damping);
  KFAC_LAUNCH_CHECK();
  return KFAC_OK;
}

extern "C" int kfac_tied_basis(const kfac_tied_item* items, int count, float damping, void* ws, size_t ws_bytes,
                               void* stream) {
  KFAC_CHECK_ARG(damping > 0.f, "tied damping");
  TiedLayout L;
  int rc = check_items(items, count, ws, ws_bytes, L, false);
  if (rc || count == 0) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  char* base = (char*)ws;
  auto F = [&](size_t off) { return (float*)(base + off); };
  TiedDev* dev = (TiedDev*)(base + L.off_dev);
  std::vector<TiedDev> tab(count);
  std::vector<GroupedGemm> st(count);
  int max_d = 1, max_ld = 1;
  for (int i = 0; i < count; ++i) {
    max_d = std::max(max_d, items[i].d); max_ld = std::max(max_ld, items[i].ld);
  }
  // X = UT diag(s)
  for (int i = 0; i < count; ++i) tab[i] = TiedDev{items[i].UT, items[i].e, F(L.x[i]), items[i].d, items[i].ld};
  KFAC_CUDA(cudaMemcpyAsync(dev, tab.data(), sizeof(TiedDev) * count, cudaMemcpyHostToDevice, s));
  scale_cols_tied_kernel<<<dim3(grid_x(max_d, max_ld), count), 256, 0, s>>>(dev, damping);
  KFAC_LAUNCH_CHECK();
  // M[i][j] = sum_k Q[i][k] X[j][k] = (Q diag(s) U)[i][j]
  for (int i = 0; i < count; ++i)
    st[i] = product(items[i].Q, F(L.x[i]), items[i].M, items[i].d, items[i].ld, L.slab[i] ? F(L.slab[i]) : nullptr);
  if ((rc = launch_grouped_gemm(st.data(), count, base + L.off_gemm, grouped_gemm_ws_bytes(count), s))) return rc;
  // MT = M^T, the same transposition kfac_transpose applies on a rank that receives M
  for (int i = 0; i < count; ++i) tab[i] = TiedDev{items[i].M, nullptr, items[i].MT, items[i].d, items[i].ld};
  KFAC_CUDA(cudaMemcpyAsync(dev, tab.data(), sizeof(TiedDev) * count, cudaMemcpyHostToDevice, s));
  const int tiles = ceil_div(max_d, 32);
  transpose_tied_kernel<<<dim3(tiles, tiles, count), dim3(32, 8), 0, s>>>(dev);
  KFAC_LAUNCH_CHECK();
  return KFAC_OK;
}
