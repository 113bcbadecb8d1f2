// Grouped wgmma GEMM: ONE launch runs a whole list of independent problems
//     D_i = epilogue_i(alpha_i * A_i B_i^T)        (A_i: M x K, B_i: N x K, row-major fp32, 3xTF32 split)
// through the persistent pipeline of tc_pipeline.cuh.  Work items are (problem, 128 x 128 tile, K split);
// the per-problem TMA descriptors live in a device table (the kernel walks it by binary search), so the
// precondition stage of ALL layers is one launch instead of one launch per layer
// (kfac/layers/eigen.py:371-385 executes 4 GEMMs per layer).  Long reductions are split
// deterministically: every split stores its partial tile into its own slab, grouped_reduce_kernel adds
// the slabs in a fixed order.
#include "common.cuh"
#include "gemm_grouped.cuh"
#include "tc_pipeline.cuh"

#include <algorithm>
#include <vector>

namespace kfac {

namespace {

constexpr int GBM = 128, GBN = 128, GBK = 32;

struct alignas(128) GProb {
  CUtensorMap tmA, tmB;
  float* D; int64_t ldd;
  int M, N, K;
  int tiles_n, splits, kb_per_split, kb_total;
  int work0;                       // first work item of this problem
  float alpha;
  int epi; const float* E; int64_t lde; const float* dg; const float* da; float damping;
  const float* pi; int pi_side_m, pi_side_n;
  int64_t slab_stride;             // != 0: D is the slab base, split sp stores to D + sp * slab_stride
  int mode;                        // 0 store, 1 read-modify-write accumulate, 2 atomicAdd
  const int* krange;               // device-side {first, end} k-block of the reduction (mode 2), or null
  float* peerD[7]; int npeer;
};

struct GroupedParams { const GProb* probs; int nprobs; };

// FACTORED: the instantiation that also takes EPI_DIV_FACTORED, launched only for a list with such a problem, so that
// the epilogue of every other launch stays as compact as it was
template <bool FACTORED>
struct GroupedPolicy {
  using Params = GroupedParams;
  struct Item { const GProb* pr; int m0, n0, kb0, kb1, sp, idx; };
  static constexpr uint32_t TX_BYTES = 2 * tc::PTILE;
  static constexpr int CHUNK = 1;
  __device__ static void reset(Item& it) { it.idx = 0; it.pr = nullptr; }
  __device__ static int total_work(const Params&, int t) { return t; }

  __device__ static bool decode(const Params& p, int w, Item& it) {
    // work indices only grow for a given CTA: continue the search from the cached problem
    int lo = it.idx, hi = p.nprobs - 1;
    while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (p.probs[mid].work0 <= w) lo = mid; else hi = mid - 1; }
    it.idx = lo;
    const GProb* pr = &p.probs[lo];
    it.pr = pr;
    const int local = w - pr->work0;
    const int tile = local / pr->splits, sp = local % pr->splits;
    it.m0 = (tile / pr->tiles_n) * GBM;
    it.n0 = (tile % pr->tiles_n) * GBN;
    it.sp = sp;
    int kb_lo = 0, kb_hi = pr->kb_total;
    if (pr->krange) { kb_lo = max(0, pr->krange[0]); kb_hi = min(kb_hi, pr->krange[1]); }
    it.kb0 = kb_lo + sp * pr->kb_per_split;
    it.kb1 = min(kb_hi, it.kb0 + pr->kb_per_split);
    return it.kb1 > it.kb0;
  }
  __device__ static int num_kb(const Params&, const Item& it) { return it.kb1 - it.kb0; }
  __device__ static void load(const Params&, const Item& it, int kbi, uint8_t* a, uint8_t* b, uint64_t* bar) {
    const int kc = (it.kb0 + kbi) * GBK;
    tc::tma_load_3d(a, &it.pr->tmA, bar, kc, it.m0, 0);
    tc::tma_load_3d(b, &it.pr->tmB, bar, kc, it.n0, 0);
  }
  // The problem table is in global memory: read once per item, not after each of the 64 stores of a thread (which
  // the compiler must assume may alias it).
  struct Out {
    float* D; int64_t ldd; int M, N, m0, n0;
    float alpha; int epi; const float* E; int64_t lde; const float* dg; const float* da; float damping;
    const float* pi; int pi_side_m, pi_side_n;
    int mode, npeer; const GProb* pr;
  };
  __device__ static Out out(const Params&, const Item& it) {
    const GProb& p = *it.pr;
    Out o;
    o.D = p.D + (int64_t)it.sp * p.slab_stride; o.ldd = p.ldd; o.M = p.M; o.N = p.N; o.m0 = it.m0; o.n0 = it.n0;
    o.alpha = p.alpha; o.epi = p.epi; o.E = p.E; o.lde = p.lde; o.dg = p.dg; o.da = p.da; o.damping = p.damping;
    o.pi = p.pi; o.pi_side_m = p.pi_side_m; o.pi_side_n = p.pi_side_n;
    o.mode = p.mode; o.npeer = p.npeer; o.pr = it.pr;
    return o;
  }
  __device__ static void store(const Params&, const Out& p, int row, int col, float (&v)[2]) {
    const int m = p.m0 + row, nb = p.n0 + col;
    if (m >= p.M || nb >= p.N) return;
    float* drow = p.D + (int64_t)m * p.ldd + nb;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      float x = p.alpha * v[j];
      if (nb + j < p.N) {
        if (p.epi == EPI_MUL) x *= p.E[(int64_t)m * p.lde + nb + j];
        else if (p.epi == EPI_DIV_OUTER) x = x / (p.dg[m] * p.da[nb + j] + p.damping);
        else if (p.epi == EPI_SQUARE) x = x * x;
        else if (FACTORED && p.epi == EPI_DIV_FACTORED)
          x = div_factored(x, p.dg[m], p.da[nb + j], p.damping, p.pi, p.pi_side_m, p.pi_side_n);
      }
      v[j] = x;
    }
    if (p.mode == 2) {
#pragma unroll
      for (int j = 0; j < 2; ++j)
        if (nb + j < p.N) atomicAdd(drow + j, v[j]);
      return;
    }
    if (((uintptr_t)drow & 7) == 0 && (p.ldd & 1) == 0 && nb + 2 <= p.N) {
      if (p.mode == 1) {
        const float2 o = *reinterpret_cast<const float2*>(drow);
        v[0] += o.x; v[1] += o.y;
      }
      *reinterpret_cast<float2*>(drow) = make_float2(v[0], v[1]);
      // fused compute + broadcast: the same tile goes straight to the peers' copies of D (P2P over NVLink)
      for (int q = 0; q < p.npeer; ++q)
        *reinterpret_cast<float2*>(p.pr->peerD[q] + (int64_t)m * p.ldd + nb) = make_float2(v[0], v[1]);
    } else {
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        if (nb + j >= p.N) continue;
        drow[j] = (p.mode == 1) ? drow[j] + v[j] : v[j];
        for (int q = 0; q < p.npeer; ++q) p.pr->peerD[q][(int64_t)m * p.ldd + nb + j] = v[j];
      }
    }
  }
};

// D[idx] = sum_sp slab[sp * stride + idx] over a list of split problems, one launch, fixed order.  The peers of a
// split problem (peers[i] for probs[i]) get the final sums here, its tiles being partials: every column of D,
// including the zero padding.  A launch without peers (PEERS = false) does not read the peer table.
struct RProb { const float* slab; float* D; int64_t stride; int splits; int N; int ldd; long long elem0; };
struct RPeers { float* peerD[7]; int npeer; };
template <bool PEERS>
__global__ void __launch_bounds__(256) grouped_reduce_kernel(const RProb* probs, const RPeers* peers, int count,
                                                             long long total) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    int lo = 0, hi = count - 1;
    while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (probs[mid].elem0 <= e) lo = mid; else hi = mid - 1; }
    const RProb& p = probs[lo];
    const long long idx = e - p.elem0;
    float t = 0.f;                       // padding columns (ld > N) stay zero: they feed the K dimension of the next GEMM
    if ((int)(idx % p.ldd) < p.N) {
      t = p.slab[idx];
      for (int sp = 1; sp < p.splits; ++sp) t += p.slab[(int64_t)sp * p.stride + idx];
    }
    p.D[idx] = t;
    if (PEERS) {
      const RPeers& r = peers[lo];
      for (int q = 0; q < r.npeer; ++q) r.peerD[q][idx] = t;
    }
  }
}

}  // namespace

int make_tmap_3d(CUtensorMap* tm, const float* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t stride1_bytes,
                 uint64_t stride2_bytes, uint32_t box_rows);

bool grouped_gemm_tc_ok(const GroupedGemm& g) {
  auto al16 = [](const void* p) { return ((uintptr_t)p & 15) == 0; };
  return g.M >= 64 && g.N >= 64 && g.K >= 32 && al16(g.A) && al16(g.B) && (g.lda & 3) == 0 && (g.ldb & 3) == 0;
}

size_t grouped_gemm_ws_bytes(int count) {
  const size_t n = (size_t)std::max(1, count);
  return align_up(sizeof(GProb) * n, 256) + align_up(sizeof(RProb) * n, 256) + align_up(sizeof(RPeers) * n, 256);
}

int launch_grouped_gemm(const GroupedGemm* probs, int count, void* ws, size_t ws_bytes, cudaStream_t s, int max_ctas,
                        HostStage* stage) {
  if (count <= 0) return KFAC_OK;
  if (!ws || ws_bytes < grouped_gemm_ws_bytes(count)) {
    set_error("grouped gemm: workspace too small (%zu < %zu)", ws_bytes, grouped_gemm_ws_bytes(count));
    return KFAC_ERR_WORKSPACE;
  }
  static bool attr = false;
  if (!attr) {
    KFAC_CUDA(cudaFuncSetAttribute(tc::pipeline_kernel<GroupedPolicy<false>>,
                                   cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tc::PSMEM));
    KFAC_CUDA(cudaFuncSetAttribute(tc::pipeline_kernel<GroupedPolicy<true>>,
                                   cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tc::PSMEM));
    attr = true;
  }
  // the arguments of every problem are checked (and every tensor map encoded) before anything is launched: a
  // rejected call leaves all outputs untouched
  std::vector<GProb> tab;
  std::vector<RProb> red;
  std::vector<RPeers> red_peers;
  bool any_peers = false;
  std::vector<int> simt;
  long long red_total = 0;
  int work = 0;
  for (int i = 0; i < count; ++i) {
    const GroupedGemm& g = probs[i];
    if (g.M <= 0 || g.N <= 0 || g.K <= 0) continue;
    const int splits = std::max(1, g.splits);
    if (g.npeer < 0 || g.npeer > 7) { set_error("grouped gemm: at most 7 peers"); return KFAC_ERR_BAD_ARG; }
    if (splits > 1 && ((!g.slab && g.mode != 2) || g.epi != EPI_NONE || g.mode == 1)) {
      set_error("grouped gemm: split-K needs a slab (or atomic mode) and the plain epilogue");
      return KFAC_ERR_BAD_ARG;
    }
    if (g.mode != 0 && (g.epi != EPI_NONE || g.npeer > 0)) { set_error("grouped gemm: accumulate modes need the plain epilogue"); return KFAC_ERR_BAD_ARG; }
    if (g.krange && (g.mode != 2 || !grouped_gemm_tc_ok(g))) {
      set_error("grouped gemm: a device-side k range needs the atomic mode on the tensor-core path");
      return KFAC_ERR_BAD_ARG;
    }
    if (!grouped_gemm_tc_ok(g)) { simt.push_back(i); continue; }
    GProb p{};
    int rc;
    if ((rc = make_tmap_3d(&p.tmA, g.A, (uint64_t)g.K, (uint64_t)g.M, 1, (uint64_t)g.lda * 4, (uint64_t)g.lda * 4 * g.M, GBM))) return rc;
    if ((rc = make_tmap_3d(&p.tmB, g.B, (uint64_t)g.K, (uint64_t)g.N, 1, (uint64_t)g.ldb * 4, (uint64_t)g.ldb * 4 * g.N, GBM))) return rc;
    p.M = g.M; p.N = g.N; p.K = g.K; p.ldd = g.ldd; p.alpha = g.alpha;
    p.epi = g.epi; p.E = g.E; p.lde = g.lde; p.dg = g.dg; p.da = g.da; p.damping = g.damping;
    p.pi = g.pi; p.pi_side_m = g.pi_side_m; p.pi_side_n = g.pi_side_n;
    p.tiles_n = ceil_div(g.N, GBN);
    const int tiles = ceil_div(g.M, GBM) * p.tiles_n;
    p.kb_total = ceil_div(g.K, GBK);
    p.kb_per_split = ceil_div(p.kb_total, splits);
    p.splits = ceil_div(p.kb_total, p.kb_per_split);
    p.mode = g.mode; p.krange = g.krange;
    if (p.splits > 1 && g.mode == 2) {
      p.D = g.D; p.slab_stride = 0;
    } else if (p.splits > 1) {
      // the tiles are partials: the peers get the final sums from the reduce pass, not from the epilogue
      p.D = g.slab; p.slab_stride = g.slab_stride;
      red.push_back(RProb{g.slab, g.D, g.slab_stride, p.splits, g.N, (int)g.ldd, red_total});
      RPeers r{{}, g.npeer};
      for (int q = 0; q < g.npeer; ++q) r.peerD[q] = g.peerD[q];
      red_peers.push_back(r);
      any_peers = any_peers || g.npeer > 0;
      red_total += (long long)g.M * g.ldd;
    } else {
      p.D = g.D; p.slab_stride = 0;
      p.npeer = g.npeer;
      for (int q = 0; q < g.npeer; ++q) p.peerD[q] = g.peerD[q];
    }
    p.work0 = work;
    work += tiles * p.splits;
    tab.push_back(p);
  }
  for (const int i : simt) {
    // small / unaligned problems: one SIMT launch each (fp32, no split needed)
    const GroupedGemm& g = probs[i];
    GemmArgs a{};
    a.A = g.A; a.sa_m = g.lda; a.sa_k = 1; a.B = g.B; a.sb_k = 1; a.sb_n = g.ldb;
    a.C = g.D; a.ldc = g.ldd; a.M = g.M; a.N = g.N; a.K = g.K; a.batch = 1; a.splitk = 1;
    a.alpha = g.alpha; a.beta = g.mode == 0 ? 0.f : 1.f; a.epi = g.epi; a.E = g.E; a.lde = g.lde; a.dg = g.dg; a.da = g.da; a.damping = g.damping;
    a.pi = g.pi; a.pi_side_m = g.pi_side_m; a.pi_side_n = g.pi_side_n;
    int rc = launch_gemm(a, s);
    if (rc) return rc;
    if (g.npeer > 0) {
      for (int q = 0; q < g.npeer; ++q)
        KFAC_CUDA(cudaMemcpy2DAsync(g.peerD[q], (size_t)g.ldd * 4, g.D, (size_t)g.ldd * 4, (size_t)g.N * 4, g.M,
                                    cudaMemcpyDeviceToDevice, s));
    }
  }
  if (tab.empty()) return KFAC_OK;
  GProb* d_tab = (GProb*)ws;
  RProb* d_red = (RProb*)((char*)ws + align_up(sizeof(GProb) * (size_t)std::max(1, count), 256));
  RPeers* d_red_peers = (RPeers*)((char*)d_red + align_up(sizeof(RProb) * (size_t)std::max(1, count), 256));
  int rc;
  if ((rc = send_table(stage, d_tab, tab.data(), sizeof(GProb) * tab.size(), s))) return rc;
  GroupedParams gp{d_tab, (int)tab.size()};
  const int sms = max_ctas > 0 ? std::min(max_ctas, tc_num_sms()) : tc_num_sms();
  const int grid = std::min(work, sms);
  const bool factored = std::any_of(tab.begin(), tab.end(), [](const GProb& p) { return p.epi == EPI_DIV_FACTORED; });
  if (factored) tc::pipeline_kernel<GroupedPolicy<true>><<<grid, tc::PTHREADS, tc::PSMEM, s>>>(gp, work);
  else tc::pipeline_kernel<GroupedPolicy<false>><<<grid, tc::PTHREADS, tc::PSMEM, s>>>(gp, work);
  KFAC_LAUNCH_CHECK();
  if (!red.empty()) {
    if ((rc = send_table(stage, d_red, red.data(), sizeof(RProb) * red.size(), s))) return rc;
    const int blocks = (int)std::min<long long>((red_total + 255) / 256, (long long)sms * 8);
    if (any_peers) {
      if ((rc = send_table(stage, d_red_peers, red_peers.data(), sizeof(RPeers) * red_peers.size(), s))) return rc;
      grouped_reduce_kernel<true><<<blocks, 256, 0, s>>>(d_red, d_red_peers, (int)red.size(), red_total);
    } else {
      grouped_reduce_kernel<false><<<blocks, 256, 0, s>>>(d_red, nullptr, (int)red.size(), red_total);
    }
    KFAC_LAUNCH_CHECK();
  }
  return KFAC_OK;
}

}  // namespace kfac

// test entry (not in the public header): the grouped engine on a list of problems, without peer stores.
// Mirrors GroupedGemm minus the peer fields.
struct kfac_stage_gemm {
  const float* A; int64_t lda;
  const float* B; int64_t ldb;
  float* D; int64_t ldd;
  int M, N, K;
  float alpha;
  int epi; const float* E; int64_t lde; const float* dg; const float* da; float damping;
  int splits; float* slab; int64_t slab_stride;
  int mode; const int* krange;
};

extern "C" size_t kfac_stage_grouped_gemm_ws_bytes(int count) { return kfac::grouped_gemm_ws_bytes(count); }

extern "C" int kfac_stage_grouped_gemm(const kfac_stage_gemm* probs, int count, void* ws, size_t ws_bytes,
                                       void* stream) {
  using namespace kfac;
  KFAC_CHECK_ARG(count >= 0 && (probs || count == 0), "grouped gemm test args");
  std::vector<GroupedGemm> g(count);
  for (int i = 0; i < count; ++i) {
    const kfac_stage_gemm& p = probs[i];
    GroupedGemm q{};
    q.A = p.A; q.lda = p.lda; q.B = p.B; q.ldb = p.ldb; q.D = p.D; q.ldd = p.ldd;
    q.M = p.M; q.N = p.N; q.K = p.K; q.alpha = p.alpha;
    q.epi = p.epi; q.E = p.E; q.lde = p.lde; q.dg = p.dg; q.da = p.da; q.damping = p.damping;
    q.splits = p.splits; q.slab = p.slab; q.slab_stride = p.slab_stride;
    q.mode = p.mode; q.krange = p.krange;
    g[i] = q;
  }
  return launch_grouped_gemm(g.data(), count, ws, ws_bytes, (cudaStream_t)stream);
}
