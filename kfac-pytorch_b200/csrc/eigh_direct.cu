// Direct symmetric eigensolver for the large K-FAC factors (replaces torch.linalg.eigh of
// kfac/layers/eigen.py:310,331 for n > 128):  F = H T H^T (sytrd.cu), T = Z L Z^T (stedc.cu),
// Q = H Z by compact-WY block reflectors of 128 Householder vectors (this file; wgmma GEMMs).
// Host side: workspace layout, the CTA-group schedule of the tridiagonalisation kernel, and the
// enqueue of all stages on ONE stream without host synchronisation.
#include "eigh_direct.cuh"

#include <math.h>

#include <algorithm>
#include <vector>

namespace kfac {

namespace {

constexpr int BT = TRD_BT;  // Householder vectors per block reflector of the back-transformation
constexpr int LB = 128;     // T factors are built for LB-wide halves and merged: T = [T1, -T1 (V1^T V2) T2; 0, T2]
static_assert(BT == 2 * LB, "block reflectors are merged from two halves");

inline int round_up(int x, int a) { return (x + a - 1) / a * a; }

struct BtBlock { float* S; float* Tm; float* TmT; const float* tau; int nb; };

// S = V^T V of one block -> T (upper triangular, forward columnwise: H_0 H_1 ... = I - V T V^T) of its two LB-wide halves
// (CTA 2 b + h: half h of block b); the off-diagonal quadrant follows from two small GEMMs (eigh_direct_run).
// TmT receives the transposes of the diagonal quadrants (operands of those GEMMs).
__global__ void __launch_bounds__(LB) larft_kernel(const BtBlock* blocks) {
  extern __shared__ float larft_smem[];
  float (*Ts)[LB + 1] = reinterpret_cast<float (*)[LB + 1]>(larft_smem);
  const BtBlock b = blocks[blockIdx.x >> 1];
  const int o = (blockIdx.x & 1) * LB;
  const int i = threadIdx.x, nb = max(0, min(LB, b.nb - o));
  for (int j = 0; j < LB; ++j) Ts[i][j] = 0.f;
  __syncthreads();
  for (int j = 0; j < nb; ++j) {
    const float tj = b.tau[o + j];
    float acc = 0.f;
    if (i < j) {
      for (int l = i; l < j; ++l) acc = fmaf(Ts[i][l], b.S[(o + l) * BT + o + j], acc);
      acc *= -tj;
    }
    __syncthreads();
    if (i < j) Ts[i][j] = acc;
    if (i == j) Ts[i][j] = tj;
    __syncthreads();
  }
  for (int j = 0; j < LB; ++j) {
    b.Tm[(o + j) * BT + o + i] = Ts[j][i];       // row j, coalesced over i
    b.TmT[(o + j) * BT + o + i] = Ts[i][j];
  }
}

// per-matrix pointers of the batched input / output kernels (one launch over all matrices of the call)
struct IoMat {
  const float* F; float* A;              // input factor (n x n, ld n) -> zero-padded working copy (np x np)
  const float* Z; float* ZT;             // eigenvectors of T (columns) -> their transpose, both np-strided
  float* Q; float* QT; int ldq;          // user outputs
  const float* dsrc; float* ddst;        // eigenvalues
  int n, np;
};

// A (np x np, zero padded) <- F (n x n, ld n), grid (x, matrix).  Entries that are not finite, or so large that the squared
// column norms of the reduction could overflow (|x| > 1e15), are replaced by 0 and reported in the status word (bit 1):
// the solve then runs on finite data (no NaN reaches the index arithmetic of the divide and conquer) and the caller
// sees the failure.
__global__ void pad_copy_kernel(const IoMat* mats, int* status) {
  const IoMat mt = mats[blockIdx.y];
  const int n = mt.n, np = mt.np;
  const int64_t total = (int64_t)np * np;
  bool bad = false;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int i = (int)(idx / np), j = (int)(idx % np);
    float x = (i < n && j < n) ? mt.F[(int64_t)i * n + j] : 0.f;
    if (!(fabsf(x) <= 1e15f)) { bad = true; x = 0.f; }
    mt.A[idx] = x;
  }
  if (bad && status) atomicOr(status, 2);
}

// ZT = Z^T for every matrix: grid (tiles, tiles, matrix)
__global__ void transpose_z_kernel(const IoMat* mats) {
  __shared__ float tile[32][33];
  const IoMat mt = mats[blockIdx.z];
  const int bx = blockIdx.x * 32, by = blockIdx.y * 32, n = mt.n;
  if (bx >= n || by >= n) return;
  for (int r = threadIdx.y; r < 32; r += 8) {
    const int i = by + r, j = bx + threadIdx.x;
    tile[r][threadIdx.x] = (i < n && j < n) ? mt.Z[(int64_t)i * mt.np + j] : 0.f;
  }
  __syncthreads();
  for (int r = threadIdx.y; r < 32; r += 8) {
    const int j = bx + r, i = by + threadIdx.x;
    if (j < n && i < n) mt.ZT[(int64_t)j * mt.np + i] = tile[threadIdx.x][r];
  }
}

// final outputs of every matrix from ZT (rows = eigenvectors): QT_user = ZT, Q_user = ZT^T (one read of the tile),
// eigenvalues clamped at 0 (eigen.py:321,344); grid (tiles, tiles, matrix)
__global__ void outputs_kernel(const IoMat* mats, int* status) {
  __shared__ float tile[32][33];
  const IoMat mt = mats[blockIdx.z];
  const int bx = blockIdx.x * 32, by = blockIdx.y * 32, n = mt.n;
  if (bx >= n || by >= n) return;
  for (int r = threadIdx.y; r < 32; r += 8) {
    const int i = by + r, j = bx + threadIdx.x;
    const float v = (i < n && j < n) ? mt.ZT[(int64_t)i * mt.np + j] : 0.f;
    tile[r][threadIdx.x] = v;
    if (mt.QT && i < n && j < n) mt.QT[(int64_t)i * mt.ldq + j] = v;
  }
  __syncthreads();
  for (int r = threadIdx.y; r < 32; r += 8) {
    const int j = bx + r, i = by + threadIdx.x;
    if (j < n && i < n) mt.Q[(int64_t)j * mt.ldq + i] = tile[threadIdx.x][r];
  }
  if (blockIdx.y == 0 && threadIdx.y == 0) {
    const int j = bx + threadIdx.x;
    if (j < n) {
      const float v = mt.dsrc[j];
      if (!isfinite(v) && status) atomicOr(status, 2);
      mt.ddst[j] = fmaxf(v, 0.f);
    }
  }
}

// single-matrix helpers of the test entries
__global__ void pad_copy_one_kernel(const float* F, int n, float* A, int np) {
  const int64_t total = (int64_t)np * np;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int i = (int)(idx / np), j = (int)(idx % np);
    A[idx] = (i < n && j < n) ? F[(int64_t)i * n + j] : 0.f;
  }
}

struct MatLayout {
  int n, np, nblk, nbt;
  size_t A, VT, Vb, Q0, Q1, P, Vp, Wp, part, col, tau, d, e, cpart, bar, fscr, iscr, S, Tm, TmT, Xt, Y, Y2, slabY, slabS;
  int ksplit;      // split count of the longest reduction of the back-transformation (K = np)
};

struct Layout {
  std::vector<MatLayout> m;
  size_t off_trd, off_jobs, off_dc, off_blocks, off_io, off_plan, plan_bytes, off_gws, gws_bytes, zero_begin, zero_end, total;
  int nblocks;
};

void make_layout(const int* n, int count, Layout& L) {
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off = align_up(off + bytes, 256); return o; };
  L.m.resize(count);
  L.off_trd = take(sizeof(TrdMat) * count);
  L.off_jobs = take(sizeof(TrdJob) * count);
  L.off_dc = take(sizeof(DcMat) * count);
  L.nblocks = 0;
  for (int i = 0; i < count; ++i) L.nblocks += ceil_div(n[i], BT);
  L.off_blocks = take(sizeof(BtBlock) * std::max(1, L.nblocks));
  L.off_io = take(sizeof(IoMat) * count);
  L.plan_bytes = stedc_plan_bytes(n, count);
  L.off_plan = take(L.plan_bytes);
  L.gws_bytes = grouped_gemm_ws_bytes(std::max(L.nblocks, count));
  L.off_gws = take(L.gws_bytes);
  const int grid = sytrd_max_grid();
  // everything that must start as zeros lies in ONE region (one memset per call): the reflector stores (their padding
  // is a GEMM reduction dimension), the panel, barrier and partial-scalar state of the tridiagonalisation, the two
  // eigenvector buffers of the divide and conquer (off-diagonal blocks), S and the T factors
  L.zero_begin = off;
  for (int i = 0; i < count; ++i) {
    MatLayout& m = L.m[i];
    m.n = n[i]; m.np = round_up(n[i], TRD_T); m.nblk = m.np / TRD_T; m.nbt = ceil_div(n[i], BT);
    m.ksplit = m.np > 1024 ? ceil_div(m.np, 512) : 1;
    const size_t sq = (size_t)m.np * m.np * sizeof(float);
    m.VT = take(sq); m.Vb = take(sq + (size_t)m.np * BT * 4); m.Q0 = take(sq); m.Q1 = take(sq);
    m.Vp = take((size_t)m.np * TRD_NB * 4); m.Wp = take((size_t)m.np * TRD_NB * 4);
    m.cpart = take((size_t)grid * TRD_CP * 4);
    m.bar = take(256);
    m.S = take((size_t)m.nbt * BT * BT * 4); m.Tm = take((size_t)m.nbt * BT * BT * 4); m.TmT = take((size_t)m.nbt * BT * BT * 4);
  }
  L.zero_end = off;
  for (int i = 0; i < count; ++i) {
    MatLayout& m = L.m[i];
    const size_t sq = (size_t)m.np * m.np * sizeof(float);
    m.A = take(sq + (size_t)m.np * BT * 4); m.P = take(sq);
    m.Y = take((size_t)m.np * BT * 4); m.Y2 = take((size_t)m.np * BT * 4);
    m.slabY = take((size_t)m.ksplit * m.np * BT * 4);
    m.slabS = take((size_t)m.nbt * m.ksplit * BT * BT * 4);
    m.part = take((size_t)m.nblk * m.np * 4);
    m.col = take((size_t)m.np * 4); m.tau = take((size_t)m.np * 4); m.d = take((size_t)m.np * 4); m.e = take((size_t)m.np * 4);
    m.fscr = take((size_t)12 * m.n * 4); m.iscr = take((size_t)12 * m.n * 4);
    m.Xt = take((size_t)m.nbt * LB * LB * 4);
  }
  L.total = off;
}

// ---- CTA-group schedule of the tridiagonalisation kernel --------------------------------------
// Time model of one matrix on a group of C CTAs, fitted (least squares on the relative error, worst 6.6 %, mean 1.9 %)
// to the sweep tests/sytrd_sweep.py over n = 256 .. 4608, C = 1 .. 132 on an H100 SXM 80 GB at a 400 W power limit
// (points below the smallest group a matrix can use left out): per column
//   T0 + T1 n            barriers, dependent cross-CTA loads, the serial vector phases
//   (B n^2 + GA n) / C   tile products of the trailing matrix (averaged over its shrinking size) + row work
//   DE log2 C            barrier and cross-CTA reduction cost growing with the group
constexpr double T0 = 6.92e-6, T1 = 2.82e-10, BETA = 1.24e-11, GAMMA = 1.6e-8, DELTA = 2.72e-7, EPS = -1.23e-6;
double job_time(int n, int C) {
  return (double)n * (T0 + T1 * n + (BETA * (double)n * n + GAMMA * n + EPS) / C + DELTA * std::log2((double)C));
}

void make_schedule(const int* n, int count, int G, std::vector<TrdJob>& jobs) {
  // smallest makespan M such that the CTA-time of all jobs (each sized to finish within M) fits into G * M
  auto ctas_for = [&](int ni, double M) {
    const int nb = (ni + TRD_T - 1) / TRD_T;
    const int cmin = std::min(G, sytrd_min_ctas(ni));
    const int cmax = std::max(cmin, std::min(G, nb * (nb + 1) / 2 / 2 + 1));   // >= 2 tiles per sub-group pays
    int fastest = cmin;
    for (int C = cmin; C <= cmax; ++C) {
      if (job_time(ni, C) <= M) return C;
      if (job_time(ni, C) < job_time(ni, fastest)) fastest = C;
    }
    return fastest;
  };
  double lo = 0, hi = 0;
  for (int i = 0; i < count; ++i) { lo = std::max(lo, job_time(n[i], ctas_for(n[i], 0.0))); hi += job_time(n[i], std::min(G, sytrd_min_ctas(n[i]))); }
  hi = std::max(hi, lo);
  for (int it = 0; it < 40; ++it) {
    const double M = 0.5 * (lo + hi);
    double area = 0;
    for (int i = 0; i < count; ++i) { const int C = ctas_for(n[i], M); area += C * job_time(n[i], C); }
    if (area <= 0.95 * G * M) hi = M; else lo = M;
  }
  std::vector<int> order(count), C(count);
  for (int i = 0; i < count; ++i) { order[i] = i; C[i] = ctas_for(n[i], hi); }
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return job_time(n[a], C[a]) > job_time(n[b], C[b]); });
  std::vector<double> avail(G, 0.0);
  struct Placed { double start; TrdJob job; };
  std::vector<Placed> placed;
  for (int i : order) {
    int best = 0; double best_t = 1e300;
    for (int c0 = 0; c0 + C[i] <= G; ++c0) {
      double t = 0;
      for (int c = c0; c < c0 + C[i]; ++c) t = std::max(t, avail[c]);
      if (t < best_t) { best_t = t; best = c0; }
    }
    for (int c = best; c < best + C[i]; ++c) avail[c] = best_t + job_time(n[i], C[i]);
    placed.push_back({best_t, TrdJob{i, best, C[i]}});
  }
  // a consistent global order (every CTA walks the list front to back) keeps the group barriers deadlock free
  std::stable_sort(placed.begin(), placed.end(), [](const Placed& a, const Placed& b) { return a.start < b.start; });
  jobs.clear();
  for (auto& p : placed) jobs.push_back(p.job);
}

}  // namespace

int StreamPool::init() {
  if (ready) return KFAC_OK;
  for (int i = 0; i < N; ++i) {
    KFAC_CUDA(cudaStreamCreateWithFlags(&st[i], cudaStreamNonBlocking));
    KFAC_CUDA(cudaEventCreateWithFlags(&ev_join[i], cudaEventDisableTiming));
  }
  KFAC_CUDA(cudaEventCreateWithFlags(&ev_fork, cudaEventDisableTiming));
  ready = true;
  return KFAC_OK;
}
int StreamPool::fork(cudaStream_t s) {
  int rc = init();
  if (rc) return rc;
  KFAC_CUDA(cudaEventRecord(ev_fork, s));
  for (int i = 0; i < N; ++i) KFAC_CUDA(cudaStreamWaitEvent(st[i], ev_fork, 0));
  return KFAC_OK;
}
int StreamPool::join(cudaStream_t s) {
  for (int i = 0; i < N; ++i) {
    KFAC_CUDA(cudaEventRecord(ev_join[i], st[i]));
    KFAC_CUDA(cudaStreamWaitEvent(s, ev_join[i], 0));
  }
  return KFAC_OK;
}
StreamPool& stream_pool() {
  static thread_local StreamPool pool;     // one per calling thread (and therefore per device context in practice)
  return pool;
}

int gemm_tn_acc(const float* A, int64_t lda, const float* B, int64_t ldb, float* D, int64_t ldd, int M, int N, int K,
                float alpha, cudaStream_t s) {
  TcGemmArgs t{};
  t.A = A; t.lda = lda; t.B = B; t.ldb = ldb; t.D = D; t.ldd = ldd; t.M = M; t.N = N; t.K = K;
  t.kbatch = 1; t.alpha = alpha; t.splits = 1; t.accumulate = 1;
  if (tc_gemm_supported(t)) return launch_tc_gemm(t, s);
  GemmArgs g{};
  g.A = A; g.sa_m = lda; g.sa_k = 1; g.B = B; g.sb_k = 1; g.sb_n = ldb;
  g.C = D; g.ldc = ldd; g.M = M; g.N = N; g.K = K; g.batch = 1; g.splitk = 1; g.alpha = alpha; g.beta = 1.f;
  return launch_gemm(g, s);
}

size_t eigh_direct_workspace_bytes(const int* n, int count) {
  if (count <= 0) return 0;
  Layout L;
  make_layout(n, count, L);
  return align_up(L.total, 1024);
}

// stage selector for tests / profiling: 1 = stop after the tridiagonalisation (d, e in the items' d / Q row 0),
// 0 = full solve
int eigh_direct_run(const kfac_eigh_item* items, int count, void* ws, size_t ws_bytes, int* status, cudaStream_t s) {
  if (count <= 0) return KFAC_OK;
  std::vector<int> ns(count);
  for (int i = 0; i < count; ++i) {
    ns[i] = items[i].n;
    // limits of the stages: the deflation scan of the top-level merge sorts n values in shared memory (6 n floats),
    // the tile lists of the tridiagonalisation hold 256 entries per sub-group
    if (ns[i] > KFAC_EIGH_MAX_N) {
      set_error("eigh(direct): n = %d exceeds the supported dimension %d", ns[i], KFAC_EIGH_MAX_N);
      return KFAC_ERR_UNSUPPORTED;
    }
    if (sytrd_min_ctas(ns[i]) > sytrd_max_grid()) {
      set_error("eigh(direct): n = %d needs %d CTAs for its tile lists, the device has %d SMs", ns[i], sytrd_min_ctas(ns[i]),
                sytrd_max_grid());
      return KFAC_ERR_UNSUPPORTED;
    }
  }
  Layout L;
  make_layout(ns.data(), count, L);
  if (!ws || ws_bytes < L.total) { set_error("eigh(direct): workspace too small (%zu < %zu)", ws_bytes, L.total); return KFAC_ERR_WORKSPACE; }
  char* base = (char*)ws;
  const int G = sytrd_max_grid();
  std::vector<TrdMat> trd(count);
  std::vector<DcMat> dc(count);
  int np_max = 0;
  for (int i = 0; i < count; ++i) {
    const MatLayout& m = L.m[i];
    TrdMat& t = trd[i];
    t.A = (float*)(base + m.A); t.VT = (float*)(base + m.VT); t.Vb = (float*)(base + m.Vb); t.tau = (float*)(base + m.tau);
    t.d = (float*)(base + m.d); t.e = (float*)(base + m.e);
    t.Vp = (float*)(base + m.Vp); t.Wp = (float*)(base + m.Wp); t.part = (float*)(base + m.part);
    t.col = (float*)(base + m.col); t.cpart = (float*)(base + m.cpart); t.bar = (unsigned int*)(base + m.bar);
    t.n = m.n; t.np = m.np; t.nblk = m.nblk; t.ldv = m.np;
    np_max = std::max(np_max, m.np);
    DcMat& d = dc[i];
    d.d = t.d; d.e = t.e; d.Q[0] = (float*)(base + m.Q0); d.Q[1] = (float*)(base + m.Q1);
    d.UT = t.A;                       // the working copy of F is dead after the tridiagonalisation
    d.P = (float*)(base + m.P);
    d.fscr = (float*)(base + m.fscr); d.iscr = (int*)(base + m.iscr);
    d.n = m.n; d.ld = m.np; d.result_buf = 0;
  }
  // inputs / zeroed state: one memset, one padding launch
  KFAC_CUDA(cudaMemsetAsync(base + L.zero_begin, 0, L.zero_end - L.zero_begin, s));
  std::vector<IoMat> io(count);
  for (int i = 0; i < count; ++i) {
    const MatLayout& m = L.m[i];
    IoMat& o = io[i];
    o.F = items[i].F; o.A = trd[i].A; o.n = m.n; o.np = m.np;
    o.Q = items[i].Q; o.QT = items[i].QT; o.ldq = items[i].ldq > 0 ? items[i].ldq : m.n;
    o.dsrc = trd[i].d; o.ddst = items[i].d;
    o.Z = nullptr; o.ZT = nullptr;
  }
  IoMat* d_io = (IoMat*)(base + L.off_io);
  KFAC_CUDA(cudaMemcpyAsync(d_io, io.data(), sizeof(IoMat) * count, cudaMemcpyHostToDevice, s));
  pad_copy_kernel<<<dim3(std::min(1024, ceil_div((int64_t)np_max * np_max, 256)), count), 256, 0, s>>>(d_io, status);
  KFAC_LAUNCH_CHECK();
  std::vector<TrdJob> jobs;
  make_schedule(ns.data(), count, G, jobs);
  TrdMat* d_trd = (TrdMat*)(base + L.off_trd);
  TrdJob* d_jobs = (TrdJob*)(base + L.off_jobs);
  DcMat* d_dc = (DcMat*)(base + L.off_dc);
  KFAC_CUDA(cudaMemcpyAsync(d_trd, trd.data(), sizeof(TrdMat) * count, cudaMemcpyHostToDevice, s));
  KFAC_CUDA(cudaMemcpyAsync(d_jobs, jobs.data(), sizeof(TrdJob) * jobs.size(), cudaMemcpyHostToDevice, s));
  KFAC_CUDA(cudaMemcpyAsync(d_dc, dc.data(), sizeof(DcMat) * count, cudaMemcpyHostToDevice, s));
  int rc;
  if ((rc = launch_sytrd(d_trd, d_jobs, (int)jobs.size(), np_max, G, s))) return rc;
  if ((rc = launch_stedc(dc.data(), d_dc, count, base + L.off_plan, L.plan_bytes, status, s, /*q_zeroed=*/true))) return rc;

  // ---- back-transformation: QT = Z^T B_{L-1}^T ... B_0^T, B_k = I - V_k T_k V_k^T
  std::vector<BtBlock> blocks;
  for (int i = 0; i < count; ++i) {
    const MatLayout& m = L.m[i];
    for (int kb = 0; kb < m.nbt; ++kb) {
      const int j0 = kb * BT, nb = std::min(BT, m.n - j0);
      blocks.push_back(BtBlock{(float*)(base + m.S) + (size_t)kb * BT * BT, (float*)(base + m.Tm) + (size_t)kb * BT * BT,
                               (float*)(base + m.TmT) + (size_t)kb * BT * BT, trd[i].tau + j0, nb});
    }
    // (S beyond the valid reflectors and the off-diagonal quadrants of T are zero: part of the zeroed region)
  }
  BtBlock* d_blocks = (BtBlock*)(base + L.off_blocks);
  KFAC_CUDA(cudaMemcpyAsync(d_blocks, blocks.data(), sizeof(BtBlock) * blocks.size(), cudaMemcpyHostToDevice, s));
  void* gws = base + L.off_gws;
  auto plain = [](const float* A, int64_t lda, const float* B, int64_t ldb, float* D, int64_t ldd, int M, int N, int K) {
    GroupedGemm g{};
    g.A = A; g.lda = lda; g.B = B; g.ldb = ldb; g.D = D; g.ldd = ldd; g.M = M; g.N = N; g.K = K;
    g.alpha = 1.f; g.epi = EPI_NONE; g.splits = 1; g.mode = 0;
    return g;
  };
  // S_k = V_k^T V_k for every block of every matrix: one grouped launch (long reductions through slabs)
  {
    std::vector<GroupedGemm> gg;
    for (int i = 0; i < count; ++i) {
      const MatLayout& m = L.m[i];
      const TrdMat& t = trd[i];
      for (int kb = 0; kb < m.nbt; ++kb) {
        const int j0 = kb * BT, nb = std::min(BT, m.n - j0), K = m.np - j0;
        const float* Vk = t.VT + (size_t)j0 * t.ldv + j0;
        GroupedGemm g = plain(Vk, t.ldv, Vk, t.ldv, (float*)(base + m.S) + (size_t)kb * BT * BT, BT, nb, nb, K);
        if (K > 1024 && grouped_gemm_tc_ok(g)) {
          g.splits = ceil_div(K, 512);
          g.slab = (float*)(base + m.slabS) + (size_t)kb * m.ksplit * BT * BT; g.slab_stride = (int64_t)nb * BT;
        }
        gg.push_back(g);
      }
    }
    if ((rc = launch_grouped_gemm(gg.data(), (int)gg.size(), gws, L.gws_bytes, s))) return rc;
  }
  {
    static bool attr = false;
    const int lsmem = LB * (LB + 1) * (int)sizeof(float);
    if (!attr) { KFAC_CUDA(cudaFuncSetAttribute(larft_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, lsmem)); attr = true; }
    larft_kernel<<<2 * (int)blocks.size(), LB, lsmem, s>>>(d_blocks);
    KFAC_LAUNCH_CHECK();
    // T12 = -T1 (S12 T2) for every block with more than LB reflectors: X^T = T2^T S12^T, then T12 = -T1 X
    std::vector<GroupedGemm> x1, x2;
    for (int i = 0; i < count; ++i) {
      const MatLayout& m = L.m[i];
      for (int kb = 0; kb < m.nbt; ++kb) {
        const int nb = std::min(BT, m.n - kb * BT);
        if (nb <= LB) continue;
        float* S = (float*)(base + m.S) + (size_t)kb * BT * BT;
        float* Tm = (float*)(base + m.Tm) + (size_t)kb * BT * BT;
        float* TmT = (float*)(base + m.TmT) + (size_t)kb * BT * BT;
        float* Xt = (float*)(base + m.Xt) + (size_t)kb * LB * LB;
        x1.push_back(plain(TmT + (size_t)LB * BT + LB, BT, S + LB, BT, Xt, LB, LB, LB, LB));
        GroupedGemm g = plain(Tm, BT, Xt, LB, Tm + LB, BT, LB, LB, LB);
        g.alpha = -1.f;
        x2.push_back(g);
      }
    }
    if (!x1.empty()) {
      if ((rc = launch_grouped_gemm(x1.data(), (int)x1.size(), gws, L.gws_bytes, s))) return rc;
      if ((rc = launch_grouped_gemm(x2.data(), (int)x2.size(), gws, L.gws_bytes, s))) return rc;
    }
  }
  int max_nbt = 0, n_max = 0;
  for (int i = 0; i < count; ++i) {
    const MatLayout& m = L.m[i];
    const DcMat& d = dc[i];
    max_nbt = std::max(max_nbt, m.nbt);
    n_max = std::max(n_max, m.n);
    io[i].Z = d.Q[d.result_buf]; io[i].ZT = d.Q[d.result_buf ^ 1];
  }
  // (the table is re-sent with the buffer parity the plan of the divide and conquer ended on)
  KFAC_CUDA(cudaMemcpyAsync(d_io, io.data(), sizeof(IoMat) * count, cudaMemcpyHostToDevice, s));
  transpose_z_kernel<<<dim3(ceil_div(n_max, 32), ceil_div(n_max, 32), count), dim3(32, 8), 0, s>>>(d_io);
  KFAC_LAUNCH_CHECK();
  // block reflectors, last block first; step t handles block (nbt - 1 - t) of every matrix that still has one:
  // three grouped launches per step instead of three GEMMs per block and matrix
  for (int tstep = 0; tstep < max_nbt; ++tstep) {
    std::vector<GroupedGemm> g1, g2, g3;
    for (int i = 0; i < count; ++i) {
      const MatLayout& m = L.m[i];
      if (m.nbt <= tstep) continue;
      const TrdMat& t = trd[i];
      const DcMat& d = dc[i];
      const int n = m.n, np = m.np, kb = m.nbt - 1 - tstep, j0 = kb * BT, nbp = std::min(BT, np - j0), K = np - j0;
      float* ZT = d.Q[d.result_buf ^ 1];
      float* Y = (float*)(base + m.Y);
      float* Y2 = (float*)(base + m.Y2);
      // Y = ZT[:, j0:] V_k[j0:, :]
      GroupedGemm a = plain(ZT + j0, np, t.VT + (size_t)j0 * t.ldv + j0, t.ldv, Y, BT, n, nbp, K);
      if (K > 1024 && grouped_gemm_tc_ok(a)) { a.splits = ceil_div(K, 512); a.slab = (float*)(base + m.slabY); a.slab_stride = (int64_t)n * BT; }
      g1.push_back(a);
      // Y2 = Y T_k^T
      g2.push_back(plain(Y, BT, (float*)(base + m.Tm) + (size_t)kb * BT * BT, BT, Y2, BT, n, nbp, nbp));
      // ZT[:, j0:] -= Y2 V_k[j0:, :]^T
      GroupedGemm c = plain(Y2, BT, t.Vb + (size_t)kb * np * BT + (size_t)j0 * BT, BT, ZT + j0, np, n, K, nbp);
      c.alpha = -1.f; c.mode = 1;
      g3.push_back(c);
    }
    if ((rc = launch_grouped_gemm(g1.data(), (int)g1.size(), gws, L.gws_bytes, s))) return rc;
    if ((rc = launch_grouped_gemm(g2.data(), (int)g2.size(), gws, L.gws_bytes, s))) return rc;
    if ((rc = launch_grouped_gemm(g3.data(), (int)g3.size(), gws, L.gws_bytes, s))) return rc;
  }
  outputs_kernel<<<dim3(ceil_div(n_max, 32), ceil_div(n_max, 32), count), dim3(32, 8), 0, s>>>(d_io, status);
  KFAC_LAUNCH_CHECK();
  return KFAC_OK;
}

}  // namespace kfac

// test / profiling entry (not in the public header): tridiagonalisation only
extern "C" int kfac_stage_sytrd(const float* F, int n, float* d, float* e, float* VT, int ldv, float* tau,
                                       void* ws, size_t ws_bytes, int ncta, void* stream) {
  using namespace kfac;
  cudaStream_t s = (cudaStream_t)stream;
  const int np = round_up(n, TRD_T), nblk = np / TRD_T;
  const int G = sytrd_max_grid();
  if (ncta <= 0 || ncta > G) ncta = G;
  ncta = std::max(ncta, std::min(G, sytrd_min_ctas(n)));
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off = align_up(off + bytes, 256); return o; };
  const size_t oA = take((size_t)np * (np + 128) * 4), oVT = take((size_t)np * np * 4), oVp = take((size_t)np * TRD_NB * 4),
               oWp = take((size_t)np * TRD_NB * 4), oPart = take((size_t)nblk * np * 4), oCol = take((size_t)np * 4),
               oTau = take((size_t)np * 4), oD = take((size_t)np * 4), oE = take((size_t)np * 4),
               oC = take((size_t)G * TRD_CP * 4), oBar = take(256), oMat = take(sizeof(TrdMat)), oJob = take(sizeof(TrdJob));
  if (!ws || ws_bytes < off) { set_error("sytrd test: workspace too small (%zu < %zu)", ws_bytes, off); return KFAC_ERR_WORKSPACE; }
  char* base = (char*)ws;
  TrdMat t;
  t.A = (float*)(base + oA); t.VT = (float*)(base + oVT); t.tau = (float*)(base + oTau); t.d = (float*)(base + oD);
  t.e = (float*)(base + oE); t.Vp = (float*)(base + oVp); t.Wp = (float*)(base + oWp); t.part = (float*)(base + oPart);
  t.col = (float*)(base + oCol); t.cpart = (float*)(base + oC); t.bar = (unsigned int*)(base + oBar);
  t.n = n; t.np = np; t.nblk = nblk; t.ldv = np; t.Vb = nullptr;
  pad_copy_one_kernel<<<std::min(1024, ceil_div((int64_t)np * np, 256)), 256, 0, s>>>(F, n, t.A, np);
  KFAC_LAUNCH_CHECK();
  KFAC_CUDA(cudaMemsetAsync(t.VT, 0, (size_t)np * np * 4, s));
  KFAC_CUDA(cudaMemsetAsync(t.Vp, 0, (size_t)np * TRD_NB * 4, s));
  KFAC_CUDA(cudaMemsetAsync(t.Wp, 0, (size_t)np * TRD_NB * 4, s));
  KFAC_CUDA(cudaMemsetAsync(t.bar, 0, 256, s));
  KFAC_CUDA(cudaMemsetAsync(t.cpart, 0, (size_t)G * TRD_CP * 4, s));
  TrdJob job{0, 0, ncta};
  KFAC_CUDA(cudaMemcpyAsync(base + oMat, &t, sizeof(t), cudaMemcpyHostToDevice, s));
  KFAC_CUDA(cudaMemcpyAsync(base + oJob, &job, sizeof(job), cudaMemcpyHostToDevice, s));
  int rc;
  if ((rc = launch_sytrd((TrdMat*)(base + oMat), (TrdJob*)(base + oJob), 1, np, G, s))) return rc;
  KFAC_CUDA(cudaMemcpyAsync(d, t.d, (size_t)n * 4, cudaMemcpyDeviceToDevice, s));
  KFAC_CUDA(cudaMemcpyAsync(e, t.e, (size_t)n * 4, cudaMemcpyDeviceToDevice, s));
  KFAC_CUDA(cudaMemcpyAsync(tau, t.tau, (size_t)n * 4, cudaMemcpyDeviceToDevice, s));
  if (VT) KFAC_CUDA(cudaMemcpy2DAsync(VT, (size_t)ldv * 4, t.VT, (size_t)np * 4, (size_t)n * 4, n, cudaMemcpyDeviceToDevice, s));
  return KFAC_OK;
}

// test entry: D&C on a given tridiagonal (d, e) -> eigenvalues (ascending) and eigenvectors (columns of Q, ld n)
extern "C" int kfac_stage_stedc(const float* d_in, const float* e_in, int n, float* evals, float* Q, void* ws,
                                       size_t ws_bytes, void* stream) {
  using namespace kfac;
  cudaStream_t s = (cudaStream_t)stream;
  const int np = round_up(n, TRD_T);
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off = align_up(off + bytes, 256); return o; };
  const size_t oQ0 = take((size_t)np * np * 4), oQ1 = take((size_t)np * np * 4), oUT = take((size_t)np * np * 4), oP = take((size_t)np * np * 4),
               oD = take((size_t)np * 4), oE = take((size_t)np * 4), oF = take((size_t)12 * n * 4), oI = take((size_t)12 * n * 4),
               oMat = take(sizeof(DcMat));
  const size_t pb = stedc_plan_bytes(&n, 1);
  const size_t oPlan = take(pb);
  if (!ws || ws_bytes < off) { set_error("stedc test: workspace too small (%zu < %zu)", ws_bytes, off); return KFAC_ERR_WORKSPACE; }
  char* base = (char*)ws;
  DcMat m;
  m.d = (float*)(base + oD); m.e = (float*)(base + oE); m.Q[0] = (float*)(base + oQ0); m.Q[1] = (float*)(base + oQ1);
  m.UT = (float*)(base + oUT); m.P = (float*)(base + oP); m.fscr = (float*)(base + oF); m.iscr = (int*)(base + oI); m.n = n; m.ld = np; m.result_buf = 0;
  KFAC_CUDA(cudaMemcpyAsync(m.d, d_in, (size_t)n * 4, cudaMemcpyDeviceToDevice, s));
  KFAC_CUDA(cudaMemsetAsync(m.e, 0, (size_t)np * 4, s));
  if (n > 1) KFAC_CUDA(cudaMemcpyAsync(m.e, e_in, (size_t)(n - 1) * 4, cudaMemcpyDeviceToDevice, s));
  KFAC_CUDA(cudaMemcpyAsync(base + oMat, &m, sizeof(m), cudaMemcpyHostToDevice, s));
  int rc;
  if ((rc = launch_stedc(&m, (DcMat*)(base + oMat), 1, base + oPlan, pb, nullptr, s))) return rc;
  KFAC_CUDA(cudaMemcpyAsync(evals, m.d, (size_t)n * 4, cudaMemcpyDeviceToDevice, s));
  KFAC_CUDA(cudaMemcpy2DAsync(Q, (size_t)n * 4, m.Q[m.result_buf], (size_t)np * 4, (size_t)n * 4, n, cudaMemcpyDeviceToDevice, s));
  return KFAC_OK;
}

extern "C" size_t kfac_stage_direct_workspace_bytes(int n) {
  const int np = (n + 63) / 64 * 64;
  return (size_t)np * np * 4 * 5 + (size_t)np * 4096 + (1u << 22);
}

// host-only: the CTA-group schedule of the tridiagonalisation kernel for a list of dimensions on `grid` CTAs
// (no device needed: tests/test_host_logic.py checks coverage, ranges and that the job order cannot deadlock)
extern "C" int kfac_stage_schedule(const int* n, int count, int grid, int* mat, int* cta0, int* ncta) {
  using namespace kfac;
  if (!n || count <= 0 || grid <= 0) return 0;
  std::vector<TrdJob> jobs;
  make_schedule(n, count, grid, jobs);
  for (size_t i = 0; i < jobs.size(); ++i) { mat[i] = jobs[i].mat; cta0[i] = jobs[i].cta0; ncta[i] = jobs[i].ncta; }
  return (int)jobs.size();
}
extern "C" int kfac_stage_sytrd_min_ctas(int n) { return kfac::sytrd_min_ctas(n); }

namespace kfac { int sytrd_profile(int on, unsigned long long* out16); }
extern "C" int kfac_stage_sytrd_profile(int on, unsigned long long* out16) { return kfac::sytrd_profile(on, out16); }
