// Direct symmetric eigensolver for the large K-FAC factors (replaces torch.linalg.eigh of
// kfac/layers/eigen.py:310,331 for n > 128):  F = H T H^T (sytrd.cu), T = Z L Z^T (stedc.cu),
// Q = H Z by compact-WY block reflectors of 128 Householder vectors (this file; wgmma GEMMs).
// Host side: workspace layout, the CTA-group schedule of the tridiagonalisation kernel, its waves, and the
// enqueue of all stages (one stream per wave) without host synchronisation.
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
  unsigned int* amax;                    // bit pattern of max|accepted entry| (zeroed workspace int)
  int n, np;
};

// amax <- max |x| over the entries of F the input rule accepts (eigh_entry_ok), grid (x, matrix)
__global__ void max_abs_kernel(const IoMat* mats) {
  const IoMat mt = mats[blockIdx.y];
  const int64_t total = (int64_t)mt.n * mt.n;
  float m = 0.f;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const float x = mt.F[idx];
    if (eigh_entry_ok(x)) m = fmaxf(m, fabsf(x));
  }
  const unsigned int bits = __reduce_max_sync(0xffffffffu, __float_as_uint(m));
  if ((threadIdx.x & 31) == 0 && bits) atomicMax(mt.amax, bits);
}

// A (np x np, zero padded) <- 2^-e F (n x n, ld n), e = eigh_scale_exponent(amax), grid (x, matrix).  Entries the input
// rule rejects are replaced by 0 and reported in the status word (bit 1): the solve then runs on finite data (no NaN
// reaches the index arithmetic of the divide and conquer) and the caller sees the failure.
__global__ void pad_copy_kernel(const IoMat* mats, int* status) {
  const IoMat mt = mats[blockIdx.y];
  const int n = mt.n, np = mt.np;
  const int ex = eigh_scale_exponent(*mt.amax);
  const int64_t total = (int64_t)np * np;
  bool bad = false;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int i = (int)(idx / np), j = (int)(idx % np);
    float x = (i < n && j < n) ? mt.F[(int64_t)i * n + j] : 0.f;
    if (!eigh_entry_ok(x)) { bad = true; x = 0.f; }
    mt.A[idx] = ldexpf(x, -ex);
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
// eigenvalues scaled back by 2^e and clamped at 0 (eigen.py:321,344); grid (tiles, tiles, matrix)
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
      const float v = ldexpf(mt.dsrc[j], eigh_scale_exponent(*mt.amax));
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

// One wave of the schedule (make_waves): a set of jobs whose CTAs no other wave's job uses.  It runs as its own
// cooperative launch, followed by the divide and conquer and back-transformation of its matrices, on its own stream.
struct Wave {
  std::vector<TrdJob> jobs;   // in the schedule's order; cta0 rebased onto the wave's grid, id = place in the schedule
  int ncta = 0;               // grid of its launch: the CTAs its jobs use
  int cap = 0;                // grid cap of its grouped GEMMs: the SMs free when it ends (by the predicted ends)
};

struct WaveLayout {
  int slot0, blk0;            // first entry of the wave in the job / DcMat / per-wave IoMat tables and in the BtBlock table
  size_t off_plan, plan_bytes, off_gws, gws_bytes;
};

struct Layout {
  std::vector<MatLayout> m;
  std::vector<WaveLayout> w;
  size_t off_trd, off_jobs, off_dc, off_blocks, off_io, off_amax, zero_begin, zero_end, total;
  int nblocks;
};

// Tables that are sent to the device are laid out in wave order, and each wave has its own plan and GEMM workspace:
// launches on different streams share no table and no workspace.
void make_layout(const int* n, int count, const std::vector<Wave>& waves, Layout& L) {
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off = align_up(off + bytes, 256); return o; };
  L.m.resize(count);
  L.off_trd = take(sizeof(TrdMat) * count);
  L.off_jobs = take(sizeof(TrdJob) * count);
  L.off_dc = take(sizeof(DcMat) * count);
  L.nblocks = 0;
  for (int i = 0; i < count; ++i) L.nblocks += ceil_div(n[i], BT);
  L.off_blocks = take(sizeof(BtBlock) * std::max(1, L.nblocks));
  L.off_io = take(sizeof(IoMat) * 2 * count);        // [0, count): the input stage, [count, 2 count): per wave
  L.w.resize(waves.size());
  int slot = 0, blk = 0;
  for (size_t k = 0; k < waves.size(); ++k) {
    WaveLayout& w = L.w[k];
    std::vector<int> nw;
    int nblk = 0;
    for (const TrdJob& j : waves[k].jobs) { nw.push_back(n[j.mat]); nblk += ceil_div(n[j.mat], BT); }
    w.slot0 = slot; w.blk0 = blk;
    slot += (int)nw.size(); blk += nblk;
    w.plan_bytes = stedc_plan_bytes(nw.data(), (int)nw.size());
    w.off_plan = take(w.plan_bytes);
    w.gws_bytes = grouped_gemm_ws_bytes(std::max(nblk, (int)nw.size()));
    w.off_gws = take(w.gws_bytes);
  }
  const int grid = sytrd_max_grid();
  // everything that must start as zeros lies in ONE region (one memset per call): the reflector stores (their padding
  // is a GEMM reduction dimension), the panel, barrier and partial-scalar state of the tridiagonalisation, the two
  // eigenvector buffers of the divide and conquer (off-diagonal blocks), S and the T factors, the max|F| of every matrix
  L.zero_begin = off;
  L.off_amax = take(sizeof(unsigned int) * count);
  for (int i = 0; i < count; ++i) {
    MatLayout& m = L.m[i];
    m.n = n[i]; m.np = round_up(n[i], TRD_T); m.nblk = m.np / TRD_T; m.nbt = ceil_div(n[i], BT);
    m.ksplit = chain_splits(m.np);
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

// start: if given, the predicted start time of every job (same order as jobs)
void make_schedule(const int* n, int count, int G, std::vector<TrdJob>& jobs, std::vector<double>* start = nullptr) {
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
  for (auto& p : placed) { p.job.id = (int)jobs.size(); jobs.push_back(p.job); }
  if (start) {
    start->clear();
    for (auto& p : placed) start->push_back(p.start);
  }
}

// ---- L2 residency plan of the tridiagonalisation -----------------------------------------------
// Phase A of every column re-reads the whole active lower triangle of its matrix, and the block column J of tiles
// stays active for min(n - 1, 64 (J + 1) - 1) columns.  The direct-solver matrices of a ResNet-50 batch hold ~280 MB of
// lower tiles at once, far more than the 50 MB L2, so under LRU nearly every tile read comes from HBM.  The plan keeps
// a trailing triangle (block columns J >= pin_j0) of selected matrices resident with evict_last and streams the rest
// evict_first.  Block columns are taken greedily by decreasing lifetime (reads per pinned byte), so each matrix's
// pinned set stays a contiguous trailing triangle, subject to: at every predicted instant (a job start of the
// schedule's time model) the pinned bytes of the running jobs fit `budget`.  A matrix whose next block column does
// not fit pins nothing more.  No L2 set-aside is used: the hints need no device-wide state.
constexpr long long TRD_PIN_BUDGET = 8ll << 20;      // bytes; see NOTES.md (L2 residency sweep)
long long g_pin_budget = -1;                          // test override (kfac_stage_sytrd_pin_budget); < 0: TRD_PIN_BUDGET

void make_pin_plan(const int* n, int count, const std::vector<TrdJob>& jobs, const std::vector<double>& start,
                   long long budget, std::vector<int>& pin_j0, std::vector<double>* t0 = nullptr,
                   std::vector<double>* t1 = nullptr) {
  pin_j0.resize(count);
  std::vector<double> js(count, 0.0), je(count, 0.0);
  for (size_t j = 0; j < jobs.size(); ++j) {
    const int i = jobs[j].mat;
    js[i] = start[j];
    je[i] = start[j] + job_time(n[i], jobs[j].ncta);
  }
  for (int i = 0; i < count; ++i) pin_j0[i] = (n[i] + TRD_T - 1) / TRD_T;
  if (t0) *t0 = js;
  if (t1) *t1 = je;
  if (budget <= 0) return;
  // instants at which the set of running jobs can grow: the job starts
  std::vector<double> inst(js);
  std::sort(inst.begin(), inst.end());
  inst.erase(std::unique(inst.begin(), inst.end()), inst.end());
  std::vector<long long> load(inst.size(), 0);
  struct Cand { int life, mat, J; };
  std::vector<Cand> cand;
  for (int i = 0; i < count; ++i) {
    const int nblk = pin_j0[i];
    for (int J = 0; J < nblk; ++J) cand.push_back({std::min(n[i] - 1, TRD_T * (J + 1) - 1), i, J});
  }
  // lifetime is strictly increasing in J within a matrix: each matrix's block columns come in decreasing J
  std::sort(cand.begin(), cand.end(), [](const Cand& a, const Cand& b) {
    if (a.life != b.life) return a.life > b.life;
    return a.mat != b.mat ? a.mat < b.mat : a.J > b.J;
  });
  std::vector<char> closed(count, 0);
  const long long tile_bytes = (long long)TRD_T * TRD_T * sizeof(float);
  for (const Cand& c : cand) {
    const int i = c.mat;
    if (closed[i]) continue;
    const long long bytes = (long long)((n[i] + TRD_T - 1) / TRD_T - c.J) * tile_bytes;   // tiles I >= J of column J
    bool fits = true;
    for (size_t k = 0; k < inst.size() && fits; ++k)
      if (inst[k] >= js[i] && inst[k] < je[i] && load[k] + bytes > budget) fits = false;
    if (!fits) { closed[i] = 1; continue; }
    for (size_t k = 0; k < inst.size(); ++k)
      if (inst[k] >= js[i] && inst[k] < je[i]) load[k] += bytes;
    pin_j0[i] = c.J;
  }
}

// ---- waves: parts of the schedule that can run on their own ---------------------------------------------------------
// Jobs that share a CTA are joined into components; no group barrier crosses from one component to another.  The
// later stages of a matrix (divide and conquer, back-transformation) can start as soon as its component is done, but
// in one launch they wait for the slowest job of the whole batch.  So the components are merged into at most
// `max_waves` waves, each a launch of its own followed by the later stages of its matrices on its own stream.  The
// waves are contiguous runs of the components sorted by predicted end, cut where the time the later-stage work waits
// for the end of its wave (weighted by n^3, the scale of that work) is smallest; of equally good cuts the one with the
// fewest waves is taken.  A wave keeps its jobs in the schedule's order, which keeps its group barriers deadlock free.
constexpr int EIGH_WAVES = StreamPool::N;
int g_max_waves = -1;                                 // test override (kfac_stage_eigh_max_waves); < 1: EIGH_WAVES

void make_waves(const int* n, int G, const std::vector<TrdJob>& jobs, const std::vector<double>& start, int max_waves,
                std::vector<Wave>& waves) {
  std::vector<int> root(G);
  for (int c = 0; c < G; ++c) root[c] = c;
  auto find = [&](int c) { while (root[c] != c) { root[c] = root[root[c]]; c = root[c]; } return c; };
  for (const TrdJob& j : jobs)
    for (int c = j.cta0 + 1; c < j.cta0 + j.ncta; ++c) root[find(c)] = find(j.cta0);
  std::vector<double> end(G, -1.0), work(G, 0.0);
  for (size_t j = 0; j < jobs.size(); ++j) {
    const int r = find(jobs[j].cta0), nj = n[jobs[j].mat];
    end[r] = std::max(end[r], start[j] + job_time(nj, jobs[j].ncta));
    work[r] += (double)nj * nj * nj;
  }
  std::vector<int> comp;
  for (int c = 0; c < G; ++c) if (end[c] >= 0.0) comp.push_back(c);
  std::stable_sort(comp.begin(), comp.end(), [&](int a, int b) { return end[a] < end[b]; });
  const int m = (int)comp.size(), K = std::max(1, std::min(max_waves, m));
  std::vector<double> W(m + 1, 0.0), WE(m + 1, 0.0);
  for (int i = 0; i < m; ++i) { W[i + 1] = W[i] + work[comp[i]]; WE[i + 1] = WE[i] + work[comp[i]] * end[comp[i]]; }
  auto wait = [&](int a, int b) { return end[comp[b]] * (W[b + 1] - W[a]) - (WE[b + 1] - WE[a]); };   // components a..b
  // f[k][b]: least wait of components 0..b in k + 1 waves; first[k][b]: first component of the last of them
  std::vector<std::vector<double>> f(K, std::vector<double>(m, 1e300));
  std::vector<std::vector<int>> first(K, std::vector<int>(m, 0));
  for (int b = 0; b < m; ++b) f[0][b] = wait(0, b);
  for (int k = 1; k < K; ++k)
    for (int b = k; b < m; ++b)
      for (int a = k; a <= b; ++a) {
        const double t = f[k - 1][a - 1] + wait(a, b);
        if (t < f[k][b]) { f[k][b] = t; first[k][b] = a; }
      }
  int k = 0;
  while (k < K - 1 && f[k][m - 1] > f[K - 1][m - 1] + 1e-9 * W[m] * end[comp[m - 1]]) ++k;
  std::vector<int> wave_of(G, -1);
  for (int b = m - 1, kk = k; b >= 0; --kk) {
    const int a = kk > 0 ? first[kk][b] : 0;
    for (int i = a; i <= b; ++i) wave_of[comp[i]] = kk;
    b = a - 1;
  }
  waves.assign(k + 1, Wave{});
  std::vector<int> used(G, -1);                        // wave of every CTA a job uses
  for (const TrdJob& j : jobs)
    for (int c = j.cta0; c < j.cta0 + j.ncta; ++c) used[c] = wave_of[find(j.cta0)];
  int freed = 0;                                       // CTAs no job uses, then those of the waves that end earlier
  for (int c = 0; c < G; ++c) freed += used[c] < 0;
  for (int w = 0; w <= k; ++w) {
    std::vector<int> rank(G, 0);                       // CTA -> its place in the wave's grid
    int nc = 0;
    for (int c = 0; c < G; ++c) if (used[c] == w) rank[c] = nc++;
    Wave& wv = waves[w];
    wv.ncta = nc;
    // the SMs free when the wave ends, by the predicted ends: its own and those of the waves before it (the last: all)
    freed += nc;
    wv.cap = freed;
    for (const TrdJob& j : jobs)
      if (used[j.cta0] == w) wv.jobs.push_back(TrdJob{j.mat, rank[j.cta0], j.ncta, j.id});
  }
}

// schedule, waves and workspace layout of one call
void make_plan(const int* n, int count, std::vector<TrdJob>& jobs, std::vector<double>& start, std::vector<Wave>& waves,
               Layout& L) {
  const int G = sytrd_max_grid();
  make_schedule(n, count, G, jobs, &start);
  make_waves(n, G, jobs, start, g_max_waves >= 1 ? g_max_waves : EIGH_WAVES, waves);
  make_layout(n, count, waves, L);
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
  std::vector<TrdJob> jobs;
  std::vector<double> start;
  std::vector<Wave> waves;
  Layout L;
  make_plan(n, count, jobs, start, waves, L);
  return align_up(L.total, 1024);
}

namespace {

// divide and conquer and back-transformation of the matrices of one wave, on stream s
int run_wave_tail(const Wave& wave, const WaveLayout& wl, const Layout& L, char* base, const std::vector<TrdMat>& trd,
                  std::vector<DcMat>& dc, std::vector<IoMat>& io, int* status, HostStage* stage, cudaStream_t s) {
  const int cnt = (int)wave.jobs.size(), cap = wave.cap;
  std::vector<int> mats(cnt);
  for (int k = 0; k < cnt; ++k) mats[k] = wave.jobs[k].mat;
  int rc;
  {
    std::vector<DcMat> dw(cnt);
    for (int k = 0; k < cnt; ++k) dw[k] = dc[mats[k]];
    DcMat* d_dc = (DcMat*)(base + L.off_dc) + wl.slot0;
    if ((rc = send_table(stage, d_dc, dw.data(), sizeof(DcMat) * cnt, s))) return rc;
    if ((rc = launch_stedc(dw.data(), d_dc, cnt, base + wl.off_plan, wl.plan_bytes, status, s, /*q_zeroed=*/true, cap, stage)))
      return rc;
    for (int k = 0; k < cnt; ++k) dc[mats[k]].result_buf = dw[k].result_buf;
  }

  // ---- back-transformation: QT = Z^T B_{L-1}^T ... B_0^T, B_k = I - V_k T_k V_k^T
  std::vector<BtBlock> blocks;
  for (const int i : mats) {
    const MatLayout& m = L.m[i];
    for (int kb = 0; kb < m.nbt; ++kb) {
      const int j0 = kb * BT, nb = std::min(BT, m.n - j0);
      blocks.push_back(BtBlock{(float*)(base + m.S) + (size_t)kb * BT * BT, (float*)(base + m.Tm) + (size_t)kb * BT * BT,
                               (float*)(base + m.TmT) + (size_t)kb * BT * BT, trd[i].tau + j0, nb});
    }
    // (S beyond the valid reflectors and the off-diagonal quadrants of T are zero: part of the zeroed region)
  }
  BtBlock* d_blocks = (BtBlock*)(base + L.off_blocks) + wl.blk0;
  if ((rc = send_table(stage, d_blocks, blocks.data(), sizeof(BtBlock) * blocks.size(), s))) return rc;
  void* gws = base + wl.off_gws;
  const size_t gws_bytes = wl.gws_bytes;
  auto plain = [](const float* A, int64_t lda, const float* B, int64_t ldb, float* D, int64_t ldd, int M, int N, int K) {
    GroupedGemm g{};
    g.A = A; g.lda = lda; g.B = B; g.ldb = ldb; g.D = D; g.ldd = ldd; g.M = M; g.N = N; g.K = K;
    g.alpha = 1.f; g.epi = EPI_NONE; g.splits = 1; g.mode = 0;
    return g;
  };
  // S_k = V_k^T V_k for every block of every matrix: one grouped launch (long reductions through slabs)
  {
    std::vector<GroupedGemm> gg;
    for (const int i : mats) {
      const MatLayout& m = L.m[i];
      const TrdMat& t = trd[i];
      for (int kb = 0; kb < m.nbt; ++kb) {
        const int j0 = kb * BT, nb = std::min(BT, m.n - j0), K = m.np - j0;
        const float* Vk = t.VT + (size_t)j0 * t.ldv + j0;
        GroupedGemm g = plain(Vk, t.ldv, Vk, t.ldv, (float*)(base + m.S) + (size_t)kb * BT * BT, BT, nb, nb, K);
        if (chain_splits(K) > 1 && grouped_gemm_tc_ok(g)) {
          g.splits = chain_splits(K);
          g.slab = (float*)(base + m.slabS) + (size_t)kb * m.ksplit * BT * BT; g.slab_stride = (int64_t)nb * BT;
        }
        gg.push_back(g);
      }
    }
    if ((rc = launch_grouped_gemm(gg.data(), (int)gg.size(), gws, gws_bytes, s, cap, stage))) return rc;
  }
  {
    static bool attr = false;
    const int lsmem = LB * (LB + 1) * (int)sizeof(float);
    if (!attr) { KFAC_CUDA(cudaFuncSetAttribute(larft_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, lsmem)); attr = true; }
    larft_kernel<<<2 * (int)blocks.size(), LB, lsmem, s>>>(d_blocks);
    KFAC_LAUNCH_CHECK();
    // T12 = -T1 (S12 T2) for every block with more than LB reflectors: X^T = T2^T S12^T, then T12 = -T1 X
    std::vector<GroupedGemm> x1, x2;
    for (const int i : mats) {
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
      if ((rc = launch_grouped_gemm(x1.data(), (int)x1.size(), gws, gws_bytes, s, cap, stage))) return rc;
      if ((rc = launch_grouped_gemm(x2.data(), (int)x2.size(), gws, gws_bytes, s, cap, stage))) return rc;
    }
  }
  int max_nbt = 0, n_max = 0;
  std::vector<IoMat> iw(cnt);
  for (int k = 0; k < cnt; ++k) {
    const int i = mats[k];
    const DcMat& d = dc[i];
    max_nbt = std::max(max_nbt, L.m[i].nbt);
    n_max = std::max(n_max, L.m[i].n);
    io[i].Z = d.Q[d.result_buf]; io[i].ZT = d.Q[d.result_buf ^ 1];
    iw[k] = io[i];
  }
  // (the wave's own table, with the buffer parity the plan of the divide and conquer ended on)
  IoMat* d_io = (IoMat*)(base + L.off_io) + L.m.size() + wl.slot0;
  if ((rc = send_table(stage, d_io, iw.data(), sizeof(IoMat) * cnt, s))) return rc;
  transpose_z_kernel<<<dim3(ceil_div(n_max, 32), ceil_div(n_max, 32), cnt), dim3(32, 8), 0, s>>>(d_io);
  KFAC_LAUNCH_CHECK();
  // block reflectors, last block first; step t handles block (nbt - 1 - t) of every matrix that still has one:
  // three grouped launches per step instead of three GEMMs per block and matrix
  for (int tstep = 0; tstep < max_nbt; ++tstep) {
    std::vector<GroupedGemm> g1, g2, g3;
    for (const int i : mats) {
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
      if (chain_splits(K) > 1 && grouped_gemm_tc_ok(a)) { a.splits = chain_splits(K); a.slab = (float*)(base + m.slabY); a.slab_stride = (int64_t)n * BT; }
      g1.push_back(a);
      // Y2 = Y T_k^T
      g2.push_back(plain(Y, BT, (float*)(base + m.Tm) + (size_t)kb * BT * BT, BT, Y2, BT, n, nbp, nbp));
      // ZT[:, j0:] -= Y2 V_k[j0:, :]^T
      GroupedGemm c = plain(Y2, BT, t.Vb + (size_t)kb * np * BT + (size_t)j0 * BT, BT, ZT + j0, np, n, K, nbp);
      c.alpha = -1.f; c.mode = 1;
      g3.push_back(c);
    }
    if ((rc = launch_grouped_gemm(g1.data(), (int)g1.size(), gws, gws_bytes, s, cap, stage))) return rc;
    if ((rc = launch_grouped_gemm(g2.data(), (int)g2.size(), gws, gws_bytes, s, cap, stage))) return rc;
    if ((rc = launch_grouped_gemm(g3.data(), (int)g3.size(), gws, gws_bytes, s, cap, stage))) return rc;
  }
  outputs_kernel<<<dim3(ceil_div(n_max, 32), ceil_div(n_max, 32), cnt), dim3(32, 8), 0, s>>>(d_io, status);
  KFAC_LAUNCH_CHECK();
  return KFAC_OK;
}

}  // namespace

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
  std::vector<TrdJob> jobs;
  std::vector<double> start;
  std::vector<Wave> waves;
  Layout L;
  make_plan(ns.data(), count, jobs, start, waves, L);
  if (!ws || ws_bytes < L.total) { set_error("eigh(direct): workspace too small (%zu < %zu)", ws_bytes, L.total); return KFAC_ERR_WORKSPACE; }
  char* base = (char*)ws;
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
    o.amax = (unsigned int*)(base + L.off_amax) + i;
    o.Z = nullptr; o.ZT = nullptr;
  }
  IoMat* d_io = (IoMat*)(base + L.off_io);
  KFAC_CUDA(cudaMemcpyAsync(d_io, io.data(), sizeof(IoMat) * count, cudaMemcpyHostToDevice, s));
  const dim3 io_grid(std::min(1024, ceil_div((int64_t)np_max * np_max, 256)), count);
  max_abs_kernel<<<io_grid, 256, 0, s>>>(d_io);
  KFAC_LAUNCH_CHECK();
  pad_copy_kernel<<<io_grid, 256, 0, s>>>(d_io, status);
  KFAC_LAUNCH_CHECK();
  std::vector<int> pin_j0;
  make_pin_plan(ns.data(), count, jobs, start, g_pin_budget >= 0 ? g_pin_budget : TRD_PIN_BUDGET, pin_j0);
  bool any_pin = false;
  for (int i = 0; i < count; ++i) any_pin |= pin_j0[i] < trd[i].nblk;
  for (int i = 0; i < count; ++i) { trd[i].pin_j0 = pin_j0[i]; trd[i].stream_first = any_pin ? 1 : 0; }
  TrdMat* d_trd = (TrdMat*)(base + L.off_trd);
  KFAC_CUDA(cudaMemcpyAsync(d_trd, trd.data(), sizeof(TrdMat) * count, cudaMemcpyHostToDevice, s));
  // one wave runs on s; several run on the side streams, which join s before the call returns (also on an error)
  const int nw = (int)waves.size();
  StreamPool& pool = stream_pool();
  // with several waves their tables go through pinned host memory: a pageable copy may make the host wait for one
  // wave's stream while the others still need their work enqueued
  HostStage* stage = nw > 1 ? &pool.stage : nullptr;
  int rc;
  if (stage && (rc = stage->begin())) return rc;
  if (nw > 1 && (rc = pool.fork(s))) return rc;
  auto wave_stream = [&](int w) { return nw > 1 ? pool.st[w] : s; };
  auto done = [&](int r) -> int {
    if (nw > 1) {
      int j = pool.join(s);
      if (!j) j = stage->end(s);
      if (!r) r = j;
    }
    return r;
  };
  // every wave's tridiagonalisation is enqueued before any later stage: the launches start together
  auto launch_wave = [&](int w) -> int {
    const Wave& wv = waves[w];
    const cudaStream_t sw = wave_stream(w);
    TrdJob* d_jobs = (TrdJob*)(base + L.off_jobs) + L.w[w].slot0;
    int np_w = 0;
    for (const TrdJob& j : wv.jobs) np_w = std::max(np_w, L.m[j.mat].np);
    const int rc = send_table(stage, d_jobs, wv.jobs.data(), sizeof(TrdJob) * wv.jobs.size(), sw);
    if (rc) return rc;
    return launch_sytrd(d_trd, d_jobs, (int)wv.jobs.size(), np_w, wv.ncta, sw);
  };
  for (int w = 0; w < nw; ++w)
    if ((rc = launch_wave(w))) return done(rc);
  for (int w = 0; w < nw; ++w)
    if ((rc = run_wave_tail(waves[w], L.w[w], L, base, trd, dc, io, status, stage, wave_stream(w)))) return done(rc);
  return done(KFAC_OK);
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
  t.pin_j0 = nblk; t.stream_first = 0;
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

// host-only: the L2 residency plan of the tridiagonalisation for the schedule of kfac_stage_schedule (same dims and
// grid) under `budget` bytes (< 0: the default).  Per matrix: pin_j0 (first pinned block column; nblk = none) and the
// predicted start / end of its job in seconds.  Returns count.
extern "C" int kfac_stage_pin_plan(const int* n, int count, int grid, long long budget, int* pin_j0, double* t0,
                                   double* t1) {
  using namespace kfac;
  if (!n || count <= 0 || grid <= 0) return 0;
  std::vector<TrdJob> jobs;
  std::vector<double> start, s0, s1;
  std::vector<int> pin;
  make_schedule(n, count, grid, jobs, &start);
  make_pin_plan(n, count, jobs, start, budget >= 0 ? budget : TRD_PIN_BUDGET, pin, &s0, &s1);
  for (int i = 0; i < count; ++i) { pin_j0[i] = pin[i]; t0[i] = s0[i]; t1[i] = s1[i]; }
  return count;
}
// test-only: the residency budget (bytes) of the following kfac_eigh_batched calls; < 0 restores the default
extern "C" void kfac_stage_sytrd_pin_budget(long long bytes) { kfac::g_pin_budget = bytes; }

// host-only: the waves of the schedule of kfac_stage_schedule (same dims and grid).  Per job of that list: its wave, its
// first CTA on the wave's grid and its place in the wave's job list.  Returns the number of waves.
extern "C" int kfac_stage_waves(const int* n, int count, int grid, int* wave, int* wave_cta0, int* wave_pos) {
  using namespace kfac;
  if (!n || count <= 0 || grid <= 0) return 0;
  std::vector<TrdJob> jobs;
  std::vector<double> start;
  std::vector<Wave> waves;
  make_schedule(n, count, grid, jobs, &start);
  make_waves(n, grid, jobs, start, g_max_waves >= 1 ? g_max_waves : EIGH_WAVES, waves);
  for (size_t w = 0; w < waves.size(); ++w)
    for (size_t k = 0; k < waves[w].jobs.size(); ++k) {
      const TrdJob& j = waves[w].jobs[k];
      wave[j.id] = (int)w; wave_cta0[j.id] = j.cta0; wave_pos[j.id] = (int)k;
    }
  return (int)waves.size();
}
// test-only: the most waves the following calls (kfac_eigh_batched, its workspace size, kfac_stage_waves) split the
// schedule into; < 1 restores the default.  1 runs every stage of every matrix on the caller's stream.
extern "C" void kfac_stage_eigh_max_waves(int w) { kfac::g_max_waves = w; }

namespace kfac {
int sytrd_profile(int on, unsigned long long* out16);
int sytrd_job_times(unsigned long long* out, int max_jobs);
}
extern "C" int kfac_stage_sytrd_profile(int on, unsigned long long* out16) { return kfac::sytrd_profile(on, out16); }
// %globaltimer (ns) at the start and end of job j of the last launch run with the profile switch on: out[2 j], out[2 j + 1]
extern "C" int kfac_stage_sytrd_job_times(unsigned long long* out, int max_jobs) { return kfac::sytrd_job_times(out, max_jobs); }
