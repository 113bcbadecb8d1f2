// K5: batched symmetric (PSD) eigendecomposition -- entry point and the small-matrix solver.
//
// Size classes
//   n <= 64 / n <= 128 : the whole matrix lives in the shared memory of ONE CTA; two-sided cyclic Jacobi with a
//                        round-robin ordering (N/2 disjoint rotations per step, N-1 steps per sweep), all such
//                        matrices of the batch in one launch on a side stream.
//   n  > 128           : direct solver (eigh_direct.cu): Householder tridiagonalisation (sytrd.cu), divide and
//                        conquer on the tridiagonal matrix (stedc.cu), block-reflector back-transformation --
//                        the same three stages as LAPACK's ssyevd behind torch.linalg.eigh
//                        (kfac/layers/eigen.py:310,331).
// Round 1 solved n > 128 by block one-sided Jacobi sweeps; the direct solver replaced it (4.4x faster on a lone
// 4608-wide factor, data-independent cost, LAPACK-class accuracy) and the sweep machinery was removed.
#include "common.cuh"
#include "eigh_direct.cuh"

#include <algorithm>
#include <vector>

namespace kfac {

struct SmallMat { const float* F; float* Q; float* QT; float* d; int n, ldq; };

// round-robin tournament: pair k of step r among nb (even) players
__device__ __forceinline__ void tournament(int r, int k, int nb, int& p, int& q) {
  const int m = nb - 1;
  int a, b;
  if (k == 0) { a = r % m; b = m; }
  else { a = (r + k) % m; b = (r - k + m) % m; }
  p = min(a, b); q = max(a, b);
}

// status word (device int in the workspace header): bit 0 = an iterative solve used up its sweeps, bit 1 = a
// non-finite eigenvalue came out (e.g. an AMP overflow step put Inf/NaN into a factor)
template <int N>
__global__ void __launch_bounds__(N * 8) jacobi_small_kernel(const SmallMat* mats, int max_sweeps, int* status) {
  extern __shared__ float sm[];
  float (*M)[N + 1] = reinterpret_cast<float (*)[N + 1]>(sm);
  float (*W)[N + 1] = reinterpret_cast<float (*)[N + 1]>(sm + N * (N + 1));
  float* cs = sm + 2 * N * (N + 1);       // c[N/2], s[N/2]
  int* pq = reinterpret_cast<int*>(cs + N);
  __shared__ int sh_big;
  __shared__ unsigned int sh_amax;
  __shared__ float sh_floor;
  __shared__ int sh_big_signal;
  constexpr int T = N * 8;   // the 2x2-block update is latency bound: more threads = fewer serial LDS/STS
  const int tid = threadIdx.x;
  const SmallMat mt = mats[blockIdx.x];
  const int n = mt.n;
  if (tid == 0) sh_amax = 0u;
  __syncthreads();
  bool bad_in = false;
  float amax = 0.f;
  for (int idx = tid; idx < N * N; idx += T) {
    const int i = idx / N, j = idx % N;
    float x = (i < n && j < n) ? mt.F[(int64_t)i * n + j] : 0.f;
    if (!eigh_entry_ok(x)) { bad_in = true; x = 0.f; }
    M[i][j] = x;
    W[i][j] = (i == j) ? 1.f : 0.f;
    amax = fmaxf(amax, fabsf(x));
  }
  if (bad_in) atomicOr(status, 2);
  atomicMax(&sh_amax, __float_as_uint(amax));
  __syncthreads();
  // normalise by an exact power of two (eigh_scale_exponent); the eigenvalues are scaled back on output
  const int ex = eigh_scale_exponent(sh_amax);
  if (ex != 0) {
    for (int idx = tid; idx < N * N; idx += T) M[idx / N][idx % N] = ldexpf(M[idx / N][idx % N], -ex);
    __syncthreads();
  }
  // noise level eps ||M||_F of the convergence test (fixed summation order: the same bits in every call)
  for (int i = tid; i < N; i += T) {
    float r = 0.f;
    for (int j = 0; j < N; ++j) r = fmaf(M[i][j], M[i][j], r);
    cs[i] = r;
  }
  __syncthreads();
  if (tid == 0) {
    float f = 0.f;
    for (int i = 0; i < N; ++i) f += cs[i];
    sh_floor = 0x1p-24f * sqrtf(f);
  }
  __syncthreads();
  const float floor_apq = sh_floor;
  bool converged = false;
  for (int sweep = 0; sweep < max_sweeps; ++sweep) {
    int rotated_sweep = 0;
    if (tid == 0) { sh_big = 0; sh_big_signal = 0; }   // set when some |sin| >= 2e-3 in this sweep
    __syncthreads();
    for (int st = 0; st < N - 1; ++st) {
      int rotated = 0;
      if (tid < N / 2) {
        int p, q;
        tournament(st, tid, N, p, q);
        const float apq = M[p][q], app = M[p][p], aqq = M[q][q];
        float c = 1.f, s = 0.f;
        if (fabsf(apq) > 1e-7f * sqrtf(fabsf(app * aqq))) {
          const float tau = (aqq - app) / (2.f * apq);
          const float t = copysignf(1.f, tau) / (fabsf(tau) + sqrtf(1.f + tau * tau));
          c = 1.f / sqrtf(1.f + t * t);   // IEEE sqrt/div: rsqrtf's bias makes column norms drift
          s = t * c;
          if (s != 0.f) {
            rotated = 1;
            if (fabsf(s) >= 2e-3f) { sh_big = 1; if (fabsf(apq) > floor_apq) sh_big_signal = 1; }
          }
        }
        cs[tid] = c;
        cs[N / 2 + tid] = s;
        pq[tid] = p | (q << 16);
      }
      // barrier + "did anybody rotate": a step without rotations is skipped entirely
      if (!__syncthreads_or(rotated)) continue;
      rotated_sweep = 1;
      // M <- J^T M J on independent 2x2 blocks (pair a rows) x (pair b columns)
      for (int idx = tid; idx < (N / 2) * (N / 2); idx += T) {
        const int b = idx % (N / 2), a = idx / (N / 2);
        const float ca = cs[a], sa = cs[N / 2 + a], cb = cs[b], sb = cs[N / 2 + b];
        if (sa == 0.f && sb == 0.f) continue;
        const int pa = pq[a] & 0xffff, qa = pq[a] >> 16, pb = pq[b] & 0xffff, qb = pq[b] >> 16;
        const float m00 = M[pa][pb], m01 = M[pa][qb], m10 = M[qa][pb], m11 = M[qa][qb];
        const float n00 = cb * m00 - sb * m01, n01 = sb * m00 + cb * m01;
        const float n10 = cb * m10 - sb * m11, n11 = sb * m10 + cb * m11;
        M[pa][pb] = ca * n00 - sa * n10;
        M[pa][qb] = ca * n01 - sa * n11;
        M[qa][pb] = sa * n00 + ca * n10;
        M[qa][qb] = sa * n01 + ca * n11;
      }
      // W <- W J
      for (int idx = tid; idx < N * (N / 2); idx += T) {
        const int i = idx % N, k = idx / N;
        const float c = cs[k], s = cs[N / 2 + k];
        if (s == 0.f) continue;
        const int p = pq[k] & 0xffff, q = pq[k] >> 16;
        const float u = W[i][p], v = W[i][q];
        W[i][p] = c * u - s * v;
        W[i][q] = s * u + c * v;
      }
      __syncthreads();
    }
    // all rotations tiny: the next sweep would only find second-order leftovers
    const int big = sh_big, big_signal = sh_big_signal;
    __syncthreads();
    if (!rotated_sweep || !big) { converged = true; break; }
    // in the null space of a rank-deficient factor app, aqq and apq are all rounding noise below eps ||M||_F: the
    // relative test keeps rotating them by large angles at an ever smaller scale and the sweeps never end.  Those
    // rotations are harmless, so a last sweep whose only large rotations are of noise counts as converged (the
    // sweeps themselves are left as they are, so every factor gets the same bits as before).
    if (sweep == max_sweeps - 1 && !big_signal) converged = true;
  }
  // M = W^T F W: rescale by the (rounding-drifted) column norms of W
  for (int j = tid; j < N; j += T) {
    float ww = 0.f;
    for (int i = 0; i < N; ++i) ww = fmaf(W[i][j], W[i][j], ww);
    cs[j] = ww > 0.f ? 1.f / sqrtf(ww) : 0.f;
  }
  __syncthreads();
  for (int idx = tid; idx < n * n; idx += T) {
    const int i = idx / n, j = idx % n;
    const float q = W[i][j] * cs[j];
    mt.Q[(int64_t)i * mt.ldq + j] = q;
    if (mt.QT) mt.QT[(int64_t)j * mt.ldq + i] = q;
  }
  int bad = 0;
  for (int j = tid; j < n; j += T) {
    const float dj = ldexpf(M[j][j] * cs[j] * cs[j], ex);
    if (!isfinite(dj)) bad = 2;
    mt.d[j] = fmaxf(dj, 0.f);      // clamp(min=0): kfac/layers/eigen.py:321,344
  }
  if (bad) atomicOr(status, 2);
  if (tid == 0 && !converged) atomicOr(status, 1);
}

}  // namespace kfac

using namespace kfac;

static const size_t SMEM64 = (2 * 64 * 65 + 64 + 32) * sizeof(float);
static const size_t SMEM128 = (2 * 128 * 129 + 128 + 64) * sizeof(float);
static const size_t HEADER = 256;     // status word

static size_t small_bytes(int count) { return align_up(sizeof(SmallMat) * (size_t)std::max(1, count), 256); }

extern "C" size_t kfac_eigh_workspace_bytes(const int* n, int count) {
  if (!n || count <= 0) return 0;
  std::vector<int> big;
  int nsmall = 0;
  for (int i = 0; i < count; ++i) { if (n[i] > 128) big.push_back(n[i]); else ++nsmall; }
  return HEADER + small_bytes(nsmall) + align_up(eigh_direct_workspace_bytes(big.data(), (int)big.size()), 1024);
}

extern "C" int kfac_eigh_batched(const kfac_eigh_item* items, int count, void* ws, size_t ws_bytes,
                                 int max_sweeps, float tol, void* stream) {
  (void)tol;
  KFAC_CHECK_ARG(count >= 0 && (items || count == 0), "items");
  if (count == 0) return KFAC_OK;
  cudaStream_t s = (cudaStream_t)stream;
  std::vector<kfac_eigh_item> big;
  std::vector<int> nbig;
  std::vector<SmallMat> s64, s128;
  for (int i = 0; i < count; ++i) {
    const kfac_eigh_item& it = items[i];
    KFAC_CHECK_ARG(it.F && it.Q && it.d && it.n > 0 && (it.ldq == 0 || it.ldq >= it.n), "eigh item");
    if (it.n > 128) { big.push_back(it); nbig.push_back(it.n); }
    else (it.n <= 64 ? s64 : s128).push_back(SmallMat{it.F, it.Q, it.QT, it.d, it.n, it.ldq > 0 ? it.ldq : it.n});
  }
  const size_t sb = small_bytes((int)(s64.size() + s128.size()));
  const size_t bd = align_up(eigh_direct_workspace_bytes(nbig.data(), (int)nbig.size()), 1024);
  if (!ws || ws_bytes < HEADER + sb + bd) {
    set_error("eigh: workspace too small (%zu < %zu)", ws_bytes, HEADER + sb + bd);
    return KFAC_ERR_WORKSPACE;
  }
  int* status = (int*)ws;
  KFAC_CUDA(cudaMemsetAsync(status, 0, HEADER, s));
  static bool attr = false;
  if (!attr) {
    KFAC_CUDA(cudaFuncSetAttribute(jacobi_small_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM128));
    KFAC_CUDA(cudaFuncSetAttribute(jacobi_small_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM64));
    attr = true;
  }
  if (max_sweeps <= 0) max_sweeps = 24;
  // the small matrices are solved by single latency-bound CTAs: a side stream overlaps them with the direct solver
  static cudaStream_t side = nullptr;
  static cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  const bool have_small = !s64.empty() || !s128.empty();
  cudaStream_t ss = s;
  if (have_small && !big.empty()) {
    if (!side) {
      KFAC_CUDA(cudaStreamCreateWithFlags(&side, cudaStreamNonBlocking));
      KFAC_CUDA(cudaEventCreateWithFlags(&ev_fork, cudaEventDisableTiming));
      KFAC_CUDA(cudaEventCreateWithFlags(&ev_join, cudaEventDisableTiming));
    }
    KFAC_CUDA(cudaEventRecord(ev_fork, s));
    KFAC_CUDA(cudaStreamWaitEvent(side, ev_fork, 0));
    ss = side;
  }
  if (have_small) {
    SmallMat* d_small = (SmallMat*)((char*)ws + HEADER);
    std::vector<SmallMat> all(s64);
    all.insert(all.end(), s128.begin(), s128.end());
    KFAC_CUDA(cudaMemcpyAsync(d_small, all.data(), sizeof(SmallMat) * all.size(), cudaMemcpyHostToDevice, ss));   // pageable: staged
    if (!s64.empty()) {
      jacobi_small_kernel<64><<<(int)s64.size(), 512, SMEM64, ss>>>(d_small, max_sweeps, status);
      KFAC_LAUNCH_CHECK();
    }
    if (!s128.empty()) {
      jacobi_small_kernel<128><<<(int)s128.size(), 1024, SMEM128, ss>>>(d_small + s64.size(), max_sweeps, status);
      KFAC_LAUNCH_CHECK();
    }
    if (ss != s) KFAC_CUDA(cudaEventRecord(ev_join, ss));
  }
  if (!big.empty()) {
    const int rc = eigh_direct_run(big.data(), (int)big.size(), (char*)ws + HEADER + sb, bd, status, s);
    if (rc) return rc;
  }
  if (ss != s) KFAC_CUDA(cudaStreamWaitEvent(s, ev_join, 0));
  return KFAC_OK;
}

extern "C" int kfac_eigh_status(const void* ws, int* host_status, void* stream) {
  KFAC_CHECK_ARG(ws && host_status, "eigh_status args");
  KFAC_CUDA(cudaMemcpyAsync(host_status, ws, sizeof(int), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  return KFAC_OK;
}
