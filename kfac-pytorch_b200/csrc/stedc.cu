// Divide and conquer for the symmetric tridiagonal eigenproblem (second stage of the direct eigensolver,
// eigh_direct.cuh) -- Cuppen's rank-one tearing with the deflation rules of LAPACK's slaed2 and the
// Gu/Eisenstat recomputation of the update vector, laid out for the GPU:
//   * T is cut into leaves of <= 64 rows (cuts at multiples of 64 keep every sub-block of Q 16-byte
//     aligned for TMA); leaves are solved by an implicit QL iteration, one warp per leaf, eigenvectors
//     accumulated in shared memory;
//   * all merges of the same tree level (of all matrices of the batch) run together:
//       deflate  (one CTA per merge: sort, z, slaed2 deflation scan)
//       rotate   (Givens rotations of close eigenvalue pairs applied to the columns of Q)
//       secular  (one warp per root: bracketing bisection on |mu| with geometric steps, pole-shifted origin)
//       zhat     (one warp per entry: Loewner product)
//       rank + build (final order; rows of U~^T: new eigenvectors in the basis of the old columns)
//       GEMM     Q_new = Q_old U~ on the wgmma engine, ONE grouped launch per level.  Merges of more than
//                DENSE_MAX rows use the structure LAPACK's slaed2/slaed3 use: only the k non-deflated columns of
//                Q_old enter the product (packed as [upper-only | mixed | lower-only] into P), the upper and lower
//                row halves are two problems over the column ranges they can see, and the deflated eigenvectors
//                are copied.  k is only known on the device: the kernel reads its k-block range from memory.
// Eigenvalues come out ascending, eigenvectors as columns of Q[result_buf].
#include "eigh_direct.cuh"

#include <algorithm>
#include <vector>

namespace kfac {

namespace {

constexpr int LEAF = 64;
constexpr int DENSE_MAX = 1024;           // merges up to this size multiply the full m x m x m product
constexpr float EPS = 5.9604645e-8f;      // relative machine epsilon (LAPACK slamch('E'))

struct DcMerge { int mat, lo, mid, hi, src; };   // src: buffer holding the children's eigenvectors
struct DcLeaf { int mat, lo, hi, buf; };
struct DcCut { int mat, pos; };

// scratch arrays (offsets in units of n)
enum { F_DL = 0, F_W, F_MU, F_LAM, F_ZHAT, F_DTMP, F_VALS, F_RC, F_RS, F_RHO, F_COUNT };
enum { I_NDCOL = 0, I_DFCOL, I_ORIG, I_INV, I_ROTA, I_ROTB, I_K, I_NROT, I_CPOS, I_CSRC, I_KR, I_COUNT };
// I_CPOS[i]: packed position of non-deflated entry i; I_CSRC[c]: column of Q_old packed at c;
// I_KR[0..3]: k-block ranges {upper begin, upper end, lower begin, lower end} of the two structured products

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_prod(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v *= __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ------------------------------------------------------------------ cuts
__global__ void dc_cut_kernel(const DcMat* mats, const DcCut* cuts, int ncuts) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ncuts) return;
  const DcMat& mt = mats[cuts[i].mat];
  const int c = cuts[i].pos;
  const float r = fabsf(mt.e[c - 1]);
  mt.d[c - 1] -= r;      // every position is touched by at most one cut
  mt.d[c] -= r;
}

// ------------------------------------------------------------------ leaves: implicit QL, one warp per leaf
__global__ void __launch_bounds__(64) dc_leaf_kernel(const DcMat* mats, const DcLeaf* leaves, int nleaves, int* status) {
  __shared__ float Z[2][LEAF][LEAF + 1];     // Z[w][col][row]
  __shared__ float sd[2][LEAF], se[2][LEAF];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int li = blockIdx.x * 2 + warp;
  if (li >= nleaves) return;
  const DcLeaf lf = leaves[li];
  const DcMat& mt = mats[lf.mat];
  const int n = lf.hi - lf.lo;
  float (*z)[LEAF + 1] = Z[warp];
  float* d = sd[warp];
  float* e = se[warp];
  for (int i = lane; i < LEAF; i += 32) {
    d[i] = i < n ? mt.d[lf.lo + i] : 0.f;
    e[i] = (i + 1 < n) ? mt.e[lf.lo + i] : 0.f;
  }
  for (int c = 0; c < n; ++c)
    for (int r = lane; r < n; r += 32) z[c][r] = (r == c) ? 1.f : 0.f;
  __syncwarp();
  // every lane runs the same scalar recurrence; lane l rotates rows l, l + 32 of the eigenvector matrix
  for (int l = 0; l < n; ++l) {
    for (int iter = 0; ; ++iter) {
      if (iter == 60) { if (lane == 0 && status) atomicOr(status, 1); break; }   // no convergence (LAPACK: info > 0)
      int m = l;
      for (; m < n - 1; ++m) {
        const float dd = fabsf(d[m]) + fabsf(d[m + 1]);
        if (fabsf(e[m]) <= EPS * dd) break;
      }
      if (m == l) break;
      float g = (d[l + 1] - d[l]) / (2.f * e[l]);
      float r = hypotf(g, 1.f);
      g = d[m] - d[l] + e[l] / (g + copysignf(r, g));
      float s = 1.f, c = 1.f, p = 0.f;
      int i = m - 1;
      bool under = false;
      for (; i >= l; --i) {
        float f = s * e[i];
        const float b = c * e[i];
        r = hypotf(f, g);
        __syncwarp();
        if (lane == 0) e[i + 1] = r;
        if (r == 0.f) {
          if (lane == 0) { d[i + 1] -= p; e[m] = 0.f; }
          under = true;
          break;
        }
        s = f / r;
        c = g / r;
        g = d[i + 1] - p;
        r = (d[i] - g) * s + 2.f * c * b;
        p = s * r;
        __syncwarp();
        if (lane == 0) d[i + 1] = g + p;
        g = c * r - b;
        for (int k = lane; k < n; k += 32) {
          const float zk1 = z[i + 1][k], zk0 = z[i][k];
          z[i + 1][k] = s * zk0 + c * zk1;
          z[i][k] = c * zk0 - s * zk1;
        }
      }
      __syncwarp();
      if (!under) {
        if (lane == 0) { d[l] -= p; e[l] = g; e[m] = 0.f; }
      }
      __syncwarp();
    }
  }
  __syncwarp();
  float* Q = mt.Q[lf.buf];
  for (int r = 0; r < n; ++r)
    for (int c = lane; c < n; c += 32) Q[(int64_t)(lf.lo + r) * mt.ld + lf.lo + c] = z[c][r];
  for (int i = lane; i < n; i += 32) mt.d[lf.lo + i] = d[i];
}

// ------------------------------------------------------------------ deflation (slaed2), one CTA per merge
__global__ void __launch_bounds__(1024) dc_deflate_kernel(const DcMat* mats, const DcMerge* merges) {
  extern __shared__ float dsm[];
  const DcMerge mg = merges[blockIdx.x];
  const DcMat& mt = mats[mg.mat];
  const int m = mg.hi - mg.lo, n1 = mg.mid - mg.lo, n = mt.n;
  float* rd = dsm;                 // raw d
  float* rz = rd + m;              // raw z
  float* sd = rz + m;              // sorted
  float* sz = sd + m;
  int* ssrc = reinterpret_cast<int*>(sz + m);
  int* ctype = ssrc + m;           // per column of Q_old: 1 = non-zero in the upper rows only, 3 = lower only, 2 = both
  __shared__ float redf[64];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const float* Q = mt.Q[mg.src];
  const float rho0 = mt.e[mg.mid - 1];
  const float sgn = rho0 < 0.f ? -1.f : 1.f;
  const float rho = 2.f * fabsf(rho0);
  float dmax = 0.f, zmax = 0.f;
  for (int i = tid; i < m; i += blockDim.x) {
    const float dv = mt.d[mg.lo + i];
    const float zv = (i < n1 ? Q[(int64_t)(mg.mid - 1) * mt.ld + mg.lo + i] : sgn * Q[(int64_t)mg.mid * mt.ld + mg.lo + i]) *
                     0.70710678118654752f;
    rd[i] = dv; rz[i] = zv;
    ctype[i] = i < n1 ? 1 : 3;
    dmax = fmaxf(dmax, fabsf(dv));
    zmax = fmaxf(zmax, fabsf(zv));
  }
  dmax = warp_max(dmax); zmax = warp_max(zmax);
  if (lane == 0) { redf[warp] = dmax; redf[32 + warp] = zmax; }
  __syncthreads();
  if (warp == 0) {
    dmax = warp_max(redf[lane]); zmax = warp_max(redf[32 + lane]);
    if (lane == 0) { redf[0] = dmax; redf[32] = zmax; }
  }
  __syncthreads();
  dmax = redf[0]; zmax = redf[32];
  // counting sort (ties by index)
  for (int i = tid; i < m; i += blockDim.x) {
    const float di = rd[i];
    int r = 0;
    for (int j = 0; j < m; ++j) { const float dj = rd[j]; r += (dj < di) || (dj == di && j < i); }
    sd[r] = di; sz[r] = rz[i]; ssrc[r] = i;
  }
  __syncthreads();
  float* fs = mt.fscr;
  int* is = mt.iscr;
  float* dl = fs + (int64_t)F_DL * n + mg.lo;
  float* w = fs + (int64_t)F_W * n + mg.lo;
  float* vals = fs + (int64_t)F_VALS * n + mg.lo;
  float* rc = fs + (int64_t)F_RC * n + mg.lo;
  float* rs = fs + (int64_t)F_RS * n + mg.lo;
  int* ndcol = is + (int64_t)I_NDCOL * n + mg.lo;
  int* dfcol = is + (int64_t)I_DFCOL * n + mg.lo;
  int* rota = is + (int64_t)I_ROTA * n + mg.lo;
  int* rotb = is + (int64_t)I_ROTB * n + mg.lo;
  int* cpos = is + (int64_t)I_CPOS * n + mg.lo;
  int* csrc = is + (int64_t)I_CSRC * n + mg.lo;
  // LAPACK slaed2's deflation rule.  zmax (|z| <= 1) does not scale with T, so the tolerance is only right for a T of
  // norm near 1: eigh_direct.cu hands over factors with max|F| in [1/16, 2) (eigh_scale_exponent), as sstedc scales T.
  const float tol = 8.f * EPS * fmaxf(dmax, zmax);
  if (tid == 0) {
    int k = 0, nd = 0, nrot = 0;
    int kt[4] = {0, 0, 0, 0};        // non-deflated columns per type
    // deflated values are written to rd[] (raw arrays are free now) in scan order, columns to rz-as-int;
    // the type and column of the non-deflated entries are kept at the far end of the same arrays (nd + k <= m)
    int* dcol_tmp = reinterpret_cast<int*>(rz);
    int* ktype_tmp = reinterpret_cast<int*>(rd);
    auto emit = [&](int pj) {
      const int col = ssrc[pj], t = ctype[col];
      dl[k] = sd[pj]; w[k] = sz[pj]; ndcol[k] = col;
      ktype_tmp[m - 1 - k] = t; dcol_tmp[m - 1 - k] = col; ++kt[t];
      ++k;
    };
    if (rho * zmax <= tol) {
      for (int j = 0; j < m; ++j) { rd[nd] = sd[j]; dcol_tmp[nd] = ssrc[j]; ++nd; }
    } else {
      int pj = -1;
      for (int j = 0; j < m; ++j) {
        const float zj = sz[j];
        if (rho * fabsf(zj) <= tol) { rd[nd] = sd[j]; dcol_tmp[nd] = ssrc[j]; ++nd; continue; }
        if (pj < 0) { pj = j; continue; }
        float s = sz[pj], c = zj;
        const float tau = hypotf(c, s);
        const float t = sd[j] - sd[pj];
        c = c / tau; s = -s / tau;
        if (fabsf(t * c * s) <= tol) {
          sz[j] = tau; sz[pj] = 0.f;
          rota[nrot] = ssrc[pj]; rotb[nrot] = ssrc[j]; rc[nrot] = c; rs[nrot] = s; ++nrot;
          if (ctype[ssrc[pj]] != ctype[ssrc[j]]) ctype[ssrc[j]] = 2;      // the surviving column now mixes both halves
          const float dp = sd[pj], dj = sd[j];
          sd[j] = dp * s * s + dj * c * c;
          sd[pj] = dp * c * c + dj * s * s;
          rd[nd] = sd[pj]; dcol_tmp[nd] = ssrc[pj]; ++nd;
          pj = j;
        } else {
          emit(pj);
          pj = j;
        }
      }
      if (pj >= 0) emit(pj);
    }
    // packed order of the non-deflated columns: [upper only | mixed | lower only]
    {
      int off[4] = {0, 0, kt[1], kt[1] + kt[2]};
      for (int i = 0; i < k; ++i) {
        const int t = ktype_tmp[m - 1 - i], c = off[t]++;
        cpos[i] = c; csrc[c] = dcol_tmp[m - 1 - i];
      }
      int* kr = is + (int64_t)I_KR * n + mg.lo;
      kr[0] = 0; kr[1] = (kt[1] + kt[2] + 31) / 32;          // upper rows see types 1 and 2
      kr[2] = kt[1] / 32; kr[3] = (k + 31) / 32;             // lower rows see types 2 and 3
      if (kt[1] + kt[2] == 0) kr[1] = 0;
      if (kt[2] + kt[3] == 0) kr[3] = kr[2];
    }
    is[(int64_t)I_K * n + mg.lo] = k;
    is[(int64_t)I_NROT * n + mg.lo] = nrot;
    fs[(int64_t)F_RHO * n + mg.lo] = rho;
    redf[1] = __int_as_float(k);
  }
  __syncthreads();
  const int k = __float_as_int(redf[1]);
  // deflated eigenpairs go behind the k roots in the list of values to be ranked
  const int* dcol_tmp = reinterpret_cast<const int*>(rz);
  for (int i = tid; i < m - k; i += blockDim.x) { vals[k + i] = rd[i]; dfcol[i] = dcol_tmp[i]; }
}

// ------------------------------------------------------------------ Givens rotations of deflated pairs
__global__ void __launch_bounds__(256) dc_rotate_kernel(const DcMat* mats, const DcMerge* merges) {
  const DcMerge mg = merges[blockIdx.y];
  const DcMat& mt = mats[mg.mat];
  const int m = mg.hi - mg.lo, n = mt.n;
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  const int nrot = mt.iscr[(int64_t)I_NROT * n + mg.lo];
  if (r >= m || nrot == 0) return;
  const int* rota = mt.iscr + (int64_t)I_ROTA * n + mg.lo;
  const int* rotb = mt.iscr + (int64_t)I_ROTB * n + mg.lo;
  const float* rc = mt.fscr + (int64_t)F_RC * n + mg.lo;
  const float* rs = mt.fscr + (int64_t)F_RS * n + mg.lo;
  float* row = mt.Q[mg.src] + (int64_t)(mg.lo + r) * mt.ld + mg.lo;
  // chains: rotation t+1 usually continues with column b of rotation t -> keep it in a register
  int cur = -1;
  float yb = 0.f;
  for (int t = 0; t < nrot; ++t) {
    const int a = rota[t], b = rotb[t];
    const float c = rc[t], s = rs[t];
    float x;
    if (a == cur) x = yb;
    else { if (cur >= 0) row[cur] = yb; x = row[a]; }
    const float y = row[b];
    row[a] = c * x + s * y;
    yb = c * y - s * x;
    cur = b;
  }
  if (cur >= 0) row[cur] = yb;
}

// ------------------------------------------------------------------ non-deflated columns of Q_old, packed by type
__global__ void __launch_bounds__(256) dc_pack_kernel(const DcMat* mats, const DcMerge* merges) {
  const DcMerge mg = merges[blockIdx.y];
  const DcMat& mt = mats[mg.mat];
  const int m = mg.hi - mg.lo, n = mt.n;
  if (m <= DENSE_MAX) return;
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= m) return;
  const int k = mt.iscr[(int64_t)I_K * n + mg.lo];
  const int kpad = (k + 31) & ~31;                            // the last k-block of the products is zero filled
  const int* csrc = mt.iscr + (int64_t)I_CSRC * n + mg.lo;
  const float* src = mt.Q[mg.src] + (int64_t)(mg.lo + r) * mt.ld + mg.lo;
  float* dst = mt.P + (int64_t)(mg.lo + r) * mt.ld + mg.lo;
  for (int c = lane; c < kpad; c += 32) dst[c] = c < k ? src[csrc[c]] : 0.f;
}

// deflated eigenvectors are columns of Q_old: copy them to their final positions (after the structured product)
__global__ void __launch_bounds__(256) dc_copy_deflated_kernel(const DcMat* mats, const DcMerge* merges) {
  const DcMerge mg = merges[blockIdx.y];
  const DcMat& mt = mats[mg.mat];
  const int m = mg.hi - mg.lo, n = mt.n;
  if (m <= DENSE_MAX) return;
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= m) return;
  const int k = mt.iscr[(int64_t)I_K * n + mg.lo];
  const int* inv = mt.iscr + (int64_t)I_INV * n + mg.lo;
  const int* dfcol = mt.iscr + (int64_t)I_DFCOL * n + mg.lo;
  const float* src = mt.Q[mg.src] + (int64_t)(mg.lo + r) * mt.ld + mg.lo;
  float* dst = mt.Q[mg.src ^ 1] + (int64_t)(mg.lo + r) * mt.ld + mg.lo;
  for (int p = lane; p < m; p += 32) {
    const int s = inv[p];
    if (s >= k) dst[p] = src[dfcol[s - k]];
  }
}

// ------------------------------------------------------------------ secular equation, one warp per root
// g(mu) = 1 + rho * sum_i w_i^2 / ((dl_i - dl_o) - mu), lambda = dl_o + mu
__device__ __forceinline__ float secular_g(const float* __restrict__ dl, const float* __restrict__ w, int k, float dlo,
                                           float rho, float mu, int lane) {
  float acc = 0.f;
  for (int i = lane; i < k; i += 32) {
    const float wi = w[i];
    acc += (wi * wi) / ((dl[i] - dlo) - mu);
  }
  return 1.f + rho * warp_sum(acc);
}

__global__ void __launch_bounds__(256) dc_secular_kernel(const DcMat* mats, const DcMerge* merges) {
  const DcMerge mg = merges[blockIdx.y];
  const DcMat& mt = mats[mg.mat];
  const int n = mt.n;
  const int k = mt.iscr[(int64_t)I_K * n + mg.lo];
  const int lane = threadIdx.x & 31;
  const int j = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (j >= k) return;
  const float* dl = mt.fscr + (int64_t)F_DL * n + mg.lo;
  const float* w = mt.fscr + (int64_t)F_W * n + mg.lo;
  const float rho = mt.fscr[(int64_t)F_RHO * n + mg.lo];
  int o;
  float sgn, thi;
  if (j < k - 1) {
    const float H = 0.5f * (dl[j + 1] - dl[j]);
    const float fm = secular_g(dl, w, k, dl[j], rho, H, lane);
    if (fm > 0.f) { o = j; sgn = 1.f; } else { o = j + 1; sgn = -1.f; }
    thi = H;
  } else {
    float ss = 0.f;
    for (int i = lane; i < k; i += 32) ss = fmaf(w[i], w[i], ss);
    o = j; sgn = 1.f; thi = rho * warp_sum(ss);
  }
  const float dlo = dl[o];
  // h(t) = sgn * g(sgn * t) is negative for small t and non-negative at thi
  float tlo = 0.f;
  {
    float t = thi;
    for (int it = 0; it < 12; ++it) {
      t *= 0.0625f;
      if (!(t > 0.f)) break;
      const float h = sgn * secular_g(dl, w, k, dlo, rho, sgn * t, lane);
      if (h < 0.f) { tlo = t; break; }
      thi = t;
    }
  }
  for (int it = 0; it < 64; ++it) {
    float tm;
    if (tlo > 0.f && thi > 4.f * tlo) tm = sqrtf(tlo) * sqrtf(thi);
    else tm = 0.5f * (tlo + thi);
    if (!(tm > tlo) || !(tm < thi)) break;
    const float h = sgn * secular_g(dl, w, k, dlo, rho, sgn * tm, lane);
    if (h < 0.f) tlo = tm; else thi = tm;
  }
  if (lane == 0) {
    const float mu = sgn * 0.5f * (tlo + thi);
    mt.fscr[(int64_t)F_MU * n + mg.lo + j] = mu;
    const float lam = dlo + mu;
    mt.fscr[(int64_t)F_LAM * n + mg.lo + j] = lam;
    mt.fscr[(int64_t)F_VALS * n + mg.lo + j] = lam;
    mt.iscr[(int64_t)I_ORIG * n + mg.lo + j] = o;
  }
}

// ------------------------------------------------------------------ Gu-Eisenstat update vector, one warp per entry
__global__ void __launch_bounds__(256) dc_zhat_kernel(const DcMat* mats, const DcMerge* merges) {
  const DcMerge mg = merges[blockIdx.y];
  const DcMat& mt = mats[mg.mat];
  const int n = mt.n;
  const int k = mt.iscr[(int64_t)I_K * n + mg.lo];
  const int lane = threadIdx.x & 31;
  const int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (i >= k) return;
  const float* dl = mt.fscr + (int64_t)F_DL * n + mg.lo;
  const float* w = mt.fscr + (int64_t)F_W * n + mg.lo;
  const float* mu = mt.fscr + (int64_t)F_MU * n + mg.lo;
  const int* orig = mt.iscr + (int64_t)I_ORIG * n + mg.lo;
  const float rho = mt.fscr[(int64_t)F_RHO * n + mg.lo];
  const float di = dl[i];
  float p = 1.f;
  for (int j = lane; j < k; j += 32) {
    const float num = (di - dl[orig[j]]) - mu[j];        // dl_i - lambda_j
    if (j == i) p *= -num;                               // lambda_i - dl_i > 0
    else p *= num / (di - dl[j]);
  }
  p = warp_prod(p);
  if (lane == 0) mt.fscr[(int64_t)F_ZHAT * n + mg.lo + i] = copysignf(sqrtf(fabsf(p) / rho), w[i]);
}

// ------------------------------------------------------------------ final order of the merged eigenvalues
__global__ void __launch_bounds__(256) dc_rank_kernel(const DcMat* mats, const DcMerge* merges) {
  const DcMerge mg = merges[blockIdx.y];
  const DcMat& mt = mats[mg.mat];
  const int m = mg.hi - mg.lo, n = mt.n;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  const float* vals = mt.fscr + (int64_t)F_VALS * n + mg.lo;
  const float vi = vals[i];
  int r = 0;
  for (int j = 0; j < m; ++j) { const float vj = vals[j]; r += (vj < vi) || (vj == vi && j < i); }
  mt.iscr[(int64_t)I_INV * n + mg.lo + r] = i;
}

// rows of U~^T (one warp per merged eigenvector, in final order)
__global__ void __launch_bounds__(256) dc_build_kernel(const DcMat* mats, const DcMerge* merges) {
  const DcMerge mg = merges[blockIdx.y];
  const DcMat& mt = mats[mg.mat];
  const int m = mg.hi - mg.lo, n = mt.n;
  const int lane = threadIdx.x & 31;
  const int p = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (p >= m) return;
  const int k = mt.iscr[(int64_t)I_K * n + mg.lo];
  const int src = mt.iscr[(int64_t)I_INV * n + mg.lo + p];
  float* row = mt.UT + (int64_t)(mg.lo + p) * mt.ld + mg.lo;
  const bool packed = m > DENSE_MAX;          // coefficients over the packed non-deflated columns only (dc_pack_kernel)
  const int width = packed ? ((k + 31) & ~31) : m;
  for (int c = lane; c < width; c += 32) row[c] = 0.f;
  __syncwarp();
  if (lane == 0) mt.fscr[(int64_t)F_DTMP * n + mg.lo + p] = mt.fscr[(int64_t)F_VALS * n + mg.lo + src];
  if (src >= k) {
    if (lane == 0 && !packed) row[mt.iscr[(int64_t)I_DFCOL * n + mg.lo + src - k]] = 1.f;
    return;
  }
  const float* dl = mt.fscr + (int64_t)F_DL * n + mg.lo;
  const float* zh = mt.fscr + (int64_t)F_ZHAT * n + mg.lo;
  const int* ndcol = mt.iscr + (int64_t)(packed ? I_CPOS : I_NDCOL) * n + mg.lo;
  const float muj = mt.fscr[(int64_t)F_MU * n + mg.lo + src];
  const float dlo = dl[mt.iscr[(int64_t)I_ORIG * n + mg.lo + src]];
  float ss = 0.f;
  for (int i = lane; i < k; i += 32) {
    const float x = zh[i] / ((dl[i] - dlo) - muj);
    ss = fmaf(x, x, ss);
  }
  const float inv = 1.f / sqrtf(warp_sum(ss));
  for (int i = lane; i < k; i += 32) row[ndcol[i]] = zh[i] / ((dl[i] - dlo) - muj) * inv;
}

__global__ void dc_copy_d_kernel(const DcMat* mats, const DcMerge* merges) {
  const DcMerge mg = merges[blockIdx.y];
  const DcMat& mt = mats[mg.mat];
  const int m = mg.hi - mg.lo;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < m) mt.d[mg.lo + i] = mt.fscr[(int64_t)F_DTMP * mt.n + mg.lo + i];
}

// ------------------------------------------------------------------ host plan
struct Node { int a, b, depth; };   // leaf-index range

struct Plan {
  std::vector<DcCut> cuts;
  std::vector<DcLeaf> leaves;
  std::vector<std::vector<DcMerge>> levels;   // levels[l-1] = merges of level l
  std::vector<int> result_buf;
};

static void build_tree(int mat, int n, int a, int b, int depth, std::vector<std::pair<Node, int>>& internal,
                       std::vector<std::pair<Node, int>>& leafs, int& maxdepth) {
  maxdepth = std::max(maxdepth, depth);
  if (b - a == 1) { leafs.push_back({Node{a, b, depth}, mat}); return; }
  internal.push_back({Node{a, b, depth}, mat});
  const int mid = (a + b) / 2;
  build_tree(mat, n, a, mid, depth + 1, internal, leafs, maxdepth);
  build_tree(mat, n, mid, b, depth + 1, internal, leafs, maxdepth);
}

static void make_plan(const int* n, int count, Plan& pl) {
  pl.result_buf.resize(count);
  for (int i = 0; i < count; ++i) {
    const int L = (n[i] + LEAF - 1) / LEAF;
    std::vector<std::pair<Node, int>> internal, leafs;
    int maxdepth = 0;
    build_tree(i, n[i], 0, L, 0, internal, leafs, maxdepth);
    auto pos = [&](int leaf) { return std::min(n[i], leaf * LEAF); };
    for (auto& lf : leafs)
      pl.leaves.push_back(DcLeaf{i, pos(lf.first.a), pos(lf.first.b), (maxdepth - lf.first.depth) & 1});
    for (auto& nd : internal) {
      const int level = maxdepth - nd.first.depth;         // >= 1
      const int mid = (nd.first.a + nd.first.b) / 2;
      if ((int)pl.levels.size() < level) pl.levels.resize(level);
      pl.levels[level - 1].push_back(DcMerge{i, pos(nd.first.a), pos(mid), pos(nd.first.b), (level - 1) & 1});
      pl.cuts.push_back(DcCut{i, pos(mid)});
    }
    pl.result_buf[i] = maxdepth & 1;
  }
}

}  // namespace

size_t stedc_plan_bytes(const int* n, int count) {
  Plan pl;
  make_plan(n, count, pl);
  size_t merges = 0;
  for (auto& l : pl.levels) merges += l.size();
  size_t widest = 1;
  for (auto& l : pl.levels) widest = std::max(widest, l.size());
  return align_up(sizeof(DcCut) * pl.cuts.size() + 256, 256) + align_up(sizeof(DcLeaf) * pl.leaves.size() + 256, 256) +
         align_up(sizeof(DcMerge) * merges + 256 * (pl.levels.size() + 1), 256) + align_up(grouped_gemm_ws_bytes(2 * (int)widest), 256);
}

int launch_stedc(DcMat* h_mats, DcMat* d_mats, int count, void* plan_ws, size_t plan_bytes, int* status, cudaStream_t s,
                 bool q_zeroed, int max_ctas, HostStage* stage) {
  std::vector<int> ns(count);
  for (int i = 0; i < count; ++i) ns[i] = h_mats[i].n;
  Plan pl;
  make_plan(ns.data(), count, pl);
  char* base = (char*)plan_ws;
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off = align_up(off + bytes, 256); return base + o; };
  DcCut* d_cuts = (DcCut*)take(sizeof(DcCut) * std::max<size_t>(1, pl.cuts.size()));
  DcLeaf* d_leaves = (DcLeaf*)take(sizeof(DcLeaf) * std::max<size_t>(1, pl.leaves.size()));
  std::vector<DcMerge*> d_levels;
  for (auto& l : pl.levels) d_levels.push_back((DcMerge*)take(sizeof(DcMerge) * l.size()));
  size_t widest = 1;
  for (auto& l : pl.levels) widest = std::max(widest, l.size());
  const size_t gws_bytes = grouped_gemm_ws_bytes(2 * (int)widest);
  void* gws = take(gws_bytes);
  if (off > plan_bytes) { set_error("stedc: plan workspace too small (%zu < %zu)", plan_bytes, off); return KFAC_ERR_WORKSPACE; }
  {
    int rc;
    if ((rc = send_table(stage, d_cuts, pl.cuts.data(), sizeof(DcCut) * pl.cuts.size(), s))) return rc;
    if ((rc = send_table(stage, d_leaves, pl.leaves.data(), sizeof(DcLeaf) * pl.leaves.size(), s))) return rc;
    for (size_t l = 0; l < pl.levels.size(); ++l)
      if ((rc = send_table(stage, d_levels[l], pl.levels[l].data(), sizeof(DcMerge) * pl.levels[l].size(), s))) return rc;
  }
  // Q buffers: off-diagonal blocks must be zero
  for (int i = 0; i < count && !q_zeroed; ++i) {
    const size_t bytes = (size_t)h_mats[i].n * h_mats[i].ld * sizeof(float);
    KFAC_CUDA(cudaMemsetAsync(h_mats[i].Q[0], 0, bytes, s));
    KFAC_CUDA(cudaMemsetAsync(h_mats[i].Q[1], 0, bytes, s));
  }
  if (!pl.cuts.empty()) {
    dc_cut_kernel<<<ceil_div(pl.cuts.size(), 256), 256, 0, s>>>(d_mats, d_cuts, (int)pl.cuts.size());
    KFAC_LAUNCH_CHECK();
  }
  dc_leaf_kernel<<<ceil_div(pl.leaves.size(), 2), 64, 0, s>>>(d_mats, d_leaves, (int)pl.leaves.size(), status);
  KFAC_LAUNCH_CHECK();
  static bool attr = false;
  if (!attr) {
    KFAC_CUDA(cudaFuncSetAttribute(dc_deflate_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr = true;
  }
  for (size_t l = 0; l < pl.levels.size(); ++l) {
    const auto& lv = pl.levels[l];
    const int nm = (int)lv.size();
    int mmax = 0;
    for (auto& mg : lv) mmax = std::max(mmax, mg.hi - mg.lo);
    const size_t dsmem = (size_t)mmax * 6 * sizeof(float);
    if (dsmem > 200 * 1024) { set_error("stedc: merge of %d rows exceeds the shared-memory sort", mmax); return KFAC_ERR_UNSUPPORTED; }
    dc_deflate_kernel<<<nm, 1024, dsmem, s>>>(d_mats, d_levels[l]);
    KFAC_LAUNCH_CHECK();
    dc_rotate_kernel<<<dim3(ceil_div(mmax, 256), nm), 256, 0, s>>>(d_mats, d_levels[l]);
    KFAC_LAUNCH_CHECK();
    if (mmax > DENSE_MAX) {
      dc_pack_kernel<<<dim3(ceil_div(mmax, 8), nm), 256, 0, s>>>(d_mats, d_levels[l]);
      KFAC_LAUNCH_CHECK();
    }
    dc_secular_kernel<<<dim3(ceil_div(mmax, 8), nm), 256, 0, s>>>(d_mats, d_levels[l]);
    KFAC_LAUNCH_CHECK();
    dc_zhat_kernel<<<dim3(ceil_div(mmax, 8), nm), 256, 0, s>>>(d_mats, d_levels[l]);
    KFAC_LAUNCH_CHECK();
    dc_rank_kernel<<<dim3(ceil_div(mmax, 256), nm), 256, 0, s>>>(d_mats, d_levels[l]);
    KFAC_LAUNCH_CHECK();
    dc_build_kernel<<<dim3(ceil_div(mmax, 8), nm), 256, 0, s>>>(d_mats, d_levels[l]);
    KFAC_LAUNCH_CHECK();
    dc_copy_d_kernel<<<dim3(ceil_div(mmax, 256), nm), 256, 0, s>>>(d_mats, d_levels[l]);
    KFAC_LAUNCH_CHECK();
    // Q_new = Q_old U~ for every merge of the level: ONE grouped wgmma launch.  Every output tile is computed by one
    // CTA over the whole reduction (its k range is read on the device) and added once into the zeroed target block,
    // so the result is the same in every run.
    std::vector<GroupedGemm> gg;
    for (auto& mg : lv) {
      const DcMat& mt = h_mats[mg.mat];
      const int m = mg.hi - mg.lo, n1 = mg.mid - mg.lo;
      const int64_t o = (int64_t)mg.lo * mt.ld + mg.lo;
      GroupedGemm g{};
      g.lda = mt.ld; g.B = mt.UT + o; g.ldb = mt.ld; g.ldd = mt.ld;
      g.N = m; g.K = m; g.alpha = 1.f; g.epi = EPI_NONE; g.splits = 1;
      if (m > DENSE_MAX) {
        // structured: packed non-deflated columns, upper and lower row halves over the k-block ranges written by the
        // deflation kernel (I_KR); deflated eigenvectors are copied afterwards
        KFAC_CUDA(cudaMemset2DAsync(mt.Q[mg.src ^ 1] + o, (size_t)mt.ld * 4, 0, (size_t)m * 4, (size_t)m, s));
        g.mode = 2;
        const int* kr = mt.iscr + (int64_t)I_KR * mt.n + mg.lo;
        g.A = mt.P + o; g.D = mt.Q[mg.src ^ 1] + o; g.M = n1; g.krange = kr;
        gg.push_back(g);
        g.A = mt.P + o + (int64_t)n1 * mt.ld; g.D = mt.Q[mg.src ^ 1] + o + (int64_t)n1 * mt.ld; g.M = m - n1; g.krange = kr + 2;
        gg.push_back(g);
      } else {
        g.A = mt.Q[mg.src] + o; g.D = mt.Q[mg.src ^ 1] + o; g.M = m;
        gg.push_back(g);
      }
    }
    { const int rc = launch_grouped_gemm(gg.data(), (int)gg.size(), gws, gws_bytes, s, max_ctas, stage); if (rc) return rc; }
    if (mmax > DENSE_MAX) {
      dc_copy_deflated_kernel<<<dim3(ceil_div(mmax, 8), nm), 256, 0, s>>>(d_mats, d_levels[l]);
      KFAC_LAUNCH_CHECK();
    }
  }
  for (int i = 0; i < count; ++i) h_mats[i].result_buf = pl.result_buf[i];
  return KFAC_OK;
}

}  // namespace kfac
