// Householder tridiagonalisation F = H T H^T of symmetric fp32 matrices (first stage of the direct
// eigensolver, eigh_direct.cuh) as ONE persistent kernel: a matrix is worked on by a group of CTAs
// that meet at two group barriers per column.
//
// Blocked formulation (LAPACK ssytrd/slatrd): inside a panel of TRD_NB columns the trailing matrix is
// NOT updated; the effective matrix is A - V W^T - W V^T with the panel's Householder vectors V and
// w-vectors W.  Per column s (x = effective column s below the diagonal):
//   phase C   beta, tau, v from x (every CTA redundantly; x and |x|^2 partials were published before)
//   phase A   symmetric product with the panel-start matrix: only the lower-triangle 64 x 64 tiles
//             (I >= J) are read -- tile (I,J) yields a partial of y_I (rows) and of y_J (columns) --
//             plus the per-CTA partials of W^T v, V^T v and v^T A v            -> group barrier 1
//   phase B   row owners: y = A v - V (W^T v) - W (V^T v), w = tau y - tau^2/2 (y^T v) v, then the next
//             effective column x' = A[:, s+1] - V W[s+1,:]^T - W V[s+1,:]^T and |x'|^2 partials -> barrier 2
// After TRD_NB columns the lower tiles get the rank-2*NB update A -= V W^T + W V^T (fp32 SIMT: the
// tensor core's 3xTF32 accumulate would cost the tridiagonal ~1e-5 of accuracy) -> one more barrier.
// The matrix (<= 42 MB of lower tiles at n = 4608) fits the 50 MB L2 of an H100; algorithmic traffic
// is 2/3 n^3 * 4 bytes of L2 reads for the products.  Everything is deterministic (no atomics on data).
#include "eigh_direct.cuh"

namespace kfac {

namespace {

constexpr int NB = TRD_NB, T = TRD_T;
constexpr int UPAD = T + 4;                 // row length of the transposed update staging
constexpr int SUB_STAGE = 4 * NB * UPAD;    // floats per sub-group: VI^T, WI^T, VJ^T, WJ^T as [NB][UPAD]

__device__ __forceinline__ unsigned ld_acquire(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

__device__ __forceinline__ void group_barrier(unsigned* bar, unsigned& epoch, int ncta) {
  __syncthreads();
  if (ncta > 1) {
    if (threadIdx.x == 0) {
      // release-increment / acquire-poll: bar.sync made the CTA's writes visible to this thread (cta scope),
      // the gpu-scope release is cumulative; no separate MEMBARs on the critical path
      epoch += 1;
      asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(bar) : "memory");
      const unsigned target = epoch * (unsigned)ncta;
      while (ld_acquire(bar) < target) {}
    }
    __syncthreads();
  }
}

__device__ __forceinline__ void sub_sync(int sg) {          // 4 sub-groups of 256 threads (tile update)
  asm volatile("bar.sync %0, %1;" ::"r"(sg + 9), "r"(256) : "memory");
}
__device__ __forceinline__ void sub_sync8(int sg8) {        // 8 sub-groups of 128 threads (symmetric product)
  asm volatile("bar.sync %0, %1;" ::"r"(sg8 + 1), "r"(128) : "memory");
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// L2 eviction-priority hints for the lower tiles of A (TrdMat::pin_j0).  The loads are __ldcg with a cache policy
// operand; the values loaded and stored are the same as without it.
__device__ __forceinline__ uint64_t l2_policy(bool pinned, bool stream_first) {
  uint64_t p;
  if (pinned) asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  else if (stream_first) asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  else asm("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ float4 ldcg_hint(const float4* ptr, uint64_t pol) {
  float4 r;
  asm("ld.global.cg.L2::cache_hint.v4.f32 {%0, %1, %2, %3}, [%4], %5;"
      : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(ptr), "l"(pol));
  return r;
}
__device__ __forceinline__ float ldcg_hint(const float* ptr, uint64_t pol) {
  float r;
  asm("ld.global.cg.L2::cache_hint.f32 %0, [%1], %2;" : "=f"(r) : "l"(ptr), "l"(pol));
  return r;
}
__device__ __forceinline__ void st_hint(float4* ptr, float4 v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.v4.f32 [%0], {%1, %2, %3, %4}, %5;"
               ::"l"(ptr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w), "l"(pol) : "memory");
}
// back to the normal priority: the 128-byte line at ptr (a pinned line must not outlive the tridiagonalisation)
__device__ __forceinline__ void l2_unpin(const float* ptr) {
  asm volatile("applypriority.global.L2::evict_normal [%0], 128;" ::"l"(ptr) : "memory");
}

// optional phase timing (CTA 0, thread 0 of every group accumulates clock64 deltas): set by kfac_stage_sytrd_profile,
// which also records %globaltimer at the start and end of every job (on the job's first CTA, at TrdJob::id)
__device__ unsigned long long g_trd_prof[16];
__device__ int g_trd_prof_on = 0;
constexpr int MAX_TIMED_JOBS = 512;
__device__ unsigned long long g_trd_jobtime[2 * MAX_TIMED_JOBS];
__device__ __forceinline__ unsigned long long globaltimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
#define TRD_STAMP(i) do { if (prof) { const long long t__ = clock64(); if (tid == 0) atomicAdd(&g_trd_prof[i], (unsigned long long)(t__ - tprev)); tprev = t__; } } while (0)

constexpr int MAXT = 256;                   // owned tiles per sub-group (list in shared memory)
constexpr int NCP = 5;                      // ceil(max CTAs per group / 32)

__device__ __forceinline__ float sum5(const float (&x)[NCP]) { return ((x[0] + x[1]) + (x[2] + x[3])) + x[4]; }

// sums of 8 per-lane values over the warp with 9 shuffles: afterwards every lane holds the complete sum
// of value number bit2 | bit3 << 1 | bit4 << 2 of its lane index
__device__ __forceinline__ float reduce8(float (&r)[8], int lane) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float keep = (lane & 16) ? r[i + 4] : r[i], send = (lane & 16) ? r[i] : r[i + 4];
    r[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const float keep = (lane & 8) ? r[i + 2] : r[i], send = (lane & 8) ? r[i] : r[i + 2];
    r[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
  }
  {
    const float keep = (lane & 4) ? r[1] : r[0], send = (lane & 4) ? r[0] : r[1];
    r[0] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
  }
  r[0] += __shfl_xor_sync(0xffffffffu, r[0], 2);
  r[0] += __shfl_xor_sync(0xffffffffu, r[0], 1);
  return r[0];
}

// sums of 8 per-lane values over each 16-lane half of the warp with 8 shuffles: afterwards every lane holds the sum
// (over its half) of value number (lane >> 1) & 7 bit-reversed, i.e. ((lane >> 3) & 1) * 4 + ((lane >> 2) & 1) * 2 + ((lane >> 1) & 1)
__device__ __forceinline__ float reduce8h(float (&r)[8], int lane) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float keep = (lane & 8) ? r[i + 4] : r[i], send = (lane & 8) ? r[i] : r[i + 4];
    r[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const float keep = (lane & 4) ? r[i + 2] : r[i], send = (lane & 4) ? r[i] : r[i + 2];
    r[i] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
  }
  {
    const float keep = (lane & 2) ? r[1] : r[0], send = (lane & 2) ? r[0] : r[1];
    r[0] = keep + __shfl_xor_sync(0xffffffffu, send, 2);
  }
  r[0] += __shfl_xor_sync(0xffffffffu, r[0], 1);
  return r[0];
}

// fp32 pairs: sm_90 has no packed fp32 instruction, so each pair is two round-to-nearest FFMA / FMUL
// (the same rounding per element as a packed pair)
__device__ __forceinline__ float2 fma2(float2 a, float2 b, float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
__device__ __forceinline__ float2 mul2(float2 a, float2 b) {
  return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y));
}

// sums of 16 per-lane values over the warp with 16 shuffles: afterwards every lane holds the complete sum of value
// number (lane >> 1) & 15
__device__ __forceinline__ float reduce16(float (&r)[16], int lane) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float keep = (lane & 16) ? r[i + 8] : r[i], send = (lane & 16) ? r[i] : r[i + 8];
    r[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float keep = (lane & 8) ? r[i + 4] : r[i], send = (lane & 8) ? r[i] : r[i + 4];
    r[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const float keep = (lane & 4) ? r[i + 2] : r[i], send = (lane & 4) ? r[i] : r[i + 2];
    r[i] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
  }
  {
    const float keep = (lane & 2) ? r[1] : r[0], send = (lane & 2) ? r[0] : r[1];
    r[0] = keep + __shfl_xor_sync(0xffffffffu, send, 2);
  }
  r[0] += __shfl_xor_sync(0xffffffffu, r[0], 1);
  return r[0];
}

// One column costs two dependent L2 round trips and two group barriers: every phase first ISSUES all its global
// loads (they are mutually independent), then computes.  cpart is stored transposed ([scalar][cta]) so that the
// cross-CTA reductions read contiguous lines.
__device__ void tridiagonalise(const TrdMat& mt, int cta, int ncta, float* smem) {
  const int n = mt.n, np = mt.np, nblk = mt.nblk;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int sg = warp >> 3;                          // update sub-group (256 threads)
  const int G = ncta * 4, sgid = cta * 4 + sg;       // tile owners of the rank-2NB update
  const int sg8 = warp >> 2, sw4 = warp & 3;         // product sub-group (128 threads) and warp within it
  const int G8 = ncta * 8, sgid8 = cta * 8 + sg8;    // tile owners of the symmetric product
  const int GW = ncta * 32, gw = cta * 32 + warp;    // row owners: rows r = gw (mod GW)
  float* stage = smem;                               // 4 * SUB_STAGE (update staging / column partial sums)
  float* red = stage + 4 * SUB_STAGE;                // 32 x 66
  float* sc = red + 32 * 66;                         // 160 scalars: [0,32) p1, [32,64) p2, 64 vAv, 66.. misc, [96,128) vrow, [128,160) wrow
  short2* tlist = reinterpret_cast<short2*>(sc + 160) + sg * MAXT;
  short2* tlist8 = reinterpret_cast<short2*>(sc + 160) + 4 * MAXT + sg8 * MAXT;
  __shared__ int s_ntile[12];
  unsigned epoch = 0;
  float* const col = mt.col;
  float* const cpart = mt.cpart;
  const float* __restrict__ A = mt.A;
  const int pin_j0 = mt.pin_j0;
  const bool sfirst = mt.stream_first != 0;

  if (n == 1) {
    if (cta == 0 && tid == 0) { mt.d[0] = mt.A[0]; mt.tau[0] = 0.f; mt.e[0] = 0.f; }
    return;
  }
  // static tile ownership.  Tiles are numbered by decreasing column block J (t = 0: (nblk-1, nblk-1); then the two
  // tiles of column nblk-2; ...) and dealt round-robin to the sub-groups: the tiles still active at step s
  // (J >= b0) are a PREFIX of that numbering, so every sub-group holds the same number of active tiles (+-1) at every
  // step, and its list needs no scan for dead entries.
  auto build_list = [&](short2* list, int first, int stride) {
    const int tiles = nblk * (nblk + 1) / 2;
    int cnt = 0;
    for (int t = first; t < tiles && cnt < MAXT; t += stride) {
      int j = (int)((sqrtf(8.f * (float)t + 1.f) - 1.f) * 0.5f);
      while ((j + 1) * (j + 2) / 2 <= t) ++j;
      while (j * (j + 1) / 2 > t) --j;
      const int J = nblk - 1 - j, I = J + (t - j * (j + 1) / 2);
      list[cnt++] = make_short2((short)I, (short)J);
    }
    return cnt;
  };
  if ((tid & 255) == 0) s_ntile[sg] = build_list(tlist, sgid, G);
  if ((tid & 127) == 0) s_ntile[4 + sg8] = build_list(tlist8, sgid8, G8);
  __syncthreads();
  const int ntile = s_ntile[sg], ntile8 = s_ntile[4 + sg8];

  // ---- column 0: x = A[1:, 0], |x[1:]|^2 partials, d[0]
  {
    float sig = 0.f;
    for (int r = gw; r < n; r += GW) {
      if (r >= 1 && lane == 0) {
        const float x = __ldcg(&A[(int64_t)r * np]);
        col[r] = x;
        if (r >= 2) sig = fmaf(x, x, sig);
      }
    }
    if (lane == 0) red[warp] = sig;
    __syncthreads();
    if (warp == 0) {
      const float t = warp_sum(red[lane]);
      if (lane == 0) { cpart[65 * ncta + cta] = t; if (cta == 0) mt.d[0] = __ldcg(&A[0]); }
    }
  }
  group_barrier(mt.bar, epoch, ncta);

  int P = 0;                                         // columns in the current panel
  const bool prof = g_trd_prof_on != 0 && cta == 0;
  long long tprev = prof ? clock64() : 0;
  // Vector work is organised in ROW BLOCKS of 32 consecutive rows; block k belongs to CTA (k mod ncta) and its rows
  // are spread over the CTA's 32 warps (warp w takes row 32 k + w).  Code paths without work are skipped by
  // WARP-UNIFORM branches (the kernel is instruction-issue bound, not bandwidth bound).
  const int nrb = (n + 31) / 32;
  float* s_vrow = sc + 96;                           // 32: V[s+1][:]
  float* s_wrow = sc + 128;                          // 32: W[s+1][:]
  const int vt_per = (n + ncta - 1) / ncta, vt_a = cta * vt_per, vt_b = min(n, vt_a + vt_per);
  constexpr int BP = 4;                              // row blocks per pass
  int kfirst = cta;                                  // first owned row block that still has an active row
  for (int s = 0; s <= n - 2; ++s) {
    const int s1 = s + 1;
    const int b0 = s1 / T, rb_first = s1 / 32;
    while (kfirst < rb_first) kfirst += ncta;
    // =========================================================== phase C: Householder scalars (warp 0)
    if (warp == 0) {
      float sgp[NCP];
#pragma unroll
      for (int j = 0; j < NCP; ++j) { const int c = lane + 32 * j; sgp[j] = c < ncta ? __ldcg(&cpart[65 * ncta + c]) : 0.f; }
      const float alpha = __ldcg(&col[s1]);
      const float sigma = warp_sum(sum5(sgp));
      if (lane == 0) {
        float beta, tau, scal;
        if (sigma == 0.f) { beta = alpha; tau = 0.f; scal = 0.f; }
        else {
          beta = -copysignf(sqrtf(fmaf(alpha, alpha, sigma)), alpha);
          tau = (beta - alpha) / beta;
          scal = 1.f / (alpha - beta);
        }
        sc[66] = tau; sc[67] = scal;
        if (cta == 0) { mt.e[s] = beta; mt.tau[s] = tau; }
      }
    }
    __syncthreads();
    TRD_STAMP(0);      // phase C (scalars)
    // =========================================================== rank-2NB update of the lower tiles
    if (P == NB) {                                     // (every CTA has published its panel column: see phase C)
      const int ub0 = b0;
      float* st = stage + sg * SUB_STAGE;
      float* VIt = st, *WIt = st + NB * UPAD, *VJt = st + 2 * NB * UPAD, *WJt = st + 3 * NB * UPAD;
      const int st_tid = tid & 255;
      for (int ti = 0; ti < ntile; ++ti) {
        const int I = tlist[ti].x, J = tlist[ti].y;
        if (J < ub0) break;                          // uniform within the sub-group: the active tiles are a prefix
        sub_sync(sg);
        // stage the four 64 x NB operand blocks transposed ([k][row])
#pragma unroll
        for (int it = 0; it < 2; ++it) {
          const int idx = st_tid + it * 256;          // 0..511: row = idx / 8, k4 = idx % 8
          const int row = idx >> 3, k4 = (idx & 7) * 4;
          const float4 vi = __ldcg(reinterpret_cast<const float4*>(&mt.Vp[(int64_t)(I * T + row) * NB + k4]));
          const float4 wi = __ldcg(reinterpret_cast<const float4*>(&mt.Wp[(int64_t)(I * T + row) * NB + k4]));
          const float4 vj = __ldcg(reinterpret_cast<const float4*>(&mt.Vp[(int64_t)(J * T + row) * NB + k4]));
          const float4 wj = __ldcg(reinterpret_cast<const float4*>(&mt.Wp[(int64_t)(J * T + row) * NB + k4]));
          VIt[(k4 + 0) * UPAD + row] = vi.x; VIt[(k4 + 1) * UPAD + row] = vi.y; VIt[(k4 + 2) * UPAD + row] = vi.z; VIt[(k4 + 3) * UPAD + row] = vi.w;
          WIt[(k4 + 0) * UPAD + row] = wi.x; WIt[(k4 + 1) * UPAD + row] = wi.y; WIt[(k4 + 2) * UPAD + row] = wi.z; WIt[(k4 + 3) * UPAD + row] = wi.w;
          VJt[(k4 + 0) * UPAD + row] = vj.x; VJt[(k4 + 1) * UPAD + row] = vj.y; VJt[(k4 + 2) * UPAD + row] = vj.z; VJt[(k4 + 3) * UPAD + row] = vj.w;
          WJt[(k4 + 0) * UPAD + row] = wj.x; WJt[(k4 + 1) * UPAD + row] = wj.y; WJt[(k4 + 2) * UPAD + row] = wj.z; WJt[(k4 + 3) * UPAD + row] = wj.w;
        }
        sub_sync(sg);
        const int tx = st_tid & 15, ty = st_tid >> 4;
        float2 acc[4][2];                              // 4 x 4 outputs as fp32 pairs
#pragma unroll
        for (int i = 0; i < 4; ++i) { acc[i][0] = make_float2(0.f, 0.f); acc[i][1] = make_float2(0.f, 0.f); }
#pragma unroll 8
        for (int k = 0; k < NB; ++k) {
          const float4 a1 = *reinterpret_cast<const float4*>(&VIt[k * UPAD + ty * 4]);
          const float4 b1 = *reinterpret_cast<const float4*>(&WJt[k * UPAD + tx * 4]);
          const float4 a2 = *reinterpret_cast<const float4*>(&WIt[k * UPAD + ty * 4]);
          const float4 b2 = *reinterpret_cast<const float4*>(&VJt[k * UPAD + tx * 4]);
          const float av1[4] = {a1.x, a1.y, a1.z, a1.w}, av2[4] = {a2.x, a2.y, a2.z, a2.w};
          const float2 b1lo = make_float2(b1.x, b1.y), b1hi = make_float2(b1.z, b1.w);
          const float2 b2lo = make_float2(b2.x, b2.y), b2hi = make_float2(b2.z, b2.w);
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float2 d1 = make_float2(av1[i], av1[i]), d2 = make_float2(av2[i], av2[i]);
            acc[i][0] = fma2(d1, b1lo, fma2(d2, b2lo, acc[i][0]));
            acc[i][1] = fma2(d1, b1hi, fma2(d2, b2hi, acc[i][1]));
          }
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          float4* p = reinterpret_cast<float4*>(&mt.A[(int64_t)(I * T + ty * 4 + i) * np + J * T + tx * 4]);
          const uint64_t pol = l2_policy(J >= pin_j0, sfirst);
          float4 a = ldcg_hint(p, pol);
          a.x -= acc[i][0].x; a.y -= acc[i][0].y; a.z -= acc[i][1].x; a.w -= acc[i][1].y;
          st_hint(p, a, pol);
        }
      }
      P = 0;
      TRD_STAMP(8);    // rank-2NB update
      group_barrier(mt.bar, epoch, ncta);
      TRD_STAMP(9);    // barrier 3
    }
    const float tau = sc[66], scal = sc[67];
    // v[r] = 0 (r <= s), 1 (r = s + 1), x[r] * scal (r > s + 1): x is read straight from `col`
#define TRD_RAW(r) (((r) > s1 && (r) < n) ? __ldcg(col + (r)) : 0.f)
#define TRD_VFIX(r, raw) ((r) == s1 ? 1.f : (raw) * scal)
    // =========================================================== phase A
    // the Householder vector is kept for the back-transformation (each CTA writes a slice of the row)
    if (vt_a + tid < vt_b) {
      float* vt = mt.VT + (int64_t)s * mt.ldv;
      float* vb = mt.Vb ? mt.Vb + (int64_t)(s / TRD_BT) * np * TRD_BT + (s % TRD_BT) : nullptr;
      for (int r = vt_a + tid; r < vt_b; r += TRD_THREADS) {
        const float raw = TRD_RAW(r);
        const float v = TRD_VFIX(r, raw);
        vt[r] = v;
        if (vb) vb[(int64_t)r * TRD_BT] = v;
      }
    }
    // symmetric product with the lower tiles of this sub-group (128 threads: a warp takes 16 rows of the tile; its lower
    // half-warp rows 0..7, the upper one rows 8..15; a lane holds 4 adjacent columns of 8 rows).  The phase is bound by
    // issue slots, not by bandwidth: 128-bit loads, fp32 pairs and half-warp reductions keep the count down.
    float vav = 0.f;
    {
      float* cs = stage + sg8 * (4 * T);             // column partial sums: [4 warps][64]
      const int st_tid = tid & 127;
      const int hl = lane & 15, h8 = (lane >> 4) * 8;
      if (s1 % T == 0 && b0 - 1 >= pin_j0) {         // block column b0 - 1 has left the active set: unpin its lines
        for (int ti = 0; ti < ntile8; ++ti) {
          const int I = tlist8[ti].x, J = tlist8[ti].y;
          if (J < b0 - 1) break;
          if (J == b0 - 1) l2_unpin(A + (int64_t)(I * T + (st_tid >> 1)) * np + J * T + (st_tid & 1) * 32);
        }
      }
      for (int ti = 0; ti < ntile8; ++ti) {
        const int I = tlist8[ti].x, J = tlist8[ti].y;
        if (J < b0) break;                           // the active tiles are a prefix of the list
        const int rb = I * T + sw4 * 16 + h8, c0 = J * T + 4 * hl;
        const float* ap = A + (int64_t)rb * np + c0;
        float4 a[8];
        const uint64_t pol = l2_policy(J >= pin_j0, sfirst);
#pragma unroll
        for (int k = 0; k < 8; ++k) a[k] = ldcg_hint(reinterpret_cast<const float4*>(ap + (int64_t)k * np), pol);
        const float4 rj = __ldcg(reinterpret_cast<const float4*>(col + c0));     // col has np >= c0 + 4 entries
        const int ri_r = rb + (lane & 7);
        const float ri = TRD_RAW(ri_r);
        float2 vj01, vj23;
        vj01.x = (c0 > s1 && c0 < n) ? rj.x * scal : (c0 == s1 ? 1.f : 0.f);
        vj01.y = (c0 + 1 > s1 && c0 + 1 < n) ? rj.y * scal : (c0 + 1 == s1 ? 1.f : 0.f);
        vj23.x = (c0 + 2 > s1 && c0 + 2 < n) ? rj.z * scal : (c0 + 2 == s1 ? 1.f : 0.f);
        vj23.y = (c0 + 3 > s1 && c0 + 3 < n) ? rj.w * scal : (c0 + 3 == s1 ? 1.f : 0.f);
        const float vi_l = TRD_VFIX(ri_r, ri);
        float rs[8];
        float2 c01 = make_float2(0.f, 0.f), c23 = make_float2(0.f, 0.f);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const float vi = __shfl_sync(0xffffffffu, vi_l, (lane & 16) + k);
          const float2 vi2 = make_float2(vi, vi);
          const float2 a01 = make_float2(a[k].x, a[k].y), a23 = make_float2(a[k].z, a[k].w);
          const float2 t = fma2(a23, vj23, mul2(a01, vj01));
          rs[k] = t.x + t.y;
          c01 = fma2(a01, vi2, c01);
          c23 = fma2(a23, vi2, c23);
        }
        const float tot = reduce8h(rs, lane);
        const int rid = ((lane >> 3) & 1) * 4 + ((lane >> 2) & 1) * 2 + ((lane >> 1) & 1);
        const float vi_r = __shfl_sync(0xffffffffu, vi_l, (lane & 16) + rid);
        if ((lane & 1) == 0) {
          mt.part[(int64_t)J * np + rb + rid] = tot;
          const float t = tot * vi_r;
          vav += (I == J) ? t : 2.f * t;
        }
        if (I != J) {
          c01.x += __shfl_xor_sync(0xffffffffu, c01.x, 16);
          c01.y += __shfl_xor_sync(0xffffffffu, c01.y, 16);
          c23.x += __shfl_xor_sync(0xffffffffu, c23.x, 16);
          c23.y += __shfl_xor_sync(0xffffffffu, c23.y, 16);
          sub_sync8(sg8);                            // previous tile's readers are done with cs
          if (lane < 16) *reinterpret_cast<float4*>(&cs[sw4 * T + 4 * hl]) = make_float4(c01.x, c01.y, c23.x, c23.y);
          sub_sync8(sg8);
          if (st_tid < T) {
            const float t = (cs[st_tid] + cs[T + st_tid]) + (cs[2 * T + st_tid] + cs[3 * T + st_tid]);
            mt.part[(int64_t)I * np + J * T + st_tid] = t;
          }
        }
      }
    }
    TRD_STAMP(1);      // VT write + tile products
    // per-CTA partials of p1 = W^T v, p2 = V^T v: warp w takes row 32 k + w of every owned block (lane = panel column)
    float p1 = 0.f, p2 = 0.f;
    if (P > 0) {
      for (int kp = kfirst; kp < nrb; kp += BP * ncta) {
        float raw[BP], wv[BP], vv[BP];
#pragma unroll
        for (int q = 0; q < BP; ++q) {               // loads of up to BP blocks first ...
          const int k = kp + q * ncta, r = k * 32 + warp;
          raw[q] = 0.f; wv[q] = 0.f; vv[q] = 0.f;
          if (k < nrb && r >= s1 && r < n) {         // warp-uniform
            raw[q] = TRD_RAW(r);
            if (lane < P) { wv[q] = __ldcg(mt.Wp + r * NB + lane); vv[q] = __ldcg(mt.Vp + r * NB + lane); }
          }
        }
#pragma unroll
        for (int q = 0; q < BP; ++q) {               // ... then their use
          const float v = TRD_VFIX((kp + q * ncta) * 32 + warp, raw[q]);
          p1 = fmaf(wv[q], v, p1);
          p2 = fmaf(vv[q], v, p2);
        }
      }
    }
    vav = warp_sum(vav);
    red[warp * 66 + lane] = p1;
    red[warp * 66 + 32 + lane] = p2;
    if (lane == 0) red[warp * 66 + 64] = vav;
    __syncthreads();
    if (tid < 65) {
      float t = 0.f;
#pragma unroll 8
      for (int w = 0; w < 32; ++w) t += red[w * 66 + tid];
      cpart[tid * ncta + cta] = t;
    }
    TRD_STAMP(2);      // dots + CTA reduction
    group_barrier(mt.bar, epoch, ncta);
    TRD_STAMP(3);      // barrier 1
    // =========================================================== phase B
    {
      // ---- every global load of the phase is issued before any of them is used (they are mutually independent);
      // blocks / tile classes without work are skipped by uniform branches
      float* Gs = stage;                               // [BP][32 warps][33]
      float g[BP], vr[BP], wr[BP], ac[BP], rw[BP];
      int kpass = kfirst;
      // own rows (written by this CTA or before the last barrier): may be loaded before the barrier completes
      auto load_rows = [&](int kp) {
#pragma unroll
        for (int q = 0; q < BP; ++q) {
          const int k = kp + q * ncta;
          vr[q] = 0.f; wr[q] = 0.f; ac[q] = 0.f; rw[q] = 0.f;
          const int r = k * 32 + warp;                 // finish: warp = row, lane = panel column
          if (k < nrb && r >= s1 && r < n) {           // uniform
            if (lane < P) { vr[q] = __ldcg(mt.Vp + r * NB + lane); wr[q] = __ldcg(mt.Wp + r * NB + lane); }
            if (r > s1) ac[q] = ldcg_hint(A + (int64_t)r * np + s1, l2_policy(b0 >= pin_j0, sfirst));
            rw[q] = TRD_RAW(r);
          }
        }
      };
      // tile partials of the other CTAs: only after the barrier
      auto load_gather = [&](int kp) {
#pragma unroll
        for (int q = 0; q < BP; ++q) {
          const int k = kp + q * ncta;
          g[q] = 0.f;
          const int rl = k * 32 + lane;                // gather: lane = row, warp = tile class
          if (k < nrb && rl < n) {
            const float* pp = mt.part + (int64_t)(b0 + warp) * np + rl;
            float g0 = 0.f, g1 = 0.f, g2 = 0.f;
            if (b0 + warp < nblk) g0 = __ldcg(pp);
            if (b0 + warp + 32 < nblk) g1 = __ldcg(pp + (int64_t)32 * np);
            if (b0 + warp + 64 < nblk) g2 = __ldcg(pp + (int64_t)64 * np);
            float gx = 0.f;                            // more than 96 active tile classes: n > 6144 only
            for (int X = b0 + warp + 96; X < nblk; X += 32) gx += __ldcg(mt.part + (int64_t)X * np + rl);
            g[q] = ((g0 + g1) + g2) + gx;
          }
        }
      };
      load_rows(kpass);
      load_gather(kpass);
      // cross-CTA sums of p1, p2, vAv: warp w owns outputs w (p1), 32 + w (p2) and (warp 0) 64
      {
        float sa = 0.f, sb = 0.f, scv = 0.f;
        if (warp < P) {
          float ca[NCP], cb[NCP];
#pragma unroll
          for (int j = 0; j < NCP; ++j) {
            const int c = lane + 32 * j;
            ca[j] = c < ncta ? __ldcg(&cpart[warp * ncta + c]) : 0.f;
            cb[j] = c < ncta ? __ldcg(&cpart[(32 + warp) * ncta + c]) : 0.f;
          }
          sa = sum5(ca); sb = sum5(cb);
        }
        if (warp == 0) {
          float cc[NCP];
#pragma unroll
          for (int j = 0; j < NCP; ++j) { const int c = lane + 32 * j; cc[j] = c < ncta ? __ldcg(&cpart[64 * ncta + c]) : 0.f; }
          scv = sum5(cc);
        }
        // row s+1 (warp 1): raw loads now, the rest after the sums are published
        float y1p = 0.f, vrow = 0.f, wrow = 0.f, a11 = 0.f;
        if (warp == 1) {
#pragma unroll
          for (int j = 0; j < 3; ++j) { const int X = b0 + lane + 32 * j; if (X < nblk) y1p += __ldcg(&mt.part[(int64_t)X * np + s1]); }
          for (int X = b0 + lane + 96; X < nblk; X += 32) y1p += __ldcg(&mt.part[(int64_t)X * np + s1]);    // n > 6144
          if (lane < P) { vrow = __ldcg(mt.Vp + s1 * NB + lane); wrow = __ldcg(mt.Wp + s1 * NB + lane); }
          a11 = ldcg_hint(&A[(int64_t)s1 * np + s1], l2_policy(b0 >= pin_j0, sfirst));
        }
        if (warp < P) { sa = warp_sum(sa); sb = warp_sum(sb); }
        if (warp == 0) scv = warp_sum(scv);
        if (lane == 0) { sc[warp] = sa; sc[32 + warp] = sb; if (warp == 0) sc[64] = scv; }
        __syncthreads();
        if (warp == 1) {
          const float p1l = (lane < P) ? sc[lane] : 0.f, p2l = (lane < P) ? sc[32 + lane] : 0.f;
          const float ytv1 = sc[64] - 2.f * warp_sum(p1l * p2l);
          const float y1 = warp_sum(y1p - (vrow * p1l + wrow * p2l));
          const float w1v = tau * (y1 - 0.5f * tau * ytv1);          // v[s+1] = 1
          if (lane == P) { vrow = 1.f; wrow = w1v; }
          s_vrow[lane] = vrow; s_wrow[lane] = wrow;
          const float dd = warp_sum(vrow * wrow);
          if (lane == 0) { sc[68] = ytv1; sc[69] = w1v; if (cta == 0) mt.d[s1] = a11 - 2.f * dd; }
        }
      }
      TRD_STAMP(4);    // phase B loads, cross-CTA sums, row s+1
      // the gathered partial sums go through shared memory: (warp = tile class, lane = row) -> (lane = class, warp = row)
#pragma unroll
      for (int q = 0; q < BP; ++q) if (kpass + q * ncta < nrb) Gs[(q * 32 + warp) * 33 + lane] = g[q];
      __syncthreads();
      TRD_STAMP(5);    // gather through shared memory
      const float ytv = sc[68], w1 = sc[69];
      const float p1l = (lane < P) ? sc[lane] : 0.f, p2l = (lane < P) ? sc[32 + lane] : 0.f;
      const float vsl = (lane < P) ? s_vrow[lane] : 0.f, wsl = (lane < P) ? s_wrow[lane] : 0.f;
      float sig = 0.f;
      for (; kpass < nrb; kpass += BP * ncta) {
        // warp w finishes row 32 k + w of each block of the pass (lane = panel column): y, w, x' and its norm partial.
        // The 2 x BP lane-partial sums of the pass are reduced together (9 shuffles instead of 2 x BP x 5 dependent ones):
        // afterwards lane 8 q holds y of row q, lane 8 q + 4 its xs.
        float red8[8];
#pragma unroll
        for (int q = 0; q < BP; ++q) {
          const int k = kpass + q * ncta;
          const float gq = (k < nrb) ? Gs[(q * 32 + lane) * 33 + warp] : 0.f;
          red8[2 * q] = gq - (vr[q] * p1l + wr[q] * p2l);
          red8[2 * q + 1] = vr[q] * wsl + wr[q] * vsl;
        }
        const float mine = reduce8(red8, lane);                    // value index bit2 | bit3 << 1 | bit4 << 2 of the lane
#pragma unroll
        for (int q = 0; q < BP; ++q) {
          const float y = __shfl_sync(0xffffffffu, mine, 8 * q), xs = __shfl_sync(0xffffffffu, mine, 8 * q + 4);
          const int k = kpass + q * ncta, r = k * 32 + warp;
          if (k >= nrb || r < s1 || r >= n || lane != 0) continue;
          const float v = TRD_VFIX(r, rw[q]);
          const float w = tau * (y - 0.5f * tau * ytv * v);
          mt.Wp[r * NB + P] = w;
          mt.Vp[r * NB + P] = v;
          if (r > s1) {
            const float x = ac[q] - xs - (v * w1 + w);             // panel column P: V[s+1][P] = 1, W[s+1][P] = w1
            col[r] = x;
            if (r > s1 + 1) sig = fmaf(x, x, sig);
          }
        }
        if (kpass + BP * ncta < nrb) {                   // another pass (small groups only): reload, regather
          __syncthreads();
          load_rows(kpass + BP * ncta);
          load_gather(kpass + BP * ncta);
#pragma unroll
          for (int q = 0; q < BP; ++q) if (kpass + (BP + q) * ncta < nrb) Gs[(q * 32 + warp) * 33 + lane] = g[q];
          __syncthreads();
        }
      }
      sig = warp_sum(sig);
      if (lane == 0) red[warp] = sig;
      __syncthreads();
      if (warp == 0) {
        const float t = warp_sum(red[lane]);
        if (lane == 0) cpart[65 * ncta + cta] = t;
      }
      P += 1;
    }
    TRD_STAMP(6);      // finish rows + norm partial
    group_barrier(mt.bar, epoch, ncta);
    TRD_STAMP(7);      // barrier 2
#undef TRD_RAW
#undef TRD_VFIX
  }
  // the block columns still active at the last column: unpin their lines
  const int b0_last = (n - 1) / T;
  if (max(b0_last, pin_j0) < nblk) {
    const int st_tid = tid & 127;
    for (int ti = 0; ti < ntile8; ++ti) {
      const int I = tlist8[ti].x, J = tlist8[ti].y;
      if (J < max(b0_last, pin_j0)) break;
      l2_unpin(A + (int64_t)(I * T + (st_tid >> 1)) * np + J * T + (st_tid & 1) * 32);
    }
  }
  if (cta == 0 && tid == 0) { mt.e[n - 1] = 0.f; mt.tau[n - 1] = 0.f; }
}

__global__ void __launch_bounds__(TRD_THREADS, 1) sytrd_kernel(const TrdMat* mats, const TrdJob* jobs, int njobs) {
  extern __shared__ __align__(16) float trd_smem[];
  for (int j = 0; j < njobs; ++j) {
    const TrdJob job = jobs[j];
    const int b = (int)blockIdx.x;
    if (b < job.cta0 || b >= job.cta0 + job.ncta) continue;
    const bool stamp = g_trd_prof_on != 0 && b == job.cta0 && threadIdx.x == 0 && job.id >= 0 && job.id < MAX_TIMED_JOBS;
    if (stamp) g_trd_jobtime[2 * job.id] = globaltimer();
    tridiagonalise(mats[job.mat], b - job.cta0, job.ncta, trd_smem);
    __syncthreads();
    if (stamp) g_trd_jobtime[2 * job.id + 1] = globaltimer();
  }
}

size_t trd_smem_bytes(int) {
  return sizeof(float) * ((size_t)4 * SUB_STAGE + 32 * 66 + 160) + sizeof(short2) * 12 * MAXT + 64;
}

}  // namespace

int sytrd_max_grid() { return tc_num_sms(); }

// smallest group that can own all lower tiles of an n x n matrix (tile list of MAXT entries per sub-group)
int sytrd_min_ctas(int n) {
  const int nblk = (n + T - 1) / T, tiles = nblk * (nblk + 1) / 2;
  if (nblk >= MAXT) return 1 << 30;
  int C = 1;
  while (tiles / (4 * C) + nblk + 1 > MAXT) ++C;
  return C;
}

int launch_sytrd(const TrdMat* d_mats, const TrdJob* d_jobs, int njobs, int np_max, int grid, cudaStream_t s) {
  if (njobs <= 0) return KFAC_OK;
  const size_t smem = trd_smem_bytes(np_max);
  if (smem > 227 * 1024) { set_error("sytrd: matrix too large for the shared-memory vector (np = %d)", np_max); return KFAC_ERR_UNSUPPORTED; }
  static size_t attr_set = 0;
  if (smem > attr_set) {
    KFAC_CUDA(cudaFuncSetAttribute(sytrd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_set = smem;
  }
  void* args[] = {(void*)&d_mats, (void*)&d_jobs, (void*)&njobs};
  // cooperative launch: every CTA of the grid is resident (the group barriers spin)
  KFAC_CUDA(cudaLaunchCooperativeKernel((const void*)sytrd_kernel, dim3(grid), dim3(TRD_THREADS), args, smem, s));
  count_launch(1);
  return KFAC_OK;
}

// test hook: switch the phase timers on / read them (cycles summed over the CTA 0 of every group)
int sytrd_profile(int on, unsigned long long* out16) {
  if (out16) KFAC_CUDA(cudaMemcpyFromSymbol(out16, g_trd_prof, sizeof(unsigned long long) * 16));
  unsigned long long zero[16] = {0};
  KFAC_CUDA(cudaMemcpyToSymbol(g_trd_prof, zero, sizeof(zero)));
  KFAC_CUDA(cudaMemcpyToSymbol(g_trd_prof_on, &on, sizeof(int)));
  return KFAC_OK;
}

int sytrd_job_times(unsigned long long* out, int max_jobs) {
  const int m = std::min(max_jobs, MAX_TIMED_JOBS);
  if (out && m > 0) KFAC_CUDA(cudaMemcpyFromSymbol(out, g_trd_jobtime, sizeof(unsigned long long) * 2 * m));
  return KFAC_OK;
}

}  // namespace kfac
