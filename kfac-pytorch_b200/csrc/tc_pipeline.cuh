// Warp-specialised persistent wgmma pipeline, parameterised by a Policy that
// says where the operand tiles come from and where the accumulator goes.
//
//   D_tile[128 x 128] = sum_kb A_kb[128 x 32] * B_kb[128 x 32]^T     (fp32-accurate)
//
// every product is the 3-term TF32 split  a*b ~= a_lo*b_hi + a_hi*b_lo + a_hi*b_hi
// accumulated in fp32 registers.  Roles (384 threads = 3 warpgroups, 1 CTA / SM):
//   warp 0       TMA producer : Policy::load() issues cp.async.bulk.tensor into the stage
//   warps 1-3    splitter     : B_lo = x - trunc_tf32(x), smem -> smem, same (swizzled) offsets
//   warps 4-11   two consumer warpgroups, rows 0-63 and 64-127 of the tile.  Per k-step of 8 each thread loads its
//                A fragment from the stage (ldmatrix), forms A_lo in registers with the same formula, and issues
//                3 wgmma m64n128k8 with A from registers and B from shared memory as one commit group (12 per
//                k-block, 3 groups in flight); then the epilogue straight from the accumulator registers ->
//                Policy::store()
// A_lo never goes through shared memory: per k-block the stage is written by TMA (32 KB) and the splitter (16 KB)
// and read by the splitter (16 KB), the fragment loads (2 x 8 KB) and the B operands of the MMAs (2 x 48 KB),
// 176 KB instead of 240 KB with A_lo staged and both A terms read by the MMAs from shared memory.
// 4 smem stages x {A, B_hi, B_lo} x 16 KB = 192 KB; the producer and the splitter run up to 4 k-blocks ahead, so
// the loads of the next tile overlap the epilogue of this one.
// The A fragments (4 k-steps x {hi, lo} x 4 = 32 registers) sit next to the 128 accumulators; setmaxnreg moves
// registers from the producer / splitter warpgroup (40) to the consumers (232), without which ptxas serialises the
// wgmmas.
//
// Bits: every output element is the same sequence of tensor-core operations as with A_lo staged in shared memory
// (same k order, same operand values, same products into the same accumulators), so the results do not change.
//
// Policy requirements:
//   struct Params;                       (passed as __grid_constant__)
//   struct Item;
//   static constexpr uint32_t TX_BYTES;  bytes landed by load() per stage
//   static constexpr int CHUNK;          consecutive items per CTA (lets decode() cache shared state in Item)
//   __device__ static int  total_work(const Params&, int host_total);   effective number of work items
//   __device__ static void reset(Item&);                          called once per role before the loop
//   __device__ static bool decode(const Params&, int w, Item&);   false -> item is skipped; Item persists
//                                                                 across calls (may cache)
//   __device__ static int  num_kb(const Params&, const Item&);    > 0
//   __device__ static void load(const Params&, const Item&, int kbi, uint8_t* a, uint8_t* b, uint64_t* bar);
//   struct Out;                          what the epilogue needs of an item, in registers
//   __device__ static Out  out(const Params&, const Item&);       once per item, before its 64 store() calls: a
//                                                                 policy whose item lives in global memory copies
//                                                                 it here, or every store() would reload it
//   __device__ static void store(const Params&, const Out&, int row, int col, float (&v)[2]);   columns col, col + 1
#pragma once
#include "tc_common.cuh"

namespace kfac {
namespace tc {

constexpr int PBM = 128, PBN = 128, PBK = 32, PSTAGES = 4;
constexpr int PTILE = PBM * PBK * 4;       // 16 KB slot
constexpr int PSTAGE = 3 * PTILE;          // 48 KB: A, B_hi, B_lo
constexpr int PTHREADS = 384;
constexpr int PSPLIT_THREADS = 96;         // warps 1-3
constexpr int PREG_PRODUCER = 40, PREG_CONSUMER = 232;   // 128 x 40 + 256 x 232 <= 64 K registers
constexpr size_t PSMEM = (size_t)PSTAGES * PSTAGE + 1024 + 256;

// This thread's A fragment of one k-step (8 reduction indices, columns 8 kk .. 8 kk + 7 of the TMA tile) in the
// layout of wgmma_tf32_m64n128k8, by one ldmatrix.x4: each 8 x 16 B matrix is 8 rows x 4 fp32, lane l receives
// word l % 4 of row l / 4 of each.  Matrices: rows +0 / +8 (bit 0 of the lane's octet) x columns +0 / +4 (bit 1).
// a_addr: this lane's row (see the consumer) at k-step 0; the tile has rows of 128 B, SWIZZLE_128B (16-byte chunk
// index xor-ed with the row index mod 8), so k-step kk is the chunk pair 2 kk: address bit 5 flipped by kk.
__device__ __forceinline__ void load_a_frag(uint32_t a_addr, int kk, float (&hi)[4]) {
  uint32_t r[4];
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(a_addr ^ ((uint32_t)kk << 5))
               : "memory");
#pragma unroll
  for (int i = 0; i < 4; ++i) hi[i] = __uint_as_float(r[i]);
}

template <class P>
__global__ void __launch_bounds__(PTHREADS, 1)
pipeline_kernel(const __grid_constant__ typename P::Params p, int total_work) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)PSTAGES * PSTAGE);
  uint64_t* full = bars;
  uint64_t* conv = bars + PSTAGES;
  uint64_t* empty = bars + 2 * PSTAGES;
  constexpr int CH = P::CHUNK;   // consecutive work items handled by one CTA (decode amortisation)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  total_work = P::total_work(p, total_work);   // a policy may shrink the host-side upper bound (device-side work list)
  if (warp == 0 && lane == 0) {
    for (int s = 0; s < PSTAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&conv[s], 3); mbar_init(&empty[s], 8); }
    fence_barrier_init();
  }
  __syncthreads();
  auto tile_ptr = [&](int s, int which) { return smem + (size_t)s * PSTAGE + (size_t)which * PTILE; };

  if (warp == 0) {
    setmaxnreg_dec<PREG_PRODUCER>();
    if (lane == 0) {
      int s = 0; uint32_t ph = 0;
      typename P::Item it;
      P::reset(it);
      for (int wb = blockIdx.x * CH; wb < total_work; wb += gridDim.x * CH)
      for (int w = wb; w < min(wb + CH, total_work); ++w) {
        if (!P::decode(p, w, it)) continue;
        const int nkb = P::num_kb(p, it);
        for (int kbi = 0; kbi < nkb; ++kbi) {
          mbar_wait(&empty[s], ph ^ 1);
          mbar_arrive_expect_tx(&full[s], P::TX_BYTES);
          P::load(p, it, kbi, tile_ptr(s, 0), tile_ptr(s, 1), &full[s]);
          if (++s == PSTAGES) { s = 0; ph ^= 1; }
        }
      }
    }
  } else if (warp < 4) {
    setmaxnreg_dec<PREG_PRODUCER>();
    const int t = threadIdx.x - 32;
    int s = 0; uint32_t ph = 0;
    typename P::Item it;
    P::reset(it);
    for (int wb = blockIdx.x * CH; wb < total_work; wb += gridDim.x * CH)
    for (int w = wb; w < min(wb + CH, total_work); ++w) {
      if (!P::decode(p, w, it)) continue;
      const int nkb = P::num_kb(p, it);
      for (int kbi = 0; kbi < nkb; ++kbi) {
        mbar_wait(&full[s], ph);
        const float4* src = reinterpret_cast<const float4*>(tile_ptr(s, 1));
        float4* dst = reinterpret_cast<float4*>(tile_ptr(s, 2));
#pragma unroll 4
        for (int i = t; i < PTILE / 16; i += PSPLIT_THREADS) {
          const float4 v = src[i];
          float4 lo;
          lo.x = v.x - __uint_as_float(__float_as_uint(v.x) & 0xffffe000u);
          lo.y = v.y - __uint_as_float(__float_as_uint(v.y) & 0xffffe000u);
          lo.z = v.z - __uint_as_float(__float_as_uint(v.z) & 0xffffe000u);
          lo.w = v.w - __uint_as_float(__float_as_uint(v.w) & 0xffffe000u);
          dst[i] = lo;
        }
        fence_proxy_async_smem();   // the generic-proxy stores above are read by wgmma (async proxy)
        __syncwarp();
        if (lane == 0) mbar_arrive(&conv[s]);
        if (++s == PSTAGES) { s = 0; ph ^= 1; }
      }
    }
  } else {
    setmaxnreg_inc<PREG_CONSUMER>();
    const int cw = (warp - 4) >> 2;          // consumer warpgroup: tile rows 64 cw .. 64 cw + 63
    const int wq = warp & 3;                 // warp within the warpgroup: accumulator rows 16 wq ..
    // ldmatrix row address of this lane: matrix j = lane / 8 holds rows 16 wq + 8 (j & 1) .. + 7 and columns
    // 4 (j >> 1) .. + 3 of the k-step
    const int lrow = cw * 64 + wq * 16 + (lane & 7) + 8 * ((lane >> 3) & 1), lchunk = lane >> 4;
    const uint32_t a_lane = (uint32_t)(lrow * 128 + ((lchunk ^ (lrow & 7)) << 4));
    int s = 0; uint32_t ph = 0;
    typename P::Item it;
    P::reset(it);
    float acc[64], cor[64];
    // A fragments, one slot per k-step: each k-step is its own commit group, so the slot of k-step kk is free
    // again once the group of the same k-step of the previous k-block has retired (3 groups stay in flight)
    float hi[4][4], lo[4][4];
    for (int wb = blockIdx.x * CH; wb < total_work; wb += gridDim.x * CH)
    for (int w = wb; w < min(wb + CH, total_work); ++w) {
      if (!P::decode(p, w, it)) continue;
      const int nkb = P::num_kb(p, it);
      int prev = -1;
      for (int kbi = 0; kbi < nkb; ++kbi) {
        mbar_wait(&full[s], ph);             // A landed (read here by ldmatrix)
        mbar_wait(&conv[s], ph);             // B_lo written
        const uint32_t a_addr = smem_u32(tile_ptr(s, 0)) + a_lane;
        const uint64_t bhi = make_kmajor_sw128_desc(smem_u32(tile_ptr(s, 1)));
        const uint64_t blo = make_kmajor_sw128_desc(smem_u32(tile_ptr(s, 2)));
#pragma unroll
        for (int kk = 0; kk < PBK / 8; ++kk) {
          wgmma_wait<3>();                   // k-step kk of the previous k-block has retired
#pragma unroll
          for (int i = 0; i < 4; ++i) { wgmma_hold(hi[kk][i]); wgmma_hold(lo[kk][i]); }
          if (kk == PBK / 8 - 1 && prev >= 0) {   // ... and with it the whole previous k-block: its stage is free
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[prev]);
          }
          load_a_frag(a_addr, kk, hi[kk]);
#pragma unroll
          for (int i = 0; i < 4; ++i) lo[kk][i] = hi[kk][i] - __uint_as_float(__float_as_uint(hi[kk][i]) & 0xffffe000u);
          wgmma_fence();
          // The two small cross terms go to their own accumulator so that the main one sees one
          // accumulate per k-step of 8 (the tensor core's fp32 adds bias long chains otherwise).
          const uint64_t adv = (uint64_t)(kk * 2);   // next 8 reduction indices: 32 B along the row
          const int accum = (kbi > 0 || kk > 0) ? 1 : 0;
          wgmma_tf32_m64n128k8(cor, lo[kk], bhi + adv, accum);
          wgmma_tf32_m64n128k8(cor, hi[kk], blo + adv, 1);
          wgmma_tf32_m64n128k8(acc, hi[kk], bhi + adv, accum);
          wgmma_commit();
        }
        prev = s;
        if (++s == PSTAGES) { s = 0; ph ^= 1; }
      }
      wgmma_wait<0>();
#pragma unroll
      for (int kk = 0; kk < PBK / 8; ++kk)
#pragma unroll
        for (int i = 0; i < 4; ++i) { wgmma_hold(hi[kk][i]); wgmma_hold(lo[kk][i]); }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[prev]);
      const int r0 = cw * 64 + wq * 16 + (lane >> 2), c0 = 2 * (lane & 3);
      const typename P::Out out = P::out(p, it);
#pragma unroll
      for (int j = 0; j < PBN / 8; ++j) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float v[2] = {acc[4 * j + 2 * h] + cor[4 * j + 2 * h], acc[4 * j + 2 * h + 1] + cor[4 * j + 2 * h + 1]};
          P::store(p, out, r0 + 8 * h, 8 * j + c0, v);
        }
      }
    }
  }
}

}  // namespace tc
}  // namespace kfac
