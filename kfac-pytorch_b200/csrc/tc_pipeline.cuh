// Warp-specialised persistent wgmma pipeline, parameterised by a Policy that
// says where the operand tiles come from and where the accumulator goes.
//
//   D_tile[128 x 128] = sum_kb A_kb[128 x 32] * B_kb[128 x 32]^T     (fp32-accurate)
//
// every product is the 3-term TF32 split  a*b ~= a_lo*b_hi + a_hi*b_lo + a_hi*b_hi
// accumulated in fp32 registers.  Roles (384 threads = 3 warpgroups, 1 CTA / SM):
//   warp 0       TMA producer : Policy::load() issues cp.async.bulk.tensor into the stage
//   warps 1-3    splitter     : lo = x - trunc_tf32(x), smem -> smem, same (swizzled) offsets
//   warps 4-11   two consumer warpgroups, rows 0-63 and 64-127 of the tile: 12 wgmma m64n128k8 per
//                k-block (one k-block in flight while the next is issued), then the epilogue straight
//                from the accumulator registers -> Policy::store()
// 3 smem stages x {A_hi, B_hi, A_lo, B_lo} x 16 KB = 192 KB; the producer and the splitter run up to
// 3 k-blocks ahead, so the loads of the next tile overlap the epilogue of this one.
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
//   __device__ static void store(const Params&, const Item&, int row, int col, float (&v)[2]);   columns col, col + 1
#pragma once
#include "tc_common.cuh"

namespace kfac {
namespace tc {

constexpr int PBM = 128, PBN = 128, PBK = 32, PSTAGES = 3;
constexpr int PTILE = PBM * PBK * 4;       // 16 KB slot
constexpr int PSTAGE = 4 * PTILE;          // 64 KB
constexpr int PTHREADS = 384;
constexpr int PSPLIT_THREADS = 96;         // warps 1-3
constexpr size_t PSMEM = (size_t)PSTAGES * PSTAGE + 1024 + 256;

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
#pragma unroll
        for (int which = 0; which < 2; ++which) {
          const float4* src = reinterpret_cast<const float4*>(tile_ptr(s, which));
          float4* dst = reinterpret_cast<float4*>(tile_ptr(s, which + 2));
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
        }
        fence_proxy_async_smem();   // the generic-proxy stores above are read by wgmma (async proxy)
        __syncwarp();
        if (lane == 0) mbar_arrive(&conv[s]);
        if (++s == PSTAGES) { s = 0; ph ^= 1; }
      }
    }
  } else {
    const int cw = (warp - 4) >> 2;          // consumer warpgroup: tile rows 64 cw .. 64 cw + 63
    const int wq = warp & 3;                 // warp within the warpgroup: accumulator rows 16 wq ..
    const uint32_t a_off = (uint32_t)cw * 64u * 128u;
    int s = 0; uint32_t ph = 0;
    typename P::Item it;
    P::reset(it);
    float acc[64], cor[64];
    for (int wb = blockIdx.x * CH; wb < total_work; wb += gridDim.x * CH)
    for (int w = wb; w < min(wb + CH, total_work); ++w) {
      if (!P::decode(p, w, it)) continue;
      const int nkb = P::num_kb(p, it);
      int prev = -1;
      for (int kbi = 0; kbi < nkb; ++kbi) {
        mbar_wait(&conv[s], ph);
        const uint64_t ahi = make_kmajor_sw128_desc(smem_u32(tile_ptr(s, 0)) + a_off);
        const uint64_t bhi = make_kmajor_sw128_desc(smem_u32(tile_ptr(s, 1)));
        const uint64_t alo = make_kmajor_sw128_desc(smem_u32(tile_ptr(s, 2)) + a_off);
        const uint64_t blo = make_kmajor_sw128_desc(smem_u32(tile_ptr(s, 3)));
        wgmma_fence();
        // The two small cross terms go to their own accumulator so that the main one sees one
        // accumulate per k-step of 8 (the tensor core's fp32 adds bias long chains otherwise).
#pragma unroll
        for (int kk = 0; kk < PBK / 8; ++kk) {
          const uint64_t adv = (uint64_t)(kk * 2);   // next 8 reduction indices: 32 B along the row
          const int accum = (kbi > 0 || kk > 0) ? 1 : 0;
          wgmma_tf32_m64n128k8(cor, alo + adv, bhi + adv, accum);
          wgmma_tf32_m64n128k8(cor, ahi + adv, blo + adv, 1);
          wgmma_tf32_m64n128k8(acc, ahi + adv, bhi + adv, accum);
        }
        wgmma_commit();
        if (prev >= 0) {                     // the previous k-block has retired: its stage is free
          wgmma_wait<1>();
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty[prev]);
        }
        prev = s;
        if (++s == PSTAGES) { s = 0; ph ^= 1; }
      }
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[prev]);
      const int r0 = cw * 64 + wq * 16 + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
      for (int j = 0; j < PBN / 8; ++j) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float v[2] = {acc[4 * j + 2 * h] + cor[4 * j + 2 * h], acc[4 * j + 2 * h + 1] + cor[4 * j + 2 * h + 1]};
          P::store(p, it, r0 + 8 * h, 8 * j + c0, v);
        }
      }
    }
  }
}

}  // namespace tc
}  // namespace kfac
