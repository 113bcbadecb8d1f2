// The diagonal A factor of an nn.EmbeddingBag layer (kfac_factor_embedding_bag): s_v = sum_b c_bv^2 over the pooled
// rows c_b of the bags, then acc[v] += alpha * s_v.
//
//   prepare   one thread per entry i: its bag (a binary search in the offsets, or i / L for 2-D indices), its sort key
//             (the token, or V for an entry equal to padding_idx) and, for the mean, the non-padding
//             count L_b of its bag (integer atomics)
//   sort      CUB's stable radix sort of (key, i) on the key: each token's entries end up contiguous, in entry order,
//             and so in bag order
//   pairs     one thread per (token, bag) pair, at its first sorted position: c_bv summed in fp64 in entry order and
//             squared, stored at that position (0 at the pair's other positions)
//   sums      one thread per token run: the run's stored squares added in position (= bag) order in fp64, rounded once
//             to s_v.  A frequent token's run is long; its walk reads one contiguous fp64 array
//   add       acc[v] = fl(acc[v] + fl(alpha * s_v)), the rounding of kfac_factor_embedding's scale-and-add
//
// No floating-point atomics and a fixed order everywhere: the same bits on every run.  Nothing is read back to the
// host.
#include "common.cuh"

#include <cub/device/device_radix_sort.cuh>

namespace kfac {
namespace {

inline int grid_for(int64_t total) {
  const int64_t b = (total + 255) / 256;
  return (int)max((int64_t)1, min(b, (int64_t)tc_num_sms() * 16));
}

// the bits of a key in [0, V]: the sentinel V must sort after every token
inline int key_bits(int V) {
  int bits = 1;
  while (bits < 32 && ((unsigned)V >> bits) != 0) ++bits;
  return bits;
}

struct BagWs {
  unsigned* keys_in; unsigned* keys_out;
  int* vals_in; int* vals_out;
  int* bag;         // the bag of entry i (-1: none)
  int* len;         // B non-padding counts (mean)
  double* sq;       // N: c_bv^2 at the first position of each (token, bag) pair, 0 elsewhere
  float* sums;      // V
  void* sort; size_t sort_bytes;
  size_t total;
};

BagWs carve(char* base, int64_t N, int64_t B, int V) {
  BagWs w{};
  size_t off = 0;
  auto take = [&](size_t bytes) { char* p = base ? base + off : nullptr; off += align_up(bytes, 256); return p; };
  w.keys_in = (unsigned*)take((size_t)N * 4);
  w.keys_out = (unsigned*)take((size_t)N * 4);
  w.vals_in = (int*)take((size_t)N * 4);
  w.vals_out = (int*)take((size_t)N * 4);
  w.bag = (int*)take((size_t)N * 4);
  w.len = (int*)take((size_t)B * 4);
  w.sq = (double*)take((size_t)N * 8);
  w.sums = (float*)take((size_t)V * 4);
  cub::DeviceRadixSort::SortPairs(nullptr, w.sort_bytes, (const unsigned*)nullptr, (unsigned*)nullptr,
                                  (const int*)nullptr, (int*)nullptr, (int)N, 0, key_bits(V));
  w.sort = take(w.sort_bytes);
  w.total = off;
  return w;
}

// the bag of entry i: the last b with offsets[b] <= i among the nsearch offsets (-1 before offsets[0])
template <typename I>
__device__ __forceinline__ int64_t bag_of(const I* __restrict__ offsets, int64_t nsearch, int64_t i) {
  int64_t lo = 0, hi = nsearch;     // the first offset > i lies in [lo, hi]
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if ((int64_t)offsets[mid] <= i) lo = mid + 1;
    else hi = mid;
  }
  return lo - 1;
}

template <typename I>
__global__ void __launch_bounds__(256) bag_prepare_kernel(const I* __restrict__ idx, const I* __restrict__ offsets,
                                                          int64_t N, int64_t B, int64_t L, int64_t padding_idx,
                                                          int mean, int V, BagWs w) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < N; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = offsets ? bag_of(offsets, B, i) : i / L;
    const int64_t t = (int64_t)idx[i];
    const bool in = b >= 0 && t != padding_idx;
    w.keys_in[i] = in ? (unsigned)t : (unsigned)V;
    w.vals_in[i] = (int)i;
    w.bag[i] = (int)b;
    if (in && mean) atomicAdd(w.len + b, 1);
  }
}

// One thread per sorted position; the first position of each (token, bag) pair walks the pair's entries in entry
// order and stores c^2 (c = n / L_b for the mean), every other position stores 0
__global__ void __launch_bounds__(256) bag_pairs_kernel(int64_t N, int V, const void* __restrict__ weights,
                                                        int weight_dtype, int mean, BagWs w) {
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < N; p += (int64_t)gridDim.x * blockDim.x) {
    const unsigned v = w.keys_out[p];
    const int b = w.bag[w.vals_out[p]];
    if (v >= (unsigned)V || (p > 0 && w.keys_out[p - 1] == v && w.bag[w.vals_out[p - 1]] == b)) {
      w.sq[p] = 0.0;
      continue;
    }
    double c = 0.0;
    for (int64_t q = p; q < N && w.keys_out[q] == v; ++q) {
      const int i = w.vals_out[q];
      if (w.bag[i] != b) break;
      c += weights ? (double)load_as_float(weights, weight_dtype, i) : 1.0;
    }
    if (mean) c = c / (double)w.len[b];
    w.sq[p] = c * c;
  }
}

// One thread per sorted position; the first position of each token's run adds the run's squares in position order
__global__ void __launch_bounds__(256) bag_sums_kernel(int64_t N, int V, BagWs w) {
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < N; p += (int64_t)gridDim.x * blockDim.x) {
    const unsigned v = w.keys_out[p];
    if (v >= (unsigned)V || (p > 0 && w.keys_out[p - 1] == v)) continue;
    double s = 0.0;
    for (int64_t q = p; q < N && w.keys_out[q] == v; ++q) s += w.sq[q];
    w.sums[v] = (float)s;
  }
}

__global__ void __launch_bounds__(256) bag_scale_add_kernel(const float* __restrict__ sums, int V, float alpha,
                                                            float* acc) {
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < V; v += gridDim.x * blockDim.x)
    acc[v] = __fadd_rn(acc[v], __fmul_rn(alpha, sums[v]));
}

}  // namespace
}  // namespace kfac

using namespace kfac;

extern "C" size_t kfac_factor_embedding_bag_workspace_bytes(int64_t N, int64_t B, int V) {
  if (N < 0 || N >= (1ll << 31) || B < 0 || B >= (1ll << 31) || V <= 0) return 0;
  return carve(nullptr, N, B, V).total;
}

extern "C" int kfac_factor_embedding_bag(const void* idx, const void* offsets, int index_dtype, int64_t N, int64_t B,
                                         int64_t padding_idx, int mode, const void* weights,
                                         int weight_dtype, int V, float alpha, float* acc, void* ws, size_t ws_bytes,
                                         void* stream) {
  KFAC_CHECK_ARG(acc && V > 0 && N >= 0 && N < (1ll << 31) && B >= 0 && B < (1ll << 31) && (idx || N == 0),
                 "embedding bag factor args");
  KFAC_CHECK_ARG(index_dtype == KFAC_I32 || index_dtype == KFAC_I64, "index dtype");
  KFAC_CHECK_ARG(mode == KFAC_BAG_SUM || mode == KFAC_BAG_MEAN, "bag mode");
  KFAC_CHECK_ARG(!weights || mode == KFAC_BAG_SUM, "per-sample weights need KFAC_BAG_SUM");
  KFAC_CHECK_ARG(!weights || weight_dtype == KFAC_F32 || weight_dtype == KFAC_F16 || weight_dtype == KFAC_BF16,
                 "weight dtype");
  KFAC_CHECK_ARG(offsets || (B > 0 ? N % B == 0 : N == 0), "2-D indices: N must be a multiple of B");
  KFAC_CHECK_ARG(padding_idx >= -1 && padding_idx < V, "padding_idx");
  const BagWs need = carve(nullptr, N, B, V);
  if (!ws || ws_bytes < need.total) {
    set_error("factor_embedding_bag: workspace too small (%zu < %zu)", ws_bytes, need.total);
    return KFAC_ERR_WORKSPACE;
  }
  if (N == 0 || B == 0) return KFAC_OK;
  cudaStream_t s = (cudaStream_t)stream;
  BagWs w = carve((char*)ws, N, B, V);
  const int mean = mode == KFAC_BAG_MEAN;
  const int64_t L = offsets ? 0 : N / B;
  if (mean) KFAC_CUDA(cudaMemsetAsync(w.len, 0, (size_t)B * sizeof(int), s));
  KFAC_CUDA(cudaMemsetAsync(w.sums, 0, (size_t)V * sizeof(float), s));
  if (index_dtype == KFAC_I32)
    bag_prepare_kernel<int><<<grid_for(N), 256, 0, s>>>((const int*)idx, (const int*)offsets, N, B, L, padding_idx,
                                                        mean, V, w);
  else
    bag_prepare_kernel<long long><<<grid_for(N), 256, 0, s>>>((const long long*)idx, (const long long*)offsets, N, B,
                                                              L, padding_idx, mean, V, w);
  KFAC_LAUNCH_CHECK();
  size_t sort_bytes = w.sort_bytes;
  KFAC_CUDA(cub::DeviceRadixSort::SortPairs(w.sort, sort_bytes, w.keys_in, w.keys_out, w.vals_in, w.vals_out, (int)N,
                                            0, key_bits(V), s));
  count_launch(1);    // the sort's own launches count as one
  bag_pairs_kernel<<<grid_for(N), 256, 0, s>>>(N, V, weights, weight_dtype, mean, w);
  KFAC_LAUNCH_CHECK();
  bag_sums_kernel<<<grid_for(N), 256, 0, s>>>(N, V, w);
  KFAC_LAUNCH_CHECK();
  bag_scale_add_kernel<<<grid_for(V), 256, 0, s>>>(w.sums, V, alpha, acc);
  KFAC_LAUNCH_CHECK();
  return KFAC_OK;
}
