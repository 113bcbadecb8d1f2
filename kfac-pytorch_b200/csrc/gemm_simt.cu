// fp32 SIMT GEMM engine: the size-class for small / oddly shaped operands
// (factor dims < 128, ragged tails, strided transposes).  Large aligned tiles
// go to the wgmma engine in gemm_tc.cu.
#include "common.cuh"

namespace kfac {

constexpr int BM = 64, BN = 64, BK = 16;

__global__ void __launch_bounds__(256) gemm_simt_kernel(GemmArgs g) {
  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Bs[BK][BN + 4];
  const int tid = threadIdx.x;
  const int bz = blockIdx.z;
  const int b = bz / g.splitk, sk = bz % g.splitk;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  int kchunk = (g.K + g.splitk - 1) / g.splitk;
  kchunk = (kchunk + BK - 1) / BK * BK;
  const int k_begin = sk * kchunk;
  const int k_end = min(g.K, k_begin + kchunk);
  const float* __restrict__ A = g.A + (int64_t)b * g.sa_b;
  const float* __restrict__ B = g.B + (int64_t)b * g.sb_b;
  float* C = g.C + (int64_t)b * g.sc_b;
  const int tx = tid % 16, ty = tid / 16;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  const bool a_m_fast = (g.sa_m == 1);
  const bool b_n_fast = (g.sb_n == 1);

  for (int k0 = k_begin; k0 < k_end; k0 += BK) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      int m, k;
      if (a_m_fast) { m = tid % 64; k = tid / 64 + 4 * i; }
      else          { k = tid % 16; m = tid / 16 + 16 * i; }
      float v = 0.f;
      if (m0 + m < g.M && k0 + k < k_end)
        v = A[(int64_t)(m0 + m) * g.sa_m + (int64_t)(k0 + k) * g.sa_k];
      As[k][m] = v;
      int n;
      if (b_n_fast) { n = tid % 64; k = tid / 64 + 4 * i; }
      else          { k = tid % 16; n = tid / 16 + 16 * i; }
      v = 0.f;
      if (n0 + n < g.N && k0 + k < k_end)
        v = B[(int64_t)(k0 + k) * g.sb_k + (int64_t)(n0 + n) * g.sb_n];
      Bs[k][n] = v;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      const float4 a4 = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      const float4 b4 = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      const float a[4] = {a4.x, a4.y, a4.z, a4.w};
      const float bb[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], bb[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= g.M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= g.N) continue;
      float v = g.alpha * acc[i][j];
      if (g.epi == EPI_MUL) v *= g.E[(int64_t)m * g.lde + n];
      else if (g.epi == EPI_DIV_OUTER) v = v / (g.dg[m] * g.da[n] + g.damping);
      float* c = &C[(int64_t)m * g.ldc + n];
      if (g.atomic) atomicAdd(c, v);
      else *c = (g.beta == 0.f) ? v : (v + g.beta * (*c));
    }
  }
}

int launch_gemm(const GemmArgs& g0, cudaStream_t stream) {
  GemmArgs g = g0;
  if (g.M <= 0 || g.N <= 0) return KFAC_OK;
  if (g.batch <= 0) g.batch = 1;
  if (g.splitk <= 0) g.splitk = 1;
  if (g.splitk > 1 && !g.atomic) {
    set_error("launch_gemm: split-K requires atomic accumulation");
    return KFAC_ERR_BAD_ARG;
  }
  if (g.atomic && g.epi != EPI_NONE) {
    set_error("launch_gemm: epilogue not allowed with atomic accumulation");
    return KFAC_ERR_BAD_ARG;
  }
  dim3 grid(ceil_div(g.N, BN), ceil_div(g.M, BM), g.batch * g.splitk);
  if (grid.z > 65535 || grid.y > 65535) {
    set_error("launch_gemm: grid too large (%u,%u,%u)", grid.x, grid.y, grid.z);
    return KFAC_ERR_BAD_ARG;
  }
  gemm_simt_kernel<<<grid, 256, 0, stream>>>(g);
  KFAC_LAUNCH_CHECK();
  return KFAC_OK;
}

}  // namespace kfac

extern "C" int kfac_gemm_f32(const float* A, int64_t sa_m, int64_t sa_k,
                             const float* B, int64_t sb_k, int64_t sb_n, float* C,
                             int64_t ldc, int M, int N, int K, float alpha,
                             float beta, void* stream) {
  using namespace kfac;
  KFAC_CHECK_ARG(A && B && C, "null pointer");
  KFAC_CHECK_ARG(M >= 0 && N >= 0 && K >= 0, "negative dims");
  GemmArgs g{};
  g.A = A; g.sa_m = sa_m; g.sa_k = sa_k;
  g.B = B; g.sb_k = sb_k; g.sb_n = sb_n;
  g.C = C; g.ldc = ldc;
  g.M = M; g.N = N; g.K = K; g.batch = 1; g.splitk = 1;
  g.alpha = alpha; g.beta = beta;
  return launch_gemm(g, (cudaStream_t)stream);
}
