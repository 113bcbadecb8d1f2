// wgmma GEMM engine: D = epilogue(alpha * A B^T), A (M x K) and B (N x K)
// row-major fp32 ("TN", both operands K-major), fp32-equivalent accuracy from a
// 3xTF32 split:  a*b ~= a_hi*b_hi + a_hi*b_lo + a_lo*b_hi  with fp32 register
// accumulation (single-pass TF32 fails the 1e-3 parity bar, SURVEY.md 7.3 H1).
//
// One persistent CTA per SM, warp-specialised (tc_pipeline.cuh):
//   warp 0      TMA producer   (cp.async.bulk.tensor 3-D tiles, SWIZZLE_128B)
//   warps 1-3   splitter       (smem -> smem: B_lo = x - trunc_tf32(x))
//   warps 4-11  two consumer warpgroups (A_hi / A_lo in registers, 12 x wgmma m64n128k8 per k-block
//               each, then the fused epilogue from the accumulator registers -> HBM)
// 4 smem stages x {A, B_hi, B_lo} x 16 KB = 192 KB.
#include "common.cuh"
#include "tc_pipeline.cuh"

namespace kfac {

constexpr int TBM = 128, TBN = 128, TBK = 32;

struct TcParams {
  CUtensorMap tmA, tmB;
  float* D; int64_t ldd;
  int M, N, K, kbatch;
  int tiles_m, tiles_n, splits, upper_only, atomic, accum;
  float alpha;
  int epi; const float* E; int64_t lde; const float* dg; const float* da; float damping;
  const float* pi; int pi_side_m, pi_side_n;
  float* peerD[7]; int npeer;
  int64_t slab_stride;             // != 0: split sp writes to D + sp * slab_stride (plain stores, no atomics)
};

// FACTORED: the instantiation that also takes EPI_DIV_FACTORED (as in the grouped engine)
template <bool FACTORED>
struct GemmPolicy {
  using Params = TcParams;
  struct Item { int m0, n0, kb0, kb1, diag, sp; };
  static constexpr uint32_t TX_BYTES = 2 * tc::PTILE;
  static constexpr int CHUNK = 1;
  __device__ static void reset(Item&) {}
  __device__ static int total_work(const Params&, int t) { return t; }

  __device__ static bool decode(const Params& p, int w, Item& it) {
    const int tile = w / p.splits, sp = w % p.splits;
    int tm, tn;
    if (p.upper_only) {
      int t = tile; tm = 0;
      while (t >= p.tiles_n - tm) { t -= p.tiles_n - tm; ++tm; }
      tn = tm + t;
    } else { tm = tile / p.tiles_n; tn = tile % p.tiles_n; }
    it.m0 = tm * TBM; it.n0 = tn * TBN; it.diag = (tm == tn); it.sp = sp;
    const int kb_total = ((p.K + TBK - 1) / TBK) * p.kbatch;
    const int per = (kb_total + p.splits - 1) / p.splits;
    it.kb0 = sp * per; it.kb1 = min(kb_total, it.kb0 + per);
    return it.kb1 > it.kb0;
  }
  __device__ static int num_kb(const Params&, const Item& it) { return it.kb1 - it.kb0; }
  using Out = Item;                // the parameters are kernel parameters already
  __device__ static Out out(const Params&, const Item& it) { return it; }
  __device__ static void load(const Params& p, const Item& it, int kbi, uint8_t* a, uint8_t* b, uint64_t* bar) {
    const int kblocks = (p.K + TBK - 1) / TBK;
    const int kb = it.kb0 + kbi;
    const int bt = kb / kblocks, kc = (kb % kblocks) * TBK;
    tc::tma_load_3d(a, &p.tmA, bar, kc, it.m0, bt);
    tc::tma_load_3d(b, &p.tmB, bar, kc, it.n0, bt);
  }
  __device__ static void store(const Params& p, const Item& it, int row, int col, float (&v)[2]) {
    const int m = it.m0 + row, nb = it.n0 + col;
    if (m >= p.M || nb >= p.N) return;
    const bool mirror = p.upper_only && !it.diag && p.slab_stride == 0;   // split partials hold the upper tiles only
    float* drow = p.D + (int64_t)it.sp * p.slab_stride + (int64_t)m * p.ldd + nb;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      float x = p.alpha * v[j];
      if (nb + j < p.N) {
        if (p.epi == EPI_MUL) x *= p.E[(int64_t)m * p.lde + nb + j];
        else if (p.epi == EPI_DIV_OUTER) x = x / (p.dg[m] * p.da[nb + j] + p.damping);
        else if (FACTORED && p.epi == EPI_DIV_FACTORED)
          x = div_factored(x, p.dg[m], p.da[nb + j], p.damping, p.pi, p.pi_side_m, p.pi_side_n);
      }
      v[j] = x;
    }
    if (!p.atomic && !mirror && ((uintptr_t)drow & 7) == 0 && (p.ldd & 1) == 0 && nb + 2 <= p.N) {
      if (p.accum) {
        const float2 o = *reinterpret_cast<const float2*>(drow);
        v[0] += o.x; v[1] += o.y;
      }
      *reinterpret_cast<float2*>(drow) = make_float2(v[0], v[1]);
      // fused compute + broadcast: the same tile goes straight to the peers' copies of D
      // (P2P stores over NVLink, overlapped with the MMAs of the next tile)
      for (int q = 0; q < p.npeer; ++q)
        *reinterpret_cast<float2*>(p.peerD[q] + (int64_t)m * p.ldd + nb) = make_float2(v[0], v[1]);
    } else {
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        if (nb + j >= p.N) continue;
        if (p.atomic) {
          atomicAdd(drow + j, v[j]);
          if (mirror) atomicAdd(p.D + (int64_t)(nb + j) * p.ldd + m, v[j]);
        } else {
          drow[j] = p.accum ? drow[j] + v[j] : v[j];
          if (mirror) {
            float* t = p.D + (int64_t)(nb + j) * p.ldd + m;
            *t = p.accum ? *t + v[j] : v[j];
          }
          for (int q = 0; q < p.npeer; ++q) p.peerD[q][(int64_t)m * p.ldd + nb + j] = v[j];
        }
      }
    }
  }
};

// ------------------------------------------------------------------ host
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  }
  return fn;
}

// generic 3-D fp32 map, SWIZZLE_128B: dims {d0, d1, d2}, byte strides of d1/d2, box {32, box_rows, 1}
int make_tmap_3d(CUtensorMap* tm, const float* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t stride1_bytes,
                 uint64_t stride2_bytes, uint32_t box_rows) {
  EncodeTiledFn enc = get_encode();
  if (!enc) { set_error("cuTensorMapEncodeTiled unavailable"); return KFAC_ERR_CUDA; }
  cuuint64_t dims[3] = {d0, d1, d2};
  cuuint64_t strides[2] = {stride1_bytes, stride2_bytes};
  cuuint32_t box[3] = {32, box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, (void*)base, dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed (%d)", (int)r); return KFAC_ERR_CUDA; }
  return KFAC_OK;
}

// 3-D map {K, rows, kbatch} over a row-major fp32 matrix (ld elements) with box {32, 128, 1}
static int make_tmap(CUtensorMap* tm, const float* base, int64_t rows, int64_t K, int64_t ld, int kbatch,
                     int64_t kb_stride) {
  EncodeTiledFn enc = get_encode();
  if (!enc) { set_error("cuTensorMapEncodeTiled unavailable"); return KFAC_ERR_CUDA; }
  cuuint64_t dims[3] = {(cuuint64_t)K, (cuuint64_t)rows, (cuuint64_t)kbatch};
  cuuint64_t strides[2] = {(cuuint64_t)ld * 4, (cuuint64_t)(kbatch > 1 ? kb_stride : ld * rows) * 4};
  cuuint32_t box[3] = {TBK, TBM, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, (void*)base, dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed (%d)", (int)r); return KFAC_ERR_CUDA; }
  return KFAC_OK;
}

int tc_num_sms() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
      n = 132;
  }
  return n;
}

bool tc_gemm_supported(const TcGemmArgs& a) {
  auto al16 = [](const void* p) { return ((uintptr_t)p & 15) == 0; };
  if (!(al16(a.A) && al16(a.B))) return false;
  if ((a.lda & 3) || (a.ldb & 3)) return false;
  if (a.kbatch > 1 && ((a.a_kb_stride & 3) || (a.b_kb_stride & 3))) return false;
  if (a.M < 1 || a.N < 1 || a.K < 1) return false;
  return true;
}

int launch_tc_gemm(const TcGemmArgs& a, cudaStream_t stream) {
  if (!tc_gemm_supported(a)) { set_error("tc_gemm: unsupported alignment/shape"); return KFAC_ERR_UNSUPPORTED; }
  static int num_sms = 0;
  static bool attr = false;
  if (!attr) {
    int dev = 0;
    KFAC_CUDA(cudaGetDevice(&dev));
    KFAC_CUDA(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev));
    KFAC_CUDA(cudaFuncSetAttribute(tc::pipeline_kernel<GemmPolicy<false>>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   (int)tc::PSMEM));
    KFAC_CUDA(cudaFuncSetAttribute(tc::pipeline_kernel<GemmPolicy<true>>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   (int)tc::PSMEM));
    attr = true;
  }
  const int kbatch = a.kbatch > 0 ? a.kbatch : 1;
  TcParams p{};
  int rc;
  if ((rc = make_tmap(&p.tmA, a.A, a.M, a.K, a.lda, kbatch, a.a_kb_stride))) return rc;
  if ((rc = make_tmap(&p.tmB, a.B, a.N, a.K, a.ldb, kbatch, a.b_kb_stride))) return rc;
  p.D = a.D; p.ldd = a.ldd; p.M = a.M; p.N = a.N; p.K = a.K; p.kbatch = kbatch;
  p.tiles_m = ceil_div(a.M, TBM); p.tiles_n = ceil_div(a.N, TBN);
  p.upper_only = a.upper_only; p.atomic = a.atomic; p.alpha = a.alpha; p.accum = a.accumulate;
  if (a.accumulate && (a.atomic || a.npeer > 0 || a.splits > 1)) { set_error("tc_gemm: accumulate needs the plain single-split epilogue"); return KFAC_ERR_BAD_ARG; }
  p.epi = a.epi; p.E = a.E; p.lde = a.lde; p.dg = a.dg; p.da = a.da; p.damping = a.damping;
  p.pi = a.pi; p.pi_side_m = a.pi_side_m; p.pi_side_n = a.pi_side_n;
  p.npeer = a.npeer;
  for (int q = 0; q < a.npeer && q < 7; ++q) p.peerD[q] = a.peerD[q];
  if (a.npeer > 0 && (a.atomic || a.upper_only)) { set_error("tc_gemm: peer stores need the plain-store epilogue"); return KFAC_ERR_BAD_ARG; }
  const int ntiles = a.upper_only ? p.tiles_m * (p.tiles_m + 1) / 2 : p.tiles_m * p.tiles_n;
  const int kb_total = ceil_div(a.K, TBK) * kbatch;
  int splits = a.splits;
  if (splits <= 0) {
    splits = 1;
    if (a.atomic && ntiles < num_sms) splits = std::max(1, std::min(num_sms / ntiles, kb_total / 8));
  }
  splits = tc_normalize_splits(splits, kb_total);
  if (splits > 1 && !a.atomic && !a.slab) { set_error("tc_gemm: split-K needs atomic accumulation or a slab workspace"); return KFAC_ERR_BAD_ARG; }
  if (a.slab && (a.atomic || a.npeer > 0 || a.epi != EPI_NONE || a.accumulate)) { set_error("tc_gemm: slab split-K needs the plain epilogue"); return KFAC_ERR_BAD_ARG; }
  p.splits = splits;
  if (a.slab) { p.D = a.slab; p.slab_stride = a.slab_stride; }
  const int total = ntiles * splits;
  const int grid = std::min(total, num_sms);
  if (p.epi == EPI_DIV_FACTORED) tc::pipeline_kernel<GemmPolicy<true>><<<grid, tc::PTHREADS, tc::PSMEM, stream>>>(p, total);
  else tc::pipeline_kernel<GemmPolicy<false>><<<grid, tc::PTHREADS, tc::PSMEM, stream>>>(p, total);
  KFAC_LAUNCH_CHECK();
  return KFAC_OK;
}

}  // namespace kfac

extern "C" int kfac_gemm_tn_tc(const float* A, int64_t lda, const float* B, int64_t ldb, float* D, int64_t ldd,
                               int M, int N, int K, float alpha, int atomic, int splits, void* stream) {
  using namespace kfac;
  KFAC_CHECK_ARG(A && B && D, "null pointer");
  TcGemmArgs a{};
  a.A = A; a.lda = lda; a.B = B; a.ldb = ldb; a.D = D; a.ldd = ldd;
  a.M = M; a.N = N; a.K = K; a.kbatch = 1; a.alpha = alpha; a.atomic = atomic; a.splits = splits;
  return launch_tc_gemm(a, (cudaStream_t)stream);
}
