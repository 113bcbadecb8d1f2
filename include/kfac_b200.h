/*
 * kfac_b200.h -- C ABI of the H100-native (sm_90a) K-FAC hot path (libkfac_b200.so).
 *
 * The reference (gpauloski/kfac-pytorch v0.4.2) has no FFI: its hot path is a
 * chain of torch calls inside Python classes.  This header is the boundary a
 * maintainer would bind (ctypes stub in INTEGRATION.md) to replace exactly
 * those call sites; each entry point cites the reference lines it replaces.
 *
 * Conventions
 *   - plain pointers + sizes only; every pointer is a DEVICE pointer unless
 *     stated otherwise; all matrices are dense row-major fp32 unless a dtype
 *     code is given (0 = f32, 1 = f16, 2 = bf16).
 *   - the library never allocates user-visible memory: workspaces are sized by
 *     the *_workspace_bytes() queries and passed in by the caller.
 *   - `stream` is a cudaStream_t passed as void*.  Calls are asynchronous.
 *   - return value: 0 = ok, <0 = kfac_status; kfac_last_error() (thread-local)
 *     gives the message.  No C++ exceptions cross this boundary.
 *   - arrays of item structs are HOST arrays (read during the call only).
 */
#ifndef KFAC_B200_H_
#define KFAC_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum kfac_status {
  KFAC_OK = 0,
  KFAC_ERR_BAD_ARG = -1,
  KFAC_ERR_NOT_READY = -2,
  KFAC_ERR_CUDA = -3,
  KFAC_ERR_WORKSPACE = -4,
  KFAC_ERR_NO_CONVERGE = -5,
  KFAC_ERR_UNSUPPORTED = -6
};

enum kfac_dtype { KFAC_F32 = 0, KFAC_F16 = 1, KFAC_BF16 = 2 };
enum kfac_method { KFAC_EIGEN = 1, KFAC_INVERSE = 2 }; /* kfac/enums.py ComputeMethod */

int kfac_version(void);
const char* kfac_last_error(void);
/* compute capability of the current device (e.g. 100) or <0 */
int kfac_device_arch(void);
/* cumulative number of CUDA kernels this library has launched in the process */
long long kfac_launch_count(void);

/* ---------------------------------------------------------------- factors
 * K3: second-moment statistics, accumulated into `acc` (d x d, fp32):
 *         acc += scale * X^T X
 * `scale` folds 1/rows (utils.py:51-55), the conv 1/spatial^2
 * (modules.py:175-177,188-190) and the AMP 1/grad_scale^2 (base.py:365-366).
 */

/* replaces LinearModuleHelper.get_a_factor / get_g_factor
 * (kfac/layers/modules.py:123-141) + append_bias_ones (utils.py:8-15):
 * x is (rows, features) row-major; d = features + append_ones. */
/* ws may be NULL (SIMT kernel).  With a workspace of kfac_factor_linear_workspace_bytes()
 * tall inputs (rows >= 512, features >= 128) are transposed once into a feature-major matrix
 * and the SYRK runs on the wgmma engine; the workspace also holds the per-split partials of a
 * reduction split over the SMs.  Every factor call is deterministic (partials are added in a
 * fixed order; without a workspace the reduction runs unsplit). */
size_t kfac_factor_linear_workspace_bytes(int64_t rows, int features, int append_ones);
int kfac_factor_linear(const void* x, int dtype, int64_t rows, int features,
                       int append_ones, float scale, float* acc, void* ws,
                       size_t ws_bytes, void* stream);

/* replaces Conv2dModuleHelper._extract_patches + get_a_factor
 * (kfac/layers/modules.py:170-178,210-237).  x is NCHW; feature order
 * (C, kh, kw) [+ ones]; d = C*kh*kw + append_ones. */
size_t kfac_factor_conv2d_input_workspace_bytes(int batch, int C, int H, int W,
                                                int kh, int kw, int sh, int sw,
                                                int ph, int pw, int append_ones);
int kfac_factor_conv2d_input(const void* x, int dtype, int batch, int C, int H,
                             int W, int kh, int kw, int sh, int sw, int ph,
                             int pw, int append_ones, float scale, float* acc,
                             void* ws, size_t ws_bytes, void* stream);

/* replaces Conv2dModuleHelper.get_g_factor (modules.py:180-192):
 * g is (batch, C, Ho, Wo); acc (C x C) += scale * sum_n Y_n Y_n^T.
 * ws (optional, kfac_factor_conv2d_gradout_workspace_bytes): maps whose rows are not
 * 16-byte multiples (7 x 7) are packed there for the tensor-core SYRK; without it they
 * take the SIMT kernel. */
size_t kfac_factor_conv2d_gradout_workspace_bytes(int batch, int C, int Ho, int Wo);
int kfac_factor_conv2d_gradout(const void* g, int dtype, int batch, int C,
                               int Ho, int Wo, float scale, float* acc,
                               void* ws, size_t ws_bytes, void* stream);

/* K4: replaces KFACBaseLayer.update_{a,g}_factor (layers/base.py:375-405) and
 * the symmetrisation of get_cov (utils.py:57):
 *   factor = alpha*(first ? I : factor)
 *          + (1-alpha)*inv_count*0.5*(batch + batch^T);   batch = 0 */
typedef struct kfac_ema_item {
  float* factor; /* d x d running average */
  float* batch;  /* d x d micro-batch sum (consumed, zeroed) */
  int d;
  int first;       /* 1: seed with identity */
  float inv_count; /* 1 / number of accumulated micro-batches */
} kfac_ema_item;
int kfac_factor_ema(const kfac_ema_item* items, int count, float alpha,
                    void* stream);

/* ------------------------------------------------------- eigendecomposition
 * K5: replaces torch.linalg.eigh + clamp(min=0) in
 * KFACEigenLayer.compute_{a,g}_inv (kfac/layers/eigen.py:295-344).
 * F (n x n, symmetric PSD) -> Q (n x n row-major, COLUMNS are eigenvectors,
 * same convention as torch.linalg.eigh) and d (n eigenvalues >= 0, in the
 * order of Q's columns: ascending for n > 128, unsorted for n <= 128).
 * All matrices of the batch are solved concurrently:
 *   n <= 128  two-sided Jacobi, the whole matrix in the shared memory of one CTA;
 *   n  > 128  Householder tridiagonalisation (one persistent kernel for the batch, CTA groups per
 *             matrix) -> divide and conquer on the tridiagonal matrix -> block-reflector
 *             back-transformation (grouped wgmma GEMMs) -- the stages of LAPACK's ssyevd. */
typedef struct kfac_eigh_item {
  const float* F; /* n x n dense (ld = n) */
  float* Q;       /* n x n, leading dimension ldq */
  float* QT;      /* optional transposed copy (rows are eigenvectors), ld = ldq; may be NULL */
  float* d;
  int n;
  int ldq;        /* 0 -> n.  Multiples of 4 let the tensor-core GEMMs consume Q directly */
  const float* V0T; /* ignored (warm start of the round-1 iterative solver; kept for ABI compatibility) */
} kfac_eigh_item;
#define KFAC_EIGH_MAX_N 8192   /* largest factor dimension (KFAC_ERR_UNSUPPORTED beyond) */
size_t kfac_eigh_workspace_bytes(const int* n, int count);
/* max_sweeps <= 0 -> default (24 sweeps of the n <= 128 Jacobi); tol is ignored.
 * The first int of the workspace is a device status word written by the call (0 = fine, bit 0 = an
 * iteration did not converge, bit 1 = a non-finite (or |x| > 1e15) factor entry, replaced by 0, or a non-finite eigenvalue): fetch it with kfac_eigh_status(). */
int kfac_eigh_batched(const kfac_eigh_item* items, int count, void* ws,
                      size_t ws_bytes, int max_sweeps, float tol, void* stream);
/* asynchronous copy of the status word of the last kfac_eigh_batched() on this workspace into
 * (pinned) host memory; valid once `stream` has passed this point.  torch.linalg.eigh raises in
 * these cases (eigen.py:310); the caller maps a non-zero word to KFAC_ERR_NO_CONVERGE. */
int kfac_eigh_status(const void* ws, int* host_status, void* stream);

/* K6: replaces eigen.py:345-348: out[i,j] = 1 / (dg[i]*da[j] + damping) */
int kfac_dgda(const float* dg, const float* da, int g, int a, float damping,
              float* out, int ld_out, void* stream);

/* K7: replaces KFACInverseLayer.compute_{a,g}_inv (kfac/layers/inverse.py:
 * 186-213): inv = (F + damping I)^-1, formed as Q diag(1/(d+damping)) Q^T from
 * the eigendecomposition of F (F is symmetric PSD). ws: n*ldq floats. */
int kfac_inverse_from_eigh(const float* Q, int ldq, const float* d, int n,
                           float damping, float* inv, int ld_inv, void* ws,
                           size_t ws_bytes, void* stream);
/* dst (cols x rows, ld_dst) = src^T (src rows x cols, ld_src): gives a rank that
 * received an eigenbasis by broadcast the K-major copy the GEMM engine wants */
int kfac_transpose(const float* src, int ld_src, float* dst, int ld_dst, int rows,
                   int cols, void* stream);

/* ---------------------------------------------------------- precondition
 * K8/K9/K10: replaces ModuleHelper.get_grad (modules.py:56-69,194-208) and
 * KFAC{Eigen,Inverse}Layer.preconditioned_grad (eigen.py:350-385,
 * inverse.py:215-234).  grad matrix = [wgrad viewed (g, a-1|a), bgrad].
 *   EIGEN  : P = Qg [ (Qg^T grad Qa) * dgda ] Qa^T     (dgda != NULL)
 *            P = Qg [ (Qg^T grad Qa) / (dg x da + damping) ] Qa^T  (else)
 *   INVERSE: P = Ginv grad Ainv */
typedef struct kfac_precond_item {
  const void* wgrad; /* (g, a - has_bias) */
  const void* bgrad; /* (g) or NULL */
  int grad_dtype;
  int g, a; /* a includes the bias column when bgrad != NULL */
  const float* qa;   /* a x a (ld = ldqa), columns are eigenvectors */
  const float* qaT;  /* its transpose (ld = ldqa) */
  const float* qg;   /* g x g (ld = ldqg) */
  const float* qgT;
  const float* dgda; /* g x a (ld = ld_dgda) or NULL */
  const float* da;
  const float* dg;
  const float* a_inv; /* a x a (ld = ldqa), symmetric */
  const float* g_inv; /* g x g (ld = ldqg), symmetric */
  int ldqa, ldqg, ld_dgda;
  float* P; /* out: g x a fp32 (ld = ldp) */
  int ldp;
  /* fused compute + broadcast (replaces KFACBaseLayer.broadcast_grad, layers/base.py:224-252):
   * HOST array of n_peers (<= 7) device pointers -- the same P entry inside the peer ranks'
   * P arenas, mapped with kfac_peer_open().  The epilogue of the last GEMM stores every tile
   * to P and to all peers (P2P over NVLink).  n_peers = 0: local only. */
  float* const* peer_P;
  int n_peers;
} kfac_precond_item;
size_t kfac_precondition_workspace_bytes(const kfac_precond_item* items, int count);
int kfac_precondition(const kfac_precond_item* items, int count, int method,
                      float damping, void* ws, size_t ws_bytes, void* stream);

/* K11: replaces BaseKFACPreconditioner._compute_grad_scale
 * (kfac/base_preconditioner.py:411-435) without host syncs:
 *   vg = sum_layers sum(P * grad) * lr^2 ;  nu = vg==0 ? 1 : min(1, sqrt(kl_clip/|vg|))
 * K12: replaces KFACBaseLayer.update_grad + ModuleHelper.set_grad
 * (layers/base.py:407-423, modules.py:87-97): grad <- nu * P, written IN PLACE
 * into the existing weight/bias .grad storage (the reference rebinds .grad). */
typedef struct kfac_grad_item {
  const float* P;
  void* wgrad;
  void* bgrad;
  int grad_dtype;
  int g, a;
  int ldp; /* leading dimension of P */
} kfac_grad_item;
/* Both calls run as ONE launch over all layers and are bitwise reproducible (fixed assignment of elements
 * to threads, fixed-order reduction; no floating-point atomics): every data-parallel replica that
 * preconditions locally gets the same nu.  ws: device workspace of kfac_grad_workspace_bytes(count) bytes
 * (item table + partial sums); scale_out: device float[1] (nu). */
size_t kfac_grad_workspace_bytes(int count);
int kfac_grad_scale(const kfac_grad_item* items, int count, float kl_clip,
                    float lr, void* ws, size_t ws_bytes, float* scale_out, void* stream);
/* scale may be NULL (no clipping: scale = 1) */
int kfac_grad_update(const kfac_grad_item* items, int count, const float* scale,
                     void* ws, size_t ws_bytes, void* stream);

/* ---------------------------------------------------------- peer memory
 * Buffers that other ranks of the node write into directly (CUDA IPC over NVLink).
 * kfac_peer_alloc: cudaMalloc + zero + export a 64-byte IPC handle (caller-owned: free with
 * kfac_peer_free).  kfac_peer_open maps a handle exported by ANOTHER process. */
int kfac_peer_alloc(size_t bytes, void** dev_ptr, void* handle64);
int kfac_peer_open(const void* handle64, void** dev_ptr);
int kfac_peer_close(void* dev_ptr);
int kfac_peer_free(void* dev_ptr);

/* ---------------------------------------------------- communication helpers
 * replaces get_triu / fill_triu (kfac/distributed.py:422-465): pack the upper
 * triangle (row-major order of torch.triu_indices) and mirror it back. */
int kfac_triu_pack(const float* F, int n, float* packed, void* stream);
int kfac_triu_unpack(const float* packed, int n, float* F, void* stream);
/* buf *= s (the 1/world averaging of distributed.py:239-241,369) */
int kfac_scale_inplace(float* buf, int64_t count, float s, void* stream);

/* ----------------------------------------------------------- dense GEMM
 * C = alpha * op(A) op(B) + beta * C, fp32 row-major with explicit element
 * strides (A(m,k) at A[m*sa_m + k*sa_k], B(k,n) at B[k*sb_k + n*sb_n]).
 * Exposed for tests / profiling of the GEMM engine used by K3/K5/K8. */
int kfac_gemm_f32(const float* A, int64_t sa_m, int64_t sa_k, const float* B,
                  int64_t sb_k, int64_t sb_n, float* C, int64_t ldc, int M,
                  int N, int K, float alpha, float beta, void* stream);

/* Tensor-core engine (wgmma / TMA, 3xTF32 split, fp32 accumulate in registers):
 * D (+)= alpha * A B^T with A (M x K) and B (N x K) row-major fp32, lda/ldb
 * multiples of 4 and 16-byte aligned bases.  atomic != 0: accumulate into D
 * with split-K (`splits` <= 0: automatic).  Exposed for tests / profiling. */
int kfac_gemm_tn_tc(const float* A, int64_t lda, const float* B, int64_t ldb,
                    float* D, int64_t ldd, int M, int N, int K, float alpha,
                    int atomic, int splits, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* KFAC_B200_H_ */
