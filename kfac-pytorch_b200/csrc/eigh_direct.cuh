// Direct (non-iterative) symmetric eigensolver for the large factors (n > 128):
//   1. sytrd.cu   Householder tridiagonalisation  F = H T H^T   (persistent multi-CTA kernel, fp32 SIMT,
//                 lower-triangle 64x64 tiles resident in L2, two group barriers per column)
//   2. stedc.cu   divide and conquer on T (Cuppen / Gu-Eisenstat): leaf solves in shared memory,
//                 rank-one merges = deflation + secular equation + one wgmma GEMM per merge
//   3. eigh_direct.cu  back-transformation Q = H Z with compact-WY block reflectors (wgmma GEMMs)
// Replaces torch.linalg.eigh of kfac/layers/eigen.py:310,331 (LAPACK ssyevd = the same three stages).
#pragma once
#include "common.cuh"
#include "gemm_grouped.cuh"

namespace kfac {

constexpr int TRD_NB = 32;        // panel width (columns per block reflector of the reduction)
constexpr int TRD_T = 64;         // tile edge of the lower-triangle tiling
constexpr int TRD_THREADS = 1024; // 4 sub-groups of 8 warps
constexpr int TRD_BT = 256;       // Householder vectors per block reflector of the back-transformation
constexpr int TRD_CP = 72;        // floats of per-CTA partial scalars: [0,32) W^T v, [32,64) V^T v, 64 v^T A v, 65 |x|^2

struct TrdMat {
  float* A;        // np x np working copy of F (zero padded); only tiles I >= J are kept up to date
  float* VT;       // n x ldv: row j = Householder vector v_j (v_j[j+1] = 1, zero for r <= j)
  float* Vb;       // optional: the same vectors as row-major blocks, block kb = reflectors [kb*TRD_BT, ..): Vb[kb*np*TRD_BT + r*TRD_BT + i]
  float* tau;      // n
  float* d;        // n     diagonal of T
  float* e;        // n     sub-diagonal of T (e[j] couples j, j+1)
  float* Vp;       // np x TRD_NB panel of Householder vectors
  float* Wp;       // np x TRD_NB panel of w vectors
  float* part;     // nblk x np partial products of the symmetric matrix-vector product
  float* col;      // np  effective next column
  float* cpart;    // 66 x ncta per-CTA partial scalars, transposed [scalar][cta]
  unsigned int* bar;  // group barrier counter (zeroed before launch)
  int n, np, nblk, ldv;
};

struct TrdJob { int mat, cta0, ncta; };

// all jobs of one launch; a CTA processes the jobs that contain it in list order
int launch_sytrd(const TrdMat* d_mats, const TrdJob* d_jobs, int njobs, int np_max, int grid, cudaStream_t s);
int sytrd_max_grid();
int sytrd_min_ctas(int n);

// ---- divide and conquer (stedc.cu)
struct DcMat {
  float* d;        // n   in: diagonal of T, out: eigenvalues (ascending)
  float* e;        // n   sub-diagonal (destroyed)
  float* Q[2];     // n x ld ping-pong eigenvector matrices (columns = eigenvectors); result in Q[result_buf]
  float* UT;       // n x ld workspace (rows = coefficient vectors of the merged eigenvectors)
  float* P;        // n x ld workspace (non-deflated columns of Q_old, packed by type, for the large merges)
  float* fscr;     // 10 n floats of scratch
  int* iscr;       // 12 n ints of scratch
  int n, ld;
  int result_buf;
};

struct DcPlanHost;   // opaque (stedc.cu)
// workspace bytes for the plan tables (merge lists, leaf descriptors) of a batch
size_t stedc_plan_bytes(const int* n, int count);   // includes the grouped-GEMM tables
// eigen-decomposition of `count` tridiagonal matrices; d_mats/h_mats describe them (device pointers inside);
// plan_ws: device scratch of stedc_plan_bytes(); all work is enqueued on `s`
// status: device int, bit 0 is set when a leaf QL iteration did not converge
// q_zeroed: the caller has already zeroed Q[0] and Q[1] of every matrix
int launch_stedc(DcMat* h_mats, DcMat* d_mats, int count, void* plan_ws, size_t plan_bytes, int* status, cudaStream_t s,
                 bool q_zeroed = false);

// plain fp32 TN GEMM on the wgmma engine: D = alpha * A B^T (+ D when accumulate)
int gemm_tn_plain(const float* A, int64_t lda, const float* B, int64_t ldb, float* D, int64_t ldd, int M, int N,
                  int K, cudaStream_t s);
// a few side streams for independent small launches (per-merge / per-matrix GEMM chains)
struct StreamPool {
  static constexpr int N = 4;
  cudaStream_t st[N];
  cudaEvent_t ev_fork, ev_join[N];
  bool ready = false;
  int init();
  int fork(cudaStream_t s);     // side streams wait for everything enqueued on s so far
  int join(cudaStream_t s);     // s waits for everything enqueued on the side streams
};
StreamPool& stream_pool();

size_t eigh_direct_workspace_bytes(const int* n, int count);
// status: device int (bit 0: an iteration did not converge, bit 1: non-finite eigenvalue); may be nullptr
int eigh_direct_run(const kfac_eigh_item* items, int count, void* ws, size_t ws_bytes, int* status, cudaStream_t s);
int gemm_tn_acc(const float* A, int64_t lda, const float* B, int64_t ldb, float* D, int64_t ldd, int M, int N,
                int K, float alpha, cudaStream_t s);

}  // namespace kfac
