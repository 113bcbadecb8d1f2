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
 * fixed order; without a workspace the reduction runs unsplit).  rows = 0 adds nothing and
 * launches nothing. */
size_t kfac_factor_linear_workspace_bytes(int64_t rows, int features, int append_ones);
int kfac_factor_linear(const void* x, int dtype, int64_t rows, int features,
                       int append_ones, float scale, float* acc, void* ws,
                       size_t ws_bytes, void* stream);
/* The same statistics on rows with a row stride ld >= features (elements), e.g. a column block
 * of a packed projection's gradient.  ld == features gives the bits of kfac_factor_linear, and a
 * column block the bits of kfac_factor_linear on a contiguous copy of it. */
size_t kfac_factor_linear_strided_workspace_bytes(int64_t rows, int features, int64_t ld,
                                                  int append_ones);
int kfac_factor_linear_strided(const void* x, int dtype, int64_t rows, int features, int64_t ld,
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

/* Geometry of a Conv1d / Conv2d / Conv3d layer's input, every per-axis array in (D, H, W)
 * order: a Conv1d is D = kd = 1, H = kh = 1; the Conv2d entries are D = kd = 1 with dilation 1
 * and symmetric padding.  The output extent of an axis is
 *     (in + pad_before + pad_after - dilation * (kernel - 1) - 1) / stride + 1,
 * and the feature order of A is (C, kd, kh, kw) [+ ones], the order of weight.reshape(out, -1).
 * Padding is zero padding (other padding modes are applied to x by the caller). */
typedef struct kfac_conv_geometry {
  int batch, C;
  int in[3];
  int kernel[3];
  int stride[3];
  int dilation[3];
  int pad_before[3];
  int pad_after[3];
} kfac_conv_geometry;

/* acc (d x d) += scale * X^T X, X the N-d dilated im2col of x (batch, C, D, H, W) in any dtype.
 * The im2col is formed in fp32, feature-major, in chunks of whole examples: the largest chunk
 * whose matrix and SYRK partials fit in ws_bytes (one example with an unsplit SYRK when only
 * its matrix fits), each chunk's SYRK added to acc in chunk order, so a call is deterministic
 * for a given ws_bytes.  The workspace query returns the bytes of the largest chunk whose
 * matrix and SYRK partials together fit in max_bytes, or of one example when even that does
 * not fit.  A kernel of all ones with unit stride and no padding reads x in place (no
 * matrix).  Conv2d: kfac_factor_conv2d_input is this call with one chunk of the whole batch. */
size_t kfac_factor_conv_input_workspace_bytes(const kfac_conv_geometry* geom, int append_ones,
                                              size_t max_bytes);
int kfac_factor_conv_input(const void* x, int dtype, const kfac_conv_geometry* geom,
                           int append_ones, float scale, float* acc, void* ws, size_t ws_bytes,
                           void* stream);

/* Geometry of a ConvTranspose1d / 2d / 3d layer's input (groups = 1) in torch's own parameters, every
 * per-axis array in (D, H, W) order (a 1-d layer is D = kd = 1, H = kh = 1).  The output extent of
 * an axis is
 *     (in - 1) * stride - 2 * padding + dilation * (kernel - 1) + output_padding + 1,
 * and output position o reads input (o + padding - k * dilation) / stride through tap k when stride
 * divides it and the quotient lies in [0, in), zero otherwise.  With the weight (C_in, C_out, k...),
 * A's feature order is (C_in, kd, kh, kw) [+ ones].  Every call refuses with KFAC_ERR_BAD_ARG an
 * empty output, output_padding >= max(stride, dilation), and batch x output positions >= 2^31. */
typedef struct kfac_conv_transpose_geometry {
  int batch, C;
  int in[3];
  int kernel[3];
  int stride[3];
  int dilation[3];
  int padding[3];
  int output_padding[3];
} kfac_conv_transpose_geometry;

/* kfac_factor_conv_input for a transposed geometry: the same chunked fp32 im2col (the taps that
 * fall between inputs are exact zeros) and the same SYRK, chunking and workspace query. */
size_t kfac_factor_conv_transpose_input_workspace_bytes(const kfac_conv_transpose_geometry* geom,
                                                        int append_ones, size_t max_bytes);
int kfac_factor_conv_transpose_input(const void* x, int dtype,
                                     const kfac_conv_transpose_geometry* geom, int append_ones,
                                     float scale, float* acc, void* ws, size_t ws_bytes,
                                     void* stream);

/* replaces Conv2dModuleHelper.get_g_factor (modules.py:180-192):
 * g is (batch, C, Ho, Wo); acc (C x C) += scale * sum_n Y_n Y_n^T.
 * ws (optional, kfac_factor_conv2d_gradout_workspace_bytes): maps whose rows are not
 * 16-byte multiples (7 x 7) are packed there for the tensor-core SYRK; without it they
 * take the SIMT kernel.  Only the plane of S = Ho * Wo elements is used, so the output
 * gradient of a Conv1d (S = Lo) or Conv3d (S = Do * Ho * Wo) layer is passed as (1, S); the
 * same holds for kfac_rows_conv2d_gradout and kfac_reduce_rows_conv2d_gradout. */
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

/* Guarded EMA for mixed-precision training with a dynamic loss scale (replaces the
 * division of the grad-outputs by grad_scaler() in layers/base.py:365-366).
 * loss_scale: HOST array of `count` DEVICE pointers to one float each (NULL array or
 * NULL entry = 1); the window of item i is multiplied by u = (1 / *loss_scale[i])^2 as it
 * is read.  A window with an entry whose unscaled value is not finite or exceeds 1e15 in
 * magnitude (the bound kfac_eigh_batched rejects) is DROPPED: its factor keeps its value
 * (becomes exactly I when `first` = 1), its batch is zeroed and *skipped (device counter,
 * may be NULL) is incremented.  Every other item gets the bits kfac_factor_ema gives on
 * batch * u (on batch itself for a NULL scale).  ws: kfac_factor_ema_guarded_workspace_bytes(count)
 * bytes of device memory (one drop flag per item).  Two launches per 40 items (scan, EMA). */
size_t kfac_factor_ema_guarded_workspace_bytes(int count);
int kfac_factor_ema_guarded(const kfac_ema_item* items, int count, float alpha,
                            const float* const* loss_scale, unsigned long long* skipped,
                            void* ws, size_t ws_bytes, void* stream);

/* Embedding layers (an extension beyond the reference, opt-in): an nn.Embedding is a Linear
 * layer whose input rows are one-hot vectors e_idx, so its A factor is DIAGONAL, the token
 * frequencies.  It is kept as a vector of V floats and never eigendecomposed.
 * kfac_factor_embedding: acc[v] += alpha * count(idx == v) over the N indices (alpha = 1/N).
 * idx: N int32 (index_dtype KFAC_I32) or int64 (KFAC_I64) indices in [0, V); they are trusted
 * (the embedding's forward pass has already checked them).  Deterministic and without a host
 * sync: an integer histogram in ws (kfac_factor_embedding_workspace_bytes(V) bytes), then one
 * fixed-order scale-and-add per entry.  No floating-point atomics. */
enum kfac_index_dtype { KFAC_I32 = 3, KFAC_I64 = 4 };
size_t kfac_factor_embedding_workspace_bytes(int V);
int kfac_factor_embedding(const void* idx, int index_dtype, int64_t N, int V, float alpha,
                          float* acc, void* ws, size_t ws_bytes, void* stream);
/* Embedding bags (nn.EmbeddingBag, opt-in): bag b of B pools its entries into the row c_b of a
 * Linear layer on R^V,
 *   KFAC_BAG_SUM:  c_bv = sum_{i in b, t_i = v} w_i      (w_i = weights[i], or 1)
 *   KFAC_BAG_MEAN: c_bv = n_bv / L_b                     (c_b = 0 for an empty bag)
 * where entries equal to padding_idx (>= 0; -1 for none) are left out and L_b counts the others.
 * kfac_factor_embedding_bag keeps the diagonal of (1/B) C^T C:  acc[v] += alpha * sum_b c_bv^2
 * (alpha = 1/B).  Bags of one index give the bits of kfac_factor_embedding on the same indices.
 * idx: N int32 / int64 indices in [0, V) (index_dtype), trusted like kfac_factor_embedding's.
 *   offsets != NULL: idx is 1-D and bag b is [offsets[b], offsets[b + 1]), the last bag ending
 *     at N.  Only the first B offsets are read (include_last_offset's extra entry is not: as in
 *     torch, the last bag ends at N).  offsets has index_dtype, is non-decreasing, starts at 0
 *     and is read on the device.
 *   offsets == NULL: idx is (B, N / B) row-major, one bag per row.
 * weights: NULL, or N per-sample weights of weight_dtype (KFAC_F32/F16/BF16), KFAC_BAG_SUM only.
 * c_bv is formed in fp64 (weights summed in entry order), squared and summed over the bags in bag
 * order in fp64, rounded once to fp32 as s_v, then acc[v] = fl(acc[v] + fl(alpha * s_v)).  The
 * (token, bag) pairs are grouped by a stable radix sort on the token (CUB): no floating-point
 * atomics, the same bits on every run, no host sync.  ws: kfac_factor_embedding_bag_workspace_bytes
 * (N, B, V) bytes (N < 2^31). */
enum kfac_bag_mode { KFAC_BAG_SUM = 0, KFAC_BAG_MEAN = 1 };
size_t kfac_factor_embedding_bag_workspace_bytes(int64_t N, int64_t B, int V);
int kfac_factor_embedding_bag(const void* idx, const void* offsets, int index_dtype, int64_t N,
                              int64_t B, int64_t padding_idx, int mode,
                              const void* weights, int weight_dtype, int V, float alpha,
                              float* acc, void* ws, size_t ws_bytes, void* stream);
/* EMA of diagonal factors (vectors of d = V floats), the schedule of kfac_factor_ema on the
 * diagonal and with the same rounding (the bits kfac_factor_ema gives on diag(batch)):
 *   factor = alpha*(first ? 1 : factor) + (1-alpha)*inv_count*batch;   batch = 0
 * A window of token counts (the A side of an embedding) is finite whatever the loss scale and
 * always takes this unguarded EMA.  One launch per 40 items. */
int kfac_factor_ema_diag(const kfac_ema_item* items, int count, float alpha, void* stream);
/* Guarded EMA of diagonal factors: the contract of kfac_factor_ema_guarded on vectors of d
 * floats (the diagonal G of a large-output Linear layer can overflow under fp16).  loss_scale:
 * HOST array of `count` DEVICE pointers (NULL array or entry = 1), u = (1 / *loss_scale[i])^2.
 * A window with an entry whose unscaled value is not finite or exceeds 1e15 is dropped: the
 * factor keeps its value (all ones when `first` = 1), the batch is zeroed and *skipped (may be
 * NULL) is incremented.  Every kept window gets the bits kfac_factor_ema_diag gives on batch * u.
 * ws: kfac_factor_ema_diag_guarded_workspace_bytes(count) bytes (one drop flag per item).
 * Two launches per 40 items (scan, EMA). */
size_t kfac_factor_ema_diag_guarded_workspace_bytes(int count);
int kfac_factor_ema_diag_guarded(const kfac_ema_item* items, int count, float alpha,
                                 const float* const* loss_scale, unsigned long long* skipped,
                                 void* ws, size_t ws_bytes, void* stream);

/* Diagonal-G Linear layers (an extension beyond the reference, opt-in): the G factor of a layer
 * with many outputs (an LM head, V = 50257) is approximated by its diagonal, kept as V floats.
 * kfac_factor_linear_diag: acc[j] += scale * sum_r x[r, j]^2 over x (rows x features, dtype
 * KFAC_F32/F16/BF16, contiguous), the diagonal of what kfac_factor_linear accumulates for the same
 * input.  Deterministic and without a host sync: the rows are split into a number of chunks that
 * depends on `rows` only, each chunk's column sums (accumulated in fp64, stored as fp32) go to ws
 * (kfac_factor_linear_diag_workspace_bytes(rows, features) bytes), and a second launch adds them
 * in a fixed order.  No floating-point atomics. */
size_t kfac_factor_linear_diag_workspace_bytes(int64_t rows, int features);
int kfac_factor_linear_diag(const void* x, int dtype, int64_t rows, int features, float scale,
                            float* acc, void* ws, size_t ws_bytes, void* stream);
/* Diagonal-A layers (an extension beyond the reference, opt-in): a Linear or convolution layer with
 * more inputs than the eigensolver takes keeps its A factor as the vector diag(A), bias entry last.
 * kfac_factor_linear_diag_ones: kfac_factor_linear_diag with the ones column of kfac_factor_linear
 * appended when append_ones: acc has features + append_ones entries, and acc[features] += scale *
 * rows (the squares of the ones column).  Same workspace query, chunking and bits on the features
 * as kfac_factor_linear_diag (which is this call with append_ones = 0). */
int kfac_factor_linear_diag_ones(const void* x, int dtype, int64_t rows, int features,
                                 int append_ones, float scale, float* acc, void* ws,
                                 size_t ws_bytes, void* stream);
/* kfac_factor_conv_input_diag: acc (d = C * kd * kh * kw + append_ones floats) += scale * the
 * diagonal of the X^T X kfac_factor_conv_input accumulates for the same geometry, without the
 * im2col: acc[(c, taps)] += scale * sum over the im2col rows of row^2, and acc[d - 1] += scale *
 * batch * Do * Ho * Wo for the ones column.  Each (b, c) volume is read once from HBM; the window
 * sums of its squares over the output lattice are formed from it (a kernel window of at most 2048
 * taps, else KFAC_ERR_BAD_ARG).  x in fp32, fp16 or bf16.  Deterministic and without a host sync:
 * every example's sums go to ws as fp32 partials (batch x (d - append_ones) floats,
 * kfac_factor_conv_input_diag_workspace_bytes), and a second launch adds them in example order in
 * fp64.  No floating-point atomics. */
size_t kfac_factor_conv_input_diag_workspace_bytes(const kfac_conv_geometry* geom);
int kfac_factor_conv_input_diag(const void* x, int dtype, const kfac_conv_geometry* geom,
                                int append_ones, float scale, float* acc, void* ws,
                                size_t ws_bytes, void* stream);
/* dst[i] = src[i] for n floats; ORs 2 (the non-finite bit of the kfac_eigh_batched status word)
 * into the DEVICE int *status when an entry is not finite or exceeds 1e15 in magnitude.  The
 * snapshot of a diagonal factor at an inverse step, checked like a decomposed factor. */
int kfac_diag_snapshot(const float* src, float* dst, int n, int* status, void* stream);

/* Normalization layers (an extension beyond the reference, opt-in): BatchNorm1d/2d, LayerNorm and
 * RMSNorm keep the exact per-channel Fisher block of their affine part y = s * xhat + b instead of
 * two Kronecker factors.  Channel c is a one-input layer with bias on xhat: rows a_r = (xhat_rc, 1)
 * (or (xhat_rc) without a bias) and g_r = dL/dy_rc, and
 *   F_c = (1/N) sum_r g_rc^2 a_r a_r^T,  packed as k = 3 floats (F_ss, F_sb, F_bb) or k = 1 (F_ss).
 * kfac_factor_norm: acc (C x k, row-major) += scale * sum_r g_rc^2 a_r a_r^T for one layer call:
 *   KFAC_NORM_BATCH  x, g are (rows = B, C, S) contiguous; xhat uses the biased statistics of each
 *                    channel over its B * S entries, plus eps;
 *   KFAC_NORM_LAYER  x, g are (rows, C) row-major (C = the product of normalized_shape); xhat uses
 *                    the mean and biased variance of each row, plus eps;
 *   KFAC_NORM_RMS    as LAYER with xhat = x / sqrt(mean(x^2) + eps) (k must be 1).
 * scale folds 1/N, the 1/S^4 of rows and gradients scaled by 1/S like a Conv2d layer's, and the
 * AMP 1/grad_scale^2.  x (the layer INPUT: xhat does not depend on the gain) and g take any of
 * KFAC_F32/F16/BF16 independently and are read once each (LAYER / RMS read x a second time for the
 * row statistics).  All sums are fp64; the chunking depends on the shape only and the chunk partials
 * are added in a fixed order, so the same input gives the same bits.  No floating-point atomics, no
 * host sync.  ws: kfac_factor_norm_workspace_bytes(kind, rows, C, S) bytes.  Three launches (two
 * for BATCH). */
enum kfac_norm_kind { KFAC_NORM_BATCH = 0, KFAC_NORM_LAYER = 1, KFAC_NORM_RMS = 2 };
size_t kfac_factor_norm_workspace_bytes(int kind, int64_t rows, int C, int64_t S);
int kfac_factor_norm(const void* x, int x_dtype, const void* g, int g_dtype, int kind, int64_t rows,
                     int C, int64_t S, int k, double eps, float scale, float* acc, void* ws,
                     size_t ws_bytes, void* stream);
/* kfac_factor_group_norm: the same contract as kfac_factor_norm for GroupNorm and InstanceNorm*
 * (groups = C): x, g are (B, C, S) contiguous; xhat uses the mean and biased variance, plus eps, of
 * each example's group, the Cg * S entries of channels [gi * Cg, (gi + 1) * Cg) with Cg = C / groups.
 * acc (C x k) += scale * sum_{b,s} g^2 a a^T.  x and g take any of KFAC_F32/F16/BF16 independently
 * and are read once each; the sums are fp64, reduced in a fixed order, so the same input gives the
 * same bits; no floating-point atomics, no host sync.  Refused: groups not dividing C, k not 1 or 3,
 * B * C * S >= 2^31.  ws: kfac_factor_group_norm_workspace_bytes(B, C, S, groups) bytes (B * C * 5
 * doubles of plane sums and B * groups (mean, 1/std) pairs).  Three launches. */
size_t kfac_factor_group_norm_workspace_bytes(int64_t B, int C, int64_t S, int groups);
int kfac_factor_group_norm(const void* x, int x_dtype, const void* g, int g_dtype, int64_t B, int C,
                           int64_t S, int groups, int k, double eps, float scale, float* acc,
                           void* ws, size_t ws_bytes, void* stream);
/* P_c = (F_c + damping I)^-1 (wgrad[c], bgrad[c]) for every channel of every item, in fp64, written
 * as P (C x np, ld = np, np = 2 with a bias, else 1): the weight in column 0 and the bias in the last
 * column, the layout kfac_grad_scale / kfac_grad_update read for g = C, a = np.  F is the C x k
 * snapshot of the running block (k = 3 with a bias, k = 1 without).  One launch over all items;
 * every channel is one thread, so the result does not depend on the other items.
 * ws: kfac_norm_precondition_workspace_bytes(count) bytes (the item table). */
typedef struct kfac_norm_item {
  const float* F;     /* C x k */
  const void* wgrad;  /* (C), grad_dtype */
  const void* bgrad;  /* (C) when k = 3, else NULL */
  int grad_dtype;
  int C, k;
  float* P;           /* out: C x np */
} kfac_norm_item;
size_t kfac_norm_precondition_workspace_bytes(int count);
int kfac_norm_precondition(const kfac_norm_item* items, int count, float damping, void* ws,
                           size_t ws_bytes, void* stream);

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
 * iteration did not converge, bit 1 = a non-finite (or |x| > 1e15) factor entry, replaced by 0, or a non-finite eigenvalue): fetch it with kfac_eigh_status().
 * Scale: a factor whose largest finite entry of magnitude at most 1e15 is m is solved as 2^-e F with 2^-e m in
 * [1, 2), and its eigenvalues are multiplied by 2^e, unless m lies in [1/16, 1) or is 0 (then e = 0, the result it
 * had before the normalisation).  So the accuracy does not depend on the magnitude of F, and replacing F by 2^k F
 * gives the same Q (and QT) bits and 2^k d whenever the largest entries of both lie outside [1/16, 1), provided the
 * entries of both are normal floats (or zero) and at most 1e15; eigenvalues that are subnormal floats may differ by one
 * subnormal ulp. */
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
 * the eigendecomposition of F (F is symmetric PSD). ws: n*ldq floats.
 * Deterministic: the same inputs give the same bits in every call.  For n > 1024 the product's
 * reduction runs as chains of at most 512 on the tensor cores, one after another into inv (the
 * first stores, each later one adds), never with floating-point atomics. */
int kfac_inverse_from_eigh(const float* Q, int ldq, const float* d, int n,
                           float damping, float* inv, int ld_inv, void* ws,
                           size_t ws_bytes, void* stream);
/* pi-adjusted (factored Tikhonov) damping (Martens & Grosse 2015, sec. 6.3; an extension beyond the reference,
 * opt-in): the damping lambda of the Kronecker product A (x) G is split between the factors by their trace norms,
 *     pi = sqrt((tr A / a) / (tr G / g)),    s = sqrt(lambda),    gamma_A = s * pi,    gamma_G = s / pi,
 * so that (A + gamma_A I) (x) (G + gamma_G I) does not depend on how the scale of the product is split between A and G.
 * kfac_pi: pi of every item, one launch per 768 items (one block each).  A factor is dense (ld >= its dimension; its
 * diagonal is read) or a vector (ld = 0: a diagonal factor, its own diagonal).  Both traces are summed in fp64 in a
 * fixed order (no atomics: repeat calls give the same bits), pi is rounded once to fp32, and it is 1 where a mean
 * trace is not a positive finite number (or pi does not round to a positive finite float).  No host sync, no
 * workspace. */
typedef struct kfac_pi_item {
  const float* A;  /* a x a (ld = lda), or a floats (lda = 0) */
  const float* G;  /* g x g (ld = ldg), or g floats (ldg = 0) */
  float* pi;       /* out: one float */
  int a, g;
  int lda, ldg;
} kfac_pi_item;
int kfac_pi(const kfac_pi_item* items, int count, void* stream);
/* kfac_dgda with pi: out[i,j] = 1 / ((dg[i] + gamma_G) * (da[j] + gamma_A)), gamma_A = s * *pi, gamma_G = s / *pi
 * (fp32, each rounded on its own); s on the host, pi a DEVICE float. */
int kfac_dgda_pi(const float* dg, const float* da, int g, int a, float s, const float* pi,
                 float* out, int ld_out, void* stream);
/* kfac_inverse_from_eigh with the damping gamma of one factor: side +1 (A) gamma = s * *pi, side -1 (G)
 * gamma = s / *pi; inv = Q diag(1 / (d + gamma)) Q^T with the same workspace, products and bits as
 * kfac_inverse_from_eigh with damping = gamma. */
int kfac_inverse_from_eigh_pi(const float* Q, int ldq, const float* d, int n, float s,
                              const float* pi, int side, float* inv, int ld_inv, void* ws,
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
 *   INVERSE: P = Ginv grad Ainv
 * Embedding items (kind = KFAC_ITEM_EMBEDDING): wgrad is the (a = V, g = d) weight gradient,
 * bgrad NULL, da the diagonal A factor (V floats; its own eigenvalues), and P (V x ldp, ldp >= d)
 * is written in the weight's layout:
 *   EIGEN  : P = [(wgrad Qg) / (da x dg + damping)] Qg^T     (qg, qgT, dg; dgda is not used)
 *   INVERSE: P = diag(1 / (da + damping)) wgrad Ginv          (g_inv)
 * qa, qaT, a_inv, dgda and ldqa are ignored.  The two (one) GEMMs join the grouped launches of
 * the dense items; the other items' results do not depend on the embedding items.
 * Diagonal-G items (kind = KFAC_ITEM_DIAG_G): wgrad (g = V, a - has_bias) and bgrad as for a
 * dense item, dg the diagonal G factor (V floats; its own eigenvalues), P (g x ldp, ldp >= a):
 *   EIGEN  : P = [(grad Qa) / (dg x da + damping)] Qa^T      (qa, qaT, da; dgda is not used)
 *   INVERSE: P = diag(1 / (dg + damping)) grad Ainv           (a_inv)
 * qg, qgT, g_inv, dgda, ldqg and ld_dgda are ignored.  This is the embedding item with the dense
 * factor on the A side.
 * Tied items (kind = KFAC_ITEM_TIED): one (V, d) weight used by an embedding (token frequencies f,
 * output-gradient factor E) and by a bias-less diagonal-G head (input factor H, diagonal G h).  With
 * M and mu from kfac_tied_whiten / kfac_tied_basis (M^T (E + tI) M = I, M^T (H + tI) M = diag(mu),
 * t = tied_damping), the row v of P is (f_v + t)(E + tI) + (h_v + t)(H + tI) solved for row v of
 * the gradient:
 *   P = [(wgrad M) / ((f + t) 1^T + (h + t) mu^T)] M^T
 * wgrad is (a = V, g = d), bgrad NULL, qg = M, qgT = M^T (ld = ldqg), da = f, dh = h (V floats each),
 * dg = mu (d floats), P (V x ldp, ldp >= d).  `method` and `damping` of the call are not used; the
 * two GEMMs join the grouped launches, the division is one more launch over all tied items (the
 * engines' epilogues are left as they are), and the other items' results do not depend on tied items.
 * Diagonal-A items (kind = KFAC_ITEM_DIAG_A): a Linear or convolution layer whose A factor is kept
 * as its diagonal.  wgrad (g, a - has_bias) and bgrad as for a dense item (fp32, fp16 or bf16; no
 * wgrad_taps), da the diagonal A factor (a floats, bias entry last; its own eigenvalues), P (g x ldp,
 * ldp >= a) in the dense layout:
 *   EIGEN  : P = Qg [(Qg^T grad) / (dg x da + damping)]       (qg, qgT, dg; dgda is not used)
 *   INVERSE: P = Ginv grad diag(1 / (da + damping))            (g_inv)
 * qa, qaT, a_inv, dgda, ldqa and ld_dgda are ignored.  The gradient is gathered transposed (one
 * more launch per item), and the products are those of an embedding item on grad^T (the division
 * is the EPI_DIV_OUTER epilogue of the first product), the last one formed transposed so that P is
 * g x a.  The two (one) GEMMs join the grouped launches; the last one is split into chains of at
 * most 512 for g > 1024 (eigen), and its peer stores give the bits of the local P.  The other
 * items' results do not depend on diagonal-A items.
 * pi-adjusted damping (pi != NULL, a DEVICE float from kfac_pi; every kind but KFAC_ITEM_TIED, which rejects it with
 * KFAC_ERR_BAD_ARG): with s = sqrtf(damping), gamma_A = s * *pi and gamma_G = s / *pi, every division by
 * (u x v + damping) above, u and v the eigenvalues (or diagonals) of the two factors, becomes a division by
 * (u + gamma_u) x (v + gamma_v) (the EPI_DIV_FACTORED epilogue), and each one-sided division of the INVERSE method
 * takes the gamma of its diagonal factor.  So
 *   dense EIGEN (no dgda):  P = Qg [(Qg^T grad Qa) / ((dg + gamma_G) x (da + gamma_A))] Qa^T
 *   embedding EIGEN:        P = [(wgrad Qg) / ((da + gamma_A) x (dg + gamma_G))] Qg^T
 *   diagonal-G INVERSE:     P = diag(1 / (dg + gamma_G)) grad Ainv,   and likewise for the other kinds.
 * dgda, a_inv and g_inv are used as given (kfac_dgda_pi and kfac_inverse_from_eigh_pi form them with pi). */
enum kfac_item_kind {
  KFAC_ITEM_DENSE = 0, KFAC_ITEM_EMBEDDING = 1, KFAC_ITEM_DIAG_G = 2, KFAC_ITEM_TIED = 3, KFAC_ITEM_DIAG_A = 4
};
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
   * P arenas, mapped with kfac_peer_open().  The last GEMM stores P to all peers too (P2P over
   * NVLink): from its tile epilogue, or, where its reduction is split (K > 1024), from the pass
   * that adds the partials.  P does not depend on n_peers: the same bits for 0 to 7 peers, and
   * columns [0, n) of every peer entry equal P (padding columns hold P's zeros or are left
   * as they were).  Every peer pointer must be the same offset into an arena with the same
   * alignment as the local one (the tiles are stored as float2 where P's row is 8-byte
   * aligned).  n_peers = 0: local only. */
  float* const* peer_P;
  int n_peers;
  int kind; /* kfac_item_kind; 0 (dense) for the positional initialisers written before it */
  const float* dh;    /* KFAC_ITEM_TIED: the head's diagonal G (V floats); else ignored */
  float tied_damping; /* KFAC_ITEM_TIED: the damping M and mu were formed with (> 0) */
  /* layout of wgrad (dense items): 0 (the initialisers written before this field) = row-major
   * (g, a - has_bias); T > 0 = a transposed convolution's (C_in, g, T) weight gradient, whose
   * grad-matrix element (r, ci * T + t) lies at wgrad[(ci * g + r) * T + t].  P stays (g, a). */
  int wgrad_taps;
  /* pi-adjusted damping: a DEVICE float (kfac_pi) or NULL (the initialisers written before this field) for the
   * damping above, with its bits */
  const float* pi;
} kfac_precond_item;
size_t kfac_precondition_workspace_bytes(const kfac_precond_item* items, int count);
int kfac_precondition(const kfac_precond_item* items, int count, int method,
                      float damping, void* ws, size_t ws_bytes, void* stream);

/* Tied embedding / LM-head pairs (an extension beyond the reference, opt-in): the d x d factors E
 * (the embedding's G) and H (the head's A) are diagonalised together.  With E = Q diag(e) Q^T
 * (kfac_eigh_batched, e >= 0) and s = (e + damping)^-1/2:
 *   kfac_tied_whiten:  C = diag(s) (Q^T H Q + damping I) diag(s), written exactly symmetric
 *                      ((X + X^T) / 2 before the scaling), dense with ld = d: the F of a
 *                      kfac_eigh_batched item whose Q / QT are U / UT below.
 *   kfac_tied_basis:   M = Q diag(s) U (U: the eigenvectors of C in its columns) and MT = M^T.
 * Then M^T (E + damping I) M = I and M^T (H + damping I) M = diag(mu), mu the eigenvalues of C.
 * Q^T H Q, the product by Q and M run on the grouped wgmma engine (3xTF32); products with d > 1024
 * are split into chains of <= 512 whose partials are added in a fixed order.  No floating-point
 * atomics: the same inputs give the same bits.  Both calls are batched over items; the fields a
 * call does not name are ignored.  ws: kfac_tied_workspace_bytes(items, count) bytes. */
typedef struct kfac_tied_item {
  const float* Q;  /* d x d (ld): eigenvectors of E in the columns (kfac_eigh_item.Q) */
  const float* QT; /* its transpose (ld) */
  const float* e;  /* d eigenvalues of E */
  const float* H;  /* d x d (ld = d), symmetric: whiten */
  float* C;        /* out of whiten: d x d (ld = d) */
  const float* UT; /* basis: d x d (ld), rows are the eigenvectors of C (kfac_eigh_item.QT) */
  float* M;        /* out of basis: d x d (ld) */
  float* MT;       /* out of basis: d x d (ld), the transpose of M */
  int d, ld;       /* ld: a multiple of 4, >= d */
} kfac_tied_item;
size_t kfac_tied_workspace_bytes(const kfac_tied_item* items, int count);
int kfac_tied_whiten(const kfac_tied_item* items, int count, float damping, void* ws,
                     size_t ws_bytes, void* stream);
int kfac_tied_basis(const kfac_tied_item* items, int count, float damping, void* ws,
                    size_t ws_bytes, void* stream);

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
  int wgrad_taps; /* layout of wgrad, as for a precondition item (0 = row-major); the sums run in P's order */
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

/* ----------------------------------------------------------------- EKFAC
 * Eigenvalue-corrected K-FAC (George et al., 2018): the Kronecker product dg x da of the
 * eigenvalues is replaced by second moments S measured in the eigenbasis,
 *   S_batch = (1/N) sum_r (Qg^T g_r)^2 (Qa^T x_r)^2^T          (g x a, element-wise squares),
 * and the eigen precondition runs with dgda = 1 / (S + damping).
 *
 * Row writers: the rows x_r / g_r of one layer, SAMPLE-major fp32 (N x ld_out, ld_out a multiple
 * of 4 and >= d; columns [d, ld_out) are written as 0).  Every value is multiplied by
 * scale / *loss_scale (loss_scale: optional DEVICE float, the AMP loss scale; NULL = 1).
 * The feature order is that of the factor calls above.  No workspace. */
int kfac_rows_linear(const void* x, int dtype, int64_t rows, int features, int append_ones,
                     float scale, const float* loss_scale, float* out, int ld_out, void* stream);
/* kfac_rows_linear on input rows with a row stride ld >= features (elements) */
int kfac_rows_linear_strided(const void* x, int dtype, int64_t rows, int features, int64_t ld,
                             int append_ones, float scale, const float* loss_scale, float* out,
                             int ld_out, void* stream);
int kfac_rows_conv2d_input(const void* x, int dtype, int batch, int C, int H, int W, int kh,
                           int kw, int sh, int sw, int ph, int pw, int append_ones, float scale,
                           float* out, int ld_out, void* stream);
/* the rows of kfac_factor_conv_input: (batch * Do * Ho * Wo) x ld_out; the Conv2d entry above is
 * this call with a depth-1, dilation-1 geometry */
int kfac_rows_conv_input(const void* x, int dtype, const kfac_conv_geometry* geom, int append_ones,
                         float scale, float* out, int ld_out, void* stream);
/* the rows of kfac_factor_conv_transpose_input: (batch * Do * Ho * Wo) x ld_out */
int kfac_rows_conv_transpose_input(const void* x, int dtype, const kfac_conv_transpose_geometry* geom,
                                   int append_ones, float scale, float* out, int ld_out,
                                   void* stream);
/* g (batch, C, Ho, Wo) -> rows (batch*Ho*Wo, C) */
int kfac_rows_conv2d_gradout(const void* g, int dtype, int batch, int C, int Ho, int Wo,
                             float scale, const float* loss_scale, float* out, int ld_out,
                             void* stream);

/* K-FAC-reduce rows (Eschenhagen et al., 2023) of a weight-shared layer: ONE row per example,
 * the sum of the example's R expand rows (those of the kfac_rows_* writer with scale 1),
 * multiplied by scale / *loss_scale (loss_scale: optional DEVICE float; NULL = 1).  Output
 * fp32, SAMPLE-major, batch x ld_out (ld_out >= d, any value; columns [d, ld_out) are written
 * as 0), usable as the rows of kfac_factor_linear (ld_out = d) or of the EKFAC statistics
 * (ld_out = ld4(d)).  Every input element is read once; the sums run in fp32 over runs of at
 * most 16 elements, then in fp64, in a fixed order (no atomics: the same bits on every run).
 * One launch each, no workspace.
 *   linear:   x (B, R, features) in f32/f16/bf16; the ones column is scale * R.
 *   conv2d_input:  x NCHW; the window sums of every (b, c) plane over the output lattice,
 *             computed from the plane (no im2col); feature order (C, kh, kw) [+ ones], the
 *             ones column scale * Ho * Wo; zero padding, dilation and groups ignored, as in
 *             kfac_factor_conv2d_input.  kh * kw <= 2048.
 *   conv2d_gradout:  g (batch, C, Ho, Wo) -> the spatial sum of every (b, c) plane. */
int kfac_reduce_rows_linear(const void* x, int dtype, int64_t B, int64_t R, int features,
                            int append_ones, float scale, const float* loss_scale, float* out,
                            int ld_out, void* stream);
/* kfac_reduce_rows_linear with the element (b, t, f) at x[b * example_stride + t * position_stride
 * + f]: a sequence-first (R, B, ld) tensor, or a column block of one, is reduced in place with
 * example_stride = ld and position_stride = B * ld.  The contiguous strides (R * features,
 * features) give the bits of kfac_reduce_rows_linear. */
int kfac_reduce_rows_linear_strided(const void* x, int dtype, int64_t B, int64_t R, int features,
                                    int64_t example_stride, int64_t position_stride,
                                    int append_ones, float scale, const float* loss_scale,
                                    float* out, int ld_out, void* stream);
int kfac_reduce_rows_conv2d_input(const void* x, int dtype, int batch, int C, int H, int W,
                                  int kh, int kw, int sh, int sw, int ph, int pw,
                                  int append_ones, float scale, float* out, int ld_out,
                                  void* stream);
int kfac_reduce_rows_conv2d_gradout(const void* g, int dtype, int batch, int C, int Ho, int Wo,
                                    float scale, const float* loss_scale, float* out,
                                    int ld_out, void* stream);
/* conv2d_input for an N-d geometry with dilation: the window sums of every (b, c) volume over
 * the output lattice, feature order (C, kd, kh, kw) [+ ones], the ones column
 * scale * Do * Ho * Wo.  kd * kh * kw <= 2048.  The Conv2d entry above is this call with a
 * depth-1, dilation-1 geometry.  A single-row input (D = H = 1, kd = kh = 1, no depth or height
 * padding: a Conv1d) spreads each window offset's sum over a CTA; the sums keep their order. */
int kfac_reduce_rows_conv_input(const void* x, int dtype, const kfac_conv_geometry* geom,
                                int append_ones, float scale, float* out, int ld_out,
                                void* stream);
/* conv_input for a transposed geometry: the sum over the output positions of tap (l, i, j) is the
 * sum of x over the box of inputs whose outputs i * stride - padding + k * dilation lie inside the
 * output on every axis, formed by the same kernels (and the same single-row path). */
int kfac_reduce_rows_conv_transpose_input(const void* x, int dtype,
                                          const kfac_conv_transpose_geometry* geom, int append_ones,
                                          float scale, float* out, int ld_out, void* stream);

/* Rows of a recurrent layer's sub-layer (nn.RNN / LSTM / GRU): position (t, b) of a sequence of T
 * steps, time-major (row t * B + b) or packed (row offsets[t] + b, offsets a DEVICE int[T + 1]
 * with offsets[0] = 0 and non-increasing batch sizes offsets[t + 1] - offsets[t] <= B, as in a
 * PackedSequence).  The source row of a position holds `features` elements of dtype `dtype`:
 *   shift  0: x[row(t, b) * ldx + col0 ...] itself;
 *   shift +1: the previous hidden state of a forward direction: row (t - 1, b) of x, h0[b * ldh]
 *             at t = 0;
 *   shift -1: that of a reverse direction: row (t + 1, b) while sequence b continues there, else
 *             h0[b * ldh].
 * With `mul` set, the columns f >= mul_col0 are multiplied by mul[row(t, b) * ldm + f - mul_col0]
 * (same dtype): the GRU's hidden-gate gradient [dr, dz, r * dn] from the input-gate gradient and r. */
typedef struct kfac_sequence_rows {
  const void* x;   int64_t ldx;  int col0;
  const void* h0;  int64_t ldh;  int shift;
  const void* mul; int64_t ldm;  int mul_col0;
  int T; int B; const int* offsets;   /* offsets NULL: T x B time-major positions */
} kfac_sequence_rows;
/* One row per position, in row(t, b) order, like kfac_rows_linear (out: rows x ld_out fp32, the
 * values times scale / *loss_scale, the ones column scale, zeros up to ld_out).  Rows: T * B, or
 * offsets[T]. */
int kfac_rows_sequence(const kfac_sequence_rows* src, int dtype, int features, int append_ones,
                       float scale, const float* loss_scale, float* out, int ld_out, void* stream);
/* K-FAC-reduce over sequences: row b (b < B) is the sum of sequence b's R_b rows times
 * scale * R_b^-power / *loss_scale (power 1: the mean, A side; 0.5: G side), the ones column R_b
 * times that factor.  R_b is T, or the number of steps whose batch size exceeds b.  The sums keep
 * the order of kfac_reduce_rows_linear. */
int kfac_reduce_rows_sequence(const kfac_sequence_rows* src, int dtype, int features,
                              int append_ones, float scale, float power,
                              const float* loss_scale, float* out, int ld_out, void* stream);

/* S_batch of every item, for all items together; no floating-point atomics, the same bits on
 * every run.  Launches: one grouped wgmma launch of the projections (x^2 epilogue), the K = N
 * product as one grouped launch, and the fixed-order sum of its split partials.  Extra launches:
 *   - a projection with K = a or g > 1024 is accumulated in place over chunks of <= 512 columns,
 *     one grouped launch per chunk round (up to 16 at K = 8192), then one squaring launch;
 *   - the grouped engine runs each problem that is too small or narrow for the tensor cores
 *     (M or N < 64) as its own SIMT launch: the projections of a layer with a or g < 64 (or with
 *     fewer than 64 rows), and its S_batch product (g or a < 64) once per 4096 rows, followed by
 *     one summing launch per such layer. */
typedef struct kfac_ekfac_stat_item {
  const float* X;   /* N x ldx: rows x_r (kfac_rows_*) */
  const float* G;   /* N x ldg: rows g_r */
  const float* qaT; /* a x a (ld = ldqa): rows are the eigenvectors of A (kfac_eigh_item.QT) */
  const float* qgT; /* g x g (ld = ldqg) */
  float* S_batch;   /* out: g x a (ld = lds); the padding columns [a, lds) are unspecified */
  int64_t N;        /* rows, < 2^31 */
  int a, g;
  int ldx, ldg, ldqa, ldqg, lds;   /* ldx, ldg, lds multiples of 4 */
} kfac_ekfac_stat_item;
size_t kfac_ekfac_statistics_workspace_bytes(const kfac_ekfac_stat_item* items, int count);
int kfac_ekfac_statistics(const kfac_ekfac_stat_item* items, int count, void* ws,
                          size_t ws_bytes, void* stream);

/* Schedule of S, one mode per call, then dgda = 1 / (S + damping) (padding columns 0):
 *   KEEP  S unchanged (the per-step damping refresh)
 *   EMA   S = alpha*S + (1-alpha)*S_batch
 *   RESET S = S_batch                     (a window measured in a new basis)
 *   SEED  S = dg x da                     (a new basis without a window: the K-FAC eigen method)
 * EMA and RESET drop the window of an item whose S_batch holds an entry that is not finite or
 * exceeds 1e15 in magnitude, or whose drop_a / drop_g flag (the drop flags kfac_factor_ema_guarded
 * leaves in its workspace) is set: EMA then keeps S, RESET falls back to SEED.  A window dropped
 * for its S_batch alone (neither flag set) increments *skipped (device counter, may be NULL); the
 * guarded EMA has counted the others.  One launch (two with the scan of S_batch in EMA / RESET). */
enum kfac_ekfac_mode { KFAC_EKFAC_KEEP = 0, KFAC_EKFAC_EMA = 1, KFAC_EKFAC_RESET = 2, KFAC_EKFAC_SEED = 3 };
typedef struct kfac_ekfac_update_item {
  float* S;             /* g x a running second moments (ld) */
  const float* S_batch; /* g x a (ld); EMA / RESET only */
  const float* dg;      /* eigenvalues of G (g) and A (a); SEED / RESET only */
  const float* da;
  float* dgda;          /* out: g x a (ld) */
  int g, a, ld;
  const int* drop_a;    /* optional DEVICE flags: non-zero drops the window */
  const int* drop_g;
} kfac_ekfac_update_item;
size_t kfac_ekfac_update_workspace_bytes(int count);
int kfac_ekfac_update(const kfac_ekfac_update_item* items, int count, float alpha, int mode,
                      float damping, unsigned long long* skipped, void* ws, size_t ws_bytes,
                      void* stream);

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
