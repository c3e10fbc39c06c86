/*
 * pipegcn_b200 -- C ABI of the H100-native (sm_90a) PipeGCN hot path (libpipegcn_b200.so).
 *
 * The reference (GATECH-EIC/PipeGCN @ 73ab949) is pure Python; it has no FFI.  Its
 * plug-in seam is a set of Python objects (helper/context.py:4-5, module/layer.py:8).
 * These entry points are what a ctypes binding of those objects calls; each one
 * names the reference code it replaces.  All pointers are raw device pointers
 * unless stated otherwise, every call is asynchronous on `stream`
 * (a cudaStream_t passed as void*), never synchronises the host, and returns 0 on
 * success or a negative pg_status; pg_last_error() describes the last failure of
 * the calling thread.  The caller owns all memory.
 */
#ifndef PIPEGCN_B200_H
#define PIPEGCN_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PG_ABI_VERSION 2

/* element types of activations / gradients */
#define PG_F32  0
#define PG_BF16 1

enum pg_status {
  PG_OK = 0,
  PG_ERR_INVALID = -1,      /* bad argument (null pointer, misaligned, unsupported width) */
  PG_ERR_CUDA = -2,         /* a CUDA runtime/driver call failed */
  PG_ERR_UNSUPPORTED = -3,  /* not available on this device / build */
  PG_ERR_TIMEOUT = -4       /* a halo flag did not arrive within the spin bound */
};

int pg_abi_version(void);
const char* pg_last_error(void);
/* writes sm major*10+minor, SM count and L2 bytes of `device`; needs a GPU */
int pg_device_info(int device, int* sm_arch, int* sm_count, int64_t* l2_bytes);
/* tuning knobs (process-wide; the defaults are the measured best, the other values keep earlier code paths selectable):
 * "agg_impl" = 1 | 2 | 3 (row-per-group, chunked, chunked + cp.async long rows); "agg_unroll" = 4 | 8 neighbour rows in
 * flight per lane group; "agg_pack_short" = 0 | 1; "agg_occ" = 4 | 5; "agg_overlap" = 0 | 1 (short rows on a side
 * stream); "agg_narrow" = 0 | 1 (sub-warp kernels for rows of <= 16 vectors); "agg_l2_hint" = 0 | 1;
 * "ln_stage" = 0 | 1 | 2 (LayerNorm rows through the cp.async ring: never / one vector per lane / always);
 * "ce_subwarp" = 0 | 1 (several cross-entropy rows per warp); "gemm_epi_slabs" = 1 | 2 (GEMM epilogue: staging
 * slabs per warp).  Unknown names return PG_ERR_INVALID. */
int pg_set_option(const char* name, int value);

/* ------------------------------------------------------------------------------------------
 * Adjacency of one partition in CSR form plus the split of its long rows.
 * Forward: rows = destination (`_V`) nodes, columns = source (`_U`) ids  (layer.py:47-49).
 * Backward: rows = source ids, columns = destinations (DGL gspmm backward on the reversed graph).
 * Rows with more than seg_len entries are cut into segments of seg_len that different
 * warps reduce into fp32 partials; a fix-up pass sums the partials in segment order, so the
 * result does not depend on scheduling.
 * ---------------------------------------------------------------------------------------- */
typedef struct pg_csr {
  const int32_t* indptr;        /* [n_rows + 1] */
  const int32_t* indices;       /* [nnz] */
  int32_t n_rows;
  int32_t seg_len;              /* > 0 */
  int32_t n_long;               /* rows longer than seg_len */
  int32_t n_seg;                /* total segments of the long rows */
  const int32_t* long_row;      /* [n_long] row id */
  const int32_t* long_seg_ptr;  /* [n_long + 1] first segment of every long row */
  const int32_t* seg_long;      /* [n_seg] index into long_row */
  const int32_t* row_order;     /* [n_rows] processing order of the rows (e.g. by falling degree), or NULL */
  int64_t nnz;                  /* number of entries (indptr[n_rows]); selects the short-row kernel shape */
  /* chunked walk (optional, chunks == NULL selects the row-per-group kernel): the rows in processing order
   * (falling length) with their entries stored contiguously, cut into chunks one warp processes */
  const int32_t* chunks;        /* [n_chunks][4] = {first entry in pidx, n, item, kind | n_rows << 2}:
                                 *   kind 0: n_rows whole rows of n entries each (n_rows * n <= 32), item = first row in prow
                                 *   kind 1: one row of n entries, item = its position in prow
                                 *   kind 2: one segment (n entries) of a long row, item = segment index (scratch slot) */
  int32_t n_chunks;
  int32_t n_chunks_long;        /* the kind 2 and kind 1 chunks come first: chunks [0, n_chunks_long) */
  const int32_t* pidx;          /* [nnz] column ids, rows concatenated in processing order; bit 31 set = "hot" source
                                 * row (referenced often): loaded with an L2 evict_last policy */
  const int32_t* prow;          /* [n_rows] row id of every position of the processing order */
} pg_csr;

/*
 * Dropout (model.py:47) without a stored mask: keep(element) is a pure function of (seed, step, element index), where
 * step = *step_dev + step_off is an epoch counter that lives on the device (CUDA-graph replay).  Every kernel that
 * writes a tensor the next layer consumes can apply it on the way out, so no [num_all, d] dropout pass is needed:
 * the LayerNorm epilogue (inner rows), the halo push (the receiver's halo rows, receiver's row index), and the
 * transposed aggregate / fix-up (the gradient of the dropped tensor).  p == 0 or a NULL pointer: no dropout.
 */
typedef struct pg_drop {
  float p;
  uint64_t seed;
  const uint32_t* step_dev;   /* may be NULL: the mask does not depend on a step */
  int32_t step_off;
} pg_drop;

/*
 * Neighbour aggregate (SURVEY.md K6/K7/K11):
 *   out[r, 0:d] = ( sum_{e in row r} x[indices[e], 0:d] ) / row_div[r]  ( + out[r, 0:d] if r < acc_rows )
 * x and out have element type `dtype`, sums are fp32.  ldx/ldo are row strides in elements.
 * row_div (fp32, [n_rows]) may be NULL (no division); the division is one IEEE reciprocal per row and a multiply per
 * element (within 1 ulp of `/`).  scratch: fp32 [n_seg * d_pad] where
 * d_pad = d rounded up to 8; may be NULL when n_seg == 0.
 * Replaces graph['_E'].update_all(fn.copy_src, fn.sum) and `/ degs` at
 * PipeGCN/module/layer.py:47-50, and their autograd.
 */
int pg_aggregate(const pg_csr* g, const void* x, int64_t ldx, void* out, int64_t ldo, int32_t d, int dtype,
                 const float* row_div, int32_t acc_rows, float* scratch, void* stream);
/* the same, with the dropout mask of `drop` applied to every output row as it is written (the backward of
 * `layer(dropout(F))`: out = mask * ((A^T g) (+ out)) / (1 - p)); element index = row * ceil(d / vec) + vector */
int pg_aggregate_drop(const pg_csr* g, const void* x, int64_t ldx, void* out, int64_t ldo, int32_t d, int dtype,
                      const float* row_div, int32_t acc_rows, float* scratch, const pg_drop* drop, void* stream);

/*
 * Neighbour aggregate with a per-source and a per-destination scale (GraphConv's symmetric norm, c = deg^-1/2):
 *   out[r, 0:d] = dst_scale[r] * ( sum_{e in row r} src_scale[indices[e]] * x[indices[e], 0:d] )  ( + bias[0:d] )
 * then, if `drop` is given, that key's dropout mask as the row is stored (as pg_aggregate_drop).  The sum is fp32 in the
 * order of pg_aggregate (CSR order within a chunk or segment, long-row segment partials merged in segment order), each
 * term one multiply-add; then the multiply by dst_scale, then the bias, then one rounding to `dtype`.  With
 * src_scale == 1 and dst_scale = 1 / row_div (fp32 IEEE division) the result has the bits of pg_aggregate.
 * src_scale: fp32 [source rows]; dst_scale: fp32 [n_rows]; bias: fp32 [d] or NULL; scratch as pg_aggregate.
 * No accumulate mode, no atomics: the same bits from run to run.
 */
int pg_aggregate_scaled(const pg_csr* g, const void* x, int64_t ldx, void* out, int64_t ldo, int32_t d, int dtype,
                        const float* src_scale, const float* dst_scale, const float* bias, float* scratch,
                        const pg_drop* drop, void* stream);
/* loads every pg_aggregate_scaled kernel (call it before any halo wait can spin: a first launch may wait for the device) */
int pg_aggregate_scaled_preload(void);

/*
 * pg_aggregate_scaled with an initial residual (GCNII):
 *   out[r, 0:d] = dst_scale[r] * ( sum_{e in row r} src_scale[indices[e]] * x[indices[e], 0:d] ) + alpha * res[r, 0:d]
 *                 ( + bias[0:d] )
 * The sum is that of pg_aggregate_scaled; after the multiply by dst_scale each element takes one fp32 multiply-add of
 * alpha * res, then the bias, then one rounding to `dtype`.  A long row gets the residual once, in its fix-up.
 * res: [n_rows, ldr] of `dtype`, ldr >= d; res == NULL is pg_aggregate_scaled (the same kernels and bits).
 * Dropout, scratch and determinism as pg_aggregate_scaled.
 */
int pg_aggregate_scaled_res(const pg_csr* g, const void* x, int64_t ldx, void* out, int64_t ldo, int32_t d, int dtype,
                            const float* src_scale, const float* dst_scale, const void* res, int64_t ldr, float alpha,
                            const float* bias, float* scratch, const pg_drop* drop, void* stream);
/* loads every pg_aggregate_scaled_res kernel (as pg_aggregate_scaled_preload) */
int pg_aggregate_scaled_res_preload(void);

/*
 * GCNII row kernels (csrc/gcnii.cu).  Rows of `dtype` are 16-byte aligned and padded to the 16-byte vector (as the
 * dropout kernels); the pad columns of every output are written as 0.  No atomics: the same bits from run to run.
 *   pg_gcnii_relu_drop: h0 = ReLU(z); if hd != NULL, hd = dropout(h0) under `drop` (element (r, c) keyed as
 *                       pg_dropout_rows with row0 = 0; drop NULL or p = 0: hd = h0).
 *   pg_gcnii_teleport:  acc[r, c] = alpha * ds[r, c] (accumulate = 0) or fma(alpha, ds[r, c], acc[r, c]), fp32 acc.
 *   pg_gcnii_relu_bwd:  dz[r, c] = h0[r, c] > 0 ? g[r, c] + (r < n_acc ? acc[r, c] : 0) : 0, the sum in fp32, one rounding.
 */
int pg_gcnii_relu_drop(const void* z, int64_t ldz, void* h0, int64_t ldh, void* hd, int64_t ldd, int32_t n_rows,
                       int32_t d, int dtype, const pg_drop* drop, void* stream);
int pg_gcnii_teleport(const void* ds, int64_t ldd, float* acc, int64_t lda, int32_t n_rows, int32_t d, int dtype,
                      float alpha, int accumulate, void* stream);
int pg_gcnii_relu_bwd(const void* g, int64_t ldg, const void* h0, int64_t ldh, const float* acc, int64_t lda,
                      int32_t n_acc, void* dz, int64_t ldz, int32_t n_rows, int32_t d, int dtype, void* stream);

/* out[r, 0:d] = x[r, 0:d] / row_div[r]   (gradient of `/ degs`, layer.py:50) */
int pg_row_div(const void* x, int64_t ldx, void* out, int64_t ldo, int32_t n_rows, int32_t d, int dtype,
               const float* row_div, void* stream);

/*
 * Dense part of the layer on the Hopper tensor cores (wgmma) (SURVEY.md K8/K10):
 *   c[m, n] = sum_s a_s[m, k_s] * b_s[n, k_s]^T  (+ bias[n])  (/ row_div[m])      1 <= n_src <= 6
 * dtype_in PG_BF16 -> bf16 wgmma, PG_F32 -> tf32 wgmma; fp32 accumulation in registers;
 * dtype_out selects the element type of c.  n <= 256.  All operands row-major with 16-byte
 * aligned rows (TMA); k tails and the m tail are zero-filled / masked.  `srcs` is a HOST array.
 * When c's rows are 16-byte aligned (base and ldc) the epilogue stores with TMA, which may also write the rest of
 * the 16-byte vector holding column n-1 (columns [n, n rounded up to 16 bytes) of every row, never past ldc);
 * other outputs are written exactly in columns [0, n).
 * Replaces `self.linear1(feat[0:num_dst]) + self.linear2(ah)` at
 * PipeGCN/module/layer.py:51 (two pairs: inner rows x W1, neighbour mean x W2,
 * bias = b1 + b2) and, with one pair, the dX products of its autograd (row_div = in_deg fuses the
 * `/ degs` gradient).  fp32 parity mode passes the hi/lo halves of pg_split_tf32 as three pairs
 * per product (hi*hi + hi*lo + lo*hi: the "3xTF32" product, fp32-grade accuracy).
 */
typedef struct pg_gemm_src {
  const void* a;   /* [m, k] */
  int64_t lda;
  const void* b;   /* [n, k] */
  int64_t ldb;
  int32_t k;
} pg_gemm_src;

int pg_linear(int dtype_in, int dtype_out, const pg_gemm_src* srcs, int32_t n_src, const float* bias,
              const float* row_div, void* c, int64_t ldc, int32_t m, int32_t n, void* stream);
/* the same with the dropout mask of `drop` applied to c as it is written; c's row 0 is row drop_row0 of the tensor the
 * mask is defined on (the gradient of a dropped tensor produced by a GEMM: transform-first layers) */
int pg_linear_drop(int dtype_in, int dtype_out, const pg_gemm_src* srcs, int32_t n_src, const float* bias,
                   const float* row_div, void* c, int64_t ldc, int32_t m, int32_t n, const pg_drop* drop,
                   int64_t drop_row0, void* stream);
/* Grouped form: n_prob (1..4) products that share their A operands, each with its own B operands and output, in one
 * launch.  `srcs` holds n_prob x n_src pairs (problem-major, n_prob * n_src <= 12); pair s of every problem has the
 * A operand (a, lda, k) of srcs[s].  Problem q writes outs[q] = sum_s A_s B_{q,s}^T (+ bias) (/ row_div), with the
 * dropout of outs[q].drop, exactly as one pg_linear_drop call on its pairs would.  The CTAs working on the same rows
 * of A run together, so A is read from HBM once for all problems (the rest from L2). */
typedef struct pg_gemm_out {
  const float* bias;     /* [n] or NULL */
  const float* row_div;  /* [m] or NULL */
  void* c;
  int64_t ldc;
  const pg_drop* drop;   /* NULL or p == 0: no dropout */
  int64_t drop_row0;
} pg_gemm_out;
int pg_linear_group(int dtype_in, int dtype_out, const pg_gemm_src* srcs, int32_t n_src, int32_t n_prob,
                    const pg_gemm_out* outs, int32_t m, int32_t n, void* stream);

/*
 * Weight gradients on the Hopper tensor cores (MN-major bf16 operands, split-K over the rows, deterministic;
 * dtype_in must be PG_BF16 -- wgmma transposes 16-bit operands only -- else PG_ERR_UNSUPPORTED):
 *   out[n, k] = sum_s sum_m a_s[m, n] * b_s[m, k]        n, k <= 256, fp32 output, 1 <= n_src <= 6
 * a_s = upstream gradient g [m, n], b_s = layer input [m, k], both row-major with 16-byte aligned rows; `srcs[s].k`
 * is ignored.  Replaces the autograd of PipeGCN/module/layer.py:51 for the weights: gW1 = g^T feat[:N_in],
 * gW2 = g^T ah (one call each; three pairs per call for the split-fp32 product).  `workspace`: fp32 scratch of
 * pg_wgrad_workspace(m, n, k, dtype_in) floats for the split-K partials.
 */
int64_t pg_wgrad_workspace(int32_t m, int32_t n, int32_t k, int dtype_in);
int pg_wgrad(int dtype_in, const pg_gemm_src* srcs, int32_t n_src, float* out, int64_t ldo, int32_t m, int32_t n,
             int32_t k, float* workspace, int64_t workspace_floats, void* stream);
/* Grouped form: n_prob (1..2) weight gradients of the same n x k shape in one launch (and one reduction launch).
 * `srcs` holds n_prob x n_src pairs, problem-major.  Problem q has its own rows (outs[q].m), split-K partition and
 * workspace (pg_wgrad_workspace(outs[q].m, n, k, dtype_in) floats) and gets the bits of a lone pg_wgrad call.  The CTAs
 * of all problems over the same row slice run side by side, so an operand the problems share (g^T x and g^T ah) is
 * read from HBM once. */
typedef struct pg_wgrad_out {
  float* out;
  int64_t ldo;
  int32_t m;
  float* workspace;
  int64_t workspace_floats;
} pg_wgrad_out;
int pg_wgrad_group(int dtype_in, const pg_gemm_src* srcs, int32_t n_src, int32_t n_prob, const pg_wgrad_out* outs,
                   int32_t n, int32_t k, void* stream);

/* hi = x with the 13 low mantissa bits cleared (a tf32 value), lo = x - hi (exact); [rows, d] fp32 */
int pg_split_tf32(const float* x, int64_t ldx, float* hi, float* lo, int64_t ld, int32_t rows, int32_t d,
                  void* stream);

/* ------------------------------------------------------------------------------------------
 * Row-wise epilogues of the layer loop (model.py:53-56, train.py:320,351).  One warp per row, every tensor
 * read once and written once; column reductions are two-stage (`partial`: fp32 scratch of
 * pg_row_grid(n_rows) * 3 * d floats for the LayerNorm backward, pg_row_grid(n) * max(c, 1) for the loss).
 * ---------------------------------------------------------------------------------------- */
int pg_row_grid(int32_t n_rows);
/* out = keep ? x / (1 - p) : 0 with keep a pure function of (seed, element index) -- the backward calls it again on
 * the gradient with the same seed instead of storing a mask (dropout of model.py:47; in place allowed) */
int pg_dropout(const void* x, int64_t ldx, void* out, int64_t ldo, int32_t n_rows, int32_t d, int dtype, float p,
               uint64_t seed, const uint32_t* step_dev, void* stream);
/* the same with the general mask key: rows are numbered from row0 (a slice of a larger tensor) */
int pg_dropout_rows(const void* x, int64_t ldx, void* out, int64_t ldo, int64_t row0, int32_t n_rows, int32_t d, int dtype,
                    const pg_drop* drop, void* stream);
/* out = relu?(LayerNorm(y) * gamma + beta), mean/rstd [n_rows] kept for the backward; d % (16/elem) == 0 */
int pg_ln_relu_fwd(const void* y, int64_t ldy, const float* gamma, const float* beta, float eps, int relu,
                   void* out, int64_t ldo, float* mean, float* rstd, int32_t n_rows, int32_t d, int dtype,
                   void* stream);
/* the same with the next layer's dropout fused: `out` receives dropout(result) (what the next layer's aggregate and
 * GEMM read), `out_clean` the result itself (what the halo push sends and the backward needs) */
int pg_ln_relu_drop_fwd(const void* y, int64_t ldy, const float* gamma, const float* beta, float eps, int relu,
                        void* out, int64_t ldo, void* out_clean, int64_t ldc, float* mean, float* rstd, int32_t n_rows,
                        int32_t d, int dtype, const pg_drop* drop, void* stream);
/* g_y, dgamma[d], dbeta[d] and colsum[d] = column sums of g_y (the bias gradient of the producing linear) */
int pg_ln_relu_bwd(const void* g_out, int64_t ldg, const void* out, int64_t ldo, const void* y, int64_t ldy,
                   const float* mean, const float* rstd, const float* gamma, int relu, void* g_y, int64_t ldgy,
                   float* dgamma, float* dbeta, float* colsum, float* partial, int32_t n_rows, int32_t d,
                   int dtype, void* stream);
/* the same; with beta given the ReLU mask is recomputed from y (the forward's expression) and `out` is not read */
int pg_ln_relu_bwd2(const void* g_out, int64_t ldg, const void* out, int64_t ldo, const void* y, int64_t ldy,
                    const float* mean, const float* rstd, const float* gamma, const float* beta, int relu, void* g_y,
                    int64_t ldgy, float* dgamma, float* dbeta, float* colsum, float* partial, int32_t n_rows, int32_t d,
                    int dtype, void* stream);
/* loss[0] = sum_rows (logsumexp(z) - z[label]) over the first n_rows rows: CrossEntropyLoss(reduction='sum') */
int pg_ce_fwd(const void* z, int64_t ld, const int64_t* labels, int32_t n_rows, int32_t c, int dtype, float* lse,
              float* partial, float* loss, void* stream);
/* g[r] = (softmax(z[r]) - onehot) * upstream[0] for r < n_rows, 0 for n_rows <= r < n_total; colsum[c] optional */
int pg_ce_bwd(const void* z, int64_t ld, const int64_t* labels, const float* lse, const float* upstream,
              int32_t n_rows, int32_t n_total, int32_t c, int dtype, void* g, int64_t ldg, float* colsum,
              float* partial, void* stream);
/*
 * Accuracy counts of the evaluation (calc_acc, train.py:11-17) on the device.  For every row r < n_rows:
 * p = argmax of the c logits z[r, 0:c] (fp32 or bf16, compared in fp32; torch.argmax's order: NaN is the maximum,
 * the first maximal index wins); pred[r] = p when pred != NULL; for every bit k < n_tags set in tag[r] (bit k: row r
 * belongs to mask k), counts[2k + 1] += 1 and counts[2k] += (p == labels[r]).  counts ([2 * n_tags] int64: correct,
 * total per mask) is overwritten; labels, tag and counts may be NULL when n_tags == 0 (labels and tag also when
 * n_rows == 0).  n_tags <= 8; any ld >= c.
 * Integer atomics: the result is deterministic.
 */
int pg_eval_count(const void* logits, int64_t ld, int32_t n_rows, int32_t c, int dtype, const int64_t* labels,
                  const uint8_t* tag, int32_t n_tags, int32_t* pred, int64_t* counts, void* stream);

/* ------------------------------------------------------------------------------------------
 * Halo exchange (feature_buffer.py:165-194).  One descriptor per message of a launch; the
 * array lives in device memory and is built once by Buffer.init_buffer.
 * A message copies n_rows rows of `src` (gathered through idx, or contiguous from src_row0)
 * to `dst` -- normally peer memory mapped over NVLink.  With `ema` set the sender first
 * updates its fp32 mirror  ema <- m*ema + (1-m)*row  (feature_buffer.py:189-191) and ships
 * the smoothed row.  When the last CTA of a message has stored its rows it publishes `value`
 * to *flag with system-scope release semantics.
 * ---------------------------------------------------------------------------------------- */
typedef struct pg_msg {
  const int32_t* idx;      /* [n_rows] source row ids, or NULL */
  int64_t src_row0;        /* first source row when idx == NULL */
  int32_t n_rows;
  int32_t cta_begin;       /* first CTA of this message inside the launch (filled by the host) */
  void* dst;               /* destination of row 0 */
  int64_t ld_dst;          /* elements */
  float* ema;              /* [n_rows, ld_ema] fp32 sender-side EMA mirror, or NULL */
  int64_t ld_ema;
  uint32_t* flag;          /* flag word to publish (peer memory), or NULL */
  uint32_t* counter;       /* local arrival counter of this message (self resetting) */
  int64_t dst_row0;        /* row index of `dst` inside the receiver's tensor (key of the receiver's dropout mask) */
} pg_msg;

/* rows per CTA used by pg_halo_push when the host fills cta_begin */
int pg_push_rows_per_cta(void);

/* momentum = m and one_minus = (float)(1 - m) evaluated in double precision by the caller, exactly the two
 * scalars of `t *= m; t += (1 - m) * recv` (feature_buffer.py:190-191) */
/* the flag value published is `value` (+ *value_dev when value_dev != NULL: an epoch counter that lives on the
 * device, so that a captured CUDA graph of an epoch can be replayed) */
/* Vectors: the widest of 16, 8, 4 and (bf16) 2 bytes that src's base address and row stride allow, V elements each
 * (V = 1 for a bf16 source of odd stride, such as a contiguous [N, d] tensor with odd d).  Row r of message m is
 * written as columns [0, round_up(d, V)) of dst + r * ld_dst -- the tail of the last vector receives src's own pad
 * columns (with `ema`, the mirror's columns [0, round_up(d, V)) are updated too) -- so ld_dst and ld_ema must be
 * >= round_up(d, V), and dst must be aligned to the vector.  Rows >= n_rows are not touched. */
int pg_halo_push(const pg_msg* msgs, int32_t n_msgs, int32_t n_ctas, const void* src, int64_t ld_src, int32_t d,
                 int dtype, float momentum, float one_minus, uint32_t value, const uint32_t* value_dev, void* stream);
/* the same with the RECEIVER's dropout applied to every row as it is stored into peer memory (after the EMA, whose
 * mirror stays clean): the halo rows arrive as the rows of dropout(cat(feat, halo)) the receiver will consume.  The
 * mask is defined on 16-byte vectors: a source that allows narrower ones is refused (PG_ERR_INVALID). */
int pg_halo_push_drop(const pg_msg* msgs, int32_t n_msgs, int32_t n_ctas, const void* src, int64_t ld_src, int32_t d,
                      int dtype, float momentum, float one_minus, uint32_t value, const uint32_t* value_dev,
                      const pg_drop* drop, void* stream);

/*
 * Block the stream until every flags[i] >= value (acquire, system scope).  A bounded spin:
 * after `timeout_ms` the kernel stores PG_ERR_TIMEOUT to *status (device word, may be NULL)
 * and returns, so a dead peer cannot hang the GPU (the reference hangs in gloo wait(),
 * feature_buffer.py:184).  wait_ns (device word, may be NULL): the nanoseconds (%globaltimer) this launch
 * spent blocked are ADDED to it -- the exposed communication time of comm_timer.py:17-27, readable after
 * a region of CUDA-graph replays where host-recorded events are not available.
 */
int pg_halo_wait(const uint32_t* const* flags, int32_t n_flags, uint32_t value, const uint32_t* value_dev,
                 int32_t timeout_ms, int32_t* status, uint64_t* wait_ns, void* stream);

/*
 * Static-layer-0 shortcut: dst[r, 0:d] = c * src[r, 0:d] with c = 0 for k <= 0, else 1 (corr == 0) or
 * 1 - m^k (corr != 0), k = k_host (+ *k_dev).  The input features never change, so the halo rows of layer 0 after
 * k EMA updates of feature_buffer.py:186-191 are the closed form (1 - m^k) * x of the one-shot exchanged rows.
 */
int pg_scale_rows(const void* src, int64_t ld_src, void* dst, int64_t ld_dst, int32_t n_rows, int32_t d, int dtype,
                  float momentum, int corr, int32_t k_host, const uint32_t* k_dev, void* stream);

/*
 * grad[urow[i], 0:d] += sum_k recv[usrc[k], 0:d]  for k in [uptr[i], uptr[i+1]), in that order
 * (peers ascending), replacing the per-peer loop at feature_buffer.py:208-217.  bf16 sums are rounded to bf16
 * after every add.  Like the push, rows are moved in the widest vectors both operands allow (bf16: at least 4
 * bytes, else PG_ERR_INVALID), and columns [0, round_up(d, V)) of the urow rows are written.
 */
int pg_boundary_add(void* grad, int64_t ld_grad, const void* recv, int64_t ld_recv, int32_t d, int dtype,
                    const int32_t* urow, const int32_t* uptr, const int32_t* usrc, int32_t n_urow, void* stream);

/* ------------------------------------------------------------------------------------------
 * Boundary-node sampling (BNS-GCN, synchronous training): in epoch t rank r keeps halo row h (its row in r's `_U`
 * space, h >= N_in) iff hash(seed, t, r, h) < thresh, thresh = round(p * 2^32); inner rows are always kept.  The
 * hash is one function (csrc/common.cuh: bns_key / bns_keep), so the receiver, the pushing owner and the owner's
 * boundary add draw the same sample from the key alone.  t = epoch (+ *epoch_dev when epoch_dev != NULL: the
 * device epoch counter of a captured CUDA graph).
 * ---------------------------------------------------------------------------------------- */
typedef struct pg_bns {
  uint64_t seed;
  uint32_t thresh;
  uint32_t epoch;
  const uint32_t* epoch_dev;
} pg_bns;

/* mask[h - num_in] = keep(rank, h) for the halo rows h in [num_in, num_all) (bytes 0 / 1), and deg[v] = the number of
 * kept sources of inner row v in the forward CSR (indptr [num_in + 1], indices = `_U` rows; the self loop counts):
 * the sampled in-degree, as fp32.  One launch, one coalesced pass over the CSR. */
int pg_bns_sample(const pg_bns* s, int32_t rank, const int32_t* indptr, const int32_t* indices, int32_t num_in,
                  int32_t num_all, uint8_t* mask, float* deg, void* stream);
/* pg_halo_push_drop (no EMA: the messages' ema must be NULL) that moves only the sampled rows: row i of message m is
 * loaded and stored iff keep(keys[2m], keys[2m + 1] + i) -- keys[2m] the rank whose `_U` space the rows are keyed in,
 * keys[2m + 1] the row of i = 0 there (the receiver and dst_row0 for a feature push, the pusher and src_row0 for a
 * gradient push).  Flags are published as by pg_halo_push, also for messages whose sample is empty.  drop may be
 * NULL. */
int pg_halo_push_bns(const pg_msg* msgs, int32_t n_msgs, int32_t n_ctas, const int32_t* keys, const void* src,
                     int64_t ld_src, int32_t d, int dtype, uint32_t value, const uint32_t* value_dev,
                     const pg_drop* drop, const pg_bns* s, void* stream);
/* pg_boundary_add over the kept slots only: slot k of recv is added iff keep(slot_keys[2k], slot_keys[2k + 1]) (the
 * receiving peer and the row the slot fills in its `_U` space). */
int pg_boundary_add_bns(void* grad, int64_t ld_grad, const void* recv, int64_t ld_recv, int32_t d, int dtype,
                        const int32_t* urow, const int32_t* uptr, const int32_t* usrc, int32_t n_urow,
                        const int32_t* slot_keys, const pg_bns* s, void* stream);
/* dst[r, 0:d] = mask[r] ? src[r, 0:d] : 0 for r < n_rows; with src == NULL the kept rows of dst are left as they
 * are (only the unkept rows are zeroed). */
int pg_bns_mask_rows(const void* src, int64_t ld_src, void* dst, int64_t ld_dst, int32_t n_rows, int32_t d, int dtype,
                     const uint8_t* mask, void* stream);

/* ------------------------------------------------------------------------------------------
 * Quantised halo messages (--halo-bits b, b = 8 or 4).  Every message row of d elements travels as b-bit codes plus an
 * fp32 pair (lo, scale): lo = min, scale = (max - lo) / (2^b - 1) over the d elements (fp32, correctly rounded),
 *   q = clamp(floor((x - lo) * inv + u), 0, 2^b - 1),  inv = (2^b - 1) / (max - lo)
 * with every operation rounded separately (no FMA; q = 0 unless scale > 0 and inv is finite), and the receiver decodes
 * lo + q * scale (a multiply, then an add).  4-bit codes pack two per byte, the even element
 * in the low nibble; a code row is padded to 16 bytes.  A row with a non-finite element or a non-finite range ships
 * lo = scale = NaN (every element decodes to NaN); a never-written (zero) row decodes to zeros.  u in [0, 1) is a pure
 * function of (seed, layer * 2 + direction, the flag value of the message, the receiving rank, the row the data fills
 * at the receiver = dst_row0 + i, the element) with 24 random bits (csrc/common.cuh: quant_key / quant_u).
 * ---------------------------------------------------------------------------------------- */
typedef struct pg_quant {
  uint64_t seed;
  int32_t bits;               /* 8 or 4 */
  int32_t stream;             /* layer * 2 + direction (0 = features, 1 = gradients) */
} pg_quant;
/* per message of a quantised push */
typedef struct pg_qmsg {
  float* pairs;               /* (lo, scale) of row 0 of the message, [n_rows][2] fp32 -- normally peer memory */
  int32_t rank;               /* the receiving rank */
  int32_t pad;
} pg_qmsg;
/* pg_halo_push without EMA and dropout, storing codes: message m's row i goes to msgs[m].dst + i * ld_dst (ld_dst in
 * BYTES, a multiple of 16; dst 16-byte aligned) and its pair to qmsgs[m].pairs + 2 i.  One warp per row.  Flags are
 * published as by pg_halo_push, also for empty messages; value (+ *value_dev) is also the noise's step. */
int pg_halo_push_q(const pg_msg* msgs, int32_t n_msgs, int32_t n_ctas, const pg_qmsg* qmsgs, const void* src,
                   int64_t ld_src, int32_t d, int dtype, uint32_t value, const uint32_t* value_dev, const pg_quant* q,
                   void* stream);
/* out[r, 0:d] = decode(codes[r], pairs[r]) for r < n_rows (activation dtype; out 16-byte aligned, ld_out >= d rounded
 * up to 8).  With `mirror` (fp32 [n_rows, ld_mirror], 16-byte aligned) the receiver's EMA first runs
 * mirror <- m * mirror + (1 - m) * decoded (two roundings, no FMA) and out receives the mirror.  With `drop` the mask
 * of that key is applied as pg_dropout_rows(row0 = drop_row0) would apply it to the undropped output. */
int pg_halo_dequant(const uint8_t* codes, int64_t ld_codes, const float* pairs, int32_t n_rows, int32_t d, int32_t bits,
                    void* out, int64_t ld_out, int dtype, float* mirror, int64_t ld_mirror, float momentum,
                    float one_minus, const pg_drop* drop, int64_t drop_row0, void* stream);
/* pg_boundary_add over code rows: grad[urow[i]] += v_k for k in [uptr[i], uptr[i+1]) in that order, v_k the decoded
 * slot usrc[k] (with `mirror`: that slot's fp32 mirror after its EMA update) rounded to the activation dtype; the sum
 * is fp32, rounded to the dtype after every add. */
int pg_boundary_add_q(void* grad, int64_t ld_grad, int32_t d, int dtype, const uint8_t* codes, int64_t ld_codes,
                      const float* pairs, int32_t bits, const int32_t* urow, const int32_t* uptr, const int32_t* usrc,
                      int32_t n_urow, float* mirror, int64_t ld_mirror, float momentum, float one_minus, void* stream);

/* ------------------------------------------------------------------------------------------
 * Graph attention (GAT, DGL GATConv with negative_slope 0.2, no attention dropout) over the `_U` rows
 * [inner | halo] of one partition.  z [num_all, H * D] (fp32 or bf16, `dtype`) holds H heads of D columns per row;
 * el [num_all, H] and er [N_in, H] are fp32 scores; for the in-edges u -> v of the forward CSR
 *   e_uv = LeakyReLU(el[u] + er[v]),  a_uv = softmax over u of e_uv,  out[v] = sum_u a_uv z[u] + bias
 * per head.  `keep` (uint8 [num_all - num_in], may be NULL) is the boundary-node sample of the halo rows: a halo row u
 * with keep[u - num_in] == 0 is absent from every softmax and gets no gradient.  The plan must carry the chunk table
 * (pg_csr::chunks); `scratch` is fp32 of n_seg * H * (D + 2) floats (may be NULL when n_seg == 0).  fp32 accumulation,
 * no atomics, no per-edge storage, D <= 512; the results are the same bits from run to run.
 * For this section, GATv2's and the graph transformer's:
 * - A destination row without a kept source (no in-edge, or every source unkept) gets m = -inf, s = 0 and the
 *   output bias (GAT), 0 (GATv2) or skip (transformer) rounded once to the dtype; its gradient terms are exactly 0,
 *   and so are the source-pass outputs of an unkept halo row and of a row that is nobody's source (except GAT's
 *   der (x) attn_r of an inner row).
 * - Every pass writes columns [0, H * D) of each row of its wide outputs, [0, H) of each row of the per-head ones,
 *   and nothing else: no pad columns, no other rows.
 * ---------------------------------------------------------------------------------------- */
/* loads every attention kernel (call it before any halo wait can spin: a first launch may wait for the device) */
int pg_gat_preload(void);
/* el[r, k] = <z[r, k, :], attn_l[k, :]> for r < n_rows, er[r, k] = <z[r, k, :], attn_r[k, :]> for r < n_er */
int pg_gat_scores(const void* z, int64_t ldz, int32_t n_rows, int32_t n_er, int32_t H, int32_t D, int dtype,
                  const float* attn_l, const float* attn_r, float* el, float* er, void* stream);
/* out[v] (activation dtype, bias fp32 [H * D] or NULL) and the softmax statistics m[v, k] (maximum) and s[v, k]
 * (sum of exp(e - m)), fp32 [N_in, H], over the forward CSR g (rows = inner rows v) */
int pg_gat_aggregate(const pg_csr* g, const void* z, int64_t ldz, int32_t H, int32_t D, int dtype, const float* el,
                     const float* er, const float* bias, const uint8_t* keep, int32_t num_in, void* out, int64_t ldo,
                     float* m, float* s, float* scratch, void* stream);
/* backward over the forward CSR, grad = dL/d out:  dv[v, k] = <grad[v, k], out[v, k] - bias[k]>, evaluated as
 * sum_u a_uv <grad[v, k], z[u, k]> (the products the second output uses, so that bf16 rounding of the stored output does
 * not enter), and der[v, k] = sum_u a_uv (<grad[v, k], z[u, k]> - dv[v, k]) LeakyReLU'(el[u, k] + er[v, k]) */
int pg_gat_bwd_dst(const pg_csr* g, const void* z, int64_t ldz, const void* grad, int64_t ldg, int32_t H, int32_t D,
                   int dtype, const float* el, const float* er, const float* m, const float* s, const uint8_t* keep,
                   int32_t num_in, float* der, float* dv, float* scratch, void* stream);
/* backward over the CSC gt (rows = all `_U` rows u, columns = destinations v):
 *   del[u, k] = sum_v a_uv (<grad[v, k], z[u, k]> - dv[v, k]) LeakyReLU'(el[u, k] + er[v, k])
 *   dz[u, k] = sum_v a_uv grad[v, k] + del[u, k] attn_l[k] (+ der[u, k] attn_r[k] for u < num_in)
 * dz in the activation dtype; unkept halo rows get dz = 0, del = 0 */
int pg_gat_bwd_src(const pg_csr* gt, const void* z, int64_t ldz, const void* grad, int64_t ldg, int32_t H, int32_t D,
                   int dtype, const float* el, const float* er, const float* m, const float* s, const float* dv,
                   const float* der, const float* attn_l, const float* attn_r, const uint8_t* keep, int32_t num_in,
                   void* dz, int64_t lddz, float* del, float* scratch, void* stream);
/* out[k * D + c] = sum_r coef[r, k] x[r, k * D + c] (coef fp32 [n_rows, H], NULL: 1) in a fixed order: the gradients
 * of attn_l / attn_r (coef = del / der) and column sums (H = 1).  partial: fp32 scratch of
 * pg_gat_colsum_blocks(n_rows) * H * D floats */
int pg_gat_colsum_blocks(int32_t n_rows);
int pg_gat_colsum(const void* x, int64_t ldx, int32_t n_rows, int32_t H, int32_t D, int dtype, const float* coef,
                  float* out, float* partial, void* stream);

/* ------------------------------------------------------------------------------------------
 * Dynamic graph attention (GATv2, DGL GATv2Conv with share_weights=False, negative_slope 0.2, no attention dropout)
 * over the `_U` rows [inner | halo] of one partition.  zs [num_all, H * D] and zd [N_in, H * D] (fp32 or bf16,
 * `dtype`) are the source and destination transforms, attn fp32 [H * D]; for the in-edges u -> v of the forward CSR,
 * per head k:
 *   t_uv = zs[u, k] + zd[v, k],  e_uv = <attn[k], LeakyReLU(t_uv)>,  a_uv = softmax over u of e_uv,
 *   out[v, k] = sum_u a_uv zs[u, k]      (a row without a kept in-edge gets 0)
 * `keep` and the chunk-table plan as for pg_gat_*; fp32 accumulation, no atomics, no per-edge storage, D <= 512; the
 * results are the same bits from run to run.  Scratch (fp32, may be NULL when n_seg == 0): n_seg * H * (D + 2) floats
 * for the aggregate, n_seg * H * (4 D + 1) for the destination pass, n_seg * H * D for the source pass.
 * ---------------------------------------------------------------------------------------- */
int pg_gatv2_preload(void);
/* out (activation dtype) and the softmax statistics m (maximum), s (sum of exp(e - m)), fp32 [N_in, H] */
int pg_gatv2_aggregate(const pg_csr* g, const void* zs, int64_t ldzs, const void* zd, int64_t ldzd, int32_t H,
                       int32_t D, int dtype, const float* attn, const uint8_t* keep, int32_t num_in, void* out,
                       int64_t ldo, float* m, float* s, float* scratch, void* stream);
/* backward over the forward CSR, grad = dL/d out, dot_uv = <grad[v, k], zs[u, k]>:
 *   dv[v, k] = D_v = sum_u a_uv dot_uv,  de_uv = a_uv (dot_uv - D_v)
 *   dzd[v, k] = sum_u de_uv attn[k] ⊙ LeakyReLU'(t_uv)                 (activation dtype)
 *   pattn[v, k] = sum_u de_uv LeakyReLU(t_uv)  (fp32 [N_in, H * D], row stride ldp: d attn is its column sum) */
int pg_gatv2_bwd_dst(const pg_csr* g, const void* zs, int64_t ldzs, const void* zd, int64_t ldzd, const void* grad,
                     int64_t ldg, int32_t H, int32_t D, int dtype, const float* attn, const float* m, const float* s,
                     const uint8_t* keep, int32_t num_in, void* dzd, int64_t lddzd, float* dv, float* pattn,
                     int64_t ldp, float* scratch, void* stream);
/* backward over the CSC gt (rows = all `_U` rows u, columns = destinations v):
 *   dzs[u, k] = sum_v a_uv grad[v, k] + de_uv attn[k] ⊙ LeakyReLU'(t_uv)   (activation dtype; unkept halo rows: 0) */
int pg_gatv2_bwd_src(const pg_csr* gt, const void* zs, int64_t ldzs, const void* zd, int64_t ldzd, const void* grad,
                     int64_t ldg, int32_t H, int32_t D, int dtype, const float* attn, const float* m, const float* s,
                     const float* dv, const uint8_t* keep, int32_t num_in, void* dzs, int64_t lddzs, float* scratch,
                     void* stream);

/* ------------------------------------------------------------------------------------------
 * Graph transformer (PyG TransformerConv with concat=True, beta=False, root_weight=True, no edge features, no
 * attention dropout) over the `_U` rows [inner | halo] of one partition.  q and skip [N_in, H * D], k and v
 * [num_all, H * D] (fp32 or bf16, `dtype`, each with its own row stride) are the four projections; for the in-edges
 * u -> v of the forward CSR, per head h:
 *   e_uv = scale <q[v, h], k[u, h]>  (scale = 1/sqrt(D), passed in fp32),  a_uv = softmax over u of e_uv,
 *   out[v, h] = sum_u a_uv v[u, h] + skip[v, h]    (attention part 0 for a row without a kept in-edge)
 * `keep` and the chunk-table plan as for pg_gat_*; fp32 accumulation, no atomics, no per-edge storage, D <= 512; the
 * results are the same bits from run to run, and both backward passes recompute a_uv with the forward's bits.
 * Scratch (fp32, may be NULL when n_seg == 0): n_seg * H * (D + 2) floats for the aggregate, n_seg * H * (2 D + 1) for
 * the destination pass, n_seg * H * 2 D for the source pass.
 * ---------------------------------------------------------------------------------------- */
int pg_tconv_preload(void);
/* out (activation dtype; skip added in fp32 before the one rounding) and the softmax statistics m (maximum), s (sum
 * of exp(e - m)), fp32 [N_in, H] */
int pg_tconv_aggregate(const pg_csr* g, const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v,
                       int64_t ldv, const void* skip, int64_t ldskip, int32_t H, int32_t D, int dtype, float scale,
                       const uint8_t* keep, int32_t num_in, void* out, int64_t ldo, float* m, float* s,
                       float* scratch, void* stream);
/* backward over the forward CSR, grad = dL/d out, gd_uv = <grad[v, h], v[u, h]>:
 *   delta[v, h] = sum_u a_uv gd_uv   (fp32 [N_in, H])
 *   dq[v, h] = scale sum_u a_uv (gd_uv - delta_v) k[u, h],  gcopy[v, h] = grad[v, h]   (activation dtype) */
int pg_tconv_bwd_dst(const pg_csr* g, const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v,
                     int64_t ldv, const void* grad, int64_t ldg, int32_t H, int32_t D, int dtype, float scale,
                     const float* m, const float* s, const uint8_t* keep, int32_t num_in, void* dq, int64_t lddq,
                     void* gcopy, int64_t ldgc, float* delta, float* scratch, void* stream);
/* backward over the CSC gt (rows = all `_U` rows u, columns = destinations v):
 *   dv[u, h] = sum_v a_uv grad[v, h],  dk[u, h] = scale sum_v a_uv (gd_uv - delta_v) q[v, h]
 *   (activation dtype; unkept halo rows: 0) */
int pg_tconv_bwd_src(const pg_csr* gt, const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v,
                     int64_t ldv, const void* grad, int64_t ldg, int32_t H, int32_t D, int dtype, float scale,
                     const float* m, const float* s, const float* delta, const uint8_t* keep, int32_t num_in,
                     void* dk, int64_t lddk, void* dv, int64_t lddv, float* scratch, void* stream);

/* ------------------------------------------------------------------------------------------
 * Max-pool GraphSAGE (DGL SAGEConv(aggregator_type='pool')) over the `_U` rows [inner | halo] of one partition.
 * Q [num_all, d] (fp32 or bf16, `dtype`) is the pooled transform h Wp^T + bp.  For the in-edges u -> v of the forward
 * CSR g (each edge once):
 *   M[v, c] = max_u Q[u, c],  A[v, c] = the u that gives it,  hn[v, c] = ReLU(M[v, c])
 * A tie goes to the first source in CSR order; the first NaN source becomes the value and the argmax; a row without
 * in-edges gets hn = 0 and A = -1.  A holds int32 `_U` row ids (bit 31 of pg_csr::pidx stripped).  Rows of q, hn, A,
 * grad and gq start on 16-byte boundaries with strides that are multiples of 16 bytes, covering the last 16-byte
 * vector of a row of q, A and grad (the padded rows of the activations).  The plans must carry the chunk table
 * (pg_csr::chunks); scratch is fp32 [n_seg][ld_scratch] (may be NULL when n_seg == 0).  No atomics: the results are the
 * same bits from run to run.
 * ---------------------------------------------------------------------------------------- */
/* loads every pool kernel (call it before any halo wait can spin: a first launch may wait for the device) */
int pg_pool_preload(void);
/* hn [N_in, d] (activation dtype) and A [N_in, d] int32 over the forward CSR g; ld_scratch >= 2 d */
int pg_max_aggregate(const pg_csr* g, const void* q, int64_t ldq, int32_t d, int dtype, void* hn, int64_t ldh,
                     int32_t* arg, int64_t lda, float* scratch, int64_t ld_scratch, void* stream);
/* gq[u, c] = [Q[u, c] > 0] * sum over the destinations v of CSC row u (gt = the transposed plan, rows = all num_all
 * `_U` rows) with A[v, c] == u of grad[v, c], accumulated in fp32 in CSC order and stored in the activation dtype;
 * a row without out-edges gets 0.  grad = dL/d hn [N_in, d]; ld_scratch >= d */
int pg_max_aggregate_bwd(const pg_csr* gt, const void* q, int64_t ldq, const int32_t* arg, int64_t lda,
                         const void* grad, int64_t ldg, int32_t d, int dtype, void* gq, int64_t ldgq, float* scratch,
                         int64_t ld_scratch, void* stream);

/* ------------------------------------------------------------------------------------------
 * Principal neighbourhood aggregation (DGL PNAConvTower, aggregators mean/max/min/std) over the `_U` rows
 * [inner | halo] of one partition.  zs [num_all, d] (fp32 or bf16, `dtype`) is the source half h W_s^T of the message
 * linear, zd [N_in, d] fp32 its destination half h W_d^T + b.  For the in-edges u -> v of the forward CSR g (each edge
 * once, D_v of them), per column:
 *   mu = mean_u zs[u],  var = mean_u (zs[u] - mu)^2,  mx / mn = max_u / min_u zs[u] with sources A+ / A-
 *   agg[v] = [mu + zd | mx + zd | mn + zd | sqrt(max(var, 0) + 1e-30)]   (zd added in fp32, one rounding to dtype)
 * The four parts start `seg` elements apart (seg >= d, a multiple of the 16-byte vector); columns [d, seg) of each part
 * are not written.  The moments use Welford's update per edge and Chan's merge across long-row segments, so a row whose
 * sources are all equal gets var = 0 exactly.  A tie of an extreme goes to the first source in CSR order; the first NaN
 * source becomes the value and the source.  A row without in-edges gets agg = 0, mu = var = 0 and A+- = -1.  A+- hold
 * int32 `_U` row ids.  mu / var (fp32) and A+ / A- may be NULL (pairwise): they are then not written.  Rows start on
 * 16-byte boundaries with strides that are multiples of 16 bytes, covering the last 16-byte vector of a row.  The plans
 * must carry the chunk table; scratch is fp32 [n_seg][ld_scratch] (may be NULL when n_seg == 0).  No atomics: the
 * results are the same bits from run to run.
 * ---------------------------------------------------------------------------------------- */
/* loads every PNA kernel (call it before any halo wait can spin: a first launch may wait for the device) */
int pg_pna_preload(void);
/* agg [N_in, 4 seg] (dtype), mu / var [N_in, d] fp32, A+ / A- [N_in, d] int32 over the forward CSR g;
 * ld_scratch >= 6 d */
int pg_pna_aggregate(const pg_csr* g, const void* zs, int64_t ldz, const float* zd, int64_t ldzd, int32_t d, int dtype,
                     void* agg, int64_t ldagg, int64_t seg, float* mu, float* var, int64_t ldst, int32_t* amax,
                     int32_t* amin, int64_t lda, float* scratch, int64_t ld_scratch, void* stream);
/* out[v, o] = fl(fl(y[v, o] + fl(a[v] z[v, o])) + fl(t[v] z[v, d_out + o])) in fp32, rounded once to dtype: the
 * degree scalers a (amplification) and t (attenuation) applied to the GEMM outputs y = [h | agg] [W_x; W_1]^T + b and
 * z = agg [W_2; W_3]^T, fp32 [n_rows, d_out] and [n_rows, 2 d_out] */
int pg_pna_combine(const float* y, int64_t ldy, const float* z, int64_t ldz, const float* a, const float* t,
                   int32_t n_rows, int32_t d_out, int dtype, void* out, int64_t ldo, void* stream);
/* out = [g | a g | t g] (dtype, each product rounded once), the three parts `seg` elements apart; columns
 * [d_out, seg) of each part are not written */
int pg_pna_grad_scale(const void* g, int64_t ldg, const float* a, const float* t, int32_t n_rows, int32_t d_out,
                      int dtype, void* out, int64_t ldo, int64_t seg, void* stream);
/* per destination element, from g_agg = [g_mu | g_mx | g_mn | g_sigma] (fp32, parts `seg` apart), mu, var and
 * D_v = indptr[v + 1] - indptr[v]:
 *   g_zd = g_mu + g_mx + g_mn,  beta = [var > 0] g_sigma / (D sigma),  alpha = g_mu / D - beta mu  (fp32)
 * g_zd, g_mx and g_mn in dtype, alpha and beta fp32; every output 0 on a row without in-edges */
int pg_pna_bwd_dst(const int32_t* indptr, const float* gagg, int64_t ldga, int64_t seg, const float* mu,
                   const float* var, int64_t ldst, int32_t n_rows, int32_t d, int dtype, void* gzd, int64_t ldgzd,
                   float* alpha, float* beta, int64_t ldab, void* gmx, void* gmn, int64_t ldgm, void* stream);
/* g_zs[u] = S1 + zs[u] S2 over the CSC row u of gt (rows = all num_all `_U` rows), with S1 = sum alpha_v + the g_mx_v
 * of the destinations whose A+ is u + the g_mn_v of those whose A- is u, and S2 = sum beta_v, each accumulated in
 * fp32 in CSC order (edge by edge: alpha, then g_mx, then g_mn); the product is applied once at the end.  A row
 * without out-edges gets exactly 0.  ld_scratch >= 2 d */
int pg_pna_bwd_src(const pg_csr* gt, const void* zs, int64_t ldz, const float* alpha, const float* beta, int64_t ldab,
                   const int32_t* amax, const int32_t* amin, int64_t lda, const void* gmx, const void* gmn,
                   int64_t ldgm, int32_t d, int dtype, void* gzs, int64_t ldgzs, float* scratch, int64_t ld_scratch,
                   void* stream);

/* ------------------------------------------------------------------------------------------
 * Softmax-aggregation graph convolution (DeeperGCN; PyG GENConv, aggr='softmax', one scalar temperature t) over the
 * `_U` rows [inner | halo] of one partition.  xs [num_all, d] (fp32 or bf16, `dtype`) is x_src = h W_src^T (or h),
 * xd [N_in, d] (dtype) x_dst.  For the in-edges u -> v of the forward CSR g whose source is kept, per column c:
 *   m_u = ReLU(xs[u]) + 1e-7,  s_u = t m_u   (fp32, one rounding each; a NaN x stays NaN)
 *   M = max_u s_u,  W = sum_u exp(s_u - M),  A = sum_u exp(s_u - M) m_u,  B = sum_u exp(s_u - M) m_u^2
 *   agg = A / W,  L = M + log W,  var = max(B / W - agg^2, 0),  S = agg + xd   (S rounded once to dtype)
 * The state is updated online, one expf per edge and element (exp(-|s - M|) weighs the new edge or rescales the old
 * state), in CSR order; long rows come as segments whose states a fix-up merges in segment order.  No atomics: the
 * results are the same bits from run to run.  A row without a kept in-edge gets agg = 0, L = -inf, var = 0 and S = xd;
 * a NaN source makes its destinations' agg, L, var and S NaN.  t is read from device memory (a captured CUDA graph
 * sees every update of it).  keep (uint8 [num_all - num_in], or NULL: every source kept) is the keep mask of the halo
 * rows: a source u >= num_in with keep[u - num_in] == 0 is skipped.  Rows start on 16-byte boundaries with strides that
 * are multiples of 16 bytes, covering the last 16-byte vector of a row; only columns [0, d) are written.  The plans
 * must carry the chunk table; scratch is fp32 [n_seg][ld_scratch] (may be NULL when n_seg == 0).
 * ---------------------------------------------------------------------------------------- */
/* fp64 block partials of pg_genconv_bwd_dst's dt: the `partial` workspace holds this many doubles */
#define PG_GENCONV_DT_PARTIALS 264
/* loads every GENConv kernel (call it before any halo wait can spin: a first launch may wait for the device) */
int pg_genconv_preload(void);
/* S [N_in, d] (dtype) over the forward CSR g; with agg != NULL also agg and L (fp32 [N_in, d], the backward's
 * operands), with var != NULL (needs agg) also var (fp32 [N_in, d], the temperature's gradient).  ld_scratch >= 3 d,
 * or 4 d with var */
int pg_genconv_aggregate(const pg_csr* g, const void* xs, int64_t ldxs, const void* xd, int64_t ldxd, int32_t d,
                         int dtype, const float* t, const uint8_t* keep, int32_t num_in, void* s, int64_t lds,
                         float* agg, int64_t ldagg, float* lse, int64_t ldlse, float* var, int64_t ldvar,
                         float* scratch, int64_t ld_scratch, void* stream);
/* per destination element, from g_S (fp32 [n_rows, d], the gradient of S) and agg:
 *   Q = fl(t fl(g_S agg))  (fp32);  gst = g_S rounded to dtype (may be NULL: not written)
 * and with var != NULL:  dt = sum_{v, c} g_S var  (fp64 products and sums: each of at most PG_GENCONV_DT_PARTIALS
 * CTAs sums its elements in grid-stride order and a fixed tree, then one CTA sums the partials in a fixed order and
 * rounds once to fp32 into the device scalar *dt).  The grid depends on n_rows * d only: the same bits from run to run.
 * var and dt are NULL together */
int pg_genconv_bwd_dst(const float* gs, int64_t ldg, const float* agg, int64_t ldagg, const float* var, int64_t ldvar,
                       const float* t, int32_t n_rows, int32_t d, int dtype, float* q, int64_t ldq, void* gst,
                       int64_t ldgst, double* partial, float* dt, void* stream);
/* dx[u] over the CSC row u of gt (rows = all num_all `_U` rows), per column:
 *   acc = sum_v exp(fl(t m_u) - L_v) (G_v (1 + t m_u) - Q_v)   (G = g_S; fp32, one multiply-add per term, CSC order;
 *                                                              long rows: segment sums added in segment order)
 *   dx  = dropout([xs[u] > 0] ? acc : 0  (+ add[u] for u < n_add))   rounded once to dtype
 * with m_u recomputed from xs.  A row without out-edges, and an unkept halo row, get acc = 0 (so 0, or add[u]).
 * add (fp32 [n_add, d], may be NULL when n_add == 0) lets the inner rows take g_S when x_src is h itself; drop (may be
 * NULL) is the dropout key of the layer input, applied as pg_dropout_rows does (row u, 16-byte vectors).
 * ld_scratch >= d */
int pg_genconv_bwd_src(const pg_csr* gt, const void* xs, int64_t ldxs, const float* t, const uint8_t* keep,
                       int32_t num_in, const float* lse, int64_t ldlse, const float* gs, int64_t ldg, const float* q,
                       int64_t ldq, const float* add, int64_t ldadd, int32_t n_add, const pg_drop* drop, int32_t d,
                       int dtype, void* dx, int64_t lddx, float* scratch, int64_t ld_scratch, void* stream);

/* ------------------------------------------------------------------------------------------
 * Residual gated graph convolution (Bresson & Laurent, 2017; PyG ResGatedGraphConv, sigmoid gate, no edge features)
 * over the `_U` rows [inner | halo] of one partition.  Every operand is fp32 or bf16 (`dtype`), and two of them are
 * paired rows with halves `half` columns apart: qv [num_all rows] holds q at columns [0, d) and val at
 * [half, half + d); ks [N_in rows] holds k at [0, d) and skip at [half, half + d) (skip carries the output bias).
 * For the in-edges u -> v of the forward CSR g whose source is kept, per column c, with x = fl(k[v] + q[u]):
 *   e = exp(-|x|),  r = 1 / (1 + e),  sigmoid(x) = x >= 0 ? r : e r,  sigmoid'(x) = e r r   (one expf per element)
 *   out[v] = skip[v] + sum_u sigmoid(x) val[u]
 * Sums are fp32 with one multiply-add per term, in CSR order (CSC order in the source pass); long rows come as
 * segments whose partials a fix-up adds in segment order.  No atomics and no per-edge storage (both backward passes
 * recompute the gate): the results are the same bits from run to run.  A row without a kept in-edge gets out = skip.
 * keep (uint8 [num_all - num_in], or NULL: every source kept) is the keep mask of the halo rows: a source
 * u >= num_in with keep[u - num_in] == 0 is skipped.  Every result is rounded once to dtype.  The kernels read and
 * write whole vectors of VB bytes, VB the widest of 16, 8, 4 (and 2 for bf16) that every operand's base, second half
 * and row stride allow; each row's last vector is written whole, the columns past d as 0, so `half` and every row
 * stride must reach round_up(d, VB / element size) (past `half` too for a paired operand).  The plans must carry the
 * chunk table; scratch is fp32 [n_seg][ld_scratch] (may be NULL when n_seg == 0).
 * ---------------------------------------------------------------------------------------- */
/* loads every ResGatedGCN kernel (call it before any halo wait can spin: a first launch may wait for the device) */
int pg_resgated_preload(void);
/* out [N_in, d] over the forward CSR g.  ld_scratch >= d */
int pg_resgated_aggregate(const pg_csr* g, const void* qv, int64_t ldqv, const void* ks, int64_t ldks, int32_t half,
                          int32_t d, int dtype, const uint8_t* keep, int32_t num_in, void* out, int64_t ldo,
                          float* scratch, int64_t ld_scratch, void* stream);
/* over the forward CSR g, with G = grad [N_in, d] the gradient of out: the paired rows dkg [N_in] get
 *   dk[v] = G[v] sum_u sigmoid'(x) val[u]  at [0, d),   a copy of G[v]  at [half, half + d)
 * (the [dk | G] operand of the input-gradient GEMM).  ld_scratch >= d */
int pg_resgated_bwd_dst(const pg_csr* g, const void* qv, int64_t ldqv, const void* ks, int64_t ldks, int32_t half,
                        const void* grad, int64_t ldg, int32_t d, int dtype, const uint8_t* keep, int32_t num_in,
                        void* dkg, int64_t lddkg, float* scratch, int64_t ld_scratch, void* stream);
/* over the CSC row u of gt (rows = all num_all `_U` rows, entries the destinations v of u): the paired rows dqv get
 *   dq[u] = val[u] sum_v G[v] sigmoid'(x)  at [0, d),   dval[u] = sum_v G[v] sigmoid(x)  at [half, half + d)
 * An unkept halo row, and a row without out-edges, get exact zeros (its val is not read).  ld_scratch >= 2 d */
int pg_resgated_bwd_src(const pg_csr* gt, const void* qv, int64_t ldqv, const void* ks, int64_t ldks, int32_t half,
                        const void* grad, int64_t ldg, int32_t d, int dtype, const uint8_t* keep, int32_t num_in,
                        void* dqv, int64_t lddqv, float* scratch, int64_t ld_scratch, void* stream);

/* ------------------------------------------------------------------------------------------
 * Symmetric heap: device memory that peers map through CUDA IPC (host pointers out).
 * ---------------------------------------------------------------------------------------- */
#define PG_IPC_HANDLE_BYTES 64
int pg_heap_alloc(size_t bytes, void** ptr);
int pg_heap_free(void* ptr);
int pg_ipc_export(void* ptr, unsigned char* handle);
int pg_ipc_import(const unsigned char* handle, void** ptr);
int pg_ipc_close(void* ptr);
int pg_enable_peer_access(int peer_device);

#ifdef __cplusplus
}
#endif
#endif /* PIPEGCN_B200_H */
