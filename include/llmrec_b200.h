/*
 * llmrec_b200 -- C ABI of the H100 (sm_90a) kernels behind the LLMRec training-and-eval hot path.
 *
 * Boundary contract (SURVEY.md section 8b): the reference has no FFI layer -- its boundary is the
 * Python API (MM_Model.forward, Trainer.bpr_loss/prune_loss, AdamW.step, test_torch).  These entry
 * points are what a ctypes/cffi binding of that API binds: plain device pointers, sizes and a
 * cudaStream_t.  No torch types.  Conventions:
 *   - every pointer is a DEVICE pointer unless the name ends in _host;
 *   - all matrices are row-major fp32 with an explicit leading dimension (elements), except the side-feature table X of the
 *     _bf16 projection entry points: raw bfloat16 bits (uint16_t), row-major, leading dimension in elements; and of the _i8
 *     entry points: the row-scaled int8 format described there, row pitch in bytes;
 *   - index arrays are int32 (CSR rowptr/col; nnz < 2^31) unless stated;
 *   - nothing is allocated, nothing synchronises the host; work is enqueued on `stream`;
 *   - return 0 on success, non-zero on error; llmrec_last_error() gives the message
 *     (the reference's only error convention is Python exceptions / sys.exit on NaN, main.py:287-289).
 * Reference citations are file:line into HKUDS/LLMRec @ 169f3614.
 */
#ifndef LLMREC_B200_H
#define LLMREC_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* llmrec_stream_t; /* cudaStream_t */

#define LLMREC_ABI_VERSION 2
#define LLMREC_MAX_SEG 16

int llmrec_abi_version(void);
const char* llmrec_last_error(void);
/* 1 when the running device is sm_90 (H100); kernels refuse to launch otherwise. */
int llmrec_device_ok(void);

/* ---------------------------------------------------------------------------------------------
 * Propagation SpMM.  Replaces torch.sparse.mm / torch.mm(COO, dense) at Models.py:57-61,152-183
 * (20 calls per forward) and their autograd transposes.
 *
 *   Y_s[r,:] (+)= epi( rs[r] * sum_{e in row r} v[e] * cs[col[e]] * X_s[col[e],:] )     s = 0..nseg-1
 *
 * One launch propagates `nseg` dense operands that share the sparsity pattern (the image / text /
 * 5 attribute / profile / ID operands of one graph direction), reading the index stream once.
 * vals, row_scale, col_scale may each be NULL (= 1).  The Trainer's graphs are binary patterns with
 * rs = (deg+1e-8)^-1/2 (main.py:114-126), so vals == NULL there.
 * seg flags: bit0 = row softmax over the d columns after scaling (Models.py:174-175); the optional
 * addend Z is added after the epilogue (used by the backward chain: g_out = g_direct + A^T g).
 * Work decomposition: `tiling` (required for the vectorised kernels; NULL falls back to the scalar
 * warp-per-row kernel) lists nnz-bounded tiles so that low-degree rows are batched and power-law rows are
 * split over several warps and reduced by a deterministic second pass.
 * --------------------------------------------------------------------------------------------- */
typedef struct {
  const float* X;   /* gathered operand  [n_cols x d], leading dimension ldx */
  float* Y;         /* output            [n_rows x d], ldy */
  const float* Z;   /* optional addend   [n_rows x d], ldz: Y = epi(...) + Z  (Z == Y accumulates in place) */
  int64_t ldx;
  int64_t ldy;
  int64_t ldz;
  int32_t flags;    /* LLMREC_SPMM_SOFTMAX */
  int32_t _pad;
} llmrec_spmm_seg;

typedef struct {
  const int32_t* tiles;       /* [n_tiles][8] = {first row, #complete rows (0 = one piece of a long row), e0, e1} followed by
                                 16 one-byte row-end offsets relative to e0 (pieces: {split index, first piece, #pieces, 0} instead);
                                 32-byte aligned; pieces of long rows are numbered first (llmrec_spmm_plan_tiles builds this) */
  const int32_t* split_row;   /* [n_split] rows that were cut into pieces */
  const int32_t* split_first; /* [n_split+1] first piece (tile id) of each split row */
  float* scratch;             /* [n_split_tiles * min(nseg,16) * d] partial sums of the pieces */
  int32_t n_tiles, n_split, n_split_tiles, _pad;
  int32_t* split_tickets;     /* optional int32[n_split * 64], zeroed once: with it the LAST piece of a long row to finish adds the row's
                                 pieces (in piece order) and runs the epilogue inside the same launch; NULL = second-pass kernel */
  const uint32_t* src_mask;   /* optional bitmask over SOURCE rows (= pattern columns): a clear bit promises that row of X is all zero;
                                 its fetch is skipped (identical sums).  NULL = every row is live. */
} llmrec_spmm_tiling;

/* Host-side planner (runs once per graph): tiles of <= tile_nnz (8..248) non-zeros, each a run of <= max_rows (<= 15)
 * complete rows or one piece of a longer row.  Call with tiles_out == NULL to get the sizes in
 * counts_out = {n_tiles, n_split, n_split_tiles}, allocate, call again.  All pointers are HOST memory. */
int llmrec_spmm_plan_tiles(const int32_t* rowptr_host, int32_t n_rows, int32_t tile_nnz, int32_t max_rows,
                           int32_t* tiles_out, int32_t* split_row_out, int32_t* split_first_out, int32_t* counts_out);

#define LLMREC_SPMM_SOFTMAX 1

int llmrec_spmm_csr_f32(const int32_t* rowptr, const int32_t* col, const float* vals,
                        const float* row_scale, const float* col_scale,
                        int32_t n_rows, int32_t n_cols, int32_t d,
                        const llmrec_spmm_seg* segs_host, int32_t nseg,
                        const llmrec_spmm_tiling* tiling_host, llmrec_stream_t stream);

/* Row-LIST form of the same product: only rows[0 .. *n_rows_dev) (device list, device-side length, capped at max_rows; entries < 0 skipped)
 * are computed and written; all other rows of Y are left untouched.  One segment, d in {32, 64, 128}.  For the products of a training
 * step that are provably consumed on a small row subset (the last propagation layer reaches the loss only through the batch's
 * neighbourhood -- dist.py "demand" mode).  Persistent grid, no host synchronisation. */
int llmrec_spmm_rows_f32(const int32_t* rowptr, const int32_t* col, const float* vals, const float* row_scale, const float* col_scale,
                         int32_t d, const llmrec_spmm_seg* seg_host, const int32_t* rows, const int32_t* n_rows_dev, int32_t max_rows,
                         const uint32_t* src_mask, int32_t cta_per_row /* 1: one CTA per listed row -- short lists of possibly very long rows */,
                         llmrec_stream_t stream);
int llmrec_row_softmax_bwd_rows_f32(const float* S, int64_t lds, const float* dS, int64_t ldds, float* dX, int64_t lddx,
                                    const int32_t* rows, const int32_t* n_rows_dev, int32_t max_rows, int32_t d, llmrec_stream_t stream);
/* Device-side row sets: mask |= {col[e] : e in rows list[.] of the CSR}, mask |= {ids}, and mask -> (unordered) id list with *count += #bits. */
int llmrec_mark_neighbors(const int32_t* rowptr, const int32_t* col, const int32_t* list, int32_t n_list, uint32_t* mask, llmrec_stream_t stream);
int llmrec_mark_ids(const int32_t* ids, int32_t n, uint32_t* mask, llmrec_stream_t stream);
/* mask |= {ids[0 .. min(*n_dev, max_n))}: the live length is read from device memory (a captured step's B', the first word of its meta row). */
int llmrec_mark_ids_rows(const int32_t* ids, const int32_t* n_dev, int32_t max_n, uint32_t* mask, llmrec_stream_t stream);
int llmrec_compact_mask(const uint32_t* mask, int32_t n_bits, int32_t* list_out, int32_t* count, llmrec_stream_t stream);
int llmrec_zero_rows_f32(float* Y, int64_t ldy, const int32_t* idx, int32_t n, int32_t d, llmrec_stream_t stream);
int llmrec_assign_rows_f32(const float* G, int64_t ldg, const int32_t* idx, int32_t n, int32_t d, float* Y, int64_t ldy, llmrec_stream_t stream);
/* Dense AdamW over one [n_rows x width] table whose gradient is row-sparse: g is read only where row_mask has the row's bit set. */
int llmrec_adamw_step_rows_f32(float* p, const float* g, float* m, float* v, int64_t n_rows, int32_t width, const uint32_t* row_mask,
                               const double* state, float lr, float beta1, float beta2, float eps, float weight_decay, llmrec_stream_t stream);

/* Row softmax Y = softmax(X, dim=-1) and its backward dX = S*(dS - sum(dS*S)) (Models.py:174-175). */
int llmrec_row_softmax_f32(const float* X, int64_t ldx, float* Y, int64_t ldy, int64_t n, int32_t d, llmrec_stream_t stream);
int llmrec_row_softmax_bwd_f32(const float* S, int64_t lds, const float* dS, int64_t ldds, float* dX, int64_t lddx,
                               int64_t n, int32_t d, llmrec_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Side-feature projection  Y = X W^T + b   (nn.Linear at Models.py:145-150; 8 per forward) and its
 * weight gradient dW = dY^T X, db = colsum(dY) (autograd of the same; features are constants so
 * there is no dX).  X:[n x k] ldx, W:[d x k] (nn.Linear layout), Y:[n x d] ldy.
 * mode: 0 = wgmma 3xTF32 (fp32-accurate, default), 1 = wgmma 1xTF32, 2 = exact fp32 SIMT.
 * --------------------------------------------------------------------------------------------- */
int llmrec_proj_fwd_f32(const float* X, int64_t ldx, const float* W, const float* bias,
                        float* Y, int64_t ldy, int64_t n, int32_t k, int32_t d, int32_t mode,
                        float* wsplit /* 2*d*k floats, mode 0 only */, llmrec_stream_t stream);
int llmrec_proj_wgrad_f32(const float* X, int64_t ldx, const float* dY, int64_t lddy,
                          float* dW, float* db, int64_t n, int32_t k, int32_t d, int32_t accumulate,
                          int32_t mode, float* scratch, int64_t scratch_elems, llmrec_stream_t stream);
/* scratch elements needed by llmrec_proj_wgrad_f32 for this shape/mode */
int64_t llmrec_proj_wgrad_scratch(int64_t n, int32_t k, int32_t d, int32_t mode);

/* Grouped forms: all projections of one step (image, text, user, 5 attribute tables) in ONE persistent
 * launch.  Problems that share W (the 5 attribute tables use item_trans) share `wsplit`; wgrad problems
 * that share dW/db list them in order with accumulate = 1 after the first. */
typedef struct {
  const float* X; const float* W; const float* bias; float* Y; float* wsplit;
  int64_t ldx, ldy, n;
  int32_t k, _reserved;       /* flags: 0 or LLMREC_PROJ_ROW_MAP */
} llmrec_proj_fwd_problem;
typedef struct {
  const float* X; const float* dY; float* dW; float* db;
  int64_t ldx, lddy, n;
  int32_t k, accumulate;      /* flags: LLMREC_WGRAD_ACCUMULATE | LLMREC_PROJ_ROW_MAP */
} llmrec_proj_wgrad_problem;
#define LLMREC_WGRAD_ACCUMULATE 1
int llmrec_proj_fwd_group_f32(const llmrec_proj_fwd_problem* probs_host, int32_t n_prob, int32_t d, int32_t mode,
                              llmrec_stream_t stream);
int llmrec_proj_wgrad_group_f32(const llmrec_proj_wgrad_problem* probs_host, int32_t n_prob, int32_t d, int32_t mode,
                                float* scratch /* zero-initialised ONCE by the caller: its FIRST word is a ticket the kernels leave at zero */,
                                int64_t scratch_elems, llmrec_stream_t stream);
/* Stream note: when any problem has db != NULL, the bias column sums (they read dY only) are enqueued on a library-owned side
 * stream forked from `stream` with an event and joined back into it before the call returns, so they overlap the persistent
 * weight-gradient kernel; inside a stream capture this becomes a parallel graph branch.  One side stream + two events per device,
 * created on first use (the only objects the library ever creates); LLMREC_BRANCHES=0 keeps everything on `stream`. */
int64_t llmrec_proj_wgrad_group_scratch(const llmrec_proj_wgrad_problem* probs_host, int32_t n_prob, int32_t d, int32_t mode);

/* bf16 feature tables (--feat_dtype bf16): the same grouped projections with X as raw bfloat16 bits (row-major, leading dimension
 * ldx in ELEMENTS); W, bias, Y, dY, dW, db stay fp32.  The result is what the fp32 entry points compute on the upcast table:
 *   mode 0: W (forward) / dY (weight gradient) split EXACTLY into three bf16 terms t0 + t1 + t2 (t0 = trunc_bf16(v), t1 =
 *           trunc_bf16(v - t0), t2 = the rest, bf16-exact); a bf16 X needs no split, every bf16 x bf16 product is exact in fp32,
 *           so only the accumulation rounds (fp32-class, no product term dropped);
 *   mode 1: one bf16 wgmma, W / dY truncated to bf16;
 *   mode 2: the exact SIMT kernels with X widened on load (forward bit-identical to mode 2 on the upcast table; the weight
 *           gradient too, up to the order of its atomics across 1024-row chunks).
 * The tensor-core path takes d = 32..256 in steps of 32, k % 8 == 0, ldx % 8 == 0 and a 16-byte aligned X; other shapes run
 * the SIMT kernels.  `wsplit` (2*d*k floats, holding the 3*d*k bf16 terms) is needed in modes 0 AND 1.  Scratch, accumulate,
 * grouping and the side-stream bias sums are as for the _f32 forms. */
typedef struct {
  const uint16_t* X; const float* W; const float* bias; float* Y; float* wsplit;
  int64_t ldx, ldy, n;
  int32_t k, _reserved;       /* flags: 0 or LLMREC_PROJ_ROW_MAP */
} llmrec_proj_fwd_problem_bf16;
typedef struct {
  const uint16_t* X; const float* dY; float* dW; float* db;
  int64_t ldx, lddy, n;
  int32_t k, accumulate;      /* flags: LLMREC_WGRAD_ACCUMULATE | LLMREC_PROJ_ROW_MAP */
} llmrec_proj_wgrad_problem_bf16;
int llmrec_proj_fwd_group_bf16(const llmrec_proj_fwd_problem_bf16* probs_host, int32_t n_prob, int32_t d, int32_t mode,
                               llmrec_stream_t stream);
int llmrec_proj_wgrad_group_bf16(const llmrec_proj_wgrad_problem_bf16* probs_host, int32_t n_prob, int32_t d, int32_t mode,
                                 float* scratch /* zero-initialised ONCE, as for llmrec_proj_wgrad_group_f32 */,
                                 int64_t scratch_elems, llmrec_stream_t stream);
int64_t llmrec_proj_wgrad_group_bf16_scratch(const llmrec_proj_wgrad_problem_bf16* probs_host, int32_t n_prob, int32_t d, int32_t mode);

/* int8 feature tables (--feat_dtype int8): the same grouped projections with X in a row-scaled 8-bit format.  Row r of a table with
 * logical width k is ldx BYTES long (the row pitch; at least roundup(k, 16) + 4 and a multiple of 4, roundup(k, 16) + 16 as built by
 * llmrec_b200/feat_int8.py) and holds
 *   bytes [0, k)                       the int8 values q (|q| <= 127),
 *   bytes [k, roundup(k, 16))          zero,
 *   bytes [roundup(k, 16), +4)         the row's fp32 scale 2^e, e in [-126, 120] (1 for an all-zero row),
 *   the rest of the row                zero.
 * Every stored value x~ = q * 2^e is exactly a bf16 number, so the table is a lossless encoding of one bf16 table X~, and the results are
 * BIT-IDENTICAL to the _bf16 entry points on X~ in every mode: the tensor-core path loads the raw q by TMA and expands q * 2^e to bf16 in
 * shared memory, in the exact layout the bf16 kernels load, before the same wgmma consumers read it; the SIMT kernels widen q * 2^e on
 * load.  k is the logical width; W, bias, Y, dY, dW, db stay fp32.  The tensor-core path takes d = 32..256 in steps of 32, k % 16 == 0,
 * ldx % 16 == 0 and a 16-byte aligned X; other shapes run the SIMT kernels.  `wsplit`, scratch, row maps, accumulate, grouping and the
 * side-stream bias sums are as for the _bf16 forms. */
typedef struct {
  const int8_t* X; const float* W; const float* bias; float* Y; float* wsplit;
  int64_t ldx, ldy, n;        /* ldx: row pitch of X in bytes */
  int32_t k, _reserved;       /* flags: 0 or LLMREC_PROJ_ROW_MAP */
} llmrec_proj_fwd_problem_i8;
typedef struct {
  const int8_t* X; const float* dY; float* dW; float* db;
  int64_t ldx, lddy, n;       /* ldx: row pitch of X in bytes */
  int32_t k, accumulate;      /* flags: LLMREC_WGRAD_ACCUMULATE | LLMREC_PROJ_ROW_MAP */
} llmrec_proj_wgrad_problem_i8;
int llmrec_proj_fwd_group_i8(const llmrec_proj_fwd_problem_i8* probs_host, int32_t n_prob, int32_t d, int32_t mode,
                             llmrec_stream_t stream);
int llmrec_proj_wgrad_group_i8(const llmrec_proj_wgrad_problem_i8* probs_host, int32_t n_prob, int32_t d, int32_t mode,
                               float* scratch /* zero-initialised ONCE, as for llmrec_proj_wgrad_group_f32 */,
                               int64_t scratch_elems, llmrec_stream_t stream);
int64_t llmrec_proj_wgrad_group_i8_scratch(const llmrec_proj_wgrad_problem_i8* probs_host, int32_t n_prob, int32_t d, int32_t mode);

/* Row maps, for X tables that hold a subset of the output's rows (the training step projects only the items with a training edge,
 * from compact copies of the item tables).  A problem whose flags word -- `_reserved` of the forward problem, `accumulate` of the
 * weight-gradient problem, _f32, _bf16 and _i8 -- has LLMREC_PROJ_ROW_MAP set takes a map from an llmrec_proj_row_map record.  The
 * records follow the n_prob problems in the same host array, one per problem in order (records of unflagged problems are ignored);
 * callers that never set the bit pass plain problem arrays as before.  rows: a DEVICE int32 list of the problem's n X rows, every
 * entry a valid row of Y / dY:
 *   forward          X row r is written to Y[rows[r]]; Y rows not in the map are left untouched.  Each written row gets the bits
 *                    of the same X row in an unmapped call (the per-row arithmetic is unchanged);
 *   weight gradient  X row r pairs with dY[rows[r]]: dW (+)= sum_r dY[rows[r]]^T X[r].  The bias sums db (+)= colsum(dY) run over
 *                    ALL n_dy rows of dY, so db gets the bits of an unmapped call on the full tables; dW differs from that call by
 *                    rounding only (the row chunks see another row sequence).
 * The _scratch queries take the same arrays (n = the X row count). */
typedef struct {
  const int32_t* rows;
  int64_t n_dy;               /* weight gradient: row count of dY (the bias sums run over all of them); unused by the forward */
} llmrec_proj_row_map;
#define LLMREC_PROJ_ROW_MAP 2

/* ---------------------------------------------------------------------------------------------
 * Fusion (Models.py:185-197):  out = mean(layer_0..layer_{L}) + sum_t coef[t] * x_t / max(||x_t||_2, 1e-12)
 * and its backward: d layer_l = g/(L+1) (written once to d_layer, may be NULL);
 * d x_t (+)= coef[t] * (g - y_t (y_t . g)) / max(||x_t||,1e-12),  y_t = x_t/max(||x_t||,1e-12).
 * Pointer tables are HOST arrays (copied into the launch parameters).
 * --------------------------------------------------------------------------------------------- */
/* rows: optional int32 device list of row ids to process (NULL = rows 0..n-1; n = list length otherwise).  Entries < 0 are skipped:
 * nothing is read or written for them, forward and backward.
 * llmrec_fuse_fwd_f32 with rows != NULL and n < 0: COMPACT form over |n| list entries -- the layer tables are read at rows[b], the
 * side operands and `out` at the compact position b (side features projected on the batch's rows only, hoisted mode); a negative
 * entry gives a zero row of `out`. */
int llmrec_fuse_fwd_f32(const float* const* layers_host, const int64_t* ld_layers_host, int32_t n_layers,
                        const float* const* sides_host, const int64_t* ld_sides_host, const float* coef_host,
                        int32_t n_sides, float* out, int64_t ldo, const int32_t* rows, int64_t n, int32_t d,
                        llmrec_stream_t stream);
int llmrec_fuse_bwd_f32(const float* g, int64_t ldg, int32_t n_layers, float* d_layer, int64_t lddl,
                        const float* const* sides_host, const int64_t* ld_sides_host, const float* coef_host,
                        float* const* d_sides_host, const int64_t* ld_dsides_host, int32_t n_sides,
                        int32_t accumulate, const int32_t* rows, int64_t n, int32_t d, llmrec_stream_t stream);
/* Row-LIST forms with a device-side length: only rows[0 .. min(*n_rows_dev, max_rows)) are processed (entries < 0 skipped), each by the
 * same per-row code as the full form, so a listed row gets the same bits; every other row of out / d_layer / d_sides is left untouched.
 * The grid is sized for max_rows, no host synchronisation.  The training step fuses only its batch's rows with these (the loss reads
 * U / I there only, and the fused-output gradient is zero elsewhere); a row listed twice would be accumulated twice by the backward. */
int llmrec_fuse_fwd_rows_f32(const float* const* layers_host, const int64_t* ld_layers_host, int32_t n_layers,
                             const float* const* sides_host, const int64_t* ld_sides_host, const float* coef_host,
                             int32_t n_sides, float* out, int64_t ldo, const int32_t* rows, const int32_t* n_rows_dev, int32_t max_rows,
                             int32_t d, llmrec_stream_t stream);
int llmrec_fuse_bwd_rows_f32(const float* g, int64_t ldg, int32_t n_layers, float* d_layer, int64_t lddl,
                             const float* const* sides_host, const int64_t* ld_sides_host, const float* coef_host,
                             float* const* d_sides_host, const int64_t* ld_dsides_host, int32_t n_sides, int32_t accumulate,
                             const int32_t* rows, const int32_t* n_rows_dev, int32_t max_rows, int32_t d, llmrec_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * BPR + prune heads (main.py:330-342 bpr_loss, :158-165 prune_loss, :232-254 the 8 heads).
 * For head h with user matrix XU_h and item matrix XI_h (row-major, ld):
 *   x_b   = <XU[u_b], XI[p_b]> - <XU[u_b], XI[n_b]>;  maxi_b = logsigmoid(x_b + 1e-8)
 *   keep  = the int((1-drop_rate)*B) smallest maxi (ties -> lower b);  mf_h = -mean(maxi[keep])
 *   emb_h = regs0/batch_size * sum_{t in u,p,n} 1/(2*sum||row_t||^2 + 1e-8)
 * loss += w_mf[h]*mf_h + w_emb[h]*emb_h.  Gradients w.r.t. the gathered rows are scatter-added
 * (atomicAdd) into GU_h / GI_h (same shapes as XU_h / XI_h; NULL = skip that head's grads).
 * out_host-visible results live in `out` (device, 4 floats per head: mf, emb, kept, _) .
 * idx are int32 device arrays of length B.  `n_keep` = int((1-drop_rate)*B) computed by the caller
 * in double arithmetic like the reference (main.py:161-162).
 * `meta` (may be NULL): DEVICE int32[2] = {live B', n_keep}.  When given, B is only the CAPACITY the launch is sized
 * for (index arrays and `work` hold B entries) and the kernels read the live length and n_keep from `meta` -- one
 * captured CUDA graph then serves every batch length <= B (the augmented-edge filter makes B' vary per step).
 * Two launches: score + per-head radix select of the kept set (ties -> lower position) + loss; scatter of row gradients.
 * --------------------------------------------------------------------------------------------- */
typedef struct {
  const float* XU; const float* XI;
  float* GU; float* GI;
  int64_t ldxu, ldxi, ldgu, ldgi;
  float w_mf, w_emb;
} llmrec_bpr_head;

int llmrec_bpr_heads_f32(const llmrec_bpr_head* heads_host, int32_t n_heads,
                         const int32_t* users, const int32_t* pos, const int32_t* neg, int32_t B,
                         int32_t n_keep, const int32_t* meta, float regs0_over_bs, int32_t d,
                         float* out /* [n_heads*4] */, float* loss_accum /* [1], += */,
                         float* work /* llmrec_bpr_work_elems() floats, zeroed once */, llmrec_stream_t stream);
int64_t llmrec_bpr_work_elems(int32_t n_heads, int32_t B);

/* Ordered (bit-reproducible) form of the heads' row gradients.  Forward values (`out`, loss) are those of llmrec_bpr_heads_f32;
 * the row gradients are gathered instead of scattered with float atomics.  Definition of the result: every element G[row, j]
 * starts from the value it holds at the call (what llmrec_grad_init_f32 left: zero, or c * X) and takes its contributions one
 * fp32 add at a time (each add flushes denormals, as the device's float atomic does), in this order:
 *   1. heads in ascending index;  2. within a head, ascending batch position b;  3. at one position, pos[b] before neg[b].
 * Each contribution is computed by the instructions of the atomic form, and its early-outs are kept (a triplet with g == 0 of a
 * head with w_emb == 0 adds nothing; a head with GU == GI == NULL is skipped), so a row with one contribution gets the atomic
 * form's bits and every result is one the atomic form could have produced.  The bits do not depend on the grid, the stream
 * schedule or timing.  Heads that accumulate into one buffer must name it by the same pointer and leading dimension (the
 * attribute heads' shared Gprof_u); gradient buffers of different pointers must not overlap.
 * llmrec_bpr_slot_plan sorts the batch's slots -- user slots b; item slots 2b (pos) and 2b + 1 (neg) -- by (row, slot) into
 * `plan` (llmrec_bpr_slot_plan_elems(B) int32).  It reads the index arrays (and meta[0]) only, so it may run on another stream
 * as soon as they are staged; the ordered call must be ordered after it.  B is the capacity as above; entries past the live
 * length are never read.  Capacity: B <= 65536 triplets (an argument error above; there is no fall-back to the atomic form).
 * Any d and leading dimensions; a row that occurs many times in one batch is walked by one warp per destination buffer. */
int64_t llmrec_bpr_slot_plan_elems(int32_t B);
int llmrec_bpr_slot_plan(const int32_t* users, const int32_t* pos, const int32_t* neg, int32_t B, const int32_t* meta,
                         int32_t* plan, llmrec_stream_t stream);
int llmrec_bpr_heads_ordered_f32(const llmrec_bpr_head* heads_host, int32_t n_heads,
                                 const int32_t* users, const int32_t* pos, const int32_t* neg, int32_t B,
                                 int32_t n_keep, const int32_t* meta, float regs0_over_bs, int32_t d,
                                 float* out /* [n_heads*4] */, float* loss_accum /* [1], += */,
                                 float* work /* llmrec_bpr_work_elems() floats, zeroed once */,
                                 const int32_t* plan /* llmrec_bpr_slot_plan of the same index arrays */, llmrec_stream_t stream);

/* First touch of every gradient buffer of a step, one launch instead of a memset per buffer: region r is written
 * G_r[n x width] = X_r ? c_r * X_r : 0, and *loss = sum_r 0.5 * c_r * sum(X_r^2) (OVERWRITTEN: this is the first term of
 * the step's loss) -- feat_reg_loss_calculation (main.py:151-156) and its gradient for the regions with X, plain zeroing
 * for the buffers the BPR heads scatter-add into.  <= 16 regions (128-bit accesses when width / ld % 4 == 0 and aligned).
 * scratch: llmrec_grad_init_scratch() floats, zeroed once by the caller (the kernel leaves its ticket at zero). */
typedef struct {
  float* G; const float* X;
  int64_t ldg, ldx, n;
  int32_t width; float c;
} llmrec_grad_region;
int llmrec_grad_init_f32(const llmrec_grad_region* regions_host, int32_t n_regions, float* loss, float* scratch, llmrec_stream_t stream);
int64_t llmrec_grad_init_scratch(void);

/* feat_reg_loss_calculation (main.py:151-156): loss += c * 0.5*sum(X^2) ; G = (accumulate? G:0) + c*X.
 * G may be NULL (loss only). */
int llmrec_sqnorm_grad_f32(const float* X, int64_t ldx, float* G, int64_t ldg, int64_t n, int32_t d,
                           float c, int32_t accumulate, float* loss_accum, float* partial /* >= 1024 floats */,
                           llmrec_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Dense AdamW over a list of tensors (torch.optim.AdamW defaults at main.py:100-104,278:
 * decoupled weight decay, bias correction).  `state` is a device block of 4 doubles
 * {step, lr/bc1, sqrt(bc2), _}; llmrec_adamw_advance increments step and recomputes the scalars
 * on device (CUDA-graph friendly).  Tensor tables are HOST arrays.
 * --------------------------------------------------------------------------------------------- */
int llmrec_adamw_advance(double* state, double lr, double beta1, double beta2, llmrec_stream_t stream);
int llmrec_adamw_step_f32(float* const* p_host, const float* const* g_host, float* const* m_host, float* const* v_host,
                          const int64_t* numel_host, int32_t n_tensors, const double* state,
                          float lr, float beta1, float beta2, float eps, float weight_decay,
                          llmrec_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Full-catalog scoring + top-K (utility/batch_test.py:149-152 scores, :21-36,100-102 ranking).
 *   score[b,i] = <U[users[b]], I[i]>;  train items of the user are excluded; top-K by score,
 *   ties -> lowest item id (heapq.nlargest over ascending candidates).
 * mask CSR: mask_rowptr int32[n_users_total+1], mask_col int32 with every row SORTED ASCENDING (the fused
 * selection walks it with a merge pointer).  users = int32[b].
 * out_idx int32 [b x K], out_val fp32 [b x K] (may be NULL; exact fp32 scores).  K <= 64.
 * mode: 0 = wgmma 3xTF32 scoring with the select fused into the epilogue + exact fp32 rescoring of the
 *           K+16.. candidates (d in {32,64,96,128}); 2 = exact fp32 SIMT.  Both return the same lists unless two
 *           scores closer than the TF32x3 rounding (~1e-5 relative) straddle rank K+16.
 * --------------------------------------------------------------------------------------------- */
int llmrec_score_topk_f32(const float* U, int64_t ldu, const float* I, int64_t ldi,
                          const int32_t* users, int32_t n_batch, int32_t n_items, int32_t d,
                          const int32_t* mask_rowptr, const int32_t* mask_col,
                          int32_t K, int32_t* out_idx, float* out_val, int32_t mode,
                          float* scratch, int64_t scratch_elems, llmrec_stream_t stream);
int64_t llmrec_score_topk_scratch(int32_t n_batch, int32_t n_items, int32_t d, int32_t K, int32_t mode);

/* Top-K over a catalog given by ids: llmrec_score_topk_f32 with the catalog replaced by the rows
 * among[0 .. n_among) of I.  among int32 STRICTLY ASCENDING, every id a row of I (not checked on the
 * device).  Mask rows and out_idx hold GLOBAL item ids (rows of I); a masked id outside `among` is
 * ignored.  Ties -> lowest global id; fewer than K survivors padded with -1 / -inf.  K is 1..64 and
 * <= n_among.  Same modes and the same returned score bits as llmrec_score_topk_f32: mode 0 gathers
 * the hi/lo copies of the n_among rows into the scratch, mode 2 scores a [b x n_among] block.  Called
 * with among = 0..n_items-1 it returns what llmrec_score_topk_f32 returns. */
int llmrec_score_topk_among_f32(const float* U, int64_t ldu, const float* I, int64_t ldi,
                                const int32_t* users, int32_t n_batch, const int32_t* among, int32_t n_among, int32_t d,
                                const int32_t* mask_rowptr, const int32_t* mask_col,
                                int32_t K, int32_t* out_idx, float* out_val, int32_t mode,
                                float* scratch, int64_t scratch_elems, llmrec_stream_t stream);
int64_t llmrec_score_topk_among_scratch(int32_t n_batch, int32_t n_among, int32_t d, int32_t K, int32_t mode);

/* Top-K for groups of users who choose together.  Group g's members are the rows
 * members[member_rowptr_host[g] .. member_rowptr_host[g+1]) of U: 1..64 per group (64 = one wgmma M tile; a group
 * never straddles a tile), ascending and distinct by the caller's convention (not checked; the order is
 * the summation order of mean).  member_rowptr_host is a HOST int32 [n_groups+1] array: the tile plan is built
 * from it and copied into the scratch from pageable memory, so unlike the other entry points this call waits
 * for the stream's earlier work before it returns.  members is device int32.  Let s(u, i) be the sequential fp32 FMA
 * chain of llmrec_score_pairs_f32.  The group score of item i is, by agg:
 *   LLMREC_AGG_MEAN: the fp32 sum 0 + s(u_0, i) + s(u_1, i) + ... in member order, then one IEEE fp32
 *                    division by the member count;
 *   LLMREC_AGG_MIN / LLMREC_AGG_MAX: the exact minimum / maximum; a NaN member score makes it NaN.
 * The catalog is I (among NULL, n_items rows) or the rows among[0 .. n_items) of I (STRICTLY ASCENDING,
 * as for llmrec_score_topk_among_f32).  Mask rows are indexed by GROUP (mask_rowptr int32[n_groups+1],
 * rows sorted ascending, NULL = no mask) and hold global ids.  out_idx int32 / out_val fp32 [n_groups x K]
 * by (group score desc, id asc); NaN and -inf group scores are never returned; short rows padded with -1 /
 * -inf.  K is 1..64 and <= n_items.  mode 0: the member rows are packed into 64-row tiles, every member is
 * scored on the tensor cores (3xTF32), each group's approximate scores are aggregated by the same rule in
 * shared memory and selected with K+16.. slack, then the candidates are rescored exactly (d in
 * {32,64,96,128}, aligned operands; other shapes take mode 2); mode 2: exact fp32 SIMT.  Both return the
 * same ids and bits unless two group scores closer than the TF32x3 rounding straddle rank K+16.  In mode 2
 * a group's row does not depend on the other groups of the call; in mode 0 it does not either, unless such
 * near ties straddle the slack (the number of catalog slices, and so of candidates per group, follows the
 * number of tiles in the call, as for llmrec_score_topk_f32).  scratch: llmrec_score_topk_group_scratch
 * with the same member_rowptr_host. */
#define LLMREC_AGG_MEAN 0
#define LLMREC_AGG_MIN 1
#define LLMREC_AGG_MAX 2
int llmrec_score_topk_group_f32(const float* U, int64_t ldu, const float* I, int64_t ldi,
                                const int32_t* member_rowptr_host, const int32_t* members, int32_t n_groups,
                                const int32_t* among, int32_t n_items, int32_t d,
                                const int32_t* mask_rowptr, const int32_t* mask_col, int32_t K, int32_t agg,
                                int32_t* out_idx, float* out_val, int32_t mode,
                                float* scratch, int64_t scratch_elems, llmrec_stream_t stream);
int64_t llmrec_score_topk_group_scratch(const int32_t* member_rowptr_host, int32_t n_groups, int32_t n_items, int32_t d, int32_t K, int32_t mode);

/* hits[b,j] = 1 if out_idx[b,j] in truth row of users[b] (test_set membership, batch_test.py:30-34). */
int llmrec_topk_hits(const int32_t* idx, int32_t n_batch, int32_t K, const int32_t* users,
                     const int32_t* truth_rowptr, const int32_t* truth_col, uint8_t* hits,
                     llmrec_stream_t stream);

/* test_flag == 'full' (utility/batch_test.py:38-68, utility/metrics.py:95-100): per-user ROC-AUC of the exact fp32 scores over the
 * candidates (all items minus the user's mask row), positives = the user's truth row; 0 when either class is empty (the
 * reference swallows sklearn's ValueError).  mask / truth rows sorted ascending.  out_auc fp32[n_batch]. */
int llmrec_user_auc_f32(const float* U, int64_t ldu, const float* I, int64_t ldi, const int32_t* users, int32_t n_batch, int32_t n_items, int32_t d,
                        const int32_t* mask_rowptr, const int32_t* mask_col, const int32_t* truth_rowptr, const int32_t* truth_col,
                        float* out_auc, llmrec_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Scores of given pairs and re-ranking of given candidate lists (no full-catalog pass).  One score is
 * the sequential fp32 FMA chain a = 0; for j in 0..d-1: a = fmaf(U[u][j], I[i][j], a) -- the order of
 * both llmrec_score_topk_f32 modes' returned scores, so the same (u, i) gets the same bits.  Any d >= 1,
 * any leading dimensions.  Exact fp32 on the SIMT cores: each candidate row is read once per query.
 *
 * score_pairs: out[p] = <U[qrow[p]], I[item[p]]> for p < n (a negative id gives NaN; ids are otherwise
 *   rows of U / I).  out fp32[n].
 * rerank: query r (< m) scores every candidate cand_col[cand_rowptr[r] .. cand_rowptr[r+1]) against
 *   U[qrow[r]], drops ids outside [0, n_catalog) (-1 = padding), drops ids of mask row qrow[r] (mask_rowptr
 *   NULL: no mask; rows SORTED ASCENDING, as for score_topk), keeps one copy of a repeated id and writes the K
 *   best by (score desc, id asc) to out_idx int32 [m x K] / out_val fp32 [m x K].  A NaN score ranks after
 *   every number; a real candidate, even at -inf or NaN, ranks before padding; fewer than K survivors are
 *   padded with -1 / -inf.  K is 1..LLMREC_RERANK_MAX_K (the selection width); rows may be any length
 *   (a long row is streamed with a running top-K in shared memory).  No scratch, no host sync.
 * --------------------------------------------------------------------------------------------- */
#define LLMREC_RERANK_MAX_K 1024
int llmrec_score_pairs_f32(const float* U, int64_t ldu, const float* I, int64_t ldi, const int32_t* qrow, const int32_t* item,
                           int32_t n, int32_t d, float* out, llmrec_stream_t stream);
int llmrec_rerank_f32(const float* U, int64_t ldu, const float* I, int64_t ldi, const int32_t* qrow, int32_t m,
                      const int32_t* cand_rowptr, const int32_t* cand_col, const int32_t* mask_rowptr, const int32_t* mask_col,
                      int32_t n_catalog, int32_t d, int32_t K, int32_t* out_idx, float* out_val, llmrec_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Explanations: the exact split of scores <U[u], I[i]> over the query's history items and the model's
 * channels (id, then the n_side side terms of the fusion in order).  With ui = diag(su) R, every user-side
 * term but two is linear in the user's history: for history item j and target i,
 *   contrib[.., 0]     = ((sum_{l < n_id} dot(id_src[l][j], I[i])) * su) * inv            (0 when n_id = 0)
 *   contrib[.., 1 + t] = dot(side_src[t][j], I[i]) * ((coef[t] / max(sqrt(ss_t), 1e-12)) * su)
 *   own = dot(own_src[u], I[i]) * inv,   last = dot(last_src[u], I[i]) * inv,   inv = 1.0f / n_layers
 * where u = qrow[b], su = su[b], ss_t = the chain of x*x over side_usr[t][u] (the side row the fusion
 * normalised), id_src = Il[0 .. L-2] (n_id = L - 1, n_layers = L + 1), own_src = Ul[0], last_src = Ul[L],
 * and dot = the sequential chain a = 0; a = fmaf(x[k], y[k], a), k = 0..d-1, of llmrec_score_pairs_f32.
 * Every product and sum is one IEEE fp32 operation in the order written, so each output has exactly one
 * value, independent of the launch's grouping; own + last + sum contrib = <U[u], I[i]> up to the rounding of
 * the propagation sums and of the fusion.
 *
 * Query b (< m) has history hist_col[hist_rowptr[b] .. hist_rowptr[b+1]) (H_b item ids; the caller
 * collapses repeats) and targets targets[b * P .. b * P + P) (ids outside [0, n_catalog), e.g. -1, are
 * padding).  contrib fp32 [P * nnz_h x (1 + n_side)]: query b's block starts at row P * hist_rowptr[b] and
 * is [P x H_b x (1 + n_side)].  own / last fp32 [m x P].  A padding target gets zeros everywhere.
 * top_n = 0: no selection; 1..LLMREC_EXPLAIN_MAX_TOP: top_ids int32 / top_vals fp32 [m x P x top_n] hold
 * the top_n history items of each (query, target) with the largest total = sum of the channels in order
 * (fp32, from 0), by (total desc, id asc) with the keys of llmrec_rerank_f32, padded with -1 / -inf (a
 * padding target: -1 / 0).  Pointer tables (side_*, id_src, ld_*, coef) are host arrays.  No scratch, no
 * host sync; one launch, and a second one with top_n > 0.
 * --------------------------------------------------------------------------------------------- */
#define LLMREC_EXPLAIN_MAX_TOP 64
int llmrec_explain_f32(const float* own_src, int64_t ld_own, const float* last_src, int64_t ld_last,
                       const float* const* side_usr, const int64_t* ld_side_usr, const float* const* side_src,
                       const int64_t* ld_side_src, const float* coef, int32_t n_side, const float* const* id_src,
                       const int64_t* ld_id, int32_t n_id, const float* I, int64_t ldi, int32_t n_catalog, int32_t d,
                       int32_t n_layers, const int32_t* qrow, const float* su, int32_t m, const int32_t* hist_rowptr,
                       const int32_t* hist_col, const int32_t* targets, int32_t P, float* contrib, float* own, float* last,
                       int32_t top_n, int32_t* top_ids, float* top_vals, llmrec_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Diversified selection: greedy maximal marginal relevance over each query's pool of scored items.
 * Query b (< m) has the pool entries p < P: (pool_ids[b * ldp + p], pool_scores[b * ldp + p]); an id outside
 * [0, n_catalog) (e.g. -1) is padding, at any position.  X fp32 [n_catalog x d] holds the normalised catalog
 * rows (llmrec_row_normalize_f32), and cos(a, b) is the sequential chain c = 0; c = fmaf(X[a][j], X[b][j], c),
 * j = 0..d-1.  mu = 1.0f - lambda (one fp32 subtract).
 *   Round 1 picks the valid entry with the smallest key (s_p, id_p) in the order of llmrec_rerank_f32 (score
 *   desc, id asc, NaN last).  After each pick k, every unpicked entry with id_k retires (a repeated id is
 *   picked once) and every other one takes m_p = c when c = cos(id_p, id_k) > m_p (m_p starts at -inf; a NaN
 *   never replaces it).  Round t >= 2 picks the smallest key (obj_p, id_p), obj_p = lambda * s_p - mu * m_p
 *   (two fp32 multiplies and one subtract, each rounded once).  Equal keys go to the lower pool position.
 * Writes K entries per query in pick order: out_idx int32 / out_val fp32 (the pick's s) / out_sim fp32 (the
 * pick's m when picked; -inf for the first) [m x K], padded with -1 / -inf / -inf when fewer than K valid
 * distinct ids remain.  Every output is one exact fp32 value, independent of the launch's grouping.
 * 1 <= K <= P <= LLMREC_RERANK_MAX_K, 0 <= lambda <= 1.  One block per query; the pool's rows are kept in
 * shared memory when P * (d | 1) * 4 <= 110 KiB, else read from L2 each round.  No scratch, no host sync.
 * --------------------------------------------------------------------------------------------- */
int llmrec_diversify_f32(const float* X, int64_t ldx, const int32_t* pool_ids, const float* pool_scores, int64_t ldp,
                         int32_t m, int32_t P, int32_t n_catalog, int32_t d, int32_t K, float lambda,
                         int32_t* out_idx, float* out_val, float* out_sim, llmrec_stream_t stream);

/* Host-side (CPU, no GPU needed) BPR item sampler, bit-identical to Data.sample()'s numpy draws
 * (utility/load_data.py:166-187): hand over numpy's legacy MT19937 state (np.random.get_state()), get the
 * positives / rejection-sampled negatives for `users` and the advanced state back.  All pointers HOST. */
int llmrec_host_sample_items(uint32_t* mt_key /* [624] */, int32_t* mt_pos, const int32_t* users, int32_t n_users_in_batch,
                             const int32_t* train_rowptr, const int32_t* train_col, int32_t n_items,
                             int32_t* pos_out, int32_t* neg_out);

/* One whole training batch on the host, bit-identical to Data.sample() followed by the augmented-edge step of
 * main.py:213-224, written straight into a (pinned) [3 x ld] int32 staging buffer (rows: users, pos, neg):
 *   users    random.sample(exist_users, batch) -- or `batch` random.choice draws when batch > n_exist (load_data.py:158-161)
 *            -- from CPython's MT19937 stream (random.getstate(): key[624] + pos)
 *   pos/neg  the np.random.randint draws of llmrec_host_sample_items from numpy's legacy global stream
 *   aug      random.sample(users, n_aug) over the batch list; (u, aug_pos[u], aug_neg[u]) appended when both ids < aug_limit
 *            (the column count of train_mat, main.py:84-85,221);
 *            INT32_MIN in the tables = uid missing from augmented_sample_dict (KeyError upstream -> return 4)
 * `*_pool_branch` = which branch of CPython's sample() applies (n <= setsize), decided by the caller in Python arithmetic.
 * stamp: int32[n_exist] zero-initialised once, `epoch` > 0 and different on every call; pool: int32[max(n_exist if
 * users_pool_branch, 0) and >= batch + n_aug].  *n_out = batch + kept augmented edges.  All pointers HOST. */
int llmrec_host_sample_batch(uint32_t* py_key, int32_t* py_pos, uint32_t* np_key, int32_t* np_pos,
                             const int32_t* exist_users, int32_t n_exist, int32_t batch, int32_t users_pool_branch,
                             const int32_t* train_rowptr, const int32_t* train_col, int32_t n_items,
                             int32_t n_aug, int32_t aug_pool_branch, const int32_t* aug_pos, const int32_t* aug_neg,
                             int32_t n_aug_table, int32_t aug_limit, int32_t* stamp, int32_t epoch, int32_t* pool,
                             int32_t* out, int64_t ld, int32_t* n_out);

/* Device-side batch sampler (SURVEY.md 8f-1; utility/load_data.py:157-195 + main.py:216-224 on the GPU): ONE kernel fills the [4 x cap]
 * int32 index buffer of a training step -- rows users / pos / neg and the meta row {B', n_keep} looked up in meta_table[2*B' ..] -- from
 * DEVICE copies of exist_users, the train CSR (rows SORTED ascending) and the augmented-edge tables (ids < 0 or >= aug_limit are dropped,
 * as upstream's filter does; INT32_MIN = uid missing, and a missing uid or one >= n_aug_table is dropped too, where upstream raises
 * KeyError).  PRECONDITION, not checked here: every exist user has 1 <= deg < n_items (a train item to be the positive and an item left to
 * be the negative) and every train row is sorted ascending; DeviceSampler checks both on the host.  The negative is never a train item.
 * state = device uint64[2] {seed, step}; the kernel advances `step`, so the launch
 * can live inside a captured CUDA graph.  NOT bit-compatible with the reference's host RNG streams (that is llmrec_host_sample_batch, the
 * default): same distributions, counter-based generator.  key_scratch: uint32[max(n_exist, batch)]. */
int llmrec_device_sample_batch(const int32_t* exist_users, int32_t n_exist, int32_t batch,
                               const int32_t* train_rowptr, const int32_t* train_col, int32_t n_items,
                               int32_t n_aug, const int32_t* aug_pos, const int32_t* aug_neg, int32_t n_aug_table, int32_t aug_limit,
                               const int32_t* meta_table, int32_t cap, uint64_t* state, int32_t* out, uint32_t* key_scratch,
                               llmrec_stream_t stream);

/* Device-side batch sampler ON the reference's streams (`--device_sampler 2`): one launch draws exactly the batch of
 * llmrec_host_sample_batch (same arguments, same users / pos / neg / augmented triplets / B', both streams left in the same state) into the
 * [4 x cap] index buffer of llmrec_device_sample_batch.  train_col: the rows in the host sampler's order (the positive indexes them);
 * train_col_sorted: the same rows sorted ascending (negative rejection).  All pointers DEVICE.
 * state: int32[LLMREC_REF_SAMPLER_STATE_ELEMS] = { CPython `random` key[624], pos, numpy global MT19937 key[624], pos, error, pad }.
 * error != 0 (set by a call, or found on entry): the host sampler's return code (2 no train item, 3 no possible negative, 4 uid missing
 * from the augmentation tables; 5 a rejection loop passed 2^24 draws); both streams keep their state before the failing call, and every
 * call writes a batch of user 0 / item 0 with B' = batch until the host clears the word.
 * work: int32[llmrec_device_sample_batch_ref_work(...)] scratch (unused when it fits in shared memory). */
#define LLMREC_REF_SAMPLER_STATE_ELEMS 1252
int64_t llmrec_device_sample_batch_ref_work(int32_t n_exist, int32_t batch, int32_t users_pool_branch, int32_t aug_pool_branch);
int llmrec_device_sample_batch_ref(const int32_t* exist_users, int32_t n_exist, int32_t batch, int32_t users_pool_branch,
                                   const int32_t* train_rowptr, const int32_t* train_col, const int32_t* train_col_sorted,
                                   int32_t n_items, int32_t n_aug, int32_t aug_pool_branch, const int32_t* aug_pos, const int32_t* aug_neg,
                                   int32_t n_aug_table, int32_t aug_limit, const int32_t* meta_table, int32_t cap,
                                   int32_t* state, int32_t* out, int32_t* work, int64_t work_elems, llmrec_stream_t stream);

/* Row helpers of the sharded (multi-GPU) path: epilogue of an item-side propagation applied AFTER the cross-rank
 * sum of per-rank partials, and gather / scatter-add of batch rows by index (idx < 0 = row not owned: zeros / skipped). */
int llmrec_row_scale_softmax_f32(const float* X, int64_t ldx, const float* scale, float* Y, int64_t ldy, int64_t n, int32_t d,
                                 int32_t softmax, llmrec_stream_t stream);
int llmrec_gather_rows_f32(const float* X, int64_t ldx, const int32_t* idx, int32_t n, int32_t d, float* out, int64_t ldo,
                           llmrec_stream_t stream);
int llmrec_scatter_add_rows_f32(const float* G, int64_t ldg, const int32_t* idx, int32_t n, int32_t d, float* Y, int64_t ldy,
                                llmrec_stream_t stream);
/* Ordered form of llmrec_scatter_add_rows_f32: Y[idx[b], :] += G[b, :] one fp32 add at a time in ascending b (idx[b] < 0
 * skipped), so the result does not depend on the schedule.  n <= 131072; scratch: llmrec_scatter_add_rows_ordered_scratch(n) int32. */
int llmrec_scatter_add_rows_ordered_f32(const float* G, int64_t ldg, const int32_t* idx, int32_t n, int32_t d, float* Y, int64_t ldy,
                                        int32_t* scratch, int64_t scratch_elems, llmrec_stream_t stream);
int64_t llmrec_scatter_add_rows_ordered_scratch(int32_t n);
/* Y[r, :] = X[r, :] / max(||X[r, :]||_2, 1e-12) for r < n (F.normalize(X, dim=1)): the unit rows of item-to-item cosine neighbours.
 * X == Y (in place) is allowed. */
int llmrec_row_normalize_f32(const float* X, int64_t ldx, float* Y, int64_t ldy, int64_t n, int32_t d, llmrec_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Hoisted side-feature mode (SURVEY.md 8f-3; Models.py:145-167 with dropout p = 0 and the mask branch off):
 * iu.ui.(X W^T + 1 b^T) = (iu.ui.X) W^T + (iu.ui.1) b^T, so the propagated TABLES are precomputed once and a step projects
 * only the gathered rows of its batch.  The three helpers below are what that needs besides gather / projection / wgrad:
 *   rank1_add      Y[r, c] += scale[r * lds] * bias[c]          (the (iu.ui.1) b^T term on the compact rows)
 *   scaled_colsum  out[c] (+)= sum_terms sum_r scale[r * lds] * G[r * ldg + c]   (bias gradient; scale == NULL means 1)
 *   feat_reg_gram  feat_reg (main.py:151-156) over ALL rows through the k x k Gram matrix of a propagated table X~ and
 *                  h = X~^T s, n2 = |s|^2:  loss += c/2 (tr(W G W^T) + 2 b^T W h + n2 |b|^2);  dW += c (W G + b h^T);
 *                  db += c (W h + n2 b).  Two launches: W G by the exact-fp32 SIMT GEMM, then one pass over [d x k].
 *                  scratch: llmrec_feat_reg_gram_scratch(d, k) floats, zeroed once (ticket re-zeroed by the kernel).
 * --------------------------------------------------------------------------------------------- */
typedef struct { float* Y; const float* scale; const float* bias; int64_t ldy, lds, n; int32_t width, _pad; } llmrec_rank1_block;
typedef struct { const float* G; const float* scale; int64_t ldg, lds, n; } llmrec_colsum_term;
int llmrec_rank1_add_f32(const llmrec_rank1_block* blocks_host, int32_t n_blocks, llmrec_stream_t stream);
int llmrec_scaled_colsum_f32(const llmrec_colsum_term* terms_host, int32_t n_terms, int32_t width, float* out, int32_t accumulate,
                             float* scratch /* llmrec_scaled_colsum_scratch(width) floats, zeroed once */, llmrec_stream_t stream);
int64_t llmrec_scaled_colsum_scratch(int32_t width);
int llmrec_feat_reg_gram_f32(const float* W, const float* bias, const float* G, const float* h, float n2, int32_t d, int32_t k, float c,
                             float* dW, float* db, float* loss_accum, float* scratch, llmrec_stream_t stream);
int64_t llmrec_feat_reg_gram_scratch(int32_t d, int32_t k);

/* small utilities used by the host mirror */
int llmrec_fill_f32(float* p, int64_t n, float v, llmrec_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* LLMREC_B200_H */
