// C-ABI entry points that pick between the wgmma kernels and the exact SIMT kernels by `mode`
// (0 = wgmma 3xTF32, 1 = wgmma TF32, 2 = fp32 SIMT) and by shape support.
#include <vector>
#include "common.cuh"
#include "proj_tc.cuh"

namespace llmrec {
int proj_fwd_simt(const float*, int64_t, const float*, const float*, float*, int64_t, int64_t, int, int, const int*, cudaStream_t);
int proj_fwd_simt(const uint16_t*, int64_t, const float*, const float*, float*, int64_t, int64_t, int, int, const int*, cudaStream_t);
int proj_wgrad_simt(const float*, int64_t, const float*, int64_t, float*, float*, int64_t, int, int, int, const int*, int64_t, cudaStream_t);
int proj_wgrad_simt(const uint16_t*, int64_t, const float*, int64_t, float*, float*, int64_t, int, int, int, const int*, int64_t, cudaStream_t);
int proj_fwd_simt(const int8_t*, int64_t, const float*, const float*, float*, int64_t, int64_t, int, int, const int*, cudaStream_t);
int proj_wgrad_simt(const int8_t*, int64_t, const float*, int64_t, float*, float*, int64_t, int, int, int, const int*, int64_t, cudaStream_t);
int score_topk_simt(const float*, int64_t, const float*, int64_t, const int*, int, const int*, int, int, const int*, const int*, int, int*, float*, float*, int64_t, cudaStream_t);
bool proj_tc_supported(int d, int64_t ldx, const void* X, int k, bool wgrad, XType xt);
int proj_fwd_tc_group(const llmrec_proj_fwd_problem*, const int32_t* const*, int, int, int, XType, cudaStream_t);
int proj_wgrad_tc_group(const llmrec_proj_wgrad_problem*, const int32_t* const*, const int64_t*, int, int, int, XType, float*, int64_t, cudaStream_t);
int64_t proj_wgrad_tc_scratch(const llmrec_proj_wgrad_problem*, int, int, int, XType);
bool score_tc_supported(int d, int K, long long ldu, long long ldi, const void* U, const void* I);
long long score_tc_scratch(int n_batch, int n_items, int d, int K);
int score_topk_tc(const float*, long long, const float*, long long, const int*, int, const int*, int, int, const int*, const int*, int, int*, float*, float*, long long, cudaStream_t);
long long score_tc_group_scratch(const int* rp, int n_groups, int n_items, int d, int K);
int score_topk_group_tc(const float*, long long, const float*, long long, const int*, const int*, int, const int*, int, int, const int*, const int*, int,
                        int, int*, float*, float*, long long, cudaStream_t);
int score_topk_group_simt(const float*, int64_t, const float*, int64_t, const int*, const int*, const int*, int, const int*, int, int, const int*,
                          const int*, int, int, int*, float*, float*, int64_t, cudaStream_t);
}  // namespace llmrec
using namespace llmrec;

// bf16 / int8 X: the bf16 and int8 problems travel in the fp32 structs (same layout; X then holds a bf16 / int8 table's address), the
// tensor-core path reads W as bf16 terms in modes 0 and 1 (wsplit needed in both)
static bool fwd_tc_ok(const llmrec_proj_fwd_problem* pr, int n, int d, int mode, XType xt) {
  if (mode == 2 || n > 8) return false;
  for (int p = 0; p < n; ++p)
    if (!proj_tc_supported(d, pr[p].ldx, pr[p].X, pr[p].k, false, xt) || pr[p].ldy % 4 != 0 || !aligned16(pr[p].Y) || !aligned16(pr[p].W) ||
        (pr[p].bias && !aligned16(pr[p].bias)) || ((mode == 0 || xt != XType::F32) && !pr[p].wsplit))
      return false;
  return true;
}
static bool wg_tc_ok(const llmrec_proj_wgrad_problem* pr, int n, int d, int mode, XType xt) {
  if (mode == 2 || n > 8) return false;
  for (int p = 0; p < n; ++p)
    if (!proj_tc_supported(d, pr[p].ldx, pr[p].X, pr[p].k, true, xt) || pr[p].lddy % 4 != 0 || !aligned16(pr[p].dY)) return false;
  return true;
}
// int8 X: every row must hold its scale at roundup(k, 16), 4-byte aligned, inside the row pitch
template <class Prob>
static int check_i8_rows(const Prob* pr, int32_t n_prob) {
  for (int p = 0; p < n_prob; ++p)
    LLMREC_CHECK_ARG(pr[p].k >= 1 && pr[p].ldx % 4 == 0 && pr[p].ldx >= i8_scale_offset(pr[p].k) + 4 && (reinterpret_cast<uintptr_t>(pr[p].X) & 3u) == 0,
                     "proj (int8 X): problem %d: row pitch %lld bytes cannot hold k = %d values and the row scale (needs a multiple of 4, "
                     ">= roundup(k, 16) + 4, and a 4-byte aligned table)", p, (long long)pr[p].ldx, pr[p].k);
  return 0;
}

// Row maps (LLMREC_PROJ_ROW_MAP): the llmrec_proj_row_map records that follow the n_prob problems of a host array (same struct size for
// the _f32 and _bf16 problems); rows / n_dy stay empty when no problem is flagged, and a flagged problem needs a non-NULL map.
struct RowMaps { std::vector<const int32_t*> rows; std::vector<int64_t> n_dy; };
static int32_t flags(const llmrec_proj_fwd_problem& p) { return p._reserved; }
static int32_t flags(const llmrec_proj_fwd_problem_bf16& p) { return p._reserved; }
static int32_t flags(const llmrec_proj_wgrad_problem& p) { return p.accumulate; }
static int32_t flags(const llmrec_proj_wgrad_problem_bf16& p) { return p.accumulate; }
static int32_t flags(const llmrec_proj_fwd_problem_i8& p) { return p._reserved; }
static int32_t flags(const llmrec_proj_wgrad_problem_i8& p) { return p.accumulate; }
template <class Prob>
static int row_maps(const Prob* pr, int32_t n_prob, bool wgrad, RowMaps& M) {
  bool any = false;
  for (int p = 0; p < n_prob; ++p) any = any || (flags(pr[p]) & LLMREC_PROJ_ROW_MAP);
  if (!any) return 0;
  const llmrec_proj_row_map* rec = reinterpret_cast<const llmrec_proj_row_map*>(pr + n_prob);
  M.rows.assign(n_prob, nullptr);
  M.n_dy.assign(n_prob, 0);
  for (int p = 0; p < n_prob; ++p) {
    M.n_dy[p] = pr[p].n;
    if (!(flags(pr[p]) & LLMREC_PROJ_ROW_MAP)) continue;
    LLMREC_CHECK_ARG(rec[p].rows || pr[p].n <= 0, "proj: problem %d is flagged LLMREC_PROJ_ROW_MAP but its map is NULL", p);
    LLMREC_CHECK_ARG(!wgrad || rec[p].n_dy >= 0, "proj_wgrad: problem %d has a negative dY row count", p);
    M.rows[p] = rec[p].rows; M.n_dy[p] = rec[p].n_dy;
  }
  return 0;
}

// rows: NULL, or n_prob optional row maps
static int proj_fwd_group(const llmrec_proj_fwd_problem* pr, const int32_t* const* rows, int32_t n_prob, int32_t d, int32_t mode, XType xt,
                          llmrec_stream_t stream) {
  LLMREC_REQUIRE_DEVICE();
  LLMREC_CHECK_ARG(n_prob >= 1 && d >= 1, "proj_fwd_group: bad sizes");
  cudaStream_t st = as_stream(stream);
  for (int p0 = 0; p0 < n_prob; p0 += 8) {
    int np = n_prob - p0 < 8 ? n_prob - p0 : 8;
    if (fwd_tc_ok(pr + p0, np, d, mode, xt)) {
      int rc = proj_fwd_tc_group(pr + p0, rows ? rows + p0 : nullptr, np, d, mode, xt, st);
      if (rc) return rc;
    } else {
      for (int p = p0; p < p0 + np; ++p) {
        if (pr[p].n <= 0) continue;
        const int32_t* map = rows ? rows[p] : nullptr;
        int rc = xt == XType::I8   ? proj_fwd_simt(reinterpret_cast<const int8_t*>(pr[p].X), pr[p].ldx, pr[p].W, pr[p].bias, pr[p].Y, pr[p].ldy, pr[p].n, pr[p].k, d, map, st)
                 : xt == XType::BF16 ? proj_fwd_simt(reinterpret_cast<const uint16_t*>(pr[p].X), pr[p].ldx, pr[p].W, pr[p].bias, pr[p].Y, pr[p].ldy, pr[p].n, pr[p].k, d, map, st)
                                     : proj_fwd_simt(pr[p].X, pr[p].ldx, pr[p].W, pr[p].bias, pr[p].Y, pr[p].ldy, pr[p].n, pr[p].k, d, map, st);
        if (rc) return rc;
      }
    }
  }
  return 0;
}
template <class Prob>   // the _bf16 / _i8 forward problem
static std::vector<llmrec_proj_fwd_problem> as_f32_layout(const Prob* pr, int32_t n_prob) {
  std::vector<llmrec_proj_fwd_problem> q(n_prob > 0 ? n_prob : 0);
  for (int p = 0; p < n_prob; ++p)
    q[p] = {reinterpret_cast<const float*>(pr[p].X), pr[p].W, pr[p].bias, pr[p].Y, pr[p].wsplit, pr[p].ldx, pr[p].ldy, pr[p].n, pr[p].k, 0};
  return q;
}
extern "C" int llmrec_proj_fwd_group_f32(const llmrec_proj_fwd_problem* pr, int32_t n_prob, int32_t d, int32_t mode, llmrec_stream_t stream) {
  LLMREC_CHECK_ARG(pr && n_prob >= 1, "proj_fwd_group: bad sizes");
  RowMaps M;
  if (int rc = row_maps(pr, n_prob, false, M)) return rc;
  return proj_fwd_group(pr, M.rows.empty() ? nullptr : M.rows.data(), n_prob, d, mode, XType::F32, stream);
}
extern "C" int llmrec_proj_fwd_group_bf16(const llmrec_proj_fwd_problem_bf16* pr, int32_t n_prob, int32_t d, int32_t mode, llmrec_stream_t stream) {
  LLMREC_CHECK_ARG(pr && n_prob >= 1, "proj_fwd_group: bad sizes");
  RowMaps M;
  if (int rc = row_maps(pr, n_prob, false, M)) return rc;
  return proj_fwd_group(as_f32_layout(pr, n_prob).data(), M.rows.empty() ? nullptr : M.rows.data(), n_prob, d, mode, XType::BF16, stream);
}
extern "C" int llmrec_proj_fwd_group_i8(const llmrec_proj_fwd_problem_i8* pr, int32_t n_prob, int32_t d, int32_t mode, llmrec_stream_t stream) {
  LLMREC_CHECK_ARG(pr && n_prob >= 1, "proj_fwd_group: bad sizes");
  if (int rc = check_i8_rows(pr, n_prob)) return rc;
  RowMaps M;
  if (int rc = row_maps(pr, n_prob, false, M)) return rc;
  return proj_fwd_group(as_f32_layout(pr, n_prob).data(), M.rows.empty() ? nullptr : M.rows.data(), n_prob, d, mode, XType::I8, stream);
}
extern "C" int llmrec_proj_fwd_f32(const float* X, int64_t ldx, const float* W, const float* bias, float* Y, int64_t ldy,
                                   int64_t n, int32_t k, int32_t d, int32_t mode, float* wsplit, llmrec_stream_t stream) {
  llmrec_proj_fwd_problem p{X, W, bias, Y, wsplit, ldx, ldy, n, k, 0};
  if (n <= 0) return 0;
  return llmrec_proj_fwd_group_f32(&p, 1, d, mode, stream);
}

static int64_t proj_wgrad_scratch(const llmrec_proj_wgrad_problem* pr, int32_t n_prob, int32_t d, int32_t mode, XType xt) {
  int64_t need = 0;
  for (int p0 = 0; p0 < n_prob; p0 += 8) {
    int np = n_prob - p0 < 8 ? n_prob - p0 : 8;
    if (wg_tc_ok(pr + p0, np, d, mode, xt)) { int64_t s = proj_wgrad_tc_scratch(pr + p0, np, d, mode, xt); need = s > need ? s : need; }
  }
  return need;
}
// rows / n_dy: NULL, or per problem an optional dY row map and the row count of dY
static int proj_wgrad_group(const llmrec_proj_wgrad_problem* pr, const int32_t* const* rows, const int64_t* n_dy, int32_t n_prob, int32_t d,
                            int32_t mode, XType xt, float* scratch, int64_t scratch_elems, llmrec_stream_t stream) {
  LLMREC_REQUIRE_DEVICE();
  LLMREC_CHECK_ARG(n_prob >= 1 && d >= 1, "proj_wgrad_group: bad sizes");
  cudaStream_t st = as_stream(stream);
  for (int p0 = 0; p0 < n_prob; p0 += 8) {
    int np = n_prob - p0 < 8 ? n_prob - p0 : 8;
    if (wg_tc_ok(pr + p0, np, d, mode, xt)) {
      int rc = proj_wgrad_tc_group(pr + p0, rows ? rows + p0 : nullptr, rows ? n_dy + p0 : nullptr, np, d, mode, xt, scratch, scratch_elems, st);
      if (rc) return rc;
    } else {
      for (int p = p0; p < p0 + np; ++p) {
        const int acc = pr[p].accumulate & LLMREC_WGRAD_ACCUMULATE;
        const int32_t* map = rows ? rows[p] : nullptr;
        const int64_t ndy = n_dy ? n_dy[p] : pr[p].n;
        int rc = xt == XType::I8   ? proj_wgrad_simt(reinterpret_cast<const int8_t*>(pr[p].X), pr[p].ldx, pr[p].dY, pr[p].lddy, pr[p].dW, pr[p].db, pr[p].n, pr[p].k, d, acc, map, ndy, st)
                 : xt == XType::BF16 ? proj_wgrad_simt(reinterpret_cast<const uint16_t*>(pr[p].X), pr[p].ldx, pr[p].dY, pr[p].lddy, pr[p].dW, pr[p].db, pr[p].n, pr[p].k, d, acc, map, ndy, st)
                                     : proj_wgrad_simt(pr[p].X, pr[p].ldx, pr[p].dY, pr[p].lddy, pr[p].dW, pr[p].db, pr[p].n, pr[p].k, d, acc, map, ndy, st);
        if (rc) return rc;
      }
    }
  }
  return 0;
}
template <class Prob>   // the _bf16 / _i8 weight-gradient problem
static std::vector<llmrec_proj_wgrad_problem> as_wgrad_f32_layout(const Prob* pr, int32_t n_prob) {
  std::vector<llmrec_proj_wgrad_problem> q(n_prob > 0 ? n_prob : 0);
  for (int p = 0; p < n_prob; ++p)
    q[p] = {reinterpret_cast<const float*>(pr[p].X), pr[p].dY, pr[p].dW, pr[p].db, pr[p].ldx, pr[p].lddy, pr[p].n, pr[p].k, pr[p].accumulate};
  return q;
}
extern "C" int64_t llmrec_proj_wgrad_group_scratch(const llmrec_proj_wgrad_problem* pr, int32_t n_prob, int32_t d, int32_t mode) {
  return proj_wgrad_scratch(pr, n_prob, d, mode, XType::F32);
}
extern "C" int64_t llmrec_proj_wgrad_group_bf16_scratch(const llmrec_proj_wgrad_problem_bf16* pr, int32_t n_prob, int32_t d, int32_t mode) {
  return proj_wgrad_scratch(as_wgrad_f32_layout(pr, n_prob).data(), n_prob, d, mode, XType::BF16);
}
extern "C" int64_t llmrec_proj_wgrad_group_i8_scratch(const llmrec_proj_wgrad_problem_i8* pr, int32_t n_prob, int32_t d, int32_t mode) {
  return proj_wgrad_scratch(as_wgrad_f32_layout(pr, n_prob).data(), n_prob, d, mode, XType::I8);
}
extern "C" int llmrec_proj_wgrad_group_f32(const llmrec_proj_wgrad_problem* pr, int32_t n_prob, int32_t d, int32_t mode,
                                           float* scratch, int64_t scratch_elems, llmrec_stream_t stream) {
  LLMREC_CHECK_ARG(pr && n_prob >= 1, "proj_wgrad_group: bad sizes");
  RowMaps M;
  if (int rc = row_maps(pr, n_prob, true, M)) return rc;
  const bool mapped = !M.rows.empty();
  return proj_wgrad_group(pr, mapped ? M.rows.data() : nullptr, mapped ? M.n_dy.data() : nullptr, n_prob, d, mode, XType::F32, scratch, scratch_elems, stream);
}
extern "C" int llmrec_proj_wgrad_group_bf16(const llmrec_proj_wgrad_problem_bf16* pr, int32_t n_prob, int32_t d, int32_t mode,
                                            float* scratch, int64_t scratch_elems, llmrec_stream_t stream) {
  LLMREC_CHECK_ARG(pr && n_prob >= 1, "proj_wgrad_group: bad sizes");
  RowMaps M;
  if (int rc = row_maps(pr, n_prob, true, M)) return rc;
  const bool mapped = !M.rows.empty();
  return proj_wgrad_group(as_wgrad_f32_layout(pr, n_prob).data(), mapped ? M.rows.data() : nullptr, mapped ? M.n_dy.data() : nullptr, n_prob, d, mode,
                          XType::BF16, scratch, scratch_elems, stream);
}
extern "C" int llmrec_proj_wgrad_group_i8(const llmrec_proj_wgrad_problem_i8* pr, int32_t n_prob, int32_t d, int32_t mode,
                                          float* scratch, int64_t scratch_elems, llmrec_stream_t stream) {
  LLMREC_CHECK_ARG(pr && n_prob >= 1, "proj_wgrad_group: bad sizes");
  if (int rc = check_i8_rows(pr, n_prob)) return rc;
  RowMaps M;
  if (int rc = row_maps(pr, n_prob, true, M)) return rc;
  const bool mapped = !M.rows.empty();
  return proj_wgrad_group(as_wgrad_f32_layout(pr, n_prob).data(), mapped ? M.rows.data() : nullptr, mapped ? M.n_dy.data() : nullptr, n_prob, d, mode,
                          XType::I8, scratch, scratch_elems, stream);
}
extern "C" int64_t llmrec_proj_wgrad_scratch(int64_t n, int32_t k, int32_t d, int32_t mode) {
  llmrec_proj_wgrad_problem p{nullptr, nullptr, nullptr, nullptr, 4, 4, n, k, 0};
  // alignment of real pointers is checked at call time; size the scratch for the tensor-core path
  if (mode == 2 || d % 32 != 0 || d > 256 || k % 4 != 0) return 0;
  return proj_wgrad_tc_scratch(&p, 1, d, mode, XType::F32);
}
extern "C" int llmrec_proj_wgrad_f32(const float* X, int64_t ldx, const float* dY, int64_t lddy, float* dW, float* db,
                                     int64_t n, int32_t k, int32_t d, int32_t accumulate, int32_t mode,
                                     float* scratch, int64_t scratch_elems, llmrec_stream_t stream) {
  llmrec_proj_wgrad_problem p{X, dY, dW, db, ldx, lddy, n, k, accumulate};
  return llmrec_proj_wgrad_group_f32(&p, 1, d, mode, scratch, scratch_elems, stream);
}

extern "C" int64_t llmrec_score_topk_scratch(int32_t n_batch, int32_t n_items, int32_t d, int32_t K, int32_t mode) {
  if (mode != 2 && (d == 32 || d == 64 || d == 96 || d == 128) && K <= 64) return score_tc_scratch(n_batch, n_items, d, K);
  int64_t want = (int64_t)n_batch * n_items;
  int64_t cap = (int64_t)1 << 28;  // 1 GiB of fp32 scores at most; the SIMT kernel loops over user sub-blocks
  if (want > cap) want = (cap / n_items) * n_items;
  if (want < n_items) want = n_items;
  return want;
}
// among: NULL (the catalog is the n_items rows of I), or n_items ascending global ids of rows of I
static int score_topk(const float* U, int64_t ldu, const float* I, int64_t ldi, const int32_t* users, int32_t n_batch, const int32_t* among,
                      int32_t n_items, int32_t d, const int32_t* mask_rowptr, const int32_t* mask_col, int32_t K, int32_t* out_idx,
                      float* out_val, int32_t mode, float* scratch, int64_t scratch_elems, llmrec_stream_t stream) {
  LLMREC_REQUIRE_DEVICE();
  LLMREC_CHECK_ARG(K >= 1 && K <= 64 && K <= n_items, among ? "score_topk_among: K=%d unsupported (1..64, <= n_among)"
                                                            : "score_topk: K=%d unsupported (1..64, <= n_items)", K);
  if (n_batch <= 0) return 0;
  if (mode != 2 && score_tc_supported(d, K, ldu, ldi, U, I))
    return score_topk_tc(U, ldu, I, ldi, users, n_batch, among, n_items, d, mask_rowptr, mask_col, K, out_idx, out_val, scratch, scratch_elems,
                         as_stream(stream));
  return score_topk_simt(U, ldu, I, ldi, users, n_batch, among, n_items, d, mask_rowptr, mask_col, K, out_idx, out_val, scratch, scratch_elems,
                         as_stream(stream));
}
extern "C" int llmrec_score_topk_f32(const float* U, int64_t ldu, const float* I, int64_t ldi, const int32_t* users, int32_t n_batch,
                                     int32_t n_items, int32_t d, const int32_t* mask_rowptr, const int32_t* mask_col, int32_t K,
                                     int32_t* out_idx, float* out_val, int32_t mode, float* scratch, int64_t scratch_elems,
                                     llmrec_stream_t stream) {
  return score_topk(U, ldu, I, ldi, users, n_batch, nullptr, n_items, d, mask_rowptr, mask_col, K, out_idx, out_val, mode, scratch, scratch_elems,
                    stream);
}
extern "C" int64_t llmrec_score_topk_among_scratch(int32_t n_batch, int32_t n_among, int32_t d, int32_t K, int32_t mode) {
  return llmrec_score_topk_scratch(n_batch, n_among, d, K, mode);
}
extern "C" int llmrec_score_topk_among_f32(const float* U, int64_t ldu, const float* I, int64_t ldi, const int32_t* users, int32_t n_batch,
                                           const int32_t* among, int32_t n_among, int32_t d, const int32_t* mask_rowptr, const int32_t* mask_col,
                                           int32_t K, int32_t* out_idx, float* out_val, int32_t mode, float* scratch, int64_t scratch_elems,
                                           llmrec_stream_t stream) {
  LLMREC_CHECK_ARG(among || n_among <= 0, "score_topk_among: among is NULL");
  return score_topk(U, ldu, I, ldi, users, n_batch, among, n_among, d, mask_rowptr, mask_col, K, out_idx, out_val, mode, scratch, scratch_elems,
                    stream);
}

// ---- groups ----------------------------------------------------------------------------------------------------------------
// mode 2: the device copy of the member CSR (rounded to 4 elements), then rows of group and member scores
static int64_t group_rowptr_elems(int32_t n_groups) { return ((int64_t)n_groups + 1 + 3) / 4 * 4; }
static int64_t group_simt_scratch(const int32_t* rp, int32_t n_groups, int32_t n_items) {
  int64_t want = ((int64_t)n_groups + (rp[n_groups] - rp[0])) * n_items;
  const int64_t cap = (int64_t)1 << 28;   // 1 GiB of fp32 scores at most; the SIMT path loops over blocks of groups
  if (want > cap) want = (cap / n_items) * n_items;
  if (want < 65LL * n_items) want = 65LL * n_items;   // one group of 64 members and its group row
  return group_rowptr_elems(n_groups) + want;
}
static bool group_tc_shape(int32_t d, int32_t K, int32_t mode) { return mode != 2 && (d == 32 || d == 64 || d == 96 || d == 128) && K <= 64; }
extern "C" int64_t llmrec_score_topk_group_scratch(const int32_t* member_rowptr_host, int32_t n_groups, int32_t n_items, int32_t d, int32_t K, int32_t mode) {
  if (!member_rowptr_host || n_groups <= 0 || n_items <= 0) return 0;
  for (int g = 0; g < n_groups; ++g)   // a malformed CSR sizes nothing; the call itself reports it
    if (member_rowptr_host[g + 1] - member_rowptr_host[g] < 1 || member_rowptr_host[g + 1] - member_rowptr_host[g] > 64) return 0;
  if (!group_tc_shape(d, K, mode)) return group_simt_scratch(member_rowptr_host, n_groups, n_items);
  // the call may still take the SIMT path (leading dimensions, alignment): leave room for its smallest block (one group of 64
  // members and its group row), not for its full 1 GiB of blocks
  const int64_t tc = score_tc_group_scratch(member_rowptr_host, n_groups, n_items, d, K);
  const int64_t simt_min = group_rowptr_elems(n_groups) + 65LL * n_items;
  return tc > simt_min ? tc : simt_min;
}
extern "C" int llmrec_score_topk_group_f32(const float* U, int64_t ldu, const float* I, int64_t ldi, const int32_t* member_rowptr_host,
                                           const int32_t* members, int32_t n_groups, const int32_t* among, int32_t n_items, int32_t d,
                                           const int32_t* mask_rowptr, const int32_t* mask_col, int32_t K, int32_t agg, int32_t* out_idx,
                                           float* out_val, int32_t mode, float* scratch, int64_t scratch_elems, llmrec_stream_t stream) {
  LLMREC_REQUIRE_DEVICE();
  LLMREC_CHECK_ARG(K >= 1 && K <= 64 && K <= n_items, "score_topk_group: K=%d unsupported (1..64, <= n_items = %d)", K, n_items);
  LLMREC_CHECK_ARG(agg == LLMREC_AGG_MEAN || agg == LLMREC_AGG_MIN || agg == LLMREC_AGG_MAX, "score_topk_group: agg=%d is not "
                   "LLMREC_AGG_MEAN / _MIN / _MAX", agg);
  LLMREC_CHECK_ARG(n_groups >= 0 && d >= 1, "score_topk_group: bad sizes");
  if (n_groups == 0) return 0;
  LLMREC_CHECK_ARG(member_rowptr_host && members && member_rowptr_host[0] == 0, "score_topk_group: member CSR missing or not starting at 0");
  for (int g = 0; g < n_groups; ++g) {
    const int n = member_rowptr_host[g + 1] - member_rowptr_host[g];
    LLMREC_CHECK_ARG(n >= 1 && n <= 64, "score_topk_group: group %d has %d members (1..64)", g, n);
  }
  cudaStream_t st = as_stream(stream);
  if (group_tc_shape(d, K, mode) && score_tc_supported(d, K, ldu, ldi, U, I))
    return score_topk_group_tc(U, ldu, I, ldi, member_rowptr_host, members, n_groups, among, n_items, d, mask_rowptr, mask_col, K, agg, out_idx,
                               out_val, scratch, scratch_elems, st);
  const int64_t head = group_rowptr_elems(n_groups);
  LLMREC_CHECK_ARG(scratch && scratch_elems >= head + 65LL * n_items, "score_topk_group(simt): scratch too small");
  int32_t* drp = reinterpret_cast<int32_t*>(scratch);
  // pageable source: the copy is staged before this returns
  LLMREC_CHECK_CUDA(cudaMemcpyAsync(drp, member_rowptr_host, ((size_t)n_groups + 1) * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  return score_topk_group_simt(U, ldu, I, ldi, member_rowptr_host, drp, members, n_groups, among, n_items, d, mask_rowptr, mask_col, K, agg, out_idx,
                               out_val, scratch + head, scratch_elems - head, st);
}
