// Exact-fp32 full-catalog scoring + top-K (utility/batch_test.py:149-152 and :21-36,100-102) and the
// hit-vector lookup (:30-34).  mode 2 of llmrec_score_topk_f32: sequential-FMA fp32 scores, exact
// selection with ties -> lowest item id.  It is the on-device checker of the wgmma kernel and the
// path for K/d the tensor-core kernel does not cover.
//
// The catalog is I, or (among != NULL, llmrec_score_topk_among_f32) the rows among[0 .. n_items) of I with ids
// ascending: column j of the score block is item among[j], mask rows and returned ids are global item ids.
#include "common.cuh"

namespace llmrec {

// position of global item id v in the ascending catalog ids among[0 .. n), or -1 when it is not there
__device__ __forceinline__ int catalog_pos(const int* __restrict__ among, int n, int v) {
  int lo = 0, hi = n;
  while (lo < hi) { const int m = (lo + hi) >> 1; const int x = __ldg(among + m); if (x < v) lo = m + 1; else hi = m; }
  return lo < n && __ldg(among + lo) == v ? lo : -1;
}

// scores for a block of users into scratch[b][n_items] (column j = catalog item j)
__global__ void __launch_bounds__(256) score_rows_kernel(const float* __restrict__ U, int64_t ldu, const float* __restrict__ I, int64_t ldi,
                                                         const int* __restrict__ users, const int* __restrict__ among, int n_items, int d,
                                                         float* __restrict__ S) {
  extern __shared__ float us[];  // d
  const int b = blockIdx.y;
  const float* u = U + (int64_t)users[b] * ldu;
  for (int j = threadIdx.x; j < d; j += blockDim.x) us[j] = u[j];
  __syncthreads();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_items) return;
  const float* it = I + (int64_t)(among ? __ldg(among + i) : i) * ldi;
  float a = 0.f;
  for (int j = 0; j < d; ++j) a = fmaf(us[j], it[j], a);
  S[(int64_t)b * n_items + i] = a;
}
// masked items -> -inf; with `among`, a masked id outside the catalog is skipped; users NULL: row b reads mask row b
__global__ void mask_rows_kernel(const int* __restrict__ users, const int* __restrict__ rowptr, const int* __restrict__ col,
                                 const int* __restrict__ among, int n_items, float* __restrict__ S) {
  const int b = blockIdx.x;
  const int u = users ? users[b] : b;
  for (int e = rowptr[u] + threadIdx.x; e < rowptr[u + 1]; e += blockDim.x) {
    int c = col[e];
    if (among) c = catalog_pos(among, n_items, c);
    if (c >= 0 && c < n_items) S[(int64_t)b * n_items + c] = -INFINITY;
  }
}
// group rows of a block of groups g0 .. g0 + gridDim.y from the scores of their members (rows of Sm from member m_base on):
// Sg[g - g0][i] = the exact group score of catalog column i (common.cuh agg_*)
__global__ void __launch_bounds__(256) aggregate_group_rows_kernel(const float* __restrict__ Sm, const int* __restrict__ grp_rowptr, int g0,
                                                                   int m_base, int n_items, int agg, float* __restrict__ Sg) {
  const int g = g0 + blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_items) return;
  const int m0 = __ldg(grp_rowptr + g), m1 = __ldg(grp_rowptr + g + 1);
  float v = agg_start(agg);
  for (int m = m0; m < m1; ++m) v = agg_fold(agg, v, Sm[(int64_t)(m - m_base) * n_items + i]);
  Sg[(int64_t)blockIdx.y * n_items + i] = agg_end(agg, v, m1 - m0);
}
// K rounds of block arg-max with (score desc, id asc) order; ascending catalog ids make the lowest column the lowest id
__global__ void __launch_bounds__(256) select_topk_kernel(float* __restrict__ S, const int* __restrict__ among, int n_items, int K,
                                                          int* __restrict__ out_idx, float* __restrict__ out_val) {
  __shared__ float bv[8]; __shared__ int bi[8];
  __shared__ int win;
  const int b = blockIdx.x;
  float* s = S + (int64_t)b * n_items;
  for (int r = 0; r < K; ++r) {
    float best = -INFINITY; int besti = 0x7fffffff;
    for (int i = threadIdx.x; i < n_items; i += blockDim.x) {
      float v = s[i];
      if (v > best || (v == best && i < besti && v != -INFINITY)) { best = v; besti = i; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      float ov = __shfl_xor_sync(0xffffffffu, best, o); int oi = __shfl_xor_sync(0xffffffffu, besti, o);
      if (ov > best || (ov == best && oi < besti)) { best = ov; besti = oi; }
    }
    if ((threadIdx.x & 31) == 0) { bv[threadIdx.x >> 5] = best; bi[threadIdx.x >> 5] = besti; }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int w = 1; w < 8; ++w) if (bv[w] > best || (bv[w] == best && bi[w] < besti)) { best = bv[w]; besti = bi[w]; }
      bool ok = besti != 0x7fffffff && best != -INFINITY;
      out_idx[(int64_t)b * K + r] = ok ? (among ? among[besti] : besti) : -1;
      if (out_val) out_val[(int64_t)b * K + r] = ok ? best : -INFINITY;
      if (ok) s[besti] = -INFINITY;
      win = besti;
    }
    __syncthreads();
  }
}

__global__ void topk_hits_kernel(const int* __restrict__ idx, int n_batch, int K, const int* __restrict__ users,
                                 const int* __restrict__ rowptr, const int* __restrict__ col, uint8_t* __restrict__ hits) {
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= (int64_t)n_batch * K) return;
  const int b = (int)(t / K);
  const int item = idx[t];
  const int u = users[b];
  uint8_t h = 0;
  if (item >= 0) for (int e = rowptr[u]; e < rowptr[u + 1]; ++e) if (col[e] == item) { h = 1; break; }
  hits[t] = h;
}

// test_flag == 'full' (batch_test.py:38-68): per-user ROC-AUC of the exact fp32 scores over the candidates (all items minus the user's
// train items), positives = the user's truth row.  roc_auc_score is the Mann-Whitney statistic:
//   AUC = sum_{p in pos} ( #{neg: s_neg < s_p} + 0.5 #{neg: s_neg == s_p} ) / (n_pos * n_neg),  0 when one class is empty
// (the reference catches sklearn's ValueError and returns 0., utility/metrics.py:95-100).  One CTA per user; mask / truth rows sorted.
constexpr int kAucMaxPos = 128;
__device__ __forceinline__ bool sorted_has(const int* __restrict__ a, int lo, int hi, int v) {
  while (lo < hi) { const int m = (lo + hi) >> 1; const int x = a[m]; if (x == v) return true; if (x < v) lo = m + 1; else hi = m; }
  return false;
}
__global__ void __launch_bounds__(256) user_auc_kernel(const float* __restrict__ U, int64_t ldu, const float* __restrict__ I, int64_t ldi,
                                                       const int* __restrict__ users, int n_items, int d,
                                                       const int* __restrict__ mrp, const int* __restrict__ mcol,
                                                       const int* __restrict__ trp, const int* __restrict__ tcol, float* __restrict__ out) {
  extern __shared__ float us[];          // d user values, then kAucMaxPos positive scores
  float* ps = us + d;
  __shared__ double red_l[8], red_e[8];
  __shared__ int red_n[8];
  __shared__ int s_npos;
  const int b = blockIdx.x, u = users[b];
  for (int j = threadIdx.x; j < d; j += blockDim.x) us[j] = U[(int64_t)u * ldu + j];
  __syncthreads();
  const int m0 = mrp ? mrp[u] : 0, m1 = mrp ? mrp[u + 1] : 0;
  const int t0 = trp[u], t1 = trp[u + 1];
  auto score = [&](int i) { const float* it = I + (int64_t)i * ldi; float a = 0.f; for (int j = 0; j < d; ++j) a = fmaf(us[j], it[j], a); return a; };
  double less = 0.0, eq = 0.0;
  int n_neg = 0, n_pos_total = 0;
  for (int tb = t0; tb < t1 || tb == t0; tb += kAucMaxPos) {      // positives in chunks of kAucMaxPos (one pass over the catalog per chunk)
    if (threadIdx.x == 0) s_npos = 0;
    __syncthreads();
    for (int e = tb + threadIdx.x; e < min(t1, tb + kAucMaxPos); e += blockDim.x) {
      const int i = tcol[e];
      if (i >= 0 && i < n_items && !sorted_has(mcol, m0, m1, i) && (e == t0 || tcol[e - 1] != i)) ps[atomicAdd(&s_npos, 1)] = score(i);
    }
    __syncthreads();
    const int np = s_npos;
    n_pos_total += np;
    int nn = 0;
    for (int i = threadIdx.x; i < n_items; i += blockDim.x) {
      if (sorted_has(mcol, m0, m1, i) || sorted_has(tcol, t0, t1, i)) continue;      // not a candidate / a positive
      ++nn;
      if (np == 0) continue;
      const float s = score(i);
      for (int q = 0; q < np; ++q) { less += (s < ps[q]) ? 1.0 : 0.0; eq += (s == ps[q]) ? 1.0 : 0.0; }
    }
    if (tb == t0) n_neg = nn;
    __syncthreads();
    if (t1 - t0 <= kAucMaxPos) break;
  }
  // block reduce (counts are exact in double)
  for (int o = 16; o > 0; o >>= 1) { less += __shfl_xor_sync(0xffffffffu, less, o); eq += __shfl_xor_sync(0xffffffffu, eq, o); n_neg += __shfl_xor_sync(0xffffffffu, n_neg, o); }
  if ((threadIdx.x & 31) == 0) { red_l[threadIdx.x >> 5] = less; red_e[threadIdx.x >> 5] = eq; red_n[threadIdx.x >> 5] = n_neg; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double L = 0.0, E = 0.0; long long NN = 0;
    for (int w = 0; w < 8; ++w) { L += red_l[w]; E += red_e[w]; NN += red_n[w]; }
    out[b] = (n_pos_total > 0 && NN > 0) ? (float)((L + 0.5 * E) / ((double)n_pos_total * (double)NN)) : 0.f;
  }
}

// among: NULL (the catalog is I), or n_items ascending ids of rows of I (the catalog is those rows)
int score_topk_simt(const float* U, int64_t ldu, const float* I, int64_t ldi, const int* users, int n_batch, const int* among, int n_items, int d,
                    const int* mask_rowptr, const int* mask_col, int K, int* out_idx, float* out_val,
                    float* scratch, int64_t scratch_elems, cudaStream_t st) {
  LLMREC_CHECK_ARG(scratch && scratch_elems >= (int64_t)n_items, "score_topk(simt): scratch too small");
  int64_t per = scratch_elems / n_items;
  if (per > 65535) per = 65535;
  for (int b0 = 0; b0 < n_batch; b0 += (int)per) {
    int nb = (int)((per < (int64_t)(n_batch - b0)) ? per : (int64_t)(n_batch - b0));
    dim3 grid((n_items + 255) / 256, nb);
    score_rows_kernel<<<grid, 256, d * sizeof(float), st>>>(U, ldu, I, ldi, users + b0, among, n_items, d, scratch);
    LLMREC_CHECK_LAUNCH("score_rows");
    if (mask_rowptr) { mask_rows_kernel<<<nb, 128, 0, st>>>(users + b0, mask_rowptr, mask_col, among, n_items, scratch); LLMREC_CHECK_LAUNCH("mask_rows"); }
    select_topk_kernel<<<nb, 256, 0, st>>>(scratch, among, n_items, K, out_idx + (int64_t)b0 * K, out_val ? out_val + (int64_t)b0 * K : nullptr);
    LLMREC_CHECK_LAUNCH("select_topk");
  }
  return 0;
}

// groups: rp is the HOST member CSR, grp_rowptr its device copy; members are rows of U; mask rows are indexed by group.  Blocks of
// groups whose group rows and member rows fit the scratch: member scores (score_rows_kernel), group rows, mask, selection.
int score_topk_group_simt(const float* U, int64_t ldu, const float* I, int64_t ldi, const int* rp, const int* grp_rowptr, const int* members,
                          int n_groups, const int* among, int n_items, int d, const int* mask_rowptr, const int* mask_col, int K, int agg,
                          int* out_idx, float* out_val, float* scratch, int64_t scratch_elems, cudaStream_t st) {
  const int64_t rows = scratch ? scratch_elems / n_items : 0;
  LLMREC_CHECK_ARG(rows >= 65, "score_topk_group(simt): scratch too small (one group of 64 members needs 65 rows of %d)", n_items);
  for (int g0 = 0; g0 < n_groups;) {
    int g1 = g0 + 1;
    while (g1 < n_groups && g1 + 1 - g0 <= 65535 && rp[g1 + 1] - rp[g0] <= 65535 && (g1 + 1 - g0) + (int64_t)(rp[g1 + 1] - rp[g0]) <= rows) ++g1;
    const int ng = g1 - g0, nm = rp[g1] - rp[g0];
    float* Sg = scratch;
    float* Sm = scratch + (int64_t)ng * n_items;
    dim3 grid_m((n_items + 255) / 256, nm), grid_g((n_items + 255) / 256, ng);
    score_rows_kernel<<<grid_m, 256, d * sizeof(float), st>>>(U, ldu, I, ldi, members + rp[g0], among, n_items, d, Sm);
    LLMREC_CHECK_LAUNCH("score_rows");
    aggregate_group_rows_kernel<<<grid_g, 256, 0, st>>>(Sm, grp_rowptr, g0, rp[g0], n_items, agg, Sg);
    LLMREC_CHECK_LAUNCH("aggregate_group_rows");
    if (mask_rowptr) { mask_rows_kernel<<<ng, 128, 0, st>>>(nullptr, mask_rowptr + g0, mask_col, among, n_items, Sg); LLMREC_CHECK_LAUNCH("mask_rows"); }
    select_topk_kernel<<<ng, 256, 0, st>>>(Sg, among, n_items, K, out_idx + (int64_t)g0 * K, out_val ? out_val + (int64_t)g0 * K : nullptr);
    LLMREC_CHECK_LAUNCH("select_topk");
    g0 = g1;
  }
  return 0;
}
}  // namespace llmrec

extern "C" int llmrec_user_auc_f32(const float* U, int64_t ldu, const float* I, int64_t ldi, const int32_t* users, int32_t n_batch, int32_t n_items, int32_t d,
                                   const int32_t* mask_rowptr, const int32_t* mask_col, const int32_t* truth_rowptr, const int32_t* truth_col,
                                   float* out_auc, llmrec_stream_t stream) {
  LLMREC_REQUIRE_DEVICE();
  LLMREC_CHECK_ARG(truth_rowptr && truth_col && d >= 1 && d <= 4096, "user_auc: truth CSR required, d=%d out of range", d);
  if (n_batch <= 0) return 0;
  llmrec::user_auc_kernel<<<n_batch, 256, (size_t)(d + llmrec::kAucMaxPos) * sizeof(float), llmrec::as_stream(stream)>>>(
      U, ldu, I, ldi, users, n_items, d, mask_rowptr, mask_col, truth_rowptr, truth_col, out_auc);
  LLMREC_CHECK_LAUNCH("user_auc");
  return 0;
}

extern "C" int llmrec_topk_hits(const int32_t* idx, int32_t n_batch, int32_t K, const int32_t* users,
                                const int32_t* truth_rowptr, const int32_t* truth_col, uint8_t* hits, llmrec_stream_t stream) {
  LLMREC_REQUIRE_DEVICE();
  int64_t total = (int64_t)n_batch * K;
  if (total <= 0) return 0;
  llmrec::topk_hits_kernel<<<(unsigned)((total + 255) / 256), 256, 0, llmrec::as_stream(stream)>>>(idx, n_batch, K, users, truth_rowptr, truth_col, hits);
  LLMREC_CHECK_LAUNCH("topk_hits");
  return 0;
}
