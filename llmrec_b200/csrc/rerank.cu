// Scores of given (user, item) pairs and per-query re-ranking of given candidate lists: the serving questions that are not a
// full-catalog top-K.  Both are gathers of embedding rows followed by per-row work, so they run on the SIMT cores in exact fp32:
// every candidate row is read once per query, the work is gather- and L2-bound, and tensor cores would add nothing.
//
// One score = one sequential fp32 FMA chain a = fmaf(u[j], i[j], a), j = 0..d-1, from a = 0 -- the arithmetic of
// score_rows_kernel (score_simt.cu) and rescore_topk_kernel (score_tc.cu), so a pair's score has the bits score_topk returns.
//
// Layout (both kernels): one warp owns 32 (query, item) rows at a time.  For every 32-column slice of d it stages the 32 gathered
// item rows (and, for pairs, the 32 user rows) in shared memory with coalesced loads -- 16-byte loads when rows and d allow -- at a
// padded pitch of 33 floats, then each lane runs its own chain over the slice from shared memory (bank = lane + column: no conflicts).
//
// Re-ranking keeps a running top-K per query in the warp's shared memory as packed 64-bit keys (rank_key.cuh: ascending keys are
// (score desc, id asc), NaN after every number, and a repeated id becomes two adjacent equal keys).  Candidates
// that cannot beat the current K-th key are dropped on arrival; the rest are appended to a staging run behind the kept list, and
// when the buffer is full (or the row ends) the warp sorts kept + staged with a bitonic network sized to the next power of two of
// that count (not to the buffer), drops repeated keys and keeps the first K.  A 10..200-candidate row is one 32..256-wide sort.
#include "common.cuh"
#include "rank_key.cuh"

namespace llmrec {

constexpr int kRrWarps = 8;          // rerank: warps per block (one query row per warp at a time)
constexpr int kPairWarps = 4;        // score_pairs: warps per block (two staged 32-row slices each, static shared memory)
constexpr int kPitch = 33;           // staged row pitch in floats

// tile[r * kPitch + c] = X[row_r * ld + j0 + c] for the 32 rows of the warp (row_r = lane r's `row`, < 0: not loaded), c < min(32, d - j0)
template <bool VEC>
__device__ __forceinline__ void stage_rows(float* tile, const float* __restrict__ X, int64_t ld, int row, int j0, int d, int lane) {
  if (VEC) {                                           // 8 float4 per row slice; ld, d and X are multiples of 4 floats
#pragma unroll
    for (int it = 0; it < 8; ++it) {
      const int r = it * 4 + (lane >> 3), q = lane & 7;
      const int rr = __shfl_sync(0xffffffffu, row, r);
      const int c = j0 + 4 * q;
      if (rr >= 0 && c < d) {
        const float4 v = ldg4(X + (int64_t)rr * ld + c);
        float* t = tile + r * kPitch + 4 * q;
        t[0] = v.x; t[1] = v.y; t[2] = v.z; t[3] = v.w;
      }
    }
  } else {
    const int c = j0 + lane;
#pragma unroll 4
    for (int r = 0; r < 32; ++r) {
      const int rr = __shfl_sync(0xffffffffu, row, r);
      if (rr >= 0 && c < d) tile[r * kPitch + lane] = __ldg(X + (int64_t)rr * ld + c);
    }
  }
}

// out[p] = <U[qrow[p]], I[item[p]]>; a negative id gives NaN
template <bool VEC>
__global__ void __launch_bounds__(kPairWarps * 32) score_pairs_kernel(const float* __restrict__ U, int64_t ldu, const float* __restrict__ I, int64_t ldi,
                                                                    const int* __restrict__ qrow, const int* __restrict__ item, int n, int d,
                                                                    float* __restrict__ out) {
  __shared__ float sm[kPairWarps][2][32 * kPitch];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  float* tu = sm[w][0];
  float* ti = sm[w][1];
  const int64_t n_groups = ((int64_t)n + 31) / 32;
  for (int64_t g = (int64_t)blockIdx.x * kPairWarps + w; g < n_groups; g += (int64_t)gridDim.x * kPairWarps) {
    const int64_t p = g * 32 + lane;
    int u = -1, i = -1;
    if (p < n) { u = qrow[p]; i = item[p]; }
    const bool ok = u >= 0 && i >= 0;
    if (!ok) u = i = -1;
    float a = 0.f;
    for (int j0 = 0; j0 < d; j0 += 32) {
      __syncwarp();
      stage_rows<VEC>(tu, U, ldu, u, j0, d, lane);
      stage_rows<VEC>(ti, I, ldi, i, j0, d, lane);
      __syncwarp();
      const int nj = min(32, d - j0);
      const float* ur = tu + lane * kPitch;
      const float* ir = ti + lane * kPitch;
      for (int j = 0; j < nj; ++j) a = fmaf(ur[j], ir[j], a);
    }
    if (p < n) out[p] = ok ? a : __int_as_float(0x7fc00000);
  }
}

__device__ __forceinline__ bool in_sorted(const int* __restrict__ a, int lo, int hi, int v) {
  while (lo < hi) { const int m = (lo + hi) >> 1; const int x = __ldg(a + m); if (x == v) return true; if (x < v) lo = m + 1; else hi = m; }
  return false;
}

template <bool VEC>
__global__ void __launch_bounds__(kRrWarps * 32) rerank_kernel(const float* __restrict__ U, int64_t ldu, const float* __restrict__ I, int64_t ldi,
                                                               const int* __restrict__ qrow, int m, const int* __restrict__ crp, const int* __restrict__ ccol,
                                                               const int* __restrict__ mrp, const int* __restrict__ mcol, int n_catalog, int d, int K,
                                                               int cap, int* __restrict__ out_idx, float* __restrict__ out_val) {
  extern __shared__ __align__(16) uint8_t rr_smem[];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  uint64_t* buf = reinterpret_cast<uint64_t*>(rr_smem) + (size_t)w * cap;
  float* ti = reinterpret_cast<float*>(reinterpret_cast<uint64_t*>(rr_smem) + (size_t)kRrWarps * cap) + (size_t)w * (32 * kPitch + 32);
  float* us = ti + 32 * kPitch;
  for (int r = blockIdx.x * kRrWarps + w; r < m; r += gridDim.x * kRrWarps) {
    const int q = qrow[r];
    const int c0 = crp[r], c1 = crp[r + 1];
    const int m0 = mrp ? mrp[q] : 0, m1 = mrp ? mrp[q + 1] : 0;
    int nb = 0, ns = 0;
    uint64_t thr = kNoKey;                          // a candidate enters only below the K-th kept key
    for (int e0 = c0; e0 < c1; e0 += 32) {
      if (nb + ns + 32 > cap) {
        flush_run(buf, &nb, ns, K, lane);
        ns = 0;
        thr = nb == K ? buf[K - 1] : kNoKey;
      }
      const int e = e0 + lane;
      int id = e < c1 ? ccol[e] : -1;
      if (id >= n_catalog || (id >= 0 && m1 > m0 && in_sorted(mcol, m0, m1, id))) id = -1;
      float a = 0.f;
      for (int j0 = 0; j0 < d; j0 += 32) {
        __syncwarp();
        us[lane] = j0 + lane < d ? __ldg(U + (int64_t)q * ldu + j0 + lane) : 0.f;
        stage_rows<VEC>(ti, I, ldi, id, j0, d, lane);
        __syncwarp();
        const int nj = min(32, d - j0);
        const float* ir = ti + lane * kPitch;
        for (int j = 0; j < nj; ++j) a = fmaf(us[j], ir[j], a);
      }
      const uint64_t key = id >= 0 ? rank_key(a, id) : kNoKey;
      const bool take = key < thr;
      const unsigned bal = __ballot_sync(0xffffffffu, take);
      if (take) buf[nb + ns + __popc(bal & ((1u << lane) - 1u))] = key;
      ns += __popc(bal);
    }
    __syncwarp();
    flush_run(buf, &nb, ns, K, lane);
    __syncwarp();
    for (int k = lane; k < K; k += 32) {
      const bool has = k < nb;
      const uint64_t key = has ? buf[k] : kNoKey;
      out_idx[(int64_t)r * K + k] = has ? (int)(uint32_t)key : -1;
      out_val[(int64_t)r * K + k] = has ? key_score(key) : -INFINITY;
    }
    __syncwarp();
  }
}

static bool vec_ok(const float* X, int64_t ld, int d) { return aligned16(X) && ld % 4 == 0 && d % 4 == 0; }

// running top-K buffer per warp: room for K kept keys and at least 32 (and up to 256) staged ones
static int rerank_cap(int K) {
  int c = 256;
  while (c < K + 32) c <<= 1;
  return c;
}

}  // namespace llmrec

extern "C" int llmrec_score_pairs_f32(const float* U, int64_t ldu, const float* I, int64_t ldi, const int32_t* qrow, const int32_t* item,
                                      int32_t n, int32_t d, float* out, llmrec_stream_t stream) {
  LLMREC_REQUIRE_DEVICE();
  LLMREC_CHECK_ARG(n >= 0 && d >= 1, "score_pairs: n = %d, d = %d (need n >= 0, d >= 1)", n, d);
  if (n == 0) return 0;
  LLMREC_CHECK_ARG(U && I && qrow && item && out && ldu >= d && ldi >= d, "score_pairs: null operand or leading dimension below d = %d", d);
  using namespace llmrec;
  const int64_t groups = ((int64_t)n + 31) / 32;
  const int64_t want = (groups + kPairWarps - 1) / kPairWarps;
  const unsigned grid = (unsigned)(want < 65535 * 16 ? want : 65535 * 16);
  cudaStream_t st = as_stream(stream);
  if (vec_ok(U, ldu, d) && vec_ok(I, ldi, d))
    score_pairs_kernel<true><<<grid, kPairWarps * 32, 0, st>>>(U, ldu, I, ldi, qrow, item, n, d, out);
  else
    score_pairs_kernel<false><<<grid, kPairWarps * 32, 0, st>>>(U, ldu, I, ldi, qrow, item, n, d, out);
  LLMREC_CHECK_LAUNCH("score_pairs");
  return 0;
}

extern "C" int llmrec_rerank_f32(const float* U, int64_t ldu, const float* I, int64_t ldi, const int32_t* qrow, int32_t m,
                                 const int32_t* cand_rowptr, const int32_t* cand_col, const int32_t* mask_rowptr, const int32_t* mask_col,
                                 int32_t n_catalog, int32_t d, int32_t K, int32_t* out_idx, float* out_val, llmrec_stream_t stream) {
  LLMREC_REQUIRE_DEVICE();
  LLMREC_CHECK_ARG(K >= 1 && K <= LLMREC_RERANK_MAX_K, "rerank: K = %d outside 1..%d", K, LLMREC_RERANK_MAX_K);
  LLMREC_CHECK_ARG(m >= 0 && d >= 1 && n_catalog >= 0, "rerank: m = %d, d = %d, n_catalog = %d (need m >= 0, d >= 1, n_catalog >= 0)", m, d, n_catalog);
  if (m == 0) return 0;
  LLMREC_CHECK_ARG(U && I && qrow && cand_rowptr && out_idx && out_val && ldu >= d && ldi >= d,
                   "rerank: null operand or leading dimension below d = %d", d);
  using namespace llmrec;
  const int cap = rerank_cap(K);
  const size_t smem = (size_t)kRrWarps * ((size_t)cap * sizeof(uint64_t) + (32 * kPitch + 32) * sizeof(float));
  const int64_t want = ((int64_t)m + kRrWarps - 1) / kRrWarps;
  const unsigned grid = (unsigned)(want < 65535 * 16 ? want : 65535 * 16);
  cudaStream_t st = as_stream(stream);
  if (vec_ok(U, ldu, d) && vec_ok(I, ldi, d)) {
    LLMREC_CHECK_CUDA(cudaFuncSetAttribute(rerank_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    rerank_kernel<true><<<grid, kRrWarps * 32, smem, st>>>(U, ldu, I, ldi, qrow, m, cand_rowptr, cand_col, mask_rowptr, mask_col, n_catalog, d, K,
                                                           cap, out_idx, out_val);
  } else {
    LLMREC_CHECK_CUDA(cudaFuncSetAttribute(rerank_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    rerank_kernel<false><<<grid, kRrWarps * 32, smem, st>>>(U, ldu, I, ldi, qrow, m, cand_rowptr, cand_col, mask_rowptr, mask_col, n_catalog, d, K,
                                                            cap, out_idx, out_val);
  }
  LLMREC_CHECK_LAUNCH("rerank");
  return 0;
}
