// Diversified recommendations: greedy maximal-marginal-relevance selection of K entries from each query's pool of P scored items.
//
// Pool entry p = (id_p, s_p).  X holds the normalised catalog rows; cos(a, b) is the sequential chain c = fmaf(X[a][j], X[b][j], c),
// j = 0..d-1, from c = 0 (the chain of similar_items' returned cosines).  With mu = 1 - lambda (one fp32 subtract):
//   round 1 picks the smallest rank_key(s_p, id_p) (score desc, id asc, NaN last);
//   after each pick k, every unpicked entry with id_k retires, every other one takes m_p = max(m_p, cos(id_p, id_k)) (m_p from -inf,
//   a NaN cosine never replaces it);
//   round t >= 2 picks the smallest rank_key(obj_p, id_p), obj_p = lambda * s_p - mu * m_p (two multiplies and a subtract, each
//   rounded once: __fmul_rn / __fsub_rn keep nvcc from contracting them into an FMA); equal keys go to the lower pool position.
// Every output is one exact fp32 value, so a query's result does not depend on the other queries of the launch.
//
// Layout: one block per query, threads own pool entries p = tid + e * blockDim (at most kDvMaxE each, state in registers).  When the
// pool's rows fit kDvPoolBudget bytes at an odd pitch (d | 1) they are staged once in shared memory and a round reads the picked row
// from there; otherwise a round stages the picked row in shared memory and each thread streams its entries' rows from L2.  A round is
// the cosine update of every owned entry (one whole chain each, K * P * d FMAs per query in all, not the P^2 * d of a Gram matrix),
// then a block-wide argmin of (64-bit key, position): warp shuffles, then one shared-memory step across warps.  SIMT by design: a
// tensor-core dot product reassociates the chain.
#include "common.cuh"
#include "rank_key.cuh"

namespace llmrec {

constexpr int kDvMaxThreads = 256;
constexpr int kDvMaxE = LLMREC_RERANK_MAX_K / kDvMaxThreads;   // pool entries per thread
constexpr int kDvWarps = kDvMaxThreads / 32;
constexpr size_t kDvPoolBudget = 110 * 1024;                   // pool rows in shared memory: two blocks still fit an SM

__device__ __forceinline__ void better(uint64_t& k, int& p, uint64_t k2, int p2) {
  if (k2 < k || (k2 == k && p2 < p)) { k = k2; p = p2; }
}

template <bool SHARED_POOL>
__global__ void __launch_bounds__(kDvMaxThreads) diversify_kernel(const float* __restrict__ X, int64_t ldx, const int* __restrict__ pool_ids,
                                                                  const float* __restrict__ pool_scores, int64_t ldp, int P, int n_catalog,
                                                                  int d, int K, float lam, int* __restrict__ out_idx,
                                                                  float* __restrict__ out_val, float* __restrict__ out_sim) {
  extern __shared__ __align__(16) float dv_smem[];
  __shared__ uint64_t red_key[2][kDvWarps];
  __shared__ int red_pos[2][kDvWarps];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, T = blockDim.x, nw = T >> 5;
  const int pitch = d | 1;
  const float mu = __fsub_rn(1.f, lam);
  float* xk = dv_smem;                                 // streamed pool: the picked row; shared pool: rows [P][pitch]

  int id[kDvMaxE];
  float s[kDvMaxE], mx[kDvMaxE];
#pragma unroll
  for (int e = 0; e < kDvMaxE; ++e) {
    const int p = tid + e * T;
    int v = -1;
    float sc = 0.f;
    if (p < P) {
      v = __ldg(pool_ids + (int64_t)b * ldp + p);
      sc = __ldg(pool_scores + (int64_t)b * ldp + p);
    }
    id[e] = (v >= 0 && v < n_catalog) ? v : -1;        // out of range = padding
    s[e] = sc;
    mx[e] = -INFINITY;
  }
  if (SHARED_POOL) {
    for (int r = warp; r < P; r += nw) {               // one warp per row, coalesced
      const int v = __ldg(pool_ids + (int64_t)b * ldp + r);
      if (v >= 0 && v < n_catalog)
        for (int j = lane; j < d; j += 32) dv_smem[r * pitch + j] = __ldg(X + (int64_t)v * ldx + j);
    }
    __syncthreads();
  }
  const int64_t o = (int64_t)b * K;
  int picked = 0;
  for (int t = 0; t < K; ++t) {
    uint64_t bk = kNoKey;
    int bp = 0x7fffffff;
#pragma unroll
    for (int e = 0; e < kDvMaxE; ++e) {
      if (id[e] < 0) continue;
      const float obj = t == 0 ? s[e] : __fsub_rn(__fmul_rn(lam, s[e]), __fmul_rn(mu, mx[e]));
      better(bk, bp, rank_key(obj, id[e]), tid + e * T);
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const uint64_t k2 = __shfl_xor_sync(0xffffffffu, bk, off);
      const int p2 = __shfl_xor_sync(0xffffffffu, bp, off);
      better(bk, bp, k2, p2);
    }
    const int par = t & 1;                             // double-buffered: round t + 1 writes the other half before all have read this one
    if (lane == 0) { red_key[par][warp] = bk; red_pos[par][warp] = bp; }
    __syncthreads();
    bk = red_key[par][0]; bp = red_pos[par][0];
    for (int w = 1; w < nw; ++w) better(bk, bp, red_key[par][w], red_pos[par][w]);
    if (bk == kNoKey) break;                           // no valid entry left: the same decision in every thread
    const int kid = (int)(uint32_t)bk;
#pragma unroll
    for (int e = 0; e < kDvMaxE; ++e) {
      if (tid + e * T == bp) {                         // the owner writes the pick: its score and its m when picked
        out_idx[o + t] = kid;
        out_val[o + t] = s[e];
        out_sim[o + t] = mx[e];
      }
      if (id[e] == kid) id[e] = -1;                    // the pick and its repeats retire
    }
    picked = t + 1;
    if (picked == K) break;
    const float* xr;
    if (SHARED_POOL) {
      xr = dv_smem + bp * pitch;
    } else {
      for (int j = tid; j < d; j += T) xk[j] = __ldg(X + (int64_t)kid * ldx + j);
      __syncthreads();
      xr = xk;
    }
#pragma unroll
    for (int e = 0; e < kDvMaxE; ++e) {
      if (id[e] < 0) continue;
      float c = 0.f;
      if (SHARED_POOL) {
        const float* xp = dv_smem + (tid + e * T) * pitch;
        for (int j = 0; j < d; ++j) c = fmaf(xp[j], xr[j], c);
      } else {
        const float* xp = X + (int64_t)id[e] * ldx;
        for (int j = 0; j < d; ++j) c = fmaf(__ldg(xp + j), xr[j], c);
      }
      if (c > mx[e]) mx[e] = c;                        // a NaN never replaces m
    }
  }
  for (int k = picked + tid; k < K; k += T) {          // fewer than K valid distinct ids: padding
    out_idx[o + k] = -1;
    out_val[o + k] = -INFINITY;
    out_sim[o + k] = -INFINITY;
  }
}

}  // namespace llmrec

extern "C" int llmrec_diversify_f32(const float* X, int64_t ldx, const int32_t* pool_ids, const float* pool_scores, int64_t ldp, int32_t m,
                                    int32_t P, int32_t n_catalog, int32_t d, int32_t K, float lambda, int32_t* out_idx, float* out_val,
                                    float* out_sim, llmrec_stream_t stream) {
  using namespace llmrec;
  LLMREC_REQUIRE_DEVICE();
  LLMREC_CHECK_ARG(K >= 1 && K <= P && P <= LLMREC_RERANK_MAX_K, "diversify: K = %d, P = %d (need 1 <= K <= P <= %d)", K, P,
                   LLMREC_RERANK_MAX_K);
  LLMREC_CHECK_ARG(lambda >= 0.f && lambda <= 1.f, "diversify: lambda = %g (need 0 <= lambda <= 1)", (double)lambda);
  LLMREC_CHECK_ARG(m >= 0 && d >= 1 && n_catalog >= 0, "diversify: m = %d, d = %d, n_catalog = %d (need m >= 0, d >= 1, n_catalog >= 0)",
                   m, d, n_catalog);
  if (m == 0) return 0;
  LLMREC_CHECK_ARG(X && pool_ids && pool_scores && out_idx && out_val && out_sim && ldx >= d && ldp >= P,
                   "diversify: null operand, ldx below d = %d or ldp below P = %d", d, P);
  const int threads = min(kDvMaxThreads, (P + 31) / 32 * 32);
  const size_t pitch = (size_t)(d | 1);
  const size_t pool_bytes = (size_t)P * pitch * sizeof(float);
  cudaStream_t st = as_stream(stream);
  if (pool_bytes <= kDvPoolBudget) {
    LLMREC_CHECK_CUDA(cudaFuncSetAttribute(diversify_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pool_bytes));
    diversify_kernel<true><<<(unsigned)m, threads, pool_bytes, st>>>(X, ldx, pool_ids, pool_scores, ldp, P, n_catalog, d, K, lambda,
                                                                     out_idx, out_val, out_sim);
  } else {
    const size_t row_bytes = (size_t)d * sizeof(float);
    LLMREC_CHECK_ARG(row_bytes <= 200 * 1024, "diversify: d = %d needs %zu bytes of shared memory for the picked row", d, row_bytes);
    LLMREC_CHECK_CUDA(cudaFuncSetAttribute(diversify_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)row_bytes));
    diversify_kernel<false><<<(unsigned)m, threads, row_bytes, st>>>(X, ldx, pool_ids, pool_scores, ldp, P, n_catalog, d, K, lambda,
                                                                      out_idx, out_val, out_sim);
  }
  LLMREC_CHECK_LAUNCH("diversify");
  return 0;
}
