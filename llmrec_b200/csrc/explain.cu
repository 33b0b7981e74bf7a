// Exact attribution of scores <U[u], I[i]> to the query's history items and the model's channels.
//
// Every user-side term of the fusion except two is linear in the user's row of ui = diag(su) R: Fu = ui.Pi, prof_u = ui.prof_i and
// Ul[l] = ui.Il[l-1] for l < L.  The fusion normalises each side row with one scale per user and channel, so a score splits into one
// term per (history item j, channel) plus the user's own ID layer and the softmax layer l = L:
//   id channel:    ((sum_{l=1..L-1} dot(Il[l-1][j], I[i])) * su) * inv                 (0 when L = 1)
//   side term t:   dot(src_t[j], I[i]) * w_t,   w_t = (coef_t / max(sqrt(ss_t), 1e-12)) * su
//   own = dot(Ul[0][u], I[i]) * inv,   last = dot(Ul[L][u], I[i]) * inv,   inv = 1 / (L + 1)
// with src_t the item-side source of side term t (a Pi block or prof_i), ss_t the squared norm of the user's fused side row, and dot
// the sequential chain a = fmaf(x[k], y[k], a), k = 0..d-1, from a = 0 (the chain of score_pairs_kernel and rerank_kernel); ss_t is
// the same chain over x[k] * x[k].  Each product and sum is one fp32 operation in the order written, so every output has one value,
// whatever the grouping of the launch.
//
// explain_kernel: one block per (query, chunk of up to kExPT targets).  The chunk's target rows I[i] are staged once in shared memory
// at an odd pitch; the history is streamed in tiles: each history item's n_id + n_side source rows are gathered once per chunk and
// every thread runs whole chains out of shared memory for (target, item, channel) outputs, consecutive threads taking consecutive
// channels and items of one target, so their writes are contiguous and their source rows fall in distinct banks.
// explain_top_kernel: one warp per (query, target) selects the N history items with the largest total (the channels summed in order,
// in fp32) by (total desc, id asc) with the running top-K of rank_key.cuh.
#include "common.cuh"
#include "rank_key.cuh"

namespace llmrec {

constexpr int kExThreads = 128;      // explain_kernel: threads per block
constexpr int kExPT = 64;            // targets per block
constexpr int kExMaxId = 7;          // id-channel sources Il[0 .. L-2]
constexpr int kExMaxSides = 16;
constexpr int kExTopWarps = 4;       // explain_top_kernel: warps per block (one (query, target) at a time each)
constexpr int kExTopCap = 128;       // running top-N buffer per warp: N <= 64 kept + 32 staged fit

struct ExplainParams {
  const float* own_src; int64_t ld_own;
  const float* last_src; int64_t ld_last;
  const float* side_usr[kExMaxSides]; int64_t ld_side_usr[kExMaxSides];
  const float* side_src[kExMaxSides]; int64_t ld_side_src[kExMaxSides]; float coef[kExMaxSides]; int n_side;
  const float* id_src[kExMaxId]; int64_t ld_id[kExMaxId]; int n_id;
  const float* I; int64_t ldi; int d; float inv;
  const int* qrow; const float* su; const int* hrp; const int* hcol;
  const int* targets; int P; int n_catalog;
  float* contrib; float* own; float* last;
  int pitch; int ht;                 // shared row pitch (odd), history items per tile
};

__device__ __forceinline__ float dot_chain(const float* x, const float* y, int d) {
  float a = 0.f;
  for (int k = 0; k < d; ++k) a = fmaf(x[k], y[k], a);
  return a;
}

// dst[k] = src[k] for k < d (src null: zeros), by one warp
__device__ __forceinline__ void stage_row(float* dst, const float* __restrict__ src, int d, int lane) {
  for (int k = lane; k < d; k += 32) dst[k] = src ? __ldg(src + k) : 0.f;
}

__global__ void __launch_bounds__(kExThreads) explain_kernel(const ExplainParams p) {
  extern __shared__ __align__(16) float ex_smem[];
  const int b = blockIdx.x, p0 = blockIdx.y * kExPT;
  const int np = min(kExPT, p.P - p0);
  const int pitch = p.pitch, d = p.d, C = 1 + p.n_side, R = p.n_id + p.n_side;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
  float* T = ex_smem;                                     // [np][pitch] target rows
  float* Uq = T + kExPT * pitch;                          // [2][pitch] Ul[0][u], Ul[L][u]
  float* w = Uq + 2 * pitch;                              // [kExMaxSides] side weights w_t
  int* tgt = reinterpret_cast<int*>(w + kExMaxSides);     // [kExPT] target ids of the chunk, -1 = padding
  int* hid = tgt + kExPT;                                 // [ht] history ids of the tile
  float* Src = reinterpret_cast<float*>(hid + p.ht);      // [ht * R][pitch] gathered source rows

  const int q = __ldg(p.qrow + b);
  const float su = __ldg(p.su + b);
  for (int x = tid; x < np; x += blockDim.x) {
    const int id = __ldg(p.targets + (int64_t)b * p.P + p0 + x);
    tgt[x] = (id >= 0 && id < p.n_catalog) ? id : -1;
  }
  if (tid < p.n_side) {
    const float* x = p.side_usr[tid] + (int64_t)q * p.ld_side_usr[tid];
    float ss = 0.f;
    for (int k = 0; k < d; ++k) { const float v = __ldg(x + k); ss = fmaf(v, v, ss); }
    w[tid] = (p.coef[tid] / fmaxf(sqrtf(ss), 1e-12f)) * su;
  }
  __syncthreads();
  for (int r = warp; r < np + 2; r += nw) {
    if (r < np) stage_row(T + r * pitch, tgt[r] >= 0 ? p.I + (int64_t)tgt[r] * p.ldi : nullptr, d, lane);
    else if (r == np) stage_row(Uq, p.own_src + (int64_t)q * p.ld_own, d, lane);
    else stage_row(Uq + pitch, p.last_src + (int64_t)q * p.ld_last, d, lane);
  }
  __syncthreads();
  for (int x = tid; x < 2 * np; x += blockDim.x) {
    const int pp = x >> 1, which = x & 1;
    const float v = tgt[pp] >= 0 ? dot_chain(Uq + which * pitch, T + pp * pitch, d) * p.inv : 0.f;
    (which ? p.last : p.own)[(int64_t)b * p.P + p0 + pp] = v;
  }
  const int h0 = __ldg(p.hrp + b), H = __ldg(p.hrp + b + 1) - h0;
  const int64_t base = (int64_t)p.P * h0;                 // the query's first contrib row: its block is [P x H x C]
  for (int t0 = 0; t0 < H; t0 += p.ht) {
    const int nh = min(p.ht, H - t0);
    __syncthreads();                                      // the previous tile's rows are read
    for (int x = tid; x < nh; x += blockDim.x) hid[x] = __ldg(p.hcol + h0 + t0 + x);
    __syncthreads();
    for (int r = warp; r < nh * R; r += nw) {
      const int hh = r / R, s = r - hh * R;
      const int64_t j = hid[hh];
      const float* src = s < p.n_id ? p.id_src[s] + j * p.ld_id[s] : p.side_src[s - p.n_id] + j * p.ld_side_src[s - p.n_id];
      stage_row(Src + r * pitch, src, d, lane);
    }
    __syncthreads();
    const int per_p = nh * C;
    for (int x = tid; x < np * per_p; x += blockDim.x) {
      const int pp = x / per_p, rem = x - pp * per_p, hh = rem / C, c = rem - hh * C;
      float v = 0.f;
      if (tgt[pp] >= 0) {
        const float* tr = T + pp * pitch;
        const float* sr = Src + hh * R * pitch;
        if (c == 0) {
          float s = 0.f;
          for (int l = 0; l < p.n_id; ++l) s += dot_chain(sr + l * pitch, tr, d);
          v = (s * su) * p.inv;
        } else {
          v = dot_chain(sr + (p.n_id + c - 1) * pitch, tr, d) * w[c - 1];
        }
      }
      p.contrib[(base + (int64_t)(p0 + pp) * H + t0 + hh) * C + c] = v;
    }
  }
}

__global__ void __launch_bounds__(kExTopWarps * 32) explain_top_kernel(const float* __restrict__ contrib, const int* __restrict__ hrp,
                                                                      const int* __restrict__ hcol, const int* __restrict__ targets,
                                                                      int m, int P, int n_catalog, int C, int N,
                                                                      int* __restrict__ top_ids, float* __restrict__ top_vals) {
  __shared__ uint64_t sbuf[kExTopWarps][kExTopCap];
  const int lane = threadIdx.x & 31, wi = threadIdx.x >> 5;
  uint64_t* buf = sbuf[wi];
  const int64_t n_pairs = (int64_t)m * P;
  for (int64_t g = (int64_t)blockIdx.x * kExTopWarps + wi; g < n_pairs; g += (int64_t)gridDim.x * kExTopWarps) {
    const int b = (int)(g / P), pp = (int)(g - (int64_t)b * P);
    const int id = __ldg(targets + g);
    int* oi = top_ids + g * N;
    float* ov = top_vals + g * N;
    if (id < 0 || id >= n_catalog) {                     // padding target: zeros, no item
      for (int k = lane; k < N; k += 32) { oi[k] = -1; ov[k] = 0.f; }
      continue;
    }
    const int h0 = __ldg(hrp + b), H = __ldg(hrp + b + 1) - h0;
    const float* rows = contrib + ((int64_t)P * h0 + (int64_t)pp * H) * C;
    int nb = 0, ns = 0;
    uint64_t thr = kNoKey;                               // an item enters only below the N-th kept key
    for (int e0 = 0; e0 < H; e0 += 32) {
      if (nb + ns + 32 > kExTopCap) {
        flush_run(buf, &nb, ns, N, lane);
        ns = 0;
        thr = nb == N ? buf[N - 1] : kNoKey;
      }
      const int e = e0 + lane;
      uint64_t key = kNoKey;
      if (e < H) {
        float t = 0.f;
        for (int c = 0; c < C; ++c) t += __ldg(rows + (int64_t)e * C + c);
        key = rank_key(t, __ldg(hcol + h0 + e));
      }
      const bool take = key < thr;
      const unsigned bal = __ballot_sync(0xffffffffu, take);
      if (take) buf[nb + ns + __popc(bal & ((1u << lane) - 1u))] = key;
      ns += __popc(bal);
    }
    __syncwarp();
    flush_run(buf, &nb, ns, N, lane);
    __syncwarp();
    for (int k = lane; k < N; k += 32) {
      const bool has = k < nb;
      const uint64_t key = has ? buf[k] : kNoKey;
      oi[k] = has ? (int)(uint32_t)key : -1;
      ov[k] = has ? key_score(key) : -INFINITY;
    }
    __syncwarp();
  }
}

// shared bytes of explain_kernel for a tile of ht history items
static size_t explain_smem(int pitch, int R, int ht) {
  return sizeof(float) * ((size_t)(kExPT + 2 + (size_t)ht * R) * pitch + kExMaxSides) + sizeof(int) * (kExPT + ht);
}

}  // namespace llmrec

extern "C" int llmrec_explain_f32(const float* own_src, int64_t ld_own, const float* last_src, int64_t ld_last,
                                  const float* const* side_usr, const int64_t* ld_side_usr, const float* const* side_src,
                                  const int64_t* ld_side_src, const float* coef, int32_t n_side, const float* const* id_src,
                                  const int64_t* ld_id, int32_t n_id, const float* I, int64_t ldi, int32_t n_catalog, int32_t d,
                                  int32_t n_layers, const int32_t* qrow, const float* su, int32_t m, const int32_t* hist_rowptr,
                                  const int32_t* hist_col, const int32_t* targets, int32_t P, float* contrib, float* own, float* last,
                                  int32_t top_n, int32_t* top_ids, float* top_vals, llmrec_stream_t stream) {
  using namespace llmrec;
  LLMREC_REQUIRE_DEVICE();
  LLMREC_CHECK_ARG(m >= 0 && P >= 0 && d >= 1 && n_catalog >= 0, "explain: m = %d, P = %d, d = %d, n_catalog = %d (need m, P, n_catalog >= 0, d >= 1)",
                   m, P, d, n_catalog);
  LLMREC_CHECK_ARG(n_side >= 0 && n_side <= kExMaxSides && n_id >= 0 && n_id <= kExMaxId && n_layers == n_id + 2,
                   "explain: n_side = %d (0..%d), n_id = %d (0..%d), n_layers = %d (L + 1 layers give L - 1 id sources: n_id + 2)", n_side, kExMaxSides, n_id, kExMaxId, n_layers);
  LLMREC_CHECK_ARG(top_n == 0 || (top_n >= 1 && top_n <= LLMREC_EXPLAIN_MAX_TOP && top_ids && top_vals),
                   "explain: top_n = %d (0, or 1..%d with both top outputs)", top_n, LLMREC_EXPLAIN_MAX_TOP);
  if (m == 0 || P == 0) return 0;
  LLMREC_CHECK_ARG(own_src && last_src && I && qrow && su && hist_rowptr && contrib && own && last && ld_own >= d && ld_last >= d && ldi >= d,
                   "explain: null operand or leading dimension below d = %d", d);
  ExplainParams p{};
  p.own_src = own_src; p.ld_own = ld_own; p.last_src = last_src; p.ld_last = ld_last;
  for (int t = 0; t < n_side; ++t) {
    LLMREC_CHECK_ARG(side_usr[t] && side_src[t] && ld_side_usr[t] >= d && ld_side_src[t] >= d, "explain: side term %d null or ld below d", t);
    p.side_usr[t] = side_usr[t]; p.ld_side_usr[t] = ld_side_usr[t];
    p.side_src[t] = side_src[t]; p.ld_side_src[t] = ld_side_src[t]; p.coef[t] = coef[t];
  }
  for (int l = 0; l < n_id; ++l) {
    LLMREC_CHECK_ARG(id_src[l] && ld_id[l] >= d, "explain: id source %d null or ld below d", l);
    p.id_src[l] = id_src[l]; p.ld_id[l] = ld_id[l];
  }
  p.n_side = n_side; p.n_id = n_id;
  p.I = I; p.ldi = ldi; p.d = d; p.inv = 1.0f / (float)n_layers;
  p.qrow = qrow; p.su = su; p.hrp = hist_rowptr; p.hcol = hist_col; p.targets = targets; p.P = P; p.n_catalog = n_catalog;
  p.contrib = contrib; p.own = own; p.last = last;
  p.pitch = d | 1;
  const int R = n_id + n_side, C = 1 + n_side;
  // history items per tile: enough (target, item, channel) outputs for every thread, within the shared-memory budget
  int ht = 1;
  while (ht < 32 && (size_t)ht * C * min(P, kExPT) < 4 * kExThreads && explain_smem(p.pitch, R, 2 * ht) <= 96 * 1024) ht *= 2;
  p.ht = ht;
  const size_t smem = explain_smem(p.pitch, R, ht);
  LLMREC_CHECK_ARG(smem <= 227 * 1024, "explain: d = %d with %d source rows per item needs %zu bytes of shared memory", d, R, smem);
  cudaStream_t st = as_stream(stream);
  LLMREC_CHECK_CUDA(cudaFuncSetAttribute(explain_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const dim3 grid((unsigned)m, (unsigned)((P + kExPT - 1) / kExPT));
  explain_kernel<<<grid, kExThreads, smem, st>>>(p);
  LLMREC_CHECK_LAUNCH("explain");
  if (top_n > 0) {
    const int64_t want = ((int64_t)m * P + kExTopWarps - 1) / kExTopWarps;
    const unsigned g = (unsigned)(want < 65535 * 16 ? want : 65535 * 16);
    explain_top_kernel<<<g, kExTopWarps * 32, 0, st>>>(contrib, hist_rowptr, hist_col, targets, m, P, n_catalog, C, top_n, top_ids, top_vals);
    LLMREC_CHECK_LAUNCH("explain_top");
  }
  return 0;
}
