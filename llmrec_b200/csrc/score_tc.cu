// Full-catalog scoring + top-K on the Hopper tensor cores (utility/batch_test.py:149-152 scores, :21-36,100-102 ranking).
//
//   score[b, i] = <U[users[b]], I[i]>   for every item i;  items of the user's train row are excluded;
//   top-K by (score desc, item id asc)  ==  heapq.nlargest over ascending candidates.
//
// The reference materialises the [2048 x n_items] score block, copies it to the host and ranks each user in Python.
// Here the score matrix never exists in memory:
//   * CTA = one warpgroup = (tile of 64 users, slice of the catalog).  The 64 user rows are gathered ONCE, split into
//     TF32 hi/lo and parked in shared memory as the K-major A operand; item rows (pre-split hi/lo copies of I) stream
//     through a TMA-fed shared-memory ring as the B operand; three tf32 wgmmas per k8 step (lo*hi + hi*lo + hi*hi, fp32
//     accumulate in registers) produce a [64 users x 128 items] score tile.
//   * the tile is staged in shared memory and the selection runs one user row per thread over items in ascending id:
//     train-item masking by a merge pointer into the user's sorted train row, threshold test against the thread's
//     current K'-th best, replace-min insertion into a per-thread candidate heap in shared memory (K' = K + 16..32
//     slack).  Ties keep the lower item id (strict > against the minimum; eviction of the largest id among equal minima).
//   * a small exact pass (rescore_topk_kernel) recomputes the K' candidates of every catalog slice in sequential fp32 FMA
//     order -- the same arithmetic as the SIMT reference kernel -- and emits the final top-K by (score desc, id asc), so
//     the 3xTF32 rounding of the selection pass (~1e-5 relative) cannot change the result unless it misranks by more
//     than the slack.
//   * the catalog may be a subset of I given by ascending ids (`among`, llmrec_score_topk_among_f32): the hi/lo copies
//     are gathered compacted, column j of the catalog offers global id among[j] (each tile's 128 ids staged once in
//     shared memory), and mask rows / returned ids stay global.  Ascending ids keep the merge pointer and the tie rule
//     valid unchanged; among == NULL is the identity map (the whole of I).
//   * groups (llmrec_score_topk_group_f32, the GROUP instantiation): the A tile holds the member rows of whole groups,
//     packed in the order given (a tile slot plan built on the host; padding slots are zero rows).  Selection thread t
//     owns group t of the tile: after staging, the whole CTA folds each group's member rows of the score tile into the first
//     of them by the group rule (mean / min / max, common.cuh agg_*), and thread t runs the threshold test, mask merge
//     pointer and heap on its group's row unchanged; mask rows and candidate rows are indexed by group.  rescore_topk_group_kernel recomputes every
//     member's exact chain per candidate and aggregates exactly.  The slack argument carries over: a member's 3xTF32 score
//     is within e of its exact chain, so the mean of n such scores is within e of the exact mean (up to the rounding of
//     an fp32 sum of n terms), and min / max move by at most the largest member error -- the aggregated error is bounded
//     by the largest member error.  Every member is scored: the tensor work equals recommending for each member.
#include <stdlib.h>
#include <string.h>
#include <vector>
#include "common.cuh"
#include "tc_common.cuh"

namespace llmrec {
using namespace tc;

constexpr int SBM = 64;        // users per tile (wgmma M)
constexpr int SBN = 128;       // items per score tile (4 x n32)
constexpr int SBK = 32;        // fp32 per 128-byte swizzle row
constexpr int kStageLd = SBN + 1;   // staged score row pitch: row-per-thread reads hit 32 distinct banks
constexpr uint32_t kTileU = SBM * SBK * 4;   // 8 KiB: one k-block of the hi or lo user tile
constexpr uint32_t kTileI = SBN * SBK * 4;   // 16 KiB: one k-block of the hi or lo item tile

struct ScoreParams {
  CUtensorMap tmIhi, tmIlo;  // [n_items x d] hi / lo copies of I, box {32, 128}, SWIZZLE_128B
  const float* U; long long ldu;
  const int* users; int n_batch, n_items, d;   // n_items: catalog size (rows of the hi / lo copies)
  const int* among;                             // NULL, or catalog column j -> global item id among[j] (ascending)
  const int* mask_rowptr; const int* mask_col;  // train rows, columns sorted ascending
  int Kc, splits, tiles_per_split, stages;
  int* cand_idx; float* cand_val;  // [n_batch][splits][Kc]  (GROUP: [n_groups][splits][Kc])
  // GROUP only (users = the members): slot r of tile t holds members[slot_pos[t * 64 + r]] (-1 = a zero row); tile t holds
  // groups tile_g0[t] .. tile_g0[t+1]; group g's members are rows gofs[g] .. gofs[g] + n of its tile, n from grp_rowptr
  const int* slot_pos; const int* tile_g0; const int* gofs; const int* grp_rowptr;
  int agg;
};

template <int D, bool GROUP>
__global__ void __launch_bounds__(128, 1) score_topk_tc_kernel(const __grid_constant__ ScoreParams P) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr int KB = D / SBK;
  constexpr uint32_t stage_bytes = 2 * kTileI;
  const int stages = P.stages, Kc = P.Kc;
  uint8_t* a_hi = smem;                                   // [KB][64 users][32] K-major, swizzled
  uint8_t* a_lo = smem + KB * kTileU;
  uint8_t* ring = smem + 2 * KB * kTileU;                 // stages x (I_hi tile | I_lo tile)
  float* stg = reinterpret_cast<float*>(ring + (size_t)stages * stage_bytes);   // [64][kStageLd] staged scores
  float* lv = stg + SBM * kStageLd;                       // heap values [Kc][64]
  int* li = reinterpret_cast<int*>(lv + (size_t)Kc * SBM);   // heap ids [Kc][64]
  uint64_t* full = reinterpret_cast<uint64_t*>(li + (size_t)Kc * SBM);
  int* tile_ids = reinterpret_cast<int*>(full + 8);       // [SBN] global ids of the current tile's columns (among only)

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int utile = blockIdx.x, split = blockIdx.y;
  const int tile0 = split * P.tiles_per_split;
  const int n_item_tiles = (P.n_items + SBN - 1) / SBN;
  const int tile1 = min(n_item_tiles, tile0 + P.tiles_per_split);
  const int n_steps = (tile1 - tile0) * KB;
  auto issue = [&](int g) {
    const int s = g % stages, t = tile0 + g / KB, kb = g % KB;
    uint8_t* dst = ring + (size_t)s * stage_bytes;
    mbar_arrive_expect_tx(&full[s], stage_bytes);
    tma_load_2d(dst, &P.tmIhi, &full[s], kb * SBK, t * SBN);
    tma_load_2d(dst + kTileI, &P.tmIlo, &full[s], kb * SBK, t * SBN);
  };
  if (tid == 0) {
    prefetch_tmap(&P.tmIhi); prefetch_tmap(&P.tmIlo);
    for (int s = 0; s < stages; ++s) mbar_init(&full[s], 1);
    fence_barrier_init();
    for (int g = 0; g < stages && g < n_steps; ++g) issue(g);
  }
  // A operand: gather the 64 user rows, split hi/lo
  for (int i = tid; i < SBM * (D / 4); i += 128) {
    const int r = i / (D / 4), c4 = i - r * (D / 4);
    float4 v;
    if constexpr (GROUP) {
      const int p = __ldg(P.slot_pos + utile * SBM + r);
      v = p >= 0 ? ldg4(P.U + (long long)__ldg(P.users + p) * P.ldu + c4 * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
    } else {
      const int b = utile * SBM + r;
      v = b < P.n_batch ? ldg4(P.U + (long long)P.users[b] * P.ldu + c4 * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    float4 h, l;
    split4(v, h, l);
    const uint32_t off = (uint32_t)(c4 >> 3) * kTileU + sw128_off(r, c4 & 7);
    *reinterpret_cast<float4*>(a_hi + off) = h;
    *reinterpret_cast<float4*>(a_lo + off) = l;
  }
  fence_proxy_async_smem();
  __syncthreads();

  // ===== selection state: thread t < 64 owns user row t of the tile (GROUP: group t of the tile) =====
  const int b = utile * SBM + tid;
  int grp = 0, r0 = tid;   // GROUP: the thread's group and the tile row of its first member
  bool live;
  if constexpr (GROUP) {
    grp = __ldg(P.tile_g0 + utile) + tid;
    live = tid < SBM && grp < __ldg(P.tile_g0 + utile + 1);
    if (live) r0 = __ldg(P.gofs + grp);
  } else {
    live = tid < SBM && b < P.n_batch;
  }
  int mp = 0, mend = 0, next_masked = 0x7fffffff;
  if (live && P.mask_rowptr) {
    const int u = GROUP ? grp : P.users[b];
    mp = P.mask_rowptr[u]; mend = P.mask_rowptr[u + 1];
    next_masked = mp < mend ? __ldg(P.mask_col + mp) : 0x7fffffff;
  }
  // Per-thread binary MIN-heap of the K' best (score, id) seen so far, in shared memory with layout [k][thread]
  // (bank = thread for every k: conflict-free however the heap paths of the 32 lanes diverge).  Heap order: a is
  // "smaller" than b when a.score < b.score, or equal scores and a.id > b.id, so the root is the entry to evict and a
  // new item enters only when strictly better than the root -> ties keep the lower item id.
  float* hv = lv + tid;
  int* hi_ = li + tid;
  auto HV = [&](int k) -> float& { return hv[(size_t)k * SBM]; };
  auto HI = [&](int k) -> int& { return hi_[(size_t)k * SBM]; };
  auto lower = [](float av, int ai, float bv, int bi) { return av < bv || (av == bv && ai > bi); };
  int count = 0;
  float thr = -INFINITY;   // root score once the heap is full
  auto sift_down = [&](int pos, float v, int id, int n) {
    for (;;) {
      int c = 2 * pos + 1;
      if (c >= n) break;
      float cv = HV(c); int ci = HI(c);
      if (c + 1 < n) {
        const float rv = HV(c + 1); const int ri = HI(c + 1);
        if (lower(rv, ri, cv, ci)) { ++c; cv = rv; ci = ri; }
      }
      if (!lower(cv, ci, v, id)) break;
      HV(pos) = cv; HI(pos) = ci;
      pos = c;
    }
    HV(pos) = v; HI(pos) = id;
  };
  // train-item test on the slow path only: merge pointer into the user's SORTED train row.  Offered items arrive in
  // ascending id, so the pointer only moves forward; the usual case is one register compare, no memory access.
  auto is_masked = [&](int item) -> bool {
    while (next_masked < item) { ++mp; next_masked = mp < mend ? __ldg(P.mask_col + mp) : 0x7fffffff; }
    return next_masked == item;
  };
  auto offer = [&](float s, int col, int item) {   // catalog column col holds global item id `item`
    if (col >= P.n_items || is_masked(item)) return;
    if (count < Kc) {
      HV(count) = s; HI(count) = item;
      if (++count == Kc) {
        for (int p = Kc / 2 - 1; p >= 0; --p) sift_down(p, HV(p), HI(p), Kc);   // heapify once
        thr = HV(0);
      }
    } else if (s > thr) {   // (equal score, larger id) never displaces: lowest id wins ties
      sift_down(0, s, item, Kc);
      thr = HV(0);
    }
  };

  float acc[4][16];
  int g = 0;
  for (int t = tile0; t < tile1; ++t) {
#pragma unroll
    for (int c = 0; c < 4; ++c)
#pragma unroll
      for (int i = 0; i < 16; ++i) acc[c][i] = 0.f;
    for (int kb = 0; kb < KB; ++kb, ++g) {
      const int s = g % stages;
      mbar_wait(&full[s], (uint32_t)(g / stages) & 1u);
      const uint32_t bh = smem_u32(ring + (size_t)s * stage_bytes), bl = bh + kTileI;
      const uint32_t ah = smem_u32(a_hi) + kb * kTileU, al = smem_u32(a_lo) + kb * kTileU;
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const uint64_t bhd = gmma_desc_sw128(bh + c * 4096u + kk * 32u);
          wgmma_m64n32k8_tf32(acc[c], gmma_desc_sw128(al + kk * 32u), bhd, 1);                                  // lo * hi
          wgmma_m64n32k8_tf32(acc[c], gmma_desc_sw128(ah + kk * 32u), gmma_desc_sw128(bl + c * 4096u + kk * 32u), 1);   // hi * lo
          wgmma_m64n32k8_tf32(acc[c], gmma_desc_sw128(ah + kk * 32u), bhd, 1);                                  // hi * hi
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      __syncthreads();   // stage s fully read
      if (tid == 0 && g + stages < n_steps) issue(g + stages);
    }
    // registers -> staged [64 users][128 items]
    {
      const int row = warp * 16 + (lane >> 2);
#pragma unroll
      for (int c = 0; c < 4; ++c)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int col = c * 32 + j * 8 + (lane & 3) * 2;
            stg[(row + 8 * h) * kStageLd + col] = acc[c][4 * j + 2 * h];
            stg[(row + 8 * h) * kStageLd + col + 1] = acc[c][4 * j + 2 * h + 1];
          }
    }
    if (P.among) {
      const int col = t * SBN + tid;
      tile_ids[tid] = col < P.n_items ? __ldg(P.among + col) : 0x7fffffff;
    }
    __syncthreads();
    if constexpr (GROUP) {   // fold each group's member rows into its first row: all 128 threads, one (group, column) per step
      const int g0 = __ldg(P.tile_g0 + utile), ng = __ldg(P.tile_g0 + utile + 1) - g0;
#pragma unroll 1
      for (int e = tid; e < ng * SBN; e += 128) {   // consecutive threads take consecutive columns of one group's rows
        const int gg = g0 + e / SBN, c = e % SBN;
        const int n = __ldg(P.grp_rowptr + gg + 1) - __ldg(P.grp_rowptr + gg);
        if (n == 1) continue;
        float* col = stg + __ldg(P.gofs + gg) * kStageLd + c;
        float v = agg_start(P.agg);
#pragma unroll 1
        for (int m = 0; m < n; ++m) v = agg_fold(P.agg, v, col[m * kStageLd]);
        col[0] = agg_end(P.agg, v, n);
      }
      __syncthreads();
    }
    if (live) {
      const float* srow = stg + r0 * kStageLd;
#pragma unroll 1
      for (int c0 = 0; c0 < SBN; c0 += 32) {
        // fast path: one compare per score builds the mask of columns that beat the current threshold
        unsigned hit = 0;
#pragma unroll
        for (int j = 0; j < 32; ++j) hit |= (srow[c0 + j] > thr ? 1u : 0u) << j;
        const int col0 = t * SBN + c0;
        while (hit) {   // slow path: set bits in ascending item id
          const int j = __ffs(hit) - 1;
          hit &= hit - 1;
          const float s = srow[c0 + j];
          if (count < Kc || s > thr) offer(s, col0 + j, P.among ? tile_ids[c0 + j] : col0 + j);
        }
      }
    }
    __syncthreads();   // staging free for the next tile
  }
  if (live) {
    const long long q = GROUP ? grp : b;
    int* oi = P.cand_idx + (q * P.splits + split) * Kc;
    float* ov = P.cand_val + (q * P.splits + split) * Kc;
    for (int k = 0; k < Kc; ++k) {
      const bool has = k < count;
      oi[k] = has ? HI(k) : -1;
      ov[k] = has ? HV(k) : -INFINITY;
    }
  }
}

// I -> hi / lo copies (hi exactly TF32-representable); rows: NULL, or row r of the copies is row rows[r] of X
__global__ void split_hi_lo_kernel(const float* __restrict__ X, long long ldx, const int* __restrict__ rows, long long n, int d,
                                   float* __restrict__ hi, float* __restrict__ lo) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n * d) return;
  const long long r = i / d; const int c = (int)(i - r * d);
  const long long src = rows ? (long long)__ldg(rows + r) : r;
  const float v = X[src * ldx + c]; const float h = tf32_hi(v);
  hi[i] = h; lo[i] = v - h;
}

// exact fp32 rescoring of the candidates of one user + final (score desc, id asc) top-K: ONE WARP per user
constexpr int kMaxCandPerLane = 20;   // 32 x 20 = 640 candidates (<= 6 slices x 96)

// the final top-K of a warp's rescored candidates (lane-owned sc / id, id -1 = none; NaN and -inf never win): K rounds of a warp
// arg-max by (score desc, id asc) -> out_idx[0 .. K) / out_val (may be NULL), padded with -1 / -inf
__device__ __forceinline__ void warp_emit_topk(float (&sc)[kMaxCandPerLane], int (&id)[kMaxCandPerLane], int K, int lane, int* out_idx,
                                               float* out_val) {
  for (int r = 0; r < K; ++r) {
    float best = -INFINITY; int besti = 0x7fffffff, bestq = -1;
#pragma unroll
    for (int q = 0; q < kMaxCandPerLane; ++q) {
      if (id[q] >= 0 && sc[q] != -INFINITY && (sc[q] > best || (sc[q] == best && id[q] < besti))) { best = sc[q]; besti = id[q]; bestq = q; }
    }
    float wb = best; int wi = besti;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, wb, o); const int oi = __shfl_xor_sync(0xffffffffu, wi, o);
      if (ov > wb || (ov == wb && oi < wi)) { wb = ov; wi = oi; }
    }
    const bool ok = wi != 0x7fffffff;
    if (lane == 0) {
      out_idx[r] = ok ? wi : -1;
      if (out_val) out_val[r] = ok ? wb : -INFINITY;
    }
    if (ok && bestq >= 0 && besti == wi) {   // the owning lane retires the winner (ids are unique per user)
#pragma unroll
      for (int q = 0; q < kMaxCandPerLane; ++q) if (q == bestq) id[q] = -1;
    }
  }
}
__global__ void __launch_bounds__(256) rescore_topk_kernel(const float* __restrict__ U, long long ldu, const float* __restrict__ I, long long ldi,
                                                           const int* __restrict__ users, int n_batch, int d, const int* __restrict__ cand_idx,
                                                           int n_cand, int K, int* __restrict__ out_idx, float* __restrict__ out_val) {
  extern __shared__ float sm[];  // 8 warps x d
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int b = blockIdx.x * 8 + w;
  if (b >= n_batch) return;
  float* us = sm + (size_t)w * d;
  const float* u = U + (long long)users[b] * ldu;
  for (int j = lane; j < d; j += 32) us[j] = u[j];
  __syncwarp();
  const int* ci = cand_idx + (long long)b * n_cand;
  float sc[kMaxCandPerLane]; int id[kMaxCandPerLane];
#pragma unroll
  for (int q = 0; q < kMaxCandPerLane; ++q) {
    const int c = q * 32 + lane;
    int item = c < n_cand ? ci[c] : -1;
    float a = -INFINITY;
    if (item >= 0) {
      const float* it = I + (long long)item * ldi;
      a = 0.f;
      for (int j = 0; j < d; ++j) a = fmaf(us[j], it[j], a);   // same order as score_rows_kernel (score_simt.cu)
    }
    sc[q] = a; id[q] = item;
  }
  warp_emit_topk(sc, id, K, lane, out_idx + (long long)b * K, out_val ? out_val + (long long)b * K : nullptr);
}

// exact rescoring for groups: ONE WARP per group; each candidate's group score is every member's fmaf chain (the order of
// score_rows_kernel) in member order, folded by the exact rule (agg_*).  Member rows are warp-uniform loads from L1 / L2.
__global__ void __launch_bounds__(256) rescore_topk_group_kernel(const float* __restrict__ U, long long ldu, const float* __restrict__ I,
                                                                 long long ldi, const int* __restrict__ grp_rowptr, const int* __restrict__ members,
                                                                 int n_groups, int d, int agg, const int* __restrict__ cand_idx, int n_cand, int K,
                                                                 int* __restrict__ out_idx, float* __restrict__ out_val) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int g = blockIdx.x * 8 + w;
  if (g >= n_groups) return;
  const int m0 = __ldg(grp_rowptr + g), m1 = __ldg(grp_rowptr + g + 1);
  const int* ci = cand_idx + (long long)g * n_cand;
  float sc[kMaxCandPerLane]; int id[kMaxCandPerLane];
#pragma unroll
  for (int q = 0; q < kMaxCandPerLane; ++q) {
    const int c = q * 32 + lane;
    const int item = c < n_cand ? ci[c] : -1;
    float v = -INFINITY;
    if (item >= 0) {
      const float* it = I + (long long)item * ldi;
      v = agg_start(agg);
      for (int m = m0; m < m1; ++m) {
        const float* u = U + (long long)__ldg(members + m) * ldu;
        float a = 0.f;
        for (int j = 0; j < d; ++j) a = fmaf(__ldg(u + j), __ldg(it + j), a);
        v = agg_fold(agg, v, a);
      }
      v = agg_end(agg, v, m1 - m0);
    }
    sc[q] = v; id[q] = item;
  }
  warp_emit_topk(sc, id, K, lane, out_idx + (long long)g * K, out_val ? out_val + (long long)g * K : nullptr);
}

bool score_tc_supported(int d, int K, long long ldu, long long ldi, const void* U, const void* I) {
  return (d == 32 || d == 64 || d == 96 || d == 128) && K <= 64 && ldu % 4 == 0 && ldi % 4 == 0 && aligned16(U) && aligned16(I);
}

static int score_kc(int K) { int kc = ((K + 16 + 7) / 8) * 8; return kc > 96 ? 96 : kc; }

static void score_plan(int n_batch, int n_items, int K, int* splits, int* tiles_per_split) {
  const int utiles = (n_batch + SBM - 1) / SBM;
  const int itiles = (n_items + SBN - 1) / SBN;
  int s = utiles >= kNumSMs / 2 ? 1 : (kNumSMs + utiles - 1) / utiles;   // cut the catalog only when user tiles cannot fill the SMs
  const int max_s = itiles / 32 > 0 ? itiles / 32 : 1;   // keep >= 4096 items per slice
  if (s > max_s) s = max_s;
  if (s > 6) s = 6;       // rescore_topk_kernel holds at most 32 x 20 candidates per user
  if (s < 1) s = 1;
  *tiles_per_split = (itiles + s - 1) / s;
  *splits = (itiles + *tiles_per_split - 1) / *tiles_per_split;
  (void)K;
}

long long score_tc_scratch(int n_batch, int n_items, int d, int K) {
  int splits, tps;
  score_plan(n_batch, n_items, K, &splits, &tps);
  return 2LL * n_items * d + 2LL * n_batch * splits * score_kc(K) + 64;
}

// The hi / lo copies of the catalog, the tensor maps, the pipeline depth and the launch of score_topk_tc_kernel<D, GROUP> over
// row_tiles x P.splits CTAs; P's plan, operands and candidate buffers are set by the caller.
template <bool GROUP>
static int launch_select(ScoreParams& P, const float* I, long long ldi, const int* among, int n_items, int d, int row_tiles, float* Ihi,
                         float* Ilo, cudaStream_t st) {
  {
    const long long n = (long long)n_items * d;
    split_hi_lo_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(I, ldi, among, n_items, d, Ihi, Ilo);
    LLMREC_CHECK_LAUNCH("split_hi_lo");
  }
  if (!make_tmap_2d_f32(&P.tmIhi, Ihi, (uint64_t)d, (uint64_t)n_items, (uint64_t)d * 4, SBK, SBN)) return 4;
  if (!make_tmap_2d_f32(&P.tmIlo, Ilo, (uint64_t)d, (uint64_t)n_items, (uint64_t)d * 4, SBK, SBN)) return 4;
  const size_t fixed = (size_t)2 * d * SBM * 4 /*A hi, lo*/ + (size_t)SBM * kStageLd * 4 + (size_t)P.Kc * SBM * 8 /*heaps*/ + 64 /*barriers*/ +
                       (among ? SBN * 4 : 0) /*tile ids*/ + 1024 /*align*/;
  int stages = (int)((227 * 1024 - fixed) / (2 * kTileI));
  if (stages > 4) stages = 4;
  LLMREC_CHECK_ARG(stages >= 2, "score_topk: not enough shared memory for the pipeline");
  P.stages = stages;
  const size_t smem = fixed + (size_t)stages * 2 * kTileI;
  dim3 grid(row_tiles, P.splits);
  switch (d) {
#define LLMREC_CASE(W)                                                                                                               \
  case W:                                                                                                                            \
    LLMREC_CHECK_CUDA(cudaFuncSetAttribute(score_topk_tc_kernel<W, GROUP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    score_topk_tc_kernel<W, GROUP><<<grid, 128, smem, st>>>(P);                                                                      \
    break;
    LLMREC_CASE(32) LLMREC_CASE(64) LLMREC_CASE(96) LLMREC_CASE(128)
#undef LLMREC_CASE
    default: LLMREC_CHECK_ARG(false, "score_topk: no tensor-core kernel for d=%d", d);
  }
  LLMREC_CHECK_LAUNCH("score_topk_tc");
  return 0;
}

// among: NULL (the catalog is I), or n_items ascending ids of rows of I (the catalog is those rows)
int score_topk_tc(const float* U, long long ldu, const float* I, long long ldi, const int* users, int n_batch, const int* among, int n_items, int d,
                  const int* mask_rowptr, const int* mask_col, int K, int* out_idx, float* out_val, float* scratch, long long scratch_elems,
                  cudaStream_t st) {
  LLMREC_CHECK_ARG(scratch && scratch_elems >= score_tc_scratch(n_batch, n_items, d, K), "score_topk: scratch too small");
  ScoreParams P;
  memset(&P, 0, sizeof(P));
  score_plan(n_batch, n_items, K, &P.splits, &P.tiles_per_split);
  P.Kc = score_kc(K);
  float* Ihi = scratch; float* Ilo = scratch + (long long)n_items * d;
  float* cval = Ilo + (long long)n_items * d;
  int* cidx = reinterpret_cast<int*>(cval + (long long)n_batch * P.splits * P.Kc);
  P.U = U; P.ldu = ldu; P.users = users; P.n_batch = n_batch; P.n_items = n_items; P.d = d; P.among = among;
  P.mask_rowptr = mask_rowptr; P.mask_col = mask_col; P.cand_idx = cidx; P.cand_val = cval;
  if (int rc = launch_select<false>(P, I, ldi, among, n_items, d, (n_batch + SBM - 1) / SBM, Ihi, Ilo, st)) return rc;
  const int n_cand = P.splits * P.Kc;
  LLMREC_CHECK_ARG(n_cand <= 32 * kMaxCandPerLane, "score_topk: %d candidates per user exceed the rescoring capacity", n_cand);
  rescore_topk_kernel<<<(n_batch + 7) / 8, 256, (size_t)8 * d * sizeof(float), st>>>(U, ldu, I, ldi, users, n_batch, d, cidx, n_cand, K, out_idx, out_val);
  LLMREC_CHECK_LAUNCH("rescore_topk");
  return 0;
}

// ---- groups ----------------------------------------------------------------------------------------------------------------
// The tile plan of llmrec_score_topk_group_f32 from the host member CSR: groups in the order given, a new tile whenever the next
// group does not fit the current one.  -> the plan's ints in one array: grp_rowptr [n_groups+1], gofs [n_groups],
// tile_g0 [n_tiles+1], slot_pos [n_tiles * 64]; returns n_tiles.
int group_tile_plan(const int* rp, int n_groups, std::vector<int>* plan) {
  std::vector<int> gofs(n_groups), g0(1, 0), slots;
  int fill = 0;
  for (int g = 0; g < n_groups; ++g) {
    const int n = rp[g + 1] - rp[g];
    if (fill + n > SBM) {   // close the tile
      slots.resize(slots.size() + (SBM - fill), -1);
      g0.push_back(g);
      fill = 0;
    }
    gofs[g] = fill;
    for (int j = 0; j < n; ++j) slots.push_back(rp[g] + j);
    fill += n;
  }
  if (fill > 0) { slots.resize(slots.size() + (SBM - fill), -1); g0.push_back(n_groups); }
  const int n_tiles = (int)g0.size() - 1;
  if (plan) {
    plan->assign(rp, rp + n_groups + 1);
    plan->insert(plan->end(), gofs.begin(), gofs.end());
    plan->insert(plan->end(), g0.begin(), g0.end());
    plan->insert(plan->end(), slots.begin(), slots.end());
  }
  return n_tiles;
}

static long long plan_elems(int n_groups, int n_tiles) { return ((2LL * n_groups + 2 + n_tiles + 1 + (long long)n_tiles * SBM) + 3) / 4 * 4; }

long long score_tc_group_scratch(const int* rp, int n_groups, int n_items, int d, int K) {
  const int n_tiles = group_tile_plan(rp, n_groups, nullptr);
  int splits, tps;
  score_plan(n_tiles * SBM, n_items, K, &splits, &tps);
  return 2LL * n_items * d + 2LL * n_groups * splits * score_kc(K) + plan_elems(n_groups, n_tiles) + 64;
}

// rp: the HOST member CSR; members: device rows of U
int score_topk_group_tc(const float* U, long long ldu, const float* I, long long ldi, const int* rp, const int* members, int n_groups,
                        const int* among, int n_items, int d, const int* mask_rowptr, const int* mask_col, int K, int agg, int* out_idx,
                        float* out_val, float* scratch, long long scratch_elems, cudaStream_t st) {
  LLMREC_CHECK_ARG(scratch && scratch_elems >= score_tc_group_scratch(rp, n_groups, n_items, d, K), "score_topk_group: scratch too small");
  std::vector<int> plan;
  const int n_tiles = group_tile_plan(rp, n_groups, &plan);
  ScoreParams P;
  memset(&P, 0, sizeof(P));
  score_plan(n_tiles * SBM, n_items, K, &P.splits, &P.tiles_per_split);
  P.Kc = score_kc(K);
  float* Ihi = scratch; float* Ilo = scratch + (long long)n_items * d;
  float* cval = Ilo + (long long)n_items * d;
  int* cidx = reinterpret_cast<int*>(cval + (long long)n_groups * P.splits * P.Kc);
  int* dplan = cidx + (long long)n_groups * P.splits * P.Kc;
  // pageable source: the copy is staged before this returns, so `plan` may go when it does
  LLMREC_CHECK_CUDA(cudaMemcpyAsync(dplan, plan.data(), plan.size() * sizeof(int), cudaMemcpyHostToDevice, st));
  P.grp_rowptr = dplan; P.gofs = dplan + n_groups + 1; P.tile_g0 = P.gofs + n_groups; P.slot_pos = P.tile_g0 + n_tiles + 1;
  P.agg = agg;
  P.U = U; P.ldu = ldu; P.users = members; P.n_batch = n_tiles * SBM; P.n_items = n_items; P.d = d; P.among = among;
  P.mask_rowptr = mask_rowptr; P.mask_col = mask_col; P.cand_idx = cidx; P.cand_val = cval;
  if (int rc = launch_select<true>(P, I, ldi, among, n_items, d, n_tiles, Ihi, Ilo, st)) return rc;
  const int n_cand = P.splits * P.Kc;
  LLMREC_CHECK_ARG(n_cand <= 32 * kMaxCandPerLane, "score_topk_group: %d candidates per group exceed the rescoring capacity", n_cand);
  rescore_topk_group_kernel<<<(n_groups + 7) / 8, 256, 0, st>>>(U, ldu, I, ldi, P.grp_rowptr, members, n_groups, d, agg, cidx, n_cand, K, out_idx,
                                                               out_val);
  LLMREC_CHECK_LAUNCH("rescore_topk_group");
  return 0;
}

}  // namespace llmrec
