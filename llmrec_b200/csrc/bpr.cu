// BPR + prune heads (main.py:330-342 bpr_loss, :158-165 prune_loss, :232-254) and
// feat_reg (main.py:151-156): forward values AND row gradients, no host round trip.
//
// The reference does, per head: 3 row gathers, mul+sum, logsigmoid, a D2H copy + CPU argsort + H2D
// (x8 per step), mean of the kept 29 %.  Here the whole loss tail of a step is THREE launches:
//   grad_init   every gradient buffer of the step is written once (zeros, or c*X for the feat_reg blocks, whose
//               0.5*c*|X|^2 is summed on the way and becomes the initial value of the loss) -- no memsets;
//   bpr_forward one warp scores a (head, triplet); the LAST CTA of a head (atomic ticket) then selects the
//               n_keep smallest log-sigmoids of that head with a 4-pass radix select over order-preserving keys
//               (O(B), ties -> lower batch position like the reference's stable argsort), sums them in a fixed
//               order, and emits the per-triplet gradient coefficients; the last head adds the weighted losses;
//   bpr_grad    scatter-add of the row gradients (float atomics), or bpr_grad_ordered: the same sums gathered in a fixed order from a
//               slot plan (slot_rank), bit-reproducible.
// The live batch length B' and n_keep may come from a 2-int DEVICE block (`meta`), so one captured CUDA graph
// serves every batch length up to the capacity the grid was sized for.
#include "common.cuh"

namespace llmrec {

constexpr int kMaxHeads = 16;
constexpr int kSelThreads = 256;

struct BprParams {
  llmrec_bpr_head head[kMaxHeads];
  int n_heads; const int* users; const int* pos; const int* neg; int cap; const int* meta; int B_host; int n_keep_host; float c_emb; int d;
  float* out; float* loss; float* work; unsigned* counters;
};
// work layout: 32 words of tickets (per-head + head counter; fixed position for every capacity), then per head h
// (stride 7*cap + 8): x[cap], maxi[cap], su[cap], sp[cap], sn[cap], gcoef[cap], keep[cap], eu, ep, en
constexpr int kWorkHdr = 32;
__device__ __forceinline__ float* work_of(const BprParams& p, int h) { return p.work + kWorkHdr + (size_t)h * (7 * (size_t)p.cap + 8); }
__device__ __forceinline__ int live_B(const BprParams& p) { int b = p.meta ? __ldg(p.meta) : p.B_host; return b < p.cap ? b : p.cap; }
__device__ __forceinline__ int live_keep(const BprParams& p) { return p.meta ? __ldg(p.meta + 1) : p.n_keep_host; }

__device__ __forceinline__ float logsigmoidf(float z) {  // min(z,0) - log1p(exp(-|z|))
  return fminf(z, 0.f) - log1pf(expf(-fabsf(z)));
}
// order-preserving float -> uint32 key (ascending)
__device__ __forceinline__ unsigned okey(float v) {
  unsigned k = __float_as_uint(v);
  return (k & 0x80000000u) ? ~k : (k | 0x80000000u);
}

__device__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  float t = 0.f;
  if (threadIdx.x == 0) for (int i = 0; i < nw; ++i) t += red[i];
  if (threadIdx.x == 0) red[0] = t;
  __syncthreads();
  return red[0];
}
__device__ int block_sum_int(int v, int* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  int t = 0;
  if (threadIdx.x == 0) for (int i = 0; i < nw; ++i) t += red[i];
  if (threadIdx.x == 0) red[0] = t;
  __syncthreads();
  return red[0];
}

// selection + head outputs for head h; runs in ONE CTA of kSelThreads threads after every score of the head is visible
__device__ void bpr_select_head(const BprParams& p, int h, int B, int n_keep) {
  __shared__ int hist[256];
  __shared__ float redf[32];
  __shared__ int redi[32];
  __shared__ unsigned s_prefix;
  __shared__ int s_want;
  float* w = work_of(p, h);
  const float* maxi = w + p.cap;
  const int tid = threadIdx.x;
  n_keep = n_keep < 0 ? 0 : (n_keep > B ? B : n_keep);
  // ---- radix select: key T of rank n_keep-1 and r = how many keys == T are kept -------------------------------
  unsigned T = 0xffffffffu;
  int r = 0;
  if (n_keep > 0 && n_keep < B) {
    if (tid == 0) { s_prefix = 0u; s_want = n_keep - 1; }
    __syncthreads();
    for (int pass = 0; pass < 4; ++pass) {
      const int shift = 24 - 8 * pass;
      hist[tid] = 0;                                        // kSelThreads == 256 bins
      __syncthreads();
      const unsigned prefix = s_prefix;
      const unsigned mask = pass == 0 ? 0u : (0xffffffffu << (shift + 8));
      for (int i = tid; i < B; i += kSelThreads) {
        const unsigned k = okey(__ldcg(maxi + i));
        if ((k & mask) == prefix) atomicAdd(&hist[(k >> shift) & 255u], 1);
      }
      __syncthreads();
      {  // which bin holds rank `want`: exclusive scan of the 256 counts (one per thread), the owning thread publishes bin and remainder
        const int cnt = hist[tid], lane = tid & 31, wp = tid >> 5;
        int inc = cnt;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
        if (lane == 31) redi[wp] = inc;
        __syncthreads();
        int before = inc - cnt;
        for (int q = 0; q < wp; ++q) before += redi[q];
        const int want = s_want;
        __syncthreads();
        if (cnt > 0 && before <= want && want < before + cnt) { s_want = want - before; s_prefix = prefix | ((unsigned)tid << shift); }
      }
      __syncthreads();
    }
    T = s_prefix;
    r = s_want + 1;                                         // the first r ties (by position) are kept
    __syncthreads();
  } else if (n_keep >= B) {
    T = 0xffffffffu; r = B;                                 // everything kept (keys < T or tie rule below admits all)
  }
  // ---- ordered tie pass + gradient coefficients + kept sum (fixed order: deterministic) ------------------------
  float kept_sum = 0.f, su = 0.f, sp = 0.f, sn = 0.f;
  int ties_before = 0;                                      // uniform across the block
  const float inv_keep = n_keep > 0 ? 1.f / (float)n_keep : 0.f;
  const float wmf = p.head[h].w_mf;
  for (int base = 0; base < B; base += kSelThreads) {
    const int i = base + tid;
    unsigned k = 0u; float mv = 0.f;
    bool tie = false, less = false;
    if (i < B) {
      mv = __ldcg(maxi + i);
      k = okey(mv);
      less = n_keep > 0 && (k < T);
      tie = n_keep > 0 && (k == T);
    }
    // exclusive prefix of `tie` within the block, in thread order
    const unsigned bal = __ballot_sync(0xffffffffu, tie);
    const int lane = tid & 31, wp = tid >> 5;
    __syncthreads();
    if (lane == 0) redi[wp] = __popc(bal);
    __syncthreads();
    int before = ties_before + __popc(bal & ((1u << lane) - 1u));
    int tot = 0;
    for (int q = 0; q < kSelThreads / 32; ++q) { const int c = redi[q]; if (q < wp) before += c; tot += c; }
    const bool keep = less || (tie && before < r);
    ties_before += tot;
    if (i < B) {
      // d(-mean(maxi[keep]))/dx = -(1/n_keep) * sigmoid(-x); torch's log_sigmoid_backward form
      const float x = __ldcg(w + i);
      const float z = expf(-fabsf(x));
      const float dls = (x < 0.f) ? (1.f - z / (1.f + z)) : (z / (1.f + z));
      w[5 * (size_t)p.cap + i] = keep ? (-wmf * dls * inv_keep) : 0.f;
      w[6 * (size_t)p.cap + i] = keep ? 1.f : 0.f;
      if (keep) kept_sum += mv;
      su += __ldcg(w + 2 * (size_t)p.cap + i); sp += __ldcg(w + 3 * (size_t)p.cap + i); sn += __ldcg(w + 4 * (size_t)p.cap + i);
    }
  }
  kept_sum = block_sum(kept_sum, redf);
  su = block_sum(su, redf); sp = block_sum(sp, redf); sn = block_sum(sn, redf);
  if (tid == 0) {
    const float mf = n_keep > 0 ? -(kept_sum / (float)n_keep) : 0.f / 0.f;  // mean of empty = nan like torch
    const float du = 2.f * su + 1e-8f, dq = 2.f * sp + 1e-8f, dn = 2.f * sn + 1e-8f;
    const float emb = p.c_emb * (1.f / du + 1.f / dq + 1.f / dn);
    p.out[h * 4 + 0] = mf; p.out[h * 4 + 1] = emb; p.out[h * 4 + 2] = (float)n_keep; p.out[h * 4 + 3] = 0.f;
    // d emb / d row = w_emb * c * (-4 row / (2S+eps)^2)
    const float we = p.head[h].w_emb * p.c_emb;
    w[7 * (size_t)p.cap + 0] = -4.f * we / (du * du);
    w[7 * (size_t)p.cap + 1] = -4.f * we / (dq * dq);
    w[7 * (size_t)p.cap + 2] = -4.f * we / (dn * dn);
  }
}

__global__ void __launch_bounds__(kSelThreads) bpr_forward_kernel(const BprParams p) {
  __shared__ bool s_last, s_last_head;
  const int h = blockIdx.y, lane = threadIdx.x & 31;
  const int B = live_B(p);
  const int b = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (b < B) {
    const llmrec_bpr_head hd = p.head[h];
    const float* u = hd.XU + (int64_t)p.users[b] * hd.ldxu;
    const float* pi = hd.XI + (int64_t)p.pos[b] * hd.ldxi;
    const float* ni = hd.XI + (int64_t)p.neg[b] * hd.ldxi;
    float dp = 0.f, dn = 0.f, su = 0.f, sp = 0.f, sn = 0.f;
    for (int j = lane; j < p.d; j += 32) {
      float a = u[j], q = pi[j], r = ni[j];
      dp = fmaf(a, q, dp); dn = fmaf(a, r, dn);
      su = fmaf(a, a, su); sp = fmaf(q, q, sp); sn = fmaf(r, r, sn);
    }
    dp = warp_sum(dp); dn = warp_sum(dn); su = warp_sum(su); sp = warp_sum(sp); sn = warp_sum(sn);
    if (lane == 0) {
      float* w = work_of(p, h);
      float x = dp - dn + 1e-8f;
      w[b] = x;
      w[p.cap + b] = logsigmoidf(x);
      w[2 * (size_t)p.cap + b] = su; w[3 * (size_t)p.cap + b] = sp; w[4 * (size_t)p.cap + b] = sn;
    }
  }
  // ---- ticket: the last CTA of this head runs the selection -------------------------------------------------
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = atomicAdd(p.counters + h, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  bpr_select_head(p, h, B, live_keep(p));
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    p.counters[h] = 0u;
    s_last_head = atomicAdd(p.counters + kMaxHeads, 1u) == (unsigned)p.n_heads - 1;
  }
  __syncthreads();
  if (s_last_head && threadIdx.x == 0) {  // fixed-order head sum -> deterministic loss
    __threadfence();
    float tot = 0.f;
    for (int k = 0; k < p.n_heads; ++k) {
      volatile float* o = p.out + k * 4;
      tot += p.head[k].w_mf * o[0] + p.head[k].w_emb * o[1];
    }
    if (p.loss) *p.loss += tot;
    p.counters[kMaxHeads] = 0u;
  }
}

__global__ void __launch_bounds__(256) bpr_grad_kernel(const BprParams p) {
  const int h = blockIdx.y, lane = threadIdx.x & 31;
  const int b = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (b >= live_B(p)) return;
  const llmrec_bpr_head hd = p.head[h];
  if (!hd.GU && !hd.GI) return;
  const float* w = work_of(p, h);
  const float g = w[5 * (size_t)p.cap + b];
  const float eu = w[7 * (size_t)p.cap + 0], ep = w[7 * (size_t)p.cap + 1], en = w[7 * (size_t)p.cap + 2];
  if (g == 0.f && hd.w_emb == 0.f) return;
  const int iu = p.users[b], ip = p.pos[b], in_ = p.neg[b];
  const float* u = hd.XU + (int64_t)iu * hd.ldxu;
  const float* pi = hd.XI + (int64_t)ip * hd.ldxi;
  const float* ni = hd.XI + (int64_t)in_ * hd.ldxi;
  for (int j = lane; j < p.d; j += 32) {
    float a = u[j], q = pi[j], r = ni[j];
    if (hd.GU) atomicAdd(hd.GU + (int64_t)iu * hd.ldgu + j, g * (q - r) + eu * a);
    if (hd.GI) {
      atomicAdd(hd.GI + (int64_t)ip * hd.ldgi + j, g * a + ep * q);
      atomicAdd(hd.GI + (int64_t)in_ * hd.ldgi + j, -g * a + en * r);
    }
  }
}

// ---- ordered row gradients (deterministic form of bpr_grad) --------------------------------------------------------
// G[row, j] starts from what grad_init left and takes its contributions one fp32 add at a time: heads in ascending index,
// within a head ascending batch position, at one position pos before neg.  Gather, not scatter: the slot plan lists the
// batch's slots sorted by (row, slot) -- user slots b, item slots 2b (pos) and 2b + 1 (neg) -- so the slots of one row are a
// run in slot order.  The warp at the first entry of a run owns that row of one destination buffer: it folds every head that
// writes the buffer, in head order, in registers and stores each element once; the warps at the other entries retire.
//
// Plan layout (int32, 6 * cap): slot_u[cap] row_u[cap] slot_i[2 cap] row_i[2 cap]; only the live prefixes are written / read.
// slot_rank_kernel: one warp per slot counts the slots that sort before it -- its rank; keys (row, slot) are unique, so the
// ranks are a permutation whatever the schedule.  O(n^2 / 32) per warp-step: 2 252 item slots at the netflix batch are 71
// iterations per warp; at the capacity limit (131 072 slots) it is milliseconds, which is why the limit is where it is.
constexpr int kOrderedMaxSlots = 1 << 17;

__device__ __forceinline__ bool sorts_before(int rt, int t, int r, int s) { return rt < r || (rt == r && t < s); }

// a (and b: slots 2i -> a[i], 2i + 1 -> b[i]); n_host entries per array, or min(*n_dev, n_host)
__global__ void __launch_bounds__(256) slot_rank_kernel(const int* __restrict__ a, const int* __restrict__ b, int n_host, const int* __restrict__ n_dev,
                                                        int* __restrict__ slot_out, int* __restrict__ row_out) {
  const int lane = threadIdx.x & 31;
  int n = n_host;
  if (n_dev) { const int c = __ldg(n_dev); n = c < n ? c : n; }
  const int s = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (s >= (b ? 2 * n : n)) return;
  const int r = b ? ((s & 1) ? b[s >> 1] : a[s >> 1]) : a[s];
  int rank = 0;
  if (b) {
    for (int i = lane; i < n; i += 32) rank += (int)sorts_before(a[i], 2 * i, r, s) + (int)sorts_before(b[i], 2 * i + 1, r, s);
  } else {
    for (int i = lane; i < n; i += 32) rank += (int)sorts_before(a[i], i, r, s);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) rank += __shfl_xor_sync(0xffffffffu, rank, o);
  if (lane == 0) { slot_out[rank] = s; row_out[rank] = r; }
}

// the float atomic of bpr_grad / scatter_add_rows is an add that flushes denormals; so is every add of the ordered forms
__device__ __forceinline__ float add_ftz(float a, float b) {
  float r;
  asm("add.rn.ftz.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}

// length of the run of `row` in rowv[q0 .. n) as seen by this warp's 32 lanes (<= 32; 32 = the run may go on)
__device__ __forceinline__ int run_ahead(const int* __restrict__ rowv, int q0, int n, int row) {
  const int q = q0 + (threadIdx.x & 31);
  const unsigned m = __ballot_sync(0xffffffffu, q < n && rowv[q] == row);
  return m == 0xffffffffu ? 32 : __ffs(~m) - 1;
}

constexpr int kMaxOrdGroups = 2 * kMaxHeads;
struct OrdGroup { float* G; int64_t ldg; unsigned heads; };      // one destination buffer and the heads (bit h) that accumulate into it
struct OrdParams { OrdGroup grp[kMaxOrdGroups]; int n_user_groups; const int* plan; };

__global__ void __launch_bounds__(256) bpr_grad_ordered_kernel(const BprParams p, const OrdParams o) {
  const int lane = threadIdx.x & 31;
  const bool item = (int)blockIdx.y >= o.n_user_groups;
  const int B = live_B(p);
  const int n = item ? 2 * B : B;
  const int q_first = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (q_first >= n) return;
  const int* slotv = o.plan + (item ? 2 * (size_t)p.cap : 0);
  const int* rowv = slotv + (item ? 2 * (size_t)p.cap : (size_t)p.cap);
  const int row = rowv[q_first];
  if (q_first > 0 && rowv[q_first - 1] == row) return;      // not the first slot of its row
  const OrdGroup gr = o.grp[blockIdx.y];
  float* dst = gr.G + (int64_t)row * gr.ldg;
  for (int jb = 0; jb < p.d; jb += 128) {                   // 4 columns per lane and pass; every lane walks (the walk shuffles)
    const int j0 = jb + lane;
    float acc[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[c] = j0 + 32 * c < p.d ? dst[j0 + 32 * c] : 0.f;
    for (unsigned hm = gr.heads; hm; hm &= hm - 1) {
      const int h = __ffs(hm) - 1;
      const float* XU = p.head[h].XU; const float* XI = p.head[h].XI;
      const int64_t ldxu = p.head[h].ldxu, ldxi = p.head[h].ldxi;
      const bool no_emb = p.head[h].w_emb == 0.f;
      const float* w = work_of(p, h);
      const float* gco = w + 5 * (size_t)p.cap;
      const float eu = w[7 * (size_t)p.cap + 0], ep = w[7 * (size_t)p.cap + 1], en = w[7 * (size_t)p.cap + 2];
      for (int q0 = q_first; q0 < n; q0 += 32) {
        const int cnt = run_ahead(rowv, q0, n, row);
        // lane k fetches what slot k of the run needs; the walk below broadcasts it
        int s_l = 0, iu_l = 0, io_l = 0; float g_l = 0.f;
        if (lane < cnt) {
          s_l = slotv[q0 + lane];
          const int b = item ? s_l >> 1 : s_l;
          g_l = gco[b]; iu_l = p.users[b];
          io_l = item ? ((s_l & 1) ? p.neg[b] : p.pos[b]) : p.pos[b];
          if (!item) s_l = p.neg[b];
        }
        for (int k = 0; k < cnt; ++k) {
          const float g = __shfl_sync(0xffffffffu, g_l, k);
          const int s = __shfl_sync(0xffffffffu, s_l, k), iu = __shfl_sync(0xffffffffu, iu_l, k), io = __shfl_sync(0xffffffffu, io_l, k);
          if (g == 0.f && no_emb) continue;                 // bpr_grad's early-out: this triplet adds nothing, not even a zero
          const float* u = XU + (int64_t)iu * ldxu;
          const float* x = XI + (int64_t)io * ldxi;         // user rows: the positive item; item rows: this slot's item
          // the three contributions below are the instructions nvcc emits for bpr_grad's g*(q-r)+eu*a, g*a+ep*q, -g*a+en*r,
          // spelled out so that the two kernels cannot contract them differently
          if (!item) {
            const float* y = XI + (int64_t)s * ldxi;        // s carries neg[b] on the user side
#pragma unroll
            for (int c = 0; c < 4; ++c) {
              const int j = j0 + 32 * c;
              if (j < p.d) acc[c] = add_ftz(acc[c], __fmaf_rn(eu, u[j], __fmul_rn(g, x[j] - y[j])));
            }
          } else if (!(s & 1)) {
#pragma unroll
            for (int c = 0; c < 4; ++c) {
              const int j = j0 + 32 * c;
              if (j < p.d) acc[c] = add_ftz(acc[c], __fmaf_rn(ep, x[j], __fmul_rn(g, u[j])));
            }
          } else {
#pragma unroll
            for (int c = 0; c < 4; ++c) {
              const int j = j0 + 32 * c;
              if (j < p.d) acc[c] = add_ftz(acc[c], __fmaf_rn(en, x[j], -__fmul_rn(g, u[j])));
            }
          }
        }
        if (cnt < 32) break;
      }
    }
#pragma unroll
    for (int c = 0; c < 4; ++c) if (j0 + 32 * c < p.d) dst[j0 + 32 * c] = acc[c];
  }
}

// The same machinery for a plain row scatter: Y[idx[b], :] += G[b, :] in ascending b (idx[b] < 0 skipped; they sort first).
// plan (int32, 2 * n): slot[n] row[n] from slot_rank_kernel over idx.
__global__ void __launch_bounds__(256) scatter_add_rows_ordered_kernel(const float* __restrict__ G, int64_t ldg, const int* __restrict__ plan, int n, int d,
                                                                       float* __restrict__ Y, int64_t ldy) {
  const int lane = threadIdx.x & 31;
  const int q_first = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (q_first >= n) return;
  const int* slotv = plan;
  const int* rowv = plan + n;
  const int row = rowv[q_first];
  if (row < 0 || (q_first > 0 && rowv[q_first - 1] == row)) return;
  float* dst = Y + (int64_t)row * ldy;
  for (int jb = 0; jb < d; jb += 128) {
    const int j0 = jb + lane;
    float acc[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[c] = j0 + 32 * c < d ? dst[j0 + 32 * c] : 0.f;
    for (int q0 = q_first; q0 < n; q0 += 32) {
      const int cnt = run_ahead(rowv, q0, n, row);
      const int s_l = lane < cnt ? slotv[q0 + lane] : 0;
      for (int k = 0; k < cnt; ++k) {
        const float* g = G + (int64_t)__shfl_sync(0xffffffffu, s_l, k) * ldg;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const int j = j0 + 32 * c;
          if (j < d) acc[c] = add_ftz(acc[c], g[j]);
        }
      }
      if (cnt < 32) break;
    }
#pragma unroll
    for (int c = 0; c < 4; ++c) if (j0 + 32 * c < d) dst[j0 + 32 * c] = acc[c];
  }
}

// feat_reg: loss += c * 0.5 * sum(X^2);  G = (acc ? G : 0) + c * X
__global__ void __launch_bounds__(256) sqnorm_grad_kernel(const float* X, int64_t ldx, float* G, int64_t ldg, int64_t n, int d,
                                                          float c, int accumulate, float* partial) {
  __shared__ float red[32];
  const int64_t total = n * d;
  float s = 0.f;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t r = i / d; int j = (int)(i - r * d);
    float v = X[r * ldx + j];
    s = fmaf(v, v, s);
    if (G) { float* gp = G + r * ldg + j; *gp = accumulate ? (*gp + c * v) : c * v; }
  }
  s = block_sum(s, red);
  if (threadIdx.x == 0) partial[blockIdx.x] = s;
}
__global__ void sqnorm_final_kernel(const float* partial, int nb, float c, float* loss) {
  __shared__ float red[32];
  float s = 0.f;
  for (int i = threadIdx.x; i < nb; i += blockDim.x) s += partial[i];
  s = block_sum(s, red);
  if (threadIdx.x == 0 && loss) *loss += c * 0.5f * s;
}

// ---- grad_init: first touch of every gradient buffer of the step ---------------------------------------------------
constexpr int kMaxRegions = 16;
constexpr int kInitBlocks = kNumSMs;          // blocks per region (x n_regions in y)
struct GradInitParams {
  llmrec_grad_region reg[kMaxRegions];
  unsigned char vec[kMaxRegions];      // 1: rows are float4-addressable (width / ld % 4 == 0, 16-byte aligned bases)
  int n; float* loss; float* partial; unsigned* counter;
};
__global__ void __launch_bounds__(256) grad_init_kernel(const GradInitParams p) {
  __shared__ float red[32];
  __shared__ bool s_last;
  const llmrec_grad_region rg = p.reg[blockIdx.y];
  float s = 0.f;
  if (p.vec[blockIdx.y]) {
    const int w4 = rg.width >> 2;
    const int64_t total = rg.n * (int64_t)w4;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
      const int64_t r = i / w4; const int q = (int)(i - r * w4);
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (rg.X) {
        const float4 x = *reinterpret_cast<const float4*>(rg.X + r * rg.ldx + 4 * q);
        s += x.x * x.x + x.y * x.y + x.z * x.z + x.w * x.w;
        v = make_float4(rg.c * x.x, rg.c * x.y, rg.c * x.z, rg.c * x.w);
      }
      st4(rg.G + r * rg.ldg + 4 * q, v);
    }
  } else {                                                  // any width / alignment
    const int64_t total = rg.n * (int64_t)rg.width;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
      const int64_t r = i / rg.width; const int q = (int)(i - r * rg.width);
      float v = 0.f;
      if (rg.X) { const float x = rg.X[r * rg.ldx + q]; s = fmaf(x, x, s); v = rg.c * x; }
      rg.G[r * rg.ldg + q] = v;
    }
  }
  s = block_sum(s, red);
  if (threadIdx.x == 0) {
    p.partial[blockIdx.y * gridDim.x + blockIdx.x] = 0.5f * rg.c * s;
    __threadfence();
    s_last = atomicAdd(p.counter, 1u) == gridDim.x * gridDim.y - 1;
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  float t = 0.f;                                           // fixed order: deterministic
  const int np = gridDim.x * gridDim.y;
  for (int i = threadIdx.x; i < np; i += blockDim.x) t += __ldcg(p.partial + i);
  t = block_sum(t, red);
  if (threadIdx.x == 0) { if (p.loss) *p.loss = t; *p.counter = 0u; }
}
}  // namespace llmrec

using namespace llmrec;

extern "C" int64_t llmrec_bpr_work_elems(int32_t n_heads, int32_t B) { return kWorkHdr + (int64_t)n_heads * (7 * (int64_t)B + 8); }

static int bpr_params(BprParams& p, const llmrec_bpr_head* heads, int32_t n_heads, const int32_t* users, const int32_t* pos, const int32_t* neg,
                      int32_t B, int32_t n_keep, const int32_t* meta, float regs0_over_bs, int32_t d, float* out, float* loss_accum, float* work) {
  LLMREC_CHECK_ARG(n_heads >= 1 && n_heads <= kMaxHeads, "bpr: n_heads=%d out of range", n_heads);
  LLMREC_CHECK_ARG(B >= 1 && B <= (1 << 24), "bpr: batch capacity %d unsupported", B);
  for (int h = 0; h < n_heads; ++h) p.head[h] = heads[h];
  p.n_heads = n_heads; p.users = users; p.pos = pos; p.neg = neg; p.cap = B; p.meta = meta; p.B_host = B; p.n_keep_host = n_keep;
  p.c_emb = regs0_over_bs; p.d = d;
  p.out = out; p.loss = loss_accum; p.work = work;
  // the head of `work` holds the per-head tickets + the head counter (zeroed by the caller once; the kernel re-zeroes them)
  static_assert(kMaxHeads + 1 <= kWorkHdr, "ticket block");
  p.counters = reinterpret_cast<unsigned*>(work);
  return 0;
}

extern "C" int llmrec_bpr_heads_f32(const llmrec_bpr_head* heads, int32_t n_heads,
                                    const int32_t* users, const int32_t* pos, const int32_t* neg, int32_t B,
                                    int32_t n_keep, const int32_t* meta, float regs0_over_bs, int32_t d,
                                    float* out, float* loss_accum, float* work, llmrec_stream_t stream) {
  LLMREC_REQUIRE_DEVICE();
  BprParams p{};
  if (int rc = bpr_params(p, heads, n_heads, users, pos, neg, B, n_keep, meta, regs0_over_bs, d, out, loss_accum, work)) return rc;
  cudaStream_t st = as_stream(stream);
  dim3 grid((B + 7) / 8, n_heads);
  bpr_forward_kernel<<<grid, kSelThreads, 0, st>>>(p);
  LLMREC_CHECK_LAUNCH("bpr_forward");
  bpr_grad_kernel<<<grid, 256, 0, st>>>(p);
  LLMREC_CHECK_LAUNCH("bpr_grad");
  return 0;
}

extern "C" int64_t llmrec_bpr_slot_plan_elems(int32_t B) { return 6 * (int64_t)B; }

extern "C" int llmrec_bpr_slot_plan(const int32_t* users, const int32_t* pos, const int32_t* neg, int32_t B, const int32_t* meta,
                                    int32_t* plan, llmrec_stream_t stream) {
  LLMREC_REQUIRE_DEVICE();
  LLMREC_CHECK_ARG(B >= 1 && 2 * (int64_t)B <= kOrderedMaxSlots, "bpr_slot_plan: batch capacity %d unsupported (the ordered form takes up to %d triplets)",
                   B, kOrderedMaxSlots / 2);
  LLMREC_CHECK_ARG(plan, "bpr_slot_plan: plan is NULL");
  cudaStream_t st = as_stream(stream);
  slot_rank_kernel<<<(B + 7) / 8, 256, 0, st>>>(users, nullptr, B, meta, plan, plan + B);
  LLMREC_CHECK_LAUNCH("slot_rank(users)");
  slot_rank_kernel<<<(2 * B + 7) / 8, 256, 0, st>>>(pos, neg, B, meta, plan + 2 * (size_t)B, plan + 4 * (size_t)B);
  LLMREC_CHECK_LAUNCH("slot_rank(items)");
  return 0;
}

extern "C" int llmrec_bpr_heads_ordered_f32(const llmrec_bpr_head* heads, int32_t n_heads,
                                            const int32_t* users, const int32_t* pos, const int32_t* neg, int32_t B,
                                            int32_t n_keep, const int32_t* meta, float regs0_over_bs, int32_t d,
                                            float* out, float* loss_accum, float* work, const int32_t* plan, llmrec_stream_t stream) {
  LLMREC_REQUIRE_DEVICE();
  BprParams p{};
  if (int rc = bpr_params(p, heads, n_heads, users, pos, neg, B, n_keep, meta, regs0_over_bs, d, out, loss_accum, work)) return rc;
  LLMREC_CHECK_ARG(2 * (int64_t)B <= kOrderedMaxSlots, "bpr_heads_ordered: batch capacity %d unsupported (the ordered form takes up to %d triplets)",
                   B, kOrderedMaxSlots / 2);
  LLMREC_CHECK_ARG(plan, "bpr_heads_ordered: plan is NULL (build it with llmrec_bpr_slot_plan)");
  // destination buffers: heads that name the same GU (or GI) are folded by one warp in head order; user-side buffers first
  OrdParams o{};
  o.plan = plan;
  int ng = 0;
  for (int side = 0; side < 2; ++side) {
    for (int h = 0; h < n_heads; ++h) {
      if (!heads[h].GU && !heads[h].GI) continue;           // bpr_grad skips such a head altogether
      float* G = side ? heads[h].GI : heads[h].GU;
      const int64_t ld = side ? heads[h].ldgi : heads[h].ldgu;
      if (!G) continue;
      int g = side ? o.n_user_groups : 0;
      while (g < ng && o.grp[g].G != G) ++g;
      if (g == ng) { o.grp[ng].G = G; o.grp[ng].ldg = ld; o.grp[ng].heads = 0u; ++ng; }
      LLMREC_CHECK_ARG(o.grp[g].ldg == ld, "bpr_heads_ordered: heads that share a gradient buffer must share its leading dimension (head %d)", h);
      o.grp[g].heads |= 1u << h;
    }
    if (!side) o.n_user_groups = ng;
  }
  cudaStream_t st = as_stream(stream);
  bpr_forward_kernel<<<dim3((B + 7) / 8, n_heads), kSelThreads, 0, st>>>(p);
  LLMREC_CHECK_LAUNCH("bpr_forward");
  if (ng) {
    bpr_grad_ordered_kernel<<<dim3((2 * B + 7) / 8, ng), 256, 0, st>>>(p, o);
    LLMREC_CHECK_LAUNCH("bpr_grad_ordered");
  }
  return 0;
}

extern "C" int64_t llmrec_scatter_add_rows_ordered_scratch(int32_t n) { return 2 * (int64_t)(n > 0 ? n : 0); }

extern "C" int llmrec_scatter_add_rows_ordered_f32(const float* G, int64_t ldg, const int32_t* idx, int32_t n, int32_t d, float* Y, int64_t ldy,
                                                   int32_t* scratch, int64_t scratch_elems, llmrec_stream_t stream) {
  LLMREC_REQUIRE_DEVICE();
  if (n <= 0) return 0;
  LLMREC_CHECK_ARG(n <= kOrderedMaxSlots, "scatter_add_rows_ordered: %d rows unsupported (the ordered form takes up to %d)", n, kOrderedMaxSlots);
  LLMREC_CHECK_ARG(scratch && scratch_elems >= 2 * (int64_t)n, "scatter_add_rows_ordered: scratch too small (%lld < %lld int32)", (long long)scratch_elems,
                   2 * (long long)n);
  cudaStream_t st = as_stream(stream);
  slot_rank_kernel<<<(n + 7) / 8, 256, 0, st>>>(idx, nullptr, n, nullptr, scratch, scratch + n);
  LLMREC_CHECK_LAUNCH("slot_rank(idx)");
  scatter_add_rows_ordered_kernel<<<(n + 7) / 8, 256, 0, st>>>(G, ldg, scratch, n, d, Y, ldy);
  LLMREC_CHECK_LAUNCH("scatter_add_rows_ordered");
  return 0;
}

extern "C" int llmrec_grad_init_f32(const llmrec_grad_region* regions, int32_t n_regions, float* loss, float* scratch, llmrec_stream_t stream) {
  LLMREC_REQUIRE_DEVICE();
  LLMREC_CHECK_ARG(n_regions >= 1 && n_regions <= kMaxRegions, "grad_init: n_regions=%d out of range", n_regions);
  GradInitParams p{};
  for (int i = 0; i < n_regions; ++i) {
    p.reg[i] = regions[i];
    const llmrec_grad_region& r = regions[i];
    LLMREC_CHECK_ARG(r.G != nullptr && r.n >= 0 && r.width >= 0, "grad_init: region %d is malformed", i);
    p.vec[i] = (r.width % 4 == 0 && r.ldg % 4 == 0 && aligned16(r.G) && (!r.X || (r.ldx % 4 == 0 && aligned16(r.X)))) ? 1 : 0;
  }
  p.n = n_regions; p.loss = loss; p.partial = scratch; p.counter = reinterpret_cast<unsigned*>(scratch + kMaxRegions * kInitBlocks);
  grad_init_kernel<<<dim3(kInitBlocks, n_regions), 256, 0, as_stream(stream)>>>(p);
  LLMREC_CHECK_LAUNCH("grad_init");
  return 0;
}
extern "C" int64_t llmrec_grad_init_scratch(void) { return kMaxRegions * kInitBlocks + 4; }

extern "C" int llmrec_sqnorm_grad_f32(const float* X, int64_t ldx, float* G, int64_t ldg, int64_t n, int32_t d,
                                      float c, int32_t accumulate, float* loss_accum, float* partial /* >= 1024 floats */,
                                      llmrec_stream_t stream) {
  LLMREC_REQUIRE_DEVICE();
  if (n <= 0) return 0;
  cudaStream_t st = as_stream(stream);
  int64_t total = n * d;
  int nb = (int)((total + 256 * 8 - 1) / (256 * 8));
  if (nb > 1024) nb = 1024;
  if (nb < 1) nb = 1;
  sqnorm_grad_kernel<<<nb, 256, 0, st>>>(X, ldx, G, ldg, n, d, c, accumulate, partial);
  LLMREC_CHECK_LAUNCH("sqnorm_grad");
  sqnorm_final_kernel<<<1, 256, 0, st>>>(partial, nb, c, loss_accum);
  LLMREC_CHECK_LAUNCH("sqnorm_final");
  return 0;
}
