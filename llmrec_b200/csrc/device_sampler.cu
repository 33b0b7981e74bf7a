// Device-side batch sampler (SURVEY.md 8f-1): the work of Data.sample() (utility/load_data.py:157-195) and of the augmented-edge step
// (main.py:216-224) as ONE kernel that writes straight into the engine's static index buffer -- users / pos / neg rows and the
// {B', n_keep} meta row the captured training step reads -- so a graph replay needs no host sampler and no H2D copy at all.
// NON-PARITY by construction: the reference draws from CPython's and numpy's MT19937 streams on the host (replayed bit for bit by
// host_sampler.cu, the default); here a counter-based generator (splitmix64 over {seed, step, lane}) gives the same DISTRIBUTIONS:
//   users   a uniformly random batch_size-subset of exist_users (the batch_size smallest of n_exist random keys, radix-selected),
//           or batch_size independent draws when batch_size > n_exist (load_data.py:158-161)
//   pos     uniform over the user's train items; neg: uniform over items, rejected while it is a train item of the user (:166-187);
//           after 2^16 rejected candidates the r-th non-member, r uniform in [0, n_items - deg), so neg is never a train item
//   aug     n_aug = min(int(batch * rate), batch) distinct batch positions (the n_aug smallest of batch random keys, ties to the lower
//           position); (u, aug_pos[u], aug_neg[u]) appended in position order when both ids are in [0, aug_limit).  A uid outside
//           [0, n_aug_table) or with an INT32_MIN entry (missing from augmented_sample_dict) is DROPPED, where upstream raises KeyError
// Precondition (checked on the host by DeviceSampler): every exist user has 1 <= deg < n_items and every train row is sorted ascending.
// One CTA of 1024 threads (a batch is ~1e3 triplets); deterministic for a given {seed, step}; the step counter lives on the device.
#include "common.cuh"

namespace llmrec {

__device__ __forceinline__ unsigned long long splitmix64(unsigned long long x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}
struct Rng {
  unsigned long long base; unsigned long long ctr;
  __device__ unsigned next() { return (unsigned)(splitmix64(base + 0xD1342543DE82EF95ull * (++ctr)) >> 32); }
  __device__ int below(int n) { return (int)(((unsigned long long)next() * (unsigned long long)n) >> 32); }   // uniform in [0, n)
};

struct SampleParams {
  const int* exist; int n_exist; int batch;
  const int* rowptr; const int* col; int n_items;
  int n_aug; const int* aug_pos; const int* aug_neg; int n_aug_table; int aug_limit;
  const int* meta_table; int cap;
  unsigned long long* state;   // {seed, step}
  int* out;                    // [4 x cap]
  unsigned* keys;              // [max(n_exist, batch)] scratch
};

// threshold of the `want`-th smallest (0-based) of n 32-bit keys read through key_of(i); ties resolved by index by the caller
template <typename KeyFn>
__device__ void radix_select(KeyFn key_of, int n, int want, unsigned& T, int& r, int* hist, unsigned* s_prefix, int* s_want) {
  const int tid = threadIdx.x;
  if (tid == 0) { *s_prefix = 0u; *s_want = want; }
  __syncthreads();
  for (int pass = 0; pass < 4; ++pass) {
    const int shift = 24 - 8 * pass;
    if (tid < 256) hist[tid] = 0;
    __syncthreads();
    const unsigned prefix = *s_prefix;
    const unsigned mask = pass == 0 ? 0u : (0xffffffffu << (shift + 8));
    for (int i = tid; i < n; i += blockDim.x) {
      const unsigned k = key_of(i);
      if ((k & mask) == prefix) atomicAdd(&hist[(k >> shift) & 255u], 1);
    }
    __syncthreads();
    if (tid < 32) {  // warp 0 walks the 256 counts 8 per lane: exclusive prefix by shuffles, the owning lane publishes bin and remainder
      int c[8], sum = 0;
#pragma unroll
      for (int q = 0; q < 8; ++q) { c[q] = hist[tid * 8 + q]; sum += c[q]; }
      int inc = sum;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, inc, o); if (tid >= o) inc += t; }
      int before = inc - sum;
      const int w = *s_want;
      __syncwarp();
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        if (c[q] > 0 && before <= w && w < before + c[q]) { *s_want = w - before; *s_prefix = prefix | ((unsigned)(tid * 8 + q) << shift); }
        before += c[q];
      }
    }
    __syncthreads();
  }
  T = *s_prefix;
  r = *s_want + 1;          // how many keys == T (in index order) belong to the selection
  __syncthreads();
}

// ordered compaction: out_pos[i] = rank among selected (selected = key < T, or key == T and among the first r ties); returns total
template <typename KeyFn, typename EmitFn>
__device__ int ordered_emit(KeyFn key_of, int n, unsigned T, int r, EmitFn emit, int* redi) {
  const int tid = threadIdx.x, lane = tid & 31, wp = tid >> 5, nw = blockDim.x >> 5;
  int ties_before = 0, sel_before = 0;
  for (int base = 0; base < n; base += blockDim.x) {
    const int i = base + tid;
    const unsigned k = i < n ? key_of(i) : 0xffffffffu;
    const bool less = i < n && k < T, tie = i < n && k == T;
    const unsigned bt = __ballot_sync(0xffffffffu, tie);
    __syncthreads();
    if (lane == 0) redi[wp] = __popc(bt);
    __syncthreads();
    int tb = ties_before + __popc(bt & ((1u << lane) - 1u)), ttot = 0;
    for (int q = 0; q < nw; ++q) { const int c = redi[q]; if (q < wp) tb += c; ttot += c; }
    const bool sel = less || (tie && tb < r);
    const unsigned bs = __ballot_sync(0xffffffffu, sel);
    __syncthreads();
    if (lane == 0) redi[wp] = __popc(bs);
    __syncthreads();
    int sb = sel_before + __popc(bs & ((1u << lane) - 1u)), stot = 0;
    for (int q = 0; q < nw; ++q) { const int c = redi[q]; if (q < wp) sb += c; stot += c; }
    if (sel) emit(i, sb);
    ties_before += ttot; sel_before += stot;
  }
  __syncthreads();
  return sel_before;
}

__global__ void __launch_bounds__(1024) device_sample_kernel(const SampleParams p) {
  __shared__ int hist[256];
  __shared__ int redi[32];
  __shared__ unsigned s_prefix;
  __shared__ int s_want;
  const int tid = threadIdx.x;
  const unsigned long long seed = p.state[0], step = p.state[1];
  const unsigned long long base = splitmix64(seed ^ splitmix64(step));
  int* users = p.out; int* pos = p.out + p.cap; int* neg = p.out + 2 * (size_t)p.cap; int* meta = p.out + 3 * (size_t)p.cap;
  const int B = p.batch;
  // ---- users ----
  if (B <= p.n_exist) {
    for (int i = tid; i < p.n_exist; i += blockDim.x) p.keys[i] = (unsigned)(splitmix64(base ^ (0xA5A5A5A5ull + (unsigned long long)i * 0x9E3779B97F4A7C15ull)) >> 32);
    __syncthreads();
    auto key_of = [&](int i) { return p.keys[i]; };
    unsigned T; int r;
    radix_select(key_of, p.n_exist, B - 1, T, r, hist, &s_prefix, &s_want);
    ordered_emit(key_of, p.n_exist, T, r, [&](int i, int slot) { users[slot] = p.exist[i]; }, redi);
  } else {
    for (int b = tid; b < B; b += blockDim.x) { Rng g{base ^ 0x1111ull, (unsigned long long)b * 4}; users[b] = p.exist[g.below(p.n_exist)]; }
  }
  __syncthreads();
  // ---- one positive, one rejection-sampled negative per user ----
  for (int b = tid; b < B; b += blockDim.x) {
    Rng g{base ^ 0x2222ull, (unsigned long long)b << 20};
    const int u = users[b];
    const int e0 = p.rowptr[u], deg = p.rowptr[u + 1] - e0;
    pos[b] = deg > 0 ? p.col[e0 + g.below(deg)] : 0;
    int c = 0; bool found = false;
    for (int tries = 0; tries < (1 << 16) && !found; ++tries) {
      c = g.below(p.n_items);
      int lo = e0, hi = e0 + deg; bool hit = false;                   // train rows are sorted ascending
      while (lo < hi) { const int m = (lo + hi) >> 1; const int x = p.col[m]; if (x == c) { hit = true; break; } if (x < c) lo = m + 1; else hi = m; }
      found = !hit;
    }
    if (!found && deg < p.n_items) {
      // 2^16 candidates were all train items (a user holding nearly every item): draw the r-th non-member directly, still uniform
      // over the n_items - deg non-members.  Walk the sorted row: every distinct member at or below the running candidate pushes it up.
      c = g.below(p.n_items - deg);
      for (int j = e0; j < e0 + deg; ++j) {
        const int x = p.col[j];
        if (x > c) break;
        if (j == e0 || x != p.col[j - 1]) ++c;
      }
    }
    neg[b] = c;
  }
  __syncthreads();
  // ---- augmented edges: n_aug distinct batch positions, kept when both ids are valid; appended in position order ----
  int kept = 0;
  if (p.n_aug > 0 && p.aug_pos) {
    auto key2 = [&](int i) { return (unsigned)(splitmix64(base ^ (0x3333ull + (unsigned long long)i * 0xD6E8FEB86659FD93ull)) >> 32); };
    unsigned T; int r;
    const int n_aug = p.n_aug < B ? p.n_aug : B;
    radix_select(key2, B, n_aug - 1, T, r, hist, &s_prefix, &s_want);
    // pass 1: the selection as radix_select defines it (key2 < T, or == T and among the first r ties in position order) writes
    // keys[i] = 0 for a selected position whose table entries are valid, 0xffffffff otherwise; the users are already emitted, so the key
    // scratch (>= batch entries) is free
    for (int i = tid; i < B; i += blockDim.x) p.keys[i] = 0xffffffffu;
    __syncthreads();
    ordered_emit(key2, B, T, r, [&](int i, int) {
      const int u = users[i];
      const bool in = u >= 0 && u < p.n_aug_table;
      const int ap = in ? p.aug_pos[u] : -1, an = in ? p.aug_neg[u] : -1;
      if (ap >= 0 && an >= 0 && ap < p.aug_limit && an < p.aug_limit) p.keys[i] = 0u;
    }, redi);
    // pass 2: the flagged positions appended in position order
    kept = ordered_emit([&](int i) { return p.keys[i]; }, B, 1u, 0, [&](int i, int slot) {
      if (B + slot < p.cap) { const int u = users[i]; users[B + slot] = u; pos[B + slot] = p.aug_pos[u]; neg[B + slot] = p.aug_neg[u]; }
    }, redi);
    if (B + kept > p.cap) kept = p.cap - B;
  }
  if (tid == 0) {
    const int Bp = B + kept;
    meta[0] = p.meta_table[2 * Bp]; meta[1] = p.meta_table[2 * Bp + 1];
    p.state[1] = step + 1;
  }
}
}  // namespace llmrec

using namespace llmrec;

extern "C" int llmrec_device_sample_batch(const int32_t* exist_users, int32_t n_exist, int32_t batch,
                                          const int32_t* train_rowptr, const int32_t* train_col, int32_t n_items,
                                          int32_t n_aug, const int32_t* aug_pos, const int32_t* aug_neg, int32_t n_aug_table, int32_t aug_limit,
                                          const int32_t* meta_table, int32_t cap, uint64_t* state, int32_t* out, uint32_t* key_scratch,
                                          llmrec_stream_t stream) {
  LLMREC_REQUIRE_DEVICE();
  LLMREC_CHECK_ARG(n_exist >= 1 && batch >= 1 && n_items >= 1 && cap >= batch + (n_aug > 0 ? n_aug : 0) && meta_table && state && out && key_scratch,
                   "device_sample_batch: bad sizes (n_exist=%d batch=%d cap=%d n_aug=%d)", n_exist, batch, cap, n_aug);
  SampleParams p{exist_users, n_exist, batch, train_rowptr, train_col, n_items, n_aug, aug_pos, aug_neg, n_aug_table, aug_limit, meta_table, cap,
                 reinterpret_cast<unsigned long long*>(state), out, key_scratch};
  device_sample_kernel<<<1, 1024, 0, as_stream(stream)>>>(p);
  LLMREC_CHECK_LAUNCH("device_sample_batch");
  return 0;
}
