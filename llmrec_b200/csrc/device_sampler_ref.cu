// Device-side batch sampler on the reference's own random streams (`--device_sampler 2`): the GPU draws exactly the batches of
// llmrec_host_sample_batch (host_sampler.cu) -- the same users, positives, negatives, augmented triplets and B' -- from device copies of
// CPython's `random` MT19937 state and numpy's global legacy MT19937 state, and leaves both states where the host sampler would.
//
// One CTA of 1024 threads.  The draws themselves form one dependent chain (every rejection shifts every later draw), so warp 0 runs
// them: its 32 lanes test 32 consecutive tempered outputs against the current draw and a ballot picks the first accepted one; the twist
// runs warp-wide in three phases and tempers all 624 outputs at once.  The block does the parallel parts around the chain:
//   users    (warp 0, `random`)  random.sample(range(n_exist), batch) in CPython's pool or set branch (the set branch finds repeats in an
//            open-addressing table of the batch's draws), or `batch` draws of _randbelow(n_exist) when batch > n_exist
//   rows     (block)  positions -> user ids, the users' train-row bounds, and a Bloom filter (2^19 bits) over (batch slot, train item)
//   pos/neg  (warp 0, numpy)  masked legacy randint(deg) (a range of 1 consumes no word) and randint(n_items) redrawn while the
//            candidate is a train item of the user.  The positive indexes the train row in its stored order (as the host sampler
//            does); membership reads a copy of the rows sorted ascending.  The Bloom filter answers "not a member" from shared memory; only its positives
//            (true members and rare false positives) binary-search the sorted train row in global memory
//   aug      (warp 0, `random`)  random.sample(range(batch), n_aug) in the pool or set branch, then (warp 0) the picks whose ids are both
//            < aug_limit are appended in pick order
// Errors (no train item / no possible negative / a uid missing from the augmentation tables / a rejection loop past 2^24 draws) set
// state[ERR] to the host sampler's return code, leave both streams as they were before the call, and fill the batch with user 0 / item 0
// so the step that reads it stays in bounds.  A call that finds state[ERR] set does the same and draws nothing.  Every loop is bounded.
#include "common.cuh"

namespace llmrec {
namespace refsample {

constexpr int N = 624, M = 397;
constexpr int kThreads = 1024;
constexpr int kBloomWords = 1 << 14;          // 2^19 bits = 64 KB
constexpr int kFixedSmem = (4 * N + kBloomWords) * 4;
constexpr int kMaxSmem = 227 * 1024 - 1024;     // dynamic shared memory, with room for the kernel's static words
constexpr unsigned kMaxDraws = 1u << 24;      // words one draw may consume before the call gives up (rc 5)

enum { kPy = 0, kNp = N + 1, kErr = 2 * (N + 1), kStateElems = kErr + 2 };
static_assert(kStateElems == LLMREC_REF_SAMPLER_STATE_ELEMS, "state layout");

struct Params {
  const int* exist; int n_exist; int batch; int users_pool;
  const int* rowptr; const int* col; const int* col_sorted; int n_items;
  int n_aug; int aug_pool; const int* aug_pos; const int* aug_neg; int n_aug_table; int aug_limit;
  const int* meta_table; int cap;
  int* state; int* out; int* work; int work_in_smem; int hcap;
};

__device__ __forceinline__ unsigned temper(unsigned y) {
  y ^= (y >> 11);
  y ^= (y << 7) & 0x9d2c5680u;
  y ^= (y << 15) & 0xefc60000u;
  y ^= (y >> 18);
  return y;
}

// One stream as warp 0 consumes it: key = the MT19937 state, tmp = its 624 tempered outputs, pos the same in every lane.  All calls are
// warp-collective and return the same values in every lane.
struct WarpMt {
  unsigned* key; unsigned* tmp; int pos;
  // the twist in three phases: i < 227 reads only words of the old state, 227 <= i < 454 words the first phase wrote, the rest words of the
  // second phase (and the new key[0]); inside a phase each chunk of 32 words is read by all lanes before any lane writes
  __device__ void regen(int lane) {
    const int bounds[4] = {0, N - M, 2 * (N - M), N};
    for (int ph = 0; ph < 3; ++ph)
      for (int base = bounds[ph]; base < bounds[ph + 1]; base += 32) {
        const int i = base + lane;
        const bool in = i < bounds[ph + 1];
        unsigned v = 0;
        if (in) {
          const unsigned y = (key[i] & 0x80000000u) | (key[i + 1 < N ? i + 1 : 0] & 0x7fffffffu);
          v = key[i + M < N ? i + M : i + M - N] ^ (y >> 1) ^ ((0u - (y & 1u)) & 0x9908b0dfu);
        }
        __syncwarp();
        if (in) key[i] = v;
        __syncwarp();
      }
    for (int i = lane; i < N; i += 32) tmp[i] = temper(key[i]);
    __syncwarp();
    pos = 0;
  }
  // the first output w from pos on with ok(w), consuming every output up to and including it: the 32 lanes test 32 consecutive outputs
  // and a ballot picks the first accepted one.  false: none within kMaxDraws outputs
  template <typename Ok>
  __device__ bool first(int lane, Ok ok, unsigned& w_out) {
    for (unsigned seen = 0; seen < kMaxDraws;) {
      if (pos == N) regen(lane);
      const int i = pos + lane;
      const unsigned w = i < N ? tmp[i] : 0u;
      const unsigned hit = __ballot_sync(0xffffffffu, i < N && ok(w));
      if (hit) {
        const int f = __ffs(hit) - 1;
        w_out = __shfl_sync(0xffffffffu, w, f);
        pos += f + 1;
        return true;
      }
      const int avail = N - pos < 32 ? N - pos : 32;
      pos += avail;
      seen += avail;
    }
    return false;
  }
  // CPython's _randbelow(n): getrandbits(n.bit_length()) -- one output >> (32 - k) -- until < n
  __device__ bool randbelow(int lane, unsigned n, unsigned& r) {
    const int sh = __clz(n);
    unsigned w;
    if (!first(lane, [&](unsigned x) { return (x >> sh) < n; }, w)) return false;
    r = w >> sh;
    return true;
  }
  // numpy's legacy masked randint(0, high) for 0 < high: a range of 1 consumes no output
  __device__ bool randint(int lane, unsigned high, unsigned& v) {
    const unsigned rng = high - 1;
    v = 0;
    if (rng == 0) return true;
    unsigned mask = rng;
    mask |= mask >> 1; mask |= mask >> 2; mask |= mask >> 4; mask |= mask >> 8; mask |= mask >> 16;
    unsigned w;
    if (!first(lane, [&](unsigned x) { return (x & mask) <= rng; }, w)) return false;
    v = w & mask;
    return true;
  }
};

// insert-if-absent into an open-addressing table of non-negative ints (-1 = empty), capacity a power of two > 2x the entries
__device__ __forceinline__ bool set_insert(int* tab, int hcap, int key) {
  unsigned h = ((unsigned)key * 0x9E3779B1u) & (unsigned)(hcap - 1);
  for (int probe = 0; probe < hcap; ++probe) {
    const int v = tab[h];
    if (v == key) return false;
    if (v < 0) { tab[h] = key; return true; }
    h = (h + 1) & (unsigned)(hcap - 1);
  }
  return false;
}

__device__ __forceinline__ unsigned long long bloom_hash(int slot, int item) {
  unsigned long long x = ((unsigned long long)(unsigned)slot << 32) | (unsigned)item;
  x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 33;
  return x;
}
__device__ __forceinline__ void bloom_add(unsigned* bloom, int slot, int item) {
  const unsigned long long h = bloom_hash(slot, item);
#pragma unroll
  for (int q = 0; q < 3; ++q) { const unsigned bit = (unsigned)(h >> (19 * q)) & ((1u << 19) - 1u); atomicOr(&bloom[bit >> 5], 1u << (bit & 31u)); }
}
__device__ __forceinline__ bool bloom_maybe(const unsigned* bloom, int slot, int item) {
  const unsigned long long h = bloom_hash(slot, item);
  bool all = true;
#pragma unroll
  for (int q = 0; q < 3; ++q) { const unsigned bit = (unsigned)(h >> (19 * q)) & ((1u << 19) - 1u); all = all && ((bloom[bit >> 5] >> (bit & 31u)) & 1u); }
  return all;
}
__device__ __forceinline__ bool row_has(const int* col, int beg, int deg, int c) {   // train rows are sorted ascending
  int lo = beg, hi = beg + deg;
  while (lo < hi) {
    const int m = (lo + hi) >> 1;
    const int x = col[m];
    if (x == c) return true;
    if (x < c) lo = m + 1; else hi = m;
  }
  return false;
}

// a poisoned batch: user 0 / item 0 everywhere, B' = batch, so a step that runs on it reads nothing out of bounds
__device__ void write_safe_batch(const Params& p) {
  int* out = p.out;
  for (int b = threadIdx.x; b < p.batch; b += blockDim.x) { out[b] = 0; out[p.cap + b] = 0; out[2 * (size_t)p.cap + b] = 0; }
  if (threadIdx.x == 0) { out[3 * (size_t)p.cap] = p.meta_table[2 * p.batch]; out[3 * (size_t)p.cap + 1] = p.meta_table[2 * p.batch + 1]; }
}

__global__ void __launch_bounds__(kThreads) ref_sample_kernel(const Params p) {
  extern __shared__ unsigned smem[];
  unsigned* py_key = smem;
  unsigned* np_key = smem + N;
  unsigned* py_tmp = smem + 2 * N;
  unsigned* np_tmp = smem + 3 * N;
  unsigned* bloom = smem + 4 * N;
  int* work = p.work_in_smem ? reinterpret_cast<int*>(smem + 4 * N + kBloomWords) : p.work;
  const int B = p.batch;
  int* s_beg = work;                 // [batch] train-row start of each slot
  int* s_deg = work + B;             // [batch] its degree; reused for the augmentation picks
  int* table = work + 2 * B;         // [hcap] repeats of the set branches
  int* pool = table + p.hcap;        // pool copies of the pool branches
  __shared__ int s_err, s_B;
  const int tid = threadIdx.x;
  int* users = p.out; int* pos = p.out + p.cap; int* neg = p.out + 2 * (size_t)p.cap; int* meta = p.out + 3 * (size_t)p.cap;

  if (tid == 0) s_err = p.state[kErr];
  __syncthreads();
  if (s_err) { write_safe_batch(p); return; }
  for (int i = tid; i < N; i += blockDim.x) {
    py_key[i] = (unsigned)p.state[kPy + i]; np_key[i] = (unsigned)p.state[kNp + i];
    py_tmp[i] = temper(py_key[i]); np_tmp[i] = temper(np_key[i]);
  }
  for (int i = tid; i < kBloomWords; i += blockDim.x) bloom[i] = 0u;
  for (int i = tid; i < p.hcap; i += blockDim.x) table[i] = -1;
  if (B <= p.n_exist && p.users_pool)
    for (int i = tid; i < p.n_exist; i += blockDim.x) pool[i] = i;
  WarpMt py{py_key, py_tmp, p.state[kPy + N]}, np{np_key, np_tmp, p.state[kNp + N]};   // warp 0's copies are the ones that advance
  const int lane = tid & 31;
  __syncthreads();

  // ---- users: positions into exist_users, from the `random` stream ----
  // (warp 0; lane 0 alone touches memory, the other lanes test outputs)
  if (tid < 32) {
    int err = 0;
    unsigned j;
    const int n = p.n_exist;
    if (B <= n && p.users_pool) {
      for (int i = 0; i < B; ++i) {
        if (!py.randbelow(lane, (unsigned)(n - i), j)) { err = 5; break; }
        if (lane == 0) { users[i] = pool[j]; pool[j] = pool[n - i - 1]; }
      }
    } else if (B <= n) {
      for (int i = 0; i < B && !err; ++i) {
        for (unsigned t = 0;; ++t) {                             // redrawn while already drawn in this call
          if (t >= kMaxDraws || !py.randbelow(lane, (unsigned)n, j)) { err = 5; break; }
          int fresh = 0;
          if (lane == 0) fresh = set_insert(table, p.hcap, (int)j);
          if (__shfl_sync(0xffffffffu, fresh, 0)) break;
        }
        if (lane == 0) users[i] = (int)j;
      }
    } else {
      for (int i = 0; i < B; ++i) {
        if (!py.randbelow(lane, (unsigned)n, j)) { err = 5; break; }
        if (lane == 0) users[i] = (int)j;
      }
    }
    if (lane == 0) s_err = err;
  }
  __syncthreads();
  if (s_err) { write_safe_batch(p); if (tid == 0) p.state[kErr] = s_err; return; }
  for (int b = tid; b < B; b += blockDim.x) {
    const int u = p.exist[users[b]];
    users[b] = u;
    const int beg = p.rowptr[u];
    s_beg[b] = beg;
    s_deg[b] = p.rowptr[u + 1] - beg;
  }
  __syncthreads();
  {
    const int lane = tid & 31, wp = tid >> 5, nw = blockDim.x >> 5;
    for (int b = wp; b < B; b += nw) {
      const int beg = s_beg[b], deg = s_deg[b];
      for (int e = lane; e < deg; e += 32) bloom_add(bloom, b, p.col[beg + e]);
    }
  }
  __syncthreads();

  // ---- one positive and one rejection-sampled negative per slot, from numpy's stream ----
  if (tid < 32) {
    int err = 0;
    unsigned v;
    for (int b = 0; b < B; ++b) {
      const int beg = s_beg[b], deg = s_deg[b];
      if (deg <= 0) { err = 2; break; }
      if (!np.randint(lane, (unsigned)deg, v)) { err = 5; break; }
      if (lane == 0) pos[b] = (int)v;                            // an offset into the row; the block resolves it below
      if (deg >= p.n_items) { err = 3; break; }
      unsigned t = 0;
      for (; t < kMaxDraws; ++t) {                               // every lane evaluates the same membership test
        if (!np.randint(lane, (unsigned)p.n_items, v)) { t = kMaxDraws; break; }
        if (!bloom_maybe(bloom, b, (int)v) || !row_has(p.col_sorted, beg, deg, (int)v)) break;
      }
      if (t >= kMaxDraws) { err = 5; break; }
      if (lane == 0) neg[b] = (int)v;
    }
    if (lane == 0) s_err = err;
  }
  __syncthreads();
  if (s_err) { write_safe_batch(p); if (tid == 0) p.state[kErr] = s_err; return; }
  for (int b = tid; b < B; b += blockDim.x) pos[b] = p.col[s_beg[b] + pos[b]];
  const int n_aug = p.n_aug;
  if (n_aug > 0) {
    if (p.aug_pool) for (int i = tid; i < B; i += blockDim.x) pool[i] = i;
    else for (int i = tid; i < p.hcap; i += blockDim.x) table[i] = -1;
  }
  __syncthreads();

  // ---- augmented edges: random.sample over the batch list's positions, from the `random` stream ----
  int* pick = s_deg;
  if (tid < 32) {
    int err = 0;
    unsigned j;
    if (n_aug > 0 && p.aug_pool) {
      for (int i = 0; i < n_aug; ++i) {
        if (!py.randbelow(lane, (unsigned)(B - i), j)) { err = 5; break; }
        if (lane == 0) { pick[i] = pool[j]; pool[j] = pool[B - i - 1]; }
      }
    } else if (n_aug > 0) {
      for (int i = 0; i < n_aug && !err; ++i) {
        for (unsigned t = 0;; ++t) {
          if (t >= kMaxDraws || !py.randbelow(lane, (unsigned)B, j)) { err = 5; break; }
          int fresh = 0;
          if (lane == 0) fresh = set_insert(table, p.hcap, (int)j);
          if (__shfl_sync(0xffffffffu, fresh, 0)) break;
        }
        if (lane == 0) pick[i] = (int)j;
      }
    }
    if (lane == 0) { s_err = err; s_B = B; }
  }
  __syncthreads();
  if (s_err) { write_safe_batch(p); if (tid == 0) p.state[kErr] = s_err; return; }
  if (tid < 32) {                                                 // keep, in pick order: both ids < aug_limit
    int Bp = B, missing = 0;
    for (int base = 0; base < n_aug; base += 32) {
      const int i = base + tid;
      int u = 0, ap = 0, an = 0;
      bool keep = false, miss = false;
      if (i < n_aug) {
        u = users[pick[i]];
        miss = u < 0 || u >= p.n_aug_table;
        if (!miss) { ap = p.aug_pos[u]; an = p.aug_neg[u]; miss = ap == INT32_MIN || an == INT32_MIN; }
        keep = !miss && ap < p.aug_limit && an < p.aug_limit;
      }
      if (__ballot_sync(0xffffffffu, miss)) { missing = 1; break; }
      const unsigned kb = __ballot_sync(0xffffffffu, keep);
      if (keep) {
        const int at = Bp + __popc(kb & ((1u << tid) - 1u));
        users[at] = u; pos[at] = ap; neg[at] = an;
      }
      Bp += __popc(kb);
    }
    if (tid == 0) { s_err = missing ? 4 : 0; s_B = Bp; }
  }
  __syncthreads();
  if (s_err) { write_safe_batch(p); if (tid == 0) p.state[kErr] = s_err; return; }
  if (tid == 0) {
    meta[0] = p.meta_table[2 * s_B]; meta[1] = p.meta_table[2 * s_B + 1];
    p.state[kPy + N] = py.pos; p.state[kNp + N] = np.pos;
  }
  for (int i = tid; i < N; i += blockDim.x) { p.state[kPy + i] = (int)py_key[i]; p.state[kNp + i] = (int)np_key[i]; }
}

int table_cap(int batch) {
  int h = 1;
  while (h < 2 * batch + 2) h <<= 1;
  return h;
}
int64_t work_elems(int n_exist, int batch, int users_pool, int aug_pool) {
  const int64_t pool = (batch <= n_exist && users_pool) ? n_exist : 0;
  return 2 * (int64_t)batch + table_cap(batch) + (pool > batch ? pool : (aug_pool ? batch : pool));
}

}  // namespace refsample
}  // namespace llmrec

using namespace llmrec;

extern "C" int64_t llmrec_device_sample_batch_ref_work(int32_t n_exist, int32_t batch, int32_t users_pool_branch, int32_t aug_pool_branch) {
  if (n_exist < 1 || batch < 1) return 0;
  return refsample::work_elems(n_exist, batch, users_pool_branch, aug_pool_branch);
}

extern "C" int llmrec_device_sample_batch_ref(const int32_t* exist_users, int32_t n_exist, int32_t batch, int32_t users_pool_branch,
                                              const int32_t* train_rowptr, const int32_t* train_col, const int32_t* train_col_sorted,
                                              int32_t n_items, int32_t n_aug, int32_t aug_pool_branch, const int32_t* aug_pos, const int32_t* aug_neg,
                                              int32_t n_aug_table, int32_t aug_limit, const int32_t* meta_table, int32_t cap,
                                              int32_t* state, int32_t* out, int32_t* work, int64_t work_elems, llmrec_stream_t stream) {
  using namespace refsample;
  LLMREC_REQUIRE_DEVICE();
  LLMREC_CHECK_ARG(n_exist >= 1 && batch >= 1 && n_items >= 1 && n_aug >= 0 && n_aug <= batch && cap >= batch + n_aug && meta_table && state &&
                   out && work && exist_users && train_rowptr && train_col && train_col_sorted,
                   "device_sample_batch_ref: bad sizes (n_exist=%d batch=%d n_items=%d cap=%d n_aug=%d)", n_exist, batch, n_items, cap, n_aug);
  LLMREC_CHECK_ARG(n_aug == 0 || (aug_pos && aug_neg && n_aug_table >= 0), "device_sample_batch_ref: n_aug=%d without augmentation tables", n_aug);
  const int64_t need = refsample::work_elems(n_exist, batch, users_pool_branch, aug_pool_branch);
  LLMREC_CHECK_ARG(work_elems >= need, "device_sample_batch_ref: work holds %lld ints, %lld needed", (long long)work_elems, (long long)need);
  const int64_t smem_all = kFixedSmem + 4 * need;
  const int in_smem = smem_all <= kMaxSmem;
  const int smem = in_smem ? (int)smem_all : kFixedSmem;
  LLMREC_CHECK_CUDA(cudaFuncSetAttribute(ref_sample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  Params p{exist_users, n_exist, batch, users_pool_branch ? 1 : 0, train_rowptr, train_col, train_col_sorted, n_items, n_aug, aug_pool_branch ? 1 : 0,
           aug_pos, aug_neg, n_aug_table, aug_limit, meta_table, cap, state, out, work, in_smem, table_cap(batch)};
  ref_sample_kernel<<<1, kThreads, smem, as_stream(stream)>>>(p);
  LLMREC_CHECK_LAUNCH("device_sample_batch_ref");
  return 0;
}
