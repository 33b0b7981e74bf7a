// Packed 64-bit ranking keys and the warp's running top-K in shared memory, shared by the re-ranking (rerank.cu) and the
// explanation (explain.cu) selections.
//   key = (~order(score) << 32) | id,   order() = the order-preserving map of the fp32 bits (-0 -> +0, every NaN above +inf),
// so ascending keys are (score desc, id asc), NaN after every number, and a repeated id becomes two adjacent equal keys.
#pragma once
#include "common.cuh"

namespace llmrec {

constexpr uint64_t kNoKey = ~0ull;   // padding: after every real candidate (a real key's id half is < 2^31)

static __device__ __forceinline__ uint64_t rank_key(float s, int id) {
  uint32_t hi;
  if (s != s) {
    hi = 0xffffffffu;                                  // NaN: after every number
  } else {
    uint32_t b = __float_as_uint(s);
    if (b == 0x80000000u) b = 0u;                      // -0 == +0: ties go to the id
    const uint32_t f = (b & 0x80000000u) ? ~b : (b | 0x80000000u);
    hi = ~f;
  }
  return ((uint64_t)hi << 32) | (uint32_t)id;
}
static __device__ __forceinline__ float key_score(uint64_t key) {
  const uint32_t f = ~(uint32_t)(key >> 32);
  return __uint_as_float((f & 0x80000000u) ? (f & 0x7fffffffu) : ~f);   // NaN keys come back as a NaN
}

// kept list buf[0, *nb) (sorted, unique, <= K) + staged run buf[*nb, *nb + ns) -> the first K unique keys of both, sorted, in buf[0, *nb)
static __device__ void flush_run(uint64_t* buf, int* nb, int ns, int K, int lane) {
  const int n = *nb + ns;
  if (ns == 0) return;
  int W = 32;
  while (W < n) W <<= 1;
  for (int i = n + lane; i < W; i += 32) buf[i] = kNoKey;
  __syncwarp();
  for (int k = 2; k <= W; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int t = lane; t < (W >> 1); t += 32) {
        const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));
        const int l = i | j;
        const uint64_t a = buf[i], b = buf[l];
        if ((a > b) == ((i & k) == 0)) { buf[i] = b; buf[l] = a; }
      }
      __syncwarp();
    }
  }
  // drop repeats and keep the first K (in place: a key moves only down, and a slice is read before it is written)
  int out = 0;
  uint64_t carry = kNoKey;
  for (int base = 0; base < n && out < K; base += 32) {
    const int i = base + lane;
    const uint64_t key = i < n ? buf[i] : kNoKey;
    uint64_t prev = __shfl_up_sync(0xffffffffu, key, 1);
    if (lane == 0) prev = carry;
    carry = __shfl_sync(0xffffffffu, key, 31);
    const bool keep = i < n && key != prev;
    const unsigned bal = __ballot_sync(0xffffffffu, keep);
    const int pos = out + __popc(bal & ((1u << lane) - 1u));
    __syncwarp();
    if (keep && pos < K) buf[pos] = key;
    out += __popc(bal);
    __syncwarp();
  }
  *nb = min(out, K);
}

}  // namespace llmrec
