// Shared device/host helpers for the llmrec_b200 kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include "../../include/llmrec_b200.h"

namespace llmrec {

void set_error(const char* fmt, ...);
bool device_ok();

#define LLMREC_CHECK_ARG(cond, ...)            \
  do {                                         \
    if (!(cond)) {                             \
      llmrec::set_error(__VA_ARGS__);          \
      return 1;                                \
    }                                          \
  } while (0)

#define LLMREC_CHECK_LAUNCH(name)                                              \
  do {                                                                         \
    cudaError_t e__ = cudaGetLastError();                                      \
    if (e__ != cudaSuccess) {                                                  \
      llmrec::set_error("%s: launch failed: %s", name, cudaGetErrorString(e__)); \
      return 2;                                                                \
    }                                                                          \
  } while (0)

#define LLMREC_CHECK_CUDA(expr)                                                \
  do {                                                                         \
    cudaError_t e__ = (expr);                                                  \
    if (e__ != cudaSuccess) {                                                  \
      llmrec::set_error("%s: %s", #expr, cudaGetErrorString(e__));             \
      return 2;                                                                \
    }                                                                          \
  } while (0)

#define LLMREC_REQUIRE_DEVICE()                                                       \
  do {                                                                                \
    if (!llmrec::device_ok()) {                                                       \
      llmrec::set_error("no sm_90 CUDA device: llmrec_b200 has no CPU / other-arch fallback"); \
      return 3;                                                                       \
    }                                                                                 \
  } while (0)

constexpr int kWarp = 32;
constexpr int kNumSMs = 132;   // H100 SXM: grid sizing of the grid-stride and persistent kernels

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
template <int G>
__device__ __forceinline__ float group_sum(float v) {
#pragma unroll
  for (int o = G / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
template <int G>
__device__ __forceinline__ float group_max(float v) {
#pragma unroll
  for (int o = G / 2; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
// streaming (read-once) 128-bit load: do not allocate in L1
__device__ __forceinline__ float4 ldg4_stream(const float* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ void fma4(float4& a, float w, const float4& x) {
  a.x = fmaf(w, x.x, a.x); a.y = fmaf(w, x.y, a.y); a.z = fmaf(w, x.z, a.z); a.w = fmaf(w, x.w, a.w);
}

// Group scores (llmrec_score_topk_group_f32): v = agg_start; v = agg_fold(v, s_m) for the members in ascending id; agg_end(v, n).
// mean: the fp32 sum 0 + s_0 + s_1 + ..., then one IEEE division by n; min / max: the exact extreme, a NaN member makes it NaN
// (fminf / fmaxf would drop the NaN).  __fadd_rn / __fdiv_rn keep nvcc from contracting or approximating them.
__device__ __forceinline__ float agg_start(int agg) { return agg == LLMREC_AGG_MEAN ? 0.f : agg == LLMREC_AGG_MIN ? INFINITY : -INFINITY; }
__device__ __forceinline__ float agg_fold(int agg, float v, float s) {
  if (agg == LLMREC_AGG_MEAN) return __fadd_rn(v, s);
  if (s != s) return s;
  return (agg == LLMREC_AGG_MIN ? s < v : s > v) ? s : v;   // once v is NaN no comparison is true: it stays NaN
}
__device__ __forceinline__ float agg_end(int agg, float v, int n) { return agg == LLMREC_AGG_MEAN ? __fdiv_rn(v, (float)n) : v; }

inline cudaStream_t as_stream(llmrec_stream_t s) { return reinterpret_cast<cudaStream_t>(s); }
inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

}  // namespace llmrec
