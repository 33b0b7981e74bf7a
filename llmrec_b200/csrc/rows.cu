// Small row-wise helpers of the sharded (multi-GPU) path:
//   * Y = [softmax]( scale[r] * X[r,:] )  -- the epilogue of an item-side propagation AFTER the cross-rank sum of
//     the per-rank partials (the single-GPU path fuses this into the SpMM store)
//   * gather / scatter-add of embedding rows by index (batch rows exchanged between ranks)
#include "common.cuh"

namespace llmrec {
__global__ void __launch_bounds__(256) row_scale_softmax_kernel(const float* __restrict__ X, int64_t ldx, const float* __restrict__ scale,
                                                                float* __restrict__ Y, int64_t ldy, int64_t n, int d, int softmax) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (blockIdx.x * (int64_t)(blockDim.x >> 5)) + (threadIdx.x >> 5);
  if (row >= n) return;
  const float s = scale ? scale[row] : 1.0f;
  const float* x = X + row * ldx;
  float* y = Y + row * ldy;
  if (!softmax) {
    for (int j = lane; j < d; j += 32) y[j] = s * x[j];
    return;
  }
  float m = -INFINITY;
  for (int j = lane; j < d; j += 32) m = fmaxf(m, s * x[j]);
  m = warp_max(m);
  float t = 0.f;
  for (int j = lane; j < d; j += 32) t += expf(s * x[j] - m);
  t = warp_sum(t);
  const float inv = 1.0f / t;
  for (int j = lane; j < d; j += 32) y[j] = expf(s * x[j] - m) * inv;
}
// Y[r,:] = X[r,:] / max(||X[r,:]||_2, 1e-12)  (F.normalize; item-to-item cosine).  One warp per row; X == Y is fine: every lane
// rewrites only the elements it read.
__global__ void __launch_bounds__(256) row_normalize_kernel(const float* X, int64_t ldx, float* Y, int64_t ldy, int64_t n, int d) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (blockIdx.x * (int64_t)(blockDim.x >> 5)) + (threadIdx.x >> 5);
  if (row >= n) return;
  const float* x = X + row * ldx;
  float* y = Y + row * ldy;
  float ss = 0.f;
  for (int j = lane; j < d; j += 32) ss = fmaf(x[j], x[j], ss);
  ss = warp_sum(ss);
  const float inv = 1.0f / fmaxf(sqrtf(ss), 1e-12f);
  for (int j = lane; j < d; j += 32) y[j] = x[j] * inv;
}
// out[b,:] = idx[b] >= 0 ? X[idx[b],:] : 0
__global__ void __launch_bounds__(256) gather_rows_kernel(const float* __restrict__ X, int64_t ldx, const int* __restrict__ idx, int n, int d,
                                                          float* __restrict__ out, int64_t ldo) {
  const int lane = threadIdx.x & 31;
  const int b = (blockIdx.x * (blockDim.x >> 5)) + (threadIdx.x >> 5);
  if (b >= n) return;
  const int r = idx[b];
  if (((d | ldx | ldo) & 3) == 0 && ((reinterpret_cast<uintptr_t>(X) | reinterpret_cast<uintptr_t>(out)) & 15) == 0) {   // 128-bit rows (wide feature tables)
    const float4* src = reinterpret_cast<const float4*>(X + (int64_t)(r >= 0 ? r : 0) * ldx);
    float4* dst = reinterpret_cast<float4*>(out + (int64_t)b * ldo);
    for (int j = lane; j < (d >> 2); j += 32) dst[j] = r >= 0 ? __ldg(src + j) : make_float4(0.f, 0.f, 0.f, 0.f);
    return;
  }
  for (int j = lane; j < d; j += 32) out[(int64_t)b * ldo + j] = r >= 0 ? X[(int64_t)r * ldx + j] : 0.f;
}
// Y[idx[b],:] += G[b,:] for idx[b] >= 0 (duplicates allowed -> atomics)
__global__ void __launch_bounds__(256) scatter_add_rows_kernel(const float* __restrict__ G, int64_t ldg, const int* __restrict__ idx, int n, int d,
                                                               float* __restrict__ Y, int64_t ldy) {
  const int lane = threadIdx.x & 31;
  const int b = (blockIdx.x * (blockDim.x >> 5)) + (threadIdx.x >> 5);
  if (b >= n) return;
  const int r = idx[b];
  if (r < 0) return;
  for (int j = lane; j < d; j += 32) atomicAdd(Y + (int64_t)r * ldy + j, G[(int64_t)b * ldg + j]);
}
// ---- row sets of the demand-driven training step (dist.py): bitmask over rows, built and compacted on the device -----------------
// mask |= bit(v) for every v in the CSR rows named by list[0..n_list) -- one CTA per listed row (hub rows have 1e5 entries)
__global__ void __launch_bounds__(256) mark_neighbors_kernel(const int* __restrict__ rowptr, const int* __restrict__ col, const int* __restrict__ list,
                                                             unsigned* __restrict__ mask) {
  const int r = list[blockIdx.x];
  if (r < 0) return;
  const int e1 = rowptr[r + 1];
  for (int e = rowptr[r] + threadIdx.x; e < e1; e += blockDim.x) {
    const int v = col[e];
    const unsigned bit = 1u << (v & 31);
    if (!(mask[v >> 5] & bit)) atomicOr(mask + (v >> 5), bit);
  }
}
// ids[0 .. n) -- or ids[0 .. min(*n_dev, n)) when the live length is only known on the device (a captured step's B')
__global__ void mark_ids_kernel(const int* __restrict__ ids, int n, const int* __restrict__ n_dev, unsigned* __restrict__ mask) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (n_dev) { const int c = __ldg(n_dev); n = c < n ? c : n; }
  if (i >= n) return;
  const int v = ids[i];
  if (v >= 0) atomicOr(mask + (v >> 5), 1u << (v & 31));
}
// set bits -> list of row ids (order unspecified), *count += number of set bits; one word per thread, one atomic per warp
__global__ void __launch_bounds__(256) compact_mask_kernel(const unsigned* __restrict__ mask, int n_words, int n_bits, int* __restrict__ out, int* __restrict__ count) {
  const int wd = blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31;
  unsigned bits = wd < n_words ? mask[wd] : 0u;
  if (wd == n_words - 1 && (n_bits & 31)) bits &= (1u << (n_bits & 31)) - 1u;
  const int c = __popc(bits);
  int pre = c;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, pre, o); if (lane >= o) pre += t; }
  int base = 0;
  if (lane == 31 && pre > 0) base = atomicAdd(count, pre);
  base = __shfl_sync(0xffffffffu, base, 31);
  int pos = base + pre - c;
  while (bits) { const int b = __ffs(bits) - 1; bits &= bits - 1; out[pos++] = wd * 32 + b; }
}
__global__ void __launch_bounds__(256) zero_rows_kernel(float* __restrict__ Y, int64_t ldy, const int* __restrict__ idx, int n, int d) {
  const int lane = threadIdx.x & 31;
  const int b = (blockIdx.x * (blockDim.x >> 5)) + (threadIdx.x >> 5);
  if (b >= n) return;
  const int r = idx[b];
  if (r < 0) return;
  for (int j = lane; j < d; j += 32) Y[(int64_t)r * ldy + j] = 0.f;
}
// Y[idx[b],:] = G[b,:] for idx[b] >= 0 (duplicates must carry identical rows)
__global__ void __launch_bounds__(256) assign_rows_kernel(const float* __restrict__ G, int64_t ldg, const int* __restrict__ idx, int n, int d,
                                                          float* __restrict__ Y, int64_t ldy) {
  const int lane = threadIdx.x & 31;
  const int b = (blockIdx.x * (blockDim.x >> 5)) + (threadIdx.x >> 5);
  if (b >= n) return;
  const int r = idx[b];
  if (r < 0) return;
  for (int j = lane; j < d; j += 32) Y[(int64_t)r * ldy + j] = G[(int64_t)b * ldg + j];
}
}  // namespace llmrec
using namespace llmrec;

extern "C" int llmrec_mark_neighbors(const int32_t* rowptr, const int32_t* col, const int32_t* list, int32_t n_list, uint32_t* mask, llmrec_stream_t stream) {
  LLMREC_REQUIRE_DEVICE();
  if (n_list <= 0) return 0;
  mark_neighbors_kernel<<<n_list, 256, 0, as_stream(stream)>>>(rowptr, col, list, mask);
  LLMREC_CHECK_LAUNCH("mark_neighbors");
  return 0;
}
extern "C" int llmrec_mark_ids(const int32_t* ids, int32_t n, uint32_t* mask, llmrec_stream_t stream) {
  LLMREC_REQUIRE_DEVICE();
  if (n <= 0) return 0;
  mark_ids_kernel<<<(n + 255) / 256, 256, 0, as_stream(stream)>>>(ids, n, nullptr, mask);
  LLMREC_CHECK_LAUNCH("mark_ids");
  return 0;
}
extern "C" int llmrec_mark_ids_rows(const int32_t* ids, const int32_t* n_dev, int32_t max_n, uint32_t* mask, llmrec_stream_t stream) {
  LLMREC_REQUIRE_DEVICE();
  LLMREC_CHECK_ARG(n_dev, "mark_ids_rows: the device-side length is required");
  if (max_n <= 0) return 0;
  mark_ids_kernel<<<(max_n + 255) / 256, 256, 0, as_stream(stream)>>>(ids, max_n, n_dev, mask);
  LLMREC_CHECK_LAUNCH("mark_ids_rows");
  return 0;
}
extern "C" int llmrec_compact_mask(const uint32_t* mask, int32_t n_bits, int32_t* list_out, int32_t* count, llmrec_stream_t stream) {
  LLMREC_REQUIRE_DEVICE();
  if (n_bits <= 0) return 0;
  const int n_words = (n_bits + 31) / 32;
  compact_mask_kernel<<<(n_words + 255) / 256, 256, 0, as_stream(stream)>>>(mask, n_words, n_bits, list_out, count);
  LLMREC_CHECK_LAUNCH("compact_mask");
  return 0;
}
extern "C" int llmrec_zero_rows_f32(float* Y, int64_t ldy, const int32_t* idx, int32_t n, int32_t d, llmrec_stream_t stream) {
  LLMREC_REQUIRE_DEVICE();
  if (n <= 0) return 0;
  zero_rows_kernel<<<(n + 7) / 8, 256, 0, as_stream(stream)>>>(Y, ldy, idx, n, d);
  LLMREC_CHECK_LAUNCH("zero_rows");
  return 0;
}
extern "C" int llmrec_assign_rows_f32(const float* G, int64_t ldg, const int32_t* idx, int32_t n, int32_t d, float* Y, int64_t ldy, llmrec_stream_t stream) {
  LLMREC_REQUIRE_DEVICE();
  if (n <= 0) return 0;
  assign_rows_kernel<<<(n + 7) / 8, 256, 0, as_stream(stream)>>>(G, ldg, idx, n, d, Y, ldy);
  LLMREC_CHECK_LAUNCH("assign_rows");
  return 0;
}

extern "C" int llmrec_row_scale_softmax_f32(const float* X, int64_t ldx, const float* scale, float* Y, int64_t ldy, int64_t n, int32_t d,
                                            int32_t softmax, llmrec_stream_t stream) {
  LLMREC_REQUIRE_DEVICE();
  if (n <= 0) return 0;
  row_scale_softmax_kernel<<<(unsigned)((n + 7) / 8), 256, 0, as_stream(stream)>>>(X, ldx, scale, Y, ldy, n, d, softmax);
  LLMREC_CHECK_LAUNCH("row_scale_softmax");
  return 0;
}
extern "C" int llmrec_row_normalize_f32(const float* X, int64_t ldx, float* Y, int64_t ldy, int64_t n, int32_t d, llmrec_stream_t stream) {
  LLMREC_REQUIRE_DEVICE();
  if (n <= 0) return 0;
  LLMREC_CHECK_ARG(X && Y && d > 0 && ldx >= d && ldy >= d, "row_normalize: need X, Y, d > 0 and leading dimensions >= d");
  row_normalize_kernel<<<(unsigned)((n + 7) / 8), 256, 0, as_stream(stream)>>>(X, ldx, Y, ldy, n, d);
  LLMREC_CHECK_LAUNCH("row_normalize");
  return 0;
}
extern "C" int llmrec_gather_rows_f32(const float* X, int64_t ldx, const int32_t* idx, int32_t n, int32_t d, float* out, int64_t ldo,
                                      llmrec_stream_t stream) {
  LLMREC_REQUIRE_DEVICE();
  if (n <= 0) return 0;
  gather_rows_kernel<<<(n + 7) / 8, 256, 0, as_stream(stream)>>>(X, ldx, idx, n, d, out, ldo);
  LLMREC_CHECK_LAUNCH("gather_rows");
  return 0;
}
extern "C" int llmrec_scatter_add_rows_f32(const float* G, int64_t ldg, const int32_t* idx, int32_t n, int32_t d, float* Y, int64_t ldy,
                                           llmrec_stream_t stream) {
  LLMREC_REQUIRE_DEVICE();
  if (n <= 0) return 0;
  scatter_add_rows_kernel<<<(n + 7) / 8, 256, 0, as_stream(stream)>>>(G, ldg, idx, n, d, Y, ldy);
  LLMREC_CHECK_LAUNCH("scatter_add_rows");
  return 0;
}
