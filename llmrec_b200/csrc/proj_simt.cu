// Exact-fp32 SIMT version of the side-feature projection and its weight gradient
// (nn.Linear at Models.py:145-150).  mode 2 of llmrec_proj_*: the bit-conservative path used as the
// on-device checker for the wgmma kernels (proj_tc.cu) and for shapes those do not cover.
// Templated on the element type of X: fp32, or bf16 (raw uint16_t bits) widened to fp32 on load -- the same FMA order, so a bf16
// table gives the bits of the fp32 kernel on its upcast copy.
#include "common.cuh"

namespace llmrec {

__device__ __forceinline__ float x_f32(float x) { return x; }
__device__ __forceinline__ float x_f32(uint16_t x) { return __uint_as_float((uint32_t)x << 16); }

// Y[n x d] = X[n x k] W^T[k x d] + b ; 64x64 tile, K step 16, 4x4 per thread
template <class T>
__global__ void __launch_bounds__(256) proj_fwd_simt_kernel(const T* __restrict__ X, int64_t ldx, const float* __restrict__ W,
                                                            const float* __restrict__ bias, float* __restrict__ Y, int64_t ldy,
                                                            int64_t n, int k, int d) {
  __shared__ float Xs[16][64 + 4];
  __shared__ float Ws[16][64 + 4];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int64_t row0 = (int64_t)blockIdx.x * 64;
  const int col0 = blockIdx.y * 64;
  float acc[4][4] = {};
  for (int k0 = 0; k0 < k; k0 += 16) {
    for (int i = threadIdx.x; i < 64 * 16; i += 256) {
      int r = i >> 4, kk = i & 15;
      int64_t gr = row0 + r;
      Xs[kk][r] = (gr < n && k0 + kk < k) ? x_f32(X[gr * ldx + k0 + kk]) : 0.f;
      int gc = col0 + r;
      Ws[kk][r] = (gc < d && k0 + kk < k) ? W[(int64_t)gc * k + k0 + kk] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { a[i] = Xs[kk][ty * 4 + i]; b[i] = Ws[kk][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    int64_t gr = row0 + ty * 4 + i;
    if (gr >= n) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int gc = col0 + tx * 4 + j;
      if (gc < d) Y[gr * ldy + gc] = acc[i][j] + (bias ? bias[gc] : 0.f);
    }
  }
}

// dW[d x k] += sum_r dY[r,:]^T X[r,:] over a row chunk ; db[d] += colsum(dY) (k-tile 0 only)
template <class T>
__global__ void __launch_bounds__(256) proj_wgrad_simt_kernel(const T* __restrict__ X, int64_t ldx, const float* __restrict__ dY, int64_t lddy,
                                                              float* __restrict__ dW, float* __restrict__ db, int64_t n, int k, int d, int rows_per_chunk) {
  __shared__ float Gs[16][64 + 4];  // dY tile  [r][dcol]
  __shared__ float Xs[16][64 + 4];  // X tile   [r][kcol]
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int d0 = blockIdx.y * 64, k0 = blockIdx.x * 64;
  const int64_t r_beg = (int64_t)blockIdx.z * rows_per_chunk;
  const int64_t r_end = min(n, r_beg + rows_per_chunk);
  float acc[4][4] = {};
  float bsum[4] = {};
  for (int64_t r0 = r_beg; r0 < r_end; r0 += 16) {
    for (int i = threadIdx.x; i < 16 * 64; i += 256) {
      int r = i >> 6, c = i & 63;
      int64_t gr = r0 + r;
      Gs[r][c] = (gr < r_end && d0 + c < d) ? dY[gr * lddy + d0 + c] : 0.f;
      Xs[r][c] = (gr < r_end && k0 + c < k) ? x_f32(X[gr * ldx + k0 + c]) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < 16; ++r) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { a[i] = Gs[r][ty * 4 + i]; b[i] = Xs[r][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if (tx == 0) bsum[i] += a[i];
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    int gd = d0 + ty * 4 + i;
    if (gd >= d) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int gk = k0 + tx * 4 + j;
      if (gk < k) atomicAdd(dW + (int64_t)gd * k + gk, acc[i][j]);
    }
    if (db && blockIdx.x == 0 && tx == 0) atomicAdd(db + gd, bsum[i]);
  }
}

template <class T>
static int fwd_simt(const T* X, int64_t ldx, const float* W, const float* bias, float* Y, int64_t ldy, int64_t n, int k, int d, cudaStream_t st) {
  dim3 grid((unsigned)((n + 63) / 64), (d + 63) / 64);
  proj_fwd_simt_kernel<T><<<grid, 256, 0, st>>>(X, ldx, W, bias, Y, ldy, n, k, d);
  LLMREC_CHECK_LAUNCH("proj_fwd_simt");
  return 0;
}
template <class T>
static int wgrad_simt(const T* X, int64_t ldx, const float* dY, int64_t lddy, float* dW, float* db, int64_t n, int k, int d, int accumulate, cudaStream_t st) {
  if (!accumulate) {
    cudaMemsetAsync(dW, 0, sizeof(float) * (size_t)d * k, st);
    if (db) cudaMemsetAsync(db, 0, sizeof(float) * d, st);
  }
  const int rows_per_chunk = 1024;
  dim3 grid((k + 63) / 64, (d + 63) / 64, (unsigned)((n + rows_per_chunk - 1) / rows_per_chunk));
  proj_wgrad_simt_kernel<T><<<grid, 256, 0, st>>>(X, ldx, dY, lddy, dW, db, n, k, d, rows_per_chunk);
  LLMREC_CHECK_LAUNCH("proj_wgrad_simt");
  return 0;
}
int proj_fwd_simt(const float* X, int64_t ldx, const float* W, const float* bias, float* Y, int64_t ldy, int64_t n, int k, int d, cudaStream_t st) {
  return fwd_simt(X, ldx, W, bias, Y, ldy, n, k, d, st);
}
int proj_fwd_simt(const uint16_t* X, int64_t ldx, const float* W, const float* bias, float* Y, int64_t ldy, int64_t n, int k, int d, cudaStream_t st) {
  return fwd_simt(X, ldx, W, bias, Y, ldy, n, k, d, st);
}
int proj_wgrad_simt(const float* X, int64_t ldx, const float* dY, int64_t lddy, float* dW, float* db, int64_t n, int k, int d, int accumulate, cudaStream_t st) {
  return wgrad_simt(X, ldx, dY, lddy, dW, db, n, k, d, accumulate, st);
}
int proj_wgrad_simt(const uint16_t* X, int64_t ldx, const float* dY, int64_t lddy, float* dW, float* db, int64_t n, int k, int d, int accumulate, cudaStream_t st) {
  return wgrad_simt(X, ldx, dY, lddy, dW, db, n, k, d, accumulate, st);
}
}  // namespace llmrec
