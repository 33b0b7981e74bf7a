// Exact-fp32 SIMT version of the side-feature projection and its weight gradient
// (nn.Linear at Models.py:145-150).  mode 2 of llmrec_proj_*: the bit-conservative path used as the
// on-device checker for the wgmma kernels (proj_tc.cu) and for shapes those do not cover.
// Templated on the element type of X: fp32, or bf16 (raw uint16_t bits) widened to fp32 on load -- the same FMA order, so a bf16
// table gives the bits of the fp32 kernel on its upcast copy -- or int8 rows (include/llmrec_b200.h: ldx is the row pitch in bytes,
// the row's scale sits at byte roundup(k, 16)) widened to q * scale, the exact value of the bf16 table the int8 one encodes.
#include "common.cuh"

namespace llmrec {

__device__ __forceinline__ float x_f32(float x) { return x; }
__device__ __forceinline__ float x_f32(uint16_t x) { return __uint_as_float((uint32_t)x << 16); }
// X[r][c] of a table of logical width k
template <class T>
__device__ __forceinline__ float x_at(const T* X, int64_t ldx, int64_t r, int c, int) { return x_f32(X[r * ldx + c]); }
__device__ __forceinline__ float x_at(const int8_t* X, int64_t ldx, int64_t r, int c, int k) {
  const int8_t* row = X + r * ldx;
  return (float)row[c] * __ldg(reinterpret_cast<const float*>(row + ((k + 15) & ~15)));
}

// Y[n x d] = X[n x k] W^T[k x d] + b ; 64x64 tile, K step 16, 4x4 per thread.  rows (optional): X row r is written to Y row rows[r]
template <class T>
__global__ void __launch_bounds__(256) proj_fwd_simt_kernel(const T* __restrict__ X, int64_t ldx, const float* __restrict__ W,
                                                            const float* __restrict__ bias, float* __restrict__ Y, int64_t ldy,
                                                            int64_t n, int k, int d, const int* __restrict__ rows) {
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
      Xs[kk][r] = (gr < n && k0 + kk < k) ? x_at(X, ldx, gr, k0 + kk, k) : 0.f;
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
    const int64_t yr = rows ? (int64_t)rows[gr] : gr;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int gc = col0 + tx * 4 + j;
      if (gc < d) Y[yr * ldy + gc] = acc[i][j] + (bias ? bias[gc] : 0.f);
    }
  }
}

// dW[d x k] += sum_r dY[r,:]^T X[r,:] over a row chunk ; db[d] += colsum(dY) (k-tile 0 only).
// rows (optional): X row r pairs with dY row rows[r] (db is then NULL: colsum_simt_kernel sums every row of dY)
template <class T>
__global__ void __launch_bounds__(256) proj_wgrad_simt_kernel(const T* __restrict__ X, int64_t ldx, const float* __restrict__ dY, int64_t lddy,
                                                              float* __restrict__ dW, float* __restrict__ db, int64_t n, int k, int d, int rows_per_chunk,
                                                              const int* __restrict__ rows) {
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
      Gs[r][c] = (gr < r_end && d0 + c < d) ? dY[(rows ? (int64_t)rows[gr] : gr) * lddy + d0 + c] : 0.f;
      Xs[r][c] = (gr < r_end && k0 + c < k) ? x_at(X, ldx, gr, k0 + c, k) : 0.f;
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

// db[d] += colsum(dY[n_dy x d]) for the row-mapped weight gradient: every row of dY, in row order within 1024-row chunks whose sums are
// added atomically -- the order of the weight-gradient kernel's own bias sums, so one chunk gives its bits
__global__ void __launch_bounds__(256) colsum_simt_kernel(const float* __restrict__ dY, int64_t lddy, float* __restrict__ db, int64_t n_dy, int d,
                                                          int rows_per_chunk) {
  const int c = blockIdx.y * 256 + threadIdx.x;
  if (c >= d) return;
  const int64_t r_beg = (int64_t)blockIdx.x * rows_per_chunk, r_end = min(n_dy, r_beg + rows_per_chunk);
  float s = 0.f;
  for (int64_t r = r_beg; r < r_end; ++r) s += dY[r * lddy + c];
  atomicAdd(db + c, s);
}

template <class T>
static int fwd_simt(const T* X, int64_t ldx, const float* W, const float* bias, float* Y, int64_t ldy, int64_t n, int k, int d, const int* rows,
                    cudaStream_t st) {
  dim3 grid((unsigned)((n + 63) / 64), (d + 63) / 64);
  proj_fwd_simt_kernel<T><<<grid, 256, 0, st>>>(X, ldx, W, bias, Y, ldy, n, k, d, rows);
  LLMREC_CHECK_LAUNCH("proj_fwd_simt");
  return 0;
}
template <class T>
static int wgrad_simt(const T* X, int64_t ldx, const float* dY, int64_t lddy, float* dW, float* db, int64_t n, int k, int d, int accumulate,
                      const int* rows, int64_t n_dy, cudaStream_t st) {
  if (!accumulate) {
    cudaMemsetAsync(dW, 0, sizeof(float) * (size_t)d * k, st);
    if (db) cudaMemsetAsync(db, 0, sizeof(float) * d, st);
  }
  const int rows_per_chunk = 1024;
  const bool mapped = rows || n_dy != n;     // the bias sums then run over the n_dy rows of dY, not beside the weight gradient
  if (n > 0) {
    dim3 grid((k + 63) / 64, (d + 63) / 64, (unsigned)((n + rows_per_chunk - 1) / rows_per_chunk));
    proj_wgrad_simt_kernel<T><<<grid, 256, 0, st>>>(X, ldx, dY, lddy, dW, mapped ? nullptr : db, n, k, d, rows_per_chunk, rows);
    LLMREC_CHECK_LAUNCH("proj_wgrad_simt");
  }
  if (mapped && db && n_dy > 0) {
    colsum_simt_kernel<<<dim3((unsigned)((n_dy + rows_per_chunk - 1) / rows_per_chunk), (d + 255) / 256), 256, 0, st>>>(dY, lddy, db, n_dy, d, rows_per_chunk);
    LLMREC_CHECK_LAUNCH("colsum_simt");
  }
  return 0;
}
int proj_fwd_simt(const float* X, int64_t ldx, const float* W, const float* bias, float* Y, int64_t ldy, int64_t n, int k, int d, const int* rows,
                  cudaStream_t st) {
  return fwd_simt(X, ldx, W, bias, Y, ldy, n, k, d, rows, st);
}
int proj_fwd_simt(const uint16_t* X, int64_t ldx, const float* W, const float* bias, float* Y, int64_t ldy, int64_t n, int k, int d, const int* rows,
                  cudaStream_t st) {
  return fwd_simt(X, ldx, W, bias, Y, ldy, n, k, d, rows, st);
}
int proj_wgrad_simt(const float* X, int64_t ldx, const float* dY, int64_t lddy, float* dW, float* db, int64_t n, int k, int d, int accumulate,
                    const int* rows, int64_t n_dy, cudaStream_t st) {
  return wgrad_simt(X, ldx, dY, lddy, dW, db, n, k, d, accumulate, rows, n_dy, st);
}
int proj_wgrad_simt(const uint16_t* X, int64_t ldx, const float* dY, int64_t lddy, float* dW, float* db, int64_t n, int k, int d, int accumulate,
                    const int* rows, int64_t n_dy, cudaStream_t st) {
  return wgrad_simt(X, ldx, dY, lddy, dW, db, n, k, d, accumulate, rows, n_dy, st);
}
int proj_fwd_simt(const int8_t* X, int64_t ldx, const float* W, const float* bias, float* Y, int64_t ldy, int64_t n, int k, int d, const int* rows,
                  cudaStream_t st) {
  return fwd_simt(X, ldx, W, bias, Y, ldy, n, k, d, rows, st);
}
int proj_wgrad_simt(const int8_t* X, int64_t ldx, const float* dY, int64_t lddy, float* dW, float* db, int64_t n, int k, int d, int accumulate,
                    const int* rows, int64_t n_dy, cudaStream_t st) {
  return wgrad_simt(X, ldx, dY, lddy, dW, db, n, k, d, accumulate, rows, n_dy, st);
}
}  // namespace llmrec
