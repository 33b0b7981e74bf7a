// Parameter blocks of the tensor-core projection kernels (proj_tc.cu).
#pragma once
#include "tc_common.cuh"

namespace llmrec {

constexpr int kMaxProb = 8;
constexpr int BK = 32;    // k (fwd) / rows (wgrad) per pipeline stage: fp32 per 128-byte swizzle row
constexpr int BK16 = 64;  // the same for bf16 X: 64 elements per 128-byte swizzle row
constexpr int stage_k(bool bf16) { return bf16 ? BK16 : BK; }
// Tile = 2 consumer warpgroups x MB blocks of wgmma M = 64: 256 rows (fwd) / features (wgrad) when MB = 2, 128 when MB = 1.
constexpr int tile_m(int mb) { return 128 * mb; }

// Element type of the side-feature table X.  I8: the int8 row format of include/llmrec_b200.h (k int8 values, zero padding to
// roundup(k, 16), the row's fp32 power-of-two scale there); the kernels expand it to bf16 in shared memory and run the bf16 pipeline.
enum class XType { F32, BF16, I8 };
constexpr int i8_scale_offset(int k) { return (k + 15) & ~15; }   // byte offset of a row's scale

// The row scales of int8 tables (fwd and wgrad): row r's scale is the fp32 at scale[p] + r * pitch[p] (NULL for other tables)
struct RowScales { const uint8_t* scale[kMaxProb]; long long pitch[kMaxProb]; };

// rows: optional output row map (X row r -> Y row rows[r]); NULL = identity
struct FwdProblem { int n, k, kblocks, tile_start; long long ldy; float* Y; const float* bias; const int* rows; };
struct FwdParams {
  CUtensorMap tmA[kMaxProb];  // X [n x k], boxes [TM rows][32 k] (bf16: [TM rows][64 k]), 128-byte swizzle
                              // int8: [TM rows][64 k] bytes, no swizzle (raw q, expanded in the kernel)
  CUtensorMap tmW[kMaxProb];  // fp32: [2d x k] (hi rows then lo rows) when SPLIT, [d x k] otherwise; boxes [d][32 k]
                              // bf16 / int8: [3d x k] (w0, w1, w2 rows) when SPLIT, [d x k] (w0) otherwise; boxes [d][64 k]
  FwdProblem prob[kMaxProb];
  RowScales xs;
  int n_prob, total_tiles, d;
};

struct WgProblem { int n, k, ft_tiles, chunks, rows_per_chunk, item_start; };
struct WgParams {
  CUtensorMap tmX[kMaxProb];  // X [n x k], boxes [32 rows][32 features] (bf16: [64 rows][64 features]), 128-byte swizzle
                              // int8: [64 rows][64 features] bytes, no swizzle (raw q, expanded in the kernel)
  CUtensorMap tmG[kMaxProb];  // bf16 / int8 X or mode 1: dY^T from dyt_split, [d x n] (bf16 split: [3d x n] bf16 terms); boxes [d][32 | 64 rows]
  const float* dY[kMaxProb];  // dY [m x d] with row stride lddy; fp32 X in mode 0: the kernel builds B (dY^T hi, lo) from it
  long long lddy[kMaxProb];
  const int* rows[kMaxProb];  // optional dY row map: X row r pairs with dY row rows[r]; NULL = identity
  WgProblem prob[kMaxProb];
  RowScales xs;
  int n_prob, total_items, d;
  float* partial;  // [total_items][TM][d]
};

}  // namespace llmrec
