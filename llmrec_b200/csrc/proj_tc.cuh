// Parameter blocks of the tensor-core projection kernels (proj_tc.cu).
#pragma once
#include "tc_common.cuh"

namespace llmrec {

constexpr int kMaxProb = 8;
constexpr int BK = 32;  // k (fwd) / rows (wgrad) per pipeline stage: fp32 per 128-byte swizzle row
// Tile = 2 consumer warpgroups x MB blocks of wgmma M = 64: 256 rows (fwd) / features (wgrad) when MB = 2, 128 when MB = 1.
constexpr int tile_m(int mb) { return 128 * mb; }

struct FwdProblem { int n, k, kblocks, tile_start; long long ldy; float* Y; const float* bias; };
struct FwdParams {
  CUtensorMap tmA[kMaxProb];  // X [n x k], boxes [TM rows][32 k], 128-byte swizzle
  CUtensorMap tmW[kMaxProb];  // [2d x k] (hi rows then lo rows) when SPLIT, [d x k] otherwise; boxes [d][32 k]
  FwdProblem prob[kMaxProb];
  int n_prob, total_tiles, d;
};

struct WgProblem { int n, k, ft_tiles, chunks, rows_per_chunk, item_start; };
struct WgParams {
  CUtensorMap tmX[kMaxProb];  // X [n x k], boxes [32 rows][32 features], 128-byte swizzle
  CUtensorMap tmG[kMaxProb];  // dY^T [2d x n] (hi rows then lo rows) when SPLIT, [d x n] otherwise; boxes [d][32 rows]
  WgProblem prob[kMaxProb];
  int n_prob, total_items, d;
  float* partial;  // [total_items][TM][d]
};

}  // namespace llmrec
