// Side-feature projection on the Hopper tensor cores (wgmma, fp32 accumulators in registers, TMA-fed).
//
//   forward  Y[n x d]  = X[n x k] W[d x k]^T + b          (nn.Linear, Models.py:145-150)
//   wgrad    dW[d x k] = dY[n x d]^T X[n x k], db = colsum(dY)   (its autograd; X is a constant feature table)
//
// Both are HBM-bound at d = 64 (the job of the kernel is to stream X once at HBM speed) with the tensor work not far behind.
// All 8 projections of a step run as ONE grouped launch: a persistent grid (one CTA per SM) walks the work units -- 256-row
// tiles (fwd) / (256-feature tile x row chunk) items (wgrad), 128 above d = 128 or when 256 would leave SMs idle -- looked up in
// a problem table, long-K problems first.
//
// Precision: fp32 operands are split  x = hi + lo  (hi = top 19 bits, exactly TF32-representable) and three tf32 wgmmas
// accumulate lo*hi + hi*lo + hi*hi in fp32 registers ("3xTF32", error ~2^-21 relative per product, i.e. fp32-class).  mode 1
// skips the split (plain TF32, ~2^-11).
//
// CTA = 3 warpgroups.  Warpgroup 0 is the producer: one thread keeps a ring of TMA stages in flight (a full and an empty
// mbarrier per stage), running ahead across work units; it hands most of its registers to the two consumer warpgroups
// (setmaxnreg).  Each consumer owns MB blocks of 64 rows (fwd) / features (wgrad) of the tile.  X goes into wgmma A-fragment
// REGISTERS straight from the stage and is split there; B (W or dY^T, hi and lo) is consumed from shared memory.  W arrives from
// TMA ready-made, split once per step by `wsplit`.  The fp32 3xTF32 weight gradient builds dY^T hi / lo in the kernel: the
// producer's warps 1..3 gather the stage's dY rows (through the row map), split them and store them in the swizzled layout TMA
// would give, so dY^T never goes through HBM (WgUnit::build).  bf16 X and mode 1 read dY^T from `dyt_split` by TMA.  One
// wgmma group (one k8 step) stays in flight while the next A fragment is loaded; no CTA-wide barrier in the main loop.
//   forward  A = X[rows][k]: the X tile [TM rows][32 k] arrives K-major with the 128-byte swizzle, exactly the A layout.
//   wgrad    A = X^T (M = features, K = rows): the fragment is read transposed out of the raw X tile, which arrives as TM/32
//            boxes [32 rows][32 features] with the 128-byte swizzle; features are permuted inside the tile so that the reads
//            are bank-conflict free (arithmetic at ld_frag_wgrad), and the epilogue undoes the permutation.
// bf16 X (--feat_dtype bf16, BF16 = true): the same pipeline with 64 k / rows per stage.  X is exact in bf16, so it is not split and
// A is read by descriptor straight from the stage (wgrad: MN-major, no permutation); W / dY^T arrive as three exact bf16 terms
// (wsplit_bf16, dyt_split<true>) and each k16 step issues X*w2 + X*w1 + X*w0: no product term is dropped (mode 1: X*w0 only).
// int8 X (--feat_dtype int8, XType::I8): every stored q * 2^e is a bf16 number, so the bf16 pipeline runs unchanged on stages that
// producer warps 1..3 expand from the raw q the TMA brings (I8Stage): the bits of the bf16 kernels on the dequantized table.
#include <mutex>
#include <stdlib.h>
#include <vector>
#include <string.h>
#include "common.cuh"
#include "tc_common.cuh"
#include "proj_tc.cuh"

namespace llmrec {

using namespace tc;


// ------------------------------------------------------------------------------------------------
// host: tensor maps
// ------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                             const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                             CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeFn get_encode() {
  static EncodeFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeFn>(p);
  }
  return fn;
}

bool make_tmap_2d(CUtensorMap* out, CUtensorMapDataType dtype, const void* base, uint64_t inner, uint64_t outer, uint64_t row_stride_bytes,
                  uint32_t box_inner, uint32_t box_outer, bool swizzle128) {
  struct Entry { TmapKey k; CUtensorMap m; };
  static std::vector<Entry> cache;
  static std::mutex mu;
  TmapKey key{base, inner, outer, row_stride_bytes, box_inner, box_outer, swizzle128 ? 1u : 0u, (uint32_t)dtype};
  std::lock_guard<std::mutex> lock(mu);
  for (auto& e : cache)
    if (memcmp(&e.k, &key, sizeof(key)) == 0) { *out = e.m; return true; }
  EncodeFn enc = get_encode();
  if (!enc) { set_error("cuTensorMapEncodeTiled entry point unavailable"); return false; }
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {row_stride_bytes};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(out, dtype, 2, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed (%d) inner=%llu outer=%llu stride=%llu box=%ux%u", (int)r,
                                     (unsigned long long)inner, (unsigned long long)outer, (unsigned long long)row_stride_bytes, box_inner, box_outer); return false; }
  if (cache.size() > 256) cache.clear();
  cache.push_back({key, *out});
  return true;
}

__device__ __forceinline__ uint8_t* align1024(uint8_t* p) {
  return reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(p) + 1023) & ~uintptr_t(1023));
}

// ------------------------------------------------------------------------------------------------
// one main loop for both directions
// ------------------------------------------------------------------------------------------------
constexpr uint32_t kSmemMax = 227u * 1024u;   // dynamic shared memory per block on sm_90

// BF16: X is a bf16 table.  A stage then covers 64 k (fwd) / rows (wgrad) in the same bytes, and a 3-way split of the fp32
// operand (W or dY^T) gives three B tiles instead of two.
template <int D, bool SPLIT, int MB, bool BF16 = false>
struct ProjCfg {
  static constexpr int TM = tile_m(MB);
  static constexpr int NB = SPLIT ? (BF16 ? 3 : 2) : 1;        // B tiles per stage
  static constexpr uint32_t kX = TM * 128u;                    // X tile of one stage: 128 bytes per row / feature
  static constexpr uint32_t kB = D * 128u;                     // one B operand tile [D][32 fp32 | 64 bf16]
  static constexpr uint32_t kStage = kX + kB * NB;
  static constexpr int kFit = (int)((kSmemMax - 1024u - 256u) / kStage);
  static constexpr int kStages = kFit > 4 ? 4 : kFit;          // 4 at d = 64, 3 at d = 128, 2 at d = 256
  static constexpr uint32_t kSmem = 1024u /*align slack*/ + kStages * kStage + 3u * kStages * 8u;   // + full, empty, raw barriers
  static_assert(kStages >= 2, "projection ring needs two stages");
};

// A fragment (4 registers, layout at WgmmaRS) of k8 step kk for m64 block `blk` (0 .. 2MB-1 over the CTA), read from the stage's X
// tile.  Forward: A(m, k) = X tile row m, column k; element (r, c) sits at r*128 + ((c/4) ^ (r%8))*16 + (c%4)*4.  A warp's 32
// lanes read rows 16w + g (r%8 = g), chunk (2kk) ^ g or (2kk+1) ^ g, word t: 8 chunks x 4 words = 32 banks, conflict free.
__device__ __forceinline__ void ld_frag_fwd(uint32_t (&a)[4], uint32_t sx, int blk, int kk, int warp, int lane) {
  const int g = lane >> 2, t = lane & 3;
  const uint32_t row = sx + (blk * 64 + warp * 16 + g) * 128 + t * 4;
  const uint32_t c0 = ((2 * kk) ^ g) << 4, c1 = c0 ^ 16;
  a[0] = lds_u32(row + c0);
  a[1] = lds_u32(row + 1024 + c0);
  a[2] = lds_u32(row + c1);
  a[3] = lds_u32(row + 1024 + c1);
}
// Wgrad: A(m, k) = X[row k][feature phi(m)] out of boxes [32 rows][32 features] (4 KiB, same swizzle, r%8 = row%8).
// Fragment row m = 16w + 8h + g (h = 0 for a0/a2, 1 for a1/a3), k = t (a0/a1) or t + 4 (a2/a3) within k8 step kk (rows 8kk..).
// Feature map inside the block's 64 features:  phi(m) = 32(w/2) + 8(w%2) + 4h + (g%4) + 16(g/4), a bijection onto 0..63
// (bits: g%4 -> 0-1, h -> 2, w%2 -> 3, g/4 -> 4, w/2 -> 5).  In box w/2 the element sits in chunk q = 2(w%2) + h + 4(g/4), word g%4.
// Banks of one load (fixed w, h, kk; lanes vary g, t): chunk q ^ (row % 8) = (2(w%2) + h + 4(g/4)) ^ t [^ 4 for k = t + 4];
// t < 4 only touches bits 0-1, so (g/4, t) -> 8 distinct chunks, times word g%4 -> 32 distinct banks: conflict free.
__device__ __forceinline__ int wgrad_feature(int blk, int warp, int h, int g) {
  return blk * 64 + 32 * (warp >> 1) + 8 * (warp & 1) + 4 * h + (g & 3) + 16 * (g >> 2);
}
__device__ __forceinline__ void ld_frag_wgrad(uint32_t (&a)[4], uint32_t sx, int blk, int kk, int warp, int lane) {
  const int g = lane >> 2, t = lane & 3;
  const uint32_t base = sx + (blk * 2 + (warp >> 1)) * 4096 + kk * 1024 + t * 128 + (g & 3) * 4;
  const uint32_t q = (2 * (warp & 1) + 4 * (g >> 2)) ^ t;
  a[0] = lds_u32(base + (q << 4));
  a[1] = lds_u32(base + ((q ^ 1) << 4));
  a[2] = lds_u32(base + 512 + ((q ^ 4) << 4));
  a[3] = lds_u32(base + 512 + ((q ^ 5) << 4));
}

// ---- int8 X: a raw stage expanded into the bf16 stage layout --------------------------------------------------------------------
// 16 int8 q (one 16-byte word) times the row scale 2^e -> 16 bf16, exactly: q * 2^e has at most 7 significant bits and is a normal
// fp32 (the format clamps e to [-126, 120]), so its top 16 bits are the bf16.  q is widened without a conversion instruction: q + 128
// goes into the low byte of 2^23's significand, and float(0x4B000000 | (q + 128)) - (2^23 + 128) = q exactly.
__device__ __forceinline__ uint32_t i8_pair_bf16(uint32_t w, int b, float s) {   // w: four q + 128; elements b, b + 1 -> packed bf16
  const float x0 = (__uint_as_float(__byte_perm(w, 0x4B000000u, 0x7650u + b)) - 8388736.0f) * s;
  const float x1 = (__uint_as_float(__byte_perm(w, 0x4B000000u, 0x7651u + b)) - 8388736.0f) * s;
  return __byte_perm(__float_as_uint(x0), __float_as_uint(x1), 0x7632u);
}
__device__ __forceinline__ void i8x16_bf16(const uint4& q, float s, uint4& lo, uint4& hi) {
  const uint32_t w0 = q.x ^ 0x80808080u, w1 = q.y ^ 0x80808080u, w2 = q.z ^ 0x80808080u, w3 = q.w ^ 0x80808080u;
  lo = make_uint4(i8_pair_bf16(w0, 0, s), i8_pair_bf16(w0, 2, s), i8_pair_bf16(w1, 0, s), i8_pair_bf16(w1, 2, s));
  hi = make_uint4(i8_pair_bf16(w2, 0, s), i8_pair_bf16(w2, 2, s), i8_pair_bf16(w3, 0, s), i8_pair_bf16(w3, 2, s));
}
__device__ __forceinline__ void converters_sync() { asm volatile("bar.sync 1, 96;" ::: "memory"); }   // producer warps 1..3

// The converter warps (producer warps 1..3, ct = 0..95) of an int8 unit.  TMA put the stage's raw q into the UPPER half of the stage's
// X area (TM * 64 bytes), as TM/64 groups of 4 KiB: group g = 64 rows (fwd) / 64 features (wgrad) at TM*64 + 4096 g.  A task expands
// 16 q at Unit::raw_off into the two 16-byte bf16 chunks at Unit::out_off -- the bytes the bf16 TMA load of the dequantized table
// writes there (128-byte swizzle; rows past n and columns past k are zeros, as TMA fills them).  Group g's bf16 output is the 8 KiB at
// 8192 g: the groups of the lower half touch no raw byte; group g >= TM/128 overwrites raw groups 2g - TM/64 and 2g - TM/64 + 1, the
// earlier one of which (and at the last group, its own) is still input.  So before writing such a group every converter has loaded the
// group's inputs, and the three warps meet at a named barrier.
template <class Unit>
struct I8Stage {
  static constexpr int kGroups = Unit::Cfg::TM / 64, kTasks = 256;   // per group: 64 x 64 q, 16 per task
  static constexpr int kPer = (kTasks + 95) / 96;                    // 3 tasks per converter thread and group
  float sc[kPer];                // wgrad: the scales of the tasks' stage rows (the same 64 rows in every group)
  const float* tile_sc = nullptr;   // fwd: the tile's TM row scales in shared memory (Unit::kScalesPerUnit)
  // wgrad: global loads, issued before the wait for the raw box
  __device__ void load_scales(const Unit& w, int kb, int ct) {
#pragma unroll
    for (int m = 0; m < kPer; ++m) {
      const int t = ct + 96 * m;
      sc[m] = t < kTasks ? w.row_scale(w.task_row(0, t, kb)) : 0.f;
    }
  }
  __device__ void expand(uint8_t* sx, int ct) const {
#pragma unroll
    for (int g = 0; g < kGroups; ++g) {
      uint4 v[kPer];
#pragma unroll
      for (int m = 0; m < kPer; ++m) {
        const int t = ct + 96 * m;
        if (t < kTasks) v[m] = *reinterpret_cast<const uint4*>(sx + Unit::Cfg::TM * 64u + g * 4096u + Unit::raw_off(t));
      }
      if (2 * g >= kGroups) converters_sync();
#pragma unroll
      for (int m = 0; m < kPer; ++m) {
        const int t = ct + 96 * m;
        if (t >= kTasks) continue;
        uint4 lo, hi;
        uint32_t o_lo, o_hi;
        i8x16_bf16(v[m], Unit::kScalesPerUnit ? tile_sc[64 * g + (t >> 2)] : sc[m], lo, hi);
        Unit::out_off(t, o_lo, o_hi);
        *reinterpret_cast<uint4*>(sx + g * 8192u + o_lo) = lo;
        *reinterpret_cast<uint4*>(sx + g * 8192u + o_hi) = hi;
      }
    }
  }
};

// task t of a group: 16 q of group row i = t / 4 (fwd: tile row 64g + i; wgrad: stage row i), columns 16 (t % 4) .. + 15 of the group
// (fwd: k; wgrad: features 64g ..); raw row i at 64 i, the bf16 row at 128 i with chunk c at ((c ^ i) % 8) * 16
__device__ __forceinline__ uint32_t i8_raw_off(int t) { return (t >> 2) * 64u + (t & 3) * 16u; }
__device__ __forceinline__ void i8_out_off(int t, uint32_t& lo, uint32_t& hi) {
  const int i = t >> 2, c = 2 * (t & 3);
  lo = i * 128u + (((c ^ i) & 7) << 4);
  hi = i * 128u + ((((c + 1) ^ i) & 7) << 4);
}

// scale of table row `row` of problem p (0 past the table: those rows load as q = 0)
__device__ __forceinline__ float i8_row_scale(const RowScales& xs, int p, int n, int row) {
  return row < n ? __ldg(reinterpret_cast<const float*>(xs.scale[p] + (long long)row * xs.pitch[p])) : 0.f;
}

// work unit -> (problem, number of k-blocks, what the producer loads for k-block kb, where the epilogue writes)
// I8 (with BF16): X is an int8 table; the bf16 pipeline runs on the stages the converter warps expand (I8Stage).
template <int D, bool SPLIT, int MB, bool BF16 = false, bool I8 = false>
struct FwdUnit {
  using Cfg = ProjCfg<D, SPLIT, MB, BF16>;
  static_assert(!I8 || BF16, "int8 X runs the bf16 pipeline");
  static constexpr int kTransA = 0;   // bf16: A = the X tile as it arrived, K-major
  struct BuildState {};               // no B to build: W arrives by TMA
  static constexpr int kBuilders = I8 ? 3 : 0;   // warps that write stage operands in the kernel: the int8 converters; W arrives by TMA
  // setmaxnreg: 128 * 40 + 256 * 232 = 384 * 168; the int8 converters hold a group's raw words in flight: 128 * 72 + 256 * 216
  static constexpr int kProducerRegs = I8 ? 72 : 40, kConsumerRegs = I8 ? 216 : 232;
  static constexpr uint32_t kRawTx = I8 ? Cfg::TM * 64u : 0u;   // raw q bytes per stage, on the stage's own raw barrier
  static constexpr uint32_t kTx = I8 ? Cfg::kStage - Cfg::kX : Cfg::kStage;   // TMA bytes per stage on `full`: X and W (int8: W)
  const FwdParams& P; int p, mblk, kb_n;
  __device__ FwdUnit(const FwdParams& P_, int u) : P(P_) {
    p = 0;
    while (p + 1 < P.n_prob && u >= P.prob[p + 1].tile_start) ++p;
    mblk = u - P.prob[p].tile_start;
    kb_n = P.prob[p].kblocks;
  }
  __device__ void issue(uint8_t* st, uint64_t* bar, uint64_t* raw_bar, int kb, uint64_t pol) const {
    constexpr int bk = stage_k(BF16);
    // fp32 / bf16 X: no evict_first.  A box row is the 128 bytes of k-block kb of one X row, and the map's 256-byte L2 promotion
    // also brings in k-block kb + 1, which this CTA reads one stage later.  Marked evict_first, that half is evidently evicted
    // before then and read from HBM again: without the hint the grouped forward at netflix takes 0.210 ms instead of 0.230
    // (H100 SXM, 700 W; DESIGN §5).
    if constexpr (I8) tma_load_2d_hint(st + Cfg::TM * 64, &P.tmA[p], raw_bar, kb * bk, mblk * Cfg::TM, pol);   // [TM rows][64 q]: the groups in order
    else tma_load_2d(st, &P.tmA[p], bar, kb * bk, mblk * Cfg::TM);
#pragma unroll
    for (int i = 0; i < Cfg::NB; ++i) tma_load_2d(st + Cfg::kX + i * Cfg::kB, &P.tmW[p], bar, kb * bk, i * D);
  }
  // int8 (I8Stage): group g = tile rows 64g .. 64g + 63, the same rows at every k-block: the converters put the tile's row scales
  // into shared memory once per unit (ts[i] = scale of tile row i)
  static constexpr bool kScalesPerUnit = true;
  __device__ void tile_scales(float* ts, int ct) const {
    for (int i = ct; i < Cfg::TM; i += 96) ts[i] = i8_row_scale(P.xs, p, P.prob[p].n, mblk * Cfg::TM + i);
  }
  static __device__ uint32_t raw_off(int t) { return i8_raw_off(t); }
  static __device__ void out_off(int t, uint32_t& lo, uint32_t& hi) { i8_out_off(t, lo, hi); }
  static __device__ void ld_frag(uint32_t (&a)[4], uint32_t sx, int blk, int kk, int warp, int lane) { ld_frag_fwd(a, sx, blk, kk, warp, lane); }
  // bf16: descriptor of m64 block `blk` (64 rows x 128 bytes), k16 step kk (+32 bytes inside the swizzled rows)
  static __device__ uint64_t a_desc(uint32_t sx, int blk, int kk) { return gmma_desc_sw128(sx + blk * 8192u + kk * 32u); }
  __device__ void store(float (&acc)[MB][D / 2], int cw, int warp, int lane) const {   // registers (+bias) -> Y (at rows[row] with a row map)
    const FwdProblem& pr = P.prob[p];
    const int g = lane >> 2, t = lane & 3;
#pragma unroll
    for (int j = 0; j < MB; ++j) {
      const int row0 = mblk * Cfg::TM + (cw * MB + j) * 64 + warp * 16 + g;
      long long yrow[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = row0 + 8 * h;
        yrow[h] = row < pr.n ? (pr.rows ? (long long)__ldg(pr.rows + row) : (long long)row) : -1;
      }
#pragma unroll
      for (int c = 0; c < D / 8; ++c) {
        const int col = c * 8 + 2 * t;
        const float2 b = pr.bias ? __ldg(reinterpret_cast<const float2*>(pr.bias + col)) : make_float2(0.f, 0.f);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (yrow[h] >= 0)
            *reinterpret_cast<float2*>(pr.Y + yrow[h] * pr.ldy + col) = make_float2(acc[j][4 * c + 2 * h] + b.x, acc[j][4 * c + 2 * h + 1] + b.y);
        }
      }
    }
  }
};

template <int D, bool SPLIT, int MB, bool BF16 = false, bool I8 = false>
struct WgUnit {
  using Cfg = ProjCfg<D, SPLIT, MB, BF16>;
  static_assert(!I8 || BF16, "int8 X runs the bf16 pipeline");
  static constexpr int kBk = stage_k(BF16);
  static constexpr int kTransA = 1;   // bf16: A = X^T, read MN-major out of the raw X tile (no feature permutation)
  const WgParams& P; int p, u, ft, r0, kb_n;
  __device__ WgUnit(const WgParams& P_, int u_) : P(P_), u(u_) {
    p = 0;
    while (p + 1 < P.n_prob && u >= P.prob[p + 1].item_start) ++p;
    const WgProblem& pr = P.prob[p];
    const int local = u - pr.item_start, chunk = local / pr.ft_tiles;
    ft = local - chunk * pr.ft_tiles;
    r0 = chunk * pr.rows_per_chunk;
    kb_n = (min(pr.n, r0 + pr.rows_per_chunk) - r0 + kBk - 1) / kBk;   // chunks are stage-aligned; rows past n load as zeros
  }
  // fp32 X, 3xTF32: producer warps 1..3 build B from dY (below).  bf16 / int8 X and mode 1 keep B = dY^T by TMA from `dyt_split`: their
  // consumers finish a stage sooner than three warps build one, measured slower at the netflix and movielens shapes (H100 SXM, 700 W).
  // int8 X: warps 1..3 expand the raw X stage instead (I8Stage).
  static constexpr bool kBuildsB = SPLIT && !BF16;
  static constexpr int kBuilders = kBuildsB || I8 ? 3 : 0;
  // kAhead (d <= 64, below): the builders hold two stages' first batches, 128 * 120 + 256 * 192 = 384 * 168 (the consumers' d/2
  // accumulators per m64 block fit); otherwise 128 * 72 + 256 * 216: the builders' loads in flight
  static constexpr bool kAhead = kBuildsB && D <= 64;
  static constexpr int kProducerRegs = kAhead ? 120 : kBuilders ? 72 : 40;
  static constexpr int kConsumerRegs = kAhead ? 192 : kBuilders ? 216 : 232;
  static constexpr uint32_t kRawTx = I8 ? Cfg::TM * 64u : 0u;   // raw q bytes per stage, on the stage's own raw barrier
  static constexpr uint32_t kTx = kBuildsB ? Cfg::kX : I8 ? Cfg::kStage - Cfg::kX : Cfg::kStage;   // TMA bytes per stage on `full`
  __device__ void issue(uint8_t* st, uint64_t* bar, uint64_t* raw_bar, int kb, uint64_t pol) const {
    const int r = r0 + kb * kBk;
    if constexpr (I8) {     // TM/64 boxes [64 rows][64 features] of raw q, 4 KiB each, into the upper half of the X area
#pragma unroll
      for (int b = 0; b < Cfg::TM / 64; ++b) tma_load_2d_hint(st + Cfg::TM * 64 + b * 4096, &P.tmX[p], raw_bar, ft * Cfg::TM + 64 * b, r, pol);
    } else if constexpr (BF16) {   // TM/64 boxes [64 rows][64 features], 8 KiB each: one per m64 block
#pragma unroll
      for (int b = 0; b < Cfg::TM / 64; ++b) tma_load_2d_hint(st + b * 8192, &P.tmX[p], bar, ft * Cfg::TM + 64 * b, r, pol);
    } else {
#pragma unroll
      for (int b = 0; b < Cfg::TM / 32; ++b) tma_load_2d_hint(st + b * 4096, &P.tmX[p], bar, ft * Cfg::TM + 32 * b, r, pol);
    }
    if constexpr (!kBuildsB) {
#pragma unroll
      for (int i = 0; i < Cfg::NB; ++i) tma_load_2d(st + Cfg::kX + i * Cfg::kB, &P.tmG[p], bar, r, i * D);
    }
  }
  // int8 (I8Stage): group g = tile features 64g .. 64g + 63 (the bf16 box of m64 block g) over the stage's 64 rows
  static constexpr bool kScalesPerUnit = false;
  __device__ void tile_scales(float*, int) const {}
  __device__ int task_row(int, int t, int kb) const { return r0 + kb * kBk + (t >> 2); }
  __device__ float row_scale(int row) const { return i8_row_scale(P.xs, p, P.prob[p].n, row); }
  static __device__ uint32_t raw_off(int t) { return i8_raw_off(t); }
  static __device__ void out_off(int t, uint32_t& lo, uint32_t& hi) { i8_out_off(t, lo, hi); }
  // B of stage kb = dY^T over the stage's kBk rows, split into hi and lo, written by builder warp bw (0 .. kBuilders-1) in the layout
  // TMA gives a [D][32] box with the 128-byte swizzle: element (column c, stage row j) at c*128 + ((j/4 ^ c) % 8)*16 + (j%4)*4.  Lane l owns
  // stage row l, so it reads its dY row through the row map once; a task is 8 columns (32 bytes of the row, two 16-byte loads),
  // the warps take every kBuilders-th task.  Each store of a warp writes one column c: chunk (l/4 ^ c) % 8, word l%4 -- 32
  // distinct banks, no conflict.  Rows at or past n are zeros, as TMA fills them.
  // The builder is latency-bound on its row map -> dY -> store chain, so the chain is software-pipelined across the stages of a unit
  // (BuildState), and no L2 load waits for the stage slot (`wait`).  kAhead (d <= 64, one batch is the whole stage): while stage kb
  // is stored, stage kb + 1's dY loads and stage kb + 2's row-map entries are in flight.  Wider stages: stage kb + 1's row-map
  // entries are loaded while stage kb is built, and stage kb's first batch of dY loads is issued before the wait.
  static constexpr int kTasks = D / 8;
  static constexpr int kBatch = 3;                   // tasks per thread whose loads are in flight together (24 floats)
  static_assert(kTasks >= kBuilders, "every builder warp has tasks in its first batch");
  static_assert(!kAhead || kTasks <= kBuilders * kBatch, "kAhead keeps a whole stage in one batch");
  struct BuildState {
    int row, next;                 // this lane's dY row of the current and of the next stage (-1 past n or past the unit)
    float4 v[kBatch][2];           // the current stage's first batch (kAhead: loaded during the previous stage)
  };
  __device__ int dy_row(int kb, int lane) const {
    if (kb >= kb_n) return -1;
    const int r = r0 + kb * kBk + lane;
    const int* __restrict__ map = P.rows[p];
    return r < P.prob[p].n ? (map ? __ldg(map + r) : r) : -1;
  }
  __device__ void load_batch(float4 (&v)[kBatch][2], int row, int t0) const {
    const float* src = row >= 0 ? P.dY[p] + (long long)row * P.lddy[p] : nullptr;
#pragma unroll
    for (int j = 0; j < kBatch; ++j) {
      const int t = t0 + kBuilders * j;
#pragma unroll
      for (int h = 0; h < 2; ++h)
        v[j][h] = t < kTasks && src ? __ldg(reinterpret_cast<const float4*>(src + 8 * t + 4 * h)) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
  __device__ void store_batch(uint8_t* st, const float4 (&v)[kBatch][2], int t0, int lane) const {
    uint8_t* b = st + Cfg::kX + (lane & 3) * 4;
    const int q = lane >> 2;
#pragma unroll
    for (int j = 0; j < kBatch; ++j) {
      const int t = t0 + kBuilders * j;
      if (t >= kTasks) break;
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float4 w = v[j][e >> 2];
        const float x = (e & 3) == 0 ? w.x : (e & 3) == 1 ? w.y : (e & 3) == 2 ? w.z : w.w, hi = tf32_hi(x);
        uint8_t* o = b + (8 * t + e) * 128 + ((q ^ e) & 7) * 16;
        *reinterpret_cast<float*>(o) = hi;
        *reinterpret_cast<float*>(o + Cfg::kB) = x - hi;
      }
    }
  }
  // the unit's first stage: its row and first batch, and the second stage's row
  __device__ void build_begin(BuildState& bs, int bw, int lane) const {
    bs.row = dy_row(0, lane);
    if constexpr (kAhead) {
      load_batch(bs.v, bs.row, bw);
      bs.next = dy_row(1, lane);
    }
  }
  template <class Wait>
  __device__ void build(uint8_t* st, int kb, int bw, int lane, BuildState& bs, Wait wait) const {
    if constexpr (kAhead) {   // one batch is the whole stage
      float4 nv[kBatch][2];
      load_batch(nv, bs.next, bw);                   // stage kb + 1's (zeros past the unit: never stored)
      const int after = dy_row(kb + 2, lane);
      wait();
      store_batch(st, bs.v, bw, lane);
#pragma unroll
      for (int j = 0; j < kBatch; ++j) { bs.v[j][0] = nv[j][0]; bs.v[j][1] = nv[j][1]; }
      bs.next = after;
    } else {
      const int row = bs.row;
      for (int t0 = bw; t0 < kTasks; t0 += kBuilders * kBatch) {
        float4 v[kBatch][2];
        load_batch(v, row, t0);
        if (t0 == bw) {
          bs.row = dy_row(kb + 1, lane);
          wait();
        }
        store_batch(st, v, t0, lane);
      }
    }
  }
  static __device__ void ld_frag(uint32_t (&a)[4], uint32_t sx, int blk, int kk, int warp, int lane) { ld_frag_wgrad(a, sx, blk, kk, warp, lane); }
  // bf16: descriptor of m64 block `blk` (its own box), k16 step kk = rows 16kk .. 16kk + 15 (+2048 bytes)
  static __device__ uint64_t a_desc(uint32_t sx, int blk, int kk) { return gmma_desc_sw128_mn(sx + blk * 8192u + kk * 2048u); }
  __device__ void store(float (&acc)[MB][D / 2], int cw, int warp, int lane) const {   // registers -> partial[item][feature][d]
    const int g = lane >> 2, t = lane & 3;
    float* out = P.partial + (long long)u * Cfg::TM * D;
#pragma unroll
    for (int j = 0; j < MB; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int f = BF16 ? (cw * MB + j) * 64 + warp * 16 + 8 * h + g : wgrad_feature(cw * MB + j, warp, h, g);
        float* o = out + (long long)f * D + 2 * t;
#pragma unroll
        for (int c = 0; c < D / 8; ++c) *reinterpret_cast<float2*>(o + c * 8) = make_float2(acc[j][4 * c + 2 * h], acc[j][4 * c + 2 * h + 1]);
      }
  }
};

template <int D, bool SPLIT, int MB, bool BF16, class Unit, class Params>
__device__ __forceinline__ void proj_pipeline(const Params& P, int total) {
  using Cfg = ProjCfg<D, SPLIT, MB, BF16>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + Cfg::kStages * Cfg::kStage);
  uint64_t* empty = full + Cfg::kStages;
  uint64_t* raw = empty + Cfg::kStages;   // int8 X: the raw q box of the stage has landed
  float* tile_sc = reinterpret_cast<float*>(raw + Cfg::kStages);   // int8 forward: the tile's TM row scales (launch_fwd sizes them)
  const int tid = threadIdx.x, wg = tid >> 7, warp = (tid >> 5) & 3, lane = tid & 31;
  if (tid == 0) {
    // full: the TMA thread's arrive (+ transaction bytes) and, when the kernel builds B or expands int8 X, one arrival per builder warp;
    // empty: one arrival per consumer warp; raw: the TMA thread's arrive (+ the raw q bytes)
    for (int s = 0; s < Cfg::kStages; ++s) { mbar_init(&full[s], 1 + Unit::kBuilders); mbar_init(&empty[s], 8); mbar_init(&raw[s], 1); }
    fence_barrier_init();
  }
  __syncthreads();

  // the CTA holds 384 x 168 registers (launch bounds): a larger split would block the consumers' setmaxnreg.inc for good
  static_assert(128 * Unit::kProducerRegs + 256 * Unit::kConsumerRegs <= 384 * 168, "setmaxnreg split exceeds the CTA's registers");
  if (wg == 0) {   // producer warpgroup: one thread issues every load, across work units; warps 1..3 build B or expand int8 X
    setmaxnreg_dec<Unit::kProducerRegs>();
    if (tid == 0) {
      const uint64_t pol = l2_policy_evict_first();
      int s = 0; uint32_t ph = 0;
      for (int u = blockIdx.x; u < total; u += gridDim.x) {
        const Unit w(P, u);
        for (int kb = 0; kb < w.kb_n; ++kb) {
          mbar_wait(&empty[s], ph ^ 1u);
          mbar_arrive_expect_tx(&full[s], Unit::kTx);
          if constexpr (Unit::kRawTx > 0) mbar_arrive_expect_tx(&raw[s], Unit::kRawTx);
          w.issue(smem + s * Cfg::kStage, &full[s], &raw[s], kb, pol);
          if (++s == Cfg::kStages) { s = 0; ph ^= 1u; }
        }
      }
    }
    if constexpr (Unit::kBuilders > 0) {
      if (warp >= 1) {
        int s = 0; uint32_t ph = 0;
        for (int u = blockIdx.x; u < total; u += gridDim.x) {
          const Unit w(P, u);
          [[maybe_unused]] I8Stage<Unit> cv;
          [[maybe_unused]] typename Unit::BuildState bs;
          if constexpr (Unit::kRawTx == 0) w.build_begin(bs, warp - 1, lane);
          if constexpr (Unit::kRawTx > 0 && Unit::kScalesPerUnit) {
            converters_sync();            // every converter is done with the previous unit's scales
            w.tile_scales(tile_sc, tid - 32);
            converters_sync();
            cv.tile_sc = tile_sc;
          }
          for (int kb = 0; kb < w.kb_n; ++kb) {
            if constexpr (Unit::kRawTx > 0) {
              // the raw box is issued after the stage was released, so its arrival also means the X area is free
              if constexpr (!Unit::kScalesPerUnit) cv.load_scales(w, kb, tid - 32);
              mbar_wait(&raw[s], ph);
              cv.expand(smem + s * Cfg::kStage, tid - 32);
            } else {
              w.build(smem + s * Cfg::kStage, kb, warp - 1, lane, bs, [&] { mbar_wait(&empty[s], ph ^ 1u); });
            }
            fence_proxy_async_smem();   // the generic-proxy stores -> visible to wgmma
            __syncwarp();
            if (lane == 0) mbar_arrive(&full[s]);
            if (++s == Cfg::kStages) { s = 0; ph ^= 1u; }
          }
        }
      }
    }
    return;
  }

  setmaxnreg_inc<Unit::kConsumerRegs>();
  const int cw = wg - 1;   // consumer warpgroup 0 / 1
  int s = 0; uint32_t ph = 0;
  float acc[MB][D / 2];
  for (int u = blockIdx.x; u < total; u += gridDim.x) {
    const Unit w(P, u);
#pragma unroll
    for (int j = 0; j < MB; ++j)
#pragma unroll
      for (int i = 0; i < D / 2; ++i) acc[j][i] = 0.f;
    int prev = -1;
    for (int kb = 0; kb < w.kb_n; ++kb) {
      mbar_wait(&full[s], ph);
      const uint32_t st = smem_u32(smem + s * Cfg::kStage), bh = st + Cfg::kX, bl = bh + Cfg::kB;
      if constexpr (BF16) {
        // X is exact in bf16: A comes straight from the stage by descriptor, B = w0 (or dY^T's first term) [+ w1 + w2], the
        // smallest term first.  One k16 step = one wgmma group; the previous group runs while this one is issued.
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
          wgmma_fence();
#pragma unroll
          for (int j = 0; j < MB; ++j) {
            const uint64_t a = Unit::a_desc(st, cw * MB + j, kk);
            if (SPLIT) {
              WgmmaSSbf16<D, Unit::kTransA>::mma(acc[j], a, gmma_desc_sw128(bl + Cfg::kB + kk * 32u));   // X * w2
              WgmmaSSbf16<D, Unit::kTransA>::mma(acc[j], a, gmma_desc_sw128(bl + kk * 32u));             // X * w1
            }
            WgmmaSSbf16<D, Unit::kTransA>::mma(acc[j], a, gmma_desc_sw128(bh + kk * 32u));               // X * w0
          }
          wgmma_commit();
          wgmma_wait<1>();
          if (kk == 0 && prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);   // the previous stage's last group is done
        }
      } else {
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {   // one k8 step = one wgmma group; the previous group runs while this one is loaded
          uint32_t ah[MB][4], al[MB][4];
#pragma unroll
          for (int j = 0; j < MB; ++j) {
            Unit::ld_frag(ah[j], st, cw * MB + j, kk, warp, lane);
            if (SPLIT)
#pragma unroll
              for (int i = 0; i < 4; ++i) {
                const float x = __uint_as_float(ah[j][i]), hi = tf32_hi(x);
                ah[j][i] = __float_as_uint(hi);
                al[j][i] = __float_as_uint(x - hi);
              }
          }
          wgmma_fence();
          const uint64_t dh = gmma_desc_sw128(bh + kk * 32u);
#pragma unroll
          for (int j = 0; j < MB; ++j) {
            if (SPLIT) {
              WgmmaRS<D>::mma(acc[j], al[j], dh);                               // lo * hi
              WgmmaRS<D>::mma(acc[j], ah[j], gmma_desc_sw128(bl + kk * 32u));   // hi * lo
            }
            WgmmaRS<D>::mma(acc[j], ah[j], dh);                                 // hi * hi
          }
          wgmma_commit();
          wgmma_wait<1>();
          if (kk == 0 && prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);   // the previous stage's last group is done
        }
      }
      prev = s;
      if (++s == Cfg::kStages) { s = 0; ph ^= 1u; }
    }
    wgmma_wait<0>();
    if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
    w.store(acc, cw, warp, lane);
  }
}

template <int D, bool SPLIT, int MB, XType XT>
__global__ void __launch_bounds__(384, 1) proj_fwd_tc_kernel(const __grid_constant__ FwdParams P) {
  constexpr bool BF16 = XT != XType::F32;
  proj_pipeline<D, SPLIT, MB, BF16, FwdUnit<D, SPLIT, MB, BF16, XT == XType::I8>>(P, P.total_tiles);
}

template <int D, bool SPLIT, int MB, XType XT>
__global__ void __launch_bounds__(384, 1) proj_wgrad_tc_kernel(const __grid_constant__ WgParams P) {
  constexpr bool BF16 = XT != XType::F32;
  proj_pipeline<D, SPLIT, MB, BF16, WgUnit<D, SPLIT, MB, BF16, XT == XType::I8>>(P, P.total_items);
}

static int num_sms() {
  static int n[64] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (!n[dev] && cudaDeviceGetAttribute(&n[dev], cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) n[dev] = 132;
  return n[dev];
}

// MB = 2 (256-wide tiles: half the W / dY^T re-reads from L2) where the accumulators fit (d <= 128) and the tiles still fill every SM
static int pick_mb(int d, long long units_at_256) { return d <= 128 && units_at_256 >= num_sms() ? 2 : 1; }

template <int D, bool SPLIT, int MB, XType XT>
static int launch_fwd(const FwdParams& P, cudaStream_t st) {
  using Cfg = ProjCfg<D, SPLIT, MB, XT != XType::F32>;
  constexpr uint32_t smem = Cfg::kSmem + (XT == XType::I8 ? Cfg::TM * 4u : 0u);   // int8: + the converters' tile scales
  static_assert(smem <= kSmemMax, "projection stages and tile scales exceed shared memory");
  LLMREC_CHECK_CUDA(cudaFuncSetAttribute(proj_fwd_tc_kernel<D, SPLIT, MB, XT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int grid = P.total_tiles < num_sms() ? P.total_tiles : num_sms();
  proj_fwd_tc_kernel<D, SPLIT, MB, XT><<<grid, 384, smem, st>>>(P);
  LLMREC_CHECK_LAUNCH("proj_fwd_tc");
  return 0;
}

template <int D, bool SPLIT, int MB, XType XT>
static int launch_wgrad(const WgParams& P, cudaStream_t st) {
  using Cfg = ProjCfg<D, SPLIT, MB, XT != XType::F32>;
  LLMREC_CHECK_CUDA(cudaFuncSetAttribute(proj_wgrad_tc_kernel<D, SPLIT, MB, XT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::kSmem));
  const int grid = P.total_items < num_sms() ? P.total_items : num_sms();
  proj_wgrad_tc_kernel<D, SPLIT, MB, XT><<<grid, 384, Cfg::kSmem, st>>>(P);
  LLMREC_CHECK_LAUNCH("proj_wgrad_tc");
  return 0;
}

// MB = 2 exists for d <= 128 only (its accumulators at d > 128 would not fit next to the fragments)
template <int D, bool SPLIT, XType XT>
static int launch_fwd_mb(const FwdParams& P, int mb, cudaStream_t st) {
  if constexpr (D <= 128) { if (mb == 2) return launch_fwd<D, SPLIT, 2, XT>(P, st); }
  return launch_fwd<D, SPLIT, 1, XT>(P, st);
}
template <int D, bool SPLIT, XType XT>
static int launch_wgrad_mb(const WgParams& P, int mb, cudaStream_t st) {
  if constexpr (D <= 128) { if (mb == 2) return launch_wgrad<D, SPLIT, 2, XT>(P, st); }
  return launch_wgrad<D, SPLIT, 1, XT>(P, st);
}

#define LLMREC_PROJ_WIDTHS(X) X(32) X(64) X(96) X(128) X(160) X(192) X(224) X(256)

static int fwd_launch(const FwdParams& P, bool split, int mb, XType xt, cudaStream_t st) {
  switch (P.d) {
#define LLMREC_CASE(W) case W: \
    if (xt == XType::I8) return split ? launch_fwd_mb<W, true, XType::I8>(P, mb, st) : launch_fwd_mb<W, false, XType::I8>(P, mb, st); \
    if (xt == XType::BF16) return split ? launch_fwd_mb<W, true, XType::BF16>(P, mb, st) : launch_fwd_mb<W, false, XType::BF16>(P, mb, st); \
    return split ? launch_fwd_mb<W, true, XType::F32>(P, mb, st) : launch_fwd_mb<W, false, XType::F32>(P, mb, st);
    LLMREC_PROJ_WIDTHS(LLMREC_CASE)
#undef LLMREC_CASE
  }
  set_error("proj_fwd: no tensor-core kernel for d=%d", P.d);
  return 1;
}

static int wgrad_launch(const WgParams& P, bool split, int mb, XType xt, cudaStream_t st) {
  switch (P.d) {
#define LLMREC_CASE(W) case W: \
    if (xt == XType::I8) return split ? launch_wgrad_mb<W, true, XType::I8>(P, mb, st) : launch_wgrad_mb<W, false, XType::I8>(P, mb, st); \
    if (xt == XType::BF16) return split ? launch_wgrad_mb<W, true, XType::BF16>(P, mb, st) : launch_wgrad_mb<W, false, XType::BF16>(P, mb, st); \
    return split ? launch_wgrad_mb<W, true, XType::F32>(P, mb, st) : launch_wgrad_mb<W, false, XType::F32>(P, mb, st);
    LLMREC_PROJ_WIDTHS(LLMREC_CASE)
#undef LLMREC_CASE
  }
  set_error("proj_wgrad: no tensor-core kernel for d=%d", P.d);
  return 1;
}

// dY -> dY^T ([d x ldt] unsplit in mode 1; the 3xTF32 fp32 kernels build their B in the kernel) for every problem of a grouped
// weight gradient in ONE launch (blockIdx.z): the B operand of the wgrad kernel, K-major (rows of dY contiguous), from strided views.
// BF16 (the bf16-X kernels): dY^T as bf16 terms [w0 ; w1 ; w2] ([3d x ldt], bf16_split3) or [d x ldt] truncated in mode 1.
// rows (optional per problem): column r of dY^T is dY row rows[r], the row that X row r pairs with (the row-mapped weight gradient).
struct DytParams { const float* dY[kMaxProb]; long long ld[kMaxProb]; int n[kMaxProb]; float* out[kMaxProb]; long long ldt[kMaxProb];
                   const int* rows[kMaxProb]; int d, split; };
template <bool BF16>
__global__ void __launch_bounds__(256) dyt_split_kernel(const DytParams P) {
  __shared__ float tile[32][33];
  const int p = blockIdx.z, n = P.n[p], r0 = blockIdx.x * 32, e0 = blockIdx.y * 32;
  if (r0 >= n) return;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const float* __restrict__ src = P.dY[p];
  const int* __restrict__ rows = P.rows[p];
#pragma unroll
  for (int i = ty; i < 32; i += 8) {
    const int r = r0 + i;
    tile[i][tx] = r < n ? __ldg(src + (long long)(rows ? __ldg(rows + r) : r) * P.ld[p] + e0 + tx) : 0.f;
  }
  __syncthreads();
  if (r0 + tx >= n) return;
  const long long ldt = P.ldt[p];
#pragma unroll
  for (int i = ty; i < 32; i += 8) {
    const float v = tile[tx][i];
    const long long at = (long long)(e0 + i) * ldt + r0 + tx;
    if constexpr (BF16) {
      uint16_t* o = reinterpret_cast<uint16_t*>(P.out[p]) + at;
      const long long lo = (long long)P.d * ldt;
      if (P.split) bf16_split3(v, o[0], o[lo], o[2 * lo]);
      else o[0] = bf16_bits(bf16_trunc(v));
    } else {
      P.out[p][at] = v;
    }
  }
}

// W -> [hi ; lo]  ([2d x k], hi exactly TF32-representable); every distinct weight matrix of a grouped launch in ONE launch (blockIdx.y)
struct WsplitParams { const float* W[kMaxProb]; float* out[kMaxProb]; long long n[kMaxProb]; };
__global__ void wsplit_kernel(const WsplitParams P) {
  const float* __restrict__ W = P.W[blockIdx.y];
  float* __restrict__ out = P.out[blockIdx.y];
  const long long n = P.n[blockIdx.y];
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float v = W[i]; const float h = tf32_hi(v); out[i] = h; out[n + i] = v - h;
  }
}
// The bf16-X kernels' B operand: W -> bf16 [w0 ; w1 ; w2] ([3d x k], W = w0 + w1 + w2 exactly) when split, else [d x k] = w0
// (W truncated to bf16).  6dk bytes: fits the 2dk-float wsplit buffer of the fp32 path.
__global__ void wsplit_bf16_kernel(const WsplitParams P, int split) {
  const float* __restrict__ W = P.W[blockIdx.y];
  uint16_t* __restrict__ out = reinterpret_cast<uint16_t*>(P.out[blockIdx.y]);
  const long long n = P.n[blockIdx.y];
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    if (split) bf16_split3(W[i], out[i], out[n + i], out[2 * n + i]);
    else out[i] = bf16_bits(bf16_trunc(W[i]));
  }
}

// dW[dc][f] = sum over (problems sharing this dW, in list order) x (row chunks, in order) of partial[item][f % tm][dc]
// One launch for every output.  Block = (output feature tile, group of feats_per_blk = 64 / (d/4) features): 64 float4
// lanes x 4 source slices; each thread sums every 4th (problem, chunk) source with independent loads in flight, the 4
// slices are combined in a fixed order -> deterministic and latency-tolerant (the naive per-element loop was latency-bound).
// When d/4 does not divide 64 (d = 96, 160, 192, 224) the last 64 - feats_per_blk * d/4 lanes would land on the next
// group's first feature, which that group's block owns: they load and store nothing (a second read-modify-write of the
// same element races under accumulate).
struct ReduceOut { float* dW; int k, n_src, accumulate, blk_start; int src[kMaxProb]; };
struct ReduceParams { ReduceOut out[kMaxProb]; int n_out; int d, tm; const float* partial; WgProblem prob[kMaxProb]; };
__global__ void __launch_bounds__(256) wgrad_reduce_kernel(const ReduceParams R) {
  __shared__ float4 part[4][64];
  int o = 0;
  while (o + 1 < R.n_out && (int)blockIdx.x >= R.out[o + 1].blk_start) ++o;
  const ReduceOut ro = R.out[o];
  const int d = R.d, f4_per_feat = d >> 2;                 // d % 32 == 0 on this path
  const int feats_per_blk = 64 / f4_per_feat;              // 8 at d = 32, 4 at d = 64, 2 at d = 96 / 128, 1 above
  const int local = blockIdx.x - ro.blk_start;
  const int tm = R.tm, groups_per_ft = tm / feats_per_blk;
  const int ft = local / groups_per_ft, fg = local - ft * groups_per_ft;
  const int e = threadIdx.x & 63, sl = threadIdx.x >> 6;
  const bool owned = e < feats_per_blk * f4_per_feat;      // every lane at d = 32, 64, 128, 256
  const int f = fg * feats_per_blk + e / f4_per_feat;      // feature inside the tm-feature tile
  const int dc4 = e - (e / f4_per_feat) * f4_per_feat;     // float4 column
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
  int idx = 0;
  for (int j = 0; owned && j < ro.n_src; ++j) {
    const WgProblem pr = R.prob[ro.src[j]];
#pragma unroll 4
    for (int c = 0; c < pr.chunks; ++c, ++idx) {
      if ((idx & 3) != sl) continue;
      const float4 v = __ldg(reinterpret_cast<const float4*>(R.partial + ((long long)(pr.item_start + c * pr.ft_tiles + ft) * tm + f) * d) + dc4);
      s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
    }
  }
  part[sl][e] = s;
  __syncthreads();
  if (sl == 0 && owned) {
    float4 a = part[0][e], b = part[1][e], c = part[2][e], g = part[3][e];
    float4 t = make_float4((a.x + b.x) + (c.x + g.x), (a.y + b.y) + (c.y + g.y), (a.z + b.z) + (c.z + g.z), (a.w + b.w) + (c.w + g.w));
    const int gf = ft * tm + f;
    if (gf < ro.k) {
      float* p = ro.dW + (long long)(dc4 * 4) * ro.k + gf;
      if (ro.accumulate) { t.x += p[0]; t.y += p[ro.k]; t.z += p[2LL * ro.k]; t.w += p[3LL * ro.k]; }
      p[0] = t.x; p[ro.k] = t.y; p[2LL * ro.k] = t.z; p[3LL * ro.k] = t.w;
    }
  }
}

// db[dc] (+)= sum_r dY[r][dc] : kColsumSlices row-slices per problem -> partial; the LAST block to finish (ticket) combines them in a fixed
// order (deterministic; problems sharing one db -- the 5 attribute matrices behind item_trans -- accumulate in problem order).  One launch.
struct ColsumParams { const float* dY[kMaxProb]; long long ld[kMaxProb]; long long n[kMaxProb]; float* db[kMaxProb]; int acc[kMaxProb]; int d; int n_prob; float* partial; unsigned* ticket; };
constexpr int kColsumSlices = 128;
__global__ void __launch_bounds__(256) colsum_kernel(const ColsumParams P) {
  __shared__ float red[256];
  __shared__ bool s_last;
  const int p = blockIdx.y, b = blockIdx.x, d = P.d;
  const int groups = 256 / d > 0 ? 256 / d : 1;  // d <= 256
  const int g = threadIdx.x / d, c = threadIdx.x - g * d;
  float s = 0.f;
  if (g < groups && P.db[p]) {
#pragma unroll 4
    for (long long r = (long long)b * groups + g; r < P.n[p]; r += (long long)kColsumSlices * groups) s += __ldg(P.dY[p] + r * P.ld[p] + c);
  }
  red[threadIdx.x] = (g < groups) ? s : 0.f;
  __syncthreads();
  if (threadIdx.x < d) {
    float t = 0.f;
    for (int gg = 0; gg < groups; ++gg) t += red[gg * d + threadIdx.x];
    P.partial[((long long)p * kColsumSlices + b) * d + threadIdx.x] = t;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = atomicAdd(P.ticket, 1u) == gridDim.x * gridDim.y - 1;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  for (int q = 0; q < P.n_prob; ++q) {          // problems in order: shared db accumulate deterministically
    if (!P.db[q]) continue;                     // uniform
    float t = 0.f;
    if (g < groups)
      for (int bb = g; bb < kColsumSlices; bb += groups) t += __ldcg(P.partial + ((long long)q * kColsumSlices + bb) * d + c);
    __syncthreads();
    red[threadIdx.x] = (g < groups) ? t : 0.f;
    __syncthreads();
    if (threadIdx.x < d) {
      float u = 0.f;
      for (int gg = 0; gg < groups; ++gg) u += red[gg * d + threadIdx.x];
      float* o = P.db[q] + threadIdx.x;
      *o = P.acc[q] ? (*o + u) : u;
    }
  }
  if (threadIdx.x == 0) *P.ticket = 0u;
}

// ------------------------------------------------------------------------------------------------
// host API (grouped)
// ------------------------------------------------------------------------------------------------
// bf16 X: a 16-byte TMA row pitch needs ldx % 8 == 0, and the bf16 W terms [3d x k] need k % 8 == 0.  int8 X (ldx = the row pitch in
// bytes): k % 16 == 0 and a 16-byte pitch, so that the raw boxes and the row scales are aligned.
bool proj_tc_supported(int d, int64_t ldx, const void* X, int k, bool wgrad, XType xt) {
  (void)wgrad;   // both directions take d in multiples of 32 (wgmma N = d)
  const int q = xt == XType::I8 ? 16 : xt == XType::BF16 ? 8 : 4;
  return d % 32 == 0 && d >= 32 && d <= 256 && ldx % q == 0 && aligned16(X) && k >= 1 && k % q == 0;
}

static CUtensorMapDataType x_type(bool bf16) { return bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32; }

// The X tensor map: fp32 / bf16 boxes with the 128-byte swizzle; int8 boxes of raw q without swizzle, over the k logical columns of the
// rows (the padding and the scale past them are never loaded: columns past k read as zeros)
static bool x_tmap(CUtensorMap* m, XType xt, const void* X, int k, int64_t n, int64_t ldx, uint32_t box_k, uint32_t box_rows) {
  if (xt == XType::I8) return make_tmap_2d(m, CU_TENSOR_MAP_DATA_TYPE_UINT8, X, (uint64_t)k, (uint64_t)n, (uint64_t)ldx, box_k, box_rows, false);
  return make_tmap_2d(m, x_type(xt == XType::BF16), X, (uint64_t)k, (uint64_t)n, (uint64_t)ldx * (xt == XType::BF16 ? 2 : 4), box_k, box_rows);
}

static void set_row_scales(RowScales& xs, int p, XType xt, const void* X, int k, int64_t ldx) {
  xs.scale[p] = xt == XType::I8 ? static_cast<const uint8_t*>(X) + i8_scale_offset(k) : nullptr;
  xs.pitch[p] = xt == XType::I8 ? ldx : 0;
}

// bf16 / int8: pr[p].X holds the address of a bf16 / int8 table (the _bf16 / _i8 problem carried in the fp32 struct's layout)
// rows: NULL, or n_prob optional output row maps (X row r of problem p -> Y row rows[p][r])
int proj_fwd_tc_group(const llmrec_proj_fwd_problem* pr, const int32_t* const* rows, int n_prob, int d, int mode, XType xt, cudaStream_t st) {
  const bool split = (mode == 0), bf16 = xt != XType::F32;    // int8 X runs the bf16 kernels on expanded stages
  const bool need_ws = split || bf16;          // bf16 kernels read W as bf16 terms in both modes
  const int es = bf16 ? 2 : 4, bk = stage_k(bf16);
  FwdParams P;
  memset(&P, 0, sizeof(P));
  P.n_prob = n_prob; P.d = d;
  WsplitParams WS;
  memset(&WS, 0, sizeof(WS));
  int n_ws = 0;
  long long ws_max = 0, tiles256 = 0;
  for (int p = 0; p < n_prob; ++p) tiles256 += (pr[p].n + tile_m(2) - 1) / tile_m(2);
  const int mb = pick_mb(d, tiles256), tm = tile_m(mb);
  int tiles = 0;
  for (int p = 0; p < n_prob; ++p) {
    const float* wsrc = need_ws ? pr[p].wsplit : pr[p].W;
    LLMREC_CHECK_ARG(!need_ws || pr[p].wsplit, "proj_fwd: 3xTF32 mode and bf16 X need a wsplit buffer of 2*d*k floats");
    bool fresh = true;
    for (int q = 0; q < p; ++q) fresh = fresh && !(pr[q].W == pr[p].W && pr[q].wsplit == pr[p].wsplit);
    if (need_ws && fresh) {
      WS.W[n_ws] = pr[p].W; WS.out[n_ws] = pr[p].wsplit; WS.n[n_ws] = (long long)d * pr[p].k;
      ws_max = WS.n[n_ws] > ws_max ? WS.n[n_ws] : ws_max;
      ++n_ws;
    }
    // an empty problem has no tiles (and a tensor map cannot have an empty dimension); its W is still split when a later problem shares it
    if (pr[p].n > 0) {
      const int pieces = split ? (bf16 ? 3 : 2) : 1;
      if (!x_tmap(&P.tmA[p], xt, pr[p].X, pr[p].k, pr[p].n, pr[p].ldx, bk, (uint32_t)tm)) return 4;
      if (!make_tmap_2d(&P.tmW[p], x_type(bf16), wsrc, (uint64_t)pr[p].k, (uint64_t)(pieces * d), (uint64_t)pr[p].k * es, bk, (uint32_t)d)) return 4;
    }
    P.prob[p].n = (int)pr[p].n; P.prob[p].k = pr[p].k; P.prob[p].kblocks = (pr[p].k + bk - 1) / bk;
    P.prob[p].tile_start = tiles; P.prob[p].ldy = pr[p].ldy; P.prob[p].Y = pr[p].Y; P.prob[p].bias = pr[p].bias;
    P.prob[p].rows = rows ? rows[p] : nullptr;
    set_row_scales(P.xs, p, xt, pr[p].X, pr[p].k, pr[p].ldx);
    tiles += (int)((pr[p].n + tm - 1) / tm);
  }
  P.total_tiles = tiles;
  if (n_ws > 0) {
    if (bf16) wsplit_bf16_kernel<<<dim3((unsigned)((ws_max + 255) / 256), n_ws), 256, 0, st>>>(WS, split ? 1 : 0);
    else wsplit_kernel<<<dim3((unsigned)((ws_max + 255) / 256), n_ws), 256, 0, st>>>(WS);
    LLMREC_CHECK_LAUNCH("wsplit");
  }
  if (tiles <= 0) return 0;
  return fwd_launch(P, split, mb, xt, st);
}

static int wg_rows_per_chunk(int64_t n) {
  int r = 2048;                       // rows per work item
  while (r > 256 && n / r < 4) r >>= 1;
  return r;
}

// Work plan of a grouped weight gradient, shared by the scratch query and the launch.  Scratch layout (floats):
//   [colsum ticket: 4] [partials: items x tm x d] [colsum partials: n_prob x kColsumSlices x d] [per problem dY^T: 2 x d x ldt]
// The last region only when `dyt_split` makes B: bf16 X (three bf16 terms, 3 x d x ldt bf16) or mode 1 (d x ldt floats).
struct WgPlan { WgProblem prob[kMaxProb]; int items, mb, tm; int64_t ldt[kMaxProb], dyt[kMaxProb], colsum, total; };
static bool wg_builds_b(int mode, bool bf16) { return mode == 0 && !bf16; }   // WgUnit::kBuilders > 0
static void wg_plan(const llmrec_proj_wgrad_problem* pr, int n_prob, int d, int mode, bool bf16, WgPlan& W) {
  long long items256 = 0;
  for (int p = 0; p < n_prob; ++p) {
    const int rpc = wg_rows_per_chunk(pr[p].n);
    items256 += (long long)((pr[p].k + tile_m(2) - 1) / tile_m(2)) * ((pr[p].n + rpc - 1) / rpc);
  }
  W.mb = pick_mb(d, items256); W.tm = tile_m(W.mb);
  W.items = 0;
  for (int p = 0; p < n_prob; ++p) {
    WgProblem& w = W.prob[p];
    w.n = (int)pr[p].n; w.k = pr[p].k; w.ft_tiles = (pr[p].k + W.tm - 1) / W.tm;
    w.rows_per_chunk = wg_rows_per_chunk(pr[p].n);
    w.chunks = (int)((pr[p].n + w.rows_per_chunk - 1) / w.rows_per_chunk);
    w.item_start = W.items;
    W.items += w.ft_tiles * w.chunks;
  }
  W.colsum = 4 + (int64_t)W.items * W.tm * d;
  int64_t off = W.colsum + (int64_t)n_prob * kColsumSlices * d;
  for (int p = 0; p < n_prob; ++p) {
    W.ldt[p] = bf16 ? (pr[p].n + 7) & ~int64_t(7) : (pr[p].n + 3) & ~int64_t(3);   // TMA row pitch: a multiple of 16 bytes
    W.dyt[p] = off;
    if (!wg_builds_b(mode, bf16)) off += 2 * (int64_t)d * W.ldt[p];
  }
  W.total = off;
}

int64_t proj_wgrad_tc_scratch(const llmrec_proj_wgrad_problem* pr, int n_prob, int d, int mode, XType xt) {
  WgPlan W;
  wg_plan(pr, n_prob, d, mode, xt != XType::F32, W);
  return W.total;   // the colsum ticket must start at zero; the kernel re-zeroes it
}

// bf16 / int8: pr[p].X holds the address of a bf16 / int8 table (the _bf16 / _i8 problem carried in the fp32 struct's layout)
// rows / n_dy: NULL, or per problem an optional dY row map (X row r pairs with dY row rows[p][r]; NULL = identity) and the row count
// of dY (n without a map), over all of which the bias sums run (the map changes only which dY rows the weight gradient reads)
int proj_wgrad_tc_group(const llmrec_proj_wgrad_problem* pr, const int32_t* const* rows, const int64_t* n_dy, int n_prob, int d, int mode,
                        XType xt, float* scratch, int64_t scratch_elems, cudaStream_t st) {
  const bool split = (mode == 0), bf16 = xt != XType::F32;    // int8 X runs the bf16 kernels on expanded stages
  const int es = bf16 ? 2 : 4, bk = stage_k(bf16), pieces = split ? (bf16 ? 3 : 2) : 1;
  const bool build_b = wg_builds_b(mode, bf16);
  WgPlan W;
  wg_plan(pr, n_prob, d, mode, bf16, W);
  LLMREC_CHECK_ARG(scratch && scratch_elems >= W.total, "proj_wgrad: scratch too small (%lld < %lld)", (long long)scratch_elems, (long long)W.total);
  WgParams P;
  memset(&P, 0, sizeof(P));
  P.n_prob = n_prob; P.d = d; P.total_items = W.items;
  P.partial = scratch + 4;                                   // word 0 of the scratch is the colsum ticket (fixed position for every problem set)
  ColsumParams C;
  memset(&C, 0, sizeof(C));
  C.d = d; C.n_prob = n_prob; C.partial = scratch + W.colsum;
  C.ticket = reinterpret_cast<unsigned*>(scratch);
  DytParams T;
  memset(&T, 0, sizeof(T));
  T.d = d; T.split = split ? 1 : 0;
  int64_t n_max = 0;
  for (int p = 0; p < n_prob; ++p) {
    P.prob[p] = W.prob[p];
    const int32_t* map = rows ? rows[p] : nullptr;
    float* dyt = scratch + W.dyt[p];
    // an empty problem has no work items (and a tensor map cannot have an empty dimension); colsum and the reduce still
    // write its dW / db: zeros, or the prior under accumulate
    if (pr[p].n > 0) {
      // boxes [bk rows][bk features] (int8: 64 x 64 bytes of raw q)
      if (!x_tmap(&P.tmX[p], xt, pr[p].X, pr[p].k, pr[p].n, pr[p].ldx, bk, bk)) return 4;
      if (!build_b &&
          !make_tmap_2d(&P.tmG[p], x_type(bf16), dyt, (uint64_t)pr[p].n, (uint64_t)(pieces * d), (uint64_t)W.ldt[p] * es, bk, (uint32_t)d)) return 4;
    }
    P.dY[p] = pr[p].dY; P.lddy[p] = pr[p].lddy; P.rows[p] = map;
    set_row_scales(P.xs, p, xt, pr[p].X, pr[p].k, pr[p].ldx);
    T.dY[p] = pr[p].dY; T.ld[p] = pr[p].lddy; T.n[p] = (int)pr[p].n; T.out[p] = dyt; T.ldt[p] = W.ldt[p]; T.rows[p] = map;
    n_max = pr[p].n > n_max ? pr[p].n : n_max;
    C.dY[p] = pr[p].dY; C.ld[p] = pr[p].lddy; C.n[p] = n_dy ? n_dy[p] : pr[p].n; C.db[p] = pr[p].db;
    C.acc[p] = pr[p].accumulate & LLMREC_WGRAD_ACCUMULATE;
  }
  // The bias gradients depend on dY only: colsum runs as a BRANCH beside the weight-gradient kernel -- fork/join through events, so inside a stream capture it becomes a parallel graph branch.
  // The side stream and the two events are per device, created on first use (never during the call that is being captured in practice:
  // callers run one eager step first); LLMREC_BRANCHES=0 keeps everything on `st`.
  bool any_db = false;
  for (int p = 0; p < n_prob; ++p) any_db = any_db || pr[p].db != nullptr;
  static const bool branches = !(getenv("LLMREC_BRANCHES") && atoi(getenv("LLMREC_BRANCHES")) == 0);
  struct Branch { cudaStream_t side; cudaEvent_t fork, join; };
  static Branch per_device[64] = {};                      // one side stream + event pair per device the process drives
  int dev = 0;
  LLMREC_CHECK_CUDA(cudaGetDevice(&dev));
  LLMREC_CHECK_ARG(dev >= 0 && dev < 64, "proj_wgrad: device ordinal %d out of range", dev);
  cudaStream_t& side = per_device[dev].side;
  cudaEvent_t& ev_fork = per_device[dev].fork;
  cudaEvent_t& ev_join = per_device[dev].join;
  bool forked = false;
  if (any_db) {
    cudaStream_t cs = st;
    if (branches) {
      if (!side) {
        LLMREC_CHECK_CUDA(cudaStreamCreateWithFlags(&side, cudaStreamNonBlocking));
        LLMREC_CHECK_CUDA(cudaEventCreateWithFlags(&ev_fork, cudaEventDisableTiming));
        LLMREC_CHECK_CUDA(cudaEventCreateWithFlags(&ev_join, cudaEventDisableTiming));
      }
      LLMREC_CHECK_CUDA(cudaEventRecord(ev_fork, st));
      LLMREC_CHECK_CUDA(cudaStreamWaitEvent(side, ev_fork, 0));
      cs = side; forked = true;
    }
    colsum_kernel<<<dim3(kColsumSlices, n_prob), 256, 0, cs>>>(C);
    LLMREC_CHECK_LAUNCH("colsum");
    if (forked) LLMREC_CHECK_CUDA(cudaEventRecord(ev_join, side));
  }
  if (W.items > 0) {   // no items: every problem is empty, and only colsum and the reduce run
    if (!build_b) {
      const dim3 grid((unsigned)((n_max + 31) / 32), (unsigned)(d / 32), (unsigned)n_prob);
      if (bf16) dyt_split_kernel<true><<<grid, 256, 0, st>>>(T);
      else dyt_split_kernel<false><<<grid, 256, 0, st>>>(T);
      LLMREC_CHECK_LAUNCH("dyt_split");
    }
    int rc = wgrad_launch(P, split, W.mb, xt, st);
    if (rc) return rc;
  }
  ReduceParams R;
  memset(&R, 0, sizeof(R));
  R.d = d; R.tm = W.tm; R.partial = scratch + 4;
  int blocks = 0;
  for (int p = 0; p < n_prob; ++p) {
    R.prob[p] = P.prob[p];
    int o = -1;
    for (int q = 0; q < R.n_out; ++q) if (R.out[q].dW == pr[p].dW) o = q;
    if (o < 0) {
      o = R.n_out++;
      R.out[o].dW = pr[p].dW; R.out[o].k = pr[p].k; R.out[o].accumulate = pr[p].accumulate & LLMREC_WGRAD_ACCUMULATE; R.out[o].n_src = 0;
    }
    LLMREC_CHECK_ARG(R.out[o].k == pr[p].k, "proj_wgrad: problems sharing dW must share k");
    R.out[o].src[R.out[o].n_src++] = p;
  }
  const int feats_per_blk = 64 / (d / 4);
  for (int o = 0; o < R.n_out; ++o) { R.out[o].blk_start = blocks; blocks += ((R.out[o].k + W.tm - 1) / W.tm) * (W.tm / feats_per_blk); }
  wgrad_reduce_kernel<<<blocks, 256, 0, st>>>(R);
  LLMREC_CHECK_LAUNCH("wgrad_reduce");
  if (forked) LLMREC_CHECK_CUDA(cudaStreamWaitEvent(st, ev_join, 0));
  return 0;
}

}  // namespace llmrec
