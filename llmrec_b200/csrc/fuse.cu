// Embedding fusion (Models.py:185-197) and its backward.
//   out = mean(layer_0..layer_L) + sum_t coef[t] * x_t / max(||x_t||_2, 1e-12)
// One (sub-)warp per row; every operand row is read once from HBM (the second touch of a side row
// hits L1), the ~40 ATen elementwise/reduction kernels of the reference collapse into one pass.
#include "common.cuh"

namespace llmrec {

constexpr int kMaxLayers = 8;
constexpr int kMaxSides = 16;
constexpr float kNormEps = 1e-12f;  // F.normalize default eps

struct FuseParams {
  const float* layers[kMaxLayers]; int64_t ld_layers[kMaxLayers]; int n_layers;
  const float* sides[kMaxSides]; int64_t ld_sides[kMaxSides]; float coef[kMaxSides]; int n_sides;
  float* dsides[kMaxSides]; int64_t ld_dsides[kMaxSides];
  float* out; int64_t ldo;           // fwd: out; bwd: d_layer (may be null)
  const float* g; int64_t ldg;       // bwd only
  const int* rows; int64_t n; int d; int accumulate;
  int compact;                       // fwd only: layers are read at rows[item], sides and out at the compact position `item`
  const int* n_dev;                  // row-list form with a device-side length: items [0, min(*n_dev, n)) of `rows`; the grid covers n
};

// Number of rows of this launch: n, or the device-side list length capped at n (the grid is sized for n).
__device__ __forceinline__ int64_t live_rows(const FuseParams& p) {
  if (!p.n_dev) return p.n;
  const int64_t c = __ldg(p.n_dev);
  return c < p.n ? c : p.n;
}

template <int LPR>
__device__ __forceinline__ float grp_sum(float v) {
#pragma unroll
  for (int o = LPR / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

template <int LPR, bool VEC>
__global__ void __launch_bounds__(256) fuse_fwd_kernel(const FuseParams p) {
  constexpr int RPW = 32 / LPR;
  __shared__ float sc[8][RPW][kMaxSides];
  const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31, sub = lane / LPR, li = lane % LPR;
  const int64_t item = ((int64_t)blockIdx.x * 8 + wib) * RPW + sub;
  const bool in_range = item < live_rows(p);
  const int64_t lrow = in_range ? (p.rows ? (int64_t)p.rows[item] : item) : 0;
  const bool valid = in_range && lrow >= 0;          // a negative list entry = "not mine": compact output row of zeros, nothing read
  const int64_t row = valid ? lrow : 0;
  const int64_t srow = (p.compact && in_range) ? item : row;
  const int nq = VEC ? p.d / 4 : p.d;
  for (int t = 0; t < p.n_sides; ++t) {
    const float* x = p.sides[t] + srow * p.ld_sides[t];
    float ss = 0.f;
    if (valid) {
      for (int q = li; q < nq; q += LPR) {
        if (VEC) { float4 v = ldg4(x + q * 4); ss += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w; }
        else { float v = x[q]; ss = fmaf(v, v, ss); }
      }
    }
    ss = grp_sum<LPR>(ss);
    if (li == 0) sc[wib][sub][t] = p.coef[t] / fmaxf(sqrtf(ss), kNormEps);
  }
  __syncwarp();
  if (!valid) {
    if (p.compact && in_range) {
      float* z = p.out + srow * p.ldo;
      for (int q = li; q < nq; q += LPR) { if (VEC) st4(z + q * 4, make_float4(0.f, 0.f, 0.f, 0.f)); else z[q] = 0.f; }
    }
    return;
  }
  const float inv_l = 1.0f / (float)p.n_layers;
  float* o = p.out + srow * p.ldo;
  for (int q = li; q < nq; q += LPR) {
    if (VEC) {
      float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int l = 0; l < p.n_layers; ++l) {
        float4 v = ldg4(p.layers[l] + row * p.ld_layers[l] + q * 4);
        a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
      }
      a.x *= inv_l; a.y *= inv_l; a.z *= inv_l; a.w *= inv_l;
      for (int t = 0; t < p.n_sides; ++t) fma4(a, sc[wib][sub][t], ldg4(p.sides[t] + srow * p.ld_sides[t] + q * 4));
      st4(o + q * 4, a);
    } else {
      float a = 0.f;
      for (int l = 0; l < p.n_layers; ++l) a += p.layers[l][row * p.ld_layers[l] + q];
      a *= inv_l;
      for (int t = 0; t < p.n_sides; ++t) a = fmaf(sc[wib][sub][t], p.sides[t][srow * p.ld_sides[t] + q], a);
      o[q] = a;
    }
  }
}

template <int LPR, bool VEC>
__global__ void __launch_bounds__(256) fuse_bwd_kernel(const FuseParams p) {
  constexpr int RPW = 32 / LPR;
  __shared__ float sa[8][RPW][kMaxSides];
  __shared__ float sb[8][RPW][kMaxSides];
  const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31, sub = lane / LPR, li = lane % LPR;
  const int64_t item = ((int64_t)blockIdx.x * 8 + wib) * RPW + sub;
  const bool in_range = item < live_rows(p);
  const int64_t lrow = in_range ? (p.rows ? (int64_t)p.rows[item] : item) : 0;
  const bool valid = in_range && lrow >= 0;          // a negative list entry = "not mine", as in the forward: nothing read or written
  const int64_t row = valid ? lrow : 0;
  const int nq = VEC ? p.d / 4 : p.d;
  const float* g = p.g + row * p.ldg;
  for (int t = 0; t < p.n_sides; ++t) {
    const float* x = p.sides[t] + row * p.ld_sides[t];
    float ss = 0.f, dt = 0.f;
    if (valid) {
      for (int q = li; q < nq; q += LPR) {
        if (VEC) {
          float4 v = ldg4(x + q * 4), gv = ldg4(g + q * 4);
          ss += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
          dt += v.x * gv.x + v.y * gv.y + v.z * gv.z + v.w * gv.w;
        } else { float v = x[q]; ss = fmaf(v, v, ss); dt = fmaf(v, g[q], dt); }
      }
    }
    ss = grp_sum<LPR>(ss);
    dt = grp_sum<LPR>(dt);
    if (li == 0) {
      float nrm = sqrtf(ss);
      if (nrm > kNormEps) { sa[wib][sub][t] = p.coef[t] / nrm; sb[wib][sub][t] = dt / (nrm * nrm); }
      else { sa[wib][sub][t] = p.coef[t] / kNormEps; sb[wib][sub][t] = 0.f; }  // clamped branch: y = x/eps
    }
  }
  __syncwarp();
  if (!valid) return;
  const float inv_l = 1.0f / (float)p.n_layers;
  for (int q = li; q < nq; q += LPR) {
    if (VEC) {
      float4 gv = ldg4(g + q * 4);
      if (p.out) st4(p.out + row * p.ldo + q * 4, make_float4(gv.x * inv_l, gv.y * inv_l, gv.z * inv_l, gv.w * inv_l));
      for (int t = 0; t < p.n_sides; ++t) {
        if (!p.dsides[t]) continue;
        float a = sa[wib][sub][t], b = sb[wib][sub][t];
        float4 x = ldg4(p.sides[t] + row * p.ld_sides[t] + q * 4);
        float4 r = make_float4(a * (gv.x - b * x.x), a * (gv.y - b * x.y), a * (gv.z - b * x.z), a * (gv.w - b * x.w));
        float* dp = p.dsides[t] + row * p.ld_dsides[t] + q * 4;
        if (p.accumulate) { float4 o = *reinterpret_cast<const float4*>(dp); r.x += o.x; r.y += o.y; r.z += o.z; r.w += o.w; }
        st4(dp, r);
      }
    } else {
      float gv = g[q];
      if (p.out) p.out[row * p.ldo + q] = gv * inv_l;
      for (int t = 0; t < p.n_sides; ++t) {
        if (!p.dsides[t]) continue;
        float r = sa[wib][sub][t] * (gv - sb[wib][sub][t] * p.sides[t][row * p.ld_sides[t] + q]);
        float* dp = p.dsides[t] + row * p.ld_dsides[t] + q;
        *dp = p.accumulate ? (*dp + r) : r;
      }
    }
  }
}

template <bool BWD>
static int launch_fuse(const FuseParams& p, bool vec, cudaStream_t st) {
  if (p.n <= 0) return 0;
  int nq = vec ? p.d / 4 : p.d;
  int lpr = nq <= 8 ? 8 : (nq <= 16 ? 16 : 32);
  int rpw = 32 / lpr;
  unsigned blocks = (unsigned)((p.n + 8 * rpw - 1) / (8 * rpw));
#define LF(L, V)                                                             \
  if (BWD) fuse_bwd_kernel<L, V><<<blocks, 256, 0, st>>>(p);               \
  else fuse_fwd_kernel<L, V><<<blocks, 256, 0, st>>>(p)
  if (vec) { if (lpr == 8) { LF(8, true); } else if (lpr == 16) { LF(16, true); } else { LF(32, true); } }
  else { if (lpr == 8) { LF(8, false); } else if (lpr == 16) { LF(16, false); } else { LF(32, false); } }
#undef LF
  LLMREC_CHECK_LAUNCH(BWD ? "fuse_bwd" : "fuse_fwd");
  return 0;
}

static int fuse_fwd(const float* const* layers, const int64_t* ld_layers, int32_t n_layers, const float* const* sides,
                    const int64_t* ld_sides, const float* coef, int32_t n_sides, float* out, int64_t ldo, const int32_t* rows,
                    const int32_t* n_dev, int64_t n, int32_t d, cudaStream_t st) {
  LLMREC_REQUIRE_DEVICE();
  LLMREC_CHECK_ARG(n_layers >= 1 && n_layers <= kMaxLayers && n_sides >= 0 && n_sides <= kMaxSides,
                   "fuse_fwd: n_layers=%d n_sides=%d out of range", n_layers, n_sides);
  FuseParams p{};
  bool vec = d % 4 == 0 && aligned16(out) && ldo % 4 == 0;
  p.n_layers = n_layers; p.n_sides = n_sides;
  for (int l = 0; l < n_layers; ++l) { p.layers[l] = layers[l]; p.ld_layers[l] = ld_layers[l]; vec = vec && aligned16(layers[l]) && ld_layers[l] % 4 == 0; }
  for (int t = 0; t < n_sides; ++t) { p.sides[t] = sides[t]; p.ld_sides[t] = ld_sides[t]; p.coef[t] = coef[t]; vec = vec && aligned16(sides[t]) && ld_sides[t] % 4 == 0; }
  p.out = out; p.ldo = ldo; p.rows = rows; p.n = n < 0 ? -n : n; p.d = d; p.n_dev = n_dev;
  p.compact = (n < 0 && rows) ? 1 : 0;
  return launch_fuse<false>(p, vec, st);
}

static int fuse_bwd(const float* g, int64_t ldg, int32_t n_layers, float* d_layer, int64_t lddl, const float* const* sides,
                    const int64_t* ld_sides, const float* coef, float* const* d_sides, const int64_t* ld_dsides, int32_t n_sides,
                    int32_t accumulate, const int32_t* rows, const int32_t* n_dev, int64_t n, int32_t d, cudaStream_t st) {
  LLMREC_REQUIRE_DEVICE();
  LLMREC_CHECK_ARG(n_layers >= 1 && n_sides >= 0 && n_sides <= kMaxSides, "fuse_bwd: n_layers=%d n_sides=%d out of range", n_layers, n_sides);
  FuseParams p{};
  bool vec = d % 4 == 0 && aligned16(g) && ldg % 4 == 0 && (!d_layer || (aligned16(d_layer) && lddl % 4 == 0));
  p.n_layers = n_layers; p.n_sides = n_sides;
  for (int t = 0; t < n_sides; ++t) {
    p.sides[t] = sides[t]; p.ld_sides[t] = ld_sides[t]; p.coef[t] = coef[t];
    p.dsides[t] = d_sides[t]; p.ld_dsides[t] = ld_dsides[t];
    vec = vec && aligned16(sides[t]) && ld_sides[t] % 4 == 0 && (!d_sides[t] || (aligned16(d_sides[t]) && ld_dsides[t] % 4 == 0));
  }
  p.out = d_layer; p.ldo = lddl; p.g = g; p.ldg = ldg; p.rows = rows; p.n = n; p.d = d; p.accumulate = accumulate; p.n_dev = n_dev;
  return launch_fuse<true>(p, vec, st);
}
}  // namespace llmrec

using namespace llmrec;

extern "C" int llmrec_fuse_fwd_f32(const float* const* layers, const int64_t* ld_layers, int32_t n_layers,
                                   const float* const* sides, const int64_t* ld_sides, const float* coef,
                                   int32_t n_sides, float* out, int64_t ldo, const int32_t* rows, int64_t n, int32_t d,
                                   llmrec_stream_t stream) {
  return fuse_fwd(layers, ld_layers, n_layers, sides, ld_sides, coef, n_sides, out, ldo, rows, nullptr, n, d, as_stream(stream));
}

extern "C" int llmrec_fuse_bwd_f32(const float* g, int64_t ldg, int32_t n_layers, float* d_layer, int64_t lddl,
                                   const float* const* sides, const int64_t* ld_sides, const float* coef,
                                   float* const* d_sides, const int64_t* ld_dsides, int32_t n_sides,
                                   int32_t accumulate, const int32_t* rows, int64_t n, int32_t d, llmrec_stream_t stream) {
  return fuse_bwd(g, ldg, n_layers, d_layer, lddl, sides, ld_sides, coef, d_sides, ld_dsides, n_sides, accumulate, rows, nullptr, n, d,
                  as_stream(stream));
}

extern "C" int llmrec_fuse_fwd_rows_f32(const float* const* layers, const int64_t* ld_layers, int32_t n_layers,
                                        const float* const* sides, const int64_t* ld_sides, const float* coef,
                                        int32_t n_sides, float* out, int64_t ldo, const int32_t* rows, const int32_t* n_rows_dev,
                                        int32_t max_rows, int32_t d, llmrec_stream_t stream) {
  LLMREC_CHECK_ARG(rows && n_rows_dev && max_rows >= 0, "fuse_fwd_rows: a row list and its device-side length are required");
  return fuse_fwd(layers, ld_layers, n_layers, sides, ld_sides, coef, n_sides, out, ldo, rows, n_rows_dev, max_rows, d, as_stream(stream));
}

extern "C" int llmrec_fuse_bwd_rows_f32(const float* g, int64_t ldg, int32_t n_layers, float* d_layer, int64_t lddl,
                                        const float* const* sides, const int64_t* ld_sides, const float* coef,
                                        float* const* d_sides, const int64_t* ld_dsides, int32_t n_sides, int32_t accumulate,
                                        const int32_t* rows, const int32_t* n_rows_dev, int32_t max_rows, int32_t d, llmrec_stream_t stream) {
  LLMREC_CHECK_ARG(rows && n_rows_dev && max_rows >= 0, "fuse_bwd_rows: a row list and its device-side length are required");
  return fuse_bwd(g, ldg, n_layers, d_layer, lddl, sides, ld_sides, coef, d_sides, ld_dsides, n_sides, accumulate, rows, n_rows_dev, max_rows,
                  d, as_stream(stream));
}
