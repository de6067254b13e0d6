// Front of the denoiser: token + positional embedding and the first block's timestep-adaptive LayerNorm;
// plus the weight packing (AdaLN (scale, shift) table, 16-bit operands, padded QKV bias) of ldm_create / ldm_load_weights.
//   h  = cat_emb[id] + pos[s]                                   T/models/common/nn_lib.py:204,220 (+ :112-127)
//   x  = LN(h) * (1 + scale_t) + shift_t                        T/models/transformer_utils.py:79-83
// One warp per token row; pad rows (s >= S of each layout's 128 R rows) are written as zeros so that every
// later tile stays finite.
#pragma once
#include "common.cuh"

namespace ldm {

// (scale|shift)[l][t][0..2d) = Linear(SiLU(Embedding[t]))   transformer_utils.py:66-69,80-81.  grid (T, L), block 256
__global__ void adaln_table_kernel(const float* __restrict__ emb /*[L][T][d]*/, const float* __restrict__ w /*[L][2d][d]*/,
                                   const float* __restrict__ b /*[L][2d]*/, float* __restrict__ out /*[L][T][2d]*/, int T, int d) {
  extern __shared__ float se[];
  const int t = blockIdx.x, l = blockIdx.y;
  const float* e = emb + (static_cast<size_t>(l) * T + t) * d;
  for (int i = threadIdx.x; i < d; i += blockDim.x) { const float v = e[i]; se[i] = v / (1.0f + expf(-v)); }
  __syncthreads();
  for (int o = threadIdx.x; o < 2 * d; o += blockDim.x) {
    const float* wr = w + (static_cast<size_t>(l) * 2 * d + o) * d;
    float acc = 0.0f;
    for (int i = 0; i < d; ++i) acc = fmaf(se[i], wr[i], acc);
    out[(static_cast<size_t>(l) * T + t) * 2 * d + o] = acc + b[static_cast<size_t>(l) * 2 * d + o];
  }
}

// fp32 -> 16-bit operand conversion with optional row/col repacking: dst[r][c] = src[src_row(r)][c] for c < src_cols,
// zero elsewhere.  row_map / col_map == nullptr: identity (maps give the source row / column, -1 = zero).  Split mode: dst is the
// hi plane and dst_lo the lo plane of the pair.
template <int MODE>
__global__ void pack_weight_kernel(const float* __restrict__ src, void* __restrict__ dst_, const int* __restrict__ row_map,
                                   const int* __restrict__ col_map, int dst_rows, int dst_cols, int src_cols, void* __restrict__ dst_lo) {
  using O = OpT<MODE>;
  typename O::T* dst = static_cast<typename O::T*>(dst_);
  const size_t n = static_cast<size_t>(dst_rows) * dst_cols;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int r = static_cast<int>(i / dst_cols), c = static_cast<int>(i % dst_cols);
    const int sr = row_map ? row_map[r] : r;
    const int sc = col_map ? col_map[c] : (c < src_cols ? c : -1);
    const float v = (sr >= 0 && sc >= 0) ? src[static_cast<size_t>(sr) * src_cols + sc] : 0.0f;
    if constexpr (kOpSplit<MODE>) O::from_pair(v, dst[i], static_cast<typename O::T*>(dst_lo)[i]);
    else dst[i] = O::from(v);
  }
}

// per-head padded QKV bias: dst[r] = src[row_map[r]] (0 where row_map[r] < 0), except column v_col of every V head (rows
// r >= v_first), which is 1: with its zero weight row it makes the attention kernel's PV MMA deliver the softmax denominator
__global__ void qkv_bias_kernel(const float* __restrict__ src, const int* __restrict__ row_map, float* __restrict__ dst, int n, int v_first,
                                int head_pad, int v_col) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const int sr = row_map[r];
  dst[r] = (r >= v_first && (r - v_first) % head_pad == v_col) ? 1.0f : (sr >= 0 ? src[sr] : 0.0f);
}

// one token row: h = cat_emb[id] + pos[s]; x = LN(h) * (1 + scale_t) + shift_t -> fp32 residual row + 16-bit operand row (whole warp;
// split mode: + the lo plane row in x16_lo)
template <int MODE>
LDM_DEVINL void embed_token_row(const long long id, const int s, const size_t row, const float* __restrict__ cat_emb, const float* __restrict__ pos,
                                const float* __restrict__ adaln /*[2d] of (layer 0, t)*/, float* __restrict__ x32, void* __restrict__ x16_, const int d, const int lane,
                                void* __restrict__ x16_lo = nullptr) {
  using O = OpT<MODE>;
  typename O::T* x16 = static_cast<typename O::T*>(x16_);
  const int nv = d / 4;                      // float4 per row (464 / 4 = 116)
  float4* o32 = reinterpret_cast<float4*>(x32 + row * d);
  uint2* o16 = reinterpret_cast<uint2*>(x16 + row * d);
  const float4* e = reinterpret_cast<const float4*>(cat_emb + static_cast<size_t>(id) * d);
  const float4* p = reinterpret_cast<const float4*>(pos + static_cast<size_t>(s) * d);
  float4 v[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int i = lane + 32 * k;
    if (i < nv) {
      const float4 a = __ldg(e + i), c = __ldg(p + i);
      v[k] = make_float4(a.x + c.x, a.y + c.y, a.z + c.z, a.w + c.w);
    } else {
      v[k] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
  // the row sum is taken of h - h[0]: its terms are of the row's spread, not of its mean, so the mean of a row far from zero
  // comes out correctly rounded too (a plain fp32 sum of 464 values near 256 is off by several ulps of the mean, which every
  // output of the row inherits)
  const float piv = __shfl_sync(0xffffffffu, v[0].x, 0);
  float sum = 0.0f;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    if (lane + 32 * k < nv) sum += ((v[k].x - piv) + (v[k].y - piv)) + ((v[k].z - piv) + (v[k].w - piv));
  }
  const float mean = piv + warp_sum(sum) / d;
  float var = 0.0f;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    if (lane + 32 * k < nv) {
      const float a = v[k].x - mean, b2 = v[k].y - mean, c = v[k].z - mean, e2 = v[k].w - mean;
      var += (a * a + b2 * b2) + (c * c + e2 * e2);
    }
  }
  const float rstd = 1.0f / sqrtf(warp_sum(var) / d + 1e-5f);
  const float4* sc = reinterpret_cast<const float4*>(adaln);
  const float4* sh = reinterpret_cast<const float4*>(adaln + d);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int i = lane + 32 * k;
    if (i < nv) {
      const float4 g = __ldg(sc + i), h = __ldg(sh + i);
      float4 r;
      r.x = (v[k].x - mean) * rstd * (1.0f + g.x) + h.x;
      r.y = (v[k].y - mean) * rstd * (1.0f + g.y) + h.y;
      r.z = (v[k].z - mean) * rstd * (1.0f + g.z) + h.z;
      r.w = (v[k].w - mean) * rstd * (1.0f + g.w) + h.w;
      o32[i] = r;
      if constexpr (kOpSplit<MODE>) {
        uint2 hi, lo;
        O::pack_pair(r.x, r.y, hi.x, lo.x);
        O::pack_pair(r.z, r.w, hi.y, lo.y);
        o16[i] = hi;
        reinterpret_cast<uint2*>(static_cast<typename O::T*>(x16_lo) + row * d)[i] = lo;
      } else {
        o16[i] = make_uint2(O::pack(r.x, r.y), O::pack(r.z, r.w));
      }
    }
  }
}

// NORM = false (instance-norm blocks): the token rows get the raw h = cat_emb[id] + pos[s] in x32 only, which
// instance_norm_kernel then normalises over the layout's tokens; pad rows as with NORM
template <int MODE, bool NORM = true>
__global__ void __launch_bounds__(256)
embed_adaln_kernel(const long long* __restrict__ ids /*[B][S]*/, const float* __restrict__ cat_emb /*[C][d]*/,
                   const float* __restrict__ pos /*[S][d]*/, const float* __restrict__ adaln_tab /*[T][2d] of layer 0*/, int t_model,
                   const int* __restrict__ t_layout /*[n_layouts] per-layout timesteps (training-side calls) or nullptr*/,
                   float* __restrict__ x32 /*[B*128R][d]*/, void* __restrict__ x16_, int n_layouts, int rows_log2 /*log2(128 R)*/, int S, int d,
                   void* __restrict__ x16_lo /*split mode: lo plane of x16*/) {
  using O = OpT<MODE>;
  typename O::T* x16 = static_cast<typename O::T*>(x16_);
  const int warp_global = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp_global >= (n_layouts << rows_log2)) return;
  pdl_sync();                                // ids come from the previous step's draw; x32 / x16 may still be read by it
  const int b = warp_global >> rows_log2, s = warp_global & ((1 << rows_log2) - 1);
  const size_t row = static_cast<size_t>(warp_global);
  if (s >= S) {                        // padding rows
    const int nv = d / 4;
    float4* o32 = reinterpret_cast<float4*>(x32 + row * d);
    uint2* o16 = reinterpret_cast<uint2*>(x16 + row * d);
    for (int i = lane; i < nv; i += 32) { o32[i] = make_float4(0.f, 0.f, 0.f, 0.f); o16[i] = make_uint2(0u, 0u); }
    if constexpr (kOpSplit<MODE>) {
      uint2* l16 = reinterpret_cast<uint2*>(static_cast<typename O::T*>(x16_lo) + row * d);
      for (int i = lane; i < nv; i += 32) l16[i] = make_uint2(0u, 0u);
    }
    return;
  }
  const long long id = ids[static_cast<size_t>(b) * S + s];
  if constexpr (NORM) {
    const float* adaln = adaln_tab + static_cast<size_t>(t_layout != nullptr ? __ldg(t_layout + b) : t_model) * 2 * d;
    embed_token_row<MODE>(id, s, row, cat_emb, pos, adaln, x32, x16_, d, lane, x16_lo);
  } else {
    const float4* e = reinterpret_cast<const float4*>(cat_emb + static_cast<size_t>(id) * d);
    const float4* p = reinterpret_cast<const float4*>(pos + static_cast<size_t>(s) * d);
    float4* o32 = reinterpret_cast<float4*>(x32 + row * d);
    for (int i = lane; i < d / 4; i += 32) {
      const float4 a = __ldg(e + i), c = __ldg(p + i);
      o32[i] = make_float4(a.x + c.x, a.y + c.y, a.z + c.z, a.w + c.w);
    }
  }
}

// norm1 of the instance-norm blocks (AdaInsNorm, transformer_utils.py:86-100): x = InstanceNorm1d(h) * (1 + scale_t) + shift_t,
// the statistics per layout and channel over the layout's S token rows (mean and biased variance, eps 1e-5, no affine), in place
// on the fp32 rows x32 (the raw embedding or FF2's pre-norm sum) -> x32 and the 16-bit operand rows (split mode: + the lo plane).
// grid (d / (4 kInCols4), n_layouts); a block holds kInCols4 float4 columns of one layout in 8 R row slices, thread (slice, col)
// rows slice, slice + 8 R, .. < S in registers (at most kInRows): one read of the rows, and the variance is taken about the mean.
// The sums run over h - h[row 0] (offset invariance, as in the LayerNorm epilogues).  Pad rows (s >= S) are neither read nor
// written: after the fused embedding of the draw kernels they may hold stale values, and the GEMMs keep them finite.
// The row stride is the compile-time kInD, so a thread's rows are immediate offsets of one address.
constexpr int kInD = 464, kInCols4 = 29, kInRows = 16;
static_assert(kInD % (4 * kInCols4) == 0, "whole column blocks");
template <int MODE, int R>
__global__ void __launch_bounds__(kInCols4 * 8 * R)
instance_norm_kernel(float* __restrict__ x32 /*[B*128R][kInD]*/, void* __restrict__ x16_, void* __restrict__ x16_lo,
                     const float* __restrict__ adaln_tab /*[T][2 kInD] of the layer*/, int t_model,
                     const int* __restrict__ t_layout /*[n_layouts] per-layout timesteps (training-side calls) or nullptr*/, int S) {
  using O = OpT<MODE>;
  constexpr int d = kInD;
  constexpr int kSlices = 8 * R;
  static_assert(kSlices * kInRows >= 128 * R, "a thread's registers cover its slice of the layout's rows");
  __shared__ float4 red[kSlices][kInCols4];
  const int col = threadIdx.x % kInCols4, slice = threadIdx.x / kInCols4, b = blockIdx.y;
  const int c = (blockIdx.x * kInCols4 + col) * 4;
  const size_t row0 = static_cast<size_t>(b) * 128 * R;
  pdl_sync();                                  // x32 comes from the previous kernel
  const float4 piv = *reinterpret_cast<const float4*>(x32 + row0 * d + c);
  float4 v[kInRows];
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int k = 0; k < kInRows; ++k) {
    const int s = slice + k * kSlices;
    if (s < S) {
      v[k] = *reinterpret_cast<const float4*>(x32 + (row0 + s) * d + c);
      acc.x += v[k].x - piv.x; acc.y += v[k].y - piv.y; acc.z += v[k].z - piv.z; acc.w += v[k].w - piv.w;
    }
  }
  // the slices' partial sums, added in slice order by every thread of the column
  const auto column_total = [&](float4 part) {
    red[slice][col] = part;
    __syncthreads();
    float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int i = 0; i < kSlices; ++i) { const float4 r = red[i][col]; t.x += r.x; t.y += r.y; t.z += r.z; t.w += r.w; }
    __syncthreads();
    return t;
  };
  const float inv_s = 1.0f / static_cast<float>(S);
  const float4 sum = column_total(acc);
  const float4 mean = make_float4(piv.x + sum.x * inv_s, piv.y + sum.y * inv_s, piv.z + sum.z * inv_s, piv.w + sum.w * inv_s);
  acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int k = 0; k < kInRows; ++k) {
    if (slice + k * kSlices < S) {
      const float a = v[k].x - mean.x, e = v[k].y - mean.y, f = v[k].z - mean.z, g = v[k].w - mean.w;
      acc.x = fmaf(a, a, acc.x); acc.y = fmaf(e, e, acc.y); acc.z = fmaf(f, f, acc.z); acc.w = fmaf(g, g, acc.w);
    }
  }
  const float4 q = column_total(acc);
  const float4 rstd = make_float4(1.0f / sqrtf(q.x * inv_s + 1e-5f), 1.0f / sqrtf(q.y * inv_s + 1e-5f), 1.0f / sqrtf(q.z * inv_s + 1e-5f),
                                  1.0f / sqrtf(q.w * inv_s + 1e-5f));
  const float* tab = adaln_tab + static_cast<size_t>(t_layout != nullptr ? __ldg(t_layout + b) : t_model) * 2 * d;
  const float4 g = __ldg(reinterpret_cast<const float4*>(tab + c)), sh = __ldg(reinterpret_cast<const float4*>(tab + d + c));
  typename O::T* x16 = static_cast<typename O::T*>(x16_);
#pragma unroll
  for (int k = 0; k < kInRows; ++k) {
    const int s = slice + k * kSlices;
    if (s < S) {
      const size_t off = (row0 + s) * d + c;
      float4 r;
      r.x = (v[k].x - mean.x) * rstd.x * (1.0f + g.x) + sh.x;
      r.y = (v[k].y - mean.y) * rstd.y * (1.0f + g.y) + sh.y;
      r.z = (v[k].z - mean.z) * rstd.z * (1.0f + g.z) + sh.z;
      r.w = (v[k].w - mean.w) * rstd.w * (1.0f + g.w) + sh.w;
      *reinterpret_cast<float4*>(x32 + off) = r;
      if constexpr (kOpSplit<MODE>) {
        uint2 hi, lo;
        O::pack_pair(r.x, r.y, hi.x, lo.x);
        O::pack_pair(r.z, r.w, hi.y, lo.y);
        *reinterpret_cast<uint2*>(x16 + off) = hi;
        *reinterpret_cast<uint2*>(static_cast<typename O::T*>(x16_lo) + off) = lo;
      } else {
        *reinterpret_cast<uint2*>(x16 + off) = make_uint2(O::pack(r.x, r.y), O::pack(r.z, r.w));
      }
    }
  }
}

}  // namespace ldm
