// Per-(layout, head, query tile) self-attention of the LayoutDM denoiser on wgmma: O = softmax(Q K^T) V, S <= 256 keys,
// head_dim 58.  (nn.MultiheadAttention inside Block._sa_block, T/models/transformer_utils.py:140-142,191-205; no masks.)
//
// A layout holds R = ceil(S / 128) row tiles of 128 rows (R in {1, 2}); rows S .. 128 R - 1 are pad rows, which no key reads.
// Input  qkv [M][1536] 16-bit, M = 128 R n_layouts, per-head column blocks padded 58 -> 64 with zeros:
//        Q_h = cols [h*64, h*64+64), K_h = 512 + ..., V_h = 1024 + ... ; Q is already scaled by 1/sqrt(58); column 58 of
//        every V_h is 1.0 (zero weight row, bias 1), which makes the PV MMA deliver the softmax denominator.
// Output att [M][512] 16-bit, head h in cols [h*64, h*64+64) (col 58 of every head is 1 = the normalised ones column, cols
//        59..63 are zeros; the out-projection weight is packed with zero columns there) = A operand of the out-projection.
//
// One CTA per (layout, head, query tile) work item, 256 threads = two warpgroups of 64 query rows each.  Thread 0 issues the
// TMA loads of the Q tile and the layout's R K and V tiles (128 x 64 each, 128B swizzle; the R tiles of K, and of V, sit back
// to back, so they read as one 128 R-row operand).  R = 1: several CTAs per SM overlap one item's loads with another's math.
//   S[64 x 128R] = Q K^T   wgmma, A = Q rows of the warpgroup, B = K tile t (both K-major, shared memory), fp32 in registers
//   exact softmax in registers over every valid key of all R tiles (a row lives in the quad of lanes that shares it); the
//   probabilities stay un-normalised, are rounded to the operand dtype and become, one 128-key chunk at a time, the register
//   A operand of
//   O[64x64]  = P V     wgmma, B = V as loaded ([key][d] rows = MN-major operand), 8 R k16 steps in key order
//   O is normalised by its ones column (the row sum of the rounded P) and stored.
// The chunks of P V accumulate into one O in the order of the keys, so the sum is the one a single pass would form; R = 2
// only bounds the registers the converted P holds.  No online (rescaling) softmax: the maximum is taken over all keys first.
// Split mode (OP_BF16X3): Q / K / V arrive as bf16 (hi, lo) plane pairs (the hi tiles, then the lo tiles).  Q K^T is three
// products per k-step (q_lo k_hi + q_hi k_lo + q_hi k_hi); the un-normalised P is split in registers into (P_hi, P_lo), and P V
// is three register-A wgmmas per k-step (P_lo V_hi + P_hi V_lo + P_hi V_hi).  V's ones column is 1 + 0, so the ones column
// of O is the row sum of P_hi + P_lo.  O is divided by it (one rounding, and x / x = 1 exactly, so column 58 of the pair is
// exactly 1 + 0; the reciprocal product of the 16-bit modes can land one fp32 ulp below 1).  The output is a pair (att, att_lo).
#pragma once
#include "common.cuh"

namespace ldm {

constexpr int kAttThreads = 256;
constexpr int kAttTile = 128 * 128;                 // one 128 x 64 16-bit tile = 16 KB
constexpr int kAttOnesCol = 58;                     // head_dim: V column that holds 1.0
constexpr int kAttOut = 8 * 64;                     // att row length
constexpr int kAttMaxR = 2;                         // row tiles per layout: S <= 256 (the exact softmax holds 64 x 256 scores)

// shared memory of the R-tile instantiation: Q | K_0 .. K_{R-1} | V_0 .. V_{R-1} per plane (split mode: the hi plane's tiles,
// then the lo plane's), then the barrier
template <int R, bool SPLIT>
struct AttSmem {
  static constexpr int kOffQ = 0, kOffK = kAttTile, kOffV = (1 + R) * kAttTile;
  static constexpr int kPlane = (1 + 2 * R) * kAttTile;
  static constexpr int kOffLo = kPlane;                            // split mode: the lo plane's tiles
  static constexpr int kOffBar = (SPLIT ? 2 : 1) * kPlane;
  static constexpr int kBytes = kOffBar + 64 + 1024;               // + alignment slack
};

// R = 1: two CTAs per SM (64 score registers per thread).  R = 2: 128 score registers per thread, one CTA per SM.
template <int MODE, int R>
__global__ void __launch_bounds__(kAttThreads, R == 1 ? 2 : 1)
attention_kernel(const __grid_constant__ OpMaps<MODE> map_qkv /*[M][1536], box 64 x 128*/, void* att /*[M][512]*/,
                 int n_valid /*S*/, int n_heads /*8*/, int n_layouts,
                 int rev /*1: walk the items from the last to the first (L2 reuse, see GemmParams::rev)*/,
                 void* att_lo /*split mode: lo plane of att*/) {
  static_assert(R >= 1 && R <= kAttMaxR, "one or two row tiles per layout");
  constexpr bool BF16 = kOpBf16<MODE>, SPLIT = kOpSplit<MODE>;
  using O = OpT<MODE>;
  using SM = AttSmem<R, SPLIT>;
  extern __shared__ uint8_t att_smem_raw[];
  uint8_t* smem = smem_align1024(att_smem_raw);
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + SM::kOffBar);

  // item = (layout * R + query tile) * n_heads + head; the R query tiles and n_heads heads of a layout are neighbours
  const int n_items = n_layouts * R * n_heads;
  const int item = rev ? n_items - 1 - static_cast<int>(blockIdx.x) : static_cast<int>(blockIdx.x);
  const int h = item % n_heads, qt = (item / n_heads) % R, layout = item / (n_heads * R);
  const int krow0 = layout * (128 * R), row0 = krow0 + qt * 128;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&map_qkv.hi);
    if constexpr (SPLIT) tma_prefetch_desc(&map_qkv.lo);
    mbar_init(bar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  pdl_sync();
  if (threadIdx.x == 0) {
    mbar_arrive_expect_tx(bar, (SPLIT ? 2 : 1) * (1 + 2 * R) * kAttTile);
    tma_load_2d(smem + SM::kOffQ, &map_qkv.hi, bar, h * 64, row0);
#pragma unroll
    for (int t = 0; t < R; ++t) {
      tma_load_2d(smem + SM::kOffK + t * kAttTile, &map_qkv.hi, bar, n_heads * 64 + h * 64, krow0 + t * 128);
      tma_load_2d(smem + SM::kOffV + t * kAttTile, &map_qkv.hi, bar, 2 * n_heads * 64 + h * 64, krow0 + t * 128);
    }
    if constexpr (SPLIT) {
      tma_load_2d(smem + SM::kOffLo + SM::kOffQ, &map_qkv.lo, bar, h * 64, row0);
#pragma unroll
      for (int t = 0; t < R; ++t) {
        tma_load_2d(smem + SM::kOffLo + SM::kOffK + t * kAttTile, &map_qkv.lo, bar, n_heads * 64 + h * 64, krow0 + t * 128);
        tma_load_2d(smem + SM::kOffLo + SM::kOffV + t * kAttTile, &map_qkv.lo, bar, 2 * n_heads * 64 + h * 64, krow0 + t * 128);
      }
    }
  }
  mbar_wait(bar, 0);

  const int wg = threadIdx.x >> 7, warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const uint32_t sbase = smem_u32(smem);
  // ---- S = Q K^T: s[t] holds the scores of key tile t ----
  float s[R][64];
#pragma unroll
  for (int t = 0; t < R; ++t)
#pragma unroll
    for (int i = 0; i < 64; ++i) s[t][i] = 0.0f;
  {
    const uint64_t da = make_smem_desc<128>(sbase + SM::kOffQ + wg * 64 * 128);
    wgmma_fence();
    if constexpr (SPLIT) {
      const uint64_t da_lo = make_smem_desc<128>(sbase + SM::kOffLo + SM::kOffQ + wg * 64 * 128);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
#pragma unroll
        for (int t = 0; t < R; ++t) {
          const uint64_t db = make_smem_desc<128>(sbase + SM::kOffK + t * kAttTile), db_lo = make_smem_desc<128>(sbase + SM::kOffLo + SM::kOffK + t * kAttTile);
          wgmma_ss_n128<true>(s[t], da_lo + 2 * k, db + 2 * k, k != 0);
          wgmma_ss_n128<true>(s[t], da + 2 * k, db_lo + 2 * k, 1);
          wgmma_ss_n128<true>(s[t], da + 2 * k, db + 2 * k, 1);
        }
      }
    } else {
#pragma unroll
      for (int k = 0; k < 4; ++k)
#pragma unroll
        for (int t = 0; t < R; ++t) wgmma_ss_n128<BF16>(s[t], da + 2 * k, make_smem_desc<128>(sbase + SM::kOffK + t * kAttTile) + 2 * k, k != 0);
    }
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int t = 0; t < R; ++t) fence_acc(s[t]);
  }
  // ---- softmax over the valid keys: rows r0 (s[t][4j], s[t][4j+1]) and r0 + 8 (s[t][4j+2], s[t][4j+3]), keys
  // 128 t + 8j + 2(lane%4) + {0,1} ----
  constexpr float kLog2e = 1.4426950408889634f;
  const int kq = 2 * (lane & 3);
  float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
  for (int t = 0; t < R; ++t) {
#pragma unroll
    for (int j = 0; j < 16; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        if (128 * t + 8 * j + kq + e < n_valid) { mx0 = fmaxf(mx0, s[t][4 * j + e]); mx1 = fmaxf(mx1, s[t][4 * j + 2 + e]); }
      }
    }
  }
#pragma unroll
  for (int o = 1; o <= 2; o <<= 1) {
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, o));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, o));
  }
  // e = 2^((s - max) log2 e) in (0, 1], rounded to the operand dtype (split mode: to a pair); V carries a column of ones, so
  // the PV MMA also produces the row sums of the rounded P and O is normalised on the way out
  const float mb0 = mx0 * kLog2e, mb1 = mx1 * kLog2e;
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.0f;
  // ---- O = P V, one 128-key chunk (key tile t) at a time ----
#pragma unroll
  for (int t = 0; t < R; ++t) {
    uint32_t pa[8][4];
    uint32_t pl[SPLIT ? 8 : 1][4];                               // split mode: P_lo
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      float e[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const bool ok = 128 * t + 8 * j + kq + (q & 1) < n_valid;
        e[q] = ok ? ex2_approx(fmaf(s[t][4 * j + q], kLog2e, (q < 2) ? -mb0 : -mb1)) : 0.0f;
      }
      // A fragment of k-step j/2: {row r0 keys +0..1, row r0+8 keys +0..1, row r0 keys +8..9, row r0+8 keys +8..9}
      if constexpr (SPLIT) {
        O::pack_pair(e[0], e[1], pa[j >> 1][(j & 1) * 2 + 0], pl[j >> 1][(j & 1) * 2 + 0]);
        O::pack_pair(e[2], e[3], pa[j >> 1][(j & 1) * 2 + 1], pl[j >> 1][(j & 1) * 2 + 1]);
      } else {
        pa[j >> 1][(j & 1) * 2 + 0] = O::pack(e[0], e[1]);
        pa[j >> 1][(j & 1) * 2 + 1] = O::pack(e[2], e[3]);
      }
    }
    wgmma_fence();
    const uint32_t vt = sbase + SM::kOffV + t * kAttTile;
    if constexpr (SPLIT) {
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const uint64_t dv = make_smem_desc<128>(vt + k * 2048), dv_lo = make_smem_desc<128>(vt + SM::kOffLo + k * 2048);
        wgmma_rs_n64_tb<true>(o, pl[k], dv, (t | k) != 0);
        wgmma_rs_n64_tb<true>(o, pa[k], dv_lo, 1);
        wgmma_rs_n64_tb<true>(o, pa[k], dv, 1);
      }
    } else {
#pragma unroll
      for (int k = 0; k < 8; ++k)                                // 16 keys per MMA: V advances 16 rows = 2 KB
        wgmma_rs_n64_tb<BF16>(o, pa[k], make_smem_desc<128>(vt + k * 2048), (t | k) != 0);
    }
    wgmma_commit();
    wgmma_wait<0>();                                             // the chunk's P registers are free again
    fence_acc(o);
  }
  // the ones column (head dim kAttOnesCol) sits in n8 block kAttOnesCol / 8 of the lane with 2 (lane % 4) = kAttOnesCol % 8
  constexpr int jd = kAttOnesCol / 8, ld = (kAttOnesCol % 8) / 2, ed = kAttOnesCol % 2;
  const float inv0 = 1.0f / __shfl_sync(0xffffffffu, o[4 * jd + ed], (lane & ~3) | ld);
  const float inv1 = 1.0f / __shfl_sync(0xffffffffu, o[4 * jd + 2 + ed], (lane & ~3) | ld);
  float den0 = 0.0f, den1 = 0.0f;                                // split mode: the row sums themselves (O / den, see the top)
  if constexpr (SPLIT) {
    den0 = __shfl_sync(0xffffffffu, o[4 * jd + ed], (lane & ~3) | ld);
    den1 = __shfl_sync(0xffffffffu, o[4 * jd + 2 + ed], (lane & ~3) | ld);
  }
  typename O::T* out = static_cast<typename O::T*>(att);
  const size_t r0 = static_cast<size_t>(row0 + wg * 64 + warp * 16 + (lane >> 2));
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = h * 64 + 8 * j + kq;
    if constexpr (SPLIT) {
      typename O::T* lo = static_cast<typename O::T*>(att_lo);
      O::pack_pair(o[4 * j] / den0, o[4 * j + 1] / den0, *reinterpret_cast<uint32_t*>(out + r0 * kAttOut + c), *reinterpret_cast<uint32_t*>(lo + r0 * kAttOut + c));
      O::pack_pair(o[4 * j + 2] / den1, o[4 * j + 3] / den1, *reinterpret_cast<uint32_t*>(out + (r0 + 8) * kAttOut + c),
                   *reinterpret_cast<uint32_t*>(lo + (r0 + 8) * kAttOut + c));
    } else {
      *reinterpret_cast<uint32_t*>(out + r0 * kAttOut + c) = O::pack(o[4 * j] * inv0, o[4 * j + 1] * inv0);
      *reinterpret_cast<uint32_t*>(out + (r0 + 8) * kAttOut + c) = O::pack(o[4 * j + 2] * inv1, o[4 * j + 3] * inv1);
    }
  }
}

}  // namespace ldm
