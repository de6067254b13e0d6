// wgmma (Hopper warpgroup MMA) GEMMs of the LayoutDM denoiser, C[M,N] = A[M,K] * W[N,K]^T (+ fused epilogue).
//
//   A : activations, row-major [M][K] 16-bit (fp16 or bf16), M = 128 * n_layouts (one 128-row block = one layout)
//   W : nn.Linear weight, row-major [N][K] 16-bit  (both operands are "K-major" for the MMA)
//   split mode (OP_BF16X3): A and W are bf16 (hi, lo) plane pairs; see below
//
// One kernel template, 384 threads; CTA b runs tiles b, b + gridDim.x, ... (the column tile varies fastest, so consecutive
// tiles share their A row block in L2).  The GEMMs with TMA-staged stores are launched persistent (min(tiles, SMs) CTAs),
// the others with one CTA per tile:
//   warps 0..7  : two consumer warpgroups (setmaxnreg: 232 registers).  Each issues m64 x BN_WG x k16 wgmmas from the
//                 shared-memory ring (fp32 accumulators in registers) and runs the epilogue on its own accumulator fragment.
//   warps 8..11 : producer warpgroup (setmaxnreg: 40 registers), one lane issues the TMA loads: cp.async.bulk.tensor 2-D
//                 tiles with the 128-byte swizzle into a STAGES-deep ring, completion on mbarriers (full: TMA bytes landed,
//                 empty: both warpgroups' MMAs have read the stage).  Ring slot and phase run on across tiles, so the
//                 producer fills the ring with the next tile while the consumers run this tile's epilogue.
// Stores: the 16-bit QKV / FF1 epilogues (one-plane modes) write the fragment into a shared-memory staging tile and one
// thread per warpgroup stores it with TMA; the consumers go on to the next tile while the store drains.  The other epilogues
// store straight from the fragment.
// Tile shapes:
//   WG_M = 2 : 128 rows x BN_WG columns, the warpgroups split the rows (QKV, FF1: 256 columns; vocabulary head: 160)
//   WG_M = 1 :  64 rows x 2 BN_WG columns, the warpgroups split the columns.  Used by the LN epilogue: 2 x 232 = 464 =
//              d_model, so a CTA holds whole rows and the LayerNorm row statistics are combined in shared memory.
// Epilogues:  QKV (bias, q-scale, 16-bit) | RELU (FF1: bias, ReLU, 16-bit) | F32 (bias; vocabulary head) |
//             LN  (out-projection / FF2: bias + residual + LayerNorm, affine or timestep-adaptive, fused).
//
// Split mode: a ring stage holds four boxes, A_hi | A_lo | W_hi | W_lo, of a 32-element k-block with the 64-byte swizzle, so a
// stage keeps the bytes (and the GEMMs their stage counts) of the 64-element one-plane k-block.  Each k16 step issues three
// wgmmas into the accumulator: a_lo w_hi, a_hi w_lo, a_hi w_hi.  16-bit outputs are written as (hi, lo) pairs (out, out_lo).
//
// Reference ops replaced: nn.Linear / nn.MultiheadAttention projections / nn.LayerNorm / AdaLayerNorm in
// T/models/transformer_utils.py:79-83,165-210 and T/models/common/nn_lib.py:187-189,235.
#pragma once
#include "common.cuh"

namespace ldm {

constexpr int kBM = 128;       // rows of one layout tile (125 tokens + 3 pad rows)
constexpr int kBK = 64;        // K elements per smem stage (= 128 B = one swizzle row)
constexpr int kBKSplit = 32;   // split mode: K elements per stage and plane (= 64 B = one 64-byte swizzle row)
constexpr int kWgK = 16;       // K per wgmma (16-bit operands)
constexpr int kGemmConsumers = 256;
constexpr int kProducerRegs = 40, kConsumerRegs = 232;   // persistent block: 128 x 40 + 256 x 232 <= the SM's 64 K registers

enum : int { EPI_QKV = 0, EPI_RELU = 1, EPI_F32 = 2, EPI_LN = 3 };

struct GemmParams {
  int M, N, K;            // M multiple of the tile rows; N <= n_tiles * tile columns (columns past N are computed on zero weights, not stored)
  int n_tiles;
  const float* bias;      // [N] or nullptr
  void* out;              // [M][ldo] 16-bit (EPI_F32: fp32)
  int ldo;
  float qscale;           // EPI_QKV: columns < qcols are scaled by qscale after the bias
  int qcols;
  // EPI_LN (N = 464): y = acc + bias + resid ; out = LayerNorm(y) * gamma + beta  (gamma = 1 + scale_t for AdaLN)
  const float* resid;     // fp32 [M][N] residual stream
  float* y_out;           // fp32 [M][N] pre-norm sum (the next residual) or nullptr
  const float* ln_scale;  // [N]
  const float* ln_shift;  // [N]
  int adaln;
  float* out32;           // fp32 [M][N] normalised output (next residual, AdaLN case) or nullptr
  const int* t_layout;    // EPI_LN + adaln: per-layout timesteps (training-side calls): ln_scale then points at the layer's whole [T][2N]
  int n_layouts;          //   AdaLN table and every layout reloads its (scale, shift) row; nullptr: one timestep for all
  int rev;                // 1: walk the row blocks from the last to the first.  Consecutive kernels alternate the direction, so a consumer starts
                          // with the rows its producer wrote last -- the part of the intermediate that is still in L2
  void* out_lo;           // split mode: lo plane of the 16-bit output (same layout as out)
};

// TMA-staged stores: the 16-bit plain epilogues of the one-plane modes (the split mode's (hi, lo) pair outputs would need two
// staging tiles, which leave too few ring stages).  These GEMMs are the persistent ones: 384 threads (producer warpgroup),
// min(tiles, SMs) CTAs.  The others store from the fragment, have nothing to overlap their epilogue with, and run one tile per
// CTA with 288 threads (one producer warp)
template <int EPI, bool SPLIT>
constexpr bool kStagedStore = (EPI == EPI_QKV || EPI == EPI_RELU) && !SPLIT;
template <int EPI, int MODE>
constexpr int kGemmThreads = kStagedStore<EPI, kOpSplit<MODE>> ? 384 : 288;

template <int BN_WG, int WG_M, int STAGES, bool SPLIT = false, bool STAGED = false>
struct GemmSmem {
  static constexpr int kWgN = 3 - WG_M;                          // warpgroups along N
  static constexpr int kPlanes = SPLIT ? 2 : 1;
  static constexpr int kKB = SPLIT ? kBKSplit : kBK;             // K elements per stage
  static constexpr int kRowBytes = kKB * 2;                      // one smem row = one swizzle row (128 B, split: 64 B)
  static constexpr int kAPlane = 64 * WG_M * kRowBytes;
  static constexpr int kABytes = kPlanes * kAPlane;              // A_hi (| A_lo)
  static constexpr int kBBytes = BN_WG * kRowBytes;              // one warpgroup's weight rows of one plane
  static constexpr int kStageBytes = kABytes + kPlanes * kWgN * kBBytes;   // ... | W_hi blocks (| W_lo blocks)
  static_assert(kBBytes % (SPLIT ? 512 : 1024) == 0, "weight block must keep the swizzle atom's alignment");
  // staging tile of a 16-bit output tile: [column block of 64][row][128 B] with the 128-byte swizzle, so warpgroup wm's rows of
  // column block cb are one TMA store box (64 columns x 64 rows) at cb * kStoreCb + wm * 8 KB
  static constexpr int kStoreCb = 64 * WG_M * 128;
  static constexpr int kStoreBytes = STAGED ? (kWgN * BN_WG / 64) * kStoreCb : 0;
  static_assert(!STAGED || BN_WG % 64 == 0, "staged stores go out in 64-column boxes");
  static constexpr int kOffStore = STAGES * kStageBytes;
  static constexpr int kOffBars = kOffStore + kStoreBytes;
  static constexpr int kOffStat = kOffBars + 256;                // LN: per-row sum, then sum of squared deviations, of each warpgroup's columns
  static constexpr int kBytes = kOffStat + 2 * 64 * 16 + 1024 /*align slack*/;
  static_assert(2 * STAGES * 8 <= 256, "barrier block overflow");
  static_assert(kBytes <= 232448, "exceeds the 227 KB of shared memory per CTA");
};

template <bool BF16, int N>
LDM_DEVINL void wgmma_ss(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t accumulate) {
  if constexpr (N == 256) wgmma_ss_n256<BF16>(d, da, db, accumulate);
  else if constexpr (N == 232) wgmma_ss_n232<BF16>(d, da, db, accumulate);
  else if constexpr (N == 160) wgmma_ss_n160<BF16>(d, da, db, accumulate);
  else { static_assert(N == 128, "unsupported wgmma width"); wgmma_ss_n128<BF16>(d, da, db, accumulate); }
}

// grid: staged (persistent): up to tiles = n_tiles * M / (64 WG_M) CTAs, otherwise exactly one CTA per tile; map_out: the TMA
// store map of a staged epilogue (box 64 x 64 rows)
template <int BN_WG, int WG_M, int STAGES, int EPI, int MODE>
__global__ void __launch_bounds__(kGemmThreads<EPI, MODE>, 1)
gemm_tc_kernel(const __grid_constant__ OpMaps<MODE> map_a /*box 64 (split: 32) x 64 WG_M rows*/,
               const __grid_constant__ OpMaps<MODE> map_b /*box 64 (split: 32) x BN_WG rows*/,
               const __grid_constant__ CUtensorMap map_out, const GemmParams p) {
  constexpr bool BF16 = kOpBf16<MODE>, SPLIT = kOpSplit<MODE>, STAGED = kStagedStore<EPI, SPLIT>;
  using SM = GemmSmem<BN_WG, WG_M, STAGES, SPLIT, STAGED>;
  using O = OpT<MODE>;
  constexpr int kKB = SM::kKB;
  constexpr int kBMt = 64 * WG_M, kAcc = BN_WG / 2;
  static_assert(EPI != EPI_LN || (WG_M == 1 && BN_WG == 232), "LN epilogue is laid out for 464 = 2 x 232 columns");
  static_assert(EPI == EPI_LN || WG_M == 2, "plain epilogues use 128-row tiles");

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + SM::kOffBars);
  uint64_t* empty = full + STAGES;

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
  const int num_kb = (p.K + kKB - 1) / kKB;
  const int n_mblk = p.M / kBMt, n_work = n_mblk * p.n_tiles;
  // tile t: row block t / n_tiles (walked from the last one down when rev), column tile t % n_tiles
  const auto tile_m0 = [&](int t) { const int mb = t / p.n_tiles; return (p.rev ? n_mblk - 1 - mb : mb) * kBMt; };
  const auto tile_n0 = [&](int t) { return (t % p.n_tiles) * BN_WG * SM::kWgN; };

  if (threadIdx.x == kGemmConsumers) {
    tma_prefetch_desc(&map_a.hi);
    tma_prefetch_desc(&map_b.hi);
    if constexpr (SPLIT) { tma_prefetch_desc(&map_a.lo); tma_prefetch_desc(&map_b.lo); }
    if constexpr (STAGED) tma_prefetch_desc(&map_out);
    for (int i = 0; i < STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], kGemmConsumers); }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_sync();                                                // everything above overlapped the previous kernel's tail

  if (warp >= kGemmConsumers / 32) {
    // ===================== TMA producer =====================
    if constexpr (STAGED) setmaxnreg_dec<kProducerRegs>();
    if (threadIdx.x == kGemmConsumers) {
      int s = 0;
      uint32_t phase = 0;                                    // ring slot and pass, carried from tile to tile
      for (int t = blockIdx.x; t < n_work; t += gridDim.x) {
        const int m0 = tile_m0(t), n0 = tile_n0(t);
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty[s], phase ^ 1);
          uint8_t* st = smem + s * SM::kStageBytes;
          mbar_arrive_expect_tx(&full[s], SM::kStageBytes);    // out-of-bounds box parts are zero-filled and still counted
          tma_load_2d(st, &map_a.hi, &full[s], kb * kKB, m0);
#pragma unroll
          for (int wn = 0; wn < SM::kWgN; ++wn) tma_load_2d(st + SM::kABytes + wn * SM::kBBytes, &map_b.hi, &full[s], kb * kKB, n0 + wn * BN_WG);
          if constexpr (SPLIT) {
            tma_load_2d(st + SM::kAPlane, &map_a.lo, &full[s], kb * kKB, m0);
#pragma unroll
            for (int wn = 0; wn < SM::kWgN; ++wn)
              tma_load_2d(st + SM::kABytes + (SM::kWgN + wn) * SM::kBBytes, &map_b.lo, &full[s], kb * kKB, n0 + wn * BN_WG);
          }
          if (++s == STAGES) { s = 0; phase ^= 1; }
        }
        if constexpr (!STAGED) break;                        // one tile per CTA
      }
    }
    return;
  }

  // ===================== consumer warpgroups =====================
  if constexpr (STAGED) setmaxnreg_inc<kConsumerRegs>();
  const int wg = warp >> 2;
  const int wm = WG_M == 2 ? wg : 0, wn = WG_M == 2 ? 0 : wg;
  float acc[kAcc];
#pragma unroll
  for (int i = 0; i < kAcc; ++i) acc[i] = 0.0f;
  int s = 0;
  uint32_t phase = 0;
  for (int t = blockIdx.x; t < n_work; t += gridDim.x) {
    const int m0 = tile_m0(t), n0 = tile_n0(t);
    for (int kb = 0; kb < num_kb; ++kb) {
      mbar_wait(&full[s], phase);
      const uint32_t st = smem_u32(smem + s * SM::kStageBytes);
      if constexpr (!SPLIT) {
        const uint64_t da = make_smem_desc<128>(st + wm * 64 * 128);
        const uint64_t db = make_smem_desc<128>(st + SM::kABytes + wn * SM::kBBytes);
        wgmma_fence();
        if (kb * kBK + kBK <= p.K) {
#pragma unroll
          for (int k = 0; k < kBK / kWgK; ++k) wgmma_ss<BF16, BN_WG>(acc, da + 2 * k, db + 2 * k, (kb | k) != 0);   // +32 B per k-step (>>4 = 2)
        } else {                                              // K tail of 16 (K % 64 is 0 or 16, checked at create): one k-step
          wgmma_ss<BF16, BN_WG>(acc, da, db, kb != 0);
        }
      } else {
        const uint64_t da = make_smem_desc<64>(st + wm * 64 * SM::kRowBytes), da_lo = make_smem_desc<64>(st + SM::kAPlane + wm * 64 * SM::kRowBytes);
        const uint64_t db = make_smem_desc<64>(st + SM::kABytes + wn * SM::kBBytes);
        const uint64_t db_lo = make_smem_desc<64>(st + SM::kABytes + (SM::kWgN + wn) * SM::kBBytes);
        wgmma_fence();
        // K % 32 is 0 or 16 (d = 464: 16): the tail k-block is a single k-step
        const int nk = kb * kKB + kKB <= p.K ? kKB / kWgK : 1;
#pragma unroll
        for (int k = 0; k < kKB / kWgK; ++k) {
          if (k < nk) {                                       // +32 B per k-step (>>4 = 2); the small terms first
            wgmma_ss<true, BN_WG>(acc, da_lo + 2 * k, db + 2 * k, (kb | k) != 0);
            wgmma_ss<true, BN_WG>(acc, da + 2 * k, db_lo + 2 * k, 1);
            wgmma_ss<true, BN_WG>(acc, da + 2 * k, db + 2 * k, 1);
          }
        }
      }
      wgmma_commit();
      // keep this k-block's MMAs in flight; once the previous k-block's have retired its stage goes back to the producer
      if (kb > 0) { wgmma_wait<1>(); mbar_arrive(&empty[s == 0 ? STAGES - 1 : s - 1]); }
      if (++s == STAGES) { s = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    fence_acc(acc);
    mbar_arrive(&empty[s == 0 ? STAGES - 1 : s - 1]);         // the tile's last stage: refilled with the next tile during the epilogue

    const int rw = (warp & 3) * 16 + (lane >> 2);           // fragment rows rw and rw + 8 of the warpgroup's 64
    const int row0 = m0 + wm * 64 + rw, row1 = row0 + 8;
    const int col0 = n0 + wn * BN_WG + 2 * (lane & 3);        // + 8 j: columns col, col + 1 of n8 block j

    if constexpr (STAGED) {
      // bias (q-scale | ReLU), 16-bit, into the staging tile; then one thread of the warpgroup stores its 64 rows with TMA
      float scale = 1.0f;
      if constexpr (EPI == EPI_QKV) scale = (n0 < p.qcols) ? p.qscale : 1.0f;   // Q tiles are whole tiles (512 % 256 == 0)
      const bool leader = (threadIdx.x & 127) == 0;
      uint8_t* stage = smem + SM::kOffStore + wm * 64 * 128;
      const uint32_t stage_u32 = smem_u32(stage);            // 32-bit shared addresses: 64-bit generic ones cost registers per column block
      // one named barrier per warpgroup, with a compile-time id
      const auto wg_bar = [&]() { if (wg == 0) named_bar_sync(2, 128); else named_bar_sync(3, 128); };
      if (leader) bulk_wait_group_read<0>();                   // the previous tile's store has read the staging tile
      wg_bar();
      const int sw = (rw & 7) << 4;                            // 128-byte swizzle: 16-byte chunk ^= row % 8 (rw + 8: the same)
#pragma unroll
      for (int j = 0; j < BN_WG / 8; ++j) {
        const int c = col0 + 8 * j;
        if (c >= p.N) continue;                               // columns past N: the TMA store clips them
        const float2 b = p.bias != nullptr ? __ldg(reinterpret_cast<const float2*>(p.bias + c)) : make_float2(0.0f, 0.0f);
        float v[4] = {acc[4 * j] + b.x, acc[4 * j + 1] + b.y, acc[4 * j + 2] + b.x, acc[4 * j + 3] + b.y};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          if constexpr (EPI == EPI_QKV) v[e] *= scale;
          if constexpr (EPI == EPI_RELU) v[e] = fmaxf(v[e], 0.0f);
        }
        const uint32_t blk = stage_u32 + (j >> 3) * SM::kStoreCb + ((((j & 7) << 4) ^ sw) | (4 * (lane & 3)));
        st_shared_u32(blk + rw * 128, O::pack(v[0], v[1]));
        st_shared_u32(blk + (rw + 8) * 128, O::pack(v[2], v[3]));
      }
      fence_proxy_async_smem();
      wg_bar();
      if (leader) {
#pragma unroll
        for (int cb = 0; cb < BN_WG / 64; ++cb)
          if (n0 + cb * 64 < p.N) tma_store_2d(&map_out, stage + cb * SM::kStoreCb, n0 + cb * 64, m0 + wm * 64);
        bulk_commit_group();
      }
    } else if constexpr (EPI != EPI_LN) {
      float scale = 1.0f;
      if constexpr (EPI == EPI_QKV) scale = (n0 < p.qcols) ? p.qscale : 1.0f;   // Q tiles are whole tiles (512 % 256 == 0)
#pragma unroll
      for (int j = 0; j < BN_WG / 8; ++j) {
        const int c = col0 + 8 * j;
        if (c >= p.N) continue;                               // N is even: the pair (c, c + 1) is in or out together
        const float2 b = p.bias != nullptr ? __ldg(reinterpret_cast<const float2*>(p.bias + c)) : make_float2(0.0f, 0.0f);
        float v[4] = {acc[4 * j] + b.x, acc[4 * j + 1] + b.y, acc[4 * j + 2] + b.x, acc[4 * j + 3] + b.y};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          if constexpr (EPI == EPI_QKV) v[e] *= scale;
          if constexpr (EPI == EPI_RELU) v[e] = fmaxf(v[e], 0.0f);
        }
        if constexpr (EPI == EPI_F32) {
          float* o = static_cast<float*>(p.out);
          *reinterpret_cast<float2*>(o + static_cast<size_t>(row0) * p.ldo + c) = make_float2(v[0], v[1]);
          *reinterpret_cast<float2*>(o + static_cast<size_t>(row1) * p.ldo + c) = make_float2(v[2], v[3]);
        } else {
          uint32_t* o0 = reinterpret_cast<uint32_t*>(static_cast<typename O::T*>(p.out) + static_cast<size_t>(row0) * p.ldo + c);
          uint32_t* o1 = reinterpret_cast<uint32_t*>(static_cast<typename O::T*>(p.out) + static_cast<size_t>(row1) * p.ldo + c);
          if constexpr (SPLIT) {
            uint32_t* l0 = reinterpret_cast<uint32_t*>(static_cast<typename O::T*>(p.out_lo) + static_cast<size_t>(row0) * p.ldo + c);
            uint32_t* l1 = reinterpret_cast<uint32_t*>(static_cast<typename O::T*>(p.out_lo) + static_cast<size_t>(row1) * p.ldo + c);
            O::pack_pair(v[0], v[1], *o0, *l0);
            O::pack_pair(v[2], v[3], *o1, *l1);
          } else {
            *o0 = O::pack(v[0], v[1]);
            *o1 = O::pack(v[2], v[3]);
          }
        }
      }
    } else {
      // ============ fused residual + LayerNorm epilogue (out-projection / FF2) ============
      //   y = acc + bias + resid (-> y_out); two-pass row statistics: the row sum over the thread's columns, the quad of lanes
      //   that shares a row, then the other warpgroup (other 232 columns) through shared memory gives the mean; the sum of
      //   (y - mean)^2 is reduced the same way.  One pass, E[y^2] - mean^2, loses the variance to cancellation once
      //   |mean| / std is large.  The sums run over y - pivot, pivot = bias[0] + resid[row][0] (y's column 0 without the GEMM
      //   term, the same in all 8 threads of a row): their terms are of the row's spread, not of its mean, so the mean of a row
      //   far from zero comes out correctly rounded too (a plain fp32 sum of 464 values near 256 is off by several ulps of the
      //   mean, which every output of the row inherits).  Normalise, 16-bit (+ fp32) outputs.
      float* ssum = reinterpret_cast<float*>(smem + SM::kOffStat);   // [warpgroup][64 rows] row sums of y - pivot
      float* ssq = ssum + 2 * 64;                                     // [warpgroup][64 rows] sums of squared deviations
      const int N = p.N;
      const float* r0p = p.resid + static_cast<size_t>(row0) * N;
      const float* r1p = p.resid + static_cast<size_t>(row1) * N;
      const float piv0 = __ldg(p.bias) + r0p[0], piv1 = __ldg(p.bias) + r1p[0];
      float s0 = 0.0f, s1 = 0.0f;
#pragma unroll
      for (int j = 0; j < BN_WG / 8; ++j) {
        const int c = col0 + 8 * j;
        const float2 b = __ldg(reinterpret_cast<const float2*>(p.bias + c));
        const float2 ra = *reinterpret_cast<const float2*>(r0p + c), rb = *reinterpret_cast<const float2*>(r1p + c);
        acc[4 * j] += b.x + ra.x; acc[4 * j + 1] += b.y + ra.y;
        acc[4 * j + 2] += b.x + rb.x; acc[4 * j + 3] += b.y + rb.y;
        if (p.y_out != nullptr) {
          *reinterpret_cast<float2*>(p.y_out + static_cast<size_t>(row0) * N + c) = make_float2(acc[4 * j], acc[4 * j + 1]);
          *reinterpret_cast<float2*>(p.y_out + static_cast<size_t>(row1) * N + c) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
        }
        acc[4 * j] -= piv0; acc[4 * j + 1] -= piv0; acc[4 * j + 2] -= piv1; acc[4 * j + 3] -= piv1;   // from here on: y - pivot
        s0 += acc[4 * j] + acc[4 * j + 1];
        s1 += acc[4 * j + 2] + acc[4 * j + 3];
      }
#pragma unroll
      for (int o = 1; o <= 2; o <<= 1) {
        s0 += __shfl_xor_sync(0xffffffffu, s0, o);
        s1 += __shfl_xor_sync(0xffffffffu, s1, o);
      }
      if ((lane & 3) == 0) { ssum[wn * 64 + rw] = s0; ssum[wn * 64 + rw + 8] = s1; }
      named_bar_sync(1, kGemmConsumers);
      const float inv_n = 1.0f / static_cast<float>(N);
      const float mean0 = (s0 + ssum[(wn ^ 1) * 64 + rw]) * inv_n, mean1 = (s1 + ssum[(wn ^ 1) * 64 + rw + 8]) * inv_n;   // mean - pivot, like acc
      float q0 = 0.0f, q1 = 0.0f;
#pragma unroll
      for (int j = 0; j < BN_WG / 8; ++j) {
        const float d0 = acc[4 * j] - mean0, d1 = acc[4 * j + 1] - mean0, d2 = acc[4 * j + 2] - mean1, d3 = acc[4 * j + 3] - mean1;
        q0 = fmaf(d0, d0, fmaf(d1, d1, q0));
        q1 = fmaf(d2, d2, fmaf(d3, d3, q1));
      }
#pragma unroll
      for (int o = 1; o <= 2; o <<= 1) {
        q0 += __shfl_xor_sync(0xffffffffu, q0, o);
        q1 += __shfl_xor_sync(0xffffffffu, q1, o);
      }
      if ((lane & 3) == 0) { ssq[wn * 64 + rw] = q0; ssq[wn * 64 + rw + 8] = q1; }
      named_bar_sync(1, kGemmConsumers);
      const float rstd0 = 1.0f / sqrtf(fmaxf((q0 + ssq[(wn ^ 1) * 64 + rw]) * inv_n, 0.0f) + 1e-5f);
      const float rstd1 = 1.0f / sqrtf(fmaxf((q1 + ssq[(wn ^ 1) * 64 + rw + 8]) * inv_n, 0.0f) + 1e-5f);
      const float* gam = p.ln_scale;
      const float* bet = p.ln_shift;
      float gadd = p.adaln ? 1.0f : 0.0f;
      if (p.t_layout != nullptr) {                             // per-layout timesteps: this layout's AdaLN (scale, shift) row
        const int layout = m0 / kBM;
        const int tl = layout < p.n_layouts ? __ldg(p.t_layout + layout) : 0;
        gam = p.ln_scale + static_cast<size_t>(tl) * 2 * N; bet = gam + N; gadd = 1.0f;
      }
      typename O::T* out16 = static_cast<typename O::T*>(p.out);
#pragma unroll
      for (int j = 0; j < BN_WG / 8; ++j) {
        const int c = col0 + 8 * j;
        const float2 g = __ldg(reinterpret_cast<const float2*>(gam + c)), h = __ldg(reinterpret_cast<const float2*>(bet + c));
        const float v0 = (acc[4 * j] - mean0) * rstd0 * (g.x + gadd) + h.x, v1 = (acc[4 * j + 1] - mean0) * rstd0 * (g.y + gadd) + h.y;
        const float v2 = (acc[4 * j + 2] - mean1) * rstd1 * (g.x + gadd) + h.x, v3 = (acc[4 * j + 3] - mean1) * rstd1 * (g.y + gadd) + h.y;
        if constexpr (SPLIT) {
          typename O::T* lo16 = static_cast<typename O::T*>(p.out_lo);
          O::pack_pair(v0, v1, *reinterpret_cast<uint32_t*>(out16 + static_cast<size_t>(row0) * N + c), *reinterpret_cast<uint32_t*>(lo16 + static_cast<size_t>(row0) * N + c));
          O::pack_pair(v2, v3, *reinterpret_cast<uint32_t*>(out16 + static_cast<size_t>(row1) * N + c), *reinterpret_cast<uint32_t*>(lo16 + static_cast<size_t>(row1) * N + c));
        } else {
          *reinterpret_cast<uint32_t*>(out16 + static_cast<size_t>(row0) * N + c) = O::pack(v0, v1);
          *reinterpret_cast<uint32_t*>(out16 + static_cast<size_t>(row1) * N + c) = O::pack(v2, v3);
        }
        if (p.out32 != nullptr) {
          *reinterpret_cast<float2*>(p.out32 + static_cast<size_t>(row0) * N + c) = make_float2(v0, v1);
          *reinterpret_cast<float2*>(p.out32 + static_cast<size_t>(row1) * N + c) = make_float2(v2, v3);
        }
      }
    }
    if constexpr (!STAGED) break;                            // one tile per CTA
  }
  if constexpr (STAGED) {
    if ((threadIdx.x & 127) == 0) bulk_wait_group_all();   // the last staged stores are complete before the CTA exits
  }
}

// ============ persistent LN GEMM: out-projection / FF2 in the one-plane modes ============
// 64 x 464 tiles (whole rows), min(tiles, SMs) CTAs of 384 threads; CTA b runs tiles b, b + gridDim.x, ...  The LayerNorm runs
// in warps of its own and the fp32 traffic goes through bulk copies, so a tile's epilogue overlaps the next tile's MMAs:
//   warps 0..7  : two MMA warpgroups, 64 rows x 232 columns each, m64n232k16 from the ring.  After a tile's last k-block they
//                 wait for the tile's residual rows in the tile buffer, replace them by y = acc + (bias + resid) and go
//                 straight on to the next tile.
//   warps 8..10 : epilogue: the row statistics, the LayerNorm / AdaLN and the 16-bit stores from the tile buffer.  Warp 8
//                 also issues the bulk copies of whole rows between the buffer and global memory: y out (the next residual),
//                 the normalised fp32 rows (written back into the buffer) out, and the next tile's residual rows in.
//   warp 11     : producer, one lane issues the TMA loads.
// 168 registers for every warp, no setmaxnreg: ptxas compiles the whole kernel under the launch bound's register count, and a
// 512-thread block (a whole producer warpgroup) would leave the m64n232 wgmma 128, fewer than it needs.  Three epilogue warps
// cannot keep enough loads and stores in flight to move a tile's ~300 KB of fp32 rows at HBM rate themselves (~40 us per
// tile); the bulk copies need no registers.  Ring: 3 stages of 32-element k-blocks with the 64-byte swizzle (the split mode's
// geometry, one plane): a 64-element k-block leaves room for only 2 stages beside the 118 KB tile buffer.  The split mode keeps
// the fragment-epilogue kernel above: its two-plane stages do not fit beside the buffer.
// The results are bit for bit those of the fragment epilogue: the same k16 MMA sequence, y = acc + (bias + resid), and the row
// statistics keep its summation order (per row 8 chains (h, q), h = column half, q = quad lane, each summing
// (y_c - piv) + (y_c+1 - piv) over c = 232 h + 8 j + 2 q, j ascending; (q0 + q1) + (q2 + q3), then half + half) and its FMA
// contractions (y - mean is one fma(-sum, 1/N, y - piv), the output fma(d * rstd, gamma + gadd, beta)).
constexpr int kLnThreads = 384, kLnEpiThreads = 96;
struct LnSmem {
  static constexpr int kRows = 64, kWgCols = 232, kCols = 2 * kWgCols, kStages = 3;
  static constexpr int kKB = kBKSplit;                           // 32-element k-blocks, 64-byte swizzle rows
  static constexpr int kABytes = kRows * kKB * 2;
  static constexpr int kBBytes = kWgCols * kKB * 2;              // one MMA warpgroup's weight rows
  static constexpr int kStageBytes = kABytes + 2 * kBBytes;
  static_assert(kABytes % 512 == 0 && kBBytes % 512 == 0, "boxes must keep the 64-byte swizzle atom's alignment");
  // tile buffer [64][kLd] fp32: the 8-float pad puts the 8 rows of a fragment access in distinct 32-byte bank groups and
  // keeps every row 16-byte aligned for the bulk copies
  static constexpr int kLd = kCols + 8;
  static constexpr int kOffBuf = kStages * kStageBytes;
  static constexpr int kOffBars = kOffBuf + kRows * kLd * 4;      // full[3], empty[3], res_full, buf_full
  static constexpr int kOffStat = kOffBars + 64;                 // per row: pivot, row sum of y - pivot, rstd
  static constexpr int kBytes = kOffStat + 3 * kRows * 4 + 1024 /*align slack*/;
  static_assert(kLd * 4 % 16 == 0, "bulk copies need 16-byte aligned rows");
  static_assert(kBytes <= 232448, "exceeds the 227 KB of shared memory per CTA");
};

template <int MODE>
__global__ void __launch_bounds__(kLnThreads, 1)
gemm_ln_kernel(const __grid_constant__ CUtensorMap map_a /*box 32 x 64 rows, 64-byte swizzle*/,
               const __grid_constant__ CUtensorMap map_b /*box 32 x 232 rows, 64-byte swizzle*/, const GemmParams p) {
  static_assert(!kOpSplit<MODE>, "the split mode runs the fragment-epilogue LN GEMM");
  constexpr bool BF16 = kOpBf16<MODE>;
  using SM = LnSmem;
  using O = OpT<MODE>;
  constexpr int kRows = SM::kRows, kWgCols = SM::kWgCols, kLd = SM::kLd, kAcc = kWgCols / 2;
  constexpr int kEpi = kGemmConsumers, kProducer = kEpi + kLnEpiThreads;   // first thread of the epilogue warps / producer warp

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + SM::kOffBars);
  uint64_t* empty = full + SM::kStages;
  uint64_t* res_full = empty + SM::kStages;                      // the tile's residual rows have landed in the buffer
  uint64_t* buf_full = res_full + 1;                             // the MMA warpgroups wrote y into the buffer
  float* buf = reinterpret_cast<float*>(smem + SM::kOffBuf);
  float* s_piv = reinterpret_cast<float*>(smem + SM::kOffStat);
  float* s_sum = s_piv + kRows;
  float* s_rstd = s_sum + kRows;

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
  const int N = p.N;
  const int num_kb = p.K / SM::kKB;                             // K % 32 == 0 (checked at create)
  const int n_work = p.M / kRows;
  const auto tile_m0 = [&](int t) { return (p.rev ? n_work - 1 - t : t) * kRows; };

  if (threadIdx.x == kProducer) {
    tma_prefetch_desc(&map_a);
    tma_prefetch_desc(&map_b);
    for (int i = 0; i < SM::kStages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], kGemmConsumers); }
    mbar_init(res_full, 1);
    mbar_init(buf_full, kGemmConsumers);
    fence_mbar_init();
  }
  __syncthreads();
  pdl_sync();                                                // everything above overlapped the previous kernel's tail

  if (threadIdx.x >= kProducer) {
    // ===================== TMA producer =====================
    if (threadIdx.x == kProducer) {
      int s = 0;
      uint32_t phase = 0;
      for (int t = blockIdx.x; t < n_work; t += gridDim.x) {
        const int m0 = tile_m0(t);
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty[s], phase ^ 1);
          uint8_t* st = smem + s * SM::kStageBytes;
          mbar_arrive_expect_tx(&full[s], SM::kStageBytes);
          tma_load_2d(st, &map_a, &full[s], kb * SM::kKB, m0);
          tma_load_2d(st + SM::kABytes, &map_b, &full[s], kb * SM::kKB, 0);
          tma_load_2d(st + SM::kABytes + SM::kBBytes, &map_b, &full[s], kb * SM::kKB, kWgCols);
          if (++s == SM::kStages) { s = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  if (threadIdx.x >= kEpi) {
    // ===================== epilogue warps =====================
    const int et = threadIdx.x - kEpi;
    const bool copier = et < 32;                             // warp 8: the bulk copies, one row per lane at a time
    const uint32_t row_bytes = static_cast<uint32_t>(N) * sizeof(float);
    const float inv_n = 1.0f / static_cast<float>(N);
    constexpr int kVec = kWgCols / 2;                        // float4 columns of a row (116)
    constexpr int kTotal = kRows * kVec;                     // float4 of a tile; element i = k * 96 + et
    constexpr int kPerThread = (kTotal + kLnEpiThreads - 1) / kLnEpiThreads;
    // the residual rows of tile t into the buffer (the buffer is free: every read of it and every bulk store from it is done)
    const auto load_resid = [&](int t) {
      if (lane == 0) mbar_arrive_expect_tx(res_full, kRows * row_bytes);
      __syncwarp();
      const float* src = p.resid + static_cast<size_t>(tile_m0(t)) * N;
      for (int r = lane; r < kRows; r += 32) bulk_copy_g2s(buf + r * kLd, src + static_cast<size_t>(r) * N, row_bytes, res_full);
    };
    const auto store_rows = [&](float* dst) {                // the buffer's rows to dst, one bulk group per lane
      for (int r = lane; r < kRows; r += 32) bulk_copy_s2g(dst + static_cast<size_t>(r) * N, buf + r * kLd, row_bytes);
      bulk_commit_group();
    };
    if (copier) load_resid(blockIdx.x);
    uint32_t bphase = 0;
    for (int t = blockIdx.x; t < n_work; t += gridDim.x) {
      const int m0 = tile_m0(t);
      mbar_wait(buf_full, bphase);
      if (copier && p.y_out != nullptr) store_rows(p.y_out + static_cast<size_t>(m0) * N);
      // row statistics, a group of 4 rows per warp at a time; lane = 8 row + 4 h + q owns chain (h, q) of its row
      {
        const int h = (lane >> 2) & 1, q = lane & 3;
#pragma unroll 1
        for (int g = et >> 5; g < kRows / 4; g += kLnEpiThreads / 32) {
          const int r = 4 * g + (lane >> 3);
          const float piv = s_piv[r];
          const float* yr = buf + r * kLd + h * kWgCols + 2 * q;
          float s = 0.0f;
#pragma unroll
          for (int j = 0; j < kWgCols / 8; ++j) {
            const float2 y = *reinterpret_cast<const float2*>(yr + 8 * j);
            s += (y.x - piv) + (y.y - piv);
          }
          s += __shfl_xor_sync(0xffffffffu, s, 1);
          s += __shfl_xor_sync(0xffffffffu, s, 2);
          s += __shfl_xor_sync(0xffffffffu, s, 4);           // the row sum of y - pivot; mean - pivot = s / N
          float v = 0.0f;
#pragma unroll
          for (int j = 0; j < kWgCols / 8; ++j) {
            const float2 y = *reinterpret_cast<const float2*>(yr + 8 * j);
            const float d0 = fmaf(-s, inv_n, y.x - piv), d1 = fmaf(-s, inv_n, y.y - piv);
            v = fmaf(d0, d0, fmaf(d1, d1, v));
          }
          v += __shfl_xor_sync(0xffffffffu, v, 1);
          v += __shfl_xor_sync(0xffffffffu, v, 2);
          v += __shfl_xor_sync(0xffffffffu, v, 4);
          if ((lane & 7) == 0) { s_sum[r] = s; s_rstd[r] = 1.0f / sqrtf(fmaxf(v * inv_n, 0.0f) + 1e-5f); }
        }
      }
      if (copier) bulk_wait_group_read<0>();                 // the y rows are out of the buffer before it is overwritten
      named_bar_sync(1, kLnEpiThreads);
      // normalise: 16-bit outputs stored here, the fp32 ones written back into the buffer for a bulk store
      const float* gam = p.ln_scale;
      const float* bet = p.ln_shift;
      float gadd = p.adaln ? 1.0f : 0.0f;
      if (p.t_layout != nullptr) {                             // per-layout timesteps: this layout's AdaLN (scale, shift) row
        const int layout = m0 / kBM;
        const int tl = layout < p.n_layouts ? __ldg(p.t_layout + layout) : 0;
        gam = p.ln_scale + static_cast<size_t>(tl) * 2 * N; bet = gam + N; gadd = 1.0f;
      }
      typename O::T* out16 = static_cast<typename O::T*>(p.out);
      const bool keep32 = p.out32 != nullptr;
#pragma unroll 6
      for (int k = 0; k < kPerThread; ++k) {
        const int i = k * kLnEpiThreads + et, r = i / kVec, c = (i - r * kVec) * 4;
        if (i >= kTotal) continue;
        float4* bp = reinterpret_cast<float4*>(buf + r * kLd + c);
        const float4 y = *bp;
        const float4 g = __ldg(reinterpret_cast<const float4*>(gam + c)), b = __ldg(reinterpret_cast<const float4*>(bet + c));
        const float piv = s_piv[r], s = s_sum[r], rstd = s_rstd[r];
        const float4 v = make_float4(fmaf(fmaf(-s, inv_n, y.x - piv) * rstd, g.x + gadd, b.x), fmaf(fmaf(-s, inv_n, y.y - piv) * rstd, g.y + gadd, b.y),
                                     fmaf(fmaf(-s, inv_n, y.z - piv) * rstd, g.z + gadd, b.z), fmaf(fmaf(-s, inv_n, y.w - piv) * rstd, g.w + gadd, b.w));
        *reinterpret_cast<uint2*>(out16 + static_cast<size_t>(m0 + r) * N + c) = make_uint2(O::pack(v.x, v.y), O::pack(v.z, v.w));
        if (keep32) *bp = v;
      }
      if (keep32) fence_proxy_async_smem();                  // the fp32 rows are visible to the bulk store
      named_bar_sync(1, kLnEpiThreads);
      if (copier) {
        if (keep32) store_rows(p.out32 + static_cast<size_t>(m0) * N);
        bulk_wait_group_read<0>();
        if (t + static_cast<int>(gridDim.x) < n_work) load_resid(t + gridDim.x);
      }
      bphase ^= 1;
    }
    if (copier) bulk_wait_group_all();                       // the last bulk stores are complete before the CTA exits
    return;
  }

  // ===================== MMA warpgroups =====================
  const int wn = warp >> 2;                                  // column half
  float acc[kAcc];
  int s = 0;
  uint32_t phase = 0, bphase = 0;
  const int rw = (warp & 3) * 16 + (lane >> 2);              // fragment rows rw and rw + 8 of the tile
  const int cw = wn * kWgCols + 2 * (lane & 3);              // + 8 j: columns c, c + 1 of n8 block j
  float* bw = buf + rw * kLd + cw;
  for (int t = blockIdx.x; t < n_work; t += gridDim.x) {
    for (int kb = 0; kb < num_kb; ++kb) {
      mbar_wait(&full[s], phase);
      const uint32_t st = smem_u32(smem + s * SM::kStageBytes);
      const uint64_t da = make_smem_desc<64>(st);
      const uint64_t db = make_smem_desc<64>(st + SM::kABytes + wn * SM::kBBytes);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < SM::kKB / kWgK; ++k) wgmma_ss<BF16, kWgCols>(acc, da + 2 * k, db + 2 * k, (kb | k) != 0);   // +32 B per k-step
      wgmma_commit();
      if (kb > 0) { wgmma_wait<1>(); mbar_arrive(&empty[s == 0 ? SM::kStages - 1 : s - 1]); }
      if (++s == SM::kStages) { s = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    fence_acc(acc);
    mbar_arrive(&empty[s == 0 ? SM::kStages - 1 : s - 1]);
    // y = acc + (bias + resid) over the residual rows in the buffer; the pivot bias[0] + resid[row][0] of rows rw, rw + 8
    mbar_wait(res_full, bphase);
    if (cw == 0) { const float b0 = __ldg(p.bias); s_piv[rw] = b0 + bw[0]; s_piv[rw + 8] = b0 + bw[8 * kLd]; }
#pragma unroll
    for (int j = 0; j < kAcc / 4; ++j) {
      const float2 b = __ldg(reinterpret_cast<const float2*>(p.bias + cw + 8 * j));
      float2* y0 = reinterpret_cast<float2*>(bw + 8 * j);
      float2* y1 = reinterpret_cast<float2*>(bw + 8 * kLd + 8 * j);
      const float2 r0 = *y0, r1 = *y1;
      *y0 = make_float2(acc[4 * j] + (b.x + r0.x), acc[4 * j + 1] + (b.y + r0.y));
      *y1 = make_float2(acc[4 * j + 2] + (b.x + r1.x), acc[4 * j + 3] + (b.y + r1.y));
    }
    fence_proxy_async_smem();                                // y is visible to the bulk store of y_out
    mbar_arrive(buf_full);
    bphase ^= 1;
  }
}

}  // namespace ldm
