// wgmma (Hopper warpgroup MMA) GEMMs of the LayoutDM denoiser, C[M,N] = A[M,K] * W[N,K]^T (+ fused epilogue).
//
//   A : activations, row-major [M][K] 16-bit (fp16 or bf16), M = 128 * n_layouts (one 128-row block = one layout)
//   W : nn.Linear weight, row-major [N][K] 16-bit  (both operands are "K-major" for the MMA)
//   split mode (OP_BF16X3): A and W are bf16 (hi, lo) plane pairs; 16-bit outputs are written as (hi, lo) pairs (out, out_lo)
//
// Every kernel runs one operand ring (Ring): a shared-memory ring of k-block stages that one producer lane fills with TMA 2-D
// boxes and two consumer warpgroups drain with m64 x N x k16 wgmmas into fp32 register accumulators (full / empty mbarriers).
// In the persistent kernels the ring slot and phase run on from tile to tile, so the producer fills the ring with the next
// tile during this tile's epilogue.  A split-mode stage holds both planes of a 32-element k-block, A_hi | A_lo | W_hi | W_lo:
// the bytes (and so the stage counts) of the one-plane 64-element stage.  Each of its k16 steps is three wgmmas: a_lo w_hi,
// a_hi w_lo, a_hi w_hi.
//
// gemm_tc_kernel adds the epilogue on the consumers' own accumulator fragment.  Tile shapes:
//   WG_M = 2 : 128 rows x BN_WG columns, the warpgroups split the rows (split-mode QKV, FF1: 256 columns; vocabulary head: 160)
//   WG_M = 1 :  64 rows x 2 BN_WG columns, the warpgroups split the columns.  Used by the split mode's LN epilogue: 2 x 232 =
//              464 = d_model, so a CTA holds whole rows and the LayerNorm row statistics are combined in shared memory.
// Epilogues:  QKV (bias, q-scale, 16-bit) | RELU (FF1: bias, ReLU, 16-bit) | F32 (bias; vocabulary head) |
//             LN  (out-projection / FF2: bias + residual + LayerNorm, affine or timestep-adaptive, fused).
// It stores from the fragment.  gemm_rowblock_kernel (QKV, FF1 in fp16 / bf16) keeps each layout's A rows resident and stores
// through staging buffers with TMA (see there).  gemm_ln_kernel (out-projection, FF2 in fp16 / bf16) runs on CTA pairs that
// split a 128-row block's columns and exchange the LayerNorm row statistics through each other's shared memory, with a tile
// buffer and epilogue warps of its own (see there).
//
// Reference ops replaced: nn.Linear / nn.MultiheadAttention projections / nn.LayerNorm / AdaLayerNorm in
// T/models/transformer_utils.py:79-83,165-210 and T/models/common/nn_lib.py:187-189,235.
#pragma once
#include "common.cuh"

namespace ldm {

constexpr int kBM = 128;       // rows of one layout tile (125 tokens + 3 pad rows)
constexpr int kWgK = 16;       // K per wgmma (16-bit operands)
constexpr int kGemmConsumers = 256;
constexpr int kProducerRegs = 40, kConsumerRegs = 232;   // persistent block: 128 x 40 + 256 x 232 <= the SM's 64 K registers

// K elements per ring k-block of gemm_tc_kernel: 64 with one plane, 32 per plane in the split mode (the stage keeps its bytes)
constexpr int gemm_kb(bool split) { return split ? 32 : 64; }

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
  int n_ranges;           // gemm_rowblock_kernel: column ranges each row block is cut into (work items = row blocks x n_ranges)
};

template <bool BF16, int N>
LDM_DEVINL void wgmma_ss(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t accumulate) {
  if constexpr (N == 256) wgmma_ss_n256<BF16>(d, da, db, accumulate);
  else if constexpr (N == 232) wgmma_ss_n232<BF16>(d, da, db, accumulate);
  else if constexpr (N == 160) wgmma_ss_n160<BF16>(d, da, db, accumulate);
  else { static_assert(N == 128, "unsupported wgmma width"); wgmma_ss_n128<BF16>(d, da, db, accumulate); }
}

struct NoKbHook { LDM_DEVINL void operator()(int) const {} };

// The operand ring: STAGES stages, each [A rows][KB] per plane | [B_ROWS weight rows][KB] per plane and column warpgroup.
// One smem row is one swizzle row of 2 KB bytes: the operand maps' boxes are KB columns with the (2 KB)-byte swizzle, read by
// make_smem_desc<2 KB>.  K_TAIL: K may end in a partial k-block (K % KB is 0 or 16: K = 464, 512, 1856); a k-block that runs
// past K issues a single k16 step.  Each role keeps its own cursor (slot s, pass phase) and passes it in.  A_ROWS = 0: the
// stages hold weights only (the row-block GEMM keeps its A rows outside the ring).  CONSUMERS: the threads that release a stage.
template <int KB, int PLANES, int A_ROWS, int B_ROWS, int WG_N, int STAGES, bool K_TAIL = true, int CONSUMERS = kGemmConsumers>
struct Ring {
  static constexpr int kKB = KB, kStages = STAGES, kWgN = WG_N;
  static constexpr int kRowBytes = 2 * KB;
  static constexpr int kAPlane = A_ROWS * kRowBytes;
  static constexpr int kABytes = PLANES * kAPlane;                  // A_hi (| A_lo)
  static constexpr int kBBytes = B_ROWS * kRowBytes;                // one warpgroup's weight rows of one plane
  static constexpr int kStageBytes = kABytes + PLANES * WG_N * kBBytes;   // ... | W_hi blocks (| W_lo blocks)
  static constexpr int kBytes = STAGES * kStageBytes;
  static_assert(kAPlane % (8 * kRowBytes) == 0 && kBBytes % (8 * kRowBytes) == 0, "boxes must keep the swizzle atom's alignment");

  uint8_t* stages;
  uint64_t* full;                                                   // [STAGES] the stage's TMA bytes have landed
  uint64_t* empty;                                                  // [STAGES] both warpgroups' MMAs have read the stage

  LDM_DEVINL Ring(uint8_t* smem, uint64_t* bars) : stages(smem), full(bars), empty(bars + STAGES) {}
  static LDM_DEVINL int num_kb(int K) { return K_TAIL ? (K + KB - 1) / KB : K / KB; }

  template <int MODE>
  static LDM_DEVINL void prefetch(const OpMaps<MODE>& a, const OpMaps<MODE>& b) {
    tma_prefetch_desc(&a.hi);
    tma_prefetch_desc(&b.hi);
    if constexpr (kOpSplit<MODE>) { tma_prefetch_desc(&a.lo); tma_prefetch_desc(&b.lo); }
  }
  LDM_DEVINL void init() const {
    for (int i = 0; i < STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], CONSUMERS); }
  }
  static LDM_DEVINL void advance(int& s, uint32_t& phase) { if (++s == STAGES) { s = 0; phase ^= 1; } }
  LDM_DEVINL void release_prev(int s) const { mbar_arrive(&empty[s == 0 ? STAGES - 1 : s - 1]); }

  // producer lane: the num_kb k-blocks of one tile, A rows m0.., weight block wn's rows n0 + wn * B_ROWS..; on_kb(kb) runs
  // before k-block kb's stage is claimed
  template <int MODE, class OnKb = NoKbHook>
  LDM_DEVINL void load_tile(int& s, uint32_t& phase, const OpMaps<MODE>& a, const OpMaps<MODE>& b, int num_kb, int m0, int n0,
                            OnKb on_kb = {}) const {
    static_assert(PLANES == (kOpSplit<MODE> ? 2 : 1), "one operand map per plane");
    for (int kb = 0; kb < num_kb; ++kb) {
      on_kb(kb);
      mbar_wait(&empty[s], phase ^ 1);
      uint8_t* st = stages + s * kStageBytes;
      mbar_arrive_expect_tx(&full[s], kStageBytes);              // out-of-bounds box parts are zero-filled and still counted
      if constexpr (A_ROWS > 0) tma_load_2d(st, &a.hi, &full[s], kb * KB, m0);
#pragma unroll
      for (int wn = 0; wn < WG_N; ++wn) tma_load_2d(st + kABytes + wn * kBBytes, &b.hi, &full[s], kb * KB, n0 + wn * B_ROWS);
      if constexpr (PLANES == 2 && A_ROWS > 0) tma_load_2d(st + kAPlane, &a.lo, &full[s], kb * KB, m0);
      if constexpr (PLANES == 2) {
#pragma unroll
        for (int wn = 0; wn < WG_N; ++wn)
          tma_load_2d(st + kABytes + (WG_N + wn) * kBBytes, &b.lo, &full[s], kb * KB, n0 + wn * B_ROWS);
      }
      advance(s, phase);
    }
  }

  // consumer warpgroup (A rows wm * 64.., weight block wn): the MMAs of one tile's num_kb k-blocks into acc.  A k-block's MMAs
  // stay in flight while the next k-block's are issued; once they have retired its stage goes back to the producer.  The
  // tile's last stage goes back before the epilogue, so the producer refills it with the next tile meanwhile.
  template <int MODE>
  LDM_DEVINL void mma_tile(int& s, uint32_t& phase, float (&acc)[B_ROWS / 2], int wm, int wn, int num_kb, int K) const {
    static_assert(PLANES == (kOpSplit<MODE> ? 2 : 1), "one operand map per plane");
    for (int kb = 0; kb < num_kb; ++kb) {
      mbar_wait(&full[s], phase);
      const uint32_t st = smem_u32(stages + s * kStageBytes);
      const uint64_t da = make_smem_desc<kRowBytes>(st + wm * 64 * kRowBytes), da_lo = make_smem_desc<kRowBytes>(st + kAPlane + wm * 64 * kRowBytes);
      const uint64_t db = make_smem_desc<kRowBytes>(st + kABytes + wn * kBBytes);
      const uint64_t db_lo = make_smem_desc<kRowBytes>(st + kABytes + (WG_N + wn) * kBBytes);
      wgmma_fence();
      // k16 step k: +32 B (>>4 = 2); two planes: three wgmmas, the small terms first
      const auto step = [&](int k) {
        if constexpr (PLANES == 2) {
          wgmma_ss<true, B_ROWS>(acc, da_lo + 2 * k, db + 2 * k, (kb | k) != 0);
          wgmma_ss<true, B_ROWS>(acc, da + 2 * k, db_lo + 2 * k, 1);
          wgmma_ss<true, B_ROWS>(acc, da + 2 * k, db + 2 * k, 1);
        } else {
          wgmma_ss<kOpBf16<MODE>, B_ROWS>(acc, da + 2 * k, db + 2 * k, (kb | k) != 0);
        }
      };
      // two-plane stages issue their first step ahead of the K-tail branch, one-plane stages inside it: other shapes of the same
      // rule change ptxas's wgmma schedule.  Without K_TAIL there is no branch (ptxas serialises the LN kernel's wgmmas around one)
      const bool whole = !K_TAIL || kb * KB + KB <= K;
      if (PLANES == 2 || !whole) step(0);
      if (whole) {
#pragma unroll
        for (int k = PLANES == 2 ? 1 : 0; k < KB / kWgK; ++k) step(k);
      }
      wgmma_commit();
      if (kb > 0) { wgmma_wait<1>(); release_prev(s); }
      advance(s, phase);
    }
    wgmma_wait<0>();
    fence_acc(acc);
    release_prev(s);
  }
};

// gemm_tc_kernel stores from the fragment and has nothing to overlap its epilogue with: one tile per CTA, 288 threads (one
// producer warp)
constexpr int kGemmThreads = 288;

template <int BN_WG, int WG_M, int STAGES, bool SPLIT = false>
struct GemmSmem {
  using R = Ring<gemm_kb(SPLIT), SPLIT ? 2 : 1, 64 * WG_M, BN_WG, 3 - WG_M, STAGES>;
  static constexpr int kOffBars = R::kBytes;
  static constexpr int kOffStat = kOffBars + 256;                // LN: per-row sum, then sum of squared deviations, of each warpgroup's columns
  static constexpr int kBytes = kOffStat + 2 * 64 * 16 + 1024 /*align slack*/;
  static_assert(2 * STAGES * 8 <= 256, "barrier block overflow");
  static_assert(kBytes <= 232448, "exceeds the 227 KB of shared memory per CTA");
};

// bias (q-scale | ReLU) of n8 block j of a plain epilogue's fragment: v = rows rw, rw + 8 x columns c, c + 1
template <int EPI, int N>
LDM_DEVINL void bias_act(const float (&acc)[N], int j, const float* bias, int c, float scale, float (&v)[4]) {
  const float2 b = bias != nullptr ? __ldg(reinterpret_cast<const float2*>(bias + c)) : make_float2(0.0f, 0.0f);
  v[0] = acc[4 * j] + b.x; v[1] = acc[4 * j + 1] + b.y; v[2] = acc[4 * j + 2] + b.x; v[3] = acc[4 * j + 3] + b.y;
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    if constexpr (EPI == EPI_QKV) v[e] *= scale;
    if constexpr (EPI == EPI_RELU) v[e] = fmaxf(v[e], 0.0f);
  }
}

// the LayerNorm's (gamma, beta) rows of the tile at row m0 and the offset added to gamma (AdaLN: gamma = 1 + scale)
struct LnAffine { const float* gam; const float* bet; float gadd; };
LDM_DEVINL LnAffine ln_affine(const float* scale, const float* shift, int adaln, const int* t_layout, int n_layouts, int m0, int N) {
  LnAffine a{scale, shift, adaln ? 1.0f : 0.0f};
  if (t_layout != nullptr) {                                 // per-layout timesteps: this layout's AdaLN (scale, shift) row
    const int layout = m0 / kBM;
    const int tl = layout < n_layouts ? __ldg(t_layout + layout) : 0;
    a.gam = scale + static_cast<size_t>(tl) * 2 * N; a.bet = a.gam + N; a.gadd = 1.0f;
  }
  return a;
}

// grid: one CTA per tile, tiles = n_tiles * M / (64 WG_M)
template <int BN_WG, int WG_M, int STAGES, int EPI, int MODE>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_tc_kernel(const __grid_constant__ OpMaps<MODE> map_a /*box KB x 64 WG_M rows*/,
               const __grid_constant__ OpMaps<MODE> map_b /*box KB x BN_WG rows*/, const GemmParams p) {
  constexpr bool SPLIT = kOpSplit<MODE>;
  using SM = GemmSmem<BN_WG, WG_M, STAGES, SPLIT>;
  using O = OpT<MODE>;
  constexpr int kBMt = 64 * WG_M, kAcc = BN_WG / 2;
  static_assert(EPI != EPI_LN || (WG_M == 1 && BN_WG == 232), "LN epilogue is laid out for 464 = 2 x 232 columns");
  static_assert(EPI == EPI_LN || WG_M == 2, "plain epilogues use 128-row tiles");

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  typename SM::R ring(smem, reinterpret_cast<uint64_t*>(smem + SM::kOffBars));

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
  const int num_kb = SM::R::num_kb(p.K);
  const int n_mblk = p.M / kBMt;
  // tile blockIdx.x: row block blockIdx.x / n_tiles (walked from the last one down when rev), column tile blockIdx.x % n_tiles
  const int mb = blockIdx.x / p.n_tiles;
  const int m0 = (p.rev ? n_mblk - 1 - mb : mb) * kBMt, n0 = (blockIdx.x % p.n_tiles) * BN_WG * SM::R::kWgN;

  if (threadIdx.x == kGemmConsumers) {
    ring.prefetch(map_a, map_b);
    ring.init();
    fence_mbar_init();
  }
  __syncthreads();
  pdl_sync();                                                // everything above overlapped the previous kernel's tail

  int s = 0;
  uint32_t phase = 0;
  if (warp >= kGemmConsumers / 32) {
    // ===================== TMA producer =====================
    if (threadIdx.x == kGemmConsumers) ring.load_tile(s, phase, map_a, map_b, num_kb, m0, n0);
    return;
  }

  // ===================== consumer warpgroups =====================
  const int wg = warp >> 2;
  const int wm = WG_M == 2 ? wg : 0, wn = WG_M == 2 ? 0 : wg;
  float acc[kAcc];
#pragma unroll
  for (int i = 0; i < kAcc; ++i) acc[i] = 0.0f;
  ring.template mma_tile<MODE>(s, phase, acc, wm, wn, num_kb, p.K);

  const int rw = (warp & 3) * 16 + (lane >> 2);           // fragment rows rw and rw + 8 of the warpgroup's 64
  const int row0 = m0 + wm * 64 + rw, row1 = row0 + 8;
  const int col0 = n0 + wn * BN_WG + 2 * (lane & 3);        // + 8 j: columns col, col + 1 of n8 block j

  if constexpr (EPI != EPI_LN) {
    float scale = 1.0f;
    if constexpr (EPI == EPI_QKV) scale = (n0 < p.qcols) ? p.qscale : 1.0f;   // Q tiles are whole tiles (512 % 256 == 0)
#pragma unroll
    for (int j = 0; j < BN_WG / 8; ++j) {
      const int c = col0 + 8 * j;
      if (c >= p.N) continue;                               // N is even: the pair (c, c + 1) is in or out together
      float v[4];
      bias_act<EPI>(acc, j, p.bias, c, scale, v);
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
    const LnAffine a = ln_affine(p.ln_scale, p.ln_shift, p.adaln, p.t_layout, p.n_layouts, m0, N);
    typename O::T* out16 = static_cast<typename O::T*>(p.out);
#pragma unroll
    for (int j = 0; j < BN_WG / 8; ++j) {
      const int c = col0 + 8 * j;
      const float2 g = __ldg(reinterpret_cast<const float2*>(a.gam + c)), h = __ldg(reinterpret_cast<const float2*>(a.bet + c));
      const float v0 = (acc[4 * j] - mean0) * rstd0 * (g.x + a.gadd) + h.x, v1 = (acc[4 * j + 1] - mean0) * rstd0 * (g.y + a.gadd) + h.y;
      const float v2 = (acc[4 * j + 2] - mean1) * rstd1 * (g.x + a.gadd) + h.x, v3 = (acc[4 * j + 3] - mean1) * rstd1 * (g.y + a.gadd) + h.y;
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
}

// ============ row-block GEMM: QKV and FF1 in the one-plane modes ============
// K = d = 464 is small enough for a layout's whole A row block (128 x 464, 119 KB) to stay in shared memory, so a CTA loads it
// once per work item and streams only the weights.  Work item = one 128-row block and a contiguous range of its 128-column
// tiles (n_ranges ranges per row block); min(items, SMs) CTAs of 384 threads, CTA b runs items b, b + gridDim.x, ...
//   warpgroup 2 : producer, one lane issues the TMA loads.  An item's A k-block kb is loaded just before the k-block kb of the
//                 item's first tile, as soon as both consumer warpgroups have released it (a_empty[kb]: their MMAs of the
//                 previous item reading it have retired), so the next item's first tile waits k-block by k-block.
//   warpgroups 0, 1 : consumers, ping-pong: the CTA's tiles are numbered in order across its items and warpgroup w takes the
//                 tiles q with q % 2 == w, each a whole 128 x 128 tile (two m64n128k16 wgmmas per k16 step, 128 fp32
//                 accumulators).  The weight ring serialises their mainloops; a named barrier hands the ring from one to the
//                 other once it has seen its tile's last stage arrive, so a warpgroup's ring waits never run a pass ahead of
//                 the slot's phase.  Each runs its epilogue (bias, q-scale | ReLU, 16-bit, through its own staging buffer, one
//                 TMA store per 64 columns) under the other's MMAs.
// Resident A: 8 k-blocks of 64 elements with the 128-byte swizzle, the 8th holding K's 16-column tail (the rest zero-filled by
// TMA; one k16 step, Ring's K_TAIL rule).  Every output element is bias + the same k16 steps in the same order as in gemm_tc_kernel.
constexpr int kRbThreads = 384;
struct RbSmem {
  static constexpr int kKB = 64, kCols = 128, kAKb = 8;            // k-block, tile columns, resident A k-blocks (K <= 512)
  // weights only, one warpgroup consumes a stage: 4 stages of 16 KB.  64-element (128-byte) box rows: with 32-element ones the
  // TMA loads ran well below the L2 rate
  using R = Ring<kKB, 1, 0, kCols, 1, 4, true, 128>;
  static constexpr int kAKbBytes = kBM * 2 * kKB;                  // 16 KB
  static constexpr int kOffRing = kAKb * kAKbBytes;                // 128 KB of A
  // staging buffer of a warpgroup: one 64-column block of its tile, [row][128 B] with the 128-byte swizzle = one TMA store box
  // (64 columns x 128 rows); the tile's two blocks go through it in turn
  static constexpr int kStoreBytes = kBM * 128;                    // 16 KB
  static constexpr int kOffStore = kOffRing + R::kBytes;
  static constexpr int kOffBars = kOffStore + 2 * kStoreBytes;     // ring full[4], empty[4]; a_full[8], a_empty[8]
  static constexpr int kBytes = kOffBars + (2 * R::kStages + 2 * kAKb) * 8 + 1024 /*align slack*/;
  static_assert(kBytes <= 232448, "exceeds the 227 KB of shared memory per CTA");
};

template <int EPI, int MODE>
__global__ void __launch_bounds__(kRbThreads, 1)
gemm_rowblock_kernel(const __grid_constant__ OpMaps<MODE> map_a /*box 32 x 128 rows*/, const __grid_constant__ OpMaps<MODE> map_b /*box 32 x 128 rows*/,
                     const __grid_constant__ CUtensorMap map_out /*box 64 x 128 rows*/, const GemmParams p) {
  static_assert(EPI == EPI_QKV || EPI == EPI_RELU, "16-bit plain epilogues only");
  static_assert(!kOpSplit<MODE>, "the split mode runs gemm_tc_kernel");
  using SM = RbSmem;
  using R = SM::R;
  using O = OpT<MODE>;
  constexpr int kKB = SM::kKB, kCols = SM::kCols;

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + SM::kOffBars);
  R ring(smem + SM::kOffRing, bars);
  uint64_t* a_full = bars + 2 * R::kStages;                      // A k-block kb of the current item has landed
  uint64_t* a_empty = a_full + SM::kAKb;                          // both warpgroups are done reading A k-block kb

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
  const int num_kb = R::num_kb(p.K);                              // <= kAKb (checked at create)
  const int n_mblk = p.M / kBM, n_items = n_mblk * p.n_ranges;
  // item w: row block w / n_ranges (walked from the last one down when rev), tiles [j0, j1) of range w % n_ranges
  const auto item = [&](int w, int& m0, int& j0, int& j1) {
    const int mb = w / p.n_ranges, r = w - mb * p.n_ranges;
    m0 = (p.rev ? n_mblk - 1 - mb : mb) * kBM;
    j0 = r * p.n_tiles / p.n_ranges; j1 = (r + 1) * p.n_tiles / p.n_ranges;
  };

  if (threadIdx.x == kGemmConsumers) {
    R::prefetch(map_a, map_b);
    tma_prefetch_desc(&map_out);
    ring.init();
    for (int kb = 0; kb < SM::kAKb; ++kb) { mbar_init(&a_full[kb], 1); mbar_init(&a_empty[kb], kGemmConsumers); }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_sync();                                                // everything above overlapped the previous kernel's tail

  if (warp >= kGemmConsumers / 32) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<kProducerRegs>();
    if (threadIdx.x == kGemmConsumers) {
      int s = 0;
      uint32_t phase = 0, ip = 0;                            // ring slot and pass; parity of the CTA's item count
      for (int w = blockIdx.x; w < n_items; w += gridDim.x, ip ^= 1) {
        int m0, j0, j1;
        item(w, m0, j0, j1);
        for (int j = j0; j < j1; ++j) {
          const auto load_a = [&](int kb) {                  // the item's A k-block kb, ahead of its first tile's k-block kb
            if (j != j0) return;
            mbar_wait(&a_empty[kb], ip ^ 1);
            mbar_arrive_expect_tx(&a_full[kb], SM::kAKbBytes);   // the tail k-block's zero-filled columns are counted too
            tma_load_2d(smem + kb * SM::kAKbBytes, &map_a.hi, &a_full[kb], kb * kKB, m0);
          };
          ring.load_tile(s, phase, map_b, map_b, num_kb, 0, j * kCols, load_a);
        }
      }
    }
    return;
  }

  // ===================== consumer warpgroups =====================
  setmaxnreg_inc<kConsumerRegs>();
  const int wg = warp >> 2;
  const bool leader = (threadIdx.x & 127) == 0;
  // ring hand-over: warpgroup wg waits on barrier 4 + wg before its tile's mainloop, the other arrives on it after its own
  // (compile-time ids; 2, 3 are the warpgroups' epilogue barriers)
  const auto wait_turn = [&]() { if (wg == 0) named_bar_sync(4, kGemmConsumers); else named_bar_sync(5, kGemmConsumers); };
  const auto pass_turn = [&]() { if (wg == 0) named_bar_arrive(5, kGemmConsumers); else named_bar_arrive(4, kGemmConsumers); };
  const auto wg_bar = [&]() { if (wg == 0) named_bar_sync(2, 128); else named_bar_sync(3, 128); };
  int n_cta_tiles = 0;
  for (int w = blockIdx.x; w < n_items; w += gridDim.x) { int m0, j0, j1; item(w, m0, j0, j1); n_cta_tiles += j1 - j0; }

  float acc[2][kCols / 2];
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int i = 0; i < kCols / 2; ++i) acc[h][i] = 0.0f;
  const uint32_t a_base = smem_u32(smem);
  uint8_t* stage = smem + SM::kOffStore + wg * SM::kStoreBytes;
  const uint32_t stage_u32 = smem_u32(stage);                  // 32-bit shared addresses: 64-bit generic ones cost registers
  const int rw = (warp & 3) * 16 + (lane >> 2);                 // fragment rows rw, rw + 8 of each 64-row half
  const int sw = (rw & 7) << 4;                                 // 128-byte swizzle: 16-byte chunk ^= row % 8 (the same for all four rows)
  int s = 0, q = 0;                                             // ring cursor; the CTA's tile count so far
  uint32_t phase = 0, ip = 0;
  for (int w = blockIdx.x; w < n_items; w += gridDim.x, ip ^= 1) {
    int m0, j0, j1;
    item(w, m0, j0, j1);
    bool mine_any = false;
    for (int j = j0; j < j1; ++j, ++q) {
      if ((q & 1) != wg) {                                      // the other warpgroup's tile: its stages pass by
        for (int kb = 0; kb < num_kb; ++kb) R::advance(s, phase);
        continue;
      }
      mine_any = true;
      const bool last_mine = j + 2 >= j1;                        // this warpgroup's last read of the item's A rows
      const int n0 = j * kCols;
      if (q > 0) wait_turn();
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&a_full[kb], ip);
        mbar_wait(&ring.full[s], phase);
        const uint64_t da = make_smem_desc<2 * kKB>(a_base + kb * SM::kAKbBytes);
        const uint64_t db = make_smem_desc<2 * kKB>(smem_u32(ring.stages + s * R::kStageBytes));
        wgmma_fence();
        // k16 step k: +32 B (>>4 = 2); rows 64.. of A are 64 rows x 128 B = 8 KB (>>4 = 512) on
        const auto step = [&](int k) {
          wgmma_ss<kOpBf16<MODE>, kCols>(acc[0], da + 2 * k, db + 2 * k, (kb | k) != 0);
          wgmma_ss<kOpBf16<MODE>, kCols>(acc[1], da + 512 + 2 * k, db + 2 * k, (kb | k) != 0);
        };
        const bool whole = kb * kKB + kKB <= p.K;
        if (!whole) step(0);
        if (whole) {
#pragma unroll
          for (int k = 0; k < kKB / kWgK; ++k) step(k);
        }
        wgmma_commit();
        if (kb > 0) {
          wgmma_wait<1>();
          ring.release_prev(s);
          if (last_mine) mbar_arrive(&a_empty[kb - 1]);
        }
        R::advance(s, phase);
      }
      if (q + 1 < n_cta_tiles) pass_turn();
      wgmma_wait<0>();
      fence_acc(acc[0]);
      fence_acc(acc[1]);
      ring.release_prev(s);
      if (last_mine) mbar_arrive(&a_empty[num_kb - 1]);

      // epilogue: bias (q-scale | ReLU), 16-bit, one 64-column block at a time into the staging buffer, which the leader then
      // stores with TMA.  N is a multiple of 64 (checked at create): a block past N (FF1's last tile) is not computed
      float scale = 1.0f;
      if constexpr (EPI == EPI_QKV) scale = (n0 < p.qcols) ? p.qscale : 1.0f;   // Q tiles are whole tiles (512 % 128 == 0)
      const int col0 = n0 + 2 * (lane & 3);                      // + 8 j: columns c, c + 1 of n8 block j
#pragma unroll
      for (int cb = 0; cb < kCols / 64; ++cb) {
        if (n0 + cb * 64 >= p.N) continue;
        if (leader) bulk_wait_group_read<0>();                 // the previous store has read the staging buffer
        wg_bar();
#pragma unroll
        for (int j8 = 8 * cb; j8 < 8 * cb + 8; ++j8) {
          const int c = col0 + 8 * j8;
          const uint32_t blk = stage_u32 + ((((j8 & 7) << 4) ^ sw) | (4 * (lane & 3)));
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float v[4];
            bias_act<EPI>(acc[h], j8, p.bias, c, scale, v);
            st_shared_u32(blk + (h * 64 + rw) * 128, O::pack(v[0], v[1]));
            st_shared_u32(blk + (h * 64 + rw + 8) * 128, O::pack(v[2], v[3]));
          }
        }
        fence_proxy_async_smem();
        wg_bar();
        if (leader) {
          tma_store_2d(&map_out, stage, n0 + cb * 64, m0);
          bulk_commit_group();
        }
      }
    }
    if (!mine_any) {                                             // no tile of this item: release its A rows unread
      for (int kb = 0; kb < num_kb; ++kb) { mbar_wait(&a_full[kb], ip); mbar_arrive(&a_empty[kb]); }
    }
  }
  if (leader) bulk_wait_group_all();                           // the last stores are complete before the CTA exits
}

// ============ persistent LN GEMM: out-projection / FF2 in the one-plane modes ============
// A cluster of two CTAs takes one layout's 128-row block at a time and splits its 464 columns: CTA rank h computes columns
// 232 h .. 232 h + 231 of all 128 rows, so every weight k-block it streams from L2 feeds 128 rows (FF2 reads 1.34 MB per CTA
// tile against 1.96 MB for a 64 x 464 tile of the same floats).  Clusters: min(row blocks, active clusters); cluster c runs the
// row blocks c, c + clusters, ...  384 threads per CTA.  The LayerNorm runs in warps of its own and the fp32 traffic goes
// through TMA, so a tile's epilogue overlaps the next tile's MMAs:
//   warps 0..7  : two MMA warpgroups, warpgroup w rows 64 w .. 64 w + 63 x the CTA's 232 columns, m64n232k16 from the ring.
//                 After a tile's last k-block warpgroup w waits for the residual rows of its row half w in the tile buffer,
//                 replaces them by y = acc + (bias + resid), sends the rows' sums of y - pivot (below) and goes straight on
//                 to the next tile.
//   warps 8..10 : epilogue: the row statistics, the LayerNorm / AdaLN and the 16-bit stores from the tile buffer, one row half
//                 at a time: (tile t, half 0), (t, 1), (t + 1, 0), ...  Thread 0 of warp 8 also moves the fp32 row halves
//                 between the buffer and global memory, one 2-D TMA box of 64 rows x the CTA's 232 columns each (map_res,
//                 map_st; no swizzle, so a box is the half's dense [64][232] rows): the half's y out (the next residual) or
//                 its normalised fp32 rows (written back into the buffer) out -- the host sets at most one of the two, so
//                 the normalise pass never overwrites rows a store still reads -- and, as soon as that store has read the
//                 half, the next tile's residual rows of the same half in.  So the load of half w and warpgroup w's y pass
//                 run while the epilogue works on the other half.
//   warp 11     : producer, one lane issues the TMA loads.
// The tile buffer is two row halves, [2][64][232] fp32, each with its own barriers: res_full[w] (its residual rows have
// landed; armed by the copying thread), buf_full[w] (warpgroup w wrote y; 128 arrivals).  A half is free again once the copying
// thread's wait_group.read of its store returns after the named barrier that ends the epilogue's pass over it; that thread
// loads the half's next residual rows only then, so the hand-off is program order in one thread.  Both warpgroups consume every ring
// stage, so one can run at most the ring's depth ahead of the other.
// 168 registers for every warp, no setmaxnreg: ptxas compiles the whole kernel under the launch bound's register count, and a
// 512-thread block (a whole producer warpgroup) would leave the m64n232 wgmma 128, fewer than it needs.  Three epilogue warps
// cannot keep enough loads and stores in flight to move a tile's fp32 rows at HBM rate themselves; the TMA copies need no
// registers.  Ring: STAGES stages of 32-element k-blocks with the 64-byte swizzle (8 KB of A + 14.5 KB of W each) beside the
// 116 KB tile buffer; 4 fit.  (With one 1-D bulk copy per 928-byte row, issuing a half's 64 loads took warp 8 about 2 us per
// row half (H100 SXM), on the epilogue's critical path.)  The split mode keeps the fragment-epilogue kernel above: its two-plane stages do not fit beside the buffer.
//
// The results are bit for bit those of the fragment epilogue: the same k16 MMA sequence, y = acc + (bias + resid), and the row
// statistics keep its summation order (per row 8 chains (h, q), h = column half, q = quad lane, each summing
// (y_c - piv) + (y_c+1 - piv) over c = 232 h + 8 j + 2 q, j ascending; (q0 + q1) + (q2 + q3), then half + half) and its FMA
// contractions (y - mean is one fma(-sum, 1/N, y - piv), the output fma(d * rstd, gamma + gadd, beta)).  The pivot is
// bias[0] + resid[row][0] in both CTAs, read from global memory (rank 1 does not hold column 0).  Column half h of a row lives
// in CTA h: each CTA forms its half's quad-combined partial, stores it into the peer's slot with st.async (completion counted
// on the peer's mbarrier) and adds the two, own + peer -- the same float in both CTAs, since addition commutes.  The row sums
// are formed by the MMA warpgroups from y in registers (a fragment thread's columns 2 q + 8 j are exactly chain q) and sent
// before the epilogue starts, so the epilogue reads the buffer once for the statistics, not twice, and rarely waits for
// the peer's sums.  The epilogue warps form and exchange the sums of squared deviations the same way.
// Exchange slots: two per statistic, by tile parity b, indexed by row; each (b, row half w) has an mbarrier that its own CTA
// arms (expect_tx) when its epilogue starts on half w of a tile of parity b; the peer's bytes may land before that, which the
// transaction count allows.  Overrun: the peer writes the row-sum slots (b, w) for tile i + 2 from its warpgroup w after that
// half's residual rows of tile i + 2 have landed, which its warp 8 loads only after its epilogue has finished (i + 1, w), and
// that needed this CTA's variance partials of (i + 1, w).  It writes the variance slots (b, w) for tile i + 2 in its
// epilogue's pass over (i + 2, w), which comes after (i + 1, w) as well.  This CTA sends its partials of (i + 1, w) only after
// every epilogue thread has passed the named barriers that end (i, w) (and (i, 1 - w)), so after every read of the slots
// (b, w) for tile i: two slots cannot be overrun.
// Cluster barriers: after the barrier init (no remote store before the peer's barriers exist) and before exit (no CTA leaves
// while its peer may still store into its shared memory); every thread reaches both.
constexpr int kLnThreads = 384, kLnEpiThreads = 96;

// Phase probe (tools/ln_phase_probe.py), compiled in only with -DLDM_LN_PROBE: rank 0 of the first kLnProbePairs pairs records
// %globaltimer stamps per tile and row half; each launch overwrites its GEMM's entries, so after a step they hold the
// step's last out-projection (K = 512) and last FF2 launch.
enum : int { LNP_MAIN = 0, LNP_RES, LNP_Y, LNP_BUF, LNP_XS, LNP_XV, LNP_NORM, LNP_WAIT, LNP_NEXT, LNP_N };
constexpr int kLnProbePairs = 8, kLnProbeTiles = 32;
#ifdef LDM_LN_PROBE
__device__ unsigned long long g_ln_probe[2][kLnProbePairs][kLnProbeTiles][2][LNP_N];
#endif
LDM_DEVINL void ln_probe(int K, uint32_t rank, int cl, int it, int half, int stamp) {
#ifdef LDM_LN_PROBE
  if (rank == 0 && cl < kLnProbePairs && it < kLnProbeTiles) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    g_ln_probe[K == 512 ? 0 : 1][cl][it][half][stamp] = t;
  }
#endif
}

template <int STAGES>
struct LnSmem {
  static constexpr int kRows = kBM, kHalf = kRows / 2, kCols = 232, kPairCols = 2 * kCols;
  using R = Ring<32, 1, kRows, kCols, 1, STAGES, false>;       // K = 512, 1856 (checked at create)
  // tile buffer [2 row halves][64][kLd] fp32, unpadded: a row is 928 bytes = 32 mod 128, so the 4 rows of a half warp's fragment
  // access fall in distinct 32-byte bank groups; a half is one TMA box (rows of 16-byte multiples, 128-byte aligned start)
  static constexpr int kLd = kCols;
  static constexpr int kOffBuf = R::kBytes;
  // ring full[4], empty[4]; res_full[2], buf_full[2]; xs_full[2][2], xv_full[2][2]
  static constexpr int kOffBars = kOffBuf + kRows * kLd * 4;
  static constexpr int kOffStat = kOffBars + 256;
  // per row: pivot, own half's sum of y - pivot, row sum, own half's sum of squared deviations (then rstd); the peer's partials
  // [2][kRows] x 2
  static constexpr int kBytes = kOffStat + 8 * kRows * 4 + 1024 /*align slack*/;
  static_assert(2 * R::kStages * 8 + 12 * 8 <= 256, "barrier block overflow");
  static_assert(kLd * 4 % 16 == 0 && kHalf * kLd * 4 % 128 == 0 && kLd * 4 % 128 == 32,
                "TMA boxes need 16-byte multiple rows and 128-byte aligned halves; fragment accesses need rows 32 mod 128 bytes");
  static_assert(kHalf * kCols * 4 < (1 << 20), "a row half's residual bytes exceed the mbarrier transaction count");
};

template <int MODE, int STAGES>
__global__ void __launch_bounds__(kLnThreads, 1)
gemm_ln_kernel(const __grid_constant__ OpMaps<MODE> map_a /*box 32 x 128 rows*/, const __grid_constant__ OpMaps<MODE> map_b /*box 32 x 232 rows*/,
               const __grid_constant__ CUtensorMap map_res /*p.resid, fp32, box 232 x 64 rows*/,
               const __grid_constant__ CUtensorMap map_st /*p.y_out or p.out32, whichever is set*/, const GemmParams p) {
  static_assert(!kOpSplit<MODE>, "the split mode runs the fragment-epilogue LN GEMM");
  using SM = LnSmem<STAGES>;
  using O = OpT<MODE>;
  constexpr int kRows = SM::kRows, kHalf = SM::kHalf, kCols = SM::kCols, kLd = SM::kLd, kAcc = kCols / 2;
  constexpr int kEpi = kGemmConsumers, kProducer = kEpi + kLnEpiThreads;   // first thread of the epilogue warps / producer warp

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  typename SM::R ring(smem, reinterpret_cast<uint64_t*>(smem + SM::kOffBars));
  uint64_t* res_full = ring.empty + SM::R::kStages;             // [2] row half w's residual rows have landed in the buffer
  uint64_t* buf_full = res_full + 2;                             // [2] MMA warpgroup w wrote y into row half w
  uint64_t* xs_full = buf_full + 2;                              // [2 b][2 w] the peer's row sums of tile parity b, row half w have landed
  uint64_t* xv_full = xs_full + 4;                               // [2][2] the peer's sums of squared deviations
  float* buf = reinterpret_cast<float*>(smem + SM::kOffBuf);
  float* s_piv = reinterpret_cast<float*>(smem + SM::kOffStat);
  float* s_own = s_piv + kRows;
  float* s_sum = s_own + kRows;
  float* s_var = s_sum + kRows;                                  // own half's sum of squared deviations, then the row's rstd
  float* x_sum = s_var + kRows;                                  // [2][kRows] written by the peer
  float* x_var = x_sum + 2 * kRows;                              // [2][kRows] written by the peer

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
  const int N = p.N;
  const int num_kb = SM::R::num_kb(p.K);
  const int n_work = p.M / kRows;
  const uint32_t rank = cluster_ctarank();
  const int col0 = kCols * static_cast<int>(rank);               // the CTA's first column
  const int cl = static_cast<int>(cluster_id_x()), n_cl = static_cast<int>(cluster_count_x());
  const auto tile_m0 = [&](int t) { return (p.rev ? n_work - 1 - t : t) * kRows; };
  const uint32_t peer = rank ^ 1;
  const uint32_t px_sum = map_peer(x_sum, peer), pxs_full = map_peer(xs_full, peer);

  if (threadIdx.x == kProducer) {
    ring.prefetch(map_a, map_b);
    tma_prefetch_desc(&map_res);
    tma_prefetch_desc(&map_st);
    ring.init();
    for (int w = 0; w < 2; ++w) { mbar_init(&res_full[w], 1); mbar_init(&buf_full[w], kGemmConsumers / 2); }
    for (int x = 0; x < 4; ++x) { mbar_init(&xs_full[x], 1); mbar_init(&xv_full[x], 1); }
    fence_mbar_init();
  }
  cluster_sync();                                            // both CTAs' barriers are initialised before any remote store
  pdl_sync();                                                // everything above overlapped the previous kernel's tail

  if (threadIdx.x >= kProducer) {
    // ===================== TMA producer =====================
    if (threadIdx.x == kProducer) {
      uint32_t phase = 0;
      int s = 0;
      for (int t = cl; t < n_work; t += n_cl) ring.load_tile(s, phase, map_a, map_b, num_kb, tile_m0(t), col0);
    }
  } else if (threadIdx.x >= kEpi) {
    // ===================== epilogue warps =====================
    const int et = threadIdx.x - kEpi;
    const bool copier = et == 0;                             // the row halves' TMA loads and stores
    constexpr uint32_t kHalfBytes = kHalf * kCols * sizeof(float);
    const float inv_n = 1.0f / static_cast<float>(N);
    constexpr int kVec = kCols / 4;                          // float4 columns of the CTA's part of a row (58)
    constexpr int kTotal = kHalf * kVec;                     // float4 of a row half; element i = k * 96 + et
    constexpr int kPerThread = (kTotal + kLnEpiThreads - 1) / kLnEpiThreads;
    const uint32_t px_var = map_peer(x_var, peer), pxv_full = map_peer(xv_full, peer);
    // the residual rows of row half w of tile t into the buffer (the half is free: every read of it and every store from it is
    // done)
    const auto load_resid = [&](int t, int w) {
      mbar_arrive_expect_tx(&res_full[w], kHalfBytes);
      tma_load_2d(buf + kHalf * w * kLd, &map_res, &res_full[w], col0, tile_m0(t) + kHalf * w);
    };
    const auto store_rows = [&](int m0, int w) {             // row half w of the buffer to map_st's rows of tile m0, one bulk group
      tma_store_2d(&map_st, buf + kHalf * w * kLd, col0, m0 + kHalf * w);
      bulk_commit_group();
    };
    if (copier) { load_resid(cl, 0); load_resid(cl, 1); }
    uint32_t bphase = 0;
    int it = 0;                                              // the CTA's tile count: exchange slot it & 1, its pass (it >> 1) & 1
    for (int t = cl; t < n_work; t += n_cl, ++it) {
      const int m0 = tile_m0(t), b = it & 1;
      const uint32_t xph = (it >> 1) & 1;
      const LnAffine a = ln_affine(p.ln_scale, p.ln_shift, p.adaln, p.t_layout, p.n_layouts, m0, N);
      const float *gam = a.gam + col0, *bet = a.bet + col0;
      typename O::T* out16 = static_cast<typename O::T*>(p.out) + col0;
      const bool keep32 = p.out32 != nullptr;
#pragma unroll 1
      for (int w = 0; w < 2; ++w) {
        const int h0 = kHalf * w, x = 2 * b + w;             // the half's first row; its exchange barriers
        if (et == 0) { mbar_arrive_expect_tx(&xs_full[x], kHalf * 4); mbar_arrive_expect_tx(&xv_full[x], kHalf * 4); }
        mbar_wait(&buf_full[w], bphase);
        if (et == 0) ln_probe(p.K, rank, cl, it, w, LNP_BUF);
        if (copier && p.y_out != nullptr) store_rows(m0, w);
        // the sums of squared deviations, a group of 8 rows per warp at a time; lane = 4 row + q owns chain q of its row's half.
        // The row sums came with y: this half's from the MMA warpgroups (s_own), the other's from the peer's
        const int q = lane & 3;
        mbar_wait(&xs_full[x], xph);
        if (et == 0) ln_probe(p.K, rank, cl, it, w, LNP_XS);
#pragma unroll 1
        for (int g = et >> 5; g < kHalf / 8; g += kLnEpiThreads / 32) {
          const int r = h0 + 8 * g + (lane >> 2);
          const float piv = s_piv[r], s = s_own[r] + x_sum[b * kRows + r];   // the row sum of y - pivot; mean - pivot = s / N
          const float* yr = buf + r * kLd + 2 * q;
          float v = 0.0f;
#pragma unroll
          for (int j = 0; j < kCols / 8; ++j) {
            const float2 y = *reinterpret_cast<const float2*>(yr + 8 * j);
            const float d0 = fmaf(-s, inv_n, y.x - piv), d1 = fmaf(-s, inv_n, y.y - piv);
            v = fmaf(d0, d0, fmaf(d1, d1, v));
          }
          v += __shfl_xor_sync(0xffffffffu, v, 1);
          v += __shfl_xor_sync(0xffffffffu, v, 2);
          if (q == 0) { s_sum[r] = s; s_var[r] = v; st_async_f32(px_var + (b * kRows + r) * 4, v, pxv_full + x * 8); }
        }
        mbar_wait(&xv_full[x], xph);
        if (et == 0) ln_probe(p.K, rank, cl, it, w, LNP_XV);
        if (q == 0) {                                        // the rows whose partials this lane sent
#pragma unroll 1
          for (int g = et >> 5; g < kHalf / 8; g += kLnEpiThreads / 32) {
            const int r = h0 + 8 * g + (lane >> 2);
            s_var[r] = 1.0f / sqrtf(fmaxf((s_var[r] + x_var[b * kRows + r]) * inv_n, 0.0f) + 1e-5f);
          }
        }
        named_bar_sync(1, kLnEpiThreads);
        // normalise: 16-bit outputs stored here, the fp32 ones written back into the buffer for a TMA store
#pragma unroll 6
        for (int k = 0; k < kPerThread; ++k) {
          const int i = k * kLnEpiThreads + et, r = h0 + i / kVec, c = (i - (r - h0) * kVec) * 4;
          if (i >= kTotal) continue;
          float4* bp = reinterpret_cast<float4*>(buf + r * kLd + c);
          const float4 y = *bp;
          const float4 g = __ldg(reinterpret_cast<const float4*>(gam + c)), h = __ldg(reinterpret_cast<const float4*>(bet + c));
          const float piv = s_piv[r], s = s_sum[r], rstd = s_var[r];
          const float4 v = make_float4(fmaf(fmaf(-s, inv_n, y.x - piv) * rstd, g.x + a.gadd, h.x), fmaf(fmaf(-s, inv_n, y.y - piv) * rstd, g.y + a.gadd, h.y),
                                       fmaf(fmaf(-s, inv_n, y.z - piv) * rstd, g.z + a.gadd, h.z), fmaf(fmaf(-s, inv_n, y.w - piv) * rstd, g.w + a.gadd, h.w));
          *reinterpret_cast<uint2*>(out16 + static_cast<size_t>(m0 + r) * N + c) = make_uint2(O::pack(v.x, v.y), O::pack(v.z, v.w));
          if (keep32) *bp = v;
        }
        if (keep32) fence_proxy_async_smem();                // the fp32 rows are visible to the TMA store
        named_bar_sync(1, kLnEpiThreads);
        if (et == 0) ln_probe(p.K, rank, cl, it, w, LNP_NORM);
        if (copier) {
          if (keep32) store_rows(m0, w);
          bulk_wait_group_read<0>();
          if (et == 0) ln_probe(p.K, rank, cl, it, w, LNP_WAIT);
          if (t + n_cl < n_work) load_resid(t + n_cl, w);
          if (et == 0) ln_probe(p.K, rank, cl, it, w, LNP_NEXT);
        }
      }
      bphase ^= 1;
    }
    if (copier) bulk_wait_group_all();                       // the last TMA stores are complete before the CTA exits
  } else {
    // ===================== MMA warpgroups =====================
    const int wg = warp >> 2;                                // row half
    float acc[kAcc];
    int s = 0;
    uint32_t phase = 0, bphase = 0;
    const int rw = kHalf * wg + (warp & 3) * 16 + (lane >> 2);   // fragment rows rw and rw + 8 of the tile
    const int cw = 2 * (lane & 3);                           // + 8 j: columns c, c + 1 of n8 block j (of the CTA's)
    const float* bias = p.bias + col0;
    float* bw = buf + rw * kLd + cw;
    int it = 0;                                              // the CTA's tile count: exchange slot it & 1
    for (int t = cl; t < n_work; t += n_cl, ++it) {
      const int m0 = tile_m0(t);
      ring.template mma_tile<MODE>(s, phase, acc, wg, 0, num_kb, p.K);
      if (threadIdx.x % 128 == 0) ln_probe(p.K, rank, cl, it, wg, LNP_MAIN);
      // the pivot bias[0] + resid[row][0] of rows rw, rw + 8 (column 0 of y without the GEMM term)
      float piv0 = 0.0f, piv1 = 0.0f;
      if (cw == 0) {
        const float b0 = __ldg(p.bias);
        piv0 = b0 + p.resid[static_cast<size_t>(m0 + rw) * N];
        piv1 = b0 + p.resid[static_cast<size_t>(m0 + rw + 8) * N];
      }
      piv0 = __shfl_sync(0xffffffffu, piv0, lane & ~3);
      piv1 = __shfl_sync(0xffffffffu, piv1, lane & ~3);
      // y = acc + (bias + resid) over the half's residual rows in the buffer.  The thread's columns 2 q + 8 j (q = lane % 4)
      // are chain q of rows rw and rw + 8: it sums (y_c - piv) + (y_c+1 - piv), j ascending, as the statistics require
      mbar_wait(&res_full[wg], bphase);
      if (threadIdx.x % 128 == 0) ln_probe(p.K, rank, cl, it, wg, LNP_RES);
      if (cw == 0) { s_piv[rw] = piv0; s_piv[rw + 8] = piv1; }
      float s0 = 0.0f, s1 = 0.0f;
#pragma unroll
      for (int j = 0; j < kAcc / 4; ++j) {
        const float2 b = __ldg(reinterpret_cast<const float2*>(bias + cw + 8 * j));
        float2* y0 = reinterpret_cast<float2*>(bw + 8 * j);
        float2* y1 = reinterpret_cast<float2*>(bw + 8 * kLd + 8 * j);
        const float2 r0 = *y0, r1 = *y1;
        const float2 v0 = make_float2(acc[4 * j] + (b.x + r0.x), acc[4 * j + 1] + (b.y + r0.y));
        const float2 v1 = make_float2(acc[4 * j + 2] + (b.x + r1.x), acc[4 * j + 3] + (b.y + r1.y));
        *y0 = v0;
        *y1 = v1;
        s0 += (v0.x - piv0) + (v0.y - piv0);
        s1 += (v1.x - piv1) + (v1.y - piv1);
      }
      s0 += __shfl_xor_sync(0xffffffffu, s0, 1);
      s1 += __shfl_xor_sync(0xffffffffu, s1, 1);
      s0 += __shfl_xor_sync(0xffffffffu, s0, 2);             // this half's sums of y - pivot of rows rw, rw + 8
      s1 += __shfl_xor_sync(0xffffffffu, s1, 2);
      if (cw == 0) {
        const int b = it & 1, x = 2 * b + wg;
        s_own[rw] = s0; s_own[rw + 8] = s1;
        st_async_f32(px_sum + (b * kRows + rw) * 4, s0, pxs_full + x * 8);
        st_async_f32(px_sum + (b * kRows + rw + 8) * 4, s1, pxs_full + x * 8);
      }
      fence_proxy_async_smem();                              // y is visible to the TMA store of y_out
      mbar_arrive(&buf_full[wg]);
      if (threadIdx.x % 128 == 0) ln_probe(p.K, rank, cl, it, wg, LNP_Y);
      bphase ^= 1;
    }
  }
  cluster_sync();                                            // the peer stores nothing into this CTA's shared memory any more
}

}  // namespace ldm
