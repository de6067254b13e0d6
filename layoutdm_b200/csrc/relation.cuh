// cond = "relation": gradient-based logit adjustment between the posterior and the draw, on the device.
// Replaces `update` (T/models/categorical_diffusion/logit_adjustment.py:88-126): `relation_num_update` SGD steps with
// lr = relation_lambda on the (B,S,C) log-probabilities for the loss  mean_{layout, f} cost_f  of the 14 relation costs of
// T/models/clg/const.py:226-241, evaluated on the EXPECTED boxes of `_stochastic_convert` (mode "average", :16-85).
// The reference differentiates with autograd; the costs are sums of ReLUs of linear / bilinear box terms, so the gradient is
// written out by hand here:
//     d loss / d logit[e, a, c] = g[e, a] * p[e, a, c] * (center[a, c] - bbox[e, a]),   g = d loss / d bbox   (softmax over the bins)
// One CTA per layout (the update never couples layouts); node 0 is the canvas (AddCanvasElement, T/data/util.py:106-120),
// nodes 1..E the layout's elements; edges come as a dense [N][N] table of the reference's edge_attr bit masks
// (RelSize / RelLoc, T/data/util.py:14-27).  Everything stays fp32 like the reference.
#pragma once
#include "common.cuh"

namespace ldm {

constexpr int kRelMaxNodes = 32;        // 1 canvas + n_elem (25) nodes
constexpr int kRelThreads = 256;

struct RelationParams {
  int n_layouts, S, C, n_attr, n_elem, n_cat, n_bins, pad_id;
  float* lp;                    // [n_layouts][S][C] log-probabilities, updated in place
  const long long* cond_seq;    // [n_layouts][S]: an element is valid when its category slot is not PAD (logit_adjustment.py:44)
  const int* adj;               // [n_layouts][1 + n_elem][1 + n_elem] edge_attr of the edge i -> j, 0 = no edge
  const float* centers;         // [4][n_bins] bin centres (x, y, w, h) or nullptr = linear quantisation
  float step;                   // relation_lambda / (batch_total * 14): SGD lr times the mean() over (layout, cost function)
  int n_update;
};

LDM_DEVINL float rel_center(const RelationParams& p, int a, int bin) {
  if (p.centers != nullptr) return __ldg(p.centers + a * p.n_bins + bin);
  // linear decode (bbox_tokenizer.py:150-156): the centres are float32(linspace), i.e. bin / n correctly rounded.  bin * (1 / n)
  // rounds twice and is an ulp off for some bins when n is not a power of two
  return __fdiv_rn(static_cast<float>(a < 2 ? bin : bin + 1), static_cast<float>(p.n_bins));
}

__global__ void __launch_bounds__(kRelThreads) relation_update_kernel(const RelationParams p) {
  pdl_sync();
  const int b = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, n_warps = kRelThreads / 32;
  const int N = 1 + p.n_elem;
  __shared__ float s_bbox[kRelMaxNodes][4];
  __shared__ float s_g[kRelMaxNodes][4];
  __shared__ int s_valid[kRelMaxNodes];
  __shared__ int s_any;
  const int* adj = p.adj + static_cast<size_t>(b) * N * N;

  if (threadIdx.x == 0) s_any = 0;
  __syncthreads();
  // validity (logit_adjustment.py:43-47) and "does this layout have an edge at all" (no edge: the costs and their gradient are 0)
  if (threadIdx.x < N) s_valid[threadIdx.x] = threadIdx.x == 0 ? 1 : (p.cond_seq[static_cast<size_t>(b) * p.S + (threadIdx.x - 1) * p.n_attr] != p.pad_id);
  {
    int any = 0;
    for (int i = threadIdx.x; i < N * N; i += kRelThreads) any |= adj[i] != 0;
    if (any) s_any = 1;
  }
  // canvas box: softmax of the log one-hot of encode([0.5, 0.5, 1, 1]) puts 1.0f on the canvas bin (the other bins carry 1e-30)
  if (warp == 0 && lane < 4) {
    const int a = lane;
    const float v = a < 2 ? 0.5f : 1.0f;
    int bin;
    if (p.centers == nullptr) {
      const float d32 = 1.0f / p.n_bins;
      const float q = a < 2 ? fminf(fmaxf(v, 0.0f), 1.0f - d32) : __fsub_rn(fminf(fmaxf(v, d32), 1.0f), d32);
      bin = __float2int_rn(__fmul_rn(static_cast<float>(p.n_bins), q));
    } else {
      float best = INFINITY; bin = 0;
      for (int k = 0; k < p.n_bins; ++k) {
        const float df = __fsub_rn(v, p.centers[a * p.n_bins + k]);
        const float dist = __fmul_rn(df, df);
        if (dist < best) { best = dist; bin = k; }
      }
    }
    s_bbox[0][a] = rel_center(p, a, bin);
  }
  __syncthreads();
  if (!s_any) return;

  // this warp's nodes: e = 1 + warp + k * n_warps; lane = bin.  Log-probs, probabilities and boxes stay in registers across the updates.
  constexpr int kPerWarp = (kRelMaxNodes + kRelThreads / 32 - 1) / (kRelThreads / 32);
  float v[kPerWarp][4], pr[kPerWarp][4], bx[kPerWarp][4], cen[4];
  const bool lane_on = lane < p.n_bins;
#pragma unroll
  for (int a = 0; a < 4; ++a) cen[a] = lane_on ? rel_center(p, a, lane) : 0.0f;
#pragma unroll
  for (int k = 0; k < kPerWarp; ++k) {
    const int e = 1 + warp + k * n_warps;
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      v[k][a] = -INFINITY;
      if (e < N && s_valid[e] && lane_on)
        v[k][a] = p.lp[(static_cast<size_t>(b) * p.S + (e - 1) * p.n_attr + 1 + a) * p.C + p.n_cat + a * p.n_bins + lane];
    }
  }

  for (int u = 0; u < p.n_update; ++u) {
    // ---- expected boxes (mode "average": softmax over the attribute's bins times the bin centres) ----
#pragma unroll
    for (int k = 0; k < kPerWarp; ++k) {
      const int e = 1 + warp + k * n_warps;
      if (e < N && s_valid[e]) {
#pragma unroll
        for (int a = 0; a < 4; ++a) {
          const float m = warp_max(v[k][a]);
          const float ex = lane_on ? expf(v[k][a] - m) : 0.0f;
          const float sm = warp_sum(ex);
          pr[k][a] = ex / sm;
          bx[k][a] = warp_sum(pr[k][a] * cen[a]);
          if (lane == 0) s_bbox[e][a] = bx[k][a];
        }
      }
    }
    __syncthreads();
    // ---- d(sum of the 14 costs) / d(box) of node n: one thread per node, fixed accumulation order ----
    if (threadIdx.x < N) {
      const int n = threadIdx.x;
      float g_area = 0.f, g_l = 0.f, g_t = 0.f, g_r = 0.f, g_b = 0.f, g_y = 0.f;
      if (n > 0 && s_valid[n]) {
        const float eps = 1e-8f, al = 1.0f - 0.1f, ah = 1.0f + 0.1f, third = 1.0f / 3, two3 = 2.0f / 3;
        const float xn = s_bbox[n][0], yn = s_bbox[n][1], wn = s_bbox[n][2], hn = s_bbox[n][3];
        const float an = wn * hn, ln = xn - wn / 2, tn = yn - hn / 2, rn = xn + wn / 2, bn = yn + hn / 2;
        for (int m = 0; m < N; ++m) {
          if (m == n || !s_valid[m]) continue;
          const float xm = s_bbox[m][0], ym = s_bbox[m][1], wm = s_bbox[m][2], hm = s_bbox[m][3];
          const float am = wm * hm, lm = xm - wm / 2, tm = ym - hm / 2, rm = xm + wm / 2, bm = ym + hm / 2;
          // role 1: n is the SOURCE i of the edge n -> m (never the canvas here: n > 0)
          int e1 = adj[n * N + m];
          if (e1) {
            if ((e1 & (1 << 1)) && am - al * an > 0.f) g_area -= al;                                   // size smaller: relu(a_j - (1-alpha) a_i)
            if (e1 & (1 << 2)) { if (al * an - am + eps > 0.f) g_area += al; if (am - ah * an + eps > 0.f) g_area -= ah; }   // size equal
            if ((e1 & (1 << 3)) && ah * an - am > 0.f) g_area += ah;                                   // size larger
            if ((e1 & (1 << 6)) && bm - tn > 0.f) g_t -= 1.f;                                          // top: relu(b_j - t_i)
            if ((e1 & (1 << 8)) && bn - tm > 0.f) g_b += 1.f;                                          // bottom: relu(b_i - t_j)
            if ((e1 & (1 << 5))) { if (rm - ln > 0.f) g_l -= 1.f; if (tn - bm + eps > 0.f) g_t += 1.f; if (tm - bn + eps > 0.f) g_b -= 1.f; }   // left
            if ((e1 & (1 << 7))) { if (rn - lm > 0.f) g_r += 1.f; if (tn - bm + eps > 0.f) g_t += 1.f; if (tm - bn + eps > 0.f) g_b -= 1.f; }   // right
            if ((e1 & (1 << 9))) {                                                                     // center
              if (ln - rm + eps > 0.f) g_l += 1.f;
              if (lm - rn + eps > 0.f) g_r -= 1.f;
              if (tn - bm + eps > 0.f) g_t += 1.f;
              if (tm - bn + eps > 0.f) g_b -= 1.f;
            }
          }
          // role 2: n is the DESTINATION j of the edge m -> n
          int e2 = adj[m * N + n];
          if (e2) {
            if ((e2 & (1 << 1)) && an - al * am > 0.f) g_area += 1.f;
            if (e2 & (1 << 2)) { if (al * am - an + eps > 0.f) g_area -= 1.f; if (an - ah * am + eps > 0.f) g_area += 1.f; }
            if ((e2 & (1 << 3)) && ah * am - an > 0.f) g_area -= 1.f;
            if (m == 0) {                                                                              // source is the canvas: const.py:101-148
              if ((e2 & (1 << 6)) && yn - third > 0.f) g_y += 1.f;
              if (e2 & (1 << 9)) { if (third - yn + eps > 0.f) g_y -= 1.f; if (yn - two3 + eps > 0.f) g_y += 1.f; }
              if ((e2 & (1 << 8)) && two3 - yn > 0.f) g_y -= 1.f;
            } else {
              if ((e2 & (1 << 6)) && bn - tm > 0.f) g_b += 1.f;                                        // top: relu(b_j - t_i), j = n
              if ((e2 & (1 << 8)) && bm - tn > 0.f) g_t -= 1.f;                                        // bottom: relu(b_i - t_j)
              if ((e2 & (1 << 5))) { if (rn - lm > 0.f) g_r += 1.f; if (tm - bn + eps > 0.f) g_b -= 1.f; if (tn - bm + eps > 0.f) g_t += 1.f; }
              if ((e2 & (1 << 7))) { if (rm - ln > 0.f) g_l -= 1.f; if (tm - bn + eps > 0.f) g_b -= 1.f; if (tn - bm + eps > 0.f) g_t += 1.f; }
              if ((e2 & (1 << 9))) {
                if (lm - rn + eps > 0.f) g_r -= 1.f;
                if (ln - rm + eps > 0.f) g_l += 1.f;
                if (tm - bn + eps > 0.f) g_b -= 1.f;
                if (tn - bm + eps > 0.f) g_t += 1.f;
              }
            }
          }
        }
        s_g[n][0] = g_l + g_r;
        s_g[n][1] = g_t + g_b + g_y;
        s_g[n][2] = g_area * hn + (g_r - g_l) / 2;
        s_g[n][3] = g_area * wn + (g_b - g_t) / 2;
      }
    }
    __syncthreads();
    // ---- SGD step on the bins of every valid element ----
#pragma unroll
    for (int k = 0; k < kPerWarp; ++k) {
      const int e = 1 + warp + k * n_warps;
      if (e < N && s_valid[e] && lane_on) {
#pragma unroll
        for (int a = 0; a < 4; ++a) v[k][a] -= p.step * (s_g[e][a] * pr[k][a] * (cen[a] - bx[k][a]));
      }
    }
    __syncthreads();     // s_bbox / s_g are rewritten by the next update
  }
#pragma unroll
  for (int k = 0; k < kPerWarp; ++k) {
    const int e = 1 + warp + k * n_warps;
    if (e < N && s_valid[e] && lane_on) {
#pragma unroll
      for (int a = 0; a < 4; ++a)
        p.lp[(static_cast<size_t>(b) * p.S + (e - 1) * p.n_attr + 1 + a) * p.C + p.n_cat + a * p.n_bins + lane] = v[k][a];
    }
  }
}

}  // namespace ldm
