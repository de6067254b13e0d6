// Step epilogue: logits -> log p(x0|xt) -> mask-and-replace posterior -> conditioning adjustments -> categorical draw.
// One warp per token, no (B,C,S) temporaries.  Replaces, per diffusion step (reference file:line):
//   predict_start                 T/models/categorical_diffusion/base.py:127-146
//   q_posterior (constrained)     T/models/categorical_diffusion/constrained.py:135-206 (+ q_pred :112-133, :92-110)
//   q_posterior (vanilla)         T/models/categorical_diffusion/vanilla.py:112-151
//   Converter f_to_p_log/p_to_f_log   T/helpers/layout_tokenizer.py:540-557  (here: compile-free vocab group test)
//   strong mask / refinement / pad-disable   base.py:243-284, T/helpers/task.py:154-224
//   sample()                      T/helpers/sampling.py:81-130 ; torch.multinomial(p,1) == argmax(p / Exp(1))
// Class ownership inside a warp (lane_classes): lane l holds classes 4l..4l+3 (one float4 of logits, one Philox block) and
// class 128+l; TokenNoise::lane_words draws the noise words of exactly these classes.
// The draw kernels take the noise contract as a template parameter: TokenNoise (the default, DESIGN.md §7) or TorchNoise
// (the numbers torch's CUDA generator would give the reference's draw).
#pragma once
#include <type_traits>

#include "common.cuh"
#include "embed.cuh"

namespace ldm {

enum : int { SAMP_DETERMINISTIC = 0, SAMP_RANDOM = 1, SAMP_TOP_K = 2, SAMP_TOP_P = 3, SAMP_GUMBEL = 4 };
enum : int { COND_HAS_MASK = 1, COND_PAD_DISABLE = 2, COND_REFINE = 4 };
constexpr int kMaxAttr = 8;

// The token layout (LayoutSequenceTokenizer / BboxTokenizer, T/helpers/layout_tokenizer.py:296-313, bbox_tokenizer.py:84-135):
// slot k of an element's n_attr tokens carries variable var[k] (0 = c, 1..4 = x, y, w, h) and draws from the full-vocabulary
// ids [start[k], start[k] + n[k]) plus PAD and MASK.  The bbox ids are [n_cat, n_cat + n_bbox_ids): n_bbox_ids = 4 n_bins with
// per-variable ranges (x-y-w-h) or n_bins shared by all four (xywh).  ldm_create builds it once; the step kernels' vocabulary
// groups, decode, make_cond and the relation update read it.
struct TokenLayout {
  int n_attr, n_cat, n_bins, n_bbox_ids;
  int var[kMaxAttr], start[kMaxAttr], n[kMaxAttr];
};

struct StepParams {
  int n_layouts, S, C, n_attr, pad_id, mask_id;
  int constrained;                       // 1: per-attribute groups, 0: vanilla (single group over all classes)
  int grp_start[kMaxAttr], grp_n[kMaxAttr];
  int T, t_post;
  const float* sched;                    // [G][8][T+1]
  const float* lae;                      // [G][T+1][4] log_add_exp terms that depend on (group, t) only (lae_table_kernel)
  const float* logits; int ld_logits;    // [n_layouts*layout_rows][ld]; row = b*layout_rows + s      (nullptr if logprob_in)
  int layout_rows;                       // rows per layout of the logits and of the fused embedding's x32 / x16: 128 R
  const float* logprob_in;               // [n_layouts][S][C] or nullptr: draw from given log-probs (relation hook)
  const float* lx0_in;                   // [n_layouts][S][C] or nullptr: log p(x0) given by the caller instead of predict_start(logits)
                                         // (q_posterior as a callable API, constrained.py:135-206; the MASK column is ignored like :191)
  float* lx0_out;                        // [n_layouts][S][C] or nullptr: tap of predict_start's output (base.py:127-146)
  const int* t_layout;                   // [n_layouts] or nullptr: per-layout posterior timestep (training-side calls) instead of t_post
  const long long* ids_in;               // [n_layouts][S]
  const long long* cond_seq; const unsigned char* cond_mask; const long long* cond_seq_orig; const float* refine_tbl;
  int cond_flags;
  int mode; float temperature; float top_p; int top_k;
  unsigned long long seed; unsigned int step_ctr; long long b_global0;
  const unsigned long long* call;        // nullptr, or device words {seed, b_global0, t_offset, t_tthr, t_delta, t_total} that override those
                                         // fields: a captured CUDA graph of the loop stays valid while the noise changes from call to call
  long long* ids_out;                    // [n_layouts][S]
  float* logprob_out;                    // [n_layouts][S][C] or nullptr
  // the front of the NEXT denoising step, fused behind the draw (the loop API only): the warp that drew a token also writes that
  // token's embedding + AdaLN_0(t_next) row, which saves the embed launch and overlaps its write stream with this issue-bound kernel
  const float* emb_cat; const float* emb_pos; const float* emb_adaln;   // cat_emb [C][d], pos [S][d], AdaLN row [2d] of (layer 0, t_next); emb_adaln == nullptr: off
  float* emb_x32; void* emb_x16; int emb_d, emb_bf16;
  // TorchNoise: the generator offset of the call's first step, the threads of torch's launch and the offset one draw advances;
  // step t_step of the call draws at t_offset + t_step * (1 or 2 draws) * t_delta; t_total: the layouts of the whole batch
  unsigned long long t_offset; unsigned int t_tthr, t_delta; int t_step; long long t_total;
};

LDM_DEVINL float log_add_exp(float a, float b) {   // util.py:19-21
  const float m = fmaxf(a, b);
  return m + logf(expf(a - m) + expf(b - m));
}

// The four log_add_exp terms of q_posterior that depend on (group, t) only -- computed once, with the same device function
// the kernels use, so the group-centric kernel reads them instead of re-evaluating 2 expf + 1 logf four times per class:
//   [0] log(q(x_t = c | x0' = c))  = lae(0      + lcat, lcbt)      [1] ... x0' != c:  lae(log eps + lcat, lcbt)
//   [2] one-step term, same class = lae(0      + lat,  lbt)        [3] ... different: lae(log eps + lat,  lbt)
__global__ void lae_table_kernel(const float* __restrict__ sched, float* __restrict__ lae, int G, int TT) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= G * TT) return;
  const int g = i / TT, t = i % TT;
  const float* tab = sched + static_cast<size_t>(g) * 8 * TT;
  const float lat = tab[0 * TT + t], lbt = tab[1 * TT + t], lcat = tab[3 * TT + t], lcbt = tab[4 * TT + t];
  float4 o;
  o.x = log_add_exp(0.0f + lcat, lcbt); o.y = log_add_exp(kLogEps + lcat, lcbt);
  o.z = log_add_exp(0.0f + lat, lbt);   o.w = log_add_exp(kLogEps + lat, lbt);
  reinterpret_cast<float4*>(lae)[i] = o;
}

// the drawn token's row of the next step's denoiser input (see StepParams::emb_*); best_c is warp-uniform
LDM_DEVINL void embed_next(const StepParams& p, const int b, const int s, const int best_c, const int lane) {
  if (p.emb_adaln == nullptr) return;
  const size_t row = static_cast<size_t>(b) * p.layout_rows + s;
  if (p.emb_bf16) embed_token_row<true>(best_c, s, row, p.emb_cat, p.emb_pos, p.emb_adaln, p.emb_x32, p.emb_x16, p.emb_d, lane);
  else embed_token_row<false>(best_c, s, row, p.emb_cat, p.emb_pos, p.emb_adaln, p.emb_x32, p.emb_x16, p.emb_d, lane);
}

LDM_DEVINL void lane_classes(const int C, const int lane, int (&cls)[5], bool (&valid)[5]) {
#pragma unroll
  for (int j = 0; j < 4; ++j) { cls[j] = 4 * lane + j; valid[j] = cls[j] < C; }
  cls[4] = 128 + lane; valid[4] = cls[4] < C;
}

// the vocabulary group of token position s: its attribute for the constrained diffusion, the single group 0 for vanilla
LDM_DEVINL int vocab_group(const StepParams& p, const int s) { return p.constrained ? s % p.n_attr : 0; }

// class c belongs to group g (Converter f_to_p_log): the attribute's own classes plus PAD and MASK; for vanilla every class
LDM_DEVINL bool in_group(const StepParams& p, const int g, const int c) {
  return !p.constrained || (c >= p.grp_start[g] && c < p.grp_start[g] + p.grp_n[g]) || c == p.pad_id || c == p.mask_id;
}

// argmax over the classes the warp holds in N slots per lane, first (smallest) class on ties; slots with on[j] false take no part
template <int N>
LDM_DEVINL int warp_argmax_first(const float (&v)[N], const int (&cls)[N], const bool (&on)[N]) {
  float best = -INFINITY; int best_c = 0x7fffffff;
#pragma unroll
  for (int j = 0; j < N; ++j) if (on[j] && (v[j] > best || (v[j] == best && cls[j] < best_c))) { best = v[j]; best_c = cls[j]; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oc = __shfl_xor_sync(0xffffffffu, best_c, o);
    if (ob > best || (ob == best && oc < best_c)) { best = ob; best_c = oc; }
  }
  return best_c;
}

// the noise of token (b, s) of this call, with the captured graph's {seed, b_global0} override (StepParams::call) resolved
LDM_DEVINL TokenNoise step_noise(const StepParams& p, const int b, const int s) {
  const unsigned long long seed = p.call ? __ldg(p.call) : p.seed, bg0 = p.call ? __ldg(p.call + 1) : static_cast<unsigned long long>(p.b_global0);
  return TokenNoise(seed, bg0, b, p.S, s);
}

// the torch-generator noise of token (b, s) of this call's step p.t_step, slot j holding class cls[j] (the same override)
template <int N>
LDM_DEVINL TorchDraw<N> torch_draw(const StepParams& p, const int b, const int s, const int (&cls)[N]) {
  const unsigned long long* w = p.call;
  const unsigned long long seed = w ? __ldg(w) : p.seed, bg0 = w ? __ldg(w + 1) : static_cast<unsigned long long>(p.b_global0);
  const unsigned long long off0 = w ? __ldg(w + 2) : p.t_offset;
  const uint32_t tthr = w ? static_cast<uint32_t>(__ldg(w + 3)) : p.t_tthr, delta = w ? static_cast<uint32_t>(__ldg(w + 4)) : p.t_delta;
  const bool single = (w ? static_cast<long long>(__ldg(w + 5)) : p.t_total) == 1;   // see TorchDraw
  const bool gum = p.mode == SAMP_GUMBEL;       // rand_like at the step's offset, then multinomial one draw later
  const unsigned long long off = off0 + static_cast<unsigned long long>(p.t_step) * (gum ? 2u : 1u) * delta;
  const uint32_t bg = static_cast<uint32_t>(bg0 + b), S = static_cast<uint32_t>(p.S), C = static_cast<uint32_t>(p.C);
  return TorchDraw<N>{TorchNoise(seed, off + (gum ? delta : 0u), tthr), TorchNoise(seed, off, tthr), single ? static_cast<uint32_t>(s) : (bg * S + s) * C,
                      single ? S : 1u, bg * C * S + s, S, cls};
}

// predict_start (base.py:127-146): the float64 log-sum-exp over the C-1 non-MASK logits of one token's row (lane classes);
// l receives the lane's logits.  lx0_of maps a logit to log p(x0), clamped to [-70, 0].
LDM_DEVINL double logit_lse(const StepParams& p, const float* lrow, const int lane, const int (&cls)[5], const bool (&valid)[5], float (&l)[5]) {
  const float4 v = __ldg(reinterpret_cast<const float4*>(lrow) + lane);
  l[0] = v.x; l[1] = v.y; l[2] = v.z; l[3] = v.w;
  l[4] = valid[4] ? __ldg(lrow + cls[4]) : 0.0f;
  float mx = -INFINITY;
#pragma unroll
  for (int j = 0; j < 5; ++j) if (valid[j] && cls[j] < p.C - 1) mx = fmaxf(mx, l[j]);
  mx = warp_max(mx);
  double dsum = 0.0;
#pragma unroll
  for (int j = 0; j < 5; ++j) if (valid[j] && cls[j] < p.C - 1) dsum += exp(static_cast<double>(l[j]) - static_cast<double>(mx));
  dsum = warp_sum_d(dsum);
  return static_cast<double>(mx) + log(dsum);
}
LDM_DEVINL float lx0_of(const float logit, const double lse) {
  return fminf(fmaxf(static_cast<float>(static_cast<double>(logit) - lse), -70.0f), 0.0f);
}

// predict_start for one token, every class (lane classes): MASK = -70
LDM_DEVINL void predict_start_token(const StepParams& p, const float* lrow, const int lane, const int (&cls)[5], const bool (&valid)[5], float (&lx0)[5]) {
  float l[5];
  const double lse = logit_lse(p, lrow, lane, cls, valid, l);
#pragma unroll
  for (int j = 0; j < 5; ++j) lx0[j] = (cls[j] < p.C - 1) ? lx0_of(l[j], lse) : -70.0f;
}

// The schedule terms of q_posterior at (group g, posterior timestep t): the log_add_exp terms of the lae table, lct / lcct at t,
// and the entries at t-1 (t = 0 wraps to T).
struct PostTerms { float4 lae; float lct, lcct, lcat1, lcbt1, lcct1, l1mcct1; };
LDM_DEVINL PostTerms post_terms(const StepParams& p, const int g, const int t) {
  const int TT = p.T + 1, tm1 = (t - 1 + TT) % TT;
  const float* tab = p.sched + static_cast<size_t>(g) * 8 * TT;
  PostTerms k;
  k.lae = __ldg(reinterpret_cast<const float4*>(p.lae) + static_cast<size_t>(g) * TT + t);
  k.lct = tab[2 * TT + t]; k.lcct = tab[5 * TT + t];
  k.lcat1 = tab[3 * TT + tm1]; k.lcbt1 = tab[4 * TT + tm1]; k.lcct1 = tab[5 * TT + tm1]; k.l1mcct1 = tab[7 * TT + tm1];
  return k;
}

// q(x_{t-1} | x_t, x0~) in log space (constrained.py:135-206 / vanilla.py:112-151) for the classes a warp holds in N slots per
// lane: lx0 = log p(x0) (its MASK entry is not used), x_t the token's current id.  The normalisation runs over the slots with
// in_grp[j]; only their lp[j] are written.
template <int N>
LDM_DEVINL void posterior_logprob(const StepParams& p, const PostTerms& k, const int x_t, const float (&lx0)[N], const int (&cls)[N],
                                  const bool (&in_grp)[N], float (&lp)[N]) {
  const bool is_mask = (x_t == p.mask_id);
  float q[N], one[N];
  float qmax = -INFINITY;
#pragma unroll
  for (int j = 0; j < N; ++j) {
    q[j] = -INFINITY; one[j] = 0.0f;
    if (in_grp[j]) {
      if (cls[j] != p.mask_id) {
        const bool same = (cls[j] == x_t);
        const float lq = is_mask ? k.lcct : (same ? k.lae.x : k.lae.y);      // = log_add_exp(v + lcat, lcbt), v = 0 / log eps
        one[j] = is_mask ? k.lct : (same ? k.lae.z : k.lae.w);               // = log_add_exp(v + lat, lbt)
        q[j] = lx0[j] - lq;
      } else {
        q[j] = kLogEps;
        one[j] = is_mask ? 0.0f : kLogEps;
      }
      qmax = fmaxf(qmax, q[j]);
    }
  }
  qmax = warp_max(qmax);
  float qs = 0.0f;
#pragma unroll
  for (int j = 0; j < N; ++j) if (in_grp[j]) qs += expf(q[j] - qmax);
  const float L = logf(warp_sum(qs)) + qmax;
#pragma unroll
  for (int j = 0; j < N; ++j) {
    if (in_grp[j]) {
      const float qn = q[j] - L;
      const float ev = (cls[j] != p.mask_id) ? log_add_exp(qn + k.lcat1, k.lcbt1) : log_add_exp(qn + k.l1mcct1, k.lcct1);
      lp[j] = fminf(fmaxf((ev + one[j]) + L, -70.0f), 0.0f);
    }
  }
}

// The posterior for one token, every class (lane classes), t the posterior timestep: classes outside the token's vocabulary
// group come out as log(1e-30) (Converter.p_to_f_log), invalid lanes as -inf.
LDM_DEVINL void posterior_token_logprob(const StepParams& p, const int s, const int x_t, const int t, const float (&lx0)[5],
                                        const int (&cls)[5], const bool (&valid)[5], float (&lp)[5]) {
  const int g = vocab_group(p, s);
  bool in_grp[5];
#pragma unroll
  for (int j = 0; j < 5; ++j) { in_grp[j] = valid[j] && in_group(p, g, cls[j]); lp[j] = valid[j] ? kLogEps : -INFINITY; }
  posterior_logprob<5>(p, post_terms(p, g, t), x_t, lx0, cls, in_grp, lp);
}

// The draw from lg = log-probs / temperature (top-k / top-p already applied), the same for any slot layout: Gumbel noise for
// name="gumbel", then probs = softmax(lg) and multinomial(probs, 1) = argmax(probs / e), e ~ Exp(1).  The noise contract's
// draw view (ContractDraw, TorchDraw) maps the lane's N slots to their Gumbel noise and Exp(1) variates; a slot with zero
// probability scores 0 whatever its e, so it needs none.
template <int N, class Draw>
LDM_DEVINL int draw_class(const StepParams& p, float (&lg)[N], const int (&cls)[N], const bool (&on)[N], const Draw& nz) {
  if (p.mode == SAMP_GUMBEL) nz.add_gumbel(on, lg);
  float m = -INFINITY;
#pragma unroll
  for (int j = 0; j < N; ++j) m = fmaxf(m, lg[j]);
  m = warp_max(m);
  float ex[N], sm = 0.0f;
#pragma unroll
  for (int j = 0; j < N; ++j) { ex[j] = on[j] ? expf(lg[j] - m) : 0.0f; sm += ex[j]; }
  sm = warp_sum(sm);
  bool live[N];
#pragma unroll
  for (int j = 0; j < N; ++j) live[j] = on[j] && ex[j] > 0.0f;
  float e[N];
  nz.exponential(live, e);
  float score[N];
#pragma unroll
  for (int j = 0; j < N; ++j) score[j] = on[j] ? (ex[j] / sm) / e[j] : -INFINITY;
  return warp_argmax_first<N>(score, cls, on);
}

// One token, every class (lane classes): any q_type, any sampling mode, log-prob in / out.
template <class Noise>
LDM_DEVINL void posterior_token_generic(const StepParams& p, const int token, const int lane) {
  const int b = token / p.S, s = token % p.S;
  const int C = p.C;
  int cls[5]; bool valid[5];
  lane_classes(C, lane, cls, valid);

  const int x_t = static_cast<int>(p.ids_in[token]);
  float lp[5];

  if (p.logprob_in != nullptr) {
#pragma unroll
    for (int j = 0; j < 5; ++j) lp[j] = valid[j] ? p.logprob_in[static_cast<size_t>(token) * C + cls[j]] : -INFINITY;
    // the log-probs were adjusted outside (cond = relation: base.py:261-269); what is left of the reference's order is disabling
    // PAD where the number of elements is known (base.py:271-284)
    if ((p.cond_flags & COND_PAD_DISABLE) && (s % p.n_attr != 0) && p.cond_seq[token] != p.pad_id) {
#pragma unroll
      for (int j = 0; j < 5; ++j) if (valid[j] && cls[j] == p.pad_id) lp[j] = kLogEps;
    }
  } else {
    float lx0[5];
    if (p.lx0_in != nullptr) {
#pragma unroll
      for (int j = 0; j < 5; ++j) lx0[j] = valid[j] ? p.lx0_in[static_cast<size_t>(token) * C + cls[j]] : -70.0f;
    } else {
      predict_start_token(p, p.logits + (static_cast<size_t>(b) * p.layout_rows + s) * p.ld_logits, lane, cls, valid, lx0);
    }
    if (p.lx0_out != nullptr) {
#pragma unroll
      for (int j = 0; j < 5; ++j) if (valid[j]) p.lx0_out[static_cast<size_t>(token) * C + cls[j]] = lx0[j];
    }
    posterior_token_logprob(p, s, x_t, p.t_layout ? __ldg(p.t_layout + b) : p.t_post, lx0, cls, valid, lp);

    // ---- conditioning adjustments, in the reference's order ----
    if (p.cond_flags) {
      const long long cs = p.cond_seq[token];
      const bool fixed = (p.cond_flags & COND_HAS_MASK) && p.cond_mask[token];
      if (fixed) {
#pragma unroll
        for (int j = 0; j < 5; ++j) if (valid[j]) lp[j] = (cls[j] == cs) ? 0.0f : kLogEps;
      }
      if ((p.cond_flags & COND_REFINE) && !fixed) {
        const float* trow = p.refine_tbl + static_cast<size_t>(p.cond_seq_orig[token]) * C;
#pragma unroll
        for (int j = 0; j < 5; ++j) if (valid[j]) lp[j] += __ldg(trow + cls[j]);
      }
      if ((p.cond_flags & COND_PAD_DISABLE) && (s % p.n_attr != 0) && cs != p.pad_id) {
#pragma unroll
        for (int j = 0; j < 5; ++j) if (valid[j] && cls[j] == p.pad_id) lp[j] = kLogEps;
      }
    }
  }

  if (p.logprob_out != nullptr) {
#pragma unroll
    for (int j = 0; j < 5; ++j) if (valid[j]) p.logprob_out[static_cast<size_t>(token) * C + cls[j]] = lp[j];
  }
  if (p.ids_out == nullptr) return;        // log-probabilities only (q_posterior / predict_start as callable APIs)

  // ---- draw ----
  int best_c;
  if (p.mode == SAMP_DETERMINISTIC) {
    best_c = warp_argmax_first<5>(lp, cls, valid);
  } else {
    float lg[5];
#pragma unroll
    for (int j = 0; j < 5; ++j) lg[j] = valid[j] ? lp[j] / p.temperature : -INFINITY;

    if (p.mode == SAMP_TOP_K || p.mode == SAMP_TOP_P) {
      float pr[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
      if (p.mode == SAMP_TOP_P) {
        float m = -INFINITY;
#pragma unroll
        for (int j = 0; j < 5; ++j) m = fmaxf(m, lg[j]);
        m = warp_max(m);
        float sm = 0.0f;
#pragma unroll
        for (int j = 0; j < 5; ++j) { pr[j] = valid[j] ? expf(lg[j] - m) : 0.0f; sm += pr[j]; }
        sm = warp_sum(sm);
#pragma unroll
        for (int j = 0; j < 5; ++j) pr[j] = pr[j] / sm;
      }
      int n_before[5] = {0, 0, 0, 0, 0};
      double cum[5];
#pragma unroll
      for (int j = 0; j < 5; ++j) cum[j] = static_cast<double>(pr[j]);
      for (int src = 0; src < 32; ++src) {
#pragma unroll
        for (int jj = 0; jj < 5; ++jj) {
          const float v2 = __shfl_sync(0xffffffffu, lg[jj], src);
          const float p2 = __shfl_sync(0xffffffffu, pr[jj], src);
          const int c2 = (jj < 4) ? 4 * src + jj : 128 + src;
          if (c2 < C) {
#pragma unroll
            for (int j = 0; j < 5; ++j) {
              // rank in a descending sort; ties broken by class index
              const bool before = (v2 > lg[j]) || (v2 == lg[j] && c2 < cls[j]);
              if (before) { n_before[j] += (p.mode == SAMP_TOP_P) ? 1 : (v2 > lg[j] ? 1 : 0); cum[j] += static_cast<double>(p2); }
            }
          }
        }
      }
      if (p.mode == SAMP_TOP_P) {
        // sampling.py:100-109: drop every class whose inclusive cumulative mass exceeds top_p, except rank 0
#pragma unroll
        for (int j = 0; j < 5; ++j) if (valid[j] && n_before[j] > 0 && static_cast<float>(cum[j]) > p.top_p) lg[j] = -INFINITY;
      } else {
        // sampling.py:73-78: threshold = k-th largest value (duplicates counted)
        float thr = INFINITY;
#pragma unroll
        for (int j = 0; j < 5; ++j) if (valid[j] && n_before[j] < p.top_k) thr = fminf(thr, lg[j]);
        thr = -warp_max(-thr);
#pragma unroll
        for (int j = 0; j < 5; ++j) if (valid[j] && lg[j] < thr) lg[j] = -INFINITY;
      }
    }
    if constexpr (std::is_same_v<Noise, TokenNoise>) {
      const TokenNoise nz = step_noise(p, b, s);
      best_c = draw_class<5>(p, lg, cls, valid, contract_draw<5>([&](uint32_t stream, uint32_t (&w)[5]) { nz.lane_words(lane, noise_ctr(p.step_ctr, stream), w); }));
    } else {
      best_c = draw_class<5>(p, lg, cls, valid, torch_draw<5>(p, b, s, cls));
    }
  }
  if (lane == 0) p.ids_out[token] = best_c;
  embed_next(p, b, s, best_c, lane);
}

// The group-centric computation of one token of the constrained (per-attribute) diffusion: outside the token's vocabulary
// group (plus PAD and MASK) the posterior is the constant log(1e-30), so only the <= 34 classes of the group are evaluated
// (lane l: class grp_start + l; lanes 0 / 1 additionally PAD / MASK); the float64 log-softmax still runs over all C-1 logits.
// A token whose best in-group log-probability is not far enough above log(1e-30) for the out-of-group classes to be
// unreachable, or whose refinement row lifts a class outside the group, is not taken: the routine returns false
// (warp-uniform) having written nothing, and the caller runs posterior_token_generic.  Otherwise it writes the id, the
// next step's embedding row and, with kTap and logprob_out set, the log-probabilities it drew from: the group's, and
// log(1e-30) plus the refinement entry outside it.  Both draw kernels run it for every token group_path_applies admits, so
// the ids do not depend on whether the log-probabilities are requested (DESIGN.md §2).
template <class Noise, bool kTap>
LDM_DEVINL bool posterior_token_group(const StepParams& p, const int token, const int lane) {
  const int b = token / p.S, s = token % p.S;
  const int C = p.C;
  const int x_t = static_cast<int>(p.ids_in[token]);

  // ---- conditioning: a fixed token is copied (its log-probabilities are 0 / log(1e-30)) ----
  long long cs = 0; bool fixed = false;
  if (p.cond_flags) {
    cs = p.cond_seq[token];
    fixed = (p.cond_flags & COND_HAS_MASK) && p.cond_mask[token];
  }

  // ---- predict_start: the log-sum-exp over all classes, log p(x0) of the group's ----
  const float* lrow = p.logits + (static_cast<size_t>(b) * p.layout_rows + s) * p.ld_logits;
  int lcls[5]; bool lvalid[5];
  lane_classes(C, lane, lcls, lvalid);
  float l[5];
  const double lse = logit_lse(p, lrow, lane, lcls, lvalid, l);

  const int g = vocab_group(p, s);
  const int gst = p.grp_start[g], gn = p.grp_n[g];
  const bool refine = (p.cond_flags & COND_REFINE) && !fixed;
  const float* trow = refine ? p.refine_tbl + static_cast<size_t>(p.cond_seq_orig[token]) * C : nullptr;

  // slot 0: group class gst + lane ; slot 1: PAD (lane 0) / MASK (lane 1)
  int cls[2]; bool on[2];
  cls[0] = gst + lane; on[0] = lane < gn;
  cls[1] = lane == 0 ? p.pad_id : p.mask_id; on[1] = lane < 2;
  float lx0[2], lp[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int j = 0; j < 2; ++j) lx0[j] = (on[j] && cls[j] != p.mask_id) ? lx0_of(__ldg(lrow + cls[j]), lse) : 0.0f;
  posterior_logprob<2>(p, post_terms(p, g, p.t_post), x_t, lx0, cls, on, lp);
  float lmax = -INFINITY;
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    if (on[j]) {
      if (fixed) lp[j] = (cls[j] == cs) ? 0.0f : kLogEps;
      if (refine) lp[j] += __ldg(trow + cls[j]);
      if ((p.cond_flags & COND_PAD_DISABLE) && (s % p.n_attr != 0) && cs != p.pad_id && cls[j] == p.pad_id) lp[j] = kLogEps;
      lmax = fmaxf(lmax, lp[j]);
    }
  }
  lmax = warp_max(lmax);
  if (refine) {
    // the refinement prior (task.py:154-224: lambda on the token's own attribute band) must not lift a class outside the group
    // above log(1e-30); a caller-supplied table that does sends the token to the all-classes routine
    float tmax = 0.0f;
#pragma unroll
    for (int j = 0; j < 5; ++j) if (lvalid[j] && !in_group(p, g, lcls[j])) tmax = fmaxf(tmax, __ldg(trow + lcls[j]));
    if (warp_max(tmax) > 0.0f) return false;
  }
  // every class outside the group sits at log(1e-30): it must be out of reach of the draw.  A fixed token whose id lies outside
  // the group leaves every group class at log(1e-30) and so always goes to the all-classes routine.
  const float margin = p.mode == SAMP_DETERMINISTIC ? 0.0f : Noise::kGroupMargin * p.temperature;
  if (!(lmax - kLogEps > margin)) return false;

  if constexpr (kTap) {
    if (p.logprob_out != nullptr) {
      float* out = p.logprob_out + static_cast<size_t>(token) * C;
#pragma unroll
      for (int j = 0; j < 5; ++j) if (lvalid[j] && !in_group(p, g, lcls[j])) out[lcls[j]] = refine ? kLogEps + __ldg(trow + lcls[j]) : kLogEps;
#pragma unroll
      for (int j = 0; j < 2; ++j) if (on[j]) out[cls[j]] = lp[j];
    }
  }

  int best_c;
  if (p.mode == SAMP_DETERMINISTIC) {
    best_c = warp_argmax_first<2>(lp, cls, on);
  } else {
    float lg[2];
#pragma unroll
    for (int j = 0; j < 2; ++j) lg[j] = on[j] ? lp[j] / p.temperature : -INFINITY;
    if (p.mode == SAMP_TOP_P) {
      // sampling.py:94-109 restricted to the group: the classes outside it carry ~1e-30 of the mass, sit at the tail of the
      // descending order with a cumulative mass of ~1 > top_p (group_path_applies requires top_p < 0.9999) and are dropped in any case.
      float m = warp_max(fmaxf(lg[0], lg[1]));
      float pr[2], sm = 0.0f;
#pragma unroll
      for (int j = 0; j < 2; ++j) { pr[j] = on[j] ? expf(lg[j] - m) : 0.0f; sm += pr[j]; }
      sm = warp_sum(sm);
      pr[0] /= sm; pr[1] /= sm;
      int n_before[2] = {0, 0};
      double cum[2] = {static_cast<double>(pr[0]), static_cast<double>(pr[1])};
      for (int src = 0; src < 32; ++src) {
#pragma unroll
        for (int jj = 0; jj < 2; ++jj) {
          const bool on2 = jj == 0 ? src < gn : src < 2;                 // warp-uniform
          if (!on2) continue;
          const float v2 = __shfl_sync(0xffffffffu, lg[jj], src);
          const float p2 = __shfl_sync(0xffffffffu, pr[jj], src);
          const int c2 = jj == 0 ? gst + src : (src == 0 ? p.pad_id : p.mask_id);
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            const bool before = (v2 > lg[j]) || (v2 == lg[j] && c2 < cls[j]);   // descending sort, ties by class index
            if (before) { n_before[j] += 1; cum[j] += static_cast<double>(p2); }
          }
        }
      }
#pragma unroll
      for (int j = 0; j < 2; ++j) if (on[j] && n_before[j] > 0 && static_cast<float>(cum[j]) > p.top_p) lg[j] = -INFINITY;
    }
    if constexpr (std::is_same_v<Noise, TokenNoise>) {
      // One Philox evaluation per noise stream serves the whole token: lanes 0..8 compute the (at most 9) blocks of the group,
      // lanes 9 / 10 the blocks of PAD / MASK, then every lane fetches its words.
      const TokenNoise nz = step_noise(p, b, s);
      const int b0 = TokenNoise::block_of(gst);
      const int my_block = lane < 9 ? b0 + lane : TokenNoise::block_of(lane == 9 ? p.pad_id : p.mask_id);
      const int src0 = TokenNoise::block_of(cls[0]) - b0, src1 = lane == 0 ? 9 : 10;
      best_c = draw_class<2>(p, lg, cls, on, contract_draw<2>([&](uint32_t stream, uint32_t (&w)[2]) {
        const uint4 r = nz.block(my_block, noise_ctr(p.step_ctr, stream));
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int src = j == 0 ? src0 : src1;
          const uint4 rs = make_uint4(__shfl_sync(0xffffffffu, r.x, src), __shfl_sync(0xffffffffu, r.y, src),
                                      __shfl_sync(0xffffffffu, r.z, src), __shfl_sync(0xffffffffu, r.w, src));
          w[j] = TokenNoise::word_of(rs, cls[j]);
        }
      }));
    } else {
      best_c = draw_class<2>(p, lg, cls, on, torch_draw<2>(p, b, s, cls));   // the group's classes only
    }
  }
  if (lane == 0) p.ids_out[token] = best_c;
  embed_next(p, b, s, best_c, lane);
  return true;
}

// The steps posterior_token_group serves: ids drawn from logits (no log-prob or log p(x0) input, no log p(x0) tap, one posterior
// timestep for the batch), the constrained diffusion, mode in {deterministic, random, gumbel, top_p with top_p < 0.9999}, every
// group <= 32 classes.  Kernel parameters only: the same answer for every token of a launch.
__host__ __device__ inline bool group_path_applies(const StepParams& p) {
  bool ok = p.constrained && p.ids_out != nullptr && p.logprob_in == nullptr && p.lx0_in == nullptr && p.lx0_out == nullptr &&
            p.t_layout == nullptr &&
            (p.mode == SAMP_DETERMINISTIC || p.mode == SAMP_RANDOM || p.mode == SAMP_GUMBEL || (p.mode == SAMP_TOP_P && p.top_p < 0.9999f));
  for (int g = 0; g < p.n_attr; ++g) ok = ok && p.grp_n[g] <= 32;
  return ok;
}

// All-classes kernel: any q_type, any sampling mode, log-prob in / out.  A token of a step group_path_applies admits takes
// posterior_token_group first, exactly as in posterior_sample_group_kernel, and fills the log-prob tap from it.
template <class Noise = TokenNoise>
__global__ void __launch_bounds__(256) posterior_sample_kernel(const StepParams p) {
  const int token = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (token >= p.n_layouts * p.S) return;
  pdl_sync();
  if (group_path_applies(p) && posterior_token_group<Noise, true>(p, token, lane)) return;
  posterior_token_generic<Noise>(p, token, lane);
}

// Group-centric kernel: posterior_token_group for every token, posterior_token_generic for the ones it does not take.  Launched
// where group_kernel_applies; its ids are the all-classes kernel's in every case, bit for bit.
template <class Noise = TokenNoise>
__global__ void __launch_bounds__(256) posterior_sample_group_kernel(const StepParams p) {
  const int token = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (token >= p.n_layouts * p.S) return;
  pdl_sync();
  if (!posterior_token_group<Noise, false>(p, token, lane)) posterior_token_generic<Noise>(p, token, lane);
}

// test tap of the torch-generator contract: out[i] = element i of one exponential_ (which = 1) or rand (which = 0) draw of
// `n` elements, through the TorchNoise the draw kernels use
__global__ void torch_noise_tap_kernel(const TorchNoise nz, const uint32_t n, const int which, float* __restrict__ out) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    out[i] = which ? TorchNoise::exponential(nz.word(i)) : TorchNoise::rand(nz.word(i));
}

// where posterior_sample_group_kernel may replace the all-classes kernel: no log-prob tap to fill
inline bool group_kernel_applies(const StepParams& p) { return group_path_applies(p) && p.logprob_out == nullptr; }

// ---------------------------------------------------------------------------------------------------------
// Training-side terms of the variational bound, per token: what `forward` computes after x_t has been drawn
// (T/models/categorical_diffusion/constrained.py:262-333, vanilla.py:177-243):
//   log_x0_recon   = predict_start(x_t, t)                       (logits of the denoiser run at per-layout timesteps)
//   log_model_prob = q_posterior(log_x0_recon, x_t, t)           log_true_prob = q_posterior(log_onehot(x0), x_t, t)
//   kl   = sum_c exp(true)(true - model) * mask_weight           util.py multinomial_kl, constrained.py:295-302
//   nll  = -sum_c exp(log_onehot(x0)) * model                    log_categorical, :304
//   aux  = sum_{c != MASK} exp(log_onehot(x0)) (log_onehot(x0) - log_x0_recon) * mask_weight     :321-325
// plus the argmax ids the reference's accuracy book-keeping uses (:273-292).  One warp per token, forward only.
struct VbParams {
  StepParams sp;                         // logits / ids_in (= x_t) / t_layout / schedule / optional logprob_out (= log_model_prob)
  const long long* x0;                   // [n_layouts][S]
  float w_mask, w_other;                 // mask_weight[0] (x_t == MASK), mask_weight[1]
  float* kl_tok; float* nll_tok; float* aux_tok;   // [n_layouts][S]; aux_tok may be nullptr
  long long* x0_recon; long long* xtm1_recon;      // [n_layouts][S] or nullptr
};

__global__ void __launch_bounds__(256) vb_terms_kernel(const VbParams v) {
  const StepParams& p = v.sp;
  const int token = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (token >= p.n_layouts * p.S) return;
  pdl_sync();
  const int b = token / p.S, s = token % p.S;
  const int C = p.C;
  int cls[5]; bool valid[5];
  lane_classes(C, lane, cls, valid);
  const int x_t = static_cast<int>(p.ids_in[token]);
  const int x0 = static_cast<int>(v.x0[token]);
  const int t = __ldg(p.t_layout + b);
  float lx0[5], lmp[5], lxs[5], ltp[5];
#pragma unroll
  for (int j = 0; j < 5; ++j) lxs[j] = (cls[j] == x0) ? 0.0f : kLogEps;            // index_to_log_onehot (util.py:34-40)
  posterior_token_logprob(p, s, x_t, t, lxs, cls, valid, ltp);
  predict_start_token(p, p.logits + (static_cast<size_t>(b) * p.layout_rows + s) * p.ld_logits, lane, cls, valid, lx0);
  posterior_token_logprob(p, s, x_t, t, lx0, cls, valid, lmp);
  float kl = 0.0f, nll = 0.0f, aux = 0.0f;
#pragma unroll
  for (int j = 0; j < 5; ++j) {
    if (valid[j]) {
      kl += expf(ltp[j]) * (ltp[j] - lmp[j]);
      nll += expf(lxs[j]) * lmp[j];
      if (cls[j] < C - 1) aux += expf(lxs[j]) * (lxs[j] - lx0[j]);
    }
  }
  kl = warp_sum(kl); nll = -warp_sum(nll); aux = warp_sum(aux);
  const float w = (x_t == p.mask_id) ? v.w_mask : v.w_other;
  if (p.logprob_out != nullptr) {
#pragma unroll
    for (int j = 0; j < 5; ++j) if (valid[j]) p.logprob_out[static_cast<size_t>(token) * C + cls[j]] = lmp[j];
  }
  const int a0 = v.x0_recon ? warp_argmax_first<5>(lx0, cls, valid) : 0;
  const int a1 = v.xtm1_recon ? warp_argmax_first<5>(lmp, cls, valid) : 0;
  if (lane == 0) {
    v.kl_tok[token] = kl * w; v.nll_tok[token] = nll;
    if (v.aux_tok) v.aux_tok[token] = aux * w;
    if (v.x0_recon) v.x0_recon[token] = a0;
    if (v.xtm1_recon) v.xtm1_recon[token] = a1;
  }
}

// mean over the S tokens of every layout (mean_except_batch, util.py:11-12): one warp per layout, fixed summation order
__global__ void row_mean_kernel(const float* __restrict__ in, float* __restrict__ out, int n_rows, int S) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (row >= n_rows) return;
  pdl_sync();
  float acc = 0.0f;
  for (int i = lane; i < S; i += 32) acc += in[static_cast<size_t>(row) * S + i];
  acc = warp_sum(acc);
  if (lane == 0) out[row] = acc / static_cast<float>(S);
}

// q_pred on full-vocabulary (n_layouts, S, C) log tensors: log q(x_t | x_0) for arbitrary log p(x_0) (constrained.py:112-133 per
// attribute on the partial vocabularies, vanilla.py:90-110); classes outside the token's group stay at log(1e-30) like
// Converter.p_to_f_log fills them.  t may be -1 (wraps to T, :115).
// one_step = 1: q_pred_one_timestep, log q(x_t | x_{t-1}) with the per-step tables (constrained.py:92-110), t in [0, T).
__global__ void q_pred_kernel(const StepParams p, const float* __restrict__ lx, float* __restrict__ out, const int one_step) {
  const size_t n = static_cast<size_t>(p.n_layouts) * p.S * p.C;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % p.C); const size_t tok = i / p.C; const int s = static_cast<int>(tok % p.S); const int b = static_cast<int>(tok / p.S);
    const int g = vocab_group(p, s);
    float r = kLogEps;
    if (in_group(p, g, c)) {
      const int TT = p.T + 1;
      const int t = (__ldg(p.t_layout + b) + TT) % TT;
      const float* tab = p.sched + static_cast<size_t>(g) * 8 * TT;
      const int ra = one_step ? 0 : 3, rb = one_step ? 1 : 4, rc = one_step ? 2 : 5, r1 = one_step ? 6 : 7;   // (at, bt, ct, 1-ct) vs their cumulative products
      r = (c != p.mask_id) ? log_add_exp(lx[i] + tab[ra * TT + t], tab[rb * TT + t]) : log_add_exp(lx[i] + tab[r1 * TT + t], tab[rc * TT + t]);
    }
    out[i] = r;
  }
}

// log_sample_categorical with train_sampling = "gumbel" (constrained.py:208-221): ids = argmax_c(logits_c + Gumbel noise) on
// (n_layouts, S, C) logits; classes the caller wants excluded carry -inf.  Noise = Philox stream 2, the stream q_sample_kernel draws
// from, so log_sample_categorical(q_pred(log_onehot(x0), t)) reproduces ldm_q_sample bit for bit.  One warp per token.
__global__ void __launch_bounds__(256) gumbel_argmax_kernel(const float* __restrict__ logits, long long* __restrict__ ids_out, int n_layouts, int S, int C,
                                                            unsigned long long seed, long long b_global0) {
  const int token = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (token >= n_layouts * S) return;
  const int b = token / S, s = token % S;
  int cls[5]; bool on[5];
  lane_classes(C, lane, cls, on);
  uint32_t w[5];
  TokenNoise(seed, b_global0, b, S, s).lane_words(lane, noise_ctr(0, 2), w);
  float score[5];
#pragma unroll
  for (int j = 0; j < 5; ++j) {
    const float l = on[j] ? logits[static_cast<size_t>(token) * C + cls[j]] : -INFINITY;
    on[j] = l > -INFINITY;
    score[j] = on[j] ? l + gumbel_of(u01_from_bits(w[j])) : -INFINITY;
  }
  const int best_c = warp_argmax_first<5>(score, cls, on);
  if (lane == 0) ids_out[token] = best_c;
}

// ---------------------------------------------------------------------------------------------------------
// Forward (corruption) process on ids: x_t ~ q(x_t | x_0) with the reference's Gumbel-argmax draw.
// q_pred  T/models/categorical_diffusion/constrained.py:112-133 (vanilla.py:90-110), log_sample_categorical :208-221,
// q_sample :223-230; the training forward applies it per attribute on the partial vocabularies (:232-260) -- here per token
// on the full ids (classes outside the token's group are impossible).  One warp per token, same class ownership as above.
__global__ void __launch_bounds__(256) q_sample_kernel(const StepParams p, const long long* __restrict__ x0, const int* __restrict__ t,
                                                       long long* __restrict__ xt) {
  const int token = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (token >= p.n_layouts * p.S) return;
  const int b = token / p.S, s = token % p.S;
  const int x0_id = static_cast<int>(x0[token]);
  const int tb = t[b];
  const int g = vocab_group(p, s);
  const int TT = p.T + 1;
  const float* tab = p.sched + static_cast<size_t>(g) * 8 * TT;
  const float lcat = tab[3 * TT + tb], lcbt = tab[4 * TT + tb], lcct = tab[5 * TT + tb], l1m = tab[7 * TT + tb];
  int cls[5]; bool on[5];
  lane_classes(p.C, lane, cls, on);
  uint32_t w[5];
  TokenNoise(p.seed, p.b_global0, b, p.S, s).lane_words(lane, noise_ctr(0, 2), w);
  float score[5];
#pragma unroll
  for (int j = 0; j < 5; ++j) {
    const int c = cls[j];
    on[j] = on[j] && in_group(p, g, c);
    const float v = (c == x0_id) ? 0.0f : kLogEps;                       // log(clamp(onehot, 1e-30))
    const float logit = (c != p.mask_id) ? log_add_exp(v + lcat, lcbt) : log_add_exp(v + l1m, lcct);
    score[j] = on[j] ? logit + gumbel_of(u01_from_bits(w[j])) : -INFINITY;
  }
  const int best_c = warp_argmax_first<5>(score, cls, on);
  if (lane == 0) xt[token] = best_c;
}

// ---------------------------------------------------------------------------------------------------------
// ids -> layouts on the device: LayoutSequenceTokenizer.decode (T/helpers/layout_tokenizer.py:255-266, :106-114) +
// BboxTokenizer.decode (T/helpers/bbox_tokenizer.py:117-174).  One thread per element; centers == nullptr: linear bins.
// An element is valid when its label is a category and every bbox slot holds a bbox id (any of the n_bbox_ids, whatever its
// variable); each slot's bin is its id minus the first id of its variable, clamped, and lands at its variable's place in xywh.
__global__ void decode_kernel(const long long* __restrict__ ids, const float* __restrict__ centers /*[4][n_bins] or null*/,
                              float* __restrict__ bbox /*[B][E][4]*/, long long* __restrict__ label /*[B][E]*/,
                              unsigned char* __restrict__ mask /*[B][E]*/, int n_layouts, int n_elem, const TokenLayout tl) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_layouts * n_elem) return;
  const int n_bins = tl.n_bins;
  const long long* tk = ids + static_cast<size_t>(i) * tl.n_attr;
  const long long lab = tk[0];
  bool valid = lab >= 0 && lab < tl.n_cat;
  float bb[4];
#pragma unroll
  for (int k = 1; k < 5; ++k) {
    const long long v = tk[k] - tl.n_cat;
    valid = valid && v >= 0 && v < tl.n_bbox_ids;
    const int a = tl.var[k] - 1;                                          // x, y, w, h
    long long bin = tk[k] - tl.start[k];
    bin = bin < 0 ? 0 : (bin > n_bins - 1 ? n_bins - 1 : bin);            // clamp (avoid OOV)
    if (centers != nullptr) bb[a] = fminf(fmaxf(centers[a * n_bins + bin], 0.0f), 1.0f);
    else bb[a] = static_cast<float>(a < 2 ? bin : bin + 1) * (1.0f / n_bins);
  }
  float4* o = reinterpret_cast<float4*>(bbox) + i;
  *o = valid ? make_float4(bb[0], bb[1], bb[2], bb[3]) : make_float4(0.f, 0.f, 0.f, 0.f);
  label[i] = valid ? lab : 0;
  mask[i] = valid ? 1 : 0;
}

// ---------------------------------------------------------------------------------------------------------
// layouts -> ids -> cond on the device: LayoutSequenceTokenizer.encode (T/helpers/layout_tokenizer.py:208-253, :96-104) +
// BboxTokenizer.encode (T/helpers/bbox_tokenizer.py:86-114) + the deterministic branches of get_cond (T/helpers/task.py:94-110
// c / cwh, :116-117 gt, :126-140 refinement with the caller's perturbed boxes).  One thread per element.
enum : int { COND_TYPE_C = 0, COND_TYPE_CWH = 1, COND_TYPE_REFINEMENT = 2, COND_TYPE_GT = 3 };

__global__ void make_cond_kernel(const long long* __restrict__ label /*[B][E]*/, const float* __restrict__ bbox /*[B][E][4]*/,
                                 const unsigned char* __restrict__ elem_mask /*[B][E]*/, const float* __restrict__ centers /*[4][n_bins] or null*/,
                                 long long* __restrict__ seq /*[B][E*5]*/, unsigned char* __restrict__ mask /*[B][E*5]*/,
                                 long long* __restrict__ seq_orig /*[B][E*5] or null*/, int n_layouts, int n_elem, const TokenLayout tl,
                                 int pad_id, int mask_id, int cond_type, float d32 /*float(1/n_bins)*/, float hi32 /*float(1 - 1/n_bins)*/) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_layouts * n_elem) return;
  const int n_bins = tl.n_bins;
  const bool valid = elem_mask[i] != 0;
  const float4 bb = reinterpret_cast<const float4*>(bbox)[i];
  const float v[4] = {bb.x, bb.y, bb.z, bb.w};
  int bins[4];
#pragma unroll
  for (int a = 0; a < 4; ++a) {
    int bin;
    if (centers == nullptr) {
      // float32 like torch: clamp, (w, h: - d), * n_bins, round half to even (bbox_tokenizer.py:90-93)
      const float q = a < 2 ? fminf(fmaxf(v[a], 0.0f), hi32) : __fsub_rn(fminf(fmaxf(v[a], d32), 1.0f), d32);
      bin = __float2int_rn(__fmul_rn(static_cast<float>(n_bins), q));
    } else {
      // nearest cluster centre, first index on ties (KMeans.predict, :95-104)
      float best = INFINITY; bin = 0;
      for (int k = 0; k < n_bins; ++k) {
        const float df = __fsub_rn(v[a], centers[a * n_bins + k]);
        const float dist = __fmul_rn(df, df);
        if (dist < best) { best = dist; bin = k; }
      }
    }
    bins[a] = bin;
  }
  // slot k: its variable's bin plus the first id of that variable (the offsets and the reorder of bbox_tokenizer.py:105-113)
  long long tok[5];
  tok[0] = label[i];
#pragma unroll
  for (int k = 1; k < 5; ++k) tok[k] = static_cast<long long>(bins[tl.var[k] - 1]) + tl.start[k];
#pragma unroll
  for (int k = 0; k < 5; ++k) {
    const long long t = valid ? tok[k] : pad_id;                          // _fix_padded_sequences
    // get_cond keeps slots by variable name (task.py:103-105): c for c / refinement, c, w, h for cwh
    const int var = tl.var[k];
    bool keep;
    if (cond_type == COND_TYPE_C) keep = var == 0;
    else if (cond_type == COND_TYPE_CWH) keep = var == 0 || var == 3 || var == 4;
    else if (cond_type == COND_TYPE_REFINEMENT) keep = var == 0;
    else keep = true;
    long long s = keep ? t : mask_id;
    if (!valid) s = pad_id;
    const size_t o = static_cast<size_t>(i) * 5 + k;
    seq[o] = s;
    mask[o] = cond_type == COND_TYPE_GT ? (valid ? 1 : 0) : ((valid && keep) || !valid ? 1 : 0);
    if (seq_orig != nullptr) seq_orig[o] = t;
  }
}

}  // namespace ldm
