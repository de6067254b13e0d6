/*
 * ldm_b200 -- C ABI of the H100-native LayoutDM sampling path (discrete-diffusion denoising loop).
 *
 * The reference (CyberAgentAILab/layout-dm) is pure Python: it has NO plugin / FFI boundary.  The seam this
 * library sits behind is the Python class API
 *     LayoutDM.sample()                               src/trainer/trainer/models/layoutdm.py:77-88
 *     BaseMaskAndReplaceDiffusion.sample()            src/trainer/trainer/models/categorical_diffusion/base.py:293-371
 *     BaseMaskAndReplaceDiffusion._sample_single_step base.py:205-291
 * and each entry point below names the reference code it replaces.  `layoutdm_b200/` (ctypes) is the host
 * mirror of that class API on top of these functions; INTEGRATION.md shows the stub a reference maintainer adds.
 *
 * Conventions
 *   - plain C types only; every pointer is caller-owned; `*_dev` = CUDA device memory on the handle's device,
 *     `*_host` = host memory (pinned or pageable).  ids are int64 like the reference's LongTensor.
 *   - all launches go to the caller's `stream` (a cudaStream_t passed as void*); no device synchronisation
 *     inside ldm_step / ldm_sample_loop; ldm_sample_host synchronises the stream before returning.
 *   - return value 0 = ok, < 0 = error (LDM_ERR_*); ldm_last_error() returns a thread-local message.
 *   - one handle may be used from one stream at a time; handles on different devices are independent.
 */
#ifndef LDM_B200_H_
#define LDM_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LDM_OK 0
#define LDM_ERR_INVALID (-1)      /* bad argument (the Python mirror raises AssertionError / NotImplementedError like the reference) */
#define LDM_ERR_CUDA (-2)         /* CUDA runtime / driver error */
#define LDM_ERR_UNSUPPORTED (-3)  /* model shape outside what the sm_90a kernels are built for */

typedef struct LdmHandle LdmHandle;

/* Model description: tokenizer vocabulary (layout_tokenizer.py:79-82,296-313) + denoiser dims
 * (config/backbone/medium.yaml shrunk by 29/32, layoutdm.py:54) + diffusion schedule (base.py:35-69). */
typedef struct {
  int32_t n_cat;          /* 25 rico25, 5 publaynet */
  int32_t n_bins;         /* 32 */
  int32_t n_elem;         /* 25 (max_seq_length) */
  int32_t n_attr;         /* 5  (c,x,y,w,h) */
  int32_t d_model;        /* 464 */
  int32_t n_heads;        /* 8 */
  int32_t d_ff;           /* 1856 */
  int32_t n_layers;       /* 4 */
  int32_t num_timesteps;  /* T (== AdaLN embedding rows) */
  int32_t q_type;         /* 0 = constrained (per-attribute transition matrices), 1 = vanilla */
  int32_t operand_dtype;  /* tensor-core operand type, accumulation is fp32: 0 = fp16, 1 = bf16, 2 = bf16x3 (every operand
                             a bf16 pair hi = bf16(x), lo = bf16(x - hi); products a_hi w_hi + a_hi w_lo + a_lo w_hi: fp32-class
                             accuracy for 3x the MMAs, 2x the operand bytes and ~1.24 MB more workspace per layout);
                             other values: LDM_ERR_INVALID */
  int32_t device;         /* CUDA device ordinal */
  double att_1, att_T, ctt_1, ctt_T;  /* alpha_schedule() endpoints, util.py:47-49 */
} LdmModelDesc;

/* fp32 arrays (host for ldm_create, device for ldm_load_weights) in the reference's own parameter layout (state_dict, SURVEY.md 8a-a5), layers stacked on dim 0.
 * C = n_cat + 4*n_bins + 2, S = n_elem*n_attr, d = d_model, f = d_ff, L = n_layers, T = num_timesteps. */
typedef struct {
  const float* cat_emb;      /* [C][d]        transformer.cat_emb.weight */
  const float* pos_table;    /* [S][d]        elem_emb[s/5] + attr_emb[s%5]  (or pos_emb[s]) */
  const float* in_proj_w;    /* [L][3d][d]    layers.l.self_attn.in_proj_weight */
  const float* in_proj_b;    /* [L][3d] */
  const float* out_proj_w;   /* [L][d][d] */
  const float* out_proj_b;   /* [L][d] */
  const float* linear1_w;    /* [L][f][d] */
  const float* linear1_b;    /* [L][f] */
  const float* linear2_w;    /* [L][d][f] */
  const float* linear2_b;    /* [L][d] */
  const float* norm1_emb;    /* [L][T][d]     layers.l.norm1.emb.weight */
  const float* norm1_w;      /* [L][2d][d]    layers.l.norm1.linear.weight */
  const float* norm1_b;      /* [L][2d] */
  const float* norm2_w;      /* [L][d] */
  const float* norm2_b;      /* [L][d] */
  const float* head_ln_w;    /* [d]           head.0.weight */
  const float* head_ln_b;    /* [d] */
  const float* head_w;       /* [C][d]        head.1.weight */
} LdmWeights;

/* Conditioning of one call (base.py:243-284; cond dict built by helpers/task.py:27-151). Device pointers, [B][S]. */
typedef struct {
  const int64_t* seq;          /* cond["seq"]; NULL = unconditional */
  const uint8_t* mask;         /* cond["mask"] (1 = token is fixed); NULL = no strong constraint */
  const int64_t* seq_orig;     /* cond["seq_orig"] (refinement) or NULL */
  const float* refine_table;   /* [C][C], already multiplied by +-refine_lambda (task.py:154-224) or NULL */
  int32_t pad_disable;         /* 1 for cond types c / cwh / refinement / relation (base.py:272-284) */
  /* cond = "relation" (base.py:261-269): gradient-based logit adjustment between the posterior and the draw, replacing
   * `update` (logit_adjustment.py:88-126; relation_mode "average").  rel_adj == NULL: off. */
  const int32_t* rel_adj;      /* [B][1+n_elem][1+n_elem] edge_attr bit masks (data/util.py:14-27) of the edge i -> j of
                                  cond["batch_w_canvas"], node 0 = canvas (AddCanvasElement), 0 = no edge */
  const float* rel_centers;    /* [4][n_bins] bbox bin centres (x, y, w, h) or NULL = linear quantisation */
  float rel_lambda;            /* sampling_cfg.relation_lambda: SGD learning rate (logit_adjustment.py:101-103) */
  int32_t rel_num_update;      /* sampling_cfg.relation_num_update (applied for t_model >= 10 only, :105) */
  int32_t rel_batch_total;     /* batch size the reference's loss.mean() runs over (the GLOBAL batch when sharded); <= 0: B */
} LdmCond;

/* helpers/sampling.py:13-59 */
#define LDM_SAMPLING_DETERMINISTIC 0
#define LDM_SAMPLING_RANDOM 1
#define LDM_SAMPLING_TOP_K 2
#define LDM_SAMPLING_TOP_P 3
#define LDM_SAMPLING_GUMBEL 4
typedef struct {
  int32_t mode;
  float temperature;
  float top_p;
  int32_t top_k;
} LdmSampling;

/* Where a draw's noise comes from (DESIGN.md §7).
 *   LDM_NOISE_CONTRACT : the project's Philox contract keyed by (seed, step_ctr, global layout, token, class); offset and
 *                        total_layouts are not read.
 *   LDM_NOISE_TORCH    : the numbers torch's CUDA generator with this seed and offset would give the reference's draw
 *                        (helpers/sampling.py:81-130 on a (total_layouts, C, S) batch: rand_like for name="gumbel", then
 *                        multinomial's exponential_), so a seeded run reproduces the reference on the GPU.  Step k of a call
 *                        draws at offset + k * (one step's advance, ldm_noise_advance); layouts [b_global0, b_global0 + B) of
 *                        total_layouts get the slice of the whole batch's draw.  offset must be a multiple of 4 (torch's
 *                        offsets are) and total_layouts * S * C < 2^31 (LDM_ERR_UNSUPPORTED otherwise: torch splits larger
 *                        draws).  Tied to torch's distribution kernels (ATen/native/cuda/DistributionTemplates.h). */
#define LDM_NOISE_CONTRACT 0
#define LDM_NOISE_TORCH 1
typedef struct {
  int32_t kind;
  uint64_t seed;
  uint64_t offset;
  int64_t total_layouts;
} LdmNoise;

/* Build a handle: uploads and repacks the weights (per-head padded QKV, 16-bit operands, AdaLN table for all t,
 * schedule tables, TMA descriptors).  Replaces model construction + .to(device) for the sampling path. */
int ldm_create(const LdmModelDesc* desc, const LdmWeights* weights, LdmHandle** out);
int ldm_destroy(LdmHandle* h);
/* Repack new weights into the handle's existing buffers on `stream` (what ldm_create does with its host arrays), so that a
 * handle follows a model being trained or given another checkpoint.  w: fp32 DEVICE pointers on the handle's device, in the
 * LdmWeights layout and the shapes of the handle's LdmModelDesc (a different shape is a new handle, not a reload).  No
 * allocation and no synchronisation; tensor maps and a captured loop graph stay valid (the addresses do not change).  Work
 * already queued on `stream` sees the old weights, later work the new ones; work on other streams must be ordered by the
 * caller, as for every call on a handle.  The arrays must stay valid until the work queued here has run.
 * A null handle, a null field or a pointer that is not device memory of the handle's device: LDM_ERR_INVALID. */
int ldm_load_weights(LdmHandle* h, const LdmWeights* weights_dev, void* stream);

/* One denoising step == BaseMaskAndReplaceDiffusion._sample_single_step (base.py:205-291) on token ids:
 *   ids_in_dev [B][S] (x_t)  ->  ids_out_dev [B][S] (x_{t-1}).
 * t_model: denoiser timestep; t_post: posterior timestep (after time_difference / skip_step, base.py:218-240).
 * Noise: Philox4x32-10 keyed by (seed, step_ctr, global layout index b_global0 + b, token, class) -- DESIGN.md.
 * Optional taps (device, may be NULL):
 *   logits_out_dev  [B][S][C] fp32  denoiser logits                 (CategoricalTransformer.forward, nn_lib.py:191-237)
 *   logprob_out_dev [B][S][C] fp32  log p(x_{t-1}|x_t) after the cond adjustments (input of sample(), base.py:287)
 *   logits_in_dev   [B][S][C] fp32  skip the denoiser and use these logits
 *   logprob_in_dev  [B][S][C] fp32  skip everything but [PAD-disable when cond->pad_disable, base.py:271-284, and] the draw
 *                                   (hook for an external logit adjustment such as the reference's own `update`) */
int ldm_step(LdmHandle* h, int32_t B, const int64_t* ids_in_dev, int32_t t_model, int32_t t_post,
             const LdmCond* cond, const LdmSampling* sampling, uint64_t seed, uint32_t step_ctr, int64_t b_global0,
             int64_t* ids_out_dev, float* logits_out_dev, float* logprob_out_dev,
             const float* logits_in_dev, const float* logprob_in_dev, void* stream);
/* ldm_step with the noise described by `noise` (step_ctr: the contract's counter; torch noise draws at noise->offset) */
int ldm_step_noise(LdmHandle* h, int32_t B, const int64_t* ids_in_dev, int32_t t_model, int32_t t_post,
                   const LdmCond* cond, const LdmSampling* sampling, const LdmNoise* noise, uint32_t step_ctr, int64_t b_global0,
                   int64_t* ids_out_dev, float* logits_out_dev, float* logprob_out_dev,
                   const float* logits_in_dev, const float* logprob_in_dev, void* stream);
/* How far a call of n_steps steps on a batch of total_layouts layouts moves torch's generator offset (0 for deterministic,
 * one draw per step, two for gumbel); < 0: LDM_ERR_*.  The one place that knows torch's launch policy. */
int64_t ldm_noise_advance(const LdmHandle* h, int64_t total_layouts, const LdmSampling* sampling, int32_t n_steps);

/* The whole loop == BaseMaskAndReplaceDiffusion.sample (base.py:293-371) for a precomputed timestep plan.
 *   t_model_host / t_post_host : n_steps entries each (host).
 *   ids_init_dev : [B][S] start state or NULL (= cond->seq if given, else all MASK, base.py:337-346)
 *   ids_out_dev  : [B][S] final ids
 *   ids_trace_dev: [n_steps][B][S] or NULL (get_intermediate_results, base.py:318-319,364-369) */
int ldm_sample_loop(LdmHandle* h, int32_t B, int32_t n_steps, const int32_t* t_model_host, const int32_t* t_post_host,
                    const LdmCond* cond, const LdmSampling* sampling, uint64_t seed, int64_t b_global0,
                    const int64_t* ids_init_dev, int64_t* ids_out_dev, int64_t* ids_trace_dev, void* stream);
/* ldm_sample_loop with the noise described by `noise`; a replayed CUDA graph takes the new seed / offset */
int ldm_sample_loop_noise(LdmHandle* h, int32_t B, int32_t n_steps, const int32_t* t_model_host, const int32_t* t_post_host,
                          const LdmCond* cond, const LdmSampling* sampling, const LdmNoise* noise, int64_t b_global0,
                          const int64_t* ids_init_dev, int64_t* ids_out_dev, int64_t* ids_trace_dev, void* stream);

/* Same loop with HOST buffers (what `LayoutDM.sample()` does around the core: H2D of cond, D2H of ids;
 * base.py:328-330,371): copies the inputs host->device, runs the loop, copies ids_out device->host and
 * synchronises.  cond_* / ids_init may be NULL.  Returns bytes moved through the optional out params. */
int ldm_sample_host(LdmHandle* h, int32_t B, int32_t n_steps, const int32_t* t_model_host, const int32_t* t_post_host,
                    const int64_t* cond_seq_host, const uint8_t* cond_mask_host, const int64_t* cond_seq_orig_host,
                    const float* refine_table_host, int32_t pad_disable, const LdmSampling* sampling, uint64_t seed,
                    int64_t b_global0, const int64_t* ids_init_host, int64_t* ids_out_host, void* stream,
                    int64_t* h2d_bytes, int64_t* d2h_bytes);

/* Forward (corruption) process on ids: x_t ~ q(x_t | x_0) at per-layout timesteps t_dev[B] with the reference's
 * Gumbel-argmax draw == q_sample / log_sample_categorical (constrained.py:208-230, vanilla.py:153-158) as the training
 * forward applies it per attribute (constrained.py:232-260).  Noise: Philox stream 2 of the contract in DESIGN.md. */
int ldm_q_sample(LdmHandle* h, int32_t B, const int64_t* x0_ids_dev, const int32_t* t_dev, uint64_t seed, int64_t b_global0,
                 int64_t* xt_ids_dev, void* stream);

/* Training-side API on (B, S, C) log tensors with PER-LAYOUT timesteps t_dev[B] (SURVEY 8b "must keep working" / 8f-3).  Layout note:
 * these tensors are token-major [B][S][C]; the reference's are (B, C, S) -- the Python mirror transposes.
 *   ldm_predict_start : log p(x0 | x_t) = predict_start(log_onehot(xt), t)  (base.py:127-146: denoiser at per-layout timesteps,
 *                       float64 log-softmax over the C-1 non-MASK classes, MASK = -70, clamp [-70, 0]); optional fp32 logits tap.
 *   ldm_q_posterior   : q(x_{t-1} | x_t, x0~) for ANY log p(x0) (constrained.py:135-206, vanilla.py:112-151), x_t as ids.
 *   ldm_q_pred        : log q(x_t | x0) for any log p(x0) (constrained.py:112-133 on each attribute's partial vocabulary,
 *                       vanilla.py:90-110), t may be -1 (wraps to T); classes outside a token's vocabulary group = log(1e-30).
 *   ldm_vb_terms      : what `forward` computes after x_t = q_sample(x0, t) (constrained.py:262-333, vanilla.py:177-243), forward
 *                       only: per layout  kl = mean_s(multinomial_kl(log_true_prob, log_model_prob) * mask_weight),
 *                       decoder_nll = mean_s(-log_categorical(log_onehot(x0), log_model_prob)),  kl_aux = mean_s(multinomial_kl(
 *                       log_onehot(x0)[:-1], log_x0_recon[:-1]) * mask_weight); optional taps: log_model_prob [B][S][C] and the
 *                       argmax ids of log_x0_recon / log_model_prob that feed the reference's accuracy book-keeping (:273-292). */
int ldm_predict_start(LdmHandle* h, int32_t B, const int64_t* xt_ids_dev, const int32_t* t_dev, float* log_x0_out_dev,
                      float* logits_out_dev, void* stream);
int ldm_q_posterior(LdmHandle* h, int32_t B, const float* log_x_start_dev, const int64_t* xt_ids_dev, const int32_t* t_dev,
                    float* log_prob_out_dev, void* stream);
int ldm_q_pred(LdmHandle* h, int32_t B, const float* log_x_start_dev, const int32_t* t_dev, float* log_prob_out_dev, void* stream);
/* q_pred_one_timestep: log q(x_t | x_{t-1}) with the per-step tables (constrained.py:92-110, vanilla.py:74-88), t in [0, T) */
int ldm_q_pred_one_timestep(LdmHandle* h, int32_t B, const float* log_x_t_dev, const int32_t* t_dev, float* log_prob_out_dev, void* stream);
/* log_sample_categorical with train_sampling "gumbel" (constrained.py:208-221): ids = argmax_c(logits + Gumbel noise) on [B][S][C]
 * logits (-inf = excluded class); noise = Philox stream 2 of the contract, the stream ldm_q_sample draws from. */
int ldm_gumbel_argmax(LdmHandle* h, int32_t B, const float* logits_dev, uint64_t seed, int64_t b_global0, int64_t* ids_out_dev, void* stream);
int ldm_vb_terms(LdmHandle* h, int32_t B, const int64_t* x0_ids_dev, const int64_t* xt_ids_dev, const int32_t* t_dev,
                 float mask_weight_mask, float mask_weight_other, float* kl_out_dev, float* decoder_nll_out_dev,
                 float* kl_aux_out_dev, float* log_model_prob_out_dev, int64_t* x0_recon_ids_out_dev,
                 int64_t* xtm1_recon_ids_out_dev, void* stream);

/* ids -> layouts on the device == LayoutSequenceTokenizer.decode (layout_tokenizer.py:255-266) + BboxTokenizer.decode
 * (bbox_tokenizer.py:117-174).  centers_dev: [4][n_bins] cluster centres (kmeans / percentile) or NULL for linear bins.
 * Outputs (device): bbox [B][n_elem][4] f32 (xywh), label [B][n_elem] i64, mask [B][n_elem] u8 (1 = valid element). */
int ldm_decode(LdmHandle* h, int32_t B, const int64_t* ids_dev, const float* centers_dev, float* bbox_out_dev,
               int64_t* label_out_dev, uint8_t* mask_out_dev, void* stream);

/* layouts -> cond on the device == LayoutSequenceTokenizer.encode (layout_tokenizer.py:208-253) + BboxTokenizer.encode
 * (bbox_tokenizer.py:86-114) + get_cond (helpers/task.py:27-151) for the deterministic types:
 *   cond_type 0 = "c" (:94-110), 1 = "cwh" (:94-110), 2 = "refinement" (:126-140; bbox_dev already carries the caller's
 *   N(0, 0.1) perturbation of :127), 3 = "gt" (:116-117).  "partial" / "random" draw host random numbers and stay in Python.
 * Inputs (device): label [B][n_elem] i64, bbox [B][n_elem][4] f32 xywh, elem_mask [B][n_elem] u8 (valid elements first),
 * centers_dev [4][n_bins] cluster centres or NULL for linear bins.  Outputs (device): seq [B][S] i64, mask [B][S] u8
 * (1 = fixed token), seq_orig [B][S] i64 (refinement only, else may be NULL) -- exactly the LdmCond fields. */
int ldm_make_cond(LdmHandle* h, int32_t B, int32_t cond_type, const int64_t* label_dev, const float* bbox_dev,
                  const uint8_t* elem_mask_dev, const float* centers_dev, int64_t* seq_out_dev, uint8_t* mask_out_dev,
                  int64_t* seq_orig_out_dev, void* stream);

/* Introspection */
int64_t ldm_launch_count(const LdmHandle* h);            /* kernels launched by this handle so far */
int32_t ldm_num_classes(const LdmHandle* h);             /* C */
int32_t ldm_seq_len(const LdmHandle* h);                 /* S */
/* copies the [G][8][T+1] fp32 schedule tables (log_at, log_bt, log_ct, log_cumprod_{at,bt,ct}, log_1_min_ct,
 * log_1_min_cumprod_ct; constrained.py:64-90) to host; returns number of floats written (or needed if dst NULL). */
int64_t ldm_get_schedule(const LdmHandle* h, float* dst_host, int64_t capacity);
/* test tap: AdaLN table [L][T][2d] fp32 to host */
int64_t ldm_get_adaln_table(const LdmHandle* h, float* dst_host, int64_t capacity);

/* Per-kernel timing for bench.py's roofline: between begin and end every launch is bracketed by a CUDA-event pair on
 * the launching stream; end() synchronises and returns the summed milliseconds and launch counts per category:
 * 0 embed+AdaLN, 1 QKV GEMM, 2 attention, 3 out-proj GEMM (+residual+LayerNorm2), 4 FF1 GEMM, 5 FF2 GEMM (+residual+AdaLN /
 * head LN), 6 head GEMM, 7 posterior+sampling epilogue, 8 misc. */
#define LDM_PROFILE_CATEGORIES 9
int ldm_profile_begin(LdmHandle* h);
int ldm_profile_end(LdmHandle* h, float* ms_per_category, int64_t* launches_per_category, int32_t n_categories);

/* test taps (tests/ and tools/ only): stop the denoiser after n launches (0 = off); read a workspace buffer
 * ("x32","y32","x16","z16","att16","qkv16","hid16","logits"; operand_dtype 2 also the lo planes "x16_lo","z16_lo","att16_lo",
 * "qkv16_lo","hid16_lo") of the first n_layouts layouts to host; returns bytes (< 0: unknown name). */
int ldm_debug_set_stop_after(LdmHandle* h, int32_t n_launches);
/* test tap of LDM_NOISE_TORCH: out_dev[numel] = the float32 values torch's CUDA generator (this seed / offset, the handle's
 * device) gives exponential_ (which = 1) or rand (which = 0) of a contiguous tensor of numel < 2^31 elements, computed by
 * the device code the draw kernels use */
int ldm_debug_torch_noise(const LdmHandle* h, int64_t numel, uint64_t seed, uint64_t offset, int32_t which, float* out_dev, void* stream);
int64_t ldm_debug_read(const LdmHandle* h, const char* name, void* dst_host, int64_t capacity_bytes, int32_t n_layouts);

const char* ldm_last_error(void);
const char* ldm_version(void);

#ifdef __cplusplus
}
#endif
#endif /* LDM_B200_H_ */
