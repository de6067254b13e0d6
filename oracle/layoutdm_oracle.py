"""
CPU ORACLE for the LayoutDM sampling hot path  --  TEST INFRASTRUCTURE, NOT PRODUCT CODE.

This file restates, in plain torch-CPU fp32 (numpy for the integer / RNG parts), the algorithm of the
reference's `LayoutDM.sample()` path.  Only `tests/`, `__graft_entry__.smoke()` and the `cpu_baseline` /
`--impl reference` legs of `bench.py` may import it; the product package `layoutdm_b200` never does, and
fails loudly when its CUDA library is missing.

Parity pin: the reference has NO tests / golden vectors of its own (SURVEY.md §4).  This restatement is
pinned against the *unmodified reference itself*, imported through `oracle/ref_shims` where it is available
(`tests/golden/make_golden.py`, `tests/test_oracle_vs_reference.py`), and against the fixtures that script
commits under `tests/golden/` (the tests compare against those without the reference).

Every function cites the reference file:line it follows.  `T/` = src/trainer/trainer/ of the layout-dm checkout.
Tensor layout here is (B, S, C) ("token-major"); the reference uses (B, C, S).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F

LOG_EPS = math.log(1e-30)  # T/models/categorical_diffusion/util.py:7-8

# --------------------------------------------------------------------------------------------------------------
# vocabulary layout
# --------------------------------------------------------------------------------------------------------------


@dataclass(frozen=True)
class VocabSpec:
    """Vocabulary of LayoutSequenceTokenizer with var_order c-x-y-w-h, shared_bbox_vocab x-y-w-h,
    special tokens (pad, mask).  T/helpers/layout_tokenizer.py:79-82,296-313; Converter :414-468."""

    n_cat: int = 25          # rico25: 25, publaynet: 5
    n_bins: int = 32
    n_elem: int = 25         # max_seq_length
    n_attr: int = 5

    @property
    def C(self) -> int:
        return self.n_cat + 4 * self.n_bins + 2

    @property
    def S(self) -> int:
        return self.n_elem * self.n_attr

    @property
    def pad_id(self) -> int:
        return self.n_cat + 4 * self.n_bins

    @property
    def mask_id(self) -> int:
        return self.pad_id + 1

    def group_start(self, g: int) -> int:
        return 0 if g == 0 else self.n_cat + (g - 1) * self.n_bins

    def group_n(self, g: int) -> int:
        """number of 'normal' classes of attribute group g (without PAD / MASK)"""
        return self.n_cat if g == 0 else self.n_bins

    def group_full_ids(self, g: int) -> List[int]:
        """partial vocab -> full ids, order [normal..., PAD, MASK]  (layout_tokenizer.py:429-467)"""
        st, n = self.group_start(g), self.group_n(g)
        return list(range(st, st + n)) + [self.pad_id, self.mask_id]


RICO25 = VocabSpec(n_cat=25)
PUBLAYNET = VocabSpec(n_cat=5)


@dataclass(frozen=True)
class ModelSpec:
    """Denoiser dimensions: T/config/backbone/medium.yaml:6-12 shrunk by 29/32 (T/models/layoutdm.py:54,
    T/models/common/util.py:36-44)."""

    d: int = 464
    heads: int = 8
    ff: int = 1856
    layers: int = 4
    T: int = 100             # num_timesteps == AdaLN embedding table size (diffusion_step)
    pos_emb: str = "elem_attr"   # or "default" (nn_lib.py:73-88)

    @property
    def dh(self) -> int:
        return self.d // self.heads


PREFIX = "model.module.transformer."

# --------------------------------------------------------------------------------------------------------------
# noise schedule (T/models/categorical_diffusion/util.py:47-70, constrained.py:56-90, vanilla.py:42-72)
# --------------------------------------------------------------------------------------------------------------


def alpha_schedule(T: int, N: int, att_1=0.99999, att_T=0.000009, ctt_1=0.000009, ctt_T=0.99999):
    att = np.arange(0, T) / (T - 1) * (att_T - att_1) + att_1
    att = np.concatenate(([1], att))
    at = att[1:] / att[:-1]
    ctt = np.arange(0, T) / (T - 1) * (ctt_T - ctt_1) + ctt_1
    ctt = np.concatenate(([0], ctt))
    one_minus_ctt = 1 - ctt
    one_minus_ct = one_minus_ctt[1:] / one_minus_ctt[:-1]
    ct = 1 - one_minus_ct
    bt = (1 - at - ct) / N
    att = np.concatenate((att[1:], [1]))
    ctt = np.concatenate((ctt[1:], [0]))
    btt = (1 - att - ctt) / N
    return at, bt, ct, att, btt, ctt


SCHED_NAMES = ("log_at", "log_bt", "log_ct", "log_cumprod_at", "log_cumprod_bt", "log_cumprod_ct",
               "log_1_min_ct", "log_1_min_cumprod_ct")


def schedule_tables(T: int, N: int) -> Dict[str, torch.Tensor]:
    """fp32 tables exactly as registered by the reference (float64 math, then .float()).
    log_at/bt/ct/log_1_min_ct have length T; the cumprod ones T+1 (index T = identity transition)."""
    at, bt, ct, att, btt, ctt = (torch.tensor(x.astype("float64")) for x in alpha_schedule(T, N))
    with np.errstate(divide="ignore"):
        log_at, log_bt, log_ct = torch.log(at), torch.log(bt), torch.log(ct)
        log_cat, log_cbt, log_cct = torch.log(att), torch.log(btt), torch.log(ctt)
    l1m = lambda a: torch.log(1 - a.exp() + 1e-40)  # util.py:15-16
    return {
        "log_at": log_at.float(), "log_bt": log_bt.float(), "log_ct": log_ct.float(),
        "log_cumprod_at": log_cat.float(), "log_cumprod_bt": log_cbt.float(), "log_cumprod_ct": log_cct.float(),
        "log_1_min_ct": l1m(log_ct).float(), "log_1_min_cumprod_ct": l1m(log_cct).float(),
    }


def group_schedules(T: int, vocab: VocabSpec, q_type: str = "constrained") -> List[Dict[str, torch.Tensor]]:
    """constrained: one schedule per attribute group with N = K-1 = n_normal+1 (constrained.py:51-59);
    vanilla: a single schedule with N = C-1 (vanilla.py:42-44)."""
    if q_type == "constrained":
        return [schedule_tables(T, vocab.group_n(g) + 1) for g in range(vocab.n_attr)]
    return [schedule_tables(T, vocab.C - 1)]


# --------------------------------------------------------------------------------------------------------------
# synthetic weights with the reference's state_dict key names (SURVEY.md §8a-a5)
# --------------------------------------------------------------------------------------------------------------


def make_weights(vocab: VocabSpec, spec: ModelSpec, seed: int = 0, scale: float = 1.0) -> Dict[str, torch.Tensor]:
    """Deterministic 'trained-like' weights: N(0, 0.02*scale) matrices (the reference's init std,
    T/models/base_model.py:108-116), small non-zero biases and LN affine params so that every term of the
    forward pass is exercised.  Keys are the reference's `state_dict` names."""
    g = torch.Generator().manual_seed(seed)
    std = 0.02 * scale
    d, ff, C, T = spec.d, spec.ff, vocab.C, spec.T
    n = lambda *shape, s=std: torch.randn(*shape, generator=g) * s
    sd: Dict[str, torch.Tensor] = {}
    sd[PREFIX + "cat_emb.weight"] = n(C, d)
    if spec.pos_emb == "elem_attr":
        sd[PREFIX + "pos_emb.elem_emb"] = torch.rand(vocab.n_elem, d, generator=g)
        sd[PREFIX + "pos_emb.attr_emb"] = torch.rand(vocab.n_attr, d, generator=g)
    else:
        sd[PREFIX + "pos_emb.pos_emb"] = torch.rand(vocab.S, d, generator=g)
    for l in range(spec.layers):
        p = f"{PREFIX}backbone.layers.{l}."
        sd[p + "self_attn.in_proj_weight"] = n(3 * d, d)
        sd[p + "self_attn.in_proj_bias"] = n(3 * d)
        sd[p + "self_attn.out_proj.weight"] = n(d, d)
        sd[p + "self_attn.out_proj.bias"] = n(d)
        sd[p + "linear1.weight"] = n(ff, d)
        sd[p + "linear1.bias"] = n(ff)
        sd[p + "linear2.weight"] = n(d, ff)
        sd[p + "linear2.bias"] = n(d)
        sd[p + "norm1.emb.weight"] = n(T, d, s=1.0)
        sd[p + "norm1.linear.weight"] = n(2 * d, d)
        sd[p + "norm1.linear.bias"] = n(2 * d)
        sd[p + "norm2.weight"] = 1.0 + n(d, s=0.1)
        sd[p + "norm2.bias"] = n(d, s=0.1)
    sd[PREFIX + "head.0.weight"] = 1.0 + n(d, s=0.1)
    sd[PREFIX + "head.0.bias"] = n(d, s=0.1)
    sd[PREFIX + "head.1.weight"] = n(C, d)
    return sd


def weights_checksum(sd: Dict[str, torch.Tensor]) -> float:
    return float(sum(v.double().abs().sum() for k, v in sorted(sd.items())))


# --------------------------------------------------------------------------------------------------------------
# denoiser forward  (T/models/common/nn_lib.py:191-237, T/models/transformer_utils.py:79-83,165-210)
# --------------------------------------------------------------------------------------------------------------


def _rnd(x: torch.Tensor, dt: Optional[torch.dtype]) -> torch.Tensor:
    """round-trip through the tensor-core operand dtype (same-rounding oracle, SURVEY.md §7.2-2)"""
    return x if dt is None else x.to(dt).float()


def positional_table(sd, vocab: VocabSpec, spec: ModelSpec) -> torch.Tensor:
    """(S, d) positional embedding: elem_emb[s // 5] + attr_emb[s % 5]  (nn_lib.py:112-127)"""
    if spec.pos_emb == "elem_attr":
        e = sd[PREFIX + "pos_emb.elem_emb"].repeat_interleave(vocab.n_attr, dim=0)
        a = sd[PREFIX + "pos_emb.attr_emb"].repeat(vocab.n_elem, 1)
        return (e + a)[: vocab.S]
    return sd[PREFIX + "pos_emb.pos_emb"][: vocab.S]


def adaln_table(sd, spec: ModelSpec, layer: int) -> torch.Tensor:
    """(T, 2d) = Linear(SiLU(Embedding[t])) for every t  (transformer_utils.py:66-69,80-81)"""
    p = f"{PREFIX}backbone.layers.{layer}."
    return F.linear(F.silu(sd[p + "norm1.emb.weight"]), sd[p + "norm1.linear.weight"], sd[p + "norm1.linear.bias"])


def denoiser_forward(sd, ids: torch.Tensor, t: int, vocab: VocabSpec, spec: ModelSpec,
                     operand_dtype: Optional[torch.dtype] = None,
                     taps: Optional[dict] = None) -> torch.Tensor:
    """ids (B,S) int64, scalar timestep t -> logits (B,S,C) fp32.

    With operand_dtype = torch.float16 / bfloat16 every GEMM operand (activations AND weights, and the
    attention probabilities) is rounded to that dtype first while accumulation stays fp32: this is the
    'same-rounding' oracle for the tensor-core path.  operand_dtype=None is the exact fp32 restatement.
    taps: optional dict that receives the intermediate tensors of every layer (for kernel-by-kernel tests)."""
    d, H, dh = spec.d, spec.heads, spec.dh
    B, S = ids.shape
    r = lambda x: _rnd(x, operand_dtype)
    tap = (lambda k, v: taps.__setitem__(k, v)) if taps is not None else (lambda k, v: None)
    h = sd[PREFIX + "cat_emb.weight"][ids] + positional_table(sd, vocab, spec)[None]   # nn_lib.py:204,220 (dropout = id in eval)
    for l in range(spec.layers):
        p = f"{PREFIX}backbone.layers.{l}."
        emb = adaln_table(sd, spec, l)[t]                       # (2d,); t may also be a (B,) tensor of per-layout timesteps (training)
        if emb.dim() == 2:
            emb = emb[:, None]                                  # .unsqueeze(1), transformer_utils.py:80
        scale, shift = emb[..., :d], emb[..., d:]               # torch.chunk(emb, 2)  transformer_utils.py:81
        x = F.layer_norm(h, (d,), eps=1e-5) * (1 + scale) + shift   # :82
        tap(f"x{l}", x)
        # MHA(x,x,x): torch.nn.MultiheadAttention, batch_first, no masks (transformer_utils.py:140-142,197-204)
        qkv = F.linear(r(x), r(sd[p + "self_attn.in_proj_weight"]), sd[p + "self_attn.in_proj_bias"])
        q, k, v = qkv.split(d, dim=-1)
        q = q.view(B, S, H, dh).transpose(1, 2) * (1.0 / math.sqrt(dh))
        k = k.view(B, S, H, dh).transpose(1, 2)
        v = v.view(B, S, H, dh).transpose(1, 2)
        tap(f"q{l}", q); tap(f"k{l}", k); tap(f"v{l}", v)       # (B,H,S,dh); q already scaled
        att = torch.softmax(r(q) @ r(k).transpose(-1, -2), dim=-1)
        o = (r(att) @ r(v)).transpose(1, 2).reshape(B, S, d)
        tap(f"att{l}", o)
        x = x + F.linear(r(o), r(sd[p + "self_attn.out_proj.weight"]), sd[p + "self_attn.out_proj.bias"])  # residual from the NORMALISED x (:175-178)
        tap(f"y{l}", x)
        z = F.layer_norm(x, (d,), sd[p + "norm2.weight"], sd[p + "norm2.bias"], eps=1e-5)
        tap(f"z{l}", z)
        f = F.relu(F.linear(r(z), r(sd[p + "linear1.weight"]), sd[p + "linear1.bias"]))
        tap(f"hid{l}", f)
        h = x + F.linear(r(f), r(sd[p + "linear2.weight"]), sd[p + "linear2.bias"])                    # :179
        tap(f"h{l}", h)
    hn = F.layer_norm(h, (d,), sd[PREFIX + "head.0.weight"], sd[PREFIX + "head.0.bias"], eps=1e-5)
    tap("hn", hn)
    logits = F.linear(r(hn), r(sd[PREFIX + "head.1.weight"]))                                          # nn_lib.py:187-189,235
    return logits


# --------------------------------------------------------------------------------------------------------------
# predict_start  (T/models/categorical_diffusion/base.py:127-146)
# --------------------------------------------------------------------------------------------------------------


def predict_start(logits: torch.Tensor) -> torch.Tensor:
    """logits (B,S,C) -> log p(x0|xt) (B,S,C): drop the MASK column, float64 log-softmax over C-1 (:137),
    back to fp32, append -70 for MASK, clamp to [-70, 0]."""
    lp = F.log_softmax(logits[..., :-1].double(), dim=-1).float()
    lp = torch.cat([lp, torch.full_like(lp[..., :1], -70.0)], dim=-1)
    return torch.clamp(lp, -70.0, 0.0)


# --------------------------------------------------------------------------------------------------------------
# q_posterior  (constrained.py:92-206, vanilla.py:74-151)
# --------------------------------------------------------------------------------------------------------------


def _log_add_exp(a, b):  # util.py:19-21
    m = torch.max(a, b)
    return m + torch.log(torch.exp(a - m) + torch.exp(b - m))


def _posterior_group(lp0: torch.Tensor, log_xt: torch.Tensor, is_mask: torch.Tensor, t: int, T: int,
                     tab: Dict[str, torch.Tensor]) -> torch.Tensor:
    """One vocabulary group.  lp0, log_xt: (..., K) in the partial vocab [normal..., PAD, MASK];
    is_mask (..., 1) bool: x_t == MASK.  Literal transcription of constrained.py:163-197 with scalar t."""
    tm1 = (t - 1 + (T + 1)) % (T + 1)                           # :114
    f = (lambda name, i: tab[name][i].view(-1, 1, 1)) if torch.is_tensor(t) else (lambda name, i: tab[name][i])   # extract(), util.py:24-27
    # q(xt|x0): q_pred(log_x_t, t)   :112-133, :166-173
    log_qt = _log_add_exp(log_xt[..., :-1] + f("log_cumprod_at", t), f("log_cumprod_bt", t))
    log_qt = torch.where(is_mask, f("log_cumprod_ct", t).expand_as(log_qt), log_qt)
    # q(xt|xt-1): q_pred_one_timestep   :92-110, :175-185
    one = _log_add_exp(log_xt[..., :-1] + f("log_at", t), f("log_bt", t))
    one = torch.cat([one, torch.full_like(one[..., :1], LOG_EPS)], dim=-1)
    ct_vec = torch.cat([f("log_ct", t).expand_as(one[..., :-1]), torch.zeros_like(one[..., :1])], dim=-1)
    one = torch.where(is_mask, ct_vec, one)
    # :188-197
    q = lp0[..., :-1] - log_qt
    q = torch.cat([q, torch.full_like(q[..., :1], LOG_EPS)], dim=-1)
    L = torch.logsumexp(q, dim=-1, keepdim=True)
    q = q - L
    ev = torch.cat([
        _log_add_exp(q[..., :-1] + f("log_cumprod_at", tm1), f("log_cumprod_bt", tm1)),
        _log_add_exp(q[..., -1:] + f("log_1_min_cumprod_ct", tm1), f("log_cumprod_ct", tm1)),
    ], dim=-1) + one + L
    return torch.clamp(ev, -70.0, 0.0)


def index_to_log_onehot(ids: torch.Tensor, C: int) -> torch.Tensor:
    """(B,S) -> (B,S,C) log(clamp(onehot, 1e-30))   util.py:34-40"""
    return torch.log(F.one_hot(ids, C).float().clamp(min=1e-30))


def q_posterior(log_x_recon: torch.Tensor, x_t: torch.Tensor, t: int, T: int, vocab: VocabSpec,
                scheds: List[Dict[str, torch.Tensor]], q_type: str = "constrained") -> torch.Tensor:
    """log_x_recon (B,S,C), x_t ids (B,S), posterior timestep t (scalar, or a (B,) tensor of per-layout timesteps as in training)
    -> log p(x_{t-1}|x_t) (B,S,C).  constrained: per attribute group gather -> maths -> scatter filled with log 1e-30
    (constrained.py:135-206; Converter.f_to_p_log / p_to_f_log, layout_tokenizer.py:540-557)."""
    assert (int(t.min()) >= 0 and int(t.max()) < T) if torch.is_tensor(t) else 0 <= t < T
    B, S, C = log_x_recon.shape
    log_xt = index_to_log_onehot(x_t, C)
    is_mask = (x_t == vocab.mask_id)[..., None]
    if q_type == "vanilla":
        return _posterior_group(log_x_recon, log_xt, is_mask, t, T, scheds[0])
    out = torch.full_like(log_x_recon, LOG_EPS)
    for g in range(vocab.n_attr):
        idx = torch.tensor(vocab.group_full_ids(g))
        sl = slice(g, S, vocab.n_attr)
        pg = _posterior_group(log_x_recon[:, sl][..., idx], log_xt[:, sl][..., idx], is_mask[:, sl], t, T, scheds[g])
        tmp = out[:, sl]
        tmp[..., idx] = pg
        out[:, sl] = tmp
    return out


def q_pred_full(log_x_start: torch.Tensor, t: torch.Tensor, T: int, vocab: VocabSpec, scheds: List[Dict[str, torch.Tensor]],
                q_type: str = "constrained") -> torch.Tensor:
    """q_pred (constrained.py:112-133 per attribute on its partial vocabulary; vanilla.py:90-110) on full-vocabulary (B,S,C) log
    tensors with per-layout timesteps t (B,) in [-1, T): classes outside a token's group stay log(1e-30) (p_to_f_log)."""
    t = (t + (T + 1)) % (T + 1)
    f = lambda tab, name: tab[name][t].view(-1, 1, 1)

    def group(lx, tab):                                                 # lx (..., K) partial vocab [normal..., PAD, MASK]
        return torch.cat([_log_add_exp(lx[..., :-1] + f(tab, "log_cumprod_at"), f(tab, "log_cumprod_bt")),
                          _log_add_exp(lx[..., -1:] + f(tab, "log_1_min_cumprod_ct"), f(tab, "log_cumprod_ct"))], dim=-1)
    if q_type == "vanilla":
        return group(log_x_start, scheds[0])
    out = torch.full_like(log_x_start, LOG_EPS)
    S = log_x_start.shape[1]
    for g in range(vocab.n_attr):
        idx = torch.tensor(vocab.group_full_ids(g))
        sl = slice(g, S, vocab.n_attr)
        tmp = out[:, sl]
        tmp[..., idx] = group(log_x_start[:, sl][..., idx], scheds[g])
        out[:, sl] = tmp
    return out


def q_pred_one_timestep_full(log_x_t: torch.Tensor, t: torch.Tensor, T: int, vocab: VocabSpec, scheds: List[Dict[str, torch.Tensor]],
                             q_type: str = "constrained") -> torch.Tensor:
    """q_pred_one_timestep (constrained.py:92-110, vanilla.py:74-88) on full-vocabulary (B,S,C) log tensors, t (B,) in [0, T)"""
    f = lambda tab, name: tab[name][t].view(-1, 1, 1)

    def group(lx, tab):
        return torch.cat([_log_add_exp(lx[..., :-1] + f(tab, "log_at"), f(tab, "log_bt")),
                          _log_add_exp(lx[..., -1:] + f(tab, "log_1_min_ct"), f(tab, "log_ct"))], dim=-1)
    if q_type == "vanilla":
        return group(log_x_t, scheds[0])
    out = torch.full_like(log_x_t, LOG_EPS)
    S = log_x_t.shape[1]
    for g in range(vocab.n_attr):
        idx = torch.tensor(vocab.group_full_ids(g))
        sl = slice(g, S, vocab.n_attr)
        tmp = out[:, sl]
        tmp[..., idx] = group(log_x_t[:, sl][..., idx], scheds[g])
        out[:, sl] = tmp
    return out


def gumbel_argmax(logits: torch.Tensor, u: np.ndarray) -> torch.Tensor:
    """log_sample_categorical, train_sampling "gumbel" (constrained.py:208-215): argmax(logits - log(-log(u + 1e-30) + 1e-30))"""
    g = -torch.log(-torch.log(torch.from_numpy(u) + 1e-30) + 1e-30)
    return (g + logits).argmax(dim=-1)


def vb_terms(logits: torch.Tensor, x0: torch.Tensor, xt: torch.Tensor, t: torch.Tensor, T: int, vocab: VocabSpec,
             scheds: List[Dict[str, torch.Tensor]], q_type: str = "constrained", mask_weight=(1.0, 1.0)) -> Dict[str, torch.Tensor]:
    """The loss terms `forward` derives from the denoiser logits at x_t (constrained.py:262-325, vanilla.py:196-236), per layout:
    kl (:295-302), decoder_nll (:304-305), kl_aux (:321-325), plus log_model_prob / log_x0_recon (B,S,C)."""
    C = vocab.C
    log_x0_recon = predict_start(logits)                                               # :263
    log_model_prob = q_posterior(log_x0_recon, xt, t, T, vocab, scheds, q_type)        # :264-266
    log_x_start = index_to_log_onehot(x0, C)
    log_true_prob = q_posterior(log_x_start, xt, t, T, vocab, scheds, q_type)          # :295-297
    kl = (log_true_prob.exp() * (log_true_prob - log_model_prob)).sum(-1)              # multinomial_kl, base.py:117-119
    mask_region = (xt == C - 1).float()
    w = mask_region * mask_weight[0] + (1.0 - mask_region) * mask_weight[1]
    nll = -(log_x_start.exp() * log_model_prob).sum(-1)                                # log_categorical, util.py:30-31
    aux = (log_x_start[..., :-1].exp() * (log_x_start[..., :-1] - log_x0_recon[..., :-1])).sum(-1)
    return {"kl": (kl * w).mean(1), "decoder_nll": nll.mean(1), "kl_aux": (aux * w).mean(1),
            "log_model_prob": log_model_prob, "log_x0_recon": log_x0_recon}


# --------------------------------------------------------------------------------------------------------------
# conditioning adjustments  (base.py:243-284, T/helpers/task.py:154-224)
# --------------------------------------------------------------------------------------------------------------


def refinement_table(vocab: VocabSpec, centers: List[np.ndarray], mode: str = "uniform",
                     offset_ratio: float = 0.1, weight: float = 3.0) -> torch.Tensor:
    """(C, C) table Tbl[orig_id, c]; weak_logits[b,s,c] = Tbl[seq_orig[b,s], c]  (task.py:154-224).
    centers: 4 arrays (n_bins,) of bbox cluster centres for x,y,w,h (float64, as the reference's
    `cluster_centers_`, bbox_tokenizer.py:72-82)."""
    w = -weight if mode == "negative" else weight          # task.py:212-214
    tbl = torch.zeros(vocab.C, vocab.C)
    tbl.fill_diagonal_(1.0)
    for i in range(4):
        cc = torch.from_numpy(np.asarray(centers[i])).view(-1)
        ii, jj = torch.meshgrid(cc, cc, indexing="ij")
        sl = slice(vocab.n_cat + i * vocab.n_bins, vocab.n_cat + (i + 1) * vocab.n_bins)
        if mode == "uniform":
            tbl[sl, sl] = (torch.abs(ii - jj) < offset_ratio).float()
        elif mode == "negative":
            tbl[sl, sl] = (torch.abs(ii - jj) >= offset_ratio).float()
        elif mode == "gaussian":
            tbl[sl, sl] = (-1.0 * (ii - jj) ** 2).float()
        else:
            raise NotImplementedError
    return tbl * w


def linear_centers(n_bins: int = 32) -> List[np.ndarray]:
    """bbox_quantization='linear' cluster centres  (bbox_tokenizer.py:72-82)"""
    d = 1 / n_bins
    xy = np.linspace(start=0.0, stop=1.0 - d, num=n_bins)
    wh = np.linspace(start=d, stop=1.0, num=n_bins)
    return [xy, xy, wh, wh]


def cond_adjust(logp: torch.Tensor, vocab: VocabSpec, cond: Optional[dict], t_model: Optional[int] = None) -> torch.Tensor:
    """base.py:243-284.  cond: seq (B,S), mask (B,S) bool, type, optional seq_orig + refine_table (C,C) already multiplied by
    refine_lambda; for type "relation" (:261-269) optional rel_adj (B,1+E,1+E) int edge table, rel_lambda, rel_num_update,
    rel_centers (4, n_bins) [default linear], rel_batch_total -- applied with relation_update when t_model is given."""
    if not cond:
        return logp
    logp = logp.clone()
    C = vocab.C
    if "mask" in cond:                                                    # :245-251
        strong = index_to_log_onehot(cond["seq"], C)
        logp = torch.where(cond["mask"][..., None], strong, logp)
    if cond.get("type") == "refinement":                                  # :254-258
        weak = cond["refine_table"][cond["seq_orig"]]                     # (B,S,C)  F.embedding, task.py:200
        logp = torch.where(cond["mask"][..., None], logp, logp + weak)
    if cond.get("type") == "relation" and cond.get("rel_adj") is not None and t_model is not None:   # :261-269
        cen = cond.get("rel_centers")
        if cen is None:
            cen = torch.stack([torch.as_tensor(c, dtype=torch.float32) for c in linear_centers(vocab.n_bins)])
        logp = relation_update(logp, cond["seq"], cond["rel_adj"], cen, vocab, t_model, cond["rel_lambda"], cond["rel_num_update"],
                               batch_total=cond.get("rel_batch_total"))
    if cond["type"] in ("c", "cwh", "refinement", "relation"):            # :272-284
        S = cond["seq"].shape[1]
        pad_mask = (torch.arange(S)[None] % vocab.n_attr != 0) & (cond["seq"] != vocab.pad_id)
        logp[..., vocab.pad_id] = torch.where(pad_mask, torch.full_like(logp[..., 0], LOG_EPS), logp[..., vocab.pad_id])
    return logp


# --------------------------------------------------------------------------------------------------------------
# noise contract (Philox4x32-10) shared with the CUDA kernels
# --------------------------------------------------------------------------------------------------------------

_PH_M0, _PH_M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_PH_W0, _PH_W1 = np.uint32(0x9E3779B9), np.uint32(0xBB67AE85)


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Vectorised Philox4x32-10 (Salmon et al. 2011). All inputs uint32 arrays (broadcastable)."""
    c0, c1, c2, c3 = (np.asarray(x, dtype=np.uint32) for x in (c0, c1, c2, c3))
    c0, c1, c2, c3 = np.broadcast_arrays(c0, c1, c2, c3)
    k0 = np.uint32(k0)
    k1 = np.uint32(k1)
    with np.errstate(over="ignore"):
        for _ in range(10):
            p0 = c0.astype(np.uint64) * _PH_M0
            p1 = c2.astype(np.uint64) * _PH_M1
            hi0, lo0 = (p0 >> np.uint64(32)).astype(np.uint32), p0.astype(np.uint32)
            hi1, lo1 = (p1 >> np.uint64(32)).astype(np.uint32), p1.astype(np.uint32)
            c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
            k0 = np.uint32((int(k0) + int(_PH_W0)) & 0xFFFFFFFF)
            k1 = np.uint32((int(k1) + int(_PH_W1)) & 0xFFFFFFFF)
    return c0, c1, c2, c3


def uniforms(seed: int, step_ctr: int, stream: int, b_global0: int, B: int, S: int, C: int) -> np.ndarray:
    """u[b,s,c] in (0,1), float32, the contract implemented by csrc (see DESIGN.md §RNG):
       counter = (c // 4, step_ctr | stream << 24, tok_lo, tok_hi), tok = (b_global0 + b) * S + s,
       key = (seed_lo, seed_hi); word = c % 4;  u = ((word >> 9) + 0.5) * 2^-23."""
    tok = (np.arange(B, dtype=np.uint64)[:, None] + np.uint64(b_global0)) * np.uint64(S) + np.arange(S, dtype=np.uint64)[None]
    tok_lo = (tok & np.uint64(0xFFFFFFFF)).astype(np.uint32)[..., None]
    tok_hi = (tok >> np.uint64(32)).astype(np.uint32)[..., None]
    n4 = (C + 3) // 4
    c4 = np.arange(n4, dtype=np.uint32)[None, None, :]
    w1 = np.uint32((step_ctr & 0xFFFFFF) | (stream << 24))
    r = philox4x32_10(c4, w1, tok_lo, tok_hi, seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    words = np.stack(r, axis=-1).reshape(B, S, n4 * 4)[..., :C]
    return (((words >> np.uint32(9)).astype(np.float32) + np.float32(0.5)) * np.float32(2.0 ** -23)).astype(np.float32)


# --------------------------------------------------------------------------------------------------------------
# categorical draw  (T/helpers/sampling.py:73-130)
# --------------------------------------------------------------------------------------------------------------


@dataclass
class SamplingCfg:
    name: str = "random"           # deterministic | random | top_k | top_p | gumbel
    temperature: float = 1.0
    top_p: float = 0.9
    top_k: int = 5
    num_timesteps: Optional[int] = None
    time_difference: float = 0.0


def draw(logp: torch.Tensor, cfg: SamplingCfg, u: Optional[np.ndarray] = None,
         u_gumbel: Optional[np.ndarray] = None) -> torch.Tensor:
    """logp (B,S,C) -> ids (B,S).  `torch.multinomial(probs, 1)` is argmax(probs / Exp(1)) (ATen multinomial
    fast path for a single sample); the Exp(1) variates are -log(u) with the injected uniforms."""
    if cfg.name == "deterministic":
        return torch.argmax(logp, dim=-1)                                   # sampling.py:87-88
    lg = logp / cfg.temperature                                             # :90
    if cfg.name == "top_k":                                                 # :73-78, :92-93
        v, _ = torch.topk(lg, cfg.top_k, dim=-1)
        lg = lg.clone()
        lg[lg < v[..., -1:]] = -float("inf")
    elif cfg.name == "top_p":                                               # :94-109
        assert 0.0 < cfg.top_p <= 1.0
        sl, si = torch.sort(lg, descending=True, dim=-1)
        cum = torch.cumsum(F.softmax(sl, dim=-1), dim=-1)
        rank = torch.arange(lg.shape[-1]).expand_as(sl)
        sl = sl.masked_fill((cum > cfg.top_p) & (rank > 0), -float("inf"))
        lg = sl.gather(-1, si.argsort(dim=-1))
    elif cfg.name == "random":
        pass
    elif cfg.name == "gumbel":                                              # :112-116
        ug = torch.from_numpy(u_gumbel)
        lg = lg + (-torch.log(-torch.log(ug + 1e-30) + 1e-30))
    else:
        raise NotImplementedError
    probs = F.softmax(lg, dim=-1)                                           # :120
    e = -torch.log(torch.from_numpy(u))
    return torch.argmax(probs / e, dim=-1)


# --------------------------------------------------------------------------------------------------------------
# the loop  (base.py:205-371)
# --------------------------------------------------------------------------------------------------------------


def timestep_plan(T: int, T_eval: int, time_difference: float = 0.0) -> List[Tuple[int, int]]:
    """[(t_model, t_posterior)] for every loop iteration  (base.py:310-315,348-358 and :218-240)."""
    assert T_eval <= T
    plan, prev = [], T
    for i in range(T_eval - 1, -1, -1):
        t = int(i * T / T_eval)
        delta = prev - t
        if delta <= 0:
            raise NotImplementedError
        skip = delta - 1
        noise_t = min(max(t - int(T * time_difference), 0), T - 1) if time_difference > 0.0 else t
        t_post = noise_t - skip if (skip > 0 and noise_t > skip) else noise_t
        plan.append((t, t_post))
        prev = t
    return plan


@dataclass
class Oracle:
    vocab: VocabSpec
    spec: ModelSpec
    sd: Dict[str, torch.Tensor]
    q_type: str = "constrained"
    operand_dtype: Optional[torch.dtype] = None
    scheds: List[Dict[str, torch.Tensor]] = field(default_factory=list)

    def __post_init__(self):
        self.scheds = group_schedules(self.spec.T, self.vocab, self.q_type)

    def step_logprob(self, x_t: torch.Tensor, t_model: int, t_post: int, cond: Optional[dict] = None):
        logits = denoiser_forward(self.sd, x_t, t_model, self.vocab, self.spec, self.operand_dtype)
        return self.logprob_from_logits(logits, x_t, t_post, cond, t_model), logits

    def logprob_from_logits(self, logits, x_t, t_post, cond=None, t_model=None):
        lx0 = predict_start(logits)
        lp = q_posterior(lx0, x_t, t_post, self.spec.T, self.vocab, self.scheds, self.q_type)
        return cond_adjust(lp, self.vocab, cond, t_model)

    def sample(self, B: int, cfg: SamplingCfg, seed: int = 0, cond: Optional[dict] = None,
               b_global0: int = 0, trace: Optional[list] = None) -> torch.Tensor:
        v = self.vocab
        x = cond["seq"].clone() if cond else torch.full((B, v.S), v.mask_id, dtype=torch.long)
        T_eval = cfg.num_timesteps or self.spec.T
        with torch.no_grad():
            for i, (t_model, t_post) in enumerate(timestep_plan(self.spec.T, T_eval, cfg.time_difference)):
                lp, logits = self.step_logprob(x, t_model, t_post, cond)
                u = ug = None
                if cfg.name != "deterministic":
                    u = uniforms(seed, i, 0, b_global0, B, v.S, v.C)
                if cfg.name == "gumbel":
                    ug = uniforms(seed, i, 1, b_global0, B, v.S, v.C)
                x_new = draw(lp, cfg, u, ug)
                if trace is not None:
                    trace.append({"t_model": t_model, "t_post": t_post, "x_in": x, "logits": logits, "logp": lp, "x_out": x_new})
                x = x_new
        return x


# --------------------------------------------------------------------------------------------------------------
# tokenizer decode / synthetic conditions (host-side neighbours of the path; used to build test inputs)
# --------------------------------------------------------------------------------------------------------------


def decode_ids(ids: torch.Tensor, vocab: VocabSpec) -> Dict[str, torch.Tensor]:
    """LayoutSequenceTokenizer.decode with linear bbox quantisation
    (layout_tokenizer.py:255-266, :106-114; bbox_tokenizer.py:117-146)."""
    x = ids.view(ids.shape[0], vocab.n_elem, vocab.n_attr)
    label, bbox = x[..., 0].clone(), x[..., 1:].clone() - vocab.n_cat
    label_valid = (0 <= label) & (label < vocab.n_cat)
    bbox_valid = ((0 <= bbox) & (bbox < 4 * vocab.n_bins)).all(dim=-1)
    invalid = ~(label_valid & bbox_valid)
    arr = bbox - torch.tensor([0, 1, 2, 3]) * vocab.n_bins
    arr = torch.clamp(arr, 0, vocab.n_bins - 1)
    d = 1 / vocab.n_bins
    out = torch.zeros(arr.shape, dtype=torch.float32)
    out[..., :2] = arr[..., :2].float() * d
    out[..., 2:] = (arr[..., 2:] + 1).float() * d
    label[invalid] = 0
    out[invalid] = 0.0
    return {"bbox": out, "label": label, "mask": ~invalid}


# --------------------------------------------------------------------------------------------------------------
# layouts -> ids -> cond  (tokenizer.encode layout_tokenizer.py:208-253 + bbox_tokenizer.py:86-114; get_cond task.py:27-151)
# --------------------------------------------------------------------------------------------------------------


def encode_layouts(label: torch.Tensor, bbox: torch.Tensor, mask: torch.Tensor, vocab: VocabSpec,
                   centers: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """LayoutSequenceTokenizer.encode for var_order c-x-y-w-h, shared_bbox_vocab x-y-w-h, pad_until_max, no BOS/EOS, no sort:
    label (B,E) i64, bbox (B,E,4) f32 xywh, mask (B,E) bool (valid elements form a prefix) -> seq (B,S) i64, mask (B,S) bool.
    Linear quantisation: bbox_tokenizer.py:90-93 (float32 clamp / subtract / multiply, torch.round = half-to-even);
    centers (4, n_bins) f32 = kmeans / percentile cluster centres: nearest centre like KMeans.predict (:95-104)."""
    B, E = label.shape
    nb = vocab.n_bins
    bbox = bbox.float()
    if centers is None:
        d = 1 / nb
        q = torch.zeros_like(bbox)
        q[..., :2] = torch.clamp(bbox[..., :2], 0.0, 1.0 - d)
        q[..., 2:] = torch.clamp(bbox[..., 2:], d, 1.0) - d
        idx = (nb * q).round().long()
    else:
        dist = (bbox[..., None] - centers.float()[None, None]) ** 2          # (B,E,4,nb)
        idx = dist.argmin(dim=-1)
    idx = idx + torch.arange(4) * nb + vocab.n_cat                            # KEY_MULT x-y-w-h offsets (:107-109) + :223
    tok = torch.cat([label[..., None], idx], dim=-1)                          # (B,E,5)
    tok[~mask] = vocab.pad_id                                                 # _fix_padded_sequences :96-104
    return tok.reshape(B, E * vocab.n_attr), mask[..., None].expand(B, E, vocab.n_attr).reshape(B, E * vocab.n_attr)


def make_cond(label: torch.Tensor, bbox: torch.Tensor, mask: torch.Tensor, vocab: VocabSpec, cond_type: str,
              centers: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
    """get_cond (task.py:27-151) for the deterministic conditioning types, model_type="LayoutDM":
    c / cwh (:94-110), gt (:116-117), refinement (:126-140; `bbox` is the already perturbed box, the caller draws the
    N(0, 0.1) noise of :127).  `partial` / `random` draw host random numbers and stay in Python."""
    seq, m = encode_layouts(label, bbox, mask, vocab, centers)
    attr = torch.arange(vocab.S)[None] % vocab.n_attr
    out: Dict[str, torch.Tensor] = {}
    if cond_type in ("c", "cwh"):
        keep = attr == 0 if cond_type == "c" else ((attr == 0) | (attr == 3) | (attr == 4))
        s2 = torch.where(keep, seq, torch.full_like(seq, vocab.mask_id))
        s2 = torch.where(m, s2, torch.full_like(seq, vocab.pad_id))
        out = {"seq": s2, "mask": (m & keep) | ~m}
    elif cond_type == "gt":
        out = {"seq": seq, "mask": m}
    elif cond_type == "refinement":
        cm = (m & (attr == 0)) | ~m
        s2 = torch.where(cm, seq, torch.full_like(seq, vocab.mask_id))
        s2 = torch.where(m, s2, torch.full_like(seq, vocab.pad_id))
        out = {"seq": s2, "mask": cm, "seq_orig": seq}
    else:
        raise NotImplementedError(cond_type)
    out["type"] = cond_type
    if cond_type in ("c", "cwh", "refinement"):
        out["num_element"] = mask.sum(dim=1)
    return out


# --------------------------------------------------------------------------------------------------------------
# forward (corruption) process on ids  (constrained.py:208-230, vanilla.py:153-158; used by training forward :232-260)
# --------------------------------------------------------------------------------------------------------------


def q_sample_ids(x0: torch.Tensor, t: torch.Tensor, T: int, vocab: VocabSpec, scheds: List[Dict[str, torch.Tensor]],
                 u: np.ndarray, q_type: str = "constrained") -> torch.Tensor:
    """x0 (B,S) ids, t (B,) per-layout timestep, u (B,S,C) uniforms of the noise contract (stream 2) -> x_t (B,S) ids.
    Per token: log q(x_t = k | x_0) = q_pred(log_onehot(x_0), t) over the token's vocabulary group, then the reference's
    Gumbel-argmax draw  argmax_k(logits_k - log(-log(u_k + 1e-30) + 1e-30))  (train_sampling="gumbel")."""
    B, S = x0.shape
    C = vocab.C
    log_x0 = index_to_log_onehot(x0, C)                                   # (B,S,C)
    ug = torch.from_numpy(u)
    gumbel = -torch.log(-torch.log(ug + 1e-30) + 1e-30)
    out = torch.empty_like(x0)
    groups = range(vocab.n_attr) if q_type == "constrained" else [0]
    for g in groups:
        idx = torch.tensor(vocab.group_full_ids(g)) if q_type == "constrained" else torch.arange(C)
        sl = slice(g, S, vocab.n_attr) if q_type == "constrained" else slice(0, S)
        lx = log_x0[:, sl][..., idx]                                       # (B,S',K)
        tab = scheds[g]
        tt = t.view(B, 1, 1)
        lcat, lcbt = tab["log_cumprod_at"][tt], tab["log_cumprod_bt"][tt]
        lcct, l1m = tab["log_cumprod_ct"][tt], tab["log_1_min_cumprod_ct"][tt]
        logits = torch.cat([_log_add_exp(lx[..., :-1] + lcat, lcbt), _log_add_exp(lx[..., -1:] + l1m, lcct)], dim=-1)
        k = (gumbel[:, sl][..., idx] + logits).argmax(dim=-1)
        out[:, sl] = idx[k]
    return out


# --------------------------------------------------------------------------------------------------------------
# cond=relation: gradient-based logit adjustment  (T/models/categorical_diffusion/logit_adjustment.py:16-126,
# losses T/models/clg/const.py:53-243, relation codes T/data/util.py:14-30)
# --------------------------------------------------------------------------------------------------------------
REL_SIZE_SM, REL_SIZE_EQ, REL_SIZE_LG = 1, 2, 3                     # RelSize  (data/util.py:14-18)
REL_LOC_L, REL_LOC_T, REL_LOC_R, REL_LOC_B, REL_LOC_C = 5, 6, 7, 8, 9   # RelLoc   (data/util.py:21-27)
REL_SIZE_ALPHA = 0.1                                                # data/util.py:30
N_REL_FUNCS = 14                                                    # len(const.relation), const.py:226-241


def relation_adjacency(edge_index: torch.Tensor, edge_attr: torch.Tensor, batch: torch.Tensor, B: int, n_slots: int) -> torch.Tensor:
    """PyG-style edges of a batch WITH canvas nodes (AddCanvasElement, data/util.py:106-120: node 0 of every layout is the
    canvas) -> dense (B, n_slots, n_slots) int32 bit masks: adj[b, i, j] = edge_attr of the edge i -> j (slot 0 = canvas)."""
    adj = torch.zeros(B, n_slots, n_slots, dtype=torch.int32)
    if edge_index.numel() == 0:
        return adj
    num = torch.zeros(B, dtype=torch.long).scatter_add_(0, batch, torch.ones_like(batch))
    cum = torch.cat([num.new_zeros(1), num.cumsum(0)])
    b = batch[edge_index[0]]
    adj[b, edge_index[0] - cum[b], edge_index[1] - cum[b]] = edge_attr.to(torch.int32)
    return adj


def relation_bbox(lp: torch.Tensor, cond_seq: torch.Tensor, centers: torch.Tensor, vocab: VocabSpec):
    """_stochastic_convert, mode='average' (logit_adjustment.py:16-85): expected box of every node.
    lp (B,S,C) log-probs, centers (4, n_bins) -> p (B, 1+E, 4, n_bins), bbox (B, 1+E, 4) xywh, valid (B, 1+E); node 0 = canvas,
    whose logits are the log one-hot of encode([0.5, 0.5, 1, 1]) (:36-41)."""
    B = lp.shape[0]
    E, A, nb, nc = vocab.n_elem, vocab.n_attr, vocab.n_bins, vocab.n_cat
    logits = torch.empty(B, 1 + E, 4, nb, dtype=lp.dtype)
    d = 1.0 / nb
    canvas = torch.tensor([0.5, 0.5, 1.0, 1.0])
    q = torch.cat([canvas[:2].clamp(0.0, 1.0 - d), canvas[2:].clamp(d, 1.0) - d])          # bbox_tokenizer.py:88-93 (linear)
    cb = (nb * q).round().long()
    if centers is not None and not torch.allclose(centers, torch.stack([torch.as_tensor(c, dtype=torch.float32) for c in linear_centers(nb)])):
        cb = (canvas[:, None] - centers).pow(2).argmin(dim=1)                               # KMeans.predict (:95-104)
    for a in range(4):
        lo = nc + a * nb
        logits[:, 1:, a] = lp[:, (a + 1)::A, lo:lo + nb]
        logits[:, 0, a] = torch.log(F.one_hot(cb[a], nb).float().clamp(min=1e-30))
    valid = torch.cat([torch.ones(B, 1, dtype=torch.bool), cond_seq[:, ::A] != vocab.pad_id], dim=1)
    p = torch.softmax(logits, dim=-1)
    bbox = (p * centers[None, None]).sum(-1)
    return p, bbox, valid


def relation_cost_and_grad(bbox: torch.Tensor, valid: torch.Tensor, adj: torch.Tensor):
    """The 14 relation costs of const.py:226-241 summed per layout, and d(sum)/d(bbox) by hand (ReLU subgradient 0 at 0, as
    autograd's).  bbox (B,N,4) xywh, adj (B,N,N) edge bit masks -> cost (B,), grad (B,N,4).  Plain loops: test sizes only."""
    B, N, _ = bbox.shape
    cost = torch.zeros(B, dtype=torch.float32)
    grad = torch.zeros_like(bbox)
    eps = torch.tensor(1e-8, dtype=torch.float32)
    al, ah = torch.tensor(1 - REL_SIZE_ALPHA, dtype=torch.float32), torch.tensor(1 + REL_SIZE_ALPHA, dtype=torch.float32)
    third, two3 = torch.tensor(1.0 / 3, dtype=torch.float32), torch.tensor(2.0 / 3, dtype=torch.float32)
    for b in range(B):
        x, y, w, h = bbox[b].unbind(-1)
        area = w * h
        l, t, r, bt = x - w / 2, y - h / 2, x + w / 2, y + h / 2
        g_area = torch.zeros(N); g_l = torch.zeros(N); g_t = torch.zeros(N); g_r = torch.zeros(N); g_b = torch.zeros(N); g_y = torch.zeros(N)

        def relu_term(v, pos, neg):
            """cost += relu(v); where v > 0 the listed (tensor, index, coefficient) gradient entries are applied"""
            nonlocal cost
            if v > 0:
                cost[b] += v
                for arr, idx, coef in pos + neg:
                    arr[idx] += coef
        for i in range(N):
            for j in range(N):
                m = int(adj[b, i, j])
                if m == 0 or not (valid[b, i] and valid[b, j]):
                    continue
                ai, aj = area[i], area[j]
                if m & (1 << REL_SIZE_SM):                                   # const.py:73-79: a_j <= (1 - alpha) a_i
                    relu_term(aj - al * ai, [(g_area, j, 1.0)], [(g_area, i, -float(al))])
                if m & (1 << REL_SIZE_EQ):                                   # :82-89
                    relu_term(al * ai - aj + eps, [(g_area, i, float(al))], [(g_area, j, -1.0)])
                    relu_term(aj - ah * ai + eps, [(g_area, j, 1.0)], [(g_area, i, -float(ah))])
                if m & (1 << REL_SIZE_LG):                                   # :92-98
                    relu_term(ah * ai - aj, [(g_area, i, float(ah))], [(g_area, j, -1.0)])
                if i == 0:                                                   # source is the canvas (y == 0): :101-148
                    yc = y[j]
                    if m & (1 << REL_LOC_T):
                        relu_term(yc - third, [(g_y, j, 1.0)], [])
                    if m & (1 << REL_LOC_C):
                        relu_term(third - yc + eps, [], [(g_y, j, -1.0)])
                        relu_term(yc - two3 + eps, [(g_y, j, 1.0)], [])
                    if m & (1 << REL_LOC_B):
                        relu_term(two3 - yc, [], [(g_y, j, -1.0)])
                else:                                                        # :150-223
                    if m & (1 << REL_LOC_T):
                        relu_term(bt[j] - t[i], [(g_b, j, 1.0)], [(g_t, i, -1.0)])
                    if m & (1 << REL_LOC_B):
                        relu_term(bt[i] - t[j], [(g_b, i, 1.0)], [(g_t, j, -1.0)])
                    for code in (REL_LOC_L, REL_LOC_R, REL_LOC_C):
                        if not m & (1 << code):
                            continue
                        if code == REL_LOC_L:
                            relu_term(r[j] - l[i], [(g_r, j, 1.0)], [(g_l, i, -1.0)])
                        elif code == REL_LOC_R:
                            relu_term(r[i] - l[j], [(g_r, i, 1.0)], [(g_l, j, -1.0)])
                        else:
                            relu_term(l[i] - r[j] + eps, [(g_l, i, 1.0)], [(g_r, j, -1.0)])
                            relu_term(l[j] - r[i] + eps, [(g_l, j, 1.0)], [(g_r, i, -1.0)])
                        relu_term(t[i] - bt[j] + eps, [(g_t, i, 1.0)], [(g_b, j, -1.0)])     # :168-170: t1 < b2 and t2 < b1
                        relu_term(t[j] - bt[i] + eps, [(g_t, j, 1.0)], [(g_b, i, -1.0)])
        grad[b, :, 0] = g_l + g_r
        grad[b, :, 1] = g_t + g_b + g_y
        grad[b, :, 2] = g_area * h + (g_r - g_l) / 2
        grad[b, :, 3] = g_area * w + (g_b - g_t) / 2
    return cost, grad


def relation_update(lp: torch.Tensor, cond_seq: torch.Tensor, adj: torch.Tensor, centers: torch.Tensor, vocab: VocabSpec, t: int,
                    relation_lambda: float, relation_num_update: int, mode: str = "average", batch_total: Optional[int] = None) -> torch.Tensor:
    """`update` (logit_adjustment.py:88-126) without autograd: `relation_num_update` SGD steps (lr = relation_lambda, :101-103) on
    the (B,S,C) log-probs for the loss mean_{b, f}(cost_f,b) (:117-120); no update for t < 10 (:105).  Returns the new log-probs."""
    if mode != "average":
        raise NotImplementedError("relation_mode 'gumbel' draws torch noise inside the update (logit_adjustment.py:76-77)")
    lp = lp.clone()
    n_up = 0 if t < 10 else relation_num_update
    B = lp.shape[0]
    A, nb, nc = vocab.n_attr, vocab.n_bins, vocab.n_cat
    has_edges = bool((adj != 0).any())
    for _ in range(n_up):
        if not has_edges:                                                    # :113-115
            continue
        p, bbox, valid = relation_bbox(lp, cond_seq, centers, vocab)
        _, g = relation_cost_and_grad(bbox, valid, adj)
        g = g / float((batch_total or B) * N_REL_FUNCS)                      # torch.stack(loss, -1).mean() over (layouts, costs)
        # d bbox_a / d logit_c = p_c (center_c - bbox_a)   (softmax over the attribute's bins, :74-85)
        dlog = g[..., None] * p * (centers[None, None] - bbox[..., None])    # (B, 1+E, 4, nb)
        dlog = dlog * valid[..., None, None]
        for a in range(4):
            lo = nc + a * nb
            lp[:, (a + 1)::A, lo:lo + nb] -= relation_lambda * dlog[:, 1:, a]
    return lp
