"""Per-kernel references of the denoiser's launch sequence (test scaffolding, imported by tests only).

Each function recomputes ONE kernel of layoutdm_b200/csrc from that kernel's own inputs, on the buffer layouts the kernels
use: Q / K / V heads padded 58 -> 64 columns (zeros, plus a ones column at 58 of every V head), the attention output padded
the same way, the out-projection weight with zero columns at the padding, logits rows padded to 160.  The precision is the
caller's: float64 for the GPU kernel tests (test_gpu_kernels_fp64.py), float32 without operand rounding for the check that
the chain of these references reproduces the oracle (test_kernel_refs.py), which pins the padding maps, the q-scale and the
residual wiring to the oracle.  Weights are rounded to the operand dtype the way the packing kernel rounds them (round to
nearest even), then widened."""
from __future__ import annotations

import math
from typing import Optional

import torch

from oracle import layoutdm_oracle as O

HP = 64           # per-head width after padding (kHeadPad in ldm_b200.cu)
LOGIT_LD = 160    # padded logits row (kLogitLd)
LN_EPS = 1e-5


def qkv_row_map(d: int, heads: int) -> torch.Tensor:
    """padded QKV row r = which * heads * 64 + head * 64 + j  <-  in_proj row which * d + head * dh + j (j < dh), else -1"""
    dh = d // heads
    m = []
    for r in range(3 * heads * HP):
        which, hh, j = r // (heads * HP), (r % (heads * HP)) // HP, r % HP
        m.append(which * d + hh * dh + j if j < dh else -1)
    return torch.tensor(m)


def att_col_map(d: int, heads: int) -> torch.Tensor:
    """padded attention column c = head * 64 + j  <-  out_proj input column head * dh + j (j < dh), else -1"""
    dh = d // heads
    return torch.tensor([(c // HP) * dh + c % HP if c % HP < dh else -1 for c in range(heads * HP)])


def gather_rows(w: torch.Tensor, m: torch.Tensor) -> torch.Tensor:
    """dst[r] = w[m[r]], zero where m[r] < 0"""
    out = torch.zeros((len(m),) + tuple(w.shape[1:]), dtype=w.dtype)
    ok = m >= 0
    out[ok] = w[m[ok]]
    return out


def unpad_heads(x: torch.Tensor, heads: int, dh: int) -> torch.Tensor:
    """(..., heads * 64) padded head blocks -> (..., heads * dh)"""
    return x.reshape(*x.shape[:-1], heads, HP)[..., :dh].reshape(*x.shape[:-1], heads * dh)


def weight_set(kind: str, vocab: O.VocabSpec, spec: O.ModelSpec, seed: int = 0):
    """synthetic weights of the kernel tests:
      ref    -- O.make_weights at the reference's init scale
      offset -- + 256 on every out_proj.bias, linear2.bias and on cat_emb: rows whose mean is ~256 standard deviations away
                from zero enter every LayerNorm (embedding, LN2, the AdaLN of FF2, the head LN)
      peaked -- the Q block of every in_proj_weight x 100: score spreads of tens, rows close to one-hot"""
    sd = O.make_weights(vocab, spec, seed=seed)
    for l in range(spec.layers):
        p = f"{O.PREFIX}backbone.layers.{l}."
        if kind == "offset":
            sd[p + "self_attn.out_proj.bias"] += 256.0
            sd[p + "linear2.bias"] += 256.0
        elif kind == "peaked":
            sd[p + "self_attn.in_proj_weight"][: spec.d] *= 100.0
        else:
            assert kind == "ref", kind
    if kind == "offset":
        sd[O.PREFIX + "cat_emb.weight"] += 256.0
    return sd


def layer_norm(h: torch.Tensor, scale: torch.Tensor, shift: torch.Tensor) -> torch.Tensor:
    """two-pass LayerNorm over the last dim (eps 1e-5, biased variance) in h's dtype, then * scale + shift"""
    c = h - h.mean(-1, keepdim=True)
    return c / torch.sqrt((c * c).mean(-1, keepdim=True) + LN_EPS) * scale + shift


class Model:
    """the packed weights of one handle, widened to `dtype` after rounding to `operand_dtype` (None: no rounding)"""

    def __init__(self, sd, vocab: O.VocabSpec, spec: O.ModelSpec, operand_dtype: Optional[torch.dtype] = None,
                 dtype: torch.dtype = torch.float64):
        P, d, H = O.PREFIX, spec.d, spec.heads
        self.vocab, self.spec, self.dt, self.dh = vocab, spec, dtype, d // H
        w = lambda t: (t if operand_dtype is None else t.to(operand_dtype)).to(dtype)
        f = lambda t: t.to(dtype)
        self.cat_emb = sd[P + "cat_emb.weight"].float()
        self.pos = O.positional_table(sd, vocab, spec).float()
        self.qscale = 1.0 / math.sqrt(self.dh)
        qm, am = qkv_row_map(d, H), att_col_map(d, H)
        self.layers = []
        for l in range(spec.layers):
            p = f"{P}backbone.layers.{l}."
            bq = gather_rows(sd[p + "self_attn.in_proj_bias"], qm)
            bq[2 * H * HP + torch.arange(H) * HP + self.dh] = 1.0        # V ones column: zero weight row, unit bias
            self.layers.append(dict(
                wqkv=w(gather_rows(sd[p + "self_attn.in_proj_weight"], qm)), bqkv=f(bq),
                wo=w(gather_rows(sd[p + "self_attn.out_proj.weight"].t(), am).t()), bo=f(sd[p + "self_attn.out_proj.bias"]),
                w1=w(sd[p + "linear1.weight"]), b1=f(sd[p + "linear1.bias"]),
                w2=w(sd[p + "linear2.weight"]), b2=f(sd[p + "linear2.bias"]),
                ln2w=f(sd[p + "norm2.weight"]), ln2b=f(sd[p + "norm2.bias"])))
        self.hlnw, self.hlnb = f(sd[P + "head.0.weight"]), f(sd[P + "head.0.bias"])
        hm = torch.tensor([r if r < vocab.C else -1 for r in range(LOGIT_LD)])
        self.whead = w(gather_rows(sd[P + "head.1.weight"], hm))


# ---- one function per kernel; x / z / hid / att / qkv are the kernel's input buffers (..., rows, cols) ----

def embed_input(m: Model, ids: torch.Tensor) -> torch.Tensor:
    """h = cat_emb[id] + pos[s]: the fp32 row the embedding kernel normalises (one fp32 addition, as the kernel does)"""
    return m.cat_emb[ids] + m.pos[: ids.shape[-1]]


def adaln(m: Model, h: torch.Tensor, rows: torch.Tensor) -> torch.Tensor:
    """LN(h) * (1 + scale) + shift; rows (..., 2d) fp32 AdaLN table rows, broadcast over the tokens"""
    d = m.spec.d
    r = rows.to(m.dt)
    return layer_norm(h.to(m.dt), 1 + r[..., :d], r[..., d:])


def qkv(m: Model, l: int, x: torch.Tensor) -> torch.Tensor:
    """QKV GEMM: padded (..., 1536) = x W^T + b, Q columns * 1/sqrt(dh)"""
    L = m.layers[l]
    y = x.to(m.dt) @ L["wqkv"].t() + L["bqkv"]
    y[..., : m.spec.heads * HP] *= m.qscale
    return y


def attention(m: Model, qkv_buf: torch.Tensor, n_valid: int):
    """attention on the padded heads: qkv_buf (B, R, 1536) -> att (B, R, heads * 64), plus the scores s, the probabilities p
    (B, H, R, n_valid) and v (B, H, n_valid, 64).  Q / K padding columns are zero, so the scores are those of the 58-wide heads;
    V's ones column makes att's column 58 the probability sum (1) and its zero columns keep 59..63 at 0."""
    B, R, _ = qkv_buf.shape
    H = m.spec.heads
    x = qkv_buf.to(m.dt).reshape(B, R, 3, H, HP)
    q = x[:, :, 0].transpose(1, 2)
    k = x[:, :n_valid, 1].transpose(1, 2)
    v = x[:, :n_valid, 2].transpose(1, 2)
    s = q @ k.transpose(-1, -2)
    p = torch.softmax(s, dim=-1)
    o = (p @ v).transpose(1, 2).reshape(B, R, H * HP)
    return o, s, p, q, k, v


def outproj(m: Model, l: int, att: torch.Tensor, x32: torch.Tensor) -> torch.Tensor:
    """out-projection + bias + residual (the normalised x of the block's input): y (..., d)"""
    L = m.layers[l]
    return att.to(m.dt) @ L["wo"].t() + L["bo"] + x32.to(m.dt)


def ln2(m: Model, l: int, y: torch.Tensor) -> torch.Tensor:
    L = m.layers[l]
    return layer_norm(y.to(m.dt), L["ln2w"], L["ln2b"])


def ff1(m: Model, l: int, z: torch.Tensor) -> torch.Tensor:
    L = m.layers[l]
    return torch.relu(z.to(m.dt) @ L["w1"].t() + L["b1"])


def ff2_pre(m: Model, l: int, hid: torch.Tensor, y32: torch.Tensor) -> torch.Tensor:
    """FF2 + bias + residual: the pre-norm sum h (..., d) the FF2 epilogue normalises"""
    L = m.layers[l]
    return hid.to(m.dt) @ L["w2"].t() + L["b2"] + y32.to(m.dt)


def ff2_norm(m: Model, l: int, h: torch.Tensor, rows: Optional[torch.Tensor]) -> torch.Tensor:
    """the FF2 epilogue's LayerNorm: the next block's AdaLN with its table rows, or the head LN after the last layer"""
    if l + 1 < m.spec.layers:
        return adaln(m, h, rows)
    return layer_norm(h.to(m.dt), m.hlnw, m.hlnb)


def head(m: Model, z: torch.Tensor) -> torch.Tensor:
    """vocabulary head: padded logits (..., 160), columns >= C on zero weight rows"""
    return z.to(m.dt) @ m.whead.t()
