"""References for the split-bf16 ("bf16x3") operand mode (test scaffolding, imported by tests and tools only).

Every 16-bit operand of the mode is a bf16 pair, hi = bf16(x) and lo = bf16(x - hi), and a product is a_lo b_hi + a_hi b_lo +
a_hi b_hi with fp32 accumulation (a_lo b_lo is dropped).  This module restates that arithmetic next to the oracle's:
  split_bf16 / matmul_bf16x3  -- the pair and the three-product matmul
  denoiser_forward_bf16x3     -- oracle.denoiser_forward with every operand split where the kernels split it
  split_model                 -- a kernel_refs.Model whose packed weights are the pairs the packing kernel writes (hi + lo)"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

import kernel_refs as R
from oracle import layoutdm_oracle as O

GEMM_WEIGHTS = ("self_attn.in_proj_weight", "self_attn.out_proj.weight", "linear1.weight", "linear2.weight")


def split_bf16(x: torch.Tensor):
    """the bf16 pair of an fp32 tensor: hi = bf16(x), lo = bf16(x - hi) (x - hi is exact in fp32); both returned as fp32"""
    x = x.float()
    hi = x.to(torch.bfloat16).float()
    return hi, (x - hi).to(torch.bfloat16).float()


def split_round(t: torch.Tensor) -> torch.Tensor:
    """the value a pair carries, hi + lo, in float64 (exact)"""
    hi, lo = split_bf16(t)
    return hi.double() + lo.double()


def matmul_bf16x3(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """a @ b on split operands: a_lo b_hi + a_hi b_lo + a_hi b_hi in fp32"""
    ah, al = split_bf16(a)
    bh, bl = split_bf16(b)
    return al @ bh + ah @ bl + ah @ bh


def denoiser_forward_bf16x3(sd, ids: torch.Tensor, t, vocab: O.VocabSpec, spec: O.ModelSpec) -> torch.Tensor:
    """O.denoiser_forward with the split operands of the tensor-core path: every GEMM operand and Q / K / V are split into bf16
    pairs at the points the kernels round them, and each product is hi hi + hi lo + lo hi.  Attention splits the un-normalised
    probabilities e = exp(s - max) and divides by the row sum of e_hi + e_lo, as the kernel does."""
    d, H, dh = spec.d, spec.heads, spec.dh
    B, S = ids.shape
    P = O.PREFIX
    lin = lambda x, w, b=None: matmul_bf16x3(x, w.t()) + (0.0 if b is None else b)
    h = sd[P + "cat_emb.weight"][ids] + O.positional_table(sd, vocab, spec)[None]
    for l in range(spec.layers):
        p = f"{P}backbone.layers.{l}."
        emb = O.adaln_table(sd, spec, l)[t]
        if emb.dim() == 2:
            emb = emb[:, None]
        x = F.layer_norm(h, (d,), eps=1e-5) * (1 + emb[..., :d]) + emb[..., d:]
        qkv = lin(x, sd[p + "self_attn.in_proj_weight"], sd[p + "self_attn.in_proj_bias"])
        q, k, v = (u.view(B, S, H, dh).transpose(1, 2) for u in qkv.split(d, dim=-1))
        s = matmul_bf16x3(q * (1.0 / math.sqrt(dh)), k.transpose(-1, -2))
        e = torch.exp(s - s.amax(-1, keepdim=True))
        eh, el = split_bf16(e)
        o = (matmul_bf16x3(e, v) / (eh + el).sum(-1, keepdim=True)).transpose(1, 2).reshape(B, S, d)
        x = x + lin(o, sd[p + "self_attn.out_proj.weight"], sd[p + "self_attn.out_proj.bias"])
        z = F.layer_norm(x, (d,), sd[p + "norm2.weight"], sd[p + "norm2.bias"], eps=1e-5)
        f = F.relu(lin(z, sd[p + "linear1.weight"], sd[p + "linear1.bias"]))
        h = x + lin(f, sd[p + "linear2.weight"], sd[p + "linear2.bias"])
    hn = F.layer_norm(h, (d,), sd[P + "head.0.weight"], sd[P + "head.0.bias"], eps=1e-5)
    return lin(hn, sd[P + "head.1.weight"])


def split_model(sd, vocab: O.VocabSpec, spec: O.ModelSpec) -> R.Model:
    """kernel_refs.Model of a split handle: the GEMM weights are the packed pairs (hi + lo, float64), everything else as in the
    unrounded model"""
    sd = dict(sd)
    for l in range(spec.layers):
        for k in GEMM_WEIGHTS:
            key = f"{O.PREFIX}backbone.layers.{l}.{k}"
            sd[key] = split_round(sd[key])
    sd[O.PREFIX + "head.1.weight"] = split_round(sd[O.PREFIX + "head.1.weight"])
    return R.Model(sd, vocab, spec, operand_dtype=None)
