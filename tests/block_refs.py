"""Test scaffolding for the denoiser block settings other than the default adalayernorm + relu: the unmodified reference
LayoutDM built with a given Block `timestep_type` / `activation` / `diffusion_step` (transformer_utils.py:103-170; oracle/ref_harness.py
builds the default), weights with the norm1 keys of each timestep_type, and the oracle's denoiser with those settings.

`block_forward` is oracle/layoutdm_oracle.py's `denoiser_forward` with norm1 and the feed-forward activation as the Block's
settings make them (transformer_utils.py:17-100):
    adalayernorm(_abs) : LN(x) (1 + scale_t) + shift_t          adainnorm(_abs) : InstanceNorm1d over the tokens, same affine
    None               : nn.LayerNorm(d) with weight / bias      *_abs           : emb(t) = SinusoidalPosEmb(diffusion_step, d)(t)
    relu | gelu (F.gelu, erf form) | gelu2 (x sigmoid(1.702 x))"""
from __future__ import annotations

import dataclasses
import glob
import json
import math
import os
from typing import Dict, Optional

import numpy as np
import torch
import torch.nn.functional as F

from oracle import layoutdm_oracle as O
from oracle import ref_harness as rh

TIMESTEP_TYPES = (None, "adalayernorm", "adainnorm", "adalayernorm_abs", "adainnorm_abs")
ACTIVATIONS = ("relu", "gelu", "gelu2")
# the 15 block configurations the reference can sample with
CONFIGS = [(tt, act) for tt in TIMESTEP_TYPES for act in ACTIVATIONS]


def config_id(tt, act) -> str:
    return f"{tt}-{act}"


def block_weights(vocab: O.VocabSpec, spec: O.ModelSpec, seed: int = 0, scale: float = 1.0, timestep_type: Optional[str] = "adalayernorm",
                  diffusion_step: Optional[int] = None) -> Dict[str, torch.Tensor]:
    """O.make_weights with each block's norm1 keys for timestep_type (transformer_utils.py:151-157): the Embedding of
    diffusion_step rows (default spec.T) and Linear of adalayernorm / adainnorm, the Linear alone for *_abs, an affine
    nn.LayerNorm (weight ~ 1 + N(0, 0.1), bias ~ N(0, 0.1), drawn from seed + 1) for None"""
    sd = O.make_weights(vocab, spec, seed=seed, scale=scale)
    g = torch.Generator().manual_seed(seed + 1)
    for l in range(spec.layers):
        p = f"{O.PREFIX}backbone.layers.{l}.norm1."
        if timestep_type is None:
            for k in ("emb.weight", "linear.weight", "linear.bias"):
                del sd[p + k]
            sd[p + "weight"] = 1.0 + torch.randn(spec.d, generator=g) * 0.1
            sd[p + "bias"] = torch.randn(spec.d, generator=g) * 0.1
        elif timestep_type.endswith("_abs"):
            del sd[p + "emb.weight"]
        elif diffusion_step is not None and diffusion_step != spec.T:
            sd[p + "emb.weight"] = torch.randn(diffusion_step, spec.d, generator=g)
    return sd


def sinusoidal(t: torch.Tensor, diffusion_step: int, d: int) -> torch.Tensor:
    """SinusoidalPosEmb(diffusion_step, d)(t) (transformer_utils.py:34-49) on long timesteps t (n,) -> (n, d)"""
    x = t / float(diffusion_step) * 4000.0
    half = d // 2
    e = torch.exp(torch.arange(half) * -(math.log(10000) / (half - 1)))
    e = x[:, None] * e[None, :]
    return torch.cat((e.sin(), e.cos()), dim=-1)


def activation_fn(activation: str):
    return {"relu": F.relu, "gelu": F.gelu, "gelu2": lambda x: x * torch.sigmoid(1.702 * x)}[activation]


def norm1(sd, l: int, h: torch.Tensor, t, timestep_type: Optional[str], diffusion_step: int) -> torch.Tensor:
    """the Block's norm1(h, t) of layer l; t an int or a (B,) tensor of per-layout timesteps"""
    p = f"{O.PREFIX}backbone.layers.{l}.norm1."
    d = h.shape[-1]
    if timestep_type is None:
        return F.layer_norm(h, (d,), sd[p + "weight"], sd[p + "bias"], eps=1e-5)
    tt = torch.as_tensor(t, dtype=torch.long).view(-1)
    e = sinusoidal(tt, diffusion_step, d) if timestep_type.endswith("_abs") else sd[p + "emb.weight"][tt]
    emb = F.linear(F.silu(e), sd[p + "linear.weight"], sd[p + "linear.bias"])[:, None]      # (1 | B, 1, 2d)
    scale, shift = emb[..., :d], emb[..., d:]
    if timestep_type.startswith("adainnorm"):
        x = F.instance_norm(h.transpose(-1, -2), eps=1e-5).transpose(-1, -2)
    else:
        x = F.layer_norm(h, (d,), eps=1e-5)
    return x * (1 + scale) + shift


def block_forward(sd, ids: torch.Tensor, t, vocab: O.VocabSpec, spec: O.ModelSpec, timestep_type: Optional[str] = "adalayernorm",
                  activation: str = "relu", diffusion_step: Optional[int] = None, operand_dtype: Optional[torch.dtype] = None) -> torch.Tensor:
    """ids (B,S) int64, timestep t (int or (B,) tensor) -> logits (B,S,C) fp32 of the denoiser with these block settings
    (operand_dtype: the same-rounding oracle, as in denoiser_forward)"""
    d, H, dh = spec.d, spec.heads, spec.dh
    B, S = ids.shape
    ds = spec.T if diffusion_step is None else diffusion_step
    r = lambda x: O._rnd(x, operand_dtype)
    act = activation_fn(activation)
    h = sd[O.PREFIX + "cat_emb.weight"][ids] + O.positional_table(sd, vocab, spec)[None]
    for l in range(spec.layers):
        p = f"{O.PREFIX}backbone.layers.{l}."
        x = norm1(sd, l, h, t, timestep_type, ds)
        qkv = F.linear(r(x), r(sd[p + "self_attn.in_proj_weight"]), sd[p + "self_attn.in_proj_bias"])
        q, k, v = qkv.split(d, dim=-1)
        q = q.view(B, S, H, dh).transpose(1, 2) * (1.0 / math.sqrt(dh))
        k = k.view(B, S, H, dh).transpose(1, 2)
        v = v.view(B, S, H, dh).transpose(1, 2)
        att = torch.softmax(r(q) @ r(k).transpose(-1, -2), dim=-1)
        o = (r(att) @ r(v)).transpose(1, 2).reshape(B, S, d)
        x = x + F.linear(r(o), r(sd[p + "self_attn.out_proj.weight"]), sd[p + "self_attn.out_proj.bias"])
        z = F.layer_norm(x, (d,), sd[p + "norm2.weight"], sd[p + "norm2.bias"], eps=1e-5)
        f = act(F.linear(r(z), r(sd[p + "linear1.weight"]), sd[p + "linear1.bias"]))
        h = x + F.linear(r(f), r(sd[p + "linear2.weight"]), sd[p + "linear2.bias"])
    hn = F.layer_norm(h, (d,), sd[O.PREFIX + "head.0.weight"], sd[O.PREFIX + "head.0.bias"], eps=1e-5)
    return F.linear(r(hn), r(sd[O.PREFIX + "head.1.weight"]))


@dataclasses.dataclass
class BlockOracle(O.Oracle):
    """O.Oracle whose denoiser is block_forward"""
    timestep_type: Optional[str] = "adalayernorm"
    activation: str = "relu"
    diffusion_step: Optional[int] = None

    def step_logprob(self, x_t: torch.Tensor, t_model: int, t_post: int, cond: Optional[dict] = None):
        logits = block_forward(self.sd, x_t, t_model, self.vocab, self.spec, self.timestep_type, self.activation, self.diffusion_step,
                               self.operand_dtype)
        return self.logprob_from_logits(logits, x_t, t_post, cond, t_model), logits


def build_reference(dataset: str = "rico25", T: int = 100, q_type: str = "constrained", state_dict=None, timestep_type="adalayernorm",
                    activation: str = "relu", diffusion_step: Optional[int] = None, max_seq_length: int = 25, num_layers: int = 4):
    """rh.build_reference with the Block's timestep_type / activation / diffusion_step (default T) and dataset.max_seq_length:
    (model, tokenizer), the reference LayoutDM in eval mode on CPU"""
    rh._setup_path()
    from omegaconf import OmegaConf
    from trainer.helpers.layout_tokenizer import LayoutSequenceTokenizer
    from trainer.models.layoutdm import LayoutDM

    data_cfg = OmegaConf.create(dict(
        batch_size=64, bbox_quantization="linear", num_bin_bboxes=32, num_workers=1, pad_until_max=True,
        shared_bbox_vocab="x-y-w-h", special_tokens=["pad", "mask"], transforms=["RandomOrder"], var_order="c-x-y-w-h"))
    target = {"rico25": "trainer.datasets.rico.Rico25Dataset", "publaynet": "trainer.datasets.publaynet.PubLayNetDataset"}[dataset]
    dataset_cfg = OmegaConf.create(dict(_target_=target, _partial_=True, dir="x", max_seq_length=max_seq_length))
    backbone_cfg = OmegaConf.create(dict(
        _target_="trainer.models.transformer_utils.TransformerEncoder", num_layers=num_layers,
        encoder_layer=dict(_target_="trainer.models.transformer_utils.Block", d_model=512, nhead=8,
                           dim_feedforward=2048, dropout=0.0, batch_first=True, norm_first=True, activation=activation,
                           timestep_type=timestep_type, diffusion_step=T if diffusion_step is None else diffusion_step)))
    tok = LayoutSequenceTokenizer(data_cfg, dataset_cfg)
    torch.manual_seed(0)
    model = LayoutDM(backbone_cfg=backbone_cfg, tokenizer=tok, q_type=q_type, num_timesteps=T).eval()
    if state_dict is not None:
        missing, unexpected = model.load_state_dict(state_dict, strict=False)
        assert all(("_log_" in k) or k.split(".")[-1].startswith(("Lt_", "log_")) for k in missing), missing
        assert not unexpected, unexpected
    return model, tok


# ---- the fixtures of tests/golden/blocks (make_block_golden.py) ------------------------------------------------------------

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "blocks")
NAMES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN, "*.npz")))


class BlockFixture:
    """a fixture of make_block_golden.py: the fields of fixtures.Fixture, with the case's vocabulary and block settings"""

    def __init__(self, name):
        z = np.load(os.path.join(GOLDEN, name + ".npz"))
        m = self.meta = json.loads(str(z["meta"]))
        self.z = z
        self.vocab = dataclasses.replace(O.RICO25 if m["dataset"] == "rico25" else O.PUBLAYNET, n_elem=m["n_elem"])
        self.spec = O.ModelSpec(T=m["T"])
        self.timestep_type, self.activation, self.diffusion_step = m["timestep_type"], m["activation"], m["diffusion_step"]
        self.plan = [tuple(p) for p in m["plan"]]
        self.B = m["B"]
        ld = lambda k: torch.from_numpy(z[k].astype(np.int64))
        self.x_in, self.x_out, self.ids_final = ld("x_in"), ld("x_out"), ld("ids_final")
        self.trace_steps = m["trace_steps"]
        self.cfg = O.SamplingCfg(name=m["sampling"], temperature=m["temperature"], top_p=m["top_p"], top_k=m["top_k"],
                                 num_timesteps=m["T_eval"], time_difference=m["time_difference"])
        self.cfg_dict = dict(name=m["sampling"], temperature=m["temperature"], top_p=m["top_p"], top_k=m["top_k"],
                             num_timesteps=m["T_eval"], time_difference=m["time_difference"])
        self.cond = None
        if m["cond"]:
            self.cond = dict(seq=ld("cond_seq"), mask=torch.from_numpy(z["cond_mask"]), type=m["cond"])

    def weights(self):
        sd = block_weights(self.vocab, self.spec, seed=self.meta["weight_seed"], scale=self.meta["weight_scale"], timestep_type=self.timestep_type)
        chk = O.weights_checksum(sd)
        assert abs(chk - self.meta["weights_checksum"]) <= 1e-6 * abs(chk), "synthetic weight generator drifted from the fixture"
        return sd

    def oracle(self, operand_dtype=None) -> BlockOracle:
        return BlockOracle(self.vocab, self.spec, self.weights(), q_type=self.meta["q_type"], operand_dtype=operand_dtype,
                           timestep_type=self.timestep_type, activation=self.activation, diffusion_step=self.diffusion_step)

    def logits(self, i):
        return torch.from_numpy(self.z[f"logits_{i}"])

    def logp(self, i):
        return torch.from_numpy(self.z[f"logp_{i}"])

    def noise(self, i):
        return O.uniforms(self.meta["noise_seed"], i, 0, 0, self.B, self.vocab.S, self.vocab.C)

    def host_vocab(self):
        from layoutdm_b200 import Vocab
        return Vocab.for_dataset(self.meta["dataset"], self.meta["n_elem"])
