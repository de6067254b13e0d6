"""Test scaffolding for the tokenizer settings other than the default x-y-w-h / c-x-y-w-h vocabulary: the unmodified reference
LayoutDM built with a given `shared_bbox_vocab`, `var_order` and `num_bin_bboxes` (oracle/ref_harness.py builds the default),
and the oracle's vocabulary restated for those settings.

The oracle (oracle/layoutdm_oracle.py) reads the vocabulary through VocabSpec's C / pad_id / group_start / group_n for the
denoiser, the posterior and the draw; LayoutSpec gives those the slot layout of BboxTokenizer (bbox_tokenizer.py:17-20,
105-113) and LayoutSequenceTokenizer.get_slice (layout_tokenizer.py:296-313).  What the oracle writes out with the x-y-w-h
offsets itself (encode / decode, get_cond, the refinement table) is restated here from the same slot layout."""
from __future__ import annotations

import dataclasses
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch

from oracle import layoutdm_oracle as O
from oracle import ref_harness as rh

BBOX_VARS = ("x", "y", "w", "h")


@dataclasses.dataclass(frozen=True)
class LayoutSpec(O.VocabSpec):
    shared_bbox_vocab: str = "x-y-w-h"
    var_order: str = "c-x-y-w-h"

    @property
    def n_bbox_ids(self) -> int:
        return self.n_bins * (1 if self.shared_bbox_vocab == "xywh" else 4)

    @property
    def C(self) -> int:
        return self.n_cat + self.n_bbox_ids + 2

    @property
    def pad_id(self) -> int:
        return self.n_cat + self.n_bbox_ids

    def var_start(self, name: str) -> int:
        if name == "c":
            return 0
        return self.n_cat + (0 if self.shared_bbox_vocab == "xywh" else BBOX_VARS.index(name) * self.n_bins)

    def slots(self) -> List[Tuple[str, int, int]]:
        """(variable, first id, ids) of each token slot, in var_order"""
        return [(v, self.var_start(v), self.n_cat if v == "c" else self.n_bins) for v in self.var_order.split("-")]

    def group_start(self, g: int) -> int:
        return self.slots()[g][1]

    def group_n(self, g: int) -> int:
        return self.slots()[g][2]


# the configurations the fixtures of tests/golden/token_layouts/ were recorded with: name -> (dataset, shared, order, bins, q_type)
CONFIGS = {
    "rico25_xywh": ("rico25", "xywh", "c-x-y-w-h", 32, "constrained"),               # C = 59
    "publaynet_cwhxy": ("publaynet", "x-y-w-h", "c-w-h-x-y", 32, "constrained"),     # C = 135
    "rico25_bins16": ("rico25", "x-y-w-h", "c-x-y-w-h", 16, "constrained"),          # C = 91
    "rico25_xywh_bins64": ("rico25", "xywh", "c-x-y-w-h", 64, "constrained"),        # C = 91, groups of 64 classes
    "rico25_vanilla_xywh_cwhxy": ("rico25", "xywh", "c-w-h-x-y", 16, "vanilla"),     # C = 43
}


def spec_of(config: str, n_elem: int = 25) -> LayoutSpec:
    dataset, shared, order, bins, _ = CONFIGS[config]
    return LayoutSpec(n_cat=(O.RICO25 if dataset == "rico25" else O.PUBLAYNET).n_cat, n_bins=bins, n_elem=n_elem,
                      shared_bbox_vocab=shared, var_order=order)


def tokenizer(dataset: str = "rico25", shared_bbox_vocab: str = "x-y-w-h", var_order: str = "c-x-y-w-h", num_bin_bboxes: int = 32):
    """the reference's LayoutSequenceTokenizer with DataConfig's shared_bbox_vocab / var_order / num_bin_bboxes
    (hydra_configs.py:64-83), linear quantisation, special tokens (pad, mask), 25 elements"""
    rh._setup_path()
    from omegaconf import OmegaConf
    from trainer.helpers.layout_tokenizer import LayoutSequenceTokenizer

    data_cfg = OmegaConf.create(dict(
        batch_size=64, bbox_quantization="linear", num_bin_bboxes=num_bin_bboxes, num_workers=1, pad_until_max=True,
        shared_bbox_vocab=shared_bbox_vocab, special_tokens=["pad", "mask"], transforms=["RandomOrder"], var_order=var_order))
    target = {"rico25": "trainer.datasets.rico.Rico25Dataset", "publaynet": "trainer.datasets.publaynet.PubLayNetDataset"}[dataset]
    return LayoutSequenceTokenizer(data_cfg, OmegaConf.create(dict(_target_=target, _partial_=True, dir="x", max_seq_length=25)))


def build_reference(dataset: str = "rico25", T: int = 100, q_type: str = "constrained", state_dict=None, shared_bbox_vocab: str = "x-y-w-h",
                    var_order: str = "c-x-y-w-h", num_bin_bboxes: int = 32, num_layers: int = 4, pos_emb: Optional[str] = None):
    """rh.build_reference with the tokenizer of `tokenizer(...)`: (model, tokenizer), the reference LayoutDM in eval mode on CPU.
    pos_emb: the transformer's positional embedding when given."""
    tok = tokenizer(dataset, shared_bbox_vocab, var_order, num_bin_bboxes)
    from omegaconf import OmegaConf
    from trainer.models.layoutdm import LayoutDM

    backbone_cfg = OmegaConf.create(dict(
        _target_="trainer.models.transformer_utils.TransformerEncoder", num_layers=num_layers,
        encoder_layer=dict(_target_="trainer.models.transformer_utils.Block", d_model=512, nhead=8,
                           dim_feedforward=2048, dropout=0.0, batch_first=True, norm_first=True,
                           timestep_type="adalayernorm", diffusion_step=T)))
    torch.manual_seed(0)
    kw = {} if pos_emb is None else {"pos_emb": pos_emb}
    model = LayoutDM(backbone_cfg=backbone_cfg, tokenizer=tok, q_type=q_type, num_timesteps=T, **kw).eval()
    if state_dict is not None:
        missing, unexpected = model.load_state_dict(state_dict, strict=False)
        assert all(("_log_" in k) or k.split(".")[-1].startswith(("Lt_", "log_")) for k in missing), missing
        assert not unexpected, unexpected
    return model, tok


def build_config(config: str, T: int = 100, state_dict=None, **kw):
    dataset, shared, order, bins, q_type = CONFIGS[config]
    return build_reference(dataset, T=T, q_type=q_type, state_dict=state_dict, shared_bbox_vocab=shared, var_order=order,
                           num_bin_bboxes=bins, **kw)


# ---- restatements of what the oracle writes with the x-y-w-h offsets ------------------------------------------------------

def refinement_table(vs: LayoutSpec, centers, mode: str = "uniform", offset_ratio: float = 0.1, weight: float = 3.0) -> torch.Tensor:
    """_index_to_smoothed_log_onehot (task.py:154-201) as a (C, C) table times +-refine_lambda (:212-223): variable i's block
    at its own ids; shared, the four write one block and h, the last, wins"""
    w = -weight if mode == "negative" else weight
    tbl = torch.zeros(vs.C, vs.C)
    tbl.fill_diagonal_(1.0)
    for i, name in enumerate(BBOX_VARS):
        cc = torch.from_numpy(np.asarray(centers[i], dtype=np.float64)).view(-1)
        ii, jj = torch.meshgrid(cc, cc, indexing="ij")
        lo = vs.var_start(name)
        sl = slice(lo, lo + vs.n_bins)
        if mode == "uniform":
            tbl[sl, sl] = (torch.abs(ii - jj) < offset_ratio).float()
        elif mode == "negative":
            tbl[sl, sl] = (torch.abs(ii - jj) >= offset_ratio).float()
        else:
            tbl[sl, sl] = (-1.0 * (ii - jj) ** 2).float()
    return tbl * w


def encode_bins(bbox: torch.Tensor, n_bins: int, centers: Optional[torch.Tensor] = None) -> torch.Tensor:
    """BboxTokenizer.encode's bins (bbox_tokenizer.py:84-103) in x, y, w, h order: (..., 4) f32 -> (..., 4) i64"""
    if centers is None:
        d = 1 / n_bins
        q = torch.zeros_like(bbox)
        q[..., :2] = torch.clamp(bbox[..., :2], 0.0, 1.0 - d)
        q[..., 2:] = torch.clamp(bbox[..., 2:], d, 1.0) - d
        return (n_bins * q).round().long()
    return (bbox[..., None] - centers.to(bbox.dtype)).pow(2).argmin(dim=-1)                 # KMeans.predict, first on ties


def encode_layouts(label: torch.Tensor, bbox: torch.Tensor, mask: torch.Tensor, vs: LayoutSpec,
                   centers: Optional[torch.Tensor] = None) -> torch.Tensor:
    """LayoutSequenceTokenizer.encode (layout_tokenizer.py:208-253) of dense layouts: (B, E) / (B, E, 4) / (B, E) -> (B, S) ids"""
    bins = encode_bins(bbox, vs.n_bins, centers)
    cols = [label.long()] + [bins[..., BBOX_VARS.index(v)] + lo for v, lo, _ in vs.slots()[1:]]
    tok = torch.stack(cols, dim=-1)
    tok[~mask] = vs.pad_id
    return tok.reshape(label.shape[0], -1)


def make_cond(label: torch.Tensor, bbox: torch.Tensor, mask: torch.Tensor, vs: LayoutSpec, cond_type: str,
              centers: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
    """get_cond (task.py:27-151) for c / cwh / refinement / gt: seq, mask (and seq_orig); slots kept by variable name"""
    seq = encode_layouts(label, bbox, mask, vs, centers)
    B, S = seq.shape
    valid = mask.repeat_interleave(vs.n_attr, dim=1)
    var = [v for v, _, _ in vs.slots()]
    names = {"c": "c", "cwh": "cwh", "refinement": "c", "gt": "cxywh"}[cond_type]
    keep = torch.tensor([var[s % vs.n_attr] in names for s in range(S)])[None].expand(B, S)
    out = {"mask": valid.clone() if cond_type == "gt" else (valid & keep) | ~valid}
    out["seq"] = torch.where(out["mask"] | ~valid, seq, torch.full_like(seq, vs.mask_id))
    out["seq"] = torch.where(valid, out["seq"], torch.full_like(seq, vs.pad_id))
    if cond_type == "refinement":
        out["seq_orig"] = seq
    return out


def decode_ids(ids: torch.Tensor, vs: LayoutSpec, centers: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
    """LayoutSequenceTokenizer.decode (layout_tokenizer.py:255-266) + BboxTokenizer.decode (bbox_tokenizer.py:117-174)"""
    x = ids.view(ids.shape[0], vs.n_elem, vs.n_attr)
    label = x[..., 0].clone()
    bb = x[..., 1:] - vs.n_cat
    invalid = ~(((0 <= label) & (label < vs.n_cat)) & ((0 <= bb) & (bb < vs.n_bbox_ids)).all(-1))
    by_var = {v: x[..., k] - lo for k, (v, lo, _) in enumerate(vs.slots()) if v != "c"}
    arr = torch.clamp(torch.stack([by_var[v] for v in BBOX_VARS], dim=-1), 0, vs.n_bins - 1)
    if centers is None:
        d = 1 / vs.n_bins
        out = torch.zeros(arr.shape, dtype=torch.float32)
        out[..., :2] = arr[..., :2].float() * d
        out[..., 2:] = (arr[..., 2:] + 1).float() * d
    else:
        out = torch.clamp(torch.stack([centers[i].double()[arr[..., i]] for i in range(4)], dim=-1), 0.0, 1.0).float()
    label[invalid] = 0
    out[invalid] = 0.0
    return {"bbox": out, "label": label, "mask": ~invalid}
