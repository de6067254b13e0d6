"""Host-side neighbours of the hot path: vocabulary layout, timestep plan, refinement table, token decode.
Mirrors (file:line under src/trainer/trainer/):
  Vocab              helpers/layout_tokenizer.py:79-82,296-313 (var_order c-x-y-w-h, shared_bbox_vocab x-y-w-h, pad+mask)
  timestep_plan      models/categorical_diffusion/base.py:310-315,348-358 (+ :218-240 posterior timestep)
  refinement_table   helpers/task.py:154-224
  decode_ids         helpers/layout_tokenizer.py:255-266 + helpers/bbox_tokenizer.py:117-174
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

DATASET_NUM_CATEGORIES = {"rico25": 25, "publaynet": 5}   # datasets/rico.py:42-68, datasets/publaynet.py:13-19


@dataclass(frozen=True)
class Vocab:
    n_cat: int = 25
    n_bins: int = 32
    n_elem: int = 25
    n_attr: int = 5

    @classmethod
    def for_dataset(cls, name: str, max_seq_length: int = 25) -> "Vocab":
        """the dataset's vocabulary for layouts of up to `max_seq_length` elements (config/dataset/*.yaml: dataset.max_seq_length)"""
        return cls(n_cat=DATASET_NUM_CATEGORIES[name], n_elem=int(max_seq_length))

    @classmethod
    def from_tokenizer(cls, tok) -> "Vocab":
        """from a reference LayoutSequenceTokenizer"""
        assert tok.var_order == "c-x-y-w-h" and list(tok.special_tokens) == ["pad", "mask"]
        assert tok.bbox_tokenizer.shared_bbox_vocab == "x-y-w-h"
        return cls(n_cat=tok.N_category, n_bins=tok.N_bbox_per_var, n_elem=tok.max_seq_length, n_attr=tok.N_var_per_element)

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


def group_full_ids(vocab: "Vocab", g: int) -> List[int]:
    """full-vocabulary ids of attribute g's partial vocabulary [its classes..., PAD, MASK] (Converter, layout_tokenizer.py:429-467)"""
    lo = 0 if g == 0 else vocab.n_cat + (g - 1) * vocab.n_bins
    n = vocab.n_cat if g == 0 else vocab.n_bins
    return list(range(lo, lo + n)) + [vocab.pad_id, vocab.mask_id]


def timestep_plan(T: int, T_eval: int, time_difference: float = 0.0) -> List[Tuple[int, int]]:
    """[(t_model, t_posterior)] per loop iteration."""
    assert T_eval <= T                                   # base.py:311
    plan, prev = [], T
    for i in range(T_eval - 1, -1, -1):
        t = int(i * T / T_eval)
        delta = prev - t
        if delta <= 0:
            raise NotImplementedError                    # base.py:361-362
        skip = delta - 1
        noise_t = min(max(t - int(T * time_difference), 0), T - 1) if time_difference > 0.0 else t
        t_post = noise_t - skip if (skip > 0 and noise_t > skip) else noise_t
        plan.append((t, t_post))
        prev = t
    return plan


def linear_centers(n_bins: int = 32) -> List[np.ndarray]:
    d = 1 / n_bins
    xy = np.linspace(start=0.0, stop=1.0 - d, num=n_bins)
    wh = np.linspace(start=d, stop=1.0, num=n_bins)
    return [xy, xy, wh, wh]


def refinement_table(vocab: Vocab, centers: Sequence[np.ndarray], mode: str = "uniform", offset_ratio: float = 0.1,
                     weight: float = 3.0) -> torch.Tensor:
    """(C, C) fp32 table, weak_logits[b, c, s] == table[seq_orig[b, s], c]; already multiplied by +-refine_lambda."""
    assert mode in ("uniform", "gaussian", "negative")
    w = -weight if mode == "negative" else weight
    tbl = torch.zeros(vocab.C, vocab.C)
    tbl.fill_diagonal_(1.0)
    for i in range(4):
        cc = torch.from_numpy(np.asarray(centers[i], dtype=np.float64)).view(-1)
        ii, jj = torch.meshgrid(cc, cc, indexing="ij")
        sl = slice(vocab.n_cat + i * vocab.n_bins, vocab.n_cat + (i + 1) * vocab.n_bins)
        if mode == "uniform":
            tbl[sl, sl] = (torch.abs(ii - jj) < offset_ratio).float()
        elif mode == "negative":
            tbl[sl, sl] = (torch.abs(ii - jj) >= offset_ratio).float()
        else:
            tbl[sl, sl] = (-1.0 * (ii - jj) ** 2).float()
    return tbl * w


def decode_ids(ids: torch.Tensor, vocab: Vocab, centers: Optional[Sequence[np.ndarray]] = None) -> Dict[str, torch.Tensor]:
    """ids (B, S) int64 (CPU) -> {"bbox": (B, n_elem, 4) f32, "label": (B, n_elem) i64, "mask": (B, n_elem) bool}.
    centers=None: linear quantisation; else per-variable cluster centres (kmeans / percentile)."""
    x = ids.view(ids.shape[0], vocab.n_elem, vocab.n_attr)
    label, bbox = x[..., 0].clone(), x[..., 1:].clone() - vocab.n_cat
    label_valid = (0 <= label) & (label < vocab.n_cat)
    bbox_valid = ((0 <= bbox) & (bbox < 4 * vocab.n_bins)).all(dim=-1)
    invalid = ~(label_valid & bbox_valid)
    arr = torch.clamp(bbox - torch.arange(4) * vocab.n_bins, 0, vocab.n_bins - 1)
    if centers is None:
        d = 1 / vocab.n_bins
        out = torch.zeros(arr.shape, dtype=torch.float32)
        out[..., :2] = arr[..., :2].float() * d
        out[..., 2:] = (arr[..., 2:] + 1).float() * d
    else:
        cols = [torch.from_numpy(np.asarray(centers[i]).reshape(-1))[arr[..., i]] for i in range(4)]
        out = torch.clamp(torch.stack(cols, dim=-1), 0.0, 1.0).float()
    label[invalid] = 0
    out[invalid] = 0.0
    return {"bbox": out, "label": label, "mask": ~invalid}


def relation_edge_table(batch, n_layouts: int, n_slots: int) -> torch.Tensor:
    """cond["batch_w_canvas"] (the PyG batch `get_cond(..., "relation")` attaches, helpers/task.py:112-114; node 0 of every
    layout is the canvas, data/util.py:106-120) -> dense (B, n_slots, n_slots) int32 table of its edge_attr bit masks
    (RelSize / RelLoc, data/util.py:14-27): table[b, i, j] = attr of the edge i -> j, 0 = no edge.  This is what LdmCond.rel_adj takes."""
    tab = torch.zeros(n_layouts, n_slots, n_slots, dtype=torch.int32)
    ei = getattr(batch, "edge_index", None)
    if ei is None or ei.numel() == 0:
        return tab
    ei, ea, bv = ei.cpu().long(), batch.edge_attr.cpu(), batch.batch.cpu().long()
    num = torch.zeros(n_layouts, dtype=torch.long).scatter_add_(0, bv, torch.ones_like(bv))
    first = torch.cat([num.new_zeros(1), num.cumsum(0)])
    b = bv[ei[0]]
    tab[b, ei[0] - first[b], ei[1] - first[b]] = ea.to(torch.int32)
    return tab
