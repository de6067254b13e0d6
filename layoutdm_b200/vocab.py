"""Host-side neighbours of the hot path: vocabulary layout, timestep plan, refinement table, token decode.
Mirrors (file:line under src/trainer/trainer/):
  Vocab              helpers/layout_tokenizer.py:79-82,296-313 + helpers/bbox_tokenizer.py:17-20,105-113 (either var_order,
                     either shared_bbox_vocab, special tokens pad+mask)
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


BBOX_VOCABS = ("x-y-w-h", "xywh")          # helpers/layout_tokenizer.py:16-20 CHOICES
VAR_ORDERS = ("c-x-y-w-h", "c-w-h-x-y")
BBOX_VARS = ("x", "y", "w", "h")              # BboxTokenizer.var_names: the order of bbox values and bin centres


@dataclass(frozen=True)
class Vocab:
    n_cat: int = 25
    n_bins: int = 32
    n_elem: int = 25
    n_attr: int = 5
    shared_bbox_vocab: str = "x-y-w-h"        # "xywh": x, y, w and h share one range of n_bins ids
    var_order: str = "c-x-y-w-h"              # the variables of an element's token slots

    def __post_init__(self):
        if self.shared_bbox_vocab not in BBOX_VOCABS:
            raise ValueError(f"shared_bbox_vocab must be one of {BBOX_VOCABS}, got {self.shared_bbox_vocab!r}")
        if self.var_order not in VAR_ORDERS:
            raise ValueError(f"var_order must be one of {VAR_ORDERS}, got {self.var_order!r}")

    @classmethod
    def for_dataset(cls, name: str, max_seq_length: int = 25, num_bin_bboxes: int = 32, shared_bbox_vocab: str = "x-y-w-h",
                    var_order: str = "c-x-y-w-h") -> "Vocab":
        """the dataset's vocabulary for layouts of up to `max_seq_length` elements (config/dataset/*.yaml: dataset.max_seq_length)
        and the tokenizer settings of DataConfig (hydra_configs.py:64-83)"""
        return cls(n_cat=DATASET_NUM_CATEGORIES[name], n_bins=int(num_bin_bboxes), n_elem=int(max_seq_length),
                   shared_bbox_vocab=shared_bbox_vocab, var_order=var_order)

    @classmethod
    def from_tokenizer(cls, tok) -> "Vocab":
        """from a reference LayoutSequenceTokenizer with special tokens (pad, mask)"""
        if list(tok.special_tokens) != ["pad", "mask"]:
            raise NotImplementedError(f"special tokens {list(tok.special_tokens)}: only ['pad', 'mask'] (the diffusion models') are supported")
        return cls(n_cat=tok.N_category, n_bins=tok.N_bbox_per_var, n_elem=tok.max_seq_length, n_attr=tok.N_var_per_element,
                   shared_bbox_vocab=tok.bbox_tokenizer.shared_bbox_vocab, var_order=tok.var_order)

    def var_slice(self, name: str) -> slice:
        """the full-vocabulary ids of variable `name` (LayoutSequenceTokenizer.get_slice, layout_tokenizer.py:296-313)"""
        if name == "c":
            return slice(0, self.n_cat)
        start = self.n_cat + (0 if self.shared_bbox_vocab == "xywh" else BBOX_VARS.index(name) * self.n_bins)
        return slice(start, start + self.n_bins)

    def slots(self) -> List[Tuple[str, slice]]:
        """(variable, full-vocabulary ids) of each token slot of an element, in var_order: the one description of the token
        layout every host consumer reads (the device builds the same table in ldm_create)"""
        return [(name, self.var_slice(name)) for name in self.var_order.split("-")]

    @property
    def n_bbox_ids(self) -> int:
        """ids of the bbox vocabulary (BboxTokenizer.bbox_vocab_len): n_bins shared, 4 n_bins per variable"""
        return self.n_bins * (1 if self.shared_bbox_vocab == "xywh" else 4)

    @property
    def C(self) -> int:
        return self.n_cat + self.n_bbox_ids + 2

    @property
    def S(self) -> int:
        return self.n_elem * self.n_attr

    @property
    def pad_id(self) -> int:
        return self.n_cat + self.n_bbox_ids

    @property
    def mask_id(self) -> int:
        return self.pad_id + 1

    @property
    def relation_on_device(self) -> bool:
        """the device relation update reads slot 1+a as variable a with one lane per bin: c-x-y-w-h and at most 32 bins"""
        return self.var_order == "c-x-y-w-h" and self.n_bins <= 32


def group_full_ids(vocab: "Vocab", g: int) -> List[int]:
    """full-vocabulary ids of slot g's partial vocabulary [its classes..., PAD, MASK] (Converter, layout_tokenizer.py:429-467)"""
    sl = vocab.slots()[g][1]
    return list(range(sl.start, sl.stop)) + [vocab.pad_id, vocab.mask_id]


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
    """(C, C) fp32 table, weak_logits[b, c, s] == table[seq_orig[b, s], c]; already multiplied by +-refine_lambda.
    centers: per variable x, y, w, h.  Each variable writes the block of its own ids; with a shared vocabulary the four write
    the same block and the last one (h) wins, as in the reference."""
    assert mode in ("uniform", "gaussian", "negative")
    w = -weight if mode == "negative" else weight
    tbl = torch.zeros(vocab.C, vocab.C)
    tbl.fill_diagonal_(1.0)
    for i, name in enumerate(BBOX_VARS):
        cc = torch.from_numpy(np.asarray(centers[i], dtype=np.float64)).view(-1)
        ii, jj = torch.meshgrid(cc, cc, indexing="ij")
        sl = vocab.var_slice(name)
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
    label = x[..., 0].clone()
    label_valid = (0 <= label) & (label < vocab.n_cat)
    bbox_valid = ((0 <= x[..., 1:] - vocab.n_cat) & (x[..., 1:] - vocab.n_cat < vocab.n_bbox_ids)).all(dim=-1)
    invalid = ~(label_valid & bbox_valid)
    # each slot's bin within its variable's ids, back in x, y, w, h order (BboxTokenizer.decode, bbox_tokenizer.py:117-141)
    bins = {name: x[..., k] - sl.start for k, (name, sl) in enumerate(vocab.slots()) if name != "c"}
    arr = torch.clamp(torch.stack([bins[name] for name in BBOX_VARS], dim=-1), 0, vocab.n_bins - 1)
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
