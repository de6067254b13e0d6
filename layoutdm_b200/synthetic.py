"""Synthetic inputs for benchmarks and smoke runs (no datasets or checkpoints are available offline):
random-init weights under the reference's `state_dict` key names and synthetic conditions shaped like
`helpers/task.py:get_cond` output."""
from __future__ import annotations

from typing import Dict, Optional

import torch

from .vocab import BBOX_VARS, Vocab, linear_centers, refinement_table

PREFIX = "model.module.transformer."


def random_state_dict(vocab: Vocab, num_timesteps: int = 100, d: int = 464, ff: int = 1856, layers: int = 4, seed: int = 0,
                      std: float = 0.02, timestep_type: Optional[str] = "adalayernorm") -> Dict[str, torch.Tensor]:
    """Weights distributed like the reference's initialisation (base_model.py:108-116: N(0, 0.02) for Linear / Embedding,
    pos-emb ~ U(0,1) nn_lib.py:109-110), with small non-zero biases / LN affine terms so no term is trivially zero.
    timestep_type: the blocks' norm1 keys (transformer_utils.py:151-157): the Embedding of adalayernorm / adainnorm, none for
    the *_abs types, an affine nn.LayerNorm for None.  The other parameters are drawn as for the default."""
    g = torch.Generator().manual_seed(seed)
    n = lambda *shape, s=std: torch.randn(*shape, generator=g) * s
    sd = {PREFIX + "cat_emb.weight": n(vocab.C, d),
          PREFIX + "pos_emb.elem_emb": torch.rand(vocab.n_elem, d, generator=g),
          PREFIX + "pos_emb.attr_emb": torch.rand(vocab.n_attr, d, generator=g)}
    for l in range(layers):
        p = f"{PREFIX}backbone.layers.{l}."
        sd[p + "self_attn.in_proj_weight"] = n(3 * d, d)
        sd[p + "self_attn.in_proj_bias"] = n(3 * d)
        sd[p + "self_attn.out_proj.weight"] = n(d, d)
        sd[p + "self_attn.out_proj.bias"] = n(d)
        sd[p + "linear1.weight"] = n(ff, d)
        sd[p + "linear1.bias"] = n(ff)
        sd[p + "linear2.weight"] = n(d, ff)
        sd[p + "linear2.bias"] = n(d)
        emb, w, b = n(num_timesteps, d, s=1.0), n(2 * d, d), n(2 * d)
        if timestep_type is None:
            sd[p + "norm1.weight"], sd[p + "norm1.bias"] = 1.0 + n(d, s=0.1), n(d, s=0.1)
        else:
            if not timestep_type.endswith("_abs"):
                sd[p + "norm1.emb.weight"] = emb
            sd[p + "norm1.linear.weight"], sd[p + "norm1.linear.bias"] = w, b
        sd[p + "norm2.weight"] = 1.0 + n(d, s=0.1)
        sd[p + "norm2.bias"] = n(d, s=0.1)
    sd[PREFIX + "head.0.weight"] = 1.0 + n(d, s=0.1)
    sd[PREFIX + "head.0.bias"] = n(d, s=0.1)
    sd[PREFIX + "head.1.weight"] = n(vocab.C, d)
    return sd


def synthetic_cond(vocab: Vocab, B: int, cond_type: str = "c", seed: int = 0, refine: Optional[dict] = None) -> Dict:
    """cond dict for `c` / `cwh` / `refinement` built from random layouts (n_elem ~ U{1..vocab.n_elem}, labels uniform, boxes uniform,
    linear quantisation), following get_cond (task.py:94-110, 126-140) and tokenizer.encode (layout_tokenizer.py:208-253)."""
    assert cond_type in ("c", "cwh", "refinement")
    g = torch.Generator().manual_seed(seed)
    E, A, nb = vocab.n_elem, vocab.n_attr, vocab.n_bins
    n_el = torch.randint(1, E + 1, (B,), generator=g)
    valid = torch.arange(E)[None] < n_el[:, None]                       # (B,E)
    label = torch.randint(0, vocab.n_cat, (B, E), generator=g)
    bbox = torch.rand(B, E, 4, generator=g)
    if cond_type == "refinement":
        bbox = bbox + torch.randn(B, E, 4, generator=g) * 0.1           # task.py:127
    d = 1.0 / nb
    q = torch.zeros_like(bbox)
    q[..., :2] = torch.clamp(bbox[..., :2], 0.0, 1.0 - d)
    q[..., 2:] = torch.clamp(bbox[..., 2:], d, 1.0) - d
    bins = (nb * q).round().long()                                      # bbox_tokenizer.py:88-91, x y w h
    slots = vocab.slots()
    # each slot: its variable's bin plus the first id of that variable (bbox_tokenizer.py:105-113 + layout_tokenizer.py:223)
    idx = torch.stack([bins[..., BBOX_VARS.index(name)] + sl.start for name, sl in slots[1:]], dim=-1)
    full = torch.cat([label[..., None], idx], dim=-1)                   # (B,E,5)
    full[~valid] = vocab.pad_id
    seq_full = full.view(B, E * A)
    elem_valid = valid[..., None].expand(B, E, A).reshape(B, E * A)
    kept = {"c": "c", "cwh": "cwh", "refinement": "c"}[cond_type]     # get_cond keeps slots by variable name (task.py:103-105)
    keep = torch.tensor([slots[s % A][0] in kept for s in range(E * A)])[None]
    mask = (elem_valid & keep) | ~elem_valid
    seq = torch.where(mask, seq_full, torch.full_like(seq_full, vocab.mask_id))
    seq = torch.where(elem_valid, seq, torch.full_like(seq, vocab.pad_id))
    cond = {"seq": seq, "mask": mask, "type": cond_type, "num_element": n_el}
    if cond_type == "refinement":
        r = dict(refine_mode="uniform", refine_offset_ratio=0.1, refine_lambda=3.0)
        r.update(refine or {})
        cond["seq_orig"] = seq_full
        cond["refine_table"] = refinement_table(vocab, linear_centers(nb), r["refine_mode"], r["refine_offset_ratio"], r["refine_lambda"])
    return cond
