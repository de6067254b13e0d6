"""Test scaffolding for layouts of more than 25 elements: the unmodified reference LayoutDM built for a given
`dataset.max_seq_length` (oracle/ref_harness.py builds it for the default 25), and the workspace tap read with a layout's
128 R rows."""
from __future__ import annotations

import torch

import gpu_helpers as G
from oracle import ref_harness as rh


def build_reference(dataset: str = "rico25", T: int = 100, q_type: str = "constrained", state_dict=None, max_seq_length: int = 25):
    """rh.build_reference with dataset.max_seq_length = max_seq_length (config/dataset/*.yaml): (model, tokenizer), the
    reference LayoutDM in eval mode on CPU whose tokenizer, positional table and sampling use S = 5 max_seq_length tokens"""
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
        _target_="trainer.models.transformer_utils.TransformerEncoder", num_layers=4,
        encoder_layer=dict(_target_="trainer.models.transformer_utils.Block", d_model=512, nhead=8,
                           dim_feedforward=2048, dropout=0.0, batch_first=True, norm_first=True,
                           timestep_type="adalayernorm", diffusion_step=T)))
    tok = LayoutSequenceTokenizer(data_cfg, dataset_cfg)
    torch.manual_seed(0)
    model = LayoutDM(backbone_cfg=backbone_cfg, tokenizer=tok, q_type=q_type, num_timesteps=T).eval()
    if state_dict is not None:
        missing, unexpected = model.load_state_dict(state_dict, strict=False)
        assert all(("_log_" in k) or k.split(".")[-1].startswith(("Lt_", "log_")) for k in missing), missing
        assert not unexpected, unexpected
    return model, tok


_debug_read = G.debug_read


def debug_read(engine, name: str, n_layouts: int, raw: bool = False) -> torch.Tensor:
    """gpu_helpers.debug_read with the rows a layout takes in the workspace: [n_layouts, 128 R, cols] (engine.layout_rows;
    ldm_debug_read returns a layout's rows contiguously, so the 128-row view is regrouped, not reordered)"""
    return _debug_read(engine, name, n_layouts, raw).reshape(n_layouts, engine.layout_rows, -1)
