"""CPU: the tokenizer settings other than the default vocabulary (shared xywh bbox vocabulary, var_order c-w-h-x-y, any bin
count with C <= 160).

The oracle, given the slot layout of those settings (token_layout_refs.LayoutSpec), reproduces the fixtures the unmodified
reference recorded with them (tests/golden/token_layouts) token for token.  Against the live reference: the host vocabulary
(Vocab.slots, C, PAD / MASK, the partial vocabularies), decode_ids, the refinement table and the restated encode / get_cond.
Host logic: the C ABI's struct layout, the checkpoint / vocabulary check and the routing of cond=relation."""
import ctypes
import glob
import json
import os
import subprocess

import numpy as np
import pytest
import torch

import token_layout_refs as TL
from oracle import layoutdm_oracle as O
from oracle import ref_harness as rh

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(REPO, "tests", "golden", "token_layouts")
NAMES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN, "*.npz")))
needs_ref = pytest.mark.skipif(not rh.reference_available(), reason="reference not available")

# every tokenizer setting the reference offers (layout_tokenizer.py:16-20), at bin counts around the default
SETTINGS = [(ds, shared, order, bins) for ds in ("rico25", "publaynet") for shared in ("x-y-w-h", "xywh")
            for order in ("c-x-y-w-h", "c-w-h-x-y") for bins in (16, 32, 64)]


class TokenFixture:
    """a fixture of make_token_layout_golden.py: the fields of fixtures.Fixture, with the case's vocabulary"""

    def __init__(self, name):
        z = np.load(os.path.join(GOLDEN, name + ".npz"))
        m = self.meta = json.loads(str(z["meta"]))
        self.z = z
        self.vocab = TL.spec_of(m["config"])
        self.spec = O.ModelSpec(T=m["T"])
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
            if "cond_seq_orig" in z:
                self.cond["seq_orig"] = ld("cond_seq_orig")
                self.cond["refine_table"] = torch.from_numpy(z["refine_table"])

    def weights(self):
        sd = O.make_weights(self.vocab, self.spec, seed=self.meta["weight_seed"], scale=self.meta["weight_scale"])
        chk = O.weights_checksum(sd)
        assert abs(chk - self.meta["weights_checksum"]) <= 1e-6 * abs(chk), "synthetic weight generator drifted from the fixture"
        return sd

    def logits(self, i):
        return torch.from_numpy(self.z[f"logits_{i}"])

    def logp(self, i):
        return torch.from_numpy(self.z[f"logp_{i}"])

    def noise(self, i):
        u = O.uniforms(self.meta["noise_seed"], i, 0, 0, self.B, self.vocab.S, self.vocab.C) if self.meta["sampling"] != "deterministic" else None
        return u, None

    def host_vocab(self):
        from layoutdm_b200 import Vocab
        m = self.meta
        return Vocab.for_dataset(m["dataset"], 25, m["num_bin_bboxes"], m["shared_bbox_vocab"], m["var_order"])


def test_token_layout_fixtures_present():
    assert NAMES == ["publaynet_cwhxy_c_top_p", "rico25_bins16_refinement", "rico25_vanilla_xywh_cwhxy_uncond",
                     "rico25_xywh_bins64_cwh", "rico25_xywh_uncond_random"]
    assert sorted(TokenFixture(n).vocab.C for n in NAMES) == [43, 59, 91, 91, 135]


@pytest.mark.parametrize("name", NAMES)
def test_oracle_matches_reference_fixture(name):
    fx = TokenFixture(name)
    orc = O.Oracle(fx.vocab, fx.spec, fx.weights(), q_type=fx.meta["q_type"])
    with torch.no_grad():
        for i in range(len(fx.plan)):
            t_model, t_post = fx.plan[i]
            lp, logits = orc.step_logprob(fx.x_in[i], t_model, t_post, fx.cond)
            if i in fx.trace_steps:
                assert (logits - fx.logits(i)).abs().max() < 2e-5
                assert (lp - fx.logp(i)).abs().max() < 2e-4
            u, ug = fx.noise(i)
            assert torch.equal(O.draw(lp, fx.cfg, u, ug), fx.x_out[i]), f"{name}: step {i} ids differ from the reference"
    assert torch.equal(fx.x_out[-1], fx.ids_final)
    if fx.cond is not None:
        m = fx.cond["mask"]
        assert all(torch.equal(fx.x_out[i][m], fx.cond["seq"][m]) for i in range(len(fx.plan)))


@pytest.mark.parametrize("name", NAMES)
def test_host_vocab_and_refinement_table_of_fixture(name):
    from layoutdm_b200.vocab import linear_centers, refinement_table
    fx = TokenFixture(name)
    v = fx.host_vocab()
    assert (v.C, v.pad_id, v.mask_id, v.S) == (fx.vocab.C, fx.vocab.pad_id, fx.vocab.mask_id, fx.vocab.S)
    if fx.cond is not None and "refine_table" in fx.cond:
        r = fx.meta["refine"]
        tb = refinement_table(v, linear_centers(v.n_bins), r["refine_mode"], r["refine_offset_ratio"], r["refine_lambda"])
        assert torch.equal(tb, fx.cond["refine_table"])


# ---- against the live reference ------------------------------------------------------------------------------------------

_tokenizer = TL.tokenizer


def _spec(dataset, shared, order, bins):
    return TL.LayoutSpec(n_cat=(O.RICO25 if dataset == "rico25" else O.PUBLAYNET).n_cat, n_bins=bins, shared_bbox_vocab=shared,
                         var_order=order)


@needs_ref
@pytest.mark.parametrize("dataset,shared,order,bins", SETTINGS)
def test_vocab_from_tokenizer_matches_reference(dataset, shared, order, bins):
    from layoutdm_b200 import Vocab
    from layoutdm_b200.vocab import group_full_ids
    tok = _tokenizer(dataset, shared, order, bins)
    from trainer.helpers.layout_tokenizer import Converter
    v = Vocab.from_tokenizer(tok)
    assert v == Vocab.for_dataset(dataset, 25, bins, shared, order)
    assert (v.C, v.pad_id, v.mask_id, v.S) == (tok.N_total, tok.name_to_id("pad"), tok.name_to_id("mask"), tok.max_token_length)
    assert [name for name, _ in v.slots()] == tok.var_names
    for name, sl in v.slots():
        assert sl == tok.get_slice(name)
    conv = Converter(tok)
    for g, name in enumerate(tok.var_names):
        assert group_full_ids(v, g) == conv.mapping[name]["full"].tolist()
    vs = _spec(dataset, shared, order, bins)
    assert [vs.group_full_ids(g) for g in range(5)] == [group_full_ids(v, g) for g in range(5)]
    assert (vs.C, vs.pad_id) == (v.C, v.pad_id)


@needs_ref
def test_vocab_from_tokenizer_refuses_other_special_tokens():
    from layoutdm_b200 import Vocab
    tok = _tokenizer("rico25", "xywh", "c-x-y-w-h", 32)
    tok._data_cfg.special_tokens = ["pad", "bos", "eos", "mask"]
    with pytest.raises(NotImplementedError, match="special tokens"):
        Vocab.from_tokenizer(tok)


@needs_ref
@pytest.mark.parametrize("dataset,shared,order,bins", SETTINGS)
def test_decode_ids_matches_tokenizer_decode(dataset, shared, order, bins):
    from layoutdm_b200 import Vocab
    from layoutdm_b200.vocab import decode_ids
    tok = _tokenizer(dataset, shared, order, bins)
    v = Vocab.from_tokenizer(tok)
    g = torch.Generator().manual_seed(bins)
    ids = torch.randint(0, v.C, (32, v.S), generator=g)
    # mostly valid elements: every slot from its own variable's ids, some from another variable's or a special id
    for k, (name, sl) in enumerate(v.slots()):
        own = torch.randint(sl.start, sl.stop, (32, v.n_elem), generator=g)
        ids[:, k::5] = torch.where(torch.rand(32, v.n_elem, generator=g) < 0.85, own, ids[:, k::5])
    ref = tok.decode(ids)
    for out in (decode_ids(ids, v), TL.decode_ids(ids, _spec(dataset, shared, order, bins))):
        for k in ("label", "mask"):
            assert torch.equal(out[k], ref[k])
        assert torch.equal(out["bbox"], ref["bbox"].float())
    assert bool(ref["mask"].any()) and not bool(ref["mask"].all())


@needs_ref
@pytest.mark.parametrize("dataset,shared,order,bins", [s for s in SETTINGS if s[0] == "rico25"])
@pytest.mark.parametrize("mode", ["uniform", "gaussian", "negative"])
def test_refinement_table_matches_reference(dataset, shared, order, bins, mode):
    from layoutdm_b200 import Vocab
    from layoutdm_b200.vocab import linear_centers, refinement_table
    tok = _tokenizer(dataset, shared, order, bins)
    from trainer.helpers.task import _index_to_smoothed_log_onehot
    v = Vocab.from_tokenizer(tok)
    ref = _index_to_smoothed_log_onehot(torch.arange(v.C)[None], tok, mode=mode, offset_ratio=0.15)[0].t() * (-3.0 if mode == "negative" else 3.0)
    assert torch.equal(refinement_table(v, linear_centers(bins), mode, 0.15, 3.0), ref)
    assert torch.equal(TL.refinement_table(_spec(dataset, shared, order, bins), O.linear_centers(bins), mode, 0.15, 3.0), ref)
    if shared == "xywh":          # the four variables share one block: the last one written (h) is what stays
        h = linear_centers(bins)[3]
        blk = ref[v.n_cat:v.n_cat + bins, v.n_cat:v.n_cat + bins] / (-3.0 if mode == "negative" else 3.0)
        hh = torch.from_numpy(h)
        if mode == "uniform":
            assert torch.equal(blk, (torch.abs(hh[:, None] - hh[None]) < 0.15).float())


@needs_ref
@pytest.mark.parametrize("dataset,shared,order,bins", [s for s in SETTINGS if s[3] != 64 or s[1] == "xywh"])
@pytest.mark.parametrize("cond_type", ["c", "cwh", "refinement", "gt"])
def test_restated_get_cond_matches_reference(dataset, shared, order, bins, cond_type):
    tok = _tokenizer(dataset, shared, order, bins)
    from trainer.data.util import sparse_to_dense
    from trainer.helpers.task import get_cond
    vs = _spec(dataset, shared, order, bins)
    batch = rh.synthetic_layouts(6, vs.n_cat, seed=bins)
    torch.manual_seed(5)
    ref = get_cond(batch, tok, cond_type, model_type="LayoutDM")
    bbox, label, _, mask = sparse_to_dense(batch)
    if cond_type == "refinement":                     # the same draw as task.py:127, on the same (B, max elements, 4) boxes
        torch.manual_seed(5)
        bbox = bbox + torch.normal(0, std=0.1, size=bbox.size())
    pad = vs.n_elem - label.shape[1]
    label = torch.nn.functional.pad(label, (0, pad))
    bbox = torch.nn.functional.pad(bbox, (0, 0, 0, pad))
    mask = torch.nn.functional.pad(mask, (0, pad))
    out = TL.make_cond(label, bbox, mask, vs, cond_type)
    assert torch.equal(out["seq"], ref["seq"]) and torch.equal(out["mask"], ref["mask"])
    if cond_type == "refinement":
        assert torch.equal(out["seq_orig"], ref["seq_orig"])


# ---- host logic ----------------------------------------------------------------------------------------------------------

def test_vocab_layouts_and_bounds():
    from layoutdm_b200 import Vocab
    assert Vocab() == Vocab.for_dataset("rico25") and Vocab().C == 155
    v = Vocab(shared_bbox_vocab="xywh", var_order="c-w-h-x-y")
    assert v.C == 25 + 32 + 2 and [(n, sl.start) for n, sl in v.slots()] == [("c", 0), ("w", 25), ("h", 25), ("x", 25), ("y", 25)]
    v = Vocab(var_order="c-w-h-x-y")
    assert [(n, sl.start) for n, sl in v.slots()] == [("c", 0), ("w", 89), ("h", 121), ("x", 25), ("y", 57)]
    with pytest.raises(ValueError, match="shared_bbox_vocab"):
        Vocab(shared_bbox_vocab="xy-wh")
    with pytest.raises(ValueError, match="var_order"):
        Vocab(var_order="c-xw-yh")


def test_model_desc_offsets_match_header(tmp_path):
    from layoutdm_b200 import _lib
    names = [n for n, _ in _lib.LdmModelDesc._fields_]
    src = tmp_path / "off.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "ldm_b200.h"\nint main(){' +
                   "".join(f'printf("%zu\\n", offsetof(LdmModelDesc, {n}));' for n in names) +
                   'printf("%zu\\n", sizeof(LdmModelDesc));return 0;}\n')
    exe = tmp_path / "off"
    subprocess.check_call(["gcc", "-I", os.path.join(REPO, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got == [getattr(_lib.LdmModelDesc, n).offset for n in names] + [ctypes.sizeof(_lib.LdmModelDesc)]
    assert names[-2:] == ["bbox_vocab", "var_order"]
    assert _lib.BBOX_VOCABS == {"x-y-w-h": 0, "xywh": 1} and _lib.VAR_ORDERS == {"c-x-y-w-h": 0, "c-w-h-x-y": 1}


def test_checkpoint_of_other_vocabulary_is_refused():
    from layoutdm_b200 import LayoutDMB200
    from layoutdm_b200.engine import Engine
    sd = O.make_weights(O.RICO25, O.ModelSpec(layers=1), seed=0)                      # C = 155
    with pytest.raises(ValueError, match=r"155 rows.*C = 59"):
        LayoutDMB200.from_state_dict(sd, "rico25", shared_bbox_vocab="xywh")
    with pytest.raises(ValueError, match=r"155 rows.*C = 91"):
        LayoutDMB200.from_state_dict(sd, "rico25", num_bin_bboxes=16)
    vs = TL.spec_of("rico25_xywh")
    sd59 = O.make_weights(vs, O.ModelSpec(layers=1), seed=0)
    w = Engine.pack_state_dict(sd59, LayoutDMB200.vocab_for(sd59, "rico25", shared_bbox_vocab="xywh"))
    assert w["cat_emb"].shape == (59, 464) and w["head_w"].shape == (59, 464)


class _StubEngine:
    def __init__(self, vocab):
        self.vocab, self.T, self.device = vocab, 100, torch.device("cpu")


def _relation_cond(v):
    from oracle.ref_harness import FakeBatch
    batch = FakeBatch(torch.rand(3, 4), torch.zeros(3, dtype=torch.long), torch.zeros(3, dtype=torch.long))
    batch.edge_index = torch.tensor([[0, 1], [1, 2]])
    batch.edge_attr = torch.tensor([1, 2])
    return dict(type="relation", seq=torch.full((1, v.S), v.mask_id), mask=torch.zeros(1, v.S, dtype=torch.bool), batch_w_canvas=batch)


@pytest.mark.parametrize("shared,order,bins,on_device", [("xywh", "c-x-y-w-h", 32, True), ("xywh", "c-x-y-w-h", 16, True),
                                                         ("x-y-w-h", "c-x-y-w-h", 16, True), ("xywh", "c-w-h-x-y", 32, False),
                                                         ("x-y-w-h", "c-w-h-x-y", 32, False), ("xywh", "c-x-y-w-h", 64, False)])
def test_relation_routing_by_vocabulary(shared, order, bins, on_device):
    """the device update reads slot 1+a as variable a with a lane per bin: c-x-y-w-h with <= 32 bins, shared or not, gets the
    edge table; otherwise the step takes the log-prob hook (the reference's own update), and without a hook sampling refuses"""
    from layoutdm_b200 import Vocab
    from layoutdm_b200.diffusion import FusedMaskAndReplaceDiffusion
    v = Vocab.for_dataset("rico25", 25, bins, shared, order)
    scfg = {"relation_mode": "average", "relation_lambda": 1e6}
    fused = FusedMaskAndReplaceDiffusion(_StubEngine(v))
    if on_device:
        out = fused._prepare_cond(_relation_cond(v), 1, scfg)
        assert out["rel_adj"].shape == (1, 26, 26) and out["rel_centers"].shape == (4, bins)
        return
    with pytest.raises(NotImplementedError, match="patch_reference_model"):
        fused._prepare_cond(_relation_cond(v), 1, scfg)
    fused.logit_adjust_fn = lambda t, cond, lp, cfg: lp
    out = fused._prepare_cond(_relation_cond(v), 1, scfg)
    assert "rel_adj" not in out
    # relation_mode "gumbel" and lambda 0 never take the device update: unchanged, no refusal
    FusedMaskAndReplaceDiffusion(_StubEngine(v))._prepare_cond(_relation_cond(v), 1, {"relation_mode": "gumbel", "relation_lambda": 1e6})
