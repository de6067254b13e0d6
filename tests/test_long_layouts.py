"""CPU: layouts of more than 25 elements (dataset.max_seq_length up to 51, S = 5 n_elem <= 256 tokens).

The oracle reproduces the fixtures the unmodified reference recorded at max_seq_length = 50 (tests/golden/long_layouts), token
for token; the host logic (vocabulary, timestep plans, the layout length read from a state_dict, synthetic conditions and the
routing of cond=relation past the on-device update's 31 elements) covers n_elem up to 51."""
import dataclasses
import glob
import json
import os

import numpy as np
import pytest
import torch

from oracle import layoutdm_oracle as O

LONG = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "long_layouts")
LONG_NAMES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(LONG, "*.npz")))


class LongFixture:
    """a fixture of make_long_golden.py: the fields of fixtures.Fixture, at the recorded n_elem"""

    def __init__(self, name):
        z = np.load(os.path.join(LONG, name + ".npz"))
        m = self.meta = json.loads(str(z["meta"]))
        self.z = z
        self.vocab = dataclasses.replace(O.RICO25 if m["dataset"] == "rico25" else O.PUBLAYNET, n_elem=m["n_elem"])
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


def test_long_fixtures_present():
    assert LONG_NAMES == ["publaynet_L50_c_top_p", "rico25_L50_refinement", "rico25_L50_uncond_random"]


@pytest.mark.parametrize("name", LONG_NAMES)
def test_oracle_matches_reference_fixture_at_50_elements(name):
    fx = LongFixture(name)
    assert fx.vocab.S == 250 and fx.x_in.shape == (len(fx.plan), fx.B, 250)
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


@pytest.mark.parametrize("n_elem", [25, 26, 31, 32, 50, 51])
def test_vocab_and_plans_at_any_layout_length(n_elem):
    from layoutdm_b200 import Vocab, timestep_plan
    v = Vocab.for_dataset("rico25", max_seq_length=n_elem)
    assert (v.n_elem, v.S, v.C) == (n_elem, 5 * n_elem, 155)
    assert Vocab.for_dataset("publaynet", n_elem).C == 135
    assert Vocab.for_dataset("rico25") == Vocab()                        # the default stays 25 elements
    assert timestep_plan(100, 20) == O.timestep_plan(100, 20)


def _sd(n_elem, pos_emb="elem_attr"):
    vo = dataclasses.replace(O.RICO25, n_elem=n_elem)
    return O.make_weights(vo, O.ModelSpec(layers=1, pos_emb=pos_emb), seed=1)


@pytest.mark.parametrize("n_elem", [25, 26, 50, 51])
@pytest.mark.parametrize("pos_emb", ["elem_attr", "default"])
def test_layout_length_from_positional_table(n_elem, pos_emb):
    from layoutdm_b200 import LayoutDMB200, Vocab
    from layoutdm_b200.engine import Engine, layout_length
    sd = _sd(n_elem, pos_emb)
    assert layout_length(sd) == n_elem
    v = LayoutDMB200.vocab_for(sd, "rico25")
    assert v == Vocab.for_dataset("rico25", n_elem)
    assert LayoutDMB200.vocab_for(sd, "rico25", max_seq_length=n_elem) == v
    with pytest.raises(ValueError, match="positional table"):
        LayoutDMB200.vocab_for(sd, "rico25", max_seq_length=n_elem + 1)
    w = Engine.pack_state_dict(sd, v)
    assert w["pos_table"].shape == (5 * n_elem, 464)
    vo = dataclasses.replace(O.RICO25, n_elem=n_elem)
    assert torch.equal(w["pos_table"], O.positional_table(sd, vo, O.ModelSpec(layers=1, pos_emb=pos_emb)))


def test_packing_refuses_a_positional_table_of_another_length():
    from layoutdm_b200 import Vocab
    from layoutdm_b200.engine import Engine
    with pytest.raises(ValueError, match="max_seq_length"):
        Engine.pack_state_dict(_sd(25), Vocab.for_dataset("rico25", 50))


@pytest.mark.parametrize("n_elem", [26, 50, 51])
def test_synthetic_cond_spans_the_layout_length(n_elem):
    from layoutdm_b200 import Vocab
    from layoutdm_b200.synthetic import synthetic_cond
    v = Vocab.for_dataset("publaynet", n_elem)
    c = synthetic_cond(v, 512, "c", seed=2)
    assert c["seq"].shape == (512, v.S)
    assert int(c["num_element"].min()) == 1 and int(c["num_element"].max()) == n_elem
    n_real = ((c["seq"][:, ::5] != v.pad_id)).sum(1)
    assert torch.equal(n_real, c["num_element"])


class _StubEngine:
    def __init__(self, vocab):
        self.vocab, self.T, self.device = vocab, 100, torch.device("cpu")


@pytest.mark.parametrize("n_elem,on_device", [(25, True), (31, True), (32, False), (50, False), (51, False)])
def test_relation_routing_by_layout_length(n_elem, on_device):
    """cond=relation builds the on-device update's edge table only up to 31 elements; past that the step takes the
    log-prob hook path (the reference's own update), as relation_mode "gumbel" does"""
    from layoutdm_b200 import Vocab
    from layoutdm_b200.diffusion import FusedMaskAndReplaceDiffusion
    from oracle.ref_harness import FakeBatch
    v = Vocab.for_dataset("rico25", n_elem)
    fused = FusedMaskAndReplaceDiffusion(_StubEngine(v))
    batch = FakeBatch(torch.rand(3, 4), torch.zeros(3, dtype=torch.long), torch.zeros(3, dtype=torch.long))
    batch.edge_index = torch.tensor([[0, 1], [1, 2]])
    batch.edge_attr = torch.tensor([1, 2])
    cond = dict(type="relation", seq=torch.full((1, v.S), v.mask_id), mask=torch.zeros(1, v.S, dtype=torch.bool), batch_w_canvas=batch)
    out = fused._prepare_cond(cond, 1, {"relation_mode": "average", "relation_lambda": 1e6})
    assert ("rel_adj" in out) == on_device
    if on_device:
        assert out["rel_adj"].shape == (1, n_elem + 1, n_elem + 1)
