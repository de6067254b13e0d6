"""GPU (-m gpu): models trained with the reference's other tokenizer settings: a shared xywh bbox vocabulary, var_order
c-w-h-x-y, 16 or 64 bins (C from 43 to 135; the fixtures of tests/golden/token_layouts).

Checked for each fixture configuration: logits against the fp32 oracle; the step epilogue id-exact on the reference's own
logits (all-classes and, where it applies, group kernel); ldm_decode / ldm_make_cond against the reference tokenizer (linear
bins) and against the restatement of token_layout_refs (explicit centre tables); a live reference model patched by
patch_reference_model.  The loop equals serialized steps under every schedule switch for one small-C and one reordered
configuration; the group kernel equals the all-classes kernel bit for bit on designed near ties with shared group tables; a
vocabulary of C = 161 is refused; on a shared vocabulary the device relation update matches the reference's own `update` on the
same log-probs, and end to end the hook path that runs it."""
import copy
import dataclasses
import functools

import pytest
import torch

import test_gpu_epilogue_paths as EP
import test_gpu_loop_schedule as LS
import token_layout_refs as TL
from oracle import layoutdm_oracle as O
from oracle import ref_harness as rh
from test_token_layouts import NAMES, TokenFixture

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(not rh.reference_available(), reason="reference archive missing: run python oracle/make_ref.py")
CONFIGS = sorted(TL.CONFIGS)


def vocab_of(config):
    from layoutdm_b200 import Vocab
    dataset, shared, order, bins, _ = TL.CONFIGS[config]
    return Vocab.for_dataset(dataset, 25, bins, shared, order)


def make_engine(sd, config, dtype="fp16", T=100):
    from layoutdm_b200 import Engine
    torch.cuda.empty_cache()
    return Engine.from_state_dict(sd, vocab_of(config), num_timesteps=T, operand_dtype=dtype, q_type=TL.CONFIGS[config][4])


def layout_ids(B, vs, seed):
    """ids with every slot drawn from its own variable's ids, a few MASK tokens and a few PAD elements"""
    g = torch.Generator().manual_seed(seed)
    ids = torch.empty(B, vs.S, dtype=torch.long)
    for k, (_, lo, n) in enumerate(vs.slots()):
        ids[:, k::5] = torch.randint(lo, lo + n, (B, vs.n_elem), generator=g)
    ids[torch.rand(B, vs.S, generator=g) < 0.2] = vs.mask_id
    ids[:, 5 * 20:] = vs.pad_id
    return ids


# ---- logits against the fp32 oracle ------------------------------------------------------------------------------------

@pytest.mark.parametrize("config", CONFIGS)
@pytest.mark.parametrize("dtype,tol", [("fp16", 1e-3), ("bf16x3", 1e-4)])
def test_logits_vs_oracle(config, dtype, tol):
    vs, spec = TL.spec_of(config), O.ModelSpec()
    sd = O.make_weights(vs, spec, seed=5, scale=1.0)
    eng = make_engine(sd, config, dtype)
    B = 6
    ids = layout_ids(B, vs, 9)
    for t in (0, 42, 99):
        _, lg, _ = eng.step(ids.cuda(), t, t, {"name": "deterministic"}, want_logits=True)
        with torch.no_grad():
            ref = O.denoiser_forward(sd, ids, t, vs, spec)
        err = (lg.cpu() - ref).abs().max().item()
        print(f"{config} {dtype} t={t}: C={vs.C} logits max |d| vs the fp32 oracle {err:.2e}")
        assert lg.shape == (B, vs.S, vs.C) and err < tol


# ---- the step epilogue on the reference's logits -----------------------------------------------------------------------

@pytest.mark.parametrize("name", NAMES)
def test_step_epilogue_is_id_exact_on_reference_logits(name):
    """the reference's fp32 logits scattered into the padded logits rows: ids bit-exact with the log-prob tap (all-classes
    kernel) and without it (group kernel where it applies), log-probs within 1e-4"""
    fx = TokenFixture(name)
    eng = make_engine(fx.weights(), fx.meta["config"], T=fx.meta["T"])
    cond = None if fx.cond is None else {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in fx.cond.items()}
    for i in sorted(set(fx.trace_steps)):
        t_model, t_post = fx.plan[i]
        out, _, lp = eng.step(fx.x_in[i].cuda(), t_model, t_post, fx.cfg_dict, cond, seed=fx.meta["noise_seed"], step_ctr=i,
                              want_logprob=True, logits_in=fx.logits(i).cuda())
        assert (lp.cpu() - fx.logp(i)).abs().max() < 1e-4
        assert torch.equal(out.cpu(), fx.x_out[i]), f"{name} step {i}: {(out.cpu() != fx.x_out[i]).sum().item()} ids differ"
        out2, _, _ = eng.step(fx.x_in[i].cuda(), t_model, t_post, fx.cfg_dict, cond, seed=fx.meta["noise_seed"], step_ctr=i,
                              logits_in=fx.logits(i).cuda())
        assert torch.equal(out2.cpu(), fx.x_out[i]), f"{name} step {i} (group kernel)"


# ---- the loop against serialized steps -----------------------------------------------------------------------------------

@dataclasses.dataclass(frozen=True)
class LayoutWorkload(LS.Workload):
    config: str = "rico25_xywh"

    @property
    def vocab(self):
        return vocab_of(self.config)


def layout_state_dict(config):
    @functools.lru_cache(maxsize=2)
    def sd(dataset, T):
        from layoutdm_b200.synthetic import random_state_dict
        return random_state_dict(vocab_of(config), num_timesteps=T, seed=0)
    return sd


SMALL_C = LayoutWorkload("rico25 shared xywh 16 bins c-w-h-x-y (C=43) vanilla, B=64", "rico25", 100, 40, 64, LS.CFG_RANDOM,
                         config="rico25_vanilla_xywh_cwhxy")
SHARED = LayoutWorkload("rico25 shared xywh (C=59) cond=cwh, B=64", "rico25", 100, 40, 64, LS.CFG_RANDOM, cond_type="cwh",
                        config="rico25_xywh")
REORDERED = LayoutWorkload("publaynet c-w-h-x-y (C=135) cond=c top_p, B=33", "publaynet", 100, 30, 33,
                           (("name", "top_p"), ("temperature", 1.0), ("top_p", 0.9)), cond_type="c", config="publaynet_cwhxy")


@pytest.mark.parametrize("wl", [SMALL_C, SHARED, REORDERED], ids=["C43-vanilla", "C59-cwh", "C135-cwhxy"])
def test_loop_equals_serialized_steps_under_every_switch(monkeypatch, wl):
    monkeypatch.setattr(LS, "state_dict", layout_state_dict(wl.config))
    cond, ids_init = LS.inputs(wl)
    ks = LS.prefixes(len(wl.plan))
    ref = LS.serialized(monkeypatch, wl, "fp16", wl.seed, wl.b_global0, cond, ids_init, keep=[k - 1 for k in ks])
    failures = LS.compare_prefixes(monkeypatch, wl, "fp16", LS.MATRIX, ks, ref, cond, ids_init)
    assert not failures, "\n".join(failures)


# ---- decode / make_cond --------------------------------------------------------------------------------------------------

def synthetic_layouts(B, vs, seed):
    g = torch.Generator().manual_seed(seed)
    n = torch.randint(1, vs.n_elem + 1, (B,), generator=g)
    mask = torch.arange(vs.n_elem)[None] < n[:, None]
    label = torch.randint(0, vs.n_cat, (B, vs.n_elem), generator=g)
    bbox = torch.rand(B, vs.n_elem, 4, generator=g) * 1.2 - 0.1                 # some boxes outside [0, 1]: the clamps
    return label, bbox, mask


@needs_ref
@pytest.mark.parametrize("config", CONFIGS)
def test_decode_and_make_cond_match_reference_tokenizer(config):
    dataset, shared, order, bins, q_type = TL.CONFIGS[config]
    vs = TL.spec_of(config)
    _, tok = TL.build_config(config, num_layers=1)
    eng = make_engine(O.make_weights(vs, O.ModelSpec(layers=1), seed=0), config)
    # decode: ids with valid elements, out-of-variable slots and specials
    ids = layout_ids(64, vs, 4)
    ids[3, 6] = vs.var_start("x") + vs.n_bins - 1 if shared == "x-y-w-h" else vs.mask_id
    ref = tok.decode(ids)
    dec = eng.decode(ids.cuda())
    for k in ("label", "mask"):
        assert torch.equal(dec[k].cpu(), ref[k]), k
    assert torch.equal(dec["bbox"].cpu(), ref["bbox"].float())
    # make_cond: the reference's encode + get_cond slot selection (by variable name), linear bins
    label, bbox, mask = synthetic_layouts(64, vs, 5)
    enc = tok.encode({"label": label, "bbox": bbox, "mask": mask})["seq"]
    for cond_type in ("c", "cwh", "refinement", "gt"):
        c = eng.cond_from_layouts(label.cuda(), bbox.cuda(), mask.cuda(), cond_type)
        want = TL.make_cond(label, bbox, mask, vs, cond_type)
        assert torch.equal(c["seq"].cpu(), want["seq"]) and torch.equal(c["mask"].cpu(), want["mask"]), cond_type
        if cond_type == "gt":
            assert torch.equal(c["seq"].cpu(), enc)
        if cond_type == "refinement":
            assert torch.equal(c["seq_orig"].cpu(), enc)


@pytest.mark.parametrize("config", CONFIGS)
def test_decode_and_make_cond_with_centre_tables(config):
    """kmeans-like centres passed explicitly: ldm_decode / ldm_make_cond against the restatement of token_layout_refs"""
    vs = TL.spec_of(config)
    eng = make_engine(O.make_weights(vs, O.ModelSpec(layers=1), seed=0), config)
    g = torch.Generator().manual_seed(vs.n_bins)
    centers = torch.sort(torch.rand(4, vs.n_bins, generator=g), dim=1).values
    ids = layout_ids(64, vs, 6)
    dec = eng.decode(ids.cuda(), centers)
    want = TL.decode_ids(ids, vs, centers)
    for k in ("bbox", "label", "mask"):
        assert torch.equal(dec[k].cpu(), want[k]), k
    label, bbox, mask = synthetic_layouts(64, vs, 7)
    for cond_type in ("c", "cwh", "gt"):
        c = eng.cond_from_layouts(label.cuda(), bbox.cuda(), mask.cuda(), cond_type, centers=centers)
        w = TL.make_cond(label, bbox, mask, vs, cond_type, centers)
        assert torch.equal(c["seq"].cpu(), w["seq"]) and torch.equal(c["mask"].cpu(), w["mask"]), cond_type


# ---- bounds ----------------------------------------------------------------------------------------------------------------

def test_vocabulary_of_161_classes_is_refused():
    from layoutdm_b200 import Engine, Vocab, _lib
    from layoutdm_b200.synthetic import random_state_dict
    v = Vocab(n_cat=31, n_bins=32)                                           # C = 31 + 128 + 2 = 161
    assert v.C == 161
    with pytest.raises(_lib.LdmError, match="C=161: the kernels hold at most C = 160"):
        Engine.from_state_dict(random_state_dict(v, layers=1), v)
    v = Vocab(n_cat=30, n_bins=32)                                           # C = 160: the largest
    Engine.from_state_dict(random_state_dict(v, layers=1), v).close()


# ---- the group kernel on designed near ties, shared vocabularies ---------------------------------------------------------

@dataclasses.dataclass(frozen=True)
class LayoutVoc(EP.Voc):
    """test_gpu_epilogue_paths.Voc with the tokenizer settings: the four bbox groups share the ids from n_cat on"""
    shared: str = "xywh"
    order: str = "c-x-y-w-h"

    @property
    def vocab(self):
        from layoutdm_b200 import Vocab
        return Vocab.for_dataset(self.dataset, 25, self.n_bins, self.shared, self.order)

    @property
    def spec(self) -> O.VocabSpec:
        return TL.LayoutSpec(n_cat=self.vocab.n_cat, n_bins=self.n_bins, shared_bbox_vocab=self.shared, var_order=self.order)

    def __str__(self):
        return f"{self.dataset}/{self.n_bins} bins {self.shared} {self.order}"


@pytest.mark.parametrize("voc,mode,noise_kind", [(LayoutVoc("rico25", 32), "random", "contract"),
                                                 (LayoutVoc("rico25", 32), "gumbel", "torch"),
                                                 (LayoutVoc("rico25", 32, order="c-w-h-x-y"), "random", "contract"),
                                                 (LayoutVoc("rico25", 64), "random", "contract")], ids=str)
def test_near_ties_same_ids_on_both_paths(voc, mode, noise_kind):
    """test_gpu_epilogue_paths' designed near ties with the shared group tables: the group kernel's ids equal the all-classes
    kernel's bit for bit; groups of 64 shared bins never take the group routine.  (The helper requires designed ties on 90 % of
    the tokens, a reach its tie designer gets with groups of 25 classes or more.)"""
    assert EP.step_applies(voc, {"name": mode}) == (voc.n_bins <= 32)
    EP._near_ties(voc, mode, noise_kind, B=4)


# ---- the relation update on a shared vocabulary, against the reference's own update -------------------------------------

def _relation_setup(B, lam, n_update):
    """a live rico25 shared-xywh reference model, patched; a relation cond from get_cond and its sampling cfg"""
    import random
    from layoutdm_b200 import patch_reference_model
    from test_oracle_relation import make_relation_batch
    fx = TokenFixture("rico25_xywh_uncond_random")
    model, tok = TL.build_config(fx.meta["config"], T=fx.meta["T"], state_dict=fx.weights())
    model = patch_reference_model(model)
    from trainer.helpers.task import get_cond
    random.seed(0); torch.manual_seed(0)
    cond = get_cond(make_relation_batch(B, fx.vocab.n_cat, 21), tok, "relation", model_type="LayoutDM")
    cfg = rh.sampling_cfg("random", num_timesteps=25, relation_lambda=lam, relation_mode="average", relation_tau=1.0,
                          relation_num_update=n_update)
    return model, tok, cond, cfg


@needs_ref
@pytest.mark.parametrize("lam", [3e6, 1e4])
def test_relation_update_matches_reference_update_on_shared_vocabulary(lam):
    """one device update against `update` (logit_adjustment.py:88-126, with its shared `slices` and canvas ids) on the same
    log-probs: the posterior with PAD-disable off, as both paths feed the update; PAD-disable applied after, as base.py:271-284"""
    B, t = 6, 50
    model, tok, cond, cfg = _relation_setup(B, lam, 1)
    fused = model.model.module._ldm_b200
    eng = fused.engine
    cond_d = fused._prepare_cond(cond, B, cfg)
    assert "rel_adj" in cond_d, "a shared c-x-y-w-h vocabulary of 32 bins takes the device update"
    g = torch.Generator().manual_seed(4)
    logits = (torch.randn(B, eng.vocab.S, eng.vocab.C, generator=g) * 3.0).cuda()
    ids = cond_d["seq"]
    pre = {k: v for k, v in cond_d.items() if not k.startswith("rel_")}
    pre["_pad_disable"] = False
    _, _, lp0 = eng.step(ids, t, t, cfg, pre, seed=1, want_logprob=True, logits_in=logits)
    _, _, lp = eng.step(ids, t, t, cfg, cond_d, seed=1, want_logprob=True, logits_in=logits)
    from trainer.models.categorical_diffusion.logit_adjustment import update
    # update's Parameter shares the storage of the tensor it is given and steps it in place: hand it a copy of its own
    want = update(t=t, cond=cond, model_log_prob=lp0.cpu().permute(0, 2, 1).contiguous(), tokenizer=tok, sampling_cfg=cfg)
    want, lp0 = want.permute(0, 2, 1).contiguous(), lp0.cpu()
    v = eng.vocab
    pad_off = (torch.arange(v.S)[None] % v.n_attr != 0) & (cond["seq"] != v.pad_id)
    for x in (want, lp0):
        x[..., v.pad_id] = torch.where(pad_off, torch.full_like(x[..., 0], O.LOG_EPS), x[..., v.pad_id])
    moved = (want - lp0).abs().max().item()
    err = (lp.cpu() - want).abs().max().item()
    print(f"lambda={lam:g}: the reference's update moved log-probs by up to {moved:.3e}; |device - reference| {err:.3e}")
    assert moved > 1e-2, "inputs do not exercise the update"
    assert err <= 1e-4 + 1e-5 * moved                                          # test_gpu_relation.py's gate for one update


@needs_ref
def test_patched_shared_vocabulary_relation_device_vs_reference_update():
    """test_gpu_dropin's end-to-end check on a shared vocabulary: the device update (default) against the reference's own
    autograd `update` through the log-prob hook (relation_on_device = False), same noise key, at the same thresholds"""
    B = 6
    model, tok, cond, cfg = _relation_setup(B, 3e6, 3)
    fused = model.model.module._ldm_b200
    res = {}
    for on_device in (True, False):
        fused.relation_on_device = on_device
        res[on_device] = model.model.sample(batch_size=B, cond=copy.copy(cond), sampling_cfg=cfg, seed=77, get_intermediate_results=True)
    fused.relation_on_device = True
    first = (res[True][0] == res[False][0]).float().mean().item()
    final = (res[True][-1] == res[False][-1]).float().mean().item()
    print(f"shared vocabulary relation: device vs reference update: identical tokens after step 0 {first:.4f}, after the last {final:.4f}")
    assert first > 0.995 and final > 0.9
    m = cond["mask"]
    assert torch.equal(res[True][-1][m], cond["seq"][m])


# ---- a live reference model of each configuration, patched ---------------------------------------------------------------

@needs_ref
@pytest.mark.parametrize("name", NAMES)
def test_patched_reference_model(name):
    from layoutdm_b200 import patch_reference_model
    fx = TokenFixture(name)
    model, tok = TL.build_config(fx.meta["config"], T=fx.meta["T"], state_dict=fx.weights())
    model = patch_reference_model(model)
    assert model.model.module._ldm_b200.vocab.C == fx.vocab.C
    scfg = rh.sampling_cfg(fx.meta["sampling"], num_timesteps=fx.meta["T_eval"])
    res = model.model.sample(batch_size=fx.B, cond=copy.deepcopy(fx.cond), sampling_cfg=scfg, get_intermediate_results=True,
                             seed=fx.meta["noise_seed"])
    assert len(res) == len(fx.plan) and res[0].shape == (fx.B, fx.vocab.S)
    first = (res[0] == fx.x_out[0]).float().mean().item()
    print(f"{name}: identical tokens after step 0: {first:.4f}")
    assert first > 0.99
    if fx.cond is not None:
        m = fx.cond["mask"]
        assert torch.equal(res[-1][m], fx.cond["seq"][m])
    ids = model.model.sample(batch_size=fx.B, cond=copy.deepcopy(fx.cond), sampling_cfg=scfg, seed=7)
    out = model.sample(batch_size=fx.B, cond=copy.deepcopy(fx.cond), sampling_cfg=scfg, seed=7)
    want = tok.decode(ids)
    for k in ("bbox", "label", "mask"):
        assert torch.equal(out[k], want[k]), k


@needs_ref
def test_patched_vanilla_model_with_default_positional_embedding():
    from layoutdm_b200 import patch_reference_model
    model, tok = TL.build_config("rico25_vanilla_xywh_cwhxy", T=50, pos_emb="default", num_layers=2)
    model = patch_reference_model(model)
    out = model.sample(batch_size=3, cond=None, sampling_cfg=rh.sampling_cfg("random", num_timesteps=10), seed=3)
    assert out["bbox"].shape == (3, 25, 4) and bool(out["mask"].any())
