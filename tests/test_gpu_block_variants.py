"""GPU (-m gpu): denoiser blocks with the reference Block's other settings: instance-norm AdaIN (adainnorm*), sinusoidal or no
timestep embedding (*_abs, None), GELU feed-forwards (gelu, gelu2); the fixtures of tests/golden/blocks.

Checked: logits against the fp32 oracle (block_refs.block_forward) for all 15 configurations in fp16, and a subset in bf16 and
bf16x3; the instance norm also at 26 elements (126 pad rows per layout: any pad row in its statistics shows) and at 50.  The loop
equals serialized steps under every schedule switch for an instance-norm and a GELU handle.  The training-side entry points at
per-layout timesteps on an adainnorm model.  ldm_load_weights of a new adainnorm_abs / None checkpoint gives a fresh handle's
logits.  A live reference model of each fixture, patched."""
import contextlib
import copy
import dataclasses
import functools

import pytest
import torch

import block_refs as BR
import test_gpu_loop_schedule as LS
from oracle import layoutdm_oracle as O
from oracle import ref_harness as rh

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(not rh.reference_available(), reason="reference archive missing: run python oracle/make_ref.py")
BF16_TOL = 1e-2     # test_gpu_parity.py's rule: bf16 operands carry 8x coarser mantissas than fp16, 10x its 1e-3 gate


def specs(n_elem=25, dataset="rico25"):
    """(oracle vocabulary, host vocabulary) of the dataset at n_elem elements"""
    from layoutdm_b200 import Vocab
    return dataclasses.replace(O.RICO25 if dataset == "rico25" else O.PUBLAYNET, n_elem=n_elem), Vocab.for_dataset(dataset, n_elem)


def make_engine(sd, vocab, tt, act, dtype="fp16", T=100, **kw):
    from layoutdm_b200 import Engine
    torch.cuda.empty_cache()
    return Engine.from_state_dict(sd, vocab, num_timesteps=T, operand_dtype=dtype, timestep_type=tt, activation=act, **kw)


def mixed_ids(B, vs, seed):
    """ids with every slot drawn from its own group, some MASK tokens and the last elements PAD"""
    g = torch.Generator().manual_seed(seed)
    ids = torch.empty(B, vs.S, dtype=torch.long)
    for a in range(vs.n_attr):
        ids[:, a::vs.n_attr] = torch.randint(vs.group_start(a), vs.group_start(a) + vs.group_n(a), (B, vs.n_elem), generator=g)
    ids[torch.rand(B, vs.S, generator=g) < 0.2] = vs.mask_id
    ids[:, vs.n_attr * (vs.n_elem - 3):] = vs.pad_id
    return ids


# ---- logits against the fp32 oracle ------------------------------------------------------------------------------------------

FP16_CASES = [(tt, act, 25) for tt, act in BR.CONFIGS] + \
             [(tt, act, n) for tt, act in BR.CONFIGS if tt is not None and tt.startswith("adainnorm") for n in (26, 50)]
SUBSET = [("adainnorm", "gelu", 25), ("adainnorm_abs", "gelu2", 26), (None, "gelu", 25), ("adalayernorm_abs", "relu", 50)]
CASES = [c + ("fp16", 1e-3) for c in FP16_CASES] + [c + ("bf16", BF16_TOL) for c in SUBSET] + [c + ("bf16x3", 1e-4) for c in SUBSET]


@pytest.mark.parametrize("tt,act,n_elem,dtype,tol", CASES, ids=[f"{BR.config_id(c[0], c[1])}-E{c[2]}-{c[3]}" for c in CASES])
def test_logits_vs_oracle(tt, act, n_elem, dtype, tol):
    vs, vocab = specs(n_elem)
    spec = O.ModelSpec()
    sd = BR.block_weights(vs, spec, seed=5, scale=1.0, timestep_type=tt)
    eng = make_engine(sd, vocab, tt, act, dtype)
    B = 6
    ids = mixed_ids(B, vs, 9)
    for t in (0, 42, 99):
        _, lg, _ = eng.step(ids.cuda(), t, t, {"name": "deterministic"}, want_logits=True)
        with torch.no_grad():
            ref = BR.block_forward(sd, ids, t, vs, spec, tt, act)
        err = (lg.cpu() - ref).abs().max().item()
        print(f"{tt} {act} E={n_elem} {dtype} t={t}: logits max |d| vs the fp32 oracle {err:.2e}")
        assert lg.shape == (B, vs.S, vs.C) and err < tol
    eng.close()


# ---- the loop against serialized steps ---------------------------------------------------------------------------------------

@contextlib.contextmanager
def _handle(tt, act, monkeypatch, wl, dtype, env):
    """LS.handle with the block settings"""
    for k in LS.SWITCHES:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    eng = make_engine(LS.state_dict(wl.dataset, wl.T), wl.vocab, tt, act, dtype, T=wl.T)
    try:
        yield eng
    finally:
        torch.cuda.synchronize()
        eng.close()
        del eng
        torch.cuda.empty_cache()


INORM = LS.Workload("rico25 adainnorm_abs + gelu, B=64", "rico25", 100, 40, 64, LS.CFG_RANDOM)
GELU = LS.Workload("rico25 adalayernorm + gelu2, cond=c, B=64", "rico25", 100, 40, 64, LS.CFG_RANDOM, cond_type="c")


@pytest.mark.parametrize("tt,act,wl", [("adainnorm_abs", "gelu", INORM), ("adalayernorm", "gelu2", GELU)], ids=["inorm", "gelu2"])
def test_loop_equals_serialized_steps_under_every_switch(monkeypatch, tt, act, wl):
    """an instance-norm handle launches its own embedding every step and one more kernel per layer (norm1)"""
    from layoutdm_b200 import Vocab
    from layoutdm_b200.synthetic import random_state_dict
    inorm = tt.startswith("adainnorm")
    monkeypatch.setattr(LS, "state_dict", functools.lru_cache(maxsize=1)(
        lambda dataset, T: random_state_dict(Vocab.for_dataset(dataset), num_timesteps=T, seed=0, timestep_type=tt)))
    monkeypatch.setattr(LS, "handle", functools.partial(_handle, tt, act))
    if inorm:
        monkeypatch.setattr(LS, "LAUNCHES_PER_STEP", 1 + 6 * LS.LAYERS + 2)
        monkeypatch.setattr(LS, "fuses", lambda dtype, env: False)
    cond, ids_init = LS.inputs(wl)
    ks = LS.prefixes(len(wl.plan))
    ref = LS.serialized(monkeypatch, wl, "fp16", wl.seed, wl.b_global0, cond, ids_init, keep=[k - 1 for k in ks])
    failures = LS.compare_prefixes(monkeypatch, wl, "fp16", LS.MATRIX, ks, ref, cond, ids_init)
    assert not failures, "\n".join(failures)


# ---- the training-side entry points at per-layout timesteps ------------------------------------------------------------------

@pytest.mark.parametrize("n_elem", [25, 50])
def test_training_api_per_layout_timesteps_instance_norm(n_elem):
    vs, vocab = specs(n_elem)
    spec = O.ModelSpec()
    sd = BR.block_weights(vs, spec, seed=6, scale=1.0, timestep_type="adainnorm")
    eng = make_engine(sd, vocab, "adainnorm", "gelu")
    B, T = 18, spec.T
    scheds = O.group_schedules(T, vs)
    g = torch.Generator().manual_seed(2)
    x0 = torch.empty(B, vs.S, dtype=torch.long)
    for a in range(5):
        grp = torch.tensor(vs.group_full_ids(a)[:-2])
        x0[:, a::5] = grp[torch.randint(0, len(grp), (B, vs.n_elem), generator=g)]
    t = torch.randint(0, T, (B,), generator=g)
    t[0], t[1] = 0, T - 1
    xt = eng.q_sample(x0.cuda(), t.cuda(), seed=3).cpu()
    lx0, logits = eng.predict_start(xt.cuda(), t.cuda(), want_logits=True)
    lx0, logits = lx0.cpu(), logits.cpu()
    with torch.no_grad():
        ref = BR.block_forward(sd, xt, t, vs, spec, "adainnorm", "gelu")
    err = (logits - ref).abs().max().item()
    print(f"adainnorm + gelu, E={n_elem}, per-layout t: logits max |d| vs the fp32 oracle {err:.2e}")
    assert err < 1e-3
    assert (lx0 - O.predict_start(logits)).abs().max() < 1e-4
    r = eng.vb_terms(x0.cuda(), xt.cuda(), t.cuda(), (1.0, 1.0), want_log_model_prob=True)
    w = O.vb_terms(logits, x0, xt, t, T, vs, scheds)
    assert (r["log_model_prob"].cpu() - w["log_model_prob"]).abs().max() < 1e-4
    for k in ("kl", "decoder_nll", "kl_aux"):
        assert ((r[k].cpu() - w[k]).abs() <= 1e-4 * (1.0 + w[k].abs())).all(), k
    # one timestep for all layouts: the same logits as the sampling path
    tt = torch.full((B,), 42)
    _, lg_t = eng.predict_start(xt.cuda(), tt.cuda(), want_logits=True)
    _, lg_s, _ = eng.step(xt.cuda(), 42, 42, {"name": "deterministic"}, want_logits=True)
    assert torch.equal(lg_t, lg_s)
    eng.close()


# ---- weight reloads ----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("tt,act", [("adainnorm_abs", "gelu"), (None, "gelu2")], ids=str)
def test_load_weights_equals_fresh_handle(tt, act):
    """a handle built from checkpoint A, then given B by load_state_dict (packed on the device), computes what a handle built
    from B computes, bit for bit"""
    vs, vocab = specs(25)
    spec = O.ModelSpec()
    sd_a = BR.block_weights(vs, spec, seed=11, timestep_type=tt)
    sd_b = BR.block_weights(vs, spec, seed=12, timestep_type=tt)
    ids = mixed_ids(4, vs, 1).cuda()
    eng = make_engine(sd_a, vocab, tt, act)
    _, lg_a, _ = eng.step(ids, 30, 30, {"name": "deterministic"}, want_logits=True)
    eng.load_state_dict({k: v.cuda() for k, v in sd_b.items()})
    _, lg_reloaded, _ = eng.step(ids, 30, 30, {"name": "deterministic"}, want_logits=True)
    fresh = make_engine(sd_b, vocab, tt, act)
    _, lg_b, _ = fresh.step(ids, 30, 30, {"name": "deterministic"}, want_logits=True)
    assert not torch.equal(lg_a, lg_b)
    assert torch.equal(lg_reloaded, lg_b)
    eng.close()
    fresh.close()


# ---- a live reference model of each fixture, patched ------------------------------------------------------------------------

@needs_ref
@pytest.mark.parametrize("name", BR.NAMES)
def test_patched_reference_model(name):
    """test_gpu_token_layouts' thresholds: > 99 % of the tokens of step 0 as the reference drew them, the fixed tokens kept,
    `model.sample` decoding what `model.model.sample` drew"""
    from layoutdm_b200 import patch_reference_model
    fx = BR.BlockFixture(name)
    m = fx.meta
    model, tok = BR.build_reference(m["dataset"], T=m["T"], q_type=m["q_type"], state_dict=fx.weights(), timestep_type=fx.timestep_type,
                                    activation=fx.activation, diffusion_step=fx.diffusion_step, max_seq_length=m["n_elem"])
    model = patch_reference_model(model)
    eng = model.model.module._ldm_b200.engine
    assert (eng.timestep_type, eng.activation, eng.diffusion_step) == (fx.timestep_type, fx.activation, fx.diffusion_step)
    scfg = rh.sampling_cfg(m["sampling"], num_timesteps=m["T_eval"])
    res = model.model.sample(batch_size=fx.B, cond=copy.deepcopy(fx.cond), sampling_cfg=scfg, get_intermediate_results=True,
                             seed=m["noise_seed"])
    assert len(res) == len(fx.plan) and res[0].shape == (fx.B, fx.vocab.S)
    first = (res[0] == fx.x_out[0]).float().mean().item()
    print(f"{name}: identical tokens after step 0: {first:.4f}")
    assert first > 0.99
    if fx.cond is not None:
        mk = fx.cond["mask"]
        assert torch.equal(res[-1][mk], fx.cond["seq"][mk])
    ids = model.model.sample(batch_size=fx.B, cond=copy.deepcopy(fx.cond), sampling_cfg=scfg, seed=7)
    out = model.sample(batch_size=fx.B, cond=copy.deepcopy(fx.cond), sampling_cfg=scfg, seed=7)
    want = tok.decode(ids)
    for k in ("bbox", "label", "mask"):
        assert torch.equal(out[k], want[k]), k


@pytest.mark.parametrize("name", BR.NAMES)
def test_from_state_dict_samples_each_fixture(name):
    """LayoutDMB200.from_state_dict with the fixture's block settings, bf16x3: the device's logits on the reference's step inputs
    against the reference's own logits, within the bf16x3 gate (1e-4 at the reference's init scale) times the fixture's
    weight scale (2 or 3)"""
    from layoutdm_b200 import LayoutDMB200
    fx = BR.BlockFixture(name)
    m = fx.meta
    dm = LayoutDMB200.from_state_dict(fx.weights(), m["dataset"], num_timesteps=m["T"], q_type=m["q_type"], operand_dtype="bf16x3",
                                      timestep_type=fx.timestep_type, activation=fx.activation, diffusion_step=fx.diffusion_step)
    eng = dm.model.engine
    assert eng.vocab.S == fx.vocab.S
    for i in fx.trace_steps:
        tm, tp = fx.plan[i]
        _, lg, _ = eng.step(fx.x_in[i].cuda(), tm, tp, {"name": "deterministic"}, want_logits=True)
        err = (lg.cpu() - fx.logits(i)).abs().max().item()
        print(f"{name} step {i}: bf16x3 logits max |d| vs the reference's {err:.2e}")
        assert err < 1e-4 * m["weight_scale"]
    out = dm.sample(batch_size=3, sampling_cfg={"name": "random", "temperature": 1.0, "num_timesteps": 10}, seed=3)
    assert out["bbox"].shape == (3, fx.vocab.n_elem, 4)
