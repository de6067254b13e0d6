"""GPU (-m gpu): noise="torch" -- the draws are the numbers torch's CUDA generator gives the reference's `sample`
(helpers/sampling.py:81-130), and every call leaves the generator where the reference would.

  1. torch's own exponential_ / rand against the numpy restatement (oracle/torch_noise.py)
  2. the draw kernels against the reference's `sample` on the same log-probs and generator state
  3. ldm_sample_loop_noise against serialized ldm_step_noise calls, graph on and off, and a sharded batch against the whole
  4. the patched reference model against the unmodified reference model on the same GPU, same torch.manual_seed"""
import copy

import numpy as np
import pytest
import torch

from fixtures import Fixture
from oracle import layoutdm_oracle as O
from oracle import ref_harness as rh
from oracle import torch_noise as TN

pytestmark = pytest.mark.gpu

needs_ref = pytest.mark.skipif(not rh.reference_available(), reason="reference archive missing: run python oracle/make_ref.py")


def gen():
    return torch.cuda.default_generators[torch.cuda.current_device()]


def device_policy():
    p = torch.cuda.get_device_properties(torch.cuda.current_device())
    return p.multi_processor_count, p.max_threads_per_multi_processor


# ---- 1. the stream --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", [155, 135])
@pytest.mark.parametrize("B", [1, 7, 301, 1024])
def test_torch_stream_matches_restatement_and_kernel(B, C):
    S, n = 125, B * 125 * C
    n_sm, mt = device_policy()
    torch.cuda.manual_seed(1000 + B)
    gen().set_offset(4 * 37)
    seed, off = gen().initial_seed(), gen().get_offset()
    e = torch.empty(n, device="cuda").exponential_()
    d = TN.delta(n, n_sm, mt)
    assert gen().get_offset() == off + d
    u = torch.rand(n, device="cuda")
    assert gen().get_offset() == off + 2 * d
    np.testing.assert_array_equal(u.cpu().numpy(), TN.rand(TN.words(seed, off + d, n, n_sm, mt)))
    # the uniforms are bit for bit; torch's exponential_ takes the fast __logf, which the restatement's correctly rounded log
    # matches to __logf's accuracy (the kernels call the same __logf: they are tied bit for bit through the draw test below)
    e_t, e_o = e.cpu().numpy().astype(np.float64), TN.exponential(TN.words(seed, off, n, n_sm, mt)).astype(np.float64)
    err = np.abs(e_t - e_o) / (2.0 ** -21 * (1.0 + e_o))
    print(f"B={B} C={C}: tthr={TN.tthr(n, n_sm, mt)} delta={d}; exponentials bit-equal to the correctly rounded log: "
          f"{float((e_t == e_o).mean()):.4f}, worst error {float(err.max()):.3f} x 2^-21 (1 + e)")
    assert err.max() <= 1.0
    # the device code of the draw kernels (TorchNoise through ldm_debug_torch_noise) gives torch's values bit for bit
    eng = fused_torch().engine
    from layoutdm_b200 import _lib
    for which, want, at in ((1, e, off), (0, u, off + d)):
        got = torch.empty(n, device="cuda")
        _lib.check(eng.lib.ldm_debug_torch_noise(eng._h, n, seed, at, which, got.data_ptr(), eng._stream()))
        assert torch.equal(got, want), ("exponential_" if which else "rand", int((got != want).sum()))


# ---- 2. the draw against the reference's sample() ------------------------------------------------------------------------
def engine_for(fx, dtype="fp16"):
    from layoutdm_b200 import Engine, Vocab
    return Engine.from_state_dict(fx.weights(), Vocab.for_dataset(fx.meta["dataset"]), num_timesteps=fx.meta["T"], q_type=fx.meta["q_type"],
                                  operand_dtype=dtype)


_ENG = {}


def fused_torch(name="rico25_uncond_random"):
    from layoutdm_b200 import FusedMaskAndReplaceDiffusion
    if name not in _ENG:
        _ENG[name] = engine_for(Fixture(name))
    return FusedMaskAndReplaceDiffusion(_ENG[name], noise="torch")


@needs_ref
@pytest.mark.parametrize("B", [1, 8])
@pytest.mark.parametrize("temperature", [1.0, 0.7])
@pytest.mark.parametrize("name", ["random", "top_p", "top_k", "gumbel"])
def test_draw_matches_reference_sample(name, temperature, B, monkeypatch):
    """B = 1 is its own case: the reference's (B S, C) probabilities are then a strided view (TorchDraw::exp_cs)"""
    fx = Fixture("rico25_uncond_random")
    C, S = fx.vocab.C, fx.vocab.S
    lp = torch.cat([fx.logp(i) for i in (1, 99)] * 4)[:B]  # the reference's own log-probs (B, S, C); each copy draws its own noise
    lp = lp if lp.shape[-1] == C else lp.permute(0, 2, 1)
    logits = lp.permute(0, 2, 1).contiguous().cuda()                  # (B, C, S) like model_log_prob
    rh._setup_path()
    from trainer.helpers.sampling import sample as ref_sample
    cfg = rh.sampling_cfg(name, temperature=temperature)
    torch.cuda.manual_seed(77)
    gen().set_offset(4 * 11)
    state = gen().get_state()
    seen = {}
    real = torch.multinomial

    def spy(probs, num_samples, *a, **k):
        seen["probs"] = probs.clone()
        return real(probs, num_samples, *a, **k)
    monkeypatch.setattr(torch, "multinomial", spy)
    want = ref_sample(logits, cfg)[:, 0].cpu()
    monkeypatch.setattr(torch, "multinomial", real)
    off_ref = gen().get_offset()
    gen().set_state(state)
    got = fused_torch().sample_logits(logits, cfg)[:, 0].cpu()
    assert gen().get_offset() == off_ref
    # the reference's Exp(1) variates, replayed from the same state
    gen().set_state(state)
    if name == "gumbel":
        torch.rand_like(logits)
    e = torch.empty_like(seen["probs"]).exponential_()
    score = (seen["probs"].double() / e.double()).reshape(B, S, C).cpu()
    top2 = score.topk(2, dim=-1)
    bad = (got != want).nonzero().tolist()
    for b, s in bad:
        s1, s2 = top2.values[b, s].tolist()
        near = top2.indices[b, s, 1].item() == got[b, s].item() and (s1 - s2) <= 1e-6 * s1
        assert near, f"token ({b}, {s}): {int(got[b, s])} vs the reference's {int(want[b, s])}, best p/e {s1:.9g} / {s2:.9g}"
    print(f"{name} T={temperature}: {len(bad)} of {B * S} tokens differ, all at fp32 near-ties")


# ---- 3. the loop against serialized steps ---------------------------------------------------------------------------------
@pytest.mark.parametrize("graph", [True, False])
def test_loop_equals_steps(graph, monkeypatch):
    from layoutdm_b200 import timestep_plan
    from layoutdm_b200._lib import LdmNoise, NOISE_KINDS
    if not graph:
        monkeypatch.setenv("LDM_GRAPH", "0")
    fx = Fixture("rico25_uncond_random")
    eng = engine_for(fx)
    plan = timestep_plan(fx.meta["T"], 6)
    torch_kind = NOISE_KINDS["torch"]
    seed = 0x5EED_0123_4567
    for B in (1, 301):                                                # the second batch grows the workspace (a new capture)
        for cfg in ({"name": "random", "temperature": 1.0}, {"name": "gumbel", "temperature": 0.8}, {"name": "top_p", "top_p": 0.9}):
            adv = eng.noise_advance(B, cfg, 1)
            assert eng.noise_advance(B, cfg, len(plan)) == adv * len(plan)
            for offset in (0, 4 * 1234):                              # a replay with a new offset
                loop = eng.sample_loop(B, plan, cfg, noise=LdmNoise(torch_kind, seed, offset, B)).cpu()
                ids = torch.full((B, fx.vocab.S), fx.vocab.mask_id, dtype=torch.long, device="cuda")
                for k, (tm, tp) in enumerate(plan):
                    ids = eng.step(ids, tm, tp, cfg, noise=LdmNoise(torch_kind, seed, offset + k * adv, B))[0]
                assert torch.equal(loop, ids.cpu()), (B, cfg, offset)
                if B > 1:                                             # two shards of the same batch
                    h = B // 2
                    lo = eng.sample_loop(h, plan, cfg, noise=LdmNoise(torch_kind, seed, offset, B)).cpu()
                    hi = eng.sample_loop(B - h, plan, cfg, b_global0=h, noise=LdmNoise(torch_kind, seed, offset, B)).cpu()
                    assert torch.equal(torch.cat([lo, hi]), loop), (cfg, offset)
    assert eng.noise_advance(301, {"name": "deterministic"}, 10) == 0


def test_torch_mode_generator_bookkeeping():
    fused = fused_torch()
    g = gen()
    torch.cuda.manual_seed(3)
    off = g.get_offset()
    fused.sample(batch_size=4, sampling_cfg={"name": "deterministic", "num_timesteps": 5})
    assert g.get_offset() == off                                      # deterministic draws nothing
    cfg = {"name": "gumbel", "temperature": 1.0, "num_timesteps": 5}
    fused.sample(batch_size=4, sampling_cfg=cfg)
    assert g.get_offset() == off + fused.engine.noise_advance(4, cfg, 5)
    with pytest.raises(ValueError):
        fused.sample(batch_size=4, sampling_cfg=cfg, seed=1)
    off = g.get_offset()
    with pytest.raises(AssertionError):                               # refused by the library: the generator stays put
        fused.sample(batch_size=4, sampling_cfg={"name": "top_k", "top_k": 1000, "num_timesteps": 5})
    assert g.get_offset() == off
    # a sharded call advances the generator as for the whole batch and draws its slice of it
    torch.cuda.manual_seed(9)
    whole = fused.sample(batch_size=6, sampling_cfg=cfg)
    torch.cuda.manual_seed(9)
    part = fused.sample(batch_size=3, sampling_cfg=cfg, b_global0=3, total_layouts=6)
    assert g.get_offset() == fused.engine.noise_advance(6, cfg, 5) and torch.equal(part, whole[3:])


# ---- 4. against the unmodified reference on the same GPU -------------------------------------------------------------------
def reference_pair(fx, dtype):
    from layoutdm_b200 import patch_reference_model
    args = dict(T=fx.meta["T"], q_type=fx.meta["q_type"], state_dict=fx.weights())
    ref, tok = rh.build_reference(fx.meta["dataset"], **args)
    pat, _ = rh.build_reference(fx.meta["dataset"], **args)
    return ref.cuda(), patch_reference_model(pat, operand_dtype=dtype, noise="torch"), tok


def ref_cfg(fx, **kw):
    kw.setdefault("num_timesteps", fx.meta["T_eval"])
    if fx.meta.get("refine"):
        kw.update(fx.meta["refine"])
    return rh.sampling_cfg(fx.meta["sampling"], **kw)


@needs_ref
@pytest.mark.parametrize("dtype,threshold", [("bf16x3", 0.999), ("fp16", 0.99)])
def test_patched_steps_match_reference_on_its_own_states(dtype, threshold):
    """every step fed the reference's own x_t and the generator state the reference had at that step"""
    fx = Fixture("rico25_uncond_random")
    ref, pat, _ = reference_pair(fx, dtype)
    core = pat.model.module
    B, T = 64, fx.meta["T"]
    cfg = ref_cfg(fx, num_timesteps=T)
    from layoutdm_b200 import timestep_plan
    plan = timestep_plan(T, T)
    adv = core._ldm_b200.engine.noise_advance(B, cfg, 1)
    same = tot = 0
    for s in (0, 1):
        torch.manual_seed(s)
        traj = ref.model.sample(batch_size=B, sampling_cfg=cfg, get_intermediate_results=True)
        assert gen().get_offset() == adv * len(plan)
        x = torch.full((B, fx.vocab.S), fx.vocab.mask_id, dtype=torch.long)
        for i, (t_model, _) in enumerate(plan):
            skip = (plan[i - 1][0] - t_model - 1) if i else (T - t_model - 1)
            torch.manual_seed(s)
            gen().set_offset(i * adv)
            log_z = torch.log(torch.nn.functional.one_hot(x, fx.vocab.C).permute(0, 2, 1).float().clamp(min=1e-30)).cuda()
            out = core._sample_single_step(log_z=log_z, model_t=torch.full((B,), t_model, device="cuda"), skip_step=skip, sampling_cfg=cfg)
            assert gen().get_offset() == (i + 1) * adv
            same += int((out.argmax(1).cpu() == traj[i]).sum()); tot += traj[i].numel()
            x = traj[i]
    rate = same / tot
    print(f"{dtype}: tokens equal to the reference's on its own states: {rate:.6f} ({tot - same} of {tot} differ)")
    assert rate > threshold


@needs_ref
@pytest.mark.parametrize("single", [False, True], ids=["fixture_batch", "one_layout"])
@pytest.mark.parametrize("name", ["rico25_uncond_T50", "publaynet_c_top_p", "rico25_refinement_T200"])
def test_patched_model_leaves_generator_where_reference_does(name, single):
    """one_layout: batch_size=1, LayoutDM.sample's default, where the reference's multinomial draws into a strided view"""
    fx = Fixture(name)
    ref, pat, tok = reference_pair(fx, "bf16x3")
    B = 1 if single else fx.B
    cond = copy.deepcopy(fx.cond)
    if cond is not None:
        cond.pop("refine_table", None)
        cond = {k: (v[:B] if isinstance(v, torch.Tensor) else v) for k, v in cond.items()}
    kw = dict(cond_type=fx.meta["cond"]) if cond is not None else {}
    res = {}
    for label, model in (("reference", ref), ("patched", pat)):
        torch.manual_seed(21)
        out = model.sample(batch_size=B, cond=copy.deepcopy(cond), sampling_cfg=ref_cfg(fx), **kw)
        off1 = gen().get_offset()
        traj = model.model.sample(batch_size=B, cond=copy.deepcopy(cond), sampling_cfg=ref_cfg(fx), get_intermediate_results=True)
        off2 = gen().get_offset()
        res[label] = (out, off1, traj, off2)
    assert res["patched"][1] == res["reference"][1] and res["patched"][3] == res["reference"][3]
    same = [all(torch.equal(a[b], r[b]) for a, r in zip(res["patched"][2], res["reference"][2])) for b in range(B)]
    frac = sum(same) / B
    final = (res["patched"][2][-1] == res["reference"][2][-1]).float().mean().item()
    print(f"{name} B={B}: whole trajectories identical to the reference's: {frac:.3f}; final tokens equal {final:.4f}")
    assert frac > 0.5                                                 # one layout: its whole trajectory
    # one _sample_single_step advances the generator by one step, like the reference's
    core_p, core_r = pat.model.module, ref.model.module
    log_z = torch.log(torch.nn.functional.one_hot(fx.x_in[0][:B], fx.vocab.C).permute(0, 2, 1).float().clamp(min=1e-30)).cuda()
    t = torch.full((B,), fx.plan[0][0], device="cuda")
    offs = []
    for core in (core_r, core_p):
        torch.manual_seed(4)
        core._sample_single_step(log_z=log_z, model_t=t, skip_step=fx.meta["T"] - fx.plan[0][0] - 1, sampling_cfg=ref_cfg(fx))
        offs.append(gen().get_offset())
    assert offs[0] == offs[1]
