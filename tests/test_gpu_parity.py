"""GPU (-m gpu): the CUDA path against the golden fixtures recorded from the reference and against the oracle.
Everything goes through the C ABI (layoutdm_b200.Engine is a thin ctypes wrapper)."""
import numpy as np
import pytest
import torch

from fixtures import NAMES, Fixture
from oracle import layoutdm_oracle as O

pytestmark = pytest.mark.gpu

LOGIT_TOL = 1e-3     # north-star gate: max-abs on the fp32 logits vs the reference's fp32 logits, at the reference's own
                     # weight scale (base_model.py:108-116, std 0.02).  For the x2 / x3 "peaked" stress weights of the
                     # fixtures the gate is applied relative to the logit scale: STRESS_REL * max|logit| (measured 0.6e-3 at
                     # x2, 1.2e-3 at x3: the fp16 operand rounding error grows with the weight scale; DESIGN.md "Precision").
STRESS_REL = 2e-3
BF16_FACTOR = 10.0   # bf16 operands (the north star's nominal dtype) carry 8x coarser mantissas; measured ~8x the fp16 error

_engines = {}


def engine_for(fx, dtype="fp16"):
    from layoutdm_b200 import Engine, Vocab
    key = (fx.meta["dataset"], fx.meta["T"], fx.meta["q_type"], fx.meta["weight_scale"], dtype)
    if key not in _engines:
        _engines.clear()
        torch.cuda.empty_cache()
        _engines[key] = Engine.from_state_dict(fx.weights(), Vocab.for_dataset(fx.meta["dataset"]), num_timesteps=fx.meta["T"],
                                               q_type=fx.meta["q_type"], operand_dtype=dtype)
    return _engines[key]


def cond_cuda(fx):
    if fx.cond is None:
        return None
    return {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in fx.cond.items()}


def test_schedule_and_adaln_tables():
    fx = Fixture("rico25_uncond_random")
    eng = engine_for(fx)
    sch, osch = eng.schedule_tables(), O.group_schedules(fx.spec.T, fx.vocab)
    for g in range(5):
        for r, name in enumerate(O.SCHED_NAMES):
            a, b = sch[g, r, : osch[g][name].shape[0]], osch[g][name]
            fin = torch.isfinite(b)
            assert torch.equal(torch.isfinite(a), fin)
            assert (a[fin] - b[fin]).abs().max() <= 1e-6 * b[fin].abs().max().clamp(min=1.0)
    ad = eng.adaln_table()
    oad = torch.stack([O.adaln_table(fx.weights(), fx.spec, l) for l in range(fx.spec.layers)])
    assert (ad - oad).abs().max() < 1e-5


@pytest.mark.parametrize("name", NAMES)
def test_step_epilogue_is_id_exact_on_reference_logits(name):
    """posterior + cond adjustments + draw, fed with the REFERENCE's fp32 logits under the shared-noise contract:
    token ids must be bit-exact, log-probs within 1e-4."""
    fx = Fixture(name)
    eng = engine_for(fx)
    cond = cond_cuda(fx)
    for i in fx.trace_steps:
        t_model, t_post = fx.plan[i]
        out, _, lp = eng.step(fx.x_in[i].cuda(), t_model, t_post, fx.cfg_dict, cond, seed=fx.meta["noise_seed"], step_ctr=i,
                              want_logprob=True, logits_in=fx.logits(i).cuda())
        torch.cuda.synchronize()
        assert (lp.cpu() - fx.logp(i)).abs().max() < 1e-4
        assert torch.equal(out.cpu(), fx.x_out[i]), f"{name} step {i}: {(out.cpu() != fx.x_out[i]).sum().item()} ids differ"
        # without the log-prob output the constrained / random|gumbel|deterministic configurations take the group-centric
        # kernel (posterior_sample_group_kernel): same ids
        out2, _, _ = eng.step(fx.x_in[i].cuda(), t_model, t_post, fx.cfg_dict, cond, seed=fx.meta["noise_seed"], step_ctr=i,
                              logits_in=fx.logits(i).cuda())
        assert torch.equal(out2.cpu(), fx.x_out[i]), f"{name} step {i} (group kernel): {(out2.cpu() != fx.x_out[i]).sum().item()} ids differ"


@pytest.mark.parametrize("name", NAMES)
def test_epilogue_every_step_against_oracle(name):
    """same check on every loop iteration (all timesteps, skip steps, time_difference), logits from the fp32 oracle"""
    fx = Fixture(name)
    eng = engine_for(fx)
    cond = cond_cuda(fx)
    orc = O.Oracle(fx.vocab, fx.spec, fx.weights(), q_type=fx.meta["q_type"])
    n = len(fx.plan)
    g = torch.Generator().manual_seed(0)
    bad = 0
    for i in sorted(set(range(0, n, max(1, n // 12))) | {n - 1}):
        t_model, t_post = fx.plan[i]
        logits = torch.randn(fx.B, fx.vocab.S, fx.vocab.C, generator=g) * 3.0
        lp_o = orc.logprob_from_logits(logits, fx.x_in[i], t_post, fx.cond)
        u, ug = fx.noise(i)
        want = O.draw(lp_o, fx.cfg, u, ug)
        out, _, lp = eng.step(fx.x_in[i].cuda(), t_model, t_post, fx.cfg_dict, cond, seed=fx.meta["noise_seed"], step_ctr=i,
                              want_logprob=True, logits_in=logits.cuda())
        assert (lp.cpu() - lp_o).abs().max() < 1e-4
        bad += int((out.cpu() != want).sum())
        out2, _, _ = eng.step(fx.x_in[i].cuda(), t_model, t_post, fx.cfg_dict, cond, seed=fx.meta["noise_seed"], step_ctr=i,
                              logits_in=logits.cuda())            # group-centric kernel where eligible
        bad += int((out2.cpu() != want).sum())
    assert bad == 0


def test_denoiser_logits_at_reference_weight_scale():
    """the 1e-3 gate proper: wgmma denoiser (fp16 operands, fp32 accumulate) vs the fp32 restatement of the reference,
    weights at the reference's init scale, several timesteps and token mixes"""
    _logits_vs_fp32_oracle("ref")


def test_denoiser_logits_row_offset_weights():
    """the same 1e-3 gate with + 256 on the out-projection / FF2 biases and the token embedding
    (kernel_refs.weight_set("offset")): every LayerNorm sees rows whose mean is far from zero"""
    _logits_vs_fp32_oracle("offset")


def _logits_vs_fp32_oracle(weights):
    from layoutdm_b200 import Engine, Vocab
    import kernel_refs as R
    vo, spec = O.RICO25, O.ModelSpec()
    sd = R.weight_set(weights, vo, spec, seed=0)
    _engines.clear()
    eng = Engine.from_state_dict(sd, Vocab.for_dataset("rico25"), num_timesteps=spec.T)
    g = torch.Generator().manual_seed(0)
    worst = 0.0
    for t in (0, 42, 99):
        ids = torch.randint(0, vo.C, (6, vo.S), generator=g)
        ids[0] = vo.mask_id
        ids[1, 60:] = vo.pad_id
        _, lg, _ = eng.step(ids.cuda(), t, t, {"name": "deterministic"}, want_logits=True)
        with torch.no_grad():
            ref = O.denoiser_forward(sd, ids, t, vo, spec)
        d = (lg.cpu() - ref).abs().max().item()
        print(f"{weights} t={t}: max|logit|={ref.abs().max():.3f} max-abs error {d:.2e}")
        worst = max(worst, d)
    assert worst < LOGIT_TOL


@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
@pytest.mark.parametrize("name", ["rico25_uncond_random", "publaynet_c_top_p", "rico25_refinement_T200"])
def test_denoiser_logits(name, dtype):
    """against the REFERENCE's recorded fp32 logits (stress weights x2..x3): error <= 1e-3 relative to the logit scale for
    fp16 operands; bf16 within its documented factor.  Also reports the distance to the same-rounding oracle."""
    fx = Fixture(name)
    eng = engine_for(fx, dtype)
    odt = torch.float16 if dtype == "fp16" else torch.bfloat16
    for i in fx.trace_steps:
        t_model, t_post = fx.plan[i]
        _, lg, _ = eng.step(fx.x_in[i].cuda(), t_model, t_post, {"name": "deterministic"}, want_logits=True)
        lg = lg.cpu()
        assert torch.isfinite(lg).all()
        with torch.no_grad():
            same = O.denoiser_forward(fx.weights(), fx.x_in[i], t_model, fx.vocab, fx.spec, operand_dtype=odt)
        ref = fx.logits(i)
        scale = max(1.0, ref.abs().max().item())
        d_same = (lg - same).abs().max().item()
        d_ref = (lg - ref).abs().max().item()
        print(f"{name} step {i} {dtype}: max|logit|={scale:.2f} |d| vs fp32 reference {d_ref:.2e} (rel {d_ref / scale:.2e}), vs same-rounding oracle {d_same:.2e}")
        tol = STRESS_REL * scale * (BF16_FACTOR if dtype == "bf16" else 1.0)
        assert d_ref < tol and d_same < tol


@pytest.mark.parametrize("name", NAMES)
def test_full_step_ids_vs_reference(name):
    """whole step (denoiser + epilogue) on the reference's own x_t: ids equal the reference's except where the 16-bit
    operand rounding moves a near-tie; fixed tokens are always exact."""
    fx = Fixture(name)
    eng = engine_for(fx)
    cond = cond_cuda(fx)
    n = len(fx.plan)
    steps = sorted(set(range(0, n, max(1, n // 10))) | {n - 1})
    mism = tot = 0
    for i in steps:
        t_model, t_post = fx.plan[i]
        out, _, _ = eng.step(fx.x_in[i].cuda(), t_model, t_post, fx.cfg_dict, cond, seed=fx.meta["noise_seed"], step_ctr=i)
        out = out.cpu()
        mism += int((out != fx.x_out[i]).sum()); tot += out.numel()
        if fx.cond is not None:
            m = fx.cond["mask"]
            assert torch.equal(out[m], fx.cond["seq"][m])
    print(f"{name}: {mism}/{tot} ids differ from the fp32 reference")
    assert mism / tot < 0.01


def test_loop_equals_stepwise_and_host_entry():
    fx = Fixture("publaynet_c_top_p")
    eng = engine_for(fx)
    cond = cond_cuda(fx)
    plan = fx.plan[:12]
    ids, trace = eng.sample_loop(fx.B, plan, fx.cfg_dict, cond, seed=5, trace=True)
    x = fx.cond["seq"].cuda()
    for i, (tm, tp) in enumerate(plan):
        x, _, _ = eng.step(x, tm, tp, fx.cfg_dict, cond, seed=5, step_ctr=i)
        assert torch.equal(x, trace[i])
    assert torch.equal(ids, trace[-1])
    ids2 = eng.sample_loop(fx.B, plan, fx.cfg_dict, cond, seed=5)
    assert torch.equal(ids2, ids)
    host_cond = {k: (v.pin_memory() if isinstance(v, torch.Tensor) else v) for k, v in fx.cond.items()}
    ids3, h2d, d2h = eng.sample_host(fx.B, plan, fx.cfg_dict, host_cond, seed=5)
    assert torch.equal(ids3, ids.cpu()) and d2h == fx.B * 125 * 8 and h2d >= fx.B * 125 * 9


def test_noise_is_keyed_by_global_layout_index():
    """shard invariance: layouts [4,8) of a B=8 call == a B=4 call with b_global0=4"""
    fx = Fixture("rico25_uncond_random")
    eng = engine_for(fx)
    plan = fx.plan[-6:]
    cfg = {"name": "random", "temperature": 1.0}
    init = torch.randint(0, fx.vocab.C, (8, 125), generator=torch.Generator().manual_seed(1)).cuda()
    full = eng.sample_loop(8, plan, cfg, seed=9, ids_init=init)
    part = eng.sample_loop(4, plan, cfg, seed=9, ids_init=init[4:], b_global0=4)
    assert torch.equal(full[4:], part)
    other = eng.sample_loop(4, plan, cfg, seed=10, ids_init=init[4:], b_global0=4)
    assert not torch.equal(other, part)


@pytest.mark.parametrize("B", [1, 5, 148, 1024])
def test_invariants_at_scale(B):
    """size-independent properties at the BASELINE batch sizes: ids in range, no MASK after t=0, fixed tokens kept,
    no PAD in bbox slots of real elements (cond=c)."""
    fx = Fixture("publaynet_c_top_p")
    eng = engine_for(fx)
    v = fx.vocab
    g = torch.Generator().manual_seed(B)
    n_el = torch.randint(1, 26, (B,), generator=g)
    seq = torch.full((B, 125), v.mask_id, dtype=torch.long)
    mask = torch.zeros(B, 125, dtype=torch.bool)
    for b in range(B):
        n = int(n_el[b])
        seq[b, 0:5 * n:5] = torch.randint(0, v.n_cat, (n,), generator=g)
        mask[b, 0:5 * n:5] = True
        seq[b, 5 * n:] = v.pad_id
        mask[b, 5 * n:] = True
    cond = dict(seq=seq.cuda(), mask=mask.cuda(), type="c")
    plan = [fx.plan[i] for i in (0, 30, 60, 90, 99)]
    ids = eng.sample_loop(B, plan, fx.cfg_dict, cond, seed=3).cpu()
    assert ids.min() >= 0 and ids.max() < v.C
    assert (ids != v.mask_id).all()
    assert torch.equal(ids[mask], seq[mask])
    real = (torch.arange(125)[None] % 5 != 0) & (seq != v.pad_id)
    assert (ids[real] != v.pad_id).all()
    # every generated attribute token lies in its own attribute's vocabulary slice
    for a in range(1, 5):
        tok = ids[:, a::5][real[:, a::5]]
        lo = v.n_cat + (a - 1) * v.n_bins
        assert ((tok >= lo) & (tok < lo + v.n_bins)).all()


def test_error_behaviour_mirrors_reference():
    fx = Fixture("rico25_uncond_random")
    eng = engine_for(fx)
    x = torch.full((2, 125), fx.vocab.mask_id, dtype=torch.long).cuda()
    with pytest.raises(AssertionError):          # constrained.py:139
        eng.step(x, 100, 100, {"name": "random"})
    with pytest.raises(AssertionError):          # util.py:35
        eng.step(torch.full_like(x, 155), 5, 5, {"name": "random"})
    with pytest.raises(NotImplementedError):     # base.py:361-362
        eng.sample_loop(2, [(5, 5), (5, 5)], {"name": "random"})
    with pytest.raises(NotImplementedError):     # sampling.py:117-118
        eng.step(x, 5, 5, {"name": "nucleus"})


def test_class_api_mirror():
    """FusedMaskAndReplaceDiffusion / LayoutDMB200 keep the reference signatures (sample, _sample_single_step, decode)"""
    from layoutdm_b200 import LayoutDMB200
    fx = Fixture("rico25_uncond_T50")
    model = LayoutDMB200.from_state_dict(fx.weights(), dataset="rico25", num_timesteps=100)
    torch.manual_seed(0)
    out = model.sample(batch_size=3, cond=None, sampling_cfg={"name": "random", "temperature": 1.0, "num_timesteps": 10}, cond_type="unconditional")
    assert out["bbox"].shape == (3, 25, 4) and out["label"].shape == (3, 25) and out["mask"].dtype == torch.bool and not out["bbox"].is_cuda
    torch.manual_seed(0)
    out2 = model.sample(batch_size=3, sampling_cfg={"name": "random", "temperature": 1.0, "num_timesteps": 10})
    assert torch.equal(out["bbox"], out2["bbox"])       # torch.manual_seed controls the noise like in the reference
    core = model.model
    res = core.sample(batch_size=2, sampling_cfg={"name": "random", "temperature": 1.0, "num_timesteps": 5}, get_intermediate_results=True)
    assert isinstance(res, list) and len(res) == 5 and res[0].shape == (2, 125) and res[0].dtype == torch.int64
    log_z = torch.log(torch.nn.functional.one_hot(torch.full((2, 125), 154), 155).permute(0, 2, 1).float().clamp(min=1e-30)).cuda()
    nxt = core._sample_single_step(log_z, torch.full((2,), 98, device="cuda"), 1, {"name": "random", "temperature": 1.0}, None)
    assert nxt.shape == (2, 155, 125)
    with pytest.raises(AssertionError):      # base.py:311
        core.sample(batch_size=1, sampling_cfg={"name": "random", "num_timesteps": 101})
    # get_cond -> sample, both on the device: label-conditioned generation keeps the given labels / element counts
    g = torch.Generator().manual_seed(1)
    n_el = torch.tensor([25, 1, 7])
    mask = torch.arange(25)[None] < n_el[:, None]
    label = torch.randint(0, 25, (3, 25), generator=g)
    cond = model.get_cond(label, torch.rand(3, 25, 4, generator=g), mask, cond_type="c")
    out3 = model.sample(batch_size=3, cond=cond, sampling_cfg={"name": "random", "temperature": 1.0, "num_timesteps": 20}, cond_type="c")
    assert torch.equal(out3["mask"], mask) and torch.equal(out3["label"][mask], label[mask])
    cond_r = model.get_cond(label, torch.rand(3, 25, 4, generator=g), mask, cond_type="refinement")
    assert set(cond_r) >= {"seq", "mask", "seq_orig", "refine_table", "num_element", "type"}


def test_q_sample_kernel_matches_oracle():
    """forward (corruption) process on ids: bit-exact against the oracle under the shared noise contract"""
    fx = Fixture("rico25_uncond_random")
    eng = engine_for(fx)
    v = fx.vocab
    B = 16
    g = torch.Generator().manual_seed(4)
    x0 = torch.empty(B, v.S, dtype=torch.long)
    for a in range(5):
        ids = torch.tensor(v.group_full_ids(a)[:-1])
        x0[:, a::5] = ids[torch.randint(0, len(ids), (B, 25), generator=g)]
    t = torch.randint(0, 100, (B,), generator=g)
    t[:3] = torch.tensor([0, 99, 50])
    want = O.q_sample_ids(x0, t, 100, v, O.group_schedules(100, v), O.uniforms(21, 0, 2, 0, B, v.S, v.C))
    got = eng.q_sample(x0.cuda(), t.cuda(), seed=21).cpu()
    assert torch.equal(got, want)
    shard = eng.q_sample(x0[8:].cuda(), t[8:].cuda(), seed=21, b_global0=8).cpu()     # keyed by the global layout index
    assert torch.equal(shard, want[8:])


def test_decode_kernel_matches_host_decode():
    from layoutdm_b200 import Vocab, decode_ids, linear_centers
    fx = Fixture("rico25_uncond_random")
    eng = engine_for(fx)
    g = torch.Generator().manual_seed(2)
    ids = torch.randint(0, fx.vocab.C, (64, 125), generator=g)
    ids[:8] = fx.ids_final.repeat(2, 1)[:8]
    want = O.decode_ids(ids, fx.vocab)
    got = {k: v.cpu() for k, v in eng.decode(ids.cuda()).items()}
    for k in want:
        assert torch.equal(got[k], want[k]), k
    centers = torch.stack([torch.as_tensor(c, dtype=torch.float32) for c in linear_centers(32)])
    got2 = {k: v.cpu() for k, v in eng.decode(ids.cuda(), centers).items()}
    assert torch.allclose(got2["bbox"], want["bbox"], atol=1e-6) and torch.equal(got2["mask"], want["mask"])


@pytest.mark.parametrize("cond_type", ["c", "cwh", "gt", "refinement"])
def test_make_cond_kernel_matches_oracle(cond_type):
    """layouts -> cond on the device (ldm_make_cond) == the oracle's restatement of tokenizer.encode + get_cond, which is pinned
    against the reference in tests/test_oracle_vs_reference.py; ids are bit-exact (linear bins incl. the .5 rounding boundaries
    and boxes outside [0, 1]; cluster centres), and the result drives sample() with the strong mask reproduced."""
    fx = Fixture("rico25_uncond_random")
    eng = engine_for(fx)
    vocab = fx.vocab
    B, E = 37, vocab.n_elem
    g = torch.Generator().manual_seed(5)
    n_el = torch.randint(1, E + 1, (B,), generator=g)
    n_el[0], n_el[1] = E, 1
    mask = torch.arange(E)[None] < n_el[:, None]
    label = torch.randint(0, vocab.n_cat, (B, E), generator=g)
    bbox = torch.rand(B, E, 4, generator=g) * 1.3 - 0.15
    bbox[::5] = (torch.arange(bbox[::5].numel()).view(bbox[::5].shape) % 33).float() / 32.0 + 1.0 / 64.0   # exact .5 boundaries
    want = O.make_cond(label, bbox, mask, vocab, cond_type)
    got = eng.cond_from_layouts(label, bbox, mask, cond_type)
    keys = ("seq", "mask") + (("seq_orig",) if cond_type == "refinement" else ())
    for k in keys:
        assert torch.equal(got[k].cpu(), want[k]), k
    if cond_type != "gt":
        assert torch.equal(got["num_element"].cpu(), want["num_element"])
    # cluster centres (kmeans / percentile quantisation): nearest centre
    centers = torch.sort(torch.rand(4, vocab.n_bins, generator=g), dim=1).values
    want_c = O.make_cond(label, bbox, mask, vocab, cond_type, centers=centers)
    got_c = eng.cond_from_layouts(label, bbox, mask, cond_type, centers=centers)
    for k in keys:
        assert torch.equal(got_c[k].cpu(), want_c[k]), k
    if cond_type in ("c", "cwh", "refinement"):
        from layoutdm_b200 import timestep_plan
        ids = eng.sample_loop(B, timestep_plan(fx.spec.T, 10), {"name": "random", "temperature": 1.0}, cond=got, seed=3, ids_init=got["seq"])
        assert torch.equal(ids[got["mask"]], got["seq"][got["mask"]])
    with pytest.raises(NotImplementedError):
        eng.cond_from_layouts(label, bbox, mask, "partial")


def test_loop_edge_plans_and_replay():
    """shortest plans (T_eval = 1, 2), alternating batch sizes on one handle (the captured graph is re-recorded when the plan or the
    batch changes and replayed otherwise), and replay == first run"""
    from layoutdm_b200 import timestep_plan
    fx = Fixture("rico25_uncond_random")
    eng = engine_for(fx)
    cfg = {"name": "random", "temperature": 1.0}
    for T_eval in (1, 2):
        plan = timestep_plan(fx.spec.T, T_eval)
        ids = eng.sample_loop(3, plan, cfg, seed=1)
        assert plan[-1][0] == 0 and (ids != fx.vocab.mask_id).all() and int(ids.max()) < fx.vocab.C
    plan = timestep_plan(fx.spec.T, 7)
    ref = {}
    for B in (3, 5, 3, 5, 3):
        ids = eng.sample_loop(B, plan, cfg, seed=11)
        assert B not in ref or torch.equal(ids, ref[B])       # same key -> same ids, whether the graph was re-recorded or replayed
        ref.setdefault(B, ids.clone())
    assert torch.equal(ref[5][:3], ref[3])                    # noise is keyed by the layout index, not by the batch size
    ids2, trace = eng.sample_loop(3, plan, cfg, seed=11, trace=True)   # plain (non-graph) path with the trace
    assert torch.equal(ids2, ref[3])
