"""GPU (-m gpu): layouts of more than 25 elements.  A layout of S = 5 n_elem tokens takes R = ceil(S / 128) row tiles of 128
rows (R = 2 for 26 .. 51 elements); attention runs one work item per (layout, query tile, head) over the keys of both tiles.

Checked at S = 250 unless stated: attention against float64 on its own inputs (the gate of test_gpu_kernels_fp64.py), with
peaked scores that cross the tile boundary; every tapped buffer finite, pad rows included; logits against the fp32 oracle;
the step epilogue id-exact on the reference's logits of the max_seq_length = 50 fixtures; the loop equal to serialized
steps under every schedule switch; the boundaries 26 / 51 elements and the refusal of 52; the training-side entry points at
per-layout timesteps; a live reference LayoutDM of 50 elements patched by patch_reference_model; B = 4096."""
import copy
import dataclasses

import pytest
import torch

import gpu_helpers as G
import kernel_refs as KR
import long_layout_refs as LR
import test_gpu_loop_schedule as LS
from oracle import layoutdm_oracle as O
from oracle import ref_harness as rh
from test_gpu_kernels_fp64 import F32, KAPPA, OPS, Report, ulp
from test_gpu_parity_large import mixed_ids
from test_long_layouts import LONG_NAMES, LongFixture

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def layout_rows_tap(monkeypatch):
    """every workspace tap of this module, the loop-schedule helpers' included, reads a layout's 128 R rows"""
    monkeypatch.setattr(G, "debug_read", LR.debug_read)

VO50 = dataclasses.replace(O.RICO25, n_elem=50)


def vocab_of(vo):
    from layoutdm_b200 import Vocab
    return Vocab(vo.n_cat, vo.n_bins, vo.n_elem, vo.n_attr)


def make_engine(sd, vo, dtype="fp16", T=100, q_type="constrained"):
    from layoutdm_b200 import Engine
    torch.cuda.empty_cache()
    return Engine.from_state_dict(sd, vocab_of(vo), num_timesteps=T, operand_dtype=dtype, q_type=q_type)


# ---- attention over two key tiles, against float64 ----------------------------------------------------------------------

@pytest.mark.parametrize("kind", ["ref", "peaked"])
@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
def test_attention_two_tiles_vs_float64(dtype, kind):
    """QKV -> attention of layer 0 tapped (stop after launch 3): the float64 attention of the kernel's own qkv rows over the S
    valid keys of both tiles, every query row of both tiles.  The peaked weight set gives rows whose dominant key lies in the
    other tile (a query of tile 0 on a key of tile 1, and the reverse); those rows are counted and required."""
    spec = O.ModelSpec()
    sd = KR.weight_set(kind, VO50, spec)
    eng = make_engine(sd, VO50, dtype)
    m = KR.Model(sd, VO50, spec, operand_dtype=OPS[dtype][0])
    B, S, t, H, dh = 12, VO50.S, 42, spec.heads, m.dh
    rows = eng.layout_rows
    assert rows == 256
    opdt, u_op, eta = OPS[dtype]
    ids = mixed_ids(B, VO50, 5).cuda()
    rep = Report(f"attention over two tiles, {kind} weights, {dtype}, B={B}")
    try:
        G.set_stop_after(eng, 1)
        eng.step(ids, t, t, {"name": "deterministic"})
        torch.cuda.synchronize()
        x32, x16 = G.debug_read(eng, "x32", B), G.debug_read(eng, "x16", B)
        rep.check("embed.pad_rows", bool((x32[:, S:] == 0).all() and (x16[:, S:] == 0).all()), "pad rows not zero")
        G.set_stop_after(eng, 3)
        eng.step(ids, t, t, {"name": "deterministic"})
        torch.cuda.synchronize()
        qkv16, att16 = G.debug_read(eng, "qkv16", B), G.debug_read(eng, "att16", B)
    finally:
        G.set_stop_after(eng, 0)
    assert qkv16.shape == (B, rows, 1536) and att16.shape == (B, rows, 512)
    for name, buf in (("qkv16", qkv16), ("att16", att16)):
        rep.check(name, bool(torch.isfinite(buf).all()), "non-finite values (pad rows included)")
    a4 = att16.view(B, rows, H, KR.HP)
    rep.check("att16.col58", bool((a4[..., dh] == 1.0).all()), f"ones column off by {(a4[..., dh] - 1).abs().max():.3e}")
    rep.check("att16.cols59+", bool((a4[..., dh + 1:] == 0).all()), "padding columns not zero")
    o, s, p, q, k, v = KR.attention(m, qkv16, S)
    ds = KAPPA * F32 * (q.abs() @ k.abs().transpose(-1, -2)).amax(-1, keepdim=True) + 2.0 ** -22 * s.abs().amax(-1, keepdim=True) + 2.0 ** -21
    gate = 2 * (u_op + ds + KAPPA * F32) * (p @ v.abs()) + 2 * eta * S * v.abs().amax(-2, keepdim=True)
    gate = gate.transpose(1, 2)[..., :dh]
    ref = o.view(B, rows, H, KR.HP)[..., :dh]
    rep.gate("att16", a4[..., :dh], ref, ulp(ref, opdt) + gate)
    # dominant keys across the tile boundary: top probability >= 0.5 on a key of the other tile
    pm, arg = p.max(-1)                                                      # (B, H, rows) over the S keys
    qtile = (torch.arange(rows) >= 128).view(1, 1, rows)
    ktile = arg >= 128
    valid_q = (torch.arange(rows) < S).view(1, 1, rows)
    cross01 = int(((pm >= 0.5) & ~qtile & ktile & valid_q).sum())
    cross10 = int(((pm >= 0.5) & qtile & ~ktile & valid_q).sum())
    rep.notes.append(f"query rows dominated (p >= 0.5) by a key of the other tile: tile 0 -> 1: {cross01}, tile 1 -> 0: {cross10}")
    rep.finish()
    if kind == "peaked":
        assert cross01 > 0 and cross10 > 0, "the peaked weight set no longer reaches cross-tile dominant keys"


# ---- logits against the fp32 oracle ------------------------------------------------------------------------------------

@pytest.mark.parametrize("dtype,tol", [("fp16", 1e-3), ("bf16x3", 1e-4)])
def test_logits_vs_oracle(dtype, tol):
    spec = O.ModelSpec()
    sd = O.make_weights(VO50, spec, seed=5, scale=1.0)
    eng = make_engine(sd, VO50, dtype)
    B = 6
    ids = mixed_ids(B, VO50, 9)
    for t in (0, 42, 99):
        _, lg, _ = eng.step(ids.cuda(), t, t, {"name": "deterministic"}, want_logits=True)
        with torch.no_grad():
            ref = O.denoiser_forward(sd, ids, t, VO50, spec)
        err = (lg.cpu() - ref).abs().max().item()
        print(f"{dtype} t={t}: logits max |d| vs the fp32 oracle {err:.2e}")
        assert err < tol
        lgw = G.debug_read(eng, "logits", B)
        assert torch.isfinite(lgw).all(), "non-finite logits (pad rows included)"


@pytest.mark.parametrize("name", LONG_NAMES)
def test_step_epilogue_is_id_exact_on_reference_logits(name):
    """the reference's fp32 logits of the 50-element fixtures scattered into the 256-row logits buffer: ids bit-exact
    (all-classes and group kernels), log-probs within 1e-4"""
    fx = LongFixture(name)
    eng = make_engine(fx.weights(), fx.vocab, T=fx.meta["T"])
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
class LongWorkload(LS.Workload):
    n_elem: int = 50

    @property
    def vocab(self):
        from layoutdm_b200 import Vocab
        return Vocab.for_dataset(self.dataset, self.n_elem)


def long_state_dict(n_elem):
    import functools

    @functools.lru_cache(maxsize=4)
    def sd(dataset, T):
        from layoutdm_b200 import Vocab
        from layoutdm_b200.synthetic import random_state_dict
        return random_state_dict(Vocab.for_dataset(dataset, n_elem), num_timesteps=T, seed=0)
    return sd


LONG1 = LongWorkload("rico25 unconditional, 50 elements, B=96", "rico25", 100, 100, 96, LS.CFG_RANDOM)
LONG2 = LongWorkload("publaynet cond=c top_p, 50 elements, B=33", "publaynet", 100, 30, 33,
                     (("name", "top_p"), ("temperature", 1.0), ("top_p", 0.9)), cond_type="c")
MATRIX = LS.MATRIX + [("LDM_GEMM_SPLIT=3", {"LDM_GEMM_SPLIT": "3"})]      # last: the handle helper does not unset it


@pytest.mark.parametrize("wl,dtype", [(LONG1, "fp16"), (LONG1, "bf16x3"), (LONG2, "fp16")], ids=["L50-fp16", "L50-bf16x3", "L50-c-fp16"])
def test_loop_equals_serialized_steps_under_every_switch(monkeypatch, wl, dtype):
    monkeypatch.setattr(LS, "state_dict", long_state_dict(wl.n_elem))
    cond, ids_init = LS.inputs(wl)
    ks = LS.prefixes(len(wl.plan))
    ref = LS.serialized(monkeypatch, wl, dtype, wl.seed, wl.b_global0, cond, ids_init, keep=[k - 1 for k in ks])
    failures = LS.compare_prefixes(monkeypatch, wl, dtype, MATRIX, ks, ref, cond, ids_init)
    assert not failures, "\n".join(failures)


def test_graph_replays_with_new_seeds(monkeypatch):
    wl = dataclasses.replace(LONG1, T_eval=10)
    monkeypatch.setattr(LS, "state_dict", long_state_dict(wl.n_elem))
    calls = [("seed 10", 10, 0, None, None), ("seed 11", 11, 0, None, None), ("seed 12, b_global0 96", 12, 96, None, None)]
    got = []
    with LS.handle(monkeypatch, wl, "fp16", {}) as eng:
        for _, seed, bg, cond, init in calls:
            got.append(eng.sample_loop(wl.B, wl.plan, wl.sampling, seed=seed, b_global0=bg).cpu())
    for (label, seed, bg, cond, init), ids in zip(calls, got):
        ser = LS.serialized(monkeypatch, wl, "fp16", seed, bg, cond, init).ids[-1]
        assert torch.equal(ids.to(torch.int16), ser), f"{label}: the replay differs from the serialized steps"


# ---- boundaries --------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n_elem", [26, 51])
def test_boundary_layout_lengths_sample_and_match_the_oracle(n_elem):
    """S = 130 (126 pad rows in the second tile) and S = 255: a traced loop, each step against the oracle's draw on the
    kernel's own inputs (same-rounding fp16 operands); mismatches only at near-ties"""
    from layoutdm_b200 import timestep_plan
    vo, spec = dataclasses.replace(O.RICO25, n_elem=n_elem), O.ModelSpec()
    sd = O.make_weights(vo, spec, seed=3, scale=2.0)
    eng = make_engine(sd, vo)
    B, plan = 4, timestep_plan(spec.T, 6)
    ids, trace = eng.sample_loop(B, plan, {"name": "random", "temperature": 1.0}, seed=11, trace=True)
    trace = trace.cpu()
    assert torch.equal(ids.cpu(), trace[-1])
    orc = O.Oracle(vo, spec, sd, operand_dtype=torch.float16)
    cfg = O.SamplingCfg(name="random", num_timesteps=len(plan))
    x = torch.full((B, vo.S), vo.mask_id, dtype=torch.long)
    mism = 0
    with torch.no_grad():
        for i, (tm, tp) in enumerate(plan):
            lp, _ = orc.step_logprob(x, tm, tp)
            mism += int((O.draw(lp, cfg, O.uniforms(11, i, 0, 0, B, vo.S, vo.C)) != trace[i]).sum())
            x = trace[i]
    frac = mism / (len(plan) * B * vo.S)
    print(f"n_elem={n_elem}: id mismatches vs the oracle {mism} ({frac:.4%})")
    assert frac < 0.01
    lg = G.debug_read(eng, "logits", B)
    assert lg.shape[1] == 256 and torch.isfinite(lg).all()


def test_52_elements_are_refused():
    from layoutdm_b200 import _lib
    vo = dataclasses.replace(O.RICO25, n_elem=52)
    sd = O.make_weights(vo, O.ModelSpec(layers=1), seed=1)
    with pytest.raises(_lib.LdmError, match="S=260 <= 256"):
        make_engine(sd, vo)


# ---- training-side entry points ----------------------------------------------------------------------------------------

def test_training_api_per_layout_timesteps():
    spec = O.ModelSpec()
    sd = O.make_weights(VO50, spec, seed=5, scale=1.0)
    eng = make_engine(sd, VO50)
    vo, B, T = VO50, 18, spec.T
    scheds = O.group_schedules(T, vo)
    g = torch.Generator().manual_seed(2)
    x0 = torch.empty(B, vo.S, dtype=torch.long)
    for a in range(5):
        grp = torch.tensor(vo.group_full_ids(a)[:-2])                        # every element valid: no PAD, no MASK
        x0[:, a::5] = grp[torch.randint(0, len(grp), (B, vo.n_elem), generator=g)]
    t = torch.randint(0, T, (B,), generator=g)
    t[0], t[1] = 0, T - 1
    xt = eng.q_sample(x0.cuda(), t.cuda(), seed=3).cpu()
    assert torch.equal(xt, O.q_sample_ids(x0, t, T, vo, scheds, O.uniforms(3, 0, 2, 0, B, vo.S, vo.C)))
    lx0, logits = eng.predict_start(xt.cuda(), t.cuda(), want_logits=True)
    lx0, logits = lx0.cpu(), logits.cpu()
    with torch.no_grad():
        ref = O.denoiser_forward(sd, xt, t, vo, spec)
    assert (logits - ref).abs().max() < 1e-3
    assert (lx0 - O.predict_start(logits)).abs().max() < 1e-4
    post = eng.q_posterior(lx0.cuda(), xt.cuda(), t.cuda()).cpu()
    assert (post - O.q_posterior(lx0, xt, t, T, vo, scheds)).abs().max() < 1e-4
    r = eng.vb_terms(x0.cuda(), xt.cuda(), t.cuda(), (1.0, 1.0), want_log_model_prob=True)
    w = O.vb_terms(logits, x0, xt, t, T, vo, scheds)
    assert (r["log_model_prob"].cpu() - w["log_model_prob"]).abs().max() < 1e-4
    for k in ("kl", "decoder_nll", "kl_aux"):
        assert ((r[k].cpu() - w[k]).abs() <= 1e-4 * (1.0 + w[k].abs())).all(), k
    # decode and cond_from_layouts: ids -> layouts -> cond round trip, against the host decode
    from layoutdm_b200 import decode_ids
    dec = eng.decode(x0.cuda())
    want = decode_ids(x0, vocab_of(vo))
    for k in ("bbox", "label", "mask"):
        assert torch.equal(dec[k].cpu(), want[k]), k
    c = eng.cond_from_layouts(want["label"].cuda(), want["bbox"].cuda(), want["mask"].cuda(), "gt")
    assert torch.equal(c["seq"].cpu(), x0)


# ---- a live reference LayoutDM of 50 elements, patched ----------------------------------------------------------------

@pytest.mark.skipif(not rh.reference_available(), reason="reference archive missing: run python oracle/make_ref.py")
@pytest.mark.parametrize("name", ["rico25_L50_uncond_random", "publaynet_L50_c_top_p"])
def test_patched_reference_model_of_50_elements(name):
    from layoutdm_b200 import patch_reference_model
    fx = LongFixture(name)
    model, tok = LR.build_reference(fx.meta["dataset"], T=fx.meta["T"], q_type=fx.meta["q_type"], state_dict=fx.weights(),
                                    max_seq_length=50)
    model = patch_reference_model(model)
    assert model.model.module._ldm_b200.vocab.S == 250
    cond = copy.deepcopy(fx.cond)
    scfg = rh.sampling_cfg(fx.meta["sampling"], num_timesteps=fx.meta["T_eval"])
    res = model.model.sample(batch_size=fx.B, cond=cond, sampling_cfg=scfg, get_intermediate_results=True, seed=fx.meta["noise_seed"])
    assert len(res) == len(fx.plan) and res[0].shape == (fx.B, 250)
    first = (res[0] == fx.x_out[0]).float().mean().item()
    print(f"{name}: identical tokens after step 0: {first:.4f}")
    assert first > 0.99
    if fx.cond is not None:
        m = fx.cond["mask"]
        assert torch.equal(res[-1][m], fx.cond["seq"][m])
    out = model.sample(batch_size=fx.B, cond=copy.deepcopy(fx.cond), sampling_cfg=scfg, seed=fx.meta["noise_seed"])
    assert out["bbox"].shape == (fx.B, 50, 4)


# ---- large batch --------------------------------------------------------------------------------------------------------

def test_loop_B4096_equals_serialized_first_two_steps(monkeypatch):
    """4096 layouts of 256 rows: 1M rows, FF1's hidden buffer 3.9 G elements; the loop's first two steps equal the serialized steps"""
    wl = dataclasses.replace(LONG1, B=4096, T_eval=2)
    monkeypatch.setattr(LS, "state_dict", long_state_dict(wl.n_elem))
    with LS.handle(monkeypatch, wl, "fp16", {}) as eng:
        ids = eng.sample_loop(wl.B, wl.plan, wl.sampling, seed=wl.seed).to(torch.int16).cpu()
    ser = LS.serialized(monkeypatch, wl, "fp16", wl.seed, 0, None, None)
    assert torch.equal(ids, ser.ids[-1])
