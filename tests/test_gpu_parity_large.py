"""GPU (-m gpu): parity of the LARGE-BATCH schedule -- the code path bench.py times.

Every kernel runs one tile per CTA (GEMMs: 128-row x 256-column tiles, 64-row whole-row tiles for the LN epilogues;
attention: one (layout, head) per CTA), so a large batch is many waves of CTAs over the 132 SMs, with the row-block order
reversed on every other kernel.  The sizes cover one to several waves, an odd batch and the 4096-layout config.  These
tests compare that steady state with the oracle on EVERY row: logits <= LOGIT_TOL at the reference's weight scale, and every
intermediate buffer of the launch sequence against the same-rounding oracle so that a failure names the kernel.
Everything goes through the C ABI."""
import numpy as np
import pytest
import torch

import gpu_helpers as G
from oracle import layoutdm_oracle as O

pytestmark = pytest.mark.gpu

LOGIT_TOL = 1e-3      # max-abs on fp32 logits vs the fp32 restatement of the reference, weights at the reference's init scale
STAGE_REL = 4e-3      # per-stage gate vs the same-rounding oracle, relative to the stage's own magnitude: 16-bit buffers carry
                      # one rounding (2^-11 relative for fp16) plus the accumulated difference of the upstream fp32 stream;
                      # for bf16 operands the gate scales with the unit roundoff (2^-8 / 2^-11 = 8x)
U_OP = {"fp16": 2.0 ** -11, "bf16": 2.0 ** -8}

_state = {}


def engine(dataset="rico25", T=100, scale=1.0, seed=0, dtype="fp16"):
    from layoutdm_b200 import Engine, Vocab
    key = (dataset, T, scale, seed, dtype)
    if _state.get("key") != key:
        _state.clear()
        torch.cuda.empty_cache()
        vo = O.RICO25 if dataset == "rico25" else O.PUBLAYNET
        spec = O.ModelSpec(T=T)
        sd = O.make_weights(vo, spec, seed=seed, scale=scale)
        _state.update(key=key, vo=vo, spec=spec, sd=sd,
                      eng=Engine.from_state_dict(sd, Vocab.for_dataset(dataset), num_timesteps=T, operand_dtype=dtype))
    return _state["eng"], _state["sd"], _state["vo"], _state["spec"]


def mixed_ids(B, vo, seed):
    """token mixes of a real trajectory: all-MASK layouts, partly denoised, PAD tails, fully random"""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, vo.C, (B, vo.S), generator=g)
    ids[0::7] = vo.mask_id
    keep = torch.rand(B, vo.S, generator=g) < 0.5
    ids[1::7] = torch.where(keep[1::7], ids[1::7], torch.full_like(ids[1::7], vo.mask_id))
    n_el = torch.randint(1, 26, (B,), generator=g)
    tail = torch.arange(vo.S)[None] >= (5 * n_el)[:, None]
    ids[2::7] = torch.where(tail[2::7], torch.full_like(ids[2::7], vo.pad_id), ids[2::7])
    return ids


def oracle_logits(sd, ids, t, vo, spec, chunk=256, **kw):
    out = []
    with torch.no_grad():
        for i in range(0, ids.shape[0], chunk):
            out.append(O.denoiser_forward(sd, ids[i:i + chunk], t, vo, spec, **kw))
    return torch.cat(out)


@pytest.mark.parametrize("B", [148, 296, 301, 1024])
def test_logits_all_rows_large_batch(B):
    """two consecutive denoising steps at the benchmarked schedule; the handle first serves a small batch, so the workspace
    grows mid-handle; odd B checks grids sized by the batch itself.  All B x 125 rows are compared."""
    eng, sd, vo, spec = engine()
    small = mixed_ids(5, vo, 1)
    _, lg_s, _ = eng.step(small.cuda(), 11, 11, {"name": "deterministic"}, want_logits=True)
    d = (lg_s.cpu() - oracle_logits(sd, small, 11, vo, spec)).abs().max().item()
    assert d < LOGIT_TOL
    ids = mixed_ids(B, vo, B)
    worst = 0.0
    for t in (57, 56):
        out, lg, _ = eng.step(ids.cuda(), t, t, {"name": "random", "temperature": 1.0}, seed=B, step_ctr=100 - t, want_logits=True)
        torch.cuda.synchronize()
        lg = lg.cpu()
        assert torch.isfinite(lg).all()
        ref = oracle_logits(sd, ids, t, vo, spec)
        err = (lg - ref).abs().amax(dim=(1, 2))                     # per layout
        bad = (err >= LOGIT_TOL).nonzero().flatten().tolist()
        print(f"B={B} t={t}: max|logit|={ref.abs().max():.3f} max-abs error {err.max():.2e} (worst layout {int(err.argmax())})")
        assert not bad, f"B={B} t={t}: {len(bad)} layouts off, first {bad[:8]}, max {err.max():.3e}"
        worst = max(worst, err.max().item())
        ids = out.cpu()                                             # the second step runs on the first step's draw
    # back to a small batch on the grown workspace
    _, lg_s2, _ = eng.step(small.cuda(), 11, 11, {"name": "deterministic"}, want_logits=True)
    assert torch.equal(lg_s2, lg_s)


def test_logits_config4_refinement_T200_B4096():
    """BASELINE config 4 shape: T=200 model, batch 4096 (8192 LN-GEMM CTAs, about 62 waves)"""
    eng, sd, vo, spec = engine(T=200)
    B = 4096
    ids = mixed_ids(B, vo, 4)
    _, lg, _ = eng.step(ids.cuda(), 150, 150, {"name": "deterministic"}, want_logits=True)
    torch.cuda.synchronize()
    lg = lg.cpu()
    ref = oracle_logits(sd, ids, 150, vo, spec)
    err = (lg - ref).abs().amax(dim=(1, 2))
    print(f"B={B} T=200 t=150: max-abs error {err.max():.2e}")
    assert err.max() < LOGIT_TOL, f"{int((err >= LOGIT_TOL).sum())} layouts off"


def test_stage_taps_large_batch():
    """every kernel of the launch sequence at B=300 (several waves of CTAs in every kernel), against the same-rounding oracle"""
    _stage_taps("fp16")


def test_stage_taps_large_batch_bf16():
    """the same with bf16 operands, against the bf16 same-rounding oracle; the gate scales with the unit roundoff"""
    _stage_taps("bf16")


def _stage_taps(dtype):
    eng, sd, vo, spec = engine(dtype=dtype)
    gate = STAGE_REL * U_OP[dtype] / U_OP["fp16"]
    B, t, S = 300, 42, vo.S
    ids = mixed_ids(B, vo, 9)
    taps = {}
    with torch.no_grad():
        for i in range(0, B, 100):
            tp = {}
            O.denoiser_forward(sd, ids[i:i + 100], t, vo, spec, operand_dtype=torch.float16 if dtype == "fp16" else torch.bfloat16, taps=tp)
            for k, v in tp.items():
                taps.setdefault(k, []).append(v)
    taps = {k: torch.cat(v) for k, v in taps.items()}
    ids_d = ids.cuda()
    report = []

    def cmp(name, got, want):
        got, want = got.float(), want.float()
        assert torch.isfinite(got).all(), name
        d = (got - want).abs()
        rel = d.max().item() / max(1.0, want.abs().max().item())
        report.append((name, d.max().item(), want.abs().max().item()))
        per_layout = d.reshape(B, -1).amax(dim=1)
        assert rel < gate, f"{name}: max-abs {d.max():.3e} (ref max {want.abs().max():.3f}), worst layouts {per_layout.topk(4).indices.tolist()}"

    def run(n):
        G.set_stop_after(eng, n)
        eng.step(ids_d, t, t, {"name": "deterministic"})
        torch.cuda.synchronize()

    try:
        stage = 1; run(stage)
        cmp("embed.x32", G.debug_read(eng, "x32", B)[:, :S], taps["x0"])
        for l in range(spec.layers):
            stage += 1; run(stage)
            q, k, v, pad = G.unpack_qkv(G.debug_read(eng, "qkv16", B))
            cmp(f"L{l}.qkv.q", q, taps[f"q{l}"]); cmp(f"L{l}.qkv.k", k, taps[f"k{l}"]); cmp(f"L{l}.qkv.v", v, taps[f"v{l}"])
            assert pad == 0.0, f"L{l} qkv padding columns off by {pad}"
            stage += 1; run(stage)
            a16 = G.debug_read(eng, "att16", B)[:, :S].view(B, S, 8, 64)
            cmp(f"L{l}.attention", a16[..., :58].reshape(B, S, 464), taps[f"att{l}"])
            stage += 1; run(stage)
            cmp(f"L{l}.outproj.y32", G.debug_read(eng, "y32", B)[:, :S], taps[f"y{l}"])
            cmp(f"L{l}.outproj.z16", G.debug_read(eng, "z16", B)[:, :S], taps[f"z{l}"])
            stage += 1; run(stage)
            cmp(f"L{l}.ff1.hid16", G.debug_read(eng, "hid16", B)[:, :S], taps[f"hid{l}"])
            stage += 1; run(stage)
            if l + 1 < spec.layers:
                cmp(f"L{l}.ff2.x32", G.debug_read(eng, "x32", B)[:, :S], taps[f"x{l + 1}"])
            else:
                cmp(f"L{l}.ff2.hn16", G.debug_read(eng, "z16", B)[:, :S], taps["hn"])
    finally:
        G.set_stop_after(eng, 0)
        for name, d, m in report:
            print(f"{dtype} {name:22s} max-abs {d:.3e}  ref max {m:.3f}")


def test_logprob_in_draw_is_bit_exact():
    """the relation hook's second call: draw from caller-supplied log-probs (ldm_step logprob_in) == O.draw on the same noise"""
    eng, sd, vo, spec = engine()
    B = 64
    g = torch.Generator().manual_seed(3)
    lp = torch.log_softmax(torch.randn(B, vo.S, vo.C, generator=g) * 4.0, dim=-1).clamp(-70.0, 0.0)
    ids = mixed_ids(B, vo, 2)
    for name, extra in (("random", {}), ("deterministic", {}), ("top_p", {"top_p": 0.8}), ("top_k", {"top_k": 3}), ("gumbel", {})):
        cfg_d = dict(name=name, temperature=0.9, **extra)
        cfg = O.SamplingCfg(name=name, temperature=0.9, top_p=extra.get("top_p", 0.9), top_k=extra.get("top_k", 5))
        u = O.uniforms(17, 6, 0, 0, B, vo.S, vo.C) if name != "deterministic" else None
        ug = O.uniforms(17, 6, 1, 0, B, vo.S, vo.C) if name == "gumbel" else None
        want = O.draw(lp, cfg, u, ug)
        out, _, _ = eng.step(ids.cuda(), 5, 5, cfg_d, seed=17, step_ctr=6, logprob_in=lp.cuda())
        assert torch.equal(out.cpu(), want), f"{name}: {(out.cpu() != want).sum().item()} ids differ"


def test_trajectory_distribution_matches_oracle():
    """16-bit operand rounding may flip near-ties, after which a trajectory diverges chaotically; it must not BIAS the samples.
    Same noise, same start: the per-attribute token histograms of the final layouts match the fp32 oracle's (total variation
    distance at the level two independent fp32 runs show), and most layouts are identical token by token."""
    eng, sd, vo, spec = engine(scale=2.0, seed=3)
    B, T_eval = 192, 20
    plan = O.timestep_plan(spec.T, T_eval)
    cfg = O.SamplingCfg(name="random", num_timesteps=T_eval)
    got = eng.sample_loop(B, plan, {"name": "random", "temperature": 1.0}, seed=23).cpu()
    orc = O.Oracle(vo, spec, sd)

    def oracle_run(seed):
        x = torch.full((B, vo.S), vo.mask_id, dtype=torch.long)
        with torch.no_grad():
            for i, (tm, tp) in enumerate(plan):
                lp, _ = orc.step_logprob(x, tm, tp)
                x = O.draw(lp, cfg, O.uniforms(seed, i, 0, 0, B, vo.S, vo.C))
        return x

    want, other = oracle_run(23), oracle_run(24)

    def hist(x):
        return torch.stack([torch.bincount(x[:, a::5].reshape(-1), minlength=vo.C).float() / x[:, a::5].numel() for a in range(5)])

    tv = 0.5 * (hist(got) - hist(want)).abs().sum(dim=1)
    tv_noise = 0.5 * (hist(other) - hist(want)).abs().sum(dim=1)
    same_tok = (got == want).float().mean().item()
    same_layout = (got == want).all(dim=1).float().mean().item()
    print(f"TV per attribute vs oracle {tv.tolist()} (two oracle seeds: {tv_noise.tolist()}); identical tokens {same_tok:.4f}, identical layouts {same_layout:.3f}")
    assert (tv <= tv_noise.max() + 0.02).all()
    assert same_tok > 0.9
