"""
Generates the committed golden fixtures under tests/golden/*.npz by running the UNMODIFIED reference
(the reference checkout, imported through oracle/ref_shims) on CPU, and checks the oracle restatement against it while
doing so.  Run in the build container only:

    python tests/golden/make_golden.py

What a fixture holds (everything the tests need where the reference is absent):
  * the case description (dataset, q_type, T, T_eval, sampling cfg, weight seed/scale, noise seed) and the
    checksum of the synthetic weights (regenerated on the box by oracle.make_weights),
  * the reference's inputs (cond seq/mask/seq_orig, refinement table) and, per loop iteration, the ids the
    REFERENCE produced under the injected-noise contract; for `trace_steps` also the reference's fp32 logits
    and post-adjustment log-probs.
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import ref_harness as rh  # noqa: E402
from oracle import layoutdm_oracle as O  # noqa: E402

CASES = [
    # name, dataset, q_type, T, T_eval, B, sampling, cond_type, extra sampling kw, weight scale
    dict(name="rico25_uncond_random", dataset="rico25", q_type="constrained", T=100, T_eval=100, B=4, samp="random", cond=None, scale=2.0),
    dict(name="rico25_uncond_T50", dataset="rico25", q_type="constrained", T=100, T_eval=50, B=8, samp="random", cond=None, scale=2.0),
    dict(name="publaynet_c_top_p", dataset="publaynet", q_type="constrained", T=100, T_eval=100, B=4, samp="top_p", cond="c", scale=3.0),
    dict(name="rico25_refinement_T200", dataset="rico25", q_type="constrained", T=200, T_eval=200, B=3, samp="random", cond="refinement", scale=2.0,
         refine=dict(refine_lambda=3.0, refine_mode="uniform", refine_offset_ratio=0.1)),
    dict(name="rico25_cwh_deterministic", dataset="rico25", q_type="constrained", T=100, T_eval=25, B=3, samp="deterministic", cond="cwh", scale=3.0),
    dict(name="rico25_partial_gumbel", dataset="rico25", q_type="constrained", T=100, T_eval=20, B=3, samp="gumbel", cond="partial", scale=2.0),
    dict(name="rico25_uncond_top_k_td", dataset="rico25", q_type="constrained", T=100, T_eval=30, B=3, samp="top_k", cond=None, scale=3.0,
         skw=dict(time_difference=0.05)),
    dict(name="rico25_vanilla_random", dataset="rico25", q_type="vanilla", T=100, T_eval=40, B=3, samp="random", cond=None, scale=2.0),
]
TRACE_STEPS = {1}             # loop iterations whose logits / log-probs are stored (plus the last one)
NOISE_SEED = 1234


def run_case(c, write=True):
    vocab = O.RICO25 if c["dataset"] == "rico25" else O.PUBLAYNET
    spec = O.ModelSpec(T=c["T"])
    sd = O.make_weights(vocab, spec, seed=7, scale=c["scale"])
    model, tok = rh.build_reference(c["dataset"], T=c["T"], q_type=c["q_type"], state_dict=sd)
    core = model.model.module
    B, S, C = c["B"], vocab.S, vocab.C
    skw = dict(c.get("skw", {}))
    skw.update(c.get("refine", {}))
    scfg = rh.sampling_cfg(c["samp"], num_timesteps=c["T_eval"], **skw)

    cond_ref = None
    if c["cond"]:
        from trainer.helpers.task import get_cond
        import random
        random.seed(0)
        torch.manual_seed(11)
        batch = rh.synthetic_layouts(B, vocab.n_cat, seed=3)
        cond_ref = get_cond(batch, tok, c["cond"], model_type="LayoutDM")

    # ---- run the reference with injected noise, recording every step ------------------------------------
    rec = []
    orig_step = core._sample_single_step
    orig_sample_fn = None

    def unif(i, rows, ncls):
        assert rows == B * S and ncls == C
        return O.uniforms(NOISE_SEED, i, 0, 0, B, S, C).reshape(B * S, C)

    import trainer.models.categorical_diffusion.base as base_mod
    state = {"i": 0}
    captured = {}

    def sample_hook(logits, sampling_cfg):
        captured["logp"] = logits.detach().clone()
        return orig_sample_fn(logits, sampling_cfg)

    orig_sample_fn = base_mod.sample
    base_mod.sample = sample_hook
    orig_rand_like = torch.rand_like

    def fake_rand_like(x, **kw):
        # only used by the gumbel sampler (sampling.py:113): x is (B, C, S)
        u = O.uniforms(NOISE_SEED, state["i"], 1, 0, B, S, C)
        return torch.from_numpy(u).permute(0, 2, 1).contiguous()

    def step_hook(log_z, model_t, skip_step, sampling_cfg=None, cond=None):
        x_in = log_z.argmax(1)
        with torch.no_grad():
            logits = core.transformer(x_in, timestep=model_t)["logits"]
        out = orig_step(log_z=log_z, model_t=model_t, skip_step=skip_step, sampling_cfg=sampling_cfg, cond=cond)
        rec.append(dict(t_model=int(model_t[0]), skip=int(skip_step), x_in=x_in.clone(), logits=logits.clone(),
                        logp=captured["logp"].permute(0, 2, 1).contiguous(), x_out=out.argmax(1).clone()))
        state["i"] += 1
        return out

    core._sample_single_step = step_hook
    if c["samp"] == "gumbel":
        torch.rand_like = fake_rand_like
    try:
        with rh.injected_multinomial(unif):
            import copy
            ids_ref = core.sample(batch_size=B, cond=copy.deepcopy(cond_ref), sampling_cfg=scfg)
    finally:
        core._sample_single_step = orig_step
        base_mod.sample = orig_sample_fn
        torch.rand_like = orig_rand_like

    # ---- oracle on the same inputs ----------------------------------------------------------------------
    cond_o = None
    if cond_ref is not None:
        cond_o = dict(seq=cond_ref["seq"].clone(), mask=cond_ref["mask"].clone(), type=cond_ref["type"])
        if c["cond"] == "refinement":
            cond_o["seq_orig"] = cond_ref["seq_orig"].clone()
            cond_o["refine_table"] = O.refinement_table(vocab, O.linear_centers(vocab.n_bins), c["refine"]["refine_mode"],
                                                        c["refine"]["refine_offset_ratio"], c["refine"]["refine_lambda"])
    ocfg = O.SamplingCfg(name=c["samp"], temperature=1.0, top_p=0.9, top_k=5, num_timesteps=c["T_eval"],
                         time_difference=skw.get("time_difference", 0.0))
    orc = O.Oracle(vocab, spec, sd, q_type=c["q_type"])
    trace = []
    ids_o = orc.sample(B, ocfg, seed=NOISE_SEED, cond=cond_o, trace=trace)

    plan = O.timestep_plan(c["T"], c["T_eval"], ocfg.time_difference)
    assert len(plan) == len(rec) == len(trace)
    n_mis, max_dl, max_dp = 0, 0.0, 0.0
    for i, (r, o) in enumerate(zip(rec, trace)):
        assert r["t_model"] == o["t_model"] == plan[i][0]
        # compare step-wise on the REFERENCE's own inputs so one flipped near-tie cannot cascade
        lp, logits = orc.step_logprob(r["x_in"], plan[i][0], plan[i][1], cond_o)
        max_dl = max(max_dl, (logits - r["logits"]).abs().max().item())
        max_dp = max(max_dp, (lp - r["logp"]).abs().max().item())
        u = O.uniforms(NOISE_SEED, i, 0, 0, B, S, C) if c["samp"] != "deterministic" else None
        ug = O.uniforms(NOISE_SEED, i, 1, 0, B, S, C) if c["samp"] == "gumbel" else None
        x_o = O.draw(lp, ocfg, u, ug)
        n_mis += int((x_o != r["x_out"]).sum())
    same_traj = bool((ids_o == ids_ref).all())
    print(f"{c['name']:28s} steps={len(rec):3d} logits|d|={max_dl:.2e} logp|d|={max_dp:.2e} "
          f"stepwise id mismatches={n_mis} full-trajectory identical={same_traj}")
    assert max_dl < 2e-5 and max_dp < 2e-4 and n_mis == 0, "oracle does not restate the reference"

    # invariants the reference satisfies (SURVEY.md §8c)
    if cond_ref is not None:
        m = cond_ref["mask"]
        assert (ids_ref[m] == cond_ref["seq"][m]).all()
    if plan[-1][1] == 0:
        assert (ids_ref != vocab.mask_id).all()

    if not write:
        return
    keep = sorted(TRACE_STEPS | {len(rec) - 1})
    out = dict(
        meta=json.dumps(dict(name=c["name"], dataset=c["dataset"], q_type=c["q_type"], T=c["T"], T_eval=c["T_eval"], B=B,
                             sampling=c["samp"], top_p=0.9, top_k=5, temperature=1.0,
                             time_difference=skw.get("time_difference", 0.0), cond=c["cond"], refine=c.get("refine"),
                             weight_seed=7, weight_scale=c["scale"], noise_seed=NOISE_SEED,
                             weights_checksum=O.weights_checksum(sd), trace_steps=keep,
                             plan=plan, ref_commit="873b5ee")),
        ids_final=ids_ref.numpy().astype(np.int16),
        x_in=np.stack([r["x_in"].numpy() for r in rec]).astype(np.int16),
        x_out=np.stack([r["x_out"].numpy() for r in rec]).astype(np.int16),
    )
    for i in keep:
        out[f"logits_{i}"] = rec[i]["logits"].numpy().astype(np.float32)
        out[f"logp_{i}"] = rec[i]["logp"].numpy().astype(np.float32)
    if cond_ref is not None:
        out["cond_seq"] = cond_ref["seq"].numpy().astype(np.int16)
        out["cond_mask"] = cond_ref["mask"].numpy()
        if "seq_orig" in cond_ref:
            out["cond_seq_orig"] = cond_ref["seq_orig"].numpy().astype(np.int16)
            out["refine_table"] = cond_o["refine_table"].numpy()
            # the reference's own weak_logits for the table check
    np.savez_compressed(os.path.join(HERE, c["name"] + ".npz"), **out)


if __name__ == "__main__":
    torch.set_num_threads(8)
    only = sys.argv[1:]
    for c in CASES:
        if only and c["name"] not in only:
            continue
        run_case(c)
