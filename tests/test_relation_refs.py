"""The float64 relation reference (tests/relation_refs.py) on the CPU: pinned to the oracle's restatement of the update (which
tests/test_oracle_relation.py pins to the reference's autograd `update()`), and proven sharp enough for the GPU gate: on the
GPU test's inputs, dropping any single ReLU term, cutting it from one of its two nodes, or flipping its sign moves the
reference by more than the gate."""
import pytest
import torch

import relation_refs as R
from oracle import layoutdm_oracle as O
from test_gpu_relation import synthetic_relation_cond

T = 50


def random_problem(vo, B, seed, centers, lam):
    """the batches of the older GPU test: random edges over boxes drawn from random logits"""
    cond = synthetic_relation_cond(vo, B, seed)
    g = torch.Generator().manual_seed(seed + 1)
    x_t = torch.where(cond["mask"], cond["seq"], torch.full((B, vo.S), vo.mask_id))
    logits = torch.randn(B, vo.S, vo.C, generator=g) * 3.0
    return cond, R.posterior_input(vo, x_t, logits, cond, T)


def designed_problem(vname, centers, lam):
    vo = R.VOCABS[vname]
    B, seed = R.one_update_case(vname, lam)
    B = min(B, 40)
    cond, x_t, logits = R.make_batch(vo, B, seed, centers)
    return cond, R.posterior_input(vo, x_t, logits, cond, T)


def oracle_centers(centers, vo):
    return R.linear_centers32(vo.n_bins) if centers is None else centers


def test_costs_and_box_gradient_match_oracle():
    """per-layout cost and d cost / d box of the autograd reference against O.relation_cost_and_grad on the same boxes"""
    vo = O.RICO25
    cond, lp = designed_problem("rico25", R.centers_for("kmeans", vo.n_bins), 1e4)
    prob = R.Problem(lp, cond["seq"], cond["rel_adj"], R.centers_for("kmeans", vo.n_bins), vo, 1e4)
    _, box = R.expected_boxes(prob.v0, prob.cen, prob.cbox)
    box = box.detach().requires_grad_(True)
    per_layout = torch.stack([R.total_cost(box[b:b + 1], [m[b:b + 1] for m in prob.masks]) for b in range(box.shape[0])])
    (g,) = torch.autograd.grad(per_layout.sum(), box)
    assert not R.kinks(prob.table())
    cost_o, g_o = O.relation_cost_and_grad(box.detach().float(), prob.valid, cond["rel_adj"])
    assert (cost_o.double() - per_layout.detach()).abs().max() <= 1e-5 * (1 + per_layout.abs().max())
    assert (g_o.double() - g).abs().max() <= 1e-5 * (1 + g.abs().max())
    assert g.abs().max() > 1.0


@pytest.mark.parametrize("cen_kind", R.CENTERS)
@pytest.mark.parametrize("kind", ["random", "designed"])
def test_reference_matches_oracle(kind, cen_kind):
    """one update within the fp32 gate of the reference (the oracle is fp32 arithmetic too), three updates within the
    multi-update gate on the well-conditioned layouts.  The random batches' boxes collapse onto bin centres after one update
    at these lambdas, where edges meet at the kinks; the designed batches keep >= 90 % of their layouts well conditioned."""
    for vname in ("rico25", "n_cat3_n_bins31"):
        vo = R.VOCABS[vname]
        cen = R.centers_for(cen_kind, vo.n_bins)
        for lam in (1e4, 3e6):
            cond, lp = random_problem(vo, 12, 5, cen, lam) if kind == "random" else designed_problem(vname, cen, lam)
            prob = R.Problem(lp, cond["seq"], cond["rel_adj"], cen, vo, lam)
            kk = R.kinks(prob.table())
            got = R.bin_logprobs(O.relation_update(lp, cond["seq"], cond["rel_adj"], oracle_centers(cen, vo), vo, T, lam, 1).double(), vo)
            gate = prob.gate()
            r = min(((got - prob.run(1, force=f)).abs() / gate).max().item() for f in R.kink_variants(prob, kk))
            if kind == "designed":
                cond, x_t, logits = R.multi_update_batch(vo, 3, cen)
                lp = R.posterior_input(vo, x_t, logits, cond, T)
                prob = R.Problem(lp, cond["seq"], cond["rel_adj"], cen, vo, lam)
            ref3, gate3, ok = R.multi_update_gate(prob, 3)
            got3 = R.bin_logprobs(O.relation_update(lp, cond["seq"], cond["rel_adj"], oracle_centers(cen, vo), vo, T, lam, 3).double(), vo)
            r3 = ((got3 - ref3).abs() / gate3).amax(dim=(1, 2, 3))
            print(f"{kind} {vname} {cen_kind} lambda={lam:g}: one update |oracle - ref| / gate {r:.3e} (kinks {len(kk)}); "
                  f"three: {r3[ok].max().item():.3e} on {int(ok.sum())}/{len(ok)} well-conditioned layouts")
            assert r <= 1.0
            assert (got - prob.v0).abs().max() > 1e-2, "the inputs do not exercise the update"
            assert ok.any() and r3[ok].max() <= 1.0
            if kind == "designed":
                assert 10 * int(ok.sum()) >= 9 * len(ok)


def test_canvas_box_rules():
    """the canvas node: linear rule for the linear centres (half-to-even at n_bins = 31), nearest centre otherwise"""
    for nb in (30, 31, 32):
        lin = R.linear_centers32(nb)
        cb = R.canvas_box(lin, nb)
        assert cb[0].item() == lin[0, round(nb * 0.5)].item() and cb[2].item() == lin[2, nb - 1].item()
        p, bbox, _ = O.relation_bbox(torch.zeros(1, O.VocabSpec(n_bins=nb).S, O.VocabSpec(n_bins=nb).C), torch.zeros(1, 125, dtype=torch.long),
                                     lin, O.VocabSpec(n_bins=nb))
        assert torch.equal(bbox[0, 0].double(), cb)
        km = R.kmeans_like_centers(nb, seed=nb)
        _, bbox, _ = O.relation_bbox(torch.zeros(1, 125, O.VocabSpec(n_bins=nb).C), torch.zeros(1, 125, dtype=torch.long), km, O.VocabSpec(n_bins=nb))
        assert torch.equal(bbox[0, 0].double(), R.canvas_box(km, nb))


MUTATIONS = ("drop", "flip", "drop_i", "drop_j")


@pytest.mark.parametrize("cen_kind", R.CENTERS)
def test_mutations_exceed_the_gpu_gate(cen_kind):
    """on the one-update GPU cases (every vocabulary, lambda = 1e4, with the oracle's fp32 posterior standing in for the
    kernel's), every single-term mutation of the reference leaves the GPU gate somewhere"""
    probs = []
    for vname, vo in R.VOCABS.items():
        cen = R.centers_for(cen_kind, vo.n_bins)
        cond, lp = designed_problem(vname, cen, 1e4)
        prob = R.Problem(lp, cond["seq"], cond["rel_adj"], cen, vo, 1e4)
        probs.append((prob, prob.run(1), prob.gate()))
    weakest = {}
    for n, (name, bit, src, cI, QI, *_r) in enumerate(R.TERMS):
        for mut in MUTATIONS:
            if mut == "drop_i" and QI is None:
                continue                                  # canvas-source terms: the canvas box is a constant
            r = max(((p.run(1, mutate=(n, mut)) - ref).abs() / gate).max().item() for p, ref, gate in probs)
            weakest[(name, mut)] = r
    lo = min(weakest, key=weakest.get)
    print(f"\ncentres {cen_kind}: smallest max |mutant - reference| / gate {weakest[lo]:.3e} ({lo[0]}, {lo[1]})")
    bad = {k: v for k, v in weakest.items() if not v > 1.0}
    assert not bad, f"mutations the GPU gate would not catch: {bad}"
