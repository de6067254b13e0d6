"""GPU (-m gpu): the relation update kernel (relation.cuh) against the float64 reference of tests/relation_refs.py on the
kernel's own input, bitwise plumbing of the path the class API takes (bin centres, batch total), and the relation loop.

Input and output of the kernel, bitwise.  A relation step runs the generic posterior kernel with PAD-disable off into its
log-prob buffer, the update in place, then the draw from that buffer with PAD-disable on.  The same posterior kernel with
the same flags runs for a step with the same cond without `rel_adj` and `_pad_disable: False` with `want_logprob=True`:
that is the update's input.  The relation step's own `want_logprob` output is the buffer after the update with only the
PAD column rewritten: its bin columns are the update's output.

Gates.  One update: |kernel - float64| <= the per-entry gate of relation_refs (derived from the fp32 arithmetic: softmax,
box sum, the step g p (c - b) product and the stores).  Where a ReLU argument lies within its fp32 error bound of 0 (a kink)
either branch is accepted: the reference is run both ways and the layout passes if one of them is within the gate.
Several updates: the intermediate states are not observable, so each layout is gated by the reference's own sensitivity:
it is rerun with every update perturbed by a uniform draw within that update's gate, and the gate is 4x the spread of the
draws (per element and attribute) plus the last update's own gate.  A layout is well conditioned when no draw changes a
ReLU branch in any update and no update meets a kink; the gate is asserted on those, and they must be >= 90 % of the batch.
Each case prints max |d| / gate, the kinks met and the share of well-conditioned layouts (pytest -s)."""
import types

import pytest
import torch

import relation_refs as R
from oracle import layoutdm_oracle as O

pytestmark = pytest.mark.gpu

T_STEP = 50
DET = {"name": "deterministic"}
VOCABS, CENTERS, centers_for = R.VOCABS, R.CENTERS, R.centers_for

_engines = {}


def engine(vo, dtype="fp16", layers=1, fresh=False):
    from layoutdm_b200 import Engine, Vocab
    key = (vo, dtype, layers)
    if fresh or key not in _engines:
        spec = O.ModelSpec(layers=layers)
        sd = O.make_weights(vo, spec, seed=3, scale=2.0)
        eng = Engine.from_state_dict(sd, Vocab(vo.n_cat, vo.n_bins, vo.n_elem, vo.n_attr), num_timesteps=spec.T, operand_dtype=dtype)
        if fresh:
            return eng
        _engines[key] = (eng, sd, spec)
    return _engines[key][0]


def dev(cond):
    return {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in cond.items()}


def rel_cond(cond, lam, n_up, centers, batch_total=None):
    c = dict(cond, rel_lambda=lam, rel_num_update=n_up)
    if centers is not None:
        c["rel_centers"] = centers
    if batch_total is not None:
        c["rel_batch_total"] = batch_total
    return c


def kernel_io(eng, cond, x_t, logits, lam, n_up, centers, batch_total=None):
    """(the update's input, the relation step's log-prob output), both (B,S,C) fp32 on the host"""
    base = {k: v for k, v in cond.items() if k != "rel_adj"}
    base["_pad_disable"] = False
    _, _, lp_in = eng.step(x_t.cuda(), T_STEP, T_STEP, DET, dev(base), want_logprob=True, logits_in=logits.cuda())
    _, _, lp_out = eng.step(x_t.cuda(), T_STEP, T_STEP, DET, dev(rel_cond(cond, lam, n_up, centers, batch_total)),
                            want_logprob=True, logits_in=logits.cuda())
    return lp_in.cpu(), lp_out.cpu()


def check_untouched(vo, lp_in, lp_out):
    """every entry the update does not own (categories, other groups' columns, PAD element rows outside their bins) is
    bitwise the input; the PAD column is PAD-disable's"""
    own = torch.zeros(vo.S, vo.C, dtype=torch.bool)
    for a in range(4):
        own[a + 1::vo.n_attr, vo.n_cat + a * vo.n_bins: vo.n_cat + (a + 1) * vo.n_bins] = True
    keep = ~own
    keep[:, vo.pad_id] = False
    assert torch.equal(lp_out[:, keep], lp_in[:, keep]), "the relation step changed entries the update does not own"


def one_update(vo, centers, lam, B, seed):
    """one update on a designed batch: -> (max |d| / gate, number of kink terms, active terms, term table)"""
    eng = engine(vo)
    cond, x_t, logits = R.make_batch(vo, B, seed, centers)
    lp_in, lp_out = kernel_io(eng, cond, x_t, logits, lam, 1, centers)
    check_untouched(vo, lp_in, lp_out)
    prob = R.Problem(lp_in, cond["seq"], cond["rel_adj"], centers, vo, lam)
    d_delta, store = prob.gate(parts=True)
    gate = d_delta + store
    tab = prob.table()
    kk = R.kinks(tab)
    got = R.bin_logprobs(lp_out.double(), vo)
    ratio = torch.full((B,), float("inf"), dtype=torch.float64)
    ratio_upd = torch.full((B,), float("inf"), dtype=torch.float64)
    upd = d_delta > store                          # entries whose gate is mostly the update's arithmetic, not the final store
    for force in R.kink_variants(prob, kk):
        rr = (got - prob.run(1, force=force)).abs() / gate
        ratio = torch.minimum(ratio, rr.amax(dim=(1, 2, 3)))
        ratio_upd = torch.minimum(ratio_upd, torch.where(upd, rr, torch.zeros_like(rr)).amax(dim=(1, 2, 3)))
    # layouts without an applying edge (no edge at all: the kernel's early return; edges to PAD only) keep their input bitwise
    quiet = torch.stack([m.flatten(1).any(1) for m in tab["applies"]]).any(0).logical_not()
    assert quiet.any()
    assert torch.equal(R.bin_logprobs(lp_out[quiet], vo), R.bin_logprobs(lp_in[quiet], vo))
    n_active = sum(int(a.sum()) for a in tab["active"])
    moved = (got - prob.v0).abs().max().item()
    assert moved > 1.0, "the inputs do not exercise the update"
    return (ratio.max().item(), ratio_upd.max().item()), len(kk), n_active, tab, moved


@pytest.mark.parametrize("cen_kind", CENTERS)
def test_relation_one_update_vs_float64(cen_kind):
    """every vocabulary x lambda 1e4 / 3e6 for one kind of bin centres; the coverage of the ReLU terms over these cases"""
    tabs, worst, kinks, active = [], 0.0, 0, 0
    print(f"\n== one update, centres {cen_kind}: max |d| / gate")
    for vname, vo in VOCABS.items():
        cen = centers_for(cen_kind, vo.n_bins)
        for lam in (1e4, 3e6):
            B, seed = R.one_update_case(vname, lam)
            (r, r_upd), nk, na, tab, moved = one_update(vo, cen, lam, B, seed)
            print(f"  {vname:18s} lambda={lam:<8g} B={B:<4d} max|d|/gate {r:9.3e} (where the update dominates the gate {r_upd:9.3e})  "
                  f"moved {moved:9.3e}  kinks {nk} of {na} active terms")
            tabs.append(tab); kinks += nk; active += na
            worst = max(worst, r)
    cov = R.coverage(tabs)
    print("  coverage (active, inactive applying edges):")
    for name, (on, off) in cov.items():
        print(f"    {name:18s} {on:7d} {off:7d}")
    assert worst <= 1.0, f"max |d| / gate = {worst:.3e}"
    assert kinks <= 0.01 * active, f"{kinks} kink terms of {active} active: redesign the inputs"
    missing = [n for n, (on, off) in cov.items() if on == 0 or off == 0]
    assert not missing, f"ReLU terms not both active and inactive: {missing}"


@pytest.mark.parametrize("n_up", [2, 3, 5])
def test_relation_several_updates_vs_float64(n_up):
    print(f"\n== {n_up} updates: max |d| / gate over the well-conditioned layouts")
    for vname in ("rico25", "n_cat10_n_bins30"):
        vo = VOCABS[vname]
        for cen_kind in CENTERS:
            cen = centers_for(cen_kind, vo.n_bins)
            for lam in (1e4, 3e6):
                B = 40
                eng = engine(vo)
                cond, x_t, logits = R.multi_update_batch(vo, n_up, cen, B)
                lp_in, lp_out = kernel_io(eng, cond, x_t, logits, lam, n_up, cen)
                check_untouched(vo, lp_in, lp_out)
                prob = R.Problem(lp_in, cond["seq"], cond["rel_adj"], cen, vo, lam)
                ref, gate, ok = R.multi_update_gate(prob, n_up)
                got = R.bin_logprobs(lp_out.double(), vo)
                r = ((got - ref).abs() / gate).amax(dim=(1, 2, 3))
                share = ok.float().mean().item()
                print(f"  {vname:18s} {cen_kind:7s} lambda={lam:<8g} well conditioned {int(ok.sum())}/{B} ({share:.0%})  "
                      f"max|d|/gate {r[ok].max().item():9.3e} (all layouts {r.max().item():9.3e})")
                assert 10 * int(ok.sum()) >= 9 * B, f"only {share:.0%} of the layouts are well conditioned"
                assert r[ok].max().item() <= 1.0


def test_relation_linear_centres_explicit_or_implied_bitwise():
    """rel_centers = float32(linspace) and no rel_centers (the kernel's own linear centres) give the same update, bit for
    bit, for every vocabulary (n_bins 30 and 31 are not powers of two; 31 puts 0.5 half-way between two centres)"""
    for vname, vo in VOCABS.items():
        eng = engine(vo)
        cond, x_t, logits = R.make_batch(vo, 24, 7, None)
        _, a = kernel_io(eng, cond, x_t, logits, 3e6, 3, None)
        _, b = kernel_io(eng, cond, x_t, logits, 3e6, 3, R.linear_centers32(vo.n_bins))
        assert torch.equal(a, b), f"{vname}: {(a != b).sum().item()} log-probs differ"


def test_relation_shard_batch_total_with_centres():
    """a shard with rel_batch_total = the full batch reproduces its rows of the full batch, bit for bit, and matches the float64
    reference run with that batch total"""
    vo = O.RICO25
    cen = centers_for("kmeans", vo.n_bins)
    eng = engine(vo)
    B, k, lam = 24, 10, 3e6
    cond, x_t, logits = R.make_batch(vo, B, 31, cen)
    lp_in, full = kernel_io(eng, cond, x_t, logits, lam, 1, cen)
    part = {key: (v[k:] if isinstance(v, torch.Tensor) else v) for key, v in cond.items()}
    lp_in2, shard = kernel_io(eng, part, x_t[k:], logits[k:], lam, 1, cen, batch_total=B)
    assert torch.equal(lp_in2, lp_in[k:])
    assert torch.equal(shard, full[k:])
    prob = R.Problem(lp_in2, part["seq"], part["rel_adj"], cen, vo, lam, batch_total=B)
    assert not R.kinks(prob.table())
    r = ((R.bin_logprobs(shard.double(), vo) - prob.run(1)).abs() / prob.gate()).max().item()
    print(f"\nshard of {B - k} with batch total {B}: max |d| / gate {r:.3e}")
    assert r <= 1.0


def fake_pyg_batch(adj, valid):
    """the `batch_w_canvas` get_cond attaches: global edge_index / edge_attr and the node -> layout vector"""
    ei, ea, bv, off = [], [], [], 0
    for b in range(adj.shape[0]):
        n = int(valid[b].sum())
        idx = adj[b, :n, :n].nonzero()
        ei.append(idx.t() + off)
        ea.append(adj[b, idx[:, 0], idx[:, 1]].long())
        bv.append(torch.full((n,), b))
        off += n
    return types.SimpleNamespace(edge_index=torch.cat(ei, 1), edge_attr=torch.cat(ea), batch=torch.cat(bv))


@pytest.mark.parametrize("cen_kind", ["linear", "kmeans"])
def test_class_api_relation_sampling_matches_engine(cen_kind):
    """LayoutDMB200 with bbox_centers (what users call) == Engine.sample_loop with the explicit cond"""
    from layoutdm_b200 import LayoutDMB200, timestep_plan
    vo = O.RICO25
    eng = engine(vo)
    cen = centers_for(cen_kind, vo.n_bins)
    B = 12
    cond, _, _ = R.make_batch(vo, B, 41, cen)
    valid = R.valid_nodes(cond["seq"], vo)
    adj = cond["rel_adj"] * (valid[:, :, None] & valid[:, None, :])
    cfg = {"name": "random", "temperature": 1.0, "num_timesteps": 10, "relation_mode": "average", "relation_lambda": 3e6,
           "relation_num_update": 3}
    dm = LayoutDMB200(eng, bbox_centers=[row.numpy() for row in cen])
    user = dict(seq=cond["seq"], mask=cond["mask"], type="relation", batch_w_canvas=fake_pyg_batch(adj, valid))
    ids = dm.sample(batch_size=B, cond=user, sampling_cfg=cfg, seed=5, get_intermediate_results=True)[-1]
    explicit = dict(seq=cond["seq"], mask=cond["mask"], type="relation", rel_adj=adj, rel_centers=cen, rel_lambda=3e6,
                    rel_num_update=3, rel_batch_total=B)
    want = eng.sample_loop(B, timestep_plan(100, 10), cfg, dev(explicit), seed=5).cpu()
    assert torch.equal(ids, want), f"{(ids != want).sum().item()} ids differ"


def test_relation_loop_with_centres_stepwise_vs_oracle():
    """each step of a relation loop with k-means-like centres, on the kernel's own x_t, against the same-rounding oracle step"""
    from layoutdm_b200 import Engine, Vocab
    vo, spec = O.RICO25, O.ModelSpec()
    sd = O.make_weights(vo, spec, seed=3, scale=2.0)
    eng = Engine.from_state_dict(sd, Vocab.for_dataset("rico25"), num_timesteps=spec.T)
    orc = O.Oracle(vo, spec, sd, operand_dtype=torch.float16)
    B = 6
    cen = centers_for("kmeans", vo.n_bins)
    cond, _, _ = R.make_batch(vo, B, 9, cen)
    cond = rel_cond(cond, 3e6, 3, cen)
    plan = O.timestep_plan(spec.T, 10)
    ids, trace = eng.sample_loop(B, plan, {"name": "random", "temperature": 1.0}, dev(cond), seed=4, trace=True)
    trace = trace.cpu()
    x = cond["seq"].clone()
    mism = 0
    with torch.no_grad():
        for i, (tm, tp) in enumerate(plan):
            lp, _ = orc.step_logprob(x, tm, tp, cond)
            want = O.draw(lp, O.SamplingCfg(name="random"), O.uniforms(4, i, 0, 0, B, vo.S, vo.C))
            mism += int((want != trace[i]).sum())
            x = trace[i]
    print(f"\nrelation loop with centres: {mism} of {len(plan) * B * vo.S} ids differ from the oracle")
    assert mism <= 0.01 * len(plan) * B * vo.S
    assert torch.equal(ids.cpu()[cond["mask"]], cond["seq"][cond["mask"]])


def test_relation_handle_growth_bitwise():
    """one handle at B = 8, then 300 (the workspace and the update's buffer are reallocated), then 8 again: each result is
    bitwise a fresh handle's"""
    vo = O.RICO25
    cen = centers_for("kmeans", vo.n_bins)
    eng = engine(vo, fresh=True)
    small = R.make_batch(vo, 8, 51, cen)
    big = R.make_batch(vo, 300, 52, cen)
    outs = [kernel_io(eng, *small, 3e6, 3, cen)[1], kernel_io(eng, *big, 3e6, 3, cen)[1], kernel_io(eng, *small, 3e6, 3, cen)[1]]
    del eng
    for (batch, got) in zip((small, big, small), outs):
        fresh = engine(vo, fresh=True)
        want = kernel_io(fresh, *batch, 3e6, 3, cen)[1]
        del fresh
        assert torch.equal(got, want)


@pytest.mark.parametrize("dtype", ["fp16", "bf16", "bf16x3"])
def test_relation_loop_equals_stepwise(dtype):
    """the relation loop (the split mode launches the embedding kernel in every step) == the same steps one by one, and the
    fixed tokens are kept"""
    from layoutdm_b200 import timestep_plan
    vo = O.RICO25
    eng = engine(vo, dtype, layers=2)
    cen = centers_for("kmeans", vo.n_bins)
    B = 10
    cond, _, _ = R.make_batch(vo, B, 61, cen)
    cond = dev(rel_cond(cond, 3e6, 3, cen))
    cfg = {"name": "random", "temperature": 1.0}
    plan = timestep_plan(100, 12)
    ids, trace = eng.sample_loop(B, plan, cfg, cond, seed=8, trace=True)
    x = cond["seq"]
    for i, (tm, tp) in enumerate(plan):
        x, _, _ = eng.step(x, tm, tp, cfg, cond, seed=8, step_ctr=i)
        assert torch.equal(x, trace[i]), f"{dtype} step {i}: {(x != trace[i]).sum().item()} ids differ"
    assert torch.equal(ids, trace[-1])
    assert torch.equal(ids[cond["mask"]], cond["seq"][cond["mask"]])
