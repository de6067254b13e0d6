"""CPU, only where the reference is available (its checkout or the packaged archive; tests/test_oracle_reference_golden.py
runs the same comparisons against stored reference outputs everywhere): pieces of the oracle against the UNMODIFIED
reference beyond what tests/golden/make_golden.py already asserts while generating the fixtures."""
import numpy as np
import pytest
import torch

import ref_harness as rh
from oracle import layoutdm_oracle as O

pytestmark = pytest.mark.skipif(not rh.reference_available(), reason="reference not available")


@pytest.fixture(scope="module")
def ref():
    vocab, spec = O.RICO25, O.ModelSpec(layers=1)
    sd = O.make_weights(vocab, O.ModelSpec(), seed=1)
    model, tok = rh.build_reference("rico25", state_dict=sd)
    return model, tok, vocab


def test_q_sample_ids_matches_reference_q_sample(ref):
    """forward (corruption) process: oracle.q_sample_ids == reference q_sample per attribute (constrained.py:223-230),
    with the Gumbel uniforms injected through torch.rand_like"""
    model, tok, vocab = ref
    core = model.model.module
    B, S, C, T = 6, vocab.S, vocab.C, 100
    g = torch.Generator().manual_seed(3)
    x0 = torch.empty(B, S, dtype=torch.long)
    for a in range(5):
        ids = torch.tensor(vocab.group_full_ids(a)[:-1])               # normal classes + PAD (no MASK in x0)
        x0[:, a::5] = ids[torch.randint(0, len(ids), (B, 25), generator=g)]
    t = torch.tensor([0, 1, 37, 64, 98, 99])
    u = O.uniforms(77, 0, 2, 0, B, S, C)
    want = O.q_sample_ids(x0, t, T, vocab, O.group_schedules(T, vocab), u)
    orig = torch.rand_like
    got = torch.empty_like(x0)
    try:
        for a, key in enumerate(tok.var_names):
            idx = torch.tensor(vocab.group_full_ids(a))
            K = len(idx)
            part = core.converter.f_to_p_id(x0[:, a::5], key)
            log_x0 = torch.log(torch.nn.functional.one_hot(part, K).permute(0, 2, 1).float().clamp(min=1e-30))
            ua = torch.from_numpy(u)[:, a::5][..., idx].permute(0, 2, 1).contiguous()      # (B, K, 25)
            torch.rand_like = lambda x, **kw: ua
            log_xt = core.q_sample(log_x_start=log_x0, t=t, key=key)
            got[:, a::5] = core.converter.p_to_f_id(log_xt.argmax(1), key)
    finally:
        torch.rand_like = orig
    assert torch.equal(got, want)
    # sanity: late timesteps are mostly MASK, early ones mostly unchanged
    assert (want[5] == vocab.mask_id).float().mean() > 0.9 and (want[0] == x0[0]).float().mean() > 0.9


def test_decode_matches_reference_tokenizer(ref):
    model, tok, vocab = ref
    g = torch.Generator().manual_seed(0)
    ids = torch.randint(0, vocab.C, (32, vocab.S), generator=g)
    a, b = tok.decode(ids.clone()), O.decode_ids(ids, vocab)
    for k in ("bbox", "label", "mask"):
        assert torch.equal(a[k], b[k]), k


@pytest.mark.parametrize("cond_type", ["c", "cwh", "gt", "refinement"])
def test_make_cond_matches_reference_get_cond(ref, cond_type):
    """cond construction: oracle.make_cond == the reference's get_cond (task.py:27-151) on a fake PyG batch, incl.
    boxes outside [0, 1] and on the rounding boundaries of the linear quantisation"""
    model, tok, vocab = ref
    rh._setup_path()
    from trainer.data.util import sparse_to_dense
    from trainer.helpers.task import get_cond
    batch = rh.synthetic_layouts(48, vocab.n_cat, seed=3)
    batch.x = batch.x * 1.3 - 0.15                              # some coordinates below 0 / above 1
    batch.x[::7] = (torch.arange(batch.x[::7].numel()).view(-1, 4) % 33).float() / 32.0 + 1.0 / 64.0   # exact .5 bin boundaries
    bbox, label, _, mask = sparse_to_dense(batch)
    torch.manual_seed(11)
    want = get_cond(batch, tok, cond_type=cond_type, model_type="LayoutDM")
    if cond_type == "refinement":
        torch.manual_seed(11)
        bbox = bbox + torch.normal(0, std=0.1, size=bbox.size())   # the draw of task.py:127
    got = O.make_cond(label, bbox, mask, vocab, cond_type)
    for k in ("seq", "mask") + (("seq_orig",) if cond_type == "refinement" else ()):
        assert torch.equal(want[k], got[k]), k
    if cond_type != "gt":
        assert torch.equal(want["num_element"], got["num_element"])


@pytest.mark.parametrize("q_type", ["constrained", "vanilla"])
def test_training_side_api_matches_reference(q_type):
    """q_posterior with ANY log p(x0) and per-layout timesteps, q_pred, and the loss terms of `forward` (constrained.py:232-333 /
    vanilla.py) -- oracle restatement vs the unmodified reference, with the reference's own x_t and (t, pt) injected"""
    vocab, spec = O.RICO25, O.ModelSpec()
    sd = O.make_weights(vocab, spec, seed=7, scale=2.0)
    model, tok = rh.build_reference("rico25", T=100, q_type=q_type, state_dict=sd)
    core = model.model.module
    scheds = O.group_schedules(100, vocab, q_type)
    B, S, C = 7, vocab.S, vocab.C
    g = torch.Generator().manual_seed(0)
    x0 = torch.empty(B, S, dtype=torch.long)
    for a in range(5):
        ids = torch.tensor(vocab.group_full_ids(a)[:-1])
        x0[:, a::5] = ids[torch.randint(0, len(ids), (B, 25), generator=g)]
    t = torch.tensor([0, 1, 50, 99, 37, 0, 98])
    xt = O.q_sample_ids(x0, t, 100, vocab, O.group_schedules(100, vocab), O.uniforms(3, 0, 2, 0, B, S, C))
    log_xt = O.index_to_log_onehot(xt, C).permute(0, 2, 1)
    # 1. q_posterior, arbitrary log p(x0)
    lx = torch.log_softmax(torch.randn(B, S, C, generator=g) * 2.0, dim=-1).clamp(-70.0, 0.0)
    with torch.no_grad():
        want = core.q_posterior(log_x_start=lx.permute(0, 2, 1), log_x_t=log_xt, t=t).permute(0, 2, 1)
    got = O.q_posterior(lx, xt, t, 100, vocab, scheds, q_type)
    assert (got - want).abs().max() < 1e-5
    # 2. q_pred (t = -1 wraps to T, constrained.py:115)
    tq = torch.tensor([-1, 0, 50, 99, 37, 5, 98])
    full = O.q_pred_full(lx, tq, 100, vocab, scheds, q_type)
    if q_type == "constrained":
        for a, key in enumerate("cxywh"):
            idx = torch.tensor(vocab.group_full_ids(a))
            part = lx[:, a::5][..., idx].permute(0, 2, 1)
            with torch.no_grad():
                w = core.q_pred(part, tq, key)
            assert (full[:, a::5][..., idx].permute(0, 2, 1) - w).abs().max() < 1e-5
    else:
        with torch.no_grad():
            w = core.q_pred(lx.permute(0, 2, 1), tq)
        assert (full.permute(0, 2, 1) - w).abs().max() < 1e-5
    # 2b. q_pred_one_timestep and log_sample_categorical (gumbel) with the noise injected through torch.rand_like
    t1 = torch.tensor([0, 1, 50, 99, 37, 5, 98])
    one = O.q_pred_one_timestep_full(lx, t1, 100, vocab, scheds, q_type)
    u_all = O.uniforms(9, 0, 2, 0, B, S, C)
    if q_type == "constrained":
        for a, key in enumerate("cxywh"):
            idx = torch.tensor(vocab.group_full_ids(a))
            part = lx[:, a::5][..., idx].permute(0, 2, 1)
            with torch.no_grad():
                w = core.q_pred_one_timestep(part, t1, key)
            assert (one[:, a::5][..., idx].permute(0, 2, 1) - w).abs().max() < 1e-5
            u_part = torch.from_numpy(u_all)[:, a::5][..., idx].permute(0, 2, 1).contiguous()
            orig = torch.rand_like
            torch.rand_like = lambda x, **kw: u_part
            try:
                got_ref = core.log_sample_categorical(part, key).argmax(1)
            finally:
                torch.rand_like = orig
            want_o = O.gumbel_argmax(part.permute(0, 2, 1), u_part.permute(0, 2, 1).numpy())
            assert torch.equal(got_ref, want_o)
    else:
        with torch.no_grad():
            w = core.q_pred_one_timestep(lx.permute(0, 2, 1), t1)
        assert (one.permute(0, 2, 1) - w).abs().max() < 1e-5
    # 3. forward: inject (t, pt) and the corruption so that the reference sees the same x_t
    pt = torch.full((B,), 1.0 / 100)
    core.sample_time = lambda b, device, method="uniform": (t, pt)
    if q_type == "constrained":
        def fake_q_sample(log_x_start, t, key):
            a = "cxywh".index(key)
            idx = torch.tensor(vocab.group_full_ids(a))
            part = (xt[:, a::5][..., None] == idx).long().argmax(-1)
            return torch.log(torch.nn.functional.one_hot(part, len(idx)).permute(0, 2, 1).float().clamp(min=1e-30))
    else:
        def fake_q_sample(log_x_start, t):
            return log_xt
    core.q_sample = fake_q_sample
    with torch.no_grad():
        outputs, losses = core.forward(x0, is_train=True)
        logits = core.transformer(xt, timestep=t)["logits"]
    r = O.vb_terms(logits, x0, xt, t, 100, vocab, scheds, q_type)
    assert (r["log_model_prob"].exp().permute(0, 2, 1) - outputs["probs"]).abs().max() < 1e-5
    mask = (t == 0).float()
    kl_loss = mask * r["decoder_nll"] + (1 - mask) * r["kl"]
    assert abs((kl_loss / pt).mean().item() - losses["kl_loss"].item()) < 1e-4 * abs(losses["kl_loss"].item())
    aux = mask * r["decoder_nll"] + (1 - mask) * r["kl_aux"]
    want_aux = (((1 - t / 100) + 1.0) * 0.1 * aux / pt).mean().item()
    assert abs(want_aux - losses["aux_loss"].item()) < 1e-4 * abs(losses["aux_loss"].item())
    # the oracle's denoiser at per-layout timesteps == the reference's transformer
    with torch.no_grad():
        lo = O.denoiser_forward(sd, xt, t, vocab, spec)
    assert (lo - logits).abs().max() < 2e-5
