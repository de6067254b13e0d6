"""CPU: the comparisons of tests/test_oracle_vs_reference.py against stored outputs of the UNMODIFIED reference, so that they
run without the reference.  tests/golden/oracle_vs_reference/*.npz hold what the reference computed on the seeded inputs
below (the large training-side tensors at the tokens of 6 of the 25 elements); `python tests/test_oracle_reference_golden.py`
re-records them where the reference is available, and test_golden_is_the_reference checks them against it there."""
import os

import numpy as np
import pytest
import torch

import ref_harness as rh
from oracle import layoutdm_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
COND_TYPES = ("c", "cwh", "gt", "refinement")
Q_TYPES = ("constrained", "vanilla")
ELEM = [0, 3, 7, 12, 18, 24]
TOK = [e * 5 + a for e in ELEM for a in range(5)]
VOCAB = O.RICO25


def golden_path(part):
    return os.path.join(GOLDEN, "oracle_vs_reference", f"{part}.npz")


def inputs_q_sample():
    B, S, C = 6, VOCAB.S, VOCAB.C
    g = torch.Generator().manual_seed(3)
    x0 = torch.empty(B, S, dtype=torch.long)
    for a in range(5):
        ids = torch.tensor(VOCAB.group_full_ids(a)[:-1])
        x0[:, a::5] = ids[torch.randint(0, len(ids), (B, 25), generator=g)]
    return x0, torch.tensor([0, 1, 37, 64, 98, 99]), O.uniforms(77, 0, 2, 0, B, S, C)


def inputs_training():
    spec = O.ModelSpec()
    sd = O.make_weights(VOCAB, spec, seed=7, scale=2.0)
    B, S, C = 7, VOCAB.S, VOCAB.C
    g = torch.Generator().manual_seed(0)
    x0 = torch.empty(B, S, dtype=torch.long)
    for a in range(5):
        ids = torch.tensor(VOCAB.group_full_ids(a)[:-1])
        x0[:, a::5] = ids[torch.randint(0, len(ids), (B, 25), generator=g)]
    t = torch.tensor([0, 1, 50, 99, 37, 0, 98])
    xt = O.q_sample_ids(x0, t, 100, VOCAB, O.group_schedules(100, VOCAB), O.uniforms(3, 0, 2, 0, B, S, C))
    lx = torch.log_softmax(torch.randn(B, S, C, generator=g) * 2.0, dim=-1).clamp(-70.0, 0.0)
    return dict(spec=spec, sd=sd, x0=x0, t=t, xt=xt, lx=lx, tq=torch.tensor([-1, 0, 50, 99, 37, 5, 98]),
                t1=torch.tensor([0, 1, 50, 99, 37, 5, 98]), u=O.uniforms(9, 0, 2, 0, B, S, C))


def record():
    """runs the reference on the inputs above: {part: {name: array}}"""
    out = {}
    model, tok = rh.build_reference("rico25", state_dict=O.make_weights(VOCAB, O.ModelSpec(), seed=1))
    core = model.model.module
    x0, t, u = inputs_q_sample()
    got = torch.empty_like(x0)
    orig = torch.rand_like
    try:
        for a, key in enumerate(tok.var_names):
            idx = torch.tensor(VOCAB.group_full_ids(a))
            part = core.converter.f_to_p_id(x0[:, a::5], key)
            log_x0 = torch.log(torch.nn.functional.one_hot(part, len(idx)).permute(0, 2, 1).float().clamp(min=1e-30))
            ua = torch.from_numpy(u)[:, a::5][..., idx].permute(0, 2, 1).contiguous()
            torch.rand_like = lambda x, **kw: ua
            got[:, a::5] = core.converter.p_to_f_id(core.q_sample(log_x_start=log_x0, t=t, key=key).argmax(1), key)
    finally:
        torch.rand_like = orig
    rec = {"q_sample_ids": got}
    ids = torch.randint(0, VOCAB.C, (32, VOCAB.S), generator=torch.Generator().manual_seed(0))
    rec.update({f"decode_{k}": v for k, v in tok.decode(ids.clone()).items() if k in ("bbox", "label", "mask")})
    rh._setup_path()
    from trainer.data.util import sparse_to_dense
    from trainer.helpers.task import get_cond
    for ct in COND_TYPES:
        batch = rh.synthetic_layouts(48, VOCAB.n_cat, seed=3)
        batch.x = batch.x * 1.3 - 0.15
        batch.x[::7] = (torch.arange(batch.x[::7].numel()).view(-1, 4) % 33).float() / 32.0 + 1.0 / 64.0
        bbox, label, _, mask = sparse_to_dense(batch)
        torch.manual_seed(11)
        want = get_cond(batch, tok, cond_type=ct, model_type="LayoutDM")
        if ct == "refinement":
            torch.manual_seed(11)
            bbox = bbox + torch.normal(0, std=0.1, size=bbox.size())
        rec.update({f"{ct}_in_label": label, f"{ct}_in_bbox": bbox, f"{ct}_in_mask": mask})
        rec.update({f"{ct}_{k}": want[k] for k in ("seq", "mask", "seq_orig", "num_element") if k in want})
    out["misc"] = rec
    for q_type in Q_TYPES:
        d = inputs_training()
        model, _ = rh.build_reference("rico25", T=100, q_type=q_type, state_dict=d["sd"])
        core = model.model.module
        x0, t, xt, lx, C = d["x0"], d["t"], d["xt"], d["lx"], VOCAB.C
        log_xt = O.index_to_log_onehot(xt, C).permute(0, 2, 1)
        rec = {}
        with torch.no_grad():
            rec["q_posterior"] = core.q_posterior(log_x_start=lx.permute(0, 2, 1), log_x_t=log_xt, t=t).permute(0, 2, 1)[:, TOK]
            for name, fn, tt in (("q_pred", core.q_pred, d["tq"]), ("q_pred_one", core.q_pred_one_timestep, d["t1"])):
                if q_type == "constrained":
                    for a, key in enumerate("cxywh"):
                        part = lx[:, a::5][..., torch.tensor(VOCAB.group_full_ids(a))].permute(0, 2, 1)
                        rec[f"{name}_{key}"] = fn(part, tt, key)[..., ELEM]
                else:
                    rec[name] = fn(lx.permute(0, 2, 1), tt).permute(0, 2, 1)[:, TOK]
        if q_type == "constrained":
            for a, key in enumerate("cxywh"):
                idx = torch.tensor(VOCAB.group_full_ids(a))
                u_part = torch.from_numpy(d["u"])[:, a::5][..., idx].permute(0, 2, 1).contiguous()
                orig = torch.rand_like
                torch.rand_like = lambda x, **kw: u_part
                try:
                    rec[f"gumbel_{key}"] = core.log_sample_categorical(lx[:, a::5][..., idx].permute(0, 2, 1), key).argmax(1)
                finally:
                    torch.rand_like = orig
        pt = torch.full((x0.shape[0],), 1.0 / 100)
        core.sample_time = lambda b, device, method="uniform": (t, pt)
        if q_type == "constrained":
            def fake_q_sample(log_x_start, t, key):
                a = "cxywh".index(key)
                part = (xt[:, a::5][..., None] == torch.tensor(VOCAB.group_full_ids(a))).long().argmax(-1)
                return torch.log(torch.nn.functional.one_hot(part, len(VOCAB.group_full_ids(a))).permute(0, 2, 1).float().clamp(min=1e-30))
        else:
            def fake_q_sample(log_x_start, t):
                return log_xt
        core.q_sample = fake_q_sample
        with torch.no_grad():
            outputs, losses = core.forward(x0, is_train=True)
            rec["logits"] = core.transformer(xt, timestep=t)["logits"][:, TOK]
        rec.update(probs=outputs["probs"][..., TOK], kl_loss=losses["kl_loss"], aux_loss=losses["aux_loss"])
        out[q_type] = rec
    return {p: {k: v.detach().numpy() for k, v in r.items()} for p, r in out.items()}


def load(part):
    with np.load(golden_path(part)) as z:
        return {k: torch.from_numpy(z[k]) for k in z.files}


def test_q_sample_ids_golden():
    x0, t, u = inputs_q_sample()
    want = O.q_sample_ids(x0, t, 100, VOCAB, O.group_schedules(100, VOCAB), u)
    assert torch.equal(load("misc")["q_sample_ids"], want)


def test_decode_golden():
    g = load("misc")
    ids = torch.randint(0, VOCAB.C, (32, VOCAB.S), generator=torch.Generator().manual_seed(0))
    got = O.decode_ids(ids, VOCAB)
    for k in ("bbox", "label", "mask"):
        assert torch.equal(got[k], g[f"decode_{k}"]), k


@pytest.mark.parametrize("cond_type", COND_TYPES)
def test_make_cond_golden(cond_type):
    g = {k[len(cond_type) + 1:]: v for k, v in load("misc").items() if k.startswith(cond_type + "_")}
    got = O.make_cond(g["in_label"], g["in_bbox"], g["in_mask"], VOCAB, cond_type)
    for k in ("seq", "mask") + (("seq_orig",) if cond_type == "refinement" else ()):
        assert torch.equal(g[k], got[k]), k
    if cond_type != "gt":
        assert torch.equal(g["num_element"], got["num_element"])


@pytest.mark.parametrize("q_type", Q_TYPES)
def test_training_side_api_golden(q_type):
    g, d = load(q_type), inputs_training()
    scheds = O.group_schedules(100, VOCAB, q_type)
    x0, t, xt, lx = d["x0"], d["t"], d["xt"], d["lx"]
    assert (O.q_posterior(lx, xt, t, 100, VOCAB, scheds, q_type)[:, TOK] - g["q_posterior"]).abs().max() < 1e-5
    for name, full in (("q_pred", O.q_pred_full(lx, d["tq"], 100, VOCAB, scheds, q_type)),
                       ("q_pred_one", O.q_pred_one_timestep_full(lx, d["t1"], 100, VOCAB, scheds, q_type))):
        if q_type == "constrained":
            for a, key in enumerate("cxywh"):
                idx = torch.tensor(VOCAB.group_full_ids(a))
                assert (full[:, a::5][..., idx].permute(0, 2, 1)[..., ELEM] - g[f"{name}_{key}"]).abs().max() < 1e-5, (name, key)
        else:
            assert (full[:, TOK] - g[name]).abs().max() < 1e-5, name
    if q_type == "constrained":
        for a, key in enumerate("cxywh"):
            idx = torch.tensor(VOCAB.group_full_ids(a))
            u_part = torch.from_numpy(d["u"])[:, a::5][..., idx]
            assert torch.equal(O.gumbel_argmax(lx[:, a::5][..., idx], u_part.numpy()), g[f"gumbel_{key}"]), key
    with torch.no_grad():
        logits = O.denoiser_forward(d["sd"], xt, t, VOCAB, d["spec"])
    assert (logits[:, TOK] - g["logits"]).abs().max() < 2e-5
    r = O.vb_terms(logits, x0, xt, t, 100, VOCAB, scheds, q_type)
    assert (r["log_model_prob"].exp().permute(0, 2, 1)[..., TOK] - g["probs"]).abs().max() < 1e-5
    mask, pt = (t == 0).float(), 1.0 / 100
    kl = ((mask * r["decoder_nll"] + (1 - mask) * r["kl"]) / pt).mean().item()
    assert abs(kl - g["kl_loss"].item()) < 1e-4 * abs(g["kl_loss"].item())
    aux = (((1 - t / 100) + 1.0) * 0.1 * (mask * r["decoder_nll"] + (1 - mask) * r["kl_aux"]) / pt).mean().item()
    assert abs(aux - g["aux_loss"].item()) < 1e-4 * abs(g["aux_loss"].item())


@pytest.mark.skipif(not rh.reference_available(), reason="reference not available")
def test_golden_is_the_reference():
    for part, rec in record().items():
        g = load(part)
        assert sorted(g) == sorted(rec), part
        for k, v in rec.items():
            assert np.allclose(g[k].numpy(), v, rtol=0, atol=1e-6), (part, k)


if __name__ == "__main__":
    for part, rec in record().items():
        np.savez_compressed(golden_path(part), **rec)
        print(golden_path(part), os.path.getsize(golden_path(part)))
