"""GPU (-m gpu): the split-bf16 operand mode (operand_dtype "bf16x3").  Every 16-bit operand is a pair hi = bf16(x),
lo = bf16(x - hi), and each product is a_hi w_hi + a_hi w_lo + a_lo w_hi with fp32 accumulation.

Per-kernel float64 checks: the checks of test_gpu_kernels_fp64.py (same kernels, same cases), with each kernel's inputs the exact
float64 sum hi + lo of both tapped planes and the weights rounded to the packed pair.  Its gates, with the pair's bounds in place of
the 16-bit operand rounding:
  u_op    -> 2^-16                    a value stored as a pair is within 2^-16 |x| of x (the softmax probabilities)
  ulp_out -> 2^-16 |ref| + ulp_fp32   a pair output: the fp32 value, then its pair
  KAPPA   -> 3 * 8 + 2^7              three k16 groups (one per wgmma) per k-step, plus the dropped a_lo w_lo <= 2^-16 |a w|
                                      = 2^7 2^-23 |a w|, which enters the same sum_k |a_k w_k| term
  2^-23   -> 2^-20 in the epilogue terms (the LayerNorm's 2^-23 |x_hat gamma|, the fp32 additions of a GEMM epilogue): eight
             fp32 roundings instead of one.  The LayerNorm epilogues round 1/n, the two-pass sums, the square root, its
             reciprocal, gamma + 1 and the products, each up to 2^-24 relative; the one-rounding allowance is hidden under a
             16-bit output's own rounding, but a pair output shows the epilogue's fp32 arithmetic.  Measured: LN2 at per-layout
             timesteps needs ~4.3 roundings (1.42x the gate with one, 1.02x with four); eight is that measurement with margin,
             not a derived bound.  KAPPA is divided by the same 8, so the accumulation term stays (3 * 8 + 2^7) 2^-23 sum |a w|.
End to end the pair's 2^-16 against fp16's 2^-11 per operand predicts 1e-4-class logits where fp16 gets 1e-3: these gates are
set from that prediction."""
import ctypes as C

import pytest
import torch

import gpu_helpers as G
import kernel_refs as R
import split_refs as SR
import test_gpu_kernels_fp64 as K
from fixtures import NAMES, Fixture
from oracle import layoutdm_oracle as O
from test_gpu_parity import cond_cuda
from test_gpu_parity_large import mixed_ids

pytestmark = pytest.mark.gpu

MODE = "bf16x3"
PAIR = 2.0 ** -16
EPI_ROUNDINGS = 8
KAPPA_SPLIT = (3 * K.KAPPA + 2 ** 7) / EPI_ROUNDINGS     # times F32 = EPI_ROUNDINGS 2^-23 below
PAIR_DT = torch.float64                   # stands for "a bf16 pair" in the gates of check_kernels
PAIRED = ("x16", "qkv16", "att16", "z16", "hid16")
LOGIT_TOL = 1e-4                          # the model's logits, reference and offset weights (fp16: 1e-3 against the fp32 oracle)
STRESS_REL = 1e-4                         # x2 / x3 golden fixtures, relative to max|logit| (fp16: 2e-3)
ID_FRAC = 1e-3                            # whole steps against the reference (fp16: 1e-2)

_state = {}


def engine(kind="ref", vo=O.RICO25, layers=4, sd=None, q_type="constrained", T=None):
    from layoutdm_b200 import Engine, Vocab
    key = (kind, vo, layers, q_type, T)
    if _state.get("key") != key:
        _state.clear()
        torch.cuda.empty_cache()
        spec = O.ModelSpec(layers=layers) if T is None else O.ModelSpec(T=T)
        sd = R.weight_set(kind, vo, spec) if sd is None else sd
        eng = Engine.from_state_dict(sd, Vocab(vo.n_cat, vo.n_bins, vo.n_elem, vo.n_attr), num_timesteps=spec.T, q_type=q_type,
                                     operand_dtype=MODE)
        _state.update(key=key, eng=eng, sd=sd, spec=spec, m=SR.split_model(sd, vo, spec))
    return _state["eng"], _state["sd"], _state["spec"], _state["m"]


def read_pair(eng, name, n, read=None):
    """(hi, lo) planes of a paired buffer, as bf16"""
    read = read or G.debug_read
    hi = read(eng, name, n, raw=True).view(torch.bfloat16)
    lo = read(eng, name + "_lo", n, raw=True).view(torch.bfloat16)
    return hi, lo


@pytest.fixture
def split_gates(monkeypatch):
    """check_kernels of test_gpu_kernels_fp64 on pairs: a paired buffer reads as hi + lo (float64, exact), the gates as above"""
    read, ulp = G.debug_read, K.ulp

    def paired_read(eng, name, n, raw=False):
        if name not in PAIRED:
            return read(eng, name, n, raw)
        hi, lo = read_pair(eng, name, n, read)
        v = hi.double() + lo.double()
        return v if raw else v.float()          # float32 holds hi + lo of a pair packed from an fp32 value exactly

    monkeypatch.setattr(G, "debug_read", paired_read)
    monkeypatch.setattr(K, "ulp", lambda ref, dt: PAIR * ref.abs() + ulp(ref, torch.float32) if dt is PAIR_DT else ulp(ref, dt))
    monkeypatch.setattr(K, "KAPPA", KAPPA_SPLIT)
    monkeypatch.setattr(K, "F32", EPI_ROUNDINGS * K.F32)
    monkeypatch.setitem(K.OPS, MODE, (PAIR_DT, PAIR, 2.0 ** -134))


def check_lo_padding(eng, B, S, dh=58, H=8):
    """the padding contracts on the lo planes (the hi + lo checks of check_kernels cover the sum): x16_lo pad rows after the
    embedding, QKV padding columns, attention columns 58..63 all exactly 0"""
    G.set_stop_after(eng, 1)
    try:
        eng.step(torch.full((B, S), 0, dtype=torch.long, device="cuda"), 5, 5, {"name": "deterministic"})
        torch.cuda.synchronize()
        _, lo = read_pair(eng, "x16", B)
        assert (lo[:, S:].float() == 0).all()
    finally:
        G.set_stop_after(eng, 0)
    eng.step(torch.full((B, S), 0, dtype=torch.long, device="cuda"), 5, 5, {"name": "deterministic"})
    torch.cuda.synchronize()
    _, qlo = read_pair(eng, "qkv16", B)
    assert (qlo.float().view(B, 128, 3, H, 64)[..., dh:] == 0).all()
    _, alo = read_pair(eng, "att16", B)
    assert (alo.float().view(B, 128, H, 64)[..., dh:] == 0).all()


# ---- 1. per-kernel float64 checks ----------------------------------------------------------------------------------

@pytest.mark.parametrize("kind,B", [("ref", 301), ("offset", 24), ("peaked", 24)])
def test_kernels_vs_float64(split_gates, kind, B):
    eng, sd, spec, m = engine(kind)
    vo, t = O.RICO25, 42
    ids = mixed_ids(B, vo, 11)
    ids_d = ids.cuda()
    table = eng.adaln_table()
    rep = K.Report(f"{kind} weights, {MODE}, B={B}, t={t}")
    spread = K.check_kernels(eng, m, ids, lambda l, sl: table[l][t], lambda: eng.step(ids_d, t, t, {"name": "deterministic"}), MODE, rep)
    rep.finish()
    if kind == "peaked":
        assert spread.max() > 10.0, "the peaked weight set no longer reaches peaked attention rows"
    check_lo_padding(eng, B, vo.S)


def test_kernels_vs_float64_per_layout_timesteps(split_gates):
    eng, sd, spec, m = engine("ref")
    vo, B = O.RICO25, 24
    ids = mixed_ids(B, vo, 12)
    t = torch.randint(0, spec.T, (B,), generator=torch.Generator().manual_seed(4))
    t[0], t[1] = 0, spec.T - 1
    ids_d, t_d = ids.cuda(), t.cuda()
    table = eng.adaln_table()
    rep = K.Report(f"predict_start, per-layout t, {MODE}, B={B}")
    K.check_kernels(eng, m, ids, lambda l, sl: table[l][t[sl]][:, None], lambda: eng.predict_start(ids_d, t_d), MODE, rep)
    rep.finish()


@pytest.mark.parametrize("shape", list(K.SHAPES))
def test_kernels_vs_float64_other_vocab_shapes(split_gates, shape):
    vo, L = K.SHAPES[shape]
    eng, sd, spec, m = engine("ref", vo, L)
    B, t = 24, 17
    ids = mixed_ids(B, vo, 13)
    ids_d = ids.cuda()
    table = eng.adaln_table()
    rep = K.Report(f"{shape}, {MODE}, B={B}, t={t}")
    K.check_kernels(eng, m, ids, lambda l, sl: table[l][t], lambda: eng.step(ids_d, t, t, {"name": "deterministic"}), MODE, rep)
    rep.finish()
    check_lo_padding(eng, B, vo.S)


# ---- 2. logits against the oracles -----------------------------------------------------------------------------------

@pytest.mark.parametrize("weights", ["ref", "offset"])
def test_denoiser_logits_vs_oracle(weights):
    """against the model's logits computed in float64: |d| <= 1e-4 + e32, e32 = the error of the fp32 oracle (the reference's own
    arithmetic) on the same inputs.  At the reference scale e32 ~ 1e-6 and the logits are also held within 1e-4 of the fp32 oracle.
    On the offset weights the residual stream sits near 256, where fp32 itself is ~1.4e-4 off the float64 logits: no
    fp32-accumulating implementation, the fp32 oracle included, is within 1e-4 of the fp32 oracle's answer there."""
    eng, sd, spec, m = engine(weights)
    sd64 = {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}
    vo = O.RICO25
    g = torch.Generator().manual_seed(0)
    for t in (0, 42, 99):
        ids = torch.randint(0, vo.C, (6, vo.S), generator=g)
        ids[0] = vo.mask_id
        ids[1, 60:] = vo.pad_id
        _, lg, _ = eng.step(ids.cuda(), t, t, {"name": "deterministic"}, want_logits=True)
        lg = lg.cpu().double()
        with torch.no_grad():
            f64 = O.denoiser_forward(sd64, ids, t, vo, spec)
            f32 = O.denoiser_forward(sd, ids, t, vo, spec).double()
            same = SR.denoiser_forward_bf16x3(sd, ids, t, vo, spec).double()
        d64, d32, ds = ((lg - r).abs().max().item() for r in (f64, f32, same))
        e32 = (f32 - f64).abs().max().item()
        print(f"{weights} t={t}: max|logit|={f64.abs().max():.3f} |d| vs float64 {d64:.2e} (gate 1e-4 + e32 = {LOGIT_TOL + e32:.2e}), "
              f"vs fp32 oracle {d32:.2e}, vs split oracle {ds:.2e}; fp32 oracle vs float64 e32 = {e32:.2e}")
        assert d64 < LOGIT_TOL + e32
        if weights == "ref":
            assert d32 < LOGIT_TOL


@pytest.mark.parametrize("name", ["rico25_uncond_random", "publaynet_c_top_p", "rico25_refinement_T200"])
def test_denoiser_logits_vs_reference_stress_weights(name):
    """the reference's recorded fp32 logits of the x2 / x3 golden fixtures: <= 1e-4 max|logit|"""
    fx = Fixture(name)
    eng, *_ = engine(("fx", name), fx.vocab, sd=fx.weights(), q_type=fx.meta["q_type"], T=fx.meta["T"])
    for i in fx.trace_steps:
        t_model, _ = fx.plan[i]
        _, lg, _ = eng.step(fx.x_in[i].cuda(), t_model, t_model, {"name": "deterministic"}, want_logits=True)
        lg = lg.cpu()
        assert torch.isfinite(lg).all()
        ref = fx.logits(i)
        scale = max(1.0, ref.abs().max().item())
        d = (lg - ref).abs().max().item()
        print(f"{name} step {i}: max|logit|={scale:.2f} |d| vs fp32 reference {d:.2e} (rel {d / scale:.2e}, gate {STRESS_REL:.0e})")
        assert d < STRESS_REL * scale


# ---- 3. whole steps against the reference --------------------------------------------------------------------------

@pytest.mark.parametrize("name", NAMES)
def test_full_step_ids_vs_reference(name):
    from layoutdm_b200 import Engine, Vocab
    fx = Fixture(name)
    cond = cond_cuda(fx)
    n = len(fx.plan)
    steps = sorted(set(range(0, n, max(1, n // 10))) | {n - 1})
    counts = {}
    for dtype in ("fp16", MODE):
        _state.clear()
        torch.cuda.empty_cache()
        eng = Engine.from_state_dict(fx.weights(), Vocab.for_dataset(fx.meta["dataset"]), num_timesteps=fx.meta["T"], q_type=fx.meta["q_type"],
                                     operand_dtype=dtype)
        mism = tot = 0
        for i in steps:
            t_model, t_post = fx.plan[i]
            out, _, _ = eng.step(fx.x_in[i].cuda(), t_model, t_post, fx.cfg_dict, cond, seed=fx.meta["noise_seed"], step_ctr=i)
            out = out.cpu()
            mism += int((out != fx.x_out[i]).sum()); tot += out.numel()
            if fx.cond is not None:
                msk = fx.cond["mask"]
                assert torch.equal(out[msk], fx.cond["seq"][msk]), f"{dtype}: fixed tokens changed"
        counts[dtype] = mism
        eng.close()
    print(f"{name}: ids that differ from the fp32 reference over {tot}: fp16 {counts['fp16']}, {MODE} {counts[MODE]}")
    assert counts[MODE] / tot < ID_FRAC


# ---- 4. everything else in the mode --------------------------------------------------------------------------------

def fixture_engine(name):
    fx = Fixture(name)
    eng, *_ = engine(("fx", name), fx.vocab, sd=fx.weights(), q_type=fx.meta["q_type"], T=fx.meta["T"])
    return fx, eng


def test_loop_equals_stepwise_and_graph_replay():
    fx, eng = fixture_engine("publaynet_c_top_p")
    cond = cond_cuda(fx)
    plan = fx.plan[:12]
    ids, trace = eng.sample_loop(fx.B, plan, fx.cfg_dict, cond, seed=5, trace=True)
    x = fx.cond["seq"].cuda()
    for i, (tm, tp) in enumerate(plan):
        x, _, _ = eng.step(x, tm, tp, fx.cfg_dict, cond, seed=5, step_ctr=i)
        assert torch.equal(x, trace[i]), f"step {i}"
    assert torch.equal(ids, trace[-1])
    for _ in range(2):                                         # captured, then replayed
        assert torch.equal(eng.sample_loop(fx.B, plan, fx.cfg_dict, cond, seed=5), ids)
    host_cond = {k: (v.pin_memory() if isinstance(v, torch.Tensor) else v) for k, v in fx.cond.items()}
    ids3, _, _ = eng.sample_host(fx.B, plan, fx.cfg_dict, host_cond, seed=5)
    assert torch.equal(ids3, ids.cpu())


def test_noise_is_keyed_by_global_layout_index():
    fx, eng = fixture_engine("rico25_uncond_random")
    plan = fx.plan[-6:]
    cfg = {"name": "random", "temperature": 1.0}
    init = torch.randint(0, fx.vocab.C, (8, 125), generator=torch.Generator().manual_seed(1)).cuda()
    full = eng.sample_loop(8, plan, cfg, seed=9, ids_init=init)
    part = eng.sample_loop(4, plan, cfg, seed=9, ids_init=init[4:], b_global0=4)
    assert torch.equal(full[4:], part)


@pytest.mark.parametrize("B", [1, 5, 148, 1024])
def test_invariants_at_scale(B):
    fx, eng = fixture_engine("publaynet_c_top_p")
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
    for a in range(1, 5):
        tok = ids[:, a::5][real[:, a::5]]
        lo = v.n_cat + (a - 1) * v.n_bins
        assert ((tok >= lo) & (tok < lo + v.n_bins)).all()


@pytest.mark.parametrize("q_type,B", [("constrained", 18), ("constrained", 301), ("vanilla", 9)])
def test_predict_start_and_vb_terms(q_type, B):
    """the training-side entry points run the same denoiser: logits within LOGIT_TOL of the fp32 oracle at per-layout timesteps"""
    import test_gpu_training_api as TA
    vo, spec = O.RICO25, O.ModelSpec()
    sd = O.make_weights(vo, spec, seed=5)
    eng, *_ = engine(("train", q_type), vo, sd=sd, q_type=q_type)
    scheds = O.group_schedules(spec.T, vo, q_type)
    x0, xt, t, g = TA.inputs(vo, B, seed=B)
    lx0, logits = eng.predict_start(xt.cuda(), t.cuda(), want_logits=True)
    lx0, logits = lx0.cpu(), logits.cpu()
    with torch.no_grad():
        ref = torch.cat([O.denoiser_forward(sd, xt[i:i + 128], t[i:i + 128], vo, spec) for i in range(0, B, 128)])
    err = (logits - ref).abs().max().item()
    print(f"{q_type} B={B}: logits max-abs error {err:.2e} (gate {LOGIT_TOL:.0e})")
    assert err < LOGIT_TOL
    assert (lx0 - O.predict_start(logits)).abs().max() < TA.TOL
    r = eng.vb_terms(x0.cuda(), xt.cuda(), t.cuda(), (1.0, 1.0), want_log_model_prob=True)
    w = O.vb_terms(logits, x0, xt, t, spec.T, vo, scheds, q_type)
    assert (r["log_model_prob"].cpu() - w["log_model_prob"]).abs().max() < TA.TOL
    for k in ("kl", "decoder_nll", "kl_aux"):
        d = (r[k].cpu() - w[k]).abs()
        assert (d <= TA.TOL * (1.0 + w[k].abs())).all(), f"{k}: {d.max():.3e}"


def test_operand_dtype_validation():
    """ldm_create rejects operand_dtype 3; Engine rejects an unknown name; the lo taps exist only in the split mode"""
    from layoutdm_b200 import Engine, Vocab, _lib
    vo, spec = O.RICO25, O.ModelSpec(layers=1)
    sd = O.make_weights(vo, spec, seed=0)
    with pytest.raises(ValueError):
        Engine.from_state_dict(sd, Vocab.for_dataset("rico25"), num_timesteps=spec.T, operand_dtype="tf32")
    lib = _lib.load()
    w = Engine.pack_state_dict(sd, Vocab.for_dataset("rico25"))
    ws = _lib.LdmWeights()
    keep = []
    for name in _lib._W_FIELDS:
        tt = w[name].contiguous()
        keep.append(tt)
        setattr(ws, name, tt.data_ptr())
    desc = _lib.LdmModelDesc(vo.n_cat, vo.n_bins, vo.n_elem, vo.n_attr, 464, 8, 1856, spec.layers, spec.T, 0, 3, torch.cuda.current_device(),
                             0.99999, 0.000009, 0.000009, 0.99999)
    h = C.c_void_p()
    assert lib.ldm_create(C.byref(desc), C.byref(ws), C.byref(h)) == _lib.LDM_ERR_INVALID
    assert b"operand_dtype" in lib.ldm_last_error()
    eng16 = Engine.from_state_dict(sd, Vocab.for_dataset("rico25"), num_timesteps=spec.T)
    eng16.step(torch.full((1, vo.S), vo.mask_id, dtype=torch.long, device="cuda"), 5, 5, {"name": "deterministic"})
    assert lib.ldm_debug_read(eng16._h, b"x16_lo", None, 0, 1) < 0 and lib.ldm_debug_read(eng16._h, b"x16", None, 0, 1) > 0
