"""GPU (-m gpu): every kernel of the denoiser's launch sequence, isolated, against float64 on its own inputs.

For kernel n the step is stopped after launch n (ldm_debug_set_stop_after) and its output buffers are read back
(ldm_debug_read); its inputs are the buffers as the launches before it left them.  kernel_refs.py recomputes that one kernel
in float64 from those exact inputs, with the weights rounded to the operand dtype the way the packing kernel rounds them.  A
kernel is judged on its own arithmetic, not on the drift it inherits from the stages before it.

Gates (u_op: unit roundoff of the operand dtype, 2^-11 fp16 / 2^-8 bf16; ulp_out(ref): spacing of the stored type at |ref|):
  GEMM        |d| <= ulp_out(ref) + KAPPA 2^-23 sum_k |a_k w_k| + 2^-23 (|bias| + |residual| + |ref|)
              (the last term: the fp32 additions of the epilogue; Q columns carry the q-scale on every term)
  LayerNorm   |d| <= ulp_out(ref) + 2 e_torch + 2^-23 |x_hat gamma|, e_torch = the row's largest error of
              torch.nn.functional.layer_norm in fp32 (same affine / AdaLN scale and shift, same fp32 input rows) against
              float64: no less accurate than the op the reference runs.  The last term is one fp32 rounding of the normalised
              value before the affine step, which the kernel and torch take at different points (at the reference scale both
              sit at a few fp32 ulps, where a per-row comparison would otherwise hinge on torch's luck in that row).
              FF2 normalises a sum it does not store, so its reference input is the float64 sum and the GEMM term above,
              carried through the normalisation, is added: |gamma| rstd max_row(E) (2 + |x_hat|).
  Attention   |d| <= ulp_out(ref) + 2 (u_op + ds + KAPPA 2^-23) sum_j P_j |v_j| + 2 eta S max_j |v_j|
              P is rounded to the operand dtype on purpose (u_op); ds bounds the score error of the fp32 Q K^T accumulation and
              of the exp2 evaluation; eta (half the operand dtype's smallest subnormal) covers probabilities that underflow.
              Column 58 of every head is exactly 1 (x * (1 / x) in fp32 rounds to 1), columns 59..63 exactly 0.
KAPPA = 8: wgmma multiplies 16-bit operands exactly into fp32 and adds each k16 group of products to the fp32 accumulator,
one rounding (<= 2^-23 relative, also for a truncating adder) per group at a magnitude <= sum |a w| of the terms so far.  The
worst case over K / 16 groups (29 for d = 464, 116 for FF2) needs every rounding to go the same way at a partial sum as large
as sum |a w|; with sign-mixed products the partial sums stay far below that and the roundings do not align, so a correct
kernel stays well under KAPPA = 8 (the printed max |d| / gate shows the headroom), while a dropped, doubled or misplaced
k-block moves an output by whole product terms.
Every tapped buffer is finite everywhere, pad rows included, and rerunning a stage gives bitwise-equal buffers (graph replay
and the stop_after taps rely on it).  Each test prints max |d| / gate per buffer (pytest -s)."""
import pytest
import torch
import torch.nn.functional as F

import gpu_helpers as G
import kernel_refs as R
from oracle import layoutdm_oracle as O
from test_gpu_parity_large import mixed_ids

pytestmark = pytest.mark.gpu

KAPPA = 8
F32 = 2.0 ** -23
OPS = {"fp16": (torch.float16, 2.0 ** -11, 2.0 ** -25), "bf16": (torch.bfloat16, 2.0 ** -8, 2.0 ** -134)}   # dtype, u_op, eta
CH = 16            # layouts per chunk of the float64 work
SHAPES = {"n_cat30_n_elem20_L2": (O.VocabSpec(n_cat=30, n_elem=20), 2),   # S = 100: n_valid != 125; C = 160 fills the logits row
          "n_cat1_L1": (O.VocabSpec(n_cat=1), 1)}                          # C = 131: lanes 0..2 own a class >= 128

_state = {}


def engine(kind, dtype, vo=O.RICO25, layers=4):
    from layoutdm_b200 import Engine, Vocab
    key = (kind, dtype, vo, layers)
    if _state.get("key") != key:
        _state.clear()
        torch.cuda.empty_cache()
        spec = O.ModelSpec(layers=layers)
        sd = R.weight_set(kind, vo, spec)
        eng = Engine.from_state_dict(sd, Vocab(vo.n_cat, vo.n_bins, vo.n_elem, vo.n_attr), num_timesteps=spec.T, operand_dtype=dtype)
        _state.update(key=key, eng=eng, sd=sd, spec=spec, m=R.Model(sd, vo, spec, operand_dtype=OPS[dtype][0]))
    return _state["eng"], _state["sd"], _state["spec"], _state["m"]


def ulp(ref, dt):
    """spacing of dt at |ref| (the subnormal spacing below the normal range)"""
    fi = torch.finfo(dt)
    _, e = torch.frexp(ref.abs().clamp(min=fi.tiny))
    return torch.ldexp(torch.full_like(ref, fi.eps), (e - 1).to(ref.dtype))


def torch_ln_err(h32, ref, fn):
    """e_torch: per-row max error of the fp32 torch LayerNorm `fn` on the fp32 rows h32, against the float64 ref"""
    return (fn(h32).double() - ref).abs().amax(-1, keepdim=True)


class Report:
    def __init__(self, title):
        self.title, self.ratio, self.fail, self.notes = title, {}, [], []

    def gate(self, name, got, ref, gate):
        r = ((got.double() - ref).abs() / gate).max().item()
        self.ratio[name] = max(self.ratio.get(name, 0.0), r if r == r else float("inf"))

    def check(self, name, ok, what):
        if not ok:
            self.fail.append(f"{name}: {what}")

    def finish(self):
        print(f"\n== {self.title}: max |d| / gate per buffer")
        for name, r in self.ratio.items():
            print(f"  {name:22s} {r:9.3e}{'   FAIL' if not r <= 1.0 else ''}")
        for n in self.notes:
            print("  " + n)
        bad = [f"{n}: max |d| / gate = {r:.3e}" for n, r in self.ratio.items() if not r <= 1.0] + self.fail
        assert not bad, f"{self.title}: " + "; ".join(bad)


def check_kernels(eng, m, ids, rows, launch, dtype, rep):
    """the launch sequence of one denoiser pass, kernel by kernel.  launch(): one pass on the handle (ldm_step or
    ldm_predict_start); rows(l, sl) -> fp32 AdaLN (scale | shift) rows of layer l for the layouts sl, broadcastable over tokens"""
    B, S = ids.shape
    L, d, H, dh, C = m.spec.layers, m.spec.d, m.spec.heads, m.dh, m.vocab.C
    opdt, u_op, eta = OPS[dtype]
    bits = lambda t: t.view(torch.int16 if t.element_size() == 2 else torch.int32)
    chunks = [slice(b, min(B, b + CH)) for b in range(0, B, CH)]

    def run(n, stage, names):
        """stop after launch n (0: the whole pass), read `names`; a second run must leave bitwise-equal buffers"""
        out = []
        for _ in range(2):
            G.set_stop_after(eng, n)
            launch()
            torch.cuda.synchronize()
            out.append({k: G.debug_read(eng, k, B, raw=True) for k in names})
        got = {}
        for k in names:
            rep.check(f"{stage}.{k}", torch.equal(bits(out[0][k]), bits(out[1][k])), "rerun of the stage is not bitwise equal")
            got[k] = out[0][k].float()
            rep.check(f"{stage}.{k}", bool(torch.isfinite(got[k]).all()), "non-finite values (pad rows included)")
        return got

    def gemm_gate(ref, absum, extra, outdt):
        return ulp(ref, outdt) + KAPPA * F32 * absum + F32 * (extra + ref.abs())

    def ln_gate(ref, outdt, e, shift):
        return ulp(ref, outdt) + 2 * e + F32 * (ref - shift).abs()

    def adaln_fn(r32):
        return lambda h: F.layer_norm(h, (d,), eps=R.LN_EPS) * (1 + r32[..., :d]) + r32[..., d:]

    try:
        # ---- embedding + AdaLN_0 ----
        g = run(1, "embed", ["x32", "x16"])
        rep.check("embed.pad_rows", bool((g["x32"][:, S:] == 0).all() and (g["x16"][:, S:] == 0).all()), "pad rows not zero")
        for sl in chunks:
            h32, r32 = R.embed_input(m, ids[sl]), rows(0, sl)
            ref = R.adaln(m, h32, r32)
            e = torch_ln_err(h32, ref, adaln_fn(r32))
            sh = r32[..., d:].double()
            rep.gate("embed.x32", g["x32"][sl, :S], ref, ln_gate(ref, torch.float32, e, sh))
            rep.gate("embed.x16", g["x16"][sl, :S], ref, ln_gate(ref, opdt, e, sh))
        x32, x16 = g["x32"], g["x16"]
        spread, tiny_p = [], []
        for l in range(L):
            Lw, n0, tag = m.layers[l], 2 + 5 * l, f"L{l}"
            # ---- QKV GEMM: bias, q-scale, padding contract ----
            qkv16 = run(n0, f"{tag}.qkv", ["qkv16"])["qkv16"]
            pad = qkv16.view(B, 128, 3, H, R.HP)[..., dh:]
            want = torch.zeros_like(pad)
            want[:, :, 2, :, 0] = 1.0
            rep.check(f"{tag}.qkv16.padding", torch.equal(pad, want), "padding columns (Q/K zero, V 1 then zeros) off")
            qs = torch.ones(3 * H * R.HP, dtype=torch.float64)
            qs[: H * R.HP] = m.qscale
            for sl in chunks:
                a = x16[sl, :S]
                ref = R.qkv(m, l, a)
                absum = (a.abs().double() @ Lw["wqkv"].abs().t()) * qs
                rep.gate(f"{tag}.qkv16", qkv16[sl, :S], ref, gemm_gate(ref, absum, Lw["bqkv"].abs() * qs, opdt))
            # ---- attention (all 128 query rows of the tile; keys < S) ----
            att16 = run(n0 + 1, f"{tag}.attention", ["att16"])["att16"]
            a4 = att16.view(B, 128, H, R.HP)
            rep.check(f"{tag}.att16.col58", bool((a4[..., dh] == 1.0).all()), f"ones column off by {(a4[..., dh] - 1).abs().max():.3e}")
            rep.check(f"{tag}.att16.cols59+", bool((a4[..., dh + 1:] == 0).all()), "padding columns not zero")
            for sl in chunks:
                o, s, p, q, k, v = R.attention(m, qkv16[sl], S)
                ds = KAPPA * F32 * (q.abs() @ k.abs().transpose(-1, -2)).amax(-1, keepdim=True) + 2.0 ** -22 * s.abs().amax(-1, keepdim=True) + 2.0 ** -21
                gate = 2 * (u_op + ds + KAPPA * F32) * (p @ v.abs()) + 2 * eta * S * v.abs().amax(-2, keepdim=True)
                gate = gate.transpose(1, 2)[..., :dh]                                # (b, 128, H, dh)
                ref = o.view(-1, 128, H, R.HP)[..., :dh]
                rep.gate(f"{tag}.att16", a4[sl][..., :dh], ref, ulp(ref, opdt) + gate)
                sv = s[:, :, :S]
                spread.append((sv.amax(-1) - sv.amin(-1)).flatten())
                tiny_p.append(((sv - sv.amax(-1, keepdim=True)).exp() < 2.0 ** -24).double().mean().view(1))
            # ---- out-projection + residual -> y32 ; LN2 -> z16 (recomputed from the kernel's own y32) ----
            g = run(n0 + 2, f"{tag}.outproj", ["y32", "z16"])
            y32, z16 = g["y32"], g["z16"]
            lnw, lnb = Lw["ln2w"].float(), Lw["ln2b"].float()
            for sl in chunks:
                a, r = att16[sl, :S], x32[sl, :S]
                ref = R.outproj(m, l, a, r)
                absum = a.abs().double() @ Lw["wo"].abs().t()
                rep.gate(f"{tag}.outproj.y32", y32[sl, :S], ref, gemm_gate(ref, absum, Lw["bo"].abs() + r.abs().double(), torch.float32))
                yk = y32[sl, :S]
                zref = R.ln2(m, l, yk)
                e = torch_ln_err(yk, zref, lambda h: F.layer_norm(h, (d,), lnw, lnb, eps=R.LN_EPS))
                rep.gate(f"{tag}.outproj.z16", z16[sl, :S], zref, ln_gate(zref, opdt, e, Lw["ln2b"]))
            # ---- FF1 + ReLU ----
            hid16 = run(n0 + 3, f"{tag}.ff1", ["hid16"])["hid16"]
            for sl in chunks:
                a = z16[sl, :S]
                ref = R.ff1(m, l, a)
                absum = a.abs().double() @ Lw["w1"].abs().t()
                rep.gate(f"{tag}.ff1.hid16", hid16[sl, :S], ref, gemm_gate(ref, absum, Lw["b1"].abs(), opdt))
            # ---- FF2 + residual -> next block's AdaLN (x32 + x16) or the head LN (z16) ----
            last = l + 1 == L
            g = run(n0 + 4, f"{tag}.ff2", ["z16"] if last else ["x32", "x16"])
            for sl in chunks:
                a, r = hid16[sl, :S], y32[sl, :S]
                hpre = R.ff2_pre(m, l, a, r)
                E = KAPPA * F32 * (a.abs().double() @ Lw["w2"].abs().t()) + F32 * (Lw["b2"].abs() + r.abs().double() + hpre.abs())
                r32 = None if last else rows(l + 1, sl)
                ref = R.ff2_norm(m, l, hpre, r32)
                if last:
                    gam, sh = m.hlnw, m.hlnb
                    e = torch_ln_err(hpre.float(), ref, lambda h: F.layer_norm(h, (d,), m.hlnw.float(), m.hlnb.float(), eps=R.LN_EPS))
                else:
                    gam, sh = 1 + r32[..., :d].double(), r32[..., d:].double()
                    e = torch_ln_err(hpre.float(), ref, adaln_fn(r32))
                c = hpre - hpre.mean(-1, keepdim=True)
                rstd = 1 / torch.sqrt((c * c).mean(-1, keepdim=True) + R.LN_EPS)
                prop = gam.abs() * rstd * E.amax(-1, keepdim=True) * (2 + (c * rstd).abs())
                if last:
                    rep.gate(f"{tag}.ff2.headln.z16", g["z16"][sl, :S], ref, ln_gate(ref, opdt, e, sh) + prop)
                else:
                    rep.gate(f"{tag}.ff2.x32", g["x32"][sl, :S], ref, ln_gate(ref, torch.float32, e, sh) + prop)
                    rep.gate(f"{tag}.ff2.x16", g["x16"][sl, :S], ref, ln_gate(ref, opdt, e, sh) + prop)
            if last:
                z16 = g["z16"]
            else:
                x32, x16 = g["x32"], g["x16"]
        # ---- vocabulary head: all 160 columns, >= C exactly 0 ----
        lg = run(0, "head", ["logits"])["logits"]
        rep.check("head.logits.cols>=C", bool((lg[..., C:] == 0).all()), "columns past C not zero")
        for sl in chunks:
            a = z16[sl, :S]
            ref = R.head(m, a)[..., :C]
            absum = a.abs().double() @ m.whead[:C].abs().t()
            rep.gate("head.logits", lg[sl, :S, :C], ref, gemm_gate(ref, absum, 0.0, torch.float32))
        sp = torch.cat(spread)
        rep.notes.append(f"attention score range per row (max - min): median {sp.median():.3g}, max {sp.max():.3g}; "
                         f"probabilities below 2^-24 of the row max: {torch.cat(tiny_p).mean():.1%}")
        return sp
    finally:
        G.set_stop_after(eng, 0)


@pytest.mark.parametrize("kind,B", [("ref", 301), ("offset", 24), ("peaked", 24)])
@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
def test_kernels_vs_float64(dtype, kind, B):
    """reference scale at B=301 (odd B, several waves of CTAs, both sweep directions); the row-offset and peaked-attention
    weight sets at a small batch"""
    eng, sd, spec, m = engine(kind, dtype)
    vo, t = O.RICO25, 42
    ids = mixed_ids(B, vo, 11)
    ids_d = ids.cuda()
    table = eng.adaln_table()
    rep = Report(f"{kind} weights, {dtype}, B={B}, t={t}")
    spread = check_kernels(eng, m, ids, lambda l, sl: table[l][t], lambda: eng.step(ids_d, t, t, {"name": "deterministic"}), dtype, rep)
    rep.finish()
    if kind == "peaked":
        assert spread.max() > 10.0, "the peaked weight set no longer reaches peaked attention rows"


@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
def test_kernels_vs_float64_per_layout_timesteps(dtype):
    """predict_start at per-layout timesteps: the t_layout rows of the embedding's AdaLN_0 and of the FF2 AdaLN epilogue"""
    eng, sd, spec, m = engine("ref", dtype)
    vo, B = O.RICO25, 24
    ids = mixed_ids(B, vo, 12)
    t = torch.randint(0, spec.T, (B,), generator=torch.Generator().manual_seed(4))
    t[0], t[1] = 0, spec.T - 1
    ids_d, t_d = ids.cuda(), t.cuda()
    table = eng.adaln_table()
    rep = Report(f"predict_start, per-layout t, {dtype}, B={B}")
    check_kernels(eng, m, ids, lambda l, sl: table[l][t[sl]][:, None], lambda: eng.predict_start(ids_d, t_d), dtype, rep)
    rep.finish()


def in_group_ids(B, vo, seed):
    """x_t of a real trajectory: every token from its own attribute's vocabulary (classes, PAD, MASK), MASK-heavy"""
    g = torch.Generator().manual_seed(seed)
    ids = torch.empty(B, vo.S, dtype=torch.long)
    for a in range(vo.n_attr):
        grp = torch.tensor(vo.group_full_ids(a))
        pick = grp[torch.randint(0, len(grp), (B, vo.n_elem), generator=g)]
        ids[:, a::vo.n_attr] = torch.where(torch.rand(B, vo.n_elem, generator=g) < 0.4, vo.mask_id, pick)
    return ids


@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_kernels_vs_float64_other_vocab_shapes(shape, dtype):
    """vocabularies ldm_create accepts beyond rico25 / publaynet: the kernel checks, then the step epilogue (posterior + draw on
    caller-given logits) bit-exact against O.draw, through the generic kernel (log-prob output) and the group kernel"""
    vo, L = SHAPES[shape]
    eng, sd, spec, m = engine("ref", dtype, vo, L)
    B, t = 24, 17
    ids = mixed_ids(B, vo, 13)
    ids_d = ids.cuda()
    table = eng.adaln_table()
    rep = Report(f"{shape}, {dtype}, B={B}, t={t}")
    check_kernels(eng, m, ids, lambda l, sl: table[l][t], lambda: eng.step(ids_d, t, t, {"name": "deterministic"}), dtype, rep)
    rep.finish()

    orc = O.Oracle(vo, spec, sd)
    g = torch.Generator().manual_seed(3)
    modes = [("deterministic", {}), ("random", {}), ("top_p", {"top_p": 0.8}), ("gumbel", {})]
    if vo.n_cat >= 3:
        modes.append(("top_k", {"top_k": 3}))
    seed = 7
    for step, (t_model, t_post) in enumerate(((60, 58), (5, 5), (0, 0))):
        x_in = in_group_ids(B, vo, 20 + step)
        logits = torch.randn(B, vo.S, vo.C, generator=g) * 3.0
        lp_o = orc.logprob_from_logits(logits, x_in, t_post)
        for name, extra in modes:
            cfg = O.SamplingCfg(name=name, temperature=0.9, top_p=extra.get("top_p", 0.9), top_k=extra.get("top_k", 5))
            u = O.uniforms(seed, step, 0, 0, B, vo.S, vo.C) if name != "deterministic" else None
            ug = O.uniforms(seed, step, 1, 0, B, vo.S, vo.C) if name == "gumbel" else None
            want = O.draw(lp_o, cfg, u, ug)
            cfg_d = dict(name=name, temperature=0.9, **extra)
            out, _, lp = eng.step(x_in.cuda(), t_model, t_post, cfg_d, seed=seed, step_ctr=step, want_logprob=True, logits_in=logits.cuda())
            assert (lp.cpu() - lp_o).abs().max() < 1e-4, f"{name} t={t_model}: log-probs"
            assert torch.equal(out.cpu(), want), f"{name} t={t_model}: {(out.cpu() != want).sum().item()} ids differ"
            out2, _, _ = eng.step(x_in.cuda(), t_model, t_post, cfg_d, seed=seed, step_ctr=step, logits_in=logits.cuda())
            assert torch.equal(out2.cpu(), want), f"{name} t={t_model} (group kernel): {(out2.cpu() != want).sum().item()} ids differ"
