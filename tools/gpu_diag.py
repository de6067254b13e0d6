"""Stage-by-stage bring-up diagnostic for the CUDA path (needs an H100):
    python tools/gpu_diag.py [--dtype fp16|bf16] [--out diag.jsonl]
For every kernel of the per-step launch sequence it stops the denoiser right after that kernel (ldm_debug_* taps),
reads the buffers it wrote and compares them with the oracle's same-rounding intermediates.  Results are appended
to a JSON-lines file after every stage, so a crash still leaves the partial record."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [REPO, os.path.join(REPO, "tests")]

from layoutdm_b200 import Engine, Vocab  # noqa: E402
from oracle import layoutdm_oracle as O  # noqa: E402
import gpu_helpers as G  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dtype", default="fp16")
    ap.add_argument("--out", default="diag.jsonl")
    ap.add_argument("--B", type=int, default=3)
    ap.add_argument("--scale", type=float, default=2.0)
    args = ap.parse_args()
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    f = open(args.out, "a")

    def rec(**kw):
        kw["dtype"] = args.dtype
        f.write(json.dumps(kw) + "\n"); f.flush()
        print(kw, flush=True)

    vo, spec = O.RICO25, O.ModelSpec()
    sd = O.make_weights(vo, spec, seed=7, scale=args.scale)
    odt = torch.float16 if args.dtype == "fp16" else torch.bfloat16
    t0 = time.time()
    eng = Engine.from_state_dict(sd, Vocab.for_dataset("rico25"), num_timesteps=spec.T, operand_dtype=args.dtype)
    rec(stage="create", seconds=time.time() - t0, device=torch.cuda.get_device_name(0))

    # schedule + AdaLN tables
    sch = eng.schedule_tables()
    osch = O.group_schedules(spec.T, vo)
    worst = 0.0
    for g in range(5):
        for r, name in enumerate(O.SCHED_NAMES):
            a, b = sch[g, r, : osch[g][name].shape[0]], osch[g][name]
            fin = torch.isfinite(b)
            assert (torch.isfinite(a) == fin).all()
            worst = max(worst, (a[fin] - b[fin]).abs().max().item())
    rec(stage="schedule", max_abs=worst)
    ad = eng.adaln_table()
    oad = torch.stack([O.adaln_table(sd, spec, l) for l in range(spec.layers)])
    rec(stage="adaln_table", max_abs=(ad - oad).abs().max().item())

    B, t = args.B, 42
    g = torch.Generator().manual_seed(5)
    ids = torch.randint(0, vo.C, (B, vo.S), generator=g)
    ids[0] = vo.mask_id
    taps = {}
    with torch.no_grad():
        ologits = O.denoiser_forward(sd, ids, t, vo, spec, operand_dtype=odt, taps=taps)
        ologits32 = O.denoiser_forward(sd, ids, t, vo, spec)
    ids_d = ids.cuda()
    samp = {"name": "deterministic"}
    S = vo.S

    def cmp(name, got, want):
        got, want = got.float(), want.float()
        d = (got - want).abs()
        bad = ~torch.isfinite(got)
        rec(stage=name, max_abs=float(d[~bad].max()) if (~bad).any() else None, mean_abs=float(d[~bad].mean()) if (~bad).any() else None,
            ref_max=float(want.abs().max()), nonfinite=int(bad.sum()))

    stage = 0
    def run(n):
        G.set_stop_after(eng, n)
        eng.step(ids_d, t, t, samp)
        torch.cuda.synchronize()

    try:
        stage = 1; run(stage)
        cmp("embed.x32", G.debug_read(eng, "x32", B)[:, :S], taps["x0"])
        cmp("embed.x16", G.debug_read(eng, "x16", B)[:, :S], taps["x0"].to(odt))
        for l in range(spec.layers):
            stage += 1; run(stage)
            q, k, v, pad = G.unpack_qkv(G.debug_read(eng, "qkv16", B))
            cmp(f"L{l}.qkv.q", q, taps[f"q{l}"]); cmp(f"L{l}.qkv.k", k, taps[f"k{l}"]); cmp(f"L{l}.qkv.v", v, taps[f"v{l}"])
            rec(stage=f"L{l}.qkv.pad_cols", max_abs=pad)
            stage += 1; run(stage)
            a16 = G.debug_read(eng, "att16", B)[:, :S].view(B, S, 8, 64)
            cmp(f"L{l}.attention", a16[..., :58].reshape(B, S, 464), taps[f"att{l}"])
            # column 58 of a head = the normalised ones column (1.0), 59..63 zeros
            rec(stage=f"L{l}.attention.pad_cols", max_abs=float(max((a16[..., 58].float() - 1.0).abs().max(), a16[..., 59:].abs().max())))
            stage += 1; run(stage)      # out-proj GEMM with fused residual + LayerNorm2
            cmp(f"L{l}.outproj.y32", G.debug_read(eng, "y32", B)[:, :S], taps[f"y{l}"])
            cmp(f"L{l}.outproj.z16", G.debug_read(eng, "z16", B)[:, :S], taps[f"z{l}"])
            stage += 1; run(stage)
            cmp(f"L{l}.ff1.hid16", G.debug_read(eng, "hid16", B)[:, :S], taps[f"hid{l}"])
            stage += 1; run(stage)      # FF2 GEMM with fused residual + AdaLN / head LN
            if l + 1 < spec.layers:
                cmp(f"L{l}.ff2.x32", G.debug_read(eng, "x32", B)[:, :S], taps[f"x{l + 1}"])
            else:
                cmp(f"L{l}.ff2.hn16", G.debug_read(eng, "z16", B)[:, :S], taps["hn"])
        G.set_stop_after(eng, 0)
        _, lg, _ = eng.step(ids_d, t, t, samp, want_logits=True)
        torch.cuda.synchronize()
        cmp("logits.vs_same_rounding", lg.cpu(), ologits)
        cmp("logits.vs_fp32", lg.cpu(), ologits32)
    except Exception as e:  # noqa: BLE001
        rec(stage=f"FAILED_at_launch_{stage}", error=repr(e))
        raise
    finally:
        f.close()


if __name__ == "__main__":
    main()
