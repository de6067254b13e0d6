"""Precision evidence for the 16-bit tensor-core operands (needs an H100):
    python tools/precision_report.py [--out precision.json]
For weight scales 1 (the reference's init scale, base_model.py:108-116), 2 and 3 ("peaked" stress weights) and both operand
dtypes (fp16, bf16 and the split bf16x3 pairs) it reports the max-abs logit error against the fp32 oracle and the same-rounding oracle, the largest magnitude every
16-bit activation buffer reaches during a step (fp16 overflows at 65504; a bf16x3 buffer is read as hi + lo) and the number of
non-finite values."""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [REPO, os.path.join(REPO, "tests")]

from layoutdm_b200 import Engine, Vocab  # noqa: E402
from oracle import layoutdm_oracle as O  # noqa: E402
import gpu_helpers as G  # noqa: E402
import split_refs as SR  # noqa: E402


def read16(eng, name, B):
    """a 16-bit activation buffer as float32 values (the split mode: hi + lo of both planes)"""
    if eng.operand_dtype != "bf16x3":
        return G.debug_read(eng, name, B)
    hi = G.debug_read(eng, name, B, raw=True).view(torch.bfloat16)
    lo = G.debug_read(eng, name + "_lo", B, raw=True).view(torch.bfloat16)
    return (hi.double() + lo.double()).float()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="precision.json")
    ap.add_argument("--B", type=int, default=32)
    args = ap.parse_args()
    vo, spec = O.RICO25, O.ModelSpec()
    g = torch.Generator().manual_seed(0)
    ids = torch.randint(0, vo.C, (args.B, vo.S), generator=g)
    ids[0] = vo.mask_id
    ids[1, 60:] = vo.pad_id
    rows = []
    for dtype in ("fp16", "bf16", "bf16x3"):
        for scale in (1.0, 2.0, 3.0):
            sd = O.make_weights(vo, spec, seed=0, scale=scale)
            eng = Engine.from_state_dict(sd, Vocab.for_dataset("rico25"), num_timesteps=spec.T, operand_dtype=dtype)
            odt = {"fp16": torch.float16, "bf16": torch.bfloat16}.get(dtype)
            worst32 = worst_same = max_logit = 0.0
            for t in (0, 42, 99):
                _, lg, _ = eng.step(ids.cuda(), t, t, {"name": "deterministic"}, want_logits=True)
                with torch.no_grad():
                    ref = O.denoiser_forward(sd, ids, t, vo, spec)
                    same = (O.denoiser_forward(sd, ids, t, vo, spec, operand_dtype=odt) if odt is not None
                            else SR.denoiser_forward_bf16x3(sd, ids, t, vo, spec))
                worst32 = max(worst32, (lg.cpu() - ref).abs().max().item())
                worst_same = max(worst_same, (lg.cpu() - same).abs().max().item())
                max_logit = max(max_logit, ref.abs().max().item())
            # largest magnitude of every 16-bit buffer over the launches of one step (stop-after taps)
            peak, nonfinite = {}, 0
            n_launch = 1 + 5 * spec.layers + 1
            stage_buf = {}
            k = 1
            stage_buf[k] = ["x16"]
            for l in range(spec.layers):
                for names in (["qkv16"], ["att16"], ["z16"], ["hid16"], ["x16"] if l + 1 < spec.layers else ["z16"]):
                    k += 1
                    stage_buf[k] = names
            for k, names in stage_buf.items():
                G.set_stop_after(eng, k)
                eng.step(ids.cuda(), 42, 42, {"name": "deterministic"})
                torch.cuda.synchronize()
                for nme in names:
                    v = read16(eng, nme, args.B)
                    nonfinite += int((~torch.isfinite(v)).sum())
                    peak[nme] = max(peak.get(nme, 0.0), float(v[torch.isfinite(v)].abs().max()))
            G.set_stop_after(eng, 0)
            rows.append({"operand_dtype": dtype, "weight_scale": scale, "max_abs_logit": round(max_logit, 3), "logit_err_vs_fp32": worst32,
                         "logit_err_rel": worst32 / max(1.0, max_logit), "logit_err_vs_same_rounding": worst_same,
                         "peak_abs_16bit_buffers": {k: round(v, 2) for k, v in peak.items()}, "nonfinite": nonfinite,
                         "fp16_headroom_x": round(65504.0 / max(peak.values()), 1)})
            print(rows[-1], flush=True)
            eng.close()
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    json.dump({"B": args.B, "timesteps": [0, 42, 99], "rows": rows}, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
