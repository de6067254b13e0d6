"""Speed of the tensor-core operand modes on the flagship workload (rico25 unconditional, T=100, batch 1024, random sampling,
random-init weights -- bench.py's main line): fp16 and the split "bf16x3" mode, alternated, `--runs` timed loops of each.
Prints the card and its power limit, layouts/s per run, and the per-category milliseconds of one profiled loop
(ldm_profile_begin / ldm_profile_end) per mode, as one JSON document.

    python tools/operand_mode_speed.py [--batch 1024] [--runs 2] [--modes fp16,bf16x3]"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card() -> dict:
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        info["power_limit_w"], info["max_sm_clock_mhz"] = float(q[0]), float(q[1])
    except (OSError, ValueError, IndexError, subprocess.TimeoutExpired):
        info["power_limit_w"] = None
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--modes", default="fp16,bf16x3")
    args = ap.parse_args()
    from layoutdm_b200 import Engine, Vocab, timestep_plan
    from layoutdm_b200.synthetic import random_state_dict

    T, B = 100, args.batch
    vocab = Vocab.for_dataset("rico25")
    sd = random_state_dict(vocab, num_timesteps=T, seed=0)
    plan = timestep_plan(T, T)
    cfg = {"name": "random", "temperature": 1.0}
    modes = args.modes.split(",")
    engines = {m: Engine.from_state_dict(sd, vocab, num_timesteps=T, operand_dtype=m) for m in modes}
    for m, eng in engines.items():                        # warm-up: graph capture, clocks
        for w in range(3):
            eng.sample_loop(B, plan, cfg, seed=100 + w)
    torch.cuda.synchronize()
    runs = {m: [] for m in modes}
    for r in range(args.runs):
        for m in modes:                                    # alternated, so drift hits both modes alike
            eng = engines[m]
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            ids = eng.sample_loop(B, plan, cfg, seed=1000 + r)
            e1.record()
            torch.cuda.synchronize()
            assert int(ids.max()) < vocab.mask_id, "MASK token survived the loop"
            runs[m].append(round(B / (e0.elapsed_time(e1) * 1e-3), 1))
    prof = {}
    for m, eng in engines.items():
        eng.profile_begin()
        eng.sample_loop(B, plan, cfg, seed=5)
        prof[m] = {k: {"ms": round(v[0], 2), "launches": v[1]} for k, v in eng.profile_end().items() if v[1] > 0}
    out = {"card": card(), "workload": f"rico25 unconditional, T={T}, batch={B}, random sampling, random-init weights",
           "layouts_per_s": runs, "profile_ms_per_loop": prof}
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
