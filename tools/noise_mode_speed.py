"""Cost of noise="torch" (draws from torch's CUDA generator stream) against the default Philox contract: the whole sampling
loop (rico25, T = 100, one CUDA graph, CUDA events) and the draw kernel alone (per-launch CUDA events of the profiled loop,
category posterior_sample), the two modes alternated.  Prints one JSON line with the card name and power limit.

    python tools/noise_mode_speed.py [--B 1024] [--dtype fp16] [--reps 5] [--sampling random]"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from layoutdm_b200 import Engine, Vocab, timestep_plan                      # noqa: E402
from layoutdm_b200._lib import NOISE_KINDS, LdmNoise                        # noqa: E402
from layoutdm_b200.synthetic import random_state_dict                        # noqa: E402


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=1024)
    ap.add_argument("--T", type=int, default=100)
    ap.add_argument("--dtype", default="fp16")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sampling", default="random")
    a = ap.parse_args()
    vocab = Vocab.for_dataset("rico25")
    eng = Engine.from_state_dict(random_state_dict(vocab, num_timesteps=a.T, seed=0), vocab, num_timesteps=a.T, operand_dtype=a.dtype)
    plan = timestep_plan(a.T, a.T)
    cfg = {"name": a.sampling, "temperature": 1.0}
    noises = {"contract": None, "torch": LdmNoise(NOISE_KINDS["torch"], 123, 0, a.B)}
    run = lambda m: eng.sample_loop(a.B, plan, cfg, seed=10, noise=noises[m])
    for m in noises:                                   # warm-up: capture both graphs
        run(m)
    torch.cuda.synchronize()
    loop_ms = {m: [] for m in noises}
    for _ in range(a.reps):
        for m in noises:
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record(); run(m); e.record(); e.synchronize()
            loop_ms[m].append(s.elapsed_time(e))
    draw_ms = {}
    for m in noises:
        eng.profile_begin()
        run(m)
        prof = eng.profile_end()
        ms, n = prof["posterior_sample"]
        draw_ms[m] = ms / max(n, 1)
    med = {m: sorted(v)[len(v) // 2] for m, v in loop_ms.items()}
    print(json.dumps({"B": a.B, "T": a.T, "dtype": a.dtype, "sampling": a.sampling, **card(),
                      "loop_ms_median": med, "loop_ms_all": loop_ms, "layouts_per_s": {m: a.B / (v / 1e3) for m, v in med.items()},
                      "draw_kernel_ms": draw_ms, "torch_over_contract_loop": med["torch"] / med["contract"],
                      "torch_over_contract_draw": draw_ms["torch"] / draw_ms["contract"]}))


if __name__ == "__main__":
    main()
