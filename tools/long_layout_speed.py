"""Speed of layouts of 50 elements (S = 250, two 128-row tiles per layout) against the default 25 (S = 125, one tile): the whole
sampling loop (rico25 unconditional, T = 100, random sampling, one CUDA graph, CUDA events), the two lengths alternated, then
the per-category milliseconds of one profiled loop each (per-launch CUDA events).  Prints the card, its power limit and SM
clock, and one JSON line.

Per layout-step the algorithmic FLOPs at S = 250 are 2.085x those at S = 125 (the GEMMs 2x, attention 4x), so about half the
layouts/s is expected; this tool measures it.

    python tools/long_layout_speed.py [--B 1024] [--T 100] [--dtype fp16] [--reps 3]"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from layoutdm_b200 import Engine, Vocab, timestep_plan                      # noqa: E402
from layoutdm_b200.synthetic import random_state_dict                        # noqa: E402


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"gpu": torch.cuda.get_device_name(0), "name_power_limit_sm_clock_max_sm_clock": q.stdout.strip()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=1024)
    ap.add_argument("--T", type=int, default=100)
    ap.add_argument("--dtype", default="fp16")
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    lengths = (25, 50)
    plan = timestep_plan(a.T, a.T)
    cfg = {"name": "random", "temperature": 1.0}
    engines = {}
    for n in lengths:
        vocab = Vocab.for_dataset("rico25", n)
        engines[n] = Engine.from_state_dict(random_state_dict(vocab, num_timesteps=a.T, seed=0), vocab, num_timesteps=a.T,
                                            operand_dtype=a.dtype)
    run = lambda n: engines[n].sample_loop(a.B, plan, cfg, seed=10)
    for n in lengths:                                  # warm-up: workspace, graph capture
        run(n)
    torch.cuda.synchronize()
    loop_ms = {n: [] for n in lengths}
    for _ in range(a.reps):
        for n in lengths:
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record(); run(n); e.record(); e.synchronize()
            loop_ms[n].append(s.elapsed_time(e))
    cat_ms = {}
    for n in lengths:
        engines[n].profile_begin()
        run(n)
        cat_ms[n] = {k: round(ms, 3) for k, (ms, _) in engines[n].profile_end().items()}
    med = {n: sorted(v)[len(v) // 2] for n, v in loop_ms.items()}
    lps = {n: a.B / (med[n] / 1e3) for n in lengths}
    print(json.dumps({"B": a.B, "T": a.T, "dtype": a.dtype, "sampling": "random", **card(),
                      "loop_ms_median": med, "loop_ms_all": loop_ms, "layouts_per_s": lps,
                      "layouts_per_s_50_over_25": lps[50] / lps[25], "profiled_loop_ms_per_category": cat_ms}))


if __name__ == "__main__":
    main()
