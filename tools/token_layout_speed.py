"""Speed of the tokenizer settings other than the default vocabulary (the configurations of tests/golden/token_layouts: shared
xywh bbox vocabulary, c-w-h-x-y, 16 or 64 bins) against the default rico25 x-y-w-h c-x-y-w-h 32 bins (C = 155): the whole
sampling loop (unconditional, T = 100, random sampling, one CUDA graph, CUDA events), the configurations alternated, then the
per-category milliseconds of one profiled loop each.  Prints the card, its power limit and SM clock, and one JSON line.

The head GEMM computes the padded 160-column logits row whatever C is, so the denoiser does the same work; the draw kernels
evaluate fewer valid classes at small C; a shared vocabulary of more than 32 bins puts 64 classes in each bbox group and so
takes the all-classes draw kernel instead of the group kernel.  This tool measures what that amounts to.

    python tools/token_layout_speed.py [--B 1024] [--T 100] [--dtype fp16] [--reps 3]"""
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

# name -> (dataset, shared_bbox_vocab, var_order, num_bin_bboxes, q_type)
CONFIGS = {
    "default_rico25": ("rico25", "x-y-w-h", "c-x-y-w-h", 32, "constrained"),
    "rico25_xywh": ("rico25", "xywh", "c-x-y-w-h", 32, "constrained"),
    "publaynet_cwhxy": ("publaynet", "x-y-w-h", "c-w-h-x-y", 32, "constrained"),
    "rico25_bins16": ("rico25", "x-y-w-h", "c-x-y-w-h", 16, "constrained"),
    "rico25_xywh_bins64": ("rico25", "xywh", "c-x-y-w-h", 64, "constrained"),
    "rico25_vanilla_xywh_cwhxy": ("rico25", "xywh", "c-w-h-x-y", 16, "vanilla"),
}


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
    plan = timestep_plan(a.T, a.T)
    cfg = {"name": "random", "temperature": 1.0}
    engines, C = {}, {}
    for name, (dataset, shared, order, bins, q_type) in CONFIGS.items():
        vocab = Vocab.for_dataset(dataset, 25, bins, shared, order)
        C[name] = vocab.C
        engines[name] = Engine.from_state_dict(random_state_dict(vocab, num_timesteps=a.T, seed=0), vocab, num_timesteps=a.T,
                                               operand_dtype=a.dtype, q_type=q_type)
    run = lambda n: engines[n].sample_loop(a.B, plan, cfg, seed=10)
    for n in CONFIGS:                                   # warm-up: workspace, graph capture
        run(n)
    torch.cuda.synchronize()
    loop_ms = {n: [] for n in CONFIGS}
    for _ in range(a.reps):
        for n in CONFIGS:
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record(); run(n); e.record(); e.synchronize()
            loop_ms[n].append(s.elapsed_time(e))
    cat_ms = {}
    for n in CONFIGS:
        engines[n].profile_begin()
        run(n)
        cat_ms[n] = {k: round(ms, 3) for k, (ms, _) in engines[n].profile_end().items()}
    med = {n: sorted(v)[len(v) // 2] for n, v in loop_ms.items()}
    lps = {n: a.B / (med[n] / 1e3) for n in CONFIGS}
    print(json.dumps({"B": a.B, "T": a.T, "dtype": a.dtype, "sampling": "random", **card(), "C": C,
                      "loop_ms_median": med, "loop_ms_all": loop_ms, "layouts_per_s": lps,
                      "layouts_per_s_over_default": {n: lps[n] / lps["default_rico25"] for n in CONFIGS},
                      "profiled_loop_ms_per_category": cat_ms}))


if __name__ == "__main__":
    main()
