"""Speed of the denoiser block settings other than the default adalayernorm + relu (the reference Block's timestep_type /
activation): the whole sampling loop (rico25 unconditional, T = 100, random sampling, one CUDA graph, CUDA events) of each
variant alternated with the default, the median of --reps runs each, then the per-category milliseconds of one profiled loop.
Prints the card, its power limit and SM clock, and one JSON line.

None and the *_abs types only fill the AdaLN table differently and run the default kernels.  GELU / GELU2 change FF1's
epilogue.  The instance-norm types add one pass per layer over the fp32 rows (instance_norm_kernel, profiled under
"embed_adaln") and launch the embedding in every step instead of fusing it into the previous draw.

    python tools/block_variant_speed.py [--B 1024] [--T 100] [--dtype fp16] [--reps 3]"""
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

DEFAULT = ("adalayernorm", "relu")
VARIANTS = [(None, "relu"), ("adalayernorm_abs", "relu"), ("adalayernorm", "gelu"), ("adalayernorm", "gelu2"), ("adainnorm", "relu"),
            ("adainnorm_abs", "gelu")]


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
    vocab = Vocab.for_dataset("rico25")
    name = lambda v: f"{v[0]}+{v[1]}"
    engines = {}
    for tt, act in [DEFAULT] + VARIANTS:
        sd = random_state_dict(vocab, num_timesteps=a.T, seed=0, timestep_type=tt)
        engines[name((tt, act))] = Engine.from_state_dict(sd, vocab, num_timesteps=a.T, operand_dtype=a.dtype, timestep_type=tt, activation=act)
    run = lambda n: engines[n].sample_loop(a.B, plan, cfg, seed=10)
    for n in engines:                                   # warm-up: workspace, graph capture
        run(n)
    torch.cuda.synchronize()
    loop_ms = {n: [] for n in engines}
    for _ in range(a.reps):
        for v in VARIANTS:                              # each variant right after the default
            for n in (name(DEFAULT), name(v)):
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record(); run(n); e.record(); e.synchronize()
                loop_ms[n].append(s.elapsed_time(e))
    cat_ms = {}
    for n in engines:
        engines[n].profile_begin()
        run(n)
        cat_ms[n] = {k: round(ms, 3) for k, (ms, _) in engines[n].profile_end().items()}
    med = {n: sorted(v)[len(v) // 2] for n, v in loop_ms.items()}
    lps = {n: a.B / (med[n] / 1e3) for n in engines}
    print(json.dumps({"B": a.B, "T": a.T, "dtype": a.dtype, "dataset": "rico25", "cond": None, "sampling": "random", **card(),
                      "loop_ms_median": med, "loop_ms_all": loop_ms, "layouts_per_s": lps,
                      "layouts_per_s_over_default": {n: lps[n] / lps[name(DEFAULT)] for n in engines},
                      "profiled_loop_ms_per_category": cat_ms}))


if __name__ == "__main__":
    main()
