"""Per-kernel timing of a few denoising steps (CUDA events via ldm_profile_*):  B=1024 STEPS=6 python tools/gemm_probe.py"""
import os, sys, json
import torch
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from layoutdm_b200 import Engine, Vocab, timestep_plan
from layoutdm_b200.synthetic import random_state_dict
B = int(os.environ.get("B", "1024")); steps = int(os.environ.get("STEPS", "6"))
vocab = Vocab.for_dataset("rico25")
eng = Engine.from_state_dict(random_state_dict(vocab), vocab)
plan = timestep_plan(100, 100)[:steps]
cfg = {"name": "random", "temperature": 1.0}
eng.sample_loop(B, plan, cfg, seed=1); torch.cuda.synchronize()
eng.profile_begin(); eng.sample_loop(B, plan, cfg, seed=2); prof = eng.profile_end()
print(json.dumps({"B": B,
                  "us_per_launch": {k: round(v[0] * 1e3 / v[1], 1) for k, v in prof.items() if v[1]}}))
