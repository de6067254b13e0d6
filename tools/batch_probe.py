import os, sys, time, json
import torch
sys.path.insert(0, os.getcwd())
from layoutdm_b200 import Engine, Vocab, timestep_plan
from layoutdm_b200.synthetic import random_state_dict
vocab = Vocab.for_dataset("rico25")
eng = Engine.from_state_dict(random_state_dict(vocab), vocab)
cfg = {"name": "random", "temperature": 1.0}
plan = timestep_plan(100, 100)
out = {}
for B in (132, 264, 528, 1024, 2048):
    for _ in range(2): eng.sample_loop(B, plan, cfg, seed=1)
    torch.cuda.synchronize(); t0 = time.perf_counter()
    n = 3
    for i in range(n): eng.sample_loop(B, plan, cfg, seed=2 + i)
    torch.cuda.synchronize(); dt = (time.perf_counter() - t0) / n
    out[B] = {"ms": round(dt * 1e3, 1), "layouts_per_s": round(B / dt, 1), "us_per_layout_step": round(dt * 1e6 / 100 / B, 3)}
print(json.dumps(out))
