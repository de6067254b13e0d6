"""Cost of following a model's weights: the device time of one ldm_load_weights (CUDA events over many back-to-back
reloads, warmed up) in fp16 and bf16x3, a whole reload from live CUDA parameters as a patched model does it (state_dict,
stacking on the GPU, ldm_load_weights; host clock to a synchronise), and the host time of the check `sample()` runs when
nothing changed.  rico25, T = 100, the paper's 4-layer denoiser.  Prints one JSON line with the card name and power limit.

    python tools/weight_reload_probe.py [--reps 200]"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import torch
from torch import nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from layoutdm_b200 import Engine, FusedMaskAndReplaceDiffusion, Vocab, _lib       # noqa: E402
from layoutdm_b200.synthetic import PREFIX, random_state_dict                     # noqa: E402

T = 100


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip()}


def module_from_state_dict(sd) -> nn.Module:
    """a module whose parameters carry the state_dict's names (the reference's CategoricalTransformer's 58 parameters)"""
    root = nn.Module()
    for key, v in sd.items():
        *path, leaf = key[len(PREFIX):].split(".")
        m = root
        for p in path:
            if not hasattr(m, p):
                m.add_module(p, nn.Module())
            m = getattr(m, p)
        m.register_parameter(leaf, nn.Parameter(v.clone()))
    return root


def load_weights_us(eng: Engine, reps: int) -> float:
    """device µs per ldm_load_weights: back-to-back reloads on one stream between two events"""
    w = {k: v.cuda() for k, v in Engine.pack_state_dict(random_state_dict(eng.vocab, num_timesteps=T, seed=1), eng.vocab).items()}
    ws = _lib.LdmWeights()
    for name in _lib._W_FIELDS:
        setattr(ws, name, w[name].data_ptr())
    stream = torch.cuda.current_stream()
    call = lambda: _lib.check(eng.lib.ldm_load_weights(eng._h, C.byref(ws), C.c_void_p(stream.cuda_stream)))
    for _ in range(10):
        call()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(reps):
        call()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) * 1e3 / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    a = ap.parse_args()
    vocab = Vocab.for_dataset("rico25")
    sd = random_state_dict(vocab, num_timesteps=T, seed=0)
    out = {**card()}
    for dtype in ("fp16", "bf16x3"):
        eng = Engine.from_state_dict(sd, vocab, num_timesteps=T, operand_dtype=dtype)
        out[f"ldm_load_weights_us_{dtype}"] = round(load_weights_us(eng, a.reps), 1)
        # a patched model's reload and its unchanged check, on live CUDA parameters
        module = module_from_state_dict(sd).cuda()
        fused = FusedMaskAndReplaceDiffusion(eng)
        fused.follow(module)
        for _ in range(5):
            fused.reload_weights()
        torch.cuda.synchronize()
        n = max(a.reps // 4, 10)
        t0 = time.perf_counter()
        for _ in range(n):
            fused.reload_weights()
        torch.cuda.synchronize()
        out[f"reload_from_module_us_{dtype}"] = round((time.perf_counter() - t0) * 1e6 / n, 1)
        reloads = fused.weight_reloads
        n = 20 * a.reps
        t0 = time.perf_counter()
        for _ in range(n):
            fused._follow_weights()
        out[f"unchanged_check_host_us_{dtype}"] = round((time.perf_counter() - t0) * 1e6 / n, 2)
        assert fused.weight_reloads == reloads, "the unchanged check reloaded"
        eng.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
