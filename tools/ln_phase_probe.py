"""Where a tile's time goes in the LN GEMMs (out-projection, FF2): median per-phase µs from %globaltimer stamps.

Builds the library with -DLDM_LN_PROBE into its own directory (--out, default a temporary one; reused while newer than the
sources), runs single denoising steps at B layouts, and after each step reads the stamps of the step's last out-projection
and FF2 launch (rank 0 of the first 8 CTA pairs, up to 32 tiles each).  Phases of a tile t and row half w, in chain order:
  mma: res wait    mainloop done -> the half's residual rows have landed (res_full passed)
  mma: y pass      res_full passed -> y written, buf_full arrived
  epi: pick-up     buf_full arrived -> the epilogue has passed buf_full
  epi: peer sums   -> the peer's row sums have landed (xs_full passed)
  epi: variance    -> the peer's variance partials have landed (xv_full passed)
  epi: normalise   -> rstd, the y store's read, the normalise pass done
  copy: fp32 store -> the normalised rows' bulk store has read the buffer (bulk_wait_group_read returned)
  copy: issue      -> the next tile's residual rows issued
  res: load        next residual issued -> res_full of tile t + 1 passed
and the tile period (mainloop done to mainloop done; normalise done to normalise done).  Needs an H100.
  python tools/ln_phase_probe.py [--batch 1024] [--steps 6] [--dtype fp16] [--out DIR]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import __graft_entry__ as G  # noqa: E402
from layoutdm_b200 import _lib  # noqa: E402

STAMPS = ("main", "res", "y", "buf", "xs", "xv", "norm", "wait", "next")   # gemm_tc.cuh LNP_*
PAIRS, TILES = 8, 32                                                      # kLnProbePairs, kLnProbeTiles
PHASES = (("mma: res wait", "main", "res"), ("mma: y pass", "res", "y"), ("epi: pick-up", "y", "buf"),
          ("epi: peer sums", "buf", "xs"), ("epi: variance", "xs", "xv"), ("epi: normalise", "xv", "norm"),
          ("copy: fp32 store", "norm", "wait"), ("copy: issue", "wait", "next"))


def build_variant(out):
    out = os.path.abspath(out)
    os.makedirs(out, exist_ok=True)
    lib = os.path.join(out, "libldm_b200_lnprobe.so")
    srcs = [os.path.join(G.CSRC, f) for f in sorted(os.listdir(G.CSRC))] + [os.path.join(REPO, "include", "ldm_b200.h")]
    if G._stale(lib, srcs):
        nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
        subprocess.check_call([nvcc] + G.NVCC_FLAGS + ["-DLDM_LN_PROBE", "-o", lib, os.path.join(G.CSRC, "ldm_b200.cu")], cwd=out)
    return lib


def phases(st):
    """st: [samples, pairs, tiles, 2 halves, stamps] ns (0 = not recorded) -> {half: {phase: median µs}}"""
    k = {n: i for i, n in enumerate(STAMPS)}
    out = {}
    for w in range(2):
        s = st[:, :, :, w].astype(np.float64)
        row = {}

        def med(a, b):
            ok = (a > 0) & (b > 0)
            return round(float(np.median((b - a)[ok])) / 1e3, 2) if ok.any() else None
        for name, a, b in PHASES:
            row[name] = med(s[..., k[a]], s[..., k[b]])
        row["res: load"] = med(s[:, :, :-1, k["next"]], s[:, :, 1:, k["res"]])
        row["period: mainloop"] = med(s[:, :, :-1, k["main"]], s[:, :, 1:, k["main"]])
        row["period: epilogue"] = med(s[:, :, :-1, k["norm"]], s[:, :, 1:, k["norm"]])
        out[f"half {w}"] = {n: v for n, v in row.items() if v is not None}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--dtype", default="fp16", choices=["fp16", "bf16"])
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    _lib.LIB_PATH = build_variant(a.out or tempfile.mkdtemp(prefix="ln_probe_"))
    from layoutdm_b200 import Engine, Vocab
    from layoutdm_b200.synthetic import random_state_dict
    lib = _lib.load()
    lib.ldm_probe_ln_read.restype, lib.ldm_probe_ln_read.argtypes = C.c_int64, [C.c_void_p, C.c_int64]
    vocab = Vocab.for_dataset("rico25")
    eng = Engine.from_state_dict(random_state_dict(vocab), vocab, operand_dtype=a.dtype)
    ids = torch.full((a.batch, vocab.S), vocab.mask_id, dtype=torch.long, device="cuda")
    buf = np.zeros((2, PAIRS, TILES, 2, len(STAMPS)), dtype=np.uint64)
    samples = []
    for i in range(a.steps + 1):
        eng.step(ids, 50, 49, {"name": "random", "temperature": 1.0})
        assert lib.ldm_probe_ln_read(C.c_void_p(buf.ctypes.data), buf.nbytes) == buf.nbytes
        if i > 0:                                                     # the first step warms up
            samples.append(buf.copy())
    st = np.stack(samples)
    props = torch.cuda.get_device_properties(0)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"device": props.name, "nvidia_smi": smi, "B": a.batch, "dtype": a.dtype, "steps": a.steps,
                      "out_projection": phases(st[:, 0]), "ff2": phases(st[:, 1])}, indent=1))
    eng.close()


if __name__ == "__main__":
    main()
