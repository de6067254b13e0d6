"""
Generates the fixtures under tests/golden/blocks/*.npz: make_golden.py's recording of the UNMODIFIED reference (on CPU, under the
injected-noise contract, checked against the oracle while doing so), for models whose denoiser Blocks have other settings than
adalayernorm + relu: instance-norm AdaIN, sinusoidal or no timestep embedding, GELU feed-forwards, one of them at 50 elements and
one with the vanilla q_type.  They live in their own directory so that the default fixture set of tests/golden/*.npz stays as it is.
Run where the reference checkout is available:

    python tests/golden/make_block_golden.py [case names]

make_golden.run_case runs unchanged; what differs is what it is handed: weights with the norm1 keys of the case's timestep_type
(block_refs.block_weights), the reference built with the case's Block settings (block_refs.build_reference), the oracle with
those settings (block_refs.BlockOracle) and the output directory.  The fixture's meta records the settings.
"""
from __future__ import annotations

import dataclasses
import functools
import json
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import block_refs as BR  # noqa: E402
import make_golden as MG  # noqa: E402
import ref_harness as rh  # noqa: E402
from oracle import layoutdm_oracle as O  # noqa: E402

OUT = os.path.join(HERE, "blocks")
CASES = [
    dict(name="rico25_adainnorm_relu_uncond", dataset="rico25", q_type="constrained", samp="random", cond=None, scale=2.0,
         timestep_type="adainnorm", activation="relu"),
    dict(name="rico25_adalayernorm_abs_gelu_c", dataset="rico25", q_type="constrained", samp="top_p", cond="c", scale=2.0,
         timestep_type="adalayernorm_abs", activation="gelu"),
    dict(name="publaynet_none_gelu2_cwh", dataset="publaynet", q_type="constrained", samp="random", cond="cwh", scale=3.0,
         timestep_type=None, activation="gelu2"),
    dict(name="rico25_L50_adainnorm_abs_gelu", dataset="rico25", q_type="constrained", samp="random", cond=None, scale=2.0,
         timestep_type="adainnorm_abs", activation="gelu", n_elem=50),
    dict(name="rico25_vanilla_adainnorm_gelu2", dataset="rico25", q_type="vanilla", samp="random", cond=None, scale=2.0,
         timestep_type="adainnorm", activation="gelu2"),
]
for c in CASES:
    c.update(T=100, T_eval=20, B=2)


def _namespace(base, **override):
    """base's attributes, with `override` in front"""
    ns = types.SimpleNamespace(**{k: getattr(base, k) for k in dir(base) if not k.startswith("__")})
    for k, v in override.items():
        setattr(ns, k, v)
    return ns


def run_case(c):
    n_elem = c.get("n_elem", 25)
    tt, act = c["timestep_type"], c["activation"]
    MG.O = _namespace(O, RICO25=dataclasses.replace(O.RICO25, n_elem=n_elem), PUBLAYNET=dataclasses.replace(O.PUBLAYNET, n_elem=n_elem),
                      make_weights=functools.partial(BR.block_weights, timestep_type=tt),
                      Oracle=functools.partial(BR.BlockOracle, timestep_type=tt, activation=act))
    MG.rh = _namespace(rh, build_reference=functools.partial(BR.build_reference, timestep_type=tt, activation=act, max_seq_length=n_elem),
                       synthetic_layouts=functools.partial(rh.synthetic_layouts, max_elem=n_elem))
    MG.HERE = OUT
    os.makedirs(OUT, exist_ok=True)
    MG.run_case(c)
    path = os.path.join(OUT, c["name"] + ".npz")
    z = dict(np.load(path))
    meta = json.loads(str(z["meta"]))
    meta.update(n_elem=n_elem, timestep_type=tt, activation=act, diffusion_step=c["T"])
    z["meta"] = json.dumps(meta)
    np.savez_compressed(path, **z)


if __name__ == "__main__":
    torch.set_num_threads(8)
    only = sys.argv[1:]
    for c in CASES:
        if not only or c["name"] in only:
            run_case(c)
