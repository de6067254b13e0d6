"""
Generates the fixtures under tests/golden/long_layouts/*.npz: make_golden.py's recording of the UNMODIFIED reference (on CPU,
under the injected-noise contract, checked against the oracle while doing so), for models of dataset.max_seq_length = 50
(S = 250 tokens: two 128-row tiles per layout in the kernels).  They live in their own directory so that the 25-element
fixture set of tests/golden/*.npz stays as it is.  Run in the build container only:

    python tests/golden/make_long_golden.py [case names]

make_golden.run_case runs unchanged; what differs is what it is handed: the oracle's vocabularies at n_elem = 50, the reference
built at max_seq_length = 50 (long_layout_refs.build_reference), synthetic cond layouts of up to 50 elements, and the output
directory.  The fixture's meta records n_elem.
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

import long_layout_refs  # noqa: E402
import make_golden as MG  # noqa: E402
import ref_harness as rh  # noqa: E402
from oracle import layoutdm_oracle as O  # noqa: E402

N_ELEM = 50
OUT = os.path.join(HERE, "long_layouts")
CASES = [
    dict(name="rico25_L50_uncond_random", dataset="rico25", q_type="constrained", T=100, T_eval=20, B=2, samp="random", cond=None, scale=2.0),
    dict(name="publaynet_L50_c_top_p", dataset="publaynet", q_type="constrained", T=100, T_eval=20, B=2, samp="top_p", cond="c", scale=3.0),
    dict(name="rico25_L50_refinement", dataset="rico25", q_type="constrained", T=100, T_eval=20, B=2, samp="random", cond="refinement",
         scale=2.0, refine=dict(refine_lambda=3.0, refine_mode="uniform", refine_offset_ratio=0.1)),
]


def _namespace(base, **override):
    """base's attributes, with `override` in front"""
    ns = types.SimpleNamespace(**{k: getattr(base, k) for k in dir(base) if not k.startswith("__")})
    for k, v in override.items():
        setattr(ns, k, v)
    return ns


def run_case(c):
    MG.O = _namespace(O, RICO25=dataclasses.replace(O.RICO25, n_elem=N_ELEM), PUBLAYNET=dataclasses.replace(O.PUBLAYNET, n_elem=N_ELEM))
    MG.rh = _namespace(rh, build_reference=functools.partial(long_layout_refs.build_reference, max_seq_length=N_ELEM),
                       synthetic_layouts=functools.partial(rh.synthetic_layouts, max_elem=N_ELEM))
    MG.HERE = OUT
    os.makedirs(OUT, exist_ok=True)
    MG.run_case(c)
    path = os.path.join(OUT, c["name"] + ".npz")
    z = dict(np.load(path))
    meta = json.loads(str(z["meta"]))
    meta["n_elem"] = N_ELEM
    z["meta"] = json.dumps(meta)
    np.savez_compressed(path, **z)


if __name__ == "__main__":
    torch.set_num_threads(8)
    only = sys.argv[1:]
    for c in CASES:
        if not only or c["name"] in only:
            run_case(c)
