"""
Generates the fixtures under tests/golden/token_layouts/*.npz: make_golden.py's recording of the UNMODIFIED reference (on CPU,
under the injected-noise contract, checked against the oracle while doing so), for models trained with tokenizer settings other
than the default: a shared xywh bbox vocabulary, var_order c-w-h-x-y, 16 or 64 bins.  They live in their own directory so that
the default fixture set of tests/golden/*.npz stays as it is.  Run where the reference checkout is available:

    python tests/golden/make_token_layout_golden.py [case names]

make_golden.run_case runs unchanged; what differs is what it is handed: the oracle's vocabulary with the slot layout of the
case's tokenizer settings (token_layout_refs.LayoutSpec), its refinement table, the reference built with those settings
(token_layout_refs.build_reference) and the output directory.  The fixture's meta records the configuration.
"""
from __future__ import annotations

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

import make_golden as MG  # noqa: E402
import ref_harness as rh  # noqa: E402
import token_layout_refs as TL  # noqa: E402
from oracle import layoutdm_oracle as O  # noqa: E402

OUT = os.path.join(HERE, "token_layouts")
CASES = [
    dict(name="rico25_xywh_uncond_random", config="rico25_xywh", samp="random", cond=None, scale=2.0),
    dict(name="publaynet_cwhxy_c_top_p", config="publaynet_cwhxy", samp="top_p", cond="c", scale=3.0),
    dict(name="rico25_bins16_refinement", config="rico25_bins16", samp="random", cond="refinement", scale=2.0,
         refine=dict(refine_lambda=3.0, refine_mode="uniform", refine_offset_ratio=0.1)),
    dict(name="rico25_xywh_bins64_cwh", config="rico25_xywh_bins64", samp="random", cond="cwh", scale=2.0),
    dict(name="rico25_vanilla_xywh_cwhxy_uncond", config="rico25_vanilla_xywh_cwhxy", samp="random", cond=None, scale=2.0),
]
for c in CASES:
    dataset, _, _, _, q_type = TL.CONFIGS[c["config"]]
    c.update(dataset=dataset, q_type=q_type, T=100, T_eval=20, B=2)


def _namespace(base, **override):
    """base's attributes, with `override` in front"""
    ns = types.SimpleNamespace(**{k: getattr(base, k) for k in dir(base) if not k.startswith("__")})
    for k, v in override.items():
        setattr(ns, k, v)
    return ns


def run_case(c):
    spec = TL.spec_of(c["config"])
    _, shared, order, bins, _ = TL.CONFIGS[c["config"]]
    MG.O = _namespace(O, RICO25=spec, PUBLAYNET=spec, refinement_table=TL.refinement_table)
    MG.rh = _namespace(rh, build_reference=functools.partial(TL.build_reference, shared_bbox_vocab=shared, var_order=order,
                                                             num_bin_bboxes=bins))
    MG.HERE = OUT
    os.makedirs(OUT, exist_ok=True)
    MG.run_case(c)
    path = os.path.join(OUT, c["name"] + ".npz")
    z = dict(np.load(path))
    meta = json.loads(str(z["meta"]))
    meta.update(config=c["config"], shared_bbox_vocab=shared, var_order=order, num_bin_bboxes=bins)
    z["meta"] = json.dumps(meta)
    np.savez_compressed(path, **z)


if __name__ == "__main__":
    torch.set_num_threads(8)
    only = sys.argv[1:]
    for c in CASES:
        if not only or c["name"] in only:
            run_case(c)
