"""CPU: host-side mirror logic and the C-ABI surface (no compute calls -- there is no GPU here)."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

import layoutdm_b200 as L
from layoutdm_b200 import _lib
from layoutdm_b200.engine import Engine, sampling_struct
from oracle import layoutdm_oracle as O

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_package_does_not_import_oracle():
    for f in os.listdir(os.path.join(REPO, "layoutdm_b200")):
        if f.endswith(".py"):
            src = open(os.path.join(REPO, "layoutdm_b200", f)).read()
            assert "oracle" not in src.replace("# oracle", ""), f"{f} must not reference the oracle"


@pytest.mark.parametrize("T,T_eval,td", [(100, 100, 0.0), (100, 50, 0.0), (100, 30, 0.05), (200, 200, 0.0), (100, 7, 0.2), (100, 1, 0.0)])
def test_timestep_plan_matches_oracle(T, T_eval, td):
    assert L.timestep_plan(T, T_eval, td) == O.timestep_plan(T, T_eval, td)


def test_timestep_plan_rejects_too_many_steps():
    with pytest.raises(AssertionError):
        L.timestep_plan(100, 101)


def test_decode_and_refinement_table_match_oracle():
    for vo, vl in ((O.RICO25, L.Vocab.for_dataset("rico25")), (O.PUBLAYNET, L.Vocab.for_dataset("publaynet"))):
        assert (vo.C, vo.S, vo.pad_id, vo.mask_id) == (vl.C, vl.S, vl.pad_id, vl.mask_id)
        g = torch.Generator().manual_seed(0)
        ids = torch.randint(0, vo.C, (16, vo.S), generator=g)
        a, b = O.decode_ids(ids, vo), L.decode_ids(ids, vl)
        for k in a:
            assert torch.equal(a[k], b[k])
        for mode in ("uniform", "gaussian", "negative"):
            ta = O.refinement_table(vo, O.linear_centers(), mode, 0.1, 3.0)
            tb = L.refinement_table(vl, L.linear_centers(), mode, 0.1, 3.0)
            assert torch.equal(ta, tb)
        # decode with explicit centres == linear decode when the centres are the linear ones
        c = L.decode_ids(ids, vl, L.linear_centers())
        assert torch.allclose(c["bbox"], b["bbox"], atol=1e-6)


def test_library_exports_every_declared_symbol():
    lib = _lib.load()
    hdr = open(os.path.join(REPO, "include", "ldm_b200.h")).read()
    declared = set(re.findall(r"\b(ldm_[a-z_0-9]+)\s*\(", hdr))
    assert declared == set(_lib.SIGNATURES), declared ^ set(_lib.SIGNATURES)
    for name in declared:
        assert hasattr(lib, name)
    assert b"sm_90a" in lib.ldm_version()


def test_struct_layout_matches_header(tmp_path):
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include "ldm_b200.h"\nint main(){printf("%zu %zu %zu %zu\\n", sizeof(LdmModelDesc), sizeof(LdmWeights), sizeof(LdmCond), sizeof(LdmSampling));return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", "-I", os.path.join(REPO, "include"), str(src), "-o", str(exe)])
    sizes = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert sizes == [ctypes.sizeof(_lib.LdmModelDesc), ctypes.sizeof(_lib.LdmWeights), ctypes.sizeof(_lib.LdmCond), ctypes.sizeof(_lib.LdmSampling)]


def test_no_cpu_fallback():
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    sd = O.make_weights(O.RICO25, O.ModelSpec(layers=1), seed=0)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        Engine.from_state_dict(sd, L.Vocab.for_dataset("rico25"))


def test_pack_state_dict_shapes_and_prefixes():
    spec = O.ModelSpec()
    sd = O.make_weights(O.RICO25, spec, seed=0)
    v = L.Vocab.for_dataset("rico25")
    w = Engine.pack_state_dict(sd, v)
    assert w["in_proj_w"].shape == (4, 3 * 464, 464) and w["pos_table"].shape == (125, 464) and w["head_w"].shape == (155, 464)
    assert torch.equal(w["pos_table"], O.positional_table(sd, O.RICO25, spec))
    # other prefixes a user may hand in (un-wrapped module, bare transformer)
    for new in ("model.transformer.", "transformer.", ""):
        sd2 = {k.replace("model.module.transformer.", new): t for k, t in sd.items()}
        w2 = Engine.pack_state_dict(sd2, v)
        assert torch.equal(w2["linear2_w"], w["linear2_w"])
    with pytest.raises(KeyError):
        Engine.pack_state_dict({"foo": torch.zeros(1)}, v)
    # vanilla-config positional embedding (nn_lib.py:73-88)
    sd3 = O.make_weights(O.RICO25, O.ModelSpec(pos_emb="default"), seed=0)
    w3 = Engine.pack_state_dict(sd3, v)
    assert torch.equal(w3["pos_table"], sd3[O.PREFIX + "pos_emb.pos_emb"])


def test_sampling_struct_mirrors_reference_errors():
    s = sampling_struct({"name": "top_p", "top_p": 0.9, "temperature": 1.0})
    assert (s.mode, round(s.top_p, 3)) == (3, 0.9)
    with pytest.raises(NotImplementedError):
        sampling_struct({"name": "top_k_top_p"})      # sampling.py:117-118
    with pytest.raises(AssertionError):
        sampling_struct({"name": "top_p", "top_p": 1.5})   # sampling.py:96

    class Cfg:   # attribute-style config (OmegaConf DictConfig behaves like both)
        name, temperature = "random", 0.7
    assert abs(sampling_struct(Cfg()).temperature - 0.7) < 1e-6


def test_relation_edge_table_matches_oracle_adjacency():
    """product-side dense edge table (LdmCond.rel_adj) == the oracle's, built from a PyG-style batch with canvas nodes"""
    import torch
    from layoutdm_b200.vocab import relation_edge_table
    from oracle import layoutdm_oracle as O

    class Batch:
        pass
    g = torch.Generator().manual_seed(0)
    sizes = [26, 2, 9]
    b = Batch()
    b.batch = torch.cat([torch.full((n,), i) for i, n in enumerate(sizes)])
    ei, ea, off = [], [], 0
    for n in sizes:
        for i in range(n):
            for j in range(i + 1, n):
                if torch.rand(1, generator=g) < 0.3:
                    ei.append((off + i, off + j)); ea.append(int(torch.randint(1, 1 << 10, (1,), generator=g)))
        off += n
    b.edge_index = torch.tensor(ei).t().contiguous()
    b.edge_attr = torch.tensor(ea)
    got = relation_edge_table(b, 3, 26)
    want = O.relation_adjacency(b.edge_index, b.edge_attr, b.batch, 3, 26)
    assert got.dtype == torch.int32 and torch.equal(got, want) and int((got != 0).sum()) == len(ea)
    b.edge_index = torch.zeros(2, 0, dtype=torch.long)
    assert int(relation_edge_table(b, 3, 26).abs().sum()) == 0


def test_duplicate_cond_keeps_shared_tables():
    """one condition, many outputs (task.py:235-248): per-layout tensors repeat, the (C,C) refinement table and the (4,n_bins)
    relation centres are shared and stay as they are"""
    import torch
    from layoutdm_b200.diffusion import duplicate_cond
    cond = {"seq": torch.zeros(1, 125, dtype=torch.long), "mask": torch.ones(1, 125, dtype=torch.bool), "refine_table": torch.zeros(155, 155),
            "rel_centers": torch.zeros(4, 32), "rel_adj": torch.zeros(1, 26, 26, dtype=torch.int32), "type": "refinement"}
    out = duplicate_cond(cond, 4)
    assert out["seq"].shape == (4, 125) and out["mask"].shape == (4, 125) and out["rel_adj"].shape == (4, 26, 26)
    assert out["refine_table"].shape == (155, 155) and out["rel_centers"].shape == (4, 32)


def test_group_full_ids_cover_the_vocabulary():
    from layoutdm_b200 import Vocab
    from layoutdm_b200.vocab import group_full_ids
    from oracle import layoutdm_oracle as O
    for name, ov in (("rico25", O.RICO25), ("publaynet", O.PUBLAYNET)):
        v = Vocab.for_dataset(name)
        for g in range(5):
            assert group_full_ids(v, g) == ov.group_full_ids(g)


def test_header_is_plain_c():
    """include/ldm_b200.h is the drop-in boundary: it must compile as C (no C++ / torch types) and declare every symbol the
    ctypes mirror binds"""
    import os, re, subprocess, tempfile
    from layoutdm_b200 import _lib
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    hdr = os.path.join(repo, "include", "ldm_b200.h")
    with tempfile.NamedTemporaryFile("w", suffix=".c", delete=False) as f:
        f.write('#include "ldm_b200.h"\nint main(void) { LdmCond c = {0}; LdmSampling s = {0}; (void)c; (void)s; return sizeof(LdmModelDesc) > 0 ? 0 : 1; }\n')
        src = f.name
    try:
        subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-fsyntax-only", "-I", os.path.dirname(hdr), src])
    finally:
        os.unlink(src)
    text = open(hdr).read()
    for name in _lib.SIGNATURES:
        assert re.search(r"\b%s\s*\(" % name, text), f"{name} is bound by the mirror but not declared in the header"
