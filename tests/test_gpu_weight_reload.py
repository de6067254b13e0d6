"""GPU (-m gpu): ldm_load_weights repacks new weights into a live handle in place, stream-ordered.

A handle built from W1 and then given W2 must compute what a fresh handle built from W2 computes, bit for bit: the AdaLN
table, a step's logits and ids, and a replay of the loop graph captured under W1.  Reloading W1 gives the first handle's
original bits back (a stale lo plane, QKV-bias ones row or AdaLN row would show there).  Loads queued between loops on one
stream apply between them.  A patched reference model follows its weights through training steps, load_state_dict and
device moves."""
from __future__ import annotations

import functools

import pytest
import torch

from oracle import ref_harness as rh

pytestmark = pytest.mark.gpu

T = 100
RANDOM = {"name": "random", "temperature": 1.0}


@functools.lru_cache(maxsize=None)
def vocab():
    from layoutdm_b200 import Vocab
    return Vocab.for_dataset("rico25")


@functools.lru_cache(maxsize=None)
def state_dict(seed: int):
    from layoutdm_b200.synthetic import random_state_dict
    return random_state_dict(vocab(), num_timesteps=T, seed=seed)


def engine(seed: int, operand_dtype: str = "fp16"):
    from layoutdm_b200 import Engine
    return Engine.from_state_dict(state_dict(seed), vocab(), num_timesteps=T, operand_dtype=operand_dtype)


def packed_on_device(seed: int):
    from layoutdm_b200 import Engine
    return {k: v.cuda() for k, v in Engine.pack_state_dict(state_dict(seed), vocab()).items()}


def plan(n: int = 25):
    from layoutdm_b200 import timestep_plan
    return timestep_plan(T, n)


def step_ids_logits(eng, B: int = 301):
    """one step at B = 301 from a fixed random state, through the logits tap"""
    g = torch.Generator().manual_seed(5)
    ids = torch.randint(0, vocab().C, (B, vocab().S), generator=g).cuda()
    out, lg, _ = eng.step(ids, 60, 59, RANDOM, seed=9, want_logits=True)
    torch.cuda.synchronize()
    return out.cpu(), lg.cpu()


def run(eng):
    """what the handle computes: AdaLN table, a step's ids + logits at B = 301, a graph-captured loop's ids"""
    ada = eng.adaln_table()
    ids, lg = step_ids_logits(eng)
    loop = eng.sample_loop(64, plan(), RANDOM, seed=21).cpu()
    return ada, ids, lg, loop


def assert_same(got, want):
    for name, a, b in zip(("AdaLN table", "step ids", "step logits", "loop ids"), got, want):
        assert a.shape == b.shape and torch.equal(a, b), f"{name} differs"


@pytest.mark.parametrize("operand_dtype", ["fp16", "bf16", "bf16x3"])
def test_reload_equals_fresh_handle(operand_dtype):
    e = engine(0, operand_dtype)
    first = run(e)                            # the loop graph is captured here, under W1
    fresh = run(engine(1, operand_dtype))
    assert not torch.equal(first[3], fresh[3])
    e.load_weights(packed_on_device(1))
    assert_same(run(e), fresh)                # the loop replays the graph captured under W1
    e.load_weights(packed_on_device(0))
    assert_same(run(e), first)


def test_loads_apply_in_stream_order():
    """loop(W1), load(W2), loop(W2), load(W1), loop(W1) queued on one side stream with no host synchronise in between"""
    B, p = 512, plan(100)
    want = {s: engine(s).sample_loop(B, p, RANDOM, seed=4).cpu() for s in (0, 1)}
    assert not torch.equal(want[0], want[1])
    e = engine(0)
    w = {s: packed_on_device(s) for s in (0, 1)}
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        a = e.sample_loop(B, p, RANDOM, seed=4)
        e.load_weights(w[1])
        b = e.sample_loop(B, p, RANDOM, seed=4)
        e.load_weights(w[0])
        c = e.sample_loop(B, p, RANDOM, seed=4)
    side.synchronize()
    assert torch.equal(a.cpu(), want[0]) and torch.equal(b.cpu(), want[1]) and torch.equal(c.cpu(), want[0])


def test_bad_loads_are_rejected():
    from layoutdm_b200 import Engine
    e = engine(0)
    w = packed_on_device(1)
    with pytest.raises(ValueError):
        e.load_weights({**w, "in_proj_w": w["in_proj_w"][:3]})            # another layer count: a new handle, not a reload
    sd = dict(state_dict(1))
    for k in [k for k in sd if ".backbone.layers.3." in k]:
        del sd[k]
    with pytest.raises(ValueError):
        e.load_state_dict(sd)
    import ctypes as C
    from layoutdm_b200 import _lib
    ws = _lib.LdmWeights()
    host = Engine.pack_state_dict(state_dict(1), vocab())
    for name in _lib._W_FIELDS:
        setattr(ws, name, host[name].data_ptr())
    assert e.lib.ldm_load_weights(e._h, C.byref(ws), None) == _lib.LDM_ERR_INVALID         # host memory
    ws.head_w = None
    assert e.lib.ldm_load_weights(e._h, C.byref(ws), None) == _lib.LDM_ERR_INVALID
    assert e.lib.ldm_load_weights(None, C.byref(ws), None) == _lib.LDM_ERR_INVALID
    assert torch.equal(e.sample_loop(8, plan(), RANDOM, seed=1).cpu(), engine(0).sample_loop(8, plan(), RANDOM, seed=1).cpu())


def test_layoutdm_b200_load_state_dict():
    from layoutdm_b200 import LayoutDMB200
    m = LayoutDMB200.from_state_dict(state_dict(0), num_timesteps=T).load_state_dict(state_dict(1))
    want = LayoutDMB200.from_state_dict(state_dict(1), num_timesteps=T)
    cfg = dict(RANDOM, num_timesteps=50)
    assert torch.equal(m.model.sample(batch_size=16, sampling_cfg=cfg, seed=3), want.model.sample(batch_size=16, sampling_cfg=cfg, seed=3))
    a, b = m.sample(batch_size=16, sampling_cfg=cfg, seed=3), want.sample(batch_size=16, sampling_cfg=cfg, seed=3)
    assert all(torch.equal(a[k], b[k]) for k in ("bbox", "label", "mask"))


@pytest.mark.skipif(not rh.reference_available(), reason="reference archive missing: run python oracle/make_ref.py")
def test_patched_model_follows_its_weights():
    """main.py's use: the patched model samples between training steps; every sample must be what a model freshly built from
    the live weights samples"""
    from layoutdm_b200 import patch_reference_model
    from layoutdm_b200.synthetic import synthetic_cond
    model, _ = rh.build_reference("rico25", T=T, state_dict=state_dict(0))
    model = patch_reference_model(model.cuda())
    core = model.model.module
    fused = core._ldm_b200
    cfg = rh.sampling_cfg("random", num_timesteps=50)
    x0 = synthetic_cond(vocab(), 8, "refinement", seed=0)["seq_orig"].cuda()      # valid layouts: every token in its group

    def sample(m, seed):
        return m.model.sample(batch_size=8, sampling_cfg=cfg, seed=seed).cpu()

    def check(what, seed):
        """sample twice after a change; returns how many reloads the first call made (the second must make none)"""
        fresh, _ = rh.build_reference("rico25", T=T, state_dict=model.state_dict())
        want = sample(patch_reference_model(fresh.cuda()), seed)
        n = fused.weight_reloads
        assert torch.equal(sample(model, seed), want), what
        reloads = fused.weight_reloads
        assert torch.equal(sample(model, seed), want), what
        assert fused.weight_reloads == reloads, f"{what}: a call with nothing changed reloaded"
        return reloads - n

    def train_step(opt):
        core.train()
        _, losses = core(x0)
        sum(v.mean() for v in losses.values()).backward()
        opt.step()
        opt.zero_grad()
        core.eval()

    assert fused.weight_reloads == 0
    sample(model, 1)
    assert fused.weight_reloads == 0
    train_step(torch.optim.AdamW(model.parameters(), lr=1e-3))
    assert check("AdamW (foreach) step", 2) == 1
    train_step(torch.optim.AdamW(model.parameters(), lr=1e-3, fused=True))
    assert check("AdamW (fused) step", 3) == 1
    model.load_state_dict(state_dict(1), strict=False)
    assert check("load_state_dict", 4) == 1
    model.cpu()
    model.cuda()
    assert check("cpu() / cuda()", 5) <= 1
