"""CPU: the closed-form restatement of torch's CUDA generator stream (oracle/torch_noise.py, csrc TorchNoise) against a literal
simulation of ATen's distribution_elementwise_grid_stride_kernel loop with curand's Philox state, and the reference's
`model_log_prob` layout the element index of `rand_like` depends on."""
import sys

import numpy as np
import pytest
import torch

from oracle import layoutdm_oracle as O
from oracle import ref_harness as rh
from oracle import torch_noise as TN

# (SMs, max threads per SM): small devices keep the literal loop short, the H100 SXM the kernels meet
DEVICES = [(1, 256), (2, 512), (3, 1024), (5, 2048)]


def simulate(seed: int, offset: int, numel: int, n_sm: int, max_threads_sm: int):
    """distribution_elementwise_grid_stride_kernel<unroll 4> with curand_uniform4, literally: every thread runs curand_init(seed,
    idx, offset) and its grid-stride loop.  Returns (subsequence, counter, word, 32-bit word) per element and the largest
    counter any thread used."""
    block = 256
    grid = min(n_sm * (max_threads_sm // block), (numel + block - 1) // block)
    threads = block * grid
    out = np.full((numel, 4), -1, dtype=np.int64)
    top = -1
    rounded = ((numel - 1) // (threads * 4) + 1) * threads * 4
    for idx in range(threads):
        ctr = offset // 4                        # skipahead(offset): offset / 4 counter steps (offset % 4 == 0)
        li = idx
        while li < rounded:
            r = O.philox4x32_10(np.uint32(ctr & 0xFFFFFFFF), np.uint32(ctr >> 32), np.uint32(idx), np.uint32(0),
                                seed & 0xFFFFFFFF, seed >> 32)
            for ii in range(4):
                e = li + threads * ii
                if e < numel:
                    out[e] = (idx, ctr, ii, int(r[ii]))
            top = max(top, ctr)
            ctr += 1                             # curand_uniform4: the next Philox block of this subsequence
            li += threads * 4
    assert (out[:, 0] >= 0).all()
    return out, top


@pytest.mark.parametrize("n_sm,max_threads_sm", DEVICES)
def test_closed_form_matches_grid_stride_loop(n_sm, max_threads_sm):
    seed, offset = 0x1234_5678_9ABC_DEF0, 4 * 1_000_003
    cap = 256 * n_sm * (max_threads_sm // 256)
    for numel in sorted({1, 7, 255, 257, cap - 3, cap, cap + 1, 4 * cap - 1, 4 * cap, 4 * cap + 1, 9 * cap + 5}):
        if numel <= 0:
            continue
        sim, top = simulate(seed, offset, numel, n_sm, max_threads_sm)
        threads = TN.tthr(numel, n_sm, max_threads_sm)
        sub, ctr, word = TN.element_coords(np.arange(numel), offset, threads)
        np.testing.assert_array_equal(sub, sim[:, 0])
        np.testing.assert_array_equal(ctr, sim[:, 1])
        np.testing.assert_array_equal(word, sim[:, 2])
        w = TN.words(seed, offset, numel, n_sm, max_threads_sm)
        np.testing.assert_array_equal(w.astype(np.int64), sim[:, 3])
        # the offset advance covers exactly the counters the draw used: the next draw starts on fresh blocks
        d = TN.delta(numel, n_sm, max_threads_sm)
        assert d == ((numel - 1) // (threads * 4) + 1) * 4          # calc_execution_policy's counter_offset
        assert top == offset // 4 + d // 4 - 1


def test_h100_policy():
    """the numbers the kernels meet at the benchmark's shape (B = 1024, S = 125, C = 155) on an H100 SXM"""
    numel = 1024 * 125 * 155
    assert TN.tthr(numel, *TN.H100_SXM) == 270_336
    assert TN.delta(numel, *TN.H100_SXM) == 76


def test_transforms():
    w = np.array([0, 1, 2 ** 31, 2 ** 32 - 256, 2 ** 32 - 129, 2 ** 32 - 128, 2 ** 32 - 1], dtype=np.uint32)
    u = TN.curand_uniform(w)
    assert u[0] == np.float32(2.0 ** -33) and u[-1] == np.float32(1.0)
    r = TN.rand(w)
    assert r[-1] == 0.0 and (r[:-2] < 1.0).all()                       # uniform_'s (0, 1] -> [0, 1)
    e = TN.exponential(w)
    assert e[-1] == np.float32(2.0 ** -24)                              # log(1) -> -eps / 2
    assert (e > 0).all() and abs(float(e[0]) - 33 * np.log(2)) < 1e-5


def test_draw_e_matches_draw_with_uniforms():
    """draw_e with e = -log(u) is layoutdm_oracle.draw on the same uniforms"""
    g = torch.Generator().manual_seed(0)
    lp = torch.log_softmax(torch.randn(3, 10, 20, generator=g) * 3, dim=-1)
    u = O.uniforms(5, 0, 0, 0, 3, 10, 20)
    ug = O.uniforms(5, 0, 1, 0, 3, 10, 20)
    e = (-torch.log(torch.from_numpy(u))).numpy()
    for cfg in (O.SamplingCfg("random"), O.SamplingCfg("top_k", top_k=4), O.SamplingCfg("top_p", top_p=0.8),
                O.SamplingCfg("gumbel", temperature=0.7)):
        assert torch.equal(TN.draw_e(lp, cfg, e, ug), O.draw(lp, cfg, u, ug)), cfg.name


@pytest.mark.skipif(not rh.reference_available(), reason="reference archive missing: run python oracle/make_ref.py")
@pytest.mark.parametrize("q_type", ["constrained", "vanilla"])
def test_reference_model_log_prob_is_contiguous_bcs(q_type, monkeypatch):
    """`sample(model_log_prob, cfg)` (base.py:287) gets a contiguous (B, C, S) tensor for both q_types, so rand_like's element
    (b, c, s) is (b C + c) S + s.  multinomial's probabilities, rearranged to (B S, C), are a contiguous copy for B > 1 (element
    (b S + s) C + c) but a view with strides (1, S) for B = 1, which empty_like keeps, so exponential_ fills element (s, c) at
    c S + s (TorchDraw::exp_cs)"""
    model, tok = rh.build_reference("rico25", T=10, q_type=q_type, state_dict=O.make_weights(O.RICO25, O.ModelSpec(T=10), seed=1))
    core = model.model.module if hasattr(model.model, "module") else model.model
    base = sys.modules[next(c for c in type(core).__mro__ if c.__name__ == "BaseMaskAndReplaceDiffusion").__module__]
    C, S = O.RICO25.C, O.RICO25.S
    real, real_multinomial = base.sample, torch.multinomial
    for B in (1, 2):
        seen, probs = [], []

        def spy(logits, cfg):
            seen.append((tuple(logits.shape), logits.is_contiguous(), logits.dtype))
            return real(logits, cfg)

        def spy_multinomial(p, *a, **k):
            probs.append((tuple(p.shape), p.stride(), torch.empty_like(p).stride()))
            return real_multinomial(p, *a, **k)
        monkeypatch.setattr(base, "sample", spy)
        monkeypatch.setattr(torch, "multinomial", spy_multinomial)
        core.sample(batch_size=B, sampling_cfg=rh.sampling_cfg("gumbel", num_timesteps=2))
        assert seen and all(s == ((B, C, S), True, torch.float32) for s in seen), seen
        want = (1, S) if B == 1 else (C, 1)
        assert probs and all(p == ((B * S, C), want, want) for p in probs), probs
