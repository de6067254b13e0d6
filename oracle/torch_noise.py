"""numpy restatement of the numbers torch's CUDA generator gives the reference's draw (the LDM_NOISE_TORCH contract of
csrc/common.cuh::TorchNoise).  Restated from ATen/native/cuda/DistributionTemplates.h (torch 2.11):

  calc_execution_policy     256-thread blocks, grid = min(SMs * (max threads per SM // 256), ceil(numel / 256)),
                            tthr = 256 * grid; the generator's offset advances by delta = ((numel - 1) // (4 tthr) + 1) * 4
  distribution_elementwise_grid_stride_kernel
                            thread idx runs curand_init(seed, idx, offset) and one curand_uniform4 per loop iteration:
                            element i is word (i // tthr) % 4 of the Philox4x32-10 block with counter
                            offset // 4 + i // (4 tthr) (64 bits, words 0-1) and subsequence i % tthr (words 2-3), key = seed
  curand_uniform            u = w 2^-32 + 2^-33 in float32, in (0, 1]
  uniform_kernel (rand)     u, with 1 -> 0
  transformation::exponential (ATen/core/TransformationHelper.h)
                            e = -(u >= 1 - eps/2 ? -eps/2 : log(u)), log = the device's fast __logf (ATen/NumericUtils.h)

The reference's helpers/sampling.py:81-130 draws multinomial(probs, 1) = argmax(probs / e) with e = exponential_ on the
(B S, C) probabilities (element (b S + s) C + c) and, for name="gumbel", first rand_like on the (B, C, S) logits (element
(b C + c) S + s)."""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch
import torch.nn.functional as F

from .layoutdm_oracle import SamplingCfg, philox4x32_10

H100_SXM = (132, 2048)          # (SMs, max threads per SM) of an H100 SXM


def tthr(numel: int, n_sm: int, max_threads_sm: int) -> int:
    return 256 * min(n_sm * (max_threads_sm // 256), (numel + 255) // 256)


def delta(numel: int, n_sm: int, max_threads_sm: int) -> int:
    return ((numel - 1) // (tthr(numel, n_sm, max_threads_sm) * 4) + 1) * 4


def element_coords(i: np.ndarray, offset: int, threads: int):
    """closed form: (subsequence, 64-bit counter, word) of elements i"""
    i = np.asarray(i, dtype=np.int64)
    return i % threads, offset // 4 + i // (4 * threads), (i // threads) % 4


def words(seed: int, offset: int, numel: int, n_sm: int, max_threads_sm: int, i: Optional[np.ndarray] = None) -> np.ndarray:
    """the 32-bit words of elements i (default: all numel) of one draw at `offset`"""
    assert offset % 4 == 0
    i = np.arange(numel, dtype=np.int64) if i is None else np.asarray(i, dtype=np.int64)
    sub, ctr, word = element_coords(i, offset, tthr(numel, n_sm, max_threads_sm))
    r = philox4x32_10((ctr & 0xFFFFFFFF).astype(np.uint32), (ctr >> 32).astype(np.uint32), sub.astype(np.uint32), np.uint32(0),
                      seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    return np.choose(word, r).astype(np.uint32)


def curand_uniform(w: np.ndarray) -> np.ndarray:
    return (w.astype(np.float32) * np.float32(2.0 ** -32) + np.float32(2.0 ** -33)).astype(np.float32)


def rand(w: np.ndarray) -> np.ndarray:
    u = curand_uniform(w)
    return np.where(u == np.float32(1.0), np.float32(0.0), u)


def exponential(w: np.ndarray) -> np.ndarray:
    """Exp(1) in float32 with a correctly rounded log; torch's __logf (lg2.approx times ln 2) is within about 2^-21 absolute /
    2^-21 relative of it, so these equal torch's values to that accuracy, not bit for bit"""
    u = curand_uniform(w)
    half_eps = np.float32(2.0 ** -24)
    return np.where(u >= np.float32(1.0) - half_eps, half_eps, (-np.log(u.astype(np.float64))).astype(np.float32))


def draw_noise(seed: int, offset: int, B: int, S: int, C: int, gumbel: bool, n_sm: int = H100_SXM[0],
               max_threads_sm: int = H100_SXM[1]):
    """(e (B,S,C), u_gumbel (B,S,C) or None, offset after the draw) of one reference `sample` on a (B, C, S) batch"""
    n = B * S * C
    d = delta(n, n_sm, max_threads_sm)
    ug = None
    if gumbel:
        ug = rand(words(seed, offset, n, n_sm, max_threads_sm)).reshape(B, C, S).transpose(0, 2, 1).copy()
        offset += d
    e = exponential(words(seed, offset, n, n_sm, max_threads_sm)).reshape(B, S, C)
    return e, ug, offset + d


def draw_e(logp: torch.Tensor, cfg: SamplingCfg, e: np.ndarray, u_gumbel: Optional[np.ndarray] = None) -> torch.Tensor:
    """layoutdm_oracle.draw with the Exp(1) variates given directly: logp (B,S,C) -> ids (B,S)"""
    if cfg.name == "deterministic":
        return torch.argmax(logp, dim=-1)
    lg = logp / cfg.temperature
    if cfg.name == "top_k":
        v, _ = torch.topk(lg, cfg.top_k, dim=-1)
        lg = lg.masked_fill(lg < v[..., -1:], -float("inf"))
    elif cfg.name == "top_p":
        sl, si = torch.sort(lg, descending=True, dim=-1)
        cum = torch.cumsum(F.softmax(sl, dim=-1), dim=-1)
        rank = torch.arange(lg.shape[-1]).expand_as(sl)
        lg = sl.masked_fill((cum > cfg.top_p) & (rank > 0), -float("inf")).gather(-1, si.argsort(dim=-1))
    elif cfg.name == "gumbel":
        lg = lg + (-torch.log(-torch.log(torch.from_numpy(u_gumbel) + 1e-30) + 1e-30))
    elif cfg.name != "random":
        raise NotImplementedError
    return torch.argmax(F.softmax(lg, dim=-1) / torch.from_numpy(e), dim=-1)
