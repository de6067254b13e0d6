"""helpers shared by the -m gpu tests and tools/gpu_diag.py (test scaffolding; uses the ldm_debug_* taps)"""
from __future__ import annotations

import ctypes as C

import torch


def debug_read(engine, name: str, n_layouts: int, raw: bool = False) -> torch.Tensor:
    """copy a workspace buffer of the first n_layouts layouts to the host; returns [n_layouts, 128, cols] float32
    (raw: in the buffer's own dtype, for bitwise comparisons)"""
    lib, h = engine.lib, engine._h
    nbytes = lib.ldm_debug_read(h, name.encode(), None, 0, n_layouts)
    assert nbytes > 0, f"unknown buffer {name}"
    is32 = name in ("x32", "y32", "logits")
    dt = torch.float32 if is32 else (torch.bfloat16 if engine.operand_dtype == "bf16" else torch.float16)
    out = torch.empty(nbytes // (4 if is32 else 2), dtype=dt)
    rc = lib.ldm_debug_read(h, name.encode(), C.c_void_p(out.data_ptr()), nbytes, n_layouts)
    assert rc == nbytes, f"ldm_debug_read failed rc={rc}"
    out = out.view(n_layouts, 128, -1)
    return out if raw else out.float()


def unpack_qkv(qkv: torch.Tensor, S: int = 125, heads: int = 8, dh: int = 58):
    """[B,128,1536] padded per-head layout -> q,k,v each (B,H,S,dh) and the max deviation of the padding columns from their
    contract: zeros, except column dh of every V head, which is 1.0 (the softmax-denominator column, attention.cuh)"""
    B = qkv.shape[0]
    x = qkv[:, :S].view(B, S, 3, heads, 64).float()
    want = torch.zeros_like(x[..., dh:])
    want[:, :, 2, :, 0] = 1.0
    pad = (x[..., dh:] - want).abs().max().item()
    q, k, v = (x[:, :, i, :, :dh].permute(0, 2, 1, 3).contiguous() for i in range(3))
    return q, k, v, pad


def set_stop_after(engine, n: int):
    rc = engine.lib.ldm_debug_set_stop_after(engine._h, n)
    assert rc == 0
