"""CPU: the per-kernel references of test_gpu_kernels_fp64.py, chained in fp32 without operand rounding, reproduce the oracle's
forward pass tap by tap.  This pins those references -- padding maps, the q-scale, the ones column, the residual wiring and the
AdaLN rows -- to the oracle, which is itself pinned to the reference."""
import pytest
import torch

import kernel_refs as R
from oracle import layoutdm_oracle as O
from test_gpu_parity_large import mixed_ids

TOL = 1e-5

SHAPES = {"rico25_L4": (O.RICO25, 4), "n_cat30_n_elem20_L2": (O.VocabSpec(n_cat=30, n_elem=20), 2), "n_cat1_L1": (O.VocabSpec(n_cat=1), 1)}


@pytest.mark.parametrize("per_layout_t", [False, True])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_kernel_reference_chain_reproduces_oracle(shape, per_layout_t):
    vo, L = SHAPES[shape]
    spec = O.ModelSpec(layers=L)
    sd = O.make_weights(vo, spec, seed=1)
    m = R.Model(sd, vo, spec, operand_dtype=None, dtype=torch.float32)
    B, S, C, H, dh = 9, vo.S, vo.C, spec.heads, spec.dh
    ids = mixed_ids(B, vo, 5)
    t = torch.randint(0, spec.T, (B,), generator=torch.Generator().manual_seed(2)) if per_layout_t else 42
    taps = {}
    with torch.no_grad():
        logits = O.denoiser_forward(sd, ids, t, vo, spec, taps=taps)
        tables = torch.stack([O.adaln_table(sd, spec, l) for l in range(L)])     # (L, T, 2d)
        rows = lambda l: tables[l][t][:, None] if per_layout_t else tables[l][t]

        def close(name, got, want):
            assert got.shape == want.shape, name
            d = (got - want).abs().max().item()
            assert d <= TOL, f"{name}: max-abs {d:.3e}"

        x = R.adaln(m, R.embed_input(m, ids), rows(0))
        close("x0", x, taps["x0"])
        for l in range(L):
            qkv = R.qkv(m, l, x)
            q, k, v = (qkv[..., i * H * R.HP:(i + 1) * H * R.HP].reshape(B, S, H, R.HP) for i in range(3))
            for name, a in (("q", q), ("k", k), ("v", v)):
                close(f"{name}{l}", a[..., :dh].transpose(1, 2), taps[f"{name}{l}"])
            pad = torch.zeros(B, S, 3, H, R.HP - dh)
            pad[:, :, 2, :, 0] = 1.0
            assert torch.equal(qkv.reshape(B, S, 3, H, R.HP)[..., dh:], pad)
            att = R.attention(m, qkv, S)[0]
            close(f"att{l}", R.unpad_heads(att, H, dh), taps[f"att{l}"])
            a = att.reshape(B, S, H, R.HP)
            assert (a[..., dh] - 1).abs().max() <= TOL and torch.equal(a[..., dh + 1:], torch.zeros_like(a[..., dh + 1:]))
            y = R.outproj(m, l, att, x)
            close(f"y{l}", y, taps[f"y{l}"])
            z = R.ln2(m, l, y)
            close(f"z{l}", z, taps[f"z{l}"])
            hid = R.ff1(m, l, z)
            close(f"hid{l}", hid, taps[f"hid{l}"])
            h = R.ff2_pre(m, l, hid, y)
            close(f"h{l}", h, taps[f"h{l}"])
            x = R.ff2_norm(m, l, h, rows(l + 1) if l + 1 < L else None)
            close(f"x{l + 1}" if l + 1 < L else "hn", x, taps[f"x{l + 1}"] if l + 1 < L else taps["hn"])
        lg = R.head(m, x)
        close("logits", lg[..., :C], logits)
        assert torch.equal(lg[..., C:], torch.zeros_like(lg[..., C:]))
