"""GPU (-m gpu): the persistent GEMMs compute every output element the same way whatever the CTA count.

The persistent GEMMs run min(tiles, SMs) CTAs, each walking tiles b, b + gridDim.x, ... through one shared-memory operand ring
whose slot and phase carry over from tile to tile:
- QKV and FF1 in fp16 / bf16, with a staging tile that the previous tile's TMA store may still be reading;
- the out-projection and FF2 in fp16 / bf16 (bias + residual + LayerNorm / AdaLN epilogue), with a tile buffer that takes the
  next tile's residual rows while the MMA warpgroups compute it.  At per-layout timesteps (predict_start) FF2's AdaLN reloads
  the (scale, shift) row of the tile's own layout, so a CTA's consecutive tiles normalise with different rows.
LDM_GEMM_CTAS caps their CTA count: with 1 CTA a single ring runs through every tile of a launch (hundreds of tiles), with 7 the
tiles of a row block spread over CTAs in a ragged last round.  Every other GEMM (and every GEMM of the split mode) runs one CTA
per tile whatever the cap.  Each GEMM's tapped output must be bitwise equal to the uncapped run's."""
import pytest
import torch

import gpu_helpers as G
from oracle import layoutdm_oracle as O
from test_gpu_parity_large import mixed_ids

pytestmark = pytest.mark.gpu

B = 301
LAYERS = 2
T = 20


def run(monkeypatch, dtype, cap, sd, taps, call):
    """taps: launch count to stop after -> the buffers that launch's GEMM writes (0: the whole pass).  Launch 1 is the
    embedding; layer l's launches are 2 + 5 l: QKV, attention, out-projection, FF1, FF2.  call(engine) runs the pass."""
    from layoutdm_b200 import Engine, Vocab
    vo = O.RICO25
    if cap is None:
        monkeypatch.delenv("LDM_GEMM_CTAS", raising=False)
    else:
        monkeypatch.setenv("LDM_GEMM_CTAS", str(cap))
    eng = Engine.from_state_dict(sd, Vocab(vo.n_cat, vo.n_bins, vo.n_elem, vo.n_attr), num_timesteps=T, operand_dtype=dtype)
    bits = lambda t: t.view(torch.int16 if t.element_size() == 2 else torch.int32).clone()
    out = {}
    try:
        for n, names in taps.items():
            G.set_stop_after(eng, n)
            call(eng)
            torch.cuda.synchronize()
            for k in names:
                out[(n, k)] = bits(G.debug_read(eng, k, B, raw=True))
        G.set_stop_after(eng, 0)
    finally:
        eng.close()
    return out


def check_caps(monkeypatch, dtype, sd, taps, call, what):
    ref = run(monkeypatch, dtype, None, sd, taps, call)
    for cap in (1, 7):
        got = run(monkeypatch, dtype, cap, sd, taps, call)
        bad = [f"launch {n} {k}" for (n, k), v in ref.items() if not torch.equal(v, got[(n, k)])]
        assert not bad, f"{dtype}, LDM_GEMM_CTAS={cap}{what}: not bitwise equal to the uncapped run: {bad}"


@pytest.mark.parametrize("dtype", ["fp16", "bf16", "bf16x3"])
def test_gemm_outputs_independent_of_cta_count(monkeypatch, dtype):
    vo, spec = O.RICO25, O.ModelSpec(layers=LAYERS, T=T)
    sd = O.make_weights(vo, spec, seed=5, scale=2.0)
    ids = mixed_ids(B, vo, B).cuda()
    lo = (lambda names: names + [n + "_lo" for n in names if n.endswith("16")]) if dtype == "bf16x3" else (lambda names: names)
    taps = {2: lo(["qkv16"]), 4: lo(["y32", "z16"]), 5: lo(["hid16"]), 6: lo(["x32", "x16"]), 1 + 5 * LAYERS: lo(["z16"]), 0: ["logits"]}
    check_caps(monkeypatch, dtype, sd, taps, lambda eng: eng.step(ids, 7, 7, {"name": "deterministic"}), "")


@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
def test_ln_gemm_outputs_independent_of_cta_count_per_layout_t(monkeypatch, dtype):
    vo, spec = O.RICO25, O.ModelSpec(layers=LAYERS, T=T)
    sd = O.make_weights(vo, spec, seed=6, scale=2.0)
    ids = mixed_ids(B, vo, 13).cuda()
    t = torch.randint(0, T, (B,), generator=torch.Generator().manual_seed(8))
    t[0], t[1] = 0, T - 1
    t = t.cuda()
    taps = {4: ["y32", "z16"], 6: ["x32", "x16"], 4 + 5 * (LAYERS - 1): ["y32", "z16"], 1 + 5 * LAYERS: ["z16"]}
    check_caps(monkeypatch, dtype, sd, taps, lambda eng: eng.predict_start(ids, t), ", per-layout timesteps")
