"""GPU (-m gpu): the persistent LN GEMMs give the same bits whatever the CTA count, at per-layout timesteps.

In fp16 / bf16 the out-projection and FF2 (bias + residual + LayerNorm / AdaLN epilogue) run min(tiles, SMs) CTAs, each
walking tiles b, b + gridDim.x, ... through one shared-memory ring and one tile buffer, which takes the next tile's
residual rows while the MMA warpgroups compute it.  At per-layout timesteps (predict_start) FF2's AdaLN reloads the (scale, shift)
row of the tile's own layout, so a CTA's consecutive tiles normalise with different rows.  With LDM_GEMM_CTAS = 1 every
tile of a launch goes through one CTA, with 7 the tiles of a layout are split between CTAs; each LN GEMM launch's tapped
output must be bitwise equal to the uncapped run's."""
import pytest
import torch

import gpu_helpers as G
from oracle import layoutdm_oracle as O
from test_gpu_parity_large import mixed_ids

pytestmark = pytest.mark.gpu

B = 301
LAYERS = 2
T = 20


def taps():
    """launch count to stop after -> the buffers that launch's LN GEMM writes.  Launch 1 is the embedding; layer l's launches
    are 2 + 5 l: QKV, attention, out-projection, FF1, FF2"""
    return {4: ["y32", "z16"], 6: ["x32", "x16"], 4 + 5 * (LAYERS - 1): ["y32", "z16"], 1 + 5 * LAYERS: ["z16"]}


def run(monkeypatch, dtype, cap, sd, ids, t):
    from layoutdm_b200 import Engine, Vocab
    vo = O.RICO25
    if cap is None:
        monkeypatch.delenv("LDM_GEMM_CTAS", raising=False)
    else:
        monkeypatch.setenv("LDM_GEMM_CTAS", str(cap))
    eng = Engine.from_state_dict(sd, Vocab(vo.n_cat, vo.n_bins, vo.n_elem, vo.n_attr), num_timesteps=T, operand_dtype=dtype)
    bits = lambda x: x.view(torch.int16 if x.element_size() == 2 else torch.int32).clone()
    out = {}
    try:
        for n, names in taps().items():
            G.set_stop_after(eng, n)
            eng.predict_start(ids, t)
            torch.cuda.synchronize()
            for k in names:
                out[(n, k)] = bits(G.debug_read(eng, k, B, raw=True))
        G.set_stop_after(eng, 0)
    finally:
        eng.close()
    return out


@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
def test_ln_gemm_outputs_independent_of_cta_count_per_layout_t(monkeypatch, dtype):
    vo, spec = O.RICO25, O.ModelSpec(layers=LAYERS, T=T)
    sd = O.make_weights(vo, spec, seed=6, scale=2.0)
    ids = mixed_ids(B, vo, 13).cuda()
    t = torch.randint(0, T, (B,), generator=torch.Generator().manual_seed(8))
    t[0], t[1] = 0, T - 1
    t = t.cuda()
    ref = run(monkeypatch, dtype, None, sd, ids, t)
    for cap in (1, 7):
        got = run(monkeypatch, dtype, cap, sd, ids, t)
        bad = [f"launch {n} {k}" for (n, k), v in ref.items() if not torch.equal(v, got[(n, k)])]
        assert not bad, f"{dtype}, LDM_GEMM_CTAS={cap}, per-layout timesteps: not bitwise equal to the uncapped run: {bad}"
