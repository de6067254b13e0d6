"""GPU (-m gpu): the persistent GEMM schedule computes every output element the same way whatever the CTA count.

QKV and FF1 in fp16 / bf16 are persistent: min(tiles, SMs) CTAs, each walking tiles b, b + gridDim.x, ... with one
shared-memory ring whose slot and phase carry over from tile to tile, and a staging tile that the previous tile's TMA store
may still be reading.  LDM_GEMM_CTAS caps their CTA count: with 1 CTA a single ring runs through every tile of a launch
(hundreds of tiles, 8 k-blocks each over 3 stages), with 7 the tiles of a row block spread over CTAs in a ragged last round.
Every other GEMM (and every GEMM of the split mode) runs one CTA per tile whatever the cap.  Each GEMM's tapped output must
be bitwise equal to the uncapped run's, in every operand mode."""
import pytest
import torch

import gpu_helpers as G
from oracle import layoutdm_oracle as O
from test_gpu_parity_large import mixed_ids

pytestmark = pytest.mark.gpu

B = 301
LAYERS = 2
T = 20


def taps(split):
    """launch count to stop after -> the buffers that launch's GEMM writes (0: the whole pass, ending with the head).
    Launch 1 is the embedding; layer l's launches are 2 + 5 l: QKV, attention, out-projection, FF1, FF2"""
    lo = (lambda names: names + [n + "_lo" for n in names if n.endswith("16")]) if split else (lambda names: names)
    last_ff2 = 1 + 5 * LAYERS
    return {2: lo(["qkv16"]), 4: lo(["y32", "z16"]), 5: lo(["hid16"]), 6: lo(["x32", "x16"]), last_ff2: lo(["z16"]), 0: ["logits"]}


def run(monkeypatch, dtype, cap, sd, ids):
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
        for n, names in taps(dtype == "bf16x3").items():
            G.set_stop_after(eng, n)
            eng.step(ids, 7, 7, {"name": "deterministic"})
            torch.cuda.synchronize()
            for k in names:
                out[(n, k)] = bits(G.debug_read(eng, k, B, raw=True))
        G.set_stop_after(eng, 0)
    finally:
        eng.close()
    return out


@pytest.mark.parametrize("dtype", ["fp16", "bf16", "bf16x3"])
def test_gemm_outputs_independent_of_cta_count(monkeypatch, dtype):
    vo, spec = O.RICO25, O.ModelSpec(layers=LAYERS, T=T)
    sd = O.make_weights(vo, spec, seed=5, scale=2.0)
    ids = mixed_ids(B, vo, B).cuda()
    ref = run(monkeypatch, dtype, None, sd, ids)
    for cap in (1, 7):
        got = run(monkeypatch, dtype, cap, sd, ids)
        bad = [f"launch {n} {k}" for (n, k), v in ref.items() if not torch.equal(v, got[(n, k)])]
        assert not bad, f"{dtype}, LDM_GEMM_CTAS={cap}: not bitwise equal to the uncapped run: {bad}"
