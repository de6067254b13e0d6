"""GPU (-m gpu): the row-block QKV / FF1 GEMMs (fp16 / bf16) compute every output element the same way whatever the work split.

A work item is one layout's 128-row block and a range of its 128-column tiles; the CTA keeps the item's A rows resident while
its two consumer warpgroups take alternate tiles.  LDM_GEMM_SPLIT=g cuts every row block into g column ranges (1: a CTA runs
all 12 QKV / 15 FF1 tiles of a layout; 5: ragged ranges of 2-3 tiles; automatic: one range per row block at large batches,
more at small ones), and LDM_GEMM_CTAS=7 makes each CTA run many items in a row, so the resident A rows are refilled while
the other warpgroup is still on the previous item's last tile.  The tapped qkv16 / hid16 must be bitwise equal in every case,
and a layout's rows must not depend on the batch it runs in (B = 8 and B = 1 take other automatic splits than B = 301)."""
import pytest
import torch

import gpu_helpers as G
from oracle import layoutdm_oracle as O
from test_gpu_parity_large import mixed_ids

pytestmark = pytest.mark.gpu

B = 301
LAYERS = 2
T = 20
# launch count to stop after -> the row-block GEMM output it leaves: layer l's QKV is launch 2 + 5 l, its FF1 launch 5 + 5 l
TAPS = {2: "qkv16", 5: "hid16", 7: "qkv16", 10: "hid16"}


def run(monkeypatch, dtype, sd, ids, split, cap):
    from layoutdm_b200 import Engine, Vocab
    vo = O.RICO25
    for name, v in (("LDM_GEMM_SPLIT", split), ("LDM_GEMM_CTAS", cap)):
        if v is None:
            monkeypatch.delenv(name, raising=False)
        else:
            monkeypatch.setenv(name, str(v))
    eng = Engine.from_state_dict(sd, Vocab(vo.n_cat, vo.n_bins, vo.n_elem, vo.n_attr), num_timesteps=T, operand_dtype=dtype)
    n = ids.shape[0]
    out = {}
    try:
        for stop, name in TAPS.items():
            G.set_stop_after(eng, stop)
            eng.step(ids, 7, 7, {"name": "deterministic"})
            torch.cuda.synchronize()
            out[stop] = G.debug_read(eng, name, n, raw=True).view(torch.int16).clone()
        G.set_stop_after(eng, 0)
    finally:
        eng.close()
    return out


def weights_and_ids(seed):
    vo, spec = O.RICO25, O.ModelSpec(layers=LAYERS, T=T)
    return O.make_weights(vo, spec, seed=seed, scale=2.0), mixed_ids(B, vo, seed).cuda()


@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
def test_rowblock_outputs_independent_of_split(monkeypatch, dtype):
    sd, ids = weights_and_ids(21)
    ref = run(monkeypatch, dtype, sd, ids, None, None)
    for split in (None, 1, 2, 5):
        for cap in (None, 7):
            if split is None and cap is None:
                continue
            got = run(monkeypatch, dtype, sd, ids, split, cap)
            bad = [f"launch {n} {TAPS[n]}" for n in TAPS if not torch.equal(ref[n], got[n])]
            assert not bad, f"{dtype}, LDM_GEMM_SPLIT={split}, LDM_GEMM_CTAS={cap}: not bitwise equal to the automatic split: {bad}"


@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
def test_rowblock_rows_independent_of_batch(monkeypatch, dtype):
    sd, ids = weights_and_ids(22)
    ref = run(monkeypatch, dtype, sd, ids, None, None)
    for n in (8, 1):
        got = run(monkeypatch, dtype, sd, ids[:n].contiguous(), None, None)
        for stop, name in TAPS.items():
            v = got[stop].view(torch.float16 if dtype == "fp16" else torch.bfloat16)
            assert torch.isfinite(v.float()).all(), f"{dtype}, B={n}: launch {stop} {name} is not finite"
            assert torch.equal(got[stop], ref[stop][:n]), f"{dtype}, B={n}: launch {stop} {name} differs from the same layouts at B={B}"
