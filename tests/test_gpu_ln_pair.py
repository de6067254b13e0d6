"""GPU (-m gpu): the out-projection / FF2 LN GEMMs in fp16 / bf16 compute every row the same way whatever CTA pair computes it.

gemm_ln_kernel runs clusters of two CTAs; a pair takes one layout's 128-row block at a time, each CTA 232 of its 464 columns,
and the two exchange their halves' LayerNorm row statistics through double-buffered slots in each other's shared memory.
LDM_GEMM_CTAS=n runs max(1, n / 2) pairs: with 1 and 2 a single pair walks every row block of a launch, with 4 and 6 the
row blocks of B = 67 and B = 301 do not divide evenly among the pairs.  At per-layout timesteps (predict_start) FF2's AdaLN
reads the (scale, shift) row of the tile's own layout, so a pair's consecutive tiles normalise with different rows and a stale
exchange slot would show.  The tapped outputs of both LN GEMMs of every layer must be bitwise equal to the uncapped run's,
and a layout's rows must be the same at every batch size."""
import pytest
import torch

import gpu_helpers as G
from oracle import layoutdm_oracle as O
from test_gpu_parity_large import mixed_ids

pytestmark = pytest.mark.gpu

LAYERS = 2
T = 20
# launch count to stop after -> what it leaves: layer l's out-projection is launch 4 + 5 l (y32, z16), its FF2 launch 6 + 5 l
# (x32, x16: the next layer's AdaLN; the last layer's FF2 writes the head LayerNorm into z16)
TAPS = {4: ("y32", "z16"), 6: ("x32", "x16"), 4 + 5 * (LAYERS - 1): ("y32", "z16"), 1 + 5 * LAYERS: ("z16",)}


def weights(seed):
    return O.make_weights(O.RICO25, O.ModelSpec(layers=LAYERS, T=T), seed=seed, scale=2.0)


def inputs(n, seed):
    ids = mixed_ids(n, O.RICO25, seed).cuda()
    t = torch.randint(0, T, (n,), generator=torch.Generator().manual_seed(seed + 1))
    t[0], t[-1] = 0, T - 1
    return ids, t.cuda()


def run(monkeypatch, dtype, sd, cap, ids, t):
    """the bits of the tapped LN GEMM outputs: one step at timestep 7 (t None) or predict_start at per-layout timesteps t"""
    from layoutdm_b200 import Engine, Vocab
    vo = O.RICO25
    if cap is None:
        monkeypatch.delenv("LDM_GEMM_CTAS", raising=False)
    else:
        monkeypatch.setenv("LDM_GEMM_CTAS", str(cap))
    eng = Engine.from_state_dict(sd, Vocab(vo.n_cat, vo.n_bins, vo.n_elem, vo.n_attr), num_timesteps=T, operand_dtype=dtype)
    n = ids.shape[0]
    out = {}
    try:
        for stop, names in TAPS.items():
            G.set_stop_after(eng, stop)
            if t is None:
                eng.step(ids, 7, 7, {"name": "deterministic"})
            else:
                eng.predict_start(ids, t)
            torch.cuda.synchronize()
            for k in names:
                v = G.debug_read(eng, k, n, raw=True)
                out[(stop, k)] = v.view(torch.int16 if v.element_size() == 2 else torch.int32).clone()
        G.set_stop_after(eng, 0)
    finally:
        eng.close()
    return out


@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
@pytest.mark.parametrize("B", [301, 67])
def test_ln_pair_outputs_independent_of_cluster_count(monkeypatch, dtype, B):
    sd = weights(31)
    ids, t = inputs(B, 32)
    for per_layout in (False, True):
        tt = t if per_layout else None
        ref = run(monkeypatch, dtype, sd, None, ids, tt)
        for cap in (1, 2, 4, 6):
            got = run(monkeypatch, dtype, sd, cap, ids, tt)
            bad = [f"launch {n} {k}" for (n, k), v in ref.items() if not torch.equal(v, got[(n, k)])]
            assert not bad, (f"{dtype}, B={B}, LDM_GEMM_CTAS={cap}{', per-layout timesteps' if per_layout else ''}: "
                             f"not bitwise equal to the uncapped run: {bad}")


@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
def test_ln_pair_rows_independent_of_batch(monkeypatch, dtype):
    sd = weights(33)
    ids, t = inputs(301, 34)
    for per_layout in (False, True):
        ref = run(monkeypatch, dtype, sd, None, ids, t if per_layout else None)
        for n in (1, 2, 67):
            got = run(monkeypatch, dtype, sd, None, ids[:n].contiguous(), t[:n].contiguous() if per_layout else None)
            bad = [f"launch {s} {k}" for (s, k), v in got.items() if not torch.equal(v, ref[(s, k)][:n])]
            assert not bad, (f"{dtype}, B={n}{', per-layout timesteps' if per_layout else ''}: "
                             f"the layouts' rows differ from the same layouts at B=301: {bad}")
