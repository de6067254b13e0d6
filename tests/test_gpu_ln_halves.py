"""GPU (-m gpu): the LN GEMMs' row-half pipeline gives every row the same bits whatever number of tiles its CTA pair runs.

gemm_ln_kernel hands its tile buffer over by row half: the epilogue walks (tile 0, half 0), (0, 1), (1, 0), ..., the next
tile's residual rows of a half are loaded as soon as the half's last bulk store has read it, and the LayerNorm exchange
barriers alternate by (tile parity, half).  The edges of that hand-off are a pair that runs exactly one tile (no next
load, one parity used) and pairs that run an odd number of tiles (the parities end unbalanced).  With B = 7 and 13 row blocks,
LDM_GEMM_CTAS = 2, 6, 10, 16 runs 1, 3, 5, 8 pairs: 7 or 13 tiles on one pair; 3 + 2 + 2 and 5 + 4 + 4; 2 + 2 + 1 + 1 + 1 and
3 + 3 + 3 + 2 + 2; seven pairs of one tile and 2 + ... + 1.  The tapped y32 / z16 / x32 / x16 must be bitwise those of the
uncapped launch, in which every pair runs one tile."""
import pytest

from test_gpu_ln_pair import inputs, run, weights

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
@pytest.mark.parametrize("B", [7, 13])
def test_ln_halves_outputs_independent_of_tiles_per_pair(monkeypatch, dtype, B):
    import torch
    sd = weights(41)
    ids, t = inputs(B, 42)
    for per_layout in (False, True):
        tt = t if per_layout else None
        ref = run(monkeypatch, dtype, sd, None, ids, tt)
        for cap in (2, 6, 10, 16):
            got = run(monkeypatch, dtype, sd, cap, ids, tt)
            bad = [f"launch {n} {k}" for (n, k), v in ref.items() if not torch.equal(v, got[(n, k)])]
            assert not bad, (f"{dtype}, B={B}, LDM_GEMM_CTAS={cap}{', per-layout timesteps' if per_layout else ''}: "
                             f"not bitwise equal to the uncapped run: {bad}")
