"""CPU: the split ("bf16x3") operand references (split_refs.py) -- the pair hi = bf16(x), lo = bf16(x - hi) and the forward built on it."""
import torch

import split_refs as SR
from oracle import layoutdm_oracle as O


def test_pair_bounds_over_the_exponent_range():
    """|lo| <= 2^-8 |x| and |x - (hi + lo)| <= 2^-16 |x| wherever lo is a normal bf16 (|x| >= 2^-118); below that lo is
    subnormal and the pair is still within half a bf16 subnormal spacing (2^-134) of x.  Up to the largest bf16 (3.39e38);
    beyond it hi rounds to inf"""
    g = torch.Generator().manual_seed(0)
    m = 1.0 + torch.rand(200_000, generator=g, dtype=torch.float64)
    e = torch.randint(-133, 127, (m.numel(),), generator=g)
    x = (torch.ldexp(m, e.double()) * torch.where(torch.rand(m.numel(), generator=g) < 0.5, -1.0, 1.0)).float()
    edge = torch.tensor([2.0 ** -126, 2.0 ** -118, 1.5 * 2.0 ** -118, 2.0 ** -126 * 1.999, 1.0 + 2.0 ** -8, 1.0 + 2.0 ** -9 + 2.0 ** -20,
                         3.38e38, 1.0 - 2.0 ** -24, 2.0 ** -127, 2.0 ** -149])
    x = torch.cat([x, edge, -edge])
    x = x[x.abs() <= 3.38e38]
    hi, lo = SR.split_bf16(x)
    assert torch.isfinite(hi).all() and torch.isfinite(lo).all()
    xd, err = x.double(), (x.double() - (hi.double() + lo.double())).abs()
    normal = xd.abs() >= 2.0 ** -118
    assert (lo.double().abs() <= 2.0 ** -8 * xd.abs()).all()
    assert (err[normal] <= 2.0 ** -16 * xd.abs()[normal]).all(), f"max rel {(err[normal] / xd.abs()[normal]).max():.3e}"
    assert (err <= torch.maximum(2.0 ** -16 * xd.abs(), torch.full_like(xd, 2.0 ** -134))).all()
    # the pair is exact where x has at most 16 significant bits
    y = torch.ldexp(torch.randint(1 << 15, 1 << 16, (1000,), generator=g).double(), torch.randint(-100, 100, (1000,), generator=g).double()).float()
    h2, l2 = SR.split_bf16(y)
    assert torch.equal(h2.double() + l2.double(), y.double())


def test_matmul_bf16x3_drops_only_lo_lo():
    g = torch.Generator().manual_seed(1)
    a, b = torch.randn(64, 464, generator=g), torch.randn(464, 96, generator=g)
    exact = a.double() @ b.double()
    got = SR.matmul_bf16x3(a, b).double()
    bound = 2.0 ** -16 * (a.double().abs() @ b.double().abs()) + 64 * 2.0 ** -24 * (a.double().abs() @ b.double().abs())
    assert ((got - exact).abs() <= bound).all()
    assert (SR.matmul_bf16x3(a, b) - a @ b).abs().max() < 1e-3 * (a.abs() @ b.abs()).max()


def test_oracle_bf16x3_forward_matches_fp32_at_reference_scale():
    """the split forward stays within 1e-4 of the fp32 forward at the reference's weight scale (fp16 operands: ~1e-3)"""
    vo, spec = O.RICO25, O.ModelSpec()
    sd = O.make_weights(vo, spec, seed=0)
    g = torch.Generator().manual_seed(0)
    worst = 0.0
    with torch.no_grad():
        for t in (0, 42, 99):
            ids = torch.randint(0, vo.C, (2, vo.S), generator=g)
            ids[0, :40] = vo.mask_id
            ref = O.denoiser_forward(sd, ids, t, vo, spec)
            got = SR.denoiser_forward_bf16x3(sd, ids, t, vo, spec)
            worst = max(worst, (got - ref).abs().max().item())
    print(f"oracle bf16x3 vs fp32 forward: max |d| {worst:.2e}")
    assert worst < 1e-4
