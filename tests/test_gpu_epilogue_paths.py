"""GPU (-m gpu): the step epilogue draws the same ids whether or not its log-probabilities are requested.

`Engine.step` takes the group-centric draw kernel (posterior_sample_group_kernel) where it applies, and the all-classes kernel
(posterior_sample_kernel) whenever the log-prob tap is requested (`want_logprob=True`, every oracle test's log-prob check).  Both
run posterior_token_group for the tokens it can prove safe and posterior_token_generic for the rest, so the ids must be equal
bit for bit.  The cases go where the two could part: near ties built from the known noise (the last bit of a reduction decides
them), the fallback's edges (temperatures around kGroupMargin, refinement rows that lift an out-of-group class, fixed tokens
outside their group, PAD-disable, top_p on both sides of 0.9999), the vocabularies ldm_create accepts with n_bins != 32, and
serialized steps at the benchmark's shapes.  Each table counts the tokens drawn, the tokens on the group path and on the
fallback (restated on the host from the log-prob tap), and the ids that differ."""
from __future__ import annotations

import functools
from dataclasses import dataclass

import numpy as np
import pytest
import torch

from oracle import layoutdm_oracle as O
from oracle import torch_noise as TN

pytestmark = pytest.mark.gpu

LOG_EPS32 = np.float32(O.LOG_EPS)
GROUP_MARGIN = {"contract": 40.0, "torch": 48.0}       # TokenNoise / TorchNoise::kGroupMargin (csrc/common.cuh)
T_DIFF = 100
MIN_PATH = 1000                                        # tokens each path must see in a case meant to reach both


@dataclass(frozen=True)
class Voc:
    dataset: str
    n_bins: int

    @property
    def vocab(self):
        from layoutdm_b200 import Vocab
        return Vocab(n_cat=Vocab.for_dataset(self.dataset).n_cat, n_bins=self.n_bins)

    @property
    def spec(self) -> O.VocabSpec:
        return O.VocabSpec(n_cat=self.vocab.n_cat, n_bins=self.n_bins)

    @property
    def group_path(self) -> bool:                      # every group <= 32 classes (group_path_applies)
        return self.vocab.n_cat <= 32 and self.n_bins <= 32

    def __str__(self):
        return f"{self.dataset}/{self.n_bins} bins"


RICO = Voc("rico25", 32)
VOCABS = [RICO, Voc("rico25", 26), Voc("rico25", 30), Voc("rico25", 33), Voc("publaynet", 31), Voc("publaynet", 38)]


@functools.lru_cache(maxsize=1)
def engine(voc: Voc):
    """a one-layer handle: every step here is fed its logits, the denoiser's weights do not matter"""
    from layoutdm_b200 import Engine
    from layoutdm_b200.synthetic import random_state_dict
    torch.cuda.empty_cache()
    return Engine.from_state_dict(random_state_dict(voc.vocab, num_timesteps=T_DIFF, layers=1, seed=0), voc.vocab, num_timesteps=T_DIFF)


def device_policy():
    p = torch.cuda.get_device_properties(torch.cuda.current_device())
    return p.multi_processor_count, p.max_threads_per_multi_processor


def in_group_table(spec: O.VocabSpec, dev="cpu") -> torch.Tensor:
    """(S, C) bool: class c belongs to token position s's vocabulary group (its attribute's classes, PAD, MASK)"""
    m = torch.zeros(spec.S, spec.C, dtype=torch.bool)
    for a in range(spec.n_attr):
        m[a::spec.n_attr, spec.group_full_ids(a)] = True
    return m.to(dev)


# ---- the noise of a call, on the host ---------------------------------------------------------------------------------------
@dataclass
class Noise:
    kind: str                  # "contract" | "torch"
    seed: int
    step_ctr: int = 0          # contract
    offset: int = 0            # torch

    def kw(self, B):
        if self.kind == "contract":
            return dict(seed=self.seed, step_ctr=self.step_ctr)
        from layoutdm_b200._lib import LdmNoise, NOISE_KINDS
        return dict(noise=LdmNoise(NOISE_KINDS["torch"], self.seed, self.offset, B))

    def variates(self, B, S, C, gumbel):
        """(e, u_gumbel or None) as float32 numpy (B, S, C): what the draw kernels use for token (b, s), class c"""
        if self.kind == "contract":
            u = O.uniforms(self.seed, self.step_ctr, 0, 0, B, S, C)
            e = (-np.log(u.astype(np.float64))).astype(np.float32)
            return e, (O.uniforms(self.seed, self.step_ctr, 1, 0, B, S, C) if gumbel else None)
        e, ug, _ = TN.draw_noise(self.seed, self.offset, B, S, C, gumbel, *device_policy())
        return e, ug

    def score_noise(self, B, S, C, gumbel, dev):
        """float64 (B, S, C) the draw adds to lp / T before its argmax: Gumbel noise (name="gumbel") - log e"""
        e, ug = self.variates(B, S, C, gumbel)
        z = -torch.from_numpy(e).double().log()
        if ug is not None:
            z = z - torch.log(-torch.log(torch.from_numpy(ug).double() + 1e-30) + 1e-30)
        return z.to(dev)


# ---- the two paths, the host's count of the group path, the oracle ------------------------------------------------------------
def step_applies(voc: Voc, cfg: dict) -> bool:
    """group_path_applies restated: constrained, every group <= 32 classes, a mode the group routine draws"""
    name = cfg["name"]
    return voc.group_path and (name in ("deterministic", "random", "gumbel") or (name == "top_p" and np.float32(cfg.get("top_p", 0.9)) < np.float32(0.9999)))


def group_path_mask(voc: Voc, cfg: dict, noise_kind: str, lp: torch.Tensor, cond=None) -> torch.Tensor:
    """(B, S) bool: the tokens posterior_token_group takes, restated from the log-prob tap (float32 like the kernel)"""
    B, S, C = lp.shape
    if not step_applies(voc, cfg):
        return torch.zeros(B, S, dtype=torch.bool, device=lp.device)
    ing = in_group_table(voc.spec, lp.device)
    lmax = lp.masked_fill(~ing[None], -float("inf")).amax(-1)
    margin = 0.0 if cfg["name"] == "deterministic" else float(np.float32(GROUP_MARGIN[noise_kind]) * np.float32(cfg.get("temperature", 1.0)))
    ok = (lmax - float(LOG_EPS32)) > margin                 # one float32 subtraction, like the kernel
    if cond is not None and cond.get("refine_table") is not None:
        fixed = cond["mask"].bool() if cond.get("mask") is not None else torch.zeros_like(ok)
        rows = cond["refine_table"].to(lp.device)[cond["seq_orig"].to(lp.device)]         # (B, S, C)
        lifts = (rows.masked_fill(ing[None], 0.0) > 0).any(-1)
        ok &= ~(lifts & ~fixed.to(lp.device))
    return ok


def both_paths(eng, x_t, t_post, cfg, noise: Noise, logits, cond=None):
    """ids without the tap (the group kernel where it applies), ids and log-probs with it (the all-classes kernel)"""
    B = x_t.shape[0]
    kw = noise.kw(B)
    ids_g, _, _ = eng.step(x_t, t_post, t_post, cfg, cond, logits_in=logits, **kw)
    ids_a, _, lp = eng.step(x_t, t_post, t_post, cfg, cond, logits_in=logits, want_logprob=True, **kw)
    torch.cuda.synchronize()
    return ids_g, ids_a, lp


class Table:
    def __init__(self, title):
        self.rows, self.title = [], title
        self.tot = dict(drawn=0, group=0, fallback=0, differ=0)

    def add(self, label, drawn, group, differ, extra=""):
        self.rows.append(f"  {label:44s} {drawn:8d} {group:8d} {drawn - group:9d} {differ:7d} {extra}")
        for k, v in (("drawn", drawn), ("group", group), ("fallback", drawn - group), ("differ", differ)):
            self.tot[k] += v

    def show(self):
        print(f"\n{self.title}\n  {'case':44s} {'drawn':>8s} {'group':>8s} {'fallback':>9s} {'differ':>7s}")
        print("\n".join(self.rows))
        t = self.tot
        print(f"  {'total':44s} {t['drawn']:8d} {t['group']:8d} {t['fallback']:9d} {t['differ']:7d}")


def cuda_cond(cond):
    return None if cond is None else {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in cond.items()}


def oracle_check(voc: Voc, cfg: dict, noise: Noise, logits, x_t, t_post, cond, ids, lp):
    """O.draw on O.logprob_from_logits under the contract noise: ids bit for bit, log-probs within 1e-4; returns the number of
    differing ids"""
    spec = voc.spec
    orc = O.Oracle(spec, O.ModelSpec(T=T_DIFF), {})
    lp_o = orc.logprob_from_logits(logits.cpu(), x_t.cpu(), t_post, cond)
    err = float((lp.cpu() - lp_o).abs().max())
    assert err < 1e-4, f"log-probs differ from the oracle's by {err:.2e}"
    ocfg = O.SamplingCfg(name=cfg["name"], temperature=cfg.get("temperature", 1.0), top_p=cfg.get("top_p", 0.9), top_k=cfg.get("top_k", 5))
    B = x_t.shape[0]
    u = O.uniforms(noise.seed, noise.step_ctr, 0, 0, B, spec.S, spec.C)
    ug = O.uniforms(noise.seed, noise.step_ctr, 1, 0, B, spec.S, spec.C) if cfg["name"] == "gumbel" else None
    want = O.draw(lp_o, ocfg, u, ug)
    return int((ids.cpu() != want).sum())


# ---- 1. near ties built from the known noise --------------------------------------------------------------------------------
def posterior64(spec: O.VocabSpec, sch64, logits64, x_t, t):
    """float64 log p(x_{t-1} | x_t) of the oracle on the handle's schedule tables"""
    lx = torch.log_softmax(logits64[..., :-1], -1).clamp(-70.0, 0.0)
    lx = torch.cat([lx, torch.full_like(lx[..., :1], -70.0)], -1)
    return O.q_posterior(lx, x_t, t, T_DIFF, spec, sch64)


def design_ties(spec, sch64, logits, x_t, t, z, temp, ing):
    """raise one in-group class's logit (bisection, per token) until its score lp / temp + z ties the winner's; the class is the
    one of the winner's runner-up and the four best-noised in-group classes that gets furthest past the winner at +40.
    Returns (logits, reachable)."""
    B, S, C = logits.shape
    score = lambda lg: posterior64(spec, sch64, lg, x_t, t) / temp + z
    sc = score(logits)
    a = sc.argmax(-1)
    movable = ing.clone()
    movable[:, spec.mask_id] = False
    cand_ok = movable[None].expand(B, -1, -1).clone()
    cand_ok.scatter_(-1, a[..., None], False)
    runner = sc.masked_fill(~cand_ok, -float("inf")).argmax(-1, keepdim=True)
    cands = torch.cat([runner, z.masked_fill(~cand_ok, -float("inf")).topk(4, -1).indices], -1)
    best_f = torch.full((B, S), -float("inf"), dtype=torch.float64, device=logits.device)
    b = runner[..., 0].clone()
    for k in range(cands.shape[-1]):
        c = cands[..., k:k + 1]
        lg = logits.clone()
        lg.scatter_add_(-1, c, torch.full(c.shape, 40.0, dtype=torch.float64, device=logits.device))
        s2 = score(lg)
        f = s2.gather(-1, c)[..., 0] - s2.gather(-1, a[..., None])[..., 0]
        f = torch.where(cand_ok.gather(-1, c)[..., 0], f, torch.full_like(f, -float("inf")))
        up = f > best_f
        best_f, b = torch.where(up, f, best_f), torch.where(up, c[..., 0], b)
    reach = best_f > 0
    x0 = logits.gather(-1, b[..., None])[..., 0]
    lo, hi = torch.zeros_like(x0), torch.full_like(x0, 40.0)
    for _ in range(64):
        mid = 0.5 * (lo + hi)
        lg = logits.clone()
        lg.scatter_(-1, b[..., None], (x0 + mid)[..., None])
        s2 = score(lg)
        f = s2.gather(-1, b[..., None])[..., 0] - s2.gather(-1, a[..., None])[..., 0]
        lo, hi = torch.where(f < 0, mid, lo), torch.where(f < 0, hi, mid)
    out = logits.clone()
    out.scatter_(-1, b[..., None], torch.where(reach, x0 + hi, x0)[..., None])
    return out, reach


def tie_gap(spec, sch64, logits, x_t, t, z, temp):
    """relative float64 gap between the two best scores of every token"""
    top = (posterior64(spec, sch64, logits, x_t, t) / temp + z).topk(2, -1).values
    return (top[..., 0] - top[..., 1]).abs() / top[..., 0].abs().clamp(min=1.0)


def near_tie_inputs(voc: Voc, eng, cfg, noise: Noise, t, B, seed):
    """logits and x_t of B layouts whose winning scores tie in float64, per token where the posterior lets them.  x_t takes
    turns over MASK, the in-group class the noise favours least and PAD; a token whose tie its own x_t kind cannot reach tries
    the others (a non-MASK x_t holds most of the posterior's mass in mid-schedule, MASK does late)."""
    dev = "cuda"
    spec = voc.spec
    S, C = spec.S, spec.C
    sch = eng.schedule_tables()
    sch64 = [{name: sch[g, r].double().to(dev) for r, name in enumerate(O.SCHED_NAMES)} for g in range(spec.n_attr)]
    ing = in_group_table(spec, dev)
    g = torch.Generator().manual_seed(seed)
    logits = (torch.randn(B, S, C, generator=g, dtype=torch.float64) * 2.0).to(dev)
    temp = float(np.float32(cfg.get("temperature", 1.0)))
    if cfg["name"] == "deterministic":
        z = torch.zeros(B, S, C, dtype=torch.float64, device=dev)
        temp = 1.0
    else:
        z = noise.score_noise(B, S, C, cfg["name"] == "gumbel", dev)
    normal = ing.clone()
    normal[:, [spec.pad_id, spec.mask_id]] = False
    worst = z.masked_fill(~normal[None], float("inf")).argmin(-1)
    options = [torch.full((B, S), spec.mask_id, device=dev), worst, torch.full((B, S), spec.pad_id, device=dev)]
    kind = (torch.arange(B * S, device=dev) % 3).view(B, S)
    x_t = torch.zeros(B, S, dtype=torch.long, device=dev)
    done = torch.zeros(B, S, dtype=torch.bool, device=dev)
    for shift in range(3):                                  # each token's own kind first, then the next ones
        k = (kind + shift) % 3
        cand = torch.where(k == 0, options[0], torch.where(k == 1, options[1], options[2]))
        _, reach = design_ties(spec, sch64, logits, cand, t, z, temp, ing)
        take = ~done & (reach | (shift == 2))
        x_t = torch.where(take, cand, x_t)
        done |= take
    logits, reach = design_ties(spec, sch64, logits, x_t, t, z, temp, ing)
    designed = reach & (tie_gap(spec, sch64, logits, x_t, t, z, temp) < 2.0 ** -20)
    return logits.float(), x_t, designed


TIE_T = [0, 1, 2, 5, 10, 25, 50, 75, 98, 99]


@pytest.mark.parametrize("noise_kind", ["contract", "torch"])
@pytest.mark.parametrize("mode", ["random", "gumbel", "deterministic"])
def test_near_ties_same_ids_on_both_paths(mode, noise_kind):
    _near_ties(RICO, mode, noise_kind, B=8)


@pytest.mark.parametrize("voc", VOCABS[1:], ids=str)
def test_near_ties_other_vocabularies(voc):
    assert engine(voc) is not None and step_applies(voc, {"name": "random"}) == (voc.n_bins <= 32)
    _near_ties(voc, "random", "contract", B=4)


def _near_ties(voc: Voc, mode: str, noise_kind: str, B: int):
    eng = engine(voc)
    cfg = {"name": mode, "temperature": 1.0}
    tab = Table(f"near ties: {voc}, {mode}, {noise_kind} noise, B={B} per timestep")
    n_tok = n_designed = 0
    bad = []
    for i, t in enumerate(TIE_T):
        noise = Noise(noise_kind, seed=1000 + i, step_ctr=i, offset=4 * 97 * i)
        logits, x_t, designed = near_tie_inputs(voc, eng, cfg, noise, t, B, seed=i)
        ids_g, ids_a, lp = both_paths(eng, x_t, t, cfg, noise, logits)
        grp = group_path_mask(voc, cfg, noise_kind, lp)
        differ = int((ids_g != ids_a).sum())
        kinds = f"designed ties {int(designed.sum())}/{designed.numel()} (x_t MASK {int((x_t == voc.spec.mask_id).sum())}, PAD {int((x_t == voc.spec.pad_id).sum())})"
        tab.add(f"t_post={t}", x_t.numel(), int(grp.sum()), differ, kinds)
        n_tok += x_t.numel()
        n_designed += int(designed.sum())
        if differ:
            bad.append(f"t_post={t}: {differ} ids differ")
    tab.show()
    assert not bad, "; ".join(bad)
    # deterministic: without noise a tie is reachable only where the posterior follows log p(x0) (t_post near 0 and T - 1); in
    # mid-schedule the x_t kinds hold a floor of the posterior's mass no logit can tie
    # (publaynet's 5-class label group offers fewer candidate classes: 85 % there)
    need = 0.15 if mode == "deterministic" else (0.9 if voc.vocab.n_cat > 5 else 0.85)
    print(f"  designed ties: {n_designed} of {n_tok} tokens ({n_designed / n_tok:.1%}, at least {need:.0%} required)")
    assert n_designed >= need * n_tok
    if voc.group_path:
        assert tab.tot["group"] >= MIN_PATH // 2
    else:
        assert tab.tot["group"] == 0


# ---- 2. the fallback and its edges ------------------------------------------------------------------------------------------
TEMPS = [0.05, 0.3, 1.0, 1.4, 1.5, 1.7, 1.75, 2.5]


def edge_inputs(voc: Voc, temp: float, noise_kind: str, B: int, seed: int):
    """tokens around the fallback's edges, one call: refinement cond at t_post = 0, x_t = a class of the token's group whose logit
    dominates (log p ~ 0), the caller's refinement rows shift the group to lmax - log(1e-30) = margin -+ 0.01 (rows of ids = 0 / 1
    mod 3 of each group), lift one out-of-group class to +0.5 (ids = 2 mod 3); every 7th token fixed, alternately to a class of
    its group and to one outside it; PAD-disabled where the seq is not PAD"""
    spec = voc.spec
    S, C, A = spec.S, spec.C, spec.n_attr
    g = torch.Generator().manual_seed(seed)
    margin = float(np.float32(GROUP_MARGIN[noise_kind]) * np.float32(temp))
    k_below, k_above = O.LOG_EPS * -1 - margin + 0.01, O.LOG_EPS * -1 - margin - 0.01
    tbl = torch.zeros(C, C)
    s = torch.arange(S)
    grp_lo = torch.tensor([spec.group_start(a) for a in range(A)])[s % A]
    grp_n = torch.tensor([spec.group_n(a) for a in range(A)])[s % A]
    for a in range(A):
        ids = spec.group_full_ids(a)[:-2]
        for j, r in enumerate(ids):
            k = k_below if j % 3 == 0 else k_above
            tbl[r, ids] = -k
            tbl[r, spec.pad_id] = -k
            tbl[r, spec.mask_id] = -k
            if j % 3 == 2:
                tbl[r, spec.group_full_ids((a + 1) % A)[0]] = 0.5
    x_t = grp_lo + (torch.rand(B, S, generator=g) * grp_n).long()
    seq_orig = grp_lo + (torch.rand(B, S, generator=g) * grp_n).long()
    logits = torch.randn(B, S, C, generator=g)
    logits.scatter_add_(-1, x_t[..., None], torch.full((B, S, 1), 40.0))
    fixed = torch.zeros(B, S, dtype=torch.bool)
    fixed.view(-1)[::7] = True
    seq = torch.full((B, S), spec.mask_id)
    inside = grp_lo + (torch.rand(B, S, generator=g) * grp_n).long()
    outside = (inside + spec.n_cat + 2 * spec.n_bins) % (C - 2)            # another attribute's class
    alt = torch.zeros(B, S, dtype=torch.bool)
    alt.view(-1)[::14] = True
    seq = torch.where(fixed, torch.where(alt, outside, inside), seq)
    seq.view(-1)[3::11] = spec.pad_id                                      # PAD-disable off for these
    cond = dict(seq=seq, mask=fixed, type="refinement", seq_orig=seq_orig, refine_table=tbl)
    return logits, x_t, cond


def natural_inputs(voc: Voc, B: int, seed: int, scale: float = 3.0):
    spec = voc.spec
    g = torch.Generator().manual_seed(seed)
    logits = torch.randn(B, spec.S, spec.C, generator=g) * scale
    x_t = torch.randint(0, spec.C, (B, spec.S), generator=g)
    return logits, x_t


def reference_cond(voc: Voc, B: int, mode: str, seed: int):
    """the reference's own refinement tables (task.py:154-224, linear centres) on a cond = refinement with a few fixed labels"""
    spec = voc.spec
    g = torch.Generator().manual_seed(seed)
    seq_orig = torch.randint(0, spec.C - 2, (B, spec.S), generator=g)
    fixed = torch.zeros(B, spec.S, dtype=torch.bool)
    fixed[:, 0::spec.n_attr] = torch.rand(B, spec.n_elem, generator=g) < 0.5
    seq = torch.where(fixed, seq_orig, torch.full_like(seq_orig, spec.mask_id))
    tbl = O.refinement_table(spec, O.linear_centers(spec.n_bins), mode=mode)
    return dict(seq=seq, mask=fixed, type="refinement", seq_orig=seq_orig, refine_table=tbl)


@pytest.mark.parametrize("voc", VOCABS, ids=str)
def test_fallback_edges(voc):
    """every case path against path, and under the contract noise against O.draw (ids bit for bit, log-probs within 1e-4)"""
    eng = engine(voc)
    B = 24
    tab = Table(f"fallback edges: {voc}, B={B}")
    bad = []
    for noise_kind in ("contract", "torch"):
        for i, temp in enumerate(TEMPS):
            for mode in ("random", "gumbel"):
                cfg = {"name": mode, "temperature": temp}
                noise = Noise(noise_kind, seed=77 + i, step_ctr=i, offset=4 * 13 * i)
                logits, x_t, cond = edge_inputs(voc, temp, noise_kind, B, seed=i)
                c = cuda_cond(cond)
                ids_g, ids_a, lp = both_paths(eng, x_t.cuda(), 0, cfg, noise, logits.cuda(), c)
                grp = group_path_mask(voc, cfg, noise_kind, lp, c)
                differ = int((ids_g != ids_a).sum())
                fixed = cond["mask"].cuda()
                assert torch.equal(ids_g[fixed], c["seq"][fixed]), "fixed tokens not kept"
                o = oracle_check(voc, cfg, noise, logits, x_t, 0, cond, ids_a, lp) if noise_kind == "contract" else 0
                tab.add(f"{noise_kind} {mode} T={temp} margin edge", x_t.numel(), int(grp.sum()), differ, f"oracle differs {o}")
                if differ or o:
                    bad.append(f"{noise_kind} {mode} T={temp}: {differ} ids differ between the paths, {o} from the oracle")
                # the rows of ids 0 mod 3 sit just below the margin, the others just above unless they lift an out-of-group class
                if voc.group_path and not (0 < int(grp.sum()) < x_t.numel()):
                    bad.append(f"{noise_kind} {mode} T={temp}: the margin edge does not split the tokens ({int(grp.sum())} on the group path)")
                if not voc.group_path and int(grp.sum()):
                    bad.append(f"{noise_kind} {mode} T={temp}: {int(grp.sum())} tokens on the group path of a vocabulary it does not serve")
    # natural logits at every temperature, the reference's own refinement tables, top_p around 0.9999, and the all-classes modes
    j = 0
    for temp in TEMPS:
        cfgs = [{"name": "random", "temperature": temp}, {"name": "top_k", "top_k": 1, "temperature": temp},
                {"name": "top_k", "top_k": voc.spec.C, "temperature": temp}]
        if temp in (0.3, 1.0, 1.4):
            cfgs += [{"name": "top_p", "top_p": p, "temperature": temp} for p in (0.05, 0.9, 0.99985, 0.9999)]
            cfgs += [{"name": "deterministic"}, {"name": "gumbel", "temperature": temp}]
        for cfg in cfgs:
            for cond_mode in (None, "uniform", "gaussian", "negative"):
                if cond_mode is not None and cfg["name"] not in ("random", "top_p"):
                    continue
                j += 1
                noise = Noise("contract", seed=500 + j, step_ctr=j)
                logits, x_t = natural_inputs(voc, B, seed=j)
                cond = reference_cond(voc, B, cond_mode, seed=j) if cond_mode else None
                t_post = (17 * j) % T_DIFF
                c = cuda_cond(cond)
                ids_g, ids_a, lp = both_paths(eng, x_t.cuda(), t_post, cfg, noise, logits.cuda(), c)
                grp = group_path_mask(voc, cfg, "contract", lp, c)
                differ = int((ids_g != ids_a).sum())
                o = oracle_check(voc, cfg, noise, logits, x_t, t_post, cond, ids_a, lp)
                label = f"{cfg['name']} T={cfg.get('temperature', 1.0)}" + (f" p={cfg['top_p']}" if "top_p" in cfg else "") + \
                        (f" k={cfg['top_k']}" if "top_k" in cfg else "") + (f" {cond_mode}" if cond_mode else "")
                tab.add(label, x_t.numel(), int(grp.sum()), differ, f"oracle differs {o}")
                if differ or o:
                    bad.append(f"{label}: {differ} ids differ between the paths, {o} from the oracle")
                if cfg["name"] == "top_p" and cfg["top_p"] >= 0.9999 and int(grp.sum()):
                    bad.append(f"{label}: top_p >= 0.9999 must take the all-classes routine")
    tab.show()
    assert not bad, "\n".join(bad)
    if voc.group_path:
        assert tab.tot["group"] >= MIN_PATH and tab.tot["fallback"] >= MIN_PATH
    else:
        assert tab.tot["group"] == 0


# ---- 4. natural inputs at the benchmark's shapes ----------------------------------------------------------------------------
BENCH = {"config0": ("rico25", 8, 50, {"name": "random", "temperature": 1.0}, None),
         "config2": ("publaynet", 1024, 100, {"name": "top_p", "temperature": 1.0, "top_p": 0.9}, "c"),
         "config2_T1.5": ("publaynet", 1024, 100, {"name": "top_p", "temperature": 1.5, "top_p": 0.9}, "c")}


@pytest.mark.parametrize("name", list(BENCH))
def test_serialized_steps_same_ids_on_both_paths(name):
    """serialized steps with the logits tap, then each step's epilogue run both ways on those logits: every id equal to the step's"""
    from layoutdm_b200 import Engine, Vocab, timestep_plan
    from layoutdm_b200.synthetic import random_state_dict, synthetic_cond
    dataset, B, T_eval, cfg, cond_type = BENCH[name]
    vocab = Vocab.for_dataset(dataset)
    voc = Voc(dataset, 32)
    engine.cache_clear()
    torch.cuda.empty_cache()
    eng = Engine.from_state_dict(random_state_dict(vocab, num_timesteps=100, seed=0), vocab, num_timesteps=100)
    cond = None
    if cond_type:
        cond = {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in synthetic_cond(vocab, B, cond_type, seed=0).items()}
        x = cond["seq"]
    else:
        x = torch.full((B, vocab.S), vocab.mask_id, dtype=torch.int64, device="cuda")
    tab = Table(f"serialized steps: {name}, B={B}, {cfg}")
    bad = []
    for i, (tm, tp) in enumerate(timestep_plan(100, T_eval)):
        nxt, lg, _ = eng.step(x, tm, tp, cfg, cond, seed=10, step_ctr=i, want_logits=True)
        ids_g, _, _ = eng.step(x, tm, tp, cfg, cond, seed=10, step_ctr=i, logits_in=lg)
        ids_a, _, lp = eng.step(x, tm, tp, cfg, cond, seed=10, step_ctr=i, logits_in=lg, want_logprob=True)
        grp = group_path_mask(voc, cfg, "contract", lp, cond)
        differ = int((ids_g != ids_a).sum())
        if i % 10 == 0 or differ:
            tab.add(f"step {i} (t_post={tp})", x.numel(), int(grp.sum()), differ)
        else:
            tab.add(f"step {i}", x.numel(), int(grp.sum()), differ)
        if differ or not torch.equal(ids_g, nxt):
            bad.append(f"step {i}: {differ} ids differ between the paths, {int((ids_g != nxt).sum())} from the step")
        x = nxt
    tab.rows = [r for r in tab.rows if "t_post" in r]
    tab.show()
    eng.close()
    assert not bad, "\n".join(bad)
    assert tab.tot["group"] >= MIN_PATH         # at T = 1.5 too: the contract noise's fallback starts above T = 69.08 / 40
