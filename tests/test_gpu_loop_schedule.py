"""GPU (-m gpu): the benchmarked sampling loop equals the serialized step path bit for bit, at the benchmark's shapes and under
every launch-schedule switch.

The per-kernel tests check each kernel against float64 through `ldm_step` / `ldm_predict_start`: plain stream launches and one
embedding launch per step.  `ldm_sample_loop`, the path bench.py times, differs from that in five ways: the T-step plan is
captured once as a CUDA graph; each replay takes its seed and `b_global0` from device words (`call_block`); the draw kernel
writes the next step's embedding rows, so no embedding kernel runs after the first step; every edge is a programmatic
dependent launch; and the kernels alternate their sweep direction, the QKV, FF1 and LN GEMMs on persistent grids.  Here the
loop is compared with a handle that has all of that switched off (`LDM_PDL=0 LDM_GRAPH=0 LDM_FUSE_EMBED=0 LDM_SWEEP=0`),
driven one `Engine.step` per plan entry with the same seed, step counter, `b_global0`, cond and start ids.

The graph path keeps no trace, so its intermediate states are read by running plan prefixes `plan[:k]`: the final ids and
the workspace logits (the last step's) of each prefix must equal the serialized step k - 1 bit for bit on every token row.
The pad rows s >= S of a layout tile are excluded where the embedding is fused: the draw writes token rows only, so from
the second step on the pad rows of x32 / x16 keep what the previous step's last AdaLN epilogue wrote, while the embedding
kernel zeroes them.  No token row reads them (attention masks keys >= S, every other kernel works row by row); they must
stay finite, and the tables print how many differ.  Without the fused embedding (the split mode, LDM_FUSE_EMBED=0) every
row must match.

One state of the loop at the benchmark shape is also tied to float64: test_loop_logits_vs_float64_at_benchmark_shape."""
from __future__ import annotations

import contextlib
import functools
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import pytest
import torch

import gpu_helpers as G
from oracle import layoutdm_oracle as O

pytestmark = pytest.mark.gpu

SWITCHES = ("LDM_PDL", "LDM_GRAPH", "LDM_FUSE_EMBED", "LDM_SWEEP", "LDM_GEMM_CTAS")
SERIAL = {"LDM_PDL": "0", "LDM_GRAPH": "0", "LDM_FUSE_EMBED": "0", "LDM_SWEEP": "0"}
MATRIX = [("default", {}), ("LDM_PDL=0", {"LDM_PDL": "0"}), ("LDM_GRAPH=0", {"LDM_GRAPH": "0"}),
          ("LDM_FUSE_EMBED=0", {"LDM_FUSE_EMBED": "0"}), ("LDM_SWEEP=0", {"LDM_SWEEP": "0"}), ("all four off", SERIAL),
          ("LDM_GEMM_CTAS=7", {"LDM_GEMM_CTAS": "7"})]
LAYERS = 4                    # random_state_dict's depth
LAUNCHES_PER_STEP = 1 + 5 * LAYERS + 2   # embedding, 5 per layer, head, draw
LOGIT_TOL = 1e-3              # test_gpu_parity.py's gate: max-abs on fp32 logits vs float64, weights at the reference's init scale
RANDOM = {"name": "random", "temperature": 1.0}


@dataclass(frozen=True)
class Workload:
    name: str
    dataset: str
    T: int
    T_eval: int
    B: int
    cfg: Tuple[Tuple[str, object], ...]
    cond_type: Optional[str] = None     # synthetic_cond type; its seq is also the start state (bench.py's configs 2 / 3)
    time_difference: float = 0.0
    seed: int = 10
    b_global0: int = 0

    @property
    def sampling(self) -> dict:
        return dict(self.cfg)

    @property
    def vocab(self):
        from layoutdm_b200 import Vocab
        return Vocab.for_dataset(self.dataset)

    @property
    def plan(self) -> List[Tuple[int, int]]:
        from layoutdm_b200 import timestep_plan
        return timestep_plan(self.T, self.T_eval, self.time_difference)


CFG_RANDOM = tuple(RANDOM.items())
CONFIG1 = Workload("config 1: rico25 unconditional, T=100, random", "rico25", 100, 100, 1024, CFG_RANDOM)
CONFIG2 = Workload("config 2: publaynet cond=c, top_p=0.9", "publaynet", 100, 100, 1024,
                   (("name", "top_p"), ("temperature", 1.0), ("top_p", 0.9)), cond_type="c")
CONFIG3 = Workload("config 3: rico25 refinement, T=200", "rico25", 200, 200, 4096, CFG_RANDOM, cond_type="refinement")
CONFIG0 = Workload("config 0 shape: T_eval=50 (skip steps)", "rico25", 100, 50, 8, CFG_RANDOM)
TAIL301 = Workload("odd tail B=301, T_eval=40, time_difference=0.05, b_global0=777", "rico25", 100, 40, 301, CFG_RANDOM,
                   time_difference=0.05, b_global0=777)
TAIL1 = Workload("odd tail B=1, top_k=5, cond=cwh", "rico25", 100, 100, 1, (("name", "top_k"), ("temperature", 1.0), ("top_k", 5)),
                 cond_type="cwh")


@functools.lru_cache(maxsize=4)
def state_dict(dataset: str, T: int):
    from layoutdm_b200 import Vocab
    from layoutdm_b200.synthetic import random_state_dict
    return random_state_dict(Vocab.for_dataset(dataset), num_timesteps=T, seed=0)


def inputs(wl: Workload, cond_seed: int = 0):
    """(cond, ids_init) on the GPU: bench.py's synthetic condition, whose seq is also the start state, or (None, None)"""
    if wl.cond_type is None:
        return None, None
    from layoutdm_b200.synthetic import synthetic_cond
    cond = {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in synthetic_cond(wl.vocab, wl.B, wl.cond_type, seed=cond_seed).items()}
    return cond, cond["seq"]


@contextlib.contextmanager
def handle(monkeypatch, wl: Workload, dtype: str, env: Dict[str, str]):
    """an Engine created with exactly the switches in env (the others unset), closed and its memory released on exit"""
    from layoutdm_b200 import Engine
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    torch.cuda.empty_cache()
    eng = Engine.from_state_dict(state_dict(wl.dataset, wl.T), wl.vocab, num_timesteps=wl.T, operand_dtype=dtype)
    try:
        yield eng
    finally:
        torch.cuda.synchronize()
        eng.close()
        del eng
        torch.cuda.empty_cache()


def prefixes(n: int) -> List[int]:
    return sorted({k for k in (1, 2, 3, n // 2, n) if 1 <= k <= n})


def bits(t: torch.Tensor) -> torch.Tensor:
    return t.contiguous().view(torch.int32)


def first_diff(a: torch.Tensor, b: torch.Tensor):
    """first differing (layout, token) of two [B][S(, ...)] tensors, compared bit for bit; None if equal"""
    if a.is_floating_point():
        a, b = bits(a), bits(b)
    d = a != b
    if d.dim() > 2:
        d = d.flatten(2).any(-1)
    idx = d.nonzero()
    return None if len(idx) == 0 else tuple(idx[0].tolist())


@dataclass
class Serial:
    """the serialized step path: ids after every step (CPU, int16), token logits and pad-row logits of the kept steps"""
    ids: List[torch.Tensor] = field(default_factory=list)
    logits: Dict[int, torch.Tensor] = field(default_factory=dict)
    pad: Dict[int, torch.Tensor] = field(default_factory=dict)


def serialized(monkeypatch, wl: Workload, dtype: str, seed: int, b_global0: int, cond, ids_init, keep=(), plan=None, B=None,
               want_logprob: bool = False) -> Serial:
    """want_logprob: every step also fills the log-prob tap, so its draw runs in the all-classes kernel"""
    plan = wl.plan if plan is None else plan
    B = wl.B if B is None else B
    v = wl.vocab
    out = Serial()
    with handle(monkeypatch, wl, dtype, SERIAL) as eng:
        if ids_init is not None:
            x = ids_init
        elif cond is not None:
            x = cond["seq"]
        else:
            x = torch.full((B, v.S), v.mask_id, dtype=torch.int64, device="cuda")
        for i, (tm, tp) in enumerate(plan):
            x, lg, _ = eng.step(x, tm, tp, wl.sampling, cond, seed=seed, step_ctr=i, b_global0=b_global0, want_logits=i in keep,
                                want_logprob=want_logprob)
            out.ids.append(x.to(torch.int16).cpu())
            if i in keep:
                out.logits[i] = lg.cpu()
                out.pad[i] = G.debug_read(eng, "logits", B, raw=True)[:, v.S:].clone()
    return out


def fuses(dtype: str, env: Dict[str, str]) -> bool:
    """the handle writes the next step's embedding rows from the draw (the split mode never does)"""
    return dtype != "bf16x3" and env.get("LDM_FUSE_EMBED", "1") != "0"


def expected_launches(k: int, wl: Workload, fused: bool) -> int:
    fill = 1 if wl.cond_type is None else 0            # the all-MASK start state
    return fill + k * LAUNCHES_PER_STEP - ((k - 1) if fused else 0)


def compare_prefixes(monkeypatch, wl: Workload, dtype: str, settings, ks: List[int], ref: Serial, cond, ids_init) -> List[str]:
    """run every setting's loop on plan[:k] for each k, compare with the serialized path and print one table row per setting;
    returns the failures"""
    v, plan, S, C = wl.vocab, wl.plan, wl.vocab.S, wl.vocab.C
    failures = []
    print(f"\n{wl.name} | {dtype} | B={wl.B} | {len(plan)} steps | prefixes k={ks} | seed {wl.seed}, b_global0 {wl.b_global0}")
    print(f"  {'setting':18s} {'launches':9s} {'ids':5s} {'token logits':13s} pad rows differing (of {wl.B * (128 - S)}) per prefix")
    for label, env in settings:
        fused = fuses(dtype, env)
        row_ids = row_lg = row_launch = "ok"
        pads = []
        with handle(monkeypatch, wl, dtype, env) as eng:
            for k in ks:
                step = k - 1
                l0 = eng.launch_count
                ids = eng.sample_loop(wl.B, plan[:k], wl.sampling, cond=cond, seed=wl.seed, b_global0=wl.b_global0, ids_init=ids_init)
                torch.cuda.synchronize()
                n_launch = eng.launch_count - l0
                if n_launch != expected_launches(k, wl, fused):
                    row_launch = "FAIL"
                    failures.append(f"{label} k={k}: {n_launch} launches, expected {expected_launches(k, wl, fused)} (fused embedding: {fused})")
                ids = ids.cpu()
                assert int(ids.min()) >= 0 and int(ids.max()) < C
                d = first_diff(ids.to(torch.int16), ref.ids[step])
                if d is not None:
                    row_ids = "FAIL"
                    failures.append(f"{label} k={k}: ids differ, first at (layout, token) {d}, step {step}, "
                                    f"{int((ids.to(torch.int16) != ref.ids[step]).sum())} tokens")
                lg = G.debug_read(eng, "logits", wl.B, raw=True)
                d = first_diff(lg[:, :S, :C], ref.logits[step])
                if d is not None:
                    row_lg = "FAIL"
                    failures.append(f"{label} k={k}: token-row logits differ, first at (layout, token) {d}, step {step}")
                pad = lg[:, S:]
                if not torch.isfinite(pad).all():
                    row_lg = "FAIL"
                    failures.append(f"{label} k={k}: non-finite pad-row logits")
                n_pad = int((bits(pad) != bits(ref.pad[step])).any(-1).sum())
                pads.append(f"k={k}: {n_pad}")
                # before the first fused row (k = 1) and without the fused embedding, the pad rows are the embedding's zeros too
                if n_pad and (k == 1 or not fused):
                    row_lg = "FAIL"
                    failures.append(f"{label} k={k}: {n_pad} pad rows differ although no fused embedding row was written")
                del lg, pad
        print(f"  {label:18s} {row_launch:9s} {row_ids:5s} {row_lg:13s} {', '.join(pads)}")
    return failures


WORKLOADS = {"config1": CONFIG1, "config2": CONFIG2, "config0": CONFIG0, "tail301": TAIL301, "tail1": TAIL1}


@pytest.mark.parametrize("name,dtype", [("config1", "fp16"), ("config1", "bf16"), ("config1", "bf16x3"), ("config2", "fp16"),
                                        ("config0", "fp16"), ("tail301", "fp16"), ("tail1", "fp16")])
def test_loop_equals_serialized_steps_under_every_switch(monkeypatch, name, dtype):
    """the switch matrix: default, each of PDL / graph / fused embedding / sweep off alone, all four off, 7 persistent CTAs"""
    wl = WORKLOADS[name]
    cond, ids_init = inputs(wl)
    ks = prefixes(len(wl.plan))
    ref = serialized(monkeypatch, wl, dtype, wl.seed, wl.b_global0, cond, ids_init, keep=[k - 1 for k in ks])
    failures = compare_prefixes(monkeypatch, wl, dtype, MATRIX, ks, ref, cond, ids_init)
    # the serialized steps with the log-prob tap (the all-classes draw kernel, which the oracle tests read log-probs from)
    tap = serialized(monkeypatch, wl, dtype, wl.seed, wl.b_global0, cond, ids_init, keep=[k - 1 for k in ks], want_logprob=True)
    for step, (a, b) in enumerate(zip(tap.ids, ref.ids)):
        d = first_diff(a, b)
        if d is not None:
            failures.append(f"serialized steps with the log-prob tap: ids differ at step {step}, first at (layout, token) {d}, "
                            f"{int((a != b).sum())} tokens")
            break
    for step in ref.logits:
        if first_diff(tap.logits[step], ref.logits[step]) is not None:
            failures.append(f"serialized steps with the log-prob tap: logits differ at step {step}")
    print(f"  {'log-prob tap':18s} {'-':9s} {'ok' if not any('log-prob tap' in f for f in failures) else 'FAIL':5s}")
    assert not failures, "\n".join(failures)


def test_loop_equals_serialized_steps_config3_B4096(monkeypatch):
    """config 3 at its own shape (T = 200, 4096 layouts, refinement): the default schedule, full plan and k = 2"""
    wl = CONFIG3
    cond, ids_init = inputs(wl)
    ks = [2, len(wl.plan)]
    ref = serialized(monkeypatch, wl, "fp16", wl.seed, wl.b_global0, cond, ids_init, keep=[k - 1 for k in ks])
    failures = compare_prefixes(monkeypatch, wl, "fp16", MATRIX[:1], ks, ref, cond, ids_init)
    assert not failures, "\n".join(failures)


# ---- replay semantics: what changes from call to call reaches the captured graph ----

def final_ids(monkeypatch, wl, seed, b_global0, cond=None, ids_init=None, B=None):
    """a fresh default handle's first (captured) run, and the serialized step path's final ids"""
    B = wl.B if B is None else B
    with handle(monkeypatch, wl, "fp16", {}) as eng:
        first = eng.sample_loop(B, wl.plan, wl.sampling, cond=cond, seed=seed, b_global0=b_global0, ids_init=ids_init).cpu()
    serial = serialized(monkeypatch, wl, "fp16", seed, b_global0, cond, ids_init, B=B).ids[-1]
    return first, serial


def check_replays(monkeypatch, wl, calls, got, title):
    """calls: (label, seed, b_global0, cond, ids_init); got: the ids the shared handle returned for each"""
    failures = []
    print(f"\n{title}")
    print(f"  {'call':34s} {'= fresh capture':16s} = serialized steps")
    for (label, seed, b0, cond, ids_init), ids in zip(calls, got):
        first, serial = final_ids(monkeypatch, wl, seed, b0, cond, ids_init, B=ids.shape[0])
        d_first, d_serial = first_diff(ids, first), first_diff(ids.to(torch.int16), serial)
        print(f"  {label:34s} {'ok' if d_first is None else 'FAIL':16s} {'ok' if d_serial is None else 'FAIL'}")
        if d_first is not None:
            failures.append(f"{label}: differs from a fresh handle's captured run, first at (layout, token) {d_first}")
        if d_serial is not None:
            failures.append(f"{label}: differs from the serialized steps, first at (layout, token) {d_serial}, step {len(wl.plan) - 1}")
    return failures


def test_replay_bench_call_sequence(monkeypatch):
    """bench.py's calls on one handle (warm-up seeds 100..102, timed seeds 1000 + k, b_global0 = rank * B for rank 1), then
    a change of b_global0 alone: every replay equals a fresh capture and the serialized steps with its own key"""
    wl, B = CONFIG1, CONFIG1.B
    calls = [(f"seed {s}, b_global0 {b0}", s, b0, None, None) for s, b0 in ((100, B), (101, B), (102, B), (1000, B), (1001, B), (1001, 0))]
    with handle(monkeypatch, wl, "fp16", {}) as eng:
        got = [eng.sample_loop(B, wl.plan, wl.sampling, seed=s, b_global0=b0).cpu() for _, s, b0, _, _ in calls]
    failures = check_replays(monkeypatch, wl, calls, got, f"replay: {wl.name}, B={B}, fp16, bench.py's call sequence")
    if torch.equal(got[-1], got[-2]):
        failures.append("a new b_global0 alone left the ids unchanged")
    assert not failures, "\n".join(failures)


def other_start(cond, vocab, seed):
    """a start state with the same fixed tokens and some MASK positions already drawn inside their attribute's vocabulary"""
    g = torch.Generator().manual_seed(seed)
    seq = cond["seq"].cpu()
    s = torch.arange(vocab.S).expand_as(seq)
    attr = s % vocab.n_attr
    lo = torch.where(attr == 0, torch.zeros_like(attr), vocab.n_cat + (attr - 1) * vocab.n_bins)
    n = torch.where(attr == 0, torch.full_like(attr, vocab.n_cat), torch.full_like(attr, vocab.n_bins))
    drawn = lo + (torch.rand(seq.shape, generator=g) * n).long()
    pick = (seq == vocab.mask_id) & (torch.rand(seq.shape, generator=g) < 0.5)
    return torch.where(pick, drawn, seq).cuda()


def test_replay_new_cond_and_ids_init(monkeypatch):
    """config 2: a second condition with the same flags and other contents, then another start state, replayed on the handle
    that captured the first; each equals a fresh capture and the serialized steps"""
    wl = CONFIG2
    cond0, init0 = inputs(wl, cond_seed=0)
    cond1, init1 = inputs(wl, cond_seed=1)
    init2 = other_start(cond1, wl.vocab, seed=2)
    assert not torch.equal(init2, init1)
    calls = [("cond seed 0", 5, 0, cond0, init0), ("cond seed 1 (same flags)", 5, 0, cond1, init1),
             ("cond seed 1, another ids_init", 5, 0, cond1, init2), ("cond seed 0 again, seed 6", 6, 0, cond0, init0)]
    with handle(monkeypatch, wl, "fp16", {}) as eng:
        got = [eng.sample_loop(wl.B, wl.plan, wl.sampling, cond=c, seed=s, b_global0=b0, ids_init=i).cpu() for _, s, b0, c, i in calls]
    failures = check_replays(monkeypatch, wl, calls, got, f"replay: {wl.name}, B={wl.B}, fp16, new cond / ids_init contents")
    for (label, _, _, c, _), ids in zip(calls, got):
        m = c["mask"].cpu()
        if not torch.equal(ids[m], c["seq"].cpu()[m]):
            failures.append(f"{label}: fixed tokens not kept")
    assert not failures, "\n".join(failures)


def test_replay_after_workspace_shrink(monkeypatch):
    """config 1 at B = 4096, then at B = 1024 on the same handle: the workspace stays at 4096 layouts and the graph is captured
    again; the B = 1024 result equals a fresh B = 1024 handle and the serialized steps"""
    wl = CONFIG1
    with handle(monkeypatch, wl, "fp16", {}) as eng:
        big = eng.sample_loop(4096, wl.plan, wl.sampling, seed=7).cpu()
        small = eng.sample_loop(1024, wl.plan, wl.sampling, seed=7).cpu()
    failures = check_replays(monkeypatch, wl, [("B=1024 after B=4096", 7, 0, None, None)], [small],
                             f"replay: {wl.name}, fp16, workspace grown to 4096 layouts")
    d = first_diff(big[:1024], small)
    if d is not None:      # the noise is keyed by the global layout index, not by the batch size
        failures.append(f"the first 1024 layouts of the B=4096 run differ from the B=1024 run, first at (layout, token) {d}")
    assert not failures, "\n".join(failures)


def test_loop_on_side_stream(monkeypatch):
    """the loop called under torch.cuda.stream(side), inputs made ready on that stream first: a replay of the graph captured
    on the default stream and a capture of a new plan both give the default stream's ids"""
    wl = CONFIG2
    cond, init = inputs(wl)
    short = wl.plan[:10]
    side = torch.cuda.Stream()
    with handle(monkeypatch, wl, "fp16", {}) as eng:
        want_full = eng.sample_loop(wl.B, wl.plan, wl.sampling, cond=cond, seed=3, ids_init=init).cpu()
        want_short = eng.sample_loop(wl.B, short, wl.sampling, cond=cond, seed=4, ids_init=init).cpu()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            got_full = eng.sample_loop(wl.B, wl.plan, wl.sampling, cond=cond, seed=3, ids_init=init)     # captured on the default stream
            got_short = eng.sample_loop(wl.B, short, wl.sampling, cond=cond, seed=4, ids_init=init)    # captured again, on the side stream
        torch.cuda.current_stream().wait_stream(side)
        got_full, got_short = got_full.cpu(), got_short.cpu()
    print(f"\nside stream: {wl.name}, B={wl.B}: full plan {'ok' if torch.equal(got_full, want_full) else 'FAIL'}, "
          f"10-step plan {'ok' if torch.equal(got_short, want_short) else 'FAIL'}")
    assert first_diff(got_full, want_full) is None, f"full plan differs at {first_diff(got_full, want_full)}"
    assert first_diff(got_short, want_short) is None, f"10-step plan differs at {first_diff(got_short, want_short)}"


# ---- anchor: one state of the loop at the benchmark shape against float64 ----

def anchor_layouts(B: int, n_sms: int, n: int = 48, seed: int = 0) -> List[int]:
    """the first and last row tiles, the layouts at the wave boundaries of the 128-row GEMM tiles and of the 64-row LN GEMM
    tiles (from the start and, for the reversed sweeps, from the end), then random layouts up to n"""
    pick = [0, 1, B - 2, B - 1]
    for m in range(1, B // n_sms + 1):
        pick += [m * n_sms - 1, m * n_sms, B - m * n_sms]          # 128-row tiles
    for m in range(1, 2 * B // n_sms + 1, 2):
        pick += [m * n_sms // 2]                                    # 64-row tiles
    out = []
    for b in pick:
        if 0 <= b < B and b not in out:
            out.append(b)
    out = out[:n]
    g = torch.Generator().manual_seed(seed)
    for b in torch.randperm(B, generator=g).tolist():
        if len(out) == n:
            break
        if b not in out:
            out.append(b)
    return sorted(out)


def test_loop_logits_vs_float64_at_benchmark_shape(monkeypatch):
    """config 1, B = 1024, prefix k = 2 (the first step whose embedding rows the draw wrote): the loop's logits of 48 layouts
    against a float64 forward of the same x_t, within test_gpu_parity.py's 1e-3 gate"""
    wl = CONFIG1
    v, spec, plan = O.RICO25, O.ModelSpec(T=wl.T), wl.plan
    with handle(monkeypatch, wl, "fp16", {}) as eng:
        x_t = eng.sample_loop(wl.B, plan[:1], wl.sampling, seed=wl.seed).cpu()
        eng.sample_loop(wl.B, plan[:2], wl.sampling, seed=wl.seed)
        torch.cuda.synchronize()
        lg = G.debug_read(eng, "logits", wl.B, raw=True)[:, : v.S, : v.C]
    picks = anchor_layouts(wl.B, torch.cuda.get_device_properties(0).multi_processor_count)
    sd64 = {k: t.double() for k, t in state_dict(wl.dataset, wl.T).items()}
    t = plan[1][0]
    err = torch.empty(len(picks), dtype=torch.float64)
    scale = 0.0
    with torch.no_grad():
        for i in range(0, len(picks), 16):
            idx = picks[i:i + 16]
            ref = O.denoiser_forward(sd64, x_t[idx], t, v, spec)
            err[i:i + len(idx)] = (lg[idx].double() - ref).abs().amax(dim=(1, 2))
            scale = max(scale, ref.abs().max().item())
    worst = int(err.argmax())
    print(f"\nanchor: {wl.name}, B={wl.B}, k=2 (t={t}), {len(picks)} layouts vs float64: max|logit| {scale:.3f}, max-abs error "
          f"{err.max():.2e} (layout {picks[worst]}), gate {LOGIT_TOL:.0e}, headroom {LOGIT_TOL / max(err.max().item(), 1e-30):.1f}x")
    assert torch.isfinite(err).all() and err.max() < LOGIT_TOL, \
        f"layouts over the gate: {[(picks[i], f'{e:.2e}') for i, e in enumerate(err.tolist()) if e >= LOGIT_TOL]}"
