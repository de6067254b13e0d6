"""Host mirror of the reference's diffusion-core class API, running on the sm_90a library.

  FusedMaskAndReplaceDiffusion   <->  BaseMaskAndReplaceDiffusion (+ Constrained / Vanilla subclasses)
                                      models/categorical_diffusion/base.py:29-371, constrained.py, vanilla.py
  LayoutDMB200                   <->  LayoutDM   models/layoutdm.py:26-97
  patch_reference_model(model)   drop-in: re-routes `model.model.sample` / `_sample_single_step` of a live reference
                                 LayoutDM instance (so src/trainer's test.py / main.py / demo notebook run unchanged).

Same signatures, argument meaning and exception types as the reference; ids are int64, results come back on the CPU
exactly where the reference returns CPU tensors.
"""
from __future__ import annotations

import copy
import weakref
from typing import Any, Dict, List, Optional, Union

import torch
import torch.nn.functional as F
from torch.optim.optimizer import register_optimizer_step_post_hook

from . import _lib
from .engine import Engine, sampling_struct
from .vocab import Vocab, decode_ids, group_full_ids, linear_centers, refinement_table, relation_edge_table, timestep_plan


def _cfg_get(cfg, key, default=None):
    if cfg is None:
        return default
    if hasattr(cfg, "get"):
        v = cfg.get(key, default)
    else:
        v = getattr(cfg, key, default)
    return default if v is None else v


def index_to_log_onehot(x: torch.Tensor, num_classes: int) -> torch.Tensor:
    """util.py:34-40 : (B, S) -> (B, C, S)"""
    assert x.max().item() < num_classes, f"Error: {x.max().item()} >= {num_classes}"
    return torch.log(F.one_hot(x, num_classes).permute(0, 2, 1).float().clamp(min=1e-30))


def duplicate_cond(cond: Dict, batch_size: int) -> Dict:
    """helpers/task.py:235-248: one condition, many outputs.  Per-layout tensors are repeated along dim 0; the (C, C)
    refinement band table is shared by all layouts and stays as it is."""
    if cond["seq"].size(0) == 1 and batch_size > 1:
        for k in cond:
            if isinstance(cond[k], torch.Tensor) and k not in ("refine_table", "rel_centers"):
                cond[k] = cond[k].repeat([batch_size] + [1] * (cond[k].dim() - 1))
    return cond


_FOLLOWERS: "weakref.WeakSet[WeightFollower]" = weakref.WeakSet()
_STEP_HOOK = None


def _optimizer_stepped(optimizer, args, kwargs):
    """optimizer step post-hook: marks the followers of the parameters it stepped dirty.  A fused AdamW step writes the
    parameters without bumping their version counters, so the fingerprint alone would miss it."""
    stepped = None
    for f in list(_FOLLOWERS):
        if stepped is None:
            stepped = {id(p) for g in optimizer.param_groups for p in g["params"]}
        if not stepped.isdisjoint(f.param_ids):
            f.dirty = True


class WeightFollower:
    """Keeps a target's packed weights equal to a live module's parameters.  target: anything with `load_weights(dict)` (the
    `Engine.pack_state_dict` dict), `vocab` and `device`, i.e. an Engine.

    `check()` reloads when the parameters may have changed since the last load: a parameter's storage (`data_ptr`: a
    parameter replaced, `model.cpu()` / `.cuda()`) or version counter (in-place writes such as `load_state_dict` or a foreach
    optimizer step) differs, or an optimizer stepped one of them (the dirty flag, set by a step post-hook).  Writes through
    `.data` bypass all of these; call `reload()` after them.  An unchanged module costs the fingerprint only."""

    def __init__(self, module: torch.nn.Module, target):
        global _STEP_HOOK
        self.module, self.target = module, target
        self.reloads = 0
        self.dirty = False
        self._fp = self._fingerprint()
        _FOLLOWERS.add(self)
        if _STEP_HOOK is None:        # one hook for every follower; it holds them only through the weak set
            _STEP_HOOK = register_optimizer_step_post_hook(_optimizer_stepped)

    def _fingerprint(self):
        params = list(self.module.parameters())
        self.param_ids = frozenset(id(p) for p in params)
        return tuple((p.data_ptr(), p._version) for p in params)

    def check(self) -> bool:
        """reload if the module may have changed; True if it did"""
        fp = self._fingerprint()
        if self.dirty or fp != self._fp:
            self.reload(fp)
            return True
        return False

    def reload(self, fp=None):
        """repack the module's current parameters into the target unconditionally"""
        sd = self.module.state_dict()
        self.target.load_weights(Engine.pack_state_dict(sd, self.target.vocab, device=self.target.device))
        self._fp = self._fingerprint() if fp is None else fp
        self.dirty = False
        self.reloads += 1


class FusedMaskAndReplaceDiffusion:
    """noise="contract": the draws use the project's Philox contract keyed by a seed (drawn from torch's generator unless
    given).  noise="torch": they are the numbers torch's CUDA generator gives the reference's `sample` on the same GPU, and
    every call advances that generator as the reference's would, so a seeded run reproduces the reference's samples."""

    def __init__(self, engine: Engine, tokenizer=None, bbox_centers=None, noise: str = "contract"):
        if noise not in _lib.NOISE_KINDS:
            raise ValueError(f"noise must be one of {', '.join(_lib.NOISE_KINDS)}, got {noise!r}")
        self.noise = noise
        self.engine = engine
        self.vocab: Vocab = engine.vocab
        self.num_classes = self.vocab.C
        self.max_token_length = self.vocab.S
        self.num_timesteps = engine.T
        self.tokenizer = tokenizer
        # cluster centres used by the refinement prior (task.py:183-189); linear quantisation by default
        if bbox_centers is None and tokenizer is not None:
            bt = tokenizer.bbox_tokenizer
            bbox_centers = [bt.clustering_models[f"{k}-{self.vocab.n_bins}"].cluster_centers_.reshape(-1) for k in ("x", "y", "w", "h")]
        self.bbox_centers = bbox_centers if bbox_centers is not None else linear_centers(self.vocab.n_bins)
        self._step_ctr = 0
        self._seed: Optional[int] = None     # noise key of `_sample_single_step` trajectories (None: drawn from torch's generator)
        self._last_t: Optional[int] = None
        self.relation_on_device = True   # cond=relation, relation_mode "average": hand-derived update kernel; False: logit_adjust_fn hook
        self.logit_adjust_fn = None      # optional hook f(t: int, cond, model_log_prob (B,C,S), sampling_cfg) for cond=relation
        self._weights: Optional[WeightFollower] = None   # the live module whose parameters the engine follows (follow())

    @property
    def device(self) -> torch.device:
        return self.engine.device

    # ---- weights -------------------------------------------------------------------------------------
    def follow(self, module: torch.nn.Module):
        """take the denoiser's weights from `module` (the reference's CategoricalTransformer, whose state_dict the engine was
        built from): every call that runs the denoiser first reloads them if they may have changed (WeightFollower)"""
        self._weights = WeightFollower(module, self.engine)

    def reload_weights(self):
        """repack the followed module's parameters now: needed after writes through `.data`, which nothing detects"""
        if self._weights is None:
            raise ValueError("no weight source: follow(module) first (patch_reference_model does)")
        self._weights.reload()

    @property
    def weight_reloads(self) -> int:
        """how many times the followed module's weights have been repacked"""
        return 0 if self._weights is None else self._weights.reloads

    def _follow_weights(self):
        if self._weights is not None:
            self._weights.check()

    # ---- helpers -------------------------------------------------------------------------------------
    def _prepare_cond(self, cond: Optional[Dict], batch_size: int, sampling_cfg) -> Optional[Dict]:
        if not cond:
            return None
        cond = dict(cond)
        if cond.get("type") == "refinement" and "refine_table" not in cond:
            # set_additional_conditions_for_refinement (task.py:204-224) without materialising (B,C,S) weak_logits
            cond["refine_table"] = refinement_table(self.vocab, self.bbox_centers, _cfg_get(sampling_cfg, "refine_mode", "uniform"),
                                                    _cfg_get(sampling_cfg, "refine_offset_ratio", 0.1),
                                                    _cfg_get(sampling_cfg, "refine_lambda", 3.0))
        if self.relation_on_device and cond.get("type") == "relation" and "batch_w_canvas" in cond and "rel_adj" not in cond \
                and _cfg_get(sampling_cfg, "relation_mode", "average") == "average" and float(_cfg_get(sampling_cfg, "relation_lambda", 0.0)) > 0.0:
            # logit_adjustment.update (:88-126) on the device: dense edge table + bin centres + SGD hyper-parameters.
            # relation_mode "gumbel" draws torch noise inside the update and stays on the reference's autograd path (logit_adjust_fn).
            cond["rel_adj"] = relation_edge_table(cond["batch_w_canvas"], cond["seq"].size(0), self.vocab.n_elem + 1)
            cond["rel_centers"] = torch.stack([torch.as_tensor(c, dtype=torch.float32).view(-1) for c in self.bbox_centers])
            cond["rel_lambda"] = float(_cfg_get(sampling_cfg, "relation_lambda", 3e6))
            cond["rel_num_update"] = int(_cfg_get(sampling_cfg, "relation_num_update", 3))
            cond.setdefault("rel_batch_total", batch_size)
        cond = duplicate_cond(cond, batch_size)
        for k in list(cond):
            if isinstance(cond[k], torch.Tensor):
                cond[k] = cond[k].to(self.device)                              # base.py:328-330
        return cond

    def _with_torch_noise(self, total_layouts: int, sampling_cfg, n_steps: int, seed: Optional[int], call):
        """call(noise) with the noise of n_steps steps from torch's CUDA generator of this device (its seed and current offset);
        once the call has succeeded the generator is advanced past its draws, where the reference would leave it"""
        if seed is not None:
            raise ValueError("seed= selects the Philox contract; with noise='torch' the draws come from torch's CUDA generator")
        if torch.cuda.is_current_stream_capturing():
            raise ValueError("noise='torch' reads and advances torch's CUDA generator, which cannot be done during a CUDA graph capture")
        gen = torch.cuda.default_generators[self.device.index]
        offset = gen.get_offset()
        advance = self.engine.noise_advance(total_layouts, sampling_cfg, n_steps)
        out = call(_lib.LdmNoise(_lib.NOISE_KINDS["torch"], gen.initial_seed(), offset, total_layouts))
        gen.set_offset(offset + advance)
        return out

    @staticmethod
    def _new_seed() -> int:
        # the reference draws from torch's global generator, so `set_seed` / torch.manual_seed keeps controlling
        # reproducibility: derive the Philox key from it
        return int(torch.randint(0, 2 ** 62, (1,)).item())

    # ---- reference API -------------------------------------------------------------------------------
    def sample(self, batch_size: Optional[int] = 1, cond: Optional[Dict] = None, sampling_cfg=None,
               get_intermediate_results: bool = False, seed: Optional[int] = None, b_global0: int = 0,
               total_layouts: Optional[int] = None, **kwargs) -> Union[torch.LongTensor, List[torch.LongTensor]]:
        """base.py:293-371.  total_layouts: the whole batch when this call samples layouts [b_global0, b_global0 + batch_size)
        of it (noise="torch": the draws are that slice of the whole batch's, and the generator advances as for the whole batch)"""
        self._follow_weights()
        total = b_global0 + batch_size if total_layouts is None else int(total_layouts)
        T_eval = _cfg_get(sampling_cfg, "num_timesteps", self.num_timesteps)
        plan = timestep_plan(self.num_timesteps, T_eval, float(_cfg_get(sampling_cfg, "time_difference", 0.0)))
        cond_d = self._prepare_cond(cond, batch_size, sampling_cfg)
        if cond_d is not None:
            assert cond_d["seq"].shape[0] == batch_size
            assert cond_d["seq"].max().item() < self.num_classes
        if self.noise == "torch" and seed is not None:
            raise ValueError("seed= selects the Philox contract; with noise='torch' the draws come from torch's CUDA generator")
        seed = self._new_seed() if seed is None and self.noise == "contract" else seed
        if cond_d is not None and cond_d.get("type") == "relation" and "rel_adj" not in cond_d and self.logit_adjust_fn is not None:
            # an external (Python) logit adjustment between posterior and draw: per-step host loop through the log-prob taps
            return self._sample_stepwise(batch_size, plan, cond_d, sampling_cfg, seed, b_global0, get_intermediate_results, total)
        loop = lambda noise: self.engine.sample_loop(batch_size, plan, sampling_cfg, cond_d, seed=seed or 0, b_global0=b_global0,
                                                     trace=get_intermediate_results, noise=noise)
        res = self._with_torch_noise(total, sampling_cfg, len(plan), None, loop) if self.noise == "torch" else loop(None)
        if get_intermediate_results:
            return [r for r in res[1].cpu()]
        return res.cpu()

    def _sample_stepwise(self, B, plan, cond, sampling_cfg, seed, b_global0, trace, total=None):
        """per-step host loop: needed when a Python hook edits the log-probs between posterior and draw (cond=relation)"""
        ids = cond["seq"].clone() if cond else torch.full((B, self.max_token_length), self.vocab.mask_id, device=self.device)
        results = []
        for i, (t_model, t_post) in enumerate(plan):
            ids = self._step_ids(ids, t_model, t_post, sampling_cfg, cond, seed, i, b_global0, total)
            if trace:
                results.append(ids.cpu())
        return results if trace else ids.cpu()

    def _step_ids(self, ids, t_model, t_post, sampling_cfg, cond, seed, step_ctr, b_global0=0, total=None):
        # noise="torch": the generator is read right before the step's draw (after the hook, which may draw from it as well)
        def draw(**kw):
            step = lambda noise: self.engine.step(ids, t_model, t_post, sampling_cfg, cond, seed, step_ctr, b_global0, noise=noise, **kw)[0]
            if self.noise != "torch":
                return step(None)
            return self._with_torch_noise(b_global0 + ids.shape[0] if total is None else total, sampling_cfg, 1, None, step)
        seed = seed or 0
        if cond is not None and cond.get("type") == "relation" and "rel_adj" not in cond and self.logit_adjust_fn is not None:
            # base.py:243-284 order: strong mask -> update() -> PAD-disable -> draw.  The first call returns the log-probs with the
            # strong mask only (PAD-disable off: `update` must see what the reference's sees), the hook edits them, PAD-disable
            # is applied here, the second call draws from the result.  `t` is an int like in the reference (base.py:262).  The first
            # call's draw is discarded: it takes the contract's noise and leaves torch's generator alone.
            pre = dict(cond); pre["_pad_disable"] = False
            _, _, lp = self.engine.step(ids, t_model, t_post, sampling_cfg, pre, seed, step_ctr, b_global0, want_logprob=True)
            lp = self.logit_adjust_fn(int(t_model), cond, lp.permute(0, 2, 1).contiguous(), sampling_cfg)      # (B,C,S) like the reference
            lp = lp.permute(0, 2, 1).contiguous()
            S = ids.shape[1]
            pad_mask = (torch.arange(S, device=ids.device)[None] % self.vocab.n_attr != 0) & (cond["seq"] != self.vocab.pad_id)
            lp[..., self.vocab.pad_id] = torch.where(pad_mask, torch.full_like(lp[..., 0], -69.07755278982137), lp[..., self.vocab.pad_id])
            return draw(logprob_in=lp)
        return draw()

    def _sample_single_step(self, log_z: torch.Tensor, model_t: torch.Tensor, skip_step: int, sampling_cfg=None,
                            cond: Optional[Dict] = None) -> torch.Tensor:
        """base.py:205-291 ; log_z (B,C,S) -> log_z (B,C,S).  Kept for API compatibility (the notebook and subclasses call it);
        `sample()` itself never materialises (B,C,S) tensors."""
        self._follow_weights()
        ids = log_z.argmax(1).to(self.device)
        t_model = int(model_t[0].item())
        assert bool((model_t == t_model).all())
        td = float(_cfg_get(sampling_cfg, "time_difference", 0.0))
        T = self.num_timesteps
        noise_t = min(max(t_model - int(T * td), 0), T - 1) if td > 0.0 else t_model            # :218-225
        t_post = noise_t - skip_step if (skip_step > 0 and noise_t > skip_step) else noise_t   # :227-240
        cond_d = None
        if cond:
            cond_d = {k: (v.to(self.device) if isinstance(v, torch.Tensor) else v) for k, v in cond.items()}
            if cond_d.get("type") == "refinement" and "refine_table" not in cond_d:
                cond_d = self._prepare_cond(cond_d, ids.shape[0], sampling_cfg)
        if self.noise == "torch":      # one step's draws from torch's CUDA generator
            out = self._step_ids(ids, t_model, t_post, sampling_cfg, cond_d, None, 0)
            return index_to_log_onehot(out, self.num_classes)
        # noise key: like the reference, the draws come from torch's global generator -- a new key is derived from it at the start
        # of every trajectory (timesteps strictly decrease inside one), unless reset_noise(seed) pinned one
        if self._seed is None or (self._last_t is not None and t_model >= self._last_t and not self._pinned):
            self._seed, self._step_ctr = self._new_seed(), 0
        self._last_t = t_model
        out = self._step_ids(ids, t_model, t_post, sampling_cfg, cond_d, self._seed, self._step_ctr)
        self._step_ctr += 1
        return index_to_log_onehot(out, self.num_classes)

    # ---- training-side API (SURVEY 8b: "signatures that must keep working"; forward only, no autograd) -----------------
    VAR_NAMES = ("c", "x", "y", "w", "h")

    def _key_index(self, key: str) -> int:
        return self.VAR_NAMES.index(key) if self.engine.q_type == "constrained" else 0

    def predict_start(self, log_x_t: torch.Tensor, t: torch.Tensor) -> torch.Tensor:
        """base.py:127-146: log_x_t (B,C,S) log one-hot, t (B,) -> log p(x0|xt) (B,C,S)"""
        self._follow_weights()
        return self.engine.predict_start(log_x_t.argmax(1), t).permute(0, 2, 1).contiguous()

    def q_posterior(self, log_x_start: torch.Tensor, log_x_t: torch.Tensor, t: torch.Tensor) -> torch.Tensor:
        """constrained.py:135-206 / vanilla.py:112-151: (B,C,S) log p(x0), (B,C,S) log one-hot x_t, t (B,) -> (B,C,S)"""
        assert t.min().item() >= 0 and t.max().item() < self.num_timesteps
        out = self.engine.q_posterior(log_x_start.permute(0, 2, 1), log_x_t.argmax(1), t)
        return out.permute(0, 2, 1).contiguous()

    def q_pred(self, log_x_start: torch.Tensor, t: torch.Tensor, key: Optional[str] = None) -> torch.Tensor:
        """constrained.py:112-133: log q(x_t|x_0) on attribute `key`'s PARTIAL vocabulary, log_x_start (B, K_key, S/5) -> same shape;
        vanilla (key=None): (B,C,S) -> (B,C,S)  (vanilla.py:90-110)"""
        v = self.vocab
        if self.engine.q_type != "constrained" or key is None:
            return self.engine.q_pred(log_x_start.permute(0, 2, 1), t).permute(0, 2, 1).contiguous()
        g = self._key_index(key)
        ids = torch.tensor(group_full_ids(v, g), device=self.device)
        B, K, Sg = log_x_start.shape
        assert K == ids.numel() and Sg == v.n_elem
        full = torch.full((B, v.S, v.C), -69.07755278982137, device=self.device)
        full[:, g::v.n_attr, ids] = log_x_start.to(self.device).permute(0, 2, 1)
        out = self.engine.q_pred(full, t)
        return out[:, g::v.n_attr][..., ids].permute(0, 2, 1).contiguous()

    def _partial_to_full(self, x: torch.Tensor, key: Optional[str], fill: float):
        """(B, K_key, S/5) tensor on attribute `key`'s partial vocabulary -> ((B, S, C) full tensor with `fill` elsewhere, group index, ids)"""
        v = self.vocab
        g = self._key_index(key)
        ids = torch.tensor(group_full_ids(v, g), device=self.device)
        B, K, Sg = x.shape
        assert K == ids.numel() and Sg == v.n_elem
        full = torch.full((B, v.S, v.C), fill, device=self.device)
        full[:, g::v.n_attr, ids] = x.to(self.device).permute(0, 2, 1)
        return full, g, ids

    def q_pred_one_timestep(self, log_x_t: torch.Tensor, t: torch.Tensor, key: Optional[str] = None) -> torch.Tensor:
        """constrained.py:92-110 / vanilla.py:74-88: log q(x_t|x_{t-1}); partial vocabulary (B, K_key, S/5) with `key`, else (B,C,S)"""
        if self.engine.q_type != "constrained" or key is None:
            return self.engine.q_pred_one_timestep(log_x_t.permute(0, 2, 1), t).permute(0, 2, 1).contiguous()
        full, g, ids = self._partial_to_full(log_x_t, key, -69.07755278982137)
        out = self.engine.q_pred_one_timestep(full, t)
        return out[:, g::self.vocab.n_attr][..., ids].permute(0, 2, 1).contiguous()

    def log_sample_categorical(self, logits: torch.Tensor, key: Optional[str] = None, seed: Optional[int] = None) -> torch.Tensor:
        """constrained.py:208-221 (train_sampling "gumbel"): log one-hot of argmax(logits + Gumbel noise) along the class dim"""
        seed = self._new_seed() if seed is None else seed
        v = self.vocab
        if self.engine.q_type != "constrained" or key is None:
            return index_to_log_onehot(self.engine.gumbel_argmax(logits.permute(0, 2, 1), seed), v.C)
        full, g, ids = self._partial_to_full(logits, key, float("-inf"))
        full[:, [a for a in range(v.S) if a % v.n_attr != g]] = 0.0        # other attributes' positions: any finite row (their draw is discarded)
        xt = self.engine.gumbel_argmax(full, seed)[:, g::v.n_attr]
        return index_to_log_onehot((xt[..., None] == ids).long().argmax(-1), ids.numel())

    def sample_logits(self, logits: torch.Tensor, sampling_cfg, seed: Optional[int] = None) -> torch.Tensor:
        """helpers/sampling.py:81-130 `sample(logits, sampling_cfg)`: (B,C,S) logits -> (B,1,S) ids.  noise="torch": the draw of
        the reference's `sample` on contiguous (B,C,S) logits, one step of torch's CUDA generator"""
        B = logits.shape[0]
        dummy = torch.zeros(B, self.vocab.S, dtype=torch.long, device=self.device)
        lp = logits.to(self.device).permute(0, 2, 1)
        if self.noise == "torch":
            out = self._with_torch_noise(B, sampling_cfg, 1, seed, lambda noise: self.engine.step(dummy, 0, 0, sampling_cfg, None, 0, 0, logprob_in=lp,
                                                                                                   noise=noise)[0])
        else:
            out = self.engine.step(dummy, 0, 0, sampling_cfg, None, self._new_seed() if seed is None else seed, 0, logprob_in=lp)[0]
        return out[:, None, :]

    def q_sample(self, log_x_start: torch.Tensor, t: torch.Tensor, key: Optional[str] = None, seed: Optional[int] = None) -> torch.Tensor:
        """constrained.py:223-230: x_t ~ q(x_t|x_0) for attribute `key` (log one-hot in, log one-hot out, partial vocabulary)"""
        v = self.vocab
        seed = self._new_seed() if seed is None else seed
        if self.engine.q_type != "constrained" or key is None:
            xt = self.engine.q_sample(log_x_start.argmax(1), t, seed)
            return index_to_log_onehot(xt, v.C)
        g = self._key_index(key)
        ids = torch.tensor(group_full_ids(v, g), device=self.device)
        x0 = torch.full((log_x_start.shape[0], v.S), v.pad_id, dtype=torch.long, device=self.device)
        x0[:, g::v.n_attr] = ids[log_x_start.to(self.device).argmax(1)]
        xt = self.engine.q_sample(x0, t, seed)[:, g::v.n_attr]
        part = (xt[..., None] == ids).long().argmax(-1)                     # full id -> index in the partial vocabulary
        return index_to_log_onehot(part, ids.numel())

    def sample_time(self, b: int, device=None, method: str = "uniform"):
        """base.py:179-203 (host-side importance sampling over the running loss history)"""
        device = self.device if device is None else device
        if method == "importance":
            if not (self.Lt_count > 10).all():
                return self.sample_time(b, device, method="uniform")
            Lt_sqrt = torch.sqrt(self.Lt_history + 1e-10) + 0.0001
            Lt_sqrt[0] = Lt_sqrt[1]
            pt_all = Lt_sqrt / Lt_sqrt.sum()
            t = torch.multinomial(pt_all, num_samples=b, replacement=True)
            return t, pt_all.gather(dim=0, index=t)
        if method == "uniform":
            t = torch.randint(0, self.num_timesteps, (b,), device=device).long()
            return t, torch.ones_like(t).float() / self.num_timesteps
        raise ValueError

    def forward(self, x: torch.Tensor, is_train: bool = True, t: Optional[torch.Tensor] = None, pt: Optional[torch.Tensor] = None,
                seed: Optional[int] = None):
        """constrained.py:232-333 / vanilla.py:177-243, FORWARD ONLY (validation loss; no autograd graph is built -- the optimiser
        step of the reference's training loop stays out of scope).  x (B,S) ids -> ({"probs": (B,C,S)}, {"kl_loss", "aux_loss"})."""
        self._follow_weights()
        if not hasattr(self, "Lt_history"):
            self.Lt_history = torch.zeros(self.num_timesteps, device=self.device)
            self.Lt_count = torch.zeros(self.num_timesteps, device=self.device)
            self.diffusion_acc_list = [0] * self.num_timesteps
            self.diffusion_keep_list = [0] * self.num_timesteps
            self.mask_weight = [1.0, 1.0]
            self.auxiliary_loss_weight = 1e-1
            self.adaptive_auxiliary_loss = True
        x = x.to(self.device)
        b = x.size(0)
        if t is None:
            t, pt = self.sample_time(b, self.device, "importance")
        t, pt = t.to(self.device), pt.to(self.device)
        xt = self.engine.q_sample(x, t, self._new_seed() if seed is None else seed)
        aux_on = self.auxiliary_loss_weight != 0 and is_train
        r = self.engine.vb_terms(x, xt, t, self.mask_weight, want_aux=aux_on, want_log_model_prob=True, want_recon_ids=True)
        same0 = (r["x0_recon"] == x).float().mean(1).cpu()
        same1 = (r["xt_1_recon"] == xt).float().mean(1).cpu()
        for i, this_t in enumerate(t.tolist()):                                               # :273-292
            self.diffusion_acc_list[this_t] = same0[i].item() * 0.1 + self.diffusion_acc_list[this_t] * 0.9
            self.diffusion_keep_list[this_t] = same1[i].item() * 0.1 + self.diffusion_keep_list[this_t] * 0.9
        mask = (t == 0).float()
        kl_loss = mask * r["decoder_nll"] + (1.0 - mask) * r["kl"]                             # :307-308
        Lt2 = kl_loss.pow(2)
        Lt2_prev = self.Lt_history.gather(dim=0, index=t)
        self.Lt_history.scatter_(dim=0, index=t, src=(0.1 * Lt2 + 0.9 * Lt2_prev))
        self.Lt_count.scatter_add_(dim=0, index=t, src=torch.ones_like(Lt2))
        losses = {"kl_loss": (kl_loss / pt).mean()}
        if aux_on:
            kl_aux_loss = mask * r["decoder_nll"] + (1.0 - mask) * r["kl_aux"]
            w = (1 - t / self.num_timesteps) + 1.0 if self.adaptive_auxiliary_loss else 1.0
            losses["aux_loss"] = (w * self.auxiliary_loss_weight * kl_aux_loss / pt).mean()
        return {"probs": r["log_model_prob"].permute(0, 2, 1).exp()}, losses

    __call__ = forward

    def q_sample_ids(self, x0: torch.Tensor, t: torch.Tensor, seed: Optional[int] = None) -> torch.Tensor:
        """corruption x_t ~ q(x_t | x_0) on ids (constrained.py:223-230 applied per attribute as in :232-260)"""
        return self.engine.q_sample(x0, t, self._new_seed() if seed is None else seed)

    _pinned = False

    def reset_noise(self, seed: Optional[int] = None):
        """pin the noise key of the following `_sample_single_step` calls (seed=None: back to torch's global generator)"""
        self._seed, self._step_ctr, self._last_t, self._pinned = seed, 0, None, seed is not None

    def predict_logits(self, ids: torch.Tensor, t: int) -> torch.Tensor:
        """CategoricalTransformer.forward (nn_lib.py:191-237): ids (B,S) -> logits (B,S,C) on the GPU"""
        self._follow_weights()
        s = sampling_struct({"name": "deterministic"})
        _, lg, _ = self.engine.step(ids.to(self.device), t, t, s, want_logits=True)
        return lg


class LayoutDMB200:
    """LayoutDM wrapper (models/layoutdm.py:26-97): `.sample()` returns decoded layouts on the CPU."""

    def __init__(self, engine: Engine, tokenizer=None, bbox_centers=None, noise: str = "contract"):
        self.model = FusedMaskAndReplaceDiffusion(engine, tokenizer, bbox_centers, noise=noise)
        self.tokenizer = tokenizer
        self.vocab = engine.vocab
        self._centers = bbox_centers

    @classmethod
    def from_state_dict(cls, sd, dataset: str = "rico25", num_timesteps: int = 100, q_type: str = "constrained",
                        operand_dtype: str = "fp16", device=None, tokenizer=None, bbox_centers=None, noise: str = "contract") -> "LayoutDMB200":
        """noise: "contract" (the project's Philox contract) or "torch" (torch's CUDA generator, FusedMaskAndReplaceDiffusion)"""
        vocab = Vocab.from_tokenizer(tokenizer) if tokenizer is not None else Vocab.for_dataset(dataset)
        eng = Engine.from_state_dict(sd, vocab, num_timesteps=num_timesteps, q_type=q_type, operand_dtype=operand_dtype, device=device)
        return cls(eng, tokenizer, bbox_centers, noise=noise)

    def eval(self):
        return self

    def load_state_dict(self, sd) -> "LayoutDMB200":
        """repack another checkpoint of the same shapes into the engine in place, like the reference's
        `model.load_state_dict(torch.load(...))` (test.py's load_model); returns self"""
        self.model.engine.load_state_dict(sd)
        return self

    def sample(self, batch_size: Optional[int] = 1, cond: Optional[Dict] = None, sampling_cfg=None, total_layouts: Optional[int] = None,
               **kwargs) -> Dict[str, torch.Tensor]:
        """layoutdm.py:77-88 (extra kwargs such as cond_type= / device= are swallowed like the reference does)"""
        kw = {k: v for k, v in kwargs.items() if k in ("seed", "b_global0", "get_intermediate_results")}
        if total_layouts is not None:
            kw["total_layouts"] = total_layouts
        ids = self.model.sample(batch_size=batch_size, cond=cond, sampling_cfg=sampling_cfg, **kw)
        if self.tokenizer is not None:
            return self.tokenizer.decode(ids)
        if kw.get("get_intermediate_results", False):
            return ids                                             # the list of per-step ids, like the core's sample()
        if kwargs.get("decode_on_device", True):                   # ids -> layouts on the GPU (ldm_decode), results back on the CPU like layoutdm.py:87
            c = None if self._centers is None else torch.stack([torch.as_tensor(x, dtype=torch.float32).view(-1) for x in self._centers])
            return {k: v.cpu() for k, v in self.model.engine.decode(ids, c).items()}
        return decode_ids(ids, self.vocab, self._centers)          # host fallback (decode_on_device=False)

    def get_cond(self, label: torch.Tensor, bbox: torch.Tensor, mask: torch.Tensor, cond_type: str = "c", refine: Optional[dict] = None) -> Dict:
        """helpers/task.py:get_cond (:27-151) for dense layouts (what `sparse_to_dense(batch)` returns: bbox (B,E,4), label (B,E),
        mask (B,E)), built on the GPU for cond_type c / cwh / gt / refinement; for refinement the N(0, 0.1) box noise of
        task.py:127 is drawn here from torch's global generator, like the reference does."""
        if cond_type == "refinement":
            bbox = bbox + torch.normal(0, std=0.1, size=bbox.size())
        c = None if self._centers is None else torch.stack([torch.as_tensor(x, dtype=torch.float32).view(-1) for x in self._centers])
        return self.model.engine.cond_from_layouts(label, bbox, mask, cond_type, centers=c, refine=refine)

    def aggregate_sampling_settings(self, sampling_cfg, args):
        """base_model.py:124-150 + layoutdm.py:90-97"""
        if args.cond == "refinement" and args.refine_lambda > 0.0:
            sampling_cfg.refine_mode = args.refine_mode
            sampling_cfg.refine_offset_ratio = args.refine_offset_ratio
            sampling_cfg.refine_lambda = args.refine_lambda
        if args.cond == "relation" and args.relation_lambda > 0.0:
            sampling_cfg.relation_mode = args.relation_mode
            sampling_cfg.relation_lambda = args.relation_lambda
            sampling_cfg.relation_tau = args.relation_tau
            sampling_cfg.relation_num_update = args.relation_num_update
        if "num_timesteps" not in sampling_cfg:
            sampling_cfg.num_timesteps = args.num_timesteps
        if args.time_difference > 0:
            sampling_cfg.time_difference = args.time_difference
        return sampling_cfg


def patch_reference_model(model, operand_dtype: str = "fp16", device=None, noise: str = "contract"):
    """Drop-in for a live reference `trainer.models.layoutdm.LayoutDM`: after `patch_reference_model(model)`,
    `model.sample(...)` (layoutdm.py:77) and `model.model.sample(...)` / `_sample_single_step(...)` run on the sm_90a library.
    Training `forward` is untouched.  The library follows the model's weights: optimizer steps, `load_state_dict` and device
    moves after patching are picked up by the next sampling call (WeightFollower); after writes through `.data`, call
    `model.model.module._ldm_b200.reload_weights()`.
    noise="torch": the draws come from torch's CUDA generator like the unpatched model's on the same GPU."""
    core = model.model.module if hasattr(model.model, "module") else model.model
    tok = model.tokenizer
    vocab = Vocab.from_tokenizer(tok)
    q_type = "vanilla" if type(core).__name__.startswith("Vanilla") else "constrained"
    eng = Engine.from_state_dict(model.state_dict(), vocab, num_timesteps=core.num_timesteps, q_type=q_type,
                                 operand_dtype=operand_dtype, device=device)
    fused = FusedMaskAndReplaceDiffusion(eng, tok, noise=noise)
    fused.follow(core.transformer)
    # cond=relation: the reference's own gradient update (logit_adjustment.py:88-126) runs between the posterior and the draw.
    # `model` is a live reference object, so its package is importable; an import failure is an error, not a silent downgrade.
    import importlib
    _update = importlib.import_module(type(core).__module__.rsplit(".", 1)[0] + ".logit_adjustment").update

    def _hook(t, cond, model_log_prob, sampling_cfg):
        return _update(t=t, cond=cond, model_log_prob=model_log_prob, tokenizer=tok, sampling_cfg=sampling_cfg)
    fused.logit_adjust_fn = _hook
    core.sample = fused.sample
    core._sample_single_step = fused._sample_single_step
    core._ldm_b200 = fused
    return model
