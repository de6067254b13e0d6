"""Engine: owns one LdmHandle (packed weights + workspace on one GPU) and exposes step / loop calls on torch
CUDA tensors.  PyTorch is only used for device memory and the current stream; all compute is in libldm_b200.so."""
from __future__ import annotations

import ctypes as C
import math
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from . import _lib
from .vocab import Vocab, linear_centers, refinement_table

PREFIXES = ("model.module.transformer.", "model.transformer.", "module.transformer.", "transformer.", "")


def _find_prefix(sd) -> str:
    for p in PREFIXES:
        if p + "cat_emb.weight" in sd:
            return p
    raise KeyError("state_dict does not contain '<prefix>cat_emb.weight' (expected the reference's LayoutDM keys)")


def layout_length(sd) -> int:
    """the layout length (max_seq_length, elements per layout) a reference state_dict was trained for: the rows of its
    ElementPositionalEmbedding's element table, or those of its PositionalEmbedding's token table / 5 (nn_lib.py:73-127)"""
    p = _find_prefix(sd)
    if p + "pos_emb.elem_emb" in sd:
        return int(sd[p + "pos_emb.elem_emb"].shape[0])
    if p + "pos_emb.pos_emb" in sd:
        rows = int(sd[p + "pos_emb.pos_emb"].shape[0])
        if rows % 5:
            raise ValueError(f"pos_emb.pos_emb has {rows} rows, not 5 tokens (c-x-y-w-h) per element")
        return rows // 5
    raise KeyError("state_dict has no positional table ('<prefix>pos_emb.elem_emb' or '<prefix>pos_emb.pos_emb')")


def block_settings(timestep_type: Optional[str], activation: str) -> Tuple[int, int]:
    """the denoiser block's timestep_type / activation (backbone.encoder_layer, transformer_utils.py:103-170) -> LdmModelDesc's
    (norm1_kind, activation), refused as the reference refuses them"""
    if isinstance(timestep_type, str) and timestep_type.endswith("_mlp"):
        raise NotImplementedError(f"timestep_type={timestep_type!r}: the reference's LayoutDM raises for it when sampling (its _AdaNorm "
                                  "MLP, nn.Linear(1, ...), is given the long timesteps base.py builds), so there is nothing to reproduce")
    assert timestep_type in _lib.NORM1_KINDS, f"timestep_type={timestep_type!r} is not one of {list(_lib.NORM1_KINDS)} (transformer_utils.py:124-132)"
    if activation not in _lib.ACTIVATIONS:
        raise RuntimeError(f"activation should be relu/gelu/gelu2, not {activation}")        # transformer_utils.py:28-31
    return _lib.NORM1_KINDS[timestep_type], _lib.ACTIVATIONS[activation]


def sinusoidal_table(num_timesteps: int, diffusion_step: int, d: int) -> torch.Tensor:
    """(T, d) fp32: SinusoidalPosEmb(diffusion_step, d)(t) for t = 0 .. T-1 (transformer_utils.py:34-49, rescale_steps 4000), the
    reference's own float32 operations on its long timesteps"""
    x = torch.arange(num_timesteps) / float(diffusion_step) * 4000.0
    half = d // 2
    e = torch.exp(torch.arange(half) * -(math.log(10000) / (half - 1)))
    e = x[:, None] * e[None, :]
    return torch.cat((e.sin(), e.cos()), dim=-1)


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else C.c_void_p(t.data_ptr())


def sampling_struct(cfg) -> _lib.LdmSampling:
    """reference sampling_cfg (DictConfig / dict / dataclass-like) -> LdmSampling (helpers/sampling.py:13-59)"""
    get = (lambda k, d=None: cfg.get(k, d)) if hasattr(cfg, "get") else (lambda k, d=None: getattr(cfg, k, d))
    name = get("name")
    if name not in _lib.SAMPLING_MODES:
        raise NotImplementedError(f"sampling '{name}'")          # sampling.py:117-118
    s = _lib.LdmSampling()
    s.mode = _lib.SAMPLING_MODES[name]
    s.temperature = float(get("temperature", 1.0) or 1.0)
    s.top_p = float(get("top_p", 0.9) or 0.9)
    s.top_k = int(get("top_k", 5) or 5)
    if name == "top_p":
        assert 0.0 < s.top_p <= 1.0                             # sampling.py:96
    return s


class Engine:
    def __init__(self, vocab: Vocab, weights: Dict[str, torch.Tensor], num_timesteps: int = 100, q_type: str = "constrained",
                 operand_dtype: str = "fp16", device: Optional[int] = None, d_model: int = 464, n_heads: int = 8, d_ff: int = 1856,
                 att_1=0.99999, att_T=0.000009, ctt_1=0.000009, ctt_T=0.99999, timestep_type: Optional[str] = "adalayernorm",
                 activation: str = "relu", diffusion_step: Optional[int] = None):
        """weights: the `pack_state_dict` arrays.  timestep_type / activation / diffusion_step: the denoiser block's settings
        (backbone.encoder_layer.*); `load_state_dict` packs later checkpoints with them.  diffusion_step: what the sinusoidal
        embedding of the *_abs types divides by (None: num_timesteps)."""
        if operand_dtype not in _lib.OPERAND_DTYPES:
            raise ValueError(f"operand_dtype must be one of {', '.join(_lib.OPERAND_DTYPES)}, got {operand_dtype!r}")
        norm1_kind, act = block_settings(timestep_type, activation)
        if not torch.cuda.is_available():
            raise RuntimeError("layoutdm_b200 needs a CUDA (sm_90a, H100) device; there is no CPU fallback")
        self.lib = _lib.load()
        self.vocab = vocab
        self.T = num_timesteps
        self.q_type = q_type
        self.operand_dtype = operand_dtype
        self.timestep_type, self.activation, self.diffusion_step = timestep_type, activation, diffusion_step
        self.device_index = torch.cuda.current_device() if device is None else int(device)
        self.device = torch.device("cuda", self.device_index)
        L = weights["in_proj_w"].shape[0]
        self.n_layers, self.d_model, self.d_ff = L, d_model, d_ff
        desc = _lib.LdmModelDesc(vocab.n_cat, vocab.n_bins, vocab.n_elem, vocab.n_attr, d_model, n_heads, d_ff, L, num_timesteps,
                                 {"constrained": 0, "vanilla": 1}[q_type], _lib.OPERAND_DTYPES[operand_dtype], self.device_index,
                                 att_1, att_T, ctt_1, ctt_T, norm1_kind, act, _lib.BBOX_VOCABS[vocab.shared_bbox_vocab],
                                 _lib.VAR_ORDERS[vocab.var_order])
        w = _lib.LdmWeights()
        keep = []
        for name in _lib._W_FIELDS:
            t = weights[name].detach().to("cpu", torch.float32).contiguous()
            keep.append(t)
            setattr(w, name, t.data_ptr())
        h = C.c_void_p()
        _lib.check(self.lib.ldm_create(C.byref(desc), C.byref(w), C.byref(h)))
        self._h = h

    @property
    def layout_rows(self) -> int:
        """rows a layout takes in the workspace (ldm_debug_read): 128 R, R = ceil(S / 128) row tiles; rows S .. are pad rows"""
        return 128 * ((self.vocab.S + 127) // 128)

    # ------------------------------------------------------------------------------------------------
    @classmethod
    def from_state_dict(cls, sd: Dict[str, torch.Tensor], vocab: Vocab, num_timesteps: int = 100, timestep_type: Optional[str] = "adalayernorm",
                        activation: str = "relu", diffusion_step: Optional[int] = None, **kw) -> "Engine":
        """sd: the reference LayoutDM `state_dict()` (keys `model.module.transformer.*`, SURVEY.md 8a-a5), of a model whose blocks
        have these timestep_type / activation / diffusion_step settings."""
        block_settings(timestep_type, activation)
        w = cls.pack_state_dict(sd, vocab, timestep_type, diffusion_step, num_timesteps=num_timesteps)
        return cls(vocab, w, num_timesteps=num_timesteps, timestep_type=timestep_type, activation=activation, diffusion_step=diffusion_step, **kw)

    @staticmethod
    def pack_state_dict(sd, vocab: Vocab, timestep_type: Optional[str] = "adalayernorm", diffusion_step: Optional[int] = None,
                        num_timesteps: Optional[int] = None, device=None) -> Dict[str, torch.Tensor]:
        """the reference's parameters in the LdmWeights layout, fp32, on `device` (default: the CPU).  Parameters already on
        `device` are stacked there, with no host round trip.

        norm1 of every timestep_type is a filling of the AdaLN arrays norm1_emb / norm1_w / norm1_b, whose table
        Linear(SiLU(norm1_emb[t])) gives (scale_t, shift_t) and norm1 = norm(x) * (1 + scale_t) + shift_t:
          adalayernorm / adainnorm          : the Embedding and Linear as they are
          adalayernorm_abs / adainnorm_abs  : norm1_emb[l][t] = SinusoidalPosEmb(diffusion_step, d)(t) (`sinusoidal_table`)
          None (nn.LayerNorm with affine)   : norm1_emb = 0, norm1_w = 0, norm1_b = [weight - 1, bias] -> (1 + scale, shift) = (w, b)
        The table has num_timesteps rows; the types without an Embedding need num_timesteps (diffusion_step defaults to it).
        norm1 keys that contradict timestep_type are a ValueError."""
        block_settings(timestep_type, "relu")          # refuses *_mlp and unknown types
        p = _find_prefix(sd)
        device = torch.device("cpu") if device is None else torch.device(device)
        g = lambda k: sd[p + k].detach().to(device, torch.float32)
        L = 0
        while f"{p}backbone.layers.{L}.linear1.weight" in sd:
            L += 1
        st = lambda k: torch.stack([g(f"backbone.layers.{l}.{k}") for l in range(L)]).contiguous()
        if sd[p + "cat_emb.weight"].shape[0] != vocab.C:
            raise ValueError(f"the state_dict's cat_emb has {sd[p + 'cat_emb.weight'].shape[0]} rows, the vocabulary has C = {vocab.C} "
                             f"({vocab.n_cat} categories, {vocab.n_bins} bins, shared_bbox_vocab {vocab.shared_bbox_vocab}): a model of "
                             "other tokenizer settings")
        if p + "pos_emb.elem_emb" in sd and sd[p + "pos_emb.elem_emb"].shape[0] != vocab.n_elem:
            raise ValueError(f"the state_dict's positional table is for {sd[p + 'pos_emb.elem_emb'].shape[0]} elements, the vocabulary "
                             f"has {vocab.n_elem}: a model of another max_seq_length")
        if p + "pos_emb.elem_emb" in sd:      # ElementPositionalEmbedding, nn_lib.py:112-127
            pos = (g("pos_emb.elem_emb").repeat_interleave(vocab.n_attr, dim=0) + g("pos_emb.attr_emb").repeat(vocab.n_elem, 1))[: vocab.S]
        else:                                  # PositionalEmbedding, nn_lib.py:73-88
            pos = g("pos_emb.pos_emb")[: vocab.S]
        if pos.shape[0] != vocab.S:
            raise ValueError(f"the state_dict's positional table covers {pos.shape[0]} tokens, the vocabulary has S = {vocab.S} "
                             f"({vocab.n_elem} elements): a model of another max_seq_length")
        n1 = f"{p}backbone.layers.0.norm1."
        kind = "None (nn.LayerNorm)" if n1 + "weight" in sd else "an Embedding timestep (adalayernorm / adainnorm)" \
            if n1 + "emb.weight" in sd else "a sinusoidal timestep (*_abs)" if n1 + "linear.weight" in sd else "no norm1"
        want = {None: "weight", "adalayernorm": "emb.weight", "adainnorm": "emb.weight"}.get(timestep_type, "linear.weight")
        if n1 + want not in sd or (want == "linear.weight" and n1 + "emb.weight" in sd):
            raise ValueError(f"timestep_type={timestep_type!r}, but the state_dict's norm1 keys are those of {kind}")
        if timestep_type in (None, "adalayernorm_abs", "adainnorm_abs"):
            if num_timesteps is None:
                raise ValueError(f"timestep_type={timestep_type!r} has no timestep table in the state_dict: give num_timesteps")
            d = sd[p + "cat_emb.weight"].shape[1]
            if timestep_type is None:
                norm1_emb = torch.zeros(L, num_timesteps, d, device=device)
                norm1_w = torch.zeros(L, 2 * d, d, device=device)
                norm1_b = torch.cat([st("norm1.weight") - 1.0, st("norm1.bias")], dim=1)
            else:
                sin = sinusoidal_table(num_timesteps, num_timesteps if diffusion_step is None else diffusion_step, d)
                norm1_emb = sin.to(device)[None].expand(L, -1, -1).contiguous()
                norm1_w, norm1_b = st("norm1.linear.weight"), st("norm1.linear.bias")
        else:
            norm1_emb, norm1_w, norm1_b = st("norm1.emb.weight"), st("norm1.linear.weight"), st("norm1.linear.bias")
            if num_timesteps is not None:      # an Embedding of diffusion_step rows: the sampler reads rows t < num_timesteps
                if norm1_emb.shape[1] < num_timesteps:
                    raise ValueError(f"norm1.emb has {norm1_emb.shape[1]} rows (diffusion_step), fewer than num_timesteps = {num_timesteps}")
                norm1_emb = norm1_emb[:, :num_timesteps].contiguous()
        return dict(
            cat_emb=g("cat_emb.weight"), pos_table=pos.contiguous(),
            in_proj_w=st("self_attn.in_proj_weight"), in_proj_b=st("self_attn.in_proj_bias"),
            out_proj_w=st("self_attn.out_proj.weight"), out_proj_b=st("self_attn.out_proj.bias"),
            linear1_w=st("linear1.weight"), linear1_b=st("linear1.bias"), linear2_w=st("linear2.weight"), linear2_b=st("linear2.bias"),
            norm1_emb=norm1_emb, norm1_w=norm1_w, norm1_b=norm1_b,
            norm2_w=st("norm2.weight"), norm2_b=st("norm2.bias"),
            head_ln_w=g("head.0.weight"), head_ln_b=g("head.0.bias"), head_w=g("head.1.weight"))

    def weight_shapes(self) -> Dict[str, Tuple[int, ...]]:
        """the shape of every LdmWeights field for this handle (include/ldm_b200.h)"""
        C, S, d, f, L, T = self.vocab.C, self.vocab.S, self.d_model, self.d_ff, self.n_layers, self.T
        return dict(cat_emb=(C, d), pos_table=(S, d), in_proj_w=(L, 3 * d, d), in_proj_b=(L, 3 * d), out_proj_w=(L, d, d),
                    out_proj_b=(L, d), linear1_w=(L, f, d), linear1_b=(L, f), linear2_w=(L, d, f), linear2_b=(L, d),
                    norm1_emb=(L, T, d), norm1_w=(L, 2 * d, d), norm1_b=(L, 2 * d), norm2_w=(L, d), norm2_b=(L, d),
                    head_ln_w=(d,), head_ln_b=(d,), head_w=(C, d))

    def load_weights(self, weights: Dict[str, torch.Tensor]):
        """Repack new weights (the `pack_state_dict` dict, on any device) into this handle in place (ldm_load_weights), on the
        current stream: sampling queued before sees the old weights, sampling after the new ones.  The shapes must be the
        handle's; a captured sampling graph stays valid."""
        want = self.weight_shapes()
        stream = torch.cuda.current_stream(self.device)
        w = _lib.LdmWeights()
        keep = []
        for name in _lib._W_FIELDS:
            t = weights[name].detach().to(self.device, torch.float32).contiguous()
            if tuple(t.shape) != want[name]:
                raise ValueError(f"weight {name}: shape {tuple(t.shape)}, the handle was built for {want[name]}")
            t.record_stream(stream)          # the packing kernels read it after this call returns
            keep.append(t)
            setattr(w, name, t.data_ptr())
        _lib.check(self.lib.ldm_load_weights(self._h, C.byref(w), C.c_void_p(stream.cuda_stream)))

    def load_state_dict(self, sd: Dict[str, torch.Tensor]):
        """load_weights from a reference LayoutDM `state_dict()` (any of the key prefixes `from_state_dict` takes)"""
        self.load_weights(self.pack_state_dict(sd, self.vocab, self.timestep_type, self.diffusion_step, num_timesteps=self.T, device=self.device))

    def close(self):
        if getattr(self, "_h", None):
            self.lib.ldm_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ------------------------------------------------------------------------------------------------
    @property
    def launch_count(self) -> int:
        return int(self.lib.ldm_launch_count(self._h))

    def profile_begin(self):
        _lib.check(self.lib.ldm_profile_begin(self._h))

    def profile_end(self) -> Dict[str, Tuple[float, int]]:
        """{category: (total ms, launches)} of everything launched since profile_begin()"""
        n = len(_lib.PROFILE_CATEGORIES)
        ms, cnt = (C.c_float * n)(), (C.c_int64 * n)()
        _lib.check(self.lib.ldm_profile_end(self._h, ms, cnt, n))
        return {name: (float(ms[i]), int(cnt[i])) for i, name in enumerate(_lib.PROFILE_CATEGORIES)}

    def schedule_tables(self) -> torch.Tensor:
        n = self.lib.ldm_get_schedule(self._h, None, 0)
        out = torch.empty(n, dtype=torch.float32)
        self.lib.ldm_get_schedule(self._h, C.c_void_p(out.data_ptr()), n)
        G = self.vocab.n_attr if self.q_type == "constrained" else 1
        return out.view(G, 8, self.T + 1)

    def adaln_table(self) -> torch.Tensor:
        n = self.lib.ldm_get_adaln_table(self._h, None, 0)
        out = torch.empty(n, dtype=torch.float32)
        self.lib.ldm_get_adaln_table(self._h, C.c_void_p(out.data_ptr()), n)
        return out.view(-1, self.T, 2 * 464)

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def make_cond(self, cond: Optional[dict]) -> Tuple[Optional[_lib.LdmCond], list]:
        """cond tensors must already be on self.device: seq (B,S) i64, mask (B,S) bool/uint8, optional seq_orig, refine_table."""
        if not cond:
            return None, []
        keep = []
        c = _lib.LdmCond()
        seq = cond["seq"].to(self.device, torch.int64).contiguous(); keep.append(seq)
        c.seq = seq.data_ptr()
        if cond.get("mask") is not None:
            m = cond["mask"].to(self.device).to(torch.uint8).contiguous(); keep.append(m)
            c.mask = m.data_ptr()
        if cond.get("seq_orig") is not None and cond.get("refine_table") is not None:
            so = cond["seq_orig"].to(self.device, torch.int64).contiguous(); keep.append(so)
            tb = cond["refine_table"].to(self.device, torch.float32).contiguous(); keep.append(tb)
            assert tb.shape == (self.vocab.C, self.vocab.C), f"refine_table must be (C, C) = ({self.vocab.C}, {self.vocab.C}), got {tuple(tb.shape)}"
            c.seq_orig, c.refine_table = so.data_ptr(), tb.data_ptr()
        c.pad_disable = 1 if cond.get("type") in ("c", "cwh", "refinement", "relation") else 0   # base.py:272
        if cond.get("rel_adj") is not None and int(cond.get("rel_num_update", 0)) > 0:
            # cond = relation on the device (logit_adjustment.py:88-126): dense edge table, bin centres, SGD hyper-parameters
            E1 = self.vocab.n_elem + 1
            adj = cond["rel_adj"].to(self.device, torch.int32).contiguous(); keep.append(adj)
            assert adj.shape == (seq.shape[0], E1, E1), f"rel_adj must be (B, {E1}, {E1}), got {tuple(adj.shape)}"
            c.rel_adj = adj.data_ptr()
            if cond.get("rel_centers") is not None:
                cen = cond["rel_centers"].to(self.device, torch.float32).contiguous(); keep.append(cen)
                assert cen.shape == (4, self.vocab.n_bins)
                c.rel_centers = cen.data_ptr()
            c.rel_lambda = float(cond["rel_lambda"])
            c.rel_num_update = int(cond["rel_num_update"])
            c.rel_batch_total = int(cond.get("rel_batch_total", 0) or 0)
        if cond.get("_pad_disable") is not None:                     # relation hook: PAD-disable comes after update() (base.py:261-284)
            c.pad_disable = 1 if cond["_pad_disable"] else 0
        return c, keep

    def noise_advance(self, total_layouts: int, sampling, n_steps: int) -> int:
        """how far `n_steps` steps on a batch of `total_layouts` layouts move torch's CUDA generator (ldm_noise_advance)"""
        s = sampling if isinstance(sampling, _lib.LdmSampling) else sampling_struct(sampling)
        adv = int(self.lib.ldm_noise_advance(self._h, int(total_layouts), C.byref(s), int(n_steps)))
        _lib.check(adv if adv < 0 else _lib.LDM_OK)
        return adv

    @staticmethod
    def _noise(noise: Optional[_lib.LdmNoise], seed: int) -> _lib.LdmNoise:
        return _lib.LdmNoise(_lib.NOISE_KINDS["contract"], seed, 0, 0) if noise is None else noise

    def step(self, ids_in: torch.Tensor, t_model: int, t_post: int, sampling, cond: Optional[dict] = None, seed: int = 0,
             step_ctr: int = 0, b_global0: int = 0, want_logits: bool = False, want_logprob: bool = False,
             logits_in: Optional[torch.Tensor] = None, logprob_in: Optional[torch.Tensor] = None, noise: Optional[_lib.LdmNoise] = None):
        """one `_sample_single_step` on ids; returns (ids_out, logits | None, logprob | None), all on the GPU.
        noise: an LdmNoise (torch-generator noise); None: the contract keyed by seed / step_ctr."""
        B, S = ids_in.shape
        assert S == self.vocab.S and ids_in.is_cuda and ids_in.dtype == torch.int64
        assert int(ids_in.max()) < self.vocab.C, f"Error: {int(ids_in.max())} >= {self.vocab.C}"     # util.py:35
        ids_in = ids_in.contiguous()
        out = torch.empty_like(ids_in)
        lg = torch.empty(B, S, self.vocab.C, device=self.device) if want_logits else None
        lp = torch.empty(B, S, self.vocab.C, device=self.device) if want_logprob else None
        c, keep = self.make_cond(cond)
        s = sampling if isinstance(sampling, _lib.LdmSampling) else sampling_struct(sampling)
        li = None if logits_in is None else logits_in.to(self.device, torch.float32).contiguous()
        pi = None if logprob_in is None else logprob_in.to(self.device, torch.float32).contiguous()
        rc = self.lib.ldm_step_noise(self._h, B, _ptr(ids_in), int(t_model), int(t_post), C.byref(c) if c else None, C.byref(s),
                                     C.byref(self._noise(noise, seed)), C.c_uint32(step_ctr), C.c_int64(b_global0), _ptr(out), _ptr(lg),
                                     _ptr(lp), _ptr(li), _ptr(pi), self._stream())
        _lib.check(rc)
        return out, lg, lp

    def sample_loop(self, B: int, plan: Sequence[Tuple[int, int]], sampling, cond: Optional[dict] = None, seed: int = 0,
                    b_global0: int = 0, ids_init: Optional[torch.Tensor] = None, trace: bool = False, noise: Optional[_lib.LdmNoise] = None):
        """whole T-step loop on the device; returns ids (B,S) [and the (n_steps,B,S) trace] as CUDA tensors.
        noise: an LdmNoise (torch-generator noise, step k at its offset + k steps); None: the contract keyed by seed."""
        n = len(plan)
        tm = (C.c_int32 * n)(*[p[0] for p in plan])
        tp = (C.c_int32 * n)(*[p[1] for p in plan])
        out = torch.empty(B, self.vocab.S, dtype=torch.int64, device=self.device)
        tr = torch.empty(n, B, self.vocab.S, dtype=torch.int64, device=self.device) if trace else None
        c, keep = self.make_cond(cond)
        s = sampling if isinstance(sampling, _lib.LdmSampling) else sampling_struct(sampling)
        if ids_init is not None:
            ids_init = ids_init.to(self.device, torch.int64).contiguous()
        rc = self.lib.ldm_sample_loop_noise(self._h, B, n, tm, tp, C.byref(c) if c else None, C.byref(s), C.byref(self._noise(noise, seed)),
                                            C.c_int64(b_global0), _ptr(ids_init), _ptr(out), _ptr(tr), self._stream())
        _lib.check(rc)
        return (out, tr) if trace else out

    def q_sample(self, x0: torch.Tensor, t: torch.Tensor, seed: int = 0, b_global0: int = 0) -> torch.Tensor:
        """forward (corruption) process: x0 (B,S) ids, t (B,) timesteps -> x_t ids (CUDA)"""
        B, S = x0.shape
        assert S == self.vocab.S and int(t.min()) >= 0 and int(t.max()) < self.T
        x0 = x0.to(self.device, torch.int64).contiguous()
        t32 = t.to(self.device, torch.int32).contiguous()
        out = torch.empty_like(x0)
        _lib.check(self.lib.ldm_q_sample(self._h, B, _ptr(x0), _ptr(t32), C.c_uint64(seed), C.c_int64(b_global0), _ptr(out), self._stream()))
        return out

    # ---- training-side API on (B, S, C) log tensors, per-layout timesteps (SURVEY 8f-3) ------------------------------
    def _t32(self, t: torch.Tensor, B: int, lo: int = 0) -> torch.Tensor:
        t = t.to(self.device).view(-1)
        assert t.numel() == B and int(t.min()) >= lo and int(t.max()) < self.T                     # constrained.py:139
        return t.to(torch.int32).contiguous()

    def predict_start(self, xt: torch.Tensor, t: torch.Tensor, want_logits: bool = False):
        """base.py:127-146 at per-layout timesteps: xt (B,S) ids, t (B,) -> log p(x0|xt) (B,S,C) [, logits (B,S,C)] on the GPU"""
        B = xt.shape[0]
        xt = xt.to(self.device, torch.int64).contiguous()
        t32 = self._t32(t, B)
        out = torch.empty(B, self.vocab.S, self.vocab.C, device=self.device)
        lg = torch.empty_like(out) if want_logits else None
        _lib.check(self.lib.ldm_predict_start(self._h, B, _ptr(xt), _ptr(t32), _ptr(out), _ptr(lg), self._stream()))
        return (out, lg) if want_logits else out

    def q_posterior(self, log_x_start: torch.Tensor, xt: torch.Tensor, t: torch.Tensor) -> torch.Tensor:
        """constrained.py:135-206 / vanilla.py:112-151: log_x_start (B,S,C) any log p(x0), xt (B,S) ids, t (B,) -> (B,S,C)"""
        B = xt.shape[0]
        lx = log_x_start.to(self.device, torch.float32).contiguous()
        assert lx.shape == (B, self.vocab.S, self.vocab.C)
        xt = xt.to(self.device, torch.int64).contiguous()
        t32 = self._t32(t, B)
        out = torch.empty_like(lx)
        _lib.check(self.lib.ldm_q_posterior(self._h, B, _ptr(lx), _ptr(xt), _ptr(t32), _ptr(out), self._stream()))
        return out

    def q_pred(self, log_x_start: torch.Tensor, t: torch.Tensor) -> torch.Tensor:
        """constrained.py:112-133 on the full vocabulary: log_x_start (B,S,C), t (B,) in [-1, T) -> log q(x_t|x_0) (B,S,C)"""
        B = log_x_start.shape[0]
        lx = log_x_start.to(self.device, torch.float32).contiguous()
        t32 = self._t32(t, B, lo=-1)
        out = torch.empty_like(lx)
        _lib.check(self.lib.ldm_q_pred(self._h, B, _ptr(lx), _ptr(t32), _ptr(out), self._stream()))
        return out

    def q_pred_one_timestep(self, log_x_t: torch.Tensor, t: torch.Tensor) -> torch.Tensor:
        """constrained.py:92-110 on the full vocabulary: log_x_t (B,S,C), t (B,) in [0, T) -> log q(x_t|x_{t-1}) (B,S,C)"""
        B = log_x_t.shape[0]
        lx = log_x_t.to(self.device, torch.float32).contiguous()
        t32 = self._t32(t, B)
        out = torch.empty_like(lx)
        _lib.check(self.lib.ldm_q_pred_one_timestep(self._h, B, _ptr(lx), _ptr(t32), _ptr(out), self._stream()))
        return out

    def gumbel_argmax(self, logits: torch.Tensor, seed: int = 0, b_global0: int = 0) -> torch.Tensor:
        """log_sample_categorical, train_sampling "gumbel" (constrained.py:208-221): logits (B,S,C) -> ids (B,S)"""
        B = logits.shape[0]
        lg = logits.to(self.device, torch.float32).contiguous()
        assert lg.shape == (B, self.vocab.S, self.vocab.C)
        out = torch.empty(B, self.vocab.S, dtype=torch.int64, device=self.device)
        _lib.check(self.lib.ldm_gumbel_argmax(self._h, B, _ptr(lg), C.c_uint64(seed), C.c_int64(b_global0), _ptr(out), self._stream()))
        return out

    def vb_terms(self, x0: torch.Tensor, xt: torch.Tensor, t: torch.Tensor, mask_weight=(1.0, 1.0), want_aux: bool = True,
                 want_log_model_prob: bool = False, want_recon_ids: bool = False) -> Dict[str, torch.Tensor]:
        """the per-layout loss terms of `forward` (constrained.py:262-333) after x_t has been drawn; tensors on the GPU"""
        B = x0.shape[0]
        x0 = x0.to(self.device, torch.int64).contiguous()
        xt = xt.to(self.device, torch.int64).contiguous()
        t32 = self._t32(t, B)
        f = lambda: torch.empty(B, device=self.device)
        kl, nll, aux = f(), f(), (f() if want_aux else None)
        lmp = torch.empty(B, self.vocab.S, self.vocab.C, device=self.device) if want_log_model_prob else None
        r0 = torch.empty_like(x0) if want_recon_ids else None
        r1 = torch.empty_like(x0) if want_recon_ids else None
        _lib.check(self.lib.ldm_vb_terms(self._h, B, _ptr(x0), _ptr(xt), _ptr(t32), C.c_float(mask_weight[0]), C.c_float(mask_weight[1]),
                                         _ptr(kl), _ptr(nll), _ptr(aux), _ptr(lmp), _ptr(r0), _ptr(r1), self._stream()))
        return {"kl": kl, "decoder_nll": nll, "kl_aux": aux, "log_model_prob": lmp, "x0_recon": r0, "xt_1_recon": r1}

    def decode(self, ids: torch.Tensor, centers: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
        """ids (B,S) on the GPU -> {"bbox" (B,E,4) f32, "label" (B,E) i64, "mask" (B,E) bool} on the GPU"""
        B = ids.shape[0]
        ids = ids.to(self.device, torch.int64).contiguous()
        E = self.vocab.n_elem
        bbox = torch.empty(B, E, 4, dtype=torch.float32, device=self.device)
        label = torch.empty(B, E, dtype=torch.int64, device=self.device)
        mask = torch.empty(B, E, dtype=torch.uint8, device=self.device)
        c = None if centers is None else centers.to(self.device, torch.float32).contiguous()
        _lib.check(self.lib.ldm_decode(self._h, B, _ptr(ids), _ptr(c), _ptr(bbox), _ptr(label), _ptr(mask), self._stream()))
        return {"bbox": bbox, "label": label, "mask": mask.bool()}

    COND_TYPES = {"c": 0, "cwh": 1, "refinement": 2, "gt": 3}

    def cond_from_layouts(self, label: torch.Tensor, bbox: torch.Tensor, mask: torch.Tensor, cond_type: str = "c",
                          centers: Optional[torch.Tensor] = None, refine: Optional[dict] = None) -> dict:
        """get_cond (helpers/task.py:27-151) on the device for cond_type c / cwh / refinement / gt: dense layouts
        (label (B,E) i64, bbox (B,E,4) f32 xywh, mask (B,E) bool with the valid elements first) -> the `cond` dict `sample()`
        takes, tensors on the GPU.  For "refinement" `bbox` must already carry the N(0, 0.1) perturbation of task.py:127;
        `refine` (refine_mode / refine_offset_ratio / refine_lambda, hydra_configs.py:39-41) builds the band table."""
        if cond_type not in self.COND_TYPES:
            raise NotImplementedError(f"cond_type {cond_type!r} is built on the host (task.py)")
        B, E = label.shape
        assert E == self.vocab.n_elem and bbox.shape == (B, E, 4) and mask.shape == (B, E)
        lab = label.to(self.device, torch.int64).contiguous()
        bb = bbox.to(self.device, torch.float32).contiguous()
        em = mask.to(self.device).to(torch.uint8).contiguous()
        c = None if centers is None else centers.to(self.device, torch.float32).contiguous()
        S = self.vocab.S
        seq = torch.empty(B, S, dtype=torch.int64, device=self.device)
        m = torch.empty(B, S, dtype=torch.uint8, device=self.device)
        so = torch.empty(B, S, dtype=torch.int64, device=self.device) if cond_type == "refinement" else None
        _lib.check(self.lib.ldm_make_cond(self._h, B, self.COND_TYPES[cond_type], _ptr(lab), _ptr(bb), _ptr(em), _ptr(c), _ptr(seq),
                                          _ptr(m), _ptr(so), self._stream()))
        cond = {"seq": seq, "mask": m.bool(), "type": cond_type}
        if cond_type != "gt":
            cond["num_element"] = em.sum(dim=1, dtype=torch.int64)
        if cond_type == "refinement":
            r = dict(refine_mode="uniform", refine_offset_ratio=0.1, refine_lambda=3.0)
            r.update(refine or {})
            cen = linear_centers(self.vocab.n_bins) if centers is None else [row.numpy() for row in centers.detach().cpu().double()]
            cond["seq_orig"] = so
            cond["refine_table"] = refinement_table(self.vocab, cen, r["refine_mode"], r["refine_offset_ratio"], r["refine_lambda"]).to(self.device)
        return cond

    def sample_host(self, B: int, plan, sampling, cond: Optional[dict] = None, seed: int = 0, b_global0: int = 0,
                    ids_init: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None):
        """host-buffer entry (ldm_sample_host): cond / ids_init are CPU tensors (ideally pinned); returns (ids CPU, h2d, d2h)."""
        n = len(plan)
        tm = (C.c_int32 * n)(*[p[0] for p in plan])
        tp = (C.c_int32 * n)(*[p[1] for p in plan])
        if out is None:
            out = torch.empty(B, self.vocab.S, dtype=torch.int64).pin_memory()
        s = sampling if isinstance(sampling, _lib.LdmSampling) else sampling_struct(sampling)
        seq = mask = so = tb = None
        pad_disable = 0
        if cond:
            seq = cond["seq"].to(torch.int64).contiguous()
            mask = cond["mask"].to(torch.uint8).contiguous() if cond.get("mask") is not None else None
            if cond.get("seq_orig") is not None and cond.get("refine_table") is not None:
                so = cond["seq_orig"].to(torch.int64).contiguous()
                tb = cond["refine_table"].to(torch.float32).contiguous()
                assert tb.shape == (self.vocab.C, self.vocab.C), f"refine_table must be (C, C), got {tuple(tb.shape)}"
            pad_disable = 1 if cond.get("type") in ("c", "cwh", "refinement", "relation") else 0
            for t in (seq, mask, so, tb):
                assert t is None or not t.is_cuda
        if ids_init is not None:
            ids_init = ids_init.to(torch.int64).contiguous()
        h2d, d2h = C.c_int64(0), C.c_int64(0)
        rc = self.lib.ldm_sample_host(self._h, B, n, tm, tp, _ptr(seq), _ptr(mask), _ptr(so), _ptr(tb), pad_disable, C.byref(s),
                                      C.c_uint64(seed), C.c_int64(b_global0), _ptr(ids_init), _ptr(out), self._stream(),
                                      C.byref(h2d), C.byref(d2h))
        _lib.check(rc)
        return out, h2d.value, d2h.value
