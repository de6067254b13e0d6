"""CPU: denoiser blocks with the reference Block's other settings (transformer_utils.py:103-210): timestep_type None /
adalayernorm / adainnorm / adalayernorm_abs / adainnorm_abs, activation relu / gelu / gelu2.

The oracle's block_forward equals the live reference's logits for all 15 configurations and reproduces the fixtures the
unmodified reference recorded with them (tests/golden/blocks) token for token.  The host side: the norm1 arrays
Engine.pack_state_dict fills give, through the AdaLN formula the kernels apply, the reference's own norm1 output; the
refusals (*_mlp, norm1 keys that contradict the timestep_type, an unknown type or activation); the settings read from a live
model; random_state_dict's keys for each type."""
import functools

import pytest
import torch
import torch.nn.functional as F

import block_refs as BR
from oracle import layoutdm_oracle as O
from oracle import ref_harness as rh

needs_ref = pytest.mark.skipif(not rh.reference_available(), reason="reference not available")
IDS = [BR.config_id(*c) for c in BR.CONFIGS]


@functools.lru_cache(maxsize=1)
def _ids_and_t():
    g = torch.Generator().manual_seed(0)
    return torch.randint(0, O.RICO25.C, (3, O.RICO25.S), generator=g), torch.tensor([0, 41, 99])


@needs_ref
@pytest.mark.parametrize("tt,act", BR.CONFIGS, ids=IDS)
def test_oracle_equals_live_reference(tt, act):
    """block_forward against the reference's own transformer, at per-layout timesteps"""
    _oracle_vs_reference(tt, act, None)


@needs_ref
def test_oracle_equals_live_reference_diffusion_step():
    """diffusion_step = 200 != num_timesteps: what the sinusoidal embedding divides by and the Embedding's row count"""
    _oracle_vs_reference("adainnorm_abs", "gelu", 200)
    _oracle_vs_reference("adalayernorm", "relu", 200)


def _oracle_vs_reference(tt, act, diffusion_step):
    v, spec = O.RICO25, O.ModelSpec()
    sd = BR.block_weights(v, spec, seed=1, scale=2.0, timestep_type=tt, diffusion_step=diffusion_step)
    model, _ = BR.build_reference(T=spec.T, state_dict=sd, timestep_type=tt, activation=act, diffusion_step=diffusion_step)
    ids, t = _ids_and_t()
    with torch.no_grad():
        ref = model.model.module.transformer(ids, timestep=t)["logits"]
        got = BR.block_forward(sd, ids, t, v, spec, tt, act, diffusion_step)
    err = (ref - got).abs().max().item()
    assert err < 2e-5, f"{tt} {act} diffusion_step={diffusion_step}: max |d| {err:.2e}"


def test_block_fixtures_present():
    assert BR.NAMES == ["publaynet_none_gelu2_cwh", "rico25_L50_adainnorm_abs_gelu", "rico25_adainnorm_relu_uncond",
                        "rico25_adalayernorm_abs_gelu_c", "rico25_vanilla_adainnorm_gelu2"]


@pytest.mark.parametrize("name", BR.NAMES)
def test_oracle_reproduces_block_fixtures(name):
    """step-wise on the reference's own inputs: logits within 2e-5, log-probs within 2e-4, every drawn id equal"""
    fx = BR.BlockFixture(name)
    orc = fx.oracle()
    with torch.no_grad():
        for i, (tm, tp) in enumerate(fx.plan):
            lp, logits = orc.step_logprob(fx.x_in[i], tm, tp, fx.cond)
            if i in fx.trace_steps:
                assert (logits - fx.logits(i)).abs().max() < 2e-5 and (lp - fx.logp(i)).abs().max() < 2e-4
            x = O.draw(lp, fx.cfg, fx.noise(i))
            assert torch.equal(x, fx.x_out[i]), f"{name} step {i}: {(x != fx.x_out[i]).sum().item()} ids differ"


# ---- the packed norm1 arrays -------------------------------------------------------------------------------------------------

@needs_ref
@pytest.mark.parametrize("tt", BR.TIMESTEP_TYPES, ids=str)
@pytest.mark.parametrize("diffusion_step", [None, 200])
def test_packed_arrays_give_reference_norm1(tt, diffusion_step):
    """(scale, shift) = Linear(SiLU(norm1_emb[t])) of the packed arrays, applied as the kernels apply it (norm(x) (1 + scale) +
    shift, norm = LayerNorm or InstanceNorm1d), equals the reference's norm1(x, t) of every layer at every t"""
    from layoutdm_b200 import Engine, Vocab
    v, spec = O.RICO25, O.ModelSpec()
    sd = BR.block_weights(v, spec, seed=2, scale=2.0, timestep_type=tt, diffusion_step=diffusion_step)
    model, _ = BR.build_reference(T=spec.T, state_dict=sd, timestep_type=tt, diffusion_step=diffusion_step)
    w = Engine.pack_state_dict(sd, Vocab.for_dataset("rico25"), tt, diffusion_step, num_timesteps=spec.T)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(spec.T, v.S, spec.d, generator=g) * 2.0 + 0.5
    t = torch.arange(spec.T)
    d = spec.d
    for l, layer in enumerate(model.model.module.transformer.backbone.layers):
        tab = F.linear(F.silu(w["norm1_emb"][l]), w["norm1_w"][l], w["norm1_b"][l])           # adaln_table_kernel
        scale, shift = tab[:, None, :d], tab[:, None, d:]
        inorm = tt is not None and tt.startswith("adainnorm")
        xn = F.instance_norm(x.transpose(1, 2), eps=1e-5).transpose(1, 2) if inorm else F.layer_norm(x, (d,), eps=1e-5)
        got = xn * (1.0 + scale) + shift
        with torch.no_grad():
            ref = layer.norm1(x) if tt is None else layer.norm1(x, t)
        err = (got - ref).abs().max().item()
        assert err < 2e-5, f"{tt} layer {l}: max |d| {err:.2e}"


def test_none_type_packs_layernorm_affine_exactly():
    """timestep_type None: the table gives scale = w - 1 and shift = b, and 1 + (w - 1) is w again in fp32 for the weights a
    LayerNorm has (w in [0.5, 2]: w - 1 is exact, Sterbenz)"""
    from layoutdm_b200 import Engine, Vocab
    v, spec = O.RICO25, O.ModelSpec()
    sd = BR.block_weights(v, spec, seed=4, timestep_type=None)
    w = Engine.pack_state_dict(sd, Vocab.for_dataset("rico25"), None, num_timesteps=spec.T)
    assert not w["norm1_emb"].any() and not w["norm1_w"].any()
    for l in range(spec.layers):
        nw = sd[f"{O.PREFIX}backbone.layers.{l}.norm1.weight"]
        assert ((nw >= 0.5) & (nw <= 2.0)).all()
        assert torch.equal(1.0 + w["norm1_b"][l, : spec.d], nw)
        assert torch.equal(w["norm1_b"][l, spec.d:], sd[f"{O.PREFIX}backbone.layers.{l}.norm1.bias"])


# ---- refusals ----------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("tt", ["adalayernorm_mlp", "adainnorm_mlp"])
def test_mlp_types_are_refused_by_name(tt):
    from layoutdm_b200 import Engine, LayoutDMB200, Vocab
    from layoutdm_b200.synthetic import random_state_dict
    v = Vocab.for_dataset("rico25")
    sd = random_state_dict(v, layers=1)
    with pytest.raises(NotImplementedError, match=f"{tt}.*the reference's LayoutDM raises"):
        Engine.pack_state_dict(sd, v, tt)
    with pytest.raises(NotImplementedError, match=tt):
        Engine.from_state_dict(sd, v, timestep_type=tt)
    with pytest.raises(NotImplementedError, match=tt):
        LayoutDMB200.from_state_dict(sd, timestep_type=tt)


def test_unknown_type_and_activation_are_refused():
    from layoutdm_b200 import Engine, Vocab
    from layoutdm_b200.engine import block_settings
    from layoutdm_b200.synthetic import random_state_dict
    v = Vocab.for_dataset("rico25")
    sd = random_state_dict(v, layers=1)
    with pytest.raises(AssertionError, match="adagroupnorm"):
        Engine.pack_state_dict(sd, v, "adagroupnorm")
    with pytest.raises(RuntimeError, match="activation should be relu/gelu/gelu2, not swish"):
        Engine.from_state_dict(sd, v, activation="swish")
    assert block_settings("adalayernorm", "relu") == (0, 0)           # the default: zero-filled struct fields
    assert block_settings("adainnorm_abs", "gelu2") == (1, 2)


@pytest.mark.parametrize("given", BR.TIMESTEP_TYPES, ids=str)
@pytest.mark.parametrize("saved", BR.TIMESTEP_TYPES, ids=str)
def test_norm1_keys_must_match_the_timestep_type(given, saved):
    """a state_dict packs under its own kind of timestep_type (Embedding: adalayernorm / adainnorm, sinusoidal: *_abs, None);
    any other is a ValueError that names both"""
    from layoutdm_b200 import Engine, Vocab
    from layoutdm_b200.synthetic import random_state_dict
    v = Vocab.for_dataset("rico25")
    sd = random_state_dict(v, layers=1, timestep_type=saved)
    kind = lambda tt: "none" if tt is None else "abs" if tt.endswith("_abs") else "emb"
    if kind(given) == kind(saved):
        Engine.pack_state_dict(sd, v, given, num_timesteps=100)
    else:
        with pytest.raises(ValueError, match=rf"timestep_type={given!r}, but the state_dict's norm1 keys are those of"):
            Engine.pack_state_dict(sd, v, given, num_timesteps=100)


def test_default_pack_is_unchanged():
    """the default settings pack the arrays the earlier packing gave: the Embedding and Linear as they are"""
    from layoutdm_b200 import Engine, Vocab
    from layoutdm_b200.synthetic import random_state_dict
    v = Vocab.for_dataset("rico25")
    sd = random_state_dict(v, layers=2)
    w = Engine.pack_state_dict(sd, v)
    p = "model.module.transformer.backbone.layers."
    for l in range(2):
        assert torch.equal(w["norm1_emb"][l], sd[f"{p}{l}.norm1.emb.weight"])
        assert torch.equal(w["norm1_w"][l], sd[f"{p}{l}.norm1.linear.weight"])
        assert torch.equal(w["norm1_b"][l], sd[f"{p}{l}.norm1.linear.bias"])


@needs_ref
@pytest.mark.parametrize("tt", BR.TIMESTEP_TYPES, ids=str)
def test_random_state_dict_keys_load_into_the_reference(tt):
    from layoutdm_b200 import Vocab
    from layoutdm_b200.synthetic import random_state_dict
    sd = random_state_dict(Vocab.for_dataset("rico25"), timestep_type=tt)
    BR.build_reference(state_dict=sd, timestep_type=tt)          # asserts no missing / unexpected parameter


# ---- the settings of a live model --------------------------------------------------------------------------------------------

@needs_ref
@pytest.mark.parametrize("tt,act", BR.CONFIGS, ids=IDS)
def test_block_settings_read_from_a_live_model(tt, act):
    from layoutdm_b200.diffusion import block_settings_of
    model, _ = BR.build_reference(timestep_type=tt, activation=act, diffusion_step=120, num_layers=2)
    assert block_settings_of(model.model.module.transformer.backbone.layers) == (tt, act, 120)


@needs_ref
def test_block_settings_must_agree_and_be_known():
    from layoutdm_b200.diffusion import block_settings_of
    model, _ = BR.build_reference(timestep_type="adainnorm", activation="gelu", num_layers=2)
    layers = model.model.module.transformer.backbone.layers
    layers[1].activation = F.relu
    with pytest.raises(ValueError, match="disagree"):
        block_settings_of(layers)
    layers[1].activation = torch.tanh
    with pytest.raises(NotImplementedError, match="activation"):
        block_settings_of(layers)
