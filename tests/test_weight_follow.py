"""CPU: when the engine behind a patched model reloads its weights (WeightFollower).  A stub stands in for the Engine and counts
the `load_weights` calls; the followed module is a small torch module under the reference's CategoricalTransformer key names.
The GPU side (what a reload computes) is tests/test_gpu_weight_reload.py."""
import pytest
import torch
from torch import nn

from layoutdm_b200 import Engine, FusedMaskAndReplaceDiffusion, Vocab
from layoutdm_b200.diffusion import WeightFollower

D, FF, LAYERS, T = 8, 16, 2, 4


class _Norm1(nn.Module):
    def __init__(self):
        super().__init__()
        self.emb = nn.Embedding(T, D)
        self.linear = nn.Linear(D, 2 * D)


class _Layer(nn.Module):
    def __init__(self):
        super().__init__()
        self.self_attn = nn.MultiheadAttention(D, 2, batch_first=True)
        self.linear1, self.linear2 = nn.Linear(D, FF), nn.Linear(FF, D)
        self.norm1, self.norm2 = _Norm1(), nn.LayerNorm(D)


class _PosEmb(nn.Module):
    def __init__(self, vocab):
        super().__init__()
        self.elem_emb = nn.Parameter(torch.rand(vocab.n_elem, D))
        self.attr_emb = nn.Parameter(torch.rand(vocab.n_attr, D))


class TinyTransformer(nn.Module):
    """the parameter names of the reference's CategoricalTransformer (nn_lib.py:137-237), tiny shapes"""

    def __init__(self, vocab):
        super().__init__()
        self.cat_emb = nn.Embedding(vocab.C, D)
        self.pos_emb = _PosEmb(vocab)
        self.backbone = nn.Module()
        self.backbone.layers = nn.ModuleList([_Layer() for _ in range(LAYERS)])
        self.head = nn.Sequential(nn.LayerNorm(D), nn.Linear(D, vocab.C))

    def forward(self, ids):
        h = self.cat_emb(ids)
        for layer in self.backbone.layers:
            h = h + layer.linear2(torch.relu(layer.linear1(h)))
        return self.head(h)


class StubEngine:
    """what WeightFollower and FusedMaskAndReplaceDiffusion need of an Engine; records every load"""

    def __init__(self, vocab):
        self.vocab, self.T, self.q_type = vocab, T, "constrained"
        self.device = torch.device("cpu")
        self.loads = []

    def load_weights(self, weights):
        self.loads.append({k: v.clone() for k, v in weights.items()})

    def step(self, ids, *args, **kwargs):
        return ids, torch.zeros(ids.shape[0], self.vocab.S, self.vocab.C), None


@pytest.fixture
def setup():
    torch.manual_seed(0)
    vocab = Vocab.for_dataset("rico25")
    module = TinyTransformer(vocab)
    eng = StubEngine(vocab)
    return vocab, module, eng, WeightFollower(module, eng)


def _train_step(module, vocab, opt):
    ids = torch.randint(0, vocab.C, (2, 6))
    module(ids).logsumexp(-1).mean().backward()
    opt.step()
    opt.zero_grad()


def test_unchanged_module_does_not_reload(setup):
    vocab, module, eng, f = setup
    assert not f.check() and not f.check()
    assert eng.loads == [] and f.reloads == 0


@pytest.mark.parametrize("fused", [False, True])
def test_optimizer_step_reloads_once(setup, fused):
    """a foreach AdamW step bumps the version counters; a fused one does not, and the step post-hook's dirty flag catches it"""
    vocab, module, eng, f = setup
    opt = torch.optim.AdamW(module.parameters(), lr=1e-2, fused=fused, foreach=None if fused else True)
    _train_step(module, vocab, opt)
    assert f.check()
    assert not f.check()
    assert f.reloads == 1 and len(eng.loads) == 1
    w = eng.loads[0]
    assert torch.equal(w["cat_emb"], module.cat_emb.weight.detach())
    assert torch.equal(w["linear1_w"][1], module.backbone.layers[1].linear1.weight.detach())
    _train_step(module, vocab, opt)                # every later step too
    assert f.check() and f.reloads == 2
    assert torch.equal(eng.loads[1]["head_w"], module.head[1].weight.detach())


def test_fused_step_leaves_versions_alone(setup):
    """why the dirty flag exists: with the hook's flag cleared, a fused step is invisible to the fingerprint"""
    vocab, module, eng, f = setup
    opt = torch.optim.AdamW(module.parameters(), lr=1e-2, fused=True)
    _train_step(module, vocab, opt)
    f.check()
    before = module.cat_emb.weight.detach().clone()
    _train_step(module, vocab, opt)
    assert not torch.equal(before, module.cat_emb.weight)
    assert f.dirty
    f.dirty = False
    assert not f.check()


def test_unrelated_optimizer_does_not_reload(setup):
    vocab, module, eng, f = setup
    other = nn.Linear(3, 3)
    opt = torch.optim.AdamW(other.parameters(), fused=True)
    other(torch.randn(2, 3)).sum().backward()
    opt.step()
    assert not f.check() and f.reloads == 0


def test_load_state_dict_reloads_once(setup):
    vocab, module, eng, f = setup
    torch.manual_seed(1)
    sd = TinyTransformer(vocab).state_dict()
    module.load_state_dict(sd)
    assert f.check() and not f.check()
    assert f.reloads == 1
    assert torch.equal(eng.loads[0]["norm1_emb"][0], sd["backbone.layers.0.norm1.emb.weight"])


def test_replaced_parameter_reloads_once(setup):
    vocab, module, eng, f = setup
    module.head[1].weight = nn.Parameter(torch.randn(vocab.C, D))
    assert f.check() and not f.check()
    assert f.reloads == 1
    assert torch.equal(eng.loads[0]["head_w"], module.head[1].weight.detach())


def test_data_write_needs_reload_weights(setup):
    """a write through .data is not detected (documented); reload_weights() repacks"""
    vocab, module, eng, _ = setup
    fused = FusedMaskAndReplaceDiffusion(eng)
    with pytest.raises(ValueError):
        fused.reload_weights()
    fused.follow(module)
    module.cat_emb.weight.data = module.cat_emb.weight.data + 1.0     # new storage, found by data_ptr ...
    fused.predict_logits(torch.zeros(1, vocab.S, dtype=torch.long), 3)
    assert fused.weight_reloads == 1
    module.cat_emb.weight.data.mul_(2.0)                                # ... an in-place write through .data is not
    fused.predict_logits(torch.zeros(1, vocab.S, dtype=torch.long), 3)
    assert fused.weight_reloads == 1
    fused.reload_weights()
    assert fused.weight_reloads == 2 and len(eng.loads) == 2
    assert torch.equal(eng.loads[-1]["cat_emb"], module.cat_emb.weight.detach())


def test_every_denoiser_call_checks(setup):
    """a denoiser call of the fused object runs the check first: one reload after a step, none on the next call"""
    vocab, module, eng, _ = setup
    fused = FusedMaskAndReplaceDiffusion(eng)
    fused.follow(module)
    opt = torch.optim.AdamW(module.parameters(), fused=True)
    ids = torch.zeros(1, vocab.S, dtype=torch.long)
    fused.predict_logits(ids, 3)
    assert fused.weight_reloads == 0
    _train_step(module, vocab, opt)
    fused.predict_logits(ids, 3)
    fused.predict_logits(ids, 3)
    assert fused.weight_reloads == 1


def test_pack_state_dict_device_argument(setup):
    """pack_state_dict(device=...) gives the same arrays as the host packing"""
    vocab, module, eng, _ = setup
    sd = module.state_dict()
    a, b = Engine.pack_state_dict(sd, vocab), Engine.pack_state_dict(sd, vocab, device="cpu")
    assert a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)
    assert a["in_proj_w"].shape == (LAYERS, 3 * D, D) and a["pos_table"].shape == (vocab.S, D)
