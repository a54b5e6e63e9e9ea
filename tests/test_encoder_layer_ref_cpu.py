"""The fp64 encoder-layer reference of the GPU tests, checked on the CPU against the model's own
torch layers: it must be the layer itself before it can judge the kernels."""
import numpy as np
import torch

from skycomputing_b200.models import BertConfig
from skycomputing_b200.models.bert_layers import (BertLayer_Body, BertLayer_Head,
                                                  BertLayer_Tail)
from skycomputing_b200.ops.dropout_ref import keep_mask
from tests import _fp64_bounds
from tests._encoder_layer_ref import PARAM_NAMES, layer_params, layer_ref

B, S, H, HEADS, I = 3, 72, 128, 2, 512


def _layer():
    torch.manual_seed(11)
    cfg = BertConfig(100, hidden_size=H, num_attention_heads=HEADS, intermediate_size=I).__dict__
    head, body, tail = BertLayer_Head(cfg), BertLayer_Body(cfg), BertLayer_Tail(cfg)
    with torch.no_grad():
        for ln in (head.attention.output.LayerNorm, tail.output.LayerNorm):
            ln.weight.add_(0.2 * torch.randn(H))
            ln.bias.add_(0.1 * torch.randn(H))
    return [m.double().eval() for m in (head, body, tail)]


def _inputs():
    x = torch.randn(B, S, H, dtype=torch.float64)
    mask = torch.zeros(B, S, dtype=torch.float64)
    mask[1, 50:] = -10000.0
    mask[2, :] = -10000.0                       # one fully padded sequence
    return x, mask


def _torch_layer(head, body, tail, x, mask):
    a = head.attention(x, mask[:, None, None, :])
    inter = body.intermediate(a)
    return tail.output(inter, a)


def _grads(y, dy, leaves):
    return torch.autograd.grad(y, leaves, dy)


def test_reference_matches_the_torch_layers():
    """All-ones keep factors: forward and every input / parameter gradient to 1e-10."""
    head, body, tail = _layer()
    x, mask = _inputs()
    x.requires_grad_(True)
    y_mod = _torch_layer(head, body, tail, x, mask)
    p = layer_params(head, body, tail)
    xr = x.detach().clone().requires_grad_(True)
    y_ref, _ = layer_ref(xr, mask, p, HEADS)
    torch.testing.assert_close(y_ref, y_mod, rtol=1e-10, atol=1e-10)

    dy = torch.randn_like(y_mod)
    mods = dict(wqkv=[m.weight for m in (head.attention.self.query, head.attention.self.key,
                                         head.attention.self.value)],
                bqkv=[m.bias for m in (head.attention.self.query, head.attention.self.key,
                                       head.attention.self.value)],
                wo=[head.attention.output.dense.weight], bo=[head.attention.output.dense.bias],
                g1=[head.attention.output.LayerNorm.weight],
                b1n=[head.attention.output.LayerNorm.bias],
                w1=[body.intermediate.dense_act.weight], b1=[body.intermediate.dense_act.bias],
                w2=[tail.output.dense.weight], b2=[tail.output.dense.bias],
                g2=[tail.output.LayerNorm.weight], b2n=[tail.output.LayerNorm.bias])
    mod_leaves = [x] + [t for n in PARAM_NAMES for t in mods[n]]
    g_mod = _grads(y_mod, dy, mod_leaves)
    g_ref = _grads(y_ref, dy, [xr] + [p[n] for n in PARAM_NAMES])
    torch.testing.assert_close(g_ref[0], g_mod[0], rtol=1e-10, atol=1e-10)
    i = 1
    for n, ref in zip(PARAM_NAMES, g_ref[1:]):
        k = len(mods[n])
        got = torch.cat(g_mod[i:i + k]) if k > 1 else g_mod[i]
        i += k
        torch.testing.assert_close(ref, got, rtol=1e-10, atol=1e-10, msg=n)


class _HandDropout(torch.nn.Module):
    """Dropout with a given boolean keep mask, scaled by 1 / (1 - p) of the fp32 p the kernels
    receive."""

    def __init__(self, keep, p):
        super().__init__()
        self.keep, self.scale = keep, 1.0 / (1.0 - float(np.float32(p)))

    def forward(self, t):
        return t * self.keep.reshape(t.shape) * self.scale


def test_keep_factors_through_the_reference_equal_hand_applied_masks(monkeypatch):
    """``_keep`` at p = 0.1 fed to the reference equals the torch layers with each dropout site
    replaced by its boolean mask from ``keep_mask``, applied by hand: the factors land on the
    right sites with the right scale."""
    monkeypatch.setattr(_fp64_bounds, "DEV", "cpu")
    head, body, tail = _layer()
    x, mask = _inputs()
    p, seed, step, base = 0.1, 1234, 5, 40
    rng = type("Rng", (), {"state": torch.tensor([seed, step], dtype=torch.int64)})()
    k_attn = _fp64_bounds._keep(rng, base + 1, (B, HEADS, S, S), p)
    k_o = _fp64_bounds._keep(rng, base + 2, (B * S, H), p)
    k_ffn = _fp64_bounds._keep(rng, base + 3, (B * S, H), p)
    assert 0.85 < float((k_o > 0).double().mean()) < 0.95
    y_ref, _ = layer_ref(x, mask, layer_params(head, body, tail), HEADS, k_attn, k_o, k_ffn)

    def hand(stream, shape):
        return _HandDropout(torch.from_numpy(keep_mask(seed, step, stream, shape, p)), p)

    head.attention.self.dropout = hand(base + 1, (B, HEADS, S, S))
    head.attention.output.dropout = hand(base + 2, (B * S, H))
    tail.output.dropout = hand(base + 3, (B * S, H))
    with torch.no_grad():
        y_mod = _torch_layer(head, body, tail, x, mask)
    torch.testing.assert_close(y_ref.detach(), y_mod, rtol=1e-10, atol=1e-10)
