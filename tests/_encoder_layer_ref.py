"""fp64 autograd reference of one BERT encoder layer (Head + Body + Tail) with explicit dropout.

The keep factors are passed in (kept-and-scaled values, 0 where dropped), so the reference applies
exactly the masks the native kernels drew: ``k_attn`` [B, heads, S, S] on the attention
probabilities, ``k_o`` [B*S, H] on the attention-output dense and ``k_ffn`` [B*S, H] on the FFN2
dense.  With all-ones factors it is the eval-mode layer of ``skycomputing_b200.models``.
"""
import math

import torch

PARAM_NAMES = ("wqkv", "bqkv", "wo", "bo", "g1", "b1n", "w1", "b1", "w2", "b2", "g2", "b2n")


def layer_params(head, body, tail, dtype=torch.float64, weights=None):
    """The layer's parameters in the order of ``PARAM_NAMES`` (Q | K | V fused as the native span
    fuses them), as leaf tensors of ``dtype`` that require grad.  ``weights`` optionally replaces
    the four weight matrices (e.g. by the bf16 compute copies the kernels multiply with)."""
    att = head.attention
    sa, so = att.self, att.output
    out = tail.output
    lin = body.intermediate.dense_act
    p = dict(wqkv=torch.cat([sa.query.weight, sa.key.weight, sa.value.weight]),
             bqkv=torch.cat([sa.query.bias, sa.key.bias, sa.value.bias]),
             wo=so.dense.weight, bo=so.dense.bias, g1=so.LayerNorm.weight, b1n=so.LayerNorm.bias,
             w1=lin.weight, b1=lin.bias, w2=out.dense.weight, b2=out.dense.bias,
             g2=out.LayerNorm.weight, b2n=out.LayerNorm.bias)
    if weights is not None:
        p.update(weights)
    return {k: p[k].detach().to(dtype).clone().requires_grad_(True) for k in PARAM_NAMES}


def layer_norm(z, g, b, eps):
    mu = z.mean(-1, keepdim=True)
    var = ((z - mu) ** 2).mean(-1, keepdim=True)
    return (z - mu) / torch.sqrt(var + eps) * g + b


def gelu(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def layer_ref(x, mask, p, heads, k_attn=None, k_o=None, k_ffn=None, eps=1e-12):
    """x [B, S, H], mask additive [B, S]; returns the layer output [B, S, H] and a dict of the
    intermediates (qkv, ctx, z1, a, h1, inter, z2) as [B*S, ...] tensors."""
    B, S, H = x.shape
    d = H // heads
    xf = x.reshape(B * S, H)
    qkv = xf @ p["wqkv"].t() + p["bqkv"]
    q, k, v = qkv.view(B, S, 3, heads, d).permute(2, 0, 3, 1, 4)
    s = q @ k.transpose(-1, -2) / math.sqrt(d) + mask[:, None, None, :]
    prob = torch.softmax(s, dim=-1)
    if k_attn is not None:
        prob = prob * k_attn
    ctx = (prob @ v).permute(0, 2, 1, 3).reshape(B * S, H)
    t1 = ctx @ p["wo"].t() + p["bo"]
    z1 = (t1 * k_o if k_o is not None else t1) + xf
    a = layer_norm(z1, p["g1"], p["b1n"], eps)
    h1 = a @ p["w1"].t() + p["b1"]
    inter = gelu(h1)
    t2 = inter @ p["w2"].t() + p["b2"]
    z2 = (t2 * k_ffn if k_ffn is not None else t2) + a
    y = layer_norm(z2, p["g2"], p["b2n"], eps)
    return y.view(B, S, H), dict(qkv=qkv, ctx=ctx, z1=z1, a=a, h1=h1, inter=inter, z2=z2)
