"""BERT layer library, split into the reference's allocatable units.

Registered names and calling conventions are those of scaelum/model/bert_layers.py:171-395:

    BertEmbeddings(config)            (input_ids, token_type_ids, attention_mask) -> (emb, ext_mask)
    BertLayer_Head(config)            (hidden, mask)            -> (attn_out, mask)
    BertLayer_Body(config)            (attn_out, mask)          -> (inter, attn_out, mask)
    BertLayer_Tail(config)            (inter, attn_out, mask)   -> (hidden, mask)
    BertPooler(config)                (hidden, mask)            -> pooled
    BertTailForClassification(hidden_dropout_prob, hidden_size, num_classes)   pooled -> logits
    BertTailForMaskedLM(config)       (hidden, mask)            -> logits [B, S, vocab]
    BertTailForMaskedLM(config, max_predictions=P)
                                      (hidden, mask, labels)    -> (logits [B*P, vocab], slot_labels [B*P])
    BertTailForMaskedLM(config, tie_word_embeddings=True)
                                      as above; decoder weight = the word-embedding table
                                      (``tie_word_embeddings``, set up by the stage / engine)
    BertTailForQuestionAnswering(config)
                                      (hidden, mask)            -> logits [B, 2, S] (start, end)

Parameter names match the reference (``attention.self.query.weight`` ...), so layer-indexed
checkpoints interchange.  Every layer has two execution paths behind the same class:

* ``torch``  - fp32 eager PyTorch with exactly the reference's math.  It is the numerics oracle for
  the kernel tests and the CPU path (BASELINE config 1 runs on it over gloo).
* ``native`` - bf16 sm_90a kernels (wgmma GEMMs / attention, fused LayerNorm, in-kernel
  dropout) through ``skycomputing_b200.ops.functions``.  Consecutive Head/Body/Tail layers of one
  block are executed as ONE autograd node (``BertSpan``); the stage runtime builds those spans.

``set_backend("auto" | "torch" | "native")`` selects the path; ``auto`` means native whenever the
input lives on a CUDA device and the extension is built.
"""
from __future__ import annotations

import math
from typing import List

import torch
import torch.nn as nn
import torch.nn.functional as F

from ..registry import LAYER
from .bert import BertConfig

_BACKEND = "auto"


def set_backend(name: str) -> None:
    global _BACKEND
    assert name in ("auto", "torch", "native"), name
    _BACKEND = name


def get_backend() -> str:
    return _BACKEND


def _nat():
    from ..ops import native

    return native


def native_active(device: torch.device) -> bool:
    """Do the sm_90a kernels run on ``device`` (CUDA, backend not "torch", extension built)?"""
    return device.type == "cuda" and _BACKEND != "torch" and _nat().available()


def _native_enabled(t: torch.Tensor) -> bool:
    if native_active(t.device):
        return True
    if _BACKEND == "torch" or not t.is_cuda:
        if _BACKEND == "native" and not t.is_cuda:
            raise RuntimeError("backend 'native' requires CUDA tensors")
        return False
    if _BACKEND == "native":
        _nat().ext()  # raises with the build hint
    raise RuntimeError(
        "CUDA tensors reached a skycomputing_b200 layer but the sm_90a extension is not built; "
        "run __graft_entry__.build() (or set_backend('torch') to use the eager oracle on purpose)"
    )


# device-resident dropout RNG shared by all native layers of this process
_RNG = {}
_RNG_STREAM_COUNTER = [0]


def default_rng(device: torch.device):
    key = (device.type, device.index)
    if key not in _RNG:
        _RNG[key] = _nat().RngState(torch.initial_seed(), device=device)
    return _RNG[key]


def advance_rng(inc: int = 1) -> None:
    """Advance the dropout step counter (one launch per device; CUDA-graph capturable)."""
    for r in _RNG.values():
        r.advance(inc)


def _next_rng_base() -> int:
    _RNG_STREAM_COUNTER[0] += 8
    return _RNG_STREAM_COUNTER[0]


# --------------------------------------------------------------------------------------------
# activations (reference: bert_layers.py:21-57)
# --------------------------------------------------------------------------------------------
def gelu(x):
    return x * 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0)))


def bias_gelu(bias, y):
    return gelu(bias + y)


def bias_gelu_training(bias, y):
    """Training-time variant of bias_gelu (scaelum bert_layers.py:36-38): bias add + library erf-GELU."""
    return torch.nn.functional.gelu(bias + y)


def bias_tanh(bias, y):
    return torch.tanh(bias + y)


def swish(x):
    return x * torch.sigmoid(x)


ACT2FN = {"gelu": gelu, "bias_gelu": bias_gelu, "bias_tanh": bias_tanh, "relu": F.relu,
          "swish": swish, "tanh": torch.tanh}


class LinearActivation(nn.Module):
    """Linear whose bias is folded into the activation (reference: bert_layers.py:60-108)."""

    def __init__(self, in_features: int, out_features: int, act="gelu", bias: bool = True):
        super().__init__()
        self.in_features, self.out_features = in_features, out_features
        self.act_name = act if isinstance(act, str) else None
        # reference semantics (bert_layers.py:73-84): with a bias, "gelu" means "bias_gelu" - the
        # bias is handed to the activation instead of to F.linear; "bias_*" names are accepted
        # directly.  `act_fn` is the plain activation, `biased_act_fn(bias, y)` the folded form.
        self.biased_act_fn = None
        if isinstance(act, str):
            base = act[5:] if act.startswith("bias_") else act
            folded = "bias_" + base
            if folded in ACT2FN:
                self.biased_act_fn = ACT2FN[folded]
            if base in ACT2FN:
                self.act_fn = ACT2FN[base]
            elif self.biased_act_fn is not None:
                fn = self.biased_act_fn
                self.act_fn = lambda y: fn(torch.zeros((), dtype=y.dtype, device=y.device), y)
            else:
                raise KeyError(f"unknown activation {act!r}; known: {sorted(ACT2FN)}")
        else:
            self.act_fn = act
        self.weight = nn.Parameter(torch.empty(out_features, in_features))
        if bias:
            self.bias = nn.Parameter(torch.empty(out_features))
        else:
            self.register_parameter("bias", None)
        self.reset_parameters()

    def reset_parameters(self) -> None:
        nn.init.kaiming_uniform_(self.weight, a=math.sqrt(5))
        if self.bias is not None:
            bound = 1 / math.sqrt(self.in_features)
            nn.init.uniform_(self.bias, -bound, bound)

    def forward(self, x):
        y = F.linear(x, self.weight, None)
        if self.bias is None:
            return self.act_fn(y)
        if self.biased_act_fn is not None:
            return self.biased_act_fn(self.bias, y)
        return self.act_fn(y + self.bias)

    def extra_repr(self) -> str:
        return f"in_features={self.in_features}, out_features={self.out_features}, bias={self.bias is not None}"


class BertLayerNorm(nn.Module):
    """TF-style LayerNorm (epsilon inside the sqrt), reference: bert_layers.py:143-168."""

    def __init__(self, hidden_size: int, eps: float = 1e-12):
        super().__init__()
        self.shape = torch.Size((hidden_size,))
        self.eps = eps
        self.weight = nn.Parameter(torch.ones(hidden_size))
        self.bias = nn.Parameter(torch.zeros(hidden_size))

    def forward(self, x):
        u = x.mean(-1, keepdim=True)
        s = (x - u).pow(2).mean(-1, keepdim=True)
        x = (x - u) / torch.sqrt(s + self.eps)
        return self.weight * x + self.bias


BertNonFusedLayerNorm = BertLayerNorm


# --------------------------------------------------------------------------------------------
# embeddings
# --------------------------------------------------------------------------------------------
@LAYER.register_module
class BertEmbeddings(nn.Module):
    def __init__(self, config):
        super().__init__()
        config = BertConfig.from_dict(config) if isinstance(config, dict) else config
        self.word_embeddings = nn.Embedding(config.vocab_size, config.hidden_size)
        self.position_embeddings = nn.Embedding(config.max_position_embeddings, config.hidden_size)
        self.token_type_embeddings = nn.Embedding(config.type_vocab_size, config.hidden_size)
        self.LayerNorm = BertLayerNorm(config.hidden_size, eps=1e-12)
        self.dropout = nn.Dropout(config.hidden_dropout_prob)
        # the tied BertTailForMaskedLM of the same stage that decodes with this table (not a
        # submodule), see tie_decoder_to_embeddings
        object.__setattr__(self, "_tied_head", None)
        self._native = None

    def _native_params(self):
        from ..ops.functions import EmbeddingParams

        if self._native is None:
            object.__setattr__(self, "_native", EmbeddingParams(self))
            self._native.rng_base = _next_rng_base()
        self._native.rng = default_rng(self.word_embeddings.weight.device)
        return self._native

    def forward(self, input_ids, token_type_ids, attention_mask):
        if _native_enabled(input_ids) and self.word_embeddings.weight.shape[1] % 4 == 0:
            from ..ops.functions import EmbeddingsFn

            ep = self._native_params()
            return EmbeddingsFn.apply(ep, self.training, None, 0, input_ids, token_type_ids,
                                      attention_mask, *ep.all_params())
        ext = attention_mask.unsqueeze(1).unsqueeze(2).to(dtype=self.word_embeddings.weight.dtype)
        ext = (1.0 - ext) * -10000.0
        seq_length = input_ids.size(1)
        position_ids = torch.arange(seq_length, dtype=torch.long, device=input_ids.device)
        position_ids = position_ids.unsqueeze(0).expand_as(input_ids)
        emb = (self.word_embeddings(input_ids) + self.position_embeddings(position_ids)
               + self.token_type_embeddings(token_type_ids))
        emb = self.dropout(self.LayerNorm(emb))
        return emb, ext


# --------------------------------------------------------------------------------------------
# transformer block pieces (oracle sub-modules keep the reference's attribute names)
# --------------------------------------------------------------------------------------------
class BertSelfAttention(nn.Module):
    def __init__(self, config):
        super().__init__()
        if config.hidden_size % config.num_attention_heads != 0:
            raise ValueError(
                "The hidden size (%d) is not a multiple of the number of attention heads (%d)"
                % (config.hidden_size, config.num_attention_heads))
        self.num_attention_heads = config.num_attention_heads
        self.attention_head_size = config.hidden_size // config.num_attention_heads
        self.all_head_size = self.num_attention_heads * self.attention_head_size
        self.query = nn.Linear(config.hidden_size, self.all_head_size)
        self.key = nn.Linear(config.hidden_size, self.all_head_size)
        self.value = nn.Linear(config.hidden_size, self.all_head_size)
        self.dropout = nn.Dropout(config.attention_probs_dropout_prob)

    def _split(self, x):
        return x.reshape(x.size()[:-1] + (self.num_attention_heads, self.attention_head_size)
                         ).permute(0, 2, 1, 3)

    def forward(self, hidden_states, attention_mask):
        q = self._split(self.query(hidden_states))
        k = self._split(self.key(hidden_states))
        v = self._split(self.value(hidden_states))
        scores = torch.matmul(q, k.transpose(-1, -2)) / math.sqrt(self.attention_head_size)
        scores = scores + attention_mask
        probs = self.dropout(F.softmax(scores, dim=-1))
        ctx = torch.matmul(probs, v).permute(0, 2, 1, 3).contiguous()
        return ctx.reshape(ctx.size()[:-2] + (self.all_head_size,))


class BertSelfOutput(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.dense = nn.Linear(config.hidden_size, config.hidden_size)
        self.LayerNorm = BertLayerNorm(config.hidden_size, eps=1e-12)
        self.dropout = nn.Dropout(config.hidden_dropout_prob)

    def forward(self, hidden_states, input_tensor):
        return self.LayerNorm(self.dropout(self.dense(hidden_states)) + input_tensor)


class BertAttention(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.self = BertSelfAttention(config)
        self.output = BertSelfOutput(config)

    def forward(self, input_tensor, attention_mask):
        return self.output(self.self(input_tensor, attention_mask), input_tensor)


class BertIntermediate(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.dense_act = LinearActivation(config.hidden_size, config.intermediate_size,
                                          act=config.hidden_act)

    def forward(self, hidden_states):
        return self.dense_act(hidden_states)


class BertOutput(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.dense = nn.Linear(config.intermediate_size, config.hidden_size)
        self.LayerNorm = BertLayerNorm(config.hidden_size, eps=1e-12)
        self.dropout = nn.Dropout(config.hidden_dropout_prob)

    def forward(self, hidden_states, input_tensor):
        return self.LayerNorm(self.dropout(self.dense(hidden_states)) + input_tensor)


class BertSpan:
    """A contiguous run of Head/Body/Tail layers of ONE block executed as a single autograd node.

    Not an ``nn.Module`` (the layers stay owned by the stage's Sequential); the stage runtime
    creates spans from adjacent layers, a lone layer creates a one-element span for itself.
    """

    def __init__(self, head=None, body=None, tail=None):
        from ..ops.functions import SpanParams

        self.head, self.body, self.tail = head, body, tail
        self.params = SpanParams(head, body, tail)
        self.params.rng_base = _next_rng_base()
        self.in_channel = None   # parallel.p2p.FusedChannel feeding this span (stage input)
        self.out_channel = None  # channel this span's LayerNorm writes into (stage output)
        self.microbatch = 0

    @property
    def layers(self) -> List[nn.Module]:
        return [m for m in (self.head, self.body, self.tail) if m is not None]

    def supports(self, hidden: torch.Tensor) -> bool:
        H = hidden.shape[-1]
        if hidden.dim() != 3 or H % 8 != 0:
            return False
        if self.head is not None:
            # wgmma attention: head size 64, any sequence length that is a multiple of 8 (S = 128
            # single-tile kernels, everything else flash-style tiles of 128 keys)
            sa = self.head.attention.self
            if sa.attention_head_size != 64 or hidden.shape[1] <= 0 or hidden.shape[1] % 8 != 0:
                return False
        if self.body is not None and self.body.intermediate.dense_act.act_name not in ("gelu", "bias_gelu"):
            return False
        return True

    def __call__(self, *inputs):
        from ..ops.functions import BertSpanFn

        sp = self.params
        first = (self.head or self.body or self.tail)
        training = first.training
        dev = inputs[0].device
        sp.rng = default_rng(dev)
        inputs = tuple(t.to(torch.bfloat16) if (torch.is_tensor(t) and t.is_floating_point()
                                                and t.dim() == 3 and t.dtype != torch.bfloat16)
                       else t for t in inputs)
        if not training and not torch.is_grad_enabled():
            # inference: nothing is kept for a backward pass that cannot happen
            out = BertSpanFn.infer(sp, self.in_channel, self.out_channel, self.microbatch, inputs)
        else:
            out = BertSpanFn.apply(sp, training, self.in_channel, self.out_channel,
                                   self.microbatch, len(inputs), *inputs, *sp.all_params())
        mask = inputs[-1]
        if self.tail is not None:
            return out, mask
        if self.body is not None:
            if self.head is not None:
                inter, attn_out = out
            else:
                inter, attn_out = out, inputs[0]
            return inter, attn_out, mask
        return out, mask


def _lone_span(layer, **kw) -> BertSpan:
    span = layer.__dict__.get("_lone_span")
    if span is None:
        span = BertSpan(**kw)
        object.__setattr__(layer, "_lone_span", span)
    return span


@LAYER.register_module
class BertLayer_Head(nn.Module):
    def __init__(self, config):
        super().__init__()
        config = BertConfig.from_dict(config) if isinstance(config, dict) else config
        self.attention = BertAttention(config)

    def forward(self, hidden_states, attention_mask):
        if _native_enabled(hidden_states):
            span = _lone_span(self, head=self)
            if span.supports(hidden_states):
                return span(hidden_states, attention_mask)
        hidden_states = hidden_states.float()
        return self.attention(hidden_states, attention_mask), attention_mask


@LAYER.register_module
class BertLayer_Body(nn.Module):
    def __init__(self, config):
        super().__init__()
        config = BertConfig.from_dict(config) if isinstance(config, dict) else config
        self.intermediate = BertIntermediate(config)

    def forward(self, attention_output, attention_mask):
        if _native_enabled(attention_output):
            span = _lone_span(self, body=self)
            if span.supports(attention_output):
                return span(attention_output, attention_mask)
        attention_output = attention_output.float()
        return self.intermediate(attention_output), attention_output, attention_mask


@LAYER.register_module
class BertLayer_Tail(nn.Module):
    def __init__(self, config):
        super().__init__()
        config = BertConfig.from_dict(config) if isinstance(config, dict) else config
        self.output = BertOutput(config)

    def forward(self, intermediate_output, attention_output, attention_mask):
        if _native_enabled(attention_output):
            span = _lone_span(self, tail=self)
            if span.supports(attention_output):
                return span(intermediate_output, attention_output, attention_mask)
        out = self.output(intermediate_output.float(), attention_output.float())
        return out, attention_mask


@LAYER.register_module
class BertPooler(nn.Module):
    def __init__(self, config):
        super().__init__()
        config = BertConfig.from_dict(config) if isinstance(config, dict) else config
        self.dense_act = LinearActivation(config.hidden_size, config.hidden_size, act="tanh")
        self._native = None

    def _native_params(self):
        from ..ops.functions import SmallLinearParams

        if self._native is None:
            object.__setattr__(self, "_native", SmallLinearParams(
                self.dense_act.weight, self.dense_act.bias, act_tanh=True, first_token=True))
        return self._native

    def forward(self, hidden_states, attention_mask):
        if _native_enabled(hidden_states) and hidden_states.dim() == 3:
            from ..ops.functions import PoolerFn, SmallLinearFn

            lp = self._native_params()
            B, _S, H = hidden_states.shape
            if B % 8 == 0 and H % 8 == 0 and hidden_states.dtype == torch.bfloat16:
                return PoolerFn.apply(lp, hidden_states, *lp.all_params())  # wgmma GEMM path
            return SmallLinearFn.apply(lp, self.training, hidden_states, *lp.all_params())
        first_token_tensor = hidden_states[:, 0].float()
        return self.dense_act(first_token_tensor)


@LAYER.register_module
class BertTailForClassification(nn.Module):
    objective = "classification"   # how Runner.evaluate scores it: runner.metrics.OBJECTIVES

    def __init__(self, hidden_dropout_prob, hidden_size, num_classes):
        super().__init__()
        self.num_classes = num_classes
        self.dropout = nn.Dropout(hidden_dropout_prob)
        self.classifier = nn.Linear(hidden_size, num_classes)
        self._native = None

    def _native_params(self):
        from ..ops.functions import SmallLinearParams

        if self._native is None:
            object.__setattr__(self, "_native", SmallLinearParams(
                self.classifier.weight, self.classifier.bias, act_tanh=False,
                first_token=False, p_drop=float(self.dropout.p)))
            self._native.rng_base = _next_rng_base()
        return self._native

    def forward(self, logits):
        if _native_enabled(logits) and logits.dim() == 2:
            from ..ops.functions import SmallLinearFn

            lp = self._native_params()
            lp.rng = default_rng(logits.device)
            return SmallLinearFn.apply(lp, self.training, logits, *lp.all_params()).view(
                -1, self.num_classes)
        logits = self.classifier(self.dropout(logits.float()))
        return logits.view(-1, self.num_classes)


class BertPredictionHeadTransform(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.dense_act = LinearActivation(config.hidden_size, config.hidden_size, act=config.hidden_act)
        self.LayerNorm = BertLayerNorm(config.hidden_size, eps=1e-12)

    def forward(self, hidden_states):
        return self.LayerNorm(self.dense_act(hidden_states))


@LAYER.register_module
class BertTailForMaskedLM(nn.Module):
    """Masked-language-model head (HF ``BertLMPredictionHead``): dense + activation + LayerNorm,
    then a decoder to vocabulary logits.  ``(hidden [B,S,H], mask) -> logits [B,S,V]``; every
    token is decoded unless ``max_predictions`` is set (below).

    By default the decoder weight is a parameter of its own.  ``tie_word_embeddings=True`` ties
    it to the word-embedding table of the model's first layer, as BERT, HF
    ``BertForPreTraining`` and NVIDIA's recipe do (the decoder bias stays the head's own).  The head
    still constructs its own ``decoder.weight``, so it can be built and benchmarked alone; whoever
    assembles the model sets up the tie: a stage that holds both layers replaces the head's
    Parameter by the table's (``tie_decoder_to_embeddings``, one Parameter and, on the GPU, one
    parameter bank), and a pipeline whose head sits on another rank keeps a bit-identical replica
    there (``parallel.engine_base``: both copies step on the summed gradient).  The native
    path needs ``H % 8 == 0`` and ``V % 8 == 0`` (GEMM output widths), which is why BERT configs
    pad the vocabulary (30522 -> 30528); other shapes run the eager path.

    ``max_predictions=P`` makes the head label-consuming (``consumes_labels``): in a pipeline the
    stage passes the micro-batch's labels ``[B, S]`` and the head decodes only the labelled
    positions, at most P per sequence, returning ``(logits [B*P, V], slot_labels [B*P])`` (slot
    layout and overflow rule: ``ops.functions.mlm_slots_ref``).  It is a data contract: choose
    ``P >= round(mask_prob * (S - 2))``, the labelled count of the BERT masking (19 at S = 128
    and 15 %).  Without labels the head decodes every position, as the dense head does; the
    parameters are the same in both modes, so checkpoints interchange.

    P is at most ``max_position_embeddings`` and at most ``MAX_PREDICTIONS_LIMIT`` (the
    ``mlm_gather`` kernel keeps a sequence's slot map in shared memory), on every backend, so that
    a config that constructs also runs on the GPU.  ``ignore_index`` must be the loss's: the head
    marks empty slots with it, and a loss with another value counts them as invalid labels."""

    MAX_PREDICTIONS_LIMIT = 8192   # csrc/kernels/api.h: kMlmMaxPredictions
    objective = "masked_lm"

    def __init__(self, config, max_predictions=None, ignore_index: int = -100,
                 tie_word_embeddings: bool = False):
        super().__init__()
        config = BertConfig.from_dict(config) if isinstance(config, dict) else config
        bound = min(config.max_position_embeddings, self.MAX_PREDICTIONS_LIMIT)
        if max_predictions is not None and (
                isinstance(max_predictions, bool) or not isinstance(max_predictions, int)
                or not 1 <= max_predictions <= bound):
            raise ValueError("max_predictions must be None or an int in [1, {}] (the sequence "
                             "length bound, at most {} slots per sequence), got {!r}".format(
                                 bound, self.MAX_PREDICTIONS_LIMIT, max_predictions))
        self.max_predictions = max_predictions
        self.ignore_index = int(ignore_index)
        self.consumes_labels = max_predictions is not None
        self.transform = BertPredictionHeadTransform(config)
        self.decoder = nn.Linear(config.hidden_size, config.vocab_size)
        self.tie_word_embeddings = bool(tie_word_embeddings)
        if self.tie_word_embeddings:
            # a replica (head on another stage) takes the table's weight-decay decisions
            self.decoder.weight.tied_name = TIED_TABLE_NAME
        # the BertEmbeddings of the same stage whose table this head's decoder shares (not a
        # submodule: the table stays the embeddings' parameter); None for an untied head or a replica
        object.__setattr__(self, "_tied_embeddings", None)
        self._native = None

    @property
    def is_replica(self) -> bool:
        """Tied, but the table lives on another stage: ``decoder.weight`` is a copy of it."""
        return self.tie_word_embeddings and self._tied_embeddings is None

    def load_state_dict(self, state_dict, strict: bool = True, assign: bool = False):
        """A head tied to the table of its own stage does not load ``decoder.weight``: the shared
        Parameter holds the embeddings' entry of the same file (loaded first, layer 0), which wins.
        A file whose decoder weight differs (saved from an untied model) is reported once."""
        key = "decoder.weight"
        if self._tied_embeddings is None or key not in state_dict:
            return super().load_state_dict(state_dict, strict=strict, assign=assign)
        if not torch.equal(state_dict[key].to(self.decoder.weight.device, torch.float32),
                           self.decoder.weight.detach().float()):
            _warn_decoder_unused()
        rest = {k: v for k, v in state_dict.items() if k != key}
        res = super().load_state_dict(rest, strict=False, assign=assign)
        missing = [k for k in res.missing_keys if k != key]
        if strict and (missing or res.unexpected_keys):
            raise RuntimeError("Error(s) in loading state_dict for {}: missing keys {}, unexpected "
                               "keys {}".format(type(self).__name__, missing, res.unexpected_keys))
        return res

    def _native_params(self):
        from ..ops.functions import MaskedLMHeadParams

        if self._native is None:
            object.__setattr__(self, "_native", MaskedLMHeadParams(self))
        return self._native

    def _supports(self, hidden: torch.Tensor) -> bool:
        H, V = self.decoder.in_features, self.decoder.out_features
        return (hidden.dim() == 3 and H % 8 == 0 and V % 8 == 0 and H <= 2048
                and self.transform.dense_act.act_name in ("gelu", "bias_gelu"))

    def forward(self, hidden_states, attention_mask=None, labels=None):
        if labels is not None and not self.consumes_labels:
            raise ValueError("labels reach a BertTailForMaskedLM without max_predictions")
        if labels is not None:
            labels = labels.to(torch.int64).reshape(hidden_states.shape[0], -1)
        if _native_enabled(hidden_states) and self._supports(hidden_states):
            from ..ops.functions import MaskedLMHeadFn

            hp = self._native_params()
            x = hidden_states.to(torch.bfloat16)
            if not self.training and not torch.is_grad_enabled():
                return MaskedLMHeadFn.infer(hp, x, labels)
            return MaskedLMHeadFn.apply(hp, x, labels, *hp.all_params())
        if labels is None:
            return self.decoder(self.transform(hidden_states.float()))
        from ..ops.functions import mlm_slots_ref

        row, _, slot_labels = mlm_slots_ref(labels, self.max_predictions, self.ignore_index,
                                            self.decoder.out_features)
        flat = hidden_states.float().reshape(-1, hidden_states.shape[-1])
        x = torch.where((row >= 0).unsqueeze(1), flat.index_select(0, row.clamp(min=0)), 0.0)
        return self.decoder(self.transform(x)), slot_labels


@LAYER.register_module
class BertTailForPreTraining(BertTailForMaskedLM):
    """Masked-LM and next-sentence-prediction heads (HF ``BertPreTrainingHeads`` plus the pooler
    it reads): the ``BertTailForMaskedLM`` head, a ``pooler`` (dense + tanh on the [CLS] row) and
    ``seq_relationship`` (``Linear(H, 2)``, no dropout).  ``(hidden, mask) -> (mlm_logits
    [B, S, V], nsp_logits [B, 2])``.

    Labels are one int64 tensor ``[B, S + 1]`` (``ops.functions.split_pretraining_labels``).
    With ``max_predictions=P`` the head takes them and returns ``(mlm_logits [B*P, V],
    slot_labels [B*P], nsp_logits)``; without labels it returns the dense outputs.  Decoder tie,
    sparse decoding, argument checks and the last-layer rule are the masked-LM head's.  The
    native path also needs the batch to be a multiple of 8 (the pooler's weight-gradient GEMM
    runs over it); other shapes run the eager path."""

    # the outputs the loss differentiates: masked-LM logits first, next-sentence logits last
    logit_outputs = (0, -1)
    objective = "pretraining"

    def __init__(self, config, max_predictions=None, ignore_index: int = -100,
                 tie_word_embeddings: bool = False):
        super().__init__(config, max_predictions, ignore_index, tie_word_embeddings)
        config = BertConfig.from_dict(config) if isinstance(config, dict) else config
        self.pooler = BertPooler(config.__dict__)
        self.seq_relationship = nn.Linear(config.hidden_size, 2)

    def _native_params(self):
        from ..ops.functions import PreTrainingHeadParams

        if self._native is None:
            object.__setattr__(self, "_native", PreTrainingHeadParams(self))
        return self._native

    def _supports(self, hidden: torch.Tensor) -> bool:
        return super()._supports(hidden) and hidden.shape[0] % 8 == 0

    def forward(self, hidden_states, attention_mask=None, labels=None):
        from ..ops.functions import split_pretraining_labels

        if labels is not None and not self.consumes_labels:
            raise ValueError("labels reach a BertTailForPreTraining without max_predictions")
        if labels is not None:
            labels = labels.to(torch.int64).reshape(hidden_states.shape[0], -1)
        if _native_enabled(hidden_states) and self._supports(hidden_states):
            from ..ops.functions import PreTrainingHeadFn

            hp = self._native_params()
            x = hidden_states.to(torch.bfloat16)
            if not self.training and not torch.is_grad_enabled():
                return PreTrainingHeadFn.infer(hp, x, labels)
            return PreTrainingHeadFn.apply(hp, x, labels, *hp.all_params())
        if native_active(hidden_states.device) and super()._supports(hidden_states):
            _warn_eager_batch(hidden_states.shape[0])
        nsp = self.seq_relationship(self.pooler.dense_act(hidden_states[:, 0].float()))
        mlm = super().forward(hidden_states, attention_mask,
                              None if labels is None else split_pretraining_labels(labels)[0])
        return (*mlm, nsp) if isinstance(mlm, tuple) else (mlm, nsp)


@LAYER.register_module
class BertTailForQuestionAnswering(nn.Module):
    """Extractive question-answering head (HF ``BertForQuestionAnswering``): ``qa_outputs =
    Linear(H, 2)`` on every token, after the last encoder block (no pooler).  ``(hidden [B,S,H],
    mask) -> logits [B, 2, S]`` in fp32, row 0 the start and row 1 the end logits (each softmax
    row contiguous); as in HF the logits are not masked.

    The native path (``QuestionAnsweringFn``) runs on a bf16 3-D input with ``H % 8 == 0``, any B
    and S; other inputs, the CPU and ``backend="torch"`` run the eager fp32 path.  Labels are the
    ``[B, 5]`` layout of ``ops.functions.split_span_labels``; the head is evaluated by span
    (``objective``), and ``max_answer_length`` bounds the predicted answer in tokens."""

    # logit shapes alone would not tell this head from a token-level one
    objective = "span"

    def __init__(self, config, max_answer_length: int = 30):
        super().__init__()
        config = BertConfig.from_dict(config) if isinstance(config, dict) else config
        if isinstance(max_answer_length, bool) or not isinstance(max_answer_length, int) \
                or max_answer_length < 1:
            raise ValueError("max_answer_length must be a positive int, got {!r}".format(
                max_answer_length))
        self.max_answer_length = max_answer_length
        self.qa_outputs = nn.Linear(config.hidden_size, 2)
        self._native = None

    def _native_params(self):
        from ..ops.functions import QuestionAnsweringParams

        if self._native is None:
            object.__setattr__(self, "_native", QuestionAnsweringParams(self))
        return self._native

    def forward(self, hidden_states, attention_mask=None):
        if (_native_enabled(hidden_states) and hidden_states.dim() == 3
                and hidden_states.dtype == torch.bfloat16 and hidden_states.shape[-1] % 8 == 0):
            from ..ops.functions import QuestionAnsweringFn

            hp = self._native_params()
            if not self.training and not torch.is_grad_enabled():
                return QuestionAnsweringFn.infer(hp, hidden_states)
            return QuestionAnsweringFn.apply(hp, hidden_states, *hp.all_params())
        return self.qa_outputs(hidden_states.float()).transpose(1, 2).contiguous()


TIED_TABLE_NAME = "word_embeddings.weight"
_WARNED_EAGER_BATCH = [False]


def _warn_eager_batch(batch: int) -> None:
    """Once per process: a pretraining head on the GPU whose batch is not a multiple of 8 runs
    the eager fp32 path (the whole vocabulary-wide decoder in fp32)."""
    if _WARNED_EAGER_BATCH[0]:
        return
    _WARNED_EAGER_BATCH[0] = True
    import warnings

    warnings.warn("BertTailForPreTraining: a batch of {} sequences is not a multiple of 8, so the "
                  "head runs its eager fp32 path, which is much slower than the native one; use "
                  "micro-batches of a multiple of 8 sequences".format(batch))


def _warn_decoder_unused() -> None:
    import warnings

    warnings.warn("the checkpoint's decoder.weight differs from its word_embeddings.weight (saved "
                  "from an untied model): the tied decoder uses the word-embedding entry, the "
                  "decoder entry is not used")


def check_tied_layers(first, head) -> None:
    """ValueError unless ``head`` (a tied BertTailForMaskedLM, or its layer config dict) can share
    the table of ``first``, the model's first layer (module or config dict)."""
    def shape(layer, kind):
        if isinstance(layer, dict):
            if layer.get("layer_type") != kind:
                return None
            c = layer.get("config")
            c = BertConfig.from_dict(c) if isinstance(c, dict) else c
            return (int(c.vocab_size), int(c.hidden_size))
        if kind == "BertEmbeddings":
            return tuple(layer.word_embeddings.weight.shape) if isinstance(layer, BertEmbeddings) else None
        return (layer.decoder.out_features, layer.decoder.in_features)

    table = shape(first, "BertEmbeddings")
    if table is None:
        got = first.get("layer_type") if isinstance(first, dict) else type(first).__name__
        raise ValueError("tie_word_embeddings=True needs a BertEmbeddings as the model's first "
                         "layer, got {}".format(got))
    dec = shape(head, head.get("layer_type") if isinstance(head, dict) else "BertTailForMaskedLM")
    if dec != table:
        raise ValueError("tie_word_embeddings=True: the decoder is [vocab, hidden] = {} but the "
                         "word-embedding table is {}".format(list(dec), list(table)))


def is_tied_head_cfg(layer_cfg: dict) -> bool:
    return (layer_cfg.get("layer_type") in MASKED_LM_HEADS
            and bool(layer_cfg.get("tie_word_embeddings", False)))


# registered names of the heads with a masked-LM decoder (BertTailForMaskedLM and its subclass)
MASKED_LM_HEADS = ("BertTailForMaskedLM", "BertTailForPreTraining")


def tie_decoder_to_embeddings(layers) -> bool:
    """Same-stage tie: when ``layers`` (one stage, in order) start with a BertEmbeddings and hold a
    ``tie_word_embeddings`` head, the head's ``decoder.weight`` becomes the table's Parameter (the
    same object; the decoder bias stays the head's).  A tied head without the embeddings in front
    is left alone: it is a replica of a table on another stage.  Returns True when it tied."""
    layers = list(layers)
    heads = [l for l in layers if isinstance(l, BertTailForMaskedLM) and l.tie_word_embeddings]
    if not heads or not isinstance(layers[0], BertEmbeddings):
        return False
    emb = layers[0]
    for head in heads:
        check_tied_layers(emb, head)
        if head._tied_embeddings is emb:
            continue
        table = emb.word_embeddings.weight
        table.tied_name = TIED_TABLE_NAME
        head.decoder.weight = table
        object.__setattr__(head, "_tied_embeddings", emb)
        object.__setattr__(head, "_native", None)
        object.__setattr__(emb, "_tied_head", head)
        if emb._native is not None:
            emb._native.tie_word_bank()
    return True


def native_param_banks(module: nn.Module):
    """All ParamBanks of `module`'s native layers (created eagerly; used by the fused optimizer).

    For a stage (``ModuleWrapper``) the banks of its fused spans are returned, so that the
    optimizer and the forward pass share the same flat fp32 / bf16 buffers.
    """
    banks = []
    covered = set()
    # every stage runtime (ModuleWrapper) below `module` - `module` itself, or the chunks of a
    # looped pipeline held in a ModuleList - contributes the banks of ITS fused spans: building
    # lone per-layer spans for them instead would give the optimizer different flat buffers than
    # the ones the forward pass reads
    for m in module.modules():
        spans = getattr(m, "spans", None)
        if callable(spans):
            for span in spans():
                banks.extend(span.params.banks)
                covered.update(id(l) for l in span.layers)
    for m in module.modules():
        if id(m) in covered:
            continue
        if isinstance(m, BertEmbeddings):
            banks.extend(m._native_params().banks)
        elif isinstance(m, BertPooler):
            banks.extend(m._native_params().banks)
        elif isinstance(m, BertTailForClassification):
            banks.extend(m._native_params().banks)
        elif isinstance(m, BertTailForMaskedLM):
            banks.extend(m._native_params().banks)
        elif isinstance(m, BertTailForQuestionAnswering):
            banks.extend(m._native_params().banks)
        elif isinstance(m, BertLayer_Head):
            banks.extend(_lone_span(m, head=m).params.banks)
        elif isinstance(m, BertLayer_Body):
            banks.extend(_lone_span(m, body=m).params.banks)
        elif isinstance(m, BertLayer_Tail):
            banks.extend(_lone_span(m, tail=m).params.banks)
    # a tied decoder's bank IS the embeddings' table bank: listed once, where the embeddings are
    return list({id(b): b for b in banks}.values())
