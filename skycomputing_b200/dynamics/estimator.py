"""Speed / FLOPs / memory estimation (capability parity with scaelum/dynamics/estimator.py:13-152).

* ``benchmark_speed``: forward loop under ``no_grad``; the result is the sum of the stage's own
  DEVICE-timed forward durations (ModuleWrapper.forward_time), optional warm-up iterations (the
  reference has none and times with wall clock + cuda.synchronize).
* ``benchmark_model``: (output, FLOPs, memory MiB).  FLOPs come from
  ``torch.utils.flop_counter.FlopCounterMode`` on the eager path (replaces the unavailable
  ``pthflops``); memory is the reference's torchsummary-style formula
  ``(2 x outputs + param_scale x params + inputs) x bytes_per_element``.
"""
from __future__ import annotations

from collections import OrderedDict

import numpy as np
import torch
import torch.nn as nn
from torch.utils.flop_counter import FlopCounterMode


class Estimator:
    @staticmethod
    def benchmark_speed(model, data, device, iterations, dtype=None, warmup: int = 0):
        data = Estimator._convert_to_tuple(data)
        if dtype:
            data = Estimator._convert_dtype(data, dtype)
        data = Estimator._move_to_device(data, device)
        model = model.to(device)
        with torch.no_grad():
            for _ in range(warmup):
                model(*data)
            if warmup and hasattr(model, "reset_timers"):
                model.reset_timers()
            for _ in range(iterations):
                model(*data)
        return float(sum(model.forward_time))

    @staticmethod
    def _convert_dtype(data, dtype):
        assert isinstance(dtype, str)
        dt = getattr(torch, dtype)
        return [d.to(dt) if torch.is_tensor(d) and d.is_floating_point() else d for d in data]

    @staticmethod
    def _move_to_device(data, device):
        return [d.to(device) if torch.is_tensor(d) else d for d in data]

    @staticmethod
    def _convert_to_tuple(data):
        return data if isinstance(data, (list, tuple)) else (data,)

    @staticmethod
    def benchmark_model(model, data, device, dtype=None, param_scale=2):
        from ..models.bert_layers import get_backend, set_backend

        data = Estimator._convert_to_tuple(data)
        if dtype:
            data = Estimator._convert_dtype(data, dtype)
        data = Estimator._move_to_device(data, device)
        model = model.to(device)
        prev = get_backend()
        set_backend("torch")  # FLOP counting / hooks need the eager oracle path
        try:
            with torch.no_grad():
                output = model(*data)
            flops = Estimator._calc_flops(model, data)
            mem_usage = Estimator._calc_memory_usage(model, data, param_scale)
        finally:
            set_backend(prev)
        return output, flops, mem_usage

    @staticmethod
    def analytic_layer_cost(layer_cfg: dict, data, param_scale: int = 2):
        """Closed-form (flops, mem_MiB, output_meta) for the registered BERT layers, or None.

        FLOPs follow FlopCounterMode's convention (2 per multiply-accumulate of every matmul);
        memory follows the reference formula (2 x forward-hook outputs + param_scale x params +
        inputs, 4 bytes each).  tests/test_core_cpu.py checks both against the measured path.
        """
        lt = layer_cfg.get("layer_type")
        data = data if isinstance(data, (list, tuple)) else (data,)
        c = layer_cfg.get("config")
        mb = 1024.0 ** 2
        f32 = torch.float32
        if lt == "BertTailForClassification":
            B, H = data[0].shape
            C = layer_cfg["num_classes"]
            params = H * C + C
            outs = B * H + 2 * B * C      # dropout, linear, the layer module itself
            mem = (2 * outs + param_scale * params + B * H) * 4 / mb
            return 2.0 * B * H * C, mem, [((B, C), f32)]
        if c is None or lt not in ("BertEmbeddings", "BertLayer_Head", "BertLayer_Body",
                                   "BertLayer_Tail", "BertPooler", "BertTailForMaskedLM",
                                   "BertTailForPreTraining", "BertTailForQuestionAnswering"):
            return None
        if lt == "BertTailForQuestionAnswering":
            # qa_outputs = Linear(H, 2) on every token: fp32 logits [B, 2, S]
            B, S, _ = data[0].shape
            H = c["hidden_size"]
            params = 2 * H + 2
            outs = 2 * B * S * 2          # the linear, the layer module itself
            mem = (2 * outs + param_scale * params + B * S * H + B * S) * 4 / mb
            return 2.0 * B * S * H * 2, mem, [((B, 2, S), f32)]
        if lt == "BertTailForPreTraining":
            # the masked-LM head, plus the pooler on the [CLS] rows and the 2-way classifier
            flops, mem, outs = Estimator.analytic_layer_cost(dict(layer_cfg, layer_type="BertTailForMaskedLM"),
                                                data, param_scale)
            B, H = data[0].shape[0], c["hidden_size"]
            params = H * H + H + 2 * H + 2
            mem += (2 * 2 * B * (H + 2) + param_scale * params) * 4 / mb
            return flops + 2.0 * B * H * (H + 2), mem, outs + [((B, 2), f32)]
        H, I, A = c["hidden_size"], c["intermediate_size"], c["num_attention_heads"]
        if lt == "BertTailForMaskedLM":
            B, S, _ = data[0].shape
            V = c["vocab_size"]
            params = H * H + H + 2 * H + V * H + V
            P = layer_cfg.get("max_predictions")
            if P is None:
                # transform dense + decoder; every token is decoded, so the decoder dominates
                # (about 2.5 encoder blocks at BERT-large with a 30K vocabulary)
                outs = 3 * B * S * H + 2 * B * S * V   # dense_act, LayerNorm, transform; decoder, layer
                mem = (2 * outs + param_scale * params + B * S * H + B * S) * 4 / mb
                return 2.0 * B * S * H * (H + V), mem, [((B, S, V), f32)]
            # sparse head: B*P slots are decoded (a fraction of a block at P = 20, S = 128); the
            # labels [B, S] are one more input and the slot labels one more output
            R = B * P
            outs = 3 * R * H + 2 * R * V + R
            mem = (2 * outs + param_scale * params + B * S * H + 2 * B * S) * 4 / mb
            return 2.0 * R * H * (H + V), mem, [((R, V), f32), ((R,), torch.int64)]
        if lt == "BertEmbeddings":
            B, S = data[0].shape
            params = (c["vocab_size"] + c["max_position_embeddings"] + c["type_vocab_size"]) * H + 2 * H
            outs = 6 * B * S * H + B * S  # 3 lookups, LayerNorm, dropout, the module's own tuple
            mem = (2 * outs + param_scale * params + 3 * B * S) * 4 / mb
            return 0.0, mem, [((B, S, H), f32), ((B, 1, 1, S), f32)]
        if lt == "BertPooler":
            B, S, _ = data[0].shape
            params = H * H + H
            mem = (2 * 2 * B * H + param_scale * params + B * S * H + B * S) * 4 / mb
            return 2.0 * B * H * H, mem, [((B, H), f32)]
        if lt == "BertLayer_Head":
            B, S, _ = data[0].shape
            flops = 4 * 2.0 * B * S * H * H + 2 * 2.0 * B * S * S * H
            params = 4 * (H * H + H) + 2 * H
            outs = 10 * B * S * H + B * A * S * S + B * S   # every sub-module output is hooked
            mem = (2 * outs + param_scale * params + B * S * H + B * S) * 4 / mb
            return flops, mem, [((B, S, H), f32), ((B, 1, 1, S), f32)]
        if lt == "BertLayer_Body":
            B, S, _ = data[0].shape
            params = H * I + I
            outs = 3 * B * S * I + B * S * H + B * S
            mem = (2 * outs + param_scale * params + B * S * H + B * S) * 4 / mb
            return 2.0 * B * S * H * I, mem, [((B, S, I), f32), ((B, S, H), f32), ((B, 1, 1, S), f32)]
        # BertLayer_Tail
        B, S, _ = data[1].shape
        params = I * H + H + 2 * H
        outs = 5 * B * S * H + B * S
        mem = (2 * outs + param_scale * params + B * S * I + B * S * H + B * S) * 4 / mb
        return 2.0 * B * S * I * H, mem, [((B, S, H), f32), ((B, 1, 1, S), f32)]

    @staticmethod
    def _calc_flops(model, data) -> float:
        data = tuple(d.detach() if torch.is_tensor(d) else d for d in data)
        with FlopCounterMode(display=False) as fc:
            model(*data)
        return float(fc.get_total_flops())

    @staticmethod
    def _calc_memory_usage(model, data, param_scale, bytes_per_element: float = 4.0) -> float:
        assert isinstance(data, (list, tuple))
        summary = OrderedDict()
        hooks = []

        def register_hook(module):
            def hook(module, inputs, output):
                key = "%s-%i" % (module.__class__.__name__, len(summary) + 1)
                outs = output if isinstance(output, (list, tuple)) else [output]
                shapes = [list(o.size()) for o in outs if torch.is_tensor(o)]
                params = 0
                if hasattr(module, "weight") and hasattr(module.weight, "size"):
                    params += int(np.prod(list(module.weight.size())))
                if hasattr(module, "bias") and hasattr(module.bias, "size"):
                    params += int(np.prod(list(module.bias.size())))
                summary[key] = dict(output_shape=shapes, nb_params=params)

            if not isinstance(module, (nn.Sequential, nn.ModuleList)):
                hooks.append(module.register_forward_hook(hook))

        model.apply(register_hook)
        try:
            with torch.no_grad():
                model(*data)
        finally:
            for h in hooks:
                h.remove()
        total_params = sum(v["nb_params"] for v in summary.values())
        total_output = sum(float(np.prod(s)) for v in summary.values() for s in v["output_shape"])
        mb = 1024.0 ** 2
        total_input_size = sum(float(np.prod(d.size())) * bytes_per_element / mb
                               for d in data if torch.is_tensor(d))
        total_output_size = 2.0 * total_output * bytes_per_element / mb  # x2 for gradients
        total_params_size = param_scale * total_params * bytes_per_element / mb
        return float(total_params_size + total_output_size + total_input_size)
