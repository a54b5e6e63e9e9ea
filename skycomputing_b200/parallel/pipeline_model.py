"""``RpcModel`` facade: the distributed model a Runner drives.

API parity with scaelum/model/rpc_model.py:16-63 and rpc_module.py:12-99 (``RpcModel(worker_
manager)``, ``.model`` list of per-stage modules in pipeline order, ``.forward``,
``.parameter_rrefs()``; ``BaseModule / LocalModule / RemoteModule`` with ``load_weights /
get_state_dict / parameter_rrefs``) on an SPMD substrate: every rank constructs the same
``RpcModel`` from the (identical) allocation result, materialises only ITS stage as a
``LocalModule`` and keeps parameter-less ``RemoteModule`` handles for the others.  There is no
per-iteration Python RPC: "remote" data moves through parallel/p2p.py or parallel/comm.py.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import torch
import torch.nn as nn

from .. import utils
from ..builder import build_module_from_cfg


def _this_rank() -> int:
    import torch.distributed as dist

    return dist.get_rank() if dist.is_available() and dist.is_initialized() else 0


class BaseModule(nn.Module):
    def __init__(self, rank, model_cfg, sequential_wrapper_cfg, device_rank: Optional[int] = None,
                 layer_range: Optional[tuple] = None):
        super().__init__()
        self.rank = rank                      # pipeline position (reference: RPC destination)
        self.device_rank = device_rank        # process / GPU that owns the stage
        self.model_cfg = model_cfg
        self.sequential_wrapper_cfg = sequential_wrapper_cfg
        self.layer_range = layer_range
        self.module = self._build_module()

    def forward(self, *args, **kwargs):
        return self._forward(*args, **kwargs)

    def _forward(self, *args):
        raise NotImplementedError

    def _build_module(self):
        raise NotImplementedError

    def load_weights(self, state_dict: List[Dict]) -> None:
        raise NotImplementedError

    def get_state_dict(self) -> Optional[List[Dict]]:
        raise NotImplementedError

    def parameter_rrefs(self) -> List:
        raise NotImplementedError

    @property
    def is_local(self) -> bool:
        return isinstance(self, LocalModule)


class LocalModule(BaseModule):
    def _forward(self, *args):
        res = self.module(*args)
        return res if isinstance(res, (tuple, list)) else (res,)

    def _build_module(self):
        return build_module_from_cfg(rank=self.rank, model_cfg=self.model_cfg,
                                     module_wrapper_cfg=self.sequential_wrapper_cfg)

    def load_weights(self, state_dict: List[Dict]) -> None:
        utils.load_weights(self.module, state_dict)

    def get_state_dict(self) -> List[Dict]:
        return utils.get_state_dict(self.module)

    def parameter_rrefs(self) -> List:
        return list(self.module.parameters())


class RemoteModule(BaseModule):
    """Handle of a stage owned by another rank (no parameters live here)."""

    def _build_module(self):
        return None

    def _forward(self, *args):
        raise RuntimeError("a RemoteModule is executed by its owner rank; use RpcModel.forward / "
                           "train_step, which run the local stage and move data between ranks")

    def load_weights(self, state_dict: List[Dict]) -> None:
        return None  # the owner loads its own span (CheckpointHook is collective)

    def get_state_dict(self) -> Optional[List[Dict]]:
        return None

    def parameter_rrefs(self) -> List:
        return []


class RpcModel(nn.Module):
    def __init__(self, worker_manager, this_rank: Optional[int] = None):
        super().__init__()
        self.worker_manager = worker_manager
        self.this_rank = _this_rank() if this_rank is None else this_rank
        self.engine = None
        self.model = self._build_model()
        assert isinstance(self.model, nn.ModuleList), "model must be iterable"

    def _build_model(self) -> nn.ModuleList:
        """One module per (virtual) pipeline stage, in pipeline order.  Plain pipelines: stage k =
        worker k.  Looped pipelines (``worker.chunks`` with v > 1 spans): virtual stage k = chunk
        k // D of worker k % D, so a rank owns v LocalModules."""
        model = nn.ModuleList()
        pool = list(self.worker_manager.worker_pool)
        D = len(pool)
        single = D == 1
        v = max((len(w.chunks) for w in pool if getattr(w, "chunks", None)), default=1)
        self.virtual_stages = v if not single else 1
        if self.virtual_stages > 1:
            assert all(w.chunks is not None and len(w.chunks) == v for w in pool), \
                "every worker of a looped pipeline needs the same number of chunks"
        for k in range(D * self.virtual_stages):
            d, c = k % D, k // D
            worker = pool[d]
            dev = worker.device if worker.device is not None else d
            cfg = dict(worker.extra_config or {})
            if self.virtual_stages > 1:
                b, e = worker.chunks[c]
                off = sum(ce - cb for cb, ce in worker.chunks[:c])
                model_cfg, layer_range = worker.model_config[off:off + (e - b)], (b, e)
            else:
                model_cfg, layer_range = worker.model_config, worker.layer_range
            if single or dev == self.this_rank:
                if cfg.get("module_to_cuda") and torch.cuda.is_available():
                    # one process per GPU: the process' current device is the stage's device
                    cfg["cuda_device"] = torch.cuda.current_device()
                module = LocalModule(rank=worker.rank, model_cfg=model_cfg,
                                     sequential_wrapper_cfg=cfg, device_rank=dev,
                                     layer_range=layer_range)
                if module.module.consumes_labels and k != D * self.virtual_stages - 1:
                    # only the last stage receives the labels
                    raise ValueError("pipeline stage {} of {} ends with a layer that consumes "
                                     "labels; it must be the model's last layer".format(
                                         k, D * self.virtual_stages))
            else:
                module = RemoteModule(rank=worker.rank, model_cfg=model_cfg,
                                      sequential_wrapper_cfg=cfg, device_rank=dev,
                                      layer_range=layer_range)
            model.append(module)
        return model

    # ---- topology -------------------------------------------------------------------------
    @property
    def num_stages(self) -> int:
        return len(self.model)

    @property
    def stage_to_rank(self) -> List[int]:
        return [m.device_rank for m in self.model]

    @property
    def local_stage_index(self) -> int:
        for i, m in enumerate(self.model):
            if m.is_local:
                return i
        raise RuntimeError("this rank owns no pipeline stage")

    @property
    def local_stage_indices(self) -> List[int]:
        """All (virtual) stages this rank owns, in pipeline order (one for a plain pipeline)."""
        return [i for i, m in enumerate(self.model) if m.is_local]

    @property
    def local_stages(self) -> List:
        return [self.model[i].module for i in self.local_stage_indices]

    @property
    def optim_module(self) -> nn.Module:
        """What the optimizer of this rank must cover: the local stage, or all local chunks of a
        looped pipeline."""
        stages = self.local_stages
        return stages[0] if len(stages) == 1 else nn.ModuleList(stages)

    @property
    def local_module(self) -> LocalModule:
        return self.model[self.local_stage_index]

    @property
    def local_stage(self):
        """The ModuleWrapper this rank executes."""
        return self.local_module.module

    # ---- execution ------------------------------------------------------------------------
    def attach_engine(self, engine) -> None:
        self.engine = engine

    def forward(self, *args):
        if len(args) == 1 and isinstance(args[0], (list, tuple)):
            args = tuple(args[0])
        if self.num_stages == 1:
            return self.local_module(*args)[0]
        if self.engine is None:
            raise RuntimeError("RpcModel spans several ranks: attach a PipelineEngine (the Runner "
                               "does this) before calling forward")
        outs = self.engine.forward_only(args if self.local_stage_index == 0 else None)
        return None if outs is None else outs[0]

    def train_step(self, data, labels):
        return self.engine.train_step(data, labels)

    def parameter_rrefs(self) -> List:
        out = []
        for m in self.model:
            out.extend(m.parameter_rrefs())
        return out
