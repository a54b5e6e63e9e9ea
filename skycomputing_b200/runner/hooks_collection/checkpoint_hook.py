"""Layer-indexed checkpoint save / resume.

Capability parity with scaelum/runner/hooks_collection/checkpoint_hook.py:13-74 (same constructor:
``load_checkpoint_from, save_path, save_interval``; ``before_run`` loads, ``after_epoch`` saves
every ``save_interval`` epochs into ``<save_path>/epoch_{n}.pth``) with the reference's broken
paths fixed (SURVEY §2.7) and a sharded, collective implementation:

* checkpoints are keyed by GLOBAL layer index (``"<idx>.<param name>"``, the ModuleList format of
  the reference's ParameterServer), so they are independent of the allocation - resume under a
  different partition works;
* every rank contributes the state_dicts of ITS layers; rank 0 (the "central server") merges them
  through the ParameterServer and writes ONE reference-compatible file, plus (new) optimizer /
  iteration / RNG state in ``epoch_{n}.extra.rank{r}.pth`` shards;
* on load every rank reads the file and picks the layers of its own span.
"""
import os
import os.path as osp
from collections import OrderedDict

import torch

from ...registry import HOOKS
from ..hooks import Hook


def _dist():
    import torch.distributed as dist

    return dist if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1 else None


@HOOKS.register_module
class CheckpointHook(Hook):
    def __init__(self, load_checkpoint_from: str = None, save_path: str = None,
                 save_interval: int = None, save_optimizer: bool = True,
                 resume_training_state: bool = False, strict_optimizer: bool = False,
                 from_pretraining: bool = False):
        # from_pretraining=True initialises a model (a classification config, typically) from a
        # file saved by a pretraining run: weights only, see _from_pretraining_entry
        # resume_training_state=True also restores optimizer state and the epoch / iteration
        # counters from the per-rank ``.extra`` shards (same world size required); the default
        # restores weights only, like the reference.
        self._resume_training_state = resume_training_state
        self._strict_optimizer = strict_optimizer
        self._load_checkpoint_from = load_checkpoint_from
        self._save_interval = save_interval
        self._save_path = save_path
        self._save_optimizer = save_optimizer
        self._from_pretraining = from_pretraining
        if from_pretraining and resume_training_state:
            raise ValueError("from_pretraining loads weights only: it cannot resume the training "
                             "state of another run")

    # ------------------------------------------------------------------ load
    def before_run(self, runner):
        if not self._load_checkpoint_from:
            return
        sd = torch.load(self._load_checkpoint_from, map_location="cpu")
        per_layer = {}
        for key, val in sd.items():
            idx, name = key.split(".", 1)
            per_layer.setdefault(int(idx), OrderedDict())[name] = val
        self._tie_rule(runner, per_layer, self._load_checkpoint_from)
        dropped, kept_init = [], []
        for module in runner.model.model:
            if not module.is_local:
                continue
            n_layers = (max(per_layer) + 1) if per_layer else 0
            if runner.parameter_server is not None:
                n_layers = max(n_layers, len(runner.parameter_server))
            b, e = module.layer_range if module.layer_range is not None else (0, n_layers)
            layers = list(module.module.layers.children())
            sds = []
            for i in range(b, e):
                # layers without parameters / buffers (ReLU, Flatten, Dropout-only ...) have no keys
                # in the file: they load an empty state dict, as in the reference's ParameterServer
                sd = per_layer.get(i, OrderedDict())
                if self._from_pretraining:
                    sd = self._from_pretraining_entry(layers[i - b], i, sd, dropped, kept_init)
                else:
                    self._check_not_pretraining(layers[i - b], i, sd)
                sds.append(sd)
            module.load_weights(sds)
        if self._from_pretraining:
            msg = ("CheckpointHook: initialised from the pretraining checkpoint {}; dropped "
                   "entries: {}; left at initialisation: {}".format(
                       self._load_checkpoint_from, "; ".join(dropped) or "none",
                       "; ".join(kept_init) or "none"))
            runner._log(msg)
            print(msg, flush=True)
        engine = getattr(runner, "engine", None)
        if engine is not None and hasattr(engine, "sync_tied_weights"):
            engine.sync_tied_weights()   # an engine that is already set up: replica := table
        if self._from_pretraining:
            # rank 0's copy takes what the workers hold now: the loaded entries and, for the
            # layers left at initialisation, the workers' own initial weights
            self._gather_to_parameter_server(runner)
        elif runner.is_rank0:
            runner.parameter_server.load_weights_from_file(self._load_checkpoint_from)
        extra = self._extra_path(self._load_checkpoint_from, runner.rank)
        if self._resume_training_state and osp.exists(extra):
            st = torch.load(extra, map_location="cpu")
            if self._save_optimizer and st.get("optimizer") is not None:
                try:
                    runner.optimizer.load_state_dict(st["optimizer"])
                except Exception as exc:  # a resume with fresh optimizer state must not be silent
                    msg = "CheckpointHook: optimizer state of {} NOT restored ({}: {})".format(
                        extra, type(exc).__name__, exc)
                    if self._strict_optimizer:
                        raise RuntimeError(msg) from exc
                    import warnings

                    warnings.warn(msg)
                    runner._log(msg)
            runner.iter = st.get("iter", runner.iter)
            runner.epoch = st.get("epoch", runner.epoch)

    @staticmethod
    def _from_pretraining_entry(layer, idx: int, sd, dropped: list, kept_init: list):
        """What layer ``idx`` of the model loads from a pretraining file's entry ``sd``: the entry
        when its names are the layer's; for a ``BertPooler``, the ``pooler.*`` entries of a
        pretraining head saved at the same index; otherwise the layer's own current state (it
        keeps its initialisation).  Entries not taken are reported in ``dropped`` (as
        ``layer idx: prefix.*``), layers left at initialisation in ``kept_init``."""
        from ...models.bert_layers import BertPooler

        own = layer.state_dict()
        take, used = None, ()
        if set(sd) == set(own):
            take, used = sd, tuple(sd)
        elif isinstance(layer, BertPooler) and all("pooler." + k in sd for k in own):
            used = tuple("pooler." + k for k in own)
            take = OrderedDict((k, sd["pooler." + k]) for k in own)
        if take is not None:
            for k, v in take.items():
                if tuple(v.shape) != tuple(own[k].shape):
                    raise ValueError(
                        "layer {} ({}): the checkpoint's {} is {} but the model's is {}; build the "
                        "model with the pretraining run's geometry (a masked-LM run pads the "
                        "vocabulary to a multiple of 8)".format(idx, type(layer).__name__, k,
                                                               list(v.shape), list(own[k].shape)))
        rest = sorted({k.split(".", 1)[0] for k in sd if k not in used})
        if rest:
            dropped.append("layer {}: {}".format(idx, ", ".join(r + ".*" for r in rest)))
        if take is None:
            if own:
                kept_init.append("layer {} ({})".format(idx, type(layer).__name__))
            return own
        return take

    @staticmethod
    def _check_not_pretraining(layer, idx: int, sd) -> None:
        """A classification layer fed a pretraining head's entry: a clear error instead of a
        ``load_state_dict`` traceback."""
        own = layer.state_dict()
        if own and set(sd) != set(own) and any(k.startswith(("transform.", "decoder.",
                                                             "seq_relationship.")) for k in sd):
            raise ValueError(
                "layer {} ({}) gets the entries of a masked-LM / pretraining head ({}): the "
                "checkpoint comes from a pretraining model; load it with CheckpointHook("
                "load_checkpoint_from=..., from_pretraining=True)".format(
                    idx, type(layer).__name__, ", ".join(sorted({k.split(".", 1)[0] for k in sd}))))

    @staticmethod
    def _tie_rule(runner, per_layer: dict, path: str) -> None:
        """A decoder tied to the word embeddings takes the file's ``word_embeddings.weight`` entry
        (layer 0), whichever stage it is on: its own ``decoder.weight`` entry is replaced by it.
        The file keeps both entries, so tied and untied checkpoints interchange; a file saved from
        an untied model (the entries differ) is reported once."""
        from ...models.bert_layers import BertTailForMaskedLM

        table = per_layer.get(0, {}).get("word_embeddings.weight")
        if table is None:
            return
        for module in runner.model.model:
            if not module.is_local:
                continue
            b = module.layer_range[0] if module.layer_range is not None else 0
            for off, layer in enumerate(module.module.layers.children()):
                if not (isinstance(layer, BertTailForMaskedLM) and layer.tie_word_embeddings):
                    continue
                sd = per_layer.get(b + off)
                if sd is None or "decoder.weight" not in sd:
                    continue
                if not torch.equal(sd["decoder.weight"].float(), table.float()):
                    msg = ("CheckpointHook: {} was saved from an untied model: the tied decoder "
                           "uses its word_embeddings.weight, its decoder.weight is not used"
                           .format(path))
                    import warnings

                    warnings.warn(msg)
                    runner._log(msg)
                sd["decoder.weight"] = table

    # ------------------------------------------------------------------ save
    @staticmethod
    def _extra_path(ckpt_path: str, rank: int) -> str:
        root, _ = osp.splitext(ckpt_path)
        return "{}.extra.rank{}.pth".format(root, rank)

    def after_epoch(self, runner):
        if not self._save_path or not self.every_n_epochs(runner, self._save_interval):
            return
        self.save(runner, osp.join(self._save_path, "epoch_{}.pth".format(runner.epoch)))

    def after_val_epoch(self, runner):
        # an evaluation pass is not a training epoch: no checkpoint
        return None

    @staticmethod
    def _gather_to_parameter_server(runner) -> None:
        """Every rank's layer weights into rank 0's ParameterServer.  Collective."""
        local = {}
        for module in runner.model.model:
            if not module.is_local:
                continue
            b, _e = module.layer_range if module.layer_range is not None else (0, 0)
            for off, layer_sd in enumerate(module.get_state_dict()):
                local[b + off] = layer_sd
        d = _dist()
        if d is not None:
            gathered = [None] * d.get_world_size()
            d.all_gather_object(gathered, local)
        else:
            gathered = [local]
        if runner.is_rank0:
            for part in gathered:
                for idx, layer_sd in part.items():
                    try:
                        runner.parameter_server.update_weights(layer_sd, idx)
                    except Exception as exc:
                        raise Exception("have {} state dicts, have {} layers, error occurs at {}".format(
                            sum(len(p) for p in gathered), len(runner.parameter_server), idx)) from exc

    def save(self, runner, file_name: str) -> None:
        if runner.is_rank0:
            os.makedirs(osp.dirname(osp.abspath(file_name)), exist_ok=True)
        self._gather_to_parameter_server(runner)
        if runner.is_rank0:
            runner.parameter_server.save_weights_to_file(file_name)
        if self._save_optimizer:
            d = _dist()
            if d is not None:
                d.barrier()
            torch.save(dict(optimizer=runner.optimizer.state_dict() if runner.optimizer else None,
                            iter=runner.iter, epoch=runner.epoch),
                       self._extra_path(file_name, runner.rank))
