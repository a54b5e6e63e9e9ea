"""Training loop + hook dispatch (capability parity with scaelum/runner/runner.py:15-156).

Same constructor contract (``model, parameter_server, worker_manager, optimizer, max_epochs,
max_iters, loss_cfg, timer_cfg, logging_cfg``), same hook call sequence (``before_run,
before_train_epoch, before_train_iter, after_train_iter, after_train_epoch, after_run``) and the
same rank-0 log lines (``epoch: e, iter: i`` / ``forward time`` / ``backward time`` /
``step time``).  Differences, all deliberate:

* SPMD: every rank runs the loop over the same (seeded) data order; the first stage consumes the
  inputs, the last stage the labels.  Rank 0 keeps the reference's "central server" duties (logs,
  ParameterServer, stop flag);
* the iteration is one ``PipelineEngine.train_step`` (micro-batched 1F1B or sequential; fused
  NVLink boundaries; CUDA graph) instead of dist_autograd + DistributedOptimizer RPC fan-out;
* times are device times (CUDA events), throughput (sequences/s) and loss are logged as well, and a
  structured ``metrics.jsonl`` is written next to ``allocation.log``;
* the reference's off-by-one (``max_iters + 1`` iterations) and the undefined ``max_epochs`` /
  ``max_iters`` attributes (SURVEY §2.7) are fixed.
"""
from __future__ import annotations

import json
import os
import time
from typing import Optional

import torch
import torch.nn as nn

from ..logger import Logger
from ..timer import DistributedTimer
from .hooks import Hook


class _NativeCrossEntropy(nn.Module):
    def forward(self, logits, labels):
        from ..ops.functions import SoftmaxCrossEntropyFn

        return SoftmaxCrossEntropyFn.apply(logits, labels)

    def fused(self, logits, labels, scale: float, loss_acc: torch.Tensor) -> torch.Tensor:
        """Engine fast path: one launch computes the micro-batch loss, adds ``loss * scale`` to
        ``loss_acc`` and returns d(loss * scale)/dlogits, which the engine feeds straight into
        ``logits.backward`` (no scalar-loss autograd nodes, no scaling / accumulation kernels)."""
        from ..ops import native as nat

        _, dlogits = nat.softmax_ce(logits.detach().contiguous().float(), labels.contiguous(),
                                    grad_scale=scale, loss_acc=loss_acc)
        return dlogits


class MaskedLMLoss(nn.Module):
    """Token-level cross entropy of a masked-language-model head: logits ``[..., V]``, labels
    ``[...]`` with ``ignore_index`` on every position that is not predicted.  The mean runs over
    the labelled positions; with none the loss is 0 (``F.cross_entropy`` would give NaN), so that
    a micro-batch without a masked token adds nothing to the step.  On the GPU the loss runs on
    the ``vocab_ce`` kernel, which supports at most 98304 classes (``ops.native.vocab_ce``)."""

    def __init__(self, ignore_index: int = -100):
        super().__init__()
        self.ignore_index = int(ignore_index)

    def forward(self, logits, labels):
        # the mean of F.cross_entropy(ignore_index=...) as sum / count, without a host sync
        flat = labels.reshape(-1)
        total = nn.functional.cross_entropy(logits.reshape(-1, logits.shape[-1]).float(), flat,
                                            ignore_index=self.ignore_index, reduction="sum")
        return total / (flat != self.ignore_index).sum().clamp(min=1)


class _NativeMaskedLMLoss(MaskedLMLoss):
    def fused(self, logits, labels, scale: float, loss_acc: torch.Tensor) -> torch.Tensor:
        """Engine fast path (see ``_NativeCrossEntropy.fused``): the ``vocab_ce`` kernel adds
        ``loss * scale`` to ``loss_acc`` and returns the bf16 gradient of the logits, written over
        them when they are a bf16 tensor of their own (no second vocabulary-sized buffer)."""
        from ..ops import native as nat

        V = logits.shape[-1]
        flat = logits.detach().reshape(-1, V)
        in_place = flat.dtype == torch.bfloat16 and flat.is_contiguous()
        if flat.dtype != torch.bfloat16:
            flat = flat.to(torch.bfloat16)
        _, dlogits = nat.vocab_ce(flat, labels.reshape(-1), grad_scale=scale, loss_acc=loss_acc,
                                  ignore_index=self.ignore_index, in_place=in_place)
        return dlogits.view(logits.shape)


class PreTrainingLoss(nn.Module):
    """BERT's pretraining loss (HF ``BertForPreTraining``'s ``total_loss``): the ``MaskedLMLoss``
    mean of the masked-LM logits plus the next-sentence cross entropy, each a mean over its
    labelled rows (0 without one).  ``logits`` = ``(mlm_logits, nsp_logits)``, ``labels`` the
    one-tensor layout of ``ops.functions.split_pretraining_labels``."""

    def __init__(self, ignore_index: int = -100):
        super().__init__()
        self.ignore_index = int(ignore_index)
        self.mlm = MaskedLMLoss(ignore_index)

    def forward(self, logits, labels):
        from ..ops.functions import split_pretraining_labels

        mlm_logits, nsp_logits = logits
        mlm_labels, nsp_labels = split_pretraining_labels(labels)
        return self.mlm(mlm_logits, mlm_labels) + self.mlm(nsp_logits, nsp_labels)


class _NativePreTrainingLoss(PreTrainingLoss):
    def __init__(self, ignore_index: int = -100):
        super().__init__(ignore_index)
        self.mlm = _NativeMaskedLMLoss(ignore_index)

    def fused(self, logits, labels, scale: float, loss_acc: torch.Tensor):
        """Engine fast path: ``vocab_ce`` and ``masked_softmax_ce`` each add their ``loss *
        scale`` into ``loss_acc``; returns the gradients of (mlm_logits, nsp_logits)."""
        from ..ops import native as nat
        from ..ops.functions import split_pretraining_labels

        mlm_logits, nsp_logits = logits
        mlm_labels, nsp_labels = split_pretraining_labels(labels)
        dmlm = self.mlm.fused(mlm_logits, mlm_labels, scale, loss_acc)
        _, dnsp = nat.masked_softmax_ce(nsp_logits.detach().float(), nsp_labels, grad_scale=scale,
                                        loss_acc=loss_acc, ignore_index=self.ignore_index)
        return dmlm, dnsp


class QuestionAnsweringLoss(nn.Module):
    """The span loss of a question-answering head (HF ``BertForQuestionAnswering``'s
    ``total_loss``): ``(mean start CE + mean end CE) / 2`` over logits ``[B, 2, S]``, each mean
    over the sequences whose label is in [0, S) (0 without one), labels the ``[B, 5]`` layout of
    ``ops.functions.split_span_labels``.  ``ignore_index`` rows add nothing; any other label
    outside [0, S) makes the loss NaN (HF clamps such positions and ignores them)."""

    def __init__(self, ignore_index: int = -100):
        super().__init__()
        self.ignore_index = int(ignore_index)

    def forward(self, logits, labels):
        from ..ops.functions import split_span_labels

        S = logits.shape[-1]
        start, end = split_span_labels(labels.reshape(-1, 5))[:2]
        total = 0.0
        for row, lab in ((logits[:, 0].float(), start), (logits[:, 1].float(), end)):
            keep = lab != self.ignore_index
            valid = keep & (lab >= 0) & (lab < S)
            ce = torch.logsumexp(row, 1) - row.gather(1, torch.where(valid, lab, 0)[:, None])[:, 0]
            mean = torch.where(valid, ce, 0.0).sum() / valid.sum().clamp(min=1)
            # an invalid label is never silent (and never used as an index)
            total = total + torch.where((keep & ~valid).any(), float("nan"), mean)
        return total / 2


class _NativeQuestionAnsweringLoss(QuestionAnsweringLoss):
    def forward(self, logits, labels):
        from ..ops.functions import SpanCrossEntropyFn

        return SpanCrossEntropyFn.apply(logits, labels, self.ignore_index)

    def fused(self, logits, labels, scale: float, loss_acc: torch.Tensor) -> torch.Tensor:
        """Engine fast path (see ``_NativeCrossEntropy.fused``): ``qa_span_ce`` adds ``loss *
        scale`` into ``loss_acc`` and returns the [B, 2, S] gradient of the logits."""
        from ..ops import native as nat

        _, dlogits = nat.qa_span_ce(logits.detach().float().contiguous(), labels,
                                    grad_scale=scale, loss_acc=loss_acc,
                                    ignore_index=self.ignore_index)
        return dlogits


_LOSSES = {
    "CrossEntropyLoss": (nn.CrossEntropyLoss, _NativeCrossEntropy),
    "MaskedLMLoss": (MaskedLMLoss, _NativeMaskedLMLoss),
    "PreTrainingLoss": (PreTrainingLoss, _NativePreTrainingLoss),
    "QuestionAnsweringLoss": (QuestionAnsweringLoss, _NativeQuestionAnsweringLoss),
}


def build_loss(loss_cfg: dict, device: torch.device) -> nn.Module:
    from ..models.bert_layers import native_active

    cfg = dict(loss_cfg)
    name = cfg.pop("type")
    # the native cross entropy takes no options (label_smoothing, weight, ...)
    if name not in _LOSSES or (name == "CrossEntropyLoss" and cfg):
        return getattr(nn, name)(**cfg)
    torch_loss, native_loss = _LOSSES[name]
    return (native_loss if native_active(device) else torch_loss)(**cfg)


class Runner:
    def __init__(self, model, parameter_server, worker_manager, optimizer, max_epochs: int,
                 max_iters: int, loss_cfg: dict, timer_cfg: dict, logging_cfg: dict,
                 micro_batches: int = 1, schedule: Optional[str] = None, boundary: str = "auto",
                 use_cuda_graph: bool = True, loss_interval: int = 1, device=None,
                 async_loss: bool = False):
        import torch.distributed as dist

        self.model = model
        self.worker_manager = worker_manager
        self.parameter_server = parameter_server
        self.optimizer = optimizer
        self._hooks = []
        self._hook_impl = {}
        self._fixed_batch = None
        self._epoch = 0
        self._iter = 0
        self._inner_iter = 0
        self._max_epochs = max_epochs
        self._max_iters = max_iters
        self._stop = False
        self.data_loader = None
        self.rank = dist.get_rank() if dist.is_available() and dist.is_initialized() else 0
        self.world_size = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
        self.is_rank0 = self.rank == 0
        self._logging_config = logging_cfg
        self._logger = Logger(**logging_cfg) if (logging_cfg and self.is_rank0) else None
        self._metrics_path = None
        if logging_cfg and self.is_rank0:
            self._metrics_path = os.path.join(os.path.dirname(os.path.abspath(logging_cfg["filename"])),
                                              "metrics.jsonl")
        self._timer_config = timer_cfg
        self._timer = DistributedTimer(**(timer_cfg or {}))
        stage = model.local_stage
        self.device = torch.device(device) if device is not None else stage.device
        self.loss_function = build_loss(loss_cfg, self.device)
        self.micro_batches = micro_batches
        self.schedule = schedule or ("sequential" if micro_batches == 1 else "1f1b")
        self.loss_interval = loss_interval
        # async_loss: the loss of step i is copied D2H asynchronously into pinned memory and
        # handed out by the call for step i+1 (flush_loss() returns the last one), so the host
        # never stalls the device between steps
        self.async_loss = async_loss
        self._loss_slots = None
        self._loss_pending = None
        self.last_loss: Optional[float] = None
        self.last_step_seconds: Optional[float] = None
        self._boundary = boundary
        self._use_cuda_graph = use_cuda_graph
        self._eval_accum = None       # kept across passes: a captured eval graph adds into it
        self.val_iter = 0             # batch index of the current evaluation pass
        self.last_eval: Optional[dict] = None
        self.engine = None
        self._build_engine()

    def _build_engine(self) -> None:
        from ..parallel.pipeline import PipelineEngine

        model = self.model
        v = getattr(model, "virtual_stages", 1)
        if v > 1:
            from ..parallel.pipeline_looped import LoopedPipelineEngine

            P = model.num_stages // v
            self.schedule = "looped"
            self.engine = LoopedPipelineEngine(
                stages=model.local_stages, virtual_indices=model.local_stage_indices, num_ranks=P,
                ring=model.stage_to_rank[:P], device=self.device, optimizer=self.optimizer,
                loss_fn=self.loss_function, micro_batches=self.micro_batches,
                # fused NVLink ring + whole-step CUDA graph by default on the native path (validated
                # on 2/4/8 GPUs); SKY_LOOPED_FUSED=0 or
                # boundary="nccl" selects torch.distributed p2p
                boundary=("auto" if (self._boundary in ("auto", "fused")
                                     and os.environ.get("SKY_LOOPED_FUSED", "1") != "0") else "dist"),
                use_cuda_graph=self._use_cuda_graph)
            model.attach_engine(self.engine)
            return
        self.engine = PipelineEngine(
            stage=model.local_stage, stage_index=model.local_stage_index,
            num_stages=model.num_stages, stage_to_rank=model.stage_to_rank, device=self.device,
            optimizer=self.optimizer, loss_fn=self.loss_function, micro_batches=self.micro_batches,
            schedule=self.schedule, boundary=self._boundary, use_cuda_graph=self._use_cuda_graph)
        model.attach_engine(self.engine)

    def rebuild(self, model, optimizer, worker_manager=None) -> None:
        """Swap in a re-partitioned model (ReallocateHook): the old engine's peer regions / CUDA
        graph are released, a new engine is built around the new local stage.  Collective."""
        if self.engine is not None:
            import torch.distributed as dist

            if self.device.type == "cuda":
                torch.cuda.synchronize(self.device)
            if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
                dist.barrier()  # every rank is done with its neighbours' regions before any is freed
            self.engine.close()
        self.model = model
        self.optimizer = optimizer
        if worker_manager is not None:
            self.worker_manager = worker_manager
        self._loss_pending = None
        self._build_engine()

    # ------------------------------------------------------------------ properties
    hooks = property(lambda self: self._hooks)
    max_epochs = property(lambda self: self._max_epochs)
    max_iters = property(lambda self: self._max_iters)
    max_iter = property(lambda self: self._max_iters)
    inner_iter = property(lambda self: self._inner_iter)

    @property
    def epoch(self) -> int:
        return self._epoch

    @epoch.setter
    def epoch(self, i: int) -> None:
        self._epoch = i

    @property
    def iter(self) -> int:
        return self._iter

    @iter.setter
    def iter(self, i: int) -> None:
        self._iter = i

    def request_stop(self) -> None:
        self._stop = True
        self._iter = self._max_iters + 1
        self._epoch = self._max_epochs + 1

    def register_hook(self, hook: Hook) -> None:
        assert isinstance(hook, Hook)
        self._hooks.append(hook)

    def _call_hook(self, fn_name: str) -> None:
        # hooks whose class does not implement `fn_name` are skipped without a Python call (the
        # set of implemented callbacks is computed once per hook class; hooks appended to
        # `runner.hooks` directly are handled the same way)
        for hook in self._hooks:
            impl = self._hook_impl.get(type(hook))
            if impl is None:
                impl = self._hook_impl[type(hook)] = type(hook).overrides()
            if fn_name in impl or fn_name in getattr(hook, "__dict__", ()):
                hook.fire(self, fn_name)

    def _log(self, msg: str) -> None:
        if self._logger is not None:
            self._logger.info(msg)

    # ------------------------------------------------------------------ one iteration
    def _to_device(self, t: torch.Tensor) -> torch.Tensor:
        if self.device.type != "cuda":
            return t
        if not t.is_pinned():
            t = t.pin_memory()
        return t.to(self.device, non_blocking=True)

    def train_iteration(self, data, labels) -> Optional[float]:
        """One optimisation step through the public API: H2D of this step's inputs (first stage)
        and labels (last stage), pipeline step, D2H of the loss (last stage).  Returns the loss as
        a Python float on the last stage (None elsewhere / when loss_interval skips it)."""
        eng = self.engine
        inputs = None
        if eng.is_first:
            data = data if isinstance(data, (list, tuple)) else (data,)
            inputs = [self._to_device(t) for t in data]
        lab = self._to_device(labels) if (eng.is_last and labels is not None) else None
        loss = eng.train_step(inputs, lab)
        out = None
        if loss is not None and self.loss_interval and (self._iter % self.loss_interval == 0):
            if self.async_loss and loss.is_cuda:
                out = self.flush_loss()  # the previous step's loss (its copy finished long ago)
                if self._loss_slots is None:
                    self._loss_slots = [torch.zeros(1, dtype=torch.float32).pin_memory()
                                        for _ in range(2)]
                    self._loss_slot_idx = 0
                slot = self._loss_slots[self._loss_slot_idx]
                self._loss_slot_idx ^= 1
                slot.copy_(loss.detach().reshape(1), non_blocking=True)  # D2H of this step's result
                ev = torch.cuda.Event()
                ev.record()
                self._loss_pending = (slot, ev)
            else:
                out = float(loss.item())  # D2H read of the step's result
                self.last_loss = out
        return out

    def flush_loss(self) -> Optional[float]:
        """async_loss mode: wait for and return the most recent step's loss."""
        if self._loss_pending is None:
            return None
        slot, ev = self._loss_pending
        self._loss_pending = None
        ev.synchronize()
        self.last_loss = float(slot[0])
        return self.last_loss

    def train(self, data_loader) -> None:
        self.data_loader = data_loader
        self.model.train(True)
        self._call_hook("before_run")
        cuda = self.device.type == "cuda"
        while self._epoch < self._max_epochs and not self._stop:
            self._call_hook("before_train_epoch")
            for batch_index, (data, labels) in enumerate(data_loader):
                if self._iter >= self._max_iters or self._stop:
                    break
                self._inner_iter = batch_index
                if not self._batch_shape_ok(data):
                    continue
                self._log("epoch: {}, iter: {}".format(self._epoch, self._iter))
                self._call_hook("before_train_iter")
                if cuda:
                    e0 = torch.cuda.Event(enable_timing=True)
                    e1 = torch.cuda.Event(enable_timing=True)
                    e0.record()
                t0 = time.time()
                loss = self.train_iteration(data, labels)
                if cuda:
                    e1.record()
                    e1.synchronize()
                    step_s = e0.elapsed_time(e1) * 1e-3
                else:
                    step_s = time.time() - t0
                self.last_step_seconds = step_s
                self._log_iteration(step_s, loss, data)
                self._iter += 1
                self._check_boundary_health()
                self._call_hook("after_train_iter")
            self._epoch += 1
            self._call_hook("after_train_epoch")
        self._call_hook("after_run")

    # ------------------------------------------------------------------ evaluation
    def evaluate(self, data_loader, name: str = "val", micro_batches: Optional[int] = None,
                 ignore_index: int = -100) -> dict:
        """Classification metrics of the model on ``data_loader`` (collective: every rank calls
        it and every rank gets the same dict, broadcast by the last stage).  For a token-level
        head (``BertTailForMaskedLM``, or a last layer without an ``objective`` whose logits are
        3-D or labels 2-D) the metrics are those of ``token_metrics``: labelled tokens, loss,
        top-1 accuracy and perplexity.  For a head evaluated by span
        (``BertTailForQuestionAnswering``) they are those of ``span_metrics`` (``n``, ``loss``,
        ``start_accuracy``, ``end_accuracy``, ``exact``, ``f1``), plus ``text_exact_match`` and
        ``text_f1`` when the loader's dataset has ``text_scores(spans, scores)``; more predictions
        than ``len(data_loader.dataset)`` rounded up to the batch raise ``ValueError``.  For a
        pretraining head (``BertTailForPreTraining``) they are those of ``pretraining_metrics``:
        the masked-LM ones with an ``mlm_`` prefix (and ``perplexity``), the next-sentence ``nsp_n``,
        ``nsp_loss`` and ``nsp_accuracy``, and ``loss`` = the sum of the two losses.

        The model runs in eval mode (the previous mode is restored) through the engine's
        forward-only pass with ``micro_batches`` chunks per batch (default: the training value;
        it must divide the batch size).  The first batch fixes the evaluation batch size; a
        shorter last batch is padded to it with zero ids / mask and ``ignore_index`` labels, so
        every example is counted exactly once.  Fires ``before/after_val_epoch`` once and
        ``before/after_val_iter`` per batch; ``val_iter`` counts the batches of the pass and
        ``iter`` does not move.  Neither the training RNG streams nor the optimizer are touched.
        """
        import torch.distributed as dist

        from .metrics import eval_accumulator, format_metrics

        eng = self.engine
        m = int(micro_batches or self.micro_batches)
        layers = getattr(eng.stages[-1], "layers", None)
        head = layers[-1] if layers is not None and len(layers) else None
        acc = self._eval_accum = eval_accumulator(head, ignore_index, data_loader,
                                                  self._eval_accum)
        was_training = self.model.training
        cpu_rng = torch.random.get_rng_state()   # iterating a DataLoader draws a base seed
        self.model.train(False)
        self.val_iter = 0
        try:
            acc.reset()
            self._call_hook("before_val_epoch")
            batch = None
            for data, labels in data_loader:
                data = list(data) if isinstance(data, (list, tuple)) else [data]
                n = int(data[0].shape[0])
                if batch is None:
                    batch = n
                    if batch % m:
                        raise ValueError("evaluation batches of {} samples cannot be split into {} "
                                         "equal micro-batches".format(batch, m))
                if n > batch:
                    raise ValueError("evaluation batch of {} samples after batches of {}".format(
                        n, batch))
                if n < batch:
                    data = [torch.cat([t, t.new_zeros((batch - n,) + tuple(t.shape[1:]))])
                            for t in data]
                    labels = torch.cat([labels, labels.new_full((batch - n,) + tuple(labels.shape[1:]),
                                                                ignore_index)])
                self._call_hook("before_val_iter")
                inputs = [self._to_device(t) for t in data] if eng.is_first else None
                lab = self._to_device(labels) if eng.is_last else None
                eng.eval_step(inputs, lab, acc, micro_batches=m)
                self.val_iter += 1
                self._call_hook("after_val_iter")
            payload = acc.payload(head, data_loader) if eng.is_last else None
            if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
                box = [payload]
                dist.broadcast_object_list(box, src=self.model.stage_to_rank[-1])
                payload = box[0]
        finally:
            self.model.train(was_training)
            torch.random.set_rng_state(cpu_rng)
        error = payload.pop("error")
        if error:
            raise ValueError("evaluation {}: {}".format(name, error))
        self._call_hook("after_val_epoch")
        self._log("eval {}: {}".format(name, format_metrics(payload)))
        if self._metrics_path is not None:
            with open(self._metrics_path, "a") as f:
                f.write(json.dumps(dict(mode="val", name=name, iter=self._iter, **payload)) + "\n")
        self.last_eval = dict(payload, name=name)
        return payload

    def _batch_shape_ok(self, data) -> bool:
        """The engine fixes the micro-batch shape on the first step (static CUDA-graph buffers,
        peer slots, cached p2p metas).  Every rank iterates the same seeded loader, so all ranks
        take the same decision here without communicating: a batch that cannot be split into
        ``micro_batches`` equal chunks is a configuration error, and a later batch of a different
        size (the short batch a loader without ``drop_last`` ends an epoch with, as the reference's
        stock data_config does) is skipped with a log line instead of hanging a neighbour stage in
        a full-size receive."""
        first = data[0] if isinstance(data, (list, tuple)) else data
        if not torch.is_tensor(first) or first.dim() == 0:
            return True
        nseq = int(first.shape[0])
        if self._fixed_batch is None:
            if nseq % max(self.micro_batches, 1) != 0:
                raise ValueError(
                    "batch of {} samples cannot be split into {} equal micro-batches".format(
                        nseq, self.micro_batches))
            self._fixed_batch = nseq
            return True
        if nseq != self._fixed_batch:
            self._log("skipping a batch of {} samples: the pipeline was set up for batches of {} "
                      "(use drop_last=True to avoid the short batch at the end of an epoch)".format(
                          nseq, self._fixed_batch))
            return False
        return True

    def _check_boundary_health(self, every: int = 50) -> None:
        """Failure detection for the in-kernel cross-GPU flag protocol: every spin-wait has a 4 s
        timeout that raises a device-side error flag instead of hanging the GPU; poll it here
        (one 4-byte D2H read every ``every`` iterations) and fail the run loudly."""
        fused = getattr(self.engine, "fused", None)
        if fused is None or self._iter % every != 0:
            return
        code = fused.error_code()
        if code == 5:
            raise RuntimeError(
                f"rank {self.rank}: the tied word-embedding gradient of the last stage did not "
                f"arrive within 4 s (error flag 5) at iteration {self._iter}: the last stage "
                "stopped producing - check its log")
        if code:
            raise RuntimeError(
                f"rank {self.rank}: fused stage-boundary wait timed out (error flag {code}) at "
                f"iteration {self._iter}: a neighbour stage stopped producing - check its log")

    def _log_iteration(self, step_s: float, loss, data) -> None:
        stage = self.model.local_stage
        fwd = bwd = None
        try:
            stage.flush_logs()
            if stage.forward_time:
                fwd = sum(stage.forward_time[-self.micro_batches:])
            if stage.backward_time:
                bwd = sum(stage.backward_time[-self.micro_batches:])
        except Exception:
            pass
        if not self.is_rank0:
            return
        if fwd is not None:
            self._log("forward time: {}".format(fwd))
        if bwd is not None:
            self._log("backward time: {}".format(bwd))
        self._log("step time: {}".format(step_s))
        first = data[0] if isinstance(data, (list, tuple)) else data
        nseq = int(first.shape[0]) if torch.is_tensor(first) else 0
        if loss is not None:
            self._log("loss: {}".format(loss))
        extra = {}
        if getattr(self.optimizer, "reports_scalars", False):
            # learning-rate schedule / clipping: this step's device scalars (the step has been
            # synchronised above; the global norm is the same on every rank)
            sc = self.optimizer.scalars()
            if sc["lr"] is not None:
                self._log("lr: {}".format(sc["lr"]))
                extra["lr"] = sc["lr"]
            if sc["grad_norm"] is not None:
                self._log("grad norm: {}".format(sc["grad_norm"]))
                extra["grad_norm"] = sc["grad_norm"]
        if self._metrics_path is not None:
            with open(self._metrics_path, "a") as f:
                f.write(json.dumps(dict(epoch=self._epoch, iter=self._iter, step_seconds=step_s,
                                        sequences_per_s=(nseq / step_s if step_s > 0 else None),
                                        forward_seconds=fwd, backward_seconds=bwd, loss=loss,
                                        **extra)) + "\n")
