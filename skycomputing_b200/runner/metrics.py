"""Classification metrics of an evaluation pass.

An accumulator collects, over every batch of the pass, the sum of the per-row cross entropies,
the number of counted rows and a ``C x C`` confusion matrix (``[label, prediction]``); rows whose
label is ``ignore_index`` (the padding of a short final batch) are skipped, and a label outside
``[0, C)`` is counted as invalid.  ``classification_metrics`` turns the totals into the numbers the
GLUE classification tasks report.

* ``TorchEvalAccumulator``: plain torch on any device, fp64 losses.  Used for CPU runs and
  ``backend="torch"``, and the oracle of the native ``ops.native.EvalAccumulator``;
* ``LazyEvalAccumulator``: what ``Runner.evaluate`` hands to the engine - picks the native or the
  torch accumulator from the first logits it sees (the class count is only known there).

Token-level outputs (a masked-language-model head: logits ``[B, S, V]``, labels ``[B, S]``) are
counted per labelled token instead, without a confusion matrix: ``TorchTokenAccumulator`` (the
oracle) and ``ops.native.TokenEvalAccumulator`` collect the loss sum, the labelled tokens, the
correct top-1 predictions and the invalid labels, and ``token_metrics`` reports ``n``, ``loss``,
``accuracy`` and ``perplexity``.
"""
from __future__ import annotations

import math

import torch


class TorchEvalAccumulator:
    """Same totals as the ``classify_eval`` kernel: loss = logsumexp(row) - row[label] (fp64),
    prediction = ``torch.argmax`` (first maximum, NaN counts as the maximum)."""

    def __init__(self, C: int, device=None):
        self.C = int(C)
        self.device = torch.device(device) if device is not None else torch.device("cpu")
        self.reset()

    def reset(self) -> None:
        self.loss_sum = torch.zeros((), dtype=torch.float64, device=self.device)
        self.count = torch.zeros((), dtype=torch.int64, device=self.device)
        self.invalid = torch.zeros((), dtype=torch.int64, device=self.device)
        self.confusion = torch.zeros(self.C * self.C, dtype=torch.int64, device=self.device)

    @torch.no_grad()
    def add(self, logits: torch.Tensor, labels: torch.Tensor, ignore_index: int = -100) -> None:
        logits = logits.detach().reshape(-1, logits.shape[-1]).to(self.device)
        labels = labels.detach().reshape(-1).to(self.device, torch.int64)
        if logits.shape[1] != self.C:
            raise ValueError("logits have {} classes, the accumulator {}".format(
                logits.shape[1], self.C))
        keep = labels != ignore_index
        valid = keep & (labels >= 0) & (labels < self.C)
        self.invalid += (keep & ~valid).sum()
        rows = logits[valid].double()
        lab = labels[valid]
        pred = torch.argmax(logits[valid], dim=1)
        loss = torch.logsumexp(rows, dim=1) - rows.gather(1, lab[:, None])[:, 0]
        self.loss_sum += loss.sum()
        self.count += lab.numel()
        self.confusion += torch.bincount(lab * self.C + pred, minlength=self.C * self.C)

    def read(self) -> dict:
        return dict(loss_sum=float(self.loss_sum), count=int(self.count),
                    invalid=int(self.invalid),
                    confusion=self.confusion.cpu().view(self.C, self.C).clone())


class TorchTokenAccumulator:
    """Same totals as the ``vocab_ce`` kernel in eval mode: loss = logsumexp(row) - row[label]
    (fp64 sum), correct = ``torch.argmax`` equals the label."""

    def __init__(self, V: int, device=None):
        self.V = int(V)
        self.device = torch.device(device) if device is not None else torch.device("cpu")
        self.reset()

    def reset(self) -> None:
        self.loss_sum = torch.zeros((), dtype=torch.float64, device=self.device)
        self.count = torch.zeros((), dtype=torch.int64, device=self.device)
        self.correct = torch.zeros((), dtype=torch.int64, device=self.device)
        self.invalid = torch.zeros((), dtype=torch.int64, device=self.device)

    @torch.no_grad()
    def add(self, logits: torch.Tensor, labels: torch.Tensor, ignore_index: int = -100) -> None:
        logits = logits.detach().reshape(-1, logits.shape[-1]).to(self.device)
        labels = labels.detach().reshape(-1).to(self.device, torch.int64)
        if logits.shape[1] != self.V:
            raise ValueError("logits have {} classes, the accumulator {}".format(
                logits.shape[1], self.V))
        keep = labels != ignore_index
        valid = keep & (labels >= 0) & (labels < self.V)
        self.invalid += (keep & ~valid).sum()
        rows = logits[valid].float()
        lab = labels[valid]
        loss = torch.logsumexp(rows, dim=1) - rows.gather(1, lab[:, None])[:, 0]
        self.loss_sum += loss.double().sum()
        self.count += lab.numel()
        self.correct += (torch.argmax(logits[valid], dim=1) == lab).sum()

    def read(self) -> dict:
        return dict(loss_sum=float(self.loss_sum), count=int(self.count),
                    correct=int(self.correct), invalid=int(self.invalid), classes=self.V)


def make_token_accumulator(V: int, device) -> object:
    """The native token accumulator where the native kernels run, the torch one elsewhere."""
    device = torch.device(device)
    if device.type == "cuda":
        from ..models.bert_layers import get_backend
        from ..ops import native as nat

        if get_backend() != "torch" and nat.available() and V <= nat.ext().vocab_ce_max_v():
            return nat.TokenEvalAccumulator(V, device)
    return TorchTokenAccumulator(V, device)


def make_accumulator(C: int, device) -> object:
    """The native accumulator where the native kernels run (CUDA, backend != "torch", C within
    the kernel's limit), the torch one elsewhere."""
    device = torch.device(device)
    if device.type == "cuda":
        from ..models.bert_layers import get_backend
        from ..ops import native as nat

        if get_backend() != "torch" and nat.available() and C <= nat.ext().eval_max_classes():
            return nat.EvalAccumulator(C, device)
    return TorchEvalAccumulator(C, device)


class LazyEvalAccumulator:
    """Creates its accumulator on the first ``add`` (from the logits' class count and device) and
    keeps it, so that a captured evaluation graph always adds into the same buffer."""

    def __init__(self, ignore_index: int = -100):
        self.ignore_index = ignore_index
        self.inner = None

    def reset(self) -> None:
        if self.inner is not None:
            self.inner.reset()

    def add(self, logits: torch.Tensor, labels: torch.Tensor) -> None:
        if self.inner is None:
            # one prediction per token (MLM head: [B, S, V] logits, [B, S] labels) or per sequence
            per_token = logits.dim() == 3 or labels.dim() == 2
            make = make_token_accumulator if per_token else make_accumulator
            self.inner = make(logits.shape[-1], logits.device)
        self.inner.add(logits, labels, self.ignore_index)

    def read(self) -> dict:
        if self.inner is None:
            return dict(loss_sum=0.0, count=0, invalid=0, confusion=torch.zeros(0, 0, dtype=torch.int64))
        return self.inner.read()


def classification_metrics(confusion, loss_sum: float, count: int) -> dict:
    """``n``, mean ``loss``, ``accuracy`` and the ``confusion`` matrix (nested lists, rows =
    labels); for two classes also ``f1`` of class 1 and the Matthews correlation ``mcc``, each 0
    when its denominator is 0 (the scikit-learn convention).  With n == 0 loss and accuracy are
    None."""
    conf = torch.as_tensor(confusion, dtype=torch.int64)
    n = int(count)
    correct = int(conf.diagonal().sum()) if conf.numel() else 0
    out = dict(n=n, loss=(float(loss_sum) / n) if n else None,
               accuracy=(correct / n) if n else None, confusion=conf.tolist())
    if conf.shape == (2, 2):
        tn, fp, fn, tp = (int(v) for v in conf.reshape(-1))
        den_f1 = 2 * tp + fp + fn
        out["f1"] = (2 * tp / den_f1) if den_f1 else 0.0
        den = (tp + fp) * (tp + fn) * (tn + fp) * (tn + fn)
        out["mcc"] = ((tp * tn - fp * fn) / den ** 0.5) if den else 0.0
    return out


def token_metrics(loss_sum: float, count: int, correct: int) -> dict:
    """``n`` labelled tokens, mean ``loss``, top-1 ``accuracy`` and ``perplexity = exp(loss)``;
    None each when n == 0."""
    n = int(count)
    loss = (float(loss_sum) / n) if n else None
    return dict(n=n, loss=loss, accuracy=(int(correct) / n) if n else None,
                perplexity=math.exp(min(loss, 700.0)) if n else None)


def format_metrics(metrics: dict) -> str:
    parts = []
    for k in ("n", "loss", "accuracy", "perplexity", "f1", "mcc"):
        if k in metrics:
            v = metrics[k]
            parts.append("{}={}".format(k, "None" if v is None else (
                "{:.6g}".format(v) if isinstance(v, float) else v)))
    return ", ".join(parts)


__all__ = ["TorchEvalAccumulator", "TorchTokenAccumulator", "LazyEvalAccumulator",
           "make_accumulator", "make_token_accumulator", "classification_metrics", "token_metrics",
           "format_metrics"]
