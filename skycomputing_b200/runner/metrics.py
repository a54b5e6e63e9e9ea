"""Classification metrics of an evaluation pass.

An accumulator collects, over every batch of the pass, the sum of the per-row cross entropies,
the number of counted rows and a ``C x C`` confusion matrix (``[label, prediction]``); rows whose
label is ``ignore_index`` (the padding of a short final batch) are skipped, and a label outside
``[0, C)`` is counted as invalid.  ``classification_metrics`` turns the totals into the numbers the
GLUE classification tasks report.

* ``TorchEvalAccumulator``: plain torch on any device, fp64 losses.  Used for CPU runs and
  ``backend="torch"``, and the oracle of the native ``ops.native.EvalAccumulator``;
* ``LazyEvalAccumulator``: what ``Runner.evaluate`` hands to the engine (``eval_accumulator``) -
  the accumulator ``OBJECTIVES`` maps the ``objective`` of the model's last layer to.

Token-level outputs (a masked-language-model head: logits ``[B, S, V]``, labels ``[B, S]``) are
counted per labelled token instead, without a confusion matrix: ``TorchTokenAccumulator`` (the
oracle) and ``ops.native.TokenEvalAccumulator`` collect the loss sum, the labelled tokens, the
correct top-1 predictions and the invalid labels, and ``token_metrics`` reports ``n``, ``loss``,
``accuracy`` and ``perplexity``.

A span head (``BertTailForQuestionAnswering``: logits ``[B, 2, S]``, labels ``[B, 5]``) is
evaluated by ``TorchSpanAccumulator`` (the oracle) or ``ops.native.SpanEvalAccumulator``: the best
answer span of every sequence and the totals ``span_metrics`` turns into ``n``, ``loss``,
``start_accuracy``, ``end_accuracy``, ``exact`` and ``f1``.
"""
from __future__ import annotations

import math
from typing import Callable, NamedTuple

import torch

from ..models.bert_layers import native_active


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


def _token_accumulator(V: int, device) -> object:
    """The native token accumulator where the native kernels run, the torch one elsewhere."""
    if native_active(device):
        from ..ops import native as nat

        if V <= nat.ext().vocab_ce_max_v():
            return nat.TokenEvalAccumulator(V, device)
    return TorchTokenAccumulator(V, device)


def _classification_accumulator(C: int, device) -> object:
    """The native accumulator where the native kernels run and take C, the torch one elsewhere."""
    if native_active(device):
        from ..ops import native as nat

        if C <= nat.ext().eval_max_classes():
            return nat.EvalAccumulator(C, device)
    return TorchEvalAccumulator(C, device)


class TorchSpanAccumulator:
    """Same totals, spans and tie rule as the ``qa_span_eval`` kernel, in plain torch with fp64
    sums (the CPU path and the kernel's oracle).  ``add`` takes logits ``[B, 2, S]`` and labels
    ``[B, 5]`` (``ops.functions.split_span_labels``).

    Best span of a sequence: the maximum of ``start[i] + end[j]`` (one fp32 add, NaN counts as
    -inf) over ``max(start_lo, 0) <= i <= min(start_hi, S - 1)`` and ``i <= j <= min(i + L - 1,
    end_hi, S - 1)``; among equal scores the smallest ``(i, j)`` wins; an empty range gives
    ``(-1, -1)`` with score -inf.  Totals run over the sequences whose gold start and end are both
    in [0, S): start / end cross entropy (fp64), top-1 start / end hits (``torch.argmax``), exact
    spans and SQuAD's token F1 on position intervals.  Predictions of the first ``capacity``
    sequences since ``reset`` are kept, later ones counted as overflow."""

    def __init__(self, max_answer_length: int = 30, capacity: int = 0, device=None):
        self.max_answer_length = int(max_answer_length)
        self.capacity = int(capacity)
        self.device = torch.device(device) if device is not None else torch.device("cpu")
        self.reset()

    def reset(self) -> None:
        self.sums = torch.zeros(3, dtype=torch.float64)
        self.counts = dict(count=0, start_correct=0, end_correct=0, exact=0, invalid=0, overflow=0)
        self.spans, self.scores = [], []
        self.seen = 0

    @staticmethod
    def best_span(start: torch.Tensor, end: torch.Tensor, lo: int, hi: int, end_hi: int, L: int):
        """``(i, j, score)`` of one sequence's fp32 start / end logits [S]."""
        S = start.numel()
        lo, hi, end_hi = max(int(lo), 0), min(int(hi), S - 1), min(int(end_hi), S - 1)
        if hi < lo:
            return -1, -1, float("-inf")
        i = torch.arange(S).view(S, 1)
        j = torch.arange(S).view(1, S)
        ok = (i >= lo) & (i <= hi) & (j >= i) & (j <= i + L - 1) & (j <= end_hi)
        if not bool(ok.any()):
            return -1, -1, float("-inf")
        score = start.float().view(S, 1) + end.float().view(1, S)
        score = torch.where(torch.isnan(score), float("-inf"), score)
        best = score[ok].max()
        k = int(torch.nonzero((ok & (score == best)).reshape(-1))[0])   # the first (i, j)
        return k // S, k % S, float(best)

    @staticmethod
    def span_f1(pi: int, pj: int, gs: int, ge: int) -> float:
        overlap = min(pj, ge) - max(pi, gs) + 1
        if pi < 0 or overlap <= 0:
            return 0.0
        p, r = overlap / (pj - pi + 1), overlap / (ge - gs + 1)
        return 2 * p * r / (p + r)

    @torch.no_grad()
    def add(self, logits: torch.Tensor, labels: torch.Tensor, ignore_index: int = -100) -> None:
        logits = logits.detach().float().cpu()
        labels = labels.detach().reshape(-1, 5).cpu().to(torch.int64)
        B, _, S = logits.shape
        for b in range(B):
            gs, ge, lo, hi, ehi = (int(v) for v in labels[b])
            st, en = logits[b, 0], logits[b, 1]
            pi, pj, score = self.best_span(st, en, lo, hi, ehi, self.max_answer_length)
            if self.seen < self.capacity:
                self.spans.append((pi, pj))
                self.scores.append(score)
            else:
                self.counts["overflow"] += 1
            self.seen += 1
            ok_s, ok_e = 0 <= gs < S, 0 <= ge < S
            if (gs != ignore_index and not ok_s) or (ge != ignore_index and not ok_e):
                self.counts["invalid"] += 1
                continue
            if not (ok_s and ok_e):
                continue
            c = self.counts
            c["count"] += 1
            c["start_correct"] += int(int(torch.argmax(st)) == gs)
            c["end_correct"] += int(int(torch.argmax(en)) == ge)
            c["exact"] += int(pi == gs and pj == ge)
            self.sums[0] += float(torch.logsumexp(st.double(), 0) - st.double()[gs])
            self.sums[1] += float(torch.logsumexp(en.double(), 0) - en.double()[ge])
            self.sums[2] += self.span_f1(pi, pj, gs, ge)

    def read(self) -> dict:
        return dict(start_loss_sum=float(self.sums[0]), end_loss_sum=float(self.sums[1]),
                    f1_sum=float(self.sums[2]), **self.counts,
                    spans=torch.tensor(self.spans, dtype=torch.int64).reshape(-1, 2),
                    scores=torch.tensor(self.scores, dtype=torch.float32))


def _span_accumulator(max_answer_length: int, capacity: int, device) -> object:
    """The native span accumulator where the native kernels run, the torch one elsewhere."""
    if native_active(device):
        from ..ops import native as nat

        return nat.SpanEvalAccumulator(max_answer_length, capacity, device)
    return TorchSpanAccumulator(max_answer_length, capacity, device)


def span_metrics(totals: dict) -> dict:
    """``n`` counted sequences, ``loss`` = (mean start CE + mean end CE) / 2, ``start_accuracy``,
    ``end_accuracy``, ``exact`` (best span == gold span) and ``f1`` (mean token F1), as fractions;
    None each when n == 0."""
    n = int(totals["count"])
    if n == 0:
        return dict(n=0, loss=None, start_accuracy=None, end_accuracy=None, exact=None, f1=None)
    return dict(n=n, loss=(totals["start_loss_sum"] + totals["end_loss_sum"]) / (2 * n),
                start_accuracy=totals["start_correct"] / n, end_accuracy=totals["end_correct"] / n,
                exact=totals["exact"] / n, f1=totals["f1_sum"] / n)


class LazyEvalAccumulator:
    """Creates the accumulator of ``objective`` from ``args`` on the first ``add`` and keeps it, so
    that a captured evaluation graph always adds into the same buffer.  A last layer that declares
    no objective is scored per token when its first logits are 3-D or its labels 2-D, per sequence
    otherwise, with the class count of those logits."""

    def __init__(self, ignore_index: int = -100, objective=None, args=None):
        self.key = (objective, ignore_index, args)
        self.ignore_index, self.objective, self.args = ignore_index, objective, args
        self.inner = None

    def reset(self) -> None:
        if self.inner is not None:
            self.inner.reset()

    def add(self, logits, labels: torch.Tensor) -> None:
        if self.inner is None:
            if self.objective is None:
                per_token = logits.dim() == 3 or labels.dim() == 2
                self.objective = "masked_lm" if per_token else "classification"
                self.args = (logits.shape[-1],)
            self.inner = OBJECTIVES[self.objective].accumulator(*self.args, labels.device)
        self.inner.add(logits, labels, self.ignore_index)

    def read(self) -> dict:
        if self.inner is None:
            return dict(loss_sum=0.0, count=0, invalid=0, confusion=torch.zeros(0, 0, dtype=torch.int64))
        return self.inner.read()

    def payload(self, head, loader) -> dict:
        """The metrics of the pass and ``error``, the text of the ValueError its labels raise."""
        objective = self.objective if self.inner is not None else "classification"
        return OBJECTIVES[objective].payload(self.read(), head, loader, self.ignore_index)


class PreTrainingAccumulator:
    """Both objectives of a pretraining head: the masked-LM token totals and the next-sentence
    classification totals (two classes), each native or torch as for a head of that kind.  ``add``
    takes ``(mlm_logits, nsp_logits)`` and the one-tensor labels of
    ``ops.functions.split_pretraining_labels``."""

    def __init__(self, V: int, device):
        self.mlm = _token_accumulator(V, device)
        self.nsp = _classification_accumulator(2, device)

    def reset(self) -> None:
        self.mlm.reset()
        self.nsp.reset()

    def add(self, logits, labels: torch.Tensor, ignore_index: int = -100) -> None:
        from ..ops.functions import split_pretraining_labels

        mlm_labels, nsp_labels = split_pretraining_labels(labels)
        self.mlm.add(logits[0], mlm_labels, ignore_index)
        self.nsp.add(logits[1], nsp_labels, ignore_index)

    def read(self) -> dict:
        return dict(mlm=self.mlm.read(), nsp=self.nsp.read())


def pretraining_metrics(totals: dict) -> dict:
    """``mlm_n``, ``mlm_loss``, ``mlm_accuracy``, ``perplexity`` (``token_metrics`` of the
    masked-LM totals), ``nsp_n``, ``nsp_loss``, ``nsp_accuracy`` (``classification_metrics`` of the
    next-sentence totals) and ``loss = mlm_loss + nsp_loss``, an objective without a labelled row
    counting 0 (None when neither has one)."""
    m, n = totals["mlm"], totals["nsp"]
    tok = token_metrics(m["loss_sum"], m["count"], m["correct"])
    cls = classification_metrics(n["confusion"], n["loss_sum"], n["count"])
    out = dict(mlm_n=tok["n"], mlm_loss=tok["loss"], mlm_accuracy=tok["accuracy"],
               perplexity=tok["perplexity"], nsp_n=cls["n"], nsp_loss=cls["loss"],
               nsp_accuracy=cls["accuracy"])
    out["loss"] = (None if tok["n"] == 0 and cls["n"] == 0
                   else (tok["loss"] or 0.0) + (cls["loss"] or 0.0))
    return out


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


def _labels_error(invalid: int, classes, ignore_index: int, *notes: str):
    """The text of the ValueError a pass with ``invalid`` labels raises; None without one."""
    return "{} labels are outside [0, {}) and not ignore_index ({}){}".format(
        invalid, classes, ignore_index, "".join(notes)) if invalid else None


def _max_predictions_note(head, V: int) -> str:
    if not getattr(head, "consumes_labels", False):
        return ""
    return ("; the sparse masked-language-model head decodes at most max_predictions = {} "
            "labelled positions per sequence, and a sequence with more gets the out-of-range "
            "label {} in its last slot: raise max_predictions or label fewer positions".format(
                head.max_predictions, V))


def _classification_payload(totals: dict, head, loader, ignore_index: int) -> dict:
    return dict(classification_metrics(totals["confusion"], totals["loss_sum"], totals["count"]),
                error=_labels_error(totals["invalid"], len(totals["confusion"]), ignore_index))


def _token_payload(totals: dict, head, loader, ignore_index: int) -> dict:
    return dict(token_metrics(totals["loss_sum"], totals["count"], totals["correct"]),
                error=_labels_error(totals["invalid"], totals["classes"], ignore_index,
                                    _max_predictions_note(head, totals["classes"])))


def _pretraining_payload(totals: dict, head, loader, ignore_index: int) -> dict:
    m, n = totals["mlm"], totals["nsp"]
    return dict(pretraining_metrics(totals), error=_labels_error(
        m["invalid"] + n["invalid"], m["classes"], ignore_index,
        " ({} of them next-sentence labels, which must be in [0, 2))".format(n["invalid"]),
        _max_predictions_note(head, m["classes"])))


def _span_args(head, loader) -> tuple:
    """``(max_answer_length, capacity)``: the prediction buffer holds every example of the loader,
    its length rounded up to the batch (a padded last batch is stored too)."""
    n = len(loader.dataset)
    bs = int(getattr(loader, "batch_size", None) or 1)
    return int(head.max_answer_length), (n + bs - 1) // bs * bs


def _span_payload(totals: dict, head, loader, ignore_index: int) -> dict:
    """Span metrics, and the dataset's ``text_scores`` (SQuAD answer-text scores) if it has any."""
    if totals["overflow"]:
        raise ValueError("evaluation: {} span predictions did not fit the prediction buffer "
                         "of {} sequences".format(totals["overflow"], len(totals["spans"])))
    payload = dict(span_metrics(totals), error=_labels_error(
        totals["invalid"], "S (the sequence length)", ignore_index))
    ds = loader.dataset
    if hasattr(ds, "text_scores"):
        n = len(ds)
        payload.update(ds.text_scores(totals["spans"][:n], totals["scores"][:n]))
    return payload


class Objective(NamedTuple):     # how an evaluation pass scores a last layer's ``objective``
    args: Callable          # (head, loader) -> the arguments the accumulator is built from
    accumulator: Callable   # (*args, device) -> the accumulator, native where the kernels run
    payload: Callable       # (totals, head, loader, ignore_index) -> the metrics and ``error``


OBJECTIVES = {
    "classification": Objective(lambda head, loader: (head.num_classes,),
                                _classification_accumulator, _classification_payload),
    "masked_lm": Objective(lambda head, loader: (head.decoder.out_features,),
                           _token_accumulator, _token_payload),
    "pretraining": Objective(lambda head, loader: (head.decoder.out_features,),
                             PreTrainingAccumulator, _pretraining_payload),
    "span": Objective(_span_args, _span_accumulator, _span_payload),
}


def eval_accumulator(head, ignore_index: int, loader, previous=None) -> LazyEvalAccumulator:
    """``previous`` if built alike (a captured evaluation graph adds into it), else a new one."""
    objective = getattr(head, "objective", None)
    args = OBJECTIVES[objective].args(head, loader) if objective else None
    if previous is None or previous.key != (objective, ignore_index, args):
        previous = LazyEvalAccumulator(ignore_index, objective, args)
    return previous


def format_metrics(metrics: dict) -> str:
    parts = []
    for k in ("n", "loss", "accuracy", "perplexity", "f1", "mcc", "mlm_n", "mlm_loss",
              "mlm_accuracy", "nsp_n", "nsp_loss", "nsp_accuracy", "start_accuracy",
              "end_accuracy", "exact", "text_exact_match", "text_f1"):
        if k in metrics:
            v = metrics[k]
            parts.append("{}={}".format(k, "None" if v is None else (
                "{:.6g}".format(v) if isinstance(v, float) else v)))
    return ", ".join(parts)


__all__ = ["TorchEvalAccumulator", "TorchTokenAccumulator", "classification_metrics",
           "token_metrics", "PreTrainingAccumulator", "pretraining_metrics",
           "TorchSpanAccumulator", "span_metrics", "OBJECTIVES", "LazyEvalAccumulator",
           "eval_accumulator", "format_metrics"]
