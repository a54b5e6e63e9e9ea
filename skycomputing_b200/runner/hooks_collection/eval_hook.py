"""Periodic evaluation on held-out data during training.

``EvalHook(datasets={name: data_loader, ...})`` runs ``Runner.evaluate`` on every named loader
every ``interval`` training iterations (0 = never), after every epoch when ``by_epoch`` is set and
once after the run when ``at_end`` is set (unless the last iteration was just evaluated).  With
``save_best=path`` it writes a checkpoint (``CheckpointHook.save``, collective) whenever metric
``key`` of the FIRST dataset improves under ``rule`` ("greater" or "less").  Every rank runs the
same schedule, and every rank receives the same metrics, so the decisions agree without
communication.  ``history`` keeps ``(iter, name, metrics)`` of every pass.
"""
from __future__ import annotations

from typing import Dict, Optional

from ...registry import HOOKS
from ..hooks import Hook
from .checkpoint_hook import CheckpointHook


@HOOKS.register_module
class EvalHook(Hook):
    def __init__(self, datasets: Dict[str, object], interval: int = 0, by_epoch: bool = False,
                 at_end: bool = True, save_best: Optional[str] = None, key: str = "accuracy",
                 rule: str = "greater"):
        if not datasets:
            raise ValueError("EvalHook needs at least one named evaluation data loader")
        if rule not in ("greater", "less"):
            raise ValueError("rule must be 'greater' or 'less', got {!r}".format(rule))
        self.datasets = dict(datasets)
        self.interval = int(interval or 0)
        self.by_epoch = by_epoch
        self.at_end = at_end
        self.save_best = save_best
        self.key = key
        self.rule = rule
        self.best: Optional[float] = None
        self.history: list = []
        self._last_iter: Optional[int] = None
        self._saver = CheckpointHook()

    def _improves(self, value) -> bool:
        if value is None:
            return False
        if self.best is None:
            return True
        return value > self.best if self.rule == "greater" else value < self.best

    def _run(self, runner) -> None:
        self._last_iter = runner.iter
        for i, (name, loader) in enumerate(self.datasets.items()):
            metrics = runner.evaluate(loader, name=name)
            self.history.append((runner.iter, name, metrics))
            if i == 0 and self.save_best and self._improves(metrics.get(self.key)):
                self.best = metrics[self.key]
                self._saver.save(runner, self.save_best)

    def after_train_iter(self, runner):
        # runner.iter already counts the iteration that just finished
        if self.interval > 0 and runner.iter % self.interval == 0:
            self._run(runner)

    def after_train_epoch(self, runner):
        if self.by_epoch and self._last_iter != runner.iter:
            self._run(runner)

    def after_run(self, runner):
        if self.at_end and self._last_iter != runner.iter:
            self._run(runner)
