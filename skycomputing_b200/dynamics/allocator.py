"""Layer -> device allocation front-end (``Allocator``).

Same public surface as scaelum/dynamics/allocator.py:12-439 - ``even_allocate()``,
``dynamic_allocate(break_iter=1000)``, ``optimal_allocate(max_time=300, threads=24)``, all
returning the (re-ranked) ``WorkerManager`` - on top of the C++ core (csrc/alloc/allocator.cc):

* ``even``     pure arithmetic, identical split to the reference;
* ``dynamic``  greedy boundary shifting after a memory pass; ``solver="compat"`` reproduces the
               reference bit-for-bit (including the dead shrink branch, SURVEY §2.7),
               the default ``"heuristic"`` runs the intended two-way refinement;
* ``optimal``  exact min-max contiguous partition (bisection + subset DP over device orders)
               instead of a time-limited MILP (PuLP/CBC are not even installable here);
               ``max_time`` / ``threads`` are accepted for API compatibility and ignored - the
               exact solver needs milliseconds for D = 8, L = 483.

Extras (all optional): ``granularity="block"`` only cuts between whole transformer blocks (the
fused NVLink boundary exists for those cuts and they carry 5x less data than a cut after
``BertLayer_Body``); ``comm_aware=True`` adds boundary-bytes / link-bandwidth to the stage cost.
"""
from __future__ import annotations

from typing import List, Optional, Sequence

from .. import _core
from .worker_manager import WorkerManager

_BLOCK_SEQ = ("BertLayer_Head", "BertLayer_Body", "BertLayer_Tail")


def group_units(model_cfg: Sequence[dict], granularity: str) -> List[tuple]:
    """[(begin, end)] index ranges of the allocatable units of the layer list.

    ``"layer"``: every list entry is a unit (the reference's granularity).  ``"block"``: a
    ``Head, Body, Tail`` triple is one unit, and the entries in front of the first / behind the
    last transformer block (embeddings; pooler, classifier) belong to that block's unit - every
    cut then sits between two whole blocks, which is where the fused NVLink boundary exists."""
    n = len(model_cfg)
    if granularity == "layer":
        return [(i, i + 1) for i in range(n)]
    units, is_block, i = [], [], 0
    while i < n:
        names = [c.get("layer_type") for c in model_cfg[i:i + 3]]
        if tuple(names) == _BLOCK_SEQ:
            units.append((i, i + 3))
            is_block.append(True)
            i += 3
        else:
            units.append((i, i + 1))
            is_block.append(False)
            i += 1
    if any(is_block):
        first, last = is_block.index(True), len(is_block) - 1 - is_block[::-1].index(True)
        head = (units[0][0], units[first][1])
        tail = (units[last][0], units[-1][1])
        if first == last:
            return [(head[0], tail[1])]
        units = [head] + units[first + 1:last] + [tail]
    return units


class Allocator:
    def __init__(self, model_cfg: list, worker_manager: WorkerManager, model_benchmarker=None,
                 device_benchmarker=None, solver: str = "heuristic", granularity: str = "layer",
                 comm_aware: bool = False, boundary_bytes: Optional[Sequence[float]] = None,
                 link_bytes_per_s: float = 340e9, device_flops_per_s: float = 7e14,
                 logger=None):
        # comm_aware cost of a cut = boundary bytes / link_bytes_per_s.  The defaults (link rate
        # for 4-8 MiB stage-boundary tensors, sustained rate of a transformer block) are carried
        # over from the B200 version and have not been re-measured on H100: pass measured values
        # where they matter.
        assert solver in ("heuristic", "compat", "exact"), solver
        assert granularity in ("layer", "block"), granularity
        self._model_cfg = model_cfg
        self._worker_manager = worker_manager
        self._model_benchmarker = model_benchmarker
        self._device_benchmarker = device_benchmarker
        self._solver = solver
        self._granularity = granularity
        self._comm_aware = comm_aware
        self._boundary_bytes = boundary_bytes
        self._link_bytes_per_s = link_bytes_per_s
        self._device_flops_per_s = device_flops_per_s
        self._logger = logger
        self.last_result: Optional[dict] = None
        self.last_device_times: dict = {}
        self.last_layer_costs: list = []

    # ------------------------------------------------------------------ helpers
    def _log(self, msg: str) -> None:
        if self._logger is not None:
            self._logger.info(msg)

    def _benchmarks(self):
        results = self._device_benchmarker.benchmark()
        names = list(results.keys())
        ranks = [int(n.replace("worker", "")) for n in names]
        dt = [float(results[n]["time"]) for n in names]
        dm = [float(results[n]["avai_mem"]) for n in names]
        lf, lm = self._model_benchmarker.benchmark()
        lf, lm = [float(x) for x in lf], [float(x) for x in lm]
        if self._comm_aware and self._boundary_bytes is None:
            # `comm_aware=True` without explicit sizes: the model benchmarker knows what every
            # layer hands to the next one (a cut after BertLayer_Body ships 5x the bytes of a cut
            # after Head / Tail: [M, I] + [M, H] instead of [M, H])
            self._boundary_bytes = getattr(self._model_benchmarker, "last_boundary_bytes", None)
        # kept for diagnostics / ReallocateHook: benchmark time per PHYSICAL device (stable across
        # re-orderings of the pool, unlike the rank-derived worker names) and the layer costs
        pool = list(self._worker_manager.worker_pool)
        self.last_device_times = {(w.device if w.device is not None else i): dt[i]
                                  for i, w in enumerate(pool)}
        self.last_layer_costs = list(lf)
        self._log("worker ranks: {}".format(ranks))
        self._log("worker time: {}".format(dt))
        return ranks, dt, dm, lf, lm

    def _unit_vectors(self, lf, lm):
        units = group_units(self._model_cfg, self._granularity)
        uf = [sum(lf[b:e]) for b, e in units]
        um = [sum(lm[b:e]) for b, e in units]
        return units, uf, um

    def _cut_penalty(self, units, dt, uf) -> List[float]:
        if not (self._comm_aware and self._boundary_bytes is not None):
            return []
        # cost unit = dev_time x flops.  The fastest device (dev_time = tmin) sustains
        # `device_flops_per_s`, so one second == tmin * device_flops_per_s cost units.
        tmin = min(dt)
        pen = [0.0] * (len(units) + 1)
        for k in range(1, len(units)):
            layer_idx = units[k][0]
            seconds = float(self._boundary_bytes[layer_idx]) / self._link_bytes_per_s
            pen[k] = seconds * self._device_flops_per_s * tmin
        return pen

    def _assign(self, order: Sequence[int], unit_bounds: Sequence[int], units) -> WorkerManager:
        """order[k] = index (in the current pool) of the worker that runs pipeline stage k."""
        pool = list(self._worker_manager.worker_pool)
        n_units = len(units)
        for k, widx in enumerate(order):
            ub, ue = unit_bounds[k], unit_bounds[k + 1]
            b = units[ub][0] if ub < n_units else len(self._model_cfg)
            e = units[ue - 1][1] if ue > ub else b
            w = pool[widx]
            w.model_config = self._model_cfg[b:e]
            w.layer_range = (b, e)
            w.order = k + 1
        self._worker_manager.reset_rank_by_order()
        for w in self._worker_manager.worker_pool:
            self._log("rank {} (device {}) has layers {} to {}".format(
                w.rank, w.device, w.layer_range[0], w.layer_range[1]))
        return self._worker_manager

    # ------------------------------------------------------------------ public API
    def even_allocate(self) -> WorkerManager:
        units = group_units(self._model_cfg, self._granularity)
        D = self._worker_manager.size
        bounds = _core.even_partition(len(units), D)
        self.last_result = dict(method="even", boundaries=bounds, order=list(range(D)))
        return self._assign(list(range(D)), bounds, units)

    def dynamic_allocate(self, break_iter: int = 1000) -> WorkerManager:
        ranks, dt, dm, lf, lm = self._benchmarks()
        units, uf, um = self._unit_vectors(lf, lm)
        if self._solver == "exact":
            res = _core.optimal_partition(uf, um, dt, dm, permute=False, min_layers=1,
                                          cut_penalty=self._cut_penalty(units, dt, uf))
        else:
            res = _core.dynamic_partition(uf, um, dt, dm, break_iter=break_iter,
                                          compat=(self._solver == "compat"),
                                          cut_penalty=[] if self._solver == "compat"
                                          else self._cut_penalty(units, dt, uf))
        self.last_result = res
        self._log("dynamic allocation: {}".format(res))
        return self._assign(res["order"], res["boundaries"], units)

    def optimal_allocate(self, max_time: int = 300, threads: int = 24,
                         permute: bool = True) -> WorkerManager:
        del max_time, threads  # the exact solver does not need a time limit
        ranks, dt, dm, lf, lm = self._benchmarks()
        units, uf, um = self._unit_vectors(lf, lm)
        res = _core.optimal_partition(uf, um, dt, dm, permute=permute, min_layers=1,
                                      cut_penalty=self._cut_penalty(units, dt, uf))
        self.last_result = res
        self._log("optimal allocation: {}".format(res))
        return self._assign(res["order"], res["boundaries"], units)

    def looped_allocate(self, alloc_type: str, virtual_stages: int) -> WorkerManager:
        """Allocation for a LOOPED pipeline: ``virtual_stages`` (v) chunks per worker, virtual
        stage k = chunk k // D of worker k % D (pool order is kept, no device permutation).

        The v x D spans come from the same solvers: ``even`` splits the units evenly; ``dynamic``
        / ``optimal`` run the exact fixed-order min-max partition over v x D virtual devices whose
        speed is the worker's and whose memory cap is 1/v of the worker's.  With v chunks the
        pipeline fill / drain shrink by v (parallel/pipeline_looped.py)."""
        v = int(virtual_stages)
        assert v >= 1
        units = group_units(self._model_cfg, self._granularity)
        pool = list(self._worker_manager.worker_pool)
        D = len(pool)
        VP = v * D
        if len(units) < VP:
            raise ValueError(f"{len(units)} allocatable units cannot fill {v} x {D} virtual stages")
        if alloc_type in ("dynamic", "optimal"):
            ranks, dt, dm, lf, lm = self._benchmarks()
            _units, uf, um = self._unit_vectors(lf, lm)
            vdt = [dt[k % D] for k in range(VP)]
            vdm = [dm[k % D] / v for k in range(VP)]
            res = _core.optimal_partition(uf, um, vdt, vdm, permute=False, min_layers=1,
                                          cut_penalty=self._cut_penalty(units, vdt, uf))
            # the exact solver balanced the most expensive CHUNK (pipeline latency); throughput
            # is set by the busiest DEVICE (sum of its v chunks): refine towards that, but never
            # past the most expensive chunk of the even split, so that the result is no worse than
            # ``even`` on either measure
            even = _core.even_partition(len(units), VP)
            even_worst = max(sum(uf[even[k]:even[k + 1]]) * dt[k % D] for k in range(VP))
            bounds = self._refine_device_loads(list(res["boundaries"]), uf, um, dt, dm, D,
                                               max_chunk=even_worst * (1.0 + 1e-12))
            self.last_result = dict(res, boundaries=bounds, virtual_stages=v)
        else:
            bounds = _core.even_partition(len(units), VP)
            self.last_result = dict(method="even", boundaries=bounds, order=list(range(VP)),
                                    virtual_stages=v)
        for d, w in enumerate(pool):
            chunks, cfg = [], []
            for c in range(v):
                k = c * D + d
                b = units[bounds[k]][0]
                e = units[bounds[k + 1] - 1][1]
                chunks.append((b, e))
                cfg += self._model_cfg[b:e]
            w.chunks = chunks
            w.model_config = cfg
            w.layer_range = chunks[0] if v == 1 else None
            w.order = d + 1
            self._log("rank {} (device {}) runs layer spans {}".format(w.rank, w.device, chunks))
        self._worker_manager.reset_rank_by_order()
        return self._worker_manager

    @staticmethod
    def _refine_device_loads(bounds: List[int], uf, um, dt, dm, D: int,
                             max_chunk: float = float("inf")) -> List[int]:
        """Hill-climb on the chunk boundaries of a looped partition (C++ core,
        csrc/alloc/allocator.cc: refine_looped_partition): repeatedly shrink a chunk of the busiest
        device by one unit (handing the unit to the neighbouring chunk, which belongs to another
        device) while that lowers the descending-sorted vector of device loads
        dt[d] x sum(flops of d's chunks); ties are broken towards the smaller most-expensive
        chunk.  Every chunk keeps >= 1 unit, device memory caps are respected, and no move makes
        a chunk cost more than ``max_chunk`` (dt x flops)."""
        assert len(dt) == D and len(dm) == D
        return list(_core.refine_looped_partition([float(x) for x in uf], [float(x) for x in um],
                                                  [float(x) for x in dt], [float(x) for x in dm],
                                                  [int(x) for x in bounds], float(max_chunk)))

    def allocate(self, alloc_type: str, virtual_stages: int = 1, **kwargs) -> WorkerManager:
        """Dispatch on ``allocator_config['type']`` (experiment/launch.py:119-138 semantics)."""
        if virtual_stages and int(virtual_stages) > 1:
            return self.looped_allocate(alloc_type, int(virtual_stages))
        if alloc_type == "dynamic":
            return self.dynamic_allocate(**kwargs)
        if alloc_type == "optimal":
            return self.optimal_allocate(**kwargs)
        return self.even_allocate()

    # ------------------------------------------------------------------ diagnostics
    @staticmethod
    def bottleneck(layer_flops, layer_mem, dev_time, dev_mem, order, boundaries) -> float:
        return _core.partition_bottleneck(list(layer_flops), list(layer_mem), list(dev_time),
                                          list(dev_mem), list(order), list(boundaries))
