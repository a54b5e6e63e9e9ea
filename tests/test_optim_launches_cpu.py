"""The fused optimizers' launch sequences, driven on CPU with a recording fake of ``native.ext()``.

For SGD (with and without momentum), Adam, AdamW and LAMB over banks plus torch-fallback
parameters, banks only and fallback parameters only; with nothing configured, a learning-rate
schedule, gradient clipping and both; on a single stage, with an ``all_reduce`` of the norm and
with a peer-memory exchange: the ordered kernel launches (and ``all_reduce`` calls) of a step and
their arguments, pointers named by the buffer they point into, the ``state_dict`` keys and a
``load_state_dict`` round trip, and the flags the engines read.  The expected values live in
``golden/optim_launches.json``; ``PYTHONPATH=. python tests/test_optim_launches_cpu.py`` rewrites
it."""
import json
import os
import struct
from types import SimpleNamespace

import pytest
import torch

from skycomputing_b200.ops import native
from skycomputing_b200.ops.functions import ParamBank
from skycomputing_b200.parallel import optim
from skycomputing_b200.parallel.engine_base import EngineBase

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "optim_launches.json")
STREAM = 7
EXCHANGE = SimpleNamespace(regions_ptr=0x51000, n_ranks=2, position=1, epoch_ptr=0x52000,
                           error_ptr=0x53000)
SENTINELS = {0x51000: "exchange.regions", 0x52000: "exchange.epoch", 0x53000: "exchange.error"}

# binding argument names (csrc/bindings_cuda.cpp) and which of them are device pointers
KERNELS = {
    "sgd_multi": ("d_tensors n max_numel lr momentum weight_decay grad_scale zero_grad stream "
                  "scalars", "d_tensors scalars"),
    "adam_multi": ("d_tensors n max_numel lr beta1 beta2 eps weight_decay decoupled step "
                   "grad_scale zero_grad stream scalars", "d_tensors step scalars"),
    "lamb_moments": ("segs chunk_seg n_chunks beta1 beta2 eps step grad_scale partials stream "
                     "scalars", "segs chunk_seg step partials scalars"),
    "lamb_update": ("segs chunk_seg n_chunks lr beta1 beta2 eps step partials ratios stream "
                    "scalars", "segs chunk_seg step partials ratios scalars"),
    "grad_sumsq_multi": ("d_tensors n blocks grad_scale partials stream", "d_tensors partials"),
    "optim_finalize": ("partials n_partials extra_sumsq regions n_ranks my_pos epoch error_flag "
                       "step step_offset schedule warmup total base_lr max_norm out stream",
                       "partials extra_sumsq regions epoch error_flag step out"),
    "advance_counter": ("counter inc stream", "counter"),
}
assert set(KERNELS) <= set(native._KERNELS_PER_CALL)


class FakeExt:
    """Records launches; packed tables carry a token that names the rows they were packed from."""
    OPTIM_SCALARS_FLOATS = 4
    LAMB_CHUNK = 4

    def __init__(self):
        self.launches, self.tables, self.opt = [], {}, None

    # ---- pointers -> names
    def _buffers(self):
        named = []
        for i, b in enumerate(self.opt.banks):
            named += [(f"bank{i}.master", b.flat), (f"bank{i}.grad", b.flat_grad),
                      (f"bank{i}.shadow", b._shadow)]
        sd = self.opt.state_dict()
        for key in ("momentum", "second_moment"):
            named += [(f"{key}{i}", t) for i, t in enumerate(sd.get(key, [])) if t is not None]
        seen = []

        def walk(v):
            if isinstance(v, torch.Tensor):
                seen.append((f"{str(v.dtype)[6:]}[{v.numel()}]", v))
            elif isinstance(v, (list, tuple)):
                for x in v:
                    walk(x)
            elif isinstance(v, dict):
                for x in v.values():
                    walk(x)
        walk(list(vars(self.opt).values()))
        return named + seen

    def _find(self, ptr):
        for name, t in self._buffers():
            if t is not None and t.numel() and 0 <= ptr - t.data_ptr() < t.numel() * t.element_size():
                return name, t, ptr - t.data_ptr()
        raise AssertionError(f"pointer {ptr:#x} into no known buffer")

    def name(self, ptr):
        if not ptr or ptr in SENTINELS:
            return SENTINELS.get(ptr, 0)
        name, t, off = self._find(ptr)
        if t.dtype == torch.uint8:            # a packed table: name it by its rows
            return self.tables[struct.unpack_from("<q", t.numpy().tobytes())[0]]
        return f"{name}+{off}" if off else name

    def _table(self, rows):
        token = len(self.tables) + 1
        ptrs = (0, 1, 2, 3, 4) if rows and len(rows[0]) == 9 else (0, 1, 2, 3, 6)
        self.tables[token] = [[self.name(x) if k in ptrs else x for k, x in enumerate(r)]
                              for r in rows]
        return struct.pack("<q", token) + bytes(56 * max(1, len(rows)))

    # ---- host calls
    def pack_sgd_descriptors(self, descs):
        return self._table(descs)

    def pack_lamb_segments(self, rows):
        chunks = [-(-r[5] // self.LAMB_CHUNK) for r in rows]
        seg = self._table(rows)
        token = len(self.tables) + 1
        self.tables[token] = ["chunks", chunks]
        return (seg, struct.pack("<q", token) + bytes(4 * sum(chunks)), sum(chunks),
                [all(r[k] % 16 == 0 for k in range(4)) for r in rows])

    def grad_sumsq_blocks(self, max_numel):
        return 1 + max_numel // 8

    # ---- launches
    def __getattr__(self, kernel):
        if kernel not in KERNELS:
            raise AttributeError(kernel)
        names, ptrs = (s.split() for s in KERNELS[kernel])

        def launch(*args, **kw):
            vals = dict(zip(names, args), **kw)
            assert set(vals) <= set(names), (kernel, sorted(vals))
            self.launches.append([kernel, {k: self.name(v) if k in ptrs else v
                                           for k, v in sorted(vals.items())}])
            if kernel == "advance_counter":
                _, t, off = self._find(vals["counter"])
                t.view(-1)[off // 8] += vals["inc"]
        return launch


KINDS = {
    "sgd": lambda m, b: optim.FusedSGD(m, lr=0.1, weight_decay=0.01, banks=b),
    "sgd_momentum": lambda m, b: optim.FusedSGD(m, lr=0.1, momentum=0.9, weight_decay=0.01,
                                                banks=b),
    "adam": lambda m, b: optim.FusedAdam(m, lr=0.01, betas=(0.8, 0.9), eps=1e-7,
                                         weight_decay=0.01, banks=b),
    "adamw": lambda m, b: optim.FusedAdam(m, lr=0.01, weight_decay=0.02, decoupled=True, banks=b),
    "lamb": lambda m, b: optim.FusedLamb(m, lr=0.02, weight_decay=0.05, banks=b),
}
LAYOUTS = ("banks+rest", "banks", "rest")
CONFIGS = {"plain": (None, None), "schedule": ("cosine", None), "clip": (None, 1.0),
           "schedule+clip": ("linear", 0.5)}
REDUCTIONS = ("single", "allreduce", "exchange")
CASES = [(k, l, c, r) for k in KINDS for l in LAYOUTS for c in CONFIGS for r in REDUCTIONS]


def _module(layout):
    torch.manual_seed(0)
    mod = torch.nn.Module()
    banks = []
    if layout != "rest":
        mod.dense_weight = torch.nn.Parameter(torch.randn(4, 3))
        mod.dense_extra = torch.nn.Parameter(torch.randn(3, 3))      # 21 elements: a scalar tail
        mod.LayerNorm_bias = torch.nn.Parameter(torch.randn(6))
        w = ParamBank([mod.dense_weight, mod.dense_extra])
        w.wgrad_target = True                                       # left un-zeroed, then fresh
        banks = [w, ParamBank([mod.LayerNorm_bias], need_shadow=False), w]   # de-duplicated
    if layout != "banks":
        mod.fallback = torch.nn.Linear(3, 2)
    return mod, banks


def run_case(kind, layout, config, reduction, monkeypatch):
    fake = FakeExt()
    monkeypatch.setattr(native, "ext", lambda: fake)
    monkeypatch.setattr(native, "cast_f32_to_bf16_", lambda s, d: d.copy_(s))
    streams = []
    monkeypatch.setattr(torch.cuda, "current_stream",
                        lambda *a, **k: streams.append(1) or SimpleNamespace(cuda_stream=STREAM))
    monkeypatch.setattr(torch.distributed, "all_reduce",
                        lambda t, group=None: fake.launches.append(["all_reduce", fake.name(
                            t.data_ptr()), t.numel(), group]))
    mod, banks = _module(layout)
    opt = KINDS[kind](mod, banks)
    fake.opt = opt
    sched, max_norm = CONFIGS[config]
    if sched or max_norm:
        opt.configure(optim.check_lr_schedule(
            sched and dict(type=sched, warmup_steps=1, total_steps=6)), max_norm)
    if reduction == "allreduce":
        opt.set_norm_reduction(group="group", allreduce=True)
    elif reduction == "exchange":
        opt.set_norm_reduction(group="group", exchange=EXCHANGE)
    flags = [opt.graph_safe, opt.needs_global_norm, opt.reports_scalars,
             list(EngineBase._norm_info(SimpleNamespace(optimizer=opt)))]
    steps = []
    for _ in range(2):
        for p in getattr(mod, "fallback", torch.nn.Linear(1, 1)).parameters():
            p.grad = torch.randn_like(p)
        fake.launches.clear()
        opt.step(grad_scale=0.5)
        steps.append(list(fake.launches))
    assert steps[0] == steps[1]
    assert steps[0] or not streams, "the stream is queried only when something is launched"
    fresh = [b.fresh for b in opt.banks]
    sd = opt.state_dict()
    return dict(launches=steps[0], flags=flags, fresh=fresh, step_count=opt.step_count(),
                state_keys=sorted(sd)), opt, sd


def _clone(x):
    if isinstance(x, torch.Tensor):
        return x.clone()
    if isinstance(x, dict):
        return {k: _clone(v) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return type(x)(_clone(v) for v in x)
    return x


def _same(a, b):
    if isinstance(a, torch.Tensor):
        return isinstance(b, torch.Tensor) and torch.equal(a, b)
    if isinstance(a, dict):
        return isinstance(b, dict) and a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    return a == b


def _golden():
    with open(GOLDEN) as f:
        return json.load(f)


@pytest.mark.parametrize("kind,layout,config,reduction", CASES)
def test_launch_sequence(kind, layout, config, reduction, monkeypatch):
    got, opt, sd = run_case(kind, layout, config, reduction, monkeypatch)
    assert json.loads(json.dumps(got)) == _golden()["/".join((kind, layout, config, reduction))]
    # load_state_dict round trip: disturb every buffer the state_dict exposes, then restore it
    saved = _clone(sd)
    for t in (t for key in ("momentum", "second_moment") for t in sd.get(key, [])):
        if t is not None:
            t.add_(1.0)
    opt.step(grad_scale=0.5)
    opt.load_state_dict(_clone(saved))
    assert _same(opt.state_dict(), saved)
    assert opt.step_count() == got["step_count"]


if __name__ == "__main__":
    class _Patch:
        def setattr(self, obj, name, value):
            setattr(obj, name, value)

    table = {}
    saved = {n: getattr(native, n) for n in ("ext", "cast_f32_to_bf16_")}
    saved_stream, saved_ar = torch.cuda.current_stream, torch.distributed.all_reduce
    try:
        for case in CASES:
            table["/".join(case)] = run_case(*case, _Patch())[0]
    finally:
        for n, v in saved.items():
            setattr(native, n, v)
        torch.cuda.current_stream, torch.distributed.all_reduce = saved_stream, saved_ar
    with open(GOLDEN, "w") as f:       # one case per line
        f.write("{\n" + ",\n".join(f"{json.dumps(k)}: {json.dumps(v, separators=(',', ':'))}"
                                    for k, v in table.items()) + "\n}\n")
    print(f"wrote {len(table)} cases to {GOLDEN}")
