"""skycomputing_b200 - H100-native load-balanced pipeline-model-parallel training.

Same user-facing surface as hpcaitech/SkyComputing (``scaelum``): python-file configs, the four
registries, builders, ``dynamics`` (Allocator / benchmarkers / Estimator / ParameterServer /
Worker / WorkerManager), ``RpcModel``, ``Runner`` + hooks, ``Logger``, ``DistributedTimer``,
``Stimulator`` - on a Hopper-first substrate (one process per GPU, hand-written sm_90a
kernels, peer-memory fused stage boundaries over NVLink, C++ allocator / benchmark loop).
"""
def _ensure_core() -> None:
    """The C++ core (allocator / stimulator) is a hard dependency of `dynamics`; build it on first
    import if the in-tree .so is missing (g++ only, a few seconds).  The CUDA module is built by
    `__graft_entry__.build()` / `python -m skycomputing_b200._build` and is only needed on GPUs."""
    import os
    import sys

    override = os.environ.get("SKY_CORE_OVERRIDE")
    if override:
        # an instrumented (ASAN / UBSAN) build of the core from tools/run_core_sanitizer.sh
        import glob
        import importlib.machinery
        import importlib.util

        path = glob.glob(os.path.join(override, "_core*.so"))[0]
        loader = importlib.machinery.ExtensionFileLoader(__name__ + "._core", path)
        spec = importlib.util.spec_from_loader(__name__ + "._core", loader)
        mod = importlib.util.module_from_spec(spec)
        loader.exec_module(mod)
        sys.modules[__name__ + "._core"] = mod
        globals()["_core"] = mod
        return
    try:
        from . import _core  # noqa: F401
    except ImportError:
        from . import _build

        _build.build_core(verbose=False)


_ensure_core()

from .builder import *  # noqa: F401,F403,E402
from .config import *  # noqa: F401,F403
from .dataset import *  # noqa: F401,F403
from .dynamics import *  # noqa: F401,F403
from .logger import *  # noqa: F401,F403
from .models import *  # noqa: F401,F403
from .parallel import (BaseModule, FusedAdam, FusedLamb, FusedSGD, Lamb, LocalModule,  # noqa: F401
                       PipelineEngine, RemoteModule, RpcModel, build_optimizer)
from .registry import *  # noqa: F401,F403
from .runner import *  # noqa: F401,F403
from .stimulator import Stimulator  # noqa: F401
from .timer import *  # noqa: F401,F403
from .version import __version__  # noqa: F401
from . import utils  # noqa: F401

# `scaelum.model` is spelled `models` here; keep the old name importable
from . import models as model  # noqa: F401,E402
