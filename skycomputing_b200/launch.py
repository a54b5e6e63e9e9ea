"""Process bootstrap + orchestration (capability parity with experiment/launch.py:20-236).

    python -m skycomputing_b200.launch -c <config.py> [-p PORT] [--spawn N]

The same config keys as the reference are consumed (``model_config, rpc_config, data_config,
logging_config, worker_config, allocator_config, train_config``); rank / world size come from
torchrun (``RANK/WORLD_SIZE/LOCAL_RANK``), Slurm (``SLURM_PROCID/SLURM_NPROCS``), Open MPI, or
``--spawn N`` (N local processes, no cluster needed).  One process per worker: the reference's
"1 master + N workers" becomes N SPMD ranks, rank 0 doubling as the central server (logs,
ParameterServer, stop flag) - a reference-style config with ``CORE_NUM = N + 1`` therefore runs on
N processes.

Every rank executes the same sequence (allocation is deterministic given the gathered
benchmarks): worker pool -> [benchmarks] -> allocator -> RpcModel (local stage only) -> optimizer
-> Runner -> hooks -> train.  Allocation failures are logged and exit non-zero instead of being
swallowed (SURVEY §2.7).
"""
from __future__ import annotations

import argparse
import copy
import os
import os.path as osp
import sys
import traceback
from typing import Optional

import torch
import torch.distributed as dist

from .builder import build_data_generator, build_dataloader_from_cfg, build_hook
from .config import load_config
from .dynamics import Allocator, DeviceBenchmarker, ModelBenchmarker, ParameterServer, WorkerManager
from .logger import Logger
from .parallel import RpcModel, build_optimizer
from .runner import Runner


def _discover_rank() -> tuple:
    env = os.environ
    for r, w in (("RANK", "WORLD_SIZE"), ("SLURM_PROCID", "SLURM_NPROCS"),
                 ("OMPI_COMM_WORLD_RANK", "OMPI_COMM_WORLD_SIZE"), ("PMI_RANK", "PMI_SIZE")):
        if r in env and w in env:
            return int(env[r]), int(env[w])
    return 0, 1


def _local_rank(rank: int) -> int:
    for k in ("LOCAL_RANK", "SLURM_LOCALID", "OMPI_COMM_WORLD_LOCAL_RANK"):
        if k in os.environ:
            return int(os.environ[k])
    n = torch.cuda.device_count() if torch.cuda.is_available() else 1
    return rank % max(n, 1)


def _seeded_loader(data_config: dict, seed: int):
    dataloader_cfg = dict(data_config["dataloader_cfg"])
    dataset_cfg = dict(data_config["dataset_cfg"])
    if dataloader_cfg.get("shuffle") and "generator" not in dataloader_cfg:
        # every rank iterates the same order (first stage reads inputs, last stage labels)
        dataloader_cfg["generator"] = torch.Generator().manual_seed(seed)
    return build_dataloader_from_cfg(dataset_cfg=dataset_cfg, dataloader_cfg=dataloader_cfg)


def run_process(rank: int, world_size: int, rpc_config: dict, model_config: list = None,
                data_config: dict = None, logging_config: dict = None,
                allocator_config: dict = None, train_config: dict = None,
                worker_config: list = None, backend: Optional[str] = None,
                seed: int = 1234) -> int:
    train_config = copy.deepcopy(train_config)
    allocator_config = copy.deepcopy(allocator_config)
    worker_config = copy.deepcopy(worker_config)
    for k, v in (rpc_config or {}).items():
        if k == "GLOO_SOCKET_IFNAME":
            # only meaningful if that NIC exists on this machine (reference: Cray `ipogif0`)
            if not osp.exists(osp.join("/sys/class/net", str(v))):
                continue
        os.environ[k] = str(v)
    wants_cuda = any((w.get("extra_config") or {}).get("module_to_cuda") for w in worker_config)
    use_cuda = wants_cuda and torch.cuda.is_available()
    local_rank = _local_rank(rank)
    if use_cuda:
        torch.cuda.set_device(local_rank)
    device = torch.device("cuda", local_rank) if use_cuda else torch.device("cpu")
    if backend is None:
        backend = "nccl" if use_cuda else "gloo"
    print("starting to initialize the process group on rank: {} ({})".format(rank, backend), flush=True)
    if not dist.is_initialized():
        # failure detection for the un-fused (NCCL) boundaries: a peer that died or hung turns into
        # an exception on the survivors after the timeout instead of a silent stall (the fused
        # boundaries have their own in-kernel 4 s flag timeouts, Runner._check_boundary_health)
        os.environ.setdefault("TORCH_NCCL_ASYNC_ERROR_HANDLING", "1")
        import datetime

        timeout_s = int(rpc_config.get("rpc_timeout", 1200)) if isinstance(rpc_config, dict) else 1200
        kwargs = dict(backend=backend, rank=rank, world_size=world_size,
                      timeout=datetime.timedelta(seconds=timeout_s))
        if use_cuda:
            kwargs["device_id"] = device
        dist.init_process_group(**kwargs)
    torch.manual_seed(seed)
    status = 0
    try:
        log_workspace = osp.dirname(logging_config["filename"])
        if rank == 0:
            if osp.exists(log_workspace):
                for f in os.listdir(log_workspace):
                    p = osp.join(log_workspace, f)
                    if osp.isfile(p):
                        os.remove(p)
            else:
                os.makedirs(log_workspace, exist_ok=True)
        dist.barrier()
        logger = Logger(**logging_config) if rank == 0 else None

        def info(msg):
            if logger is not None:
                logger.info(msg)

        info("logger initialized")
        if len(worker_config) != world_size:
            raise RuntimeError(
                "worker_config has {} workers but {} processes were launched: launch one process "
                "per worker (a reference-style CORE_NUM = workers + 1 config runs on `workers` "
                "ranks; rank 0 doubles as the central server)".format(len(worker_config), world_size))
        for i, w in enumerate(worker_config):
            ec = w.setdefault("extra_config", {})
            if not use_cuda:
                ec["module_to_cuda"] = False
                ec["output_to_cpu"] = False
                ec["cuda_device"] = -1
            else:
                ec["cuda_device"] = local_rank if i == rank else ec.get("cuda_device", 0)
                ec["output_to_cpu"] = False  # boundaries never stage through the host
            w.setdefault("device", i)
        worker_manager = WorkerManager(first_rank=0)
        worker_manager.load_worker_pool_from_config(worker_config)

        parameter_server = ParameterServer(model_config, lazy=True) if rank == 0 else None
        data_loader = _seeded_loader(data_config, seed)
        info("created data loader")

        alloc_type = allocator_config.get("type", "even")
        alloc_opts = {k: allocator_config[k] for k in ("solver", "granularity", "comm_aware")
                      if k in allocator_config}
        model_benchmarker = device_benchmarker = None
        if alloc_type in ("dynamic", "optimal"):
            benchmark_cfg = copy.deepcopy(allocator_config["benchmark_config"])
            mcfg = benchmark_cfg["model"]
            data_cfg_for_model = mcfg.pop("data_generator_cfg")
            gen_type = data_cfg_for_model.pop("generator_type")
            model_benchmarker = ModelBenchmarker(
                model_config=model_config,
                data_generator=build_data_generator(gen_type, **data_cfg_for_model), **mcfg)
            dcfg = benchmark_cfg["device"]
            data_cfg_for_device = dcfg.pop("data_generator_cfg", None)
            gen = None
            if data_cfg_for_device is not None:
                gen_type = data_cfg_for_device.pop("generator_type")
                gen = build_data_generator(gen_type, **data_cfg_for_device)
            device_benchmarker = DeviceBenchmarker(worker_manager=worker_manager,
                                                   data_generator=gen, **dcfg)
        allocator = Allocator(model_cfg=model_config, worker_manager=worker_manager,
                              model_benchmarker=model_benchmarker,
                              device_benchmarker=device_benchmarker, logger=logger, **alloc_opts)
        try:
            worker_manager = allocator.allocate(
                alloc_type, virtual_stages=int(allocator_config.get("virtual_stages", 1)))
        except Exception:
            info("allocation FAILED:\n" + traceback.format_exc())
            raise
        info({"dynamic": "dynamically allocated model layers based on benchmarking",
              "optimal": "use optimal strategy to allocate model layers"}.get(
                  alloc_type, "Evenly allocated model layers"))
        for worker in worker_manager.worker_pool:
            info("rank: {}, number of layers: {}".format(worker.rank, len(worker.model_config)))

        model = RpcModel(worker_manager=worker_manager, this_rank=rank)
        info("created model")
        # optional learning-rate schedule / global-norm gradient clipping (None = off)
        step_cfg = dict(lr_schedule=train_config.get("lr_schedule_cfg"),
                        grad_clip=train_config.get("grad_clip_cfg"))
        optimizer = build_optimizer(model.optim_module, dict(train_config["optim_cfg"]), **step_cfg)
        info("created distrubted optimizer")
        runner = Runner(model=model, parameter_server=parameter_server,
                        worker_manager=worker_manager, optimizer=optimizer,
                        loss_cfg=dict(train_config["loss_cfg"]),
                        timer_cfg=dict(train_config["timer_config"]),
                        logging_cfg=dict(logging_config), device=device,
                        **dict(train_config["runner_cfg"]))
        info("created runner")
        def allocator_factory(pool):
            """Same benchmarkers / options as the initial allocation, around a copy of the pool
            (used by ReallocateHook to re-benchmark and re-allocate during training)."""
            mb = model_benchmarker
            db = None
            if device_benchmarker is not None:
                db = copy.copy(device_benchmarker)
                db._worker_manager = pool
            return Allocator(model_cfg=model_config, worker_manager=pool, model_benchmarker=mb,
                             device_benchmarker=db, logger=logger, **alloc_opts)

        for cfg in train_config.get("hook_config", []):
            cfg = dict(cfg)
            if cfg.get("type") == "ReallocateHook":
                if model_benchmarker is None:
                    info("ReallocateHook needs allocator_config.type dynamic|optimal: skipped")
                    continue
                cfg.setdefault("allocator_factory", allocator_factory)
                cfg.setdefault("optimizer_cfg", dict(train_config["optim_cfg"]))
                cfg.setdefault("lr_schedule", step_cfg["lr_schedule"])
                cfg.setdefault("grad_clip", step_cfg["grad_clip"])
                cfg.setdefault("allocate_type", alloc_type)
            runner.register_hook(build_hook(cfg.pop("type"), **cfg))
        info("register hooks")
        runner.train(data_loader)
        runner.engine.close()
    except Exception:
        traceback.print_exc()
        status = 1
    finally:
        try:
            if dist.is_initialized():
                dist.destroy_process_group()
        except Exception:
            pass
    print("finish (rank {}, status {})".format(rank, status), flush=True)
    return status


def parse_args(argv=None):
    parser = argparse.ArgumentParser()
    parser.add_argument("-c", "--config", type=str, required=True, help="path to config file")
    parser.add_argument("-p", "--port", type=int, default=29500)
    parser.add_argument("--spawn", type=int, default=0,
                        help="spawn N local processes instead of relying on a launcher")
    parser.add_argument("--backend", type=str, default=None, choices=[None, "nccl", "gloo"])
    return parser.parse_args(argv)


def _entry(rank: int, world_size: int, args) -> int:
    config = load_config(args.config)
    rpc_config = dict(config.get("rpc_config", {}))
    host_file = "./HOST"
    if osp.exists(host_file):  # reference convention (experiment/launch.py:212-217)
        with open(host_file, "r") as f:
            rpc_config["MASTER_ADDR"] = f.readline().strip()
    rpc_config.setdefault("MASTER_ADDR", os.environ.get("MASTER_ADDR", "127.0.0.1"))
    if rpc_config["MASTER_ADDR"] == "localhost":
        rpc_config["MASTER_ADDR"] = "127.0.0.1"
    rpc_config["MASTER_PORT"] = os.environ.get("MASTER_PORT", args.port)
    os.environ["MASTER_ADDR"] = str(rpc_config["MASTER_ADDR"])
    os.environ["MASTER_PORT"] = str(rpc_config["MASTER_PORT"])
    return run_process(rank=rank, world_size=world_size, rpc_config=rpc_config,
                       model_config=config["model_config"], data_config=config["data_config"],
                       logging_config=config["logging_config"],
                       allocator_config=config["allocator_config"],
                       train_config=config["train_config"], worker_config=config["worker_config"],
                       backend=args.backend)


def _spawn_entry(local_rank: int, world_size: int, args) -> None:
    os.environ["RANK"] = str(local_rank)
    os.environ["LOCAL_RANK"] = str(local_rank)
    os.environ["WORLD_SIZE"] = str(world_size)
    code = _entry(local_rank, world_size, args)
    if code != 0:
        sys.exit(code)


def main(argv=None) -> int:
    args = parse_args(argv)
    if args.spawn and args.spawn > 0:
        import torch.multiprocessing as mp

        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ["MASTER_PORT"] = str(args.port)
        mp.spawn(_spawn_entry, args=(args.spawn, args), nprocs=args.spawn, join=True)
        return 0
    rank, world_size = _discover_rank()
    return _entry(rank, world_size, args)


if __name__ == "__main__":
    sys.exit(main())
