"""Evaluate a small BERT over an N-GPU pipeline (one process per GPU) and print the metrics.

    python -m torch.distributed.run --nproc-per-node N tools/check_eval.py [--steps K]

Rank 0 prints one line ``CHECK {json}``: the metrics of an evaluation before training (seeded
weights: the same on any number of stages), after ``--steps`` training steps, and whether the
training step used fused peer-memory boundaries.  ``--boundary nccl`` trains over NCCL p2p instead.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import skycomputing_b200 as sky  # noqa: E402


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=4)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--micro-batches", type=int, default=2)
    ap.add_argument("--boundary", default="auto")
    args = ap.parse_args()
    rank = int(os.environ.get("RANK", 0))
    world = int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    cfg = sky.BertConfig(1000, hidden_size=256, num_hidden_layers=args.layers, num_attention_heads=4,
                         intermediate_size=1024, hidden_dropout_prob=0.1,
                         attention_probs_dropout_prob=0.1)
    enc = [dict(layer_type="BertLayer_Head", config=cfg.__dict__),
           dict(layer_type="BertLayer_Body", config=cfg.__dict__),
           dict(layer_type="BertLayer_Tail", config=cfg.__dict__)] * args.layers
    mc = ([dict(layer_type="BertEmbeddings", config=cfg.__dict__)] + enc
          + [dict(layer_type="BertPooler", config=cfg.__dict__),
             dict(layer_type="BertTailForClassification", hidden_dropout_prob=0.1,
                  hidden_size=256, num_classes=3)])
    wm = sky.WorkerManager(first_rank=0)
    wm.load_worker_pool_from_config([dict(
        name=f"gpu-{i}", server_config={}, device=i,
        extra_config=dict(module_to_cuda=True, cuda_device=i, slowdown=0, mem_limit=-1,
                          timer_config=dict(root="/tmp/sky_check_eval"))) for i in range(world)])
    wm = sky.Allocator(mc, wm, granularity="block").allocate("even")
    model = sky.RpcModel(wm, this_rank=rank)
    for mod in model.model:
        if not mod.is_local:
            continue
        for off, layer in enumerate(mod.module.layers.children()):
            gen = torch.Generator().manual_seed(500 + mod.layer_range[0] + off)
            with torch.no_grad():
                for n, p in layer.named_parameters():
                    p.copy_((torch.randn(p.shape, generator=gen) * 0.02).to(p.device))
                    if n.endswith("LayerNorm.weight"):
                        p.fill_(1.0)
    opt = sky.build_optimizer(model.optim_module, dict(optim_type="SGD", lr=0.05, momentum=0.9))
    runner = sky.Runner(model=model, parameter_server=None, worker_manager=wm, optimizer=opt,
                        max_epochs=1, max_iters=args.steps, loss_cfg=dict(type="CrossEntropyLoss"),
                        timer_cfg=dict(root="/tmp/sky_check_eval"), logging_cfg=None,
                        micro_batches=args.micro_batches, boundary=args.boundary, device=dev)
    # token ids must stay below the model's vocabulary: the embedding kernels do not check them
    dev_set = sky.SynthMNLIDataset(num_samples=3 * args.batch + 5, max_seq_length=128,
                                   vocab_size=cfg.vocab_size, seed=11,
                                   label_rule="token")
    dev_loader = torch.utils.data.DataLoader(dev_set, batch_size=args.batch)
    before = runner.evaluate(dev_loader, name="dev")
    train = sky.SynthMNLIDataset(num_samples=args.batch * args.steps, max_seq_length=128,
                                 vocab_size=cfg.vocab_size, seed=3,
                                 label_rule="token")
    runner.train(torch.utils.data.DataLoader(train, batch_size=args.batch, drop_last=True))
    after = runner.evaluate(dev_loader, name="dev")
    fused = runner.engine.fused is not None
    flags = [None] * world
    if world > 1:
        dist.all_gather_object(flags, (fused, before, after))
    else:
        flags = [(fused, before, after)]
    runner.engine.close()
    if rank == 0:
        print("CHECK " + json.dumps(dict(fused_any=any(f[0] for f in flags), before=before,
                                         after=after,
                                         same_on_all_ranks=all(f[1:] == flags[0][1:] for f in flags))),
              flush=True)
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
