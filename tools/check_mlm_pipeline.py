"""Masked-language-model pipeline check (run under torchrun): trains a BERT with the
BertTailForMaskedLM head and MaskedLMLoss for a few steps on SynthMLMDataset and prints the
per-step losses of the last stage as one JSON line (``CHECK {...}``), so that a 1-GPU run and
pipelines cut at different places can be compared (dropout off => the same math everywhere).

    --cut blocks   an even split of whole blocks: the cut sits between two blocks, where the
                   stage boundary is fused (peer-memory slots, one CUDA graph per step)
    --cut head     the last stage is the head alone: the cut sits directly in front of it, and the
                   boundary runs over torch.distributed p2p (the head does not consume a fused slot)
    --max-predictions P
                   the sparse head: only the labelled positions (at most P per sequence) are
                   decoded; the labels reach the head on the last stage
    --virtual-stages v
                   a looped pipeline (v chunks per rank on a ring; fused ring by default,
                   torch.distributed p2p with --boundary nccl): the head sits in the last chunk of
                   the last rank
    --max-grad-norm x
                   global-norm gradient clipping (the norm is printed per step: ``grad_norms``)
    --tie          the decoder weight is tied to the word embeddings: on 2+ GPUs the last stage
                   holds a replica of the first stage's table; the checksum of both copies is
                   printed for every step (``tied_checksums``: [first rank's, last rank's])
    --nsp          the pretraining head (BertTailForPreTraining: masked-LM + next-sentence
                   prediction) with PreTrainingLoss on SynthPretrainingDataset
    --qa           the question-answering head (BertTailForQuestionAnswering) with
                   QuestionAnsweringLoss on SynthQADataset at --seq tokens (default 384 with --qa)
"""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import skycomputing_b200 as sky  # noqa: E402
from skycomputing_b200.dynamics.allocator import group_units  # noqa: E402
from skycomputing_b200.models import BertConfig, set_backend  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cut", default="blocks", choices=["blocks", "head"])
    ap.add_argument("--boundary", default="auto")
    ap.add_argument("--micro-batches", type=int, default=2)
    ap.add_argument("--layers", type=int, default=4)
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--max-predictions", type=int, default=None)
    ap.add_argument("--tie", action="store_true")
    ap.add_argument("--nsp", action="store_true")
    ap.add_argument("--qa", action="store_true")
    ap.add_argument("--seq", type=int, default=None)
    ap.add_argument("--optim", default="SGD")
    ap.add_argument("--virtual-stages", type=int, default=1)
    ap.add_argument("--max-grad-norm", type=float, default=None)
    a = ap.parse_args()
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    set_backend("native")
    torch.manual_seed(7)
    cfg = BertConfig(30528, hidden_size=1024, num_hidden_layers=a.layers, num_attention_heads=16,
                     intermediate_size=4096, hidden_dropout_prob=0.0,
                     attention_probs_dropout_prob=0.0)
    enc = [dict(layer_type="BertLayer_Head", config=cfg.__dict__),
           dict(layer_type="BertLayer_Body", config=cfg.__dict__),
           dict(layer_type="BertLayer_Tail", config=cfg.__dict__)] * a.layers
    head = dict(layer_type="BertTailForPreTraining" if a.nsp else "BertTailForMaskedLM",
                config=cfg.__dict__)
    if a.qa:
        head = dict(layer_type="BertTailForQuestionAnswering", config=cfg.__dict__)
    if a.max_predictions is not None:
        head["max_predictions"] = a.max_predictions
    if a.tie:
        head["tie_word_embeddings"] = True
    model_config = [dict(layer_type="BertEmbeddings", config=cfg.__dict__)] + enc + [head]
    workers = [dict(name=f"gpu-{i}", server_config={}, device=i,
                    extra_config=dict(module_to_cuda=True, cuda_device=local, slowdown=0,
                                      mem_limit=-1, timer_config=dict(root="/tmp/sky_check_mlm")))
               for i in range(world)]
    wm = sky.WorkerManager(first_rank=0)
    wm.load_worker_pool_from_config(workers)
    if a.virtual_stages > 1 and world > 1:
        wm = sky.Allocator(model_config, wm, granularity="block").allocate(
            "even", virtual_stages=a.virtual_stages)
    elif a.cut == "blocks" or world == 1:
        wm = sky.Allocator(model_config, wm, granularity="block").allocate("even")
    else:
        # every layer but the head on the first world - 1 stages, the head alone on the last
        alloc = sky.Allocator(model_config, wm, granularity="layer")
        units = group_units(model_config, "layer")
        n = len(units)
        body = [round(i * (n - 1) / (world - 1)) for i in range(world)]
        wm = alloc._assign(list(range(world)), body + [n], units)
    # identical initial weights regardless of the partition: seed per GLOBAL layer index
    model = sky.RpcModel(wm, this_rank=rank)
    for mod in model.model:
        if not mod.is_local:
            continue
        b0 = mod.layer_range[0]
        for off, layer in enumerate(mod.module.layers.children()):
            g = torch.Generator(device="cpu").manual_seed(1000 + b0 + off)
            # a tied decoder is the table (one GPU) or its replica, synchronised by the engine
            skip = {id(layer.decoder.weight)} if getattr(layer, "tie_word_embeddings", False) else set()
            with torch.no_grad():
                for p in layer.parameters():
                    if id(p) in skip:
                        continue
                    p.copy_((torch.randn(p.shape, generator=g) * 0.02).to(p.device))
                for n_, p in layer.named_parameters():
                    if n_.endswith("LayerNorm.weight"):
                        p.fill_(1.0)
    lr = 0.01 if a.optim == "SGD" else 1e-3
    loss = ("QuestionAnsweringLoss" if a.qa else "PreTrainingLoss" if a.nsp else "MaskedLMLoss")
    opt = sky.build_optimizer(model.optim_module, dict(optim_type=a.optim, lr=lr),
                              grad_clip=(dict(max_norm=a.max_grad_norm)
                                         if a.max_grad_norm is not None else None))
    runner = sky.Runner(model=model, parameter_server=None, worker_manager=wm, optimizer=opt,
                        max_epochs=1, max_iters=10 ** 9, loss_cfg=dict(type=loss),
                        timer_cfg=dict(root="/tmp/sky_check_mlm"), logging_cfg=None,
                        micro_batches=a.micro_batches, schedule="1f1b", boundary=a.boundary,
                        device=dev)
    model.train(True)
    seq = a.seq or (384 if a.qa else 128)
    if a.qa:
        ds = sky.SynthQADataset(num_samples=a.batch * 2, max_seq_length=seq, vocab_size=30528,
                                seed=3)
    else:
        data_cls = sky.SynthPretrainingDataset if a.nsp else sky.SynthMLMDataset
        ds = data_cls(num_samples=a.batch * 2, max_seq_length=seq, vocab_size=30528, seed=3)
    batches = list(torch.utils.data.DataLoader(ds, batch_size=a.batch))
    losses, checksums, norms = [], [], []
    eng = runner.engine
    for step in range(a.steps):
        data, labels = batches[step % 2]
        out = runner.train_iteration(data, labels)
        if out is not None:
            losses.append(out)
        if a.max_grad_norm is not None:
            norms.append(opt.scalars()["grad_norm"])
        if a.tie:
            # the bits of this rank's copy of the table (table on the first rank, replica on the
            # last): equal checksums on both ranks every step
            table, head_mod = eng._local_tied_params()
            copy = head_mod.decoder.weight if (head_mod is not None and not eng.is_first) else table
            checksums.append(None if copy is None else
                             int(copy.detach().view(torch.int32).to(torch.int64).sum()))
    torch.cuda.synchronize()
    looped = getattr(model, "virtual_stages", 1) > 1
    info = dict(cut=a.cut, world=world, fused=(eng.in_fused or eng.out_fused),
                layers=[len(w.model_config) for w in wm.worker_pool],
                last_stage_first_layer=None if looped else model_config[
                    max(w.layer_range for w in wm.worker_pool)[0]]["layer_type"],
                engine=type(eng).__name__, grad_norms=norms,
                graph=eng._graph is not None, losses=losses,
                err=eng.fused.error_code() if eng.fused is not None else 0,
                first=eng.is_first, checksums=checksums,
                tied_exchange=("peer" if eng._tied_exchange is not None else
                               "all_reduce" if eng._tied_group is not None else None))
    gathered = [None] * world
    dist.all_gather_object(gathered, info)
    if rank == 0:
        last = [g for g in gathered if g["losses"]][0]
        last["fused_any"] = any(g["fused"] for g in gathered)
        last["graph_all"] = all(g["graph"] for g in gathered)
        last["err_any"] = max(g["err"] for g in gathered)
        if a.tie:
            first = [g for g in gathered if g["first"]][0]
            last["tied_checksums"] = [first["checksums"], last["checksums"]]
            last["tied_exchange"] = first["tied_exchange"]
        print("CHECK " + json.dumps(last), flush=True)
    eng.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
