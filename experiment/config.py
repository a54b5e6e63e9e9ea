"""Example config, same knobs as the reference's experiment/config.py (PROJECT, ALLOCATE_TYPE,
CORE_NUM, LAYER_NUM) with synthetic MNLI-shaped data (no network for GLUE) and env overrides so
the five BASELINE.json configs are this one file:

  1. 4-layer BERT, CORE_NUM=2, even, CPU/gloo:
       LAYER_NUM=4 CORE_NUM=2 DEVICE=cpu python -m skycomputing_b200.launch -c experiment/config.py --spawn 1
  2. BERT-large even on 8xH100:
       LAYER_NUM=24 CORE_NUM=9 torchrun --nproc-per-node 8 -m skycomputing_b200.launch -c experiment/config.py
  3. ... ALLOCATE_TYPE=dynamic     4. LAYER_NUM=160 ALLOCATE_TYPE=optimal
  5. SLOW_RANK=3 SLOWDOWN=1.0 ALLOCATE_TYPE=dynamic   (device-side throttle on one GPU)

CORE_NUM keeps the reference meaning "workers + 1 central server"; WORKER_NUM = CORE_NUM - 1
processes are launched and rank 0 doubles as the central server.
"""
import os
import os.path as osp

from skycomputing_b200.models.bert import BertConfig

PROJECT = os.getenv("PROJECT", "/tmp/skycomputing_b200")
ALLOCATE_TYPE = os.getenv("ALLOCATE_TYPE", "even")          # even | dynamic | optimal
CORE_NUM = int(os.getenv("CORE_NUM", "2"))                   # workers + 1
LAYER_NUM = int(os.getenv("LAYER_NUM", "4"))
DEVICE = os.getenv("DEVICE", "auto")                         # auto | cpu | cuda
BATCH_SIZE = int(os.getenv("BATCH_SIZE", "32"))
MICRO_BATCHES = int(os.getenv("MICRO_BATCHES", "1"))
MAX_ITERS = int(os.getenv("MAX_ITERS", "30"))
SLOW_RANK = int(os.getenv("SLOW_RANK", "-1"))
SLOWDOWN = float(os.getenv("SLOWDOWN", "0"))
# optional learning-rate schedule (constant | linear | cosine, HF transformers formulas) and
# global-norm gradient clipping; unset = constant lr, no clipping
LR_SCHEDULE = os.getenv("LR_SCHEDULE")
WARMUP_STEPS = int(os.getenv("WARMUP_STEPS", "0"))
TOTAL_STEPS = int(os.getenv("TOTAL_STEPS", str(MAX_ITERS)))
MAX_GRAD_NORM = float(os.getenv("MAX_GRAD_NORM")) if os.getenv("MAX_GRAD_NORM") else None
# EVAL_EVERY=N: train on the learnable synthetic task (label_rule="token") and evaluate on a
# held-out split of it (EVAL_SAMPLES samples of another seed) every N iterations and after the
# run; unset = random labels, no evaluation
EVAL_EVERY = int(os.getenv("EVAL_EVERY")) if os.getenv("EVAL_EVERY") else None
EVAL_SAMPLES = int(os.getenv("EVAL_SAMPLES", "256"))
TINY = os.getenv("TINY", "0") == "1"                          # shrink the geometry for CPU smoke runs
# TASK=mlm: masked-language-model pretraining (RoBERTa style, no next-sentence head) on the
# learnable SynthMLMDataset with a BertTailForMaskedLM head and MaskedLMLoss; the vocabulary is
# padded to a multiple of 8 (30522 -> 30528) for the head's GEMMs.  Default: classification
TASK = os.getenv("TASK", "cls")
if TASK not in ("cls", "mlm"):
    raise ValueError("TASK must be 'cls' or 'mlm', got {!r}".format(TASK))
# MLM_MAX_PREDICTIONS=P (TASK=mlm): the head decodes only the labelled positions, at most P per
# sequence (P >= round(0.15 * (SEQ_LEN - 2)): 20 at 128 tokens); unset = every position decoded
MLM_MAX_PREDICTIONS = int(os.getenv("MLM_MAX_PREDICTIONS")) if os.getenv("MLM_MAX_PREDICTIONS") else None

_config = BertConfig.bert_large()                              # wwm_uncased_L-24_H-1024_A-16 geometry
if TINY:
    _config = BertConfig(1000, hidden_size=64, num_hidden_layers=LAYER_NUM, num_attention_heads=4,
                         intermediate_size=128, max_position_embeddings=128)
_SEQ = int(os.getenv("SEQ_LEN", "128" if not TINY else "16"))
if TASK == "mlm":
    _config.vocab_size = (_config.vocab_size + 7) // 8 * 8

_ENCODER = [
    dict(layer_type="BertLayer_Head", config=_config.__dict__),
    dict(layer_type="BertLayer_Body", config=_config.__dict__),
    dict(layer_type="BertLayer_Tail", config=_config.__dict__),
] * LAYER_NUM

_TAIL = [
    dict(layer_type="BertPooler", config=_config.__dict__),
    dict(layer_type="BertTailForClassification",
         hidden_dropout_prob=_config.hidden_dropout_prob,
         hidden_size=_config.hidden_size, num_classes=3),
]
if TASK == "mlm":
    _TAIL = [dict(layer_type="BertTailForMaskedLM", config=_config.__dict__)]
    if MLM_MAX_PREDICTIONS is not None:
        _TAIL[0]["max_predictions"] = MLM_MAX_PREDICTIONS

model_config = [dict(layer_type="BertEmbeddings", config=_config.__dict__)] + _ENCODER + _TAIL

rpc_config = dict(MASTER_ADDR="127.0.0.1", MASTER_PORT="29500", GLOO_SOCKET_IFNAME="ipogif0")

_LOG_ROOT = f"{PROJECT}/logs/{CORE_NUM}nodes_{LAYER_NUM}layers/{ALLOCATE_TYPE}"
logging_config = dict(mode="a", filename=osp.join(_LOG_ROOT, "allocation.log"))

WORKER_NUM = CORE_NUM - 1
_use_cuda = DEVICE != "cpu"
worker_config = []
for _i in range(1, WORKER_NUM + 1):
    worker_config.append(
        dict(
            name=f"gpu-{_i}",
            server_config=dict(host="localhost", port="8001"),
            extra_config=dict(
                slowdown=SLOWDOWN if (_i - 1) == SLOW_RANK else 0,
                logging_config=dict(mode="a", filename=osp.join(_LOG_ROOT, f"node-{_i}-train.log")),
                mem_limit=-1,
                cuda_device=0,
                module_to_cuda=_use_cuda,
                output_to_cpu=False,
                timer_config=dict(root=_LOG_ROOT),
            ),
        )
    )

data_config = dict(
    dataset_cfg=dict(type="SynthMNLIDataset", num_samples=BATCH_SIZE * (MAX_ITERS + 2),
                     max_seq_length=_SEQ, vocab_size=_config.vocab_size, num_classes=3, seed=0),
    dataloader_cfg=dict(batch_size=BATCH_SIZE, shuffle=True, num_workers=0, drop_last=True),
)
if TASK == "mlm":
    data_config["dataset_cfg"] = dict(type="SynthMLMDataset", num_samples=BATCH_SIZE * (MAX_ITERS + 2),
                                      max_seq_length=_SEQ, vocab_size=_config.vocab_size, seed=0)
    if EVAL_EVERY is not None:  # the held-out split: another seed of the same task
        data_config["eval_datasets"] = dict(
            dev=dict(type="SynthMLMDataset", num_samples=EVAL_SAMPLES, max_seq_length=_SEQ,
                     vocab_size=_config.vocab_size, seed=1))
elif EVAL_EVERY is not None:
    # a learnable task (label = first token after [CLS] mod 3) for training and the held-out split,
    # so that the dev accuracy measures something; random labels stay at chance
    data_config["dataset_cfg"]["label_rule"] = "token"
    data_config["eval_datasets"] = dict(
        dev=dict(type="SynthMNLIDataset", num_samples=EVAL_SAMPLES, max_seq_length=_SEQ,
                 vocab_size=_config.vocab_size, num_classes=3, seed=1, label_rule="token"))

allocator_config = dict(
    type=ALLOCATE_TYPE,
    granularity=os.getenv("GRANULARITY", "block"),
    solver=os.getenv("SOLVER", "heuristic"),
    # COMM_AWARE=1: charge every cut boundary-bytes / link bandwidth (sizes from the model
    # benchmarker); matters at GRANULARITY=layer, where a cut after BertLayer_Body ships 5x
    comm_aware=os.getenv("COMM_AWARE", "0") == "1",
    # VIRTUAL_STAGES=v > 1: looped pipeline, every worker runs v non-adjacent chunks of the model
    # (pipeline fill / drain shrink by v; parallel/pipeline_looped.py)
    virtual_stages=int(os.getenv("VIRTUAL_STAGES", "1")),
    benchmark_config=dict(
        model=dict(device="cpu", param_scale=2,
                   data_generator_cfg=dict(generator_type="DataloaderGenerator",
                                           generator_cfg=data_config)),
        device=dict(
            # proxy="bert_block": C++ loop over the block's real forward + backward kernels (GPU only);
            # proxy="model": the reference's Conv2d stack (parity, also works on CPU)
            proxy=os.getenv("BENCH_PROXY", "bert_block" if _use_cuda else "model"),
            model_config=[dict(layer_type="Conv2d", in_channels=256 if not TINY else 8,
                               out_channels=256 if not TINY else 8, kernel_size=3, padding=1)] * 10,
            iterations=30 if not TINY else 2,
            warmup=3 if not TINY else 0,
            data_generator_cfg=dict(generator_type="RandomTensorGenerator",
                                    generator_cfg=dict(size=(32, 256, 64, 64) if not TINY
                                                       else (2, 8, 8, 8))),
        ),
    ),
)

train_config = dict(
    optim_cfg=dict(optim_type="SGD", lr=0.001),
    lr_schedule_cfg=(dict(type=LR_SCHEDULE, warmup_steps=WARMUP_STEPS, total_steps=TOTAL_STEPS)
                     if LR_SCHEDULE else None),
    grad_clip_cfg=dict(max_norm=MAX_GRAD_NORM) if MAX_GRAD_NORM is not None else None,
    loss_cfg=dict(type="MaskedLMLoss" if TASK == "mlm" else "CrossEntropyLoss"),
    runner_cfg=dict(max_epochs=1, max_iters=MAX_ITERS, micro_batches=MICRO_BATCHES),
    hook_config=[dict(type="StopHook", root=_LOG_ROOT), dict(type="DistributedTimerHelperHook")]
    # REALLOCATE_EVERY=N: re-benchmark the devices and re-run the allocator every N iterations,
    # migrating layers when the predicted bottleneck improves (needs ALLOCATE_TYPE dynamic|optimal)
    + ([dict(type="ReallocateHook", interval=int(os.getenv("REALLOCATE_EVERY")))]
       if os.getenv("REALLOCATE_EVERY") else []),
    timer_config=dict(root=_LOG_ROOT),
)
if EVAL_EVERY is not None:
    train_config["eval_cfg"] = dict(interval=EVAL_EVERY, at_end=True)
