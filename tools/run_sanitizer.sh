#!/bin/bash
# compute-sanitizer over the kernel numerics tests (SURVEY §5.2: the in-kernel producer / consumer
# flag protocol, the mbarrier pipelines and the DSMEM statistics exchange are the race surface).
#   tools/run_sanitizer.sh [memcheck|racecheck|synccheck|initcheck] [suite]
# suite:  gemm     wgmma GEMM incl. the GEMM + LayerNorm cluster kernel
#         rows     LayerNorm fwd/bwd, column sums, softmax-CE, fused optimizers
#         attn     attention fwd/bwd
#         layers   embeddings + block + pooler + classifier through the layer classes (embed_fwd /
#                  embed_bwd / small_linear kernels) and the flag handshake (peer_copy_signal,
#                  wait_flags, flag-gated GEMM) on one GPU
#         mlm      the sparse masked-language-model slot kernels (mlm_gather / mlm_scatter) over
#                  the shape grid, and one graph replayed with different label counts
#         tied     the tied word-embedding gradient exchange (tied_grad_push / tied_grad_reduce)
#                  in loopback on one GPU, and the tied masked-language-model head
#         pretrain the pretraining head's kernels: mlm_scatter with the [CLS]-row gradient,
#                  cls_grad_add, softmax_ce on the next-sentence labels, and the native head
#                  forward / backward
#         qa       the question-answering kernels: qa_logits_fwd / qa_logits_bwd (+ finalize),
#                  softmax_ce on the start / end rows, qa_span_eval, and their graph replays
#         all      everything above (default)
# Runs on ONE GPU; reports land in bench_out/sanitizer_<tool>_<suite>.log.  The sanitizer slows
# kernels 10-100x: the 4 s flag-wait timeouts are only meaningful under memcheck / synccheck.
set -uo pipefail
TOOL=${1:-memcheck}
SUITE=${2:-all}
mkdir -p bench_out
run() {  # name, pytest args...
  local name=$1; shift
  compute-sanitizer --tool "$TOOL" --print-limit 50 --error-exitcode 7 \
    --log-file "bench_out/sanitizer_${TOOL}_${name}.log" \
    python -m pytest -x -q -p no:cacheprovider "$@" 2>&1 | tail -3
  echo "[sanitizer] tool=$TOOL suite=$name exit=$? $(grep -c 'ERROR SUMMARY: 0 errors' bench_out/sanitizer_${TOOL}_${name}.log) clean-summaries"
  tail -n 2 "bench_out/sanitizer_${TOOL}_${name}.log"
}
case "$SUITE" in gemm|all)
  run gemm tests/test_kernels_gpu.py -k "(gemm_kk and 1024-1024-1024) or gelu_dual or residual_and_dgelu or dgrad_layout or wgrad_layout or layernorm_epilogue" ;;
esac
case "$SUITE" in rows|all)
  run rows tests/test_kernels_gpu.py tests/test_optim_gpu.py -k "layernorm_fwd_bwd or colsum or softmax_ce or dropout_mask_consistent or fused_optimizer" ;;
esac
case "$SUITE" in attn|all)
  run attn tests/test_kernels_gpu.py -k "attention" ;;
esac
case "$SUITE" in mlm|all)
  run mlm tests/test_mlm_sparse_gpu.py -k "gather_and_scatter or different_label_counts" ;;
esac
case "$SUITE" in tied|all)
  run tied tests/test_mlm_tied_gpu.py -k "loopback or reject_bad_arguments or matches_eager" ;;
esac
case "$SUITE" in layers|all)
  run layers tests/test_layers_gpu.py tests/test_kernels_gpu.py -k "embeddings_pooler_classifier or handshake or signals_panels" ;;
esac
case "$SUITE" in pretrain|all)
  run pretrain tests/test_pretraining_gpu.py -k "scatter_joins or next_sentence_softmax_ce or native_head_matches" ;;
esac
case "$SUITE" in qa|all)
  run qa tests/test_qa_gpu.py -k "against_fp64 or matches_the_torch_accumulator or replays_are_bit_equal_and_append" ;;
esac
