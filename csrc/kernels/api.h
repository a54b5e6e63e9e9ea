// C++ launch API of the sm_90a kernel library (no torch dependency: compiled by nvcc alone,
// bound to Python in csrc/bindings_cuda.cpp).  All launchers are asynchronous on `stream`.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace sky {

// ---------------------------------------------------------------------------------------------
// GEMM  out[M,N] = epilogue( sum_k A[m,k] * B[n,k] )   bf16 operands, fp32 accumulation in registers
// ---------------------------------------------------------------------------------------------
enum GemmAct : int { ACT_NONE = 0, ACT_GELU = 1, ACT_DGELU_MUL_AUX = 2, ACT_TANH = 3 };

struct GemmArgs {
  const void* A = nullptr;  // bf16
  const void* B = nullptr;  // bf16
  int M = 0, N = 0, K = 0;
  // a_mn == false: A stored row-major [M, K] (K contiguous), lda = row stride in elements
  // a_mn == true : A stored row-major [K, M] (M contiguous), lda = row stride in elements
  int lda = 0, ldb = 0;
  bool a_mn = false, b_mn = false;

  void* out = nullptr;  // bf16 (default) or fp32 when out_f32; may be a peer-GPU pointer
  int ldo = 0;
  bool out_f32 = false;
  bool accumulate = false;  // out += result (fp32 outputs only)
  void* out2 = nullptr;     // optional bf16 copy of the pre-activation (bias added)
  int ldo2 = 0;

  const float* bias = nullptr;  // [N] fp32
  const void* aux = nullptr;    // bf16 [M,N]: residual (add_aux) or pre-activation (DGELU_MUL_AUX)
  int ldaux = 0;
  int act = ACT_NONE;
  bool add_aux = false;

  float dropout_p = 0.f;                // applied after bias/activation, before add_aux
  const uint64_t* rng_state = nullptr;  // device: {seed, step}; required when dropout_p > 0
  uint32_t rng_stream = 0;              // per-call-site stream id

  // Stage-boundary fusion.  signal_flags[m_blk] (possibly in peer memory) is incremented with
  // release.sys semantics once per finished output tile.  wait_flags[m_blk] (local memory) is
  // polled with acquire.sys by the TMA producer before it loads A rows of that 128-row panel; the
  // expected value is (*wait_epoch) * wait_mult.
  uint32_t* signal_flags = nullptr;
  const uint32_t* wait_flags = nullptr;
  const uint32_t* wait_epoch = nullptr;
  uint32_t wait_mult = 0;
  int* error_flag = nullptr;  // set to non-zero on flag-wait timeout
  // LayerNorm epilogue (ln_gamma != nullptr): out = LN(dropout(A B^T + bias) + aux) * gamma + beta,
  // out2 = the pre-LN sum (bf16, saved for backward), ln_mean / ln_rstd = row statistics.  The
  // N / BLOCK_N CTAs of a 128-row panel (at N = 1024 and BLOCK_N = 256: the CTA pairs of its two
  // 64-row halves) form thread-block clusters (row statistics through DSMEM); `out` may be peer
  // memory, signal_flags[panel] then receives N / BLOCK_N signals.
  const float* ln_gamma = nullptr;
  const float* ln_beta = nullptr;
  float* ln_mean = nullptr;
  float* ln_rstd = nullptr;
  float ln_eps = 1e-12f;
  int block_n = 0;            // 0 = auto (128 or 256)
  int stream_k = -1;          // stream-K schedule: -1 auto, 0 off, 1 on
  int pair = -1;              // -1 auto, 0 single CTAs, 1 = 2-CTA clusters (B multicast), 2 = 4-CTA clusters (A and B multicast)
  // perf triage: 1 = full main loop, the epilogue discards the tile; 2 = epilogue math but no
  // stores; 3 = MMAs only (no TMA loads: the MMAs read stale shared memory), no epilogue; 4 = TMA
  // loads only (no MMAs), no epilogue.  With clusters (pair != 0), 3 and 4 only drop the epilogue.
  int debug = 0;
  int max_ctas = 0;           // 0 = all SMs
  // SGD update in the epilogue of a weight gradient (sgd_master != nullptr).  The fp32 result g (or
  // out + g when accumulate) is NOT stored; the epilogue applies sgd_multi's plain update with it,
  //   sgd_master -= sgd_lr * (g * sgd_grad_scale + sgd_weight_decay * sgd_master),
  // and writes the new value to the bf16 sgd_shadow, both laid out as `out` ([M, N], row stride
  // ldo).  Only with out_f32, a_mn and b_mn, and without bias / aux / out2 / act / dropout / flags
  // or an explicit stream-K or cluster schedule (980); sgd_shadow must be non-null and out,
  // sgd_master and sgd_shadow 16-byte aligned with ldo % 8 == 0 (981).
  float* sgd_master = nullptr;
  void* sgd_shadow = nullptr;
  float sgd_lr = 0.f, sgd_weight_decay = 0.f, sgd_grad_scale = 1.f;
};

// Returns 0 on success, a cudaError_t / CUresult-like code otherwise.
int launch_gemm(const GemmArgs& args, cudaStream_t stream);
int launch_gemm_ln(const GemmArgs& args, cudaStream_t stream);
// tile width the fused LN epilogue would use (0 = use GEMM + standalone LayerNorm instead; with
// `force` only when the kernel cannot run the shape at all) / signals per 128-row panel
int gemm_ln_block_n(int M, int N, bool force = false);
int gemm_ln_tiles_per_panel(int M, int N, bool force = false);
int gemm_tiles_per_panel(int N, int block_n);  // number of signals per 128-row panel
// clusters of the GEMM + LayerNorm kernel for width N and tile width block_n that the device can
// hold at once (cudaOccupancyMaxActiveClusters); *cluster = CTAs per cluster; < 0 on error
int gemm_ln_max_active_clusters(int N, int block_n, int* cluster);
int gemm_pick_block_n(int M, int N);

// ---------------------------------------------------------------------------------------------
// LayerNorm (rows of H), bf16 in/out, fp32 statistics
// ---------------------------------------------------------------------------------------------
struct LayerNormFwdArgs {
  const void* z = nullptr;  // bf16 [M,H]
  void* y = nullptr;        // bf16 [M,H]
  float* mean = nullptr;    // [M]
  float* rstd = nullptr;    // [M]
  const float* gamma = nullptr;
  const float* beta = nullptr;
  int M = 0, H = 0;
  float eps = 1e-12f;
  // optional: wait for 128-row panels written by a peer
  const uint32_t* wait_flags = nullptr;
  const uint32_t* wait_epoch = nullptr;
  uint32_t wait_mult = 0;
  int* error_flag = nullptr;
  // optional: y is (peer) boundary memory; every CTA (8 rows) bumps signal_flags[row/128] once
  // with release.sys, i.e. a 128-row panel is complete at 16 signals (kLnSignalsPerPanel)
  uint32_t* signal_flags = nullptr;
};
constexpr int kLnSignalsPerPanel = 16;
int launch_layernorm_fwd(const LayerNormFwdArgs& a, cudaStream_t stream);

struct LayerNormBwdArgs {
  const void* dy = nullptr;  // bf16 [M,H]
  const void* z = nullptr;   // bf16 [M,H] pre-LN input saved by forward
  const float* mean = nullptr;
  const float* rstd = nullptr;
  const float* gamma = nullptr;
  void* dz = nullptr;         // bf16 [M,H]
  void* dz_dropped = nullptr; // optional bf16 [M,H]: dz * keep/(1-p) with the GEMM-epilogue mask
  float* dgamma = nullptr;    // fp32 [H], accumulated (+=)
  float* dbeta = nullptr;     // fp32 [H], accumulated (+=)
  int M = 0, H = 0;
  float dropout_p = 0.f;
  const uint64_t* rng_state = nullptr;
  uint32_t rng_stream = 0;
  const uint32_t* wait_flags = nullptr;
  const uint32_t* wait_epoch = nullptr;
  uint32_t wait_mult = 0;
  int* error_flag = nullptr;
};
int launch_layernorm_bwd(const LayerNormBwdArgs& a, cudaStream_t stream);
// dgamma += sum_rows dy * xhat, dbeta += sum_rows dy; out2 += sum_rows x2 when x2 != null.
// H % 8 != 0 returns 916.
int launch_ln_param_grad(const void* dy, const void* z, const float* mean, const float* rstd,
                         float* dgamma, float* dbeta, int M, int H, const void* x2, float* out2,
                         cudaStream_t stream);

// y[i] = g[i] * gelu'(h[i])  (bf16, n % 8 == 0): only used when a stage cut separates FFN1 | FFN2
int launch_dgelu_mul(const void* g, const void* h, void* y, long long n, cudaStream_t stream);

// column sums: out[n] += sum_m x[m,n]   (bias gradients)
int launch_colsum(const void* x_bf16, int M, int N, int ldx, float* out, cudaStream_t stream);

// ---------------------------------------------------------------------------------------------
// Attention (head_dim = 64; S = 128 single-tile kernels, any other S % 8 == 0 tiled), wgmma
// ---------------------------------------------------------------------------------------------
struct AttnArgs {
  const void* qkv = nullptr;   // bf16 [B*S, 3*H]  (Q | K | V), head h at columns h*64
  const float* mask = nullptr; // fp32 additive [B, S] or null
  void* ctx = nullptr;         // bf16 [B*S, H] (fwd: output, bwd: saved forward output)
  float* lse = nullptr;        // fp32 [B*heads, S] log2-domain log-sum-exp (fwd: out, bwd: in)
  const void* dctx = nullptr;  // bwd: bf16 [B*S, H]
  void* dqkv = nullptr;        // bwd: bf16 [B*S, 3*H]
  int B = 0, S = 0, heads = 0, head_dim = 0;
  float scale = 0.125f;
  float dropout_p = 0.f;
  const uint64_t* rng_state = nullptr;
  uint32_t rng_stream = 0;
};
int launch_attention_fwd(const AttnArgs& a, cudaStream_t stream);
int launch_attention_bwd(const AttnArgs& a, cudaStream_t stream);
bool attention_supported(int S, int head_dim);

// ---------------------------------------------------------------------------------------------
// Embeddings: word + position + token-type gather, LayerNorm, dropout; and its backward
// ---------------------------------------------------------------------------------------------
struct EmbedArgs {
  const int64_t* input_ids = nullptr;   // [B*S]
  const int64_t* token_type = nullptr;  // [B*S]
  const int64_t* attn_mask = nullptr;   // [B*S] (0/1) or null
  const float* word = nullptr;          // [V,H] fp32 master weights
  const float* pos = nullptr;           // [P,H]
  const float* type = nullptr;          // [T,H]
  const float* gamma = nullptr;
  const float* beta = nullptr;
  void* out = nullptr;        // bf16 [B*S,H]
  float* ext_mask = nullptr;  // fp32 [B*S] = (1-mask)*-10000
  float* xhat = nullptr;      // optional fp32? (unused) kept null
  float* mean = nullptr;      // [B*S]
  float* rstd = nullptr;      // [B*S]
  int B = 0, S = 0, H = 0;
  float eps = 1e-12f;
  float dropout_p = 0.f;
  const uint64_t* rng_state = nullptr;
  uint32_t rng_stream = 0;
};
int launch_embed_fwd(const EmbedArgs& a, cudaStream_t stream);

struct EmbedBwdArgs {
  const void* dout = nullptr;  // bf16 [B*S,H]
  const int64_t* input_ids = nullptr;
  const int64_t* token_type = nullptr;
  const float* word = nullptr;
  const float* pos = nullptr;
  const float* type = nullptr;
  const float* gamma = nullptr;
  const float* mean = nullptr;
  const float* rstd = nullptr;
  float* dword = nullptr;  // fp32 [V,H] (+=, atomics)
  float* dpos = nullptr;
  float* dtype_ = nullptr;
  float* dgamma = nullptr;
  float* dbeta = nullptr;
  int B = 0, S = 0, H = 0;
  int type_rows = 2;  // rows of the token-type table (accumulated in shared memory when <= 4)
  float dropout_p = 0.f;
  const uint64_t* rng_state = nullptr;
  uint32_t rng_stream = 0;
  const uint32_t* wait_flags = nullptr;
  const uint32_t* wait_epoch = nullptr;
  uint32_t wait_mult = 0;
  int* error_flag = nullptr;
};
int launch_embed_bwd(const EmbedBwdArgs& a, cudaStream_t stream);

// ---------------------------------------------------------------------------------------------
// Small dense layers (pooler / classifier) + softmax cross-entropy, CUDA-core (latency bound)
// ---------------------------------------------------------------------------------------------
// y[m,n] = act( sum_k x[m*ldx + k] * w[n,k] + b[n] ); x bf16 or fp32, w/b fp32, y fp32
int launch_small_linear_fwd(const void* x, bool x_bf16, int ldx, const float* w, const float* b,
                            float* y, int M, int N, int K, int act_tanh, float dropout_p,
                            const uint64_t* rng_state, uint32_t rng_stream, cudaStream_t stream);
// dx[m,k] = sum_n dy'[m,n] w[n,k];  dw[n,k] += sum_m dy'[m,n] x[m,k];  db[n] += sum_m dy'[m,n]
// where dy' = dy * (1 - y^2) if act_tanh.  Input dropout mask is re-applied to x and dx.
int launch_small_linear_bwd(const void* x, bool x_bf16, int ldx, const float* w, const float* y,
                            const float* dy, void* dx, bool dx_bf16, int lddx, float* dw, float* db,
                            int M, int N, int K, int act_tanh, float dropout_p,
                            const uint64_t* rng_state, uint32_t rng_stream, cudaStream_t stream);
// loss = mean_m CE(logits[m,:], labels[m]);  dlogits = (softmax - onehot) / M * grad_scale
int launch_softmax_ce(const float* logits, const int64_t* labels, float* loss, float* dlogits,
                      int M, int C, float grad_scale, float* loss_acc, cudaStream_t stream);
// Evaluation accumulator: the header is followed by C x C confusion counters [label * C + pred].
struct EvalAccum {
  double loss_sum;                  // sum of the per-row cross entropies (fp32 rows, fp64 sum)
  unsigned long long count;         // rows with a label in [0, C)
  unsigned long long invalid;       // rows whose label is neither ignore_index nor in [0, C)
  unsigned long long confusion[];   // C * C
};
constexpr int kEvalMaxClasses = 1024;
// Adds one batch of fp32 logits [M, C] (row stride ldl) into *acc: per row lse - logit[label] and
// pred = argmax (first maximum, NaN counts as the maximum).  Rows with label == ignore_index are
// skipped.  One CTA, fixed reduction order: deterministic, no host sync, graph-capturable.
// C > kEvalMaxClasses returns 940.
int launch_classify_eval(const float* logits, int ldl, const int64_t* labels, int M, int C,
                         long long ignore_index, EvalAccum* acc, cudaStream_t stream);

// Vocabulary cross entropy over bf16 logits [M, V] (row stride ldl), the masked-language-model
// loss.  Rows labelled ignore_index are neither read nor counted; n_valid = the other rows.
// Training mode (dlogits != null, acc == null):
//   dlogits = (softmax - onehot) * grad_scale / n_valid as bf16, with row stride ldl; it may be
//   the logits buffer itself (in place), otherwise it must not overlap it.  Ignored rows get an
//   exact 0.  loss_out[0] = mean loss, loss_acc[0] += mean * grad_scale (either may be null).
//   n_valid == 0 gives loss 0 and an all-zero gradient (torch's mean reduction gives NaN).  A
//   label outside [0, V) that is not ignore_index makes the loss NaN and its gradient row 0.
// Eval mode (acc != null, dlogits == null): adds {fp64 loss sum, labelled rows, top-1 correct,
//   invalid labels} into *acc; argmax as torch.argmax (first maximum, NaN is the maximum).
// One CTA per row reads the row from HBM once into shared memory; per-row results are summed by
// one CTA in a fixed order (no float atomics: graph replays are bit-identical); no host sync.
// Launches: 3 in training mode, 2 in eval mode (vocab_ce_launches).  workspace: vocab_ce_workspace_bytes(M), any
// contents; an empty batch (M == 0) may pass null data pointers.  Errors: 950 V outside [1, kVocabCeMaxV], 951 bad shape / null pointer, 952 not
// exactly one of dlogits / acc, 953 dlogits partially overlaps logits.
struct VocabEvalAccum {
  double loss_sum;
  unsigned long long count;    // labelled rows with a label in [0, V)
  unsigned long long correct;  // ... whose argmax is the label
  unsigned long long invalid;  // rows whose label is neither ignore_index nor in [0, V)
};
constexpr int kVocabCeMaxV = 98304;  // the bf16 row must fit in shared memory (192 KiB)
struct VocabCeArgs {
  const void* logits = nullptr;  // bf16
  long long ldl = 0;
  const int64_t* labels = nullptr;
  int M = 0, V = 0;
  long long ignore_index = -100;
  void* dlogits = nullptr;       // bf16, training mode
  float grad_scale = 1.f;
  float* loss_out = nullptr;
  float* loss_acc = nullptr;
  VocabEvalAccum* acc = nullptr;  // eval mode
  void* workspace = nullptr;
};
size_t vocab_ce_workspace_bytes(int M);
int launch_vocab_ce(const VocabCeArgs& a, cudaStream_t stream);
// kernels a successful launch_vocab_ce(a) issues: 3 (training), 2 (eval), fewer when M == 0
int vocab_ce_launches(const VocabCeArgs& a);

// Sparse masked-language-model decoding.  Sequence b owns slots [b*P, (b+1)*P); its labelled
// positions (label != ignore_index), in position order, fill them from the front.
// mlm_gather (one launch, one CTA per sequence):
//   slot_of_row[B*S] (int32) = the row's slot, -1 where the row is not decoded;
//   slot_labels[B*P] = the slot's label, ignore_index in an empty slot; when a sequence has more
//   than P labelled positions the extra ones are dropped and its last slot gets the label V (out
//   of range: the vocab_ce loss turns NaN and the eval accumulator counts it as invalid);
//   x_c[B*P, H] (bf16) = hidden[row_of_slot] (hidden is [B*S, H] bf16), zeros in an empty slot.
// mlm_scatter (one launch): dhidden[r] = dx_c[slot_of_row[r]] for a decoded row, zeros otherwise;
//   every row of dhidden [rows, H] is written exactly once.
// Both: H % 8 == 0, hidden / x_c / dx_c / dhidden 16-byte aligned; integer scans and copies only
// (deterministic), no host sync.  Errors: 960 bad shape (B, S, P >= 1, P <= kMlmMaxPredictions,
// H a positive multiple of 8), 961 null pointer, 962 a bf16 buffer is not 16-byte aligned.
constexpr int kMlmMaxPredictions = 8192;  // slot map of one sequence in shared memory
int launch_mlm_gather(const void* hidden, const int64_t* labels, int B, int S, int H, int P,
                      long long ignore_index, int V, int* slot_of_row, int64_t* slot_labels,
                      void* x_c, cudaStream_t stream);
// With dcls ([rows / S, H] bf16, 16-byte aligned; S divides rows) row b*S, the [CLS] position of
// sequence b, gets dcls[b] added (each lane rounded once from fp32; dcls[b] exactly when the row
// is not decoded): the pooler branch's input gradient joins the head's in the same pass.
int launch_mlm_scatter(const void* dx_c, const int* slot_of_row, long long rows, int H,
                       void* dhidden, cudaStream_t stream, const void* dcls = nullptr, int S = 1);
// cls_grad_add (one launch): dhidden[b*S] += dcls[b] in place (bf16 [B*S, H] and [B, H], lanes
// rounded once from fp32), the dense head's [CLS]-row join.  Errors: 982 bad shape (B, S >= 1, H a
// positive multiple of 8), 983 null pointer, 984 a buffer is not 16-byte aligned.
int launch_cls_grad_add(void* dhidden, const void* dcls, int B, int S, int H, cudaStream_t stream);

// Cross entropy over fp32 logits [M, C] (row stride ldl) with ignore_index, the next-sentence-
// prediction loss.  n_valid = rows whose label is in [0, C).  dlogits [M, C] (contiguous) =
// (softmax - onehot) * grad_scale / n_valid on those rows and an exact 0 on every other row.
// loss[0] = mean over the n_valid rows (0 when n_valid == 0), NaN when any label is neither
// ignore_index nor in [0, C) (such a label is never used as an index); loss_acc[0] += loss *
// grad_scale.  loss / loss_acc may be null.  One CTA, fixed-order fp64 reduction, no host sync,
// graph-capturable.  Errors: 985 bad shape (M < 0, C < 1, ldl < C), 986 null pointer.
int launch_masked_softmax_ce(const float* logits, int ldl, const int64_t* labels, int M, int C,
                             long long ignore_index, float* dlogits, float grad_scale,
                             float* loss, float* loss_acc, cudaStream_t stream);

// Question-answering span head (HF BertForQuestionAnswering's qa_outputs = Linear(H, 2)).
// logits / dlogits are fp32 [B, 2, S]: row 2b holds sequence b's start logits, row 2b + 1 its end
// logits.  labels are int64 [B, kQaLabelCols] per sequence: start, end (the gold answer's first and
// last token), start_lo, start_hi (where a predicted answer may start), end_hi (the last position
// where it may end).  All four kernels use fixed reduction orders and no float atomics (two calls
// or graph replays give identical bits) and never synchronise with the host.
// Errors: 990 bad shape (B, S >= 1, H a positive multiple of 8, B * S within int range,
// max_answer_length >= 1, capacity >= 0), 991 null pointer, 992 hidden / dhidden / w not 16-byte
// aligned.
constexpr int kQaLabelCols = 5;
constexpr int kQaRowsPerCta = 128;  // rows of one partial dW / db in qa_logits_bwd
// logits[b, c, s] = dot(hidden[b*S + s], w[c]) + bias[c] (hidden bf16 [B*S, H], w fp32 [2, H]).
// One launch.
int launch_qa_logits_fwd(const void* hidden, int B, int S, int H, const float* w, const float* b,
                         float* logits, cudaStream_t stream);
// dhidden[r] = g[b, 0, s] * w[0] + g[b, 1, s] * w[1] (bf16, every row written once), dw [2, H] +=
// sum_r g_c[r] hidden[r], db [2] += sum_r g_c[r].  The first launch stores per-128-row partials in
// `workspace` (qa_logits_bwd_workspace_bytes), the second adds them in row-block order (fp64).
int launch_qa_logits_bwd(const void* hidden, const float* dlogits, int B, int S, int H,
                         const float* w, void* dhidden, float* workspace, float* dw, float* db,
                         cudaStream_t stream);
size_t qa_logits_bwd_workspace_bytes(int B, int S, int H);
// Span loss: (mean start CE + mean end CE) / 2, each mean over the sequences whose label is in
// [0, S) (0 without one).  dlogits = d(loss * grad_scale)/dlogits, an exact 0 on a row whose label
// is ignore_index or invalid; any label neither ignore_index nor in [0, S) makes the loss NaN and
// is never used as an index.  loss[0] = the loss, loss_acc[0] += loss * grad_scale (either may be
// null).  One CTA, one launch.
int launch_qa_span_ce(const float* logits, const int64_t* labels, int B, int S,
                      long long ignore_index, float* dlogits, float grad_scale, float* loss,
                      float* loss_acc, cudaStream_t stream);
// Evaluation accumulator of a span head.  Totals over the sequences whose gold start and end are
// both in [0, S); `invalid` counts sequences with a gold label that is neither ignore_index nor in
// [0, S).  Predictions go to pred_spans[cursor + b] / pred_scores[cursor + b] while that is below
// the capacity (else `overflow` is counted); the cursor lives here, so a replayed graph appends.
struct SpanEvalAccum {
  double start_loss_sum;           // lse - logit[gold] of the start rows (fp32 rows, fp64 sum)
  double end_loss_sum;
  double f1_sum;                   // SQuAD token F1 of the best span against the gold interval
  unsigned long long count;
  unsigned long long start_correct;  // argmax (first maximum, NaN is the maximum) == gold start
  unsigned long long end_correct;
  unsigned long long exact;          // best span == gold span
  unsigned long long invalid;
  unsigned long long cursor;         // sequences seen since the last reset
  unsigned long long overflow;       // of them, not stored: past the capacity
};
// Best span of each sequence: the maximum of start[i] + end[j] (one fp32 add; NaN counts as -inf)
// over max(start_lo, 0) <= i <= min(start_hi, S - 1), i <= j <= min(i + L - 1, end_hi, S - 1);
// among equal scores the smallest (i, j) wins; an empty range gives (-1, -1) and score -inf.
// pred_spans int32 [capacity, 2], pred_scores fp32 [capacity].  One CTA, one launch.
int launch_qa_span_eval(const float* logits, const int64_t* labels, int B, int S,
                        int max_answer_length, long long ignore_index, SpanEvalAccum* acc,
                        int* pred_spans, float* pred_scores, long long capacity,
                        cudaStream_t stream);

// ---------------------------------------------------------------------------------------------
// Optimizer / parameter maintenance
// ---------------------------------------------------------------------------------------------
// Multi-tensor fused SGD: p -= lr * (g + wd * p) (optional momentum buffer), then refresh the
// bf16 compute copy and zero the gradient.  `n_tensors` descriptors in device memory.
struct SgdTensor {
  float* p;
  float* g;
  float* mom;         // may be null
  void* p_bf16;       // may be null
  long long numel;
  int skip_zero;      // the first gradient write of the next step OVERWRITES g: do not zero it
  int pad_;
  float* mom2;        // Adam second moment (null for SGD)
};
// Device-side optimizer scalars, written by launch_optim_finalize once per step.  When the
// optimizer kernels get a non-null pointer to it they take `lr` from here (instead of the host
// argument) and multiply the gradient by `clip_coef` first, so that a CUDA graph captured once
// replays a learning-rate schedule and global-norm clipping correctly.
struct OptimScalars {
  float lr;
  float clip_coef;    // min(1, max_norm / (grad_norm + 1e-6)); NaN / 0 propagate as in torch
  float grad_norm;    // global L2 norm of the (scaled) gradients over every pipeline stage
  float local_sumsq;  // this rank's share of grad_norm^2
};
int launch_sgd_multi(const SgdTensor* d_tensors, int n_tensors, long long max_numel, float lr,
                     float momentum, float weight_decay, float grad_scale, bool zero_grad,
                     cudaStream_t stream, const OptimScalars* scalars = nullptr);
// Multi-tensor fused Adam / AdamW (torch.optim.Adam(W) semantics, amsgrad=False): moments in
// `mom` / `mom2`, the step count lives in DEVICE memory (`step`, advanced by the caller with
// launch_advance_counter before this launch) so that the whole update is CUDA-graph capturable.
int launch_adam_multi(const SgdTensor* d_tensors, int n_tensors, long long max_numel, float lr,
                      float beta1, float beta2, float eps, float weight_decay, bool decoupled,
                      const uint64_t* step, float grad_scale, bool zero_grad, cudaStream_t stream,
                      const OptimScalars* scalars = nullptr);
// Sum of squares of g * grad_scale over the descriptors' gradients.  Grid (blocks, n_tensors);
// block (x, y) writes its fp32 partial to partials[y * blocks + x] (no atomics: the result is the
// same on every replay).  `blocks` must come from grad_sumsq_blocks(max_numel).
int grad_sumsq_blocks(long long max_numel);
int launch_grad_sumsq_multi(const SgdTensor* d_tensors, int n_tensors, int blocks,
                            float grad_scale, float* partials, cudaStream_t stream);
// LAMB (You et al. 2019, apex FusedLAMB defaults: adam_w_mode, grad averaging, bias correction,
// no NVLAMB).  One segment per nn.Parameter inside the flat banks, each with its own trust ratio:
//   g = grad * grad_scale * clip_coef,  m = b1 m + (1-b1) g,  v = b2 v + (1-b2) g^2,
//   u = (m / (1-b1^t)) / (sqrt(v / (1-b2^t)) + eps) + wd p,
//   r = ||p|| / ||u|| if use_ratio and both norms > 0, else 1,   p -= lr r u.
// Work is handed out in kLambChunk-element chunks of the segments (chunk c belongs to segment
// chunk_seg[c]); each block takes a contiguous range of chunks.
constexpr int kLambChunk = 16384;
struct LambSegment {
  float* p;           // fp32 master (the segment's first element)
  float* g;           // fp32 gradient
  float* m;           // first moment
  float* v;           // second moment
  void* p_bf16;       // bf16 shadow, may be null
  long long numel;
  float weight_decay; // lambda (0 for a tensor excluded from weight decay)
  int use_ratio;      // apply the trust ratio (lambda != 0)
  int skip_zero;      // leave g as it is: the next step's first wgrad overwrites it
  int vec;            // float4 path (p, g, m, v 16-byte, p_bf16 8-byte aligned); set by lamb_prepare
  int chunk0;         // index of the segment's first chunk
  int n_chunks;
};
// Host side, once per table: checks the segments, sets vec / chunk0 / n_chunks and fills
// chunk_seg[0 .. *n_chunks) (capacity `cap`).  Errors: 970 null pointer, numel < 1, a fp32 pointer
// not 4-byte aligned or more than `cap` / INT_MAX chunks; 972 a bf16 shadow not 2-byte aligned.
int lamb_prepare(LambSegment* segs, int n_segments, int* chunk_seg, long long cap, int* n_chunks);
long long lamb_chunks(long long numel);
// Pass 1: m and v, and the fp32 partials {sum p^2, sum u^2} of every chunk into partials[c]
// (fixed slots, fixed in-block order: bit-identical on every call); zeroes g unless skip_zero.
// Pass 2: r from the segment's partials (summed in fp64 in a fixed order), p -= lr r u (u
// recomputed from the new m, v and the old p), the bf16 shadow from the new p; the block holding a
// segment's first chunk writes its r to ratios[segment].  `step` is the device step counter
// (1-based, advanced before pass 1); with `scalars` lr and clip_coef come from the device.
// Errors: 970 bad table / null buffer, 971 null step counter.
int launch_lamb_moments(const LambSegment* segs, const int* chunk_seg, int n_chunks, float beta1,
                        float beta2, float eps, const uint64_t* step, float grad_scale,
                        float2* partials, cudaStream_t stream,
                        const OptimScalars* scalars = nullptr);
int launch_lamb_update(const LambSegment* segs, const int* chunk_seg, int n_chunks, float lr,
                       float beta1, float beta2, float eps, const uint64_t* step,
                       const float2* partials, float* ratios, cudaStream_t stream,
                       const OptimScalars* scalars = nullptr);
// Learning-rate schedules f(k) of launch_optim_finalize (lr = base_lr * f(k)).
enum LrScheduleType : int { kLrNone = 0, kLrConstant = 1, kLrLinear = 2, kLrCosine = 3 };
// Cross-rank exchange of the local sums of squares through peer memory (CUDA IPC).  Every rank
// owns one region, mapped by all the others: `uint32 flags[n_ranks]` in the first 256 bytes, then
// `float slots[2][n_ranks]`.  `regions` is a device array of the n_ranks region bases as mapped in
// this process (own region included), indexed by pipeline position.
struct NormExchangeArgs {
  void* const* regions = nullptr;
  int n_ranks = 0;
  int my_pos = 0;
  const uint32_t* epoch = nullptr;  // device step epoch, advanced once per step
  int* error_flag = nullptr;        // set to 4 when a peer's slot did not arrive in time
};
// One block: sums `partials` in a fixed order (+ *extra_sumsq when non-null), optionally sums
// the ranks' shares through `ex` in position order (bit-identical on every rank), then writes
// *out: grad_norm, clip_coef (1 when max_norm <= 0) and lr = base_lr * f(k), k = *step (0 when
// `step` is null) + step_offset.
int launch_optim_finalize(const float* partials, int n_partials, const float* extra_sumsq,
                          NormExchangeArgs ex, const uint64_t* step, long long step_offset,
                          int schedule, int warmup,
                          int total, double base_lr, float max_norm, OptimScalars* out,
                          cudaStream_t stream);
// Round-to-nearest-even casts, bit-identical to torch's .to(torch.bfloat16) / .float() for every
// non-NaN input.  Subnormals are converted, not flushed, even under --use_fast_math (neither
// conversion has a flush-to-zero form); a NaN stays a NaN, its payload may differ from torch's.
int launch_cast_f32_to_bf16(const float* src, void* dst, long long n, cudaStream_t stream);
int launch_cast_bf16_to_f32(const void* src, float* dst, long long n, cudaStream_t stream);

// ---------------------------------------------------------------------------------------------
// Runtime helpers
// ---------------------------------------------------------------------------------------------
int launch_advance_counter(uint64_t* counter, uint64_t inc, cudaStream_t stream);   // rng step
int launch_advance_epoch(uint32_t* counter, uint32_t inc, cudaStream_t stream);     // flag epochs
int launch_signal_flags(uint32_t* flags, int n, uint32_t inc, cudaStream_t stream); // release.sys
int launch_wait_flags(const uint32_t* flags, int n, const uint32_t* epoch, uint32_t mult,
                      int* error_flag, cudaStream_t stream);
// Device-side throttle used by the stimulator / `slowdown`: spins for `ns` nanoseconds, or for
// factor * (elapsed since *t_start_ns) when factor > 0 (simulated slow device).
int launch_spin_ns(uint64_t ns, cudaStream_t stream);
int launch_record_time(uint64_t* slot, cudaStream_t stream);
int launch_spin_factor(const uint64_t* t_start_slot, float factor, cudaStream_t stream);
// Peer copy with flags (unfused boundary over NVLink): copies n bytes (16B multiple) to dst
// (peer pointer) and bumps `n_flags` counters with release.sys.
int launch_peer_copy_signal(const void* src, void* dst, long long nbytes, uint32_t* flags,
                            int n_flags, uint32_t inc, cudaStream_t stream);
// Tied word-embedding gradient exchange between the first and the last pipeline rank (parallel/
// p2p.py: TiedGradExchange).  push (last rank): dst[0:n] = src[0:n] with 16-byte peer stores, then
// the last block to finish adds 1 to *flag (release.sys).  reduce (first rank): waits until
// *wait_flag >= *epoch (acquire.sys; after 4 s *error_flag = 5 and the sum is skipped), then
// s = g + inbox once per element, stored into g and peer_g, then the last block adds 1 to
// *publish_flag.  `done`: a zeroed device counter private to the launching rank.  Pointers 16-byte
// aligned (931); null pointers or n <= 0: 930.
int launch_tied_grad_push(const float* src, float* dst, long long n, uint32_t* flag,
                          unsigned int* done, cudaStream_t stream);
int launch_tied_grad_reduce(float* g, const float* inbox, float* peer_g, long long n,
                            const uint32_t* wait_flag, const uint32_t* epoch, int* error_flag,
                            uint32_t* publish_flag, unsigned int* done, cudaStream_t stream);

}  // namespace sky
