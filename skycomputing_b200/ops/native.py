"""Tensor-level wrappers of the sm_90a kernel library (``skycomputing_b200._cuda``).

Every function validates dtype / layout in Python, then hands raw device pointers and the current
CUDA stream to the C++ launcher (which is torch-free, see csrc/bindings_cuda.cpp).  Outputs are
pre-allocated by the caller or allocated here through torch's caching allocator, so everything is
CUDA-graph capturable.

These wrappers FAIL LOUDLY when the extension is missing on a GPU machine: there is no silent
PyTorch fallback on the hot path (the eager oracle lives in ``skycomputing_b200.models`` and is
selected explicitly with ``backend="torch"``).
"""
from __future__ import annotations

from typing import Optional

import torch

_cuda = None
_import_error: Optional[BaseException] = None
try:  # the .so is built in-tree by skycomputing_b200._build / __graft_entry__.build()
    from .. import _cuda as _cuda_mod  # type: ignore

    _cuda = _cuda_mod
except Exception as e:  # pragma: no cover - exercised only when the build is missing
    _import_error = e

ACT_NONE, ACT_GELU, ACT_DGELU_MUL_AUX, ACT_TANH = 0, 1, 2, 3


def available() -> bool:
    """True iff the native extension is importable AND a CUDA device is present."""
    return _cuda is not None and torch.cuda.is_available()


# ---- launch accounting (bench.py reports how many of OUR kernels ran in the timed region) ----
# kernels per call; -1: the binding returns the number of kernels it launched
_KERNELS_PER_CALL = {
    "gemm": 1, "layernorm_fwd": 1, "layernorm_bwd": 1, "ln_param_grad": 1, "colsum": 1, "dgelu_mul": 1,
    "attention_fwd": 1, "attention_bwd": 1, "embed_fwd": 1, "embed_bwd": 1,
    "small_linear_fwd": 1, "small_linear_bwd": 2, "softmax_ce": 1, "classify_eval": 1,
    "vocab_ce": -1, "mlm_gather": 1, "mlm_scatter": 1, "cls_grad_add": 1,
    "qa_logits_fwd": 1, "qa_logits_bwd": 2, "qa_span_eval": 1,
    "sgd_multi": 1, "adam_multi": 1, "lamb_moments": 1, "lamb_update": 1,
    "grad_sumsq_multi": 1, "optim_finalize": 1,
    "cast_f32_to_bf16": 1, "cast_bf16_to_f32": 1, "advance_counter": 1, "advance_epoch": 1,
    "signal_flags": 1, "wait_flags": 1, "spin_ns": 1, "record_time": 1, "spin_factor": 1,
    "peer_copy_signal": 1, "tied_grad_push": 1, "tied_grad_reduce": 1,
}
_launches = [0]
_counting_proxy = None


class _CountingExt:
    """Attribute proxy of the extension module that counts kernel launches per call."""

    def __init__(self, mod):
        self._mod = mod
        self._cache = {}

    def __getattr__(self, name):
        fn = self._cache.get(name)
        if fn is None:
            target = getattr(self._mod, name)
            n = _KERNELS_PER_CALL.get(name, 0)
            if n < 0 and callable(target):
                def fn(*a, __t=target, **k):
                    launched = __t(*a, **k)
                    _launches[0] += launched
                    return launched
            elif n and callable(target):
                def fn(*a, __t=target, __n=n, **k):
                    _launches[0] += __n
                    return __t(*a, **k)
            else:
                fn = target
            self._cache[name] = fn
        return fn


def enable_launch_counter() -> None:
    global _counting_proxy
    if _counting_proxy is None and _cuda is not None:
        _counting_proxy = _CountingExt(_cuda)


def reset_launch_counter() -> None:
    _launches[0] = 0


def launch_count() -> int:
    return _launches[0]


def ext():
    if _counting_proxy is not None:
        return _counting_proxy
    if _cuda is None:
        raise RuntimeError(
            "skycomputing_b200._cuda is not built/importable "
            f"({_import_error!r}); run `python -m skycomputing_b200._build` "
            "(or __graft_entry__.build()) first"
        )
    return _cuda


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t: Optional[torch.Tensor]) -> int:
    return 0 if t is None else t.data_ptr()


def _check(t: torch.Tensor, dtype: torch.dtype, name: str) -> None:
    if not t.is_cuda:
        raise ValueError(f"{name} must be a CUDA tensor")
    if t.dtype != dtype:
        raise ValueError(f"{name} must be {dtype}, got {t.dtype}")
    if t.dim() >= 1 and t.stride(-1) != 1:
        raise ValueError(f"{name} must have a unit inner stride")


class RngState:
    """Device-resident dropout RNG state {seed, step}; ``advance()`` is a captured kernel."""

    def __init__(self, seed: int, device: torch.device | str = "cuda"):
        # int64 storage, interpreted as uint64 on the device
        self.state = torch.tensor([int(seed) & 0x7FFFFFFFFFFFFFFF, 0], dtype=torch.int64,
                                  device=device)

    @property
    def ptr(self) -> int:
        return self.state.data_ptr()

    def advance(self, inc: int = 1) -> None:
        ext().advance_counter(self.state.data_ptr() + 8, inc, _stream())


def gemm(
    a: torch.Tensor,
    b: torch.Tensor,
    *,
    a_mn: bool = False,
    b_mn: bool = False,
    out: Optional[torch.Tensor] = None,
    out_dtype: torch.dtype = torch.bfloat16,
    accumulate: bool = False,
    bias: Optional[torch.Tensor] = None,
    aux: Optional[torch.Tensor] = None,
    act: int = ACT_NONE,
    add_aux: bool = False,
    out2: Optional[torch.Tensor] = None,
    dropout_p: float = 0.0,
    rng: Optional[RngState] = None,
    rng_stream: int = 0,
    out_ptr: int = 0,
    out_ld: int = 0,
    signal_flags: int = 0,
    wait_flags: int = 0,
    wait_epoch: int = 0,
    wait_mult: int = 0,
    error_flag: int = 0,
    block_n: int = 0,
    pair: int = -1,
    stream_k: int = -1,
    max_ctas: int = 0,
    debug: int = 0,
    sgd_master: Optional[torch.Tensor] = None,
    sgd_shadow: Optional[torch.Tensor] = None,
    sgd_lr: float = 0.0,
    sgd_weight_decay: float = 0.0,
    sgd_grad_scale: float = 1.0,
) -> Optional[torch.Tensor]:
    """out[M,N] = epilogue(sum_k A[m,k] B[n,k]) on the wgmma kernel.

    ``a``: [M,K] (or [K,M] when ``a_mn``); ``b``: [N,K] (or [K,N] when ``b_mn``), both bf16 with
    unit inner stride.  ``out_ptr``/``out_ld`` redirect the store to a raw (peer) pointer.

    ``sgd_master`` (fp32) / ``sgd_shadow`` (bf16), laid out like the fp32 ``out`` of a weight
    gradient (``a_mn`` and ``b_mn``): the gradient g (``out + g`` when ``accumulate``) is not
    stored, the epilogue applies ``sgd_multi``'s plain update to the master and refreshes the
    shadow (see GemmArgs::sgd_master in csrc/kernels/api.h).
    """
    _check(a, torch.bfloat16, "a")
    _check(b, torch.bfloat16, "b")
    if a.dim() != 2 or b.dim() != 2:
        raise ValueError("gemm operands must be 2-D")
    if a_mn:
        K, M = a.shape
    else:
        M, K = a.shape
    if b_mn:
        Kb, N = b.shape
    else:
        N, Kb = b.shape
    if K != Kb:
        raise ValueError(f"inner dimensions differ: {K} vs {Kb}")
    out_f32 = out_dtype == torch.float32 if out is None else out.dtype == torch.float32
    if out_ptr:
        o_ptr, ldo = out_ptr, out_ld
    else:
        if out is None:
            out = torch.empty((M, N), dtype=out_dtype, device=a.device)
        _check(out, torch.float32 if out_f32 else torch.bfloat16, "out")
        if tuple(out.shape) != (M, N):
            raise ValueError(f"out has shape {tuple(out.shape)}, expected {(M, N)}")
        o_ptr, ldo = out.data_ptr(), out.stride(0)
    if bias is not None:
        _check(bias, torch.float32, "bias")
    if aux is not None:
        _check(aux, torch.bfloat16, "aux")
    if out2 is not None:
        _check(out2, torch.bfloat16, "out2")
    if sgd_master is not None:
        if sgd_shadow is None:
            raise ValueError("the SGD epilogue needs sgd_shadow")
        _check(sgd_master, torch.float32, "sgd_master")
        _check(sgd_shadow, torch.bfloat16, "sgd_shadow")
        for t, what in ((sgd_master, "sgd_master"), (sgd_shadow, "sgd_shadow")):
            if t.dim() != 2 or tuple(t.shape) != (M, N) or t.stride(0) != ldo:
                raise ValueError(f"{what} must be [{M}, {N}] with the row stride of out")
    ext().gemm(
        A=a.data_ptr(), B=b.data_ptr(), M=M, N=N, K=K, lda=a.stride(0), ldb=b.stride(0),
        a_mn=a_mn, b_mn=b_mn, out=o_ptr, ldo=ldo, out_f32=out_f32, accumulate=accumulate,
        out2=_ptr(out2), ldo2=0 if out2 is None else out2.stride(0), bias=_ptr(bias),
        aux=_ptr(aux), ldaux=0 if aux is None else aux.stride(0), act=act, add_aux=add_aux,
        dropout_p=float(dropout_p), rng_state=0 if rng is None else rng.ptr,
        rng_stream=rng_stream, signal_flags=signal_flags, wait_flags=wait_flags,
        wait_epoch=wait_epoch, wait_mult=wait_mult, error_flag=error_flag, block_n=block_n, pair=pair, stream_k=stream_k,
        max_ctas=max_ctas, debug=debug, sgd_master=_ptr(sgd_master), sgd_shadow=_ptr(sgd_shadow),
        sgd_lr=float(sgd_lr), sgd_weight_decay=float(sgd_weight_decay),
        sgd_grad_scale=float(sgd_grad_scale), stream=_stream(),
    )
    return out


def _fuse_ln_mode() -> str:
    import os

    return os.environ.get("SKY_FUSE_LN", "1")


def gemm_ln_supported(M: int, N: int) -> bool:
    """Should ``dense + LayerNorm`` of this output shape run as the one-kernel GEMM + LayerNorm
    epilogue?  Default: where it is faster than GEMM + standalone LayerNorm (csrc: gemm_ln_block_n);
    ``SKY_FUSE_LN=force``: wherever the kernel can run; ``SKY_FUSE_LN=0``: never."""
    mode = _fuse_ln_mode()
    if mode == "0":
        return False
    return ext().gemm_ln_block_n(int(M), int(N), mode == "force") != 0


def gemm_ln_tiles_per_panel(M: int, N: int) -> int:
    """Flag signals per 128-row panel when the fused kernel writes a stage boundary."""
    return ext().gemm_ln_tiles_per_panel(int(M), int(N), _fuse_ln_mode() == "force")


def gemm_ln(a: torch.Tensor, b: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, *,
            eps: float = 1e-12, bias: Optional[torch.Tensor] = None,
            residual: Optional[torch.Tensor] = None, dropout_p: float = 0.0,
            rng: Optional[RngState] = None, rng_stream: int = 0, save_z: bool = True,
            y_ptr: int = 0, y_ld: int = 0, signal_flags: int = 0, wait_flags: int = 0,
            wait_epoch: int = 0, wait_mult: int = 0, error_flag: int = 0, block_n: int = 0,
            debug: int = 0):
    """y = LayerNorm(dropout(a b^T + bias) + residual) * gamma + beta in ONE wgmma kernel
    (cluster-wide row statistics through DSMEM, see csrc/kernels/gemm_sm100.cu).

    Returns ``(y, z, mean, rstd)``: ``z`` is the bf16 pre-LayerNorm sum saved for backward (None
    when ``save_z`` is False), ``y`` is None when ``y_ptr`` redirects the store to raw (peer)
    memory; ``signal_flags`` then receives ``gemm_ln_tiles_per_panel`` signals per 128-row panel.
    ``debug=1`` (timing only) runs the main loop and skips the epilogue: nothing is written."""
    _check(a, torch.bfloat16, "a")
    _check(b, torch.bfloat16, "b")
    _check(gamma, torch.float32, "gamma")
    _check(beta, torch.float32, "beta")
    M, K = a.shape
    N, Kb = b.shape
    if K != Kb:
        raise ValueError(f"inner dimensions differ: {K} vs {Kb}")
    if bias is not None:
        _check(bias, torch.float32, "bias")
    if residual is not None:
        _check(residual, torch.bfloat16, "residual")
    dev = a.device
    y = None
    if y_ptr:
        o_ptr, ldo = y_ptr, (y_ld or N)
    else:
        y = torch.empty((M, N), dtype=torch.bfloat16, device=dev)
        o_ptr, ldo = y.data_ptr(), N
    z = torch.empty((M, N), dtype=torch.bfloat16, device=dev) if save_z else None
    mean = torch.empty(M, dtype=torch.float32, device=dev)
    rstd = torch.empty(M, dtype=torch.float32, device=dev)
    ext().gemm(
        A=a.data_ptr(), B=b.data_ptr(), M=M, N=N, K=K, lda=a.stride(0), ldb=b.stride(0),
        out=o_ptr, ldo=ldo, out2=_ptr(z), ldo2=0 if z is None else N, bias=_ptr(bias),
        aux=_ptr(residual), ldaux=0 if residual is None else residual.stride(0),
        add_aux=residual is not None, dropout_p=float(dropout_p),
        rng_state=0 if rng is None else rng.ptr, rng_stream=rng_stream,
        signal_flags=signal_flags, wait_flags=wait_flags, wait_epoch=wait_epoch,
        wait_mult=wait_mult, error_flag=error_flag, block_n=block_n, debug=debug,
        ln_gamma=gamma.data_ptr(), ln_beta=beta.data_ptr(), ln_mean=mean.data_ptr(),
        ln_rstd=rstd.data_ptr(), ln_eps=float(eps), stream=_stream(),
    )
    return y, z, mean, rstd


def layernorm_fwd(z, gamma, beta, eps: float = 1e-12, *, y=None, wait_flags: int = 0,
                  wait_epoch: int = 0, wait_mult: int = 0, error_flag: int = 0):
    _check(z, torch.bfloat16, "z")
    M, H = z.shape
    if not z.is_contiguous():
        raise ValueError("z must be contiguous")
    y = torch.empty_like(z) if y is None else y
    mean = torch.empty(M, dtype=torch.float32, device=z.device)
    rstd = torch.empty(M, dtype=torch.float32, device=z.device)
    ext().layernorm_fwd(z=z.data_ptr(), y=y.data_ptr(), mean=mean.data_ptr(), rstd=rstd.data_ptr(),
                        gamma=gamma.data_ptr(), beta=beta.data_ptr(), M=M, H=H, eps=eps,
                        wait_flags=wait_flags, wait_epoch=wait_epoch, wait_mult=wait_mult,
                        error_flag=error_flag, stream=_stream())
    return y, mean, rstd


def layernorm_bwd(dy, z, mean, rstd, gamma, dgamma, dbeta, *, dropout_p: float = 0.0,
                  rng: Optional[RngState] = None, rng_stream: int = 0, wait_flags: int = 0,
                  wait_epoch: int = 0, wait_mult: int = 0, error_flag: int = 0):
    """Returns (dz, dz_dropped or None); dgamma/dbeta (fp32) are accumulated in place, or left to a
    later `ln_param_grad` call when passed as None."""
    _check(dy, torch.bfloat16, "dy")
    _check(z, torch.bfloat16, "z")
    M, H = z.shape
    dz = torch.empty_like(z)
    dzd = torch.empty_like(z) if dropout_p > 0 else None
    ext().layernorm_bwd(dy=dy.data_ptr(), z=z.data_ptr(), mean=mean.data_ptr(),
                        rstd=rstd.data_ptr(), gamma=gamma.data_ptr(), dz=dz.data_ptr(),
                        dz_dropped=_ptr(dzd), dgamma=_ptr(dgamma), dbeta=_ptr(dbeta),
                        M=M, H=H, dropout_p=float(dropout_p),
                        rng_state=0 if rng is None else rng.ptr, rng_stream=rng_stream,
                        wait_flags=wait_flags, wait_epoch=wait_epoch, wait_mult=wait_mult,
                        error_flag=error_flag, stream=_stream())
    return dz, dzd


def ln_param_grad(dy, z, mean, rstd, dgamma, dbeta, x2=None, out2=None) -> None:
    """dgamma += sum_rows dy * xhat, dbeta += sum_rows dy (the second half of layernorm_bwd);
    optionally also out2 += column sums of x2 ([M,H] bf16): the bias gradient of the dense layer
    in front of the LayerNorm, fused to save a launch."""
    M, H = z.shape
    if x2 is not None:
        _check(x2, torch.bfloat16, "x2")
        if tuple(x2.shape) != (M, H) or not x2.is_contiguous():
            raise ValueError("x2 must be a contiguous [M,H] tensor")
    ext().ln_param_grad(dy=dy.data_ptr(), z=z.data_ptr(), mean=mean.data_ptr(), rstd=rstd.data_ptr(),
                        dgamma=dgamma.data_ptr(), dbeta=dbeta.data_ptr(), M=M, H=H, x2=_ptr(x2),
                        out2=_ptr(out2), stream=_stream())


def colsum_(x: torch.Tensor, out: torch.Tensor) -> None:
    """out[n] += sum_m x[m, n]  (x bf16, out fp32)."""
    _check(x, torch.bfloat16, "x")
    _check(out, torch.float32, "out")
    M, N = x.shape
    ext().colsum(x=x.data_ptr(), M=M, N=N, ldx=x.stride(0), out=out.data_ptr(), stream=_stream())


def attention_fwd(qkv, mask, B: int, S: int, heads: int, *, dropout_p: float = 0.0,
                  rng: Optional[RngState] = None, rng_stream: int = 0, save_lse: bool = True):
    """Returns ``(ctx, lse)``; ``lse`` (kept for backward) is None when ``save_lse`` is False."""
    _check(qkv, torch.bfloat16, "qkv")
    H = qkv.shape[1] // 3
    d = H // heads
    ctx = torch.empty((B * S, H), dtype=torch.bfloat16, device=qkv.device)
    lse = torch.empty((B * heads * S,), dtype=torch.float32, device=qkv.device) if save_lse else None
    ext().attention_fwd(qkv=qkv.data_ptr(), mask=_ptr(mask), ctx=ctx.data_ptr(),
                        lse=_ptr(lse), B=B, S=S, heads=heads, head_dim=d,
                        scale=1.0 / (d ** 0.5), dropout_p=float(dropout_p),
                        rng_state=0 if rng is None else rng.ptr, rng_stream=rng_stream,
                        stream=_stream())
    return ctx, lse


def attention_bwd(qkv, mask, ctx, lse, dctx, B: int, S: int, heads: int, *,
                  dropout_p: float = 0.0, rng: Optional[RngState] = None, rng_stream: int = 0):
    _check(dctx, torch.bfloat16, "dctx")
    if not dctx.is_contiguous():
        dctx = dctx.contiguous()
    H = qkv.shape[1] // 3
    d = H // heads
    dqkv = torch.empty_like(qkv)
    ext().attention_bwd(qkv=qkv.data_ptr(), mask=_ptr(mask), ctx=ctx.data_ptr(),
                        lse=lse.data_ptr(), dctx=dctx.data_ptr(), dqkv=dqkv.data_ptr(), B=B, S=S,
                        heads=heads, head_dim=d, scale=1.0 / (d ** 0.5),
                        dropout_p=float(dropout_p), rng_state=0 if rng is None else rng.ptr,
                        rng_stream=rng_stream, stream=_stream())
    return dqkv


def cast_f32_to_bf16_(src: torch.Tensor, dst: torch.Tensor) -> None:
    ext().cast_f32_to_bf16(src.data_ptr(), dst.data_ptr(), src.numel(), _stream())


def softmax_ce(logits: torch.Tensor, labels: torch.Tensor, grad_scale: float = 1.0,
               loss_acc: Optional[torch.Tensor] = None, ignore_index: int = -100):
    """Cross entropy over fp32 logits ``[N, C]``, or ``[N, G, C]`` with G = 2 groups of rows per
    item (the span loss's start and end rows), with labels ``[N]`` or ``[N, G]`` int64 (unit
    column stride, any row stride: a column of a wider label tensor is read in place).

    Returns ``(loss [1], dlogits)``: the mean CE over each group's rows whose label is in
    [0, C), averaged over the groups (a group without such a row adds 0), and d(loss *
    grad_scale)/dlogits in the logits' shape, an exact 0 on every other row.  A label neither
    ``ignore_index`` nor in [0, C) makes the loss NaN and is never used as an index.
    ``loss_acc[0] += loss * grad_scale`` when given (the step loss of a micro-batched step,
    accumulated without extra launches).  One launch, no host synchronisation, deterministic."""
    _check(logits, torch.float32, "logits")
    if logits.dim() not in (2, 3):
        raise ValueError("logits must be [N, C] or [N, G, C]")
    N, C = logits.shape[0], logits.shape[-1]
    G = logits.shape[1] if logits.dim() == 3 else 1
    if not labels.is_cuda or labels.dtype != torch.int64 or labels.numel() != N * G:
        raise ValueError("labels must be a CUDA int64 tensor with one entry per logits row")
    rows = logits.reshape(N * G, C)
    labels = labels.reshape(N, G)
    if G > 1 and labels.stride(1) != 1:
        raise ValueError("labels must have a unit column stride")
    loss = torch.empty(1, dtype=torch.float32, device=logits.device)
    dlogits = torch.empty(logits.shape, dtype=torch.float32, device=logits.device)
    # a single row's stride is arbitrary: it is never stepped over
    ext().softmax_ce(logits=rows.data_ptr(), ldl=rows.stride(0) if N * G > 1 else C,
                     labels=labels.data_ptr(), label_ld=labels.stride(0) if N > 1 else G, N=N,
                     G=G, C=C, ignore_index=int(ignore_index), dlogits=dlogits.data_ptr(),
                     grad_scale=float(grad_scale), loss=loss.data_ptr(), loss_acc=_ptr(loss_acc),
                     stream=_stream())
    return loss, dlogits


def classify_eval(logits: torch.Tensor, labels: torch.Tensor, accum: torch.Tensor,
                  ignore_index: int = -100) -> None:
    """Adds one batch of fp32 logits [M, C] into the device accumulator ``accum`` (the int64
    buffer of an ``EvalAccumulator``): per-row cross entropy, argmax and confusion counts.  One
    launch, no host synchronisation, deterministic."""
    _check(logits, torch.float32, "logits")
    if logits.dim() != 2:
        raise ValueError("logits must be 2-D [M, C]")
    M, C = logits.shape
    if not labels.is_cuda or labels.dtype != torch.int64 or labels.numel() != M:
        raise ValueError("labels must be a CUDA int64 tensor with one entry per logits row")
    if accum.dtype != torch.int64 or accum.numel() < 3 + C * C:
        raise ValueError("accum is not an EvalAccumulator buffer for {} classes".format(C))
    ext().classify_eval(logits=logits.data_ptr(), ldl=logits.stride(0),
                        labels=labels.contiguous().data_ptr(), M=M, C=C,
                        ignore_index=int(ignore_index), acc=accum.data_ptr(), stream=_stream())


def _vocab_ce_check(logits: torch.Tensor, labels: torch.Tensor):
    _check(logits, torch.bfloat16, "logits")
    if logits.dim() != 2:
        raise ValueError("logits must be 2-D [M, V]")
    M, V = logits.shape
    if not labels.is_cuda or labels.dtype != torch.int64 or labels.numel() != M:
        raise ValueError("labels must be a CUDA int64 tensor with one entry per logits row")
    if V > ext().vocab_ce_max_v():
        raise ValueError("vocab_ce stages a logits row in shared memory and supports at most {} "
                         "classes, got {}".format(ext().vocab_ce_max_v(), V))
    ws = torch.empty(ext().vocab_ce_workspace_bytes(M), dtype=torch.uint8, device=logits.device)
    return M, V, labels.reshape(-1).contiguous(), ws


def vocab_ce(logits: torch.Tensor, labels: torch.Tensor, grad_scale: float = 1.0,
             loss_acc: Optional[torch.Tensor] = None, ignore_index: int = -100,
             in_place: bool = False):
    """Masked-language-model cross entropy over bf16 logits ``[M, V]`` (row stride may exceed V).

    Returns ``(loss, dlogits)``: the mean loss over the rows whose label is not ``ignore_index``
    (fp32 ``[1]``) and ``d(loss * grad_scale)/dlogits`` as bf16, 0 on ignored rows; with
    ``in_place`` the gradient overwrites ``logits``.  ``loss_acc[0] += loss * grad_scale`` when
    given.  With no labelled row the loss and the gradient are 0, where torch gives NaN.  Three
    launches, no host synchronisation, deterministic."""
    M, V, labels, ws = _vocab_ce_check(logits, labels)
    dlogits = logits if in_place else torch.empty_strided(logits.shape, logits.stride(),
                                                          dtype=torch.bfloat16,
                                                          device=logits.device)
    loss = torch.empty(1, dtype=torch.float32, device=logits.device)
    ext().vocab_ce(logits=logits.data_ptr(), ldl=logits.stride(0), labels=labels.data_ptr(), M=M,
                   V=V, ignore_index=int(ignore_index), dlogits=dlogits.data_ptr(),
                   grad_scale=float(grad_scale), loss_out=loss.data_ptr(),
                   loss_acc=_ptr(loss_acc), workspace=ws.data_ptr(), stream=_stream())
    return loss, dlogits


def mlm_gather(hidden: torch.Tensor, labels: torch.Tensor, P: int, V: int,
               ignore_index: int = -100):
    """The rows a sparse masked-language-model head decodes (slot layout: ``functions.
    mlm_slots_ref``).  ``hidden`` [B*S, H] bf16, ``labels`` [B, S] int64.  Returns ``(x_c
    [B*P, H] bf16, slot_of_row [B*S] int32, slot_labels [B*P] int64)``; one launch."""
    _check(hidden, torch.bfloat16, "hidden")
    if not labels.is_cuda or labels.dtype != torch.int64 or labels.dim() != 2:
        raise ValueError("labels must be a CUDA int64 [B, S] tensor")
    B, S = labels.shape
    H = hidden.shape[-1]
    if hidden.dim() != 2 or hidden.shape[0] != B * S or not hidden.is_contiguous():
        raise ValueError("hidden must be a contiguous [B*S, H] tensor")
    dev = hidden.device
    x_c = torch.empty((B * P, H), dtype=torch.bfloat16, device=dev)
    slot_of_row = torch.empty(B * S, dtype=torch.int32, device=dev)
    slot_labels = torch.empty(B * P, dtype=torch.int64, device=dev)
    ext().mlm_gather(hidden=hidden.data_ptr(), labels=labels.contiguous().data_ptr(), B=B, S=S,
                     H=H, P=int(P), ignore_index=int(ignore_index), V=int(V),
                     slot_of_row=slot_of_row.data_ptr(), slot_labels=slot_labels.data_ptr(),
                     x_c=x_c.data_ptr(), stream=_stream())
    return x_c, slot_of_row, slot_labels


def mlm_scatter(dx_c: torch.Tensor, slot_of_row: torch.Tensor,
                dcls: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The input gradient of a sparse head: ``dhidden[r] = dx_c[slot_of_row[r]]`` for a decoded
    row, zeros otherwise; ``dhidden`` [len(slot_of_row), H] bf16, every row written once.  With
    ``dcls`` [B, H] bf16 (a pooler branch's input gradient) the [CLS] row b*S of each sequence
    also gets ``dcls[b]`` added, S = len(slot_of_row) / B."""
    _check(dx_c, torch.bfloat16, "dx_c")
    if slot_of_row.dtype != torch.int32 or not slot_of_row.is_cuda:
        raise ValueError("slot_of_row must be a CUDA int32 tensor")
    dx_c = dx_c.contiguous()
    H = dx_c.shape[-1]
    S = 1
    if dcls is not None:
        _check(dcls, torch.bfloat16, "dcls")
        if dcls.dim() != 2 or dcls.shape[1] != H or slot_of_row.numel() % dcls.shape[0]:
            raise ValueError("dcls must be [B, H] with B dividing the number of rows")
        dcls = dcls.contiguous()
        S = slot_of_row.numel() // dcls.shape[0]
    dhidden = torch.empty((slot_of_row.numel(), H), dtype=torch.bfloat16, device=dx_c.device)
    ext().mlm_scatter(dx_c=dx_c.data_ptr(), slot_of_row=slot_of_row.data_ptr(),
                      rows=slot_of_row.numel(), H=H, dhidden=dhidden.data_ptr(), stream=_stream(),
                      dcls=_ptr(dcls), S=S)
    return dhidden


def cls_grad_add_(dhidden: torch.Tensor, dcls: torch.Tensor) -> torch.Tensor:
    """``dhidden[b, 0] += dcls[b]`` in place (bf16 [B, S, H] and [B, H]): the [CLS]-row join of a
    dense head with a pooler branch.  One launch."""
    _check(dhidden, torch.bfloat16, "dhidden")
    _check(dcls, torch.bfloat16, "dcls")
    B, S, H = dhidden.shape
    if not dhidden.is_contiguous() or tuple(dcls.shape) != (B, H):
        raise ValueError("dhidden must be a contiguous [B, S, H] tensor and dcls [B, H]")
    dcls = dcls.contiguous()
    ext().cls_grad_add(dhidden=dhidden.data_ptr(), dcls=dcls.data_ptr(), B=B, S=S, H=H,
                       stream=_stream())
    return dhidden


def _qa_labels(labels: torch.Tensor, B: int) -> torch.Tensor:
    if not labels.is_cuda or labels.dtype != torch.int64 or labels.numel() != B * 5:
        raise ValueError("labels must be a CUDA int64 tensor [B, 5] (ops.functions."
                         "split_span_labels)")
    return labels.reshape(B, 5).contiguous()


def _qa_logits_check(logits: torch.Tensor):
    _check(logits, torch.float32, "logits")
    if logits.dim() != 3 or logits.shape[1] != 2 or not logits.is_contiguous():
        raise ValueError("logits must be a contiguous [B, 2, S] tensor")
    return logits.shape[0], logits.shape[2]


def qa_logits(hidden: torch.Tensor, w: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """Start / end logits of a question-answering head: ``hidden`` bf16 [B, S, H] (H % 8 == 0),
    ``w`` fp32 [2, H], ``b`` fp32 [2] -> fp32 [B, 2, S] (row 0 start, row 1 end).  One launch."""
    _check(hidden, torch.bfloat16, "hidden")
    _check(w, torch.float32, "w")
    _check(b, torch.float32, "b")
    if hidden.dim() != 3 or not hidden.is_contiguous():
        raise ValueError("hidden must be a contiguous [B, S, H] tensor")
    B, S, H = hidden.shape
    if tuple(w.shape) != (2, H) or not w.is_contiguous() or b.numel() != 2:
        raise ValueError("w must be a contiguous [2, {}] tensor and b [2]".format(H))
    logits = torch.empty((B, 2, S), dtype=torch.float32, device=hidden.device)
    ext().qa_logits_fwd(hidden=hidden.data_ptr(), B=B, S=S, H=H, w=w.data_ptr(), b=b.data_ptr(),
                        logits=logits.data_ptr(), stream=_stream())
    return logits


def qa_logits_bwd(hidden: torch.Tensor, dlogits: torch.Tensor, w: torch.Tensor,
                  dw: torch.Tensor, db: torch.Tensor) -> torch.Tensor:
    """Backward of ``qa_logits``: returns ``dhidden`` bf16 [B, S, H] and adds the weight and bias
    gradients into the fp32 ``dw`` [2, H] / ``db`` [2] in a fixed order.  Two launches."""
    _check(hidden, torch.bfloat16, "hidden")
    _check(w, torch.float32, "w")
    _check(dw, torch.float32, "dw")
    _check(db, torch.float32, "db")
    B, S, H = hidden.shape
    dlogits = dlogits.float().contiguous()
    if tuple(dlogits.shape) != (B, 2, S):
        raise ValueError("dlogits must be [B, 2, S] = {}".format([B, 2, S]))
    if tuple(dw.shape) != (2, H) or not dw.is_contiguous() or db.numel() != 2:
        raise ValueError("dw must be a contiguous [2, H] tensor and db [2]")
    dhidden = torch.empty_like(hidden)
    ws = torch.empty(ext().qa_logits_bwd_workspace_bytes(B, S, H) // 4, dtype=torch.float32,
                     device=hidden.device)
    ext().qa_logits_bwd(hidden=hidden.data_ptr(), dlogits=dlogits.data_ptr(), B=B, S=S, H=H,
                        w=w.data_ptr(), dhidden=dhidden.data_ptr(), workspace=ws.data_ptr(),
                        dw=dw.data_ptr(), db=db.data_ptr(), stream=_stream())
    return dhidden


class SpanEvalAccumulator:
    """Device-side accumulator of a span head's evaluation pass (``sky::SpanEvalAccum``): fp64
    start / end cross-entropy and F1 sums, the counted sequences, top-1 start / end hits, exact
    spans, invalid labels, and the best span and score of every sequence, stored at a device
    cursor in buffers of ``capacity`` sequences (later ones are counted as overflow).

    ``reset()`` is two memsets and ``add()`` one ``qa_span_eval`` launch, capturable into a CUDA
    graph (a replay appends at the cursor); ``read()`` copies the totals and predictions once."""

    def __init__(self, max_answer_length: int, capacity: int, device=None):
        if max_answer_length < 1 or capacity < 0:
            raise ValueError("max_answer_length must be >= 1 and capacity >= 0")
        dev = device if device is not None else "cuda"
        self.max_answer_length = int(max_answer_length)
        self.capacity = int(capacity)
        self.buffer = torch.zeros(ext().qa_span_eval_accum_bytes() // 8, dtype=torch.int64,
                                  device=dev)
        self.spans = torch.full((max(self.capacity, 1), 2), -1, dtype=torch.int32, device=dev)
        self.scores = torch.zeros(max(self.capacity, 1), dtype=torch.float32, device=dev)

    def reset(self) -> None:
        self.buffer.zero_()
        self.spans.fill_(-1)

    def add(self, logits: torch.Tensor, labels: torch.Tensor, ignore_index: int = -100) -> None:
        logits = logits.detach().float().contiguous()
        B, S = _qa_logits_check(logits)
        labels = _qa_labels(labels, B)
        ext().qa_span_eval(logits=logits.data_ptr(), labels=labels.data_ptr(), B=B, S=S,
                           max_answer_length=self.max_answer_length,
                           ignore_index=int(ignore_index), acc=self.buffer.data_ptr(),
                           pred_spans=self.spans.data_ptr(), pred_scores=self.scores.data_ptr(),
                           capacity=self.capacity, stream=_stream())

    def read(self) -> dict:
        host = self.buffer.cpu()
        f = host[0:3].view(torch.float64)
        n = min(int(host[8]), self.capacity)
        return dict(start_loss_sum=float(f[0]), end_loss_sum=float(f[1]), f1_sum=float(f[2]),
                    count=int(host[3]), start_correct=int(host[4]), end_correct=int(host[5]),
                    exact=int(host[6]), invalid=int(host[7]), overflow=int(host[9]),
                    spans=self.spans[:n].cpu().long(), scores=self.scores[:n].cpu())


class TokenEvalAccumulator:
    """Device-side token accumulator of one evaluation pass over a vocabulary-sized output:
    ``{loss_sum (fp64), count, correct, invalid}`` in one int64 buffer (``sky::VocabEvalAccum``).

    ``reset()`` is one memset and ``add()`` two kernel launches of ``vocab_ce`` in eval mode,
    all capturable into a CUDA graph; ``read()`` is the single device-to-host copy of the pass."""

    def __init__(self, V: int, device=None):
        if V < 1 or V > ext().vocab_ce_max_v():
            raise ValueError("TokenEvalAccumulator supports 1 <= V <= {}, got {}".format(
                ext().vocab_ce_max_v(), V))
        self.V = int(V)
        self.buffer = torch.zeros(4, dtype=torch.int64,
                                  device=device if device is not None else "cuda")

    def reset(self) -> None:
        self.buffer.zero_()

    def add(self, logits: torch.Tensor, labels: torch.Tensor, ignore_index: int = -100) -> None:
        logits = logits.detach().reshape(-1, logits.shape[-1])
        if logits.dtype != torch.bfloat16:
            logits = logits.to(torch.bfloat16)
        if logits.shape[1] != self.V:
            raise ValueError("logits have {} classes, the accumulator {}".format(
                logits.shape[1], self.V))
        M, V, labels, ws = _vocab_ce_check(logits, labels)
        ext().vocab_ce(logits=logits.data_ptr(), ldl=logits.stride(0), labels=labels.data_ptr(),
                       M=M, V=V, ignore_index=int(ignore_index), acc=self.buffer.data_ptr(),
                       workspace=ws.data_ptr(), stream=_stream())

    def read(self) -> dict:
        host = self.buffer.cpu()
        return dict(loss_sum=float(host[0:1].view(torch.float64)[0]), count=int(host[1]),
                    correct=int(host[2]), invalid=int(host[3]), classes=self.V)


class EvalAccumulator:
    """Device-side classification accumulator of one evaluation pass: ``{loss_sum (fp64), count,
    invalid, confusion[C, C]}`` in one int64 buffer (the layout of ``sky::EvalAccum``).

    ``reset()`` is one memset and ``add()`` one ``classify_eval`` launch, both capturable into a
    CUDA graph; ``read()`` is the single device-to-host copy of the pass."""

    def __init__(self, C: int, device=None):
        if C < 1 or C > ext().eval_max_classes():
            raise ValueError("EvalAccumulator supports 1 <= C <= {} classes, got {}".format(
                ext().eval_max_classes(), C))
        self.C = int(C)
        self.buffer = torch.zeros(3 + self.C * self.C, dtype=torch.int64,
                                  device=device if device is not None else "cuda")

    def reset(self) -> None:
        self.buffer.zero_()

    def add(self, logits: torch.Tensor, labels: torch.Tensor, ignore_index: int = -100) -> None:
        logits = logits.detach().reshape(-1, logits.shape[-1])
        if logits.dtype != torch.float32:
            logits = logits.float()
        if logits.shape[1] != self.C:
            raise ValueError("logits have {} classes, the accumulator {}".format(
                logits.shape[1], self.C))
        classify_eval(logits, labels.reshape(-1), self.buffer, ignore_index)

    def read(self) -> dict:
        host = self.buffer.cpu()
        return dict(loss_sum=float(host[0:1].view(torch.float64)[0]), count=int(host[1]),
                    invalid=int(host[2]), confusion=host[3:].view(self.C, self.C).clone())
