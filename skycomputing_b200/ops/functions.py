"""Autograd functions that run the BERT layer library on the sm_90a kernels.

One ``torch.autograd.Function`` per *span* of registered layers, so a whole transformer block
(Head + Body + Tail of the reference's layer list) is 7 forward and ~17 backward kernel launches
with no framework work in between; spans that are cut by a stage boundary (Head | Body | Tail
alone or pairs) run the corresponding subset.

Conventions
-----------
* activations are bf16 ``[B, S, H]`` (viewed as ``[B*S, H]``), parameters are fp32 masters with
  bf16 shadows (``ParamBank``); weight/bias gradients are accumulated by the kernels straight into
  the fp32 ``.grad`` buffers (wgrad GEMM epilogue / colsum / LN param-grad kernels), so autograd
  receives ``None`` for every parameter input;
* dropout masks are never stored: every site has an RNG stream id and the backward kernels
  regenerate the forward mask from ``{seed, step}`` kept in device memory;
* stage-boundary fusion: ``in_ch`` / ``out_ch`` (``parallel.p2p.FusedChannel``) make the first
  GEMM wait on panel flags of the received activation, the last LayerNorm write into the next
  stage's HBM, the first dgrad GEMM write its input-gradient tiles into the previous stage's HBM,
  and the last LayerNorm-backward wait on the panels of the gradient it receives.

Reference parity: the math is that of scaelum/model/bert_layers.py:171-395 (see the per-op
citations in csrc/kernels/*.cu); tests/test_layers_gpu.py checks every span against the fp32
PyTorch oracle in ``skycomputing_b200.models.bert_layers``.
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import torch

from . import native as nat


# --------------------------------------------------------------------------------------------
# parameter bank: fp32 masters (possibly several nn.Parameters fused into one flat buffer) with a
# bf16 shadow and a flat fp32 gradient buffer
# --------------------------------------------------------------------------------------------
class ParamBank:
    """Fuses ``params`` (same trailing shape) along dim 0 into one flat fp32 master + grad buffer.

    The original ``nn.Parameter`` objects keep their names/shapes (state_dict compatibility) but
    become views into the flat storage; ``shadow()`` returns the bf16 compute copy, refreshed when
    a master was modified through torch (version counter) - the fused optimizer refreshes it
    itself in the same kernel that applies the update.
    """

    def __init__(self, params: Sequence[torch.nn.Parameter], need_shadow: bool = True):
        self.params = list(params)
        self.need_shadow = need_shadow
        self.flat: Optional[torch.Tensor] = None
        self.flat_grad: Optional[torch.Tensor] = None
        self._shadow: Optional[torch.Tensor] = None
        self._versions: List[int] = []
        self._ptrs: List[int] = []
        # weight banks whose gradient is produced by the wgrad GEMM: the fused optimizer may leave
        # the gradient un-zeroed (`overwrite_first`) and flag it `fresh`; the first wgrad of the
        # next step then STORES instead of accumulating (saves 4 B/parameter of SGD traffic and
        # turns that epilogue's red.add into plain stores)
        self.wgrad_target = False
        self.overwrite_first = False
        self.fresh = False
        # encoder weight banks (SpanParams) may have the plain SGD update applied by the epilogue
        # of their wgrad GEMM instead of by the optimizer (`update_in_wgrad_ok`); `wgrad_sgd` =
        # (lr, weight_decay, grad_scale) while an engine arms the backward that produces the
        # step's last gradient of the bank (EngineBase._arm_wgrad_sgd)
        self.update_in_wgrad_ok = False
        self.wgrad_sgd: Optional[tuple] = None
        # the word-embedding table shared with a masked-language-model decoder on the same stage:
        # it has two gradient writers (embed_bwd's atomics, the decoder wgrad's red.add, possibly
        # on the side stream or deferred), so it is never `overwrite_first` and never updated
        # inside a wgrad GEMM
        self.tied = False

    def _materialise(self) -> None:
        p0 = self.params[0]
        rows = sum(p.shape[0] for p in self.params)
        shape = (rows,) + tuple(p0.shape[1:])
        flat = torch.empty(shape, dtype=torch.float32, device=p0.device)
        off = 0
        with torch.no_grad():
            for p in self.params:
                n = p.shape[0]
                flat[off:off + n].copy_(p.data.float())
                p.data = flat[off:off + n]
                off += n
        self.flat = flat
        self.flat_grad = torch.zeros_like(flat)
        self._bind_grads()
        self._ptrs = [p.data_ptr() for p in self.params]
        self._shadow = None

    def _bind_grads(self) -> None:
        off = 0
        for p in self.params:
            n = p.shape[0]
            p.grad = self.flat_grad[off:off + n]
            off += n

    def ensure(self) -> None:
        if self.flat is None or any(p.data_ptr() != q for p, q in zip(self.params, self._ptrs)) \
                or self.flat.device != self.params[0].device:
            self._materialise()
        elif any(p.grad is None or p.grad.data_ptr() < self.flat_grad.data_ptr()
                 or p.grad.data_ptr() >= self.flat_grad.data_ptr() + self.flat_grad.numel() * 4
                 for p in self.params):
            # optimizer.zero_grad(set_to_none=True) or a foreign grad tensor: rebind (zeroed)
            self.flat_grad.zero_()
            self._bind_grads()

    def master(self) -> torch.Tensor:
        self.ensure()
        return self.flat

    def grad(self) -> torch.Tensor:
        self.ensure()
        return self.flat_grad

    def shadow(self) -> torch.Tensor:
        self.ensure()
        versions = [p._version for p in self.params]
        if self._shadow is None or versions != self._versions:
            if self._shadow is None:
                self._shadow = torch.empty(self.flat.shape, dtype=torch.bfloat16,
                                           device=self.flat.device)
            nat.cast_f32_to_bf16_(self.flat, self._shadow)
            self._versions = versions
        return self._shadow

    def mark_shadow_fresh(self) -> None:
        self._versions = [p._version for p in self.params]

    def sgd_descriptor(self, momentum_buf: Optional[torch.Tensor] = None,
                       second_moment: Optional[torch.Tensor] = None):
        self.ensure()
        if self.need_shadow and self._shadow is None:
            self.shadow()
        return (self.flat.data_ptr(), self.flat_grad.data_ptr(),
                0 if momentum_buf is None else momentum_buf.data_ptr(),
                self._shadow.data_ptr() if (self.need_shadow and self._shadow is not None) else 0,
                self.flat.numel(), 1 if self.overwrite_first else 0,
                0 if second_moment is None else second_moment.data_ptr())


class SpanParams:
    """Parameter banks + hyper-parameters of one transformer-block span (any of Head/Body/Tail)."""

    def __init__(self, head=None, body=None, tail=None):
        self.has_head = head is not None
        self.has_body = body is not None
        self.has_tail = tail is not None
        self.banks: List[ParamBank] = []
        self.heads = 0
        self.p_attn = 0.0
        self.p_hidden = 0.0
        self.eps = 1e-12
        self.rng: Optional[nat.RngState] = None
        self.rng_base = 0
        if head is not None:
            att = head.attention
            self.heads = att.self.num_attention_heads
            self.p_attn = float(att.self.dropout.p)
            self.p_hidden = float(att.output.dropout.p)
            self.eps = float(att.output.LayerNorm.eps)
            self.wqkv = self._bank([att.self.query.weight, att.self.key.weight, att.self.value.weight])
            self.bqkv = self._bank([att.self.query.bias, att.self.key.bias, att.self.value.bias], False)
            self.wo = self._bank([att.output.dense.weight])
            self.bo = self._bank([att.output.dense.bias], False)
            self.g1 = self._bank([att.output.LayerNorm.weight], False)
            self.b1n = self._bank([att.output.LayerNorm.bias], False)
        if body is not None:
            lin = body.intermediate.dense_act
            self.w1 = self._bank([lin.weight])
            self.b1 = self._bank([lin.bias], False)
        if tail is not None:
            out = tail.output
            self.p_hidden = float(out.dropout.p)
            self.eps = float(out.LayerNorm.eps)
            self.w2 = self._bank([out.dense.weight])
            self.b2 = self._bank([out.dense.bias], False)
            self.g2 = self._bank([out.LayerNorm.weight], False)
            self.b2n = self._bank([out.LayerNorm.bias], False)

    def _bank(self, params, need_shadow: bool = True) -> ParamBank:
        b = ParamBank(params, need_shadow)
        # the weights (the banks with a shadow): BertSpanFn.backward enqueues an armed wgrad
        # behind the dgrad that reads the shadow it rewrites
        b.update_in_wgrad_ok = need_shadow
        self.banks.append(b)
        return b

    def all_params(self) -> List[torch.nn.Parameter]:
        return [p for b in self.banks for p in b.params]


def _flat2d(t: torch.Tensor) -> torch.Tensor:
    return t.reshape(-1, t.shape[-1])


def _ch_kwargs_wait(ch, mb: int) -> dict:
    return dict(wait_flags=ch.act_flags_ptr(mb), wait_epoch=ch.epoch_ptr, wait_mult=ch.act_wait_mult,
                error_flag=ch.error_ptr)


class BertSpanFn(torch.autograd.Function):
    """forward(ctx, sp, training, in_ch, out_ch, mb, n_in, *inputs_then_params)."""

    @staticmethod
    def forward(ctx, sp: SpanParams, training: bool, in_ch, out_ch, mb: int, n_in: int, *tensors):
        out, saved, shape3 = BertSpanFn._run(sp, training, in_ch, out_ch, mb, tensors[:n_in], True)
        ctx.sp, ctx.saved, ctx.training = sp, saved, training
        ctx.in_ch, ctx.out_ch, ctx.mb, ctx.n_in = in_ch, out_ch, mb, n_in
        ctx.n_tensors = len(tensors)
        ctx.shape3 = shape3
        return out

    @staticmethod
    def infer(sp: SpanParams, in_ch, out_ch, mb: int, inputs):
        """Inference forward (eval mode, no autograd): the same kernels and outputs as
        ``forward(training=False)``, without what only backward reads - no FFN1 pre-activation
        copy, no pre-LayerNorm sums, no attention LSE - and without an autograd node."""
        return BertSpanFn._run(sp, False, in_ch, out_ch, mb, inputs, False)[0]

    @staticmethod
    def _run(sp: SpanParams, training: bool, in_ch, out_ch, mb, inputs, keep: bool):
        """Returns (outputs, tensors saved for backward, (B, S, H)); ``keep`` = False skips every
        buffer that only backward needs."""
        # slot index on the inbound link / on the outbound link: the same number in a plain
        # pipeline (micro-batch j), different ones on the wrap-around link of a looped pipeline
        mb_in, mb_out = mb if isinstance(mb, tuple) else (mb, mb)
        rng = sp.rng
        p_attn = sp.p_attn if training else 0.0
        p_hid = sp.p_hidden if training else 0.0
        if (p_attn > 0 or p_hid > 0) and rng is None:
            raise RuntimeError("dropout requested but the span has no RngState attached")
        saved = {}
        if sp.has_head:
            x3, mask = inputs[0], inputs[1]
            B, S, H = x3.shape
            x = _flat2d(x3)
            mask2 = None if mask is None else mask.reshape(B, S)
            wait = _ch_kwargs_wait(in_ch, mb_in) if in_ch is not None else {}
            qkv = nat.gemm(x, sp.wqkv.shadow(), bias=sp.bqkv.master(), **wait)
            ctxt, lse = nat.attention_fwd(qkv, mask2, B, S, sp.heads, dropout_p=p_attn, rng=rng,
                                          rng_stream=sp.rng_base + 1, save_lse=keep)
            ln_out = {}
            if out_ch is not None and not sp.has_body:
                ln_out = dict(y_ptr=out_ch.peer_act_ptr(mb_out), signal_flags=out_ch.peer_act_flags_ptr(mb_out))
            y1, z1, mean1, rstd1 = _gemm_ln(ctxt, sp.wo, sp.bo, x, sp.g1, sp.b1n, sp.eps, p_hid, rng,
                                            sp.rng_base + 2, ln_out, save_z=keep)
            if keep:
                saved.update(x=x, mask2=mask2, qkv=qkv, ctxt=ctxt, lse=lse, z1=z1, mean1=mean1,
                             rstd1=rstd1)
            a = y1
            shape3 = (B, S, H)
        else:
            mask = inputs[-1]
            if sp.has_body:
                a3 = inputs[0]
                B, S, H = a3.shape
                a = _flat2d(a3)
            else:
                inter3, a3 = inputs[0], inputs[1]
                B, S, H = a3.shape
                a = _flat2d(a3)
            shape3 = (B, S, H)
        if sp.has_body:
            wait = _ch_kwargs_wait(in_ch, mb_in) if (in_ch is not None and not sp.has_head) else {}
            I = sp.w1.master().shape[0]
            h1 = torch.empty((a.shape[0], I), dtype=torch.bfloat16, device=a.device) if keep else None
            inter = nat.gemm(a, sp.w1.shadow(), bias=sp.b1.master(), act=nat.ACT_GELU, out2=h1, **wait)
            if keep:
                saved.update(h1=h1)
        elif sp.has_tail:
            inter = _flat2d(inputs[0])
        if sp.has_tail:
            wait = _ch_kwargs_wait(in_ch, mb_in) if (in_ch is not None and not sp.has_body) else {}
            ln_out = {}
            if out_ch is not None:
                ln_out = dict(y_ptr=out_ch.peer_act_ptr(mb_out), signal_flags=out_ch.peer_act_flags_ptr(mb_out))
            y2, z2, mean2, rstd2 = _gemm_ln(inter, sp.w2, sp.b2, a, sp.g2, sp.b2n, sp.eps, p_hid, rng,
                                            sp.rng_base + 3, ln_out, save_z=keep, **wait)
            if keep:
                saved.update(z2=z2, mean2=mean2, rstd2=rstd2)
        if keep and (sp.has_body or sp.has_tail):
            saved.update(a=a, inter=inter)
        B, S, H = shape3
        if sp.has_tail:
            out = y2.view(B, S, H) if y2 is not None else _dummy_out(a)
        elif sp.has_body:
            # the pass-through attention output is only returned when this span produced it;
            # a span that starts at Body lets the caller forward its own input tensor
            out = (inter.view(B, S, -1), a.view(B, S, H)) if sp.has_head else inter.view(B, S, -1)
        else:
            out = y1.view(B, S, H) if y1 is not None else _dummy_out(x)
        return out, saved, shape3

    @staticmethod
    def backward(ctx, *grads):
        sp, sv = ctx.sp, ctx.saved
        in_ch, out_ch = ctx.in_ch, ctx.out_ch
        mb_in, mb_out = ctx.mb if isinstance(ctx.mb, tuple) else (ctx.mb, ctx.mb)
        rng = sp.rng
        p_attn = sp.p_attn if ctx.training else 0.0
        p_hid = sp.p_hidden if ctx.training else 0.0
        B, S, H = ctx.shape3
        M = B * S
        d_a_extra = None  # gradient flowing into `a` (attention output) besides the FFN1 dgrad
        d_inter = None
        g_in: List[Optional[torch.Tensor]] = [None] * ctx.n_in
        if sp.has_tail:
            wait = {}
            if out_ch is not None:
                dy2 = out_ch.grad_view(mb_out, M, H)
                wait = dict(wait_flags=out_ch.grad_flags_ptr(mb_out), wait_epoch=out_ch.epoch_ptr,
                            wait_mult=out_ch.grad_wait_mult, error_flag=out_ch.error_ptr)
            else:
                dy2 = _flat2d(grads[0]).contiguous()
            dz2, dz2d = nat.layernorm_bwd(dy2, sv["z2"], sv["mean2"], sv["rstd2"], sp.g2.master(),
                                          None, None, dropout_p=p_hid, rng=rng,
                                          rng_stream=sp.rng_base + 3, **wait)
            g2 = dz2d if dz2d is not None else dz2
            _ln_pgrad(dy2, sv["z2"], sv["mean2"], sv["rstd2"], sp.g2, sp.b2n, g2, sp.b2)
            if sp.has_body:
                d_h1 = _wgrad_dgrad(g2, sv["inter"], sp.w2, None, lambda: nat.gemm(
                    g2, sp.w2.shadow(), b_mn=True, aux=sv["h1"], act=nat.ACT_DGELU_MUL_AUX))
            else:
                send = _grad_send_kwargs(in_ch, mb_in, which=0)
                d_inter = _wgrad_dgrad(g2, sv["inter"], sp.w2, None,
                                       lambda: nat.gemm(g2, sp.w2.shadow(), b_mn=True, **send))
            d_a_extra = dz2
        elif sp.has_body:
            # span ends after Body: grads = (d_inter, d_attn_out)
            gi = _flat2d(grads[0]).contiguous()
            d_h1 = torch.empty_like(gi)
            nat.ext().dgelu_mul(gi.data_ptr(), sv["h1"].data_ptr(), d_h1.data_ptr(), gi.numel(),
                                torch.cuda.current_stream().cuda_stream)
            d_a_extra = None
            if sp.has_head and len(grads) > 1 and grads[1] is not None:
                d_a_extra = _flat2d(grads[1]).contiguous()
        if sp.has_body:
            send = _grad_send_kwargs(in_ch, mb_in, which=0) if not sp.has_head else {}
            d_a = _wgrad_dgrad(d_h1, sv["a"], sp.w1, sp.b1, lambda: nat.gemm(
                d_h1, sp.w1.shadow(), b_mn=True, aux=d_a_extra, add_aux=d_a_extra is not None,
                **send))
        elif sp.has_tail:
            d_a = d_a_extra  # tail-only span: grad of the attn_out input is dz2
        else:
            d_a = None
        if sp.has_head:
            wait = {}
            if not sp.has_body:
                if out_ch is not None:
                    dy1 = out_ch.grad_view(mb_out, M, H)
                    wait = dict(wait_flags=out_ch.grad_flags_ptr(mb_out), wait_epoch=out_ch.epoch_ptr,
                                wait_mult=out_ch.grad_wait_mult, error_flag=out_ch.error_ptr)
                else:
                    dy1 = _flat2d(grads[0]).contiguous()
            else:
                dy1 = d_a
            dz1, dz1d = nat.layernorm_bwd(dy1, sv["z1"], sv["mean1"], sv["rstd1"], sp.g1.master(),
                                          None, None, dropout_p=p_hid, rng=rng,
                                          rng_stream=sp.rng_base + 2, **wait)
            g1 = dz1d if dz1d is not None else dz1
            _ln_pgrad(dy1, sv["z1"], sv["mean1"], sv["rstd1"], sp.g1, sp.b1n, g1, sp.bo)
            dctx = _wgrad_dgrad(g1, sv["ctxt"], sp.wo, None,
                                lambda: nat.gemm(g1, sp.wo.shadow(), b_mn=True))
            dqkv = nat.attention_bwd(sv["qkv"], sv["mask2"], sv["ctxt"], sv["lse"], dctx, B, S,
                                     sp.heads, dropout_p=p_attn, rng=rng, rng_stream=sp.rng_base + 1)
            send = _grad_send_kwargs(in_ch, mb_in, which=0)
            dx = _wgrad_dgrad(dqkv, sv["x"], sp.wqkv, sp.bqkv, lambda: nat.gemm(
                dqkv, sp.wqkv.shadow(), b_mn=True, aux=dz1, add_aux=True, **send))
            g_in[0] = None if dx is None else dx.view(B, S, H)
        elif sp.has_body:
            g_in[0] = None if d_a is None else d_a.view(B, S, H)
        else:  # tail only: inputs (inter, attn_out, mask)
            g_in[0] = None if d_inter is None else d_inter.view(B, S, -1)
            g_in[1] = d_a.view(B, S, H)
        ctx.saved = None
        return (None, None, None, None, None, None, *g_in, *([None] * (ctx.n_tensors - ctx.n_in)))


# Weight-gradient deferral ("B before W"): the input-gradient chain of a stage is on the critical
# path of the pipeline (the previous stage waits for it), the weight / bias gradients are not.
# With deferral on, backward only queues them; the engine flushes the queue right after the
# stage's last dgrad GEMM has published its tiles to the previous stage.
_DEFER_WGRAD = [False]
_WGRAD_QUEUE: list = []
# "immediate" mode: every weight gradient is launched at once, but on a side stream that forks
# from the current point of the main stream, so it overlaps the rest of the dgrad chain.
_WGRAD_STREAM: list = [None]
_WGRAD_KEEP: list = []


def set_wgrad_stream(stream) -> None:
    _WGRAD_STREAM[0] = stream


def wgrad_keepalive() -> list:
    return _WGRAD_KEEP


def set_wgrad_deferral(on: bool) -> None:
    _DEFER_WGRAD[0] = bool(on)
    if not on:
        flush_wgrads()


def flush_wgrads() -> list:
    """Launch every queued weight / bias gradient on the CURRENT stream; returns the queued
    tensors so that a caller that flushed onto a side stream can keep them alive until it joins."""
    q = list(_WGRAD_QUEUE)
    _WGRAD_QUEUE.clear()
    for item in q:
        _run_param_grad(item)
    return q


def _run_param_grad(item) -> None:
    if item[0] == "ln":
        _, dy, z, mean, rstd, gbank, bbank, x2, bias_bank = item
        nat.ln_param_grad(dy, z, mean, rstd, gbank.grad(), bbank.grad(), x2,
                          None if bias_bank is None else bias_bank.grad())
    else:
        g, act, wbank, bbank, sgd = item
        wbank.wgrad_target = True
        first = wbank.overwrite_first and wbank.fresh
        wbank.fresh = False
        if sgd is None:
            nat.gemm(g, act, a_mn=True, b_mn=True, out=wbank.grad(), accumulate=not first)
        else:
            # the step's last gradient of the bank: the epilogue applies the SGD update to the
            # master and its shadow and does not store the gradient
            lr, weight_decay, grad_scale = sgd
            nat.gemm(g, act, a_mn=True, b_mn=True, out=wbank.grad(), accumulate=not first,
                     sgd_master=wbank.master(), sgd_shadow=wbank.shadow(), sgd_lr=lr,
                     sgd_weight_decay=weight_decay, sgd_grad_scale=grad_scale)
        if bbank is not None:  # else: the column sum rides in the LayerNorm parameter-gradient kernel
            nat.colsum_(g, bbank.grad())


def _ln_pgrad(dy, z, mean, rstd, gbank: ParamBank, bbank: ParamBank, x2=None,
              bias_bank: Optional[ParamBank] = None) -> None:
    """LayerNorm gamma / beta gradients: like the weight gradients they are not needed by the
    previous stage, so they follow the same deferral / side-stream policy."""
    item = ("ln", dy, z, mean, rstd, gbank, bbank, x2, bias_bank)
    if _DEFER_WGRAD[0]:
        _WGRAD_QUEUE.append(item)
        return
    side = _WGRAD_STREAM[0]
    if side is not None:
        side.wait_stream(torch.cuda.current_stream(dy.device))
        with torch.cuda.stream(side):
            _run_param_grad(item)
        _WGRAD_KEEP.append((dy, z, mean, rstd, x2))
        return
    _run_param_grad(item)


def pending_wgrads() -> int:
    return len(_WGRAD_QUEUE)


def _wgrad(g: torch.Tensor, act: torch.Tensor, wbank: ParamBank,
           bbank: Optional[ParamBank]) -> None:
    """dW += g^T act (both operands MN-major over the token dimension), db += colsum(g) unless
    ``bbank`` is None (the column sum then rides in the LayerNorm parameter-gradient kernel).
    An armed bank (``wbank.wgrad_sgd``) gets its SGD update in the same GEMM; the arming is read
    here, so that a deferred gradient applies the update it was queued with."""
    item = (g, act, wbank, bbank, wbank.wgrad_sgd)
    if _DEFER_WGRAD[0]:
        _WGRAD_QUEUE.append(item)
        return
    side = _WGRAD_STREAM[0]
    if side is not None:
        side.wait_stream(torch.cuda.current_stream(g.device))
        with torch.cuda.stream(side):
            _run_param_grad(item)
        _WGRAD_KEEP.append((g, act))
        return
    _run_param_grad(item)


def _wgrad_dgrad(g: torch.Tensor, act: torch.Tensor, wbank: ParamBank,
                 bbank: Optional[ParamBank], dgrad):
    """``_wgrad(g, act, wbank, bbank)`` and ``dgrad()``, the input-gradient GEMM that reads
    ``wbank``'s shadow; returns what ``dgrad()`` returns.  The weight gradient is enqueued first,
    so that on the side stream it overlaps the dgrad, unless it is armed: then it rewrites the
    shadow and must fork after the dgrad has been enqueued."""
    if wbank.wgrad_sgd is None:
        _wgrad(g, act, wbank, bbank)
        return dgrad()
    out = dgrad()
    _wgrad(g, act, wbank, bbank)
    return out


def _dummy_out(like: torch.Tensor) -> torch.Tensor:
    """Stand-in output for spans whose real output was written into the next stage's HBM."""
    return torch.zeros(1, dtype=torch.bfloat16, device=like.device)


def _gemm_ln(a, wbank, bbank, residual, gbank, betabank, eps, p_drop, rng, rng_stream,
             ln_out: dict, save_z: bool = True, **wait):
    """Dense + bias + dropout + residual + LayerNorm (the reference's BertSelfOutput / BertOutput,
    scaelum/model/bert_layers.py:285-289,323-327).  ONE wgmma kernel with the LayerNorm in the
    GEMM epilogue whenever the row fits a thread-block cluster; with ``ln_out`` (peer pointer + panel
    flags of a fused stage boundary) that kernel stores y straight into the next stage's HBM.  Otherwise GEMM, then the standalone LayerNorm.
    Returns (y | None, z, mean, rstd); ``z`` is None when ``save_z`` is False and the fused kernel
    runs (the unfused path needs z as the LayerNorm input anyway)."""
    M, N = a.shape[0], wbank.master().shape[0]
    # both ends of a fused boundary evaluate the same predicate on the same (rows, cols): the
    # consumer's expected signal count per panel follows from it (parallel/p2p.py)
    if nat.gemm_ln_supported(M, N):
        return nat.gemm_ln(a, wbank.shadow(), gbank.master(), betabank.master(), eps=eps,
                           bias=bbank.master(), residual=residual, dropout_p=p_drop, rng=rng,
                           rng_stream=rng_stream, save_z=save_z, y_ld=N, **ln_out, **wait)
    z = nat.gemm(a, wbank.shadow(), bias=bbank.master(), aux=residual, add_aux=True,
                 dropout_p=p_drop, rng=rng, rng_stream=rng_stream, **wait)
    y, mean, rstd = _ln_fwd(z, gbank.master(), betabank.master(), eps, **ln_out)
    return y, z, mean, rstd


def _ln_fwd(z, gamma, beta, eps, y_ptr: int = 0, signal_flags: int = 0):
    M, H = z.shape
    mean = torch.empty(M, dtype=torch.float32, device=z.device)
    rstd = torch.empty(M, dtype=torch.float32, device=z.device)
    if y_ptr:
        y = None
        yp = y_ptr
    else:
        y = torch.empty_like(z)
        yp = y.data_ptr()
    nat.ext().layernorm_fwd(z=z.data_ptr(), y=yp, mean=mean.data_ptr(), rstd=rstd.data_ptr(),
                            gamma=gamma.data_ptr(), beta=beta.data_ptr(), M=M, H=H, eps=eps,
                            signal_flags=signal_flags,
                            stream=torch.cuda.current_stream().cuda_stream)
    return y, mean, rstd


def _grad_send_kwargs(in_ch, mb: int, which: int) -> dict:
    """dgrad GEMM epilogue writes the input gradient straight into the previous stage's HBM."""
    if in_ch is None:
        return {}
    return dict(out_ptr=in_ch.peer_grad_ptr(mb), out_ld=in_ch.grad_ld,
                signal_flags=in_ch.peer_grad_flags_ptr(mb))


# --------------------------------------------------------------------------------------------
# embeddings / pooler / classifier / loss
# --------------------------------------------------------------------------------------------
def _flat_int64(t: torch.Tensor) -> torch.Tensor:
    """The embedding kernels read ids, token types and the attention mask as contiguous int64:
    int32 ids or a bool / int32 mask (as HF-style pipelines produce) are converted, not
    reinterpreted."""
    return t.reshape(-1).to(torch.int64).contiguous()


class EmbeddingsFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, emb, training: bool, out_ch, mb: int, input_ids, token_type_ids,
                attention_mask, *params):
        B, S = input_ids.shape
        H = emb.word.master().shape[1]
        dev = input_ids.device
        ids, tts, am = (_flat_int64(t) for t in (input_ids, token_type_ids, attention_mask))
        out = torch.empty((B * S, H), dtype=torch.bfloat16, device=dev)
        ext_mask = torch.empty((B * S,), dtype=torch.float32, device=dev)
        mean = torch.empty(B * S, dtype=torch.float32, device=dev)
        rstd = torch.empty(B * S, dtype=torch.float32, device=dev)
        p = emb.p_drop if training else 0.0
        nat.ext().embed_fwd(ids=ids.data_ptr(), tts=tts.data_ptr(), amask=am.data_ptr(),
                            word=emb.word.master().data_ptr(), pos=emb.pos.master().data_ptr(),
                            type=emb.type.master().data_ptr(), gamma=emb.gamma.master().data_ptr(),
                            beta=emb.beta.master().data_ptr(), out=out.data_ptr(),
                            ext_mask=ext_mask.data_ptr(), mean=mean.data_ptr(), rstd=rstd.data_ptr(),
                            B=B, S=S, H=H, eps=emb.eps, dropout_p=p,
                            rng_state=0 if emb.rng is None else emb.rng.ptr,
                            rng_stream=emb.rng_base, stream=torch.cuda.current_stream().cuda_stream)
        ctx.emb, ctx.training = emb, training
        ctx.saved = (ids, tts, mean, rstd)
        ctx.dims = (B, S, H)
        ctx.n_params = len(params)
        ctx.mark_non_differentiable(ext_mask)
        return out.view(B, S, H), ext_mask.view(B, 1, 1, S)

    @staticmethod
    def backward(ctx, dout, _dmask):
        emb = ctx.emb
        ids, tts, mean, rstd = ctx.saved
        B, S, H = ctx.dims
        p = emb.p_drop if ctx.training else 0.0
        dout = dout.reshape(B * S, H).contiguous()
        nat.ext().embed_bwd(dout=dout.data_ptr(), ids=ids.data_ptr(), tts=tts.data_ptr(),
                            word=emb.word.master().data_ptr(), pos=emb.pos.master().data_ptr(),
                            type=emb.type.master().data_ptr(), gamma=emb.gamma.master().data_ptr(),
                            mean=mean.data_ptr(), rstd=rstd.data_ptr(),
                            dword=emb.word.grad().data_ptr(), dpos=emb.pos.grad().data_ptr(),
                            dtype=emb.type.grad().data_ptr(), dgamma=emb.gamma.grad().data_ptr(),
                            dbeta=emb.beta.grad().data_ptr(), B=B, S=S, H=H,
                            type_rows=emb.type.master().shape[0], dropout_p=p,
                            rng_state=0 if emb.rng is None else emb.rng.ptr,
                            rng_stream=emb.rng_base, stream=torch.cuda.current_stream().cuda_stream)
        ctx.saved = None
        return (None, None, None, None, None, None, None, *([None] * ctx.n_params))


class EmbeddingParams:
    def __init__(self, mod):
        self.word = ParamBank([mod.word_embeddings.weight], False)
        if getattr(mod, "_tied_head", None) is not None:
            self.tie_word_bank()
        self.pos = ParamBank([mod.position_embeddings.weight], False)
        self.type = ParamBank([mod.token_type_embeddings.weight], False)
        self.gamma = ParamBank([mod.LayerNorm.weight], False)
        self.beta = ParamBank([mod.LayerNorm.bias], False)
        self.banks = [self.word, self.pos, self.type, self.gamma, self.beta]
        self.eps = float(mod.LayerNorm.eps)
        self.p_drop = float(mod.dropout.p)
        self.rng: Optional[nat.RngState] = None
        self.rng_base = 0

    def tie_word_bank(self) -> None:
        """The table is also the decoder weight of a tied head on this stage: the decoder GEMMs
        read a bf16 shadow, which the fused optimizers keep fresh; the embedding kernels keep
        reading the fp32 master."""
        self.word.need_shadow = True
        self.word.tied = True

    def all_params(self):
        return [p for b in self.banks for p in b.params]


class SmallLinearFn(torch.autograd.Function):
    """Pooler (first-token gather + dense + tanh) and classifier (input dropout + dense)."""

    @staticmethod
    def forward(ctx, lp, training: bool, x, *params):
        w, b = lp.w.master(), lp.b.master()
        N, K = w.shape
        if lp.first_token:
            B, S, H = x.shape
            M, ldx = B, S * H
            xs = x.contiguous()
        else:
            xs = x.contiguous()
            M, ldx = xs.shape[0], xs.shape[1]
        x_bf16 = xs.dtype == torch.bfloat16
        y = torch.empty((M, N), dtype=torch.float32, device=xs.device)
        p = lp.p_drop if training else 0.0
        nat.ext().small_linear_fwd(x=xs.data_ptr(), x_bf16=x_bf16, ldx=ldx, w=w.data_ptr(),
                                   b=b.data_ptr(), y=y.data_ptr(), M=M, N=N, K=K,
                                   act_tanh=1 if lp.act_tanh else 0, dropout_p=p,
                                   rng_state=0 if lp.rng is None else lp.rng.ptr,
                                   rng_stream=lp.rng_base, stream=torch.cuda.current_stream().cuda_stream)
        ctx.lp, ctx.training = lp, training
        ctx.saved = (xs, y, M, ldx, x_bf16)
        ctx.n_params = len(params)
        return y

    @staticmethod
    def backward(ctx, dy):
        lp = ctx.lp
        xs, y, M, ldx, x_bf16 = ctx.saved
        w = lp.w.master()
        N, K = w.shape
        dy = dy.contiguous().float()
        p = lp.p_drop if ctx.training else 0.0
        if lp.first_token:
            dx = torch.zeros_like(xs)
            lddx = ldx
        else:
            dx = torch.empty_like(xs)
            lddx = K
        nat.ext().small_linear_bwd(x=xs.data_ptr(), x_bf16=x_bf16, ldx=ldx, w=w.data_ptr(),
                                   y=y.data_ptr(), dy=dy.data_ptr(), dx=dx.data_ptr(),
                                   dx_bf16=x_bf16, lddx=lddx, dw=lp.w.grad().data_ptr(),
                                   db=lp.b.grad().data_ptr(), M=M, N=N, K=K,
                                   act_tanh=1 if lp.act_tanh else 0, dropout_p=p,
                                   rng_state=0 if lp.rng is None else lp.rng.ptr,
                                   rng_stream=lp.rng_base, stream=torch.cuda.current_stream().cuda_stream)
        ctx.saved = None
        return (None, None, dx, *([None] * ctx.n_params))


class PoolerFn(torch.autograd.Function):
    """BertPooler on the tensor-core GEMM: first-token rows are read through a strided TMA view
    (no gather copy), bias + tanh run in the epilogue; backward = two more GEMMs.

    Reference: scaelum/model/bert_layers.py:381-395.
    """

    @staticmethod
    def forward(ctx, lp, hidden, *params):
        B, S, H = hidden.shape
        hidden = hidden.contiguous()
        x0 = hidden.view(B, S * H)[:, :H]          # [B, H] view, row stride S*H
        y = nat.gemm(x0, lp.w.shadow(), bias=lp.b.master(), act=nat.ACT_TANH,
                     out_dtype=torch.float32)
        ctx.lp = lp
        ctx.saved = (hidden, y)
        ctx.n_params = len(params)
        return y

    @staticmethod
    def backward(ctx, dy):
        lp = ctx.lp
        hidden, y = ctx.saved
        B, S, H = hidden.shape
        x0 = hidden.view(B, S * H)[:, :H]
        g = (dy.float() * (1.0 - y * y))
        lp.b.grad().add_(g.sum(0))
        gb = g.to(torch.bfloat16)
        # dW[n,k] += sum_b g[b,n] x0[b,k]  (both operands MN-major over the batch dimension)
        nat.gemm(gb, x0, a_mn=True, b_mn=True, out=lp.w.grad(), accumulate=True)
        dhidden = torch.zeros_like(hidden)
        nat.gemm(gb, lp.w.shadow(), b_mn=True, out=dhidden.view(B, S * H)[:, :H])
        ctx.saved = None
        return (None, dhidden, *([None] * ctx.n_params))


class SmallLinearParams:
    def __init__(self, weight, bias, act_tanh: bool, first_token: bool, p_drop: float = 0.0):
        # the pooler (first_token) also runs on the GEMM kernel -> keep a bf16 shadow of its weight
        self.w = ParamBank([weight], need_shadow=first_token)
        self.b = ParamBank([bias], False)
        self.banks = [self.w, self.b]
        self.act_tanh = act_tanh
        self.first_token = first_token
        self.p_drop = p_drop
        self.rng: Optional[nat.RngState] = None
        self.rng_base = 0

    def all_params(self):
        return [p for b in self.banks for p in b.params]


def mlm_slots_ref(labels: torch.Tensor, P: int, ignore_index: int = -100, V: int = 0):
    """The slot layout of a sparse masked-language-model head, in plain torch (the eager path and
    the reference of the ``mlm_gather`` / ``mlm_scatter`` kernels).

    ``labels`` [B, S].  Sequence b owns slots [b*P, (b+1)*P); its labelled positions (label !=
    ``ignore_index``), in position order, fill them from the front.  Returns ``(row_of_slot [B*P],
    slot_of_row [B*S], slot_labels [B*P])``, all int64: the flat row (b*S + position) decoded in a
    slot or -1 for an empty slot, the slot of a row or -1 for a row that is not decoded, and the
    label of each slot (``ignore_index`` when empty).  A sequence with more than P labelled
    positions drops the extra ones and gets the out-of-range label ``V`` in its last slot, so that
    the overflow is never silent."""
    B, S = labels.shape
    dev = labels.device
    keep = labels != ignore_index
    rank = keep.long().cumsum(1) - 1
    fit = keep & (rank < P)
    slot = (torch.arange(B, device=dev).unsqueeze(1) * P + rank)[fit]
    rows = torch.arange(B * S, device=dev).view(B, S)[fit]
    row_of_slot = torch.full((B * P,), -1, dtype=torch.int64, device=dev)
    slot_of_row = torch.full((B * S,), -1, dtype=torch.int64, device=dev)
    slot_labels = torch.full((B * P,), int(ignore_index), dtype=torch.int64, device=dev)
    row_of_slot[slot] = rows
    slot_of_row[rows] = slot
    slot_labels[slot] = labels[fit].to(torch.int64)
    slot_labels.view(B, P)[keep.sum(1) > P, P - 1] = int(V)
    return row_of_slot, slot_of_row, slot_labels


def split_pretraining_labels(labels: torch.Tensor):
    """The labels of a masked-LM + next-sentence item are ONE int64 tensor ``[..., S + 1]``:
    columns 0..S-1 are the token labels (``ignore_index`` where a position is not predicted),
    column S is the next-sentence label (0: B follows A, 1: B is random).  Returns ``(mlm [...,
    S], nsp [...])`` as views.  One tensor keeps the engine's chunking, label buffers and label
    routing unchanged; this function and ``join_pretraining_labels`` are the only places that
    know the layout."""
    return labels[..., :-1], labels[..., -1]


def join_pretraining_labels(mlm: torch.Tensor, nsp: torch.Tensor) -> torch.Tensor:
    """Inverse of ``split_pretraining_labels``: ``mlm`` [B, S'] (or flat B*S') and ``nsp`` [B]
    -> [B, S' + 1] int64."""
    nsp = nsp.reshape(-1, 1).to(torch.int64)
    return torch.cat([mlm.reshape(nsp.shape[0], -1).to(torch.int64), nsp], dim=1)


class MaskedLMHeadParams:
    """Parameter banks of ``BertTailForMaskedLM``: transform dense (+ GELU), LayerNorm, decoder;
    and the head's slot contract (``max_predictions``, ``ignore_index``)."""

    def __init__(self, mod):
        tr = mod.transform
        self.w_t = ParamBank([tr.dense_act.weight])
        self.b_t = ParamBank([tr.dense_act.bias], False)
        self.gamma = ParamBank([tr.LayerNorm.weight], False)
        self.beta = ParamBank([tr.LayerNorm.bias], False)
        emb = getattr(mod, "_tied_embeddings", None)
        if emb is not None:
            # one Parameter, one bank: a second bank around the table would re-materialise it
            self.w_dec = emb._native_params().word
            emb._native_params().tie_word_bank()
        else:
            # untied, or the replica of a table on another stage.  A replica is not `tied`: its
            # gradient has one writer on this rank (the decoder wgrads, stream-ordered like any
            # weight bank's), and the exchange of the summed gradient stores over it before the
            # optimizer, so overwrite-first zeroing stays valid for it
            self.w_dec = ParamBank([mod.decoder.weight])
        self.b_dec = ParamBank([mod.decoder.bias], False)
        self.banks = [self.w_t, self.b_t, self.gamma, self.beta, self.w_dec, self.b_dec]
        self.eps = float(tr.LayerNorm.eps)
        self.max_predictions = mod.max_predictions
        self.ignore_index = mod.ignore_index

    def all_params(self):
        return [p for b in self.banks for p in b.params]


class MaskedLMHeadFn(torch.autograd.Function):
    """BertTailForMaskedLM on the wgmma GEMM: dense with bias + GELU in the epilogue (the
    pre-activation kept for backward), LayerNorm, decoder GEMM with bias to bf16 logits.
    Backward: decoder dgrad GEMM, LayerNorm backward, GELU derivative, transform dgrad GEMM;
    the weight / bias / LayerNorm parameter gradients go straight into the fp32 bank gradients
    and follow the same deferral / side-stream policy as the encoder's.

    With ``labels`` (a sparse head, ``hp.max_predictions`` = P) the ``mlm_gather`` kernel first
    compacts the labelled rows into B*P slots, the same chain runs on them and the result is
    ``(logits [B*P, V], slot_labels [B*P])``; backward ends with ``mlm_scatter`` into the
    [B, S, H] input gradient."""

    @staticmethod
    def _run(hp: MaskedLMHeadParams, hidden: torch.Tensor, keep: bool, labels=None):
        B, S, H = hidden.shape
        x = hidden.contiguous().view(B * S, H)
        slots = None
        if labels is not None:
            x, slot_of_row, slot_labels = nat.mlm_gather(
                x, labels, hp.max_predictions, hp.w_dec.master().shape[0], hp.ignore_index)
            slots = (slot_of_row, slot_labels)
        h1 = torch.empty_like(x) if keep else None
        t = nat.gemm(x, hp.w_t.shadow(), bias=hp.b_t.master(), act=nat.ACT_GELU, out2=h1)
        y, mean, rstd = _ln_fwd(t, hp.gamma.master(), hp.beta.master(), hp.eps)
        logits = nat.gemm(y, hp.w_dec.shadow(), bias=hp.b_dec.master())
        if slots is None:
            logits = logits.view(B, S, -1)
        return logits, (x, h1, t, mean, rstd, y), slots

    @staticmethod
    def infer(hp: MaskedLMHeadParams, hidden: torch.Tensor, labels=None):
        """Eval-mode forward without autograd: the same outputs, nothing kept for backward."""
        logits, _, slots = MaskedLMHeadFn._run(hp, hidden, False, labels)
        return logits if slots is None else (logits, slots[1])

    @staticmethod
    def forward(ctx, hp, hidden, labels, *params):
        logits, saved, slots = MaskedLMHeadFn._run(hp, hidden, True, labels)
        ctx.hp, ctx.saved, ctx.shape3 = hp, saved, tuple(hidden.shape)
        ctx.slot_of_row = None if slots is None else slots[0]
        ctx.n_params = len(params)
        if slots is None:
            return logits
        ctx.mark_non_differentiable(slots[1])
        return logits, slots[1]

    @staticmethod
    def backward(ctx, dlogits, *_dslot_labels):
        dx = MaskedLMHeadFn._backward(ctx.hp, ctx.saved, ctx.shape3, ctx.slot_of_row, dlogits)
        ctx.saved = ctx.slot_of_row = None
        return (None, dx, None, *([None] * ctx.n_params))

    @staticmethod
    def _backward(hp, saved, shape3, slot_of_row, dlogits, dcls=None) -> torch.Tensor:
        """The head's chain backward to the [B, S, H] input gradient.  ``dcls`` [B, H] (the
        pooler branch of the pretraining head) is added into the [CLS] rows as the gradient is
        written: in ``mlm_scatter`` for the sparse head, in place after the dgrad GEMM for the
        dense one."""
        x, h1, t, mean, rstd, y = saved
        B, S, H = shape3
        g = _flat2d(dlogits)
        if g.dtype != torch.bfloat16:
            g = g.to(torch.bfloat16)
        g = g.contiguous()
        _wgrad(g, y, hp.w_dec, hp.b_dec)
        dy = nat.gemm(g, hp.w_dec.shadow(), b_mn=True)
        dt, _ = nat.layernorm_bwd(dy, t, mean, rstd, hp.gamma.master(), None, None)
        _ln_pgrad(dy, t, mean, rstd, hp.gamma, hp.beta)
        dh1 = torch.empty_like(dt)
        nat.ext().dgelu_mul(dt.data_ptr(), h1.data_ptr(), dh1.data_ptr(), dt.numel(),
                            torch.cuda.current_stream().cuda_stream)
        _wgrad(dh1, x, hp.w_t, hp.b_t)
        dx = nat.gemm(dh1, hp.w_t.shadow(), b_mn=True)
        if slot_of_row is not None:
            return nat.mlm_scatter(dx, slot_of_row, dcls).view(B, S, H)
        dx = dx.view(B, S, H)
        if dcls is not None:
            nat.cls_grad_add_(dx, dcls)
        return dx


class PreTrainingHeadParams(MaskedLMHeadParams):
    """Banks of ``BertTailForPreTraining``: the masked-LM head's, then the pooler's (the banks of
    its ``BertPooler`` submodule, shared, so every bank exists once) and the next-sentence
    classifier's."""

    def __init__(self, mod):
        super().__init__(mod)
        self.pool = mod.pooler._native_params()
        self.nsp = SmallLinearParams(mod.seq_relationship.weight, mod.seq_relationship.bias,
                                     act_tanh=False, first_token=False)
        self.banks = self.banks + self.pool.banks + self.nsp.banks


class PreTrainingHeadFn(torch.autograd.Function):
    """BertTailForPreTraining as ONE autograd node: the masked-LM chain of ``MaskedLMHeadFn`` and
    the next-sentence branch (the pooler's wgmma GEMM with the tanh epilogue on the strided
    [CLS]-row view, then ``small_linear`` to 2 logits).  Outputs ``(mlm_logits, nsp_logits
    [B, 2])``, or ``(mlm_logits [B*P, V], slot_labels, nsp_logits)`` with labels [B, S + 1].
    Backward writes the input gradient once: the pooler's [B, H] input gradient joins the MLM
    gradient in the [CLS] rows (``MaskedLMHeadFn._backward``)."""

    @staticmethod
    def _run(hp: PreTrainingHeadParams, hidden: torch.Tensor, keep: bool, labels=None):
        mlm_labels = None if labels is None else split_pretraining_labels(labels)[0].contiguous()
        logits, saved, slots = MaskedLMHeadFn._run(hp, hidden, keep, mlm_labels)
        B, S, H = hidden.shape
        x0 = hidden.contiguous().view(B, S * H)[:, :H]
        pooled = nat.gemm(x0, hp.pool.w.shadow(), bias=hp.pool.b.master(), act=nat.ACT_TANH,
                          out_dtype=torch.float32)
        w, b = hp.nsp.w.master(), hp.nsp.b.master()
        nsp = torch.empty((B, w.shape[0]), dtype=torch.float32, device=hidden.device)
        nat.ext().small_linear_fwd(x=pooled.data_ptr(), x_bf16=False, ldx=H, w=w.data_ptr(),
                                   b=b.data_ptr(), y=nsp.data_ptr(), M=B, N=w.shape[0], K=H,
                                   act_tanh=0, dropout_p=0.0, rng_state=0, rng_stream=0,
                                   stream=torch.cuda.current_stream().cuda_stream)
        return logits, saved, slots, (x0, pooled, nsp)

    @staticmethod
    def infer(hp: PreTrainingHeadParams, hidden: torch.Tensor, labels=None):
        logits, _, slots, (_, _, nsp) = PreTrainingHeadFn._run(hp, hidden, False, labels)
        return (logits, nsp) if slots is None else (logits, slots[1], nsp)

    @staticmethod
    def forward(ctx, hp, hidden, labels, *params):
        logits, saved, slots, nsp_saved = PreTrainingHeadFn._run(hp, hidden, True, labels)
        ctx.hp, ctx.saved, ctx.nsp_saved = hp, saved, nsp_saved
        ctx.shape3 = tuple(hidden.shape)
        ctx.slot_of_row = None if slots is None else slots[0]
        ctx.n_params = len(params)
        nsp = nsp_saved[2]
        if slots is None:
            return logits, nsp
        ctx.mark_non_differentiable(slots[1])
        return logits, slots[1], nsp

    @staticmethod
    def backward(ctx, dlogits, *rest):
        hp = ctx.hp
        dnsp = rest[-1]
        x0, pooled, nsp = ctx.nsp_saved
        B, S, H = ctx.shape3
        # next-sentence classifier, then the pooler (bias + tanh derivative as in PoolerFn)
        w = hp.nsp.w.master()
        dpooled = torch.empty_like(pooled)
        nat.ext().small_linear_bwd(x=pooled.data_ptr(), x_bf16=False, ldx=H, w=w.data_ptr(),
                                   y=nsp.data_ptr(), dy=dnsp.contiguous().float().data_ptr(),
                                   dx=dpooled.data_ptr(), dx_bf16=False, lddx=H,
                                   dw=hp.nsp.w.grad().data_ptr(), db=hp.nsp.b.grad().data_ptr(),
                                   M=B, N=w.shape[0], K=H, act_tanh=0, dropout_p=0.0,
                                   rng_state=0, rng_stream=0,
                                   stream=torch.cuda.current_stream().cuda_stream)
        g = dpooled * (1.0 - pooled * pooled)
        hp.pool.b.grad().add_(g.sum(0))
        gb = g.to(torch.bfloat16)
        nat.gemm(gb, x0, a_mn=True, b_mn=True, out=hp.pool.w.grad(), accumulate=True)
        dcls = nat.gemm(gb, hp.pool.w.shadow(), b_mn=True)
        dx = MaskedLMHeadFn._backward(hp, ctx.saved, ctx.shape3, ctx.slot_of_row, dlogits, dcls)
        ctx.saved = ctx.nsp_saved = ctx.slot_of_row = None
        return (None, dx, None, *([None] * ctx.n_params))


def split_span_labels(labels: torch.Tensor):
    """The labels of a question-answering item are ONE int64 tensor ``[..., 5]``: the gold
    answer's first and last token positions ``start`` and ``end``, the positions ``start_lo`` ..
    ``start_hi`` where a predicted answer may start, and ``end_hi``, the last position where it
    may end.  Returns ``(start, end, start_lo, start_hi, end_hi)`` as views.  A padded evaluation
    row is ``ignore_index`` in every column.  One tensor keeps the engine's chunking, label
    buffers, label routing and evaluation padding unchanged; this function and
    ``span_answer_labels`` are the only places that know the layout."""
    return labels[..., 0], labels[..., 1], labels[..., 2], labels[..., 3], labels[..., 4]


def span_answer_labels(labels: torch.Tensor) -> torch.Tensor:
    """``(start, end)`` of ``split_span_labels``' layout as one ``[B, 2]`` view of ``labels``
    (``[B, 5]`` or flat): the labels of the span loss's start and end logit rows."""
    return labels.reshape(-1, 5)[:, :2]


class QuestionAnsweringParams:
    """Parameter banks of ``BertTailForQuestionAnswering``: ``qa_outputs`` (fp32 weight [2, H] and
    bias [2], read by the kernels as they are, so no bf16 shadow)."""

    def __init__(self, mod):
        self.w = ParamBank([mod.qa_outputs.weight], False)
        self.b = ParamBank([mod.qa_outputs.bias], False)
        self.banks = [self.w, self.b]

    def all_params(self):
        return [p for b in self.banks for p in b.params]


class QuestionAnsweringFn(torch.autograd.Function):
    """BertTailForQuestionAnswering on sm_90a: ``qa_logits_fwd`` reads the bf16 hidden states once
    and writes fp32 logits [B, 2, S]; backward (``qa_logits_bwd``) writes the bf16 input gradient
    in one pass over the rows and adds dW / db into the fp32 bank gradients in a fixed order."""

    @staticmethod
    def infer(hp: QuestionAnsweringParams, hidden: torch.Tensor) -> torch.Tensor:
        """Eval-mode forward without autograd: the same logits, nothing kept for backward."""
        return nat.qa_logits(hidden.contiguous(), hp.w.master(), hp.b.master())

    @staticmethod
    def forward(ctx, hp, hidden, *params):
        hidden = hidden.contiguous()
        ctx.hp, ctx.hidden = hp, hidden
        ctx.n_params = len(params)
        return nat.qa_logits(hidden, hp.w.master(), hp.b.master())

    @staticmethod
    def backward(ctx, dlogits):
        hp = ctx.hp
        dx = nat.qa_logits_bwd(ctx.hidden, dlogits, hp.w.master(), hp.w.grad(), hp.b.grad())
        ctx.hidden = None
        return (None, dx, *([None] * ctx.n_params))


class SoftmaxCrossEntropyFn(torch.autograd.Function):
    """``nat.softmax_ce`` as an autograd node: the classification loss on [M, C] logits, and the
    span loss (``runner.QuestionAnsweringLoss``) on [B, 2, S] logits with [B, 2] labels
    (``span_answer_labels``)."""

    @staticmethod
    def forward(ctx, logits, labels, ignore_index: int):
        loss, dlogits = nat.softmax_ce(logits.float().contiguous(), labels,
                                       ignore_index=ignore_index)
        ctx.save_for_backward(dlogits)
        return loss.reshape(())

    @staticmethod
    def backward(ctx, dloss):
        (dlogits,) = ctx.saved_tensors
        return dlogits * dloss, None, None
