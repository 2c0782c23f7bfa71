"""One torch.autograd.Function per operator of the training step (SURVEY.md section 8 row a13; reference train.py:255-281 SDModel.forward
under autograd, :573-605 loss + backward). torch autograd only ORDERS the backward pass and accumulates fan-out gradients;
every forward and backward computation below is a kernel of libimagd_b200.so:

  Linear      y = x W^T + b (+ residual)        dX = dY W            (wgmma GEMM on W^T)
                                                dW = dY^T X          (wgmma GEMM on the two transposed operands, K = tokens)
                                                db = column sum of dY
  Conv3x3     implicit-GEMM conv                dX = conv3x3(dY, flipped / transposed taps)    (the same wgmma conv kernel)
                                                dW = dY^T im2col(X)^T (wgmma GEMM), db / d(time-embedding row) = column sums
  Attention   two-stream flash forward          dQ / dK / dV / dK_ref / dV_ref: attention_bwd.cu (recompute-S)
  GroupNorm(+SiLU), LayerNorm, SiLU / GELU, GEGLU, nearest-2x upsample, stride-2 im2col, channel concat, MSE: train_ops.cu

Activations are bf16 token-major exactly as on the inference path; gradients are bf16 (fp32 accumulation inside every kernel),
the reference's bf16 mixed-precision regime (train.py:455-465). Gradients with respect to parameters come back in the
parameter's dtype.
"""
from __future__ import annotations

from typing import Optional

import torch
from torch.autograd import Function

from . import ops
from ._lib import ACT_GELU, ACT_SILU

BF16 = torch.bfloat16

_frozen_cache = {}


def _cached(kind: str, w: torch.Tensor, frozen: bool, build):
    """Derived operands of FROZEN weights (the denoising UNet: transposed / flipped copies for dgrad, fp32 biases) are built
    once. Keyed by address + in-place version; every entry also HOLDS the source's storage, so the address cannot be recycled
    for another tensor while the entry lives (saved tensors reach backward() as new Python objects, identity is no key).
    clear_cache() drops everything (models deleted, checkpoints loaded)."""
    if not frozen:
        return build()
    key = (kind, w.data_ptr(), w._version, tuple(w.shape), tuple(w.stride()))
    hit = _frozen_cache.get(key)
    if hit is None:
        hit = _frozen_cache[key] = (build(), w.untyped_storage())
    return hit[0]


def clear_cache():
    _frozen_cache.clear()


def _bf(t: torch.Tensor) -> torch.Tensor:
    return t if t.dtype == BF16 else t.to(BF16)


def _f32c(t: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
    """fp32 contiguous copy of a bias / norm parameter for the kernels' fp32 arguments: itself, a cached conversion (frozen
    parameters), or a conversion. (The optimizer's fp32 master weights are deliberately NOT used here: the model the
    reference trains in bf16 mode sees the bf16-rounded bias, and so does every path of this repo.)"""
    if t is None:
        return None
    if t.dtype == torch.float32 and t.is_contiguous():
        return t.detach()
    if not t.requires_grad:
        return _cached("f32", t, True, lambda: t.detach().float().contiguous())
    return t.detach().float().contiguous()


def _gdt(p: Optional[torch.Tensor]):
    """dtype in which a bias / affine gradient is produced: the parameter's own when it is bf16 (no conversion launch)."""
    return BF16 if p is not None and p.dtype == BF16 else torch.float32


def _as(t: Optional[torch.Tensor], like: torch.Tensor) -> Optional[torch.Tensor]:
    return None if t is None else t.to(like.dtype).reshape(like.shape)


class Linear(Function):
    """y[..., N] = x[..., K] @ w[N, K]^T + bias (+ residual).  x: bf16, contiguous or a 2-D row-strided view."""

    @staticmethod
    def forward(ctx, x, w, bias, residual, out_fp32):
        y = ops.gemm(x, w, bias=_f32c(bias), residual=residual, out_fp32=bool(out_fp32))
        ctx.save_for_backward(x, w)
        ctx.bias = bias
        ctx.res = residual
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w = ctx.saved_tensors
        N, K = w.shape
        need_x, need_w, need_b, need_r = ctx.needs_input_grad[:4]
        dy2 = _bf(dy).reshape(-1, N).contiguous()
        dx = dw = db = dr = None
        if need_x:
            wt = _cached("wt", w, not need_w, lambda: ops.transpose(w))  # [K, N]
            dx = ops.gemm(dy2, wt[:, :N] if wt.shape[1] != N else wt).view(x.shape)
        if need_w:
            x2 = x if x.dim() == 2 else x.reshape(-1, K)
            dw = ops.gemm(ops.transpose(dy2), ops.transpose(x2))  # [N, K], reduction over the (zero-padded) tokens
        if need_b and ctx.bias is not None:
            db = _as(ops.colsum(dy2, None, _gdt(ctx.bias))[0], ctx.bias)
        if need_r and ctx.res is not None:
            dr = dy2.view(ctx.res.shape)
        return dx, dw, db, dr, None


def linear(x, w, bias=None, residual=None, out_fp32=False):
    return Linear.apply(x, _bf(w), bias, residual, out_fp32)


class PackConv(Function):
    """[Cout, Cin, 3, 3] -> tap-major [Cout, 9*Cin] (and the packed gradient back), one layout kernel each way."""

    @staticmethod
    def forward(ctx, w):
        return ops.conv_weight_layout(w.contiguous(), 0)

    @staticmethod
    def backward(ctx, dwp):
        return ops.conv_weight_layout(_bf(dwp).contiguous(), 1)


def pack_conv3x3(w: torch.Tensor) -> torch.Tensor:
    """[Cout, Cin, 3, 3] -> tap-major [Cout, 9*Cin] bf16, differentiable."""
    if 9 * w.shape[1] * 2 > 48 * 1024:  # (no such layer in SD1.5: Cin <= 2560)
        co, ci = w.shape[:2]
        return _bf(w).permute(0, 2, 3, 1).reshape(co, 9 * ci).contiguous()
    return PackConv.apply(_bf(w))


def _flip_taps(wp: torch.Tensor, cin: int) -> torch.Tensor:
    """Packed forward weight [Cout, 9*Cin] -> the dgrad weight [Cin, 9*Cout]: W'[ci, 8 - tap, co] = W[co, tap, ci]."""
    return ops.conv_weight_flip(wp.contiguous(), cin)


class Conv3x3(Function):
    """ResnetBlock2D.conv1 / conv2, Upsample2D.conv: y = conv3x3(x) + bias + rowvec[sample] (+ residual)."""

    @staticmethod
    def forward(ctx, x, wp, bias, rowvec, residual):
        y = ops.conv3x3(x, wp, bias=_f32c(bias), rowvec=rowvec, residual=residual)
        ctx.save_for_backward(x, wp)
        ctx.bias, ctx.has_rowvec, ctx.res = bias, rowvec is not None, residual
        return y

    @staticmethod
    def backward(ctx, dy):
        x, wp = ctx.saved_tensors
        NB, H, W, Cin = x.shape
        Cout = wp.shape[0]
        need_x, need_w, need_b, need_v, need_r = ctx.needs_input_grad
        dy = _bf(dy).contiguous()
        dy2 = dy.view(NB * H * W, Cout)
        dx = dw = db = dv = dr = None
        if need_x:
            wf = _cached("flip", wp, not need_w, lambda: _flip_taps(wp.detach(), Cin))
            dx = ops.conv3x3(dy, wf)
        if need_w:
            dw = ops.gemm(ops.transpose(dy2), ops.im2col3x3_t(x))[:, :9 * Cin]
        if need_b and ctx.bias is not None:
            db = _as(ops.colsum(dy2, None, _gdt(ctx.bias))[0], ctx.bias)
        if need_v and ctx.has_rowvec:
            dv = ops.colsum(dy2, H * W)  # fp32 [NB, Cout]
        if need_r and ctx.res is not None:
            dr = dy
        return dx, dw, db, dv, dr


def conv3x3(x, wp, bias=None, rowvec=None, residual=None):
    return Conv3x3.apply(x, wp, bias, rowvec, residual)


class ConvIn(Function):
    """conv_in (4 -> 320, direct SIMT kernel forward). The input latents carry no gradient; dW via the transposed-im2col
    GEMM (9*4 = 36 weight columns, padded to 40 for the tensor core), db = column sum."""

    @staticmethod
    def forward(ctx, x, wp, bias):
        y = ops.conv3x3_direct(x, wp, _f32c(bias))
        ctx.save_for_backward(x, wp)
        ctx.bias = bias
        return y

    @staticmethod
    def backward(ctx, dy):
        x, wp = ctx.saved_tensors
        NB, H, W, Cin = x.shape
        Cout = wp.shape[0]
        if ctx.needs_input_grad[0]:
            raise NotImplementedError("conv_in: the latents are data, not a trainable tensor")
        dy2 = _bf(dy).contiguous().view(NB * H * W, Cout)
        dw = db = None
        if ctx.needs_input_grad[1]:
            dw = ops.gemm(ops.transpose(dy2), ops.im2col3x3_t(x))[:, :9 * Cin].contiguous()
        if ctx.needs_input_grad[2] and ctx.bias is not None:
            db = _as(ops.colsum(dy2, None, _gdt(ctx.bias))[0], ctx.bias)
        return None, dw, db


class ConvOut(Function):
    """conv_out (320 -> 4, fp32 NCHW eps). dX = the direct 4 -> 320 conv of dY with flipped taps. Weight gradients are not
    needed anywhere in the reference's training set-up (the denoising UNet is frozen, the garment UNet's output is discarded)."""

    @staticmethod
    def forward(ctx, x, wp, bias):
        y = ops.conv3x3_direct(x, wp, _f32c(bias), out_nchw_f32=True)
        ctx.save_for_backward(wp)
        ctx.cin = x.shape[-1]
        return y

    @staticmethod
    def backward(ctx, dy):
        (wp,) = ctx.saved_tensors
        if ctx.needs_input_grad[1] or ctx.needs_input_grad[2]:
            raise NotImplementedError("conv_out weight gradients: train.py freezes the denoising UNet")
        wf = _cached("flip_out", wp, True, lambda: _flip_taps(wp.detach(), ctx.cin))  # [320, 9*4]
        dy_t = ops.nchw_f32_to_nhwc_bf16(dy.float().contiguous())
        return ops.conv3x3_direct(dy_t, wf, None), None, None


class GroupNorm(Function):
    @staticmethod
    def forward(ctx, x, gamma, beta, groups, eps, silu):
        g32, b32 = _f32c(gamma), _f32c(beta)
        stats = torch.empty(x.shape[0], int(groups), 2, device=x.device, dtype=torch.float32)
        y = ops.groupnorm(x, g32, b32, groups, eps, silu=bool(silu), stats_out=stats)
        ctx.save_for_backward(x, g32, b32, stats)
        ctx.cfg = (int(groups), bool(silu), gamma, beta)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, g32, b32, stats = ctx.saved_tensors
        groups, silu, gamma, beta = ctx.cfg
        need_aff = ctx.needs_input_grad[1] or ctx.needs_input_grad[2]
        dx, dg, db = ops.groupnorm_bwd(x, _bf(dy).contiguous(), g32, b32, groups, stats, silu, need_aff, _gdt(gamma))
        return (dx if ctx.needs_input_grad[0] else None, _as(dg, gamma) if ctx.needs_input_grad[1] else None,
                _as(db, beta) if ctx.needs_input_grad[2] else None, None, None, None)


def groupnorm(x, norm: torch.nn.GroupNorm, silu: bool):
    return GroupNorm.apply(x, norm.weight, norm.bias, norm.num_groups, norm.eps, silu)


class LayerNorm(Function):
    @staticmethod
    def forward(ctx, x, gamma, beta, eps):
        g32, b32 = _f32c(gamma), _f32c(beta)
        y = ops.layernorm(x, g32, b32, eps)
        ctx.save_for_backward(x, g32)
        ctx.cfg = (float(eps), gamma, beta)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, g32 = ctx.saved_tensors
        eps, gamma, beta = ctx.cfg
        need_aff = ctx.needs_input_grad[1] or ctx.needs_input_grad[2]
        dx, dg, db = ops.layernorm_bwd(x, _bf(dy).contiguous(), g32, eps, need_aff, _gdt(gamma))
        return (dx if ctx.needs_input_grad[0] else None, _as(dg, gamma) if ctx.needs_input_grad[1] else None,
                _as(db, beta) if ctx.needs_input_grad[2] else None, None)


def layernorm(x, norm: torch.nn.LayerNorm):
    return LayerNorm.apply(x.contiguous(), norm.weight, norm.bias, norm.eps)


class Act(Function):
    @staticmethod
    def forward(ctx, x, mode):
        x = x.contiguous()
        ctx.save_for_backward(x)
        ctx.mode = int(mode)
        return ops.act(x, ctx.mode)

    @staticmethod
    def backward(ctx, dy):
        (x,) = ctx.saved_tensors
        return ops.act(x, ctx.mode, _bf(dy).contiguous()), None


def silu(x):
    return Act.apply(x, ACT_SILU)


def gelu(x):
    return Act.apply(x, ACT_GELU)


class Geglu(Function):
    """[..., 2F] = [value | gate] -> value * gelu(gate)  (diffusers-0.24 GEGLU, BasicTransformerBlock.ff)."""

    @staticmethod
    def forward(ctx, h):
        h = h.contiguous()
        ctx.save_for_backward(h)
        return ops.geglu(h)

    @staticmethod
    def backward(ctx, dy):
        (h,) = ctx.saved_tensors
        return ops.geglu(h, _bf(dy).contiguous())


class Upsample2x(Function):
    @staticmethod
    def forward(ctx, x):
        return ops.upsample2x(x)

    @staticmethod
    def backward(ctx, dy):
        return ops.downsum2x(_bf(dy).contiguous())


class Im2colS2(Function):
    """Stride-2 pad-1 3x3 patches (Downsample2D = this + Linear); adjoint = col2im gather."""

    @staticmethod
    def forward(ctx, x):
        ctx.hw = (x.shape[1], x.shape[2])
        return ops.im2col3x3_s2(x)

    @staticmethod
    def backward(ctx, dcol):
        return ops.col2im3x3_s2(_bf(dcol).contiguous(), *ctx.hw)


class Concat(Function):
    """torch.cat([a, b], -1) of token-major tensors (the up-block skip concat)."""

    @staticmethod
    def forward(ctx, a, b):
        ctx.ca = a.shape[-1]
        ctx.shapes = (a.shape, b.shape)
        return ops.concat_add(a, b)

    @staticmethod
    def backward(ctx, dy):
        dy = _bf(dy).contiguous()
        C = dy.shape[-1]
        d2 = dy.view(-1, C)
        da = ops.concat_add(d2[:, :ctx.ca], None).view(ctx.shapes[0]) if ctx.needs_input_grad[0] else None
        db = ops.concat_add(d2[:, ctx.ca:], None).view(ctx.shapes[1]) if ctx.needs_input_grad[1] else None
        return da, db


class Attention(Function):
    """Two-stream attention over the projection outputs.

    q_src:  fused [B, L, 3C] (q | k | v of self-attention; kv0 is None then) or q [B, L, C]
    kv0:    [B, L0, 2C] fused k | v of stream 0 (cross-attention context projection) or None
    kv1:    [B, L1, 2C] fused k | v of the second (garment) stream or None;  w1 = its out_scale
    len0:   visited keys of stream 0 (a prefix of kv0's tokens; None = all)."""

    @staticmethod
    def forward(ctx, q_src, kv0, kv1, heads, w1, len0):
        B, L = q_src.shape[:2]
        fused = kv0 is None
        C = q_src.shape[-1] // 3 if fused else q_src.shape[-1]
        hd = C // heads
        q2, s0, s1 = Attention._streams(q_src, kv0, kv1, C, w1, len0)
        out, saved = ops.attention_train(q2, B, L, heads, hd, s0, s1)
        ctx.save_for_backward(q_src, kv0, kv1)
        ctx.saved, ctx.cfg = saved, (heads, float(w1), len0)
        return out.view(B, L, C)

    @staticmethod
    def _streams(q_src, kv0, kv1, C, w1, len0):
        B, L = q_src.shape[:2]
        flat = q_src.view(B * L, q_src.shape[-1])
        if kv0 is None:
            q2 = flat[:, :C]
            s0 = ops.kv_stream(flat[:, C:2 * C], flat[:, 2 * C:], L)
        else:
            q2 = flat
            f0 = kv0.view(-1, 2 * C)
            n0 = kv0.shape[1] if len0 is None else int(len0)
            s0 = ops.kv_stream(f0[:, :C], f0[:, C:], n0, sample_rows=kv0.shape[1] if n0 != kv0.shape[1] else 0)
        s1 = None
        if kv1 is not None:
            f1 = kv1.view(-1, 2 * C)
            s1 = ops.kv_stream(f1[:, :C], f1[:, C:], kv1.shape[1], out_scale=w1)
        return q2, s0, s1

    @staticmethod
    def backward(ctx, d_out):
        q_src, kv0, kv1 = ctx.saved_tensors
        heads, w1, len0 = ctx.cfg
        B, L = q_src.shape[:2]
        fused = kv0 is None
        C = q_src.shape[-1] // 3 if fused else q_src.shape[-1]
        hd = C // heads
        q2, s0, s1 = Attention._streams(q_src, kv0, kv1, C, w1, len0)
        d2 = _bf(d_out).contiguous().view(B * L, C)
        need_q, need_kv0, need_kv1 = ctx.needs_input_grad[:3]
        dq_src = dkv0 = dkv1 = None
        dq = pair0 = pair1 = None
        if fused:
            if need_q:
                dq_src = torch.empty_like(q_src)
                f = dq_src.view(B * L, 3 * C)
                dq, pair0 = f[:, :C], (f[:, C:2 * C], f[:, 2 * C:])
        else:
            if need_q:
                dq_src = torch.empty_like(q_src)
                dq = dq_src.view(B * L, C)
            if need_kv0:
                dkv0 = torch.zeros_like(kv0)  # tokens outside the visited window get no gradient
                f = dkv0.view(-1, 2 * C)
                pair0 = (f[:, :C], f[:, C:])
        if kv1 is not None and need_kv1:
            dkv1 = torch.empty_like(kv1)
            f = dkv1.view(-1, 2 * C)
            pair1 = (f[:, :C], f[:, C:])
        ops.attention_bwd(q2, d2, B, L, heads, hd, s0, s1, ctx.saved, dq=dq, dkv0=pair0, dkv1=pair1)
        return dq_src, dkv0, dkv1, None, None, None


def attention(q_src, kv0, kv1, heads: int, w1: float = 1.0, len0: Optional[int] = None):
    return Attention.apply(q_src, kv0, kv1, heads, w1, len0)


class MseLoss(Function):
    """mean((pred - target)^2) over fp32 tensors (train.py:577); the gradient is produced in the same pass."""

    @staticmethod
    def forward(ctx, pred, target):
        loss, grad = ops.mse_loss_grad(pred.float().contiguous(), target.float().contiguous())
        ctx.save_for_backward(grad)
        ctx.dtype = pred.dtype
        return loss[0]

    @staticmethod
    def backward(ctx, dl):
        (grad,) = ctx.saved_tensors
        return (grad * dl).to(ctx.dtype), None


def mse_loss(pred, target):
    return MseLoss.apply(pred, target)
