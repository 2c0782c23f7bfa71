"""Tensor-level wrappers over the C ABI: torch owns device memory and the stream, the kernels do the arithmetic.

Every function takes CUDA tensors, passes raw pointers / strides / the current stream to libimagd_b200.so and
returns the output tensor. Nothing here computes on the CPU and nothing falls back to torch ops.
"""
from __future__ import annotations

import ctypes
from typing import Optional, Tuple

import torch

from . import _lib
from ._lib import ACT_GEGLU, ACT_GELU, ACT_NONE, ACT_QUICK_GELU, ACT_RELU, ACT_SILU, Epilogue, KVStream

BF16 = torch.bfloat16


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _rows2d(t: torch.Tensor) -> Tuple[int, int, int]:
    """(rows, cols, ld) of a token-major view whose last dim is contiguous."""
    assert t.stride(-1) == 1, "last dim must be contiguous"
    if t.dim() == 2:
        return t.shape[0], t.shape[1], t.stride(0)
    assert t.is_contiguous() or t.dim() == 2, "higher-rank activations must be contiguous"
    rows = 1
    for s in t.shape[:-1]:
        rows *= s
    return rows, t.shape[-1], t.shape[-1]


def _pixel_ld(t: torch.Tensor) -> int:
    """Pixel (row) stride of a channel-last [NB, H, W, C] view whose pixels are equally spaced: a contiguous tensor or a
    channel slice of a wider NHWC buffer (e.g. the concat buffer of an up block)."""
    assert t.dim() == 4 and t.stride(-1) == 1, "channel-last [NB, H, W, C] view with contiguous channels"
    NB, H, W, C = t.shape
    ld = t.stride(-2)
    for size, stride, want in ((W, ld, ld), (H, t.stride(-3), W * ld), (NB, t.stride(-4), H * W * ld)):
        assert size == 1 or stride == want, f"pixels of a {tuple(t.shape)} view with strides {t.stride()} are not equally spaced"
    assert ld >= C
    return ld


def _conv_epilogue(bias, rowvec, residual, act, NB: int, out: torch.Tensor) -> Epilogue:
    """Epilogue of a conv launch writing `out` [NB, H, W, Cout]: rowvec [>= NB, >= Cout] fp32 (one row per sample),
    residual a channel-last view of the output's shape."""
    _, H, W, Cout = out.shape
    if rowvec is not None:
        assert rowvec.dim() == 2 and rowvec.dtype == torch.float32 and rowvec.stride(1) == 1
        assert rowvec.shape[0] >= NB and rowvec.shape[1] >= Cout, f"rowvec {tuple(rowvec.shape)} for {NB} x {Cout}"
    ep = _epilogue(bias, rowvec, H * W, None, act, 1.0, False)
    if residual is not None:
        assert residual.shape == out.shape and residual.dtype == BF16, f"residual {tuple(residual.shape)} vs {tuple(out.shape)}"
        ep.residual = residual.data_ptr()
        ep.ldr = _pixel_ld(residual)
    return ep


class LnFold:
    """LayerNorm folded into the consuming GEMM (include/imagd_b200.h, DESIGN.md section 8): `stats` [M, ld, 2] fp32
    holds the producer's per-row {sum, sum of squares} partials (`parts` of them), `colsum` [N] the column sums of the
    gamma-scaled weight; the GEMM's `bias` must be the folded bias b + W beta."""

    __slots__ = ("stats", "parts", "dim", "eps", "colsum")

    def __init__(self, stats: torch.Tensor, parts: int, dim: int, eps: float, colsum: torch.Tensor):
        self.stats, self.parts, self.dim, self.eps, self.colsum = stats, int(parts), int(dim), float(eps), colsum


def gemm_tile_count_n(M: int, N: int, K: int) -> int:
    """How many row-statistics partials a producer GEMM of this shape writes per row."""
    n = _lib.load().imagd_gemm_tile_count_n(int(M), int(N), int(K))
    if n <= 0:
        _lib.check(n if n < 0 else -1, "imagd_gemm_tile_count_n")
    return n


def _epilogue(bias, rowvec, rows_per_group, residual, act, alpha, out_fp32) -> Epilogue:
    ep = Epilogue()
    ep.bias = _ptr(bias)
    ep.rowvec = _ptr(rowvec)
    ep.rowvec_ld = rowvec.stride(0) if rowvec is not None else 0
    ep.rows_per_group = int(rows_per_group)
    ep.act = int(act)
    ep.residual = _ptr(residual)
    ep.ldr = _rows2d(residual)[2] if residual is not None else 0
    ep.alpha = float(alpha)
    ep.out_fp32 = 1 if out_fp32 else 0
    return ep


def gemm(a: torch.Tensor, w: torch.Tensor, *, out: Optional[torch.Tensor] = None, bias=None, rowvec=None,
         rows_per_group: int = 0, residual=None, act: int = ACT_NONE, alpha: float = 1.0,
         out_fp32: bool = False, stats_out: Optional[torch.Tensor] = None, ln: Optional[LnFold] = None,
         scale_table: Optional[torch.Tensor] = None, scale_step: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out[M, N] = epilogue(a[M, K] @ w[N, K]^T); a / w / residual bf16, bias / rowvec fp32.
    stats_out [M, ld, 2] fp32: also emit per-row {sum, sum of squares} of the rounded outputs, one slot per N tile.
    ln: the rows of `a` are the RAW input of a LayerNorm that has been folded into `w` / `bias` (LnFold).
    scale_table: fp32 device column view [S, K][:, k] (or a 1-D [S] table); the kernel reads s = scale_table[scale_step[0]]
    (row 0 without scale_step, an int32 device tensor) and computes s * acc + s * bias + residual in place of alpha."""
    if scale_table is not None:  # the kernel sees only a pointer: dtype, rank and device are checked here
        if scale_table.dtype != torch.float32 or scale_table.dim() != 1 or not scale_table.is_cuda:
            raise ValueError(f"scale_table must be a 1-D fp32 CUDA tensor (a column view [S, K][:, k]), got "
                             f"{scale_table.dtype} {tuple(scale_table.shape)} on {scale_table.device}")
        if scale_step is not None and (scale_step.dtype != torch.int32 or not scale_step.is_cuda):
            raise ValueError(f"scale_step must be an int32 CUDA tensor, got {scale_step.dtype} on {scale_step.device}")
    lib = _lib.load()
    M, K, lda = _rows2d(a)
    N, Kw = w.shape
    assert Kw == K and a.dtype == BF16 and w.dtype == BF16
    n_out = N // 2 if act == ACT_GEGLU else N
    if out is None:
        out = torch.empty(*a.shape[:-1], n_out, device=a.device, dtype=torch.float32 if out_fp32 else BF16)
    ldd = _rows2d(out)[2]
    ep = _epilogue(bias, rowvec, rows_per_group, residual, act, alpha, out_fp32)
    if stats_out is not None:
        assert stats_out.dtype == torch.float32 and stats_out.dim() == 3 and stats_out.shape[0] == M and \
            stats_out.shape[2] == 2 and stats_out.is_contiguous()
        ep.row_stats_out = stats_out.data_ptr()
        ep.stats_ld = stats_out.shape[1]
    if ln is not None:
        assert ln.stats.dtype == torch.float32 and ln.stats.shape[0] == M and ln.stats.is_contiguous() and ln.dim == K
        assert ln.colsum.dtype == torch.float32 and ln.colsum.numel() == N and bias is not None
        ep.row_stats_in = ln.stats.data_ptr()
        ep.stats_in_ld = ln.stats.shape[1]
        ep.stats_parts = ln.parts
        ep.ln_dim = ln.dim
        ep.ln_eps = ln.eps
        ep.colsum = ln.colsum.data_ptr()
    if scale_table is not None:
        ep.scale_table = scale_table.data_ptr()
        ep.scale_step = _ptr(scale_step)
        ep.scale_ld = scale_table.stride(0)
    rc = lib.imagd_gemm_bf16(a.data_ptr(), lda, w.data_ptr(), w.stride(0), out.data_ptr(), ldd, M, N, K,
                             ctypes.byref(ep), _stream())
    _lib.check(rc, "imagd_gemm_bf16")
    return out


def conv3x3(x: torch.Tensor, w: torch.Tensor, *, out: Optional[torch.Tensor] = None, bias=None, rowvec=None,
            residual=None, act: int = ACT_NONE) -> torch.Tensor:
    """x: [NB, H, W, Cin] bf16 (token-major), w: [Cout, 9*Cin] tap-major. Stride 1, zero pad 1. x, out and residual may
    be channel slices of wider NHWC buffers (equally spaced pixels); rowvec [>= NB, >= Cout] fp32 is added per sample."""
    lib = _lib.load()
    NB, H, W, Cin = x.shape
    assert x.dtype == BF16 and w.dtype == BF16
    Cout = w.shape[0]
    assert w.shape[1] == 9 * Cin and w.is_contiguous()
    if out is None:
        out = torch.empty(NB, H, W, Cout, device=x.device, dtype=BF16)
    assert out.shape == (NB, H, W, Cout) and out.dtype == BF16
    ep = _conv_epilogue(bias, rowvec, residual, act, NB, out)
    rc = lib.imagd_conv3x3_bf16(x.data_ptr(), _pixel_ld(x), NB, H, W, Cin, w.data_ptr(), out.data_ptr(), _pixel_ld(out), Cout,
                                ctypes.byref(ep), _stream())
    _lib.check(rc, "imagd_conv3x3_bf16")
    return out


def upconv3x3(x: torch.Tensor, w_phase: torch.Tensor, *, bias=None, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Upsample2D (nearest 2x) + 3x3 conv as four 2x2 phase convs on the low-resolution input (modeling.pack_upconv3x3).
    x: [NB, H, W, Cin] bf16, w_phase: [4*Cout, 4*Cin] bf16 -> [NB, 2H, 2W, Cout]; x and out may be channel slices of wider
    NHWC buffers."""
    lib = _lib.load()
    NB, H, W, Cin = x.shape
    assert x.dtype == BF16 and w_phase.dtype == BF16 and w_phase.shape[1] == 4 * Cin and w_phase.is_contiguous()
    Cout = w_phase.shape[0] // 4
    if out is None:
        out = torch.empty(NB, 2 * H, 2 * W, Cout, device=x.device, dtype=BF16)
    assert out.shape == (NB, 2 * H, 2 * W, Cout) and out.dtype == BF16
    ep = _epilogue(bias, None, 0, None, ACT_NONE, 1.0, False)
    rc = lib.imagd_upconv3x3_bf16(x.data_ptr(), _pixel_ld(x), NB, H, W, Cin, w_phase.data_ptr(), out.data_ptr(), _pixel_ld(out),
                                  Cout, ctypes.byref(ep), _stream())
    _lib.check(rc, "imagd_upconv3x3_bf16")
    return out


def kv_stream(k: torch.Tensor, v: torch.Tensor, length: int, *, sample_rows: int = 0, broadcast: bool = False,
              n_query_samples: int = 1 << 30, out_scale: float = 1.0) -> KVStream:
    """k / v: 2-D views [rows, C] whose row 0 is the first visited key of sample 0; `sample_rows` = rows between
    samples when that differs from `length` (a window of a longer context)."""
    s = KVStream()
    s.sample_rows = int(sample_rows)
    assert k.stride(-1) == 1 and v.stride(-1) == 1 and k.dtype == BF16 and v.dtype == BF16
    ld = k.stride(-2)
    assert v.stride(-2) == ld
    s.k, s.v, s.ld, s.len = k.data_ptr(), v.data_ptr(), ld, int(length)
    s.broadcast = 1 if broadcast else 0
    s.n_query_samples = int(min(n_query_samples, 1 << 30))
    s.out_scale = float(out_scale)
    return s


def attention(q: torch.Tensor, B: int, Lq: int, heads: int, head_dim: int, s0: KVStream,
              s1: Optional[KVStream] = None, *, sm_scale: Optional[float] = None,
              out: Optional[torch.Tensor] = None, causal: bool = False) -> torch.Tensor:
    """q: [B*Lq, >= heads*head_dim] bf16 view (row stride arbitrary). Returns [B*Lq, heads*head_dim] bf16.
    causal: query i attends to keys 0..i of stream 0 (CLIP text encoder); no second stream then."""
    lib = _lib.load()
    assert q.dtype == BF16 and q.stride(-1) == 1
    q_ld = q.stride(-2)
    if out is None:
        out = torch.empty(B * Lq, heads * head_dim, device=q.device, dtype=BF16)
    if sm_scale is None:
        sm_scale = head_dim ** -0.5
    if causal:
        assert s1 is None
        rc = lib.imagd_attention_causal_bf16(q.data_ptr(), q_ld, out.data_ptr(), out.stride(-2), B, Lq, heads, head_dim,
                                             ctypes.byref(s0), float(sm_scale), _stream())
        _lib.check(rc, "imagd_attention_causal_bf16")
        return out
    rc = lib.imagd_attention_bf16(q.data_ptr(), q_ld, out.data_ptr(), out.stride(-2), B, Lq, heads, head_dim,
                                  ctypes.byref(s0), ctypes.byref(s1) if s1 is not None else None, float(sm_scale),
                                  _stream())
    _lib.check(rc, "imagd_attention_bf16")
    return out


_gn_ws = {}


def _gn_workspace(device, nbytes: int) -> torch.Tensor:
    ws = _gn_ws.get(device)
    if ws is None or ws.numel() < nbytes:
        ws = torch.zeros(max(nbytes, 1 << 20), device=device, dtype=torch.uint8)  # counters must start at 0
        _gn_ws[device] = ws
    return ws


def groupnorm(x: torch.Tensor, gamma, beta, groups: int, eps: float, *, silu: bool, out: Optional[torch.Tensor] = None,
              ws: Optional[torch.Tensor] = None, stats_out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """x: [NB, HW..., C] bf16 token-major (contiguous). GroupNorm over (HW, C/groups) per sample, optional SiLU.
    stats_out: fp32 [NB, groups, 2] that receives {mean, rstd} (training-mode forward)."""
    lib = _lib.load()
    assert x.is_contiguous() and x.dtype == BF16
    NB, C = x.shape[0], x.shape[-1]
    HW = x.numel() // (NB * C)
    if out is None:
        out = torch.empty_like(x)
    if ws is None:
        ws = _gn_workspace(x.device, lib.imagd_groupnorm_ws_bytes(NB, HW, C, groups))
    if stats_out is not None:
        assert stats_out.dtype == torch.float32 and stats_out.is_contiguous() and stats_out.numel() == NB * groups * 2
        rc = lib.imagd_groupnorm_stats_bf16(x.data_ptr(), C, out.data_ptr(), C, NB, HW, C, groups, _ptr(gamma), _ptr(beta),
                                            float(eps), 1 if silu else 0, ws.data_ptr(), stats_out.data_ptr(), _stream())
        _lib.check(rc, "imagd_groupnorm_stats_bf16")
        return out
    rc = lib.imagd_groupnorm_bf16(x.data_ptr(), C, out.data_ptr(), C, NB, HW, C, groups, _ptr(gamma), _ptr(beta),
                                  float(eps), 1 if silu else 0, ws.data_ptr(), _stream())
    _lib.check(rc, "imagd_groupnorm_bf16")
    return out


def layernorm(x: torch.Tensor, gamma, beta, eps: float = 1e-5, *, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    lib = _lib.load()
    rows, C, ldx = _rows2d(x)
    assert x.dtype == BF16
    if out is None:
        out = torch.empty(*x.shape, device=x.device, dtype=BF16)
    rc = lib.imagd_layernorm_bf16(x.data_ptr(), ldx, out.data_ptr(), _rows2d(out)[2], rows, C, _ptr(gamma), _ptr(beta),
                                  float(eps), _stream())
    _lib.check(rc, "imagd_layernorm_bf16")
    return out


def concat_add(a: torch.Tensor, b: Optional[torch.Tensor] = None, *, res_a=None, res_b=None,
               out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """cat([a (+res_a), b (+res_b)], -1) over token-major tensors of equal row count."""
    lib = _lib.load()
    rows, Ca, lda = _rows2d(a)
    Cb, ldb = 0, 0
    if b is not None:
        rb, Cb, ldb = _rows2d(b)
        assert rb == rows
    if out is None:
        out = torch.empty(*a.shape[:-1], Ca + Cb, device=a.device, dtype=BF16)
    rc = lib.imagd_concat_add_bf16(a.data_ptr(), lda, Ca, _ptr(res_a), _rows2d(res_a)[2] if res_a is not None else 0,
                                   _ptr(b), ldb, Cb, _ptr(res_b), _rows2d(res_b)[2] if res_b is not None else 0,
                                   out.data_ptr(), _rows2d(out)[2], rows, _stream())
    _lib.check(rc, "imagd_concat_add_bf16")
    return out


def upsample2x(x: torch.Tensor) -> torch.Tensor:
    lib = _lib.load()
    NB, H, W, C = x.shape
    assert x.is_contiguous() and x.dtype == BF16
    out = torch.empty(NB, 2 * H, 2 * W, C, device=x.device, dtype=BF16)
    _lib.check(lib.imagd_upsample2x_bf16(x.data_ptr(), out.data_ptr(), NB, H, W, C, _stream()), "imagd_upsample2x_bf16")
    return out


def pixel_unshuffle8(x: torch.Tensor) -> torch.Tensor:
    """fp32 NCHW [n, C, H, W] -> bf16 NHWC [n, H/8, W/8, C*64], torch.nn.PixelUnshuffle(8) channel order."""
    lib = _lib.load()
    NB, C, H, W = x.shape
    assert x.is_contiguous() and x.dtype == torch.float32
    out = torch.empty(NB, H // 8, W // 8, C * 64, device=x.device, dtype=BF16)
    _lib.check(lib.imagd_pixel_unshuffle8_bf16(x.data_ptr(), out.data_ptr(), NB, C, H, W, _stream()),
               "imagd_pixel_unshuffle8_bf16")
    return out


def avgpool2x2(x: torch.Tensor) -> torch.Tensor:
    """2x2 / stride-2 average pool of bf16 [NB, H, W, C] (H, W even)."""
    lib = _lib.load()
    NB, H, W, C = x.shape
    assert x.is_contiguous() and x.dtype == BF16
    out = torch.empty(NB, H // 2, W // 2, C, device=x.device, dtype=BF16)
    _lib.check(lib.imagd_avgpool2x2_bf16(x.data_ptr(), out.data_ptr(), NB, H, W, C, _stream()), "imagd_avgpool2x2_bf16")
    return out


def scaled_add_bcast(x: torch.Tensor, f: torch.Tensor, scale: torch.Tensor) -> torch.Tensor:
    """In place: x[s] += scale[0] * f[s % n_src] over channel-last x [NB, H, W, C] (pixels equally spaced, e.g. a channel
    slice) and contiguous f [n_src, H, W, C] bf16; scale is a device fp32 scalar."""
    lib = _lib.load()
    NB, H, W, C = x.shape
    assert x.dtype == BF16 and f.dtype == BF16 and f.is_contiguous() and tuple(f.shape[1:]) == (H, W, C)
    assert scale.dtype == torch.float32 and scale.numel() == 1 and NB % f.shape[0] == 0
    _lib.check(lib.imagd_scaled_add_bcast_bf16(x.data_ptr(), _pixel_ld(x), f.data_ptr(), scale.data_ptr(), NB, f.shape[0],
                                               H * W, C, _stream()), "imagd_scaled_add_bcast_bf16")
    return x


def im2col3x3_s2(x: torch.Tensor, pad_lo: int = 1) -> torch.Tensor:
    """Stride-2 3x3 patches, tap-major. pad_lo = 1: symmetric padding 1 (UNet Downsample2D); pad_lo = 0: the VAE
    encoder's (0,1,0,1) right/bottom-only padding."""
    lib = _lib.load()
    NB, H, W, C = x.shape
    assert x.is_contiguous() and x.dtype == BF16
    out = torch.empty(NB, H // 2, W // 2, 9 * C, device=x.device, dtype=BF16)
    if pad_lo == 1:
        _lib.check(lib.imagd_im2col3x3_s2_bf16(x.data_ptr(), out.data_ptr(), NB, H, W, C, _stream()),
                   "imagd_im2col3x3_s2_bf16")
    else:
        _lib.check(lib.imagd_im2col3x3_s2_pad_bf16(x.data_ptr(), out.data_ptr(), NB, H, W, C, int(pad_lo), _stream()),
                   "imagd_im2col3x3_s2_pad_bf16")
    return out


def softmax_rows(s: torch.Tensor, scale: float = 1.0, *, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """softmax(scale * s) over the last dim: fp32 [rows, cols] -> bf16 [rows, cols]."""
    lib = _lib.load()
    assert s.dtype == torch.float32 and s.dim() == 2 and s.stride(1) == 1
    rows, cols = s.shape
    if out is None:
        out = torch.empty(rows, cols, device=s.device, dtype=BF16)
    _lib.check(lib.imagd_softmax_rows(s.data_ptr(), s.stride(0), out.data_ptr(), out.stride(0), rows, cols, float(scale),
                                      _stream()), "imagd_softmax_rows")
    return out


def conv3x3_direct(x: torch.Tensor, w: torch.Tensor, bias, *, stride: int = 1, act: int = ACT_NONE,
                   out_nchw_f32: bool = False, add: Optional[torch.Tensor] = None,
                   out: Optional[torch.Tensor] = None) -> torch.Tensor:
    lib = _lib.load()
    NB, H, W, Cin = x.shape
    assert x.is_contiguous() and x.dtype == BF16 and w.dtype == BF16
    Cout = w.shape[0]
    Ho, Wo = (H + stride - 1) // stride, (W + stride - 1) // stride
    if out is None:
        if out_nchw_f32:
            out = torch.empty(NB, Cout, Ho, Wo, device=x.device, dtype=torch.float32)
        else:
            out = torch.empty(NB, Ho, Wo, Cout, device=x.device, dtype=BF16)
    rc = lib.imagd_conv3x3_direct_bf16(x.data_ptr(), NB, H, W, Cin, w.data_ptr(), _ptr(bias), out.data_ptr(), Cout,
                                       stride, act, 1 if out_nchw_f32 else 0, _ptr(add), _stream())
    _lib.check(rc, "imagd_conv3x3_direct_bf16")
    return out


def nchw_f32_to_nhwc_bf16(x: torch.Tensor, cpad: Optional[int] = None, *, repeat: int = 1, out=None) -> torch.Tensor:
    lib = _lib.load()
    NB, C, H, W = x.shape
    assert x.is_contiguous() and x.dtype == torch.float32
    cpad = cpad or C
    if out is None:
        out = torch.empty(NB * repeat, H, W, cpad, device=x.device, dtype=BF16)
    _lib.check(lib.imagd_nchw_f32_to_nhwc_bf16(x.data_ptr(), out.data_ptr(), NB, C, H, W, cpad, repeat, _stream()),
               "imagd_nchw_f32_to_nhwc_bf16")
    return out


def timestep_embedding(timesteps: torch.Tensor, step_ptr: Optional[torch.Tensor], NB: int, dim: int, *,
                       out=None) -> torch.Tensor:
    lib = _lib.load()
    assert timesteps.dtype == torch.float32
    if out is None:
        out = torch.empty(NB, dim, device=timesteps.device, dtype=torch.float32)
    _lib.check(lib.imagd_timestep_embedding(timesteps.data_ptr(), _ptr(step_ptr), out.data_ptr(), NB, dim, _stream()),
               "imagd_timestep_embedding")
    return out


def linear_small_m(x: torch.Tensor, w: torch.Tensor, bias, *, act_in: int = ACT_NONE, act_out: int = ACT_NONE,
                   out=None) -> torch.Tensor:
    lib = _lib.load()
    M, K = x.shape
    N = w.shape[0]
    assert x.dtype == torch.float32 and w.dtype == BF16 and x.stride(1) == 1 and w.shape[1] == K
    if out is None:
        out = torch.empty(M, N, device=x.device, dtype=torch.float32)
    rc = lib.imagd_linear_small_m(x.data_ptr(), x.stride(0), w.data_ptr(), w.stride(0), _ptr(bias), out.data_ptr(),
                                  out.stride(0), M, N, K, act_in, act_out, _stream())
    _lib.check(rc, "imagd_linear_small_m")
    return out


def cfg_ddim_step(eps_cond: torch.Tensor, eps_uncond: Optional[torch.Tensor], guidance: float, latents: torch.Tensor,
                  coef: torch.Tensor, step_ptr: torch.Tensor, *, mask=None, image_latents=None, noise=None,
                  blend_coef=None) -> torch.Tensor:
    """In-place on `latents` (fp32 NCHW). step_ptr: int32[2] device tensor {step, scratch}."""
    lib = _lib.load()
    NB, C, H, W = latents.shape
    assert latents.dtype == torch.float32 and latents.is_contiguous() and eps_cond.dtype == torch.float32
    assert step_ptr.dtype == torch.int32 and step_ptr.numel() >= 2
    rc = lib.imagd_cfg_ddim_step(eps_cond.data_ptr(), _ptr(eps_uncond), float(guidance), latents.data_ptr(),
                                 coef.data_ptr(), step_ptr.data_ptr(), _ptr(mask), _ptr(image_latents), _ptr(noise),
                                 _ptr(blend_coef), NB, C, H * W, _stream())
    _lib.check(rc, "imagd_cfg_ddim_step")
    return latents


def nchw_f32_to_nhwc_bf16_scaled(x: torch.Tensor, scale_table: torch.Tensor, step_ptr: Optional[torch.Tensor], *,
                                 repeat: int = 1, out=None) -> torch.Tensor:
    """nchw_f32_to_nhwc_bf16 times scale_table[step_ptr[0]] (device-side read; step 0 without a step_ptr)."""
    lib = _lib.load()
    NB, C, H, W = x.shape
    assert x.is_contiguous() and x.dtype == torch.float32 and scale_table.dtype == torch.float32
    if out is None:
        out = torch.empty(NB * repeat, H, W, C, device=x.device, dtype=BF16)
    _lib.check(lib.imagd_nchw_f32_to_nhwc_bf16_scaled(x.data_ptr(), out.data_ptr(), NB, C, H, W, C, repeat,
                                                      scale_table.data_ptr(), _ptr(step_ptr), _stream()),
               "imagd_nchw_f32_to_nhwc_bf16_scaled")
    return out


def cfg_sampler_step(eps_cond: torch.Tensor, eps_uncond: Optional[torch.Tensor], guidance: float, latents: torch.Tensor,
                     coef: torch.Tensor, step_ptr: torch.Tensor, *, history=None, step_noise=None, mask=None,
                     image_latents=None, noise=None, blend_coef=None) -> torch.Tensor:
    """In-place on `latents` (fp32 NCHW) and `history`. coef: fp32 [S, 6] rows {dx, de, cx, ce, ch, cz}
    (include/imagd_b200.h); step_noise: fp32 [S, *latents.shape]; step_ptr: int32[2] device tensor {step, scratch}."""
    lib = _lib.load()
    NB, C, H, W = latents.shape
    assert latents.dtype == torch.float32 and latents.is_contiguous() and eps_cond.dtype == torch.float32
    assert step_ptr.dtype == torch.int32 and step_ptr.numel() >= 2 and coef.shape[-1] == 6
    assert history is None or (history.shape == latents.shape and history.is_contiguous())
    assert step_noise is None or (step_noise.shape[1:] == latents.shape and step_noise.is_contiguous())
    rc = lib.imagd_cfg_sampler_step(eps_cond.data_ptr(), _ptr(eps_uncond), float(guidance), latents.data_ptr(),
                                    _ptr(history), _ptr(step_noise), coef.data_ptr(), step_ptr.data_ptr(), _ptr(mask),
                                    _ptr(image_latents), _ptr(noise), _ptr(blend_coef), NB, C, H * W, _stream())
    _lib.check(rc, "imagd_cfg_sampler_step")
    return latents


PC_SLOTS = 4


def cfg_sampler_pc_step(eps_cond: torch.Tensor, eps_uncond: Optional[torch.Tensor], guidance: float,
                        latents: torch.Tensor, coef: torch.Tensor, step_ptr: torch.Tensor, bank: torch.Tensor, *,
                        mask=None, image_latents=None, noise=None, blend_coef=None) -> torch.Tensor:
    """In-place on `latents` (fp32 NCHW) and `bank` (fp32 [PC_SLOTS, *latents.shape], caller-owned). coef: fp32
    [S, 16] rows {dx, de, ax, am, a0..a3, bc, bm, b0..b3, w_m, w_c} (include/imagd_b200.h); step_ptr: int32[2]
    device tensor {step, scratch}."""
    lib = _lib.load()
    NB, C, H, W = latents.shape
    assert latents.dtype == torch.float32 and latents.is_contiguous() and eps_cond.dtype == torch.float32
    assert step_ptr.dtype == torch.int32 and step_ptr.numel() >= 2 and coef.shape[-1] == 16
    assert bank.dtype == torch.float32 and bank.shape == (PC_SLOTS, *latents.shape) and bank.is_contiguous()
    rc = lib.imagd_cfg_sampler_pc_step(eps_cond.data_ptr(), _ptr(eps_uncond), float(guidance), latents.data_ptr(),
                                       bank.data_ptr(), coef.data_ptr(), step_ptr.data_ptr(), _ptr(mask),
                                       _ptr(image_latents), _ptr(noise), _ptr(blend_coef), NB, C, H * W, _stream())
    _lib.check(rc, "imagd_cfg_sampler_pc_step")
    return latents


def embed_tokens(ids: torch.Tensor, tok: torch.Tensor, pos: torch.Tensor) -> torch.Tensor:
    """ids int64 [B, T]; tok bf16 [V, C]; pos bf16 [>= T, C] -> bf16 [B, T, C] = tok[ids] + pos[:T]."""
    lib = _lib.load()
    B, T = ids.shape
    assert ids.dtype == torch.int64 and ids.is_contiguous() and tok.dtype == BF16 and pos.dtype == BF16
    assert tok.is_contiguous() and pos.is_contiguous() and pos.shape[0] >= T and pos.shape[1] == tok.shape[1]
    out = torch.empty(B, T, tok.shape[1], device=ids.device, dtype=BF16)
    _lib.check(lib.imagd_embed_tokens_bf16(ids.data_ptr(), tok.data_ptr(), pos.data_ptr(), out.data_ptr(), B * T, T,
                                           tok.shape[1], tok.shape[0], _stream()), "imagd_embed_tokens_bf16")
    return out


def patchify(x: torch.Tensor, patch: int, kpad: int) -> torch.Tensor:
    """fp32 [B, 3, H, W] -> bf16 [B * (H/patch) * (W/patch), kpad] patch rows (column = (c*patch + iy)*patch + ix)."""
    lib = _lib.load()
    B, C, H, W = x.shape
    assert C == 3 and x.dtype == torch.float32 and x.is_contiguous()
    out = torch.empty(B * (H // patch) * (W // patch), kpad, device=x.device, dtype=BF16)
    _lib.check(lib.imagd_patchify_bf16(x.data_ptr(), out.data_ptr(), B, H, W, patch, kpad, _stream()), "imagd_patchify_bf16")
    return out


def broadcast_row(vec: torch.Tensor, out: torch.Tensor, row: int) -> torch.Tensor:
    """out[b, row, :] = vec for every sample of out [B, rows, C] (bf16, contiguous)."""
    lib = _lib.load()
    B, R, C = out.shape
    assert out.is_contiguous() and out.dtype == BF16 and vec.dtype == BF16 and vec.numel() == C
    _lib.check(lib.imagd_broadcast_row_bf16(vec.data_ptr(), out.data_ptr(), B, R, row, C, _stream()),
               "imagd_broadcast_row_bf16")
    return out


# ====================================================================================================== training step
# Wrappers of the backward / training kernels (include/imagd_b200.h "Training step"; SURVEY.md section 8 row a13). They are
# called by the torch.autograd.Function classes of imagdressing_b200/autograd.py.
_ws_cache = {}


def _workspace(device, nbytes: int) -> torch.Tensor:
    ws = _ws_cache.get(device)
    if ws is None or ws.numel() < nbytes:
        ws = torch.empty(max(int(nbytes), 1 << 20), device=device, dtype=torch.uint8)
        _ws_cache[device] = ws
    return ws


class AttnSaved:
    """What a training-mode attention forward keeps for its backward."""

    __slots__ = ("lse", "o0", "o1", "lq_pad", "out")

    def __init__(self, lse, o0, o1, lq_pad, out):
        self.lse, self.o0, self.o1, self.lq_pad, self.out = lse, o0, o1, lq_pad, out


def attention_train(q: torch.Tensor, B: int, Lq: int, heads: int, head_dim: int, s0: KVStream, s1: Optional[KVStream] = None,
                    *, sm_scale: Optional[float] = None):
    """attention() that also returns AttnSaved (per-stream log-sum-exp rows and un-weighted per-stream outputs)."""
    lib = _lib.load()
    assert q.dtype == BF16 and q.stride(-1) == 1
    C = heads * head_dim
    out = torch.empty(B * Lq, C, device=q.device, dtype=BF16)
    lq_pad = (Lq + 127) // 128 * 128
    lse = torch.full((2, B, heads, lq_pad), float("inf"), device=q.device, dtype=torch.float32)
    two = s1 is not None
    o0 = torch.empty_like(out) if two else None
    o1 = torch.empty_like(out) if two else None
    aux = _lib.AttnTrain()
    aux.lse, aux.out_s0, aux.out_s1, aux.ld_s, aux.lq_pad = lse.data_ptr(), _ptr(o0), _ptr(o1), C, lq_pad
    if sm_scale is None:
        sm_scale = head_dim ** -0.5
    rc = lib.imagd_attention_train_fwd_bf16(q.data_ptr(), q.stride(-2), out.data_ptr(), C, B, Lq, heads, head_dim,
                                            ctypes.byref(s0), ctypes.byref(s1) if two else None, float(sm_scale),
                                            ctypes.byref(aux), _stream())
    _lib.check(rc, "imagd_attention_train_fwd_bf16")
    return out, AttnSaved(lse, o0, o1, lq_pad, out)


def attention_bwd(q: torch.Tensor, d_out: torch.Tensor, B: int, Lq: int, heads: int, head_dim: int, s0: KVStream,
                  s1: Optional[KVStream], saved: AttnSaved, *, sm_scale: Optional[float] = None, dq=None, dkv0=None, dkv1=None):
    """dq: [B*Lq, >= C] view to receive dQ (or None); dkv0 / dkv1: (dk_view, dv_view) laid out like the stream's k / v (same
    row stride and sample stride) or None. d_out: [B*Lq, C] bf16 (row stride arbitrary)."""
    lib = _lib.load()
    assert d_out.dtype == BF16 and d_out.stride(-1) == 1 and q.dtype == BF16
    two = s1 is not None
    dsum = torch.zeros_like(saved.lse)
    if two:
        rc = lib.imagd_attention_bwd_prep(d_out.data_ptr(), d_out.stride(-2), saved.o0.data_ptr(), saved.o1.data_ptr(),
                                          saved.o0.stride(-2), float(s0.out_scale), float(s1.out_scale), dsum.data_ptr(), B, Lq,
                                          heads, head_dim, saved.lq_pad, _stream())
    else:  # out = w0 * O_0, so D_0 = rowsum(dO o out)
        rc = lib.imagd_attention_bwd_prep(d_out.data_ptr(), d_out.stride(-2), saved.out.data_ptr(), None,
                                          saved.out.stride(-2), 1.0, 0.0, dsum.data_ptr(), B, Lq, heads, head_dim,
                                          saved.lq_pad, _stream())
    _lib.check(rc, "imagd_attention_bwd_prep")
    if sm_scale is None:
        sm_scale = head_dim ** -0.5

    def kvp(pair):
        if pair is None:
            return None, None, 0
        dk, dv = pair
        assert dk.dtype == BF16 and dk.stride(-1) == 1 and dv.stride(-2) == dk.stride(-2)
        return dk.data_ptr(), dv.data_ptr(), dk.stride(-2)

    k0p, v0p, ld0 = kvp(dkv0)
    k1p, v1p, ld1 = kvp(dkv1)
    rc = lib.imagd_attention_bwd_bf16(q.data_ptr(), q.stride(-2), d_out.data_ptr(), d_out.stride(-2), B, Lq, heads, head_dim,
                                      ctypes.byref(s0), ctypes.byref(s1) if two else None, float(sm_scale),
                                      saved.lse.data_ptr(), dsum.data_ptr(), saved.lq_pad, _ptr(dq),
                                      dq.stride(-2) if dq is not None else 0, k0p, v0p, ld0, k1p, v1p, ld1, _stream())
    _lib.check(rc, "imagd_attention_bwd_bf16")


def transpose(x: torch.Tensor, pad_to: int = 8, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """x: [rows, cols] bf16 (row stride arbitrary) -> [cols, rows_pad] with zero columns up to a multiple of `pad_to`.
    out: a [cols, rows] view (row stride arbitrary) to write into instead (no padding then)."""
    lib = _lib.load()
    assert x.dim() == 2 and x.dtype == BF16 and x.stride(1) == 1
    rows, cols = x.shape
    if out is not None:
        assert out.shape == (cols, rows) and out.dtype == BF16 and out.stride(1) == 1
        _lib.check(lib.imagd_transpose_bf16(x.data_ptr(), x.stride(0), out.data_ptr(), out.stride(0), rows, cols, rows, _stream()),
                   "imagd_transpose_bf16")
        return out
    rows_pad = (rows + pad_to - 1) // pad_to * pad_to
    out = torch.empty(cols, rows_pad, device=x.device, dtype=BF16)
    _lib.check(lib.imagd_transpose_bf16(x.data_ptr(), x.stride(0), out.data_ptr(), rows_pad, rows, cols, rows_pad, _stream()),
               "imagd_transpose_bf16")
    return out


def conv_weight_layout(w: torch.Tensor, mode: int) -> torch.Tensor:
    """mode 0: [Cout, Cin, 3, 3] -> tap-major [Cout, 9*Cin]; mode 1: packed [Cout, 9*Cin] -> [Cout, Cin, 3, 3]. bf16, contiguous."""
    lib = _lib.load()
    assert w.dtype == BF16 and w.is_contiguous()
    if mode == 0:
        co, ci = w.shape[:2]
        out = torch.empty(co, 9 * ci, device=w.device, dtype=BF16)
    else:
        co, ci = w.shape[0], w.shape[1] // 9
        out = torch.empty(co, ci, 3, 3, device=w.device, dtype=BF16)
    _lib.check(lib.imagd_conv_weight_layout_bf16(w.data_ptr(), out.data_ptr(), co, ci, int(mode), _stream()),
               "imagd_conv_weight_layout_bf16")
    return out


def conv_weight_flip(wp: torch.Tensor, cin: int) -> torch.Tensor:
    """Packed [Cout, 9*Cin] -> the dgrad weight [Cin, 9*Cout] (taps reversed, channel roles swapped)."""
    lib = _lib.load()
    assert wp.dtype == BF16 and wp.is_contiguous() and wp.shape[1] == 9 * cin
    co = wp.shape[0]
    out = torch.empty(cin, 9 * co, device=wp.device, dtype=BF16)
    _lib.check(lib.imagd_conv_weight_flip_bf16(wp.data_ptr(), out.data_ptr(), co, cin, _stream()), "imagd_conv_weight_flip_bf16")
    return out


def im2col3x3_t(x: torch.Tensor) -> torch.Tensor:
    """x: [NB, H, W, C] bf16 -> [roundup(9*C, 8), roundup(NB*H*W, 8)] transposed stride-1 pad-1 patches (tap-major rows)."""
    lib = _lib.load()
    NB, H, W, C = x.shape
    assert x.is_contiguous() and x.dtype == BF16
    P = NB * H * W
    ldo = (P + 7) // 8 * 8
    rows = (9 * C + 7) // 8 * 8
    out = (torch.zeros if rows != 9 * C else torch.empty)(rows, ldo, device=x.device, dtype=BF16)
    _lib.check(lib.imagd_im2col3x3_t_bf16(x.data_ptr(), out.data_ptr(), ldo, NB, H, W, C, _stream()), "imagd_im2col3x3_t_bf16")
    return out


def col2im3x3_s2(dcol: torch.Tensor, H: int, W: int) -> torch.Tensor:
    """Adjoint of im2col3x3_s2: dcol [NB, H/2, W/2, 9*C] -> [NB, H, W, C]."""
    lib = _lib.load()
    NB, C = dcol.shape[0], dcol.shape[-1] // 9
    assert dcol.is_contiguous() and dcol.dtype == BF16
    out = torch.empty(NB, H, W, C, device=dcol.device, dtype=BF16)
    _lib.check(lib.imagd_col2im3x3_s2_bf16(dcol.data_ptr(), out.data_ptr(), NB, H, W, C, _stream()), "imagd_col2im3x3_s2_bf16")
    return out


def downsum2x(dy: torch.Tensor) -> torch.Tensor:
    """Adjoint of upsample2x: [NB, 2H, 2W, C] -> [NB, H, W, C]."""
    lib = _lib.load()
    NB, H2, W2, C = dy.shape
    assert dy.is_contiguous() and dy.dtype == BF16
    out = torch.empty(NB, H2 // 2, W2 // 2, C, device=dy.device, dtype=BF16)
    _lib.check(lib.imagd_downsum2x_bf16(dy.data_ptr(), out.data_ptr(), NB, H2 // 2, W2 // 2, C, _stream()), "imagd_downsum2x_bf16")
    return out


def colsum(x: torch.Tensor, rows_per_group: Optional[int] = None, out_dtype=torch.float32) -> torch.Tensor:
    """x: [rows, C] bf16 -> [groups, C] column sums over consecutive groups of rows_per_group rows (fp32 or bf16 out)."""
    lib = _lib.load()
    rows, C, ldx = _rows2d(x)
    rpg = rows if rows_per_group is None else int(rows_per_group)
    groups = rows // rpg
    assert groups * rpg == rows and x.dtype == BF16 and out_dtype in (torch.float32, BF16)
    out = torch.empty(groups, C, device=x.device, dtype=out_dtype)
    ws = _workspace(x.device, lib.imagd_colreduce_ws_bytes(rpg, groups, C))
    _lib.check(lib.imagd_colsum_bf16(x.data_ptr(), ldx, rpg, groups, C, out.data_ptr(), 1 if out_dtype == BF16 else 0,
                                     ws.data_ptr(), _stream()), "imagd_colsum_bf16")
    return out


def layernorm_bwd(x: torch.Tensor, dy: torch.Tensor, gamma, eps: float, need_affine: bool, out_dtype=torch.float32):
    """-> (dx bf16 like x, dgamma [C] | None, dbeta [C] | None); the affine gradients in out_dtype (fp32 or bf16)."""
    lib = _lib.load()
    rows, C, ldx = _rows2d(x)
    _, _, lddy = _rows2d(dy)
    dx = torch.empty(*x.shape, device=x.device, dtype=BF16)
    rowstat = torch.empty(rows, 2, device=x.device, dtype=torch.float32)
    dg = torch.empty(C, device=x.device, dtype=out_dtype) if need_affine else None
    db = torch.empty(C, device=x.device, dtype=out_dtype) if need_affine else None
    ws = _workspace(x.device, lib.imagd_colreduce_ws_bytes(rows, 1, C))
    rc = lib.imagd_layernorm_bwd_bf16(x.data_ptr(), ldx, dy.data_ptr(), lddy, dx.data_ptr(), _rows2d(dx)[2], rows, C, _ptr(gamma),
                                      float(eps), _ptr(dg), _ptr(db), 1 if out_dtype == BF16 else 0, rowstat.data_ptr(),
                                      ws.data_ptr(), _stream())
    _lib.check(rc, "imagd_layernorm_bwd_bf16")
    return dx, dg, db


def groupnorm_bwd(x: torch.Tensor, dy: torch.Tensor, gamma, beta, groups: int, stats: torch.Tensor, silu: bool,
                  need_affine: bool, out_dtype=torch.float32):
    """x, dy: contiguous [NB, HW..., C] bf16; stats: the forward's {mean, rstd} [NB, groups, 2] fp32 (groupnorm(stats_out=))
    -> (dx, dgamma | None, dbeta | None); the affine gradients in out_dtype (fp32 or bf16)."""
    lib = _lib.load()
    assert x.is_contiguous() and dy.is_contiguous() and x.dtype == BF16 and dy.dtype == BF16
    NB, C = x.shape[0], x.shape[-1]
    HW = x.numel() // (NB * C)
    assert stats.dtype == torch.float32 and stats.is_contiguous() and stats.numel() == NB * groups * 2
    dx = torch.empty_like(x)
    dg = torch.empty(C, device=x.device, dtype=out_dtype) if need_affine else None
    db = torch.empty(C, device=x.device, dtype=out_dtype) if need_affine else None
    ws = _workspace(x.device, lib.imagd_groupnorm_bwd_ws_bytes(NB, HW, C, groups))
    rc = lib.imagd_groupnorm_bwd_bf16(x.data_ptr(), dy.data_ptr(), dx.data_ptr(), NB, HW, C, groups, _ptr(gamma), _ptr(beta),
                                      stats.data_ptr(), 1 if silu else 0, _ptr(dg), _ptr(db), 1 if out_dtype == BF16 else 0,
                                      ws.data_ptr(), _stream())
    _lib.check(rc, "imagd_groupnorm_bwd_bf16")
    return dx, dg, db


def act(x: torch.Tensor, mode: int, dy: Optional[torch.Tensor] = None) -> torch.Tensor:
    """mode ACT_SILU / ACT_GELU. dy None: act(x); else dy * act'(x). Contiguous bf16."""
    lib = _lib.load()
    assert x.is_contiguous() and x.dtype == BF16 and (dy is None or (dy.is_contiguous() and dy.dtype == BF16))
    y = torch.empty_like(x)
    _lib.check(lib.imagd_act_bf16(x.data_ptr(), _ptr(dy), y.data_ptr(), x.numel(), int(mode), _stream()), "imagd_act_bf16")
    return y


def geglu(h: torch.Tensor, dout: Optional[torch.Tensor] = None) -> torch.Tensor:
    """h: [..., 2F] = [value | gate]. dout None: value * gelu(gate) [..., F]; else dh [..., 2F]."""
    lib = _lib.load()
    assert h.is_contiguous() and h.dtype == BF16
    F2 = h.shape[-1]
    M = h.numel() // F2
    if dout is None:
        out = torch.empty(*h.shape[:-1], F2 // 2, device=h.device, dtype=BF16)
        ldo = F2 // 2
    else:
        assert dout.is_contiguous() and dout.dtype == BF16
        out = torch.empty_like(h)
        ldo = F2
    _lib.check(lib.imagd_geglu_bf16(h.data_ptr(), F2, _ptr(dout), out.data_ptr(), ldo, M, F2 // 2, _stream()), "imagd_geglu_bf16")
    return out


def mse_loss_grad(pred: torch.Tensor, target: torch.Tensor, grad_scale: float = 1.0):
    """-> (loss fp32 [1], grad fp32 like pred) of mean((pred - target)^2)."""
    lib = _lib.load()
    assert pred.dtype == torch.float32 and target.dtype == torch.float32 and pred.is_contiguous() and target.is_contiguous()
    grad = torch.empty_like(pred)
    loss = torch.empty(1, device=pred.device, dtype=torch.float32)
    ws = _workspace(pred.device, 4096)
    _lib.check(lib.imagd_mse_loss_grad(pred.data_ptr(), target.data_ptr(), grad.data_ptr(), loss.data_ptr(), pred.numel(),
                                       float(grad_scale), ws.data_ptr(), _stream()), "imagd_mse_loss_grad")
    return loss, grad


def adamw_step(master: torch.Tensor, param: torch.Tensor, grad: torch.Tensor, m: torch.Tensor, v: torch.Tensor, *, lr: float,
               beta1: float, beta2: float, eps: float, weight_decay: float, step: int, grad_scale: float = 1.0) -> None:
    """In place: fp32 master / moments, bf16 gradient, bf16 working copy (flat, contiguous, equal length)."""
    lib = _lib.load()
    n = master.numel()
    assert master.dtype == torch.float32 and m.dtype == torch.float32 and v.dtype == torch.float32
    assert param.dtype == BF16 and grad.dtype == BF16 and param.numel() == n and grad.numel() == n
    _lib.check(lib.imagd_adamw_step(master.data_ptr(), param.data_ptr(), grad.data_ptr(), m.data_ptr(), v.data_ptr(), n, float(lr),
                                    float(beta1), float(beta2), float(eps), float(weight_decay), int(step), float(grad_scale),
                                    _stream()), "imagd_adamw_step")


def adamw_step_dev(master: torch.Tensor, param: torch.Tensor, grad: torch.Tensor, m: torch.Tensor, v: torch.Tensor,
                   hyper: torch.Tensor, *, beta1: float, beta2: float, eps: float) -> None:
    """adamw_step with {lr, weight_decay, step, grad_scale} in the fp32 device tensor `hyper` (CUDA-graph replayable)."""
    lib = _lib.load()
    n = master.numel()
    assert master.dtype == torch.float32 and m.dtype == torch.float32 and v.dtype == torch.float32
    assert param.dtype == BF16 and grad.dtype == BF16 and param.numel() == n and grad.numel() == n
    assert hyper.dtype == torch.float32 and hyper.numel() >= 4 and hyper.is_contiguous()
    _lib.check(lib.imagd_adamw_step_dev(master.data_ptr(), param.data_ptr(), grad.data_ptr(), m.data_ptr(), v.data_ptr(), n,
                                        float(beta1), float(beta2), float(eps), hyper.data_ptr(), _stream()), "imagd_adamw_step_dev")


def grad_norm_ws_bytes(n: int) -> int:
    """Bytes of the workspace grad_norm_clip needs for an n-element gradient (allocate once, zeroed)."""
    return int(_lib.load().imagd_grad_norm_ws_bytes(int(n)))


def grad_norm_clip(grad: torch.Tensor, hyper: torch.Tensor, state: torch.Tensor, ws: torch.Tensor, *, max_norm: float) -> None:
    """Global-norm clipping pass over the flat bf16 gradient: state (fp64 [4]) = {norm of hyper[3] * grad, coef =
    min(1, max_norm / (norm + 1e-6)), finite, skipped updates}; hyper[2] advances only when the norm is finite. ws: a zeroed
    uint8 tensor of grad_norm_ws_bytes(grad.numel()) bytes kept for every call (CUDA-graph replayable)."""
    lib = _lib.load()
    assert grad.dtype == BF16 and grad.is_contiguous()
    assert hyper.dtype == torch.float32 and hyper.numel() >= 4 and hyper.is_contiguous()
    assert state.dtype == torch.float64 and state.numel() >= 4 and state.is_contiguous()
    assert ws.numel() * ws.element_size() >= grad_norm_ws_bytes(grad.numel())
    _lib.check(lib.imagd_grad_norm_clip(grad.data_ptr(), grad.numel(), float(max_norm), hyper.data_ptr(), state.data_ptr(),
                                        ws.data_ptr(), _stream()), "imagd_grad_norm_clip")


def adamw_step_clip(master: torch.Tensor, param: torch.Tensor, grad: torch.Tensor, m: torch.Tensor, v: torch.Tensor,
                    hyper: torch.Tensor, clip_state: torch.Tensor, *, beta1: float, beta2: float, eps: float) -> None:
    """adamw_step_dev with the gradient scale hyper[3] * coef of grad_norm_clip's state; a non-finite gradient (state
    finite == 0) leaves master / param / m / v untouched."""
    lib = _lib.load()
    n = master.numel()
    assert master.dtype == torch.float32 and m.dtype == torch.float32 and v.dtype == torch.float32
    assert param.dtype == BF16 and grad.dtype == BF16 and param.numel() == n and grad.numel() == n
    assert hyper.dtype == torch.float32 and hyper.numel() >= 4 and hyper.is_contiguous()
    assert clip_state.dtype == torch.float64 and clip_state.numel() >= 4 and clip_state.is_contiguous()
    _lib.check(lib.imagd_adamw_step_clip(master.data_ptr(), param.data_ptr(), grad.data_ptr(), m.data_ptr(), v.data_ptr(), n,
                                         float(beta1), float(beta2), float(eps), hyper.data_ptr(), clip_state.data_ptr(),
                                         _stream()), "imagd_adamw_step_clip")
