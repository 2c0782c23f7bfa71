"""Host-side mirror of the diffusers-0.24 SD1.5 UNet2DConditionModel / ControlNetModel surface the reference
drives (SURVEY.md §8b "Host-model surface"), executing on the sm_90a kernels of libimagd_b200.so.

The nn.Module tree only *holds* parameters under the diffusers state_dict key names (so the reference's
checkpoint routing, `.to()`, `.state_dict()`, `set_attn_processor` keep working); arithmetic never goes through
torch.nn forward. On first use the weights are repacked once for the kernels (bf16, token-major: 3x3 convs
tap-major, q/k/v fused, GEGLU rows interleaved, all time_emb_proj layers concatenated) and activations stay
bf16 [N, H, W, C] end to end — the transformer blocks read the same memory as [N, H*W, C], so the reference's
NCHW<->tokens permutes do not exist here.

Reference call sites: dressing_sd/pipelines/IMAGDressing_v1_pipeline.py:466,499,511 (UNet),
IMAGDressing_v1_pipeline_ipa_controlnet.py:651 (ControlNet), inference_IMAGdressing.py:50,68-94 (construction,
processor registration). Architecture: SURVEY.md Appendix A (diffusers 0.24.0, requirements.txt:12).
"""
from __future__ import annotations

import contextlib
import os
from typing import Dict, List, Optional, Sequence

import torch
import torch.nn as nn

from . import ops
from ._lib import ACT_GEGLU, ACT_NONE, ACT_SILU

BF16 = torch.bfloat16

SD15_CONFIG = dict(
    in_channels=4, out_channels=4, sample_size=64, block_out_channels=(320, 640, 1280, 1280), layers_per_block=2,
    cross_attention_dim=768, attention_head_dim=8, norm_num_groups=32, time_cond_proj_dim=None,
    down_block_types=("CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "DownBlock2D"),
    up_block_types=("UpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D"),
    addition_embed_type=None, global_pool_conditions=False,
)


class FrozenConfig(dict):
    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e


@contextlib.contextmanager
def skip_default_init():
    """Construct modules without running nn.Linear / nn.Conv2d default initialisation (kaiming_uniform over 860 M
    parameters costs ~40 s of CPU per UNet). Only for call sites that overwrite EVERY parameter right after —
    `load_state_dict`, `init_synthetic_`, `init_synthetic_fast_`, `from_pretrained`; parameters are torch.empty until then."""
    saved = (nn.Linear.reset_parameters, nn.Conv2d.reset_parameters)
    nn.Linear.reset_parameters = lambda self: None
    nn.Conv2d.reset_parameters = lambda self: None
    try:
        yield
    finally:
        nn.Linear.reset_parameters, nn.Conv2d.reset_parameters = saved


# LayerNorm folded into the consuming GEMMs of the transformer blocks (48 fewer launches per step): on by default,
# IMAGD_FOLD_LN=0 switches it off; tests flip the module attribute.
FOLD_LN = os.environ.get("IMAGD_FOLD_LN", "1") == "1"


def fold_layernorm(w: torch.Tensor, b: Optional[torch.Tensor], gamma: torch.Tensor, beta: torch.Tensor):
    """LN(x) W^T + b == rstd * (x W'^T - mean * colsum(W')) + b'  with  W' = W diag(gamma), b' = b + W beta.
    Returns (W' bf16 [N, K], b' fp32 [N], colsum fp32 [N]); colsum is taken over the ROUNDED W' the tensor core sees."""
    w32 = w.detach().float()
    wp = (w32 * gamma.detach().float()[None, :]).to(BF16).contiguous()
    bp = w32 @ beta.detach().float()
    if b is not None:
        bp = bp + b.detach().float()
    return wp, bp.contiguous(), wp.float().sum(1).contiguous()


class _RowStats:
    """Per-module row-statistics buffers at stable addresses (one per LayerNorm site and row count)."""

    def __init__(self):
        self._bufs: Dict[tuple, tuple] = {}

    def get(self, site: str, M: int, C: int, device) -> tuple:
        key = (site, M, str(device))
        hit = self._bufs.get(key)
        if hit is None:
            parts = ops.gemm_tile_count_n(M, C, C)
            hit = (torch.zeros(M, parts, 2, device=device, dtype=torch.float32), parts)
            self._bufs[key] = hit
        return hit


def _f32(p: torch.Tensor) -> torch.Tensor:
    return p.detach().float().contiguous()


def _bf(p: torch.Tensor) -> torch.Tensor:
    return p.detach().to(BF16).contiguous()


def pack_conv3x3(w: torch.Tensor) -> torch.Tensor:
    """[Cout, Cin, 3, 3] -> tap-major [Cout, 9*Cin] bf16."""
    co, ci = w.shape[:2]
    return w.detach().permute(0, 2, 3, 1).reshape(co, 9 * ci).to(BF16).contiguous()


# Upsample2D + conv as four 2x2 phase convs on the low-resolution input (2.25x fewer MACs, no upsampled tensor).
# On by default, IMAGD_UPCONV_PHASE=0 switches it off.
UPCONV_PHASE = os.environ.get("IMAGD_UPCONV_PHASE", "1") == "1"


def pack_upconv3x3(w: torch.Tensor) -> torch.Tensor:
    """[Cout, Cin, 3, 3] -> phase weight matrix [4*Cout, 4*Cin] bf16 for nearest-2x upsample followed by the conv:
    output pixel (2y+py, 2x+px) = sum over taps (ty, tx) of Wp[py,px,ty,tx] . in[y+py-1+ty, x+px-1+tx], where
    Wp sums the 3x3 taps (ky, kx) whose upsampled source pixel floor((2y+py+ky-1)/2) is that input row (same for x):
    py = 0: ty 0 <- ky {0}, ty 1 <- ky {1, 2};  py = 1: ty 0 <- ky {0, 1}, ty 1 <- ky {2}."""
    co, ci = w.shape[:2]
    w32 = w.detach().float()
    sel = {(0, 0): [0], (0, 1): [1, 2], (1, 0): [0, 1], (1, 1): [2]}  # (phase bit, tap bit) -> 3x3 indices
    out = torch.zeros(4, co, 4, ci, dtype=torch.float32, device=w.device)
    for py in (0, 1):
        for px in (0, 1):
            for ty in (0, 1):
                for tx in (0, 1):
                    acc = 0
                    for ky in sel[(py, ty)]:
                        for kx in sel[(px, tx)]:
                            acc = acc + w32[:, :, ky, kx]
                    out[py * 2 + px, :, ty * 2 + tx, :] = acc
    return out.reshape(4 * co, 4 * ci).to(BF16).contiguous()


def pack_geglu(w: torch.Tensor, b: torch.Tensor):
    """GEGLU.proj [2F, K] (value rows then gate rows) -> per 128 rows: 64 value + their 64 gate rows."""
    F2, K = w.shape
    Fh = F2 // 2
    wv, wg = w[:Fh].reshape(Fh // 64, 64, K), w[Fh:].reshape(Fh // 64, 64, K)
    bv, bg = b[:Fh].reshape(Fh // 64, 64), b[Fh:].reshape(Fh // 64, 64)
    return (torch.cat([wv, wg], 1).reshape(F2, K).detach().to(BF16).contiguous(),
            torch.cat([bv, bg], 1).reshape(F2).detach().float().contiguous())


class _Packed:
    """Per-module cache of kernel-layout weights, rebuilt when parameters change (load_state_dict / .to())."""

    def __init__(self):
        self._pk = None

    def _invalidate(self):
        self._pk = None


# ================================================================================================ attention
class Attention(nn.Module):
    """The plugin boundary: `processor(attn, hidden_states, encoder_hidden_states=None, attention_mask=None,
    **cross_attention_kwargs)` exactly as diffusers-0.24 Attention.forward dispatches (reference processors read
    attn.to_q/to_k/to_v/to_out/heads/... — adapter/attention_processor.py:545-625)."""

    def __init__(self, query_dim: int, cross_attention_dim: Optional[int], heads: int):
        super().__init__()
        self.heads = heads
        self.query_dim = query_dim
        self.is_cross = cross_attention_dim is not None
        kv = cross_attention_dim or query_dim
        self.to_q = nn.Linear(query_dim, query_dim, bias=False)
        self.to_k = nn.Linear(kv, query_dim, bias=False)
        self.to_v = nn.Linear(kv, query_dim, bias=False)
        self.to_out = nn.ModuleList([nn.Linear(query_dim, query_dim), nn.Dropout(0.0)])
        self.spatial_norm = None
        self.group_norm = None
        self.norm_cross = False
        self.residual_connection = False
        self.rescale_output_factor = 1.0
        self.scale = (query_dim // heads) ** -0.5
        self._pk: Dict[str, torch.Tensor] = {}
        self._fused_residual: Optional[torch.Tensor] = None  # set by BasicTransformerBlock, consumed by our processors
        # LayerNorm fold handshake (same protocol): (LnFold-less tuple) set by the block when hidden_states is the RAW
        # stream: (stats, parts, gamma, beta, eps, stats_out_for_my_output | None); consumed by attention_forward
        self._ln_fold = None
        from .processors import AttnProcessor2_0

        self.processor = AttnProcessor2_0()

    # --- diffusers API
    def set_processor(self, processor, _remove_lora: bool = False):
        if isinstance(getattr(self, "processor", None), nn.Module) and not isinstance(processor, nn.Module):
            self._modules.pop("processor")
        self.processor = processor

    def get_processor(self, return_deprecated_lora: bool = False):
        return self.processor

    def prepare_attention_mask(self, attention_mask, target_length, batch_size, out_dim=3):
        if attention_mask is not None:
            raise NotImplementedError("attention masks are not on the IMAGDressing hot path (SURVEY.md A.6)")
        return None

    def forward(self, hidden_states, encoder_hidden_states=None, attention_mask=None, **cross_attention_kwargs):
        return self.processor(self, hidden_states, encoder_hidden_states=encoder_hidden_states,
                              attention_mask=attention_mask, **cross_attention_kwargs)

    # --- kernel-layout weights
    def _apply(self, fn, *a, **k):
        self._pk = {}
        return super()._apply(fn, *a, **k)

    def packed(self, key: str, build):
        """Cache of derived weights (fused q/k/v, LoRA-merged, ...). `key` must encode every mutable input."""
        t = self._pk.get(key)
        if t is None:
            t = build()
            self._pk[key] = t
        return t

    def invalidate_packed(self):
        self._pk = {}


class FeedForward(nn.Module):
    def __init__(self, dim):
        super().__init__()

        class GEGLU(nn.Module):
            def __init__(s):
                super().__init__()
                s.proj = nn.Linear(dim, dim * 8)

        self.net = nn.ModuleList([GEGLU(), nn.Dropout(0.0), nn.Linear(dim * 4, dim)])


class BasicTransformerBlock(nn.Module, _Packed):
    def __init__(self, dim, heads, cross_dim):
        nn.Module.__init__(self)
        _Packed.__init__(self)
        self.norm1 = nn.LayerNorm(dim)
        self.attn1 = Attention(dim, None, heads)
        self.norm2 = nn.LayerNorm(dim)
        self.attn2 = Attention(dim, cross_dim, heads)
        self.norm3 = nn.LayerNorm(dim)
        self.ff = FeedForward(dim)

    def _apply(self, fn, *a, **k):
        self._invalidate()
        return super()._apply(fn, *a, **k)

    def _packed(self):
        if self._pk is None:
            w1, b1 = pack_geglu(self.ff.net[0].proj.weight, self.ff.net[0].proj.bias)
            self._pk = dict(
                ln=[(_f32(n.weight), _f32(n.bias)) for n in (self.norm1, self.norm2, self.norm3)],
                w1=w1, b1=b1, w2=_bf(self.ff.net[2].weight), b2=_f32(self.ff.net[2].bias))
            if FOLD_LN:  # norm3 folded into the GEGLU projection: fold first, then interleave value / gate rows
                proj = self.ff.net[0].proj
                wf = proj.weight.detach().float() * self.norm3.weight.detach().float()[None, :]
                bf = proj.bias.detach().float() + proj.weight.detach().float() @ self.norm3.bias.detach().float()
                w1f, b1f = pack_geglu(wf, bf)
                self._pk.update(w1f=w1f, b1f=b1f, c1f=w1f.float().sum(1).contiguous())
        return self._pk

    def _can_fold(self) -> bool:
        return FOLD_LN and all(getattr(a.processor, "_accepts_ln_fold", False) for a in (self.attn1, self.attn2))

    def _attend(self, attn: Attention, normed, residual, ctx, kw):
        attn._fused_residual = residual
        out = attn(normed, encoder_hidden_states=ctx, **kw)
        if attn._fused_residual is None:  # consumed: the processor's out-projection already added it
            return out
        attn._fused_residual = None  # foreign processor: add here (bf16)
        return ops.concat_add(out.to(BF16).contiguous(), None, res_a=residual)

    def _attend_folded(self, attn: Attention, x, ctx, kw, stats, parts, norm: nn.LayerNorm, stats_next):
        attn._fused_residual = x
        attn._ln_fold = (stats, parts, norm.weight, norm.bias, norm.eps, stats_next)
        out = attn(x, encoder_hidden_states=ctx, **kw)
        if attn._ln_fold is not None or attn._fused_residual is not None:
            attn._ln_fold = attn._fused_residual = None
            raise RuntimeError("processor advertised _accepts_ln_fold but did not consume the LayerNorm fold")
        return out

    def run(self, x: torch.Tensor, ctx, kw, x_stats=None) -> torch.Tensor:
        """x: [B, L, C] bf16. x += attn1(LN(x)); x += attn2(LN(x), ctx); x += FF(LN(x))  (SURVEY.md A.2).
        x_stats = (stats, parts) of x's rows when the producing GEMM emitted them (LayerNorm fold)."""
        pk = self._packed()
        if x_stats is not None and self._can_fold():
            B, L, C = x.shape
            if not hasattr(self, "_row_stats"):
                self._row_stats = _RowStats()
            s1, p1 = self._row_stats.get("x1", B * L, C, x.device)
            s2, p2 = self._row_stats.get("x2", B * L, C, x.device)
            x1 = self._attend_folded(self.attn1, x, None, kw, x_stats[0], x_stats[1], self.norm1, s1)
            x2 = self._attend_folded(self.attn2, x1, ctx, kw, s1, p1, self.norm2, s2)
            h = ops.gemm(x2, pk["w1f"], bias=pk["b1f"], act=ACT_GEGLU,
                         ln=ops.LnFold(s2, p2, C, self.norm3.eps, pk["c1f"]))
            return ops.gemm(h, pk["w2"], bias=pk["b2"], residual=x2)
        x = self._attend(self.attn1, ops.layernorm(x, *pk["ln"][0]), x, None, kw)
        x = self._attend(self.attn2, ops.layernorm(x, *pk["ln"][1]), x, ctx, kw)
        h = ops.gemm(ops.layernorm(x, *pk["ln"][2]), pk["w1"], bias=pk["b1"], act=ACT_GEGLU)
        return ops.gemm(h, pk["w2"], bias=pk["b2"], residual=x)


class Transformer2DModel(nn.Module, _Packed):
    def __init__(self, dim, heads, cross_dim, groups):
        nn.Module.__init__(self)
        _Packed.__init__(self)
        self.norm = nn.GroupNorm(groups, dim, eps=1e-6)
        self.proj_in = nn.Conv2d(dim, dim, 1)
        self.transformer_blocks = nn.ModuleList([BasicTransformerBlock(dim, heads, cross_dim)])
        self.proj_out = nn.Conv2d(dim, dim, 1)
        self.groups = groups

    def _apply(self, fn, *a, **k):
        self._invalidate()
        return super()._apply(fn, *a, **k)

    def _packed(self):
        if self._pk is None:
            c = self.proj_in.weight.shape[0]
            self._pk = dict(gn=(_f32(self.norm.weight), _f32(self.norm.bias)),
                            wi=_bf(self.proj_in.weight.reshape(c, c)), bi=_f32(self.proj_in.bias),
                            wo=_bf(self.proj_out.weight.reshape(c, c)), bo=_f32(self.proj_out.bias))
        return self._pk

    def run(self, x: torch.Tensor, ctx, kw) -> torch.Tensor:
        pk = self._packed()
        NB, H, W, C = x.shape
        h = ops.groupnorm(x, *pk["gn"], self.groups, 1e-6, silu=False)
        x_stats = None
        if FOLD_LN and all(b._can_fold() for b in self.transformer_blocks):
            if not hasattr(self, "_row_stats"):
                self._row_stats = _RowStats()
            x_stats = self._row_stats.get("x0", NB * H * W, C, x.device)
        h = ops.gemm(h, pk["wi"], bias=pk["bi"], stats_out=None if x_stats is None else x_stats[0]).view(NB, H * W, C)
        for blk in self.transformer_blocks:
            h = blk.run(h, ctx, kw, x_stats)
            x_stats = None  # (SD1.5 has one block per Transformer2DModel; a second one would need FF-out statistics)
        return ops.gemm(h.view(NB, H, W, C), pk["wo"], bias=pk["bo"], residual=x)


# ================================================================================================ conv blocks
class ResnetBlock2D(nn.Module, _Packed):
    def __init__(self, cin, cout, temb_dim, groups):
        nn.Module.__init__(self)
        _Packed.__init__(self)
        self.norm1 = nn.GroupNorm(groups, cin, eps=1e-5)
        self.conv1 = nn.Conv2d(cin, cout, 3, padding=1)
        self.time_emb_proj = nn.Linear(temb_dim, cout)
        self.norm2 = nn.GroupNorm(groups, cout, eps=1e-5)
        self.conv2 = nn.Conv2d(cout, cout, 3, padding=1)
        self.conv_shortcut = nn.Conv2d(cin, cout, 1) if cin != cout else None
        self.groups = groups
        self.cout = cout
        self.temb_offset = 0  # column offset into the concatenated time_emb_proj output (set by the owner)

    def _apply(self, fn, *a, **k):
        self._invalidate()
        return super()._apply(fn, *a, **k)

    def _packed(self):
        if self._pk is None:
            pk = dict(gn1=(_f32(self.norm1.weight), _f32(self.norm1.bias)), w1=pack_conv3x3(self.conv1.weight),
                      b1=_f32(self.conv1.bias), gn2=(_f32(self.norm2.weight), _f32(self.norm2.bias)),
                      w2=pack_conv3x3(self.conv2.weight), b2=_f32(self.conv2.bias))
            if self.conv_shortcut is not None:
                co, ci = self.conv_shortcut.weight.shape[:2]
                pk["ws"] = _bf(self.conv_shortcut.weight.reshape(co, ci))
                pk["bs"] = _f32(self.conv_shortcut.bias)
            self._pk = pk
        return self._pk

    def run(self, x: torch.Tensor, temb_all: torch.Tensor) -> torch.Tensor:
        """h = conv1(silu(gn(x))) + time_emb_proj(silu(temb)); out = shortcut(x) + conv2(silu(gn(h)))."""
        pk = self._packed()
        h = ops.groupnorm(x, *pk["gn1"], self.groups, 1e-5, silu=True)
        h = ops.conv3x3(h, pk["w1"], bias=pk["b1"], rowvec=temb_all[:, self.temb_offset:self.temb_offset + self.cout])
        h = ops.groupnorm(h, *pk["gn2"], self.groups, 1e-5, silu=True)
        sc = x if self.conv_shortcut is None else ops.gemm(x, pk["ws"], bias=pk["bs"])
        return ops.conv3x3(h, pk["w2"], bias=pk["b2"], residual=sc)


class Downsample2D(nn.Module, _Packed):
    def __init__(self, c):
        nn.Module.__init__(self)
        _Packed.__init__(self)
        self.conv = nn.Conv2d(c, c, 3, stride=2, padding=1)

    def _apply(self, fn, *a, **k):
        self._invalidate()
        return super()._apply(fn, *a, **k)

    def run(self, x):
        if self._pk is None:
            self._pk = dict(w=pack_conv3x3(self.conv.weight), b=_f32(self.conv.bias))
        NB, H, W, C = x.shape
        col = ops.im2col3x3_s2(x)
        return ops.gemm(col, self._pk["w"], bias=self._pk["b"])  # [NB, H/2, W/2, C]


class Upsample2D(nn.Module, _Packed):
    def __init__(self, c):
        nn.Module.__init__(self)
        _Packed.__init__(self)
        self.conv = nn.Conv2d(c, c, 3, padding=1)

    def _apply(self, fn, *a, **k):
        self._invalidate()
        return super()._apply(fn, *a, **k)

    def run(self, x):
        if self._pk is None:
            self._pk = dict(w=pack_conv3x3(self.conv.weight), b=_f32(self.conv.bias))
            if UPCONV_PHASE and x.shape[-1] % 64 == 0:
                self._pk["wp"] = pack_upconv3x3(self.conv.weight)
        if "wp" in self._pk and UPCONV_PHASE:
            return ops.upconv3x3(x, self._pk["wp"], bias=self._pk["b"])
        return ops.conv3x3(ops.upsample2x(x), self._pk["w"], bias=self._pk["b"])


class DownBlock(nn.Module):
    def __init__(self, cin, cout, temb, groups, layers, attn, heads, cross, downsample):
        super().__init__()
        if attn:
            self.attentions = nn.ModuleList([Transformer2DModel(cout, heads, cross, groups) for _ in range(layers)])
        self.resnets = nn.ModuleList([ResnetBlock2D(cin if i == 0 else cout, cout, temb, groups) for i in range(layers)])
        self.has_attn = attn
        if downsample:
            self.downsamplers = nn.ModuleList([Downsample2D(cout)])
        self.has_down = downsample

    def run(self, x, temb_all, ctx, kw, adapter_res=None):
        """adapter_res: (feature [n_src, h, w, C] bf16, device fp32 scale) of a T2I-Adapter, added in place to the output of
        the last (resnet, attention) pair before the downsampler, so it reaches both the skip and the onward path."""
        outs = []
        for i, res in enumerate(self.resnets):
            x = res.run(x, temb_all)
            if self.has_attn:
                x = self.attentions[i].run(x, ctx, kw)
            if adapter_res is not None and i == len(self.resnets) - 1:
                ops.scaled_add_bcast(x, *adapter_res)
            outs.append(x)
        if self.has_down:
            x = self.downsamplers[0].run(x)
            outs.append(x)
        return x, outs


class MidBlock(nn.Module):
    def __init__(self, c, temb, groups, heads, cross):
        super().__init__()
        self.attentions = nn.ModuleList([Transformer2DModel(c, heads, cross, groups)])
        self.resnets = nn.ModuleList([ResnetBlock2D(c, c, temb, groups), ResnetBlock2D(c, c, temb, groups)])

    def run(self, x, temb_all, ctx, kw):
        x = self.resnets[0].run(x, temb_all)
        x = self.attentions[0].run(x, ctx, kw)
        return self.resnets[1].run(x, temb_all)


class UpBlock(nn.Module):
    def __init__(self, cin, cout, prev, temb, groups, layers, attn, heads, cross, upsample):
        super().__init__()
        if attn:
            self.attentions = nn.ModuleList([Transformer2DModel(cout, heads, cross, groups) for _ in range(layers)])
        rs = []
        for i in range(layers):
            skip = cin if i == layers - 1 else cout
            inp = prev if i == 0 else cout
            rs.append(ResnetBlock2D(inp + skip, cout, temb, groups))
        self.resnets = nn.ModuleList(rs)
        self.has_attn = attn
        if upsample:
            self.upsamplers = nn.ModuleList([Upsample2D(cout)])
        self.has_up = upsample

    def run(self, x, skips: List[torch.Tensor], skip_res: Optional[List[torch.Tensor]], temb_all, ctx, kw):
        for i, res in enumerate(self.resnets):
            skip = skips.pop()
            r = skip_res.pop() if skip_res is not None else None
            # torch.cat([hidden, skip], 1) with the ControlNet residual folded into the skip half
            x = res.run(ops.concat_add(x, skip, res_b=r), temb_all)
            if self.has_attn:
                x = self.attentions[i].run(x, ctx, kw)
        if self.has_up:
            x = self.upsamplers[0].run(x)
        return x


class TimestepEmbedding(nn.Module):
    def __init__(self, cin, dim):
        super().__init__()
        self.linear_1 = nn.Linear(cin, dim)
        self.linear_2 = nn.Linear(dim, dim)


# ================================================================================================ model base
class _ModelBase(nn.Module):
    """Shared by UNet2DConditionModel and ControlNetModel: processor registry, time conditioning, dtype/device."""

    config: FrozenConfig

    # ---- registration API (inference_IMAGdressing.py:70,85,93-94; IMAGDressing_v1_pipeline.py:343,477)
    @property
    def attn_processors(self) -> Dict[str, object]:
        procs: Dict[str, object] = {}

        def walk(name, module):
            if hasattr(module, "get_processor"):
                procs[f"{name}.processor"] = module.get_processor(return_deprecated_lora=True)
            for sub, child in module.named_children():
                walk(f"{name}.{sub}", child)

        for name, module in self.named_children():
            walk(name, module)
        return procs

    def set_attn_processor(self, processor, _remove_lora: bool = False):
        count = len(self.attn_processors.keys())
        if isinstance(processor, dict) and len(processor) != count:
            raise ValueError(
                f"A dict of processors was passed, but the number of processors {len(processor)} does not match the"
                f" number of attention layers: {count}. Please make sure to pass {count} processor classes.")
        processor = dict(processor) if isinstance(processor, dict) else processor

        def walk(name, module):
            if hasattr(module, "set_processor"):
                if not isinstance(processor, dict):
                    module.set_processor(processor)
                else:
                    module.set_processor(processor.pop(f"{name}.processor"))
            for sub, child in module.named_children():
                if sub != "processor":
                    walk(f"{name}.{sub}", child)

        for name, module in self.named_children():
            walk(name, module)

    # ---- torch-module conveniences the scripts use
    @property
    def dtype(self) -> torch.dtype:
        return next(self.parameters()).dtype

    @property
    def device(self) -> torch.device:
        return next(self.parameters()).device

    @property
    def in_channels(self):
        return self.config.in_channels

    def _apply(self, fn, *a, **k):
        self._time_pk = None
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, state_dict, strict: bool = True, **kw):
        out = super().load_state_dict(state_dict, strict=strict, **kw)
        self.invalidate_packed()
        return out

    def invalidate_packed(self):
        self._time_pk = None
        for m in self.modules():
            if isinstance(m, _Packed):
                m._invalidate()
            if isinstance(m, Attention):
                m.invalidate_packed()
            proc = getattr(m, "processor", None)
            if hasattr(proc, "invalidate_packed"):
                proc.invalidate_packed()

    @classmethod
    def from_config(cls, config=None, **kw):
        return cls(**{**(config or {}), **kw})

    @classmethod
    def from_pretrained(cls, path, subfolder: Optional[str] = None, torch_dtype=None, allow_random_init: bool = False,
                        **kw):
        """Local directory with config.json + diffusion_pytorch_model{,.fp16}.safetensors (or .bin). Offline only.
        A directory without a weight file raises FileNotFoundError — a silently random-initialised UNet samples noise —
        unless `allow_random_init=True` (synthetic-weight tests / benchmarks)."""
        import json
        import os

        d = os.path.join(path, subfolder) if subfolder else path
        if not os.path.isdir(d):
            raise FileNotFoundError(f"{cls.__name__}.from_pretrained: no such directory {d!r} (offline: local paths only)")
        cfg = {}
        cj = os.path.join(d, "config.json")
        if os.path.exists(cj):
            raw = json.load(open(cj))
            cfg = {k: (tuple(v) if isinstance(v, list) else v) for k, v in raw.items() if k in SD15_CONFIG}
        with skip_default_init():
            model = cls(**cfg)
        loaded = False
        for fn in ("diffusion_pytorch_model.safetensors", "diffusion_pytorch_model.fp16.safetensors",
                   "diffusion_pytorch_model.bin", "diffusion_pytorch_model.fp16.bin"):
            fp = os.path.join(d, fn)
            if os.path.exists(fp):
                if fn.endswith(".safetensors"):
                    from safetensors.torch import load_file

                    sd = load_file(fp)
                else:
                    sd = torch.load(fp, map_location="cpu", weights_only=True)
                model.load_state_dict(sd)
                loaded = True
                break
        if not loaded:
            if not allow_random_init:
                raise FileNotFoundError(f"{cls.__name__}.from_pretrained: no diffusion_pytorch_model(.fp16).safetensors / "
                                        f".bin under {d!r}; pass allow_random_init=True for synthetic weights")
            for mod in model.modules():  # skip_default_init left torch.empty parameters
                if isinstance(mod, (nn.Linear, nn.Conv2d)):
                    mod.reset_parameters()
        if torch_dtype is not None:
            model = model.to(dtype=torch_dtype)
        return model

    # ---- time conditioning
    def _resnets(self) -> List[ResnetBlock2D]:
        return [m for m in self.modules() if isinstance(m, ResnetBlock2D)]

    def _time_packed(self):
        if getattr(self, "_time_pk", None) is None:
            res = self._resnets()
            off = 0
            ws, bs = [], []
            for r in res:
                r.temb_offset = off
                off += r.cout
                ws.append(r.time_emb_proj.weight)
                bs.append(r.time_emb_proj.bias)
            te = self.time_embedding
            self._time_pk = dict(w1=_bf(te.linear_1.weight), b1=_f32(te.linear_1.bias), w2=_bf(te.linear_2.weight),
                                 b2=_f32(te.linear_2.bias), wp=_bf(torch.cat([w.detach() for w in ws], 0)),
                                 bp=_f32(torch.cat([b.detach() for b in bs], 0)))
        return self._time_pk

    def time_conditioning(self, NB: int, timestep, device, timestep_table=None) -> torch.Tensor:
        """sinusoid(320) -> linear -> SiLU -> linear = temb[NB,1280]; then EVERY ResnetBlock2D.time_emb_proj in
        one weight-streaming pass: [NB, sum(Cout)] fp32, sliced per block by column offset."""
        pk = self._time_packed()
        dim = self.config.block_out_channels[0]
        if timestep_table is not None:
            table, step_ptr = timestep_table
            emb = ops.timestep_embedding(table, step_ptr, NB, dim)
        else:
            if not torch.is_tensor(timestep):
                timestep = torch.tensor([float(timestep)], device=device, dtype=torch.float32)
            t = timestep.reshape(-1).to(device=device, dtype=torch.float32)
            if t.numel() == 1:
                emb = ops.timestep_embedding(t, None, NB, dim)
            else:
                assert t.numel() == NB, "per-sample timesteps must match the batch"
                emb = torch.cat([ops.timestep_embedding(t[i:i + 1], None, 1, dim) for i in range(NB)], 0)
        temb = ops.linear_small_m(emb, pk["w1"], pk["b1"], act_out=ACT_SILU)
        temb = ops.linear_small_m(temb, pk["w2"], pk["b2"])
        return ops.linear_small_m(temb, pk["wp"], pk["bp"], act_in=ACT_SILU)

    @staticmethod
    def _ctx(encoder_hidden_states: torch.Tensor) -> torch.Tensor:
        return encoder_hidden_states.to(BF16).contiguous()


def _to_tokens(sample: torch.Tensor, repeat: int = 1, input_scale=None, step_ptr=None) -> torch.Tensor:
    """[N, C, H, W] (any float dtype) -> bf16 [N*repeat, H, W, C] via the layout kernel. input_scale: fp32 device table
    of the sampler's model-input scale, read at step_ptr[0] (scale_model_input of the sigma-space schedulers)."""
    if input_scale is not None:
        return ops.nchw_f32_to_nhwc_bf16_scaled(sample.float().contiguous(), input_scale, step_ptr, repeat=repeat)
    return ops.nchw_f32_to_nhwc_bf16(sample.float().contiguous(), repeat=repeat)


# ================================================================================================ UNet
class UNet2DConditionModel(_ModelBase):
    def __init__(self, **overrides):
        super().__init__()
        cfg = FrozenConfig({**SD15_CONFIG, **overrides})
        self.config = cfg
        boc = tuple(cfg.block_out_channels)
        temb = boc[0] * 4
        g, heads, cross, layers = cfg.norm_num_groups, cfg.attention_head_dim, cfg.cross_attention_dim, cfg.layers_per_block
        self.conv_in = nn.Conv2d(cfg.in_channels, boc[0], 3, padding=1)
        self.time_embedding = TimestepEmbedding(boc[0], temb)
        self.down_blocks = nn.ModuleList([])
        self.up_blocks = nn.ModuleList([])  # registered before mid_block: attn_processors order = down, up, mid
        out = boc[0]
        for i, c in enumerate(boc):
            inp, out = out, c
            self.down_blocks.append(DownBlock(inp, out, temb, g, layers, "CrossAttn" in cfg.down_block_types[i], heads,
                                              cross, i < len(boc) - 1))
        self.mid_block = MidBlock(boc[-1], temb, g, heads, cross)
        rev = list(reversed(boc))
        out = rev[0]
        for i, c in enumerate(rev):
            prev, out = out, c
            inp = rev[min(i + 1, len(boc) - 1)]
            self.up_blocks.append(UpBlock(inp, out, prev, temb, g, layers + 1, "CrossAttn" in cfg.up_block_types[i], heads,
                                          cross, i < len(boc) - 1))
        self.conv_norm_out = nn.GroupNorm(g, boc[0], eps=1e-5)
        self.conv_out = nn.Conv2d(boc[0], cfg.out_channels, 3, padding=1)
        self._io_pk = None
        self._time_pk = None
        self._unit_scale = None

    def _apply(self, fn, *a, **k):
        self._io_pk = None
        return super()._apply(fn, *a, **k)

    def invalidate_packed(self):
        self._io_pk = None
        super().invalidate_packed()

    def adapter_tokens(self, features, hw) -> List[torch.Tensor]:
        """T2I-Adapter features -> one bf16 [n_src, h, w, C] tensor per down block for a latent of size hw: accepts the
        token-major bf16 output of T2IAdapter.forward_tokens and NCHW tensors ([C, h, w] is one sample)."""
        boc = self.config.block_out_channels
        if len(features) != len(boc):
            raise ValueError(f"{len(features)} adapter features for {len(boc)} down blocks")
        out = []
        for k, r in enumerate(features):
            h, w, C = hw[0] >> k, hw[1] >> k, boc[k]
            if r.dtype == BF16 and r.dim() == 4 and tuple(r.shape[1:]) == (h, w, C):
                out.append(r.contiguous())
                continue
            r = r[None] if r.dim() == 3 else r
            if r.dim() != 4 or tuple(r.shape[1:]) != (C, h, w):
                raise ValueError(f"adapter feature {k} of shape {tuple(r.shape)} does not match [n, {C}, {h}, {w}]")
            out.append(ops.nchw_f32_to_nhwc_bf16(r.float().contiguous()))
        return out

    def _io_packed(self):
        if self._io_pk is None:
            self._io_pk = dict(wi=pack_conv3x3(self.conv_in.weight), bi=_f32(self.conv_in.bias),
                               gn=(_f32(self.conv_norm_out.weight), _f32(self.conv_norm_out.bias)),
                               wo=pack_conv3x3(self.conv_out.weight), bo=_f32(self.conv_out.bias))
        return self._io_pk

    def forward(self, sample, timestep, encoder_hidden_states, class_labels=None, timestep_cond=None,
                attention_mask=None, cross_attention_kwargs=None, added_cond_kwargs=None,
                down_block_additional_residuals=None, mid_block_additional_residual=None,
                down_intrablock_additional_residuals=None,
                encoder_attention_mask=None, return_dict: bool = True, timestep_table=None, out=None):
        """eps = UNet(sample [N,4,h,w], t, text [N,77|81,768]); returns (eps [N,4,h,w] in sample.dtype,).
        ControlNet residuals may be token-major bf16 tensors (from our ControlNetModel) or NCHW tensors, and so may the
        four T2I-Adapter features of down_intrablock_additional_residuals (batch N, or 1 broadcast over N)."""
        if getattr(self, "_train_path", False) and torch.is_grad_enabled():
            # training step (SURVEY.md 8 row a13; reference train.py:259-264,272-279): autograd operators, no CUDA graph
            if down_block_additional_residuals is not None or mid_block_additional_residual is not None:
                raise NotImplementedError("the reference's training step has no ControlNet (train.py:255-281)")
            if down_intrablock_additional_residuals is not None:
                raise NotImplementedError("adapter residuals under autograd: the training step has no T2I-Adapter")
            from .train import unet_forward_train

            eps32 = unet_forward_train(self, sample, timestep, encoder_hidden_states, cross_attention_kwargs)
            res = eps32 if sample.dtype == torch.float32 else eps32.to(sample.dtype)
            return (res,) if not return_dict else UNet2DConditionOutput(sample=res)
        adapter_res = adapter_scale = None
        if down_intrablock_additional_residuals is not None:
            adapter_res = self.adapter_tokens(down_intrablock_additional_residuals, sample.shape[-2:])
            if self._unit_scale is None or self._unit_scale.device != sample.device:
                self._unit_scale = torch.ones(1, device=sample.device, dtype=torch.float32)
            adapter_scale = self._unit_scale
        eps32 = self.forward_tokens(sample, timestep, encoder_hidden_states, cross_attention_kwargs,
                                    down_block_additional_residuals, mid_block_additional_residual,
                                    timestep_table=timestep_table, out=out, adapter_res=adapter_res,
                                    adapter_scale=adapter_scale)
        res = eps32 if sample.dtype == torch.float32 else eps32.to(sample.dtype)
        if not return_dict:
            return (res,)
        return UNet2DConditionOutput(sample=res)

    @torch.no_grad()
    def forward_tokens(self, sample, timestep, encoder_hidden_states, cross_attention_kwargs=None,
                       down_res=None, mid_res=None, timestep_table=None, out=None, sample_repeat: int = 1,
                       input_scale=None, adapter_res=None, adapter_scale=None) -> torch.Tensor:
        """The hot path. Returns eps as fp32 NCHW (written by the conv_out kernel). sample_repeat=2 evaluates the
        CFG-duplicated batch [sample, sample] without materialising the duplicate. input_scale: per-step fp32 table of
        the model-input scale, indexed by the step pointer of `timestep_table`. adapter_res: one bf16 [n_src, h, w, C]
        T2I-Adapter feature per down block (n_src divides the batch; sample s reads feature s % n_src), each added
        times the device fp32 scalar `adapter_scale` (adapter_tokens)."""
        kw = cross_attention_kwargs or {}
        pk = self._io_packed()
        NB = sample.shape[0] * sample_repeat
        ctx = self._ctx(encoder_hidden_states)
        temb_all = self.time_conditioning(NB, timestep, sample.device, timestep_table)
        step_ptr = timestep_table[1] if timestep_table is not None else None
        x = ops.conv3x3_direct(_to_tokens(sample, sample_repeat, input_scale, step_ptr), pk["wi"], pk["bi"])
        skips = [x]
        if adapter_res is not None and len(adapter_res) != len(self.down_blocks):
            raise ValueError(f"{len(adapter_res)} adapter features for {len(self.down_blocks)} down blocks")
        for k, blk in enumerate(self.down_blocks):
            x, outs = blk.run(x, temb_all, ctx, kw, None if adapter_res is None else (adapter_res[k], adapter_scale))
            skips += outs
        skip_res = None
        if down_res is not None:
            skip_res = [_as_tokens_bf16(r, s) for r, s in zip(down_res, skips)]
        x = self.mid_block.run(x, temb_all, ctx, kw)
        if mid_res is not None:
            x = ops.concat_add(x, None, res_a=_as_tokens_bf16(mid_res, x))
        for blk in self.up_blocks:
            x = blk.run(x, skips, skip_res, temb_all, ctx, kw)
        x = ops.groupnorm(x, *pk["gn"], self.config.norm_num_groups, 1e-5, silu=True)
        return ops.conv3x3_direct(x, pk["wo"], pk["bo"], out_nchw_f32=True, out=out)


class UNet2DConditionOutput:
    def __init__(self, sample):
        self.sample = sample

    def __getitem__(self, i):
        return (self.sample,)[i]


def _as_tokens_bf16(r: torch.Tensor, like: torch.Tensor) -> torch.Tensor:
    """ControlNet residual -> bf16 [N,H,W,C] matching `like`; accepts our token-major tensors, NCHW, and the
    reference's batch-stripped [C,H,W] (IMAGDressing_v1_pipeline_ipa_controlnet.py:662-666, SURVEY.md B6)."""
    NB, H, W, C = like.shape
    if r.dtype == BF16 and r.shape == like.shape:
        return r.contiguous()
    if r.dim() == 3:
        r = r.unsqueeze(0)
    if r.shape[1] == C and r.shape[-2:] == (H, W):
        t = ops.nchw_f32_to_nhwc_bf16(r.float().contiguous())
        return t.expand(NB, -1, -1, -1).contiguous() if t.shape[0] != NB else t
    raise ValueError(f"ControlNet residual shape {tuple(r.shape)} does not match {tuple(like.shape)}")


# ================================================================================================ ControlNet
class ControlNetConditioningEmbedding(nn.Module):
    def __init__(self, out_ch, cond_ch=3, chans=(16, 32, 96, 256)):
        super().__init__()
        self.conv_in = nn.Conv2d(cond_ch, chans[0], 3, padding=1)
        self.blocks = nn.ModuleList([])
        for i in range(len(chans) - 1):
            self.blocks.append(nn.Conv2d(chans[i], chans[i], 3, padding=1))
            self.blocks.append(nn.Conv2d(chans[i], chans[i + 1], 3, padding=1, stride=2))
        self.conv_out = nn.Conv2d(chans[-1], out_ch, 3, padding=1)


class ControlNetModel(_ModelBase):
    """diffusers-0.24 ControlNetModel (v1.1, SD1.5): conditioning embedding + encoder half + mid + 13 1x1 convs
    (SURVEY.md A.3). Returns token-major bf16 residuals that UNet2DConditionModel folds into its skip concat."""

    def __init__(self, **overrides):
        super().__init__()
        cfg = FrozenConfig({**SD15_CONFIG, **overrides})
        self.config = cfg
        boc = tuple(cfg.block_out_channels)
        temb = boc[0] * 4
        g, heads, cross, layers = cfg.norm_num_groups, cfg.attention_head_dim, cfg.cross_attention_dim, cfg.layers_per_block
        self.conv_in = nn.Conv2d(cfg.in_channels, boc[0], 3, padding=1)
        self.time_embedding = TimestepEmbedding(boc[0], temb)
        self.controlnet_cond_embedding = ControlNetConditioningEmbedding(boc[0])
        self.down_blocks = nn.ModuleList([])
        self.controlnet_down_blocks = nn.ModuleList([nn.Conv2d(boc[0], boc[0], 1)])
        out = boc[0]
        for i, c in enumerate(boc):
            inp, out = out, c
            last = i == len(boc) - 1
            self.down_blocks.append(DownBlock(inp, out, temb, g, layers, "CrossAttn" in cfg.down_block_types[i], heads,
                                              cross, not last))
            for _ in range(layers + (0 if last else 1)):
                self.controlnet_down_blocks.append(nn.Conv2d(out, out, 1))
        self.controlnet_mid_block = nn.Conv2d(boc[-1], boc[-1], 1)
        self.mid_block = MidBlock(boc[-1], temb, g, heads, cross)
        self._cn_pk = None
        self._time_pk = None
        self._cond_cache = None

    def _apply(self, fn, *a, **k):
        self._cn_pk = None
        self._cond_cache = None
        return super()._apply(fn, *a, **k)

    def invalidate_packed(self):
        self._cn_pk = None
        self._cond_cache = None
        super().invalidate_packed()

    def _cn_packed(self):
        if self._cn_pk is None:
            ce = self.controlnet_cond_embedding
            convs = [ce.conv_in] + list(ce.blocks) + [ce.conv_out]
            self._cn_pk = dict(
                wi=pack_conv3x3(self.conv_in.weight), bi=_f32(self.conv_in.bias),
                ce=[(pack_conv3x3(c.weight), _f32(c.bias), c.stride[0]) for c in convs],
                zw=[_bf(c.weight.reshape(c.weight.shape[0], -1)) for c in self.controlnet_down_blocks],
                zb=[_f32(c.bias) for c in self.controlnet_down_blocks],
                mw=_bf(self.controlnet_mid_block.weight.reshape(self.controlnet_mid_block.weight.shape[0], -1)),
                mb=_f32(self.controlnet_mid_block.bias))
        return self._cn_pk

    def cond_embedding(self, controlnet_cond: torch.Tensor, NB: int) -> torch.Tensor:
        """conv stack 3->16->16->32(s2)->32->96(s2)->96->256(s2)->320, SiLU between (SURVEY.md A.3). The
        conditioning image is constant over the 50 steps, so the result (tiled to the model batch NB) is cached
        per input tensor."""
        key = (controlnet_cond.data_ptr(), controlnet_cond._version, tuple(controlnet_cond.shape), NB)
        if self._cond_cache is not None and self._cond_cache[0] == key and self._cond_cache[2] is controlnet_cond:
            return self._cond_cache[1]
        pk = self._cn_packed()
        x = _to_tokens(controlnet_cond)
        n = len(pk["ce"])
        for i, (w, b, stride) in enumerate(pk["ce"]):
            x = ops.conv3x3_direct(x, w, b, stride=stride, act=ACT_SILU if i < n - 1 else ACT_NONE)
        if x.shape[0] != NB:  # batch-1 (or per-sample) cond against the CFG-duplicated latents (ipa_controlnet.py:476-492)
            x = x.repeat(NB // x.shape[0], 1, 1, 1).contiguous()
        old = self._cond_cache[1] if self._cond_cache is not None else None
        if old is not None and old.shape == x.shape:  # keep the address stable for captured graphs
            old.copy_(x)
            x = old
        self._cond_cache = (key, x, controlnet_cond)
        return x

    @torch.no_grad()
    def forward(self, sample, timestep, encoder_hidden_states, controlnet_cond, conditioning_scale: float = 1.0,
                class_labels=None, timestep_cond=None, attention_mask=None, added_cond_kwargs=None,
                cross_attention_kwargs=None, guess_mode: bool = False, return_dict: bool = True,
                timestep_table=None, sample_repeat: int = 1, input_scale=None, scale_table=None, scale_step=None,
                residuals=None):
        """scale_table / scale_step / residuals: the multi-ControlNet path (MultiControlNetModel, DenoiseEngine). The 13
        zero convs then read their scale on the device from scale_table (an fp32 column view [S, K][:, k]) at row
        scale_step[0] (row 0 without a step pointer) instead of the host float conditioning_scale, and each adds the
        matching residual of `residuals` = (down list, mid) - the previous net's outputs - so the last net of a chain
        returns the sum of all of them, rounded to bf16 once per net."""
        assert not guess_mode, "guess_mode is False in every reference script (SURVEY.md B14)"
        pk = self._cn_packed()
        NB = sample.shape[0] * sample_repeat
        ctx = self._ctx(encoder_hidden_states)
        temb_all = self.time_conditioning(NB, timestep, sample.device, timestep_table)
        cond = self.cond_embedding(controlnet_cond, NB)
        step_ptr = timestep_table[1] if timestep_table is not None else None
        x = ops.conv3x3_direct(_to_tokens(sample, sample_repeat, input_scale, step_ptr), pk["wi"], pk["bi"], add=cond)
        skips = [x]
        for blk in self.down_blocks:
            x, outs = blk.run(x, temb_all, ctx, cross_attention_kwargs or {})
            skips += outs
        x = self.mid_block.run(x, temb_all, ctx, cross_attention_kwargs or {})
        if scale_table is not None:
            prev_down, prev_mid = residuals if residuals is not None else ([None] * len(skips), None)
            tab = dict(scale_table=scale_table, scale_step=scale_step)
            down = [ops.gemm(t, w, bias=b, residual=r, **tab) for t, w, b, r in zip(skips, pk["zw"], pk["zb"], prev_down)]
            mid = ops.gemm(x, pk["mw"], bias=pk["mb"], residual=prev_mid, **tab)
            return (down, mid) if not return_dict else ControlNetOutput(down, mid)
        s = float(conditioning_scale)
        sb = pk.get(("scaled", s))
        if sb is None:  # conditioning_scale folded into the 1x1 "zero conv" epilogues: alpha * acc + (s * bias)
            sb = pk[("scaled", s)] = ([b * s for b in pk["zb"]], pk["mb"] * s)
        down = [ops.gemm(t, w, bias=b, alpha=s) for t, w, b in zip(skips, pk["zw"], sb[0])]
        mid = ops.gemm(x, pk["mw"], bias=sb[1], alpha=s)
        if not return_dict:
            return down, mid
        return ControlNetOutput(down, mid)


class ControlNetOutput:
    def __init__(self, down, mid):
        self.down_block_res_samples = down
        self.mid_block_res_sample = mid

    def __iter__(self):
        return iter((self.down_block_res_samples, self.mid_block_res_sample))


class MultiControlNetModel(nn.Module):
    """diffusers-0.24 MultiControlNetModel (pipelines/controlnet/multicontrolnet.py): several ControlNets in one call,
    their residuals summed. `nets` is a ModuleList, so state_dict keys are `nets.{k}.*` and .to() moves every net.
    Each net's zero convs add the previous net's outputs in their epilogue (ControlNetModel.forward `residuals=`), so
    the sum costs no extra pass; it is rounded to bf16 once per net where diffusers rounds twice (output, then sum)."""

    def __init__(self, controlnets):
        super().__init__()
        nets = list(controlnets)
        if not nets or not all(isinstance(n, ControlNetModel) for n in nets):
            raise ValueError("MultiControlNetModel takes a non-empty list of ControlNetModel")
        if len({id(n) for n in nets}) != len(nets):
            # one module object holds one cached conditioning embedding: two images cannot share it
            raise ValueError("each ControlNetModel object may appear once in a MultiControlNetModel")
        self.nets = nn.ModuleList(nets)

    @property
    def attn_processors(self) -> Dict[str, object]:
        return {f"nets.{k}.{name}": p for k, net in enumerate(self.nets) for name, p in net.attn_processors.items()}

    @property
    def config(self):
        return self.nets[0].config

    @property
    def dtype(self) -> torch.dtype:
        return self.nets[0].dtype

    @property
    def device(self) -> torch.device:
        return self.nets[0].device

    def load_state_dict(self, state_dict, strict: bool = True, **kw):
        out = super().load_state_dict(state_dict, strict=strict, **kw)
        self.invalidate_packed()
        return out

    def invalidate_packed(self):
        for net in self.nets:
            net.invalidate_packed()

    @torch.no_grad()
    def forward(self, sample, timestep, encoder_hidden_states, controlnet_cond: List[torch.Tensor],
                conditioning_scale: List[float], class_labels=None, timestep_cond=None, attention_mask=None,
                added_cond_kwargs=None, cross_attention_kwargs=None, guess_mode: bool = False, return_dict: bool = True,
                timestep_table=None, sample_repeat: int = 1, input_scale=None):
        """Returns the summed (down residuals, mid residual) as diffusers does. The scales are staged into a [1, K]
        device table that the zero convs read."""
        K = len(self.nets)
        if len(controlnet_cond) != K or len(conditioning_scale) != K:
            raise ValueError(f"{len(controlnet_cond)} images and {len(conditioning_scale)} scales for {K} ControlNets")
        table = torch.tensor([[float(s) for s in conditioning_scale]], dtype=torch.float32, device=sample.device)
        res = None
        for k, (net, image) in enumerate(zip(self.nets, controlnet_cond)):
            res = net(sample, timestep, encoder_hidden_states, image, cross_attention_kwargs=cross_attention_kwargs,
                      guess_mode=guess_mode, return_dict=False, timestep_table=timestep_table,
                      sample_repeat=sample_repeat, input_scale=input_scale, scale_table=table[:, k], residuals=res)
        return res


def init_synthetic_(model: nn.Module, seed: int = 0) -> nn.Module:
    """Deterministic synthetic weights (no checkpoints offline; SURVEY.md §8d): each parameter is drawn from a
    generator seeded by (seed, crc32(parameter name)), so any two module trees with the same state_dict keys get
    identical values regardless of registration order. Fan-in scaled N(0, 1/fan_in) for matrices / convs, small
    biases, norm gamma ~ 1 — keeps activations O(1) through the 60-odd layers."""
    import math
    import zlib

    with torch.no_grad():
        for name, p in model.named_parameters():
            g = torch.Generator().manual_seed((seed * 1000003 + zlib.crc32(name.encode())) % (2 ** 63))
            if p.dim() >= 2:
                v = torch.randn(p.shape, generator=g) * (1.0 / math.sqrt(p[0].numel()))
            elif "norm" in name and name.endswith("weight"):
                v = 1.0 + 0.05 * torch.randn(p.shape, generator=g)
            else:
                v = 0.02 * torch.randn(p.shape, generator=g)
            p.copy_(v.to(p.dtype))
    if hasattr(model, "invalidate_packed"):
        model.invalidate_packed()
    return model


def init_synthetic_fast_(model: nn.Module, seed: int = 0) -> nn.Module:
    """Same distribution as init_synthetic_ but drawn with the device generator of wherever the parameters live
    (seconds instead of a minute for 860 M parameters); used by bench.py, where oracle-equal values are not needed."""
    import math
    import zlib

    with torch.no_grad():
        for name, p in model.named_parameters():
            g = torch.Generator(device=p.device).manual_seed((seed * 1000003 + zlib.crc32(name.encode())) % (2 ** 63))
            if p.dim() >= 2:
                p.copy_(torch.randn(p.shape, generator=g, device=p.device) * (1.0 / math.sqrt(p[0].numel())))
            elif "norm" in name and name.endswith("weight"):
                p.copy_(1.0 + 0.05 * torch.randn(p.shape, generator=g, device=p.device))
            else:
                p.copy_(0.02 * torch.randn(p.shape, generator=g, device=p.device))
    if hasattr(model, "invalidate_packed"):
        model.invalidate_packed()
    return model
