"""Second, independently written restatement of the diffusers-0.24 SD1.5 UNet2DConditionModel / ControlNetModel forward
— TEST INFRASTRUCTURE ONLY (an anchor for oracle/unet.py, VERDICT r1 "next round" item 1b).

Why it exists: `diffusers` is a third-party dependency of the reference (requirements.txt:12, `diffusers==0.24.0`) that
is not installed where the suite runs, so oracle/unet.py cannot be pinned against the real classes
(PARITY UNPINNED for the UNet / ControlNet arithmetic; DESIGN.md section 4). A transcription error shared by
oracle/unet.py and the product's modeling.py (same nn.Module tree, same author) would pass every test that compares
the two. This file removes that shared structure: it is a flat FUNCTION over a plain `state_dict` with the diffusers
key names, written from the architecture description (SURVEY.md Appendix A: block list, skip order, norm epsilons,
time embedding, GEGLU split, zero-conv placement) in NCHW with torch.nn.functional calls only — no module classes, no
processors, no shared helper with oracle/unet.py. tests/test_oracle_anchor_cpu.py requires the two restatements to agree
to fp32 round-off (reduced widths on the CPU; tests/test_oracle_anchor_gpu.py at full SD1.5 widths, 512x512) and pins
per-block activation checksums of this one in tests/golden/unet_functional_checksums.json.

Reference call sites restated: dressing_sd/pipelines/IMAGDressing_v1_pipeline.py:466 (garment pass), :499,:511
(denoising passes), IMAGDressing_v1_pipeline_ipa_controlnet.py:651 (ControlNet). Attention here is plain SDPA
(AttnProcessor2_0) plus, optionally, the RefS garment stream restated from adapter/attention_processor.py:589-612.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F

HEADS = 8
GROUPS = 32


def _gn(sd, key, x, eps):
    return F.group_norm(x, GROUPS, sd[key + ".weight"], sd[key + ".bias"], eps)


def _conv(sd, key, x, stride=1, padding=1):
    return F.conv2d(x, sd[key + ".weight"], sd.get(key + ".bias"), stride=stride, padding=padding)


def _lin(sd, key, x):
    return F.linear(x, sd[key + ".weight"], sd.get(key + ".bias"))


def time_embedding(sd, t: torch.Tensor, batch: int) -> torch.Tensor:
    """Sinusoid [cos | sin] (flip_sin_to_cos=True, downscale_freq_shift=0) of width block_out_channels[0] (320 for
    SD1.5; read off linear_1's input width) -> linear_1 -> SiLU -> linear_2."""
    dim = sd["time_embedding.linear_1.weight"].shape[1]
    t = t.reshape(-1).float().expand(batch) if t.numel() == 1 else t.reshape(-1).float()
    k = torch.arange(dim // 2, dtype=torch.float32, device=t.device)
    ang = t[:, None] * torch.exp(-math.log(10000.0) * k / (dim // 2))[None, :]
    emb = torch.cat([ang.cos(), ang.sin()], dim=1)
    return _lin(sd, "time_embedding.linear_2", F.silu(_lin(sd, "time_embedding.linear_1", emb)))


def resnet(sd, p, x, temb):
    h = _conv(sd, p + ".conv1", F.silu(_gn(sd, p + ".norm1", x, 1e-5)))
    h = h + _lin(sd, p + ".time_emb_proj", F.silu(temb))[:, :, None, None]
    h = _conv(sd, p + ".conv2", F.silu(_gn(sd, p + ".norm2", h, 1e-5)))
    if p + ".conv_shortcut.weight" in sd:
        x = _conv(sd, p + ".conv_shortcut", x, padding=0)
    return x + h


def _sdpa(q, k, v):
    B, L, C = q.shape
    d = C // HEADS
    sp = lambda t: t.reshape(B, -1, HEADS, d).permute(0, 2, 1, 3)
    w = torch.softmax(sp(q) @ sp(k).transpose(-1, -2) / math.sqrt(d), dim=-1)
    return (w @ sp(v)).permute(0, 2, 1, 3).reshape(B, L, C)


def attention(sd, p, x, ctx=None, garment=None, scale=1.0, taps=None):
    """p = '...attn1' | '...attn2'. `garment` = cached garment features for this layer -> RefS stream added with `scale`
    through the processor's to_k_ref / to_v_ref (state_dict keys p + '.processor.to_k_ref.weight')."""
    if taps is not None:
        taps[p + ".processor"] = x
    src = x if ctx is None else ctx
    q = _lin(sd, p + ".to_q", x)
    o = _sdpa(q, _lin(sd, p + ".to_k", src), _lin(sd, p + ".to_v", src))
    if garment is not None:
        o = o + scale * _sdpa(q, _lin(sd, p + ".processor.to_k_ref", garment), _lin(sd, p + ".processor.to_v_ref", garment))
    return _lin(sd, p + ".to_out.0", o)


def transformer(sd, p, x, ctx, garments=None, scale=1.0, taps=None):
    B, C, H, W = x.shape
    h = _conv(sd, p + ".proj_in", _gn(sd, p + ".norm", x, 1e-6), padding=0)
    h = h.permute(0, 2, 3, 1).reshape(B, H * W, C)
    b = p + ".transformer_blocks.0"
    g = None if garments is None else garments.get(b + ".attn1.processor")
    h = h + attention(sd, b + ".attn1", F.layer_norm(h, (C,), sd[b + ".norm1.weight"], sd[b + ".norm1.bias"]), None, g,
                      scale, taps)
    h = h + attention(sd, b + ".attn2", F.layer_norm(h, (C,), sd[b + ".norm2.weight"], sd[b + ".norm2.bias"]), ctx,
                      taps=taps)
    n3 = F.layer_norm(h, (C,), sd[b + ".norm3.weight"], sd[b + ".norm3.bias"])
    val, gate = _lin(sd, b + ".ff.net.0.proj", n3).chunk(2, dim=-1)
    h = h + _lin(sd, b + ".ff.net.2", val * F.gelu(gate))
    h = h.reshape(B, H, W, C).permute(0, 3, 1, 2)
    return _conv(sd, p + ".proj_out", h, padding=0) + x


def encoder(sd, x, temb, ctx, garments, scale, taps, probe):
    """conv_in output + the 12 skip tensors, in creation order."""
    skips = [x]
    for i in range(4):
        for j in range(2):
            x = resnet(sd, f"down_blocks.{i}.resnets.{j}", x, temb)
            if i < 3:
                x = transformer(sd, f"down_blocks.{i}.attentions.{j}", x, ctx, garments, scale, taps)
            skips.append(x)
        if i < 3:
            x = _conv(sd, f"down_blocks.{i}.downsamplers.0.conv", x, stride=2)
            skips.append(x)
        probe(f"down_blocks.{i}", x)
    return x, skips


def middle(sd, x, temb, ctx, garments, scale, taps, probe):
    x = resnet(sd, "mid_block.resnets.0", x, temb)
    x = transformer(sd, "mid_block.attentions.0", x, ctx, garments, scale, taps)
    x = resnet(sd, "mid_block.resnets.1", x, temb)
    probe("mid_block", x)
    return x


def unet_forward(sd: Dict[str, torch.Tensor], sample, t, ctx, garments=None, scale: float = 1.0,
                 down_res: Optional[List[torch.Tensor]] = None, mid_res: Optional[torch.Tensor] = None,
                 taps: Optional[dict] = None, checks: Optional[dict] = None) -> torch.Tensor:
    """eps = UNet(sample [B,4,h,w], t, ctx [B,T,768]). `taps` collects every attention processor's input (what
    CacheAttnProcessor2_0 stores, adapter/attention_processor.py:34); `checks` collects per-block activation sums."""
    def probe(name, v):
        if checks is not None:
            checks[name] = [float(v.double().sum()), float(v.double().abs().sum())]

    temb = time_embedding(sd, t, sample.shape[0])
    x = _conv(sd, "conv_in", sample)
    probe("conv_in", x)
    x, skips = encoder(sd, x, temb, ctx, garments, scale, taps, probe)
    x = middle(sd, x, temb, ctx, garments, scale, taps, probe)
    if down_res is not None:
        skips = [s + r for s, r in zip(skips, down_res)]
        x = x + mid_res
    for i in range(4):
        for j in range(3):
            x = resnet(sd, f"up_blocks.{i}.resnets.{j}", torch.cat([x, skips.pop()], dim=1), temb)
            if i > 0:
                x = transformer(sd, f"up_blocks.{i}.attentions.{j}", x, ctx, garments, scale, taps)
        if i < 3:
            x = _conv(sd, f"up_blocks.{i}.upsamplers.0.conv", F.interpolate(x, scale_factor=2.0, mode="nearest"))
        probe(f"up_blocks.{i}", x)
    out = _conv(sd, "conv_out", F.silu(_gn(sd, "conv_norm_out", x, 1e-5)))
    probe("conv_out", out)
    return out


def controlnet_forward(sd, sample, t, ctx, cond, conditioning_scale: float = 1.0) -> Tuple[List[torch.Tensor], torch.Tensor]:
    """12 down residuals + mid residual (SURVEY.md A.3): cond-embedding conv stack added to conv_in, encoder + mid with
    the ControlNet's own weights, one 1x1 'zero conv' per skip, everything times conditioning_scale."""
    e = "controlnet_cond_embedding"
    c = F.silu(_conv(sd, e + ".conv_in", cond))
    for k in range(6):
        c = F.silu(_conv(sd, f"{e}.blocks.{k}", c, stride=2 if k % 2 else 1))
    c = _conv(sd, e + ".conv_out", c)
    temb = time_embedding(sd, t, sample.shape[0])
    x = _conv(sd, "conv_in", sample) + c
    noprobe = lambda *a: None
    x, skips = encoder(sd, x, temb, ctx, None, 1.0, None, noprobe)
    x = middle(sd, x, temb, ctx, None, 1.0, None, noprobe)
    down = [_conv(sd, f"controlnet_down_blocks.{i}", s, padding=0) * conditioning_scale for i, s in enumerate(skips)]
    return down, _conv(sd, "controlnet_mid_block", x, padding=0) * conditioning_scale
