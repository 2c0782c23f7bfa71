"""AutoencoderKL (the SD VAE) on the sm_90a kernels — SURVEY.md §8f row 1, the step either side of the denoising loop:

    ref_image_latents = vae.encode(ref_image).latent_dist.mean * 0.18215   dressing_sd/pipelines/IMAGDressing_v1_pipeline.py:454-458
    image             = vae.decode(latents / vae.config.scaling_factor)    :544
    image_latents     = latent_dist.sample(generator) * scaling_factor     IMAGDressing_v1_pipeline_controlnet_inpainting.py (prepare_latents)

Same surface as diffusers-0.24 `AutoencoderKL` for what the reference touches: `from_pretrained`, `.to()`, `.dtype`,
`.device`, `.config.{scaling_factor, block_out_channels, latent_channels}`, `encode(x).latent_dist.{mean, sample(), mode()}`,
`decode(z, return_dict=False, generator=None)`, the diffusers state_dict key names (both the current `to_q / to_k / to_v /
to_out.0` and the deprecated `query / key / value / proj_attn` attention names are accepted on load).

Arithmetic (activations bf16 token-major [N, H, W, C], exactly as modeling.py):
  ResnetBlock2D       GroupNorm+SiLU kernel -> implicit-GEMM conv3x3 (wgmma) x2, 1x1 shortcut GEMM, residual in the epilogue
  Downsample2D        im2col(pad (0,1,0,1)) -> GEMM;     Upsample2D   the four-phase conv on the low-resolution input
  mid-block attention one head of width 512 does not fit the flash kernel's register budget (O alone would be 512 columns), and
                      it runs once per image: S = Q K^T (GEMM, fp32 out), row softmax kernel (fp32 statistics, the
                      reference upcasts too), O = P V as a GEMM against V^T — V^T = W_v X^T comes straight out of a GEMM
                      with the operands swapped, and its bias moves into the out-projection (softmax rows sum to one)
  thin ends           conv_in 3->128 / 4->512 and conv_out 128->3 / 512->8 on the direct-conv kernels; quant_conv folded
                      into the encoder's conv_out at pack time (exact: 1x1 after 3x3); post_quant_conv stays a 1x1.
There is no torch fallback: every op goes through the C ABI.
"""
from __future__ import annotations

import json
import math
import os
from typing import Optional

import torch
import torch.nn as nn

from . import ops
from .modeling import FrozenConfig, _bf, _f32, pack_conv3x3, pack_upconv3x3, skip_default_init

BF16 = torch.bfloat16

VAE_CONFIG = dict(in_channels=3, out_channels=3, latent_channels=4, block_out_channels=(128, 256, 512, 512),
                  layers_per_block=2, norm_num_groups=32, scaling_factor=0.18215, sample_size=512, act_fn="silu",
                  force_upcast=True)
_DEPRECATED_ATTN = {"query": "to_q", "key": "to_k", "value": "to_v", "proj_attn": "to_out.0"}


class _Pk:
    def _apply(self, fn, *a, **k):
        self._pk = None
        return super()._apply(fn, *a, **k)


class ResnetBlock2D(_Pk, nn.Module):
    def __init__(self, cin, cout, groups):
        super().__init__()
        self.norm1 = nn.GroupNorm(groups, cin, eps=1e-6)
        self.conv1 = nn.Conv2d(cin, cout, 3, padding=1)
        self.norm2 = nn.GroupNorm(groups, cout, eps=1e-6)
        self.conv2 = nn.Conv2d(cout, cout, 3, padding=1)
        self.conv_shortcut = nn.Conv2d(cin, cout, 1) if cin != cout else None
        self.groups = groups
        self._pk = None

    def run(self, x):
        if self._pk is None:
            pk = dict(g1=(_f32(self.norm1.weight), _f32(self.norm1.bias)), w1=pack_conv3x3(self.conv1.weight),
                      b1=_f32(self.conv1.bias), g2=(_f32(self.norm2.weight), _f32(self.norm2.bias)),
                      w2=pack_conv3x3(self.conv2.weight), b2=_f32(self.conv2.bias))
            if self.conv_shortcut is not None:
                co, ci = self.conv_shortcut.weight.shape[:2]
                pk["ws"], pk["bs"] = _bf(self.conv_shortcut.weight.reshape(co, ci)), _f32(self.conv_shortcut.bias)
            self._pk = pk
        pk = self._pk
        h = ops.groupnorm(x, *pk["g1"], self.groups, 1e-6, silu=True)
        h = ops.conv3x3(h, pk["w1"], bias=pk["b1"])
        h = ops.groupnorm(h, *pk["g2"], self.groups, 1e-6, silu=True)
        sc = x if self.conv_shortcut is None else ops.gemm(x, pk["ws"], bias=pk["bs"])
        return ops.conv3x3(h, pk["w2"], bias=pk["b2"], residual=sc)


class AttnBlock(_Pk, nn.Module):
    """diffusers-0.24 Attention(_from_deprecated_attn_block=True, heads=1, residual_connection=True, upcast_softmax)."""

    def __init__(self, c, groups):
        super().__init__()
        self.group_norm = nn.GroupNorm(groups, c, eps=1e-6)
        self.to_q, self.to_k, self.to_v = nn.Linear(c, c), nn.Linear(c, c), nn.Linear(c, c)
        self.to_out = nn.ModuleList([nn.Linear(c, c), nn.Dropout(0.0)])
        self.groups = groups
        self._pk = None

    def run(self, x):
        NB, H, W, C = x.shape
        if self._pk is None:
            wo = self.to_out[0].weight.detach().float()
            self._pk = dict(g=(_f32(self.group_norm.weight), _f32(self.group_norm.bias)),
                            wqk=_bf(torch.cat([self.to_q.weight, self.to_k.weight], 0)),
                            bqk=_f32(torch.cat([self.to_q.bias, self.to_k.bias], 0)),
                            wv=_bf(self.to_v.weight), wo=_bf(self.to_out[0].weight),
                            # O = P (V + 1 b_v^T) = P V + b_v^T (rows of P sum to 1): b_v rides in the out-projection bias
                            bo=(wo @ self.to_v.bias.detach().float() + self.to_out[0].bias.detach().float()).contiguous())
        pk = self._pk
        L = H * W
        t = ops.groupnorm(x, *pk["g"], self.groups, 1e-6, silu=False).view(NB, L, C)
        qk = ops.gemm(t, pk["wqk"], bias=pk["bqk"])  # [NB, L, 2C]
        out = torch.empty(NB, L, C, device=x.device, dtype=BF16)
        xr = x.view(NB, L, C)
        s = torch.empty(L, L, device=x.device, dtype=torch.float32)
        prob = torch.empty(L, L, device=x.device, dtype=BF16)
        for n in range(NB):  # once per image, per sample: the L x L score matrix of one sample at a time (64 MB at 512x512)
            q, k = qk[n, :, :C], qk[n, :, C:]
            ops.gemm(q, k, out=s, out_fp32=True)                    # S = Q K^T
            ops.softmax_rows(s, 1.0 / math.sqrt(C), out=prob)       # fp32 statistics (upcast_softmax)
            vt = ops.gemm(pk["wv"], t[n])                           # V^T [C, L] = W_v X^T (bias folded into bo)
            o = ops.gemm(prob, vt)                                  # O = P V
            ops.gemm(o, pk["wo"], bias=pk["bo"], residual=xr[n], out=out[n])
        return out.view(NB, H, W, C)


class MidBlock(nn.Module):
    def __init__(self, c, groups):
        super().__init__()
        self.attentions = nn.ModuleList([AttnBlock(c, groups)])
        self.resnets = nn.ModuleList([ResnetBlock2D(c, c, groups), ResnetBlock2D(c, c, groups)])

    def run(self, x):
        return self.resnets[1].run(self.attentions[0].run(self.resnets[0].run(x)))


class _Sampler(_Pk, nn.Module):
    def __init__(self, c, down):
        super().__init__()
        self.conv = nn.Conv2d(c, c, 3, stride=2 if down else 1, padding=0 if down else 1)
        self.down = down
        self._pk = None

    def run(self, x):
        if self._pk is None:
            self._pk = dict(w=pack_conv3x3(self.conv.weight), b=_f32(self.conv.bias))
            if not self.down:
                self._pk["wp"] = pack_upconv3x3(self.conv.weight)
        if self.down:  # F.pad(x, (0,1,0,1)) + conv stride 2 padding 0
            return ops.gemm(ops.im2col3x3_s2(x, pad_lo=0), self._pk["w"], bias=self._pk["b"])
        return ops.upconv3x3(x, self._pk["wp"], bias=self._pk["b"])  # nearest 2x + conv3x3 as four phase convs


class _Block(nn.Module):
    def __init__(self, cin, cout, groups, layers, sampler: Optional[str]):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(cin if i == 0 else cout, cout, groups) for i in range(layers)])
        if sampler == "down":
            self.downsamplers = nn.ModuleList([_Sampler(cout, True)])
        elif sampler == "up":
            self.upsamplers = nn.ModuleList([_Sampler(cout, False)])
        self.sampler = sampler

    def run(self, x):
        for r in self.resnets:
            x = r.run(x)
        if self.sampler == "down":
            x = self.downsamplers[0].run(x)
        elif self.sampler == "up":
            x = self.upsamplers[0].run(x)
        return x


class Encoder(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        boc, g = tuple(cfg.block_out_channels), cfg.norm_num_groups
        self.conv_in = nn.Conv2d(cfg.in_channels, boc[0], 3, padding=1)
        self.down_blocks = nn.ModuleList([_Block(boc[max(i - 1, 0)], c, g, cfg.layers_per_block,
                                                 "down" if i < len(boc) - 1 else None) for i, c in enumerate(boc)])
        self.mid_block = MidBlock(boc[-1], g)
        self.conv_norm_out = nn.GroupNorm(g, boc[-1], eps=1e-6)
        self.conv_out = nn.Conv2d(boc[-1], 2 * cfg.latent_channels, 3, padding=1)
        self.groups = g


class Decoder(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        boc, g = list(reversed(cfg.block_out_channels)), cfg.norm_num_groups
        self.conv_in = nn.Conv2d(cfg.latent_channels, boc[0], 3, padding=1)
        self.mid_block = MidBlock(boc[0], g)
        self.up_blocks = nn.ModuleList([_Block(boc[max(i - 1, 0)], c, g, cfg.layers_per_block + 1,
                                               "up" if i < len(boc) - 1 else None) for i, c in enumerate(boc)])
        self.conv_norm_out = nn.GroupNorm(g, boc[-1], eps=1e-6)
        self.conv_out = nn.Conv2d(boc[-1], cfg.out_channels, 3, padding=1)
        self.groups = g


class DiagonalGaussianDistribution:
    """mean / logvar (clamped to [-30, 20]) / sample(generator) / mode() of diffusers-0.24."""

    def __init__(self, moments: torch.Tensor):
        self.mean, logvar = moments.chunk(2, dim=1)
        self.logvar = logvar.clamp(-30.0, 20.0)
        self.std = torch.exp(0.5 * self.logvar)
        self.var = torch.exp(self.logvar)

    def sample(self, generator=None):
        from .pipelines import randn_tensor

        noise = randn_tensor(self.mean.shape, generator=generator, device=self.mean.device, dtype=self.mean.dtype)
        return self.mean + self.std * noise

    def mode(self):
        return self.mean


class AutoencoderKLOutput:
    def __init__(self, latent_dist):
        self.latent_dist = latent_dist

    def __getitem__(self, i):
        return (self.latent_dist,)[i]


class DecoderOutput:
    def __init__(self, sample):
        self.sample = sample

    def __getitem__(self, i):
        return (self.sample,)[i]


class AutoencoderKL(nn.Module):
    def __init__(self, **overrides):
        super().__init__()
        self.config = FrozenConfig({**VAE_CONFIG, **{k: v for k, v in overrides.items() if k in VAE_CONFIG}})
        self.encoder = Encoder(self.config)
        self.decoder = Decoder(self.config)
        lc = self.config.latent_channels
        self.quant_conv = nn.Conv2d(2 * lc, 2 * lc, 1)
        self.post_quant_conv = nn.Conv2d(lc, lc, 1)
        self._io = None

    # ---- torch-module conveniences
    @property
    def dtype(self):
        return next(self.parameters()).dtype

    @property
    def device(self):
        return next(self.parameters()).device

    def _apply(self, fn, *a, **k):
        self._io = None
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, state_dict, strict: bool = True, **kw):
        sd = {}
        for k, v in state_dict.items():  # pre-0.18 checkpoints: query/key/value/proj_attn with [C, C, 1, 1] or [C, C]
            parts = k.split(".")
            if "attentions" in parts and len(parts) >= 2 and parts[-2] in _DEPRECATED_ATTN:
                parts[-2:-1] = _DEPRECATED_ATTN[parts[-2]].split(".")
                k = ".".join(parts)
                if v.dim() == 4:
                    v = v[:, :, 0, 0]
            sd[k] = v
        out = super().load_state_dict(sd, strict=strict, **kw)
        self.invalidate_packed()
        return out

    def invalidate_packed(self):
        self._io = None
        for m in self.modules():
            if hasattr(m, "_pk"):
                m._pk = None

    @classmethod
    def from_config(cls, config=None, **kw):
        return cls(**{**(config or {}), **kw})

    @classmethod
    def from_pretrained(cls, path, subfolder: Optional[str] = None, torch_dtype=None, allow_random_init: bool = False, **kw):
        """Local diffusers directory (config.json + diffusion_pytorch_model{,.fp16}.{safetensors,bin}); offline only."""
        d = os.path.join(path, subfolder) if subfolder else path
        if not os.path.isdir(d):
            raise FileNotFoundError(f"AutoencoderKL.from_pretrained: no such directory {d!r} (offline: local paths only)")
        cfg = {}
        cj = os.path.join(d, "config.json")
        if os.path.exists(cj):
            cfg = {k: (tuple(v) if isinstance(v, list) else v) for k, v in json.load(open(cj)).items() if k in VAE_CONFIG}
        with skip_default_init():
            model = cls(**cfg)
        for fn in ("diffusion_pytorch_model.safetensors", "diffusion_pytorch_model.fp16.safetensors",
                   "diffusion_pytorch_model.bin", "diffusion_pytorch_model.fp16.bin"):
            fp = os.path.join(d, fn)
            if os.path.exists(fp):
                if fn.endswith(".safetensors"):
                    from safetensors.torch import load_file

                    model.load_state_dict(load_file(fp))
                else:
                    model.load_state_dict(torch.load(fp, map_location="cpu", weights_only=True))
                break
        else:
            if not allow_random_init:
                raise FileNotFoundError(f"AutoencoderKL.from_pretrained: no diffusion_pytorch_model weights under {d!r}")
            for mod in model.modules():
                if isinstance(mod, (nn.Linear, nn.Conv2d)):
                    mod.reset_parameters()
        return model.to(dtype=torch_dtype) if torch_dtype is not None else model

    # ---- kernel-layout weights of the thin ends
    def _io_packed(self):
        if self._io is None:
            e, d, lc = self.encoder, self.decoder, self.config.latent_channels

            def pad_in(w, cpad):  # [Cout, Cin, 3, 3] -> Cin zero-padded (the layout kernel pads the activation alike)
                co, ci = w.shape[:2]
                wp = torch.zeros(co, cpad, 3, 3, dtype=torch.float32, device=w.device)
                wp[:, :ci] = w.detach().float()
                return pack_conv3x3(wp)

            # quant_conv (1x1) after the encoder's conv_out (3x3): W'[o] = sum_m Wq[o, m] Wc[m], b' = Wq bc + bq (exact)
            wq = self.quant_conv.weight.detach().float()[:, :, 0, 0]
            wc = e.conv_out.weight.detach().float()
            w_eq = torch.einsum("om,mikl->oikl", wq, wc)
            b_eq = wq @ e.conv_out.bias.detach().float() + self.quant_conv.bias.detach().float()
            # post_quant_conv as the centre tap of a 3x3 on the 4-channel latents (cannot be folded into conv_in: the
            # zero padding of conv_in applies AFTER its bias)
            wpq = torch.zeros(lc, lc, 3, 3, dtype=torch.float32, device=wq.device)
            wpq[:, :, 1, 1] = self.post_quant_conv.weight.detach().float()[:, :, 0, 0]
            # conv_out 128 -> 3 padded to 4 output channels for the Cout = 4 warp kernel (fp32 NCHW out, sliced to 3)
            oc = self.config.out_channels
            wdo = torch.zeros(4, d.conv_out.weight.shape[1], 3, 3, dtype=torch.float32, device=wq.device)
            wdo[:oc] = d.conv_out.weight.detach().float()
            bdo = torch.zeros(4, dtype=torch.float32, device=wq.device)
            bdo[:oc] = d.conv_out.bias.detach().float()
            self._io = dict(
                e_in=pad_in(e.conv_in.weight, 4), e_in_b=_f32(e.conv_in.bias),
                e_gn=(_f32(e.conv_norm_out.weight), _f32(e.conv_norm_out.bias)),
                e_out=pack_conv3x3(w_eq), e_out_b=b_eq.contiguous(),
                pq=pack_conv3x3(wpq), pq_b=_f32(self.post_quant_conv.bias),
                d_in=pack_conv3x3(d.conv_in.weight), d_in_b=_f32(d.conv_in.bias),
                d_gn=(_f32(d.conv_norm_out.weight), _f32(d.conv_norm_out.bias)),
                d_out=pack_conv3x3(wdo), d_out_b=bdo.contiguous())
        return self._io

    # ---- the two calls of the reference
    @torch.no_grad()
    def encode(self, x: torch.Tensor, return_dict: bool = True):
        """x [N, 3, H, W] in [-1, 1] (any float dtype) -> latent_dist over [N, 4, H/8, W/8] (fp32 moments)."""
        pk = self._io_packed()
        e = self.encoder
        t = ops.nchw_f32_to_nhwc_bf16(x.float().contiguous(), cpad=4)
        h = ops.conv3x3_direct(t, pk["e_in"], pk["e_in_b"])
        for blk in e.down_blocks:
            h = blk.run(h)
        h = e.mid_block.run(h)
        h = ops.groupnorm(h, *pk["e_gn"], e.groups, 1e-6, silu=True)
        moments = ops.conv3x3_direct(h, pk["e_out"], pk["e_out_b"], out_nchw_f32=True)  # conv_out + quant_conv
        dist = DiagonalGaussianDistribution(moments)
        return AutoencoderKLOutput(dist) if return_dict else (dist,)

    @torch.no_grad()
    def decode(self, z: torch.Tensor, return_dict: bool = True, generator=None):
        """z [N, 4, h, w] (already divided by scaling_factor) -> image [N, 3, 8h, 8w] fp32 in about [-1, 1]."""
        pk = self._io_packed()
        d = self.decoder
        t = ops.nchw_f32_to_nhwc_bf16(z.float().contiguous())
        t = ops.conv3x3_direct(t, pk["pq"], pk["pq_b"])          # post_quant_conv
        h = ops.conv3x3_direct(t, pk["d_in"], pk["d_in_b"])      # conv_in 4 -> 512
        h = d.mid_block.run(h)
        for blk in d.up_blocks:
            h = blk.run(h)
        h = ops.groupnorm(h, *pk["d_gn"], d.groups, 1e-6, silu=True)
        img = ops.conv3x3_direct(h, pk["d_out"], pk["d_out_b"], out_nchw_f32=True)[:, : self.config.out_channels]
        img = img.to(z.dtype) if z.dtype != torch.float32 else img
        return DecoderOutput(img) if return_dict else (img,)

    def forward(self, sample, sample_posterior: bool = False, generator=None):
        dist = self.encode(sample).latent_dist
        return self.decode(dist.sample(generator) if sample_posterior else dist.mode())
