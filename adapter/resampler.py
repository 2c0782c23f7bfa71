"""Drop-in for the reference's `adapter/resampler.py`: `Resampler` (the garment `ImgProj`,
inference_IMAGdressing.py:55-65) and `ProjPlusModel` (FaceID-Plus projector,
IMAGDressing_v1_pipeline_ipa_controlnet.py:79-86) with the reference's constructor arguments and state_dict keys,
executing on the sm_90a kernels: LayerNorm kernel, wgmma GEMMs (GELU / residual epilogues) and the same
attention kernel as the UNet (16 or 4 latent queries against 257 CLIP tokens + the latents, 64-wide heads;
`(q d^-1/4)(k d^-1/4)^T` == `q k^T / sqrt(d)`, softmax statistics in fp32 — adapter/resampler.py:62-78).
"""
from __future__ import annotations

import torch
import torch.nn as nn

from imagdressing_b200 import ops
from imagdressing_b200._lib import ACT_GELU, ACT_NONE

BF16 = torch.bfloat16


def FeedForward(dim, mult=4):
    """adapter/resampler.py:13-20 (parameter container; keys 0.weight/0.bias, 1.weight, 3.weight)."""
    inner_dim = int(dim * mult)
    return nn.Sequential(nn.LayerNorm(dim), nn.Linear(dim, inner_dim, bias=False), nn.GELU(),
                         nn.Linear(inner_dim, dim, bias=False))


class PerceiverAttention(nn.Module):
    """adapter/resampler.py:34-78."""

    def __init__(self, *, dim, dim_head=64, heads=8):
        super().__init__()
        self.scale = dim_head ** -0.5
        self.dim_head = dim_head
        self.heads = heads
        inner_dim = dim_head * heads
        self.norm1 = nn.LayerNorm(dim)
        self.norm2 = nn.LayerNorm(dim)
        self.to_q = nn.Linear(dim, inner_dim, bias=False)
        self.to_kv = nn.Linear(dim, inner_dim * 2, bias=False)
        self.to_out = nn.Linear(inner_dim, dim, bias=False)


def _f32(p):
    return p.detach().float().contiguous()


def _bf(p):
    return p.detach().to(BF16).contiguous()


class _PerceiverStack(nn.Module):
    """`layers` = [PerceiverAttention, FeedForward] x depth + proj_in / proj_out / norm_out, run on the kernels."""

    def _build(self, dim, depth, dim_head, heads, embedding_dim, output_dim, ff_mult):
        self.proj_in = nn.Linear(embedding_dim, dim)
        self.proj_out = nn.Linear(dim, output_dim)
        self.norm_out = nn.LayerNorm(output_dim)
        self.layers = nn.ModuleList([])
        for _ in range(depth):
            self.layers.append(nn.ModuleList([PerceiverAttention(dim=dim, dim_head=dim_head, heads=heads),
                                              FeedForward(dim=dim, mult=ff_mult)]))
        self._pk = None

    def _apply(self, fn, *a, **k):
        self._pk = None
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, *a, **k):
        self._pk = None
        return super().load_state_dict(*a, **k)

    def _packed(self):
        if self._pk is None:
            ls = []
            for attn, ff in self.layers:
                ls.append(dict(n1=(_f32(attn.norm1.weight), _f32(attn.norm1.bias)),
                               n2=(_f32(attn.norm2.weight), _f32(attn.norm2.bias)), wq=_bf(attn.to_q.weight),
                               wkv=_bf(attn.to_kv.weight), wo=_bf(attn.to_out.weight),
                               fn=(_f32(ff[0].weight), _f32(ff[0].bias)), w1=_bf(ff[1].weight), w2=_bf(ff[3].weight),
                               heads=attn.heads, dh=attn.dim_head))
            self._pk = dict(layers=ls, wi=_bf(self.proj_in.weight), bi=_f32(self.proj_in.bias),
                            wo=_bf(self.proj_out.weight), bo=_f32(self.proj_out.bias),
                            no=(_f32(self.norm_out.weight), _f32(self.norm_out.bias)))
        return self._pk

    @torch.no_grad()
    def _run_stack(self, x: torch.Tensor, latents: torch.Tensor) -> torch.Tensor:
        """x: [B, n1, embedding_dim], latents: [B, n2, dim] (bf16). Returns [B, n2, output_dim] bf16."""
        pk = self._packed()
        B, n1, _ = x.shape
        n2, D = latents.shape[1], latents.shape[2]
        x = ops.gemm(x.contiguous(), pk["wi"], bias=pk["bi"])  # proj_in
        for L in pk["layers"]:
            inner = L["heads"] * L["dh"]
            xn = ops.layernorm(x, *L["n1"])
            ln = ops.layernorm(latents, *L["n2"])
            q = ops.gemm(ln, L["wq"])  # [B, n2, inner]
            kv = torch.empty(B, n1 + n2, 2 * inner, device=x.device, dtype=BF16)  # to_kv(cat(x, latents))
            for b in range(B):
                ops.gemm(xn[b], L["wkv"], out=kv[b, :n1])
                ops.gemm(ln[b], L["wkv"], out=kv[b, n1:])
            kv2 = kv.view(B * (n1 + n2), 2 * inner)
            s0 = ops.kv_stream(kv2[:, :inner], kv2[:, inner:], n1 + n2)
            o = ops.attention(q.view(B * n2, inner), B, n2, L["heads"], L["dh"], s0)
            latents = ops.gemm(o.view(B, n2, inner), L["wo"], residual=latents)  # attn(x, latents) + latents
            h = ops.gemm(ops.layernorm(latents, *L["fn"]), L["w1"], act=ACT_GELU)
            latents = ops.gemm(h, L["w2"], residual=latents)  # ff(latents) + latents
        out = ops.gemm(latents, pk["wo"], bias=pk["bo"])
        return ops.layernorm(out, *pk["no"])


class Resampler(_PerceiverStack):
    """adapter/resampler.py:170-236 (apply_pos_emb / num_latents_mean_pooled are unused by the reference scripts)."""

    def __init__(self, dim=1024, depth=8, dim_head=64, heads=16, num_queries=8, embedding_dim=768, output_dim=1024,
                 ff_mult=4, max_seq_len: int = 257, apply_pos_emb: bool = False, num_latents_mean_pooled: int = 0):
        super().__init__()
        if apply_pos_emb or num_latents_mean_pooled:
            raise NotImplementedError("apply_pos_emb / num_latents_mean_pooled are not used by IMAGDressing")
        self.pos_emb = None
        self.to_latents_from_mean_pooled_seq = None
        self.latents = nn.Parameter(torch.randn(1, num_queries, dim) / dim ** 0.5)
        self._build(dim, depth, dim_head, heads, embedding_dim, output_dim, ff_mult)

    def forward(self, x):
        in_dtype = x.dtype
        if getattr(self, "_train_path", False) and torch.is_grad_enabled():
            # training step (SURVEY.md 8 row a13; reference train.py:257): grad-enabled operators
            from imagdressing_b200.train import resampler_forward_train

            out = resampler_forward_train(self, x)
            return out if in_dtype == BF16 else out.to(in_dtype)
        lat = self.latents.detach().to(BF16).repeat(x.size(0), 1, 1).contiguous()
        out = self._run_stack(x.to(BF16), lat)
        return out if in_dtype == BF16 else out.to(in_dtype)


class FacePerceiverResampler(_PerceiverStack):
    """adapter/resampler.py:128-167."""

    def __init__(self, *, dim=768, depth=4, dim_head=64, heads=16, embedding_dim=1280, output_dim=768, ff_mult=4):
        super().__init__()
        self._build(dim, depth, dim_head, heads, embedding_dim, output_dim, ff_mult)

    def forward(self, latents, x):
        return self._run_stack(x.to(BF16), latents.to(BF16).contiguous())


class ProjPlusModel(nn.Module):
    """adapter/resampler.py:250-281."""

    def __init__(self, cross_attention_dim=768, id_embeddings_dim=512, clip_embeddings_dim=1280, num_tokens=4):
        super().__init__()
        self.cross_attention_dim = cross_attention_dim
        self.num_tokens = num_tokens
        self.proj = nn.Sequential(nn.Linear(id_embeddings_dim, id_embeddings_dim * 2), nn.GELU(),
                                  nn.Linear(id_embeddings_dim * 2, cross_attention_dim * num_tokens))
        self.norm = nn.LayerNorm(cross_attention_dim)
        self.perceiver_resampler = FacePerceiverResampler(
            dim=cross_attention_dim, depth=4, dim_head=64, heads=cross_attention_dim // 64,
            embedding_dim=clip_embeddings_dim, output_dim=cross_attention_dim, ff_mult=4)

    @torch.no_grad()
    def forward(self, id_embeds, clip_embeds, shortcut=False, scale=1.0):
        in_dtype = id_embeds.dtype
        p0, p2 = self.proj[0], self.proj[2]
        h = ops.linear_small_m(id_embeds.float().contiguous(), _bf(p0.weight), _f32(p0.bias), act_out=ACT_GELU)
        h = ops.linear_small_m(h, _bf(p2.weight), _f32(p2.bias))
        x = h.reshape(-1, self.num_tokens, self.cross_attention_dim).to(BF16)
        x = ops.layernorm(x.contiguous(), _f32(self.norm.weight), _f32(self.norm.bias))
        out = self.perceiver_resampler(x, clip_embeds)
        if shortcut:
            out = (x.float() + scale * out.float()).to(BF16)
        return out if in_dtype == BF16 else out.to(in_dtype)
