"""CLIP text / vision encoders on the sm_90a kernels (SURVEY.md §8f row 3).

The reference builds them with `transformers` (`CLIPTextModel`, `CLIPVisionModelWithProjection`,
inference_IMAGdressing.py:44-49) and calls them at the edges of the path:

    prompt_embeds = text_encoder(input_ids)[0]                                        IMAGDressing_v1_pipeline.py:396-405 (encode_prompt)
    image_embeds  = image_encoder(ref_clip_image, output_hidden_states=True).hidden_states[-2]    :407-415

Those modules stay the PARAMETER CONTAINERS (so `from_pretrained`, `.to()`, `state_dict()` and the checkpoints keep
working unchanged); `accelerate(module)` wraps one in an executor that runs the forward on this library's kernels instead of
torch / cuBLAS: token + position embedding gather, patch embedding as a wgmma GEMM over patch rows, pre-LN transformer
layers = LayerNorm kernel -> fused QKV GEMM (+bias) -> the attention kernel (causal for text; head_dim 64 text / 80 ViT-H)
-> out-projection GEMM with bias + residual in the epilogue -> LayerNorm -> fc1 GEMM with bias + (quick_)GELU in the
epilogue -> fc2 GEMM with bias + residual. The pipelines wrap CUDA-resident CLIP modules automatically (IMAGD_CLIP_KERNELS=0
keeps the torch modules); the outputs mirror the transformers return objects for what the pipelines read (`[0]`,
`.last_hidden_state`, `.hidden_states`, `text_model.final_layer_norm`).

Parity is PINNED for this row: the oracle is the installed transformers implementation itself (tests/test_clip_*.py).
"""
from __future__ import annotations

import os
from typing import List, Optional

import torch
import torch.nn as nn

from . import ops
from ._lib import ACT_GELU, ACT_NONE, ACT_QUICK_GELU

BF16 = torch.bfloat16


def _f32(t):
    return t.detach().float().contiguous()


def _bf(t):
    return t.detach().to(BF16).contiguous()


class _Out:
    """The slice of transformers' BaseModelOutputWithPooling / CLIPVisionModelOutput the pipelines read."""

    def __init__(self, last_hidden_state, hidden_states=None):
        self.last_hidden_state = last_hidden_state
        self.hidden_states = hidden_states

    def __getitem__(self, i):
        items = (self.last_hidden_state,) + ((self.hidden_states,) if self.hidden_states is not None else ())
        return items[i]


class _Encoder(nn.Module):
    """Shared pre-LN transformer stack over a transformers CLIPEncoder's layers."""

    def __init__(self, hf_module, encoder, heads: int, act: str, causal: bool):
        super().__init__()
        self.hf = hf_module  # registered: .to() / state_dict() / parameters() go through to the transformers module
        self._layers = encoder.layers
        self.heads = heads
        if act not in ("gelu", "quick_gelu"):
            raise NotImplementedError(f"CLIP hidden_act {act!r} (the reference's encoders use gelu / quick_gelu)")
        self.act = ACT_QUICK_GELU if act == "quick_gelu" else ACT_GELU
        self.causal = causal
        self._pk = None
        self._pk_ver = None

    # ---- passthroughs the scripts / pipelines touch
    @property
    def config(self):
        return self.hf.config

    @property
    def dtype(self):
        return next(self.hf.parameters()).dtype

    @property
    def device(self):
        return next(self.hf.parameters()).device

    def _version(self):
        return tuple((p.data_ptr(), p._version) for p in self.hf.parameters())

    def _layer_packs(self):
        ver = self._version()
        if self._pk is None or self._pk_ver != ver:
            packs = []
            for lyr in self._layers:
                a = lyr.self_attn
                packs.append(dict(
                    ln1=(_f32(lyr.layer_norm1.weight), _f32(lyr.layer_norm1.bias), lyr.layer_norm1.eps),
                    wqkv=_bf(torch.cat([a.q_proj.weight, a.k_proj.weight, a.v_proj.weight], 0)),
                    bqkv=_f32(torch.cat([a.q_proj.bias, a.k_proj.bias, a.v_proj.bias], 0)),
                    wo=_bf(a.out_proj.weight), bo=_f32(a.out_proj.bias),
                    ln2=(_f32(lyr.layer_norm2.weight), _f32(lyr.layer_norm2.bias), lyr.layer_norm2.eps),
                    w1=_bf(lyr.mlp.fc1.weight), b1=_f32(lyr.mlp.fc1.bias), w2=_bf(lyr.mlp.fc2.weight), b2=_f32(lyr.mlp.fc2.bias)))
            self._pk = dict(layers=packs, extra=self._extra_packs())
            self._pk_ver = ver
        return self._pk

    def _extra_packs(self):
        return {}

    def _run_layers(self, x: torch.Tensor, n_layers: int, keep: bool) -> List[torch.Tensor]:
        """x [B, L, C] bf16 -> hidden states after each of the first n_layers layers (only the last one unless `keep`)."""
        pk = self._layer_packs()["layers"]
        B, L, C = x.shape
        hd = C // self.heads
        states = []
        for i in range(n_layers):
            p = pk[i]
            h = ops.layernorm(x, p["ln1"][0], p["ln1"][1], p["ln1"][2])
            qkv = ops.gemm(h, p["wqkv"], bias=p["bqkv"])  # [B, L, 3C]
            flat = lambda t: t.as_strided((B * L, C), (t.stride(1), 1), t.storage_offset())
            s0 = ops.kv_stream(flat(qkv[..., C:2 * C]), flat(qkv[..., 2 * C:]), L)
            o = ops.attention(flat(qkv[..., :C]), B, L, self.heads, hd, s0, causal=self.causal)
            x = ops.gemm(o.view(B, L, C), p["wo"], bias=p["bo"], residual=x)
            h = ops.layernorm(x, p["ln2"][0], p["ln2"][1], p["ln2"][2])
            h = ops.gemm(h, p["w1"], bias=p["b1"], act=self.act)
            x = ops.gemm(h, p["w2"], bias=p["b2"], residual=x)
            if keep or i == n_layers - 1:
                states.append(x)
        return states


class ClipTextEncoder(_Encoder):
    """transformers CLIPTextModel on the kernels: `enc(input_ids)[0]` = final_layer_norm(last layer)."""

    def __init__(self, hf: nn.Module):
        tm = hf.text_model
        cfg = hf.config
        super().__init__(hf, tm.encoder, cfg.num_attention_heads, cfg.hidden_act, causal=True)
        self.text_model = tm  # the pipelines' clip_skip branch calls text_model.final_layer_norm

    def _extra_packs(self):
        e, tm = self.text_model.embeddings, self.text_model
        return dict(tok=_bf(e.token_embedding.weight), pos=_bf(e.position_embedding.weight),
                    lnf=(_f32(tm.final_layer_norm.weight), _f32(tm.final_layer_norm.bias), tm.final_layer_norm.eps))

    @torch.no_grad()
    def forward(self, input_ids, attention_mask=None, output_hidden_states: bool = False, **kw):
        ex = self._layer_packs()["extra"]
        ids = input_ids.to(device=self.device, dtype=torch.int64).contiguous()
        x = ops.embed_tokens(ids, ex["tok"], ex["pos"])
        states = self._run_layers(x, len(self._layers), output_hidden_states)
        last = ops.layernorm(states[-1], ex["lnf"][0], ex["lnf"][1], ex["lnf"][2])
        dt = self.dtype
        cast = (lambda t: t) if dt == BF16 else (lambda t: t.to(dt))
        hs = tuple(cast(t) for t in [x] + states) if output_hidden_states else None
        return _Out(cast(last), hs)


class ClipVisionEncoder(_Encoder):
    """transformers CLIPVisionModel(WithProjection) on the kernels. The pipelines read `hidden_states[-2]` (the input of the
    last layer), so without `output_hidden_states` nothing beyond the patch embedding is needed and with it only the first
    N-1 layers run — unless `last_hidden_state` is asked for (post-LN pooling / projection are not on the path)."""

    def __init__(self, hf: nn.Module):
        vm = hf.vision_model
        cfg = hf.config
        super().__init__(hf, vm.encoder, cfg.num_attention_heads, cfg.hidden_act, causal=False)
        self.vision_model = vm
        self.patch = cfg.patch_size

    def _extra_packs(self):
        e, vm = self.vision_model.embeddings, self.vision_model
        w = e.patch_embedding.weight.detach().float()  # [C, 3, p, p]
        C = w.shape[0]
        K = w[0].numel()
        kpad = (K + 7) // 8 * 8
        wp = torch.zeros(C, kpad, dtype=torch.float32, device=w.device)
        wp[:, :K] = w.reshape(C, K)
        pos = e.position_embedding.weight.detach().float()
        pre = getattr(vm, "pre_layrnorm", None) or getattr(vm, "pre_layernorm")
        return dict(wp=wp.to(BF16).contiguous(), kpad=kpad, pos_patches=pos[1:].to(BF16).contiguous(),
                    cls=(e.class_embedding.detach().float() + pos[0]).to(BF16).contiguous(),
                    pre=(_f32(pre.weight), _f32(pre.bias), pre.eps))

    @torch.no_grad()
    def forward(self, pixel_values, output_hidden_states: bool = False, **kw):
        ex = self._layer_packs()["extra"]
        x = pixel_values.to(device=self.device, dtype=torch.float32).contiguous()
        B, _, H, W = x.shape
        n = (H // self.patch) * (W // self.patch)
        if ex["pos_patches"].shape[0] != n:
            raise ValueError(f"image {H}x{W} gives {n} patches, the position table holds {ex['pos_patches'].shape[0]}")
        C = ex["wp"].shape[0]
        rows = ops.patchify(x, self.patch, ex["kpad"]).view(B, n, ex["kpad"])
        tokens = torch.empty(B, n + 1, C, device=x.device, dtype=BF16)
        for b in range(B):  # patch rows + position embedding straight into rows 1.. of each sample (GEMM epilogue)
            ops.gemm(rows[b], ex["wp"], residual=ex["pos_patches"], out=tokens[b, 1:])
        ops.broadcast_row(ex["cls"], tokens, 0)
        h0 = ops.layernorm(tokens, ex["pre"][0], ex["pre"][1], ex["pre"][2])
        n_layers = len(self._layers) - 1 if output_hidden_states else len(self._layers)
        states = self._run_layers(h0, n_layers, output_hidden_states)
        dt = self.dtype
        cast = (lambda t: t) if dt == BF16 else (lambda t: t.to(dt))
        if output_hidden_states:
            # hidden_states = (embeddings, layer 1, ..., layer N): the tuple is completed with a placeholder for layer N so
            # that [-2] indexes the penultimate state exactly as with transformers, without computing the last layer
            hs = tuple(cast(t) for t in [h0] + states) + (None,)
            return _Out(None, hs)
        return _Out(cast(states[-1]), None)


def accelerate(module):
    """Wrap a transformers CLIPTextModel / CLIPVisionModel(WithProjection) in its kernel-backed executor; anything else
    (None, an already wrapped encoder, a foreign module) is returned unchanged."""
    if module is None or isinstance(module, _Encoder):
        return module
    if hasattr(module, "text_model") and hasattr(module.text_model, "encoder"):
        return ClipTextEncoder(module)
    if hasattr(module, "vision_model") and hasattr(module.vision_model, "encoder"):
        return ClipVisionEncoder(module)
    return module


def auto_accelerate(module):
    """What the pipelines do with the encoders they are given: CUDA-resident CLIP modules run on the kernels
    (IMAGD_CLIP_KERNELS=0 keeps torch); CPU-resident ones are left alone (the library has no CPU path)."""
    if module is None or os.environ.get("IMAGD_CLIP_KERNELS", "1") == "0":
        return module
    try:
        on_cuda = next(module.parameters()).is_cuda
    except (StopIteration, AttributeError):
        return module
    return accelerate(module) if on_cuda else module
