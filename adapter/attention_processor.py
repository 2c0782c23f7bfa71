"""Drop-in for the reference's `adapter/attention_processor.py`: same module path, class names, constructor
signatures, parameter names (state_dict keys `to_k_ref.weight`, `to_k_ip.weight`, `to_q_lora.down.weight`, ...),
mutable attributes (`scale`, `lora_scale`, `name`, `cache`) and call signature — executing on the sm_90a
kernels through imagdressing_b200.processors.attention_forward. See that module for how the arithmetic maps to
kernels; every class cites the reference lines it replaces (relative to /root/reference).

What is intentionally different from the reference (SURVEY.md Appendix B):
  * per-step-invariant projections (text K/V, garment K/V) and LoRA merges are computed once and cached;
  * `ref_samples=n` (extra cross_attention_kwarg) marks a CFG-batched call whose first n samples carry the
    garment stream (B4); without it every sample does, as in the reference;
  * the unused / malformed `attn_map` of IPAttnProcessor2_0 (B10) is not reproduced.
"""
from __future__ import annotations

from typing import Optional

import torch
from torch import nn

from imagdressing_b200.processors import AttnProcessor2_0, _ProcState, attention_forward, ref_stream

__all__ = ["AttnProcessor2_0", "CacheAttnProcessor2_0", "SAttnProcessor2_0", "CAttnProcessor2_0", "BaseSAttnProcessor2_0",
           "LoraRefSAttnProcessor2_0", "RefSAttnProcessor2_0", "RefCAttnProcessor2_0", "LoRAIPAttnProcessor2_0",
           "IPAttnProcessor2_0", "RefLoraSAttnProcessor2_0", "LoRALinearLayer"]


class LoRALinearLayer(nn.Module):
    """diffusers-0.24 models.lora.LoRALinearLayer (parameter container: `down.weight` [rank, in], `up.weight`
    [out, rank]); merged into the projection weights at pack time: W' = W + lora_scale * up @ down."""

    def __init__(self, in_features, out_features, rank=4, network_alpha=None, device=None, dtype=None):
        super().__init__()
        if network_alpha is not None:
            raise NotImplementedError("network_alpha is None everywhere in the reference (SURVEY.md A.5)")
        self.down = nn.Linear(in_features, rank, bias=False, device=device, dtype=dtype)
        self.up = nn.Linear(rank, out_features, bias=False, device=device, dtype=dtype)
        self.network_alpha = network_alpha
        self.rank = rank
        nn.init.normal_(self.down.weight, std=1 / rank)
        nn.init.zeros_(self.up.weight)


class _ModuleProc(nn.Module, _ProcState):
    def __init__(self):
        nn.Module.__init__(self)
        self._init_state()

    def _apply(self, fn, *a, **k):
        self.invalidate_packed()
        return super()._apply(fn, *a, **k)

    def _lora(self):
        return dict(q=self.to_q_lora, k=self.to_k_lora, v=self.to_v_lora, out=self.to_out_lora)


class CacheAttnProcessor2_0(_ProcState):
    """reference :13-100 — garment-UNet feature tap: stash the processor input (`cache["hidden_states"]`, :34),
    then plain SDPA."""

    _accepts_ln_fold = False  # the tap is the LayerNorm OUTPUT: it has to be materialised for this processor

    def __init__(self):
        self._init_state()
        self.cache = {}

    def __call__(self, attn, hidden_states, encoder_hidden_states=None, attention_mask=None, temb=None, scale=1.0,
                 **kwargs):
        if kwargs.get("_prepare_only", False):
            return attention_forward(self, attn, hidden_states, encoder_hidden_states, prepare_only=True)
        self.cache["hidden_states"] = hidden_states
        return attention_forward(self, attn, hidden_states, encoder_hidden_states)


class RefSAttnProcessor2_0(_ModuleProc):
    """reference :513-627 — hybrid attention: self SDPA + scale * SDPA(q, to_k_ref(g), to_v_ref(g)), one kernel."""

    def __init__(self, name, hidden_size, cross_attention_dim=None, scale=1.0):
        super().__init__()
        self.name = name
        self.hidden_size = hidden_size
        self.cross_attention_dim = cross_attention_dim
        self.to_k_ref = nn.Linear(cross_attention_dim or hidden_size, hidden_size, bias=False)
        self.to_v_ref = nn.Linear(cross_attention_dim or hidden_size, hidden_size, bias=False)
        self.scale = scale

    def __call__(self, attn, hidden_states, encoder_hidden_states=None, attention_mask=None, temb=None, scale=1.0,
                 num_images_per_prompt=1, cond_hidden_states=None, sa_hidden_states=None, ref_samples=None, **kwargs):
        return attention_forward(self, attn, hidden_states, encoder_hidden_states,
                                 second=ref_stream(self, hidden_states, sa_hidden_states, ref_samples),
                                 prepare_only=kwargs.get("_prepare_only", False))


class CAttnProcessor2_0(_ModuleProc):
    """reference :202-295 — plain (text) cross-attention; receives and ignores sa_hidden_states."""

    def __init__(self, name, hidden_size, cross_attention_dim=None, scale=1.0):
        super().__init__()
        self.name = name
        self.hidden_size = hidden_size
        self.cross_attention_dim = cross_attention_dim
        self.scale = scale

    def __call__(self, attn, hidden_states, encoder_hidden_states=None, attention_mask=None, temb=None, scale=1.0,
                 num_images_per_prompt=1, cond_hidden_states=None, sa_hidden_states=None, **kwargs):
        return attention_forward(self, attn, hidden_states, encoder_hidden_states,
                                 prepare_only=kwargs.get("_prepare_only", False))


class _LoraRefBase(_ModuleProc):
    def __init__(self, name, hidden_size, cross_attention_dim=None, scale=1.0, rank=128, network_alpha=None,
                 lora_scale=1.0):
        _ModuleProc.__init__(self)
        self.name = name
        self.hidden_size = hidden_size
        self.cross_attention_dim = cross_attention_dim
        kv = cross_attention_dim or hidden_size
        self.to_k_ref = nn.Linear(kv, hidden_size, bias=False)
        self.to_v_ref = nn.Linear(kv, hidden_size, bias=False)
        self.scale = scale
        self.rank = rank
        self.lora_scale = lora_scale
        self.to_q_lora = LoRALinearLayer(hidden_size, hidden_size, rank, network_alpha)
        self.to_k_lora = LoRALinearLayer(kv, hidden_size, rank, network_alpha)
        self.to_v_lora = LoRALinearLayer(kv, hidden_size, rank, network_alpha)
        self.to_out_lora = LoRALinearLayer(hidden_size, hidden_size, rank, network_alpha)

    def __call__(self, attn, hidden_states, encoder_hidden_states=None, attention_mask=None, temb=None, scale=1.0,
                 num_images_per_prompt=1, cond_hidden_states=None, sa_hidden_states=None, ref_samples=None, **kwargs):
        return attention_forward(self, attn, hidden_states, encoder_hidden_states, lora=self._lora(),
                                 lora_scale=float(self.lora_scale),
                                 second=ref_stream(self, hidden_states, sa_hidden_states, ref_samples),
                                 prepare_only=kwargs.get("_prepare_only", False))


class LoraRefSAttnProcessor2_0(_LoraRefBase):
    """reference :391-511 — RefS + lora_scale * rank-r LoRA on q / k / v / out (merged into the weights)."""


class RefLoraSAttnProcessor2_0(_LoraRefBase):
    """reference :1006-1128 — app.py's variant; identical arithmetic (it forwards `scale` to LoRACompatibleLinear,
    a numerical no-op, SURVEY.md A.5). Deliberately NOT a subclass of LoraRefSAttnProcessor2_0 so the reference's
    isinstance checks behave the same (set_scale ignores it, B9)."""


class LoRAIPAttnProcessor2_0(_ModuleProc):
    """reference :746-871 — text stream (context minus the last num_tokens, LoRA on q/k/v) + scale * IP stream
    (to_k_ip / to_v_ip over the last num_tokens tokens), out projection + LoRA. With no face the reference still
    strips the last 4 *text* tokens (B11); reproduced."""

    def __init__(self, hidden_size, cross_attention_dim=None, rank=4, network_alpha=None, lora_scale=1.0, scale=1.0,
                 num_tokens=4):
        super().__init__()
        self.rank = rank
        self.lora_scale = lora_scale
        self.num_tokens = num_tokens
        kv = cross_attention_dim or hidden_size
        self.to_q_lora = LoRALinearLayer(hidden_size, hidden_size, rank, network_alpha)
        self.to_k_lora = LoRALinearLayer(kv, hidden_size, rank, network_alpha)
        self.to_v_lora = LoRALinearLayer(kv, hidden_size, rank, network_alpha)
        self.to_out_lora = LoRALinearLayer(hidden_size, hidden_size, rank, network_alpha)
        self.hidden_size = hidden_size
        self.cross_attention_dim = cross_attention_dim
        self.scale = scale
        self.to_k_ip = nn.Linear(kv, hidden_size, bias=False)
        self.to_v_ip = nn.Linear(kv, hidden_size, bias=False)

    def __call__(self, attn, hidden_states, encoder_hidden_states=None, attention_mask=None, scale=1.0, temb=None,
                 *args, **kwargs):
        if encoder_hidden_states is None:
            raise ValueError("LoRAIPAttnProcessor2_0 needs encoder_hidden_states (reference :807-815, B11)")
        end_pos = encoder_hidden_states.shape[1] - self.num_tokens
        second = (encoder_hidden_states, self.to_k_ip, self.to_v_ip, float(self.scale), hidden_states.shape[0],
                  end_pos, self.num_tokens)
        return attention_forward(self, attn, hidden_states, encoder_hidden_states, lora=self._lora(),
                                 lora_scale=float(self.lora_scale), second=second, text_len=end_pos,
                                 prepare_only=kwargs.get("_prepare_only", False))


class IPAttnProcessor2_0(_ModuleProc):
    """reference :873-1003 — IP-Adapter without LoRA (no script uses it; kept for import / isinstance compat)."""

    def __init__(self, hidden_size, cross_attention_dim=None, scale=1.0, num_tokens=4):
        super().__init__()
        self.hidden_size = hidden_size
        self.cross_attention_dim = cross_attention_dim
        self.scale = scale
        self.num_tokens = num_tokens
        kv = cross_attention_dim or hidden_size
        self.to_k_ip = nn.Linear(kv, hidden_size, bias=False)
        self.to_v_ip = nn.Linear(kv, hidden_size, bias=False)

    def __call__(self, attn, hidden_states, encoder_hidden_states=None, attention_mask=None, temb=None, *args,
                 **kwargs):
        if encoder_hidden_states is None:
            raise ValueError("IPAttnProcessor2_0 needs encoder_hidden_states")
        end_pos = encoder_hidden_states.shape[1] - self.num_tokens
        second = (encoder_hidden_states, self.to_k_ip, self.to_v_ip, float(self.scale), hidden_states.shape[0],
                  end_pos, self.num_tokens)
        return attention_forward(self, attn, hidden_states, encoder_hidden_states, second=second, text_len=end_pos,
                                 prepare_only=kwargs.get("_prepare_only", False))


class BaseSAttnProcessor2_0(_ModuleProc):
    """reference :298-389 — plain self-attention (unused by the scripts)."""

    def __init__(self, name=None, hidden_size=None, cross_attention_dim=None, scale=1.0):
        super().__init__()
        self.name, self.hidden_size, self.cross_attention_dim, self.scale = name, hidden_size, cross_attention_dim, scale

    def __call__(self, attn, hidden_states, encoder_hidden_states=None, attention_mask=None, temb=None, scale=1.0,
                 **kwargs):
        return attention_forward(self, attn, hidden_states, encoder_hidden_states)


class SAttnProcessor2_0(_ModuleProc):
    """reference :103-200 — the concat-KV single-softmax variant: for self-attention with garment features the keys / values
    are to_k / to_v of cat([hidden_states, sa_hidden_states[name]], dim=1) (:155-161), ONE softmax over both. No reference
    script installs it (SURVEY.md section 0.3); on the kernels it is the one-stream attention over the concatenated context."""

    def __init__(self, name=None, hidden_size=None, cross_attention_dim=None, scale=1.0):
        super().__init__()
        self.name, self.hidden_size, self.cross_attention_dim, self.scale = name, hidden_size, cross_attention_dim, scale

    def __call__(self, attn, hidden_states, encoder_hidden_states=None, attention_mask=None, temb=None, scale=1.0,
                 cond_hidden_states=None, sa_hidden_states=None, **kwargs):
        if encoder_hidden_states is None and sa_hidden_states is not None:
            ref = sa_hidden_states[self.name]
            encoder_hidden_states = torch.cat([hidden_states.to(ref.dtype), ref], dim=1)
        return attention_forward(self, attn, hidden_states, encoder_hidden_states,
                                 prepare_only=kwargs.get("_prepare_only", False))


class RefCAttnProcessor2_0(_ModuleProc):
    """reference :630-744 — (cross-)attention plus the reference branch scale * SDPA(q, to_k_ref(g), to_v_ref(g)) on the
    same query: the two-stream kernel with the context as stream 0 (unused by the scripts)."""

    def __init__(self, name=None, hidden_size=None, cross_attention_dim=None, scale=1.0):
        super().__init__()
        self.name, self.hidden_size, self.cross_attention_dim, self.scale = name, hidden_size, cross_attention_dim, scale
        self.to_k_ref = nn.Linear(hidden_size, hidden_size, bias=False)  # :643-644: hidden_size inputs
        self.to_v_ref = nn.Linear(hidden_size, hidden_size, bias=False)

    def __call__(self, attn, hidden_states, encoder_hidden_states=None, attention_mask=None, temb=None, scale=1.0,
                 cond_hidden_states=None, sa_hidden_states=None, ref_samples=None, **kwargs):
        return attention_forward(self, attn, hidden_states, encoder_hidden_states,
                                 second=ref_stream(self, hidden_states, sa_hidden_states, ref_samples),
                                 prepare_only=kwargs.get("_prepare_only", False))
