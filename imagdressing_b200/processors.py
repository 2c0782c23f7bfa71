"""CUDA implementations behind the reference's attention-processor plugin API.

`attention_forward` is the one routine all processors share: projection GEMMs (wgmma), the two-stream attention
kernel, and the output projection with bias (+ the transformer block's residual when the caller offered it).
What differs per processor is only which weights are merged (LoRA) and what the second KV stream is:

  RefSAttnProcessor2_0      self stream + garment stream (to_k_ref/to_v_ref of the cached garment features)
  LoRAIPAttnProcessor2_0    text stream + IP-token stream (to_k_ip/to_v_ip of the last num_tokens context tokens)
  CAttnProcessor2_0 / AttnProcessor2_0 / CacheAttnProcessor2_0   one stream

Work that the reference repeats every denoising step but that does not depend on the step is done once and
cached by tensor identity: text K/V projections, garment K/V projections, LoRA-merged weights
(W' = W + lora_scale * up @ down, SURVEY.md A.5).

Reference: adapter/attention_processor.py (RefS :513-627, LoraRefS :391-511, C :202-295, LoRAIP :746-871,
Cache :13-100, RefLoraS :1006-1128).
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import torch
import torch.nn as nn

from . import ops

BF16 = torch.bfloat16


class TensorMemo:
    """One-entry memo keyed by tensor identity + in-place version (holds a reference so the address cannot be
    recycled under it)."""

    __slots__ = ("src", "ver", "extra", "val")

    def __init__(self):
        self.src = None
        self.ver = -1
        self.extra = None
        self.val = None

    def get(self, t: torch.Tensor, extra=None):
        if self.src is not None and self.src is t and self.ver == t._version and self.extra == extra:
            return self.val
        return None

    def put(self, t: torch.Tensor, val, extra=None):
        self.src, self.ver, self.extra, self.val = t, t._version, extra, val
        return val

    def clear(self):
        self.src = None  # keep `val`: its storage is reused so captured CUDA graphs keep valid addresses

    def reusable(self, shape, dtype=BF16):
        """Previous value's storage when the shape matches — recomputing in place keeps device addresses stable
        across images, which is what lets one captured step graph be replayed for every image."""
        v = self.val
        if v is not None and tuple(v.shape) == tuple(shape) and v.dtype == dtype:
            return v
        return None


def as_bf16(t: torch.Tensor, memo: Optional[TensorMemo] = None) -> torch.Tensor:
    if t.dtype == BF16 and t.is_contiguous():
        return t
    if memo is not None:
        v = memo.get(t)
        if v is not None:
            return v
        buf = memo.reusable(t.shape)
        if buf is not None:
            buf.copy_(t)
            return memo.put(t, buf)
        return memo.put(t, t.to(BF16).contiguous())
    return t.to(BF16).contiguous()


def _w(lin: nn.Linear) -> torch.Tensor:
    return lin.weight.detach().float()


def _merged(lin: nn.Linear, lora, lora_scale: float) -> torch.Tensor:
    """W + lora_scale * up @ down (network_alpha is None everywhere in the reference)."""
    w = _w(lin)
    if lora is not None and lora_scale != 0.0:
        w = w + float(lora_scale) * (lora.up.weight.detach().float() @ lora.down.weight.detach().float())
    return w


def _ver(*mods) -> tuple:
    """Identity + in-place version of every weight a derived (packed) tensor is built from: `load_state_dict`,
    `copy_` and optimizer steps bump `_version`, `.to()` / re-assignment change `data_ptr` (ADVICE r1: a reference-style
    `ModuleList(unet.attn_processors.values()).load_state_dict(...)` must not leave stale packed weights behind)."""
    out = []
    for m in mods:
        if m is None:
            continue
        for w in ((m.weight,) if hasattr(m, "weight") else (m.down.weight, m.up.weight)):
            out.append((w.data_ptr(), w._version))
        b = getattr(m, "bias", None)
        if b is not None:
            out.append((b.data_ptr(), b._version))
    return tuple(out)


def _packer(proc, attn):
    """packed(key, build, ver) -> derived tensor, cached per (attention module, key) and rebuilt when `ver` changes
    (one entry per key: an old lora_scale / weight version is evicted, not accumulated). The cache lives on our own
    `modeling.Attention` (cleared by its `_apply` / `invalidate_packed`); on a FOREIGN host module — e.g. a stock
    diffusers `Attention`, which has no such cache — it lives on the processor, keyed by the host's id."""
    store = getattr(attn, "_pk", None)
    if not isinstance(store, dict) or not hasattr(attn, "packed"):
        store = proc.__dict__.setdefault("_foreign_pk", {}).setdefault(id(attn), {})

    def packed(key, build, ver=()):
        hit = store.get(key)
        if hit is not None and hit[0] == ver:
            return hit[1]
        val = build()
        store[key] = (ver, val)
        return val

    return packed


def _flat(t: torch.Tensor) -> torch.Tensor:
    """[B, L, C] -> [B*L, C] view (keeps a column-slice's row stride)."""
    B, L, C = t.shape
    return t.as_strided((B * L, C), (t.stride(1), 1), t.storage_offset())


class _ProcState:
    """Mixin: caches owned by a processor instance."""

    # processors built on attention_forward can take the RAW residual stream + row statistics instead of the
    # LayerNorm output (Attention._ln_fold); the garment tap (CacheAttnProcessor2_0) needs the normed tensor itself
    _accepts_ln_fold = True

    def _init_state(self):
        self._ctx_memo = TensorMemo()   # context tensor -> bf16 copy
        self._kv_memo = TensorMemo()    # context tensor -> projected K|V
        self._kv2_memo = TensorMemo()   # second stream source -> projected K|V
        self._g_memo = TensorMemo()     # garment feature tensor -> bf16 copy

    def invalidate_packed(self):
        for m in (self._ctx_memo, self._kv_memo, self._kv2_memo, self._g_memo):
            m.clear()
        self.__dict__.pop("_foreign_pk", None)


def attention_forward(proc, attn, hidden_states: torch.Tensor, encoder_hidden_states: Optional[torch.Tensor], *,
                      lora: Optional[dict] = None, lora_scale: float = 0.0,
                      second: Optional[tuple] = None, text_len: Optional[int] = None,
                      prepare_only: bool = False) -> Optional[torch.Tensor]:
    """hidden_states [B, L, C]; returns [B, L, C] in hidden_states.dtype.

    second = (source [Bs, Ls, Cs], to_k, to_v, out_scale, n_query_samples[, first, length]): the extra KV stream,
    optionally a [first, first+length) token window of the source.
    prepare_only: compute (in place) only what is invariant over the denoising steps — the context K|V projection
    and the second stream's K|V projection — and return None (DenoiseEngine refreshes these once per image and
    replays a captured CUDA graph for the steps).
    text_len: use only the first text_len context tokens for stream 0 (LoRAIP strips the IP tokens, :811-815).
    """
    if getattr(attn, "_train_path", False) and torch.is_grad_enabled() and not prepare_only:
        # training step (SURVEY.md 8 row a13): autograd operators instead of the fused, cached inference sequence
        if lora is not None or text_len is not None:
            raise NotImplementedError("training path: the reference trains RefS / C processors only (train.py:338-366)")
        from .train import train_attention_forward

        return train_attention_forward(proc, attn, hidden_states, encoder_hidden_states, second)
    in_dtype = hidden_states.dtype
    B, L, C = hidden_states.shape
    heads = attn.heads
    hd = C // heads
    x = as_bf16(hidden_states)
    packed = _packer(proc, attn)
    lq, lk, lv, lo = ((lora["q"], lora["k"], lora["v"], lora["out"]) if lora else (None,) * 4)
    ls = float(lora_scale) if lora else 0.0
    lkey = f"{id(proc)}" if lora else "base"
    v_q, v_k, v_v = _ver(attn.to_q, lq) + (ls,), _ver(attn.to_k, lk) + (ls,), _ver(attn.to_v, lv) + (ls,)
    fold = getattr(attn, "_ln_fold", None)  # (stats, parts, gamma, beta, eps, stats_out): hidden_states is the RAW stream
    stats_out = None
    if fold is not None:
        attn._ln_fold = None  # consumed
        f_stats, f_parts, f_gamma, f_beta, f_eps, stats_out = fold
        v_ln = ((f_gamma.data_ptr(), f_gamma._version), (f_beta.data_ptr(), f_beta._version))

        def folded(key, build_w, ver):
            """(W' bf16, b' fp32, colsum fp32) of a projection that reads LN(hidden_states)."""
            from .modeling import fold_layernorm

            pk = packed("ln:" + key, lambda: fold_layernorm(build_w(), None, f_gamma, f_beta), ver + v_ln)
            return pk, ops.LnFold(f_stats, f_parts, C, f_eps, pk[2])

    if encoder_hidden_states is None and prepare_only:
        q2 = s0 = None
    elif encoder_hidden_states is None:
        build_qkv = lambda: torch.cat(
            [_merged(attn.to_q, lq, ls), _merged(attn.to_k, lk, ls), _merged(attn.to_v, lv, ls)], 0)
        if fold is not None:
            (wf, bf_, _), ln = folded("qkv:" + lkey, build_qkv, v_q + v_k + v_v)
            qkv = ops.gemm(x, wf, bias=bf_, ln=ln)
        else:
            wqkv = packed("qkv:" + lkey, lambda: build_qkv().to(BF16).contiguous(), v_q + v_k + v_v)
            qkv = ops.gemm(x, wqkv)  # [B, L, 3C]
        q2 = _flat(qkv[..., :C])
        s0 = ops.kv_stream(_flat(qkv[..., C:2 * C]), _flat(qkv[..., 2 * C:]), L)
    else:
        build_q = lambda: _merged(attn.to_q, lq, ls)
        if prepare_only:
            q2 = None
        elif fold is not None:
            (wf, bf_, _), ln = folded("q:" + lkey, build_q, v_q)
            q2 = _flat(ops.gemm(x, wf, bias=bf_, ln=ln))
        else:
            q2 = _flat(ops.gemm(x, packed("q:" + lkey, lambda: build_q().to(BF16).contiguous(), v_q)))
        ctx_src = encoder_hidden_states
        Lc = ctx_src.shape[1] if text_len is None else text_len
        kv = proc._kv_memo.get(ctx_src, (lkey, Lc, v_k, v_v))
        if kv is None:
            wkv = packed("kv:" + lkey, lambda: torch.cat([_merged(attn.to_k, lk, ls), _merged(attn.to_v, lv, ls)],
                                                         0).to(BF16).contiguous(), v_k + v_v)
            ctx = as_bf16(ctx_src, proc._ctx_memo)
            buf = proc._kv_memo.reusable((*ctx.shape[:-1], 2 * C))
            kv = proc._kv_memo.put(ctx_src, ops.gemm(ctx, wkv, out=buf), (lkey, Lc, v_k, v_v))  # [B, Lctx, 2C]
        # per-sample row stride stays the full context length; only the first Lc keys are visited
        s0 = _stream_from_kv(kv, C, Lc)

    s1 = None
    if second is not None:
        src, to_k, to_v, out_scale, n_q = second[:5]
        first = second[5] if len(second) > 5 else 0
        v_2 = _ver(to_k, to_v)
        kv2 = proc._kv2_memo.get(src, v_2)
        if kv2 is None:
            w2 = packed(f"kv2:{id(to_k)}", lambda: torch.cat([_w(to_k), _w(to_v)], 0).to(BF16).contiguous(), v_2)
            src_bf = as_bf16(src, proc._g_memo)
            buf = proc._kv2_memo.reusable((*src_bf.shape[:-1], 2 * C))
            kv2 = proc._kv2_memo.put(src, ops.gemm(src_bf, w2, out=buf), v_2)
        bcast = kv2.shape[0] == 1 and n_q > 1
        if not bcast and kv2.shape[0] < n_q:
            raise ValueError(f"second KV stream has batch {kv2.shape[0]} but {n_q} query samples use it")
        length = second[6] if len(second) > 6 else kv2.shape[1] - first
        s1 = _stream_from_kv(kv2, C, length, first, broadcast=bcast, n_query_samples=n_q, out_scale=out_scale)
    if prepare_only:
        return None

    o = ops.attention(q2, B, L, heads, hd, s0, s1)  # [B*L, C]

    out_lin = attn.to_out[0]
    wo = packed("o:" + lkey, lambda: _merged(out_lin, lo, ls).to(BF16).contiguous(), _ver(out_lin, lo) + (ls,))
    bo = packed("bo", lambda: out_lin.bias.detach().float().contiguous(), _ver(out_lin))
    # our own Attention offers the transformer block's residual for the out-projection epilogue; a foreign host module
    # (stock diffusers Attention) has no such attribute: the block adds the residual itself, as diffusers does
    residual = getattr(attn, "_fused_residual", None)
    if residual is not None and residual.dtype == BF16 and residual.shape == hidden_states.shape:
        attn._fused_residual = None  # consumed: fused into the out-projection epilogue
        y = ops.gemm(o, wo, bias=bo, residual=residual.reshape(B * L, C), stats_out=stats_out)
    else:
        if stats_out is not None:
            raise RuntimeError("LayerNorm fold needs the residual fused into the out-projection (bf16 stream)")
        y = ops.gemm(o, wo, bias=bo)
    y = y.view(B, L, C)
    return y if in_dtype == BF16 else y.to(in_dtype)


def _stream_from_kv(kv: torch.Tensor, C: int, length: int, first: int = 0, **kw):
    """kv: [Bk, Lk, 2C] fused K|V projection; the stream visits keys [first, first+length) of each sample."""
    Bk, Lk, _ = kv.shape
    ld = kv.stride(1)
    off = kv.storage_offset() + first * ld
    k = kv.as_strided((Bk * Lk - first, C), (ld, 1), off)
    v = kv.as_strided((Bk * Lk - first, C), (ld, 1), off + C)
    return ops.kv_stream(k, v, length, sample_rows=Lk if length != Lk else 0, **kw)


# ------------------------------------------------------------------------------------------------ processors
class AttnProcessor2_0(_ProcState):
    """Default processor: plain SDPA (diffusers-0.24 AttnProcessor2_0)."""

    def __init__(self):
        self._init_state()

    def __call__(self, attn, hidden_states, encoder_hidden_states=None, attention_mask=None, temb=None, scale=1.0,
                 **kwargs):
        return attention_forward(self, attn, hidden_states, encoder_hidden_states,
                                 prepare_only=kwargs.get("_prepare_only", False))


def ref_stream(proc, hidden_states, sa_hidden_states, ref_samples):
    """(source, to_k_ref, to_v_ref, scale, n_query_samples) or None — adapter/attention_processor.py:597-612."""
    if sa_hidden_states is None:
        return None
    g = sa_hidden_states[proc.name]
    n_q = hidden_states.shape[0] if ref_samples is None else int(ref_samples)
    return (g, proc.to_k_ref, proc.to_v_ref, float(proc.scale), n_q)
