"""Training step of IMAGDressing-v1 on the sm_90a kernels (SURVEY.md section 8 row a13, BASELINE.json configs[4]).

Mirrors /root/reference/train.py:
  * SDModel                      train.py:244-281  (Resampler -> garment UNet at t = 0 with the cache processors, EVERY batch row
                                                    kept and grad-enabled -> denoising UNet with the hybrid processors)
  * trainable set                train.py:368-379  (image projection + garment UNet + adapter modules; denoising UNet frozen)
  * loss / backward              train.py:573-605  (MSE on the epsilon target, backward through both UNets)
  * optimizer                    train.py:386-398  (AdamW; DeepSpeed bf16: fp32 master weights, bf16 working copy)
  * data parallelism             train.py:601-609  (DeepSpeed ZeRO-2 gradient reduction) -> bucketed NCCL all-reduce of one flat
                                                    bf16 gradient buffer, launched per bucket from gradient-ready hooks so that
                                                    the reduction overlaps the rest of the backward pass

The same nn.Module trees as inference (imagdressing_b200.modeling, adapter.*) hold the parameters; with the training path
enabled and grad mode on, their forward walks the operators through imagdressing_b200.autograd (un-fused where a fused
inference epilogue would lose what the backward needs: GEGLU pre-activations, LayerNorm outputs). torch autograd orders the
backward; all arithmetic is in libimagd_b200.so.
"""
from __future__ import annotations

import math
import weakref
from typing import Dict, Iterable, List, Optional

import torch
import torch.nn as nn

from . import autograd as ag
from . import modeling, ops
from .processors import _packer, _ver

BF16 = torch.bfloat16


def enable_training_path(model: nn.Module, on: bool = True) -> nn.Module:
    """Route `model.forward` (UNet2DConditionModel / Resampler) and its attention processors through the autograd operators
    whenever grad mode is enabled. Inference calls (torch.no_grad) keep the fused / CUDA-graph path."""
    model._train_path = bool(on)
    for m in model.modules():
        if isinstance(m, modeling.Attention):
            m._train_path = bool(on)
    return model


def _frozen(*params) -> bool:
    return not any(p is not None and p.requires_grad for p in params)


def _bfc(t: torch.Tensor) -> torch.Tensor:
    t = t if t.dtype == BF16 else t.to(BF16)
    return t if t.is_contiguous() else t.contiguous()


# ------------------------------------------------------------------------------------------------ attention processors
def train_attention_forward(proc, attn, hidden_states, encoder_hidden_states, second=None) -> torch.Tensor:
    """The grad-enabled counterpart of processors.attention_forward (adapter/attention_processor.py:531-627 under autograd):
    projection GEMMs, two-stream attention, output projection (+ the block's residual when offered)."""
    in_dtype = hidden_states.dtype
    B, L, C = hidden_states.shape
    x = _bfc(hidden_states)
    packed = _packer(proc, attn)

    def cat_w(key, *lins):
        if _frozen(*[l.weight for l in lins]):
            return packed("train:" + key, lambda: torch.cat([l.weight.detach() for l in lins], 0).to(BF16).contiguous(),
                          _ver(*lins))
        return torch.cat([ag._bf(l.weight) for l in lins], 0)

    if encoder_hidden_states is None:
        q_src, kv0 = ag.linear(x, cat_w("qkv", attn.to_q, attn.to_k, attn.to_v)), None
    else:
        q_src = ag.linear(x, attn.to_q.weight)
        kv0 = ag.linear(_bfc(encoder_hidden_states), cat_w("kv", attn.to_k, attn.to_v))
    kv1, w1 = None, 1.0
    if second is not None:
        src, to_k, to_v, w1, n_q = second[:5]
        if len(second) > 5 or src.shape[0] != B or n_q < B:
            raise NotImplementedError("training: the second stream must cover every sample with its own keys "
                                      "(train.py:266-268 keeps every cache row)")
        kv1 = ag.linear(_bfc(src), cat_w(f"kv2:{id(to_k)}", to_k, to_v))
    o = ag.attention(q_src, kv0, kv1, attn.heads, float(w1))
    residual = getattr(attn, "_fused_residual", None)
    if residual is not None and residual.dtype == BF16 and residual.shape == hidden_states.shape:
        attn._fused_residual = None
    else:
        residual = None
    y = ag.linear(o, attn.to_out[0].weight, attn.to_out[0].bias, residual)
    return y if in_dtype == BF16 else y.to(in_dtype)


# ------------------------------------------------------------------------------------------------ UNet
def _conv_w(conv: nn.Conv2d, owner=None, key: Optional[str] = None) -> torch.Tensor:
    """Tap-major bf16 weight of a 3x3 conv: the module's inference pack when frozen, a differentiable repack otherwise."""
    if owner is not None and _frozen(conv.weight):
        return owner._packed()[key]
    return ag.pack_conv3x3(conv.weight)


def _w1x1(conv: nn.Conv2d) -> torch.Tensor:
    return conv.weight.reshape(conv.weight.shape[0], -1)


def _resnet(res: modeling.ResnetBlock2D, x, temb_all):
    """h = conv1(silu(gn(x))) + time_emb_proj(silu(temb)); out = shortcut(x) + conv2(silu(gn(h)))  (SURVEY.md A.2)."""
    h = ag.groupnorm(x, res.norm1, True)
    h = ag.conv3x3(h, _conv_w(res.conv1, res, "w1"), res.conv1.bias,
                   rowvec=temb_all[:, res.temb_offset:res.temb_offset + res.cout])
    h = ag.groupnorm(h, res.norm2, True)
    sc = x if res.conv_shortcut is None else ag.linear(x, _w1x1(res.conv_shortcut), res.conv_shortcut.bias)
    return ag.conv3x3(h, _conv_w(res.conv2, res, "w2"), res.conv2.bias, residual=sc)


def _attend(attn: modeling.Attention, normed, residual, ctx, kw):
    attn._fused_residual = residual
    out = attn(normed, encoder_hidden_states=ctx, **kw)
    if attn._fused_residual is None:
        return out
    attn._fused_residual = None
    return out.to(BF16) + residual  # foreign processor: plain residual add


def _block(blk: modeling.BasicTransformerBlock, x, ctx, kw):
    x = _attend(blk.attn1, ag.layernorm(x, blk.norm1), x, None, kw)
    x = _attend(blk.attn2, ag.layernorm(x, blk.norm2), x, ctx, kw)
    proj = blk.ff.net[0].proj
    h = ag.Geglu.apply(ag.linear(ag.layernorm(x, blk.norm3), proj.weight, proj.bias))
    return ag.linear(h, blk.ff.net[2].weight, blk.ff.net[2].bias, x)


def _transformer(t2d: modeling.Transformer2DModel, x, ctx, kw):
    NB, H, W, C = x.shape
    h = ag.groupnorm(x, t2d.norm, False)
    h = ag.linear(h, _w1x1(t2d.proj_in), t2d.proj_in.bias).view(NB, H * W, C)
    for blk in t2d.transformer_blocks:
        h = _block(blk, h, ctx, kw)
    return ag.linear(h.view(NB, H, W, C), _w1x1(t2d.proj_out), t2d.proj_out.bias, x)


def _downsample(ds: modeling.Downsample2D, x):
    return ag.linear(ag.Im2colS2.apply(x), ag.pack_conv3x3(ds.conv.weight), ds.conv.bias)


def _upsample(us: modeling.Upsample2D, x):
    return ag.conv3x3(ag.Upsample2x.apply(x), ag.pack_conv3x3(us.conv.weight), us.conv.bias)


def _time_conditioning(unet, NB: int, timestep, device) -> torch.Tensor:
    """[NB, sum(Cout)] fp32: every ResnetBlock2D.time_emb_proj(silu(temb)) in one GEMM (M = batch rows on the tensor core).
    Frozen model: the inference routine; trainable (garment UNet): autograd operators."""
    te = unet.time_embedding
    res = unet._resnets()
    off = 0
    for r in res:
        r.temb_offset = off
        off += r.cout
    if _frozen(te.linear_1.weight, te.linear_2.weight, *[r.time_emb_proj.weight for r in res]):
        with torch.no_grad():
            return unet.time_conditioning(NB, timestep, device)
    dim = unet.config.block_out_channels[0]
    if not torch.is_tensor(timestep):
        timestep = torch.tensor([float(timestep)], device=device)
    t = timestep.reshape(-1).to(device=device, dtype=torch.float32)
    if t.numel() == 1:
        emb = ops.timestep_embedding(t, None, NB, dim)
    else:
        assert t.numel() == NB, "per-sample timesteps must match the batch"
        emb = torch.cat([ops.timestep_embedding(t[i:i + 1], None, 1, dim) for i in range(NB)], 0)
    h = ag.silu(ag.linear(emb.to(BF16), te.linear_1.weight, te.linear_1.bias))
    h = ag.silu(ag.linear(h, te.linear_2.weight, te.linear_2.bias))
    w = torch.cat([ag._bf(r.time_emb_proj.weight) for r in res], 0)
    b = torch.cat([r.time_emb_proj.bias for r in res], 0)
    return ag.linear(h, w, b, None, True)


def unet_forward_train(unet: modeling.UNet2DConditionModel, sample, timestep, encoder_hidden_states,
                       cross_attention_kwargs=None) -> torch.Tensor:
    """Grad-enabled UNet2DConditionModel.forward (diffusers-0.24, called at train.py:259-264 and :272-279): eps fp32 NCHW."""
    kw = cross_attention_kwargs or {}
    NB = sample.shape[0]
    ctx = _bfc(encoder_hidden_states)
    temb_all = _time_conditioning(unet, NB, timestep, sample.device)
    x = ag.ConvIn.apply(modeling._to_tokens(sample.detach()), ag.pack_conv3x3(unet.conv_in.weight), unet.conv_in.bias)
    skips = [x]
    for blk in unet.down_blocks:
        for i, res in enumerate(blk.resnets):
            x = _resnet(res, x, temb_all)
            if blk.has_attn:
                x = _transformer(blk.attentions[i], x, ctx, kw)
            skips.append(x)
        if blk.has_down:
            x = _downsample(blk.downsamplers[0], x)
            skips.append(x)
    mid = unet.mid_block
    x = _resnet(mid.resnets[0], x, temb_all)
    x = _transformer(mid.attentions[0], x, ctx, kw)
    x = _resnet(mid.resnets[1], x, temb_all)
    for blk in unet.up_blocks:
        for i, res in enumerate(blk.resnets):
            x = _resnet(res, ag.Concat.apply(x, skips.pop()), temb_all)
            if blk.has_attn:
                x = _transformer(blk.attentions[i], x, ctx, kw)
        if blk.has_up:
            x = _upsample(blk.upsamplers[0], x)
    x = ag.groupnorm(x, unet.conv_norm_out, True)
    return ag.ConvOut.apply(x, ag.pack_conv3x3(unet.conv_out.weight), unet.conv_out.bias)


# ------------------------------------------------------------------------------------------------ Resampler
def resampler_forward_train(rs, x: torch.Tensor) -> torch.Tensor:
    """Grad-enabled Resampler.forward (adapter/resampler.py:216-236, PerceiverAttention :49-78, FeedForward :13-20)."""
    B = x.shape[0]
    lat = ag._bf(rs.latents).repeat(B, 1, 1).contiguous()
    x = ag.linear(_bfc(x), rs.proj_in.weight, rs.proj_in.bias)
    for attn, ff in rs.layers:
        xn, ln = ag.layernorm(x, attn.norm1), ag.layernorm(lat, attn.norm2)
        q = ag.linear(ln, attn.to_q.weight)
        kv = ag.linear(torch.cat([xn, ln], 1).contiguous(), attn.to_kv.weight)  # to_kv(cat(x, latents)): [B, n1+n2, k | v]
        o = ag.attention(q, kv, None, attn.heads)  # (q d^-1/4)(k d^-1/4)^T == q k^T / sqrt(d)
        lat = ag.linear(o, attn.to_out.weight, None, lat)
        h = ag.gelu(ag.linear(ag.layernorm(lat, ff[0]), ff[1].weight))
        lat = ag.linear(h, ff[3].weight, None, lat)
    return ag.layernorm(ag.linear(lat, rs.proj_out.weight, rs.proj_out.bias), rs.norm_out)


# ------------------------------------------------------------------------------------------------ SDModel
class SDModel(nn.Module):
    """train.py:244-281, same constructor and forward signature."""

    def __init__(self, unet, ref_unet, proj, adapter_modules) -> None:
        super().__init__()
        self.unet = unet
        self.ref_unet = ref_unet
        self.proj = proj
        self.adapter_modules = adapter_modules
        for m in (unet, ref_unet, proj):
            enable_training_path(m)

    def forward(self, encoder_hidden_states, latents, ref_latents, clip_image_embeddings, timesteps):
        ref_timesteps = torch.zeros_like(timesteps)
        cloth_proj_embed = self.proj(clip_image_embeddings)                                      # :257
        _ = self.ref_unet(ref_latents, ref_timesteps, cloth_proj_embed, return_dict=False)      # :259-264
        sa_hidden_states = {name: proc.cache["hidden_states"]                                    # :266-268
                            for name, proc in self.ref_unet.attn_processors.items()}
        return self.unet(latents, timesteps, encoder_hidden_states=encoder_hidden_states,        # :272-279
                         cross_attention_kwargs={"sa_hidden_states": sa_hidden_states}).sample


def hidden_size_of(name: str, block_out_channels) -> int:
    """train.py:341-348."""
    if name.startswith("mid_block"):
        return block_out_channels[-1]
    if name.startswith("up_blocks"):
        return list(reversed(block_out_channels))[int(name[len("up_blocks.")])]
    return block_out_channels[int(name[len("down_blocks.")])]


def install_training_processors(unet, ref_unet) -> nn.ModuleList:
    """train.py:338-366: RefS processors on attn1 (to_k_ref / to_v_ref start as copies of the layer's to_k / to_v), C
    processors on attn2, cache processors on the garment UNet. Returns `adapter_modules`."""
    from adapter.attention_processor import CacheAttnProcessor2_0, CAttnProcessor2_0, RefSAttnProcessor2_0

    st = unet.state_dict()
    procs = {}
    for name in unet.attn_processors.keys():
        hidden = hidden_size_of(name, unet.config.block_out_channels)
        if name.endswith("attn1.processor"):
            p = RefSAttnProcessor2_0(name, hidden)
            layer = name.split(".processor")[0]
            p.load_state_dict({"to_k_ref.weight": st[layer + ".to_k.weight"], "to_v_ref.weight": st[layer + ".to_v.weight"]})
            procs[name] = p
        else:
            procs[name] = CAttnProcessor2_0(name, hidden, unet.config.cross_attention_dim)
    unet.set_attn_processor(procs)
    ref_unet.set_attn_processor({n: CacheAttnProcessor2_0() for n in ref_unet.attn_processors.keys()})
    return nn.ModuleList(unet.attn_processors.values())


def set_trainable(unet, ref_unet, proj, adapter_modules) -> List[nn.Parameter]:
    """train.py:368-379 (order matters: freezing the UNet also freezes the adapter modules registered inside it)."""
    unet.requires_grad_(False)
    proj.requires_grad_(True)
    ref_unet.requires_grad_(True)
    adapter_modules.requires_grad_(True)
    return [*proj.parameters(), *ref_unet.parameters(), *adapter_modules.parameters()]


# ------------------------------------------------------------------------------------------------ optimizer + data parallelism
class FlatAdamW:
    """AdamW over ONE flat buffer: the parameters become bf16 views of `self.param`, their .grad views of `self.grad`;
    fp32 master weights and moments live beside them. With torch.distributed initialised, the gradient buffer is reduced in
    buckets: each parameter's post-accumulate hook counts its bucket down and the completed bucket's all-reduce is launched
    at once (NCCL over NVLink on its own stream), overlapping the remaining backward pass; step() waits for the handles and
    applies the update with the 1/world scale folded into the kernel.

    accumulation_steps = k (train.py:106-111, :606 `--gradient_accumulation_steps`): k micro-steps share one update. The first
    micro-step's gradients are copied into the flat buffer, the following ones added to it (bf16 sums), the bucket all-reduces
    are launched by the LAST micro-step only, step() returns False without touching the weights until then, and 1/k joins
    1/world in the kernel's gradient scale."""

    def __init__(self, params: Iterable[nn.Parameter], lr=1e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2,
                 bucket_bytes: int = 256 << 20, step_fn=None, shard_states: bool = False, accumulation_steps: int = 1):
        seen = set()
        self.params = [p for p in params if p.requires_grad and not (id(p) in seen or seen.add(id(p)))]  # de-duplicated
        assert self.params, "no trainable parameters"
        dev = self.params[0].device
        self.lr, self.betas, self.eps, self.wd = lr, betas, eps, weight_decay
        self.t = 0
        self.accum = max(1, int(accumulation_steps))
        self._micro = 0  # index of the running micro-step inside its accumulation window
        self._step_fn = step_fn  # test hook with the host-scalar signature of ops.adamw_step; None = the device-scalar kernel
        # backward produces gradients roughly in reverse registration order: lay the buffer out reversed so that buckets
        # complete front to back
        order = list(reversed(self.params))
        sizes = [(p.numel() + 7) // 8 * 8 for p in order]  # 16-byte aligned views
        self._dist = torch.distributed.is_available() and torch.distributed.is_initialized() and \
            torch.distributed.get_world_size() > 1
        world = torch.distributed.get_world_size() if self._dist else 1
        rank = torch.distributed.get_rank() if self._dist else 0
        total = (sum(sizes) + 8 * world - 1) // (8 * world) * (8 * world)  # equal, 16-byte aligned shards
        # shard_states (ZeRO-1 style, the reference trains under DeepSpeed ZeRO, train.py:386-398): every rank keeps fp32
        # master weights and moments only for its own 1/world slice of the flat buffer, updates that slice, and the updated
        # bf16 slices meet in one all-gather; without it every rank holds and updates everything (plain data parallelism)
        self.shard = bool(shard_states) and self._dist
        per = total // world
        self._own = (rank * per, (rank + 1) * per) if self.shard else (0, total)
        n_own = self._own[1] - self._own[0]
        self.param = torch.zeros(total, device=dev, dtype=BF16)
        self.grad = torch.zeros(total, device=dev, dtype=BF16)
        self.master = torch.zeros(n_own, device=dev, dtype=torch.float32)
        self.m = torch.zeros(n_own, device=dev, dtype=torch.float32)
        self.v = torch.zeros(n_own, device=dev, dtype=torch.float32)
        # {lr, weight_decay, step, grad_scale} in device memory: what the update kernel reads, so a captured CUDA graph of the
        # step replays with a moving step count / learning-rate schedule (set_lr rewrites it between replays)
        self.hyper = torch.tensor([lr, weight_decay, 0.0, 1.0 / (world * self.accum)], device=dev, dtype=torch.float32)
        off = 0
        self._spans = []
        self._gviews = []  # per parameter: its slot of the flat gradient buffer
        with torch.no_grad():
            for p, n in zip(order, sizes):
                view = self.param[off:off + p.numel()].view(p.shape)
                view.copy_(p.detach())
                p.data = view
                p.grad = None
                self._gviews.append(self.grad[off:off + p.numel()].view(p.shape))
                self._spans.append((off, off + n))
                off += n
            self.master.copy_(self.param[self._own[0]:self._own[1]].float())
        # buckets: contiguous spans of ~bucket_bytes
        per = max(1, bucket_bytes // 2)
        self._buckets, self._bucket_of = [], []
        lo, cnt = 0, 0
        for i, (a, b) in enumerate(self._spans):
            self._bucket_of.append(len(self._buckets))
            cnt += 1
            if b - lo >= per or i == len(self._spans) - 1:
                self._buckets.append([lo, b, cnt])
                lo, cnt = b, 0
        self._pending = [b[2] for b in self._buckets]
        self._ready = [[] for _ in self._buckets]  # per bucket: indices of the parameters whose gradient has arrived
        self._handles = []
        # .grad is None before every backward, so autograd hands each gradient over without an accumulation kernel; the
        # hook of a bucket's last parameter moves the whole bucket into the flat buffer with ONE fused copy and, data
        # parallel, launches its all-reduce at once
        for i, p in enumerate(order):
            p.register_post_accumulate_grad_hook(self._make_hook(i, self._bucket_of[i]))
        self._order = order

    def _flush_bucket(self, bucket: int):
        idx = self._ready[bucket]
        if idx:
            with torch.no_grad():
                if self._micro == 0:
                    torch._foreach_copy_([self._gviews[i] for i in idx], [self._order[i].grad for i in idx])
                else:
                    torch._foreach_add_([self._gviews[i] for i in idx], [self._order[i].grad for i in idx])
            self._ready[bucket] = []
        if self._dist and self._micro == self.accum - 1:
            lo, hi, _ = self._buckets[bucket]
            self._handles.append(torch.distributed.all_reduce(self.grad[lo:hi], async_op=True))

    def _make_hook(self, index: int, bucket: int):
        # weak: a parameter keeps its hooks in the autograd engine's tables, where the garbage collector cannot see a
        # parameter -> hook -> optimizer -> parameter cycle, so a strong reference would keep every flat buffer alive
        ref = weakref.ref(self)

        def hook(_p):
            opt = ref()
            if opt is None:
                return
            opt._ready[bucket].append(index)
            opt._pending[bucket] -= 1
            if opt._pending[bucket] == 0:
                opt._flush_bucket(bucket)
        return hook

    def zero_grad(self):
        """Start of a micro-step. Inside an accumulation window (after its first micro-step) the flat buffer keeps its sums."""
        if self._micro == 0:
            self.grad.zero_()
        for p in self.params:
            p.grad = None
        self._pending = [b[2] for b in self._buckets]
        self._ready = [[] for _ in self._buckets]
        self._handles = []

    def reduce_remaining(self):
        """Buckets whose parameters did not all receive a gradient this step (unused parameters) are completed here."""
        for i, n in enumerate(self._pending):
            if n > 0:
                self._flush_bucket(i)
                self._pending[i] = 0
        for h in self._handles:
            h.wait()
        self._handles = []

    def step(self) -> bool:
        """End of a micro-step; True when the weights were updated (the accumulation window closed)."""
        self.reduce_remaining()
        if self._micro < self.accum - 1:
            self._micro += 1
            return False
        self._micro = 0
        self.t += 1
        world = (torch.distributed.get_world_size() if self._dist else 1) * self.accum
        lo, hi = self._own
        self.hyper[2:3].add_(1.0)  # device-side step count (a kernel, so it is part of a captured graph)
        if self._step_fn is not None:
            self._step_fn(self.master, self.param[lo:hi], self.grad[lo:hi], self.m, self.v, lr=self.lr, beta1=self.betas[0],
                          beta2=self.betas[1], eps=self.eps, weight_decay=self.wd, step=self.t, grad_scale=1.0 / world)
        else:
            ops.adamw_step_dev(self.master, self.param[lo:hi], self.grad[lo:hi], self.m, self.v, self.hyper,
                               beta1=self.betas[0], beta2=self.betas[1], eps=self.eps)
        if self.shard:  # every rank updated its own slice: gather the bf16 working copy
            torch.distributed.all_gather_into_tensor(self.param, self.param[lo:hi].clone())
        # the kernel wrote through raw pointers: bump the version counters so that weight-derived caches keyed on
        # (data_ptr, _version) — processors._ver, autograd._cached — see the update
        torch.autograd.graph.increment_version([self.param, *self.params])
        return True

    def set_lr(self, lr: float, weight_decay: Optional[float] = None) -> None:
        """Learning-rate schedule hook: rewrites the device-side scalars (outside any graph capture)."""
        self.lr = float(lr)
        self.hyper[0:1].fill_(self.lr)
        if weight_decay is not None:
            self.wd = float(weight_decay)
            self.hyper[1:2].fill_(self.wd)

    def reset_state(self) -> None:
        """Moments and step count back to zero (after the warm-up steps of a graph capture)."""
        self.m.zero_()
        self.v.zero_()
        self.hyper[2:3].zero_()
        self.t = 0
        self._micro = 0

    def state_dict(self) -> Dict[str, object]:
        return {"t": self.t, "own": self._own, "master": self.master, "m": self.m, "v": self.v,
                "hyper": dict(lr=self.lr, betas=self.betas, eps=self.eps, weight_decay=self.wd)}

    def load_state_dict(self, sd: Dict[str, object]) -> None:
        if tuple(sd["own"]) != tuple(self._own):
            raise ValueError(f"optimizer shard {tuple(sd['own'])} does not match this rank's {self._own}")
        self.t = int(sd["t"])
        self.hyper[2:3].fill_(float(self.t))
        for name in ("master", "m", "v"):
            getattr(self, name).copy_(sd[name])
        with torch.no_grad():
            self.param[self._own[0]:self._own[1]].copy_(self.master.to(BF16))
        if self.shard:
            torch.distributed.all_gather_into_tensor(self.param, self.param[self._own[0]:self._own[1]].clone())
        torch.autograd.graph.increment_version([self.param, *self.params])


# ------------------------------------------------------------------------------------------------ learning-rate schedule
LR_SCHEDULES = ("linear", "cosine", "cosine_with_restarts", "polynomial", "constant", "constant_with_warmup")  # train.py:129


def lr_multiplier(name: str, step: int, num_warmup_steps: int = 0, num_training_steps: Optional[int] = None,
                  num_cycles: Optional[float] = None, power: float = 1.0, lr_init: float = 1.0, lr_end: float = 1e-7) -> float:
    """The factor on the base learning rate after `step` updates, for the six schedule names train.py:125-130 accepts and
    hands to diffusers.optimization.get_scheduler (train.py:433-439; diffusers==0.24.0 per requirements.txt:12 — not in this
    image; its schedules are the published transformers ones, and tests pin this restatement against
    transformers.optimization.get_scheduler): linear warm-up from 0 over num_warmup_steps, then
      constant / constant_with_warmup : 1
      linear                          : (T - s) / (T - W), floored at 0
      cosine                          : 0.5 (1 + cos(2 pi c p)), c = 0.5 cycles, p = (s - W) / (T - W)
      cosine_with_restarts            : 0.5 (1 + cos(pi (c p mod 1))), c = 1 cycle, 0 once p >= 1
      polynomial                      : ((lr_init - lr_end) (1 - p)^power + lr_end) / lr_init, lr_end / lr_init after T."""
    if name not in LR_SCHEDULES:
        raise ValueError(f"unknown lr scheduler {name!r}; one of {LR_SCHEDULES}")
    s, W = int(step), int(num_warmup_steps)
    if name == "constant":
        return 1.0
    if s < W:
        return s / float(max(1, W))
    if name == "constant_with_warmup":
        return 1.0
    if num_training_steps is None:
        raise ValueError(f"lr scheduler {name!r} needs num_training_steps")
    T = int(num_training_steps)
    if name == "linear":
        return max(0.0, (T - s) / float(max(1, T - W)))
    progress = (s - W) / float(max(1, T - W))
    if name == "cosine":
        c = 0.5 if num_cycles is None else float(num_cycles)
        return max(0.0, 0.5 * (1.0 + math.cos(math.pi * c * 2.0 * progress)))
    if name == "cosine_with_restarts":
        c = 1.0 if num_cycles is None else float(num_cycles)
        if progress >= 1.0:
            return 0.0
        return max(0.0, 0.5 * (1.0 + math.cos(math.pi * ((c * progress) % 1.0))))
    # polynomial
    if s > T:
        return lr_end / lr_init
    remaining = 1.0 - (s - W) / float(T - W)
    return ((lr_init - lr_end) * remaining ** power + lr_end) / lr_init


class LRScheduler:
    """What train.py:433-439 builds and :608 / :618 use: `.step()` after every optimizer update, `.get_lr()[0]` for the log
    line. The new rate goes into FlatAdamW's device-side scalar (set_lr), so a captured step graph replays with it."""

    def __init__(self, name: str, optimizer: FlatAdamW, num_warmup_steps: int = 0, num_training_steps: Optional[int] = None,
                 num_cycles: Optional[float] = None, power: float = 1.0):
        self.name, self.opt = name, optimizer
        self.base_lr = float(optimizer.lr)
        self.kw = dict(num_warmup_steps=num_warmup_steps, num_training_steps=num_training_steps, num_cycles=num_cycles,
                       power=power, lr_init=self.base_lr)
        self.last_epoch = 0
        self._apply()

    def _apply(self) -> None:
        self._lr = self.base_lr * lr_multiplier(self.name, self.last_epoch, **self.kw)
        self.opt.set_lr(self._lr)

    def step(self) -> None:
        self.last_epoch += 1
        self._apply()

    def get_last_lr(self) -> List[float]:
        return [self._lr]

    get_lr = get_last_lr

    def state_dict(self) -> Dict[str, object]:
        return {"last_epoch": self.last_epoch, "base_lr": self.base_lr}

    def load_state_dict(self, sd: Dict[str, object]) -> None:
        self.last_epoch, self.base_lr = int(sd["last_epoch"]), float(sd["base_lr"])
        self.kw["lr_init"] = self.base_lr
        self._apply()


# ------------------------------------------------------------------------------------------------ the callers' side of the step
@torch.no_grad()
def prepare_batch(batch: Dict[str, object], vae, image_encoder, text_encoder, scheduler, device, noise_offset: float = 0.05,
                  generator: Optional[torch.Generator] = None) -> Dict[str, torch.Tensor]:
    """train.py:519-560: the frozen encoders either side of SDModel. VAE-encode person and garment images (latent_dist.sample()
    * 0.18215), draw the noise (+ noise_offset per-channel offset, :530-535) and uniform timesteps, CLIP-vision
    hidden_states[-2] of the garment image (zeros where drop_image_embed, :546-551), CLIP-text last hidden state.
    Returns the keyword arguments of train_step."""
    dt = next(vae.parameters()).dtype if hasattr(vae, "parameters") else torch.float32
    lat = vae.encode(batch["vae_person"].to(device, dtype=dt)).latent_dist.sample() * 0.18215
    ref = vae.encode(batch["vae_clothes"].to(device, dtype=dt)).latent_dist.sample() * 0.18215
    noise = torch.randn(lat.shape, device=device, dtype=torch.float32, generator=generator)
    if noise_offset > 0:
        noise = noise + noise_offset * torch.randn((lat.shape[0], lat.shape[1], 1, 1), device=device, dtype=torch.float32,
                                                   generator=generator)
    n_t = getattr(scheduler, "num_train_timesteps", None) or scheduler.config.num_train_timesteps
    timesteps = torch.randint(0, int(n_t), (lat.shape[0],), device=device, generator=generator).long()
    clip = torch.stack([torch.zeros_like(c) if int(d) == 1 else c
                        for c, d in zip(batch["clip_image"], batch["drop_image_embed"])], 0)
    cdt = next(image_encoder.parameters()).dtype
    image_embeds = image_encoder(clip.to(device, dtype=cdt), output_hidden_states=True).hidden_states[-2]
    text = text_encoder(batch["input_ids"].to(device))[0]
    return dict(latents=lat.float(), ref_latents=ref.float(), clip_image_embeddings=image_embeds,
                encoder_hidden_states=text, noise=noise, timesteps=timesteps)


def save_checkpoint(folder: str, ckpt_id: str, sd_model: "SDModel", optimizer: Optional[FlatAdamW], epoch: int,
                    last_global_step: int, **client_state) -> str:
    """train.py:179-193 (DeepSpeed `model.save_checkpoint(folder, ckpt_id, client_state)`): writes
    `<folder>/<ckpt_id>/mp_rank_00_model_states.pt` whose `["module"]` is SDModel.state_dict() — the `unet.` / `ref_unet.` /
    `proj.` / `adapter_modules.` key layout that inference_IMAGdressing.py:97-117 routes — plus the client state, and one
    optimizer-state file per rank. Returns the model-states path."""
    import os

    d = os.path.join(folder, str(ckpt_id))
    os.makedirs(d, exist_ok=True)
    rank = torch.distributed.get_rank() if torch.distributed.is_available() and torch.distributed.is_initialized() else 0
    path = os.path.join(d, "mp_rank_00_model_states.pt")
    if rank == 0:
        module = {k: v.detach().to("cpu").clone() for k, v in sd_model.state_dict().items()}
        torch.save({"module": module, "epoch": int(epoch), "last_global_step": int(last_global_step), **client_state}, path)
        with open(os.path.join(folder, "latest"), "w") as f:
            f.write(str(ckpt_id))
    if optimizer is not None:
        osd = {k: (v.detach().to("cpu") if torch.is_tensor(v) else v) for k, v in optimizer.state_dict().items()}
        torch.save(osd, os.path.join(d, f"zero_pp_rank_{rank}_mp_rank_00_optim_states.pt"))
    return path


def load_checkpoint(load_dir: str, sd_model: "SDModel", optimizer: Optional[FlatAdamW] = None, tag: Optional[str] = None):
    """train.py:196-207: restores the module (and this rank's optimizer shard); returns (epoch, last_global_step)."""
    import os

    if tag is None:
        with open(os.path.join(load_dir, "latest")) as f:
            tag = f.read().strip()
    d = os.path.join(load_dir, tag)
    st = torch.load(os.path.join(d, "mp_rank_00_model_states.pt"), map_location="cpu", weights_only=False)
    with torch.no_grad():
        own = sd_model.state_dict()
        for k, v in st["module"].items():
            own[k].copy_(v)  # in place: the parameters stay views of the optimizer's flat buffer
    for m in (sd_model.unet, sd_model.ref_unet):
        m.invalidate_packed()
    rank = torch.distributed.get_rank() if torch.distributed.is_available() and torch.distributed.is_initialized() else 0
    if optimizer is not None:
        optimizer.load_state_dict(torch.load(os.path.join(d, f"zero_pp_rank_{rank}_mp_rank_00_optim_states.pt"),
                                             map_location=optimizer.master.device, weights_only=False))
    ag.clear_cache()
    return int(st["epoch"]), int(st["last_global_step"])


def compute_snr(scheduler, timesteps: torch.Tensor) -> torch.Tensor:
    """SNR(t) = abar_t / (1 - abar_t)   (train.py:214-241)."""
    a = scheduler.alphas_cumprod.to(timesteps.device)[timesteps].float()
    return a / (1.0 - a)


def training_loss(pred: torch.Tensor, target: torch.Tensor, scheduler=None, timesteps=None, snr_gamma: float = 0.0):
    """train.py:573-596 for the epsilon objective: plain MSE (snr_gamma == 0, the script's default) or min-SNR-gamma weighting,
    mean_b( mean((pred_b - target_b)^2) * min(snr_b, gamma) / snr_b ) — the per-sample weight enters as sqrt(w_b) on both
    operands of the MSE kernel (mean over all elements of w_b d^2 is the same number)."""
    if snr_gamma == 0:
        return ag.mse_loss(pred.float(), target.float())
    snr = compute_snr(scheduler, timesteps)
    w = (torch.minimum(snr, torch.full_like(snr, float(snr_gamma))) / snr).sqrt().view(-1, *([1] * (pred.dim() - 1)))
    return ag.mse_loss(pred.float() * w, target.float() * w)


def train_step(sd_model: SDModel, scheduler, latents, ref_latents, clip_image_embeddings, encoder_hidden_states, noise,
               timesteps, optimizer: Optional[FlatAdamW] = None, snr_gamma: float = 0.0) -> torch.Tensor:
    """One micro-batch of train.py:527-609 after the frozen VAE / CLIP encoders: add noise, predict, MSE against the noise
    (optionally min-SNR-gamma weighted), backward, (optimizer step). Returns the detached loss."""
    if optimizer is not None:
        optimizer.zero_grad()
    noisy = scheduler.add_noise(latents, noise, timesteps)                                                        # :545
    pred = sd_model(encoder_hidden_states, noisy, ref_latents, clip_image_embeddings, timesteps)                  # :565-571
    loss = training_loss(pred, noise, scheduler, timesteps, snr_gamma)                                             # :575-596
    loss.backward()                                                                                                # :603
    if optimizer is not None:
        optimizer.step()                                                                                           # :604
    return loss.detach()


class GraphedTrainStep:
    """The whole micro-step — optimizer.zero_grad, SDModel forward, MSE, backward (with its gradient hand-over copies and, data
    parallel, the bucket all-reduces), AdamW — captured ONCE as a CUDA graph and replayed per batch: ~5 000 launches per step
    stop costing host time (the eager step is bound by Python + launch overhead, not by the GPU). Inputs live in static
    buffers; the step count and learning rate are device scalars the update kernel reads (FlatAdamW.hyper).

    Warm-up steps (required before capture: lazily built caches, workspace growth, split-K scratch) run with lr = 0 and the
    optimizer state is reset afterwards, so training starts from the given weights at step 1. Construct it BEFORE any eager
    backward of the same parameters on the default stream: autograd's gradient accumulators remember the stream they were
    created on, and one created on the legacy stream cannot take part in a capture (the warm-up here runs on a side stream)."""

    def __init__(self, sd_model: SDModel, scheduler, optimizer: FlatAdamW, example: Dict[str, torch.Tensor], warmup: int = 3):
        self.sd, self.sched, self.opt = sd_model, scheduler, optimizer
        if optimizer.accum != 1:
            raise ValueError("GraphedTrainStep captures one whole update; gradient accumulation runs through train_step")
        self.static = {k: v.detach().clone() for k, v in example.items()}
        self.static["noisy"] = scheduler.add_noise(example["latents"], example["noise"], example["timesteps"]).detach().clone()
        lr = optimizer.lr
        optimizer.set_lr(0.0)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(max(1, warmup)):
                self._body()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        optimizer.zero_grad()
        from . import _lib

        self.graph = torch.cuda.CUDAGraph()
        before = _lib.launch_count
        with torch.cuda.graph(self.graph):
            self.loss = self._body()
        self.launches_per_step = _lib.launch_count - before  # library kernels inside the graph (replays add them to the count)
        torch.cuda.synchronize()
        optimizer.reset_state()
        optimizer.set_lr(lr)

    def _body(self) -> torch.Tensor:
        st = self.static
        self.opt.zero_grad()
        pred = self.sd(st["encoder_hidden_states"], st["noisy"], st["ref_latents"], st["clip_image_embeddings"], st["timesteps"])
        loss = ag.mse_loss(pred.float(), st["noise"].float())
        loss.backward()
        self.opt.step()
        return loss.detach()

    def __call__(self, latents, ref_latents, clip_image_embeddings, encoder_hidden_states, noise, timesteps) -> torch.Tensor:
        st = self.static
        st["noisy"].copy_(self.sched.add_noise(latents, noise, timesteps))  # train.py:545 (outside the graph: table lookup)
        for k, v in (("ref_latents", ref_latents), ("clip_image_embeddings", clip_image_embeddings),
                     ("encoder_hidden_states", encoder_hidden_states), ("noise", noise), ("timesteps", timesteps)):
            st[k].copy_(v)
        self.graph.replay()
        from . import _lib

        _lib.launch_count += self.launches_per_step
        self.opt.t += 1  # (the device-side count advanced inside the graph)
        torch.autograd.graph.increment_version([self.opt.param, *self.opt.params])
        return self.loss
