"""Torch emulations of what the C-ABI kernels compute (bf16 storage, fp32 arithmetic), with the SAME Python signatures
as imagdressing_b200.ops. TEST INFRASTRUCTURE for the CPU suite only: `install(monkeypatch)` swaps them in so the whole
host mirror (modeling.py / processors.py / adapter/*) can be executed — and compared with the oracle — without a GPU.
This checks the host WIRING (weight packing, layouts, fused-epilogue arguments, processor handshake, CFG batching); the
kernels themselves are checked on the GPU against the same oracle."""
import math

import torch
import torch.nn.functional as F

BF = torch.bfloat16
ACT_NONE, ACT_GEGLU, ACT_SILU, ACT_GELU, ACT_QUICK_GELU = 0, 1, 2, 3, 4


def _act(y, act):
    if act == ACT_SILU:
        return F.silu(y)
    if act == ACT_GELU:
        return F.gelu(y)
    if act == ACT_QUICK_GELU:
        return y * torch.sigmoid(1.702 * y)
    return y


def _store(y, out):
    if out is not None:
        out.copy_(y.reshape(out.shape))
        return out
    return y


TILE = 160  # emulated N tile of a row-statistics producer


def gemm_tile_count_n(M, N, K):
    return (N + TILE - 1) // TILE


def gemm(a, w, *, out=None, bias=None, rowvec=None, rows_per_group=0, residual=None, act=ACT_NONE, alpha=1.0,
         out_fp32=False, stats_out=None, ln=None):
    lead = a.shape[:-1]
    y = alpha * (a.reshape(-1, a.shape[-1]).float() @ w.float().T)
    if ln is not None:  # LayerNorm folded into this GEMM: rstd * (acc - mean * colsum) + folded bias
        s = ln.stats[:, :ln.parts].sum(1)
        mean = s[:, 0] / ln.dim
        rstd = torch.rsqrt((s[:, 1] / ln.dim - mean * mean).clamp_min(0) + ln.eps)
        y = rstd[:, None] * (y - mean[:, None] * ln.colsum[None, :]) + bias.float()[None, :]
    elif bias is not None:
        y = y + bias.float()[None, :]
    if rowvec is not None:
        y = y + rowvec.float()[torch.arange(y.shape[0]) // rows_per_group]
    if act == ACT_GEGLU:  # packed rows: per 128, 64 value then their 64 gate
        z = y.view(y.shape[0], -1, 2, 64)
        y = (z[:, :, 0] * F.gelu(z[:, :, 1])).reshape(y.shape[0], -1)
    else:
        y = _act(y, act)
    if residual is not None:
        y = y + residual.reshape(-1, residual.shape[-1]).float()
    if stats_out is not None:  # per-row {sum, sum of squares} of the ROUNDED outputs, one slot per N tile
        yr = y.to(BF).float()
        stats_out.zero_()
        for i, c in enumerate(range(0, yr.shape[1], TILE)):
            stats_out[:, i, 0] = yr[:, c:c + TILE].sum(1)
            stats_out[:, i, 1] = (yr[:, c:c + TILE] ** 2).sum(1)
    y = y.reshape(*lead, y.shape[-1])
    return _store(y if out_fp32 else y.to(BF), out)


def _unpack3x3(w, cin):
    co = w.shape[0]
    return w.float().view(co, 3, 3, cin).permute(0, 3, 1, 2)


def conv3x3(x, w, *, out=None, bias=None, rowvec=None, residual=None, act=ACT_NONE):
    NB, H, W, Cin = x.shape
    y = F.conv2d(x.float().permute(0, 3, 1, 2), _unpack3x3(w, Cin), bias.float() if bias is not None else None, padding=1)
    if rowvec is not None:
        y = y + rowvec.float()[:, :, None, None]
    y = _act(y, act).permute(0, 2, 3, 1)
    if residual is not None:
        y = y + residual.float()
    return _store(y.to(BF).contiguous(), out)


def upconv3x3(x, w_phase, *, bias=None, out=None):
    """Four 2x2 phase convs with the kernel's conventions: phase = py*2+px, tap = ty*2+tx reads (y+py-1+ty, x+px-1+tx)."""
    NB, H, W, Cin = x.shape
    Cout = w_phase.shape[0] // 4
    xin = F.pad(x.float().permute(0, 3, 1, 2), (1, 1, 1, 1))  # zero frame: input row -1 / H, column -1 / W
    wp = w_phase.float().view(4, Cout, 4, Cin)
    y = torch.zeros(NB, Cout, 2 * H, 2 * W)
    for py in (0, 1):
        for px in (0, 1):
            k = wp[py * 2 + px].view(Cout, 2, 2, Cin).permute(0, 3, 1, 2)  # [Cout, Cin, ty, tx]
            win = xin[:, :, py:py + H + 1, px:px + W + 1]  # rows y+py-1 .. y+py (shifted by the pad of 1)
            y[:, :, py::2, px::2] = F.conv2d(win, k)
    if bias is not None:
        y = y + bias.float()[None, :, None, None]
    return _store(y.permute(0, 2, 3, 1).to(BF).contiguous(), out)


def conv3x3_direct(x, w, bias, *, stride=1, act=ACT_NONE, out_nchw_f32=False, add=None, out=None):
    NB, H, W, Cin = x.shape
    y = F.conv2d(x.float().permute(0, 3, 1, 2), _unpack3x3(w, Cin), bias.float() if bias is not None else None,
                 stride=stride, padding=1)
    y = _act(y, act)
    if add is not None:
        y = y + add.float().permute(0, 3, 1, 2)
    if out_nchw_f32:
        return _store(y.contiguous(), out)
    return _store(y.permute(0, 2, 3, 1).to(BF).contiguous(), out)


def groupnorm(x, gamma, beta, groups, eps, *, silu, out=None, ws=None, stats_out=None):
    if stats_out is not None:
        xg = x.float().reshape(x.shape[0], -1, groups, x.shape[-1] // groups)
        stats_out[:, :, 0] = xg.mean((1, 3))
        stats_out[:, :, 1] = torch.rsqrt(xg.var((1, 3), unbiased=False) + eps)
    y = F.group_norm(x.float().movedim(-1, 1), groups, gamma, beta, eps)
    if silu:
        y = F.silu(y)
    return _store(y.movedim(1, -1).to(BF).contiguous(), out)


def layernorm(x, gamma, beta, eps=1e-5, *, out=None):
    return _store(F.layer_norm(x.float(), (x.shape[-1],), gamma, beta, eps).to(BF), out)


class Stream:
    def __init__(self, k, v, length, sample_rows=0, broadcast=False, n_query_samples=1 << 30, out_scale=1.0):
        self.k, self.v, self.length, self.sample_rows = k, v, length, sample_rows or length
        self.broadcast, self.n_query_samples, self.out_scale = broadcast, n_query_samples, out_scale


def kv_stream(k, v, length, **kw):
    return Stream(k, v, length, **kw)


def attention(q, B, Lq, heads, head_dim, s0, s1=None, *, sm_scale=None, out=None, causal=False):
    C = heads * head_dim
    scale = sm_scale if sm_scale is not None else head_dim ** -0.5
    qf = q[:, :C].float().reshape(B, Lq, heads, head_dim).transpose(1, 2)

    def one(s, b):
        src = 0 if s.broadcast else b
        rows = slice(src * s.sample_rows, src * s.sample_rows + s.length)
        k = s.k[rows, :C].float().reshape(s.length, heads, head_dim).transpose(0, 1)
        v = s.v[rows, :C].float().reshape(s.length, heads, head_dim).transpose(0, 1)
        # 4-D inputs select torch's fused CPU kernel (no Lq x L matrix; ~10x faster than the 3-D math path)
        return F.scaled_dot_product_attention(qf[b][None], k[None], v[None], scale=scale, is_causal=causal)[0]

    rows = []
    for b in range(B):
        o = s0.out_scale * one(s0, b)
        if s1 is not None and b < s1.n_query_samples:
            o = o + s1.out_scale * one(s1, b)
        rows.append(o.transpose(0, 1).reshape(Lq, C))
    return _store(torch.stack(rows).reshape(B * Lq, C).to(BF), out)


def concat_add(a, b=None, *, res_a=None, res_b=None, out=None):
    add = lambda t, r: t if r is None else (t.float() + r.float()).to(BF)
    parts = [add(a, res_a)] + ([add(b, res_b)] if b is not None else [])
    return _store(torch.cat(parts, -1).contiguous(), out)


def upsample2x(x):
    return x.repeat_interleave(2, 1).repeat_interleave(2, 2).contiguous()


def embed_tokens(ids, tok, pos):
    return (tok.float()[ids] + pos.float()[: ids.shape[1]][None]).to(BF)


def patchify(x, patch, kpad):
    B, C, H, W = x.shape
    cols = F.unfold(x.float(), patch, stride=patch).transpose(1, 2).reshape(-1, C * patch * patch)  # (c, iy, ix) order
    return F.pad(cols, (0, kpad - cols.shape[1])).to(BF).contiguous()


def broadcast_row(vec, out, row):
    out[:, row, :] = vec
    return out


def softmax_rows(s, scale=1.0, *, out=None):
    return _store(torch.softmax(s.float() * scale, -1).to(BF), out)


def im2col3x3_s2(x, pad_lo=1):
    NB, H, W, C = x.shape
    xin = x.float().permute(0, 3, 1, 2)
    if pad_lo == 0:  # VAE encoder: right / bottom padding only
        xin = F.pad(xin, (0, 1, 0, 1))
    cols = F.unfold(xin, 3, padding=1 if pad_lo == 1 else 0, stride=2)  # [NB, C*9, L], channel-major (c*9 + tap)
    cols = cols.view(NB, C, 9, H // 2, W // 2).permute(0, 3, 4, 2, 1)          # -> tap-major (tap*C + c)
    return cols.reshape(NB, H // 2, W // 2, 9 * C).to(BF).contiguous()


def nchw_f32_to_nhwc_bf16(x, cpad=None, *, repeat=1, out=None):
    NB, C, H, W = x.shape
    y = x.permute(0, 2, 3, 1)
    if cpad and cpad > C:
        y = F.pad(y, (0, cpad - C))
    return _store(y.repeat(repeat, 1, 1, 1).to(BF).contiguous(), out)


def timestep_embedding(timesteps, step_ptr, NB, dim, *, out=None):
    t = timesteps[int(step_ptr[0])] if step_ptr is not None else timesteps[0]
    half = dim // 2
    freqs = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=torch.float32) / half)
    args = t.float() * freqs
    return _store(torch.cat([torch.cos(args), torch.sin(args)])[None].repeat(NB, 1), out)


def linear_small_m(x, w, bias, *, act_in=ACT_NONE, act_out=ACT_NONE, out=None):
    y = _act(x.float(), act_in) @ w.float().T
    if bias is not None:
        y = y + bias.float()
    return _store(_act(y, act_out), out)


def cfg_ddim_step(eps_cond, eps_uncond, guidance, latents, coef, step_ptr, *, mask=None, image_latents=None, noise=None,
                  blend_coef=None):
    i = int(step_ptr[0])
    c = coef[i]
    eps = eps_cond if eps_uncond is None else eps_uncond + guidance * (eps_cond - eps_uncond)
    x0 = (latents - c[1] * eps) / c[0]
    new = c[2] * x0 + c[3] * eps
    if mask is not None:  # inpaint blend with the original latents re-noised to the NEXT timestep (last step: clean)
        b = blend_coef[i]
        new = (1 - mask) * (b[0] * image_latents + b[1] * noise) + mask * new
    latents.copy_(new)
    step_ptr[0] += 1
    return latents


# ====================================================================================================== training step
# Emulations of the backward / training kernels with EXPLICIT formulas (the ones the CUDA kernels implement), not torch
# autograd: the CPU training tests then check both the autograd wiring and the backward algebra against the oracle's autograd.
class AttnSaved:
    def __init__(self, lse, o0, o1, lq_pad, out):
        self.lse, self.o0, self.o1, self.lq_pad, self.out = lse, o0, o1, lq_pad, out


def _heads(t, rows, heads, hd):
    return t.float().reshape(rows, heads, hd).transpose(0, 1)  # [heads, rows, hd]


def _stream_kv(s, b, C, heads, hd):
    rows = slice(b * s.sample_rows, b * s.sample_rows + s.length)
    return _heads(s.k[rows, :C], s.length, heads, hd), _heads(s.v[rows, :C], s.length, heads, hd)


def attention_train(q, B, Lq, heads, head_dim, s0, s1=None, *, sm_scale=None):
    C = heads * head_dim
    scale = sm_scale if sm_scale is not None else head_dim ** -0.5
    lq_pad = (Lq + 127) // 128 * 128
    lse = torch.full((2, B, heads, lq_pad), float("inf"))
    outs = [torch.zeros(B * Lq, C), torch.zeros(B * Lq, C)]
    for b in range(B):
        qh = _heads(q[b * Lq:(b + 1) * Lq, :C], Lq, heads, head_dim)
        for si, s in enumerate((s0, s1)):
            if s is None:
                continue
            assert not s.broadcast and s.n_query_samples >= B
            k, v = _stream_kv(s, b, C, heads, head_dim)
            sc = qh @ k.transpose(1, 2) * scale
            lse[si, b, :, :Lq] = torch.logsumexp(sc, -1) / math.log(2.0)
            o = torch.softmax(sc, -1) @ v
            outs[si][b * Lq:(b + 1) * Lq] = o.transpose(0, 1).reshape(Lq, C)
    out = s0.out_scale * outs[0] + (s1.out_scale * outs[1] if s1 is not None else 0)
    two = s1 is not None
    return out.to(BF), AttnSaved(lse, outs[0].to(BF) if two else None, outs[1].to(BF) if two else None, lq_pad, out.to(BF))


def attention_bwd(q, d_out, B, Lq, heads, head_dim, s0, s1, saved, *, sm_scale=None, dq=None, dkv0=None, dkv1=None):
    """P = exp2(S s log2e - lse2); dP = w dO V^T; D = w rowsum(dO o O_s); dS = P (dP - D); dQ += s dS K; dK = s dS^T Q; dV = w P^T dO
    with P and dS rounded to bf16 before the second products, as in the kernels."""
    C = heads * head_dim
    scale = sm_scale if sm_scale is not None else head_dim ** -0.5
    r = lambda t: t.to(BF).float()
    for b in range(B):
        rows = slice(b * Lq, (b + 1) * Lq)
        qh = _heads(q[rows, :C], Lq, heads, head_dim)
        doh = _heads(d_out[rows, :C], Lq, heads, head_dim)
        dq_acc = torch.zeros(heads, Lq, head_dim)
        for si, (s, pair) in enumerate(((s0, dkv0), (s1, dkv1))):
            if s is None:
                continue
            w = s.out_scale
            k, v = _stream_kv(s, b, C, heads, head_dim)
            if s1 is not None:
                os_ = (saved.o0 if si == 0 else saved.o1)[rows].float()
                D = w * (doh * _heads(os_, Lq, heads, head_dim)).sum(-1, keepdim=True)
            else:
                D = (doh * _heads(saved.out[rows], Lq, heads, head_dim)).sum(-1, keepdim=True)
            P = torch.exp2(qh @ k.transpose(1, 2) * scale * math.log2(math.e) - saved.lse[si, b, :, :Lq, None])
            dS = r(P * (w * (doh @ v.transpose(1, 2)) - D))
            dq_acc += dS @ k
            if pair is not None:
                krows = slice(b * s.sample_rows, b * s.sample_rows + s.length)
                pair[0][krows, :C] = (scale * (dS.transpose(1, 2) @ qh)).transpose(0, 1).reshape(s.length, C).to(BF)
                pair[1][krows, :C] = (w * (r(P).transpose(1, 2) @ doh)).transpose(0, 1).reshape(s.length, C).to(BF)
        if dq is not None:
            dq[rows, :C] = (scale * dq_acc).transpose(0, 1).reshape(Lq, C).to(BF)


def transpose(x, pad_to=8, out=None):
    rows, cols = x.shape
    if out is not None:
        out.copy_(x.t())
        return out
    rp = (rows + pad_to - 1) // pad_to * pad_to
    out = torch.zeros(cols, rp, dtype=BF)
    out[:, :rows] = x.t()
    return out


def conv_weight_flip(wp, cin):
    co = wp.shape[0]
    return wp.view(co, 9, cin).flip(1).permute(2, 1, 0).reshape(cin, 9 * co).contiguous()


def conv_weight_layout(w, mode):
    if mode == 0:
        co, ci = w.shape[:2]
        return w.permute(0, 2, 3, 1).reshape(co, 9 * ci).contiguous()
    co, ci = w.shape[0], w.shape[1] // 9
    return w.view(co, 3, 3, ci).permute(0, 3, 1, 2).contiguous()


def im2col3x3_t(x):
    NB, H, W, C = x.shape
    P = NB * H * W
    cols = F.unfold(x.float().permute(0, 3, 1, 2), 3, padding=1).view(NB, C, 9, H * W).permute(2, 1, 0, 3).reshape(9 * C, P)
    out = torch.zeros((9 * C + 7) // 8 * 8, (P + 7) // 8 * 8, dtype=BF)
    out[:9 * C, :P] = cols.to(BF)
    return out


def col2im3x3_s2(dcol, H, W):
    NB, Ho, Wo, C9 = dcol.shape
    C = C9 // 9
    cols = dcol.float().view(NB, Ho * Wo, 9, C).permute(0, 3, 2, 1).reshape(NB, C * 9, Ho * Wo)  # channel-major for fold
    return F.fold(cols, (H, W), 3, padding=1, stride=2).permute(0, 2, 3, 1).to(BF).contiguous()


def downsum2x(dy):
    NB, H2, W2, C = dy.shape
    return dy.float().view(NB, H2 // 2, 2, W2 // 2, 2, C).sum((2, 4)).to(BF)


def colsum(x, rows_per_group=None, out_dtype=torch.float32):
    x2 = x.reshape(-1, x.shape[-1]).float()
    rpg = x2.shape[0] if rows_per_group is None else rows_per_group
    return x2.view(-1, rpg, x2.shape[1]).sum(1).to(out_dtype)


def layernorm_bwd(x, dy, gamma, eps, need_affine, out_dtype=torch.float32):
    xf, g = x.float(), dy.float() * (gamma.float() if gamma is not None else 1.0)
    mean = xf.mean(-1, keepdim=True)
    rstd = torch.rsqrt(xf.var(-1, unbiased=False, keepdim=True) + eps)
    xh = (xf - mean) * rstd
    dx = rstd * (g - g.mean(-1, keepdim=True) - xh * (g * xh).mean(-1, keepdim=True))
    C = x.shape[-1]
    if not need_affine:
        return dx.to(BF), None, None
    return dx.to(BF), (dy.float() * xh).reshape(-1, C).sum(0).to(out_dtype), dy.float().reshape(-1, C).sum(0).to(out_dtype)


def _dsilu(z):
    s = torch.sigmoid(z)
    return s * (1 + z * (1 - s))


def groupnorm_bwd(x, dy, gamma, beta, groups, stats, silu, need_affine, out_dtype=torch.float32):
    NB, C = x.shape[0], x.shape[-1]
    xf = x.float().reshape(NB, -1, groups, C // groups)
    mean = stats[:, :, 0].reshape(NB, 1, groups, 1)
    rstd = stats[:, :, 1].reshape(NB, 1, groups, 1)
    xh = ((xf - mean) * rstd).reshape(NB, -1, C)
    dz = dy.float().reshape(NB, -1, C)
    if silu:
        dz = dz * _dsilu(xh * gamma.float() + beta.float())
    g = (dz * gamma.float()).reshape(NB, -1, groups, C // groups)
    xg = xh.reshape(NB, -1, groups, C // groups)
    dx = rstd * (g - g.mean((1, 3), keepdim=True) - xg * (g * xg).mean((1, 3), keepdim=True))
    dx = dx.reshape(x.shape).to(BF)
    if not need_affine:
        return dx, None, None
    return dx, (dz * xh).sum((0, 1)).to(out_dtype), dz.sum((0, 1)).to(out_dtype)


def _dgelu(x):
    return 0.5 * (1 + torch.erf(x / math.sqrt(2.0))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)


def act(x, mode, dy=None):
    xf = x.float()
    if dy is None:
        return _act(xf, mode).to(BF)
    return (dy.float() * (_dsilu(xf) if mode == ACT_SILU else _dgelu(xf))).to(BF)


def geglu(h, dout=None):
    v, g = h.float().chunk(2, -1)
    if dout is None:
        return (v * F.gelu(g)).to(BF)
    d = dout.float()
    return torch.cat([d * F.gelu(g), d * v * _dgelu(g)], -1).to(BF)


def mse_loss_grad(pred, target, grad_scale=1.0):
    d = pred - target
    return (d * d).mean().reshape(1), grad_scale * 2.0 * d / d.numel()


def adamw_step(master, param, grad, m, v, *, lr, beta1, beta2, eps, weight_decay, step, grad_scale=1.0):
    g = grad.float() * grad_scale
    m.mul_(beta1).add_(g, alpha=1 - beta1)
    v.mul_(beta2).addcmul_(g, g, value=1 - beta2)
    master.mul_(1 - lr * weight_decay)
    master.addcdiv_(m / (1 - beta1 ** step), (v / (1 - beta2 ** step)).sqrt() + eps, value=-lr)
    param.copy_(master.to(BF))


def adamw_step_dev(master, param, grad, m, v, hyper, *, beta1, beta2, eps):
    adamw_step(master, param, grad, m, v, lr=float(hyper[0]), beta1=beta1, beta2=beta2, eps=eps, weight_decay=float(hyper[1]),
               step=int(round(float(hyper[2]))), grad_scale=float(hyper[3]))


TRAIN_OPS = ("adamw_step_dev", "attention_train", "attention_bwd", "transpose", "conv_weight_layout", "conv_weight_flip", "im2col3x3_t", "col2im3x3_s2", "downsum2x", "colsum",
             "layernorm_bwd", "groupnorm_bwd", "act", "geglu", "mse_loss_grad", "adamw_step")


def install(monkeypatch):
    from imagdressing_b200 import ops

    for name in ("gemm", "conv3x3", "conv3x3_direct", "groupnorm", "layernorm", "kv_stream", "attention", "concat_add",
                 "upsample2x", "im2col3x3_s2", "nchw_f32_to_nhwc_bf16", "timestep_embedding", "linear_small_m",
                 "cfg_ddim_step", "gemm_tile_count_n", "upconv3x3", "softmax_rows", "embed_tokens", "patchify", "broadcast_row",
                 *TRAIN_OPS):
        monkeypatch.setattr(ops, name, globals()[name])
