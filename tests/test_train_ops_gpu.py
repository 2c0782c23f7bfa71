"""GPU parity of the training-step kernels (SURVEY.md section 8 row a13) through the C ABI, each against torch fp32 autograd of the
same operator on the same bf16-rounded inputs: two-stream attention backward (dQ, dK, dV, dK_ref, dV_ref) at every head
dim / ragged length the UNets and the Resampler use, GroupNorm / LayerNorm / activation backward, the layout kernels that
feed the dgrad / wgrad GEMMs, column sums, MSE loss + gradient, AdamW. Tolerances: bf16 outputs of fp32 accumulations ->
rel-L2 <= 1e-2 (attention 2e-2: P and dS are rounded to bf16 before the second products, as in every flash backward)."""
import math

import pytest
import torch
import torch.nn.functional as F

from conftest import rel_l2

pytestmark = pytest.mark.gpu
BF = torch.bfloat16


def rnd(shape, dev, seed, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(BF).to(dev)


def ref_attention(q, k0, v0, k1, v1, heads, w0, w1):
    """fp32 torch: q [B, L, C]; k*, v* [B, Lk, C]."""
    B, L, C = q.shape
    hd = C // heads
    sp = lambda t: t.reshape(t.shape[0], t.shape[1], heads, hd).transpose(1, 2)
    o = w0 * F.scaled_dot_product_attention(sp(q), sp(k0), sp(v0))
    if k1 is not None:
        o = o + w1 * F.scaled_dot_product_attention(sp(q), sp(k1), sp(v1))
    return o.transpose(1, 2).reshape(B, L, C)


@pytest.mark.parametrize("heads,hd,B,L,Lk1,w1", [
    (8, 40, 2, 256, 256, 1.0),      # level 0, two streams, full tiles
    (8, 40, 2, 200, 150, 0.7),      # ragged query / key tiles
    (8, 80, 2, 320, 320, 1.0),      # level 1 (640 x 512 latents: 1280 / 4)
    (8, 160, 2, 80, 80, 0.9),       # level 3 (one ragged tile)
    (8, 160, 1, 320, 320, 1.0),     # level 2
    (8, 40, 2, 384, 0, 0.0),        # self-attention, one stream
    (12, 64, 2, 16, 0, 0.0),        # Perceiver geometry (Lq 16; keys 273 below)
])
def test_attention_backward_matches_autograd(cuda_device, heads, hd, B, L, Lk1, w1):
    from imagdressing_b200 import ops

    dev = cuda_device
    C = heads * hd
    perceiver = heads == 12
    Lk0 = 273 if perceiver else L
    if perceiver:
        qbuf = rnd((B, L, C), dev, 1)
        kv0 = rnd((B, Lk0, 2 * C), dev, 2)
        q2 = qbuf.view(B * L, C)
        k0v, v0v = kv0.view(B * Lk0, 2 * C)[:, :C], kv0.view(B * Lk0, 2 * C)[:, C:]
        qf, k0f, v0f = qbuf.float(), kv0[..., :C].float(), kv0[..., C:].float()
    else:  # fused q|k|v projection output, as the processors produce it
        qkv = rnd((B, L, 3 * C), dev, 1)
        flat = qkv.view(B * L, 3 * C)
        q2, k0v, v0v = flat[:, :C], flat[:, C:2 * C], flat[:, 2 * C:]
        qf, k0f, v0f = qkv[..., :C].float(), qkv[..., C:2 * C].float(), qkv[..., 2 * C:].float()
    s0 = ops.kv_stream(k0v, v0v, Lk0)
    s1 = None
    k1f = v1f = None
    if Lk1 > 0:
        kv1 = rnd((B, Lk1, 2 * C), dev, 3)
        f1 = kv1.view(B * Lk1, 2 * C)
        s1 = ops.kv_stream(f1[:, :C], f1[:, C:], Lk1, out_scale=w1)
        k1f, v1f = kv1[..., :C].float(), kv1[..., C:].float()
    d_out = rnd((B * L, C), dev, 4)

    out, saved = ops.attention_train(q2, B, L, heads, hd, s0, s1)
    base = ops.attention(q2, B, L, heads, hd, s0, s1)
    leaves = [t.clone().requires_grad_(True) for t in (qf, k0f, v0f)] + (
        [k1f.clone().requires_grad_(True), v1f.clone().requires_grad_(True)] if Lk1 > 0 else [])
    ref = ref_attention(leaves[0], leaves[1], leaves[2], leaves[3] if Lk1 > 0 else None, leaves[4] if Lk1 > 0 else None,
                        heads, 1.0, w1)
    assert rel_l2(out.view(B, L, C), ref) < 1e-2
    assert torch.equal(out, base)  # the inference and training forwards run the same kernel
    # log-sum-exp rows (log2 domain) of stream 0
    sp = lambda t: t.reshape(t.shape[0], t.shape[1], heads, hd).transpose(1, 2)
    lse_ref = torch.logsumexp(sp(qf) @ sp(k0f).transpose(-1, -2) * hd ** -0.5, -1) / math.log(2.0)
    assert torch.allclose(saved.lse[0, :, :, :L], lse_ref, atol=2e-2, rtol=1e-3)
    assert torch.isinf(saved.lse[0, :, :, L:]).all()

    ref.backward(d_out.view(B, L, C).float())
    if perceiver:
        dq = torch.zeros(B * L, C, device=dev, dtype=BF)
        dkv0 = torch.zeros(B * Lk0, 2 * C, device=dev, dtype=BF)
        ops.attention_bwd(q2, d_out, B, L, heads, hd, s0, s1, saved, dq=dq, dkv0=(dkv0[:, :C], dkv0[:, C:]))
        got = [dq.view(B, L, C), dkv0.view(B, Lk0, 2 * C)[..., :C], dkv0.view(B, Lk0, 2 * C)[..., C:]]
    else:
        dqkv = torch.zeros(B * L, 3 * C, device=dev, dtype=BF)
        dkv1 = torch.zeros(B * Lk1, 2 * C, device=dev, dtype=BF) if Lk1 > 0 else None
        ops.attention_bwd(q2, d_out, B, L, heads, hd, s0, s1, saved, dq=dqkv[:, :C],
                          dkv0=(dqkv[:, C:2 * C], dqkv[:, 2 * C:]),
                          dkv1=(dkv1[:, :C], dkv1[:, C:]) if Lk1 > 0 else None)
        v = dqkv.view(B, L, 3 * C)
        got = [v[..., :C], v[..., C:2 * C], v[..., 2 * C:]]
        if Lk1 > 0:
            w = dkv1.view(B, Lk1, 2 * C)
            got += [w[..., :C], w[..., C:]]
    names = ["dq", "dk", "dv", "dk_ref", "dv_ref"]
    for name, g, leaf in zip(names, got, leaves):
        assert torch.isfinite(g.float()).all(), name
        err = rel_l2(g, leaf.grad)
        assert err < 2e-2, f"{name}: rel-L2 {err}"


def test_cross_attention_backward_windowed_context(cuda_device):
    """77 text keys inside an 81-token context (sample_rows > len), query gradient only — the frozen UNet's attn2."""
    from imagdressing_b200 import ops

    dev = cuda_device
    heads, hd, B, L, Lc, Lt = 8, 40, 2, 256, 81, 77
    C = heads * hd
    q = rnd((B, L, C), dev, 1)
    kv = rnd((B, Lc, 2 * C), dev, 2)
    f = kv.view(B * Lc, 2 * C)
    s0 = ops.kv_stream(f[:, :C], f[:, C:], Lt, sample_rows=Lc)
    d_out = rnd((B * L, C), dev, 3)
    out, saved = ops.attention_train(q.view(B * L, C), B, L, heads, hd, s0)
    ql = q.float().clone().requires_grad_(True)
    ref = ref_attention(ql, kv[:, :Lt, :C].float(), kv[:, :Lt, C:].float(), None, None, heads, 1.0, 0.0)
    ref.backward(d_out.view(B, L, C).float())
    dq = torch.zeros(B * L, C, device=dev, dtype=BF)
    ops.attention_bwd(q.view(B * L, C), d_out, B, L, heads, hd, s0, None, saved, dq=dq)
    assert rel_l2(out.view(B, L, C), ref) < 1e-2
    assert rel_l2(dq.view(B, L, C), ql.grad) < 2e-2


def test_layout_kernels(cuda_device):
    from imagdressing_b200 import ops

    dev = cuda_device
    x = rnd((203, 136), dev, 1)
    t = ops.transpose(x)
    assert t.shape == (136, 208) and torch.equal(t[:, :203], x.t()) and (t[:, 203:] == 0).all()
    xs = rnd((100, 400), dev, 2)[:, 64:192]  # column slice (row stride 400)
    assert torch.equal(ops.transpose(xs)[:, :100], xs.t())

    big = rnd((1000, 328), dev, 21)                      # ragged in both directions, 16-byte-aligned strides
    assert torch.equal(ops.transpose(big)[:, :1000], big.t())
    w = rnd((96, 64, 3, 3), dev, 22)
    wp = ops.conv_weight_layout(w, 0)
    assert torch.equal(wp, w.permute(0, 2, 3, 1).reshape(96, 576))
    assert torch.equal(ops.conv_weight_layout(wp, 1), w)
    dst = torch.zeros(64, 9 * 96, device=dev, dtype=BF)
    for t in range(9):                                   # the dgrad tap flip: strided source and destination views
        ops.transpose(wp[:, t * 64:(t + 1) * 64], out=dst[:, (8 - t) * 96:(9 - t) * 96])
    assert torch.equal(dst, wp.view(96, 9, 64).flip(1).permute(2, 1, 0).reshape(64, 864))
    assert torch.equal(ops.conv_weight_flip(wp, 64), dst)
    w4 = rnd((4, 9 * 320), dev, 23)                      # conv_out's dgrad weight: Cout = 4
    assert torch.equal(ops.conv_weight_flip(w4, 320), w4.view(4, 9, 320).flip(1).permute(2, 1, 0).reshape(320, 36))

    a = rnd((2, 6, 10, 64), dev, 3)
    col = ops.im2col3x3_t(a)
    ref = F.unfold(a.float().permute(0, 3, 1, 2), 3, padding=1)          # [NB, C*9, HW], row = c*9 + tap
    ref = ref.view(2, 64, 9, 60).permute(2, 1, 0, 3).reshape(9 * 64, 120)  # row = tap*C + c, col = n*HW + p
    assert torch.equal(col.float(), ref)
    a4 = rnd((2, 4, 4, 4), dev, 4)                                         # conv_in geometry: C = 4 -> 36 rows padded to 40
    col4 = ops.im2col3x3_t(a4)
    ref4 = F.unfold(a4.float().permute(0, 3, 1, 2), 3, padding=1).view(2, 4, 9, 16).permute(2, 1, 0, 3).reshape(36, 32)
    assert col4.shape == (40, 32) and torch.equal(col4[:36].float(), ref4) and (col4[36:] == 0).all()

    # col2im is the adjoint of im2col3x3_s2: <im2col(x), d> == <x, col2im(d)>
    xi = rnd((2, 8, 12, 64), dev, 5)
    d = rnd((2, 4, 6, 9 * 64), dev, 6)
    lhs = (ops.im2col3x3_s2(xi).float() * d.float()).sum()
    rhs = (xi.float() * ops.col2im3x3_s2(d, 8, 12).float()).sum()
    assert abs(float(lhs - rhs)) < 2e-2 * abs(float(lhs)) + 1.0
    xr = xi.float().permute(0, 3, 1, 2).clone().requires_grad_(True)
    colr = F.unfold(xr, 3, padding=1, stride=2).view(2, 64, 9, 4, 6).permute(0, 3, 4, 2, 1).reshape(2, 4, 6, 576)
    colr.backward(d.float())
    assert rel_l2(ops.col2im3x3_s2(d, 8, 12), xr.grad.permute(0, 2, 3, 1)) < 5e-3

    up = rnd((2, 8, 12, 64), dev, 7)
    want = up.float().view(2, 4, 2, 6, 2, 64).sum((2, 4))
    assert rel_l2(ops.downsum2x(up), want) < 5e-3

    y = rnd((2 * 96, 320), dev, 8)
    assert rel_l2(ops.colsum(y), y.float().sum(0, keepdim=True)) < 1e-5
    assert rel_l2(ops.colsum(y, 96), y.float().view(2, 96, 320).sum(1)) < 1e-5
    big = rnd((4 * 5120, 320), dev, 9)
    assert rel_l2(ops.colsum(big, 5120), big.float().view(4, 5120, 320).sum(1)) < 1e-5
    assert torch.equal(ops.colsum(big), ops.colsum(big))  # fixed-order: bit-reproducible
    assert torch.equal(ops.colsum(big, None, BF), ops.colsum(big).to(BF))  # bf16 output = the rounded fp32 result


@pytest.mark.parametrize("C,HW,groups,silu", [(320, 320, 32, True), (640, 80, 32, True), (1280, 20, 32, False),
                                               (1920, 80, 32, True), (960, 320, 32, True), (2560, 20, 32, True)])
def test_groupnorm_backward(cuda_device, C, HW, groups, silu):
    from imagdressing_b200 import ops

    dev = cuda_device
    x = (rnd((2, HW, C), dev, 1) * 1.5 + 0.5).to(BF)
    dy = rnd((2, HW, C), dev, 2)
    gamma = (1 + 0.1 * torch.randn(C, generator=torch.Generator().manual_seed(3))).to(dev)
    beta = (0.1 * torch.randn(C, generator=torch.Generator().manual_seed(4))).to(dev)
    xl, gl, bl = x.float().clone().requires_grad_(True), gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    y = F.group_norm(xl.movedim(-1, 1), groups, gl, bl, 1e-5)
    if silu:
        y = F.silu(y)
    y.movedim(1, -1).backward(dy.float())
    stats = torch.empty(2, groups, 2, device=dev, dtype=torch.float32)
    fwd = ops.groupnorm(x, gamma, beta, groups, 1e-5, silu=silu, stats_out=stats)
    assert rel_l2(fwd, y.detach().movedim(1, -1)) < 1e-2
    xg = x.float().view(2, HW, groups, C // groups)
    assert rel_l2(stats[:, :, 0], xg.mean((1, 3))) < 1e-4
    assert rel_l2(stats[:, :, 1], torch.rsqrt(xg.var((1, 3), unbiased=False) + 1e-5)) < 1e-4
    dx, dg, db = ops.groupnorm_bwd(x, dy, gamma, beta, groups, stats, silu, True)
    assert rel_l2(dx, xl.grad) < 1e-2
    assert rel_l2(dg, gl.grad) < 2e-3 and rel_l2(db, bl.grad) < 2e-3
    dx2, none_g, _ = ops.groupnorm_bwd(x, dy, gamma, beta, groups, stats, silu, False)
    assert none_g is None and torch.equal(dx, dx2)


@pytest.mark.parametrize("rows,C", [(640, 320), (77, 768), (1000, 1280), (32, 1280)])
def test_layernorm_backward(cuda_device, rows, C):
    from imagdressing_b200 import ops

    dev = cuda_device
    x = (rnd((rows, C), dev, 1) * 2 + 1).to(BF)
    dy = rnd((rows, C), dev, 2)
    gamma = (1 + 0.1 * torch.randn(C, generator=torch.Generator().manual_seed(3))).to(dev)
    beta = (0.1 * torch.randn(C, generator=torch.Generator().manual_seed(4))).to(dev)
    xl, gl, bl = x.float().clone().requires_grad_(True), gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    F.layer_norm(xl, (C,), gl, bl, 1e-5).backward(dy.float())
    dx, dg, db = ops.layernorm_bwd(x, dy, gamma, 1e-5, True)
    assert rel_l2(dx, xl.grad) < 1e-2
    assert rel_l2(dg, gl.grad) < 2e-3 and rel_l2(db, bl.grad) < 2e-3


def test_activations_and_geglu(cuda_device):
    from imagdressing_b200 import ops
    from imagdressing_b200._lib import ACT_GELU, ACT_SILU

    dev = cuda_device
    x = rnd((333, 129), dev, 1, 2.0).contiguous()
    dy = rnd((333, 129), dev, 2)
    for mode, fn in ((ACT_SILU, F.silu), (ACT_GELU, F.gelu)):
        xl = x.float().clone().requires_grad_(True)
        y = fn(xl)
        y.backward(dy.float())
        assert rel_l2(ops.act(x, mode), y) < 5e-3
        assert rel_l2(ops.act(x, mode, dy), xl.grad) < 5e-3
    h = rnd((50, 2 * 1280), dev, 3, 1.5)
    d = rnd((50, 1280), dev, 4)
    hl = h.float().clone().requires_grad_(True)
    v, g = hl.chunk(2, -1)
    out = v * F.gelu(g)
    out.backward(d.float())
    assert rel_l2(ops.geglu(h), out) < 5e-3
    assert rel_l2(ops.geglu(h, d), hl.grad) < 5e-3


def test_mse_and_adamw(cuda_device):
    from imagdressing_b200 import ops

    dev = cuda_device
    g = torch.Generator().manual_seed(0)
    pred, tgt = torch.randn(4, 4, 80, 64, generator=g).to(dev), torch.randn(4, 4, 80, 64, generator=g).to(dev)
    pl = pred.clone().requires_grad_(True)
    loss = F.mse_loss(pl, tgt)
    loss.backward()
    l, gr = ops.mse_loss_grad(pred, tgt)
    assert abs(float(l) - float(loss)) < 1e-5 * float(loss) and rel_l2(gr, pl.grad) < 1e-6
    assert float(ops.mse_loss_grad(pred, tgt)[0]) == float(l)  # deterministic

    n = 10007
    w0 = torch.randn(n, generator=g).to(dev)
    p_ref = torch.nn.Parameter(w0.clone())
    opt = torch.optim.AdamW([p_ref], lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2)
    master, m, v = w0.clone(), torch.zeros(n, device=dev), torch.zeros(n, device=dev)
    param = w0.to(BF)
    # the device-scalar variant (CUDA-graph replayable: step / lr read from memory; 4 elements per thread + scalar tail)
    master2, m2, v2, param2 = w0.clone(), torch.zeros(n, device=dev), torch.zeros(n, device=dev), w0.to(BF)
    hyper = torch.tensor([1e-3, 1e-2, 0.0, 1.0], device=dev)
    for step in range(1, 4):
        grad = (torch.randn(n, generator=g) * 0.1).to(BF).to(dev)
        p_ref.grad = grad.float()
        opt.step()
        ops.adamw_step(master, param, grad, m, v, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=1e-2, step=step)
        hyper[2:3].add_(1.0)
        ops.adamw_step_dev(master2, param2, grad, m2, v2, hyper, beta1=0.9, beta2=0.999, eps=1e-8)
    assert rel_l2(master, p_ref.detach()) < 1e-5
    assert torch.equal(param, master.to(BF))
    assert rel_l2(master2, p_ref.detach()) < 1e-5 and torch.equal(param2, master2.to(BF))
