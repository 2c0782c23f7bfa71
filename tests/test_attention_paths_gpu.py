"""GPU parity of every attention path against an fp64 reference computed from the same bf16 inputs: both forward kernels
(chosen through imagd_attention_debug_force), the automatic choice between them, the training forward's saved outputs
(per-stream log-sum-exp and outputs) and the backward at the lengths of the training step.

The automatic choice runs the TMA / wgmma kernel for non-causal head_dim 40 / 80 calls with >= 1024 keys in stream 0 and
the mma.sync kernel otherwise. Here every head_dim 40 / 80 case runs on both kernels, including the shapes the automatic
choice never sends to the wgmma kernel: one query row, Lq < 64 (the second consumer warpgroup has no rows), streams
shorter than one key block (128 keys at head_dim 40, 64 at 80) and a stream of a single key.

Every comparison reports the worst tile next to the global rel-L2. A tile is 64 query rows of one (sample, head) for the
outputs and dQ, and 128 keys of one (sample, head) for dK / dV (the dK / dV kernel's CTA tile): at [1, 4096, 8 x 40] one
wrong tile is 1/512 of the tensor, and a global rel-L2 alone dilutes its error by about 23x.

The kernels take bf16 inputs and write bf16 outputs, keep scores and softmax statistics in fp32 and round P to bf16 before
P V; the backward also rounds P and dS to bf16 before its second products. The bounds are about twice the worst values
measured over this file on an H100 80GB HBM3 (700 W power limit): forward 3.1e-3 per tile / 2.3e-3 global, backward
2.7e-3 / 2.4e-3, log-sum-exp 1.9e-6 (log2 units). The kernels are deterministic, so a rerun measures the same values.
"""
import math
from contextlib import contextmanager
from dataclasses import dataclass, replace
from typing import Optional

import pytest
import torch

BF = torch.bfloat16
gpu = pytest.mark.gpu
AUTO, MMA, WGMMA = 0, 1, 2
KERNEL = {AUTO: "auto", MMA: "mma", WGMMA: "wgmma"}
FWD_TILE, FWD_GLOBAL = 6e-3, 5e-3   # forward outputs, o0 / o1: worst (sample, head, 64 rows) tile, whole tensor
BWD_TILE, BWD_GLOBAL = 6e-3, 5e-3   # dQ (64-row tiles), dK / dV (128-key tiles)
LSE_ATOL = 4e-6                     # log-sum-exp rows, log2 units
SENTINEL = -1024.0


@contextmanager
def forced(kernel):
    from imagdressing_b200 import _lib

    lib = _lib.load()
    assert lib.imagd_attention_debug_force(kernel) == 0
    try:
        yield
    finally:
        lib.imagd_attention_debug_force(0)


def _rand(shape, dev, seed, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(BF).to(dev)


def _flat(t):
    """[n, rows, C] view with uniform row stride -> 2-D [n * rows, C] view sharing storage."""
    n, rows, C = t.shape
    assert t.stride(0) == rows * t.stride(1)
    return t.as_strided((n * rows, C), (t.stride(1), 1), t.storage_offset())


# ------------------------------------------------------------------------------------------------ reference and metric
def tile_errors(got, ref, tile):
    """got / ref: [B, L, heads, hd]. Returns (the largest rel-L2 over (sample, head, `tile` rows), the global rel-L2).
    A NaN anywhere in `got` makes both NaN, which fails every bound."""
    d2 = (got.double() - ref.double()).square().sum(-1)
    r2 = ref.double().square().sum(-1)
    B, L, H = r2.shape
    pad = (-L) % tile
    d2t = torch.nn.functional.pad(d2, (0, 0, 0, pad)).view(B, -1, tile, H).sum(2)
    r2t = torch.nn.functional.pad(r2, (0, 0, 0, pad)).view(B, -1, tile, H).sum(2)
    worst = (d2t / r2t.clamp_min(1e-300)).sqrt().max()
    return float(worst), float((d2.sum() / r2.sum()).sqrt())


def check(name, got, ref, tile, tile_bound, global_bound):
    worst, glob = tile_errors(got, ref, tile)
    print(f"{name}: worst tile rel-L2 {worst:.2e}, global {glob:.2e}")
    assert worst <= tile_bound and glob <= global_bound, (
        f"{name}: worst tile rel-L2 {worst:.3e} (bound {tile_bound}), global {glob:.3e} (bound {global_bound})")


def sdpa64(q, k, v, heads, hd, scale, causal=False):
    """fp64 softmax(q k^T scale) v per (sample, head): q [B, Lq, C], k / v [B, L, C] -> O [B, Lq, heads, hd] and the
    natural-log log-sum-exp rows [B, heads, Lq]. One (sample, head group) at a time, so 4096 x 4096 scores fit."""
    B, Lq, _ = q.shape
    L = k.shape[1]
    sp = lambda t: t.reshape(t.shape[0], t.shape[1], heads, hd).transpose(1, 2)
    qh, kh, vh = sp(q), sp(k), sp(v)
    o = torch.empty(B, heads, Lq, hd, dtype=torch.float64, device=q.device)
    lse = torch.empty(B, heads, Lq, dtype=torch.float64, device=q.device)
    step = max(1, (1 << 25) // (Lq * L))
    future = torch.ones(Lq, L, dtype=torch.bool, device=q.device).triu(1) if causal else None
    for b in range(B):
        for h in range(0, heads, step):
            hs = slice(h, h + step)
            s = qh[b, hs].double() @ kh[b, hs].double().transpose(-1, -2) * scale
            if causal:
                s.masked_fill_(future, -math.inf)
            lse[b, hs] = torch.logsumexp(s, -1)
            o[b, hs] = torch.exp(s - lse[b, hs, :, None]) @ vh[b, hs].double()
    return o.transpose(1, 2), lse


# ------------------------------------------------------------------------------------------------ cases
@dataclass
class Case:
    name: str
    B: int
    Lq: int
    heads: int
    hd: int
    L0: int
    L1: int = 0                 # 0: one stream
    n1: Optional[int] = None    # stream 1 applies to query samples [0, n1)
    bcast1: bool = False        # one stream-1 sample shared by the query samples
    w0: float = 1.0
    w1: float = 1.0
    rows0: int = 0              # sample_rows > L: the keys are a window of a longer context; the gap rows hold NaN
    rows1: int = 0
    sm_scale: Optional[float] = None
    causal: bool = False

    @property
    def C(self):
        return self.heads * self.hd

    @property
    def scale(self):
        return self.sm_scale if self.sm_scale is not None else self.hd ** -0.5

    @property
    def nq1(self):
        return min(self.n1 or self.B, self.B) if self.L1 else 0

    def wgmma_ok(self):
        return self.hd in (40, 80) and not self.causal

    def auto_kernel(self):
        return WGMMA if self.wgmma_ok() and self.L0 >= 1024 else MMA


def make_inputs(c, dev, seed=0):
    """q [B, Lq, C]; kv0 [B, rows0, 2C] and kv1 [n, rows1, 2C] (K | V side by side, as the projections produce them)."""
    q = _rand((c.B, c.Lq, c.C), dev, seed + 1)
    kv0 = _rand((c.B, c.rows0 or c.L0, 2 * c.C), dev, seed + 2)
    kv0[:, c.L0:] = float("nan")
    kv1 = None
    if c.L1:
        kv1 = _rand((1 if c.bcast1 else c.nq1, c.rows1 or c.L1, 2 * c.C), dev, seed + 3)
        kv1[:, c.L1:] = float("nan")
    return q, kv0, kv1


def kv_streams(c, kv0, kv1):
    from imagdressing_b200 import ops

    C = c.C
    s0 = ops.kv_stream(_flat(kv0[..., :C]), _flat(kv0[..., C:]), c.L0, sample_rows=c.rows0, out_scale=c.w0)
    s1 = None
    if kv1 is not None:
        s1 = ops.kv_stream(_flat(kv1[..., :C]), _flat(kv1[..., C:]), c.L1, sample_rows=c.rows1, broadcast=c.bcast1,
                           n_query_samples=c.n1 or c.B, out_scale=c.w1)
    return s0, s1


class Reference:
    """fp64 per-stream outputs O_s [B, Lq, heads, hd], natural-log lse rows [B, heads, Lq] and out = w0 O_0 + w1 O_1
    (stream 1 on samples [0, nq1) only)."""

    def __init__(self, c, q, kv0, kv1):
        C = c.C
        self.o0, self.lse0 = sdpa64(q, kv0[:, :c.L0, :C], kv0[:, :c.L0, C:], c.heads, c.hd, c.scale, c.causal)
        self.out = c.w0 * self.o0
        self.o1 = self.lse1 = None
        if kv1 is not None:
            n = c.nq1
            k1, v1 = kv1[:, :c.L1, :C], kv1[:, :c.L1, C:]
            if c.bcast1:
                k1, v1 = k1.expand(n, -1, -1), v1.expand(n, -1, -1)
            self.o1, self.lse1 = sdpa64(q[:n], k1[:n], v1[:n], c.heads, c.hd, c.scale)
            self.out = self.out.clone()
            self.out[:n] += c.w1 * self.o1


def run_forward(c, q, s0, s1, kernel, out=None):
    from imagdressing_b200 import ops

    with forced(kernel):
        o = ops.attention(_flat(q), c.B, c.Lq, c.heads, c.hd, s0, s1, sm_scale=c.sm_scale, out=out, causal=c.causal)
    return o.view(c.B, c.Lq, c.heads, c.hd)


def run_train(c, q, s0, s1, kernel):
    from imagdressing_b200 import ops

    with forced(kernel):
        return ops.attention_train(_flat(q), c.B, c.Lq, c.heads, c.hd, s0, s1, sm_scale=c.sm_scale)


FWD_CASES = [
    # head_dim 40 (wgmma key block 128)
    Case("hd40_q1_w0", 1, 1, 8, 40, 1024, w0=0.8),                                  # one query row, single-stream weight
    Case("hd40_exact_s1_127", 2, 129, 3, 40, 256, L1=127, w0=0.6, w1=-0.4),
    Case("hd40_257_s1_128", 1, 65, 8, 40, 257, L1=128, w1=0.9),
    Case("hd40_1023_s1_129", 2, 63, 1, 40, 1023, L1=129),                           # Lq < 64, just under the dispatch
    Case("hd40_1024_ip4", 2, 1000, 8, 40, 1024, L1=4, w1=0.9),                      # text + 4 IP tokens shape
    Case("hd40_1100_text77", 1, 300, 8, 40, 1100, L1=77),
    Case("hd40_s1_longer", 1, 300, 8, 40, 1100, L1=2200, w1=0.7),
    Case("hd40_cfg", 2, 1000, 8, 40, 1100, L1=1100, n1=1, w1=0.9),                  # stream 1 on sample 0 of 2
    Case("hd40_bcast", 3, 129, 3, 40, 1024, L1=300, n1=2, bcast1=True),
    Case("hd40_windows", 3, 200, 8, 40, 1037, L1=100, n1=2, w1=0.7, rows0=1100, rows1=160),
    Case("hd40_B5_scale", 5, 65, 1, 40, 128, sm_scale=0.05),                        # one key block in all
    Case("hd40_one_key", 1, 1, 3, 40, 1, L1=1, w0=0.6, w1=-0.4),
    # head_dim 80 (wgmma key block 64)
    Case("hd80_exact_s1_63", 2, 129, 8, 80, 128, L1=63, w0=0.6, w1=-0.4),
    Case("hd80_65_s1_64", 1, 63, 3, 80, 65, L1=64),
    Case("hd80_1023_s1_65", 1, 65, 8, 80, 1023, L1=65),
    Case("hd80_1024_text77", 2, 1000, 8, 80, 1024, L1=77),
    Case("hd80_windows", 3, 129, 8, 80, 1100, L1=40, n1=2, rows0=1164, rows1=81),
    Case("hd80_clip_h", 1, 257, 16, 80, 257),                                       # CLIP ViT-H self-attention
    Case("hd80_B5_q1_w0", 5, 1, 1, 80, 64, w0=1.3),
    # shapes only the mma.sync kernel serves
    Case("hd64_perceiver", 2, 16, 12, 64, 273),
    Case("hd160_level2", 1, 432, 8, 160, 432, L1=432),
    Case("hd160_q1", 2, 1, 8, 160, 432),
    Case("hd160_1100", 1, 200, 8, 160, 1100),
    Case("hd64_causal", 2, 77, 12, 64, 77, causal=True),
    Case("hd80_causal", 1, 100, 4, 80, 100, causal=True),
]
CASE = {c.name: c for c in FWD_CASES}


# ------------------------------------------------------------------------------------------------ A. forward matrix
@gpu
@pytest.mark.parametrize("c", FWD_CASES, ids=lambda c: c.name)
def test_forward_kernels_match_fp64(cuda_device, c):
    """Automatic, forced mma and (where it is legal) forced wgmma, each against fp64 and against each other. The automatic
    output is bitwise the output of the kernel the dispatch rule names. Forcing wgmma where it cannot run fails and leaves
    the output untouched."""
    from imagdressing_b200 import _lib

    q, kv0, kv1 = make_inputs(c, cuda_device)
    s0, s1 = kv_streams(c, kv0, kv1)
    ref = Reference(c, q, kv0, kv1)
    got = {k: run_forward(c, q, s0, s1, k) for k in ((AUTO, MMA, WGMMA) if c.wgmma_ok() else (AUTO, MMA))}
    for k, o in got.items():
        assert torch.isfinite(o).all(), KERNEL[k]
        check(f"A {c.name} {KERNEL[k]}", o, ref.out, 64, FWD_TILE, FWD_GLOBAL)
    assert torch.equal(got[AUTO], got[c.auto_kernel()])
    if c.wgmma_ok():
        check(f"A {c.name} wgmma vs mma", got[WGMMA], got[MMA], 64, FWD_TILE, FWD_GLOBAL)
    else:
        out = torch.full((c.B * c.Lq, c.C), SENTINEL, device=cuda_device, dtype=BF)
        with pytest.raises(_lib.ImagdError, match="wgmma"):
            run_forward(c, q, s0, s1, WGMMA, out=out)
        torch.cuda.synchronize()
        assert (out == SENTINEL).all()


def test_tile_metric_sees_one_wrong_tile():
    """CPU: the fp64 reference agrees with the emulated operator (fp32 SDPA, bf16 output) under the forward bounds, and
    one 64-row tile of one head that is 2 % off fails the per-tile bound of a [1, 1024, 8 x 40] output while its global
    rel-L2 stays under the global bound."""
    import emulated_ops

    c = Case("cpu", 1, 1024, 8, 40, 1024, L1=77, w0=0.6, w1=-0.4)
    q, kv0, kv1 = make_inputs(c, "cpu")
    ref = Reference(c, q, kv0, kv1).out
    C = c.C
    s0 = emulated_ops.kv_stream(_flat(kv0[..., :C]), _flat(kv0[..., C:]), c.L0, out_scale=c.w0)
    s1 = emulated_ops.kv_stream(_flat(kv1[..., :C]), _flat(kv1[..., C:]), c.L1, out_scale=c.w1)
    got = emulated_ops.attention(_flat(q), c.B, c.Lq, c.heads, c.hd, s0, s1).view(c.B, c.Lq, c.heads, c.hd)
    worst, glob = tile_errors(got, ref, 64)
    assert worst <= FWD_TILE and glob <= FWD_GLOBAL, (worst, glob)
    bad = got.float()
    bad[0, 128:192, 5] *= 1.02
    worst, glob = tile_errors(bad, ref, 64)
    assert worst > FWD_TILE and glob <= FWD_GLOBAL, (worst, glob)


def test_debug_force_rejects_unknown_kernels():
    from imagdressing_b200 import _lib

    lib = _lib.load()
    for bad in (-1, 3):
        assert lib.imagd_attention_debug_force(bad) != 0
        assert b"attention_debug_force" in lib.imagd_last_error()
    assert lib.imagd_attention_debug_force(0) == 0


# ------------------------------------------------------------------------------------------------ B. dispatch boundary
@gpu
@pytest.mark.parametrize("hd,L0,expect", [(40, 1023, MMA), (40, 1024, WGMMA), (80, 1023, MMA), (80, 1024, WGMMA),
                                          (64, 4096, MMA), (160, 4096, MMA)])
def test_dispatch_boundary(cuda_device, hd, L0, expect):
    """Both kernels are deterministic and round differently, so bitwise equality shows which one the automatic call ran."""
    c = Case(f"boundary_hd{hd}_{L0}", 1, 129, 2, hd, L0)
    q, kv0, _ = make_inputs(c, cuda_device, seed=20)
    s0, _ = kv_streams(c, kv0, None)
    auto = run_forward(c, q, s0, None, AUTO)
    assert torch.equal(auto, run_forward(c, q, s0, None, expect))
    if c.wgmma_ok():
        assert not torch.equal(auto, run_forward(c, q, s0, None, WGMMA if expect == MMA else MMA))
    check(f"B {c.name}", auto, Reference(c, q, kv0, None).out, 64, FWD_TILE, FWD_GLOBAL)


# ------------------------------------------------------------------------------------------------ C. hard softmax
@gpu
@pytest.mark.parametrize("kernel", [MMA, WGMMA], ids=lambda k: KERNEL[k])
@pytest.mark.parametrize("hd", [40, 80])
def test_hard_softmax(cuda_device, hd, kernel):
    """Large logits (Q and K x4, keys from 512 on x3 more), row maxima that move from block to block (K grows by 10 % per
    64 keys) and, in stream 1, rows whose maximum is the last key, inside the ragged last block."""
    c = Case(f"hard_hd{hd}", 1, 300, 8, hd, 1100, L1=1037, w1=0.8)
    q, kv0, kv1 = make_inputs(c, cuda_device, seed=30)
    C = c.C
    q.mul_(4.0)
    ramp = 1.0 + 0.1 * (torch.arange(c.L0, device=cuda_device) // 64).float()
    ramp[512:] *= 3.0
    kv0[0, :, :C] = (kv0[0, :, :C].float() * 4.0 * ramp[:, None]).to(BF)
    kv1[0, c.L1 - 1, :C] = q[0, 7] * 0.5
    kv1[0, c.L1 - 2, :C] = q[0, 11] * 0.5
    s0, s1 = kv_streams(c, kv0, kv1)
    ref = Reference(c, q, kv0, kv1)
    assert float(ref.o1[0, 7].sub(kv1[0, c.L1 - 1, C:].double().view(c.heads, hd)).abs().max()) < 1e-3  # max is last key
    out = run_forward(c, q, s0, s1, kernel)
    assert torch.isfinite(out).all()
    check(f"C {c.name} {KERNEL[kernel]}", out, ref.out, 64, FWD_TILE, FWD_GLOBAL)


# ------------------------------------------------------------------------------------------------ D. training forward
TRAIN_CASES = [CASE[n] for n in ("hd40_exact_s1_127", "hd40_1023_s1_129", "hd40_s1_longer", "hd40_q1_w0",
                                 "hd80_exact_s1_63", "hd80_1024_text77", "hd80_B5_q1_w0", "hd64_perceiver", "hd160_level2",
                                 "hd160_1100")] + [
    # the windowed cases with stream 1 on every sample (a training forward needs that)
    replace(CASE["hd40_windows"], name="hd40_windows_all", n1=None),
    replace(CASE["hd80_windows"], name="hd80_windows_all", n1=None),
]


@gpu
@pytest.mark.parametrize("c", TRAIN_CASES, ids=lambda c: c.name)
def test_train_forward_saved_outputs(cuda_device, c):
    """attention_train on each kernel: `out` is bitwise the inference output of the same kernel; the log2-domain
    log-sum-exp rows of both streams match fp64, padding rows and samples a stream skips stay +inf; the un-weighted
    per-stream outputs match fp64; a second run is bitwise equal."""
    q, kv0, kv1 = make_inputs(c, cuda_device, seed=40)
    s0, s1 = kv_streams(c, kv0, kv1)
    ref = Reference(c, q, kv0, kv1)
    n1, Lq = c.nq1, c.Lq
    for k in (MMA, WGMMA) if c.wgmma_ok() else (MMA,):
        name = f"D {c.name} {KERNEL[k]}"
        out, saved = run_train(c, q, s0, s1, k)
        assert torch.equal(out.view(c.B, Lq, c.heads, c.hd), run_forward(c, q, s0, s1, k)), name
        lse = saved.lse
        refs = [(ref.lse0, c.B)] + ([(ref.lse1, n1)] if s1 is not None else [])
        for s, (lr, n) in enumerate(refs):
            err = float((lse[s, :n, :, :Lq].double() - lr / math.log(2.0)).abs().max())
            print(f"{name}: stream {s} lse max |err| {err:.2e} (log2 units)")
            assert err <= LSE_ATOL, f"{name}: stream {s} lse off by {err:.3e}"
        assert torch.isinf(lse[..., Lq:]).all() and (lse[..., Lq:] > 0).all()  # padding rows
        assert torch.isposinf(lse[1, n1:]).all()  # stream 1 absent / skipped
        if s1 is not None:
            check(f"{name} o0", saved.o0.view(c.B, Lq, c.heads, c.hd), ref.o0, 64, FWD_TILE, FWD_GLOBAL)
            check(f"{name} o1", saved.o1.view(c.B, Lq, c.heads, c.hd)[:n1], ref.o1, 64, FWD_TILE, FWD_GLOBAL)
        again, saved2 = run_train(c, q, s0, s1, k)
        assert torch.equal(again, out) and torch.equal(saved2.lse, lse), name
        if s1 is not None:
            assert torch.equal(saved2.o0, saved.o0), name
            assert torch.equal(saved2.o1[:n1 * Lq], saved.o1[:n1 * Lq]), name


@gpu
@pytest.mark.parametrize("kernel", [MMA, WGMMA], ids=lambda k: KERNEL[k])
def test_train_forward_rejects_partial_stream(cuda_device, kernel):
    """A training forward whose stream 1 skips query samples (the CFG layout) would leave O_0 of the skipped samples
    unwritten (it is stored when stream 1 starts); the call is rejected instead, as the backward rejects it."""
    from imagdressing_b200 import _lib

    c = CASE["hd40_cfg"]
    q, kv0, kv1 = make_inputs(c, cuda_device)
    s0, s1 = kv_streams(c, kv0, kv1)
    with pytest.raises(_lib.ImagdError, match="every query sample"):
        run_train(c, q, s0, s1, kernel)


# ------------------------------------------------------------------------------------------------ E. backward
def ref_backward(c, q, kv0, kv1, d_out):
    """fp64 autograd of w0 SDPA(q, k0, v0) + w1 SDPA(q, k1, v1), one (sample, head) at a time.
    Returns [dQ, dK0, dV0(, dK1, dV1)] as [B, L, heads, hd]."""
    C, hd = c.C, c.hd
    streams = [(kv0, c.L0, c.w0)] + ([(kv1, c.L1, c.w1)] if kv1 is not None else [])
    grads = [torch.zeros(c.B, c.Lq, c.heads, hd, dtype=torch.float64, device=q.device)]
    for _, L, _ in streams:
        grads += [torch.zeros(c.B, L, c.heads, hd, dtype=torch.float64, device=q.device) for _ in range(2)]
    for b in range(c.B):
        for h in range(c.heads):
            cols = slice(h * hd, (h + 1) * hd)
            vcols = slice(C + h * hd, C + (h + 1) * hd)
            leaves = [q[b, :, cols].double().requires_grad_(True)]
            out = 0.0
            for kv, L, w in streams:
                k = kv[b, :L, cols].double().requires_grad_(True)
                v = kv[b, :L, vcols].double().requires_grad_(True)
                leaves += [k, v]
                out = out + w * (torch.softmax(leaves[0] @ k.t() * c.scale, -1) @ v)
            for g, leaf in zip(grads, torch.autograd.grad(out, leaves, d_out[b, :, cols].double())):
                g[b, :, h] = leaf
    return grads


BWD_CASES = [
    Case("hd40_B2_1280", 2, 1280, 8, 40, 1280, L1=1280),                            # 320 x 256 px training, level 0
    Case("hd40_B1_4096", 1, 4096, 8, 40, 4096, L1=4096),                            # 512 x 512 px training, level 0
    Case("hd80_B1_1024_w", 1, 1024, 8, 80, 1024, L1=1024, w0=0.7, w1=1.3),
    Case("hd40_1100_window_w", 2, 1100, 8, 40, 1100, L1=1037, rows1=1100, w0=0.7, w1=1.3),
]


@gpu
@pytest.mark.parametrize("fwd", [MMA, WGMMA], ids=lambda k: KERNEL[k])
@pytest.mark.parametrize("c", BWD_CASES, ids=lambda c: c.name)
def test_backward_training_lengths(cuda_device, c, fwd):
    """attention_train (forward forced to each kernel: their lse rows differ in the last bits) then attention_bwd, against
    fp64 autograd. dQ goes into a column slice of a wider buffer and dK / dV into buffers laid out like the streams; every
    element the backward must not write (other columns, the gap rows of a windowed stream) keeps its sentinel. A second
    backward is bitwise equal."""
    from imagdressing_b200 import ops

    dev = cuda_device
    C, hd, B, Lq = c.C, c.hd, c.B, c.Lq
    q, kv0, kv1 = make_inputs(c, dev, seed=50)
    s0, s1 = kv_streams(c, kv0, kv1)
    d_out = _rand((B, Lq, C), dev, 60)
    _, saved = run_train(c, q, s0, s1, fwd)

    def backward():
        dq_buf = torch.full((B * Lq, C + 2 * hd), SENTINEL, device=dev, dtype=BF)
        dkv = [torch.full_like(kv0, SENTINEL), torch.full_like(kv1, SENTINEL)]
        ops.attention_bwd(_flat(q), _flat(d_out), B, Lq, c.heads, hd, s0, s1, saved, sm_scale=c.sm_scale,
                          dq=dq_buf[:, hd:hd + C], dkv0=(_flat(dkv[0][..., :C]), _flat(dkv[0][..., C:])),
                          dkv1=(_flat(dkv[1][..., :C]), _flat(dkv[1][..., C:])))
        return dq_buf, dkv

    dq_buf, dkv = backward()
    ref = ref_backward(c, q, kv0, kv1, d_out)
    name = f"E {c.name} fwd {KERNEL[fwd]}"
    check(f"{name} dq", dq_buf[:, hd:hd + C].reshape(B, Lq, c.heads, hd), ref[0], 64, BWD_TILE, BWD_GLOBAL)
    for s, L in enumerate((c.L0, c.L1)):
        for j, part in enumerate(("dk", "dv")):
            got = dkv[s][:, :L, j * C:(j + 1) * C].reshape(B, L, c.heads, hd)
            check(f"{name} {part}{s}", got, ref[1 + 2 * s + j], 128, BWD_TILE, BWD_GLOBAL)
        assert (dkv[s][:, L:] == SENTINEL).all(), f"{name}: gap rows of stream {s} written"
    assert (dq_buf[:, :hd] == SENTINEL).all() and (dq_buf[:, hd + C:] == SENTINEL).all(), f"{name}: dQ outside its slice"
    dq2, dkv2 = backward()
    assert torch.equal(dq2, dq_buf) and torch.equal(dkv2[0], dkv[0]) and torch.equal(dkv2[1], dkv[1]), name
