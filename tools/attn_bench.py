"""Times every attention shape of the denoising step in isolation: CUDA events on the launching stream, L2 flushed
between launches, median of 20 launches.
    python tools/attn_bench.py            B=1 python tools/attn_bench.py
Shapes (per sample: a CFG pair = B conditional samples + B unconditional):
  hybrid l0 / l1 / l2 / mid / l1-768   self-attention over L tokens; the conditional samples add the garment stream (L keys)
  text l0 / l1 / l2 / mid / l1-768     cross-attention over the 77 text tokens
For each shape it prints the median kernel time, algorithmic TFLOP/s (4 Lq Lk head_dim per head and stream) and two
floors computed from the shape: the tensor floor (Q K^T at head_dim padded to 16, P V at head_dim, over the dense bf16
peak) and the exp2 floor (one MUFU ex2 per score, 16 per clock per SM at the maximum SM clock)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from imagdressing_b200 import ops

PEAK_BF16 = 989e12  # H100 SXM data sheet, dense bf16
SM_CLOCK = 1.98e9   # H100 SXM maximum SM clock
# levels of the 512x512 step, plus level 1 of the 768x576 workload (1728 tokens: not a multiple of the key block)
LEVELS = (("l0", 4096, 320), ("l1", 1024, 640), ("l2", 256, 1280), ("mid", 64, 1280), ("l1-768", 1728, 640))
HEADS = 8

dev = torch.device("cuda:0")
n_sm = torch.cuda.get_device_properties(dev).multi_processor_count
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)


def flat(t):
    return t.as_strided((t.shape[0] * t.shape[1], t.shape[2]), (t.stride(1), 1), t.storage_offset())


def time_ms(run, n=20):
    for _ in range(3):
        run()
    ts = []
    for _ in range(n):
        flush.zero_()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        run()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return sorted(ts)[len(ts) // 2]


def report(name, ms, pairs):
    """pairs: one (Lq, Lk, head_dim) triple per (sample, stream) of the launch."""
    scores = sum(lq * lk for lq, lk, _ in pairs) * HEADS
    flops = 4.0 * HEADS * sum(lq * lk * hd for lq, lk, hd in pairs)
    tensor_us = HEADS * sum(lq * lk * (2 * ((hd + 15) // 16 * 16) + 2 * hd) for lq, lk, hd in pairs) / PEAK_BF16 * 1e6
    exp_us = scores / (16 * n_sm * SM_CLOCK) * 1e6
    print(f"{name:<16} {ms * 1e3:9.1f} us {flops / (ms * 1e-3) / 1e12:7.1f} TFLOP/s   tensor floor {tensor_us:7.1f} us"
          f"   exp2 floor {exp_us:7.1f} us", flush=True)


for B in [int(b) for b in os.environ.get("B", "1,8").split(",")]:
    NB = 2 * B
    for lvl, L, C in LEVELS:
        hd = C // HEADS
        qkv = torch.randn(NB, L, 3 * C, device=dev).bfloat16()
        kvr = torch.randn(B, L, 2 * C, device=dev).bfloat16()
        s0 = ops.kv_stream(flat(qkv[..., C:2 * C]), flat(qkv[..., 2 * C:]), L)
        s1 = ops.kv_stream(flat(kvr[..., :C]), flat(kvr[..., C:]), L, n_query_samples=B)
        out = torch.empty(NB * L, C, device=dev, dtype=torch.bfloat16)
        ms = time_ms(lambda: ops.attention(flat(qkv[..., :C]), NB, L, HEADS, hd, s0, s1, out=out))
        report(f"B={B} hybrid {lvl}", ms, [(L, L, hd)] * (NB + B))
        txt = torch.randn(NB, 77, 2 * C, device=dev).bfloat16()
        st = ops.kv_stream(flat(txt[..., :C]), flat(txt[..., C:]), 77)
        ms = time_ms(lambda: ops.attention(flat(qkv[..., :C]), NB, L, HEADS, hd, st, None, out=out))
        report(f"B={B} text {lvl}", ms, [(L, 77, hd)] * NB)
