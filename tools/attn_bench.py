"""Times the level-0 hybrid attention (head_dim 40, L = 4096, CFG pair per sample: B conditional samples with the garment
stream + B unconditional) in isolation: CUDA events on the launching stream, L2 flushed between launches.
    B=1 python tools/attn_bench.py        B=8 python tools/attn_bench.py
Prints algorithmic TFLOP/s (4 L (L + L_ref) C per conditional sample, 4 L L C per unconditional) and the fraction of the
measured burst bf16 peak (MEASURED_PEAKS.json)."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from imagdressing_b200 import ops

dev = torch.device("cuda:0")
peak = 989.0  # H100 SXM data sheet, dense bf16 (MEASURED_PEAKS.json overrides)
try:
    peak = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")))["bf16_tflops"]
except Exception:
    pass
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
flat = lambda t: t.as_strided((t.shape[0] * t.shape[1], t.shape[2]), (t.stride(1), 1), t.storage_offset())
for B in [int(b) for b in os.environ.get("B", "1,8").split(",")]:
    for (L, C, heads) in ((4096, 320, 8), (1024, 640, 8), (256, 1280, 8)):
        NB = 2 * B
        qkv = torch.randn(NB, L, 3 * C, device=dev).bfloat16()
        kvr = torch.randn(B, L, 2 * C, device=dev).bfloat16()
        s0 = ops.kv_stream(flat(qkv[..., C:2 * C]), flat(qkv[..., 2 * C:]), L)
        s1 = ops.kv_stream(flat(kvr[..., :C]), flat(kvr[..., C:]), L, n_query_samples=B)
        out = torch.empty(NB * L, C, device=dev, dtype=torch.bfloat16)
        run = lambda: ops.attention(flat(qkv[..., :C]), NB, L, heads, C // heads, s0, s1, out=out)
        for _ in range(3):
            run()
        ts = []
        for _ in range(10):
            flush.zero_()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        ms = sorted(ts)[len(ts) // 2]
        fl = 4.0 * L * L * C * (NB + B)
        tf = fl / (ms * 1e-3) / 1e12
        print(f"B={B} L={L} hd={C // heads}: {ms * 1e3:.1f} us  {tf:.1f} TFLOP/s  "
              f"{tf / peak:.3f} of measured burst peak", flush=True)
