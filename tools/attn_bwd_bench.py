"""Times the two-stream attention backward at the level-0 shape of the training step (micro-batch 4, 5120 tokens, 8 x 40):
CUDA events on the launching stream, L2 flushed between launches; dQ kernel + dK/dV kernel per stream + the D prep.
    python tools/attn_bwd_bench.py"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from imagdressing_b200 import ops

dev = torch.device("cuda:0")
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
for (B, L, C, heads) in ((4, 5120, 320, 8), (4, 1280, 640, 8), (4, 320, 1280, 8)):
    r = lambda *s: torch.randn(*s, device=dev).bfloat16()
    qkv, kv1, d_out = r(B, L, 3 * C), r(B, L, 2 * C), r(B * L, C)
    flat, f1 = qkv.view(B * L, 3 * C), kv1.view(B * L, 2 * C)
    s0 = ops.kv_stream(flat[:, C:2 * C], flat[:, 2 * C:], L)
    s1 = ops.kv_stream(f1[:, :C], f1[:, C:], L)
    out, saved = ops.attention_train(flat[:, :C], B, L, heads, C // heads, s0, s1)
    dqkv, dkv1 = torch.empty_like(flat), torch.empty_like(f1)
    cases = {
        "dq+dkv0+dkv1": lambda: ops.attention_bwd(flat[:, :C], d_out, B, L, heads, C // heads, s0, s1, saved, dq=dqkv[:, :C],
                                                  dkv0=(dqkv[:, C:2 * C], dqkv[:, 2 * C:]), dkv1=(dkv1[:, :C], dkv1[:, C:])),
        "dq only": lambda: ops.attention_bwd(flat[:, :C], d_out, B, L, heads, C // heads, s0, s1, saved, dq=dqkv[:, :C]),
        "dkv1 only": lambda: ops.attention_bwd(flat[:, :C], d_out, B, L, heads, C // heads, s0, s1, saved,
                                               dkv1=(dkv1[:, :C], dkv1[:, C:])),
        "forward (train)": lambda: ops.attention_train(flat[:, :C], B, L, heads, C // heads, s0, s1),
    }
    for name, fn in cases.items():
        for _ in range(2):
            fn()
        ts = []
        for _ in range(7):
            flush.zero_()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        print(f"B={B} L={L} hd={C // heads} "
              f"{name:16s}: {sorted(ts)[3] * 1e3:8.1f} us", flush=True)
