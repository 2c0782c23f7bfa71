"""Per-CTA timeline of the wgmma GEMM (imagd_gemm_debug_timeline): where a CTA's lifetime goes for the short-K
transformer GEMMs. Prints the median clocks of each phase over all CTAs + the event-timed kernel duration."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from imagdressing_b200 import _lib, ops

dev = torch.device("cuda:0")
lib = _lib.load()
buf = torch.zeros(8 * 65536, device=dev, dtype=torch.int64)
flush = torch.empty(64 * 1024 * 1024, device=dev, dtype=torch.int32)
r = lambda *s: torch.randn(*s, device=dev).bfloat16()


def ev_time(fn, cold, iters=7):
    ts = []
    for _ in range(iters):
        if cold:
            flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3)
    ts.sort()
    return ts[len(ts) // 2]


def case(name, M, N, K, bias=True, residual=True, act=ops.ACT_NONE, force=None):
    a = r(M, K)
    w = (torch.randn(N, K, device=dev) * K ** -0.5).bfloat16()
    b = torch.randn(N, device=dev) if bias else None
    n_out = N // 2 if act == ops.ACT_GEGLU else N
    res = r(M, n_out) if residual else None
    out = torch.empty(M, n_out, device=dev, dtype=torch.bfloat16)
    fn = lambda: ops.gemm(a, w, out=out, bias=b, residual=res, act=act)
    if force:
        lib.imagd_gemm_debug_force(*force)
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    lib.imagd_gemm_debug_timeline(None)
    warm, cold = ev_time(fn, False), ev_time(fn, True)
    buf.zero_()
    lib.imagd_gemm_debug_timeline(buf.data_ptr())
    fn()
    torch.cuda.synchronize()
    lib.imagd_gemm_debug_timeline(None)
    lib.imagd_gemm_debug_force(0, 0, 0)
    t = buf.view(-1, 8).cpu()
    t = t[t[:, 0] != 0]
    d = lambda i, j: float((t[:, j] - t[:, i]).float().median())
    gt = t[:, 6] - t[:, 6].min()
    flops = 2.0 * M * N * K
    print(f"{name:34s} M={M} N={N} K={K} ctas={len(t):5d} warm {warm:7.1f} us ({flops / warm / 1e6:6.0f} TF/s) cold {cold:7.1f} us | "
          f"clk: prologue {d(0, 1):6.0f} first-tile {d(1, 2):6.0f} mainloop {d(2, 3):6.0f} acc-ready {d(3, 4):6.0f} "
          f"epilogue {d(4, 5):6.0f} total {d(0, 5):6.0f} | last CTA start {float(gt.max()) / 1e3:6.1f} us, SMs {len(set(t[:, 7].tolist()))}")


for B in (1, 8):
    M = 2 * B * 4096
    print(f"---- level-0 transformer GEMMs, batch {B} (CFG batch {2 * B})")
    case("to_out (bias+res)", M, 320, 320)
    case("to_out plain", M, 320, 320, bias=False, residual=False)
    case("to_out bias only", M, 320, 320, residual=False)
    case("to_out res only", M, 320, 320, bias=False)
    case("to_out (bias+res) 128/3", M, 320, 320, force=(128, 3, 1))
    case("to_out (bias+res) 64/4", M, 320, 320, force=(64, 4, 1))
    case("qkv plain", M, 960, 320, bias=False, residual=False)
    case("geglu", M, 2560, 320, residual=False, act=ops.ACT_GEGLU)
    case("ff_out (bias+res)", M, 320, 1280)
    case("ff_out plain", M, 320, 1280, bias=False, residual=False)
M = 2 * 8 * 1024
print("---- level-1, batch 8")
case("to_out (bias+res)", M, 640, 640)
case("geglu", M, 5120, 640, residual=False, act=ops.ACT_GEGLU)
case("ff_out (bias+res)", M, 640, 2560)
