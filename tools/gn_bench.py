"""GroupNorm(+SiLU) launch time over the UNet's GroupNorm shapes. Per shape of three workloads (512 x 512 at batch 1 and
batch 8, 768 x 576 at batch 8): microseconds per launch, the bytes moved (2 x numel x 2), the implied GB/s, the kernel and
plan the library chose (imagd_groupnorm_plan), and the launch-weighted total of one denoising step. CUDA events around 10
replays of a 20-launch CUDA graph per shape after a warm-up, three times; the median is printed with the spread of the
three. The card's name and power limit are printed first: every number below belongs to them.

    python tools/gn_bench.py                  the table
    python tools/gn_bench.py --sweep          also every legal forced plan per shape (imagd_groupnorm_debug_force)
    python tools/gn_bench.py --root DIR       time the library of another checkout of this project (the parent commit's,
                                              say) in the same session; one that predates the plan hooks prints "-"
    python tools/gn_bench.py --json FILE      also write the rows as JSON
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

# (latent H = W, C, launches per step): ResnetBlock2D norm1 / norm2 and Transformer2DModel.norm of the SD1.5 UNet; the
# latent side is relative to a 64 x 64 level 0
SHAPES = [(64, 320, 9), (32, 320, 1), (32, 640, 9), (16, 640, 1), (16, 1280, 10), (8, 1280, 11), (8, 2560, 2), (16, 2560, 2),
          (16, 1920, 1), (32, 1920, 1), (32, 1280, 1), (32, 960, 1), (64, 960, 1), (64, 640, 2)]
# (name, batch, level-0 latent H, W)
WORKLOADS = [("512x512 batch 1", 1, 64, 64), ("512x512 batch 8", 8, 64, 64), ("768x576 batch 8", 8, 96, 72)]
KERNELS = {1: "rendezvous", 2: "cluster"}


def card() -> str:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=60)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "nvidia-smi unavailable"


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--sweep", action="store_true")
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch

    sys.path.insert(0, os.path.abspath(args.root))
    from imagdressing_b200 import _lib, ops

    lib = _lib.load()
    hooks = hasattr(lib, "imagd_groupnorm_plan")
    dev = torch.device("cuda:0")
    print(f"card: {card()}   library: {_lib.LIB_PATH}", flush=True)
    if hooks:
        cap = (ctypes.c_int * 8)()
        assert lib.imagd_groupnorm_cluster_capacity(cap) == 0
        print("co-resident clusters (size 2 / 4 / 8 / 16 at 1, 2 CTAs per SM):", list(cap), flush=True)

    def plan(NB, HW, C):
        if not hooks:
            return None
        out = (ctypes.c_int * 5)()
        return list(out) if lib.imagd_groupnorm_plan(NB, HW, C, 32, None, out) == 0 else None

    def fmt(p):
        if p is None:
            return "-"
        return KERNELS[p[0]] + (f" {p[1]} x {p[2]} ch, {p[3] / 1024:.0f} KB, {p[4]} wave(s)" if p[0] == 2 else "")

    def time_us(x, gamma, beta, out):
        for _ in range(3):
            ops.groupnorm(x, gamma, beta, 32, 1e-5, silu=True, out=out)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()  # 20 launches per replay: the python call (~11 us) would hide the kernel otherwise
        with torch.cuda.graph(graph):
            for _ in range(20):
                ops.groupnorm(x, gamma, beta, 32, 1e-5, silu=True, out=out)
        graph.replay()
        torch.cuda.synchronize()
        runs = []
        for _ in range(3):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(10):
                graph.replay()
            b.record()
            torch.cuda.synchronize()
            runs.append(a.elapsed_time(b) * 1000.0 / 200)
        runs.sort()
        return runs[1], runs[2] - runs[0]

    rows = []
    for name, batch, H0, W0 in WORKLOADS:
        NB = 2 * batch
        total = 0.0
        print(f"{name} ({NB} samples with CFG)", flush=True)
        for side, C, n in SHAPES:
            H, W = H0 * side // 64, W0 * side // 64
            x = torch.randn(NB, H, W, C, device=dev).bfloat16()
            gamma, beta = torch.ones(C, device=dev), torch.zeros(C, device=dev)
            out = torch.empty_like(x)
            mb = 2 * x.numel() * 2 / 1e6
            us, spread = time_us(x, gamma, beta, out)
            p = plan(NB, H * W, C)
            total += us * n
            print(f"  [{NB},{H}x{W},{C}] x{n:2d}: {us:7.2f} us +-{spread:5.2f}  {mb:7.2f} MB  {mb / us * 1e3:7.0f} GB/s  {fmt(p)}",
                  flush=True)
            row = dict(workload=name, NB=NB, H=H, W=W, C=C, launches=n, us=us, spread=spread, mb=mb, plan=p, forced=[])
            rows.append(row)
            if args.sweep and hooks:
                variants = [(1, 0, 0)] + [(2, cs, gps * C // 32) for cs in (2, 4, 8, 16) for gps in (1, 2, 4, 8, 16, 32)
                                        if gps * C // 32 % 8 == 0]
                for v in variants:
                    assert lib.imagd_groupnorm_debug_force(*v) == 0
                    fp = plan(NB, H * W, C)
                    if fp is not None:  # legal under the forced values
                        fus, fspread = time_us(x, gamma, beta, out)
                        row["forced"].append(dict(plan=fp, us=fus, spread=fspread))
                        print(f"      {fmt(fp):44s} {fus:7.2f} us +-{fspread:5.2f}", flush=True)
                    lib.imagd_groupnorm_debug_force(0, 0, 0)
        print(f"  launch-weighted total per step: {total:8.1f} us", flush=True)
        rows.append(dict(workload=name, total_us=total))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(card=card(), rows=rows), f)


if __name__ == "__main__":
    main()
