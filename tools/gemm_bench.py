"""Per-launch table of the wgmma GEMM / implicit-GEMM conv kernel at the shapes one denoising step issues.

The launch keys come from the library itself (imagd_gemm_debug_log) during one eager step at each batch size, so the
shape list is never written by hand. Every key is then timed with the automatic configuration and with each forced
variant (N tile, ring depth, split-K). Each timing is a CUDA graph of --iters back-to-back launches (no host launch
gaps), after a warm-up replay; operands stay in L2 between launches as they partly do in the step.

Printed per variant: time per launch, useful TFLOP/s, the modelled L2 -> shared-memory operand bytes and the rate
they imply. The model: every CTA streams kb k-blocks of A (128 pixels x 64 channels, 16 KB) and B (BLOCK_N x 64,
BLOCK_N x 128 B).

    python tools/gemm_bench.py [--batches 1,8] [--iters 50] [--json OUT.json] [--no-variants]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ["IMAGD_DDIM_STEPS"] = os.environ.get("IMAGD_DDIM_STEPS", "2")
import torch

STAGES = {64: (4, 8), 128: (3, 6), 160: (3, 5), 256: (2, 4)}  # (shallow, deep) ring depths the library instantiates


def step_keys(lib, pipe, B, dev):
    """Launch keys (with the automatic configuration and launch count) of one eager denoising step at batch B."""
    import bench

    x = bench.synth_inputs(B, dev)
    bench.run_pipe(pipe, x)
    eng = pipe._engine
    st = next(iter(eng._states.values()))
    st["step_ptr"].zero_()
    lib.imagd_gemm_debug_log(1, None, 0)
    eng._step(st)
    torch.cuda.synchronize()
    n = lib.imagd_gemm_debug_log(0, None, 0)
    buf = bytes(256 * (n + 1))
    lib.imagd_gemm_debug_log(-1, buf, len(buf))
    st["step_ptr"].zero_()
    out = []
    for line in buf.split(b"\0", 1)[0].decode().splitlines():
        key, cfg, count = (s.split() for s in line.split("|"))
        out.append(([int(v) for v in key], [int(v) for v in cfg], int(count[0])))
    return out


def model(key, bn):
    """(useful FLOP, modelled L2 -> SMEM operand bytes) of one launch."""
    taps, NB, H, W, Cin, N, geglu, m_tiles, kb, fp32 = key
    n_tiles = -(-N // bn) * (4 if taps == 4 else 1)
    pixels = NB * H * W * (4 if taps == 4 else 1)
    flop = 2.0 * pixels * N * taps * Cin
    return flop, m_tiles * n_tiles * kb * (16384.0 + bn * 128.0)


def make_call(key, dev):
    from imagdressing_b200 import ops

    taps, NB, H, W, Cin, N, geglu, m_tiles, kb, fp32 = key
    g = torch.Generator(device="cpu").manual_seed(0)
    r = lambda *s: torch.randn(*s, generator=g).to(dev, torch.bfloat16)
    if taps == 1:
        a, w, bias = r(W, Cin), r(N, Cin), torch.randn(N, generator=g).to(dev)
        act = ops.ACT_GEGLU if geglu else ops.ACT_NONE
        out = torch.empty(W, N // 2 if geglu else N, device=dev, dtype=torch.float32 if fp32 else torch.bfloat16)
        return lambda: ops.gemm(a, w, out=out, bias=bias, act=act, out_fp32=bool(fp32))
    x, bias = r(NB, H, W, Cin), torch.randn(N, generator=g).to(dev)
    if taps == 9:
        w, out = r(N, 9 * Cin), torch.empty(NB, H, W, N, device=dev, dtype=torch.bfloat16)
        return lambda: ops.conv3x3(x, w, out=out, bias=bias)
    w, out = r(4 * N, 4 * Cin), torch.empty(NB, 2 * H, 2 * W, N, device=dev, dtype=torch.bfloat16)
    return lambda: ops.upconv3x3(x, w, out=out, bias=bias)


def time_call(fn, iters):
    fn()  # eager first: allocates the split-K scratch outside the capture
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(iters):
            fn()
    graph.replay()
    best = 1e30
    for _ in range(3):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        graph.replay()
        e1.record()
        torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1) * 1e3 / iters)
    del graph
    return best


def variants(key):
    taps, NB, H, W, Cin, N, geglu, m_tiles, kb, fp32 = key
    base = []
    for bn in ((128,) if geglu else (64, 128, 160, 256)):
        for st in STAGES[bn]:
            base.append((bn, st, 1))
    if kb >= 60 and taps != 4 and not geglu:
        for bn in (64, 128, 160):
            for sp in (2, 3, 4, 6):
                base.append((bn, STAGES[bn][1], sp))
    return base


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,8")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--json", default=None)
    ap.add_argument("--no-variants", action="store_true", help="time the automatic configuration only")
    args = ap.parse_args()

    import bench
    from imagdressing_b200 import _lib

    dev = torch.device("cuda:0")
    lib = _lib.load()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                          "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"# {smi} | {torch.cuda.get_device_name(0)}", flush=True)
    pipe = bench.build_product(dev)
    records = []
    for B in [int(b) for b in args.batches.split(",")]:
        keys = step_keys(lib, pipe, B, dev)
        tot_launch, tot_auto = sum(c for _, _, c in keys), 0.0
        print(f"## batch {B}: {len(keys)} distinct launch keys, {tot_launch} launches per step", flush=True)
        for key, cfg, count in keys:
            fn = make_call(key, dev)
            rows = []
            todo = [("auto", None)] + ([] if args.no_variants else [(None, v) for v in variants(key)])
            for name, v in todo:
                try:
                    if v is not None:
                        lib.imagd_gemm_debug_force(*v)
                    lib.imagd_gemm_debug_log(1, None, 0)
                    fn()
                    lib.imagd_gemm_debug_log(0, None, 0)
                    buf = bytes(1024)
                    lib.imagd_gemm_debug_log(-1, buf, len(buf))
                    ran = [int(t) for t in buf.split(b"\0", 1)[0].decode().split("|")[1].split()]
                    us = time_call(fn, args.iters)
                except Exception as e:  # a variant the library rejects for this shape (e.g. scratch capacity)
                    print(f"   skip {v}: {str(e)[:100]}")
                    continue
                finally:
                    lib.imagd_gemm_debug_force(0, 0, 0)
                flop, byt = model(key, ran[0])
                rows.append(dict(name=name or "forced", bn=ran[0], stages=ran[1], splits=ran[2], us=us,
                                 tflops=flop / us / 1e6, model_mb=byt / 1e6, gbps=byt / us / 1e3))
            if not rows:
                continue
            auto = rows[0]
            tot_auto += auto["us"] * count
            best = min(rows, key=lambda r: r["us"])
            taps, NB, H, W, Cin, N = key[:6]
            desc = (f"gemm M={W} N={N} K={Cin}" + (" geglu" if key[6] else "") + (" fp32" if key[9] else "")) if taps == 1 \
                else f"{'conv' if taps == 9 else 'upconv'} {NB}x{H}x{W} {Cin}->{N}"
            print(f"{desc:40s} x{count:<3d} m_tiles {key[7]:4d} kb {key[8]:4d}", flush=True)
            for r in sorted(rows, key=lambda r: r["us"]):
                tag = "auto" if r is auto else ("best" if r is best else "")
                print(f"   {tag:4s} bn {r['bn']:3d} st {r['stages']} sp {r['splits']}: "
                      f"{r['us']:8.1f} us {r['tflops']:6.1f} TF/s {r['model_mb']:8.1f} MB {r['gbps']:7.0f} GB/s")
            records.append(dict(batch=B, key=key, auto_cfg=cfg, count=count, rows=rows))
        print(f"## batch {B}: automatic configuration, launch-weighted sum {tot_auto / 1e3:.3f} ms per step", flush=True)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(dict(gpu=smi, records=records), f)


if __name__ == "__main__":
    main()
