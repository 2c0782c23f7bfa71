"""Cost of global-norm gradient clipping (FlatAdamW(max_grad_norm=)) on the training step of BASELINE.json configs[4].

1. The norm pass alone (imagd_grad_norm_clip) over the real flat gradient buffer of SDModel's trainable set (random-init
   weights), CUDA events over --launches launches: time per pass and achieved bytes/s against the H100 SXM data-sheet
   3.35 TB/s (the pass reads the bf16 buffer once; its other traffic is a few KB).
2. The captured training step (GraphedTrainStep, micro-batch --batch at --height x --width) with clipping off and on,
   alternated for --rounds rounds. Each arm is captured afresh in its round (one graph's memory pool at a time) and timed
   over --steps replays after the capture's warm-up.

The card's name, power limit and max SM clock are printed first: every number below belongs to them. Needs an H100."""
import argparse
import gc
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import bench

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def card() -> str:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "nvidia-smi unavailable"


def events(fn, n: int) -> float:
    """ms per call of fn over n calls, CUDA events around the whole run."""
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def build(dev, max_grad_norm):
    """bench.build_train's SDModel, with FlatAdamW holding the clipping state (max_grad_norm)."""
    from adapter.resampler import Resampler
    from imagdressing_b200 import modeling, train

    pipe = bench.build_product(dev, "base")
    unet, ref = pipe.unet, pipe.reference_unet
    proj = Resampler(dim=768, depth=4, dim_head=64, heads=12, num_queries=16, embedding_dim=1280, output_dim=768, ff_mult=4)
    proj = proj.to(dev, torch.bfloat16)
    modeling.init_synthetic_fast_(proj, 3)
    adapters = torch.nn.ModuleList(unet.attn_processors.values())
    params = train.set_trainable(unet, ref, proj, adapters)
    sd = train.SDModel(unet, ref, proj, adapters)
    opt = train.FlatAdamW(params, lr=1e-5, weight_decay=1e-2, max_grad_norm=max_grad_norm)
    return sd, opt, pipe.scheduler


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--height", type=int, default=640)
    ap.add_argument("--width", type=int, default=512)
    ap.add_argument("--max-grad-norm", type=float, default=1.0)
    a = ap.parse_args()

    from imagdressing_b200 import _lib, ops, train

    _lib.require_b200()
    dev = torch.device("cuda:0")
    info = card()
    print(f"card (name, power limit, max SM clock): {info}", flush=True)
    sd, opt, sched = build(dev, a.max_grad_norm)
    n = opt.grad.numel()

    # ---- 1. the norm pass alone, on the real buffer (its own state: the optimizer's stays untouched)
    grad = (torch.randn(n, device=dev) * 1e-4).to(torch.bfloat16)
    hyper = opt.hyper.clone()
    state = torch.zeros(4, device=dev, dtype=torch.float64)
    ws = torch.zeros(ops.grad_norm_ws_bytes(n), device=dev, dtype=torch.uint8)
    run = lambda: ops.grad_norm_clip(grad, hyper, state, ws, max_norm=a.max_grad_norm)
    events(run, 10)
    ms_norm = events(run, a.launches)
    del grad
    norm_pass = {"elements": n, "bytes": 2 * n, "launches": a.launches, "us_per_pass": round(ms_norm * 1e3, 1),
                 "TB_per_s": round(2 * n / (ms_norm * 1e-3) / 1e12, 3),
                 "frac_of_3.35TB/s": round(2 * n / (ms_norm * 1e-3) / HBM_BYTES_PER_S, 3)}
    print("norm pass:", json.dumps(norm_pass), flush=True)

    # ---- 2. the captured step, clipping off / on alternated (the same optimizer: max_grad_norm = None takes the plain path)
    x = bench.synth_train_batch(a.batch, dev, 0, False, a.height // 8, a.width // 8)
    arms = {"off": [], "on": []}
    launches, norms = {}, []
    for r in range(a.rounds):
        for arm in ("off", "on"):
            opt.max_grad_norm = None if arm == "off" else a.max_grad_norm
            step = train.GraphedTrainStep(sd, sched, opt, x)
            launches[arm] = step.launches_per_step
            step(**x)
            ms = events(lambda: step(**x), a.steps)
            arms[arm].append(ms)
            if arm == "on":
                norms.append(float(opt.last_grad_norm))
            print(f"round {r} clipping {arm}: {ms:.2f} ms per step", flush=True)
            del step
            gc.collect()
            torch.cuda.empty_cache()
    off, on = statistics.median(arms["off"]), statistics.median(arms["on"])
    result = {"card": info, "norm_pass": norm_pass,
              "step": {"batch": a.batch, "height": a.height, "width": a.width, "steps_per_round": a.steps,
                       "ms_off": [round(v, 2) for v in arms["off"]], "ms_on": [round(v, 2) for v in arms["on"]],
                       "median_ms_off": round(off, 2), "median_ms_on": round(on, 2),
                       "overhead_frac": round((on - off) / off, 4), "library_launches": launches,
                       "max_grad_norm": a.max_grad_norm, "pre_clip_norms": [round(v, 4) for v in norms]}}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
