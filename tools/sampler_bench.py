"""Images/s of the base pipeline (512x512, synthetic SD1.5-shaped weights) per sampler, the per-launch time of the
sampler-step kernels next to the CFG+DDIM kernel, and the solver error of the few-step samplers.
    python tools/sampler_bench.py [--rounds 3] [--reps 3]
Arms: DDIM-50, DPM-Solver++ 2M-20, DPM-Solver++ 2M-25, Euler-ancestral-30, UniPC-10 / 15 / 20 (bh2, order 2), at batch
1 and 8. Each round runs every arm in turn (a warm-up call that captures the arm's step graph, then `reps` timed calls);
rounds alternate the arms so clock drift hits them alike. Times are CUDA events around whole pipeline calls (garment
pass + denoising loop, output latents); the median over rounds is reported. The card name and its power limit are
printed with the figures.
Accuracy (reported, not asserted): the final-latent rel-L2 of UniPC-10, DPM++2M-10 and DPM++2M-20 against a 250-step
DPM++2M run of the same random-init pipeline, inputs and seed at batch 1. Every accuracy run uses trailing spacing, so
all of them integrate the same initial-value problem, from t = 999 down to alphas_cumprod[0] (with the DDIM config's
leading spacing the first timestep depends on the step count). That is the solver error on this model's
probability-flow ODE; it says nothing about image quality with trained weights."""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import bench
from imagdressing_b200 import ops
from imagdressing_b200.samplers import (DPMSolverMultistepScheduler, EulerAncestralDiscreteScheduler,
                                        UniPCMultistepScheduler)

ARMS = (("DDIM-50", None, 50), ("DPM++2M-20", DPMSolverMultistepScheduler, 20),
        ("DPM++2M-25", DPMSolverMultistepScheduler, 25), ("Euler-a-30", EulerAncestralDiscreteScheduler, 30),
        ("UniPC-10", UniPCMultistepScheduler, 10), ("UniPC-15", UniPCMultistepScheduler, 15),
        ("UniPC-20", UniPCMultistepScheduler, 20))


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        q = f"nvidia-smi unavailable ({type(e).__name__})"
    return name, q


def time_call(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def step_kernels(dev, B, launches=100):
    """Mean µs per launch of cfg_ddim_step, of the sampler step with a history row (DPM-Solver++ 2M) and with a noise
    row (Euler-ancestral), and of the predictor-corrector step with a UniPC-20 middle row (corrector and order-2
    predictor: three slot reads, two slot writes), on the CFG batch of B 512x512 latents."""
    shape = (B, 4, 64, 64)
    eps = torch.randn(2 * B, *shape[1:], device=dev)
    lat, hist = torch.randn(shape, device=dev), torch.zeros(shape, device=dev)
    z = torch.randn(launches, *shape, device=dev)
    step = torch.zeros(2, dtype=torch.int32, device=dev)
    ddim = torch.tensor([[0.9, 0.4, 0.95, 0.3]], device=dev).repeat(launches, 1)
    dpm = torch.tensor([[1.1, -0.3, 0.8, 0.1, 0.35, 0.0]], device=dev).repeat(launches, 1)
    ea = torch.tensor([[0.0, 0.0, 1.0, -0.2, 0.0, 0.1]], device=dev).repeat(launches, 1)
    unipc = UniPCMultistepScheduler()
    unipc.set_timesteps(20)
    pc = torch.tensor([unipc._row(5, 5)], device=dev).repeat(launches, 1)
    bank = torch.randn(ops.PC_SLOTS, *shape, device=dev)
    runs = {"cfg_ddim_step": lambda: ops.cfg_ddim_step(eps[:B], eps[B:], 7.5, lat, ddim, step),
            "cfg_sampler_step (history)": lambda: ops.cfg_sampler_step(eps[:B], eps[B:], 7.5, lat, dpm, step,
                                                                        history=hist),
            "cfg_sampler_step (noise)": lambda: ops.cfg_sampler_step(eps[:B], eps[B:], 7.5, lat, ea, step,
                                                                      step_noise=z),
            "cfg_sampler_pc_step (UniPC)": lambda: ops.cfg_sampler_pc_step(eps[:B], eps[B:], 7.5, lat, pc, step, bank)}
    out = {}
    for name, run in runs.items():
        step.zero_()
        run()
        step.zero_()
        torch.cuda.synchronize()

        def loop():
            for _ in range(launches):
                run()
        out[name] = round(time_call(loop) * 1000.0 / launches, 2)
    return out


def accuracy(pipe, ddim, dev):
    """Final-latent rel-L2 of the few-step arms against DPM++2M-250 on the same inputs and seed (batch 1), all on
    trailing spacing: the same start (t = 999) and end (alphas_cumprod[0]) for every step count."""
    x = bench.synth_inputs(1, dev, 0, False, "base", 64, 64)

    def run(cls, steps):
        pipe.scheduler = cls.from_config(ddim.config, timestep_spacing="trailing")
        return pipe(prompt=None, null_prompt=None, negative_prompt=None, ref_image=None, width=512, height=512,
                    num_inference_steps=steps, guidance_scale=bench.GUIDANCE, image_scale=1.0, output_type="latent",
                    prompt_embeds=x["prompt"], negative_prompt_embeds=x["negative"], latents=x["latents"],
                    garment_tokens=x["gtok"], ref_image_latents=x["garment"],
                    generator=torch.Generator().manual_seed(0)).images.float()

    ref = run(DPMSolverMultistepScheduler, 250)
    out = {}
    arms = (("UniPC-10", UniPCMultistepScheduler, 10), ("DPM++2M-10", DPMSolverMultistepScheduler, 10),
            ("DPM++2M-20", DPMSolverMultistepScheduler, 20))
    for label, cls, steps in arms:
        out[label] = round(float((run(cls, steps) - ref).norm() / ref.norm()), 5)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--batches", default="1,8")
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    torch.backends.cuda.matmul.allow_tf32 = False
    name, limits = card()
    print(f"card: {name}; power limit, max SM clock: {limits}")
    pipe = bench.build_product(dev, "base")
    ddim = pipe.scheduler
    scheds = {label: (ddim if cls is None else cls.from_config(ddim.config)) for label, cls, _ in ARMS}
    result = {"card": name, "power_limit_max_sm_clock": limits, "arms": {}, "step_kernel_us": {}}
    for B in [int(b) for b in a.batches.split(",")]:
        x = bench.synth_inputs(B, dev, 0, False, "base", 64, 64)
        times = {label: [] for label, _, _ in ARMS}
        for _ in range(a.rounds):
            for label, _, steps in ARMS:
                pipe.scheduler = scheds[label]

                def call():
                    pipe(prompt=None, null_prompt=None, negative_prompt=None, ref_image=None, width=512, height=512,
                         num_inference_steps=steps, guidance_scale=bench.GUIDANCE, image_scale=1.0,
                         output_type="latent", prompt_embeds=x["prompt"], negative_prompt_embeds=x["negative"],
                         latents=x["latents"], garment_tokens=x["gtok"], ref_image_latents=x["garment"],
                         generator=torch.Generator().manual_seed(0))
                time_call(call)  # warm-up: captures this arm's step graph (one resident graph per pipeline)
                ms = statistics.median(time_call(call) for _ in range(a.reps))
                times[label].append(ms)
        for label, _, steps in ARMS:
            ms = statistics.median(times[label])
            ips = B * 1000.0 / ms
            result["arms"][f"{label} B={B}"] = {"ms_per_call": round(ms, 1), "images_per_s": round(ips, 3),
                                                "ms_per_step": round(ms / steps, 2), "rounds_ms": [round(t, 1) for t in times[label]]}
            print(f"B={B:<2} {label:<11} {ms:9.1f} ms/call  {ips:7.3f} img/s  {ms / steps:6.2f} ms/step  "
                  f"rounds {[round(t, 1) for t in times[label]]}")
        result["step_kernel_us"][f"B={B}"] = k = step_kernels(dev, B)
        print(f"B={B:<2} step kernels (µs per launch): {k}")
    result["accuracy_rel_l2_vs_dpm2m_250"] = acc = accuracy(pipe, ddim, dev)
    print(f"final-latent rel-L2 vs DPM++2M-250 (B=1, random-init weights): {acc}")
    pipe.scheduler = ddim
    print(json.dumps(result))


if __name__ == "__main__":
    main()
