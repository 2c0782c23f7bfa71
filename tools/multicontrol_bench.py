"""Cost of several ControlNets in one call, with the card it ran on (name, power limit, max SM clock read in the same run):

  1. images/s and ms/step of the ControlNet-pose pipeline at 512x512, batch 1 and 8, DDIM-50 and UniPC-10, for the arms
       single   one ControlNetModel (host-float scale, the step graph of the single-net path)
       multi1   MultiControlNetModel([cn])                 (scale table, one graph per active set)
       multi2   MultiControlNetModel([cn, cn2])
       window2  the same pair with complementary guidance windows [0, 0.5] / [0.5, 1]
       inpaint2 the inpainting pipeline with an inpaint-style and a pose ControlNet
     all arms alternated in one process, `reps` calls each;
  2. the peak reserved memory of each arm's first call (step-graph and garment-pass captures included), measured after
     every arm has run once (so all weights are packed and every per-net cache exists) and then every arm's captured
     graphs have been released: `max_reserved_mb` is the peak, `own_mb` the peak minus what was reserved before the call
     (weights and caches), i.e. the memory the arm's own graphs and activations need;
  3. the per-launch device time of a level-0 and the mid zero-conv GEMM reading its scale from the table, with and
     without the chained residual, against the host-alpha launch, alternated over many launches.

    python tools/multicontrol_bench.py [--out results/multicontrol_bench.json] [--reps 3]
Synthetic weights. Prints one JSON object."""
import argparse
import gc
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

HW = 64  # latent side: 512 x 512 images


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def zero_conv_launches(dev, reps=200):
    """Device time per launch (us; mean, min and max of 5 blocks, the arms alternated block by block) of the level-0 and
    mid zero-conv GEMMs at batch 1 and 8. Each block replays a CUDA graph of `reps` launches, as the step graph does, so
    the host-side cost of the Python wrapper is not in the figure."""
    from imagdressing_b200 import ops

    out = {}
    for B in (1, 8):
        for name, (hw, C) in (("level0", (HW, 320)), ("mid", (HW // 8, 1280))):
            NB = 2 * B  # the CFG batch
            g = torch.Generator(device=dev).manual_seed(0)
            x = torch.randn(NB, hw, hw, C, device=dev, generator=g).to(torch.bfloat16)
            w = (torch.randn(C, C, device=dev, generator=g) / C ** 0.5).to(torch.bfloat16)
            b = torch.randn(C, device=dev, generator=g) * 0.02
            res = torch.randn(NB, hw, hw, C, device=dev, generator=g).to(torch.bfloat16)
            table = torch.full((50, 2), 0.8, device=dev)
            step = torch.tensor([17, 0], dtype=torch.int32, device=dev)
            y = torch.empty_like(x)
            bs = b * 0.8
            arms = {"host_alpha": lambda: ops.gemm(x, w, bias=bs, alpha=0.8, out=y),
                    "table": lambda: ops.gemm(x, w, bias=b, scale_table=table[:, 1], scale_step=step, out=y),
                    "table_residual": lambda: ops.gemm(x, w, bias=b, residual=res, scale_table=table[:, 1],
                                                       scale_step=step, out=y)}
            times = {k: [] for k in arms}
            graphs = {}
            for k, fn in arms.items():
                fn()  # eager first: sizes the split-K scratch outside the capture
                torch.cuda.synchronize()
                graphs[k] = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graphs[k]):
                    for _ in range(reps):
                        fn()
                graphs[k].replay()
            torch.cuda.synchronize()
            for _ in range(5):
                for k in arms:
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    graphs[k].replay()
                    e1.record()
                    torch.cuda.synchronize()
                    times[k].append(e0.elapsed_time(e1) * 1e3 / reps)
            out[f"{name}_b{B}"] = {k: {"us_mean": round(sum(v) / len(v), 2), "us_min": round(min(v), 2),
                                       "us_max": round(max(v), 2)} for k, v in times.items()}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    import bench
    from dressing_sd.pipelines.IMAGDressing_v1_pipeline_controlnet import IMAGDressing_v1 as PPose
    from dressing_sd.pipelines.IMAGDressing_v1_pipeline_controlnet_inpainting import IMAGDressing_v1 as PInpaint
    from imagdressing_b200 import _lib, modeling
    from imagdressing_b200.modeling import MultiControlNetModel
    from imagdressing_b200.samplers import UniPCMultistepScheduler
    from imagdressing_b200.scheduler import DDIMScheduler

    _lib.require_b200()
    dev = torch.device("cuda:0")
    res = dict(card=card(), size="512x512")
    res["zero_conv_us"] = zero_conv_launches(dev)

    base = bench.build_product(dev, "inpaint")  # denoising UNet, garment UNet, one ControlNet
    unet, ref, cn = base.unet, base.reference_unet, base.controlnet
    with modeling.skip_default_init():
        cn2 = modeling.ControlNetModel().to(dev, torch.bfloat16)
    modeling.init_synthetic_fast_(cn2, 3)

    def ddim():
        return DDIMScheduler(num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear",
                             clip_sample=False, set_alpha_to_one=False, steps_offset=1)

    def make(cls, controlnet, sched):
        return cls(vae=None, reference_unet=ref, unet=unet, tokenizer=None, text_encoder=None, controlnet=controlnet,
                   image_encoder=None, ImgProj=None, scheduler=sched, safety_checker=None, feature_extractor=None)

    configs = [(1, "ddim", 50), (1, "unipc", 10), (8, "ddim", 50), (8, "unipc", 10)]
    rows = []
    for B, sampler, steps in configs:
        sch = ddim() if sampler == "ddim" else UniPCMultistepScheduler.from_config(ddim().config)
        x = bench.synth_inputs(B, dev, 0, False, "inpaint", HW, HW)
        pose2 = torch.rand_like(x["pose"])
        kw = dict(prompt=None, null_prompt=None, negative_prompt=None, ref_image=None, num_inference_steps=steps,
                  guidance_scale=7.5, output_type="latent", prompt_embeds=x["prompt"], negative_prompt_embeds=x["negative"],
                  latents=x["latents"], garment_tokens=x["gtok"], ref_image_latents=x["garment"])
        pose_kw = dict(width=HW * 8, height=HW * 8, **kw)
        arms = {
            "single": (make(PPose, cn, sch), dict(pose_image=x["pose"], controlnet_conditioning_scale=1.0, **pose_kw)),
            "multi1": (make(PPose, MultiControlNetModel([cn]), sch),
                       dict(pose_image=[x["pose"]], controlnet_conditioning_scale=1.0, **pose_kw)),
            "multi2": (make(PPose, [cn, cn2], sch),
                       dict(pose_image=[x["pose"], pose2], controlnet_conditioning_scale=[1.0, 0.8], **pose_kw)),
            "window2": (make(PPose, [cn, cn2], sch),
                        dict(pose_image=[x["pose"], pose2], controlnet_conditioning_scale=[1.0, 0.8],
                             control_guidance_start=[0.0, 0.5], control_guidance_end=[0.5, 1.0], **pose_kw)),
            "inpaint2": (make(PInpaint, [cn, cn2], sch),
                         dict(control_image=[x["pose"], pose2], controlnet_conditioning_scale=[0.5, 1.0], strength=1.0,
                              image_latents=x["image_latents"], mask_latents=x["mask"], **kw)),
        }

        def drop_graphs():  # every engine's step graphs and its garment-pass graph, each in its own pool
            for p, _ in arms.values():
                p._engine._states = {}
                p._engine._garment = None
            gc.collect()
            torch.cuda.empty_cache()

        # 2. each arm's peak reserved memory, alone
        for p, call in arms.values():  # packs every net's weights and fills the per-net caches once
            p(**call)
        mem = {}
        for name, (p, call) in arms.items():
            drop_graphs()
            before = torch.cuda.memory_reserved()
            torch.cuda.reset_peak_memory_stats()
            p(**call)
            torch.cuda.synchronize()
            peak = torch.cuda.max_memory_reserved()
            mem[name] = (peak / 2 ** 20, (peak - before) / 2 ** 20)
        drop_graphs()
        for p, call in arms.values():  # capture every arm's graphs (they then stay resident together)
            p(**call)
        torch.cuda.synchronize()
        # 1. alternated timed calls
        t = {k: [] for k in arms}
        for _ in range(a.reps):
            for name, (p, call) in arms.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                p(**call)
                torch.cuda.synchronize()
                t[name].append(time.perf_counter() - t0)
        for name in arms:
            best, worst = min(t[name]), max(t[name])
            rows.append(dict(arm=name, batch=B, sampler=f"{sampler}-{steps}", img_s=round(B / best, 3),
                             img_s_slowest=round(B / worst, 3), ms_step=round(best * 1e3 / steps, 2),
                             ms_step_slowest=round(worst * 1e3 / steps, 2), max_reserved_mb=round(mem[name][0]),
                             own_mb=round(mem[name][1])))
            print(json.dumps(rows[-1]), file=sys.stderr)
        drop_graphs()
        del arms
        gc.collect()
        torch.cuda.empty_cache()
    res["pipelines"] = rows
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
