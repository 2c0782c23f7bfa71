"""GPU: the generic CFG + sampler-step kernel and the scaled layout kernel against torch fp32 statements of the same
arithmetic, then the public pipelines with DPM-Solver++, Euler and Euler-ancestral (CUDA-graph replayed) against the
oracle loop with the step-by-step oracle schedulers (oracle/samplers.py). Sizes and builders of test_pipeline_gpu.py;
tolerance rel-L2 <= 4e-2 as calibrated there for the bf16 chain."""
import pytest
import torch

from conftest import rel_l2

pytestmark = pytest.mark.gpu
STEPS = 6  # DPM-Solver++ 2M: first-order start, second-order middle, first-order end (lower_order_final)


def _ref_row(eps_c, eps_u, g, x, h, z, row, mask=None, img=None, noise=None, blend=None):
    dx, de, cx, ce, ch, cz = [float(v) for v in row]
    eps = eps_u + g * (eps_c - eps_u)
    new = cx * x + ce * eps + (ch * h if ch != 0 else 0) + (cz * z if cz != 0 else 0)
    d = dx * x + de * eps
    if mask is not None:
        new = (1 - mask) * (float(blend[0]) * img + float(blend[1]) * noise) + mask * new
    return new, d


@torch.no_grad()
def test_sampler_step_kernel_rows_and_graph_counter(cuda_device):
    from imagdressing_b200 import ops

    dev = cuda_device
    g = torch.Generator().manual_seed(0)
    r = lambda *s: torch.randn(*s, generator=g).to(dev)
    n, shape = 2, (2, 4, 24, 20)
    eps_c, eps_u, x0, img, noise = r(*shape), r(*shape), r(*shape), r(*shape), r(*shape)
    z = r(3, *shape)
    mask = (torch.rand(n, 1, 24, 20, generator=g) > 0.5).float().to(dev)
    # row 0: first order, no history read (the history holds NaN: ch = 0 must not read it); row 1: history;
    # row 2: noise; blend rows exercise the inpaint path
    coef = torch.tensor([[1.3, -0.4, 0.9, 0.2, 0.0, 0.0], [1.1, -0.3, 0.8, 0.1, 0.35, 0.0],
                         [0.0, 0.0, 1.0, -0.7, 0.0, 0.45]], device=dev)
    blend = torch.tensor([[0.8, 0.6], [0.9, 0.4], [1.0, 0.0]], device=dev)
    for use_mask in (False, True):
        x = x0.clone()
        h = torch.full(shape, float("nan"), device=dev)
        step = torch.zeros(2, dtype=torch.int32, device=dev)
        xr, hr = x0.clone(), None
        for i in range(3):
            mk = dict(mask=mask, image_latents=img, noise=noise, blend_coef=blend) if use_mask else {}
            ops.cfg_sampler_step(eps_c, eps_u, 6.5, x, coef, step, history=h, step_noise=z, **mk)
            rk = dict(mask=mask, img=img, noise=noise, blend=blend[i]) if use_mask else {}
            xr, hr = _ref_row(eps_c, eps_u, 6.5, xr, hr, z[i], coef[i], **rk)
            assert torch.isfinite(x).all()
            assert rel_l2(x, xr) < 1e-6 and rel_l2(h, hr) < 1e-6
        assert int(step[0]) == 3 and int(step[1]) == 0
    # the step counter across three replays of one captured launch
    x, h = x0.clone(), torch.zeros(shape, device=dev)
    step = torch.zeros(2, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.cfg_sampler_step(eps_c, eps_u, 6.5, x, coef, step, history=h, step_noise=z)
    x.copy_(x0)
    step.zero_()
    xr, hr = x0.clone(), None
    for i in range(3):
        graph.replay()
        xr, hr = _ref_row(eps_c, eps_u, 6.5, xr, hr, z[i], coef[i])
    torch.cuda.synchronize()
    assert int(step[0]) == 3 and rel_l2(x, xr) < 1e-6


@torch.no_grad()
def test_scaled_layout_kernel(cuda_device):
    from imagdressing_b200 import ops

    dev = cuda_device
    x = torch.randn(2, 4, 12, 10, generator=torch.Generator().manual_seed(1)).to(dev)
    scale = torch.tensor([0.25, 0.5, 0.125], device=dev)
    step = torch.tensor([2, 0], dtype=torch.int32, device=dev)
    y = ops.nchw_f32_to_nhwc_bf16_scaled(x, scale, step, repeat=2)
    ref = (x * 0.125).permute(0, 2, 3, 1).repeat(2, 1, 1, 1).to(torch.bfloat16)
    assert y.shape == (4, 12, 10, 4) and torch.equal(y, ref)
    y0 = ops.nchw_f32_to_nhwc_bf16_scaled(x, scale, None)
    assert torch.equal(y0, (x * 0.25).permute(0, 2, 3, 1).to(torch.bfloat16))


def _product(kind):
    """`X.from_config(ddim.config)` of the reference's DDIM configuration (what a user of the scripts would write)."""
    from imagdressing_b200 import samplers
    from imagdressing_b200.scheduler import DDIMScheduler

    cls = dict(dpm=samplers.DPMSolverMultistepScheduler, euler=samplers.EulerDiscreteScheduler,
               ea=samplers.EulerAncestralDiscreteScheduler)[kind]
    ddim = DDIMScheduler(num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear",
                         clip_sample=False, set_alpha_to_one=False, steps_offset=1)
    return cls.from_config(ddim.config)


def _oracle(kind, seed=None):
    from oracle.samplers import DPMSolverOracle, EulerOracle

    if kind == "dpm":
        return DPMSolverOracle()
    return EulerOracle(ancestral=kind == "ea", generator=torch.Generator().manual_seed(seed) if seed is not None else None)


def _call(pipe, x, steps, **kw):
    from test_pipeline_gpu import H, W

    return pipe(prompt=None, null_prompt=None, negative_prompt=None, ref_image=None, width=W * 8, height=H * 8,
                num_inference_steps=steps, guidance_scale=7.5, image_scale=1.0, output_type="latent",
                prompt_embeds=x["prompt"], negative_prompt_embeds=x["negative"], latents=x["latents"],
                garment_tokens=x["gtok"], ref_image_latents=x["garment"], **kw).images


@torch.no_grad()
def test_base_pipeline_each_sampler_and_switching(cuda_device):
    from dressing_sd.pipelines.IMAGDressing_v1_pipeline import IMAGDressing_v1
    from oracle.samplers import sample_one
    from test_pipeline_gpu import build, inputs

    dev = cuda_device
    (o, ro, _), (p, rp, _), sched = build(dev)
    pipe = IMAGDressing_v1(vae=None, reference_unet=rp, unet=p, tokenizer=None, text_encoder=None, image_encoder=None,
                           ImgProj=None, scheduler=sched, safety_checker=None, feature_extractor=None)
    x = inputs(dev, 42)
    ddim_first = _call(pipe, x, STEPS)
    for kind in ("dpm", "euler", "ea"):
        pipe.scheduler = _product(kind)
        outs = []
        for seed in (42, 43):  # two images back to back: no history or noise leaks from the first into the second
            xi = inputs(dev, seed)
            ref = sample_one(o, ro, xi["latents"], xi["prompt"], xi["negative"], xi["gtok"], xi["garment"], 7.5, STEPS,
                             _oracle(kind, 7))
            out = _call(pipe, xi, STEPS, generator=torch.Generator().manual_seed(7))
            err = rel_l2(out, ref)
            print(f"{kind} seed {seed}: final-latent rel-L2 {err:.4f}")
            assert torch.isfinite(out).all() and err < 4e-2
            outs.append(out)
        assert rel_l2(outs[1], outs[0]) > 0.3
    # DDIM -> DPM-Solver++ / Euler / Euler-a -> DDIM on one pipeline object: the last DDIM result is bit-identical to a fresh pipeline's
    pipe.scheduler = sched
    again = _call(pipe, x, STEPS)
    fresh = IMAGDressing_v1(vae=None, reference_unet=rp, unet=p, tokenizer=None, text_encoder=None, image_encoder=None,
                            ImgProj=None, scheduler=type(sched).from_config(sched.config), safety_checker=None, feature_extractor=None)
    assert torch.equal(again, ddim_first) and torch.equal(_call(fresh, x, STEPS), ddim_first)


@torch.no_grad()
def test_inpainting_euler_and_controlnet_dpm(cuda_device):
    from dressing_sd.pipelines.IMAGDressing_v1_pipeline_controlnet import IMAGDressing_v1 as PControl
    from dressing_sd.pipelines.IMAGDressing_v1_pipeline_controlnet_inpainting import IMAGDressing_v1 as PInpaint
    from oracle.samplers import sample_one
    from test_pipeline_gpu import H, W, build, inputs

    dev = cuda_device
    (o, ro, co), (p, rp, cp), _ = build(dev, controlnet=True)
    # ControlNet pose pipeline with DPM-Solver++ 2M
    pc = PControl(vae=None, reference_unet=rp, unet=p, tokenizer=None, text_encoder=None, controlnet=cp, image_encoder=None,
                  ImgProj=None, scheduler=_product("dpm"), safety_checker=None, feature_extractor=None)
    x = inputs(dev, 44)
    ref = sample_one(o, ro, x["latents"], x["prompt"], x["negative"], x["gtok"], x["garment"], 7.0, STEPS, _oracle("dpm"),
                     controlnet=co, control_cond=x["pose"], control_scale=0.8)
    out = pc(prompt=None, null_prompt=None, negative_prompt=None, ref_image=None, width=W * 8, height=H * 8,
             num_inference_steps=STEPS, guidance_scale=7.0, pose_image=x["pose"], output_type="latent",
             prompt_embeds=x["prompt"], negative_prompt_embeds=x["negative"], latents=x["latents"],
             garment_tokens=x["gtok"], ref_image_latents=x["garment"], controlnet_conditioning_scale=0.8).images
    err = rel_l2(out, ref)
    print(f"controlnet dpm: final-latent rel-L2 {err:.4f}")
    assert err < 4e-2
    # inpainting with Euler: sigma-space blend, scaled ControlNet input, start = noise * init_noise_sigma
    pin = PInpaint(vae=None, reference_unet=rp, unet=p, tokenizer=None, text_encoder=None, controlnet=cp,
                   image_encoder=None, ImgProj=None, scheduler=_product("euler"), safety_checker=None,
                   feature_extractor=None)
    x = inputs(dev, 48)
    g = torch.Generator().manual_seed(49)
    img_lat = torch.randn(1, 4, H, W, generator=g).to(dev)
    mask = torch.zeros(1, 1, H, W, device=dev)
    mask[:, :, H // 4: 3 * H // 4, W // 4: 3 * W // 4] = 1.0
    noise = x["latents"]
    ref = sample_one(o, ro, noise, x["prompt"], x["negative"], x["gtok"], x["garment"], 5.0, STEPS, _oracle("euler"),
                     controlnet=co, control_cond=x["pose"], control_scale=0.5, mask=mask, image_latents=img_lat,
                     noise=noise)
    out = pin(prompt=None, null_prompt=None, negative_prompt=None, ref_image=None, control_image=x["pose"], height=H * 8,
              width=W * 8, strength=1.0, num_inference_steps=STEPS, guidance_scale=5.0, latents=noise,
              prompt_embeds=x["prompt"], negative_prompt_embeds=x["negative"], output_type="latent",
              controlnet_conditioning_scale=0.5, garment_tokens=x["gtok"], ref_image_latents=x["garment"],
              image_latents=img_lat, mask_latents=mask).images
    err = rel_l2(out, ref)
    print(f"inpainting euler: final-latent rel-L2 {err:.4f}")
    assert err < 4e-2
    keep = (mask == 0).expand_as(out)
    assert rel_l2(out[keep], img_lat[keep]) < 1e-5
