"""GPU: the CFG + predictor-corrector step kernel (imagd_cfg_sampler_pc_step) against a torch fp32 statement of the same
arithmetic, then the public pipelines with UniPCMultistepScheduler (CUDA-graph replayed) against the oracle loop with
the diffusers-style UniPC oracle (unipc_oracle.py). Sizes and builders of test_pipeline_gpu.py; tolerance rel-L2 <= 4e-2
as calibrated there for the bf16 chain."""
import pytest
import torch

from conftest import rel_l2

pytestmark = pytest.mark.gpu
STEPS = 6  # order 2 / 3: first-order start, the corrector from step 1, lower orders at the end (lower_order_final)

# rows {dx, de, ax, am, a0..a3, bc, bm, b0..b3, w_m, w_c}: row 0 reads no slot (the bank holds NaN), later rows read
# more slots, row 3 overwrites the slots it reads and swaps the stash / data-prediction roles, row 4 reads them back
ROWS = [[1.3, -0.4, 1.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.9, 0.2, 0.0, 0.0, 0.0, 0.0, 0, 3],
        [1.1, -0.3, 0.0, 0.25, 0.3, 0.0, 0.0, 0.5, 0.8, 0.1, -0.2, 0.0, 0.0, 0.0, 1, 3],
        [0.9, -0.2, 0.0, 0.2, 0.1, -0.15, 0.0, 0.6, 0.85, 0.05, 0.1, -0.3, 0.0, 0.0, 2, 3],
        [1.2, -0.5, 0.0, 0.3, -0.1, 0.2, 0.15, 0.4, 0.7, 0.15, 0.05, 0.1, -0.25, 0.0, 3, 0],
        [1.0, -0.1, 0.0, 0.1, 0.35, 0.0, 0.0, 0.45, 0.95, -0.05, 0.0, 0.0, 0.0, 0.2, 1, 2]]


def _ref_row(eps_c, eps_u, g, x, bank, row, mask=None, img=None, noise=None, blend=None):
    r = [float(v) for v in row]
    eps = eps_u + g * (eps_c - eps_u)
    m = r[0] * x + r[1] * eps
    c = r[2] * x + r[3] * m
    new = r[9] * m
    for k in range(4):
        if r[4 + k] != 0 or r[10 + k] != 0:
            c = c + r[4 + k] * bank[k]
            new = new + r[10 + k] * bank[k]
    new = new + r[8] * c
    bank = bank.clone()
    bank[int(r[14])], bank[int(r[15])] = m, c
    if mask is not None:
        new = (1 - mask) * (float(blend[0]) * img + float(blend[1]) * noise) + mask * new
    return new, bank, c


@torch.no_grad()
def test_pc_step_kernel_rows_slots_and_graph_counter(cuda_device):
    from imagdressing_b200 import ops

    dev = cuda_device
    g = torch.Generator().manual_seed(0)
    r = lambda *s: torch.randn(*s, generator=g).to(dev)
    shape = (2, 4, 24, 20)
    eps_c, eps_u, x0, img, noise = r(*shape), r(*shape), r(*shape), r(*shape), r(*shape)
    mask = (torch.rand(2, 1, 24, 20, generator=g) > 0.5).float().to(dev)
    coef = torch.tensor(ROWS, device=dev)
    S = len(ROWS)
    blend = torch.tensor([[0.8, 0.6], [0.9, 0.4], [0.95, 0.3], [0.99, 0.1], [1.0, 0.0]], device=dev)
    for use_mask in (False, True):
        x = x0.clone()
        bank = torch.full((4, *shape), float("nan"), device=dev)
        step = torch.zeros(2, dtype=torch.int32, device=dev)
        xr, br, written = x0.clone(), bank.clone(), set()
        for i in range(S):
            mk = dict(mask=mask, image_latents=img, noise=noise, blend_coef=blend) if use_mask else {}
            ops.cfg_sampler_pc_step(eps_c, eps_u, 6.5, x, coef, step, bank, **mk)
            rk = dict(mask=mask, img=img, noise=noise, blend=blend[i]) if use_mask else {}
            xr, br, cr = _ref_row(eps_c, eps_u, 6.5, xr, br, coef[i], **rk)
            written |= {int(ROWS[i][14]), int(ROWS[i][15])}
            assert torch.isfinite(x).all()
            assert rel_l2(x, xr) < 1e-6
            for k in written:
                assert rel_l2(bank[k], br[k]) < 1e-6
            if use_mask:  # the stash is the corrected sample before the blend
                w_c = int(ROWS[i][15])
                assert rel_l2(bank[w_c], cr) < 1e-6
                assert not torch.allclose(bank[w_c], x)
        assert int(step[0]) == S and int(step[1]) == 0
    # three replays of one captured launch equal three eager launches
    x, bank = x0.clone(), torch.full((4, *shape), float("nan"), device=dev)
    step = torch.zeros(2, dtype=torch.int32, device=dev)
    for _ in range(3):
        ops.cfg_sampler_pc_step(eps_c, eps_u, 6.5, x, coef, step, bank)
    x_eager, bank_eager = x.clone(), bank.clone()
    x.copy_(x0)
    bank.fill_(float("nan"))
    step.zero_()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.cfg_sampler_pc_step(eps_c, eps_u, 6.5, x, coef, step, bank)
    for _ in range(3):
        graph.replay()
    torch.cuda.synchronize()
    assert int(step[0]) == 3 and int(step[1]) == 0
    assert torch.equal(x, x_eager) and torch.equal(bank.nan_to_num(), bank_eager.nan_to_num())


def _unipc(**kw):
    """`UniPCMultistepScheduler.from_config(ddim.config)` of the reference's DDIM configuration."""
    from imagdressing_b200.samplers import UniPCMultistepScheduler
    from imagdressing_b200.scheduler import DDIMScheduler

    ddim = DDIMScheduler(num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear",
                         clip_sample=False, set_alpha_to_one=False, steps_offset=1)
    return UniPCMultistepScheduler.from_config(ddim.config, **kw)


def _call(pipe, x, steps, **kw):
    from test_pipeline_gpu import H, W

    return pipe(prompt=None, null_prompt=None, negative_prompt=None, ref_image=None, width=W * 8, height=H * 8,
                num_inference_steps=steps, guidance_scale=7.5, image_scale=1.0, output_type="latent",
                prompt_embeds=x["prompt"], negative_prompt_embeds=x["negative"], latents=x["latents"],
                garment_tokens=x["gtok"], ref_image_latents=x["garment"], **kw).images


@torch.no_grad()
def test_base_pipeline_unipc_and_switching(cuda_device):
    from dressing_sd.pipelines.IMAGDressing_v1_pipeline import IMAGDressing_v1
    from imagdressing_b200.samplers import DPMSolverMultistepScheduler
    from oracle.samplers import sample_one
    from test_pipeline_gpu import build, inputs
    from unipc_oracle import UniPCOracle

    dev = cuda_device
    (o, ro, _), (p, rp, _), sched = build(dev)
    pipe = IMAGDressing_v1(vae=None, reference_unet=rp, unet=p, tokenizer=None, text_encoder=None, image_encoder=None,
                           ImgProj=None, scheduler=sched, safety_checker=None, feature_extractor=None)
    x = inputs(dev, 42)
    ddim_first = _call(pipe, x, STEPS)
    for bh, order in (("bh2", 2), ("bh1", 3)):
        pipe.scheduler = _unipc(solver_type=bh, solver_order=order)
        outs = []
        for seed in (42, 43):  # two images back to back: nothing leaks from the first into the second through the bank
            xi = inputs(dev, seed)
            ref = sample_one(o, ro, xi["latents"], xi["prompt"], xi["negative"], xi["gtok"], xi["garment"], 7.5, STEPS,
                             UniPCOracle(solver_type=bh, solver_order=order))
            out = _call(pipe, xi, STEPS)
            err = rel_l2(out, ref)
            print(f"unipc {bh} order {order} seed {seed}: final-latent rel-L2 {err:.4f}")
            assert torch.isfinite(out).all() and err < 4e-2
            outs.append(out)
        assert rel_l2(outs[1], outs[0]) > 0.3
        # the eager path (a callback forces it) computes what the replayed step graph computes
        eager = _call(pipe, inputs(dev, 43), STEPS, callback=lambda *a: None)
        print(f"unipc {bh} order {order}: eager vs graph rel-L2 {rel_l2(eager, outs[1]):.3e}")
        assert torch.equal(eager, outs[1])
    # DDIM -> UniPC -> DPM-Solver++ -> DDIM on one pipeline object: the DPM-Solver++ result and the last DDIM result
    # are bit-identical to fresh pipelines' (no UniPC state, bank or kernel choice carries over)
    def fresh(scheduler):
        return IMAGDressing_v1(vae=None, reference_unet=rp, unet=p, tokenizer=None, text_encoder=None,
                               image_encoder=None, ImgProj=None, scheduler=scheduler, safety_checker=None,
                               feature_extractor=None)

    pipe.scheduler = DPMSolverMultistepScheduler.from_config(sched.config)
    dpm_after = _call(pipe, x, STEPS)
    dpm_fresh = _call(fresh(DPMSolverMultistepScheduler.from_config(sched.config)), x, STEPS)
    print(f"DPM-Solver++ after UniPC vs fresh pipeline: rel-L2 {rel_l2(dpm_after, dpm_fresh):.3e}")
    assert torch.equal(dpm_after, dpm_fresh)
    pipe.scheduler = sched
    again = _call(pipe, x, STEPS)
    assert torch.equal(again, ddim_first) and torch.equal(_call(fresh(type(sched).from_config(sched.config)), x, STEPS),
                                                          ddim_first)


@torch.no_grad()
def test_host_step_through_the_kernel_matches_oracle(cuda_device):
    """UniPCMultistepScheduler.step() (one-row table, the scheduler's own bank, no unconditional operand) on the device
    against the oracle's step() on the CPU, step by step, on a smooth state-dependent stand-in for the model."""
    from unipc_oracle import UniPCOracle

    dev = cuda_device
    for bh, order in (("bh2", 2), ("bh1", 3)):
        p, o = _unipc(solver_type=bh, solver_order=order), UniPCOracle(solver_type=bh, solver_order=order)
        p.set_timesteps(8, device=dev)
        o.set_timesteps(8)
        x = torch.randn(2, 4, 16, 16, generator=torch.Generator().manual_seed(11))
        xg = x.to(dev)
        for tp, to in zip(p.timesteps, o.timesteps):
            x = o.step(0.6 * x + 0.2 * torch.cos(x + float(to) / 300.0), to, x)[0]
            xg = p.step(0.6 * xg + 0.2 * torch.cos(xg + float(tp) / 300.0), tp, xg).prev_sample
            assert torch.isfinite(xg).all() and rel_l2(xg.cpu(), x) < 5e-5
        assert p.step_index == 8


class _Windowed:
    """The oracle ControlNet with `controlnet_keep` applied as a zero conditioning scale outside the guidance window."""

    def __init__(self, controlnet, keep):
        self.controlnet, self.keep, self.i = controlnet, keep, 0

    def __call__(self, *args, conditioning_scale, **kw):
        scale = conditioning_scale * self.keep[self.i]
        self.i += 1
        return self.controlnet(*args, conditioning_scale=scale, **kw)


@torch.no_grad()
def test_controlnet_window_and_inpainting_unipc(cuda_device):
    from dressing_sd.pipelines.IMAGDressing_v1_pipeline_controlnet import IMAGDressing_v1 as PControl
    from dressing_sd.pipelines.IMAGDressing_v1_pipeline_controlnet_inpainting import IMAGDressing_v1 as PInpaint
    from oracle.samplers import sample_one
    from test_pipeline_gpu import H, W, build, inputs
    from unipc_oracle import UniPCOracle

    dev = cuda_device
    (o, ro, co), (p, rp, cp), _ = build(dev, controlnet=True)
    # ControlNet pose pipeline inside a guidance window: both step graphs (with / without residuals) share one bank
    pc = PControl(vae=None, reference_unet=rp, unet=p, tokenizer=None, text_encoder=None, controlnet=cp,
                  image_encoder=None, ImgProj=None, scheduler=_unipc(), safety_checker=None, feature_extractor=None)
    x = inputs(dev, 44)
    start, end = 0.2, 0.8
    keep = [1.0 - float(i / STEPS < start or (i + 1) / STEPS > end) for i in range(STEPS)]
    assert 0.0 in keep and 1.0 in keep
    ref = sample_one(o, ro, x["latents"], x["prompt"], x["negative"], x["gtok"], x["garment"], 7.0, STEPS,
                     UniPCOracle(), controlnet=_Windowed(co, keep), control_cond=x["pose"], control_scale=0.8)
    out = pc(prompt=None, null_prompt=None, negative_prompt=None, ref_image=None, width=W * 8, height=H * 8,
             num_inference_steps=STEPS, guidance_scale=7.0, pose_image=x["pose"], output_type="latent",
             prompt_embeds=x["prompt"], negative_prompt_embeds=x["negative"], latents=x["latents"],
             garment_tokens=x["gtok"], ref_image_latents=x["garment"], controlnet_conditioning_scale=0.8,
             control_guidance_start=start, control_guidance_end=end).images
    err = rel_l2(out, ref)
    print(f"controlnet unipc, window {start}-{end}: final-latent rel-L2 {err:.4f}")
    assert err < 4e-2
    # inpainting: VP blend rows, start latents at strength 1 and below (the sliced schedule restarts the warm-up)
    pin = PInpaint(vae=None, reference_unet=rp, unet=p, tokenizer=None, text_encoder=None, controlnet=cp,
                   image_encoder=None, ImgProj=None, scheduler=_unipc(), safety_checker=None, feature_extractor=None)
    x = inputs(dev, 48)
    g = torch.Generator().manual_seed(49)
    img_lat = torch.randn(1, 4, H, W, generator=g).to(dev)
    mask = torch.zeros(1, 1, H, W, device=dev)
    mask[:, :, H // 4: 3 * H // 4, W // 4: 3 * W // 4] = 1.0
    noise = x["latents"]
    for strength in (1.0, 0.6):
        ref = sample_one(o, ro, noise, x["prompt"], x["negative"], x["gtok"], x["garment"], 5.0, STEPS, UniPCOracle(),
                         controlnet=co, control_cond=x["pose"], control_scale=0.5, mask=mask, image_latents=img_lat,
                         noise=noise, strength=strength)
        out = pin(prompt=None, null_prompt=None, negative_prompt=None, ref_image=None, control_image=x["pose"],
                  height=H * 8, width=W * 8, strength=strength, num_inference_steps=STEPS, guidance_scale=5.0,
                  latents=noise, prompt_embeds=x["prompt"], negative_prompt_embeds=x["negative"], output_type="latent",
                  controlnet_conditioning_scale=0.5, garment_tokens=x["gtok"], ref_image_latents=x["garment"],
                  image_latents=img_lat, mask_latents=mask).images
        err = rel_l2(out, ref)
        print(f"inpainting unipc strength {strength}: final-latent rel-L2 {err:.4f}")
        assert err < 4e-2
        keep_px = (mask == 0).expand_as(out)
        assert rel_l2(out[keep_px], img_lat[keep_px]) < 1e-5
