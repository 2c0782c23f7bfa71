"""CPU: UniPCMultistepScheduler (imagdressing_b200/samplers.py) with the predictor-corrector kernel emulated in torch.

- identities that hold without diffusers: UniPC order 1 without a corrector is DPM-Solver++ order 1 (and DDIM on the
  trailing grid); bh2 order 2 without a corrector is DPM-Solver++ 2M; the schedules are DPM-Solver's;
- convergence order on the Gaussian toy of test_samplers_cpu.py: the corrector raises the order by one;
- product host step() sequences vs the diffusers-style oracle (unipc_oracle.py) for bh1 / bh2, orders 1-3, every
  spacing, Karras on / off, 6 and 20 steps, disable_corrector and a sliced schedule;
- every slot a row reads was written by an earlier row of the same sequence (unwritten slots may hold NaN);
- surface, refusals, compat imports;
- the base and inpainting pipelines under emulated kernels vs oracle.samplers.sample_one with the oracle."""
import math

import pytest
import torch

import emulated_ops
from oracle.samplers import sample_one
from test_samplers_cpu import _cfg_sampler_step, _ddim, _gaussian_error, _nchw_scaled, _product, _run, rel
from unipc_oracle import UniPCOracle

SPACINGS = ("leading", "linspace", "trailing")


def _cfg_sampler_pc_step(eps_cond, eps_uncond, guidance, latents, coef, step_ptr, bank, *, mask=None,
                         image_latents=None, noise=None, blend_coef=None):
    i = int(step_ptr[0])
    r = [float(v) for v in coef[i]]
    dx, de, ax, am, a, bc, bm, b = r[0], r[1], r[2], r[3], r[4:8], r[8], r[9], r[10:14]
    eps = eps_cond if eps_uncond is None else eps_uncond + guidance * (eps_cond - eps_uncond)
    m = dx * latents + de * eps
    c = ax * latents + am * m
    new = bm * m
    for k in range(4):
        if a[k] != 0 or b[k] != 0:
            c = c + a[k] * bank[k]
            new = new + b[k] * bank[k]
    new = new + bc * c
    bank[int(r[14])].copy_(m)
    bank[int(r[15])].copy_(c)
    if mask is not None:
        bl = blend_coef[i]
        new = (1 - mask) * (bl[0] * image_latents + bl[1] * noise) + mask * new
    latents.copy_(new)
    step_ptr[0] += 1
    return latents


@pytest.fixture
def emu(monkeypatch):
    emulated_ops.install(monkeypatch)
    from imagdressing_b200 import modeling, ops

    monkeypatch.setattr(ops, "cfg_sampler_step", _cfg_sampler_step)
    monkeypatch.setattr(ops, "cfg_sampler_pc_step", _cfg_sampler_pc_step)
    monkeypatch.setattr(ops, "nchw_f32_to_nhwc_bf16_scaled", _nchw_scaled)
    return modeling


def _unipc(**kw):
    from imagdressing_b200.samplers import UniPCMultistepScheduler

    return UniPCMultistepScheduler.from_config(_ddim().config, **kw)


# ---------------------------------------------------------------------------------------------------- identities
def test_order1_without_corrector_is_dpm_order1_and_ddim(emu):
    n = 20
    u = _unipc(solver_order=1, disable_corrector=list(range(n)), timestep_spacing="trailing")
    p = _product("dpm", solver_order=1, timestep_spacing="trailing")
    d = _ddim(timestep_spacing="trailing")
    for s in (u, p, d):
        s.set_timesteps(n)
    assert torch.equal(u.timesteps, p.timesteps) and torch.equal(u.timesteps, d.timesteps)
    x = torch.randn(2, 4, 8, 8, generator=torch.Generator().manual_seed(0))
    for a, b, c in zip(_run(u, x, n), _run(p, x, n), _run(d, x, n)):
        assert rel(a, b) < 2e-5 and rel(a, c) < 2e-5


@pytest.mark.parametrize("n", [6, 12])
@pytest.mark.parametrize("spacing", SPACINGS)
def test_bh2_order2_without_corrector_is_dpm_2m(emu, spacing, n):
    """The bh2 order-2 predictor is the midpoint 2M update; at n < 15 both take a first-order last step."""
    u = _unipc(solver_type="bh2", solver_order=2, disable_corrector=list(range(n)), timestep_spacing=spacing)
    p = _product("dpm", timestep_spacing=spacing)
    u.set_timesteps(n)
    p.set_timesteps(n)
    x = torch.randn(1, 4, 8, 8, generator=torch.Generator().manual_seed(1))
    for a, b in zip(_run(u, x, n), _run(p, x, n)):
        assert rel(a, b) < 2e-5


@pytest.mark.parametrize("karras", [False, True])
@pytest.mark.parametrize("spacing", SPACINGS)
def test_schedule_is_dpm_solvers(spacing, karras):
    for n in (6, 10, 20, 25, 50):
        u, p = _unipc(timestep_spacing=spacing, use_karras_sigmas=karras), _product("dpm", timestep_spacing=spacing,
                                                                                    use_karras_sigmas=karras)
        try:
            p.set_timesteps(n)
        except NotImplementedError:  # both refuse a Karras schedule that loses rows to duplicate timesteps
            with pytest.raises(NotImplementedError):
                u.set_timesteps(n)
            continue
        u.set_timesteps(n)
        assert torch.equal(u.timesteps, p.timesteps) and torch.equal(u.sigmas, p.sigmas)
        tu, tp = u.sampler_tables("cpu"), p.sampler_tables("cpu")
        assert torch.equal(tu.t, tp.t) and torch.equal(tu.blend, tp.blend) and tu.scale is None


# ---------------------------------------------------------------------------------------------------- convergence order
@pytest.mark.parametrize("order,lo,hi", [(1, 3.5, 4.8), (2, 7.0, 10.0)])
def test_corrector_raises_the_order_on_gaussian(emu, order, lo, hi):
    """Error ratio 16 -> 32 steps with Karras sigmas: UniC adds one order to UniP, so about 4 for UniPC-1 and about 8
    for UniPC-2 (bh2). At 16 steps UniPC-2 beats DPM-Solver++ 2M."""
    errs = [_gaussian_error(_unipc(solver_order=order, use_karras_sigmas=True), n) for n in (16, 32)]
    ratio = errs[0] / errs[1]
    dpm16 = _gaussian_error(_product("dpm", use_karras_sigmas=True), 16)
    print(f"UniPC-{order}: error {errs[0]:.3e} -> {errs[1]:.3e}, ratio {ratio:.2f}; DPM++2M at 16: {dpm16:.3e}")
    assert lo < ratio < hi
    if order == 2:
        assert errs[0] < dpm16


# ---------------------------------------------------------------------------------------------------- product vs oracle
CASES = [(bh, order, sp, karras, n) for bh in ("bh1", "bh2") for order in (1, 2, 3) for sp in SPACINGS
         for karras in (False, True) for n in (6, 20)]


@pytest.mark.parametrize("bh,order,spacing,karras,n", CASES)
def test_host_step_matches_oracle(emu, bh, order, spacing, karras, n):
    kw = dict(solver_type=bh, solver_order=order, timestep_spacing=spacing, use_karras_sigmas=karras)
    p, o = _unipc(**kw), UniPCOracle(**kw)
    p.set_timesteps(n)
    o.set_timesteps(n)
    assert p.timesteps.tolist() == o.timesteps.tolist() and torch.equal(p.sigmas, o.sigmas)
    x = torch.randn(1, 4, 8, 8, generator=torch.Generator().manual_seed(2))
    for a, b in zip(_run(p, x, n), _run(o, x, n)):
        assert rel(a, b) < 5e-5


@pytest.mark.parametrize("bh,order", [("bh1", 3), ("bh2", 2), ("bh2", 3)])
def test_disable_corrector_and_lower_order_final_off_match_oracle(emu, bh, order):
    kw = dict(solver_type=bh, solver_order=order, disable_corrector=[0, 3, 4, 9], lower_order_final=False)
    p, o = _unipc(**kw), UniPCOracle(**kw)
    p.set_timesteps(12)
    o.set_timesteps(12)
    x = torch.randn(1, 4, 8, 8, generator=torch.Generator().manual_seed(3))
    for a, b in zip(_run(p, x, 12), _run(o, x, 12)):
        assert rel(a, b) < 5e-5


@pytest.mark.parametrize("order", [2, 3])
def test_sliced_schedule_restarts_the_warm_up(emu, order):
    """A step sequence that starts at step k (inpainting, strength < 1) is first order without a corrector at its first
    step, so its rows differ from rows k.. of the full table; the run matches the oracle over the same slice."""
    p = _unipc(solver_order=order)
    p.set_timesteps(20)
    k = 8
    full, part = p.sampler_tables("cpu"), p.sampler_tables("cpu", p.timesteps[k:])
    assert part.coef.shape == (20 - k, 16) and part.predictor_corrector
    assert float(part.coef[0, 2]) == 1.0 and float(full.coef[k, 2]) == 0.0  # no corrector at the slice's first step
    assert not torch.equal(part.coef[1], full.coef[k + 1])
    assert torch.equal(part.t, full.t[k:]) and torch.equal(part.blend, full.blend[k:])
    o = UniPCOracle(solver_order=order)
    o.set_timesteps(20)
    x = torch.randn(1, 4, 8, 8, generator=torch.Generator().manual_seed(5))
    a = _run(p, x, 12, timesteps=p.timesteps[k:])[-1]
    b = _run(o, x, 12, timesteps=o.timesteps[k:])[-1]
    assert rel(a, b) < 5e-5


def _slot_reads_follow_writes(coef):
    written = set()
    for j, row in enumerate(coef.tolist()):
        reads = {k for k in range(4) if row[4 + k] != 0.0 or row[10 + k] != 0.0}
        assert reads <= written, f"row {j} reads slots {sorted(reads - written)} before any row wrote them"
        written |= {int(row[14]), int(row[15])}


@pytest.mark.parametrize("order", [1, 2, 3])
def test_rows_read_only_written_slots(order):
    for bh in ("bh1", "bh2"):
        for karras in (False, True):
            for dc in ([], [1, 2, 5]):
                p = _unipc(solver_order=order, solver_type=bh, use_karras_sigmas=karras, disable_corrector=dc)
                for n in (1, 2, 3, 7, 20):
                    p.set_timesteps(n)
                    for k in range(n):
                        tb = p.sampler_tables("cpu", p.timesteps[k:])
                        _slot_reads_follow_writes(tb.coef)
                        assert torch.isfinite(tb.coef).all()


def test_eager_step_ignores_nan_in_unwritten_slots(emu):
    p, o = _unipc(solver_order=3), UniPCOracle(solver_order=3)
    p.set_timesteps(8)
    o.set_timesteps(8)
    x = torch.randn(1, 4, 8, 8, generator=torch.Generator().manual_seed(6))
    p._bank = torch.full((4, *x.shape), float("nan"))
    outs = _run(p, x, 8)
    assert all(torch.isfinite(y).all() for y in outs)
    assert rel(outs[-1], _run(o, x, 8)[-1]) < 5e-5


# ---------------------------------------------------------------------------------------------------- surface
def test_surface_and_refusals():
    from imagdressing_b200.samplers import UniPCMultistepScheduler as U

    for kw in (dict(predict_x0=False), dict(solver_p=object()), dict(thresholding=True),
               dict(prediction_type="v_prediction"), dict(prediction_type="sample"), dict(solver_order=4),
               dict(solver_type="bh3")):
        with pytest.raises(NotImplementedError):
            U(**kw)
    d = U()
    assert (d.config.solver_order, d.config.solver_type, d.config.predict_x0, d.config.lower_order_final,
            d.config.disable_corrector, d.config.timestep_spacing) == (2, "bh2", True, True, [], "linspace")
    assert U(solver_type="midpoint").config.solver_type == "bh2"
    with pytest.raises(NotImplementedError):
        _unipc(use_karras_sigmas=True).set_timesteps(500)  # Karras rows lost to duplicate timesteps
    u = U.from_config(_ddim().config)  # foreign keys (clip_sample, set_alpha_to_one) are dropped
    assert u.config.timestep_spacing == "leading" and u.config.steps_offset == 1 and u.order == 1
    assert u.config.beta_schedule == "scaled_linear" and u.init_noise_sigma == 1.0
    x = torch.randn(1, 4, 4, 4)
    with pytest.raises(ValueError):
        u.step(x, 1, x)  # set_timesteps not called
    u.set_timesteps(15)
    assert u.step_index is None
    assert u.sampler_tables("cpu").coef is u.sampler_tables("cpu").coef  # cached: stable device addresses
    assert u.sampler_tables("cpu").predictor_corrector and not u.sampler_tables("cpu").history
    assert u.scale_model_input(x, u.timesteps[0]) is x
    n = torch.randn_like(x)
    t = u.timesteps[3:4]
    a = float(u.alphas_cumprod[int(t)])
    assert torch.allclose(u.add_noise(x, n, t), math.sqrt(a) * x + math.sqrt(1 - a) * n)


def test_existing_samplers_keep_their_tables():
    """The shared VP schedule leaves DPM-Solver++ on its 6-wide rows and the generic kernel."""
    p = _product("dpm")
    p.set_timesteps(20)
    tb = p.sampler_tables("cpu")
    assert tb.coef.shape == (20, 6) and tb.history and not tb.predictor_corrector


def test_compat_imports():
    import importlib
    import sys

    sys.path.insert(0, "imagdressing_b200/compat")
    try:
        from imagdressing_b200.compat import diffusers as cd
        from imagdressing_b200.compat.diffusers import schedulers as cs
        from imagdressing_b200.samplers import UniPCMultistepScheduler

        importlib.reload(cs)
        assert cs.UniPCMultistepScheduler is cd.UniPCMultistepScheduler is UniPCMultistepScheduler
        s = cs.UniPCMultistepScheduler.from_config(_ddim().config)
        assert s.config.timestep_spacing == "leading" and s.config.steps_offset == 1
        for cls in (cs.PNDMScheduler, cs.LMSDiscreteScheduler):
            with pytest.raises(NotImplementedError, match="UniPCMultistepScheduler"):
                cls()
    finally:
        sys.path.remove("imagdressing_b200/compat")


# ---------------------------------------------------------------------------------------------------- pipelines
@torch.no_grad()
@pytest.mark.parametrize("bh,order", [("bh2", 2), ("bh1", 3)])
def test_base_pipeline_unipc(emu, bh, order):
    from dressing_sd.pipelines.IMAGDressing_v1_pipeline import IMAGDressing_v1
    from test_pipelines_cpu import build, common, eager, inputs, rel as rel_l2

    (o, ro, _), (p, rp, _), sched = build(emu)
    pipe = eager(IMAGDressing_v1(vae=None, reference_unet=rp, unet=p, tokenizer=None, text_encoder=None,
                                 image_encoder=None, ImgProj=None, scheduler=sched, safety_checker=None,
                                 feature_extractor=None))
    pipe.scheduler = _unipc(solver_type=bh, solver_order=order)
    steps = 6
    x = inputs(42)
    ref = sample_one(o, ro, x["latents"], x["prompt"], x["negative"], x["gtok"], x["garment"], 7.5, steps,
                     UniPCOracle(solver_type=bh, solver_order=order))
    kw = common(x)
    kw["num_inference_steps"] = steps
    out = pipe(guidance_scale=7.5, **kw).images
    assert rel_l2(out, ref) < 4e-2


@torch.no_grad()
@pytest.mark.parametrize("strength", [1.0, 0.6])
def test_inpainting_pipeline_unipc(emu, strength):
    """VP blend rows, the start latents (noise at strength 1, add_noise(image_latents, noise, t_start) below) and the
    warm-up restart of the sliced schedule."""
    from dressing_sd.pipelines.IMAGDressing_v1_pipeline_controlnet_inpainting import IMAGDressing_v1 as PInpaint
    from test_pipelines_cpu import H, W, build, common, eager, inputs, rel as rel_l2

    (o, ro, co), (p, rp, cp), _ = build(emu)
    pin = eager(PInpaint(vae=None, reference_unet=rp, unet=p, tokenizer=None, text_encoder=None, controlnet=cp,
                         image_encoder=None, ImgProj=None, scheduler=_unipc(), safety_checker=None,
                         feature_extractor=None))
    x = inputs(44)
    g = torch.Generator().manual_seed(49)
    img = torch.randn(1, 4, H, W, generator=g)
    mask = torch.zeros(1, 1, H, W)
    mask[..., H // 4: 3 * H // 4, W // 4: 3 * W // 4] = 1.0
    steps = 5
    kw = common(x)
    kw["num_inference_steps"] = steps
    out = pin(guidance_scale=5.0, control_image=x["pose"], strength=strength, controlnet_conditioning_scale=0.5,
              image_latents=img, mask_latents=mask, **kw).images
    lat = sample_one(o, ro, x["latents"], x["prompt"], x["negative"], x["gtok"], x["garment"], 5.0, steps,
                     UniPCOracle(), controlnet=co, control_cond=x["pose"], control_scale=0.5, mask=mask,
                     image_latents=img, noise=x["latents"], strength=strength)
    assert rel_l2(out, lat) < 4e-2
    keep = (mask == 0).expand_as(out)
    assert rel_l2(out[keep], img[keep]) < 1e-5
