"""CPU: the multistep samplers (imagdressing_b200/samplers.py) with their two kernels emulated in torch.

- identities that hold without diffusers: DPM-Solver++ order 1 == DDIM (eta 0), Euler == DDIM rescaled by
  sqrt(1 + sigma^2), Euler-ancestral's sigma_up^2 + sigma_down^2 = sigma_{i+1}^2;
- convergence order on a Gaussian toy whose probability-flow solution is closed form;
- product host step() sequences vs the step-by-step oracle (oracle/samplers.py) for every spacing, Karras on / off,
  lower_order_final at 6 and 20 steps, and sliced schedules;
- known-answer timesteps / sigmas / init_noise_sigma derived here from the closed-form alpha-bar;
- the base and inpainting pipelines under emulated ops vs the oracle loop oracle.samplers.sample_one;
- compat imports and X.from_config(ddim.config)."""
import math

import numpy as np
import pytest
import torch

import emulated_ops
from oracle.samplers import DPMSolverOracle, EulerOracle, sample_one

REF = dict(num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear")


def _cfg_sampler_step(eps_cond, eps_uncond, guidance, latents, coef, step_ptr, *, history=None, step_noise=None,
                      mask=None, image_latents=None, noise=None, blend_coef=None):
    i = int(step_ptr[0])
    dx, de, cx, ce, ch, cz = coef[i]
    eps = eps_cond if eps_uncond is None else eps_uncond + guidance * (eps_cond - eps_uncond)
    new = cx * latents + ce * eps
    if history is not None:
        if ch != 0:
            new = new + ch * history
        history.copy_(dx * latents + de * eps)
    if step_noise is not None and cz != 0:
        new = new + cz * step_noise[i]
    if mask is not None:
        b = blend_coef[i]
        new = (1 - mask) * (b[0] * image_latents + b[1] * noise) + mask * new
    latents.copy_(new)
    step_ptr[0] += 1
    return latents


def _nchw_scaled(x, scale_table, step_ptr, *, repeat=1, out=None):
    s = scale_table[int(step_ptr[0]) if step_ptr is not None else 0]
    return emulated_ops.nchw_f32_to_nhwc_bf16(x * s, repeat=repeat, out=out)


@pytest.fixture
def emu(monkeypatch):
    emulated_ops.install(monkeypatch)
    from imagdressing_b200 import modeling, ops

    monkeypatch.setattr(ops, "cfg_sampler_step", _cfg_sampler_step)
    monkeypatch.setattr(ops, "nchw_f32_to_nhwc_bf16_scaled", _nchw_scaled)
    return modeling


def _ddim(**kw):
    from imagdressing_b200.scheduler import DDIMScheduler

    return DDIMScheduler(**{**REF, "clip_sample": False, "set_alpha_to_one": False, "steps_offset": 1, **kw})


def _product(kind, **kw):
    from imagdressing_b200 import samplers

    cls = dict(dpm=samplers.DPMSolverMultistepScheduler, euler=samplers.EulerDiscreteScheduler,
               ea=samplers.EulerAncestralDiscreteScheduler)[kind]
    return cls.from_config(_ddim().config, **kw)


def _eps_fn(x, t):
    """A smooth, state-dependent stand-in for the model."""
    return 0.6 * x + 0.2 * torch.cos(x + float(t) / 300.0)


def _prev(out):
    return out[0] if isinstance(out, tuple) else out.prev_sample


def _run(sch, x, steps, generator=None, timesteps=None):
    """The reference loop: scale_model_input -> model -> step, over `timesteps` (default: the whole schedule)."""
    ts = sch.timesteps if timesteps is None else timesteps
    xs = [x]
    for t in ts:
        eps = _eps_fn(sch.scale_model_input(x, t), t)
        kw = {"generator": generator} if generator is not None else {}
        x = _prev(sch.step(eps, t, x, **kw))
        xs.append(x)
    return xs


def rel(a, b):
    return float((a - b).norm() / b.norm())


# ---------------------------------------------------------------------------------------------------- identities
def test_dpm_order1_equals_ddim(emu):
    """First-order DPM-Solver++ is DDIM (eta = 0) on the same timesteps: with trailing spacing and 20 | 1000 both walk
    999, 949, ..., 49 and end at alphas_cumprod[0]."""
    d, p = _ddim(timestep_spacing="trailing"), _product("dpm", solver_order=1, timestep_spacing="trailing")
    d.set_timesteps(20)
    p.set_timesteps(20)
    assert torch.equal(d.timesteps, p.timesteps)
    x = torch.randn(2, 4, 8, 8, generator=torch.Generator().manual_seed(0))
    for a, b in zip(_run(d, x, 20), _run(p, x, 20)):
        assert rel(b, a) < 2e-5


def test_euler_equals_rescaled_ddim(emu):
    """Euler on DDIM's timestep grid (trailing, final alpha-bar 1) is DDIM in sigma space: x_euler = x_ddim sqrt(1+sigma^2)."""
    d, e = _ddim(timestep_spacing="trailing", set_alpha_to_one=True), _product("euler", timestep_spacing="trailing")
    d.set_timesteps(25)
    e.set_timesteps(25)
    assert d.timesteps.tolist() == e.timesteps.tolist()
    x = torch.randn(2, 4, 8, 8, generator=torch.Generator().manual_seed(1))
    xd = _run(d, x, 25)
    xe = _run(e, x * math.sqrt(1 + float(e.sigmas[0]) ** 2), 25)
    for i, (a, b) in enumerate(zip(xd, xe)):
        assert rel(b, a * math.sqrt(1 + float(e.sigmas[i]) ** 2)) < 2e-5


def test_euler_ancestral_noise_split():
    ea = _product("ea")
    ea.set_timesteps(30)
    s = ea.sigmas.double()
    for i in range(30):
        up, down = ea.sigma_up_down(i)
        assert up ** 2 + down ** 2 == pytest.approx(float(s[i + 1]) ** 2, rel=1e-9, abs=1e-12)
    coef = ea.sampler_tables("cpu").coef
    assert float(coef[-1, 5]) == 0.0 and float(coef[-2, 5]) > 0.0  # the last step adds no noise
    assert ea.sampler_tables("cpu").noise and not ea.sampler_tables("cpu").history


# ---------------------------------------------------------------------------------------------------- convergence order
def _gaussian_error(sch, steps, mu=0.7, s=1.0):
    """Data N(mu, s^2): in sigma space x~ = x / sqrt(abar) the marginal is N(mu, s^2 + sigma^2), eps is exact and the
    probability-flow ODE keeps (x~ - mu) / sqrt(s^2 + sigma^2) constant. Returns the final-state relative error."""
    from imagdressing_b200.scheduler import DDIMScheduler

    sch.set_timesteps(steps)
    ac = sch.alphas_cumprod.double()

    def sigma_at(i):  # the sigma of step i (i = steps: the final one)
        if isinstance(sch, DDIMScheduler):
            t = int(sch.timesteps[i]) if i < steps else -1
            a = float(ac[t]) if t >= 0 else float(sch.final_alpha_cumprod)
            return math.sqrt((1 - a) / a)
        return float(sch.sigmas[i])

    vp = "Euler" not in type(sch).__name__  # DDIM / DPM carry VP latents; Euler carries sigma-space latents
    z = torch.randn(4096, generator=torch.Generator().manual_seed(3), dtype=torch.float64).float()
    s0 = sigma_at(0)
    xt = mu + z * math.sqrt(s ** 2 + s0 ** 2)
    x = xt / math.sqrt(1 + s0 ** 2) if vp else xt
    for i, t in enumerate(sch.timesteps):
        sg = sigma_at(i)
        xin = x if vp else x / math.sqrt(1 + sg ** 2)  # VP latents
        a = 1 / (1 + sg ** 2)
        eps = math.sqrt(1 - a) * (xin - math.sqrt(a) * mu) / (a * s ** 2 + 1 - a)
        x = _prev(sch.step(eps, t, x))
    se = sigma_at(steps)
    exact = mu + z * math.sqrt(s ** 2 + se ** 2)
    if vp:
        exact = exact / math.sqrt(1 + se ** 2)
    return rel(x, exact)


@pytest.mark.parametrize("kind,lo,hi", [("dpm", 3.5, 6.0), ("ddim", 1.6, 2.4), ("euler", 1.6, 2.4)])
def test_convergence_order_on_gaussian(emu, kind, lo, hi):
    """Error ratio when the step count doubles (16 -> 32): about 4 for DPM-Solver++ 2M, about 2 for DDIM and Euler.
    Karras sigmas keep the step sizes in lambda balanced (uniform spacing in t ends with one large step in lambda, far
    from the asymptotic regime); DDIM has no Karras option and walks the trailing grid."""
    errs = []
    for n in (16, 32):
        sch = _ddim(timestep_spacing="trailing") if kind == "ddim" else _product(kind, use_karras_sigmas=True)
        errs.append(_gaussian_error(sch, n))
    ratio = errs[0] / errs[1]
    print(f"{kind}: error {errs[0]:.3e} -> {errs[1]:.3e}, ratio {ratio:.2f}")
    assert lo < ratio < hi


# ---------------------------------------------------------------------------------------------------- product vs oracle
CASES = [(kind, sp, karras, n) for kind in ("dpm", "euler", "ea") for sp in ("leading", "linspace", "trailing")
         for karras in (False, True) for n in (6, 20) if not (karras and kind == "ea")]


@pytest.mark.parametrize("kind,spacing,karras,n", CASES)
def test_host_step_matches_oracle(emu, kind, spacing, karras, n):
    kw = dict(timestep_spacing=spacing)
    okw = dict(timestep_spacing=spacing, use_karras_sigmas=karras)
    if karras:
        kw["use_karras_sigmas"] = True
    p = _product(kind, **kw)
    if kind == "dpm":
        o = DPMSolverOracle(**okw)
    else:
        o = EulerOracle(ancestral=kind == "ea", generator=torch.Generator().manual_seed(9), **okw)
    p.set_timesteps(n)
    o.set_timesteps(n)
    assert p.timesteps.tolist() == o.timesteps.tolist()
    assert torch.equal(p.sigmas, o.sigmas)
    assert p.init_noise_sigma == pytest.approx(o.init_noise_sigma, rel=1e-6)
    x = torch.randn(1, 4, 8, 8, generator=torch.Generator().manual_seed(2)) * p.init_noise_sigma
    g = torch.Generator().manual_seed(9) if kind == "ea" else None
    for a, b in zip(_run(p, x, n, generator=g), _run(o, x, n)):
        assert rel(a, b) < 5e-5


@pytest.mark.parametrize("kind", ["dpm", "euler", "ea"])
def test_sliced_schedule_rows_are_full_schedule_rows(emu, kind):
    """Inpainting with strength < 1 samples timesteps[k:]: the table rows are rows k.. of the full schedule, and the
    first sliced DPM step is first order (lower_order_nums restarts at 0)."""
    p = _product(kind)
    p.set_timesteps(20)
    k = 8
    full, part = p.sampler_tables("cpu"), p.sampler_tables("cpu", p.timesteps[k:])
    if kind == "dpm":
        assert float(part.coef[0, 4]) == 0.0 and float(full.coef[k, 4]) != 0.0
        assert torch.equal(part.coef[1:], full.coef[k + 1:])
    else:
        assert torch.equal(part.coef, full.coef[k:])
        assert torch.equal(part.scale, full.scale[k:])
    assert torch.equal(part.t, full.t[k:]) and torch.equal(part.blend, full.blend[k:])
    with pytest.raises(ValueError):
        p.sampler_tables("cpu", p.timesteps[2:5])  # not a suffix
    o = DPMSolverOracle() if kind == "dpm" else EulerOracle(ancestral=kind == "ea", generator=torch.Generator().manual_seed(4))
    o.set_timesteps(20)
    x = torch.randn(1, 4, 8, 8, generator=torch.Generator().manual_seed(5))
    g = torch.Generator().manual_seed(4) if kind == "ea" else None
    a = _run(p, x, 12, generator=g, timesteps=p.timesteps[k:])[-1]
    b = _run(o, x, 12, timesteps=o.timesteps[k:])[-1]
    assert rel(a, b) < 5e-5


def test_dpm_lower_order_final_rule():
    for n, first_order_last in ((6, True), (14, True), (15, False), (20, False)):
        p = _product("dpm")
        p.set_timesteps(n)
        coef = p.sampler_tables("cpu").coef
        assert float(coef[0, 4]) == 0.0 and float(coef[1, 4]) != 0.0
        assert (float(coef[-1, 4]) == 0.0) == first_order_last


# ---------------------------------------------------------------------------------------------------- known answers
def _abar():
    b = np.linspace(0.00085 ** 0.5, 0.012 ** 0.5, 1000, dtype=np.float64) ** 2
    return np.cumprod(1 - b)


@pytest.mark.parametrize("n", [20, 25])
def test_known_answer_schedules(n):
    ab = _abar()
    sig = np.sqrt((1 - ab) / ab)
    # DPM-Solver++ leading (from a DDIM config, steps_offset 1): n + 1 points spaced by 1000 // (n + 1), top one dropped
    p = _product("dpm")
    p.set_timesteps(n)
    r = 1000 // (n + 1)
    assert p.timesteps.tolist() == [r * k + 1 for k in range(n, 0, -1)]
    assert np.allclose(p.sigmas[:-1].double().numpy(), sig[p.timesteps.numpy()], rtol=1e-5)
    assert float(p.sigmas[-1]) == pytest.approx(sig[0], rel=1e-4)  # final sigma: sigma at t = 0, not 0 (fp32 1 - abar)
    assert p.init_noise_sigma == 1.0
    # Euler leading: 1000 // n spacing, float timesteps, init_noise_sigma = sqrt(sigma_max^2 + 1)
    e = _product("euler")
    e.set_timesteps(n)
    r = 1000 // n
    assert e.timesteps.dtype == torch.float32 and e.timesteps.tolist() == [float(r * k + 1) for k in range(n - 1, -1, -1)]
    assert float(e.sigmas[-1]) == 0.0
    assert e.init_noise_sigma == pytest.approx(math.sqrt(sig[r * (n - 1) + 1] ** 2 + 1), rel=1e-5)
    # Euler linspace: fractional timesteps linspace(0, 999, n), sigma interpolated, init_noise_sigma = sigma_max
    e = _product("euler", timestep_spacing="linspace")
    e.set_timesteps(n)
    ts = np.linspace(0, 999, n)[::-1]
    assert np.allclose(e.timesteps.double().numpy(), ts, rtol=1e-6)
    assert any(abs(t - round(t)) > 1e-3 for t in ts)
    assert np.allclose(e.sigmas[:-1].double().numpy(), np.interp(ts, np.arange(1000), sig), rtol=1e-4)
    assert e.init_noise_sigma == pytest.approx(sig[999], rel=1e-5)
    tb = e.sampler_tables("cpu")
    assert np.allclose(tb.scale.double().numpy(), 1 / np.sqrt(e.sigmas[:-1].double().numpy() ** 2 + 1), rtol=1e-6)
    assert tb.blend[:-1, 1].tolist() == e.sigmas[1:-1].tolist() and tb.blend[-1].tolist() == [1.0, 0.0]


def test_surface_and_refusals():
    from imagdressing_b200 import samplers

    for kw in (dict(solver_order=3), dict(algorithm_type="sde-dpmsolver++"), dict(algorithm_type="dpmsolver"),
               dict(prediction_type="v_prediction"), dict(thresholding=True)):
        with pytest.raises(NotImplementedError):
            samplers.DPMSolverMultistepScheduler(**kw)
    e = _product("euler")
    e.set_timesteps(10)
    x = torch.randn(1, 4, 4, 4)
    with pytest.raises(NotImplementedError):
        e.step(x, e.timesteps[0], x, s_churn=1.0)
    with pytest.raises(NotImplementedError):
        samplers.EulerAncestralDiscreteScheduler(prediction_type="v_prediction")
    p = _product("dpm")
    with pytest.raises(ValueError):
        p.step(x, 1, x)  # set_timesteps not called
    assert p.config.timestep_spacing == "leading" and p.config.steps_offset == 1 and p.order == 1
    p.set_timesteps(20)
    assert p.sampler_tables("cpu").coef is p.sampler_tables("cpu").coef  # cached: stable device addresses
    # add_noise: VP for DPM-Solver, x + sigma noise for Euler (sigma looked up by the timestep's position)
    n = torch.randn_like(x)
    t = p.timesteps[3:4]
    a = float(p.alphas_cumprod[int(t)])
    assert torch.allclose(p.add_noise(x, n, t), math.sqrt(a) * x + math.sqrt(1 - a) * n)
    assert torch.allclose(e.add_noise(x, n, e.timesteps[2:3]), x + float(e.sigmas[2]) * n)


def test_compat_imports_and_from_config():
    import importlib
    import sys

    sys.path.insert(0, "imagdressing_b200/compat")
    try:
        from imagdressing_b200.compat.diffusers import schedulers as cs
        from imagdressing_b200.compat import diffusers as cd

        importlib.reload(cs)
        for name in ("DPMSolverMultistepScheduler", "EulerDiscreteScheduler", "EulerAncestralDiscreteScheduler"):
            assert getattr(cs, name) is getattr(cd, name)
        s = cs.DPMSolverMultistepScheduler.from_config(_ddim().config)
        assert s.config.timestep_spacing == "leading" and s.config.steps_offset == 1
        assert cs.EulerDiscreteScheduler.from_config(_ddim().config).config.beta_schedule == "scaled_linear"
        for cls in (cs.PNDMScheduler, cs.LMSDiscreteScheduler):
            with pytest.raises(NotImplementedError, match="DPMSolverMultistepScheduler"):
                cls()
    finally:
        sys.path.remove("imagdressing_b200/compat")


# ---------------------------------------------------------------------------------------------------- pipelines
@torch.no_grad()
@pytest.mark.parametrize("kind", ["dpm", "euler", "ea"])
def test_base_pipeline_each_sampler(emu, kind):
    from dressing_sd.pipelines.IMAGDressing_v1_pipeline import IMAGDressing_v1
    from test_pipelines_cpu import build, common, eager, inputs, rel as rel_l2

    (o, ro, _), (p, rp, _), sched = build(emu)
    pipe = eager(IMAGDressing_v1(vae=None, reference_unet=rp, unet=p, tokenizer=None, text_encoder=None,
                                 image_encoder=None, ImgProj=None, scheduler=sched, safety_checker=None,
                                 feature_extractor=None))
    pipe.scheduler = _product(kind)
    steps = 6
    x = inputs(42)
    osch = DPMSolverOracle() if kind == "dpm" else EulerOracle(ancestral=kind == "ea",
                                                               generator=torch.Generator().manual_seed(7))
    ref = sample_one(o, ro, x["latents"], x["prompt"], x["negative"], x["gtok"], x["garment"], 7.5, steps, osch)
    kw = common(x)
    kw["num_inference_steps"] = steps
    out = pipe(guidance_scale=7.5, generator=torch.Generator().manual_seed(7), **kw).images
    assert rel_l2(out, ref) < 4e-2


@torch.no_grad()
@pytest.mark.parametrize("strength", [1.0, 0.6])
def test_inpainting_pipeline_euler(emu, strength):
    """sigma-space blend rows (1, sigma_{i+1}), the scaled ControlNet input, and the start latents: noise *
    init_noise_sigma at strength 1, add_noise(image_latents, noise, t_start) below."""
    from dressing_sd.pipelines.IMAGDressing_v1_pipeline_controlnet_inpainting import IMAGDressing_v1 as PInpaint
    from test_pipelines_cpu import H, W, build, common, eager, inputs, rel as rel_l2

    (o, ro, co), (p, rp, cp), sched = build(emu)
    pin = eager(PInpaint(vae=None, reference_unet=rp, unet=p, tokenizer=None, text_encoder=None, controlnet=cp,
                         image_encoder=None, ImgProj=None, scheduler=_product("euler"), safety_checker=None,
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
    lat = sample_one(o, ro, x["latents"], x["prompt"], x["negative"], x["gtok"], x["garment"], 5.0, steps, EulerOracle(),
                     controlnet=co, control_cond=x["pose"], control_scale=0.5, mask=mask, image_latents=img,
                     noise=x["latents"], strength=strength)
    assert rel_l2(out, lat) < 4e-2
    keep = (mask == 0).expand_as(out)
    assert rel_l2(out[keep], img[keep]) < 1e-5
