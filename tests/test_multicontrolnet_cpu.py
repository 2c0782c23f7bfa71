"""CPU: several ControlNets in one call (modeling.MultiControlNetModel, the engine's per-net state and scale table, the
pipelines' per-net arguments) with the kernel wrappers emulated in torch (tests/emulated_ops.py, plus the table-scaled
zero-conv GEMM below) against the fp32 multi-ControlNet oracle (tests/multicontrolnet_oracle.py). The kernels and the
CUDA-graph path are checked on the GPU by tests/test_multicontrolnet_gpu.py."""
import os
import subprocess
import sys

import pytest
import torch

import emulated_ops
from multicontrolnet_oracle import MultiControlNetOracle, keep_window
from oracle import unet as ou
from oracle.pipeline import sample_one
from test_pipelines_cpu import CFG, H, STEPS, W, build, common, eager, inputs, rel

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def gemm_table(a, w, *, scale_table=None, scale_step=None, bias=None, alpha=1.0, **kw):
    """emulated_ops.gemm plus the scale-table epilogue: s = scale_table[scale_step[0]] replaces alpha and scales the bias
    (fp32 product, as the kernel rounds it)."""
    if scale_table is None:
        return emulated_ops.gemm(a, w, bias=bias, alpha=alpha, **kw)
    s = float(scale_table[int(scale_step[0]) if scale_step is not None else 0])
    return emulated_ops.gemm(a, w, bias=None if bias is None else bias.float() * s, alpha=s, **kw)


@pytest.fixture
def emu(monkeypatch):
    emulated_ops.install(monkeypatch)
    from imagdressing_b200 import modeling, ops

    monkeypatch.setattr(ops, "gemm", gemm_table)
    return modeling


def extra_nets(modeling, seeds):
    """(oracle, host) ControlNet pairs with the same synthetic weights, one per seed."""
    pairs = []
    for seed in seeds:
        co, cp = ou.ControlNetModel(**CFG), modeling.ControlNetModel(**CFG)
        ou.init_synthetic_(co, seed)
        modeling.init_synthetic_(cp, seed)
        pairs.append((co.eval(), cp.eval()))
    return pairs


def pose_pipe(rp, p, controlnet, sched):
    from dressing_sd.pipelines.IMAGDressing_v1_pipeline_controlnet import IMAGDressing_v1 as PControl

    return eager(PControl(vae=None, reference_unet=rp, unet=p, tokenizer=None, text_encoder=None, controlnet=controlnet,
                          image_encoder=None, ImgProj=None, scheduler=sched, safety_checker=None, feature_extractor=None))


def images(n, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.rand(1, 3, H * 8, W * 8, generator=g) for _ in range(n)]


# ---------------------------------------------------------------------------------------------------- construction
def test_list_wrapping_state_dict_and_processors(emu):
    from imagdressing_b200.modeling import MultiControlNetModel

    (_, _, _), (p, rp, cp), sched = build(emu)
    (_, cp2), = extra_nets(emu, [3])
    pipe = pose_pipe(rp, p, [cp, cp2], sched)
    multi = pipe.controlnet
    assert isinstance(multi, MultiControlNetModel) and list(multi.nets) == [cp, cp2]
    assert pipe._engine.controlnet is multi and pipe._engine._nets() == [cp, cp2]
    keys = list(multi.state_dict())
    want = [f"nets.{k}.{n}" for k, net in enumerate((cp, cp2)) for n in net.state_dict()]
    assert keys == want
    procs = multi.attn_processors
    assert len(procs) == len(cp.attn_processors) + len(cp2.attn_processors)
    assert all(n.startswith(("nets.0.", "nets.1.")) for n in procs)
    assert multi.config is cp.config and multi.dtype == cp.dtype
    # a state dict round trip invalidates every net's packed weights
    cp._cn_packed()
    multi.load_state_dict(multi.state_dict())
    assert cp._cn_pk is None and cp2._cn_pk is None
    # a tuple wraps too, in every ControlNet pipeline class
    from dressing_sd.pipelines.IMAGDressing_v1_pipeline_controlnet_inpainting import IMAGDressing_v1 as PInpaint

    pin = PInpaint(vae=None, reference_unet=rp, unet=p, tokenizer=None, text_encoder=None, controlnet=(cp, cp2),
                   image_encoder=None, ImgProj=None, scheduler=sched, safety_checker=None, feature_extractor=None)
    assert isinstance(pin.controlnet, MultiControlNetModel)


def test_constructor_errors(emu):
    from imagdressing_b200.modeling import MultiControlNetModel

    (_, cp), = extra_nets(emu, [3])
    with pytest.raises(ValueError, match="non-empty list"):
        MultiControlNetModel([])
    with pytest.raises(ValueError, match="non-empty list"):
        MultiControlNetModel([cp, torch.nn.Linear(2, 2)])
    with pytest.raises(ValueError, match="may appear once"):
        MultiControlNetModel([cp, cp])


def test_compat_imports():
    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r);"
            "from diffusers.pipelines.controlnet import MultiControlNetModel as A;"
            "from diffusers.pipelines.controlnet.multicontrolnet import MultiControlNetModel as B;"
            "import imagdressing_b200.modeling as m; assert A is B is m.MultiControlNetModel; print('ok')"
            ) % (ROOT, os.path.join(ROOT, "imagdressing_b200", "compat"))
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "ok" in out.stdout, out.stderr[-2000:]


@torch.no_grad()
def test_public_forward_sums_the_nets(emu):
    """MultiControlNetModel.forward (the eager, public path: host scales staged into a [1, K] device table, nets chained)
    against the fp32 sum of the oracle nets' residuals, each at its own scale."""
    from imagdressing_b200.modeling import MultiControlNetModel

    (_, _, co), (_, _, cp), _ = build(emu)
    (co2, cp2), = extra_nets(emu, [3])
    x = inputs(46)
    ims, scales, t = images(2, 11), [0.7, 1.3], torch.tensor([601.0])
    down, mid = MultiControlNetModel([cp, cp2])(x["latents"], t, x["prompt"], ims, scales)
    ref_down, ref_mid = MultiControlNetOracle([co, co2], scales)(x["latents"], t, x["prompt"], ims)
    tok = lambda r: r.permute(0, 2, 3, 1)  # oracle NCHW -> the host's token-major layout
    assert len(down) == len(ref_down) == 12
    for got, ref in zip(down + [mid], ref_down + [ref_mid]):
        assert got.dtype == torch.bfloat16 and got.shape == tok(ref).shape
        assert rel(got, tok(ref)) < 4e-2
    # each net counts: the sum is not either net alone
    alone, _ = MultiControlNetOracle([co], scales[:1])(x["latents"], t, x["prompt"], ims[:1])
    assert rel(down[0], tok(alone[0])) > 5e-2
    with pytest.raises(ValueError, match="1 images and 2 scales for 2 ControlNets"):
        MultiControlNetModel([cp, cp2])(x["latents"], t, x["prompt"], ims[:1], scales)


@pytest.mark.parametrize("table,match", [
    (torch.zeros(4, dtype=torch.float64), "1-D fp32 CUDA tensor"),
    (torch.zeros(4, 2), "1-D fp32 CUDA tensor"),
    (torch.zeros(4), "1-D fp32 CUDA tensor"),
])
def test_gemm_table_argument_errors(table, match):
    """The kernel sees only a pointer, so the wrapper rejects a table of the wrong dtype, rank or device."""
    from imagdressing_b200 import ops

    a, w = torch.zeros(8, 64, dtype=torch.bfloat16), torch.zeros(8, 64, dtype=torch.bfloat16)
    with pytest.raises(ValueError, match=match):
        ops.gemm(a, w, scale_table=table)


# ---------------------------------------------------------------------------------------------------- arguments
def test_argument_normalisation():
    from imagdressing_b200.pipelines import _multi_control_args

    ims = ["a", "b", "c"]
    # scalars broadcast to every net; a float scale too
    assert _multi_control_args(3, False, ims, 0.5, 0.0, 1.0) == (ims, [0.5] * 3, [0.0] * 3, [1.0] * 3)
    # a scalar start follows the end list's length, and the other way round (ipa_controlnet.py:443-454)
    assert _multi_control_args(3, False, ims, [1, 0.5, 0.25], 0.1, [0.5, 0.6, 1.0]) == (
        ims, [1.0, 0.5, 0.25], [0.1] * 3, [0.5, 0.6, 1.0])
    assert _multi_control_args(3, False, tuple(ims), (0.2, 0.3, 0.4), [0.0, 0.5, 0.25], 0.9)[2:] == (
        [0.0, 0.5, 0.25], [0.9] * 3)


@pytest.mark.parametrize("args,match", [
    (("x", 1.0, 0.0, 1.0), "takes a list of 2 control images"),
    ((["x"], 1.0, 0.0, 1.0), "1 control images for 2 ControlNets"),
    ((["x", "y"], [1.0], 0.0, 1.0), "1 controlnet_conditioning_scale for 2"),
    ((["x", "y"], 1.0, [0.0, 0.1, 0.2], 1.0), "3 control_guidance_start for 2"),
    ((["x", "y"], 1.0, [0.0, 0.1], [1.0, 0.9, 0.8]), "2 control_guidance_start for 2|3 control_guidance_end"),
    ((["x", "y"], 1.0, [0.0, 0.6], [1.0, 0.5]), r"window \[0.6, 0.5\]"),
    ((["x", "y"], 1.0, -0.1, 1.0), r"window \[-0.1, 1.0\]"),
])
def test_argument_errors(args, match):
    from imagdressing_b200.pipelines import _multi_control_args

    with pytest.raises(ValueError, match=match):
        _multi_control_args(2, False, *args)


def test_guess_mode_and_pipeline_errors(emu):
    (_, _, _), (p, rp, cp), sched = build(emu)
    (_, cp2), = extra_nets(emu, [3])
    pipe = pose_pipe(rp, p, [cp, cp2], sched)
    x = inputs(44)
    ims = images(2, 7)
    with pytest.raises(NotImplementedError, match="guess_mode"):
        pipe(guidance_scale=7.0, pose_image=ims, guess_mode=True, **common(x))
    with pytest.raises(ValueError, match="1 control images for 2"):
        pipe(guidance_scale=7.0, pose_image=ims[:1], **common(x))
    with pytest.raises(ValueError, match="3 controlnet_conditioning_scale for 2"):
        pipe(guidance_scale=7.0, pose_image=ims, controlnet_conditioning_scale=[1.0, 1.0, 1.0], **common(x))
    # the inpainting size check applies to each image
    from dressing_sd.pipelines.IMAGDressing_v1_pipeline_controlnet_inpainting import IMAGDressing_v1 as PInpaint

    pin = eager(PInpaint(vae=None, reference_unet=rp, unet=p, tokenizer=None, text_encoder=None, controlnet=[cp, cp2],
                         image_encoder=None, ImgProj=None, scheduler=sched, safety_checker=None, feature_extractor=None))
    img, mask = torch.randn(1, 4, H, W), torch.ones(1, 1, H, W)
    small = torch.rand(1, 3, H * 4, W * 4)
    kw = {k: v for k, v in common(x).items() if k not in ("width", "height")}
    with pytest.raises(ValueError, match="does not match the image"):
        pin(guidance_scale=5.0, control_image=[ims[0], small], image_latents=img, mask_latents=mask, **kw)
    # the engine checks the per-net keep lists
    eng = pipe._engine
    with pytest.raises(ValueError, match="one 0/1 entry per step for each ControlNet"):
        eng.sample(x["latents"], x["prompt"], x["negative"], None, 7.0, STEPS, control_cond=ims, control_scale=[1.0, 1.0],
                   control_keep=[[1.0] * STEPS, [1.0] * (STEPS - 1)])
    with pytest.raises(ValueError, match="for 2 ControlNets"):
        eng.sample(x["latents"], x["prompt"], x["negative"], None, 7.0, STEPS, control_cond=ims, control_scale=[1.0])


# ---------------------------------------------------------------------------------------------------- against the oracle
@torch.no_grad()
def test_pose_pipeline_windows_vs_oracle(emu):
    """K = 3 with windows [0, 0.5] / [0.5, 1] / [0.25, 1]: every step has a different active set from its neighbour."""
    (o, ro, co), (p, rp, cp), sched = build(emu)
    (co2, cp2), (co3, cp3) = extra_nets(emu, [3, 4])
    pipe = pose_pipe(rp, p, [cp, cp2, cp3], sched)
    x = inputs(44)
    ims, scales = images(3, 8), [0.8, 0.6, 1.1]
    starts, ends = [0.0, 0.5, 0.25], [0.5, 1.0, 1.0]
    keeps = [keep_window(STEPS, s, e) for s, e in zip(starts, ends)]
    ref = sample_one(o, ro, x["latents"], x["prompt"], x["negative"], x["gtok"], x["garment"], 7.0, STEPS,
                     controlnet=MultiControlNetOracle([co, co2, co3], scales, keeps), control_cond=ims, control_scale=1.0)
    out = pipe(guidance_scale=7.0, pose_image=ims, controlnet_conditioning_scale=scales, control_guidance_start=starts,
               control_guidance_end=ends, **common(x)).images
    assert rel(out, ref) < 4e-2
    # one net, and a second net at scale 0, both reproduce the single-ControlNet pipeline exactly
    single = pose_pipe(rp, p, cp, sched)(guidance_scale=7.0, pose_image=ims[0], controlnet_conditioning_scale=0.8,
                                         **common(x)).images
    from imagdressing_b200.modeling import MultiControlNetModel

    one = pose_pipe(rp, p, MultiControlNetModel([cp]), sched)(
        guidance_scale=7.0, pose_image=ims[:1], controlnet_conditioning_scale=0.8, **common(x)).images
    assert torch.equal(one, single)
    zero = pose_pipe(rp, p, [cp, cp2], sched)(guidance_scale=7.0, pose_image=ims[:2],
                                              controlnet_conditioning_scale=[0.8, 0.0], **common(x)).images
    assert torch.equal(zero, single)


@torch.no_grad()
def test_inpainting_pipeline_two_nets_vs_oracle(emu):
    from dressing_sd.pipelines.IMAGDressing_v1_pipeline_controlnet_inpainting import IMAGDressing_v1 as PInpaint

    (o, ro, co), (p, rp, cp), sched = build(emu)
    (co2, cp2), = extra_nets(emu, [3])
    pin = eager(PInpaint(vae=None, reference_unet=rp, unet=p, tokenizer=None, text_encoder=None, controlnet=[cp, cp2],
                         image_encoder=None, ImgProj=None, scheduler=sched, safety_checker=None, feature_extractor=None))
    x = inputs(45)
    ims = images(2, 9)
    g = torch.Generator().manual_seed(49)
    img = torch.randn(1, 4, H, W, generator=g)
    mask = torch.zeros(1, 1, H, W)
    mask[..., H // 4: 3 * H // 4, W // 4: 3 * W // 4] = 1.0
    for strength in (1.0, 0.5):  # strength < 1: keep over the sliced timesteps
        steps = STEPS if strength == 1.0 else int(STEPS * strength)
        keeps = [keep_window(steps, 0.0, 1.0), keep_window(steps, 0.0, 0.5)]
        from oracle.samplers import sample_one as sample_one_sched

        from oracle.ddim import DDIMOracle

        ref = sample_one_sched(o, ro, x["latents"], x["prompt"], x["negative"], x["gtok"], x["garment"], 5.0, STEPS,
                               DDIMOracle(), controlnet=MultiControlNetOracle([co, co2], [0.5, 0.8], keeps),
                               control_cond=ims, control_scale=1.0, mask=mask, image_latents=img, noise=x["latents"],
                               strength=strength)
        out = pin(guidance_scale=5.0, control_image=ims, strength=strength, controlnet_conditioning_scale=[0.5, 0.8],
                  control_guidance_end=[1.0, 0.5], image_latents=img, mask_latents=mask, **common(x)).images
        assert rel(out, ref) < 4e-2, strength
