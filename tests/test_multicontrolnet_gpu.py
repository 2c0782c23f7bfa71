"""GPU: several ControlNets in one call.

Kernel: the scale-table epilogue of the wgmma GEMM (imagd_epilogue.scale_table) element by element against fp64
(tests/gemm_fp64_ref.py) in every kernel variant and split count of tests/test_gemm_fp64_gpu.py, and bitwise against the
host-alpha launch with the bias pre-scaled (alpha = s, bias = fp32(b * s)); every combination the table does not
support is rejected.

Pipelines: the MultiControlNetModel path of the engine (per-step scale table, chained zero convs, one step graph per
active set) through the public pipeline classes against the fp32 multi-ControlNet oracle (tests/multicontrolnet_oracle.py),
at the sizes and tolerance of tests/test_pipeline_gpu.py (32 x 32 latents, 4 steps, rel-L2 < 4e-2)."""
import pytest
import torch

import gemm_fp64_ref as R
from conftest import rel_l2
from multicontrolnet_oracle import MultiControlNetOracle, keep_window
from test_gemm_fp64_gpu import GK, GM, GN, SPLITS, VARIANTS, _gemm_inputs, _vid, check_cfg, forced, launch
from test_pipeline_gpu import STEPS, H, W, build, inputs

pytestmark = pytest.mark.gpu
BF = torch.bfloat16


# ============================================================================================== kernel
def _table(dev):
    """[S = 4, K = 3] scale table and a step counter pointing at row 2 (the sampler's int32[2] step_ptr layout)."""
    t = torch.tensor([[0.3, -1.25, 2.0], [0.75, 1.5, -0.5], [1.1, 0.6125, 0.9], [-0.2, 2.5, 0.05]], device=dev)
    return t, torch.tensor([2, 0], dtype=torch.int32, device=dev)


@pytest.mark.parametrize("mode", ["residual_step2", "plain_step2", "residual_row0"])
@pytest.mark.parametrize("splits", SPLITS, ids=lambda s: f"splits{s}")
@pytest.mark.parametrize("variant", VARIANTS, ids=_vid)
def test_table_epilogue(cuda_device, variant, splits, mode):
    from imagdressing_b200 import ops

    a, w, bias, _, res = _gemm_inputs(cuda_device)
    table, step = _table(cuda_device)
    row = 2 if mode.endswith("step2") else 0
    s = float(table[row, 1])
    residual = res if mode.startswith("residual") else None
    with forced(*variant, splits):
        out, cfg, line = launch(lambda: ops.gemm(a, w, out=R.sentinel_buffer((GM, GN), BF, cuda_device), bias=bias,
                                                 residual=residual, scale_table=table[:, 1],
                                                 scale_step=step if row else None))
        legacy = ops.gemm(a, w, bias=bias * s, alpha=s, residual=residual)
    check_cfg(cfg, variant, splits, -(-GK // 64))
    ref = R.gemm(a, w, alpha=s, bias=bias.double() * s, residual=residual)
    R.check(f"table {_vid(variant)} splits {splits} {mode}", out, ref, bn=variant[0], cfg=line, family="table")
    assert torch.equal(out, legacy), "the table launch must be bitwise the host-alpha launch with a pre-scaled bias"


def test_table_follows_the_step_counter(cuda_device):
    """One launch per step row: the scale read is the row the device counter points at."""
    from imagdressing_b200 import ops

    a, w, bias, _, res = _gemm_inputs(cuda_device)
    table, step = _table(cuda_device)
    for row in range(4):
        step[0] = row
        s = float(table[row, 2])
        got = ops.gemm(a, w, bias=bias, residual=res, scale_table=table[:, 2], scale_step=step)
        assert torch.equal(got, ops.gemm(a, w, bias=bias * s, alpha=s, residual=res)), row


def test_table_rejections(cuda_device):
    import ctypes

    from imagdressing_b200 import _lib, ops

    dev = cuda_device
    a, w, bias, rowvec, _ = _gemm_inputs(dev)
    table, step = _table(dev)
    tab = dict(scale_table=table[:, 0], scale_step=step)
    msg = "a scale table needs a plain bf16 epilogue"
    wg = torch.randn(256, GK, device=dev).to(BF)
    for kw in (dict(act=ops.ACT_GEGLU), dict(act=ops.ACT_SILU), dict(act=ops.ACT_GELU), dict(act=ops.ACT_QUICK_GELU),
               dict(rowvec=rowvec, rows_per_group=77), dict(out_fp32=True),
               dict(stats_out=torch.zeros(GM, 16, 2, device=dev))):
        with pytest.raises(_lib.ImagdError, match=msg):
            ops.gemm(a, wg if kw.get("act") == ops.ACT_GEGLU else w, bias=bias, **kw, **tab)
    # the wrapper checks what the kernel cannot see: the table's dtype and rank, the step counter's dtype
    for bad in (dict(scale_table=table[:, 0].to(BF)), dict(scale_table=table),
                dict(scale_table=table[:, 0], scale_step=step.long())):
        with pytest.raises(ValueError, match="must be"):
            ops.gemm(a, w, bias=bias, **bad)
    ln = ops.LnFold(torch.zeros(GM, 1, 2, device=dev), 1, GK, 1e-5, torch.zeros(GN, device=dev))
    with pytest.raises(_lib.ImagdError, match=msg):
        ops.gemm(a, w, bias=bias, ln=ln, **tab)
    # convolutions take no table
    lib = _lib.load()
    x = torch.randn(1, 8, 8, 64, device=dev).to(BF)
    for fn, wt, cout, out_hw in ((lib.imagd_conv3x3_bf16, torch.randn(64, 9 * 64, device=dev).to(BF), 64, 8),
                                 (lib.imagd_upconv3x3_bf16, torch.randn(4 * 64, 4 * 64, device=dev).to(BF), 64, 16)):
        y = torch.empty(1, out_hw, out_hw, cout, device=dev, dtype=BF)
        ep = ops._epilogue(None, None, 0, None, ops.ACT_NONE, 1.0, False)
        ep.scale_table = table.data_ptr()
        ep.scale_ld = 3
        rc = fn(x.data_ptr(), 64, 1, 8, 8, 64, wt.data_ptr(), y.data_ptr(), cout, cout, ctypes.byref(ep), ops._stream())
        with pytest.raises(_lib.ImagdError, match="the scale table is a GEMM epilogue only"):
            _lib.check(rc, "conv")
    torch.cuda.synchronize()


# ============================================================================================== pipelines
@pytest.fixture(scope="module")
def models(cuda_device):
    """(oracle, host) UNets, garment UNets and three ControlNets of different synthetic weights; scheduler."""
    from imagdressing_b200 import modeling
    from oracle import unet as ou

    (o, ro, co), (p, rp, cp), sched = build(cuda_device, controlnet=True)
    nets = [(co, cp)]
    for seed in (3, 4):
        with modeling.skip_default_init():
            co_k, cp_k = ou.ControlNetModel(), modeling.ControlNetModel()
        co_k = modeling.init_synthetic_fast_(co_k.to(cuda_device), seed).eval()
        cp_k.to(cuda_device).load_state_dict(co_k.state_dict())
        nets.append((co_k, cp_k.eval()))
    return (o, ro), (p, rp), nets, sched


def _pose(models, controlnet, scheduler=None):
    from dressing_sd.pipelines.IMAGDressing_v1_pipeline_controlnet import IMAGDressing_v1

    (_, _), (p, rp), _, sched = models
    return IMAGDressing_v1(vae=None, reference_unet=rp, unet=p, tokenizer=None, text_encoder=None, controlnet=controlnet,
                           image_encoder=None, ImgProj=None, scheduler=scheduler or sched, safety_checker=None,
                           feature_extractor=None)


def _inpaint(models, controlnet):
    from dressing_sd.pipelines.IMAGDressing_v1_pipeline_controlnet_inpainting import IMAGDressing_v1

    (_, _), (p, rp), _, sched = models
    return IMAGDressing_v1(vae=None, reference_unet=rp, unet=p, tokenizer=None, text_encoder=None, controlnet=controlnet,
                           image_encoder=None, ImgProj=None, scheduler=sched, safety_checker=None, feature_extractor=None)


def _common(x, **kw):
    return dict(prompt=None, null_prompt=None, negative_prompt=None, ref_image=None, width=W * 8, height=H * 8,
                num_inference_steps=STEPS, output_type="latent", prompt_embeds=x["prompt"],
                negative_prompt_embeds=x["negative"], latents=x["latents"], garment_tokens=x["gtok"],
                ref_image_latents=x["garment"], **kw)


def _poses(dev, n, seed, batch=1):
    g = torch.Generator().manual_seed(seed)
    return [torch.rand(batch, 3, H * 8, W * 8, generator=g).to(dev) for _ in range(n)]


def _mask_inputs(dev):
    g = torch.Generator().manual_seed(49)
    img_lat = torch.randn(1, 4, H, W, generator=g).to(dev)
    mask = torch.zeros(1, 1, H, W, device=dev)
    mask[:, :, H // 4: 3 * H // 4, W // 4: 3 * W // 4] = 1.0
    return img_lat, mask


@torch.no_grad()
def test_inpainting_two_nets_vs_oracle(cuda_device, models):
    from oracle.pipeline import sample_one

    (o, ro), _, nets, _ = models
    (co, cp), (co2, cp2) = nets[0], nets[1]
    x = inputs(cuda_device, 48)
    ims = _poses(cuda_device, 2, 50)
    img_lat, mask = _mask_inputs(cuda_device)
    kw = dict(strength=1.0, guidance_scale=5.0, height=H * 8, width=W * 8, image_latents=img_lat, mask_latents=mask)
    common = {k: v for k, v in _common(x).items() if k not in ("width", "height")}
    ref = sample_one(o, ro, x["latents"], x["prompt"], x["negative"], x["gtok"], x["garment"], 5.0, STEPS,
                     controlnet=MultiControlNetOracle([co, co2], [0.5, 0.8]), control_cond=ims, control_scale=1.0,
                     mask=mask, image_latents=img_lat, noise=x["latents"])
    out = _inpaint(models, [cp, cp2])(control_image=ims, controlnet_conditioning_scale=[0.5, 0.8], **kw, **common).images
    err = rel_l2(out, ref)
    print(f"inpainting, two ControlNets: final-latent rel-L2 {err:.4f}")
    assert err < 4e-2
    # both nets count: the pair differs from either net alone
    for net, im, s in ((cp, ims[0], 0.5), (cp2, ims[1], 0.8)):
        one = _inpaint(models, net)(control_image=im, controlnet_conditioning_scale=s, **kw, **common).images
        assert rel_l2(out, one) > 5e-2


@torch.no_grad()
def test_pose_windows_graphs_eager_and_scale_change(cuda_device, models):
    from oracle.pipeline import sample_one

    (o, ro), _, nets, _ = models
    x = inputs(cuda_device, 44)
    ims = _poses(cuda_device, 3, 51)
    starts, ends, scales = [0.0, 0.5, 0.25], [0.5, 1.0, 1.0], [0.8, 0.6, 1.1]
    keeps = [keep_window(STEPS, s, e) for s, e in zip(starts, ends)]
    ref = sample_one(o, ro, x["latents"], x["prompt"], x["negative"], x["gtok"], x["garment"], 7.0, STEPS,
                     controlnet=MultiControlNetOracle([n[0] for n in nets], scales, keeps), control_cond=ims,
                     control_scale=1.0)
    pipe = _pose(models, [n[1] for n in nets])
    kw = dict(guidance_scale=7.0, pose_image=ims, control_guidance_start=starts, control_guidance_end=ends)
    out = pipe(controlnet_conditioning_scale=scales, **kw, **_common(x)).images
    err = rel_l2(out, ref)
    print(f"pose, three windowed ControlNets: final-latent rel-L2 {err:.4f}")
    assert err < 4e-2
    (st,) = pipe._engine._states.values()
    active = {tuple(k for k in range(3) if keeps[k][i]) for i in range(STEPS)}
    assert set(st["graphs"]) == active and len(active) == 3
    # the eager (callback) path runs the same grouping
    seen = []
    eager = pipe(controlnet_conditioning_scale=scales, callback=lambda i, t, lat: seen.append(i), **kw,
                 **_common(x)).images
    assert seen == list(range(STEPS)) and torch.equal(eager, out)
    # a new scale list replays the same graph objects, and equals a fresh pipeline's result at that scale
    graphs = {a: g for a, (g, _) in st["graphs"].items()}
    new = [1.2, 0.3, 0.7]
    out2 = pipe(controlnet_conditioning_scale=new, **kw, **_common(x)).images
    (st2,) = pipe._engine._states.values()
    assert st2 is st and {a: g for a, (g, _) in st["graphs"].items()} == graphs
    fresh = _pose(models, [n[1] for n in nets])(controlnet_conditioning_scale=new, **kw, **_common(x)).images
    assert torch.equal(out2, fresh) and not torch.equal(out2, out)


@torch.no_grad()
def test_one_net_and_zero_scale_match_single_controlnet(cuda_device, models):
    from dressing_sd.pipelines.IMAGDressing_v1_pipeline_ipa_controlnet import IMAGDressing_v1 as PIpa
    from imagdressing_b200.modeling import MultiControlNetModel

    (_, _), (p, rp), nets, sched = models
    (_, a), (_, b) = nets[0], nets[1]
    x = inputs(cuda_device, 45)
    pose, other = _poses(cuda_device, 2, 52)
    single = _pose(models, a)(guidance_scale=7.0, pose_image=pose, controlnet_conditioning_scale=0.8, **_common(x)).images
    one = _pose(models, MultiControlNetModel([a]))(guidance_scale=7.0, pose_image=[pose], controlnet_conditioning_scale=0.8,
                                                   **_common(x)).images
    assert torch.equal(one, single)
    zero = _pose(models, [a, b])(guidance_scale=7.0, pose_image=[pose, other], controlnet_conditioning_scale=[0.8, 0.0],
                                 **_common(x)).images
    assert torch.equal(zero, single)
    # IP-Adapter pipeline with face tokens
    gq = torch.Generator().manual_seed(47)
    face, face_null = torch.randn(1, 4, 768, generator=gq).to(p.device), torch.randn(1, 4, 768, generator=gq).to(p.device)
    outs = []
    for cn, im in ((a, pose), (MultiControlNetModel([a]), [pose])):
        pipe = PIpa(vae=None, reference_unet=rp, unet=p, tokenizer=None, text_encoder=None, controlnet=cn,
                    image_encoder=None, ImgProj=None, ip_ckpt=None, scheduler=sched, safety_checker=None,
                    feature_extractor=None)
        outs.append(pipe(guidance_scale=7.0, pose_image=im, image_scale=0.9, ipa_scale=0.8, face_tokens=face,
                         face_null_tokens=face_null, controlnet_conditioning_scale=0.7, **_common(x)).images)
    assert torch.equal(outs[0], outs[1])
    # inpainting pipeline
    img_lat, mask = _mask_inputs(cuda_device)
    common = {k: v for k, v in _common(x).items() if k not in ("width", "height")}
    kw = dict(strength=1.0, guidance_scale=5.0, height=H * 8, width=W * 8, image_latents=img_lat, mask_latents=mask,
              controlnet_conditioning_scale=0.5)
    ins = [_inpaint(models, cn)(control_image=im, **kw, **common).images
           for cn, im in ((a, pose), (MultiControlNetModel([a]), [pose]))]
    assert torch.equal(ins[0], ins[1])


@torch.no_grad()
def test_unipc_two_windowed_nets_vs_oracle(cuda_device, models):
    """A multistep sampler reads scale-table row i at step i through the same step counter."""
    from oracle.samplers import sample_one
    from test_unipc_gpu import _unipc
    from unipc_oracle import UniPCOracle

    (o, ro), _, nets, _ = models
    x = inputs(cuda_device, 53)
    ims = _poses(cuda_device, 2, 54)
    starts, ends, scales = [0.0, 0.5], [0.5, 1.0], [0.9, 0.7]
    keeps = [keep_window(STEPS, s, e) for s, e in zip(starts, ends)]
    ref = sample_one(o, ro, x["latents"], x["prompt"], x["negative"], x["gtok"], x["garment"], 7.0, STEPS, UniPCOracle(),
                     controlnet=MultiControlNetOracle([nets[0][0], nets[2][0]], scales, keeps), control_cond=ims,
                     control_scale=1.0)
    out = _pose(models, [nets[0][1], nets[2][1]], scheduler=_unipc())(
        guidance_scale=7.0, pose_image=ims, controlnet_conditioning_scale=scales, control_guidance_start=starts,
        control_guidance_end=ends, **_common(x)).images
    err = rel_l2(out, ref)
    print(f"UniPC bh2, two windowed ControlNets: final-latent rel-L2 {err:.4f}")
    assert err < 4e-2


@torch.no_grad()
def test_batch_two_per_sample_and_broadcast_images(cuda_device, models):
    from oracle.pipeline import sample_one

    (o, ro), _, nets, _ = models
    xs = [inputs(cuda_device, 55), inputs(cuda_device, 56)]
    per_sample = _poses(cuda_device, 1, 57, batch=2)[0]
    shared = _poses(cuda_device, 1, 58)[0]
    xb = {k: torch.cat([xs[0][k], xs[1][k]]) for k in ("latents", "garment", "prompt", "negative", "gtok")}
    out = _pose(models, [nets[0][1], nets[1][1]])(guidance_scale=7.0, pose_image=[per_sample, shared],
                                                  controlnet_conditioning_scale=[0.8, 0.6], **_common(xb)).images
    for i, x in enumerate(xs):
        ref = sample_one(o, ro, x["latents"], x["prompt"], x["negative"], x["gtok"], x["garment"], 7.0, STEPS,
                         controlnet=MultiControlNetOracle([nets[0][0], nets[1][0]], [0.8, 0.6]),
                         control_cond=[per_sample[i:i + 1], shared], control_scale=1.0)
        err = rel_l2(out[i:i + 1], ref)
        print(f"batch 2, sample {i}: final-latent rel-L2 {err:.4f}")
        assert err < 4e-2
