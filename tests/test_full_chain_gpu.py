"""GPU parity on the METRIC's own configurations (VERDICT r1 weak #1, SURVEY.md §8c "50-step final latents"):

* BASELINE configs[1]: batch-1 512x512, 50 DDIM steps, CFG 7.5, garment-conditioned, through the public
  `dressing_sd.pipelines.IMAGDressing_v1_pipeline.IMAGDressing_v1` (CUDA-graph replayed engine);
* BASELINE configs[3] shape: 768x576 ControlNet-inpainting chain, batch 2, 50 steps, through
  `...IMAGDressing_v1_pipeline_controlnet_inpainting.IMAGDressing_v1`.

Oracle = `oracle/pipeline.sample_one` in fp32 ON THE GPU (reference-style batch-1 calls, two UNet calls per step).
Calibration, not an assumed tolerance: the SAME oracle is also run with its modules in torch bf16 and torch fp16
(latents kept fp32 between steps, as the product does) and the kernel path must stay within 2x the torch-bf16 drift
(floor 3e-2). rel-L2 and cosine of the final latents of all three are printed and written to
parity_full_chain.json in $IMAGD_PARITY_OUT (default: the system temporary directory).
"""
import json
import os
import tempfile

import pytest
import torch

from conftest import rel_l2
from test_pipeline_gpu import build

pytestmark = pytest.mark.gpu
STEPS = 50


class Cast:
    """Runs an oracle module in `dtype` behind an fp32 interface (tensor args cast in, tensor outputs cast back)."""

    def __init__(self, module, dtype):
        self.m, self.dtype = module, dtype

    @property
    def attn_processors(self):
        return self.m.attn_processors

    def _in(self, v):
        if torch.is_tensor(v):
            return v.to(self.dtype) if v.is_floating_point() else v
        if isinstance(v, dict):
            return {k: self._in(x) for k, x in v.items()}
        if isinstance(v, (list, tuple)):
            return type(v)(self._in(x) for x in v)
        return v

    def _out(self, v):
        if torch.is_tensor(v):
            return v.float()
        if isinstance(v, (list, tuple)):
            return type(v)(self._out(x) for x in v)
        return v

    def __call__(self, *a, **kw):
        return self._out(self.m(*self._in(a), **self._in(kw)))


def cosine(a, b):
    return float(torch.nn.functional.cosine_similarity(a.flatten().float(), b.flatten().float(), dim=0))


def record(name, **vals):
    path = os.environ.get("IMAGD_PARITY_OUT", tempfile.gettempdir())
    os.makedirs(path, exist_ok=True)
    f = os.path.join(path, "parity_full_chain.json")
    data = json.load(open(f)) if os.path.exists(f) else {}
    data[name] = vals
    json.dump(data, open(f, "w"), indent=1)


def make_inputs(dev, seed, h, w):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g).to(dev)
    return dict(latents=r(1, 4, h, w), garment=r(1, 4, h, w) * 0.9, prompt=r(1, 77, 768), negative=r(1, 77, 768),
                gtok=r(1, 16, 768), pose=torch.rand(1, 3, h * 8, w * 8, generator=g).to(dev))


@torch.no_grad()
def test_base_512_50_steps(cuda_device):
    from dressing_sd.pipelines.IMAGDressing_v1_pipeline import IMAGDressing_v1
    from oracle.pipeline import sample_one

    dev = cuda_device
    (o, ro, _), (p, rp, _), sched = build(dev)
    x = make_inputs(dev, 42, 64, 64)
    args = (x["latents"], x["prompt"], x["negative"], x["gtok"], x["garment"], 7.5, STEPS)
    ref = sample_one(o, ro, *args)
    pipe = IMAGDressing_v1(vae=None, reference_unet=rp, unet=p, tokenizer=None, text_encoder=None, image_encoder=None,
                           ImgProj=None, scheduler=sched, safety_checker=None, feature_extractor=None)
    out = pipe(prompt=None, null_prompt=None, negative_prompt=None, ref_image=None, width=512, height=512,
               num_inference_steps=STEPS, guidance_scale=7.5, image_scale=1.0, output_type="latent",
               prompt_embeds=x["prompt"], negative_prompt_embeds=x["negative"], latents=x["latents"],
               garment_tokens=x["gtok"], ref_image_latents=x["garment"]).images
    del pipe, p, rp
    drift = {}
    for name, dt in (("bf16", torch.bfloat16), ("fp16", torch.float16)):
        ob, rob = Cast(o.to(dt), dt), Cast(ro.to(dt), dt)
        drift[name] = sample_one(ob, rob, *args)
    e_k, e_b, e_h = rel_l2(out, ref), rel_l2(drift["bf16"], ref), rel_l2(drift["fp16"], ref)
    c_k, c_b, c_h = cosine(out, ref), cosine(drift["bf16"], ref), cosine(drift["fp16"], ref)
    print(f"512x512, 50 steps, final latents vs fp32 oracle: kernels rel-L2 {e_k:.4f} cos {c_k:.5f} | torch-bf16 "
          f"{e_b:.4f} cos {c_b:.5f} | torch-fp16 {e_h:.4f} cos {c_h:.5f}")
    record("base_512x512_50steps", kernel_rel_l2=e_k, kernel_cos=c_k, torch_bf16_rel_l2=e_b, torch_bf16_cos=c_b,
           torch_fp16_rel_l2=e_h, torch_fp16_cos=c_h, steps=STEPS, guidance=7.5)
    assert torch.isfinite(out).all()
    assert e_k <= max(2 * e_b, 3e-2), f"kernel chain error {e_k} vs torch-bf16 drift {e_b}"
    assert c_k > 0.98


@torch.no_grad()
def test_inpaint_768x576_batch2_50_steps(cuda_device):
    from dressing_sd.pipelines.IMAGDressing_v1_pipeline_controlnet_inpainting import IMAGDressing_v1
    from oracle.pipeline import sample_one

    dev = cuda_device
    h, w = 96, 72
    (o, ro, co), (p, rp, cp), sched = build(dev, controlnet=True)
    xs = [make_inputs(dev, s, h, w) for s in (50, 51)]
    g = torch.Generator().manual_seed(52)
    img_lat = [torch.randn(1, 4, h, w, generator=g).to(dev) for _ in xs]
    mask = torch.zeros(1, 1, h, w, device=dev)
    mask[:, :, h // 4: 3 * h // 4, w // 4: 3 * w // 4] = 1.0

    def run_oracle(u, r, c):
        return torch.cat([sample_one(u, r, x["latents"], x["prompt"], x["negative"], x["gtok"], x["garment"], 5.0, STEPS,
                                     controlnet=c, control_cond=x["pose"], control_scale=0.5, mask=mask,
                                     image_latents=il, noise=x["latents"]) for x, il in zip(xs, img_lat)])

    ref = run_oracle(o, ro, co)
    cat = lambda k: torch.cat([x[k] for x in xs])
    pipe = IMAGDressing_v1(vae=None, reference_unet=rp, unet=p, tokenizer=None, text_encoder=None, controlnet=cp,
                           image_encoder=None, ImgProj=None, scheduler=sched, safety_checker=None, feature_extractor=None)
    out = pipe(prompt=None, null_prompt=None, negative_prompt=None, ref_image=None, control_image=cat("pose"),
               height=h * 8, width=w * 8, strength=1.0, num_inference_steps=STEPS, guidance_scale=5.0,
               latents=cat("latents"), prompt_embeds=cat("prompt"), negative_prompt_embeds=cat("negative"),
               output_type="latent", controlnet_conditioning_scale=0.5, garment_tokens=cat("gtok"),
               ref_image_latents=cat("garment"), image_latents=torch.cat(img_lat), mask_latents=mask.expand(2, -1, -1, -1)
               ).images
    del pipe, p, rp, cp
    dt = torch.bfloat16
    bf = run_oracle(Cast(o.to(dt), dt), Cast(ro.to(dt), dt), Cast(co.to(dt), dt))
    keep = (mask == 0).expand_as(out)
    rep = (mask == 1).expand_as(out)
    e_k, e_b = rel_l2(out[rep], ref[rep]), rel_l2(bf[rep], ref[rep])
    c_k, c_b = cosine(out[rep], ref[rep]), cosine(bf[rep], ref[rep])
    print(f"768x576 inpaint, batch 2, 50 steps, repainted region vs fp32 oracle: kernels rel-L2 {e_k:.4f} cos {c_k:.5f} | "
          f"torch-bf16 {e_b:.4f} cos {c_b:.5f}")
    record("inpaint_768x576_b2_50steps", kernel_rel_l2=e_k, kernel_cos=c_k, torch_bf16_rel_l2=e_b, torch_bf16_cos=c_b,
           steps=STEPS, guidance=5.0)
    assert torch.isfinite(out).all()
    assert rel_l2(out[keep], torch.cat(img_lat)[keep]) < 1e-5  # unmasked region = the original latents, exactly
    assert e_k <= max(2 * e_b, 3e-2), f"kernel chain error {e_k} vs torch-bf16 drift {e_b}"
    assert c_k > 0.98
