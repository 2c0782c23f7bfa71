"""The four `IMAGDressing_v1` pipeline classes of the reference (dressing_sd/pipelines/IMAGDressing_v1_pipeline*.py)
behind their own constructor / `__call__` signatures, driving DenoiseEngine (batched CFG, CUDA-graph replayed
steps on the sm_90a kernels). The thin modules under dressing_sd/pipelines/ re-export these at the reference's
import paths so `inference_IMAGdressing*.py` import them unchanged.

Scope (SURVEY.md §8): the hot path is the garment pass + denoising loop. The edges — CLIP text/vision encoders
and the VAE — are caller-supplied modules invoked exactly where the reference invokes them (§8f "next" rows);
every edge can be bypassed with precomputed tensors (`prompt_embeds`, `negative_prompt_embeds`, `garment_tokens`,
`ref_image_latents`, `output_type="latent"`), which is how the offline benchmark and tests drive it.

Extensions over the reference (which hard-codes batch 1, SURVEY.md B1): any batch n = latents / prompt_embeds
batch or `num_images_per_prompt`; per-sample or shared (batch-1, broadcast) garment.
"""
from __future__ import annotations

from typing import Any, Callable, Dict, List, Optional, Union

import torch

from .engine import DenoiseEngine


class StableDiffusionPipelineOutput:
    def __init__(self, images, nsfw_content_detected=None):
        self.images = images
        self.nsfw_content_detected = nsfw_content_detected


def randn_tensor(shape, generator=None, device=None, dtype=torch.float32):
    """diffusers.utils.torch_utils.randn_tensor: CPU generators draw on the CPU then move (seed-42 parity,
    inference_IMAGdressing.py:43)."""
    gdev = generator.device.type if isinstance(generator, torch.Generator) else (device.type if device else "cpu")
    if isinstance(generator, (list, tuple)):
        return torch.cat([randn_tensor((1,) + tuple(shape[1:]), g, device, dtype) for g in generator], 0)
    if gdev == "cpu":
        return torch.randn(shape, generator=generator, dtype=dtype).to(device)
    return torch.randn(shape, generator=generator, device=device, dtype=dtype)


def _control_window(guess_mode, start, end):
    """Scalar (start, end) of the ControlNet guidance window; a one-element list is what diffusers normalises a single
    ControlNet's arguments to (ipa_controlnet.py:443-461)."""
    if guess_mode:
        raise NotImplementedError("guess_mode=True: every reference script runs guess_mode=False (the pose pipelines "
                                  "cannot even evaluate it, SURVEY.md B14); the cond-only ControlNet pass is not built")
    one = lambda v: float(v[0] if isinstance(v, (list, tuple)) else v)
    start, end = one(start), one(end)
    if not 0.0 <= start <= end <= 1.0:
        raise ValueError(f"control guidance window [{start}, {end}] must satisfy 0 <= start <= end <= 1")
    return start, end


def _image_batch(image, width, height, *, gray: bool = False) -> torch.Tensor:
    """PIL image(s) / HWC uint8-or-float arrays / CHW tensors -> float32 [n, 3|1, height, width] in [0, 1], resized
    with lanczos as diffusers-0.24 `VaeImageProcessor(resample="lanczos")` does for PIL input (tensors are resized
    bilinearly like its tensor path)."""
    import numpy as np

    if torch.is_tensor(image):
        t = image.float()
        t = t[None] if t.dim() == 3 else t
        if gray and t.shape[1] == 3:
            t = (0.299 * t[:, 0:1] + 0.587 * t[:, 1:2] + 0.114 * t[:, 2:3])
        if tuple(t.shape[-2:]) != (height, width):
            t = torch.nn.functional.interpolate(t, size=(height, width), mode="bilinear", align_corners=False)
        return t
    from PIL import Image

    imgs = list(image) if isinstance(image, (list, tuple)) else [image]
    out = []
    for im in imgs:
        if isinstance(im, np.ndarray):
            im = Image.fromarray((im * 255).round().astype("uint8") if im.dtype.kind == "f" else im)
        im = im.convert("L" if gray else "RGB").resize((width, height), resample=Image.LANCZOS)
        a = np.asarray(im).astype("float32") / 255.0
        out.append(a[None] if gray else a.transpose(2, 0, 1))
    return torch.from_numpy(np.stack(out))


class _DressingPipelineBase:
    """Shared implementation; subclasses fix the constructor signature and which side paths are active."""

    _has_controlnet = False
    _has_ipa = False
    _inpaint = False

    # ------------------------------------------------------------------ construction helpers
    def register_modules(self, **modules):
        for k, v in modules.items():
            setattr(self, k, v)

    def _encoder(self, name):
        """The CLIP text / vision encoder under `name`, running on the kernels once it lives on a CUDA device (clip.py;
        the wrapped transformers module stays the parameter container)."""
        from .clip import auto_accelerate

        enc = auto_accelerate(getattr(self, name, None))
        setattr(self, name, enc)
        return enc

    def _finish_init(self):
        vae = getattr(self, "vae", None)
        self.vae_scale_factor = 2 ** (len(vae.config.block_out_channels) - 1) if vae is not None else 8
        self._engine = DenoiseEngine(self.unet, self.reference_unet, getattr(self, "controlnet", None), self.scheduler)
        self._cross_attention_kwargs = None
        self._clip_skip = None

    @property
    def device(self):
        return self.unet.device

    _execution_device = device

    @property
    def cross_attention_kwargs(self):
        return self._cross_attention_kwargs

    @property
    def clip_skip(self):
        return self._clip_skip

    def to(self, *a, **k):
        for name in ("vae", "reference_unet", "unet", "controlnet", "text_encoder", "image_encoder", "ImgProj",
                     "image_proj_model"):
            m = getattr(self, name, None)
            if isinstance(m, torch.nn.Module):
                m.to(*a, **k)
        return self

    def progress_bar(self, iterable=None, total=None):
        class _Bar:
            def __enter__(s):
                return s

            def __exit__(s, *e):
                return False

            def update(s, *a):
                pass

        return _Bar()

    def maybe_free_model_hooks(self):
        pass

    # ------------------------------------------------------------------ scales (reference set_scale / set_ipa_scale)
    def set_scale(self, scale, lora_scale=None):
        from adapter.attention_processor import LoraRefSAttnProcessor2_0, RefSAttnProcessor2_0

        for p in self.unet.attn_processors.values():
            if isinstance(p, RefSAttnProcessor2_0):  # IMAGDressing_v1_pipeline.py:342-345
                p.scale = scale
            elif isinstance(p, LoraRefSAttnProcessor2_0) and lora_scale is not None:  # ipa_controlnet.py:379-383
                p.scale = scale
                p.lora_scale = lora_scale

    def set_ipa_scale(self, ipa_scale, lora_scale):
        from adapter.attention_processor import IPAttnProcessor2_0, LoRAIPAttnProcessor2_0

        for p in self.unet.attn_processors.values():  # ipa_controlnet.py:385-393
            if isinstance(p, (LoRAIPAttnProcessor2_0, IPAttnProcessor2_0)):
                p.scale = ipa_scale
                p.lora_scale = lora_scale

    # ------------------------------------------------------------------ edges (caller-supplied encoders)
    def encode_prompt(self, prompt, device, num_images_per_prompt, do_classifier_free_guidance, negative_prompt=None,
                      prompt_embeds=None, negative_prompt_embeds=None, lora_scale=None, clip_skip=None):
        """CLIP text encode of prompt / negative prompt (IMAGDressing_v1_pipeline.py:125-274) unless embeddings are
        supplied. Returns ([n,77,768], [n,77,768])."""

        def enc(texts):
            if self.tokenizer is None or self.text_encoder is None:
                raise ValueError("no tokenizer/text_encoder: pass prompt_embeds and negative_prompt_embeds")
            text_encoder = self._encoder("text_encoder")
            texts = [texts] if isinstance(texts, str) else list(texts)
            ids = self.tokenizer(texts, padding="max_length", max_length=self.tokenizer.model_max_length,
                                 truncation=True, return_tensors="pt").input_ids.to(device)
            if clip_skip is None:
                return text_encoder(ids)[0]
            hs = text_encoder(ids, output_hidden_states=True)[-1][-(clip_skip + 1)]
            return text_encoder.text_model.final_layer_norm(hs)

        if prompt_embeds is None:
            prompt_embeds = enc(prompt)
        if do_classifier_free_guidance and negative_prompt_embeds is None:
            n = prompt_embeds.shape[0]
            neg = negative_prompt if negative_prompt is not None else ""
            negative_prompt_embeds = enc([neg] * n if isinstance(neg, str) else neg)
        if num_images_per_prompt > 1 and prompt_embeds.shape[0] == 1:
            prompt_embeds = prompt_embeds.repeat(num_images_per_prompt, 1, 1)
            if negative_prompt_embeds is not None:
                negative_prompt_embeds = negative_prompt_embeds.repeat(num_images_per_prompt, 1, 1)
        return prompt_embeds, negative_prompt_embeds

    def prepare_latents(self, batch_size, num_channels_latents, width, height, dtype, device, generator, latents=None):
        shape = (batch_size, num_channels_latents, height // self.vae_scale_factor, width // self.vae_scale_factor)
        if isinstance(generator, list) and len(generator) != batch_size:
            raise ValueError(f"You have passed a list of generators of length {len(generator)}, but requested an "
                             f"effective batch size of {batch_size}.")
        if latents is None:
            latents = randn_tensor(shape, generator=generator, device=device, dtype=torch.float32)
        else:
            latents = latents.to(device=device, dtype=torch.float32)
        return latents * self.scheduler.init_noise_sigma

    def _garment_tokens(self, ref_clip_image, garment_tokens, device, dtype, prompt_embeds=None):
        """CLIP-vision penultimate hidden states -> ImgProj (Resampler) -> [n,16,768]
        (IMAGDressing_v1_pipeline.py:407-415). The null-image branch is not needed: the reference discards index 0
        of the garment pass (B2).

        `ref_clip_image is None` (reference :416-427): the reference calls
        `encode_prompt(null_prompt, ..., prompt_embeds=prompt_embeds, ...)` with the ALREADY ENCODED prompt embeddings,
        and diffusers' encode_prompt only tokenises when `prompt_embeds is None` — so `null_prompt` is never encoded and
        the garment UNet's text slot (index 1 of `cat([negative, null_prompt_embeds])`, :432-435) is the positive
        prompt's [n,77,768] embedding. Reproduced as is (quirk B19, DESIGN.md)."""
        if garment_tokens is not None:
            return garment_tokens
        if ref_clip_image is None:
            if prompt_embeds is None:
                raise ValueError("pass ref_clip_image (with an image_encoder), garment_tokens, or a prompt")
            return prompt_embeds
        if self.image_encoder is None:
            raise ValueError("no image_encoder: pass garment_tokens")
        enc = self._encoder("image_encoder")
        hs = enc(ref_clip_image.to(device, dtype=dtype), output_hidden_states=True).hidden_states[-2]
        return self.ImgProj(hs)

    def _ref_latents(self, ref_image, ref_image_latents, device):
        if ref_image_latents is not None:
            return ref_image_latents.to(device=device, dtype=torch.float32)
        if self.vae is None:
            raise ValueError("no vae: pass ref_image_latents")
        x = ref_image.to(dtype=self.vae.dtype, device=self.vae.device)
        return (self.vae.encode(x).latent_dist.mean * 0.18215).float()  # IMAGDressing_v1_pipeline.py:454-458

    def _decode(self, latents, output_type, generator=None):
        if output_type == "latent" or self.vae is None:
            return latents
        image = self.vae.decode((latents / self.vae.config.scaling_factor).to(self.vae.dtype), return_dict=False)[0]
        image = (image.float() / 2 + 0.5).clamp(0, 1)
        if output_type == "pt":
            return image
        arr = (image.permute(0, 2, 3, 1).cpu().numpy() * 255).round().astype("uint8")
        if output_type == "np":
            return arr
        from PIL import Image

        return [Image.fromarray(a) for a in arr]

    # ------------------------------------------------------------------ the call
    @torch.no_grad()
    def _run(self, *, prompt, negative_prompt, ref_image, width, height, num_inference_steps, guidance_scale,
             ref_clip_image=None, num_images_per_prompt=1, image_scale=1.0, generator=None, output_type="pil",
             return_dict=True, clip_skip=None, callback=None, prompt_embeds=None, negative_prompt_embeds=None,
             cross_attention_kwargs=None, latents=None, garment_tokens=None, ref_image_latents=None,
             # ControlNet
             control_image=None, controlnet_conditioning_scale=1.0, control_guidance_start=0.0,
             control_guidance_end=1.0,
             # IP-Adapter
             face_tokens=None, face_null_tokens=None,
             # inpainting
             mask=None, image_latents=None, strength=1.0, noise=None, latents_scaled=False):
        """latents_scaled: `latents` is already the sampler's start (the inpainting pipeline builds it as
        noise * init_noise_sigma or add_noise(image_latents, noise, t_start)), so it is not rescaled here."""
        device = self._execution_device
        scheduler = self.scheduler
        self._cross_attention_kwargs = cross_attention_kwargs
        self._clip_skip = clip_skip
        if guidance_scale <= 1.0:
            raise NotImplementedError("the reference always samples with classifier-free guidance (scale 5-7.5)")
        height = height or self.unet.config.sample_size * self.vae_scale_factor
        width = width or self.unet.config.sample_size * self.vae_scale_factor

        prompt_embeds, negative_prompt_embeds = self.encode_prompt(
            prompt, device, num_images_per_prompt, True, negative_prompt, prompt_embeds=prompt_embeds,
            negative_prompt_embeds=negative_prompt_embeds, clip_skip=clip_skip)
        n = latents.shape[0] if latents is not None else max(prompt_embeds.shape[0], num_images_per_prompt)
        control_pe, control_ne = prompt_embeds, negative_prompt_embeds  # ControlNet sees text only (ipa_controlnet.py:550)
        if face_tokens is not None:  # ipa_controlnet.py:555-557: append the 4 face tokens to the text
            fn = face_null_tokens if face_null_tokens is not None else torch.zeros_like(face_tokens)
            prompt_embeds = torch.cat([prompt_embeds, face_tokens.to(prompt_embeds).expand(prompt_embeds.shape[0], -1, -1)], 1)
            negative_prompt_embeds = torch.cat(
                [negative_prompt_embeds, fn.to(prompt_embeds).expand(negative_prompt_embeds.shape[0], -1, -1)], 1)

        scheduler.set_timesteps(num_inference_steps, device=device)
        timesteps = scheduler.timesteps
        if self._inpaint and strength < 1.0:
            init = min(int(num_inference_steps * strength), num_inference_steps)
            timesteps = timesteps[max(num_inference_steps - init, 0):]

        if latents_scaled:
            latents = latents.to(device=device, dtype=torch.float32)
        else:
            latents = self.prepare_latents(n, self.unet.config.in_channels, width, height, torch.float32, device,
                                           generator, latents)
        step_noise = None
        if getattr(scheduler, "_needs_noise", False):
            # Euler-ancestral: the reference loop's step() draws one latents-shaped tensor per step from `generator`,
            # in step order after prepare_latents; drawn here in the same order and staged for the captured graph
            step_noise = torch.stack([randn_tensor(latents.shape, generator=generator, device=device)
                                      for _ in range(len(timesteps))])
        gtok = self._garment_tokens(ref_clip_image, garment_tokens, device, prompt_embeds.dtype, control_pe)
        if gtok.shape[0] != n:
            gtok = gtok.expand(n, -1, -1)
        ref_lat = self._ref_latents(ref_image, ref_image_latents, device)
        sa = self._engine.garment_features(ref_lat, gtok)

        keep = None
        if control_image is not None and (control_guidance_start != 0.0 or control_guidance_end != 1.0):
            T = len(timesteps)  # controlnet_keep, ipa_controlnet.py:584-590 / inpainting.py:373-379
            keep = [1.0 - float(i / T < control_guidance_start or (i + 1) / T > control_guidance_end) for i in range(T)]
        out = self._engine.sample(
            latents, prompt_embeds, negative_prompt_embeds, sa, guidance_scale, len(timesteps), timesteps=timesteps,
            control_keep=keep,
            control_cond=control_image, control_prompt_embeds=control_pe, control_negative_embeds=control_ne,
            control_scale=controlnet_conditioning_scale, mask=mask, image_latents=image_latents, noise=noise,
            callback=callback, scheduler=scheduler, step_noise=step_noise)
        image = self._decode(out, output_type, generator)
        if not return_dict:
            return (image, None)
        return StableDiffusionPipelineOutput(images=image, nsfw_content_detected=None)


# ====================================================================================================== base
class IMAGDressing_v1_Base(_DressingPipelineBase):
    """dressing_sd/pipelines/IMAGDressing_v1_pipeline.py:18 — constructor :21-65, __call__ :347-547."""

    def __init__(self, vae, reference_unet, unet, tokenizer, text_encoder, image_encoder, ImgProj, scheduler,
                 safety_checker=None, feature_extractor=None, requires_safety_checker: bool = False):
        self.register_modules(vae=vae, reference_unet=reference_unet, unet=unet, scheduler=scheduler,
                              tokenizer=tokenizer, text_encoder=text_encoder, image_encoder=image_encoder,
                              ImgProj=ImgProj, safety_checker=safety_checker, feature_extractor=feature_extractor)
        self._finish_init()

    def __call__(self, prompt, null_prompt, negative_prompt, ref_image, width, height, num_inference_steps,
                 guidance_scale, ref_clip_image=None, num_images_per_prompt=1, image_scale=1.0, num_samples=1,
                 eta: float = 0.0, generator=None, output_type: Optional[str] = "pil", return_dict: bool = True,
                 clip_skip: Optional[int] = None, callback: Optional[Callable] = None, callback_steps: Optional[int] = 1,
                 prompt_embeds=None, negative_prompt_embeds=None, cross_attention_kwargs: Optional[Dict[str, Any]] = None,
                 latents=None, garment_tokens=None, ref_image_latents=None, **kwargs):
        self.set_scale(image_scale)  # :374
        return self._run(prompt=prompt, negative_prompt=negative_prompt, ref_image=ref_image, width=width, height=height,
                         num_inference_steps=num_inference_steps, guidance_scale=guidance_scale,
                         ref_clip_image=ref_clip_image, num_images_per_prompt=num_images_per_prompt,
                         image_scale=image_scale, generator=generator, output_type=output_type, return_dict=return_dict,
                         clip_skip=clip_skip, callback=callback, prompt_embeds=prompt_embeds,
                         negative_prompt_embeds=negative_prompt_embeds, cross_attention_kwargs=cross_attention_kwargs,
                         latents=latents, garment_tokens=garment_tokens, ref_image_latents=ref_image_latents)


# ====================================================================================================== ControlNet pose
class IMAGDressing_v1_ControlNet(_DressingPipelineBase):
    """dressing_sd/pipelines/IMAGDressing_v1_pipeline_controlnet.py:22 — __call__ :357-677."""

    _has_controlnet = True

    def __init__(self, vae, reference_unet, unet, tokenizer, text_encoder, controlnet, image_encoder, ImgProj, scheduler,
                 safety_checker=None, feature_extractor=None, requires_safety_checker: bool = False):
        self.register_modules(vae=vae, reference_unet=reference_unet, unet=unet, controlnet=controlnet,
                              scheduler=scheduler, tokenizer=tokenizer, text_encoder=text_encoder,
                              image_encoder=image_encoder, ImgProj=ImgProj, safety_checker=safety_checker,
                              feature_extractor=feature_extractor)
        self._finish_init()

    def prepare_image(self, image, width, height, device):
        """Pose image -> [n,3,H,W] in [0,1] (StableDiffusionControlNetPipeline.prepare_image, do_normalize=False)."""
        if torch.is_tensor(image):
            return image.to(device=device, dtype=torch.float32)
        return _image_batch(image, width, height).to(device)  # control_image_processor: lanczos, no normalisation

    def __call__(self, prompt, null_prompt, negative_prompt, ref_image, width, height, num_inference_steps,
                 guidance_scale, pose_image=None, ref_clip_image=None, num_images_per_prompt=1, image_scale=1.0,
                 num_samples=1, eta: float = 0.0, generator=None, output_type: Optional[str] = "pil",
                 return_dict: bool = True, clip_skip=None, callback=None, callback_steps=1, prompt_embeds=None,
                 negative_prompt_embeds=None, cross_attention_kwargs=None,
                 controlnet_conditioning_scale: Union[float, List[float]] = 1.0, guess_mode: bool = False,
                 control_guidance_start=0.0, control_guidance_end=1.0, latents=None, garment_tokens=None,
                 ref_image_latents=None, **kwargs):
        start, end = _control_window(guess_mode, control_guidance_start, control_guidance_end)
        self.set_scale(image_scale)
        ctrl = self.prepare_image(pose_image, width, height, self._execution_device) if pose_image is not None else None
        return self._run(prompt=prompt, negative_prompt=negative_prompt, ref_image=ref_image, width=width, height=height,
                         num_inference_steps=num_inference_steps, guidance_scale=guidance_scale,
                         ref_clip_image=ref_clip_image, num_images_per_prompt=num_images_per_prompt,
                         generator=generator, output_type=output_type, return_dict=return_dict, clip_skip=clip_skip,
                         callback=callback, prompt_embeds=prompt_embeds, negative_prompt_embeds=negative_prompt_embeds,
                         cross_attention_kwargs=cross_attention_kwargs, latents=latents, garment_tokens=garment_tokens,
                         ref_image_latents=ref_image_latents, control_image=ctrl,
                         controlnet_conditioning_scale=float(controlnet_conditioning_scale),
                         control_guidance_start=start, control_guidance_end=end)


# ====================================================================================================== IPA + ControlNet
class IMAGDressing_v1_IPAControlNet(IMAGDressing_v1_ControlNet):
    """dressing_sd/pipelines/IMAGDressing_v1_pipeline_ipa_controlnet.py:24 — ctor :27-86, load_ip_adapter :88-101,
    get_image_embeds :366-377, scales :379-393, __call__ :396-742."""

    _has_ipa = True

    def __init__(self, vae, reference_unet, unet, tokenizer, text_encoder, controlnet, image_encoder, ImgProj, ip_ckpt,
                 scheduler, safety_checker=None, feature_extractor=None, requires_safety_checker: bool = False):
        super().__init__(vae, reference_unet, unet, tokenizer, text_encoder, controlnet, image_encoder, ImgProj,
                         scheduler, safety_checker, feature_extractor)
        self.ip_ckpt = ip_ckpt
        self.num_tokens = 4
        self.image_proj_model = self.init_proj()
        if ip_ckpt is not None:
            self.load_ip_adapter()

    def init_proj(self):
        from adapter.resampler import ProjPlusModel

        clip_dim = self.image_encoder.config.hidden_size if self.image_encoder is not None else 1280
        return ProjPlusModel(cross_attention_dim=self.unet.config.cross_attention_dim, id_embeddings_dim=512,
                             clip_embeddings_dim=clip_dim, num_tokens=self.num_tokens).to(self.unet.device)

    def load_ip_adapter(self):
        """FaceID checkpoint: `image_proj.*` -> ProjPlusModel, `ip_adapter.{i}.*` -> processors by ModuleList index
        (attn2 processors sit at odd indices, SURVEY.md A.2), strict=False (:88-101). Implemented in checkpoint.py."""
        from .checkpoint import load_ip_adapter_checkpoint

        load_ip_adapter_checkpoint(self.ip_ckpt, image_proj_model=self.image_proj_model, unet=self.unet)

    @torch.no_grad()
    def get_image_embeds(self, face_clip_image=None, faceid_embeds=None, face_clip_embeds=None):
        """(:366-377) ProjPlusModel(faceid, CLIP hidden_states[-2], shortcut=False); uncond = zeros inputs (B12)."""
        dev = self.device
        if face_clip_embeds is None:
            enc = self._encoder("image_encoder")
            face_clip_embeds = enc(face_clip_image.to(dev, dtype=enc.dtype), output_hidden_states=True).hidden_states[-2]
            zero_clip = enc(torch.zeros_like(face_clip_image).to(dev, dtype=enc.dtype),
                            output_hidden_states=True).hidden_states[-2]
        else:
            zero_clip = torch.zeros_like(face_clip_embeds)
        fid = faceid_embeds.to(dev)
        cond = self.image_proj_model(fid, face_clip_embeds.to(dev), shortcut=False, scale=1.0)
        unc = self.image_proj_model(torch.zeros_like(fid), zero_clip.to(dev), shortcut=False, scale=1.0)
        return cond, unc

    def __call__(self, prompt, null_prompt, negative_prompt, ref_image, width, height, num_inference_steps,
                 guidance_scale, pose_image=None, ref_clip_image=None, face_clip_image=None, faceid_embeds=None,
                 num_images_per_prompt=1, image_scale=1.0, ipa_scale=0.0, s_lora_scale=0.0, c_lora_scale=0.0,
                 num_samples=1, eta: float = 0.0, generator=None, output_type: Optional[str] = "pil",
                 return_dict: bool = True, clip_skip=None, callback=None, callback_steps=1, prompt_embeds=None,
                 negative_prompt_embeds=None, cross_attention_kwargs=None,
                 controlnet_conditioning_scale: Union[float, List[float]] = 1.0, guess_mode: bool = False,
                 control_guidance_start=0.0, control_guidance_end=1.0, latents=None, garment_tokens=None,
                 ref_image_latents=None, face_clip_embeds=None, face_tokens=None, face_null_tokens=None, **kwargs):
        start, end = _control_window(guess_mode, control_guidance_start, control_guidance_end)
        has_face = faceid_embeds is not None or face_tokens is not None
        if has_face:  # :433-438
            self.set_scale(image_scale, lora_scale=s_lora_scale)
            self.set_ipa_scale(ipa_scale, c_lora_scale)
            if face_tokens is None:
                face_tokens, face_null_tokens = self.get_image_embeds(face_clip_image, faceid_embeds, face_clip_embeds)
        else:
            self.set_scale(image_scale, lora_scale=0.0)
            self.set_ipa_scale(0.0, 0.0)
        ctrl = self.prepare_image(pose_image, width, height, self._execution_device) if pose_image is not None else None
        return self._run(prompt=prompt, negative_prompt=negative_prompt, ref_image=ref_image, width=width, height=height,
                         num_inference_steps=num_inference_steps, guidance_scale=guidance_scale,
                         ref_clip_image=ref_clip_image, num_images_per_prompt=num_images_per_prompt,
                         generator=generator, output_type=output_type, return_dict=return_dict, clip_skip=clip_skip,
                         callback=callback, prompt_embeds=prompt_embeds, negative_prompt_embeds=negative_prompt_embeds,
                         cross_attention_kwargs=cross_attention_kwargs, latents=latents, garment_tokens=garment_tokens,
                         ref_image_latents=ref_image_latents, control_image=ctrl,
                         controlnet_conditioning_scale=float(controlnet_conditioning_scale), face_tokens=face_tokens,
                         face_null_tokens=face_null_tokens, control_guidance_start=start, control_guidance_end=end)


# ====================================================================================================== inpainting
class IMAGDressing_v1_ControlNetInpaint(IMAGDressing_v1_ControlNet):
    """dressing_sd/pipelines/IMAGDressing_v1_pipeline_controlnet_inpainting.py:13 — __call__ :117-548: 4-channel
    UNet, per-step blend latents = (1-m)*add_noise(image_latents, noise, t_{i+1}) + m*latents (:487-500)."""

    _inpaint = True

    def __call__(self, prompt=None, null_prompt=None, negative_prompt=None, ref_image=None, image=None, mask_image=None,
                 control_image=None, height=None, width=None, strength: float = 1.0, num_inference_steps: int = 50,
                 guidance_scale: float = 7.5, ref_clip_image=None, num_images_per_prompt: int = 1, image_scale=1.0,
                 eta: float = 0.0, generator=None, latents=None, prompt_embeds=None, negative_prompt_embeds=None,
                 output_type: Optional[str] = "pil", return_dict: bool = True, callback=None, callback_steps: int = 1,
                 cross_attention_kwargs=None, controlnet_conditioning_scale: Union[float, List[float]] = 0.5,
                 guess_mode: bool = False, control_guidance_start=0.0, control_guidance_end=1.0, clip_skip=None,
                 garment_tokens=None, ref_image_latents=None, image_latents=None, mask_latents=None, **kwargs):
        cg_start, cg_end = _control_window(guess_mode, control_guidance_start, control_guidance_end)
        dev = self._execution_device
        self.set_scale(image_scale)
        ctrl = self.prepare_image(control_image, width, height, dev) if control_image is not None else None
        if image_latents is None:
            if self.vae is None:
                raise ValueError("no vae: pass image_latents and mask_latents")
            if height is None or width is None:
                raise ValueError("height and width are required to preprocess `image`")
            # image_processor.preprocess (:301-304): resize to (height, width), [0,1] -> [-1,1]
            img = (_image_batch(image, width, height) * 2.0 - 1.0).to(device=dev, dtype=self.vae.dtype)
            dist = self.vae.encode(img).latent_dist  # _encode_vae_image: latent_dist.sample(generator) * scaling_factor
            z = dist.sample(generator) if hasattr(dist, "sample") else dist.mean
            image_latents = (z * self.vae.config.scaling_factor).float()
        n = image_latents.shape[0]
        h, w = image_latents.shape[-2:]
        if mask_latents is None:
            # mask_processor.preprocess (:306-308): grayscale, resize, binarise at 0.5; prepare_mask_latents (:352-362)
            # then resizes to the latent grid with F.interpolate's default nearest mode
            m = _image_batch(mask_image, w * self.vae_scale_factor, h * self.vae_scale_factor, gray=True)
            m = (m >= 0.5).to(device=dev, dtype=torch.float32)
            mask_latents = torch.nn.functional.interpolate(m, size=(h, w))
        if ctrl is not None and tuple(ctrl.shape[-2:]) != (h * self.vae_scale_factor, w * self.vae_scale_factor):
            raise ValueError(f"control_image {tuple(ctrl.shape[-2:])} does not match the image "
                             f"{(h * self.vae_scale_factor, w * self.vae_scale_factor)}")
        if mask_latents.shape[0] != n:
            mask_latents = mask_latents.expand(n, -1, -1, -1)
        noise = randn_tensor(image_latents.shape, generator=generator, device=dev) if latents is None else latents.to(dev)
        # is_strength_max: pure noise start scaled by init_noise_sigma; else add_noise(image_latents, noise, t_start),
        # not rescaled (inherited prepare_latents); _run takes the start as is
        self.scheduler.set_timesteps(num_inference_steps, device=dev)
        ts = self.scheduler.timesteps
        if strength < 1.0:
            init = min(int(num_inference_steps * strength), num_inference_steps)
            t0 = ts[max(num_inference_steps - init, 0)]
            start = self.scheduler.add_noise(image_latents, noise, t0.reshape(1).expand(n))
        else:
            start = noise * self.scheduler.init_noise_sigma
        return self._run(prompt=prompt, negative_prompt=negative_prompt, ref_image=ref_image, width=width, height=height,
                         num_inference_steps=num_inference_steps, guidance_scale=guidance_scale,
                         ref_clip_image=ref_clip_image, num_images_per_prompt=num_images_per_prompt,
                         generator=generator, output_type=output_type, return_dict=return_dict, clip_skip=clip_skip,
                         callback=callback, prompt_embeds=prompt_embeds, negative_prompt_embeds=negative_prompt_embeds,
                         cross_attention_kwargs=cross_attention_kwargs, latents=start, garment_tokens=garment_tokens,
                         ref_image_latents=ref_image_latents, control_image=ctrl,
                         controlnet_conditioning_scale=float(controlnet_conditioning_scale), mask=mask_latents,
                         image_latents=image_latents, strength=strength, noise=noise, control_guidance_start=cg_start,
                         control_guidance_end=cg_end, latents_scaled=True)
