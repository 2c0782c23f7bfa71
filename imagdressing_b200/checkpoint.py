"""Checkpoint / weight-format loader for the IMAGDressing-v1 hot path (SURVEY.md §8f-2).

Three on-disk formats reach the reference's models, all restated here so real weights can run on the sm_90a kernels:

1. The DeepSpeed training checkpoint `IMAGDressing-v1_512.pt`: `torch.load(path)["module"]` is the state_dict of
   `train.py`'s `SDModel` (members `unet`, `ref_unet`, `proj`, `adapter_modules`, train.py:244-253), routed by key
   prefix exactly as inference_IMAGdressing.py:97-114 does — `ref_unet.*` -> the garment UNet, `proj.*` -> the
   Resampler, `adapter_modules.{i}.*` -> the i-th entry of `ModuleList(unet.attn_processors.values())` (attn1 processors
   at even indices: `to_k_ref.weight`, `to_v_ref.weight`), and `unet.*` collected but NEVER loaded (quirk B8: the
   denoising UNet keeps its base Realistic-Vision weights, :106-107,115-117).
2. The IP-Adapter-FaceID checkpoint (`.bin` or `.safetensors`): `image_proj.*` -> ProjPlusModel, `ip_adapter.{i}.*` ->
   the same processor ModuleList with strict=False (IMAGDressing_v1_pipeline_ipa_controlnet.py:88-101; attn2 processors
   at odd indices: `to_k_ip.weight`, `to_v_ip.weight`, `to_{q,k,v,out}_lora.{down,up}.weight`).
3. diffusers model directories (`config.json` + `diffusion_pytorch_model{,.fp16}.{safetensors,bin}`):
   `modeling._ModelBase.from_pretrained`.

All of them end in `load_state_dict` on modules that hold parameters under the diffusers key names; the kernel-layout
copies (bf16, tap-major convs, fused q/k/v, interleaved GEGLU rows, LayerNorm-folded and LoRA-merged projections) are
derived lazily and are versioned on the source parameters (processors._ver), so a load after a forward can never leave a
stale packed weight behind. `export_module_checkpoint` writes format 1 (for tests and for round-tripping fine-tuned
adapters); nothing here needs a GPU.
"""
from __future__ import annotations

import os
from typing import Dict, Iterable, Optional, Tuple

import torch
import torch.nn as nn

PREFIXES = ("ref_unet", "unet", "proj", "adapter_modules")  # checked in THIS order (inference_IMAGdressing.py:103-110)


def split_module_checkpoint(model_sd: Dict[str, torch.Tensor]) -> Tuple[Dict[str, Dict[str, torch.Tensor]], list]:
    """Route SDModel keys by prefix. Returns ({"ref_unet": {...}, "unet": {...}, "proj": {...},
    "adapter_modules": {...}}, unrouted_keys). Mirrors the reference down to its `str.replace` (which removes EVERY
    occurrence of the prefix string, not only the leading one; harmless for real key names)."""
    out = {p: {} for p in PREFIXES}
    other = []
    for k, v in model_sd.items():
        if k.startswith("ref_unet"):
            out["ref_unet"][k.replace("ref_unet.", "")] = v
        elif k.startswith("unet"):
            out["unet"][k.replace("unet.", "")] = v
        elif k.startswith("proj"):
            out["proj"][k.replace("proj.", "")] = v
        elif k.startswith("adapter_modules"):
            out["adapter_modules"][k.replace("adapter_modules.", "")] = v
        else:
            other.append(k)
    return out, other


def processor_list(unet) -> nn.ModuleList:
    """`torch.nn.ModuleList(unet.attn_processors.values())` (inference_IMAGdressing.py:87): the index of a processor in
    this list is the `{i}` of `adapter_modules.{i}.*` / `ip_adapter.{i}.*` keys, so the order must be the diffusers
    module-tree order (down, up, mid; attn1 even, attn2 odd — SURVEY.md A.2)."""
    return nn.ModuleList(list(unet.attn_processors.values()))


def load_module_checkpoint(ckpt, *, reference_unet, image_proj, unet, strict: bool = True,
                           load_denoising_unet: bool = False) -> dict:
    """inference_IMAGdressing.py:97-114 on already-constructed modules. `ckpt`: a path, the loaded dict, or its
    `["module"]`. `load_denoising_unet=False` reproduces quirk B8 (the `unet.*` entries are not applied); True applies
    them (what a fine-tune that DID train the denoising UNet would need). Returns a small report."""
    if isinstance(ckpt, (str, os.PathLike)):
        ckpt = torch.load(ckpt, map_location="cpu", weights_only=True)
    model_sd = ckpt["module"] if "module" in ckpt and isinstance(ckpt["module"], dict) else ckpt
    parts, other = split_module_checkpoint(model_sd)
    reference_unet.load_state_dict(parts["ref_unet"], strict=strict)
    image_proj.load_state_dict(parts["proj"], strict=strict)
    layers = processor_list(unet)
    layers.load_state_dict(parts["adapter_modules"], strict=strict)
    if load_denoising_unet and parts["unet"]:
        own = {k: v for k, v in parts["unet"].items() if ".processor." not in k}
        unet.load_state_dict(own, strict=False)
    for m in (reference_unet, unet):
        if hasattr(m, "invalidate_packed"):
            m.invalidate_packed()
    return {"ref_unet": len(parts["ref_unet"]), "unet_ignored": 0 if load_denoising_unet else len(parts["unet"]),
            "proj": len(parts["proj"]), "adapter_modules": len(parts["adapter_modules"]), "unrouted": other}


def export_module_checkpoint(path, *, reference_unet, image_proj, unet, include_denoising_unet: bool = True) -> None:
    """Write format 1: {"module": SDModel-style state_dict}. The `unet.*` block carries the denoising UNet INCLUDING its
    processors' parameters under `unet.<layer>.processor.*`, as SDModel.state_dict() does (the processors are
    submodules of the UNet's Attention layers as well as members of `adapter_modules`)."""
    sd = {}
    for k, v in reference_unet.state_dict().items():
        sd["ref_unet." + k] = v.detach().cpu()
    if include_denoising_unet:
        for k, v in unet.state_dict().items():
            sd["unet." + k] = v.detach().cpu()
    for k, v in image_proj.state_dict().items():
        sd["proj." + k] = v.detach().cpu()
    for k, v in processor_list(unet).state_dict().items():
        sd["adapter_modules." + k] = v.detach().cpu()
    torch.save({"module": sd}, path)


def read_ip_adapter_checkpoint(path) -> Dict[str, Dict[str, torch.Tensor]]:
    """{"image_proj": {...}, "ip_adapter": {...}} from a FaceID `.bin` (already nested) or `.safetensors` (flat keys with
    the two prefixes) — IMAGDressing_v1_pipeline_ipa_controlnet.py:89-98."""
    if os.path.splitext(str(path))[-1] == ".safetensors":
        from safetensors import safe_open

        sd = {"image_proj": {}, "ip_adapter": {}}
        with safe_open(str(path), framework="pt", device="cpu") as f:
            for key in f.keys():
                if key.startswith("image_proj."):
                    sd["image_proj"][key.replace("image_proj.", "")] = f.get_tensor(key)
                elif key.startswith("ip_adapter."):
                    sd["ip_adapter"][key.replace("ip_adapter.", "")] = f.get_tensor(key)
        return sd
    return torch.load(str(path), map_location="cpu", weights_only=True)


def load_ip_adapter_checkpoint(path_or_sd, *, image_proj_model, unet) -> None:
    """IMAGDressing_v1_pipeline_ipa_controlnet.py:99-101: strict load of the projection model, strict=False load of the
    processor list (the checkpoint only holds the attn2 / LoRA entries)."""
    sd = path_or_sd if isinstance(path_or_sd, dict) else read_ip_adapter_checkpoint(path_or_sd)
    image_proj_model.load_state_dict(sd["image_proj"])
    processor_list(unet).load_state_dict(sd["ip_adapter"], strict=False)
    if hasattr(unet, "invalidate_packed"):
        unet.invalidate_packed()


def copy_self_attention_into_ref_projections(unet) -> int:
    """train.py:355-359: `to_k_ref` / `to_v_ref` start as copies of the layer's own `to_k` / `to_v` (how a fresh adapter
    is initialised before fine-tuning). Returns the number of processors touched."""
    n = 0
    sd = unet.state_dict()
    for name, proc in unet.attn_processors.items():
        if hasattr(proc, "to_k_ref") and name.endswith("attn1.processor"):
            layer = name[: -len(".processor")]
            with torch.no_grad():
                proc.to_k_ref.weight.copy_(sd[layer + ".to_k.weight"])
                proc.to_v_ref.weight.copy_(sd[layer + ".to_v.weight"])
            n += 1
    if hasattr(unet, "invalidate_packed"):
        unet.invalidate_packed()
    return n
