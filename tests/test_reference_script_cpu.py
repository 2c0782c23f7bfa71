"""CPU, BASELINE.json configs[0] / VERDICT r1 item 7-8: the reference's UNMODIFIED `inference_IMAGdressing.py` is executed
as `__main__` (runpy) — `prepare()` + `pipe(...)` + the image grid it saves — against this repo's drop-ins:

  * `dressing_sd.pipelines.IMAGDressing_v1_pipeline.IMAGDressing_v1`, `adapter.attention_processor.*`,
    `adapter.resampler.Resampler` resolve to this repo (same module paths);
  * `from diffusers import UNet2DConditionModel, AutoencoderKL, DDIMScheduler` resolves to the opt-in stand-in
    (imagdressing_b200/compat), i.e. the kernel-backed UNet / VAE / scheduler;
  * `transformers` (real, installed) provides CLIPTextModel / CLIPTokenizer / CLIPVisionModelWithProjection /
    CLIPImageProcessor; torchvision (real) the transforms.

Test infrastructure only: the hub ids the script hard-codes ("stabilityai/sd-vae-ft-mse", "SG161222/Realistic_Vision_V4.0_noVAE",
"h94/IP-Adapter") are satisfied by directories of those names under a temporary working directory holding small random-init
models (a relative path that exists is a local directory for both transformers and our from_pretrained), a toy CLIP BPE
vocabulary, and a synthetic `{"module": ...}` checkpoint with the `ref_unet.` / `unet.` / `proj.` / `adapter_modules.`
layout; the kernel wrappers are emulated in torch (tests/emulated_ops.py) because this suite has no GPU.

The script is reference source and is not copied into this repository. With a reference checkout named by
$IMAGD_REFERENCE_DIR the script itself runs, and every call it makes across the boundary into this repo (the
from_pretrained loads, the Resampler / processor / scheduler / pipeline constructors, the dtypes it casts to, the pipeline
call, the saved grid) is recorded and compared with tests/golden/inference_script_trace.json. Without a checkout the same
sequence is replayed from that recorded trace (`replay` restates the script's steps, inference_IMAGdressing.py:42-197,
with every value taken from the trace) and the same assertions run. IMAGD_WRITE_TRACE=1 rewrites the trace from a live run.
"""
import json
import os
import runpy
import sys

import pytest
import torch

import emulated_ops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REFERENCE_DIR = os.environ.get("IMAGD_REFERENCE_DIR")
SCRIPT = os.path.join(REFERENCE_DIR, "inference_IMAGdressing.py") if REFERENCE_DIR else None
TRACE = os.path.join(ROOT, "tests", "golden", "inference_script_trace.json")

UNET_CFG = dict(block_out_channels=[32, 64, 64, 64], cross_attention_dim=64, attention_head_dim=8, norm_num_groups=8)
VAE_CFG = dict(block_out_channels=[32, 32, 64, 64], norm_num_groups=8)


def make_tokenizer(d):
    """A CLIP-style byte-level BPE vocabulary with NO merges (every byte, bare and word-final), built and saved through the
    installed transformers so the files are in whatever format that version reads back."""
    from transformers import CLIPTokenizer

    # GPT-2 / CLIP byte -> printable unicode table
    bs = list(range(ord("!"), ord("~") + 1)) + list(range(0xA1, 0xAD)) + list(range(0xAE, 0x100))
    cs = bs[:]
    n = 0
    for b in range(256):
        if b not in bs:
            bs.append(b)
            cs.append(256 + n)
            n += 1
    chars = [chr(c) for c in cs]
    vocab = {}
    for c in chars:
        vocab[c] = len(vocab)
    for c in chars:
        vocab[c + "</w>"] = len(vocab)
    vocab["<|startoftext|>"] = len(vocab)
    vocab["<|endoftext|>"] = len(vocab)
    tok = CLIPTokenizer(vocab=vocab, merges=[], model_max_length=77)
    tok.save_pretrained(d)
    ids = CLIPTokenizer.from_pretrained(d)("a cat", padding="max_length", max_length=77, truncation=True).input_ids
    assert len(ids) == 77 and ids[0] == vocab["<|startoftext|>"] and vocab["<|endoftext|>"] in ids
    return len(vocab)


def make_hub(tmp):
    from safetensors.torch import save_file
    from transformers import CLIPTextConfig, CLIPTextModel, CLIPVisionConfig, CLIPVisionModelWithProjection

    from imagdressing_b200 import modeling, vae

    torch.manual_seed(0)
    rv = os.path.join(tmp, "SG161222", "Realistic_Vision_V4.0_noVAE")
    n_vocab = make_tokenizer(os.path.join(rv, "tokenizer"))
    CLIPTextModel(CLIPTextConfig(vocab_size=n_vocab, hidden_size=64, intermediate_size=128, num_hidden_layers=2,
                                 num_attention_heads=4, max_position_embeddings=77, projection_dim=64,
                                 bos_token_id=n_vocab - 2, eos_token_id=n_vocab - 1, pad_token_id=n_vocab - 1)
                  ).save_pretrained(os.path.join(rv, "text_encoder"))
    unet = modeling.UNet2DConditionModel(**UNET_CFG)
    modeling.init_synthetic_(unet, 0)
    os.makedirs(os.path.join(rv, "unet"))
    json.dump(UNET_CFG, open(os.path.join(rv, "unet", "config.json"), "w"))
    save_file({k: v.contiguous() for k, v in unet.state_dict().items()},
              os.path.join(rv, "unet", "diffusion_pytorch_model.safetensors"))
    CLIPVisionModelWithProjection(CLIPVisionConfig(hidden_size=48, intermediate_size=96, num_hidden_layers=2,
                                                   num_attention_heads=4, image_size=224, patch_size=14, projection_dim=32)
                                  ).save_pretrained(os.path.join(tmp, "h94", "IP-Adapter", "models", "image_encoder"))
    v = vae.AutoencoderKL(**VAE_CFG)
    modeling.init_synthetic_(v, 3)
    vd = os.path.join(tmp, "stabilityai", "sd-vae-ft-mse")
    os.makedirs(vd)
    json.dump(VAE_CFG, open(os.path.join(vd, "config.json"), "w"))
    save_file({k: v_.contiguous() for k, v_ in v.state_dict().items()}, os.path.join(vd, "diffusion_pytorch_model.safetensors"))
    return unet


def make_checkpoint(tmp, unet):
    """SDModel-style DeepSpeed checkpoint (train.py:244-253 member names) with fresh 'trained' values."""
    from adapter.attention_processor import CAttnProcessor2_0, RefSAttnProcessor2_0
    from adapter.resampler import Resampler
    from imagdressing_b200 import modeling

    g = torch.Generator().manual_seed(1)
    ref = modeling.UNet2DConditionModel(**UNET_CFG)
    modeling.init_synthetic_(ref, 1)
    proj = Resampler(dim=64, depth=4, dim_head=64, heads=12, num_queries=16, embedding_dim=48, output_dim=64, ff_mult=4)
    sd = {"ref_unet." + k: v for k, v in ref.state_dict().items()}
    sd.update({"unet." + k: v for k, v in unet.state_dict().items()})
    sd.update({"proj." + k: v + 0.01 * torch.randn(v.shape, generator=g) for k, v in proj.state_dict().items()})
    boc = UNET_CFG["block_out_channels"]
    for i, name in enumerate(unet.attn_processors.keys()):
        if name.endswith("attn1.processor"):
            hidden = boc[-1] if name.startswith("mid") else (list(reversed(boc))[int(name[len("up_blocks.")])]
                                                             if name.startswith("up") else boc[int(name[len("down_blocks.")])])
            for w in ("to_k_ref.weight", "to_v_ref.weight"):
                sd[f"adapter_modules.{i}.{w}"] = torch.randn(hidden, hidden, generator=g) * hidden ** -0.5
    path = os.path.join(tmp, "ckpt", "IMAGDressing-v1_512.pt")
    os.makedirs(os.path.dirname(path))
    torch.save({"module": sd}, path)
    return path


def _plain(v):
    """JSON summary of a boundary value: plain values as they are, tensors by shape / dtype, generators by seed."""
    if v is None or isinstance(v, (bool, int, float, str)):
        return v
    if isinstance(v, torch.Tensor):
        return {"tensor": list(v.shape), "dtype": str(v.dtype)}
    if isinstance(v, torch.Generator):
        return {"generator_seed": v.initial_seed()}
    if isinstance(v, type):
        return {"class": v.__name__}
    return {"object": type(v).__name__}


def _dtype(m):
    return str(next(m.parameters()).dtype)


def install_recorder(monkeypatch, trace):
    """Wrap the boundary the script calls into, recording (never altering) what it asks for."""
    import transformers

    import adapter.attention_processor as ap
    import adapter.resampler as rs
    import dressing_sd.pipelines.IMAGDressing_v1_pipeline as dp
    from imagdressing_b200 import modeling, scheduler, vae

    trace.update(from_pretrained=[], resampler=None, scheduler=None)
    loaded = []  # (object, index in trace["from_pretrained"])

    for cls in (vae.AutoencoderKL, modeling.UNet2DConditionModel, transformers.CLIPTokenizer, transformers.CLIPTextModel,
                transformers.CLIPVisionModelWithProjection):
        def wrap(cls, orig):
            def from_pretrained(klass, path, *a, **kw):
                obj = orig.__func__(klass, path, *a, **kw)
                trace["from_pretrained"].append([cls.__name__, path, kw.get("subfolder")])
                loaded.append((obj, len(trace["from_pretrained"]) - 1))
                return obj
            return classmethod(from_pretrained)
        monkeypatch.setattr(cls, "from_pretrained", wrap(cls, cls.from_pretrained))

    def ctor(cls, key):
        orig = cls.__init__

        def init(self, *a, **kw):
            orig(self, *a, **kw)
            if key is None:
                object.__setattr__(self, "_trace_ctor", [list(a), kw])
            else:
                trace[key] = [list(a), {k: _plain(v) for k, v in kw.items()}]
        monkeypatch.setattr(cls, "__init__", init)

    for cls in (ap.RefSAttnProcessor2_0, ap.CAttnProcessor2_0, ap.CacheAttnProcessor2_0):
        ctor(cls, None)
    ctor(rs.Resampler, "resampler")
    ctor(scheduler.DDIMScheduler, "scheduler")

    def role(v):
        for obj, i in loaded:
            if v is obj:
                return {"from_pretrained": i, "dtype": _dtype(v) if isinstance(v, torch.nn.Module) else None}
        if isinstance(v, rs.Resampler):
            return {"resampler": True, "dtype": _dtype(v)}
        return _plain(v)

    orig_init, orig_call = dp.IMAGDressing_v1.__init__, dp.IMAGDressing_v1.__call__

    def pipe_init(self, *a, **kw):
        trace["pipeline"] = {k: role(v) for k, v in kw.items()}
        trace["processors"] = {}
        for part in ("unet", "reference_unet"):
            procs = kw[part].attn_processors
            trace["processors"][part] = {n: [type(p).__name__] + p.__dict__.get("_trace_ctor", [[], {}]) for n, p in
                                         procs.items()}
        trace["processor_dtype"] = _dtype(torch.nn.ModuleList(kw["unet"].attn_processors.values()))
        orig_init(self, *a, **kw)

    def pipe_call(self, *a, **kw):
        trace["call"] = {k: _plain(v) for k, v in kw.items()}
        return orig_call(self, *a, **kw)

    monkeypatch.setattr(dp.IMAGDressing_v1, "__init__", pipe_init)
    monkeypatch.setattr(dp.IMAGDressing_v1, "__call__", pipe_call)


def replay(trace, ckpt, cloth, out_dir):
    """inference_IMAGdressing.py:42-197 restated, every value taken from the recorded trace."""
    import transformers
    from PIL import Image
    from torchvision import transforms

    import adapter.attention_processor as ap
    from adapter.resampler import Resampler
    from dressing_sd.pipelines.IMAGDressing_v1_pipeline import IMAGDressing_v1
    from imagdressing_b200 import checkpoint, modeling, scheduler, vae

    classes = {"AutoencoderKL": vae.AutoencoderKL, "UNet2DConditionModel": modeling.UNet2DConditionModel,
               "CLIPTokenizer": transformers.CLIPTokenizer, "CLIPTextModel": transformers.CLIPTextModel,
               "CLIPVisionModelWithProjection": transformers.CLIPVisionModelWithProjection}
    dt = lambda s: getattr(torch, s.split(".")[-1])
    loaded = [classes[c].from_pretrained(p, **({"subfolder": sub} if sub else {})) for c, p, sub in trace["from_pretrained"]]
    pipe_kw = {}
    for k, r in trace["pipeline"].items():
        if "from_pretrained" in r:
            obj = loaded[r["from_pretrained"]]
            pipe_kw[k] = obj.to(dtype=dt(r["dtype"])) if r["dtype"] else obj
        elif "resampler" in r:
            a, kw = trace["resampler"]
            pipe_kw[k] = Resampler(*a, **kw).to(dtype=dt(r["dtype"]))
        elif r.get("object") == "DDIMScheduler":
            a, kw = trace["scheduler"]
            pipe_kw[k] = scheduler.DDIMScheduler(*a, **kw)
        elif "class" in r:
            pipe_kw[k] = r["class"]  # classes handed over unused (safety checker / feature extractor)
    for part in ("unet", "reference_unet"):
        pipe_kw[part].set_attn_processor({n: getattr(ap, c)(*a, **kw) for n, (c, a, kw) in trace["processors"][part].items()})
    checkpoint.processor_list(pipe_kw["unet"]).to(dtype=dt(trace["processor_dtype"]))
    checkpoint.load_module_checkpoint(ckpt, reference_unet=pipe_kw["reference_unet"], image_proj=pipe_kw["ImgProj"],
                                      unet=pipe_kw["unet"])
    pipe = IMAGDressing_v1(**pipe_kw)

    call = dict(trace["call"])
    w, h = call["width"], call["height"]
    garment = Image.open(cloth).convert("RGB")
    call["ref_image"] = transforms.Compose([transforms.Resize([h, w]), transforms.ToTensor(),
                                            transforms.Normalize([0.5], [0.5])])(garment).unsqueeze(0)
    call["ref_clip_image"] = transformers.CLIPImageProcessor()(images=garment, return_tensors="pt").pixel_values
    call["generator"] = torch.Generator().manual_seed(call["generator"]["generator_seed"])
    for k in ("ref_image", "ref_clip_image"):
        assert list(call[k].shape) == trace["call"][k]["tensor"], k
    out = pipe(**call).images
    tiles = [garment.resize((w, h), Image.BICUBIC), out[0]]
    grid = Image.new("RGB", size=(len(tiles) * w, h))
    for i, t in enumerate(tiles):
        grid.paste(t, box=(i * w, 0))
    os.makedirs(out_dir, exist_ok=True)
    grid.save(os.path.join(out_dir, os.path.basename(cloth)))


def test_unmodified_inference_script_runs_end_to_end(tmp_path, monkeypatch):
    import numpy as np
    from PIL import Image

    tmp = str(tmp_path)
    emulated_ops.install(monkeypatch)
    unet = make_hub(tmp)
    ckpt = make_checkpoint(tmp, unet)
    cloth = os.path.join(tmp, "cloth.png")
    rng = np.random.default_rng(0)
    Image.fromarray(rng.integers(0, 255, (300, 240, 3), dtype=np.uint8)).save(cloth)

    # the stand-in diffusers is opt-in: visible only inside this test
    compat = os.path.join(ROOT, "imagdressing_b200", "compat")
    monkeypatch.syspath_prepend(compat)
    monkeypatch.syspath_prepend(ROOT)
    for m in [m for m in sys.modules if m == "diffusers" or m.startswith("diffusers.")]:
        monkeypatch.delitem(sys.modules, m)
    monkeypatch.chdir(tmp)
    monkeypatch.setenv("HF_HUB_OFFLINE", "1")
    monkeypatch.setattr(sys, "argv", ["inference_IMAGdressing.py", "--cloth_path", cloth, "--model_ckpt", ckpt,
                                      "--output_path", os.path.join(tmp, "out"), "--device", "cpu"])
    seen = {}
    import imagdressing_b200.pipelines as pl

    real_run = pl._DressingPipelineBase._run

    def spy(self, **kw):  # observe (not alter) what the script asked for
        seen.update(steps=kw["num_inference_steps"], size=(kw["height"], kw["width"]), guidance=kw["guidance_scale"],
                    prompt=kw["prompt"], has_clip=kw["ref_clip_image"] is not None)
        seen["garment_unet_loaded"] = float(self.reference_unet.conv_in.weight.float().abs().sum())
        return real_run(self, **kw)

    monkeypatch.setattr(pl._DressingPipelineBase, "_run", spy)
    stored = json.load(open(TRACE)) if os.path.exists(TRACE) else None
    if SCRIPT is not None:  # the reference's own script, its boundary calls checked against the stored trace
        trace = {}
        install_recorder(monkeypatch, trace)
        try:
            runpy.run_path(SCRIPT, run_name="__main__")
        finally:
            for m in [m for m in sys.modules if m == "diffusers" or m.startswith("diffusers.")]:
                sys.modules.pop(m, None)
        trace = json.loads(json.dumps(trace))  # tuples -> lists, as stored
        if os.environ.get("IMAGD_WRITE_TRACE") == "1":
            json.dump(trace, open(TRACE, "w"), indent=1, sort_keys=True)
        assert trace == stored
    else:  # no reference checkout: the recorded script replayed through the same boundary
        replay(stored, ckpt, cloth, os.path.join(tmp, "out"))
    out = os.path.join(tmp, "out", "cloth.png")
    assert os.path.exists(out)
    grid = Image.open(out)
    assert grid.size == (1024, 640)  # [resized garment | generated 512x640 image]
    arr = np.asarray(grid)[:, 512:]
    assert arr.std() > 1.0  # a real decoded image, not a constant
    assert seen == dict(steps=50, size=(640, 512), guidance=7.5, prompt="A beautiful woman, best quality, high quality",
                        has_clip=True, garment_unet_loaded=seen["garment_unet_loaded"])
    # the garment UNet really carries the checkpoint's `ref_unet.` weights (seed 1), not the base UNet's (seed 0)
    from imagdressing_b200 import modeling

    ref = modeling.UNet2DConditionModel(**UNET_CFG)
    modeling.init_synthetic_(ref, 1)
    want = float(ref.conv_in.weight.half().float().abs().sum())
    assert abs(seen["garment_unet_loaded"] - want) < 1e-3 * want
