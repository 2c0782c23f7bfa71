"""The denoising loop of IMAGDressing-v1, batched and CUDA-graph replayed.

Reference loop body: dressing_sd/pipelines/IMAGDressing_v1_pipeline.py:463-541 (variants
IMAGDressing_v1_pipeline_ipa_controlnet.py:595-736, IMAGDressing_v1_pipeline_controlnet_inpainting.py:387-517):
  garment pass once (ref-UNet at t=0, feature taps)  ->  per step: [ControlNet] -> UNet(cond, garment stream)
  -> UNet(uncond, plain) -> CFG -> DDIM step [-> inpaint blend].

Differences that do not change per-sample results (SURVEY.md Appendix B): the two batch-1 UNet calls run as one
CFG batch [cond.., uncond..] whose first n samples carry the garment stream (B1/B4); the garment pass runs at
batch n on the garment tokens only (B2); only the 16 attn1 taps are kept (B3); one captured CUDA graph is
replayed for all steps — the step index lives in device memory and the fused CFG+DDIM kernel (or, for the
multistep samplers of samplers.py, the generic CFG+sampler-step kernel or UniPC's predictor-corrector kernel)
advances it.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import torch

from . import _lib, ops
from .scheduler import DDIMScheduler


class DenoiseEngine:
    def __init__(self, unet, reference_unet=None, controlnet=None, scheduler: Optional[DDIMScheduler] = None,
                 use_cuda_graph: bool = True):
        self.unet = unet
        self.reference_unet = reference_unet
        self.controlnet = controlnet
        self.scheduler = scheduler
        self.use_cuda_graph = use_cuda_graph
        self._states = {}
        self._garment = None
        self._dummy = {}
        self._zero_t = None

    def _nets(self) -> list:
        """The ControlNets this engine drives: the `nets` of a MultiControlNetModel, a single ControlNetModel, or none."""
        from .modeling import MultiControlNetModel

        if self.controlnet is None:
            return []
        return list(self.controlnet.nets) if isinstance(self.controlnet, MultiControlNetModel) else [self.controlnet]

    # ------------------------------------------------------------------ garment pass
    @torch.no_grad()
    def garment_features(self, ref_latents: torch.Tensor, garment_tokens: torch.Tensor) -> Dict[str, torch.Tensor]:
        """ref-UNet forward at t = 0 with the garment tokens in the text slot; returns the attn1 processor inputs
        (post-LayerNorm hidden states) keyed by processor name (IMAGDressing_v1_pipeline.py:465-479)."""
        ru = self.reference_unet
        dev = ref_latents.device

        def collect():
            return {name: proc.cache["hidden_states"] for name, proc in ru.attn_processors.items() if "attn1" in name}

        def run(lat, tok):
            ru.forward_tokens(lat, self._zero_t, tok)

        if getattr(self, "_zero_t", None) is None or self._zero_t.device != dev:
            self._zero_t = torch.zeros(1, device=dev, dtype=torch.float32)
        if not (self.use_cuda_graph and dev.type == "cuda"):  # (graphs need a CUDA device; the kernels raise without one)
            run(ref_latents.float().contiguous(), garment_tokens)
            return collect()
        key = (tuple(ref_latents.shape), tuple(garment_tokens.shape))
        g = self._garment
        if g is None or g["key"] != key:
            # first call for this shape: eager (packs weights, sizes workspaces), then capture the pass once;
            # its feature taps are tensors of the graph's pool, so their addresses are stable across images
            g = dict(key=key, lat=ref_latents.float().contiguous().clone(),
                     tok=garment_tokens.to(torch.bfloat16).contiguous().clone())
            run(g["lat"], g["tok"])
            for proc in ru.attn_processors.values():  # the token K|V projection must be IN the graph: force a miss
                if hasattr(proc, "invalidate_packed"):
                    proc.invalidate_packed()
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            before = _lib.launch_count
            with torch.cuda.graph(graph):
                run(g["lat"], g["tok"])
            g["launches"] = _lib.launch_count - before
            _lib.launch_count = before
            g["graph"], g["sa"] = graph, collect()
            self._garment = g
        g["lat"].copy_(ref_latents)
        g["tok"].copy_(garment_tokens)
        g["graph"].replay()
        _lib.launch_count += g["launches"]
        return g["sa"]

    # ------------------------------------------------------------------ what a captured step graph froze
    def _frozen_signature(self) -> tuple:
        """Everything a captured step graph bakes in besides shapes: the processors' mutable scales (`scale` is a host
        float in the kernel's KV-stream struct, `lora_scale` selects the merged q/out weights) and the identity +
        in-place version of every weight (packed / LoRA-merged copies are separate device buffers). A second call
        with a different `image_scale` / `ipa_scale` / `s_lora_scale` / `c_lora_scale`, or after a
        `load_state_dict`, must not replay the old graph (ADVICE r1, high)."""
        sig = []
        for model in (self.unet, *self._nets()):
            for name, proc in model.attn_processors.items():
                sig.append((getattr(proc, "scale", None), getattr(proc, "lora_scale", None)))
            sig.append(sum(p._version for p in model.parameters()))
            sig.append(next(model.parameters()).data_ptr())  # .to() / re-assignment
        return tuple(sig)

    # ------------------------------------------------------------------ one step
    def _step(self, st, use_control: bool = True, active: tuple = ()):
        """One step. A single ControlNetModel runs when use_control is set; the nets of a MultiControlNetModel run when
        their index is in `active`, chained in net order, their zero convs scaled by row step_ptr[0] of st["cn_scale"]."""
        n = st["n"]
        lat = st["latents"]
        table = (st["t_table"], st["step_ptr"])
        down = mid = None
        if "cn_scale" in st:
            nets, res = self._nets(), None
            for k in active:
                res = nets[k](lat, None, st["control_text"], st["control_cond"][k], return_dict=False,
                              timestep_table=table, sample_repeat=2, input_scale=st.get("scale"),
                              scale_table=st["cn_scale"][:, k], scale_step=st["step_ptr"], residuals=res)
            if res is not None:
                down, mid = res
        elif use_control and self.controlnet is not None and st.get("control_cond") is not None:
            down, mid = self.controlnet(lat, None, st["control_text"], st["control_cond"],
                                        conditioning_scale=st["control_scale"], return_dict=False,
                                        timestep_table=table, sample_repeat=2, input_scale=st.get("scale"))
        eps = self.unet.forward_tokens(lat, None, st["text"], st["kwargs"], down, mid, timestep_table=table,
                                       out=st["eps"], sample_repeat=2, input_scale=st.get("scale"),
                                       adapter_res=st.get("adapter"), adapter_scale=st.get("adapter_scale"))
        if st["ddim"]:
            ops.cfg_ddim_step(eps[:n], eps[n:], st["guidance"], lat, st["coef"], st["step_ptr"], mask=st.get("mask"),
                              image_latents=st.get("image_latents"), noise=st.get("noise"), blend_coef=st.get("blend"))
        elif "bank" in st:
            ops.cfg_sampler_pc_step(eps[:n], eps[n:], st["guidance"], lat, st["coef"], st["step_ptr"], st["bank"],
                                    mask=st.get("mask"), image_latents=st.get("image_latents"), noise=st.get("noise"),
                                    blend_coef=st.get("blend"))
        else:
            ops.cfg_sampler_step(eps[:n], eps[n:], st["guidance"], lat, st["coef"], st["step_ptr"],
                                 history=st.get("history"), step_noise=st.get("step_noise"), mask=st.get("mask"),
                                 image_latents=st.get("image_latents"), noise=st.get("noise"),
                                 blend_coef=st.get("blend"))

    def _refresh(self, st) -> bool:
        """Per-image refresh of the step-invariant projections without running a step. Returns False when a
        processor outside this package is installed (then the caller runs a full eager step instead)."""
        from .modeling import Attention

        n = st["n"]
        jobs = [(self.unet, st["text"], st["kwargs"])]
        if self.controlnet is not None and st.get("control_cond") is not None:
            jobs += [(net, st["control_text"], {}) for net in self._nets()]
        for model, _, _ in jobs:
            for m in model.modules():
                if isinstance(m, Attention) and not hasattr(m.processor, "_kv2_memo"):
                    return False
        for model, text, kw in jobs:
            for m in model.modules():
                if isinstance(m, Attention):
                    proc = m.processor
                    proc._kv2_memo.clear()  # garment taps are rewritten by a graph replay: identity says nothing
                    dummy = self._dummy.get(m.query_dim)
                    if dummy is None or dummy.shape[0] != 2 * n:
                        dummy = self._dummy[m.query_dim] = torch.empty(2 * n, 1, m.query_dim, device=text.device,
                                                                       dtype=torch.bfloat16)
                    proc(m, dummy, encoder_hidden_states=text if m.is_cross else None, _prepare_only=True, **kw)
        if len(jobs) > 1:
            conds = st["control_cond"] if "cn_scale" in st else [st["control_cond"]]
            for net, cond in zip(self._nets(), conds):
                net.cond_embedding(cond, 2 * n)
        return True

    # ------------------------------------------------------------------ sampling
    @torch.no_grad()
    def sample(self, latents: torch.Tensor, prompt_embeds: torch.Tensor, negative_prompt_embeds: torch.Tensor,
               sa_hidden_states: Optional[Dict[str, torch.Tensor]], guidance_scale: float, num_inference_steps: int,
               *, timesteps: Optional[torch.Tensor] = None, control_cond: Optional[torch.Tensor] = None,
               control_prompt_embeds: Optional[torch.Tensor] = None, control_negative_embeds: Optional[torch.Tensor] = None,
               control_scale: float = 1.0, mask: Optional[torch.Tensor] = None,
               image_latents: Optional[torch.Tensor] = None, noise: Optional[torch.Tensor] = None,
               callback=None, control_keep: Optional[List[float]] = None, scheduler=None,
               step_noise: Optional[torch.Tensor] = None, adapter_states: Optional[List[torch.Tensor]] = None,
               adapter_conditioning_scale: float = 1.0) -> torch.Tensor:
        """latents [n,4,h,w] (already scaled by the scheduler's init_noise_sigma); embeds [n,T,768] (or [1,T,768],
        broadcast). control_keep: per-step 0/1 ControlNet guidance window (`controlnet_keep` of
        IMAGDressing_v1_pipeline_ipa_controlnet.py:584-590,643-649); steps with 0 run the UNet without residuals (what
        a zero conditioning scale computes) from a second captured graph. scheduler: the sampler to run (default: the
        one given at construction); DDIMScheduler runs the fused CFG+DDIM kernel, the multistep samplers
        (samplers.py) the generic sampler-step kernel, UniPC the predictor-corrector kernel over a resident slot
        bank. step_noise: [S,n,4,h,w], one noise draw per step, for samplers
        that add noise (Euler-ancestral). adapter_states: the four T2I-Adapter features of this call (token-major bf16
        [1 or n, h, w, C], or NCHW), added to both CFG halves at every step times adapter_conditioning_scale; the scale
        lives in device memory, so changing it replays the same graph. Returns the final latents as a new fp32 tensor.

        With a MultiControlNetModel of K nets, control_cond is a list of K images (batch 1 or n each), control_scale a
        list of K floats and control_keep None or a list of K per-step 0/1 lists. The scales times the keeps are staged
        into a resident [S, K] table that the zero convs read on the device, so new scales replay the same graphs. Steps
        are grouped by their active set (the nets kept at that step); each distinct set has its own step graph, captured
        on first use into the memory pool of the first one, which runs only those nets, chained in net order."""
        dev = latents.device
        n = latents.shape[0]
        sch = scheduler if scheduler is not None else self.scheduler
        if timesteps is None:
            sch.set_timesteps(num_inference_steps, device=dev)
            timesteps = sch.timesteps
        ddim = isinstance(sch, DDIMScheduler)
        if ddim:
            t_table, coef, blend = sch.step_tables(dev, timesteps)
            tables = None
        else:
            tables = sch.sampler_tables(dev, timesteps)
            t_table, coef, blend = tables.t, tables.coef, tables.blend
            if tables.noise and (step_noise is None or tuple(step_noise.shape) != (t_table.numel(), *latents.shape)):
                raise ValueError(f"{type(sch).__name__} needs step_noise of shape [steps, *latents.shape]")
        S = t_table.numel()

        def bn(t):
            return t if t.shape[0] == n else t.expand(n, -1, -1)

        has_control = self.controlnet is not None and control_cond is not None
        from .modeling import MultiControlNetModel

        multi = has_control and isinstance(self.controlnet, MultiControlNetModel)
        if multi:
            K = len(self.controlnet.nets)
            control_cond, control_scale = list(control_cond), [float(s) for s in control_scale]
            keeps = [[1.0] * S] * K if control_keep is None else [[float(k) for k in kk] for kk in control_keep]
            if len(control_cond) != K or len(control_scale) != K or len(keeps) != K:
                raise ValueError(f"{len(control_cond)} images, {len(control_scale)} scales and {len(keeps)} guidance "
                                 f"windows for {K} ControlNets")
            if any(len(kk) != S or any(k not in (0.0, 1.0) for k in kk) for kk in keeps):
                raise ValueError("control_keep must hold one 0/1 entry per step for each ControlNet")
            active = [tuple(k for k in range(K) if keeps[k][i] > 0) for i in range(S)]
        if adapter_states is not None:
            adapter_states = self.unet.adapter_tokens(adapter_states, latents.shape[-2:])
            if any(f.shape[0] not in (1, n) for f in adapter_states):
                raise ValueError(f"adapter features must hold 1 or {n} samples")
        cond_shape = None
        if has_control:
            cond_shape = tuple(tuple(c.shape) for c in control_cond) if multi else tuple(control_cond.shape)
        key = (n, tuple(latents.shape[1:]), prompt_embeds.shape[1], has_control, mask is not None,
               float(guidance_scale), None if multi else float(control_scale), bool(sa_hidden_states), id(t_table),
               id(coef), cond_shape, self._frozen_signature(),
               tuple(tuple(f.shape) for f in adapter_states) if adapter_states is not None else None)
        keep = [1.0] * S if control_keep is None or not has_control or multi else [float(k) for k in control_keep]
        if len(keep) != S or any(k not in (0.0, 1.0) for k in keep):
            raise ValueError("control_keep must hold one 0/1 entry per step")
        st = self._states.get(key)
        if st is None:
            f32 = dict(device=dev, dtype=torch.float32)
            st = dict(n=n, latents=torch.empty(n, *latents.shape[1:], **f32), lat0=torch.empty(n, *latents.shape[1:], **f32),
                      text=torch.empty(2 * n, prompt_embeds.shape[1], prompt_embeds.shape[2], device=dev, dtype=torch.bfloat16),
                      guidance=float(guidance_scale), coef=coef, t_table=t_table,
                      step_ptr=torch.zeros(2, dtype=torch.int32, device=dev),
                      eps=torch.empty(2 * n, *latents.shape[1:], **f32), kwargs={}, graph=None, graph_nc=None,
                      ddim=ddim)
            if tables is not None:  # (the key holds id(coef) of these live tables: no other sampler replays this graph)
                st.update(scale=tables.scale)
                if tables.history:
                    st.update(history=torch.empty(n, *latents.shape[1:], **f32))
                if tables.noise:
                    st.update(step_noise=torch.empty(S, n, *latents.shape[1:], **f32))
                if tables.predictor_corrector:  # one bank for both step graphs; a row reads only slots written before
                    st.update(bank=torch.empty(ops.PC_SLOTS, n, *latents.shape[1:], **f32))
            if has_control:
                cp = control_prompt_embeds if control_prompt_embeds is not None else prompt_embeds
                st.update(control_text=torch.empty(2 * n, cp.shape[1], cp.shape[2], device=dev, dtype=torch.bfloat16))
                if multi:  # graphs: active set -> (graph, launches); pool: the first capture's memory pool
                    st.update(control_cond=[torch.empty(c.shape, **f32) for c in control_cond],
                              cn_scale=torch.empty(S, K, **f32), graphs={}, pool=None)
                else:
                    st.update(control_cond=torch.empty(control_cond.shape, **f32), control_scale=float(control_scale))
            if mask is not None:
                st.update(mask=torch.empty(mask.shape, **f32), image_latents=torch.empty(image_latents.shape, **f32),
                          noise=torch.empty(noise.shape, **f32), blend=blend)
            if adapter_states is not None:
                st.update(adapter=[torch.empty_like(f) for f in adapter_states], adapter_scale=torch.empty(1, **f32))
            self._states = {key: st}  # one resident configuration (its graph holds the activation pool)
        # ---- stage this call's inputs into the persistent buffers (addresses stay fixed for the captured graph)
        lat = st["latents"]
        st["lat0"].copy_(latents)
        lat.copy_(st["lat0"])
        st["text"][:n].copy_(bn(prompt_embeds))
        st["text"][n:].copy_(bn(negative_prompt_embeds))
        st["kwargs"] = {"sa_hidden_states": sa_hidden_states, "ref_samples": n} if sa_hidden_states else {}
        if has_control:
            cp = control_prompt_embeds if control_prompt_embeds is not None else prompt_embeds
            cn = control_negative_embeds if control_negative_embeds is not None else negative_prompt_embeds
            if multi:
                for buf, c in zip(st["control_cond"], control_cond):
                    buf.copy_(c)
                st["cn_scale"].copy_(torch.tensor([[control_scale[k] * keeps[k][i] for k in range(K)] for i in range(S)],
                                                  dtype=torch.float32))
            else:
                st["control_cond"].copy_(control_cond)
            st["control_text"][:n].copy_(bn(cp))
            st["control_text"][n:].copy_(bn(cn))
        if mask is not None:
            st["mask"].copy_(mask)
            st["image_latents"].copy_(image_latents)
            st["noise"].copy_(noise)
        if "step_noise" in st:
            st["step_noise"].copy_(step_noise)
        if adapter_states is not None:
            for buf, f in zip(st["adapter"], adapter_states):
                buf.copy_(f)
            st["adapter_scale"].fill_(float(adapter_conditioning_scale))
        st["step_ptr"].zero_()
        if sa_hidden_states:
            # the garment taps are rewritten in place by the captured garment pass: tensor identity/version say
            # nothing about their contents, so the cached garment K|V projections are always recomputed per image
            from .modeling import Attention

            for m in self.unet.modules():
                if isinstance(m, Attention) and hasattr(m.processor, "_kv2_memo"):
                    m.processor._kv2_memo.clear()

        if not (self.use_cuda_graph and dev.type == "cuda") or callback is not None:
            for i in range(S):
                self._step(st, use_control=keep[i] > 0, active=active[i] if multi else ())
                if callback is not None:
                    callback(i, int(timesteps[i]), lat)
            return lat.clone()

        # Refresh everything that is per-image but step-invariant (text and garment K/V projections, ControlNet
        # conditioning embedding) — recomputed IN PLACE, so the device addresses the captured graph holds stay
        # valid. The first call for a configuration runs one full eager step instead (packs weights, sizes
        # workspaces) and then captures the step graph, which is replayed for every step of every later image.
        if multi:
            return self._sample_multi(st, active)
        if st["graph"] is None or not self._refresh(st):
            self._step(st)
            lat.copy_(st["lat0"])
            st["step_ptr"].zero_()
        if st["graph"] is None:
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            before = _lib.launch_count
            with torch.cuda.graph(graph):
                self._step(st)
            st["graph_launches"] = _lib.launch_count - before
            _lib.launch_count = before  # capture launched nothing
            st["graph"] = graph
        if min(keep) == 0.0 and st["graph_nc"] is None:  # steps outside the ControlNet window: no-residual graph
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            before = _lib.launch_count
            with torch.cuda.graph(graph):
                self._step(st, use_control=False)
            st["graph_nc_launches"] = _lib.launch_count - before
            _lib.launch_count = before
            st["graph_nc"] = graph
        for i in range(S):
            if keep[i] > 0:
                st["graph"].replay()
                _lib.launch_count += st["graph_launches"]
            else:
                st["graph_nc"].replay()
                _lib.launch_count += st["graph_nc_launches"]
        return lat.clone()

    def _sample_multi(self, st, active: List[tuple]) -> torch.Tensor:
        """The graph-replayed loop of a MultiControlNetModel: one step graph per distinct active set."""
        lat = st["latents"]
        graphs = st["graphs"]
        if not graphs or not self._refresh(st):
            self._step(st, active=tuple(range(len(self._nets()))))  # every net: packs weights, sizes workspaces
            lat.copy_(st["lat0"])
            st["step_ptr"].zero_()
        for a in dict.fromkeys(active):  # distinct active sets, in order of first use
            if a in graphs:
                continue
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            before = _lib.launch_count
            with torch.cuda.graph(graph, pool=st["pool"]):  # the sets' steps never overlap: one activation pool
                self._step(st, active=a)
            graphs[a] = (graph, _lib.launch_count - before)
            _lib.launch_count = before
            if st["pool"] is None:
                st["pool"] = graph.pool()
        for a in active:
            graph, launches = graphs[a]
            graph.replay()
            _lib.launch_count += launches
        return lat.clone()
