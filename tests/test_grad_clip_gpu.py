"""GPU: global-norm gradient clipping on the kernels (imagd_grad_norm_clip, imagd_adamw_step_clip; FlatAdamW(max_grad_norm=)).

- the norm pass against torch.linalg.vector_norm in fp64 at ragged sizes, one element and the real trainable-buffer size of
  SDModel; bit-identical reruns; Inf / NaN at the first, a middle and the last element detected (step count held, skip
  count advanced); values near the bf16 maximum give a finite norm;
- the clipped AdamW: coef == 1 is bitwise imagd_adamw_step_dev, coef < 1 is bitwise imagd_adamw_step_dev at the product
  scale, a non-finite state leaves every buffer bitwise untouched;
- the real training step with clipping engaged tracks clip_grad_norm_ + torch AdamW on the fp32 oracle, and the captured
  step graph with clipping equals the eager clipped step."""
import pytest
import torch

from test_train_step_gpu import batch, build, rel

pytestmark = pytest.mark.gpu
BF = torch.bfloat16


def _trainable_elements() -> int:
    """Length of FlatAdamW's flat buffer over SDModel's trainable set (Resampler + garment UNet + adapter modules,
    train.py:368-379), counted on the meta device."""
    from adapter.attention_processor import CAttnProcessor2_0, RefSAttnProcessor2_0
    from adapter.resampler import Resampler
    from imagdressing_b200 import modeling, train

    with torch.device("meta"):
        ref = modeling.UNet2DConditionModel()
        proj = Resampler(dim=768, depth=4, dim_head=64, heads=12, num_queries=16, embedding_dim=1280, output_dim=768, ff_mult=4)
        boc = ref.config.block_out_channels
        ad = [RefSAttnProcessor2_0(n, train.hidden_size_of(n, boc)) if n.endswith("attn1.processor")
              else CAttnProcessor2_0(n, train.hidden_size_of(n, boc), ref.config.cross_attention_dim)
              for n in ref.attn_processors.keys()]
    params = [*proj.parameters(), *ref.parameters(), *[p for a in ad for p in a.parameters()]]
    return sum((p.numel() + 7) // 8 * 8 for p in params)


def _norm64(g: torch.Tensor) -> float:
    return float(sum(torch.linalg.vector_norm(c.double()) ** 2 for c in g.split(1 << 26)) ** 0.5)


class _Pass:
    """One norm pass's device state, as FlatAdamW holds it."""

    def __init__(self, n, dev, scale=1.0):
        from imagdressing_b200 import ops

        self.hyper = torch.tensor([1e-4, 1e-2, 0.0, scale], device=dev, dtype=torch.float32)
        self.state = torch.zeros(4, device=dev, dtype=torch.float64)
        self.ws = torch.zeros(ops.grad_norm_ws_bytes(n), device=dev, dtype=torch.uint8)

    def __call__(self, g, max_norm=1.0):
        from imagdressing_b200 import ops

        ops.grad_norm_clip(g, self.hyper, self.state, self.ws, max_norm=max_norm)
        torch.cuda.synchronize()
        return [float(v) for v in self.state.cpu()], float(self.hyper[2])


@pytest.mark.parametrize("n", [1, 7, 9, 8192 * 5 + 3, 1_000_003, "model"])
def test_grad_norm_matches_fp64(cuda_device, n):
    dev = cuda_device
    n = _trainable_elements() if n == "model" else n
    g = (torch.randn(n, device=dev) * 1e-3).to(BF)
    want = _norm64(g)
    p = _Pass(n, dev, scale=0.25)
    (norm, coef, finite, skipped), step = p(g, max_norm=1e-5)
    print(f"n={n}: norm {norm:.9e} fp64 reference {0.25 * want:.9e}")
    assert finite == 1.0 and skipped == 0.0 and step == 1.0
    assert abs(norm - 0.25 * want) <= 1e-5 * 0.25 * want
    f32max = float(torch.tensor(1e-5, dtype=torch.float32))
    assert coef == pytest.approx(min(1.0, f32max / (norm + 1e-6)), rel=1e-12)
    first = p.state.clone()
    (norm2, coef2, _, _), step = p(g, max_norm=1e-5)  # the arrival counter was reset: the pass replays
    assert step == 2.0 and torch.equal(p.state, first)  # bit-identical rerun
    (_, coef3, _, _), _ = p(g, max_norm=1e3)
    assert coef3 == 1.0


@pytest.mark.parametrize("bad", [float("nan"), float("inf"), float("-inf")])
def test_grad_norm_detects_non_finite(cuda_device, bad):
    dev = cuda_device
    n = 1_000_003
    g = torch.randn(n, device=dev).to(BF)
    p = _Pass(n, dev)
    skipped = 0
    for pos in (0, n // 2 + 5, n - 1):
        h = g.clone()
        h[pos] = bad
        (norm, coef, finite, sk), step = p(h)
        skipped += 1
        assert finite == 0.0 and sk == skipped and step == 0.0, (pos, norm)
    (norm, _, finite, sk), step = p(g)
    assert finite == 1.0 and sk == 3 and step == 1.0 and norm == pytest.approx(_norm64(g), rel=1e-5)


def test_grad_norm_near_bf16_max_is_finite(cuda_device):
    dev = cuda_device
    n = 4099
    g = torch.full((n,), 3.0e38, device=dev).to(BF)  # squares ~1e77: far beyond fp32, well inside fp64
    g[::3] = -g[::3]
    assert torch.isfinite(g).all()
    (norm, coef, finite, _), step = _Pass(n, dev)(g)
    want = _norm64(g)
    assert finite == 1.0 and step == 1.0 and norm > 1e40
    assert abs(norm - want) <= 1e-5 * want and 0.0 < coef < 1e-39


def _adam_buffers(n, dev, seed):
    gen = torch.Generator(device=dev).manual_seed(seed)
    r = lambda: torch.randn(n, device=dev, generator=gen)
    master = r()
    return dict(master=master, param=master.to(BF), grad=r().to(BF), m=r() * 1e-2, v=r().abs() * 1e-4)


@pytest.mark.parametrize("n", [1_000_003, 4096])
def test_adamw_clip_against_adamw_dev(cuda_device, n):
    from imagdressing_b200 import ops

    dev = cuda_device
    hp = dict(beta1=0.9, beta2=0.999, eps=1e-8)
    hyper = torch.tensor([1e-3, 1e-2, 3.0, 0.5], device=dev, dtype=torch.float32)
    for coef in (1.0, 0.3):
        a, b = _adam_buffers(n, dev, 1), _adam_buffers(n, dev, 1)
        state = torch.tensor([7.0, coef, 1.0, 0.0], device=dev, dtype=torch.float64)
        ops.adamw_step_clip(*a.values(), hyper, state, **hp)
        scaled = hyper.clone()
        scaled[3] = hyper[3] * torch.tensor(coef, dtype=torch.float32, device=dev)  # the kernel's fp32 product
        ops.adamw_step_dev(*b.values(), scaled, **hp)
        for k in ("master", "param", "m", "v"):
            assert torch.equal(a[k], b[k]), (coef, k)
        assert not torch.equal(a["master"], _adam_buffers(n, dev, 1)["master"])
    # a non-finite gradient: nothing moves
    a, ref = _adam_buffers(n, dev, 2), _adam_buffers(n, dev, 2)
    state = torch.tensor([float("inf"), 0.0, 0.0, 1.0], device=dev, dtype=torch.float64)
    ops.adamw_step_clip(*a.values(), hyper, state, **hp)
    torch.cuda.synchronize()
    for k in ("master", "param", "m", "v"):
        assert torch.equal(a[k], ref[k]), k


def _oracle_step(o_unet, o_ref, o_proj, o_params, o_opt, b, max_norm_frac, max_norm=None):
    """One step of the oracle in the mixed-precision regime of test_adamw_steps_track_the_oracle_trajectory (fp32 master
    weights, forward / backward on their bf16-rounded values), clipped with clip_grad_norm_ -> (loss, pre-clip norm)."""
    from oracle import train_step as ts
    from oracle.ddim import DDIMOracle

    o_opt.zero_grad(set_to_none=True)
    master = [p.detach().clone() for p in o_params]
    with torch.no_grad():
        for p in o_params:
            p.copy_(p.to(BF).float())
    loss = float(ts.train_step(o_unet, o_ref, o_proj, DDIMOracle(), **b))
    with torch.no_grad():
        for p, m in zip(o_params, master):
            p.copy_(m)
    norm = float(torch.linalg.vector_norm(torch.stack([p.grad.norm() for p in o_params if p.grad is not None])))
    if max_norm is None:
        max_norm = max_norm_frac * norm
    torch.nn.utils.clip_grad_norm_(o_params, max_norm)
    o_opt.step()
    return loss, norm, max_norm


def test_clipped_steps_track_the_oracle_trajectory(cuda_device):
    """test_adamw_steps_track_the_oracle_trajectory with clipping engaged on every step: max_grad_norm is half the oracle's
    first gradient norm; the oracle clips with torch.nn.utils.clip_grad_norm_ before torch AdamW."""
    from imagdressing_b200 import train
    from imagdressing_b200.scheduler import DDIMScheduler
    from oracle import train_step as ts

    dev = cuda_device
    (o_unet, o_ref, o_proj, o_ad), (p_unet, p_ref, p_proj, p_ad) = build(dev)
    b = batch(dev, 2, 16, 16)
    hp = dict(lr=2e-5, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2)
    o_params = ts.set_trainable(o_unet, o_ref, o_proj, o_ad)
    o_opt = torch.optim.AdamW(o_params, **hp)
    sd = train.SDModel(p_unet, p_ref, p_proj, p_ad)
    sched = DDIMScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False)
    lo, lp, no, np_ = [], [], [], []
    max_norm, p_opt = None, None
    for _ in range(3):
        loss, norm, max_norm = _oracle_step(o_unet, o_ref, o_proj, o_params, o_opt, b, 0.5, max_norm)
        lo.append(loss)
        no.append(norm)
        if p_opt is None:
            p_opt = train.FlatAdamW(train.set_trainable(p_unet, p_ref, p_proj, p_ad), max_grad_norm=max_norm, **hp)
        lp.append(float(train.train_step(sd, sched, optimizer=p_opt, **b)))
        np_.append(float(p_opt.last_grad_norm))
    print(f"max_grad_norm {max_norm:.5g}; pre-clip norms: oracle {[round(v, 5) for v in no]} | kernels "
          f"{[round(v, 5) for v in np_]}; losses: oracle {[round(v, 5) for v in lo]} | kernels {[round(v, 5) for v in lp]}")
    assert p_opt.t == 3 and float(p_opt.skipped_steps) == 0
    for a, g in zip(no, np_):
        assert g > max_norm and a > max_norm  # engaged on both sides, every step
        assert abs(a - g) < 5e-2 * a
    for a, g in zip(lo, lp):
        assert abs(a - g) < 2e-2 * abs(a)
    assert rel(p_ref.conv_in.weight, o_ref.conv_in.weight.to(BF)) < 2e-3


def test_graphed_clipped_step_equals_eager_clipped_step(cuda_device):
    """test_graphed_step_equals_eager_step with max_grad_norm engaged: the norm pass is captured with the rest of the step."""
    from imagdressing_b200 import train
    from imagdressing_b200.scheduler import DDIMScheduler
    from oracle import train_step as ts

    dev = cuda_device
    (o_unet, o_ref, o_proj, o_ad), (p_unet, p_ref, p_proj, p_ad) = build(dev)
    b1, b2 = batch(dev, 2, 16, 16), batch(dev, 2, 16, 16)
    b2 = {k: (v.flip(0) if k != "timesteps" else torch.tensor([300, 650], device=dev)) for k, v in b2.items()}
    # a limit below both batches' norms, from the oracle (separate parameters: no eager backward of the graphed ones)
    o_params = ts.set_trainable(o_unet, o_ref, o_proj, o_ad)
    o_opt = torch.optim.SGD(o_params, lr=0.0)
    max_norm = 0.2 * min(_oracle_step(o_unet, o_ref, o_proj, o_params, o_opt, bb, 1.0)[1] for bb in (b1, b2))
    del o_unet, o_ref, o_proj, o_ad, o_params, o_opt

    sd = train.SDModel(p_unet, p_ref, p_proj, p_ad)
    opt = train.FlatAdamW(train.set_trainable(p_unet, p_ref, p_proj, p_ad), lr=2e-5, weight_decay=1e-2, max_grad_norm=max_norm)
    sched = DDIMScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False)
    start = (opt.param.clone(), opt.master.clone())
    step = train.GraphedTrainStep(sd, sched, opt, b1)
    assert torch.equal(opt.param, start[0]) and opt.t == 0 and float(opt.last_grad_norm) == 0.0
    graphed, g_norms = [], []
    for b in (b1, b2):
        graphed.append(float(step(**b)))
        g_norms.append(float(opt.last_grad_norm))
    assert opt.t == 2 and float(opt.skipped_steps) == 0
    after_graphed = opt.param.clone()
    with torch.no_grad():
        opt.param.copy_(start[0])
        opt.master.copy_(start[1])
    opt.reset_state()
    eager, e_norms = [], []
    for b in (b1, b2):
        eager.append(float(train.train_step(sd, sched, optimizer=opt, **b)))
        e_norms.append(float(opt.last_grad_norm))
    print(f"max_grad_norm {max_norm:.5g}; eager losses {eager} norms {e_norms} | graphed losses {graphed} norms {g_norms}")
    assert opt.t == 2
    for a, g in zip(eager, graphed):
        assert abs(a - g) <= 1e-5 * abs(a)
    for a, g in zip(e_norms, g_norms):
        assert g > max_norm and abs(a - g) <= 1e-4 * a
    assert rel(after_graphed, opt.param) < 1e-4
