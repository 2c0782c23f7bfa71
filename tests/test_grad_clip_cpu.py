"""CPU: global-norm gradient clipping in FlatAdamW (max_grad_norm; the reference's DeepSpeed "gradient_clipping": 1.0) with its
two kernels emulated in torch: the norm pass (ops.grad_norm_clip) and the update that reads its state (ops.adamw_step_clip).

- clipped steps == torch.nn.utils.clip_grad_norm_ + torch.optim.AdamW on fp32 copies, with clipping engaged on every step;
- accumulation k = 2 == the whole-batch clipped step;
- gloo world 2, plain and shard_states: ranks bit-identical, and equal to the single-process whole-batch clipped step;
- a non-finite gradient skips the update (weights, moments, step count untouched; skipped_steps + 1) and the next finite
  step proceeds as if it had never happened; state_dict round trip across a skipped step."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import emulated_ops

BF = torch.bfloat16
MAX = 0.05  # below every gradient norm of these toy problems: clipping is engaged on every compared step
HP = dict(lr=1e-2, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.1)


def _grad_norm_ws_bytes(n):
    return 16


def _grad_norm_clip(grad, hyper, state, ws, *, max_norm):
    """imagd_grad_norm_clip: fp64 sum of squares, norm of hyper[3] * grad, coef, finite flag, step / skip counts."""
    s = float(grad.double().square().sum())
    finite = s == s and s != float("inf")
    norm = s ** 0.5 * float(hyper[3])
    max_norm = float(torch.tensor(max_norm, dtype=torch.float32))  # the kernel takes it as a float
    state[0] = norm
    state[1] = min(1.0, max_norm / (norm + 1e-6)) if finite else 0.0
    state[2] = 1.0 if finite else 0.0
    if finite:
        hyper[2:3].add_(1.0)
    else:
        state[3] += 1.0


def _adamw_step_clip(master, param, grad, m, v, hyper, clip_state, *, beta1, beta2, eps):
    """imagd_adamw_step_clip: nothing on a non-finite gradient, else the update with scale hyper[3] * (float)coef."""
    if float(clip_state[2]) == 0.0:
        return
    scale = float(hyper[3] * clip_state[1].float())
    emulated_ops.adamw_step(master, param, grad, m, v, lr=float(hyper[0]), beta1=beta1, beta2=beta2, eps=eps,
                            weight_decay=float(hyper[1]), step=int(round(float(hyper[2]))), grad_scale=scale)


CLIP_OPS = {"grad_norm_ws_bytes": _grad_norm_ws_bytes, "grad_norm_clip": _grad_norm_clip, "adamw_step_clip": _adamw_step_clip,
            "adamw_step_dev": emulated_ops.adamw_step_dev}


def _install(setter):
    from imagdressing_b200 import ops

    for name, fn in CLIP_OPS.items():
        setter(ops, name, fn)


@pytest.fixture
def clip_ops(monkeypatch):
    _install(monkeypatch.setattr)


def _net(seed=0):
    torch.manual_seed(seed)
    return torch.nn.Sequential(torch.nn.Linear(6, 5), torch.nn.Tanh(), torch.nn.Linear(5, 4)).to(BF)


def _x(n=8, seed=1):
    return torch.randn(n, 6, generator=torch.Generator().manual_seed(seed)).to(BF)


def _loss(net, x):
    return (net(x).float() + 1.0).square().mean()


def _micro_step(net, opt, x):
    opt.zero_grad()
    _loss(net, x).backward()
    return opt.step()


def _state(opt):
    return [t.clone() for t in (opt.master, opt.param, opt.m, opt.v, opt.hyper)]


def test_clipped_steps_equal_clip_grad_norm_and_torch_adamw(clip_ops):
    from imagdressing_b200 import train

    net = _net()
    opt = train.FlatAdamW(net.parameters(), bucket_bytes=32, max_grad_norm=MAX, **HP)
    ref_params = [p.detach().float().clone() for p in opt.params]
    ref = torch.optim.AdamW(ref_params, **HP)
    spans = {id(p): opt._spans[i][0] for i, p in enumerate(opt._order)}
    x = _x()
    for step in range(4):
        opt.zero_grad()
        _loss(net, x).backward()
        for rp, p in zip(ref_params, opt.params):
            rp.grad = p.grad.float()  # the same (bf16) gradient both sides
        ref_norm = float(torch.nn.utils.clip_grad_norm_(ref_params, MAX))
        ref.step()
        assert opt.step()
        norm = float(opt.last_grad_norm)
        assert norm > MAX, (step, norm)  # clipping engaged: coef < 1
        assert abs(norm - ref_norm) <= 1e-5 * ref_norm
        assert float(opt.clip_state[1]) < 1.0
        for rp, p in zip(ref_params, opt.params):
            o = spans[id(p)]
            got = opt.master[o:o + p.numel()].view(p.shape)
            torch.testing.assert_close(got, rp.detach(), rtol=2e-6, atol=2e-7)
    assert opt.t == 4 and float(opt.skipped_steps) == 0


def test_no_clipping_keeps_the_plain_update(monkeypatch):
    """max_grad_norm=None: no norm pass, no clipped update, no extra state."""
    from imagdressing_b200 import ops, train

    def boom(*a, **k):
        raise AssertionError("clipping path used with max_grad_norm=None")

    monkeypatch.setattr(ops, "adamw_step_dev", emulated_ops.adamw_step_dev)
    monkeypatch.setattr(ops, "grad_norm_clip", boom)
    monkeypatch.setattr(ops, "adamw_step_clip", boom)
    net = _net()
    opt = train.FlatAdamW(net.parameters(), bucket_bytes=32, **HP)
    assert opt.clip_state is None and opt.last_grad_norm is None and opt.skipped_steps is None
    _micro_step(net, opt, _x())
    assert opt.t == 1 and "skipped_steps" not in opt.state_dict()


def test_clip_arguments_are_checked():
    from imagdressing_b200 import train

    for bad in (0.0, -1.0, float("nan")):
        with pytest.raises(ValueError):
            train.FlatAdamW(_net().parameters(), max_grad_norm=bad)
    with pytest.raises(ValueError):
        train.FlatAdamW(_net().parameters(), max_grad_norm=1.0, step_fn=emulated_ops.adamw_step)


def test_accumulation_equals_the_whole_batch_clipped_step(clip_ops):
    from imagdressing_b200 import train

    x = _x()
    net_a, net_w = _net(), _net()
    opt_a = train.FlatAdamW(net_a.parameters(), bucket_bytes=32, max_grad_norm=MAX, accumulation_steps=2, **HP)
    opt_w = train.FlatAdamW(net_w.parameters(), bucket_bytes=32, max_grad_norm=MAX, **HP)
    for _ in range(3):
        assert not _micro_step(net_a, opt_a, x[:4])
        assert _micro_step(net_a, opt_a, x[4:])
        assert _micro_step(net_w, opt_w, x)
        na, nw = float(opt_a.last_grad_norm), float(opt_w.last_grad_norm)
        assert na > MAX and nw > MAX
        assert abs(na - nw) < 1e-2 * nw  # bf16 sums of the two micro-batch gradients vs the batch gradient
    assert opt_a.t == opt_w.t == 3
    assert float((opt_a.master - opt_w.master).abs().max()) < 2e-3  # 3 updates of ~lr = 1e-2 each


@pytest.mark.parametrize("bad", [float("nan"), float("inf"), float("-inf")])
def test_non_finite_gradient_skips_the_update(clip_ops, bad):
    from imagdressing_b200 import train

    x = _x()
    net, twin = _net(), _net()
    opt = train.FlatAdamW(net.parameters(), bucket_bytes=32, max_grad_norm=MAX, **HP)
    ref = train.FlatAdamW(twin.parameters(), bucket_bytes=32, max_grad_norm=MAX, **HP)
    _micro_step(net, opt, x)
    _micro_step(twin, ref, x)
    before = _state(opt)
    # a poisoned gradient: the flat buffer after the backward's hand-over, before the update
    opt.zero_grad()
    _loss(net, x[:4]).backward()
    opt.grad[3] = bad
    assert opt.step()
    for a, b in zip(_state(opt), before):
        assert torch.equal(a, b)  # master, param, m, v and the step count untouched
    assert float(opt.clip_state[2]) == 0.0 and float(opt.skipped_steps) == 1 and opt.t == 1
    # the next finite step proceeds as if the bad one had never happened
    _micro_step(net, opt, x)
    _micro_step(twin, ref, x)
    for a, b in zip(_state(opt), _state(ref)):
        assert torch.equal(a, b)
    assert opt.t == 2 and float(opt.skipped_steps) == 1 and float(opt.clip_state[2]) == 1.0


def test_state_dict_round_trip_across_a_skipped_step(clip_ops):
    from imagdressing_b200 import train

    x = _x()
    net = _net()
    opt = train.FlatAdamW(net.parameters(), bucket_bytes=32, max_grad_norm=MAX, **HP)
    _micro_step(net, opt, x)
    opt.zero_grad()
    _loss(net, x).backward()
    opt.grad[0] = float("nan")
    opt.step()
    sd = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in opt.state_dict().items()}
    assert sd["t"] == 1 and sd["skipped_steps"] == 1  # the device count: the skipped update did not advance it

    net2 = _net(seed=5)  # other initial weights: everything must come from the state dict
    opt2 = train.FlatAdamW(net2.parameters(), bucket_bytes=32, max_grad_norm=MAX, **HP)
    opt2.load_state_dict(sd)
    assert opt2.t == 1 and float(opt2.skipped_steps) == 1 and float(opt2.hyper[2]) == 1.0
    assert torch.equal(opt2.param, opt.param)
    _micro_step(net, opt, x)
    _micro_step(net2, opt2, x)  # bias correction of step 2 on both
    for a, b in zip(_state(opt), _state(opt2)):
        assert torch.equal(a, b)
    assert opt.t == opt2.t == 2


# ------------------------------------------------------------------------------------------------ gloo world 2
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _dp_worker(rank, world, port, out_q):
    """Each rank back-propagates its half of the batch; the flat gradient is all-reduced, every rank computes the norm of the
    whole averaged gradient itself. Plain data parallelism and shard_states (each rank updates its slice)."""
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    _install(setattr)
    from imagdressing_b200 import train

    x = _x()
    lo, hi = rank * 4, rank * 4 + 4
    res = []
    for shard in (False, True):
        net = _net()
        opt = train.FlatAdamW(net.parameters(), bucket_bytes=32, max_grad_norm=MAX, shard_states=shard, **HP)
        norms = []
        for _ in range(3):
            _micro_step(net, opt, x[lo:hi])
            norms.append(float(opt.last_grad_norm))
        res.append((opt.param.float().numpy().copy(), norms, opt.t))
    out_q.put((rank, res))
    dist.barrier()
    dist.destroy_process_group()


def test_clipping_world2_plain_and_sharded(clip_ops):
    from imagdressing_b200 import train

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_dp_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=180) for _ in procs], key=lambda t: t[0])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    (_, (plain0, shard0)), (_, (plain1, shard1)) = res
    for a, b in ((plain0, plain1), (shard0, shard1), (plain0, shard0)):
        assert (a[0] == b[0]).all()  # parameters bit for bit
        assert a[1] == b[1]  # the same norms (hence coefficients) on both ranks
        assert a[2] == b[2] == 3

    net = _net()  # single process, whole batch
    opt = train.FlatAdamW(net.parameters(), bucket_bytes=32, max_grad_norm=MAX, **HP)
    norms = []
    for _ in range(3):
        _micro_step(net, opt, _x())
        norms.append(float(opt.last_grad_norm))
    assert all(n > MAX for n in norms)
    for a, b in zip(plain0[1], norms):
        assert abs(a - b) < 1e-2 * b
    n = opt.param.numel()
    assert float((torch.from_numpy(plain0[0])[:n] - opt.param.float()).abs().max()) < 2e-2
