"""GPU: the GroupNorm(+SiLU) / LayerNorm forward kernels (csrc/norm.cu) and the GroupNorm backward, LayerNorm backward
and column-sum kernels (csrc/train_ops.cu) element by element against fp64 references (tests/norm_fp64_ref.py).

Every output element must lie within halfulp_bf16(|ref| + E) + E of the fp64 reference (fp32 outputs: E + 2^-22 |ref|),
and every emitted GroupNorm statistic within dmu / drho of the fp64 statistic; E and dmu / drho are the allowances
derived in norm_fp64_ref under the plan that ran (its chunks / cluster ranks and their pivots). GroupNorm plans are
forced through imagd_groupnorm_debug_force (always restored to the automatic choice) and the plan that ran is read back
from imagd_groupnorm_debug_log.

  a. GroupNorm forward, every legal plan (the rendezvous kernel, each cluster size x slice width), with and without
     SiLU: the step shapes at batch 2, the training shapes at batch 4 (80 x 64 latents: HW 5120 / 1280 / 320 / 80 with
     the channel counts of the UNet's down / mid / up blocks), the VAE's full-resolution shape (64 chunks of 4096
     pixels), HW = 1025 (empty trailing chunks), HW = 5 (empty cluster CTAs); group means of 300 and 2000 in every
     plan; a strided input and output through the C ABI with sentinel columns;
  b. GroupNorm backward at the training shapes and HW = 1025, SiLU on / off, dgamma / dbeta in fp32 and bf16 and not
     requested, fed by the statistics of every forward plan and of large-mean inputs; dx bit-identical with and without
     the affine gradients and across launches;
  c. LayerNorm forward, each (VPL, R) instantiation at C = 256 ... 2048 including the C just past each one's limit,
     rows ragged against 8 R (1, 7, 20481), and a row-strided input / output;
  d. LayerNorm backward at C = 320 (20480 rows: the training transformer at level 0), 640, 768, 1280, 2048, rows 1 to
     20480, dgamma / dbeta in fp32 and bf16, with gamma and without;
  e. column sums at the bias-gradient shapes (whole-tensor and per-sample sums), split counts 1 to 64, fp32 and bf16.

The module prints the worst (|got - ref| - output rounding allowance) / E per family at its end (with -s); E is the
allowance, so a passing run is <= 1 everywhere ("stats": max of |mu_k - mu| / dmu and |rho_k / rho - 1| / drho).
Measured on an H100 80GB HBM3 (700 W power limit, 1980 MHz max SM clock), 123 tests, module 41 s (50 s under pytest):

  a. GN fwd step 1.7e-3 (stats 3.6e-3)   train 2.1e-3 (4.7e-3)   VAE 3.0e-3 (6.4e-3)   edge 1.6e-3 (3.5e-3)
     large mean 2.3e-3 (3.8e-3)   strided 9.3e-4 (2.9e-3)
  b. GN bwd dx 3.8e-2   dgamma / dbeta fp32 3.4e-3, bf16 1.1e-3
  c. LN fwd 8.5e-3   strided 4.2e-3
  d. LN bwd dx 7.3e-3   dgamma / dbeta fp32 5.1e-3, bf16 <= 0 (within the output rounding)
  e. colsum fp32 4.5e-3, bf16 <= 0

Every family stays at least 26x under its allowance; the statistics stay >= 150x under dmu / drho, which a dropped
chunk or row slot exceeds by tens to hundreds (test_norm_fp64_cpu.py). No case failed: no kernel change came of it.
"""
import subprocess
import time

import pytest
import torch

import gemm_fp64_ref as G
import norm_fp64_ref as R

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
CLUSTER_SIZES = (2, 4, 8, 16)
EPS = 1e-5


def _rand(shape, dev, seed, scale=1.0, offset=0.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale + offset).to(dev)


def _gn_input(NB, HW, C, dev, seed, mean=0.3, std=1.5):
    """bf16 [NB, HW, C]; for large means every group gets its own offset (10 % spread) so the group means are large."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    if abs(mean) < 10:
        x = torch.randn(NB, HW, C, generator=g) * std + mean
    else:
        offs = mean * (1.0 + 0.1 * torch.randn(NB, 1, 32, 1, generator=g))
        x = (torch.randn(NB, HW, 32, C // 32, generator=g) * std + offs).reshape(NB, HW, C)
    return x.to(dev).to(BF)


@pytest.fixture(scope="module")
def lib():
    from imagdressing_b200 import _lib

    lib = _lib.load()
    yield lib
    lib.imagd_groupnorm_debug_force(0, 0, 0)
    lib.imagd_groupnorm_debug_log(0, None, 0)


@pytest.fixture(scope="module", autouse=True)
def _report():
    R.WORST.clear()
    t0 = time.time()
    yield
    card = torch.cuda.get_device_name(0) if torch.cuda.is_available() else "?"
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:  # noqa: BLE001 - the report is informational
        power = "?"
    print(f"\n{card} ({power}); module {time.time() - t0:.1f} s")
    print("worst (|got - ref| - output rounding) / E per family (bound: 1):")
    for fam, v in sorted(R.WORST.items()):
        print(f"  {fam:28s} {v: .3e}")


def _plans(lib, NB, HW, C, groups):
    """Every distinct plan the forced-variant hook can select at this shape (the library decides what is legal)."""
    import ctypes

    cpg = C // groups
    forced = [(1, 0, 0)] + [(2, cs, gps * cpg) for cs in CLUSTER_SIZES for gps in range(1, groups + 1)
                            if groups % gps == 0 and gps * cpg % 8 == 0]
    out = (ctypes.c_int * 5)()
    plans = []
    try:
        for f in forced:
            assert lib.imagd_groupnorm_debug_force(*f) == 0
            if lib.imagd_groupnorm_plan(NB, HW, C, groups, None, out) == 0:
                assert (out[0], out[1], out[2]) == f
                plans.append(R.Plan(*f))
    finally:
        lib.imagd_groupnorm_debug_force(0, 0, 0)
    return plans


def _forced(lib, plan, fn):
    """Run fn under the forced plan; -> (result, the launch's debug-log line). The plan that ran must be `plan`."""
    assert lib.imagd_groupnorm_debug_force(plan.kernel, plan.cs, plan.sc) == 0
    lib.imagd_groupnorm_debug_log(1, None, 0)
    try:
        out = fn()
    finally:
        lib.imagd_groupnorm_debug_force(0, 0, 0)
        lib.imagd_groupnorm_debug_log(0, None, 0)
    buf = bytes(4096)
    n = lib.imagd_groupnorm_debug_log(-1, buf, len(buf))
    line = buf.split(b"\0", 1)[0].decode().strip()
    assert n == 1, line
    run = [int(v) for v in line.split("|")[1].split()]
    assert (run[0], run[1], run[2]) == (plan.kernel, plan.cs, plan.sc), (line, plan)
    return out, line


def _gn_fwd_all_plans(lib, dev, NB, HW, C, seed, *, family, mean=0.3, std=1.5, silus=(False, True)):
    from imagdressing_b200 import ops

    x = _gn_input(NB, HW, C, dev, seed, mean, std)
    gamma = _rand((C,), dev, seed + 1, 0.1, 1.0)
    beta = _rand((C,), dev, seed + 2, 0.1)
    plans = _plans(lib, NB, HW, C, 32)
    assert plans and plans[0].kernel == 1
    outs = {}
    for plan in plans:
        st = R.gn_stats(x, 32, EPS, plan)
        for silu in silus:
            stats = torch.full((NB, 32, 2), G.SENTINEL, device=dev)
            y, line = _forced(lib, plan, lambda: ops.groupnorm(x, gamma, beta, 32, EPS, silu=silu, stats_out=stats))
            ref, _ = R.gn_forward(x, gamma, beta, 32, EPS, silu, plan, st=st)
            R.check_gn_forward(f"groupnorm {NB}x{HW}x{C} silu={silu} {plan}", y, stats, ref, st, plan, 32,
                               family=family, cfg=line)
            outs[(plan.kernel, plan.cs, plan.sc, silu)] = stats
    return x, gamma, beta, plans, outs


# ================================================================================= a. GroupNorm forward
STEP_SHAPES = [(2, 4096, 320), (2, 1024, 640), (2, 64, 1280), (2, 256, 2560), (2, 1024, 960), (2, 256, 1920)]
TRAIN_SHAPES = [(4, 5120, 320), (4, 5120, 640), (4, 5120, 960), (4, 1280, 320), (4, 1280, 640), (4, 1280, 960),
                (4, 1280, 1280), (4, 1280, 1920), (4, 320, 640), (4, 320, 1280), (4, 320, 1920), (4, 320, 2560),
                (4, 80, 1280), (4, 80, 2560)]
EDGE_SHAPES = [(2, 1025, 320), (4, 1025, 640), (2, 5, 640), (1, 5, 320)]


@pytest.mark.parametrize("NB,HW,C", STEP_SHAPES + TRAIN_SHAPES + EDGE_SHAPES)
def test_groupnorm_forward_every_plan(cuda_device, lib, NB, HW, C):
    fam = "a. GN fwd " + ("edge" if (NB, HW, C) in EDGE_SHAPES else "step" if NB == 2 else "train")
    _gn_fwd_all_plans(lib, cuda_device, NB, HW, C, 100 + C + HW, family=fam)


def test_groupnorm_forward_vae_full_resolution(cuda_device, lib):
    """512 x 512 x 128: 64 rendezvous chunks of 4096 pixels (the longest per-thread chains); no cluster plan fits."""
    _gn_fwd_all_plans(lib, cuda_device, 1, 512 * 512, 128, 7, family="a. GN fwd VAE")


@pytest.mark.parametrize("mean,std", [(300.0, 4.0), (2000.0, 0.5)])
@pytest.mark.parametrize("NB,HW,C", [(2, 1024, 320), (4, 1280, 640), (2, 1025, 320)])
def test_groupnorm_forward_large_mean_every_plan(cuda_device, lib, NB, HW, C, mean, std):
    _gn_fwd_all_plans(lib, cuda_device, NB, HW, C, 31, mean=mean, std=std, family="a. GN fwd large mean")


def test_groupnorm_forward_strided(cuda_device, lib):
    """ldx > C and ldy > C through the C ABI: the sentinel columns around the output keep their value in every plan."""
    from imagdressing_b200 import _lib, ops

    NB, HW, C, padx, pady = 2, 1024, 640, 24, 16
    xb = _rand((NB, HW, C + padx), cuda_device, 41, 1.5, 0.3).to(BF)
    x = xb[..., 8:8 + C]
    gamma = _rand((C,), cuda_device, 42, 0.1, 1.0)
    beta = _rand((C,), cuda_device, 43, 0.1)
    ws = ops._gn_workspace(x.device, lib.imagd_groupnorm_ws_bytes(NB, HW, C, 32))
    for plan in _plans(lib, NB, HW, C, 32):
        y = G.sentinel_buffer((NB, HW, C + pady), BF, cuda_device)
        yv = y[..., 8:8 + C]
        stats = torch.full((NB, 32, 2), G.SENTINEL, device=cuda_device)

        def run():
            rc = lib.imagd_groupnorm_stats_bf16(x.data_ptr(), C + padx, yv.data_ptr(), C + pady, NB, HW, C, 32,
                                                gamma.data_ptr(), beta.data_ptr(), EPS, 1, ws.data_ptr(), stats.data_ptr(),
                                                torch.cuda.current_stream().cuda_stream)
            _lib.check(rc, "imagd_groupnorm_stats_bf16")

        _, line = _forced(lib, plan, run)
        ref, st = R.gn_forward(x.contiguous(), gamma, beta, 32, EPS, True, plan)
        R.check_gn_forward(f"strided groupnorm {plan}", yv, stats, ref, st, plan, 32, family="a. GN fwd strided", cfg=line)
        G.assert_outside_untouched(f"strided groupnorm {plan}", y, (slice(None), slice(None), slice(8, 8 + C)))


# ================================================================================= b. GroupNorm backward
def _gn_bwd_check(dev, x, gamma, beta, stats, silu, tag, seed):
    from imagdressing_b200 import ops

    NB, HW, C = x.shape
    dy = _rand((NB, HW, C), dev, seed, 1.0).to(BF)
    ref = R.gn_backward(x, dy, gamma, beta, 32, EPS, silu, stats)
    dx0, dg0, db0 = ops.groupnorm_bwd(x, dy, gamma, beta, 32, stats, silu, False)
    dx1, dg1, db1 = ops.groupnorm_bwd(x, dy, gamma, beta, 32, stats, silu, True, torch.float32)
    dx2, dg2, db2 = ops.groupnorm_bwd(x, dy, gamma, beta, 32, stats, silu, True, BF)
    dx3, _, _ = ops.groupnorm_bwd(x, dy, gamma, beta, 32, stats, silu, False)
    assert dg0 is None and db0 is None
    name = f"groupnorm_bwd {NB}x{HW}x{C} silu={silu} {tag}"
    R.G.check(name + " dx", dx1, ref.dx, family="b. GN bwd dx",
              locate=R.gn_locate(HW, C, 32, ref.parts, "chunk"))
    for t in (dx0, dx2, dx3):
        assert torch.equal(t, dx1), name + ": dx not bit-identical across need_affine / launches"
    R.check_affine(name + " dgamma fp32", dg1, ref.dgamma, ref.cands_a, family="b. GN bwd dgamma/dbeta fp32")
    R.check_affine(name + " dbeta fp32", db1, ref.dbeta, ref.cands_b, family="b. GN bwd dgamma/dbeta fp32")
    bf = lambda r: G.Ref(r.ref, r.E, r.P, False)
    R.check_affine(name + " dgamma bf16", dg2, bf(ref.dgamma), ref.cands_a, family="b. GN bwd dgamma/dbeta bf16")
    R.check_affine(name + " dbeta bf16", db2, bf(ref.dbeta), ref.cands_b, family="b. GN bwd dgamma/dbeta bf16")


@pytest.mark.parametrize("silu", [False, True])
@pytest.mark.parametrize("NB,HW,C", TRAIN_SHAPES + [(2, 1025, 320), (4, 1025, 640)])
def test_groupnorm_backward(cuda_device, lib, NB, HW, C, silu):
    from imagdressing_b200 import ops

    x = _gn_input(NB, HW, C, cuda_device, 200 + C + HW)
    gamma = _rand((C,), cuda_device, 3, 0.1, 1.0)
    beta = _rand((C,), cuda_device, 4, 0.1)
    stats = torch.empty(NB, 32, 2, device=cuda_device)
    ops.groupnorm(x, gamma, beta, 32, EPS, silu=silu, stats_out=stats)
    _gn_bwd_check(cuda_device, x, gamma, beta, stats, silu, "auto plan stats", 300 + C)


@pytest.mark.parametrize("mean,std", [(0.3, 1.5), (300.0, 4.0), (2000.0, 0.5)])
@pytest.mark.parametrize("NB,HW,C", [(4, 1280, 640), (2, 1025, 320)])
def test_groupnorm_backward_fed_by_every_forward_plan(cuda_device, lib, NB, HW, C, mean, std):
    x, gamma, beta, plans, outs = _gn_fwd_all_plans(lib, cuda_device, NB, HW, C, 51, mean=mean, std=std,
                                                    family="a. GN fwd large mean" if mean > 10 else "a. GN fwd train",
                                                    silus=(True,))
    for plan in plans:
        _gn_bwd_check(cuda_device, x, gamma, beta, outs[(plan.kernel, plan.cs, plan.sc, True)], True,
                      f"stats of {plan}", 61)


def test_groupnorm_backward_without_affine(cuda_device, lib):
    """gamma = beta = None (the identity affine)."""
    from imagdressing_b200 import ops

    NB, HW, C = 4, 1280, 640
    x = _gn_input(NB, HW, C, cuda_device, 71)
    stats = torch.empty(NB, 32, 2, device=cuda_device)
    ops.groupnorm(x, None, None, 32, EPS, silu=True, stats_out=stats)
    _gn_bwd_check(cuda_device, x, None, None, stats, True, "no affine", 72)


# ================================================================================= c. LayerNorm forward
@pytest.mark.parametrize("rows", [1, 7, 20481])
@pytest.mark.parametrize("C", [256, 512, 520, 768, 776, 1280, 1288, 2048])
def test_layernorm_forward(cuda_device, C, rows):
    from imagdressing_b200 import ops

    x = _rand((rows, C), cuda_device, C + rows, 1.2, 0.4).to(BF)
    gamma = _rand((C,), cuda_device, 5, 0.1, 1.0)
    beta = _rand((C,), cuda_device, 6, 0.1)
    y = ops.layernorm(x, gamma, beta, EPS)
    ref = R.ln_forward(x, gamma, beta, EPS)
    G.check(f"layernorm {rows}x{C}", y, ref, family="c. LN fwd", locate=lambda r, c: f"row {r}, channel {c}")


@pytest.mark.parametrize("C", [320, 1288])
def test_layernorm_forward_strided_and_large_mean(cuda_device, C):
    from imagdressing_b200 import ops

    rows, pad = 333, 40
    xb = (_rand((rows, C + pad), cuda_device, 8, 2.0) + _rand((rows, 1), cuda_device, 9, 50.0, 200.0)).to(BF)
    x = xb[:, 16:16 + C]
    out = G.sentinel_buffer((rows, C + pad), BF, cuda_device)
    ov = out[:, 8:8 + C]
    gamma = _rand((C,), cuda_device, 10, 0.1, 1.0)
    ops.layernorm(x, gamma, None, EPS, out=ov)
    ref = R.ln_forward(x, gamma, None, EPS)
    G.check(f"strided layernorm {C}", ov, ref, family="c. LN fwd strided", locate=lambda r, c: f"row {r}, channel {c}")
    G.assert_outside_untouched("strided layernorm", out, (slice(None), slice(8, 8 + C)))


# ================================================================================= d. LayerNorm backward
@pytest.mark.parametrize("C,rows", [(320, 20480), (320, 1), (320, 77), (640, 5120), (640, 7), (768, 1000), (768, 333),
                                    (1280, 1280), (1280, 20480), (2048, 320), (2048, 4097)])
def test_layernorm_backward(cuda_device, C, rows):
    from imagdressing_b200 import ops

    x = _rand((rows, C), cuda_device, C + rows, 1.2, 0.4).to(BF)
    dy = _rand((rows, C), cuda_device, C + rows + 1, 1.0).to(BF)
    gamma = _rand((C,), cuda_device, 11, 0.1, 1.0)
    for g, tag in ((gamma, "gamma"), (None, "no gamma")):
        ref = R.ln_backward(x, dy, g, EPS)
        dx0, dg0, db0 = ops.layernorm_bwd(x, dy, g, EPS, False)
        dx1, dg1, db1 = ops.layernorm_bwd(x, dy, g, EPS, True, torch.float32)
        dx2, dg2, db2 = ops.layernorm_bwd(x, dy, g, EPS, True, BF)
        name = f"layernorm_bwd {rows}x{C} {tag}"
        G.check(name + " dx", dx1, ref.dx, family="d. LN bwd dx", locate=lambda r, c: f"row {r}, channel {c}")
        assert torch.equal(dx0, dx1) and torch.equal(dx2, dx1), name + ": dx not bit-identical"
        R.check_affine(name + " dgamma fp32", dg1, ref.dgamma, ref.cands_a, family="d. LN bwd dgamma/dbeta fp32")
        R.check_affine(name + " dbeta fp32", db1, ref.dbeta, ref.cands_b, family="d. LN bwd dgamma/dbeta fp32")
        bf = lambda r: G.Ref(r.ref, r.E, r.P, False)
        R.check_affine(name + " dgamma bf16", dg2, bf(ref.dgamma), ref.cands_a, family="d. LN bwd dgamma/dbeta bf16")
        R.check_affine(name + " dbeta bf16", db2, bf(ref.dbeta), ref.cands_b, family="d. LN bwd dgamma/dbeta bf16")


# ================================================================================= e. column sums
# (rows, C, rows_per_group): bias gradients of the training UNet's convs / linears (whole-tensor sums) and the
# per-sample time-embedding row vectors (rows_per_group = H W); the split count is colreduce_splits of the shape
COLSUM_SHAPES = [(20480, 320, None), (20480, 640, 5120), (5120, 640, None), (5120, 1280, 1280), (1280, 1280, None),
                 (1280, 2560, 320), (320, 2560, None), (320, 1280, 80), (308, 768, None), (64, 320, None),
                 (20480, 64, None), (4096, 40, None), (200, 320, None), (20480, 1280, None)]


def test_colsum_split_range():
    splits = {R.colreduce_splits(rpg or rows, rows // (rpg or rows), C) for rows, C, rpg in COLSUM_SHAPES}
    assert min(splits) == 1 and max(splits) == 64 and len(splits) >= 8, sorted(splits)


@pytest.mark.parametrize("rows,C,rpg", COLSUM_SHAPES)
def test_colsum(cuda_device, rows, C, rpg):
    from imagdressing_b200 import ops

    x = _rand((rows, C), cuda_device, rows + C, 1.0, 0.2).to(BF)
    for dt in (torch.float32, BF):
        got = ops.colsum(x, rpg, dt)
        ref, cands = R.colsum(x, rpg or rows, out_bf16=dt == BF)
        R.check_affine(f"colsum {rows}x{C} rpg={rpg} {dt}", got, ref, cands,
                       family="e. colsum " + ("bf16" if dt == BF else "fp32"))
