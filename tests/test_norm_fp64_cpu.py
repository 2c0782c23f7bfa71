"""CPU: the norm checker of norm_fp64_ref is sensitive. fp32 emulations of each kernel's reduction order pass it at the
shapes test_norm_fp64_gpu.py runs (scaled down), and each emulated kernel fault (a mutant) fails it with a report that
names the chunk, cluster rank, fold lane, split, group or channel at fault. The references themselves are checked
against torch.nn.functional in fp64.

The emulations follow the kernels' decomposition, not their exact instruction order:
  - GroupNorm forward: parts (rendezvous chunks or cluster ranks) x row slots, each channel shifted by its value at the
    part's first pixel, channels -> group and parts -> sample merged with Chan's formula relative to the first part's
    mean; empty parts write {0, 0} and count 0 (the `npix > 0` guard and the clamped `cnt_k`);
  - GroupNorm backward: per-chunk partials over row slots, the fold's 4 chunk lanes, S1 / S2 per group, the apply step;
  - LayerNorm backward: per-row statistics and sums, then the column reduction's splits and their fold.
"""
import pytest
import torch

import gemm_fp64_ref as G
import norm_fp64_ref as R

BF = torch.bfloat16
EPS = 1e-5
F = torch.nn.functional


def _rand(shape, seed, scale=1.0, offset=0.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(shape, generator=g) * scale + offset


def _gn_input(NB, HW, C, seed, mean=0.3, std=1.5):
    g = torch.Generator().manual_seed(seed)
    if abs(mean) < 10:
        return (torch.randn(NB, HW, C, generator=g) * std + mean).to(BF)
    offs = mean * (1.0 + 0.1 * torch.randn(NB, 1, 32, 1, generator=g))
    return (torch.randn(NB, HW, 32, C // 32, generator=g) * std + offs).reshape(NB, HW, C).to(BF)


# ------------------------------------------------------------------------------------------------ emulations
def emu_gn_forward(x, gamma, beta, groups, eps, silu, plan, mut=None, at=None):
    """fp32 emulation of groupnorm_fused_kernel (plan.kernel 1) / groupnorm_cluster_kernel (2) -> (y bf16, stats)."""
    NB, HW, C = x.shape
    cpg = C // groups
    X = x.float()
    parts = plan.parts(HW, NB)
    slots = plan.row_slots(C)
    means, m2s = [], []
    for k, (b, e) in enumerate(parts):
        n = max(e - b, 0)
        if n == 0 and mut != "no npix guard":
            means.append(torch.zeros(NB, groups))
            m2s.append(torch.zeros(NB, groups))
            continue
        piv = X[:, b, :] if n > 0 else torch.zeros(NB, C)
        a = torch.zeros(NB, C)
        q = torch.zeros(NB, C)
        end = e - 1 if (mut == "pixel edge" and k == at) else e
        for s in range(slots):
            if mut == "row slot" and (k, s) == at:
                continue
            seg = X[:, b + s:end:slots] - piv[:, None]
            a = a + seg.sum(1)
            q = q + (seg * seg).sum(1)
        npix = torch.tensor(float(n))
        inv = 1.0 / npix  # inf for an empty part: only reached without the guard
        t = piv + a * inv
        mean_g = t.reshape(NB, groups, cpg).sum(-1) / cpg
        d = t.reshape(NB, groups, cpg) - mean_g[..., None]
        m2 = ((q - a * a * inv).reshape(NB, groups, cpg) + npix * d * d).sum(-1)
        means.append(mean_g)
        m2s.append(m2)
    pivot = means[0]
    ta = torch.zeros(NB, groups)
    tb = torch.zeros(NB, groups)
    first_empty = next((k for k, (b, e) in enumerate(parts) if e <= b), None)
    nominal = -(-HW // len(parts))
    for k, (b, e) in enumerate(parts):
        cnt_k = float(cpg * max(e - b, 0))
        if mut == "empty count" and k == first_empty:
            cnt_k = float(cpg * nominal)
        reps = 0 if (mut == "drop chunk" and k == at) else 2 if (mut == "chunk twice" and k == at) else 1
        for _ in range(reps):
            d = means[k] - pivot
            ta = ta + cnt_k * d
            tb = tb + m2s[k] + cnt_k * d * d
    cnt = float(cpg * HW)
    dm = ta / cnt
    var = ((tb - ta * dm) / cnt).clamp_min(0.0)
    mu, rstd = pivot + dm, torch.rsqrt(var + eps)
    if mut == "raw moments":  # one-pass E[x^2] - mean^2 on the raw values
        Xg = X.reshape(NB, HW, groups, cpg)
        mu = Xg.sum((1, 3)) / cnt
        rstd = torch.rsqrt(((Xg * Xg).sum((1, 3)) / cnt - mu * mu).clamp_min(0.0) + eps)
    ga = gamma.float().clone() if gamma is not None else torch.ones(C)
    be = beta.float().clone() if beta is not None else torch.zeros(C)
    if mut == "gamma beta swap":
        ga[at], be[at] = be[at].clone(), ga[at].clone()
    sc = ga * rstd.repeat_interleave(cpg, 1)
    sh = be - mu.repeat_interleave(cpg, 1) * sc
    f = X * sc[:, None] + sh[:, None]
    if silu:
        f = f / (1.0 + torch.exp(-f))
    return f.to(BF), torch.stack([mu, rstd], -1)


def _silu_grad(z):
    s = 1.0 / (1.0 + torch.exp(-z))
    return s * (1.0 + z * (1.0 - s))


def emu_gn_backward(x, dy, gamma, beta, groups, silu, stats, mut=None, at=None, out_bf16=False):
    """fp32 emulation of groupnorm_bwd_partial / _fold / _apply and the affine fold -> (dx bf16, dgamma, dbeta)."""
    NB, HW, C = x.shape
    cpg = C // groups
    X, DY = x.float(), dy.float()
    parts = R.bwd_parts(HW, NB)
    slots = 512 // (C // 8)
    ga = gamma.float() if gamma is not None else torch.ones(C)
    be = beta.float() if beta is not None else torch.zeros(C)
    mean = stats[..., 0].repeat_interleave(cpg, 1)[:, None]
    rstd = stats[..., 1].repeat_interleave(cpg, 1)[:, None]
    xh = X * rstd + (-mean * rstd)
    dz = DY * _silu_grad(xh * ga + be) if silu else DY
    part_a, part_b = [], []
    for b, e in parts:
        a = torch.zeros(NB, C)
        q = torch.zeros(NB, C)
        for s in range(slots):
            a = a + (dz[:, b + s:e:slots] * xh[:, b + s:e:slots]).sum(1)
            q = q + dz[:, b + s:e:slots].sum(1)
        part_a.append(a)
        part_b.append(q)
    la, lb = [torch.zeros(NB, C) for _ in range(4)], [torch.zeros(NB, C) for _ in range(4)]
    for k in range(len(parts)):
        if mut == "drop lane" and k % 4 == at:
            continue
        la[k % 4] = la[k % 4] + part_a[k]
        lb[k % 4] = lb[k % 4] + part_b[k]
    pa = (la[0] + la[1]) + (la[2] + la[3])
    pb = (lb[0] + lb[1]) + (lb[2] + lb[3])
    m = float(HW * cpg)
    S1 = (ga * pb).reshape(NB, groups, cpg).sum(-1) / m
    S2 = (ga * pa).reshape(NB, groups, cpg).sum(-1) / m
    gid = torch.arange(C) // cpg
    if mut == "group off":  # the apply step reads the statistics of the next group for one group's channels
        gid = torch.where(gid == at, gid + 1, gid)
    st_m, st_r = stats[..., 0][:, gid][:, None], stats[..., 1][:, None][:, :, gid]
    s1, s2 = S1[:, gid][:, None], S2[:, gid][:, None]
    if mut == "swap s1 s2":
        sel = (torch.arange(C) // cpg == at)
        s1, s2 = torch.where(sel, s2, s1), torch.where(sel, s1, s2)
    xh2 = (X - st_m) * st_r
    dz2 = DY * _silu_grad(xh2 * ga + be) if silu else DY
    if mut == "no silu grad":
        dz2 = torch.where(torch.arange(C) // cpg == at, DY, dz2)
    dx = (st_r * (dz2 * ga - s1 - xh2 * s2)).to(BF)
    if mut == "double round":
        dg = pa.to(BF).float().sum(0).to(BF)
        db = pb.to(BF).float().sum(0).to(BF)
    else:
        dg, db = pa.sum(0), pb.sum(0)
        if out_bf16:
            dg, db = dg.to(BF), db.to(BF)
    return dx, dg, db


def emu_ln_forward(x, gamma, beta, eps):
    X = x.float()
    C = X.shape[-1]
    mean = X.sum(-1, keepdim=True) / C
    rstd = torch.rsqrt(((X - mean) ** 2).sum(-1, keepdim=True) / C + eps)
    return ((X - mean) * rstd * gamma.float() + beta.float()).to(BF)


def emu_ln_backward(x, dy, gamma, eps, mut=None, out_bf16=False):
    """fp32 emulation of layernorm_bwd_kernel + colreduce_kernel<1> + colreduce_fold_kernel."""
    X, DY = x.float(), dy.float()
    rows, C = X.shape
    ga = gamma.float() if gamma is not None else torch.ones(C)
    mean = X.sum(-1, keepdim=True) / C
    rstd = torch.rsqrt(((X - mean) ** 2).sum(-1, keepdim=True) / C + eps)
    xh = (X - mean) * rstd
    g = DY * ga
    s1 = g.sum(-1, keepdim=True) / C
    s2 = (g * xh).sum(-1, keepdim=True) / C
    dx = (rstd * (g - s1 - xh * s2)).to(BF)
    if mut == "nan":
        dx[rows // 2, C // 3] = float("nan")
    splits = R.colreduce_splits(rows, 1, C)
    span = -(-rows // splits)
    pa = [(DY[s * span:(s + 1) * span] * xh[s * span:(s + 1) * span]).sum(0) for s in range(splits)]
    pb = [DY[s * span:(s + 1) * span].sum(0) for s in range(splits)]
    n = splits - 1 if mut == "split short" else splits
    dg, db = torch.zeros(C), torch.zeros(C)
    for s in range(n):
        dg, db = dg + pa[s], db + pb[s]
    if out_bf16:
        dg, db = dg.to(BF), db.to(BF)
    return dx, dg, db


def emu_colsum(x, rpg, out_bf16=False):
    X = x.float()
    rows, C = X.shape
    groups = rows // rpg
    splits = R.colreduce_splits(rpg, groups, C)
    span = -(-rpg // splits)
    out = torch.zeros(groups, C)
    for s in range(splits):
        out = out + X.reshape(groups, rpg, C)[:, s * span:(s + 1) * span].sum(1)
    return out.to(BF) if out_bf16 else out


# ------------------------------------------------------------------------------------------------ references
def test_references_match_torch_functional():
    NB, HW, C = 2, 96, 320
    x = _gn_input(NB, HW, C, 1)
    dy = _rand((NB, HW, C), 2).to(BF)
    ga, be = _rand((C,), 3, 0.1, 1.0), _rand((C,), 4, 0.1)
    xd = x.double().requires_grad_()
    gd, bd = ga.double().requires_grad_(), be.double().requires_grad_()
    z = F.group_norm(xd.permute(0, 2, 1), 32, gd, bd, EPS).permute(0, 2, 1)
    y = z * torch.sigmoid(z)
    (y * dy.double()).sum().backward()
    ref, st = R.gn_forward(x, ga, be, 32, EPS, True, R.Plan(1))
    assert torch.allclose(ref.ref, y.detach().reshape(-1, C), rtol=1e-12, atol=1e-12)
    xg = x.double().reshape(NB, HW, 32, C // 32)
    assert torch.allclose(st.rho, 1 / torch.sqrt(xg.var((1, 3), unbiased=False) + EPS), rtol=1e-12)
    stats = torch.stack([st.mu, st.rho], -1).float()
    b = R.gn_backward(x, dy, ga, be, 32, EPS, True, stats)
    assert torch.allclose(b.dx.ref, xd.grad.reshape(-1, C), rtol=1e-10, atol=1e-12)
    assert torch.allclose(b.dgamma.ref.flatten(), gd.grad, rtol=1e-10, atol=1e-10)
    assert torch.allclose(b.dbeta.ref.flatten(), bd.grad, rtol=1e-10, atol=1e-10)
    x2, dy2 = x.reshape(-1, C), dy.reshape(-1, C)
    xd = x2.double().requires_grad_()
    gd, bd = ga.double().requires_grad_(), be.double().requires_grad_()
    yl = F.layer_norm(xd, (C,), gd, bd, EPS)
    (yl * dy2.double()).sum().backward()
    assert torch.allclose(R.ln_forward(x2, ga, be, EPS).ref, yl.detach(), rtol=1e-12, atol=1e-12)
    lb = R.ln_backward(x2, dy2, ga, EPS)
    assert torch.allclose(lb.dx.ref, xd.grad, rtol=1e-10, atol=1e-12)
    assert torch.allclose(lb.dgamma.ref.flatten(), gd.grad, rtol=1e-10, atol=1e-10)
    assert torch.allclose(lb.dbeta.ref.flatten(), bd.grad, rtol=1e-10, atol=1e-10)
    cs, _ = R.colsum(x2, HW)
    assert torch.allclose(cs.ref, x2.double().reshape(NB, HW, C).sum(1))


# ------------------------------------------------------------------------------------------------ emulations pass
# the GPU file's shapes scaled down: step / training (several chunks per sample), VAE-like (64 chunks of 64 pixels),
# HW = 1025 (empty trailing chunks), HW = 5 (empty cluster ranks)
FWD_SHAPES = [(2, 256, 320), (4, 320, 640), (4, 80, 1280), (1, 4096, 128), (2, 1025, 64), (2, 5, 640)]


def _cpu_plans(C):
    cpg = C // 32
    sc = next(g * cpg for g in range(1, 33) if (g * cpg) % 8 == 0 and 32 % g == 0)
    return [R.Plan(1), R.Plan(2, 2, C), R.Plan(2, 16, sc)]


@pytest.mark.parametrize("NB,HW,C", FWD_SHAPES)
def test_emulated_forward_passes(NB, HW, C):
    x = _gn_input(NB, HW, C, HW + C)
    ga, be = _rand((C,), 5, 0.1, 1.0), _rand((C,), 6, 0.1)
    for plan in _cpu_plans(C):
        st = R.gn_stats(x, 32, EPS, plan)
        for silu in (False, True):
            y, stats = emu_gn_forward(x, ga, be, 32, EPS, silu, plan)
            ref, _ = R.gn_forward(x, ga, be, 32, EPS, silu, plan, st=st)
            R.check_gn_forward(f"emulated {plan}", y, stats, ref, st, plan, 32)


@pytest.mark.parametrize("mean,std", [(300.0, 4.0), (2000.0, 0.5)])
def test_emulated_forward_passes_at_large_means(mean, std):
    NB, HW, C = 2, 256, 320
    x = _gn_input(NB, HW, C, 9, mean, std)
    ga, be = _rand((C,), 5, 0.1, 1.0), _rand((C,), 6, 0.1)
    for plan in _cpu_plans(C):
        y, stats = emu_gn_forward(x, ga, be, 32, EPS, True, plan)
        ref, st = R.gn_forward(x, ga, be, 32, EPS, True, plan)
        R.check_gn_forward(f"emulated {plan}", y, stats, ref, st, plan, 32)
        dy = _rand((NB, HW, C), 10).to(BF)
        _check_bwd(x, dy, ga, be, True, stats)


def _check_bwd(x, dy, ga, be, silu, stats, mut=None, at=None, out_bf16=False):
    NB, HW, C = x.shape
    ref = R.gn_backward(x, dy, ga, be, 32, EPS, silu, stats, affine_bf16=out_bf16)
    dx, dg, db = emu_gn_backward(x, dy, ga, be, 32, silu, stats, mut, at, out_bf16)
    G.check("emulated groupnorm_bwd dx", dx, ref.dx, locate=R.gn_locate(HW, C, 32, ref.parts, "chunk"))
    R.check_affine("emulated groupnorm_bwd dgamma", dg, ref.dgamma, ref.cands_a)
    R.check_affine("emulated groupnorm_bwd dbeta", db, ref.dbeta, ref.cands_b)


@pytest.mark.parametrize("NB,HW,C", [(4, 320, 640), (4, 80, 1280), (2, 1025, 64), (4, 1280, 64)])
@pytest.mark.parametrize("silu", [False, True])
@pytest.mark.parametrize("out_bf16", [False, True])
def test_emulated_backward_passes(NB, HW, C, silu, out_bf16):
    x = _gn_input(NB, HW, C, 11)
    dy = _rand((NB, HW, C), 12).to(BF)
    ga, be = _rand((C,), 5, 0.1, 1.0), _rand((C,), 6, 0.1)
    _, stats = emu_gn_forward(x, ga, be, 32, EPS, silu, R.Plan(1))
    _check_bwd(x, dy, ga, be, silu, stats, out_bf16=out_bf16)


@pytest.mark.parametrize("C,rows", [(320, 2048), (640, 7), (768, 333), (1288, 65), (2048, 129)])
def test_emulated_layernorm_passes(C, rows):
    x = _rand((rows, C), C, 1.2, 0.4).to(BF)
    dy = _rand((rows, C), C + 1).to(BF)
    ga, be = _rand((C,), 5, 0.1, 1.0), _rand((C,), 6, 0.1)
    G.check("emulated layernorm", emu_ln_forward(x, ga, be, EPS), R.ln_forward(x, ga, be, EPS),
            locate=lambda r, c: f"row {r}, channel {c}")
    for g in (ga, None):
        for bf in (False, True):
            ref = R.ln_backward(x, dy, g, EPS, affine_bf16=bf)
            dx, dg, db = emu_ln_backward(x, dy, g, EPS, out_bf16=bf)
            G.check("emulated layernorm_bwd dx", dx, ref.dx, locate=lambda r, c: f"row {r}, channel {c}")
            R.check_affine("emulated dgamma", dg, ref.dgamma, ref.cands_a)
            R.check_affine("emulated dbeta", db, ref.dbeta, ref.cands_b)


@pytest.mark.parametrize("rows,C,rpg", [(4096, 320, None), (4096, 64, 1024), (64, 320, None), (1280, 1280, 320)])
def test_emulated_colsum_passes(rows, C, rpg):
    x = _rand((rows, C), rows, 1.0, 0.2).to(BF)
    for bf in (False, True):
        ref, cands = R.colsum(x, rpg or rows, out_bf16=bf)
        R.check_affine("emulated colsum", emu_colsum(x, rpg or rows, bf), ref, cands)


# ------------------------------------------------------------------------------------------------ mutants fail
def _fwd_mutant(mut, at, pattern, *, NB=2, HW=320, C=64, plan=R.Plan(1), mean=0.3, std=1.5):
    x = _gn_input(NB, HW, C, 21, mean, std)
    ga, be = _rand((C,), 5, 0.1, 1.0), _rand((C,), 6, 0.1)
    ref, st = R.gn_forward(x, ga, be, 32, EPS, True, plan)
    y, stats = emu_gn_forward(x, ga, be, 32, EPS, True, plan, mut, at)
    with pytest.raises(AssertionError, match=pattern):
        R.check_gn_forward(f"mutant {mut}", y, stats, ref, st, plan, 32)


def test_mutant_dropped_chunk():
    _fwd_mutant("drop chunk", 5, r"statistics out of bound.*explained by chunk 5 \(x-")


def test_mutant_chunk_counted_twice():
    _fwd_mutant("chunk twice", 7, r"statistics out of bound.*explained by chunk 7 \(x\+")


def test_mutant_dropped_cluster_rank():
    _fwd_mutant("drop chunk", 3, r"statistics out of bound.*explained by rank 3 \(x-", plan=R.Plan(2, 8, 16))


def test_mutant_dropped_row_slot():
    # C 64: 64 row slots, 16 pixels per chunk -> slot 2 of chunk 4 is one pixel
    _fwd_mutant("row slot", (4, 2), r"statistics out of bound.*explained by chunk 4 row slot 2 \(x-")


def test_mutant_pixel_off_by_one_at_chunk_edge():
    _fwd_mutant("pixel edge", 9, r"statistics out of bound.*explained by chunk 9 last pixel \(x-")


def test_mutant_empty_chunk_counted():
    # HW 1025 at NB 2: 64 chunks of 17 pixels, chunks 61-63 empty
    _fwd_mutant("empty count", None, r"statistics out of bound.*explained by empty chunk 61", HW=1025)


def test_mutant_npix_guard_removed():
    _fwd_mutant("no npix guard", None, r"statistics out of bound", HW=1025)
    _fwd_mutant("no npix guard", None, r"statistics out of bound", HW=5, C=640, plan=R.Plan(2, 16, 40))


def test_mutant_raw_moments_at_large_mean():
    _fwd_mutant("raw moments", None, r"statistics out of bound.*group", HW=256, C=320, mean=2000.0, std=0.5)


def test_mutant_gamma_beta_swapped_for_one_channel():
    _fwd_mutant("gamma beta swap", 37, r"channel 37, group 18, chunk")


def _bwd_mutant(mut, at, pattern, *, NB=4, HW=1280, C=64, out_bf16=False):
    x = _gn_input(NB, HW, C, 23)
    dy = _rand((NB, HW, C), 24).to(BF)
    ga, be = _rand((C,), 5, 0.1, 1.0), _rand((C,), 6, 0.1)
    _, stats = emu_gn_forward(x, ga, be, 32, EPS, True, R.Plan(1))
    with pytest.raises(AssertionError, match=pattern):
        _check_bwd(x, dy, ga, be, True, stats, mut, at, out_bf16)


def test_mutant_fold_lane_dropped():
    # NB 4, HW 1280: 64 chunks, 16 per fold lane; dx fails too (S1 / S2 lose a quarter), dbeta names the lane
    NB, HW, C = 4, 1280, 64
    x = _gn_input(NB, HW, C, 23)
    dy = _rand((NB, HW, C), 24).to(BF)
    ga, be = _rand((C,), 5, 0.1, 1.0), _rand((C,), 6, 0.1)
    _, stats = emu_gn_forward(x, ga, be, 32, EPS, True, R.Plan(1))
    ref = R.gn_backward(x, dy, ga, be, 32, EPS, True, stats)
    dx, dg, db = emu_gn_backward(x, dy, ga, be, 32, True, stats, "drop lane", 2)
    with pytest.raises(AssertionError, match=r"dx: "):
        G.check("mutant drop lane dx", dx, ref.dx, locate=R.gn_locate(HW, C, 32, ref.parts, "chunk"))
    for got, r, cands in ((dg, ref.dgamma, ref.cands_a), (db, ref.dbeta, ref.cands_b)):
        with pytest.raises(AssertionError, match=r"explained by fold lane 2 \(x-"):
            R.check_affine("mutant drop lane", got, r, cands)


def test_mutant_group_index_off_by_one():
    _bwd_mutant("group off", 11, r"dx: .*group 11, chunk")


def test_mutant_s1_s2_swapped():
    _bwd_mutant("swap s1 s2", 20, r"dx: .*group 20, chunk")


def test_mutant_silu_derivative_omitted():
    _bwd_mutant("no silu grad", 3, r"dx: .*group 3, chunk")


def test_mutant_bf16_affine_double_rounded():
    _bwd_mutant("double round", None, r"dgamma: .*channel", out_bf16=True)


def test_mutant_split_summed_short():
    rows, C = 20480, 64
    x = _rand((rows, C), 25, 1.2, 0.4).to(BF)
    dy = _rand((rows, C), 26).to(BF)
    ref = R.ln_backward(x, dy, None, EPS)
    _, dg, db = emu_ln_backward(x, dy, None, EPS, "split short")
    last = R.colreduce_splits(rows, 1, C) - 1
    with pytest.raises(AssertionError, match=rf"explained by split {last} \(x-"):
        R.check_affine("mutant split short", db, ref.dbeta, ref.cands_b)


def test_mutant_nan():
    rows, C = 333, 768
    x = _rand((rows, C), 27, 1.2, 0.4).to(BF)
    dy = _rand((rows, C), 28).to(BF)
    ref = R.ln_backward(x, dy, None, EPS)
    dx, _, _ = emu_ln_backward(x, dy, None, EPS, "nan")
    with pytest.raises(AssertionError, match=rf"row {rows // 2}, channel {C // 3}.*got nan"):
        G.check("mutant nan", dx, ref.dx, locate=lambda r, c: f"row {r}, channel {c}")
