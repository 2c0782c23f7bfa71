"""fp64 references, allowances and a per-element checker for the GroupNorm(+SiLU) / LayerNorm forward kernels
(csrc/norm.cu) and the GroupNorm backward, LayerNorm backward and column-sum kernels (csrc/train_ops.cu). TEST
INFRASTRUCTURE ONLY: importable without a GPU, used by test_norm_fp64_cpu.py (which proves the checker's sensitivity on
fp32 emulations of the kernels' reduction orders) and test_norm_fp64_gpu.py.

References are computed in fp64 from the exact bf16 / fp32 operands the kernel was given: GroupNorm
y = act(gamma (x - mu) rho + beta) with rho = 1 / sqrt(var + eps) per (sample, group); its backward dx / dgamma / dbeta
(with the SiLU derivative when fused); LayerNorm forward and backward per row; the grouped column sums. The backward
references use the fp64 statistics of x, i.e. the true gradient; the kernel's use of the fp32 forward statistics it was
handed is covered by the allowance (their measured distance from the fp64 statistics is carried through the formula).

Allowances, first order, in the style of gemm_fp64_ref:
  - Sums. Every fixed-order fp32 sum gets SUM_REL = 2^-16 of the sum of its terms' magnitudes. The longest serial chains
    are about 200 adds: the rendezvous GroupNorm's per-thread pixel loop (<= 128 pixels of a VAE chunk) + 32 row slots
    + 64 chunks; the column reduction's per-thread rows (<= 213) + 8 row lanes + the split fold; the GroupNorm
    backward's per-thread pixels + row slots + 16 chunks per fold lane + 4 lanes. Linear worst-case growth is
    n 2^-24 < 2^-16 for n <= 256, so the allowance holds without assuming random rounding.
  - Variance. The GroupNorm kernels sum (x - pivot) and (x - pivot)^2 with the pivot taken from the data (each channel's
    value at the first pixel of each chunk / cluster rank), and merge (count, mean, M2) triples with Chan's formula
    relative to the first part's mean. The reference recomputes those pivots exactly for the plan that ran, so the
    cancellation of sum (x - pivot)^2 against (mean - pivot)^2 enters the variance allowance with its real factor.
    LayerNorm is two-pass about its fp32 mean: the mean's error enters only squared.
  - Statistics bound. |mu_k - mu| <= dmu and |rho_k / rho - 1| <= drho for every (sample, group): the sharp detectors
    (a dropped 1/64 of the pixels moves rho by 1/128, hundreds of drho).
  - Per element. dmu, drho and the sum allowances are carried through the formula (for the backward: S1 = sum gamma dz,
    S2 = sum gamma dz xhat and the xhat recomputed from fp32 statistics), plus ARITH_REL = 2^-20 of the magnitudes
    involved for the fp32 arithmetic, rsqrtf and the approximate __expf.
  - Bounds: bf16 outputs |got - ref| <= halfulp_bf16(|ref| + E) + E; fp32 outputs (dgamma / dbeta, column sums)
    E + 2^-22 |ref|; bf16 dgamma / dbeta the bf16 bound on the same E (gemm_fp64_ref.bound).

The worst-ratio statistic of gemm_fp64_ref.check is kept with P = E, so WORST holds (|got - ref| - output rounding) / E:
at most 1 for anything that passes, and how far under 1 it stays is how much of the allowance the kernel uses.

On failure the report names the worst element (sample, pixel, channel, group) and its chunk / cluster rank under the plan
that ran, the worst group's statistic errors in units of dmu / drho, and the reduction units (chunk, row slot, fold lane,
split) whose own partial sums best explain the error (`attribute`).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Callable, List, Optional, Sequence, Tuple

import torch

import gemm_fp64_ref as G

SUM_REL = 2.0 ** -16
ARITH_REL = 2.0 ** -20
RND = 2.0 ** -24         # one fp32 rounding
SILU2 = 0.5              # max |silu''|
NUM_SMS = 132            # kNumSms (csrc/common.cuh): the grid caps below
WORST = G.WORST


# ------------------------------------------------------------------------------------------------ kernel geometry
def gn_chunks(HW: int, NB: int) -> int:
    """Chunks per sample of the rendezvous forward (gn_chunks) and of the backward (gn_bwd_chunks): the same rule."""
    return max(1, min((HW + 15) // 16, 64, (NUM_SMS * 2) // max(NB, 1)))


def colreduce_splits(rows_per_group: int, groups: int, C: int) -> int:
    slabs = (C + 63) // 64
    s = (NUM_SMS * 2) // max(slabs * groups, 1)
    return max(1, min(s, (rows_per_group + 63) // 64, 64))


@dataclass
class Plan:
    """A GroupNorm forward launch: kernel 1 = rendezvous, 2 = cluster of `cs` CTAs over slices of `sc` channels."""
    kernel: int
    cs: int = 0
    sc: int = 0

    def parts(self, HW: int, NB: int) -> List[Tuple[int, int]]:
        """[begin, end) pixel range of each chunk (rendezvous) / rank (cluster); end <= begin is an empty part."""
        if self.kernel == 1:
            k = gn_chunks(HW, NB)
            ppc = -(-HW // k)
            return [(c * ppc, min(HW, (c + 1) * ppc)) for c in range(k)]
        rpc = -(-HW // self.cs)
        return [(min(HW, r * rpc), min(HW, min(HW, r * rpc) + rpc)) for r in range(self.cs)]

    def row_slots(self, C: int) -> int:
        return 512 // ((C if self.kernel == 1 else self.sc) // 8)

    def unit(self) -> str:
        return "chunk" if self.kernel == 1 else "rank"

    def __str__(self):
        return "rendezvous" if self.kernel == 1 else f"cluster {self.cs} x {self.sc} ch"


def bwd_parts(HW: int, NB: int) -> List[Tuple[int, int]]:
    return Plan(1).parts(HW, NB)


def part_of(parts: Sequence[Tuple[int, int]], pix: int) -> int:
    for k, (b, e) in enumerate(parts):
        if b <= pix < e:
            return k
    return -1


# ------------------------------------------------------------------------------------------------ attribution
def attribute(resid: torch.Tensor, cands: Sequence[Tuple[str, torch.Tensor]], top: int = 4) -> str:
    """Which reduction units explain an error: resid is got - ref of a reduced quantity, each candidate the change that
    counting its unit once more would make. Ranks units by |<c, r>| / |c| (the part of the error along c) and reports
    the best with the coefficient <c, r> / <c, c> (-1: the unit is missing, +1: it is counted twice)."""
    r = torch.nan_to_num(resid.double().flatten(), nan=0.0, posinf=0.0, neginf=0.0)
    scored = []
    for name, c in cands:
        c = c.double().flatten().to(r.device)
        nn = float((c * c).sum())
        if nn <= 0.0:
            continue
        dot = float((c * r).sum())
        scored.append((abs(dot) / math.sqrt(nn), dot / nn, name))
    scored.sort(key=lambda t: -t[0])
    return "explained by " + ", ".join(f"{n} (x{coef:+.2f})" for _, coef, n in scored[:top]) if scored else "no unit"


# ------------------------------------------------------------------------------------------------ GroupNorm forward
def act_grad_silu(z):
    s = torch.sigmoid(z)
    return s * (1.0 + z * (1.0 - s))


@dataclass
class GnStats:
    mu: torch.Tensor          # [NB, G] fp64
    rho: torch.Tensor
    dmu: torch.Tensor         # absolute allowance
    drho: torch.Tensor        # relative allowance
    parts: List[Tuple[int, int]] = field(default_factory=list)
    cands: Optional[Callable[[], list]] = None   # attribution candidates of the mean's error


def gn_stats(x: torch.Tensor, groups: int, eps: float, plan: Plan) -> GnStats:
    """fp64 statistics of x [NB, HW, C] and their allowance under `plan`'s parts, pivots and Chan merge."""
    X = x.double()
    NB, HW, C = X.shape
    cpg = C // groups
    Xg = X.reshape(NB, HW, groups, cpg)
    mu = Xg.mean((1, 3))
    var = (Xg - mu[:, None, :, None]).square().mean((1, 3))
    rho = 1.0 / torch.sqrt(var + eps)
    parts = plan.parts(HW, NB)
    cnt = float(cpg * HW)
    e_m0 = mean0 = None
    ta = tb = e_ta = e_tb = sa = sb = 0.0
    for k, (b, e) in enumerate(parts):
        n = max(e - b, 0)
        if n == 0:
            continue  # a zero-count partial: contributes nothing, and the kernel writes {0, 0}
        seg = X[:, b:e, :]
        piv = seg[:, 0, :]
        D = seg - piv[:, None, :]
        a, A, B = D.sum(1), D.abs().sum(1), D.square().sum(1)
        t = piv + a / n
        e_t = SUM_REL * A / n + ARITH_REL * (piv.abs() + a.abs() / n)
        tg = t.reshape(NB, groups, cpg)
        mean_k = tg.mean(-1)
        e_mk = (e_t.reshape(NB, groups, cpg).sum(-1) + SUM_REL * tg.abs().sum(-1)) / cpg + ARITH_REL * mean_k.abs()
        d = tg - mean_k[..., None]
        e_d = e_t.reshape(NB, groups, cpg) + e_mk[..., None] + ARITH_REL * tg.abs()
        ag, Bg = a.reshape(NB, groups, cpg), B.reshape(NB, groups, cpg)
        term = (Bg - ag * ag / n) + n * d * d
        e_term = (SUM_REL * Bg + 2 * ag.abs() * SUM_REL * A.reshape(NB, groups, cpg) / n + ARITH_REL * (Bg + ag * ag / n)
                  + n * (2 * d.abs() * e_d + e_d * e_d) + ARITH_REL * n * d * d)
        m2 = term.sum(-1)
        e_m2 = e_term.sum(-1) + SUM_REL * term.abs().sum(-1)
        if mean0 is None:
            mean0, e_m0 = mean_k, e_mk
        ck = cpg * n
        Dk = mean_k - mean0
        e_D = e_mk + e_m0 + ARITH_REL * mean_k.abs()
        ta, e_ta, sa = ta + ck * Dk, e_ta + ck * e_D, sa + (ck * Dk).abs()
        tbk = m2 + ck * Dk * Dk
        tb, e_tb, sb = tb + tbk, e_tb + e_m2 + ck * (2 * Dk.abs() * e_D + e_D * e_D), sb + tbk.abs()
    e_ta = e_ta + SUM_REL * sa
    e_tb = e_tb + SUM_REL * sb
    dm = ta / cnt
    e_mu = e_m0 + e_ta / cnt + ARITH_REL * (mean0.abs() + dm.abs())
    e_var = (e_tb + 2 * dm.abs() * e_ta) / cnt + ARITH_REL * (tb.abs() + (ta * dm).abs()) / cnt
    drho = e_var / (2 * (var + eps)) + ARITH_REL
    return GnStats(mu, rho, e_mu, drho, parts, lambda: gn_mean_cands(X, mu, mean0, groups, plan, parts))


def gn_mean_cands(X, mu, mean0, groups, plan, parts):
    """Attribution candidates for a wrong mean, each as the kernel's merge would see it: a part counted once more adds
    its pixels' deviation from the first part's mean; a row slot or pixel of part k its deviation from part k's pivots;
    an empty part given its nominal count adds that count at mean 0 (built only when a check fails)."""
    NB, HW, C = X.shape
    cpg = C // groups
    cnt = float(cpg * HW)
    slots = plan.row_slots(C)
    gsum = lambda t: t.reshape(NB, -1, groups, cpg).sum((1, 3)) / cnt
    cands = []
    for k, (b, e) in enumerate(parts):
        if e <= b:
            cands.append((f"empty {plan.unit()} {k}", -(-HW // len(parts)) * cpg * (0.0 - mean0) / cnt))
            continue
        piv = X[:, b:b + 1]
        cands.append((f"{plan.unit()} {k}", gsum(X[:, b:e]) - (e - b) * cpg * mean0 / cnt))
        cands.append((f"{plan.unit()} {k} last pixel", gsum(X[:, e - 1:e] - piv)))
        for s in range(min(slots, e - b)):
            cands.append((f"{plan.unit()} {k} row slot {s}", gsum(X[:, b + s:e:slots] - piv)))
    return cands


def gn_forward(x, gamma, beta, groups: int, eps: float, silu: bool, plan: Plan,
               st: Optional[GnStats] = None) -> Tuple[G.Ref, GnStats]:
    """-> (Ref of y [NB HW, C], the statistics with their allowance; `st` reuses gn_stats of the same x and plan)."""
    st = st or gn_stats(x, groups, eps, plan)
    X = x.double()
    NB, HW, C = X.shape
    cpg = C // groups
    ga = gamma.double().reshape(1, 1, C) if gamma is not None else torch.ones(1, 1, C, dtype=torch.float64, device=X.device)
    be = beta.double().reshape(1, 1, C) if beta is not None else torch.zeros(1, 1, C, dtype=torch.float64, device=X.device)
    per_c = lambda t: t.repeat_interleave(cpg, dim=1)[:, None, :]  # [NB, G] -> [NB, 1, C]
    mu, rho, dmu, drho = per_c(st.mu), per_c(st.rho), per_c(st.dmu), per_c(st.drho)
    xh = (X - mu) * rho
    zz = xh * ga + be
    e_z = ga.abs() * (xh.abs() * drho + rho * dmu) + ARITH_REL * ((X * rho * ga).abs() + be.abs() + (mu * rho * ga).abs()
                                                                + zz.abs())
    if silu:
        y = zz * torch.sigmoid(zz)
        E = G.ACT_SLOPE * e_z + ARITH_REL * y.abs() * (1.0 + zz.abs())
    else:
        y, E = zz, e_z
    y, E = y.reshape(-1, C), E.reshape(-1, C)
    return G.Ref(y, E, E), st


def gn_locate(HW: int, C: int, groups: int, parts, unit: str, st: Optional[GnStats] = None, stats_got=None):
    """locate(row, col) for G.check over [NB HW, C] GroupNorm tensors."""
    def f(row, col):
        n, p = divmod(row, HW)
        g = col // (C // groups)
        s = f"sample {n}, pixel {p}, channel {col}, group {g}, {unit} {part_of(parts, p)}"
        if st is not None and stats_got is not None:
            rm, rr = _stat_ratios(st, stats_got)
            s += f"; that group's mean error {float(rm[n, g]):.2f} dmu, rstd error {float(rr[n, g]):.2f} drho"
        return s
    return f


def _stat_ratios(st: GnStats, stats_got):
    sg = stats_got.detach().to(st.mu.device, torch.float64).reshape(*st.mu.shape, 2)
    rm = (sg[..., 0] - st.mu).abs() / st.dmu
    rr = (sg[..., 1] / st.rho - 1.0).abs() / st.drho
    return torch.nan_to_num(rm, nan=math.inf), torch.nan_to_num(rr, nan=math.inf)


def check_gn_stats(name: str, stats_got, st: GnStats, *, family: Optional[str] = None, cfg: str = "") -> float:
    """|mu_k - mu| <= dmu and |rho_k / rho - 1| <= drho for every (sample, group). Returns the worst ratio."""
    rm, rr = _stat_ratios(st, stats_got)
    worst = float(torch.maximum(rm, rr).max())
    if family is not None:
        WORST[family + " stats"] = max(WORST.get(family + " stats", -math.inf), worst)
    if worst <= 1.0:
        return worst
    w = torch.maximum(rm, rr)
    n, g = divmod(int(torch.argmax(w)), w.shape[1])
    sg = stats_got.detach().to(st.mu.device, torch.float64).reshape(*st.mu.shape, 2)
    why = attribute(sg[..., 0] - st.mu, st.cands())
    raise AssertionError(
        f"{name}: statistics out of bound [launch {cfg or '?'}]: worst sample {n} group {g}: mean {float(sg[n, g, 0])!r} vs "
        f"{float(st.mu[n, g])!r} ({float(rm[n, g]):.2f} dmu), rstd {float(sg[n, g, 1])!r} vs {float(st.rho[n, g])!r} "
        f"({float(rr[n, g]):.2f} drho); {int((w > 1).sum())} of {w.numel()} groups out; mean error {why}")


def check_gn_forward(name: str, y, stats_got, ref: G.Ref, st: GnStats, plan: Plan, groups: int, *, family=None,
                     cfg: str = "") -> float:
    NB, G_ = st.mu.shape
    C = ref.ref.shape[1]
    HW = ref.ref.shape[0] // NB
    if stats_got is not None:
        check_gn_stats(name, stats_got, st, family=family, cfg=cfg)
    return G.check(name, y, ref, family=family, cfg=cfg or str(plan),
                   locate=gn_locate(HW, C, groups, st.parts, plan.unit(), st, stats_got))


# ------------------------------------------------------------------------------------------------ GroupNorm backward
@dataclass
class GnBwdRef:
    dx: G.Ref
    dgamma: G.Ref
    dbeta: G.Ref
    parts: List[Tuple[int, int]]
    cands_b: List[Tuple[str, torch.Tensor]]   # attribution of dbeta's error
    cands_a: List[Tuple[str, torch.Tensor]]   # attribution of dgamma's error


def gn_backward(x, dy, gamma, beta, groups: int, eps: float, silu: bool, stats_given, *, affine_bf16=False) -> GnBwdRef:
    """The true gradient of y = act(gamma xhat + beta) at x (fp64 statistics); the allowance carries the distance of the
    fp32 statistics the kernel was handed (`stats_given` [NB, G, 2]) from them. Sample by sample (memory)."""
    NB, HW, C = x.shape
    dev = x.device
    cpg = C // groups
    m = float(HW * cpg)
    parts = bwd_parts(HW, NB)
    ga = gamma.double().reshape(1, C) if gamma is not None else torch.ones(1, C, dtype=torch.float64, device=dev)
    be = beta.double().reshape(1, C) if beta is not None else torch.zeros(1, C, dtype=torch.float64, device=dev)
    sg = stats_given.detach().to(dev, torch.float64).reshape(NB, groups, 2)
    dxs, Edxs = [], []
    A = torch.zeros(NB, C, dtype=torch.float64, device=dev)
    B, EA, EB = torch.zeros_like(A), torch.zeros_like(A), torch.zeros_like(A)
    chunk_a = torch.zeros(NB, len(parts), C, dtype=torch.float64, device=dev)
    chunk_b = torch.zeros_like(chunk_a)
    pid = torch.zeros(HW, dtype=torch.long, device=dev)
    for k, (b, e) in enumerate(parts):
        if e > b:
            pid[b:e] = k
    rep = lambda t: t.repeat_interleave(cpg).reshape(1, C)
    for n in range(NB):
        X = x[n].double().reshape(HW, C)
        DY = dy[n].double().reshape(HW, C)
        Xg = X.reshape(HW, groups, cpg)
        mu_g = Xg.mean((0, 2))
        rho_g = 1.0 / torch.sqrt((Xg - mu_g[None, :, None]).square().mean((0, 2)) + eps)
        e_mu_g = (sg[n, :, 0] - mu_g).abs() + RND * sg[n, :, 0].abs()
        e_rho_g = (sg[n, :, 1] / rho_g - 1.0).abs() + RND
        mu, rho, e_mu, e_rho = rep(mu_g), rep(rho_g), rep(e_mu_g), rep(e_rho_g)
        xh = (X - mu) * rho
        e_xh = xh.abs() * e_rho + rho * e_mu + ARITH_REL * ((X * rho).abs() + (mu * rho).abs() + xh.abs())
        zz = xh * ga + be
        if silu:
            e_z = ga.abs() * e_xh + ARITH_REL * ((xh * ga).abs() + be.abs())
            dz = DY * act_grad_silu(zz)
            e_dz = DY.abs() * (SILU2 * e_z + ARITH_REL * (1.0 + zz.abs()))
        else:
            dz, e_dz = DY, torch.zeros_like(DY)
        a_t = dz * xh
        a, b = a_t.sum(0), dz.sum(0)
        ea = SUM_REL * a_t.abs().sum(0) + (dz.abs() * e_xh + e_dz * xh.abs()).sum(0)
        eb = SUM_REL * dz.abs().sum(0) + e_dz.sum(0)
        A[n], B[n], EA[n], EB[n] = a, b, ea, eb
        chunk_a[n].index_add_(0, pid, a_t)
        chunk_b[n].index_add_(0, pid, dz)
        S1 = (ga[0] * b).reshape(groups, cpg).sum(-1) / m
        S2 = (ga[0] * a).reshape(groups, cpg).sum(-1) / m
        E1 = ((ga[0].abs() * eb).reshape(groups, cpg).sum(-1) + SUM_REL * (ga[0] * b).abs().reshape(groups, cpg).sum(-1)) / m
        E2 = ((ga[0].abs() * ea).reshape(groups, cpg).sum(-1) + SUM_REL * (ga[0] * a).abs().reshape(groups, cpg).sum(-1)) / m
        E1, E2 = E1 + ARITH_REL * S1.abs(), E2 + ARITH_REL * S2.abs()
        S1, S2, E1, E2 = rep(S1), rep(S2), rep(E1), rep(E2)
        dxv = rho * (dz * ga - S1 - xh * S2)
        E = (dxv.abs() * e_rho + rho * (ga.abs() * e_dz + E1 + e_xh * S2.abs() + xh.abs() * E2)
             + ARITH_REL * rho * ((dz * ga).abs() + S1.abs() + (xh * S2).abs()))
        dxs.append(dxv)
        Edxs.append(E)
    dxr = torch.cat(dxs, 0)
    Edx = torch.cat(Edxs, 0)
    dg, db = A.sum(0), B.sum(0)
    Edg = EA.sum(0) + SUM_REL * A.abs().sum(0)
    Edb = EB.sum(0) + SUM_REL * B.abs().sum(0)
    out32 = not affine_bf16
    cands_b = [(f"chunk {k}", chunk_b[:, k].sum(0)) for k in range(len(parts))]
    cands_b += [(f"fold lane {l}", chunk_b[:, l::4].sum((0, 1))) for l in range(4)]
    cands_a = [(f"chunk {k}", chunk_a[:, k].sum(0)) for k in range(len(parts))]
    cands_a += [(f"fold lane {l}", chunk_a[:, l::4].sum((0, 1))) for l in range(4)]
    return GnBwdRef(G.Ref(dxr, Edx, Edx), G.Ref(dg.reshape(1, C), Edg.reshape(1, C), Edg.reshape(1, C), out32),
                    G.Ref(db.reshape(1, C), Edb.reshape(1, C), Edb.reshape(1, C), out32), parts, cands_b, cands_a)


def check_affine(name: str, got, ref: G.Ref, cands, *, family=None, cfg: str = "") -> float:
    """A reduced [C] output (dgamma / dbeta / column sums): per element, and on failure the units that explain it."""
    C = ref.ref.shape[-1]
    try:
        return G.check(name, got, ref, family=family, cfg=cfg, locate=lambda r, c: f"channel {c}")
    except AssertionError as e:
        g = got.detach().reshape(-1, C).to(ref.ref.device, torch.float64)
        raise AssertionError(f"{e}; error {attribute(g - ref.ref, cands)}") from None


# ------------------------------------------------------------------------------------------------ LayerNorm
def _ln_stats(X, eps):
    C = X.shape[1]
    mu = X.mean(1, keepdim=True)
    d = X - mu
    var = d.square().mean(1, keepdim=True)
    rho = 1.0 / torch.sqrt(var + eps)
    e_mu = SUM_REL * X.abs().sum(1, keepdim=True) / C + ARITH_REL * mu.abs()
    e_var = (SUM_REL * d.square().sum(1, keepdim=True) + C * e_mu * e_mu) / C + ARITH_REL * var
    drho = e_var / (2 * (var + eps)) + ARITH_REL
    return mu, rho, e_mu, drho


def ln_forward(x, gamma, beta, eps: float, block: int = 8192) -> G.Ref:
    """x [rows, C] (any row stride) -> Ref of y [rows, C]."""
    C = x.shape[-1]
    X2 = x.reshape(-1, C)
    dev = x.device
    ga = gamma.double().reshape(1, C) if gamma is not None else torch.ones(1, C, dtype=torch.float64, device=dev)
    be = beta.double().reshape(1, C) if beta is not None else torch.zeros(1, C, dtype=torch.float64, device=dev)
    ys, Es = [], []
    for r0 in range(0, X2.shape[0], block):
        X = X2[r0:r0 + block].double()
        mu, rho, e_mu, drho = _ln_stats(X, eps)
        xh = (X - mu) * rho
        y = xh * ga + be
        E = ga.abs() * (xh.abs() * drho + rho * e_mu) + ARITH_REL * ((xh * ga).abs() + be.abs() + y.abs())
        ys.append(y)
        Es.append(E)
    y, E = torch.cat(ys), torch.cat(Es)
    return G.Ref(y, E, E)


@dataclass
class LnBwdRef:
    dx: G.Ref
    dgamma: Optional[G.Ref]
    dbeta: Optional[G.Ref]
    cands_b: List[Tuple[str, torch.Tensor]]
    cands_a: List[Tuple[str, torch.Tensor]]


def ln_backward(x, dy, gamma, eps: float, *, affine_bf16=False, block: int = 4096) -> LnBwdRef:
    """The true gradient of y = gamma xhat + beta per row; dgamma = sum_r dy xhat, dbeta = sum_r dy over all rows."""
    C = x.shape[-1]
    X2, D2 = x.reshape(-1, C), dy.reshape(-1, C)
    rows = X2.shape[0]
    dev = x.device
    ga = gamma.double().reshape(1, C) if gamma is not None else torch.ones(1, C, dtype=torch.float64, device=dev)
    splits = colreduce_splits(rows, 1, C)
    span = -(-rows // splits)
    sid = (torch.arange(rows, device=dev) // span)
    dxs, Es = [], []
    dg = torch.zeros(C, dtype=torch.float64, device=dev)
    db, Edg, Edb, mag_g, mag_b = (torch.zeros_like(dg) for _ in range(5))
    split_a = torch.zeros(splits, C, dtype=torch.float64, device=dev)
    split_b = torch.zeros_like(split_a)
    for r0 in range(0, rows, block):
        X, DY = X2[r0:r0 + block].double(), D2[r0:r0 + block].double()
        mu, rho, e_mu, drho = _ln_stats(X, eps)
        xh = (X - mu) * rho
        e_xh = xh.abs() * drho + rho * e_mu + ARITH_REL * ((X - mu).abs() * rho + xh.abs())
        g = DY * ga
        s1 = g.mean(1, keepdim=True)
        s2 = (g * xh).mean(1, keepdim=True)
        E1 = SUM_REL * g.abs().sum(1, keepdim=True) / C + ARITH_REL * s1.abs()
        E2 = (SUM_REL * (g * xh).abs().sum(1, keepdim=True) + (g.abs() * e_xh).sum(1, keepdim=True)) / C + ARITH_REL * s2.abs()
        dxv = rho * (g - s1 - xh * s2)
        E = (dxv.abs() * drho + rho * (E1 + e_xh * s2.abs() + xh.abs() * E2)
             + ARITH_REL * rho * (g.abs() + s1.abs() + (xh * s2).abs()))
        dxs.append(dxv)
        Es.append(E)
        at = DY * xh
        dg += at.sum(0)
        db += DY.sum(0)
        Edg += (DY.abs() * e_xh).sum(0)
        mag_g += at.abs().sum(0)
        mag_b += DY.abs().sum(0)
        split_a.index_add_(0, sid[r0:r0 + block], at)
        split_b.index_add_(0, sid[r0:r0 + block], DY)
    Edg = Edg + SUM_REL * mag_g + ARITH_REL * mag_g
    Edb = SUM_REL * mag_b
    out32 = not affine_bf16
    dxr, Edx = torch.cat(dxs), torch.cat(Es)
    return LnBwdRef(G.Ref(dxr, Edx, Edx), G.Ref(dg.reshape(1, C), Edg.reshape(1, C), Edg.reshape(1, C), out32),
                    G.Ref(db.reshape(1, C), Edb.reshape(1, C), Edb.reshape(1, C), out32),
                    [(f"split {s}", split_b[s]) for s in range(splits)], [(f"split {s}", split_a[s]) for s in range(splits)])


# ------------------------------------------------------------------------------------------------ column sums
def colsum(x, rows_per_group: int, *, out_bf16=False) -> Tuple[G.Ref, list]:
    """x [rows, C] -> sums of each consecutive group of rows_per_group rows [groups, C]; candidates: each split of each
    group."""
    C = x.shape[-1]
    X = x.reshape(-1, C).double()
    groups = X.shape[0] // rows_per_group
    Xg = X.reshape(groups, rows_per_group, C)
    ref = Xg.sum(1)
    E = SUM_REL * Xg.abs().sum(1)
    splits = colreduce_splits(rows_per_group, groups, C)
    span = -(-rows_per_group // splits)
    cands = []
    for s in range(splits):
        c = torch.zeros_like(ref)
        c[:, :] = Xg[:, s * span:(s + 1) * span].sum(1)
        cands.append((f"split {s}", c))
    return G.Ref(ref, E, E, not out_bf16), cands
