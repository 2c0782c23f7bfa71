"""fp64 references and a per-element checker for the wgmma GEMM / implicit-GEMM conv3x3 / upsample-phase conv kernel
(csrc/gemm_tc.cu). TEST INFRASTRUCTURE ONLY: importable without a GPU, used by test_gemm_fp64_cpu.py (which proves the
checker's sensitivity on a CPU emulation of the kernel) and test_gemm_fp64_gpu.py.

References. Every reference is computed in fp64 from the exact bf16 / fp32 operands the kernel was given:
  - GEMM     alpha * A W^T + bias + rowvec[r // rows_per_group], then the activation, then + residual;
  - conv3x3  sum over the nine taps of X_shift(tap) W_tap^T on a zero-padded input (shifted matmuls, no F.conv2d);
  - upsample-phase conv: the four 2x2 phase convs of the PACKED phase weight (modeling.pack_upconv3x3), i.e. what the
    kernel is asked to compute; how far the packing itself is from the 3x3 conv of the upsampled input is a separate test;
  - GEGLU    value * gelu_erf(gate) on the packed layout (per 128 weight rows: 64 value rows, then their 64 gate rows);
  - LayerNorm-fold consumer  rstd * (alpha * acc - mean * colsum) + bias, mean / rstd folded in fp64 from the statistics
    the kernel was given.

Allowance. The kernel multiplies bf16 operands exactly and accumulates in fp32 (tensor-core chunks of k = 16, split-K
partials summed in fp32). IEEE fp32 accumulation in k16 chunks keeps |acc - ref| / P near 2^-24 at K = 8 ... 16384,
with P = (|A| |W|^T)[r, c] (the CPU emulation in test_gemm_fp64_cpu.py measures it). The allowance is E = 2^-16 P: a
factor of about 250 over that for the tensor core's own accumulation order and rounding, which IEEE does not specify.
E is carried through the epilogue: times |alpha|, times 1.13 (a bound on |act'| of SiLU / GELU / quick-GELU), for GEGLU
|gelu(g)| E_a + 1.13 |a| E_g, for the LayerNorm consumer times rstd. The epilogue's own fp32 arithmetic (the adds,
the approximate exp / erf of the activations, the fp32 fold of the statistics) adds 2^-19 of the magnitudes involved,
about 2^-10 of a bf16 half ulp, so it costs the bound no sensitivity.

Bound per element:
  bf16 output   |got - ref| <= halfulp_bf16(|ref| + E) + E  (the half ulp at the upper end: a value on a binade edge)
  fp32 output   |got - ref| <= E + 2^-22 |ref|
A dropped 64-wide k-block moves an element by about |ref| / sqrt(K / 64), hundreds of E: the bound catches it on
nearly every affected element, where a global rel-L2 of 1e-2 lets a whole wrong row through.

On an H100 80GB HBM3 the worst (|got - ref| - output rounding) / P over test_gemm_fp64_gpu.py is 7.2e-7 = 2^-20.4 (its
docstring lists the families): the tensor core keeps the accumulation within a few bits of fp32 summation, so the 2^-16
allowance stands with a factor of about 20 to spare.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Optional, Sequence

import torch

ACC_REL = 2.0 ** -16    # accumulation allowance per unit of P
EPI_REL = 2.0 ** -19    # fp32 epilogue arithmetic per unit of the magnitudes involved
FP32_REL = 2.0 ** -22   # fp32 outputs: the output's own rounding and the epilogue's
ACT_SLOPE = 1.13        # max |act'| of SiLU (1.0998), GELU (1.1289) and quick-GELU (1.0998)
SENTINEL = -1024.0      # prefill of every output buffer; no output of these tests comes near it
KBLOCK = 64             # the kernel's k-block (a split-K partial is a whole number of them)

# worst (|got - ref| - output rounding allowance) / P per test family, filled by check()
WORST: dict = {}


# ------------------------------------------------------------------------------------------------------ activations
def act_fp64(x: torch.Tensor, act: str) -> torch.Tensor:
    if act == "none":
        return x
    if act == "silu":
        return x / (1.0 + torch.exp(-x))
    if act == "gelu":
        return 0.5 * x * (1.0 + torch.erf(x * 0.5 ** 0.5))
    if act == "quick_gelu":
        return x / (1.0 + torch.exp(-1.702 * x))
    raise ValueError(act)


def halfulp_bf16(x: torch.Tensor) -> torch.Tensor:
    """Half a bf16 ulp at |x| (fp64): bf16 keeps 8 significant bits, so for 2^e <= |x| < 2^(e+1) it is 2^(e-8)."""
    x = x.abs()
    _, e = torch.frexp(x)  # x = m 2^e, m in [0.5, 1): floor(log2 x) = e - 1
    h = torch.ldexp(torch.ones_like(x), (e - 9).clamp_min(-133))
    return torch.where(x > 0, h, torch.zeros_like(x))


# ------------------------------------------------------------------------------------------------------ references
@dataclass
class Ref:
    """ref, E (allowance), P (|A| |W|^T of the accumulation) as fp64 [rows, cols]; out_fp32 selects the bound."""
    ref: torch.Tensor
    E: torch.Tensor
    P: torch.Tensor
    out_fp32: bool = False


def _rows(t: Optional[torch.Tensor], rows: int) -> Optional[torch.Tensor]:
    return None if t is None else t.double().reshape(rows, -1)


def epilogue(acc, P, *, alpha=1.0, bias=None, rowvec_rows=None, residual=None, act="none", out_fp32=False) -> Ref:
    """acc / P fp64 [rows, N]; rowvec_rows: the row vector already gathered per row ([rows, N]); residual [rows, N]."""
    f = alpha * acc
    mag = f.abs()
    if bias is not None:
        f = f + bias.double().reshape(1, -1)
        mag = mag + bias.double().abs().reshape(1, -1)
    if rowvec_rows is not None:
        f = f + rowvec_rows
        mag = mag + rowvec_rows.abs()
    E = ACC_REL * abs(alpha) * P
    if act != "none":
        E = ACT_SLOPE * E
        f = act_fp64(f, act)
        mag = mag + f.abs()
    if residual is not None:
        f = f + residual
        mag = mag + residual.abs()
    return Ref(f, E + EPI_REL * mag, P, out_fp32)


def gemm(a, w, *, alpha=1.0, bias=None, rowvec=None, rows_per_group=0, residual=None, act="none",
         out_fp32=False) -> Ref:
    """a [M, K] bf16 (any row stride), w [N, K] bf16, bias [N] / rowvec [groups, >= N] fp32, residual [M, N]."""
    A, W = a.double(), w.double()
    M, N = A.shape[0], W.shape[0]
    acc, P = A @ W.t(), A.abs() @ W.abs().t()
    rv = None
    if rowvec is not None:
        g = torch.arange(M, device=A.device) // rows_per_group
        rv = rowvec.double()[g, :N]
    return epilogue(acc, P, alpha=alpha, bias=bias, rowvec_rows=rv, residual=_rows(residual, M), act=act,
                    out_fp32=out_fp32)


def conv3x3_acc(x, wp):
    """x [NB, H, W, Cin] bf16 (channel-last view), wp [Cout, 9 Cin] tap-major (tap = ky * 3 + kx reads input pixel
    (y + ky - 1, x + kx - 1)) -> (acc, P) fp64 [NB H W, Cout]."""
    NB, H, W, Cin = x.shape
    X = torch.nn.functional.pad(x.double(), (0, 0, 1, 1, 1, 1))
    Wd = wp.double()
    acc = P = 0
    for tap in range(9):
        ky, kx = divmod(tap, 3)
        xs = X[:, ky:ky + H, kx:kx + W, :].reshape(-1, Cin)
        wt = Wd[:, tap * Cin:(tap + 1) * Cin]
        acc = acc + xs @ wt.t()
        P = P + xs.abs() @ wt.abs().t()
    return acc, P


def conv3x3(x, wp, *, bias=None, rowvec=None, residual=None, act="none") -> Ref:
    """ops.conv3x3 / imagd_conv3x3_bf16: rowvec [>= NB, >= Cout] indexed by sample, residual [NB, H, W, Cout]."""
    NB, H, W, _ = x.shape
    Cout = wp.shape[0]
    acc, P = conv3x3_acc(x, wp)
    rv = None
    if rowvec is not None:
        rv = rowvec.double()[:NB, :Cout].repeat_interleave(H * W, 0)
    return epilogue(acc, P, bias=bias, rowvec_rows=rv, residual=_rows(residual, NB * H * W), act=act)


def upconv3x3(x, w_phase, *, bias=None) -> Ref:
    """Four 2x2 phase convs of the packed weight [4 Cout, 4 Cin] (rows phase * Cout + co, phase = py * 2 + px; columns
    tap * Cin + ci, tap = ty * 2 + tx reading input pixel (y + py - 1 + ty, x + px - 1 + tx)) -> output pixel
    (2y + py, 2x + px) of [NB, 2H, 2W, Cout], flattened to rows."""
    NB, H, W, Cin = x.shape
    Cout = w_phase.shape[0] // 4
    X = torch.nn.functional.pad(x.double(), (0, 0, 1, 1, 1, 1))
    Wd = w_phase.double()
    acc = torch.zeros(NB, 2 * H, 2 * W, Cout, dtype=torch.float64, device=x.device)
    P = torch.zeros_like(acc)
    for py in (0, 1):
        for px in (0, 1):
            ph = py * 2 + px
            a = p = 0
            for t in range(4):
                ty, tx = divmod(t, 2)
                xs = X[:, py + ty:py + ty + H, px + tx:px + tx + W, :].reshape(-1, Cin)
                wt = Wd[ph * Cout:(ph + 1) * Cout, t * Cin:(t + 1) * Cin]
                a = a + xs @ wt.t()
                p = p + xs.abs() @ wt.abs().t()
            acc[:, py::2, px::2, :] = a.reshape(NB, H, W, Cout)
            P[:, py::2, px::2, :] = p.reshape(NB, H, W, Cout)
    return epilogue(acc.reshape(-1, Cout), P.reshape(-1, Cout), bias=bias)


def geglu_from_acc(acc, P, *, alpha=1.0, bias=None, ln=None) -> Ref:
    """acc / P [M, N] on the packed layout -> value * gelu_erf(gate) [M, N / 2]. ln: (mean, rstd, colsum, stat_rel) of the
    LayerNorm consumer, applied to value and gate before the GELU."""
    M, N = acc.shape
    f = alpha * acc
    E = ACC_REL * abs(alpha) * P
    mag = f.abs()
    b = bias.double().reshape(1, N) if bias is not None else torch.zeros(1, N, dtype=torch.float64, device=acc.device)
    if ln is not None:
        f, E, mag = _ln_apply(f, E, b, *ln)
    else:
        f = f + b
        mag = mag + b.abs()
    split = lambda t: (t.reshape(M, N // 128, 2, 64)[:, :, 0].reshape(M, N // 2),
                       t.reshape(M, N // 128, 2, 64)[:, :, 1].reshape(M, N // 2))
    (va, ga), (Ea, Eg), (ma, mg) = split(f), split(E), split(mag)
    gg = act_fp64(ga, "gelu")
    out = va * gg
    E_out = gg.abs() * Ea + ACT_SLOPE * va.abs() * Eg + ACT_SLOPE * Ea * Eg
    mag_out = ma + mg + gg.abs() * ma + out.abs()
    Pv, Pg = split(P)
    return Ref(out, E_out + EPI_REL * mag_out, torch.maximum(Pv, Pg))


def geglu(a, wp, *, alpha=1.0, bias=None) -> Ref:
    A, W = a.double(), wp.double()
    return geglu_from_acc(A @ W.t(), A.abs() @ W.abs().t(), alpha=alpha, bias=bias)


def ln_fold_stats(stats: torch.Tensor, dim: int, eps: float):
    """The consumer's mean / rstd from the producer's {sum, sum of squares} partials [M, parts, 2] (fp64), and the
    relative error bound of the kernel's fp32 fold of them (it sums the parts, then E[x^2] - mean^2: the cancellation
    there is amplified by E[x^2] / var)."""
    s = stats.double().sum(1)
    mean = s[:, 0] / dim
    ex2 = s[:, 1] / dim
    var = (ex2 - mean * mean).clamp_min(0.0)
    rstd = 1.0 / torch.sqrt(var + eps)
    cond = ex2 / (var + eps)
    stat_rel = EPI_REL * (stats.shape[1] + 2) * cond
    return mean.reshape(-1, 1), rstd.reshape(-1, 1), stat_rel.reshape(-1, 1)


def _ln_apply(f, E, b, mean, rstd, colsum, stat_rel):
    cs = colsum.double().reshape(1, -1)
    inner = f - mean * cs
    out = rstd * inner + b
    E = rstd * (E + EPI_REL * (f.abs() + (mean * cs).abs())) + stat_rel * rstd * inner.abs()
    return out, E, out.abs() + b.abs()


def ln_consumer(a, w, stats, dim, eps, colsum, bias, *, alpha=1.0, act="none") -> Ref:
    """The LayerNorm-folded consumer GEMM (LINEAR or GEGLU) given the statistics partials the kernel reads."""
    A, W = a.double(), w.double()
    acc, P = A @ W.t(), A.abs() @ W.abs().t()
    mean, rstd, stat_rel = ln_fold_stats(stats, dim, eps)
    if act == "geglu":
        return geglu_from_acc(acc, P, alpha=alpha, bias=bias, ln=(mean, rstd, colsum, stat_rel))
    f, E, mag = _ln_apply(alpha * acc, ACC_REL * abs(alpha) * P, bias.double().reshape(1, -1), mean, rstd, colsum,
                          stat_rel)
    return Ref(f, E + EPI_REL * mag, P)


# ------------------------------------------------------------------------------------------------------ tile geometry
def choose_pixel_box(W: int, H: int, NB: int):
    """The kernel's split of 128 output pixels into a (bw, bh, bn) box of powers of two (choose_pixel_box in
    csrc/gemm_tc.cu): the fewest wasted tile slots, wider boxes on ties."""
    best, box = -1.0, (1, 1, 1)
    w = 1
    while w <= 128:
        h = 1
        while w * h <= 128:
            n = 128 // (w * h)
            tiles = -(-W // w) * -(-H // h) * -(-NB // n)
            eff = W * H * NB / (tiles * 128.0)
            if eff > best + 1e-9 or (eff > best - 1e-9 and w > box[0]):
                best, box = eff, (w, h, n)
            h *= 2
        w *= 2
    return box


@dataclass
class Geom:
    """Output pixel geometry of a launch: a GEMM is (NB, H, W) = (1, 1, M); ups: the rows are the output pixels of the
    upsample-phase conv, [NB, 2H, 2W], tiled over the low-resolution (NB, H, W)."""
    NB: int
    H: int
    W: int
    ups: bool = False

    def box(self):
        return choose_pixel_box(self.W, self.H, self.NB)

    def m_tiles(self):
        bw, bh, bn = self.box()
        return -(-self.W // bw) * -(-self.H // bh) * -(-self.NB // bn)

    def tile_of_rows(self, rows: torch.Tensor):
        """(m-tile, phase) of output rows (int64 tensors; phase is 0 except for the upsample-phase conv)."""
        bw, bh, bn = self.box()
        tiles_x, tiles_y = -(-self.W // bw), -(-self.H // bh)
        if self.ups:
            X2 = rows % (2 * self.W)
            Y2 = (rows // (2 * self.W)) % (2 * self.H)
            n = rows // (4 * self.W * self.H)
            x, y, phase = X2 // 2, Y2 // 2, (Y2 % 2) * 2 + X2 % 2
        else:
            x, y, n = rows % self.W, (rows // self.W) % self.H, rows // (self.W * self.H)
            phase = torch.zeros_like(rows)
        return (x // bw) + tiles_x * ((y // bh) + tiles_y * (n // bn)), phase


# ------------------------------------------------------------------------------------------------------ checking
def bound(r: Ref) -> torch.Tensor:
    if r.out_fp32:
        return r.E + FP32_REL * r.ref.abs()
    return halfulp_bf16(r.ref.abs() + r.E) + r.E


def check(name: str, got: torch.Tensor, r: Ref, *, bn: int = 128, geom: Optional[Geom] = None, cfg: str = "",
          family: Optional[str] = None) -> float:
    """Assert |got - ref| <= bound on every element of got ([rows, cols] after flattening the leading dims); a NaN
    anywhere fails. On failure: the worst element's (row, col), its (m-tile, n-tile) under the launch's pixel box
    (geom; default: 128-row tiles of a GEMM) with `bn` output columns per N tile (64 for GEGLU), the launch
    configuration `cfg` (the imagd_gemm_debug_log line), the worst-tile and the global rel-L2. Returns the worst
    (|got - ref| - output rounding allowance) / P, also kept in WORST[family]."""
    ref = r.ref
    cols = ref.shape[-1]
    g = got.detach().reshape(-1, cols).to(ref.device, torch.float64)
    assert g.shape == ref.shape, f"{name}: shape {tuple(g.shape)} vs reference {tuple(ref.shape)}"
    err = (g - ref).abs()
    lim = bound(r)
    excess = torch.where(torch.isnan(err), torch.full_like(err, math.inf), err - lim)
    rounding = torch.zeros_like(ref) if r.out_fp32 else halfulp_bf16(ref.abs() + r.E)
    ratio = ((err - rounding) / r.P).masked_fill(r.P == 0, -math.inf)
    worst_ratio = float(torch.nan_to_num(ratio, nan=math.inf).max())
    if family is not None:
        WORST[family] = max(WORST.get(family, -math.inf), worst_ratio)
    n_bad = int((excess > 0).sum())
    if n_bad == 0:
        return worst_ratio
    flat = int(torch.argmax(excess))
    row, col = divmod(flat, cols)
    geom = geom or Geom(1, 1, ref.shape[0])
    rows = torch.arange(ref.shape[0], device=ref.device)
    mt, phase = geom.tile_of_rows(rows)
    n_tiles = -(-cols // bn)
    tile_id = (mt * 4 + phase).reshape(-1, 1) * n_tiles + (torch.arange(cols, device=ref.device) // bn).reshape(1, -1)
    d2 = torch.nan_to_num((g - ref).square(), nan=math.inf).flatten()
    r2 = ref.square().flatten()
    nt_total = int(tile_id.max()) + 1
    d2t = torch.zeros(nt_total, dtype=torch.float64, device=ref.device).index_add_(0, tile_id.flatten(), d2)
    r2t = torch.zeros(nt_total, dtype=torch.float64, device=ref.device).index_add_(0, tile_id.flatten(), r2)
    worst_tile = float((d2t / r2t.clamp_min(1e-300)).sqrt().max())
    glob = float((d2.sum() / r2.sum().clamp_min(1e-300)).sqrt())
    ph = int(phase[row])
    where = f"tile (m {int(mt[row])}, n {col // bn})" + (f" phase {ph}" if geom.ups else "")
    raise AssertionError(
        f"{name}: {n_bad} of {err.numel()} elements out of bound; worst at (row {row}, col {col}) in {where} "
        f"[box {geom.box()}, N tile {bn}, launch {cfg or '?'}]: got {float(g[row, col])!r}, ref {float(ref[row, col])!r}, "
        f"bound {float(lim[row, col]):.3e}, E {float(r.E[row, col]):.3e}; worst-tile rel-L2 {worst_tile:.3e}, "
        f"global rel-L2 {glob:.3e}")


def sentinel_buffer(shape: Sequence[int], dtype, device) -> torch.Tensor:
    return torch.full(tuple(shape), SENTINEL, dtype=dtype, device=device)


def assert_outside_untouched(name: str, buf: torch.Tensor, index) -> None:
    """Every element of buf outside buf[index] still holds SENTINEL."""
    rest = buf.detach().clone()
    rest[index] = SENTINEL
    bad = (rest != SENTINEL).nonzero()
    assert bad.shape[0] == 0, (f"{name}: {bad.shape[0]} elements written outside the output view, first at "
                               f"{tuple(int(v) for v in bad[0])}: {float(rest[tuple(bad[0])])!r}")
