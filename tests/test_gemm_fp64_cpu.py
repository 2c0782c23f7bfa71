"""CPU: the per-element fp64 checker of tests/gemm_fp64_ref.py against an emulation of the GEMM / conv3x3 kernel.

The emulation does what csrc/gemm_tc.cu does, in torch on the CPU: exact bf16 products accumulated in fp32 in chunks of
k = 16 (one wgmma k-step), 64-wide k-blocks dealt out to split-K partials that are summed in split order, the epilogue
in fp32, one rounding to bf16. It must pass the bound for every epilogue form at K = 8 ... 16384. Each mutant below is a
bug this kernel could have; the checker must fail it and, where the bug sits in one tile, name that tile.
"""
import math

import pytest
import torch
import torch.nn.functional as F

import gemm_fp64_ref as R

BF = torch.bfloat16


def _rand(shape, seed, scale=1.0, offset=0.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(shape, generator=g) * scale + offset


# ------------------------------------------------------------------------------------------------------ the emulation
def emu_partials(a, w, splits=1):
    """fp32 split-K partials of a [M, K] @ w[N, K]^T in k16 chunks; the kernel's split rule (no empty splits)."""
    K = a.shape[1]
    kb_total = -(-K // R.KBLOCK)
    kps = -(-kb_total // splits)
    splits = -(-kb_total // kps)
    af, wf = a.float(), w.float()
    parts = []
    for s in range(splits):
        acc = torch.zeros(a.shape[0], w.shape[0])
        for k0 in range(s * kps * R.KBLOCK, min(K, (s + 1) * kps * R.KBLOCK), 16):
            acc += af[:, k0:k0 + 16] @ wf[:, k0:k0 + 16].t()
        parts.append(acc)
    return parts


def emu_sum(parts):
    acc = torch.zeros_like(parts[0])
    for p in parts:
        acc += p
    return acc


def emu_act(f, act):
    if act == "silu":
        return F.silu(f)
    if act == "gelu":
        return F.gelu(f)
    if act == "quick_gelu":
        return f * torch.sigmoid(1.702 * f)
    return f


def emu_epilogue(acc, *, alpha=1.0, bias=None, rowvec_rows=None, residual=None, act="none", out_fp32=False):
    f = alpha * acc
    if bias is not None:
        f = f + bias
    if rowvec_rows is not None:
        f = f + rowvec_rows
    f = emu_act(f, act)
    if residual is not None:
        f = f + residual.float()
    return f if out_fp32 else f.to(BF)


def emu_geglu(acc, *, bias=None):
    M, N = acc.shape
    f = acc + (bias if bias is not None else 0.0)
    v = f.reshape(M, N // 128, 2, 64)[:, :, 0].reshape(M, N // 2)
    g = f.reshape(M, N // 128, 2, 64)[:, :, 1].reshape(M, N // 2)
    return (v * F.gelu(g)).to(BF)


def emu_conv_acc(x, wp):
    """fp32 accumulation of the implicit-GEMM conv in the kernel's order: tap-major k-blocks, k16 chunks."""
    NB, H, W, Cin = x.shape
    X = F.pad(x.float(), (0, 0, 1, 1, 1, 1))
    wf = wp.float()
    acc = torch.zeros(NB * H * W, wp.shape[0])
    for tap in range(9):
        ky, kx = divmod(tap, 3)
        xs = X[:, ky:ky + H, kx:kx + W, :].reshape(-1, Cin)
        for k0 in range(0, Cin, 16):
            acc += xs[:, k0:k0 + 16] @ wf[:, tap * Cin + k0:tap * Cin + k0 + 16].t()
    return acc


# ------------------------------------------------------------------------------------------------------ fixtures
M, N = 160, 256  # two 128-row tiles (the second ragged); N % 128 == 0 for the GEGLU form
RPG = 77         # rows per row-vector group: the groups straddle the tile boundary
_cache = {}


def _gemm_case(K):
    if K not in _cache:
        a = _rand((M, K), 1).to(BF)
        w = _rand((N, K), 2, K ** -0.5).to(BF)
        _cache[K] = (a, w, emu_partials(a, w))
    return _cache[K]


def _epi_inputs():
    bias = _rand((N,), 3)
    rowvec = _rand((-(-M // RPG), N), 4)
    res = _rand((M, N), 5).to(BF)
    return bias, rowvec, res


EPILOGUES = ["linear", "silu", "gelu", "quick_gelu", "fp32_residual", "geglu", "ln_linear", "ln_geglu"]


def _run_clean(form, K):
    """(got, ref) of the emulated kernel and the fp64 reference for one epilogue form."""
    a, w, parts = _gemm_case(K)
    acc = emu_sum(parts)
    bias, rowvec, res = _epi_inputs()
    rv_rows = rowvec[torch.arange(M) // RPG]
    if form == "linear":
        got = emu_epilogue(acc, alpha=0.75, bias=bias, rowvec_rows=rv_rows, residual=res)
        return got, R.gemm(a, w, alpha=0.75, bias=bias, rowvec=rowvec, rows_per_group=RPG, residual=res)
    if form in ("silu", "gelu", "quick_gelu"):
        got = emu_epilogue(acc, bias=bias, act=form)
        return got, R.gemm(a, w, bias=bias, act=form)
    if form == "fp32_residual":
        got = emu_epilogue(acc, bias=bias, residual=res, out_fp32=True)
        return got, R.gemm(a, w, bias=bias, residual=res, out_fp32=True)
    if form == "geglu":
        return emu_geglu(acc, bias=bias * 0.1), R.geglu(a, w, bias=bias * 0.1)
    # LayerNorm-folded consumer: `a` is the raw residual stream; its statistics come in 3 column slots
    stats = torch.stack([torch.stack([a.float()[:, s].sum(1), a.float()[:, s].square().sum(1)], -1)
                         for s in torch.arange(K).tensor_split(3)], 1)
    colsum = w.float().sum(1)
    s = stats.sum(1)
    mean = s[:, :1] / K
    rstd = torch.rsqrt((s[:, 1:] / K - mean * mean).clamp_min(0) + 1e-5)
    f = rstd * (acc - mean * colsum) + bias * 0.1
    if form == "ln_linear":
        got = f.to(BF)
    else:
        v = f.reshape(M, N // 128, 2, 64)[:, :, 0].reshape(M, N // 2)
        g = f.reshape(M, N // 128, 2, 64)[:, :, 1].reshape(M, N // 2)
        got = (v * F.gelu(g)).to(BF)
    ref = R.ln_consumer(a, w, stats, K, 1e-5, colsum, bias * 0.1, act="geglu" if form == "ln_geglu" else "none")
    return got, ref


@pytest.mark.parametrize("K", [8, 72, 1000, 2880, 16384])
@pytest.mark.parametrize("form", EPILOGUES)
def test_emulated_kernel_passes(form, K):
    got, ref = _run_clean(form, K)
    R.check(f"emulated {form} K={K}", got, ref, bn=64 if "geglu" in form else 128)


@pytest.mark.parametrize("K", [8, 320, 2880, 16384])
@pytest.mark.parametrize("splits", [1, 3])
def test_fp32_accumulation_error_is_far_below_the_allowance(K, splits):
    """IEEE fp32 accumulation in k16 chunks stays near 2^-24 P: the 2^-16 allowance leaves ~250x for the tensor core."""
    a, w = _rand((64, K), 6).to(BF), _rand((64, K), 7, K ** -0.5).to(BF)
    acc = emu_sum(emu_partials(a, w, splits)).double()
    A, W = a.double(), w.double()
    worst = float(((acc - A @ W.t()).abs() / (A.abs() @ W.abs().t())).max())
    assert worst < 2.0 ** -21, worst


def test_emulated_conv_passes():
    x = _rand((3, 12, 9, 64), 8).to(BF)
    wp = _rand((200, 9 * 64), 9, (9 * 64) ** -0.5).to(BF)
    bias, temb, res = _rand((200,), 10), _rand((3, 200), 11), _rand((3, 12, 9, 200), 12).to(BF)
    acc = emu_conv_acc(x, wp)
    got = emu_epilogue(acc, bias=bias, rowvec_rows=temb.repeat_interleave(108, 0), residual=res.reshape(-1, 200))
    R.check("emulated conv", got, R.conv3x3(x, wp, bias=bias, rowvec=temb, residual=res), geom=R.Geom(3, 12, 9))


# ------------------------------------------------------------------------------------------------------ mutants
def _fails(fn, match):
    with pytest.raises(AssertionError, match=match) as e:
        fn()
    print(str(e.value).splitlines()[0])


@pytest.mark.parametrize("K", [1000, 2880, 16384])
def test_mutant_dropped_k_block_in_one_tile(K):
    a, w, parts = _gemm_case(K)
    acc = emu_sum(parts)
    rows, cols, kb = slice(128, 160), slice(128, 256), 1  # tile (m 1, n 1), second k-block
    k = slice(kb * 64, min(K, kb * 64 + 64))
    acc[rows, cols] -= a.float()[rows, k] @ w.float()[cols, k].t()
    got = emu_epilogue(acc)
    _fails(lambda: R.check("dropped k-block", got, R.gemm(a, w)), r"tile \(m 1, n 1\)")


def test_mutant_dropped_split_partial_in_one_tile():
    a, w, _ = _gemm_case(1000)
    parts = emu_partials(a, w, 7)
    assert len(parts) == 6  # 16 k-blocks, 3 per split: the "no empty splits" clamp
    rows, cols = slice(0, 128), slice(0, 128)
    parts[4][rows, cols] = 0.0
    got = emu_epilogue(emu_sum(parts))
    _fails(lambda: R.check("dropped split-K partial", got, R.gemm(a, w)), r"tile \(m 0, n 0\)")


def test_mutant_conv_missing_halo_tap_at_a_corner():
    NB, H, W, Cin, Cout = 3, 12, 9, 64, 200
    x = _rand((NB, H, W, Cin), 13).to(BF)
    wp = _rand((Cout, 9 * Cin), 14, (9 * Cin) ** -0.5).to(BF)
    acc = emu_conv_acc(x, wp)
    n, y, xx, tap = 2, H - 1, W - 1, 0  # bottom-right corner of sample 2 without its top-left (in-image) tap
    row = (n * H + y) * W + xx
    acc[row, 128:] -= x.float()[n, y - 1, xx - 1] @ wp.float()[128:, tap * Cin:(tap + 1) * Cin].t()
    geom = R.Geom(NB, H, W)
    m_tile = int(geom.tile_of_rows(torch.tensor([row]))[0])
    assert geom.box() == (2, 16, 4) and m_tile == 4
    got = emu_epilogue(acc)
    _fails(lambda: R.check("conv corner tap", got, R.conv3x3(x, wp), geom=geom), r"tile \(m 4, n 1\)")


def test_mutant_row_with_the_neighbouring_samples_row_vector():
    a, w, parts = _gemm_case(1000)
    _, rowvec, _ = _epi_inputs()
    g = torch.arange(M) // RPG
    g[2 * RPG] = 1  # first row of group 2 (row 154, tile m 1) reads group 1's vector
    got = emu_epilogue(emu_sum(parts), rowvec_rows=rowvec[g])
    _fails(lambda: R.check("row vector", got, R.gemm(a, w, rowvec=rowvec, rows_per_group=RPG)), r"tile \(m 1, n \d\)")


def test_mutant_geglu_value_gate_swapped_in_one_tile():
    a, w, parts = _gemm_case(1000)
    acc = emu_sum(parts)
    sw = acc.clone()
    sw[:128, 128:192], sw[:128, 192:256] = acc[:128, 192:256], acc[:128, 128:192]  # packed tile n 1 of m-tile 0
    _fails(lambda: R.check("geglu swap", emu_geglu(sw), R.geglu(a, w), bn=64), r"tile \(m 0, n 1\)")


def test_mutant_output_rounded_twice():
    a, w, parts = _gemm_case(1000)
    _, _, res = _epi_inputs()
    got = (emu_epilogue(emu_sum(parts)).float() + res.float()).to(BF)  # bf16 GEMM output, then a bf16 residual add
    _fails(lambda: R.check("double rounding", got, R.gemm(a, w, residual=res)), "out of bound")


def test_mutant_column_past_a_ragged_n_edge():
    a, w = _rand((M, 128), 15).to(BF), _rand((200, 128), 16, 128 ** -0.5).to(BF)
    out = emu_epilogue(emu_sum(emu_partials(a, w)))
    buf = R.sentinel_buffer((M, 216), BF, "cpu")
    buf[:, 8:208] = out
    R.check("ragged N", buf[:, 8:208], R.gemm(a, w))
    R.assert_outside_untouched("ragged N", buf, (slice(None), slice(8, 208)))
    buf[128:, 208] = 1.0  # the last (ragged) N tile of m-tile 1 stores one column too many
    _fails(lambda: R.assert_outside_untouched("ragged N", buf, (slice(None), slice(8, 208))), r"\(128, 208\)")


def test_nan_fails():
    a, w, parts = _gemm_case(72)
    got = emu_epilogue(emu_sum(parts))
    got[3, 5] = float("nan")
    _fails(lambda: R.check("nan", got, R.gemm(a, w)), r"row 3, col 5")


# ------------------------------------------------------------------------------------------------------ the references
def test_conv_reference_is_the_convolution():
    x = _rand((2, 7, 5, 16), 17).to(BF)
    w = _rand((24, 16, 3, 3), 18, 0.2).to(BF)
    b = _rand((24,), 19)
    from oracle import ops_ref

    r = R.conv3x3(x, ops_ref.conv3x3_pack(w), bias=b)
    ref = F.conv2d(x.double().permute(0, 3, 1, 2), w.double(), b.double(), padding=1).permute(0, 2, 3, 1)
    assert torch.allclose(r.ref, ref.reshape(-1, 24), rtol=1e-12, atol=1e-12)


def test_geglu_reference_is_the_unpacked_geglu():
    from oracle import ops_ref

    a = _rand((40, 64), 20).to(BF)
    w, b = _rand((256, 64), 21, 0.125).to(BF), _rand((256,), 22, 0.1)
    wp, bp = ops_ref.geglu_pack(w, b)
    h, g = (a.double() @ w.double().t() + b.double()).chunk(2, -1)
    ref = h * 0.5 * g * (1 + torch.erf(g / math.sqrt(2)))
    assert torch.allclose(R.geglu(a, wp, bias=bp).ref, ref, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("NB,H,W", [(1, 4, 4), (3, 5, 3), (2, 1, 1)])
def test_upconv_packing_against_the_conv_of_the_upsampled_input(NB, H, W):
    """Separates "the packing rounds sums of taps to bf16" from "the kernel is wrong": with 3x3 weights whose phase
    sums are exact in bf16 the phase reference of the packed weight IS the conv of the nearest-2x upsampled input (to
    fp64 rounding); with general weights the two differ by at most the bf16 rounding of the packed sums."""
    from imagdressing_b200.modeling import pack_upconv3x3
    from oracle import ops_ref

    Cin, Cout = 64, 32
    x = _rand((NB, H, W, Cin), 23).to(BF)
    up = x.repeat_interleave(2, 1).repeat_interleave(2, 2)
    g = torch.Generator().manual_seed(24)
    w_exact = torch.randint(-8, 9, (Cout, Cin, 3, 3), generator=g).float() / 16  # sums of <= 4 taps: <= 6 bits
    r = R.upconv3x3(x, pack_upconv3x3(w_exact))
    conv = R.conv3x3(up, ops_ref.conv3x3_pack(w_exact))
    assert torch.allclose(r.ref, conv.ref, rtol=0, atol=1e-12 * float(conv.P.max()))
    w = _rand((Cout, Cin, 3, 3), 25, (9 * Cin) ** -0.5).to(BF)
    r, conv = R.upconv3x3(x, pack_upconv3x3(w)), R.conv3x3(up, ops_ref.conv3x3_pack(w))
    assert float(((r.ref - conv.ref).abs() - 2.0 ** -9 * conv.P).max()) <= 0  # packed sums within a half ulp each


@pytest.mark.parametrize("shape,box", [((128, 1, 1), (128, 1, 1)), ((64, 64, 1), (64, 2, 1)), ((80, 64, 1), (16, 8, 1)),
                                       ((9, 12, 3), (2, 16, 4)), ((1, 200, 1), (1, 128, 1)), ((1, 1, 300), (1, 1, 128))])
def test_pixel_box_port(shape, box):
    """The port of the kernel's pixel-box rule that maps rows to m-tiles in failure reports (W, H, NB) -> box."""
    assert R.choose_pixel_box(*shape) == box


# ------------------------------------------------------------------------------------------------------ the conv wrappers
class _RecordingLib:
    """Stands in for the library: records each call's arguments and reports success."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*args):
            self.calls.append((name, args))
            return 0

        return fn


@pytest.fixture
def recording_lib(monkeypatch):
    from imagdressing_b200 import _lib, ops

    lib = _RecordingLib()
    monkeypatch.setattr(_lib, "load", lambda: lib)
    monkeypatch.setattr(ops, "_stream", lambda: 0)
    return lib


def test_conv_wrappers_pass_the_views_pixel_strides(recording_lib):
    """ops.conv3x3 / ops.upconv3x3 hand the kernel the pixel strides of channel-slice views (ldx, ldy, ldr), not their
    channel counts: an output written into channels [64, 64 + Cout) of a wider NHWC buffer lands there."""
    from imagdressing_b200 import ops

    NB, H, W, Cin, Cout = 2, 5, 3, 64, 72
    x = torch.zeros(NB, H, W, Cin + 64, dtype=BF)[..., 32:32 + Cin]
    wp = torch.zeros(Cout, 9 * Cin, dtype=BF)
    buf = torch.zeros(NB, H, W, 64 + Cout + 24, dtype=BF)
    res = torch.zeros(NB, H, W, Cout + 8, dtype=BF)[..., 8:]
    temb = torch.zeros(NB + 1, Cout + 16)[:, 4:4 + Cout]
    ops.conv3x3(x, wp, out=buf[..., 64:64 + Cout], residual=res, rowvec=temb)
    name, args = recording_lib.calls[-1]
    ep = args[10]._obj
    assert name == "imagd_conv3x3_bf16"
    assert args[1] == Cin + 64 and args[2:6] == (NB, H, W, Cin) and args[8] == 64 + Cout + 24 and args[9] == Cout
    assert args[7] == buf[..., 64:].data_ptr() and ep.ldr == Cout + 8 and ep.residual == res.data_ptr()
    assert ep.rowvec_ld == Cout + 16 and ep.rows_per_group == H * W
    up = torch.zeros(NB, 2 * H, 2 * W, Cout + 40, dtype=BF)
    ops.upconv3x3(x, torch.zeros(4 * Cout, 4 * Cin, dtype=BF), out=up[..., 16:16 + Cout])
    name, args = recording_lib.calls[-1]
    assert name == "imagd_upconv3x3_bf16" and args[1] == Cin + 64 and args[8] == Cout + 40


def test_conv_wrappers_reject_views_the_kernel_cannot_address(recording_lib):
    from imagdressing_b200 import ops

    x = torch.zeros(2, 6, 6, 64, dtype=BF)
    wp = torch.zeros(32, 9 * 64, dtype=BF)
    bad = [dict(x=x[:, :, :4]),                                     # a window: rows of pixels not equally spaced
           dict(out=torch.zeros(2, 6, 8, 32, dtype=BF)[:, :, :6]),
           dict(out=torch.zeros(2, 6, 6, 16, dtype=BF)),            # wrong channel count
           dict(rowvec=torch.zeros(1, 32)),                         # fewer rows than samples
           dict(rowvec=torch.zeros(2, 24)),                         # fewer columns than Cout
           dict(residual=torch.zeros(1, 6, 6, 32, dtype=BF))]       # not the output's shape
    for kw in bad:
        args = dict(x=x)
        args.update(kw)
        with pytest.raises(AssertionError):
            ops.conv3x3(args.pop("x"), wp, **args)
    assert recording_lib.calls == []
