"""GPU: the wgmma GEMM / implicit-GEMM conv3x3 / upsample-phase conv kernel (csrc/gemm_tc.cu) element by element against
fp64 references (tests/gemm_fp64_ref.py), in every kernel variant, epilogue form, split count and pixel-box class.

Every output element must lie within halfulp_bf16(|ref| + E) + E of the fp64 reference (fp32 outputs: E + 2^-22 |ref|),
E = 2^-16 (|A| |W|^T)[r, c] carried through the epilogue; outputs are written into sentinel-filled buffers and
everything outside the written view must keep the sentinel. Configurations are forced through imagd_gemm_debug_force
(always restored to the automatic choice) and the configuration that ran is read back from imagd_gemm_debug_log.

  a. the 8 kernels (N tile 64 / 128 / 160 / 256, shallow and deep operand ring) x splits {1, 2, 3, 7} x each epilogue
     form, on a ragged GEMM (M 300, N 648, K 1000: a partial last k-block) and a ragged conv (3 x 12 x 9, Cin 192,
     Cout 328); at splits 1 the eight kernels' outputs are compared bit for bit;
  b. every pixel-box class and border, the row vector staged in shared memory (<= 4 groups per tile) and read from
     global memory (> 4), GEMM rows_per_group 16 / 77 / 128 / 1000;
  c. degenerate extents; d. strided operands (and the conv wrappers' output-stride regression);
  e. the step's, the training step's and the VAE attention's product shapes at the automatic choice;
  f. split-K arrival counters re-arming; g. the LayerNorm-fold statistics under forced N tiles; h. the upsample-phase
     conv in every kernel.

The module prints the worst (|got - ref| - output rounding allowance) / P per family at its end (with -s), the ratio
the 2^-16 allowance is a bound for. Measured on an H100 80GB HBM3 (700 W power limit, 1980 MHz max SM clock), whole file
in about 65 s:

  a. matrix 2.8e-7   b. geometry 1.0e-7   c. degenerate <= 0   d. strided 3.5e-8   f. split-K 3.3e-8
  g. LayerNorm fold 5.1e-8   h. upsample-phase conv 6.4e-8
  e. step shapes 7.2e-7, training wgrad (K up to 8192) 2.1e-7, conv dgrad 4.4e-7, VAE S = Q K^T (fp32 out) 2.9e-7,
     VAE P V (K 5120) 5.6e-7

The worst, 7.2e-7 = 2^-20.4, is 21x under the allowance: the tensor core's accumulation costs a few bits over IEEE fp32
summation (2^-24), nowhere near 2^-16. At splits 1 the eight kernels' outputs were bit-identical for every GEMM and conv
form, so test_matrix_cross_variant_bitwise asserts it.
"""
import math
from contextlib import contextmanager

import pytest
import torch

import gemm_fp64_ref as R

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
VARIANTS = [(64, 4), (64, 8), (128, 3), (128, 6), (160, 3), (160, 5), (256, 2), (256, 4)]
SPLITS = [1, 2, 3, 7]
DEEP = {64: 8, 128: 6, 160: 5, 256: 4}


def _vid(v):
    return f"bn{v[0]}-{'deep' if DEEP[v[0]] == v[1] else 'shallow'}"


def _rand(shape, dev, seed, scale=1.0, offset=0.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale + offset).to(dev)


def _lib():
    from imagdressing_b200 import _lib

    return _lib.load()


@contextmanager
def forced(bn=0, stages=0, splits=0):
    lib = _lib()
    assert lib.imagd_gemm_debug_force(bn, stages, splits) == 0
    try:
        yield
    finally:
        lib.imagd_gemm_debug_force(0, 0, 0)


def launch(fn):
    """Run fn (one kernel launch) with the launch log on -> (its result, the logged configuration dict, the log line)."""
    lib = _lib()
    lib.imagd_gemm_debug_log(1, None, 0)
    try:
        out = fn()
    finally:
        lib.imagd_gemm_debug_log(0, None, 0)
    buf = bytes(4096)
    n = lib.imagd_gemm_debug_log(-1, buf, len(buf))
    line = buf.split(b"\0", 1)[0].decode().strip()
    assert n == 1, f"expected one launch key, got {n}: {line}"
    key, run, count = line.split("|")
    names = ["taps", "NB", "H", "W", "K", "N", "geglu", "m_tiles", "kb", "out_fp32"]
    cfg = dict(zip(names, map(int, key.split())))
    cfg.update(zip(["bn", "stages", "splits"], map(int, run.split())))
    assert int(count) == 1
    return out, cfg, line


def split_count(kb_total, forced_splits):
    """Splits a launch runs with when `forced_splits` are asked for: never more than k-blocks, and no empty split."""
    s = min(forced_splits, kb_total)
    kps = -(-kb_total // s)
    return -(-kb_total // kps)


def check_cfg(cfg, variant, splits, kb_total):
    """The launch ran the forced (N tile, stages) and the split count the forced splits come to."""
    assert (cfg["bn"], cfg["stages"]) == tuple(variant), cfg
    assert cfg["splits"] == split_count(kb_total, splits), (cfg, split_count(kb_total, splits))


@pytest.fixture(scope="module", autouse=True)
def _report():
    R.WORST.clear()
    yield
    print("\nworst (|got - ref| - output rounding) / P per family (bound: 2^-16 = 1.53e-05):")
    for fam, v in sorted(R.WORST.items()):
        print(f"  {fam:24s} {v: .3e}   ({'<= 0: within the output rounding' if v <= 0 else f'2^{math.log2(v):.1f}'})")
    if _BITWISE:
        print("cross-variant bitwise at splits 1: " + ", ".join(f"{k}: {v}" for k, v in sorted(_BITWISE.items())))


_BITWISE = {}
_cache = {}


# ================================================================================= a. variant x epilogue matrix
GM, GN, GK, GRPG = 300, 648, 1000, 77
CONV = (3, 12, 9, 192, 328)
FORMS = ["linear", "silu", "gelu", "quick_gelu", "fp32_residual"]
ACTS = {"linear": "none", "silu": "silu", "gelu": "gelu", "quick_gelu": "quick_gelu", "fp32_residual": "none"}


def _gemm_inputs(dev):
    if "gemm" not in _cache:
        a = _rand((GM, GK), dev, 1).to(BF)
        w = _rand((GN, GK), dev, 2, GK ** -0.5).to(BF)
        bias, rowvec = _rand((GN,), dev, 3), _rand((-(-GM // GRPG), GN), dev, 4)
        res = _rand((GM, GN), dev, 5).to(BF)
        _cache["gemm"] = (a, w, bias, rowvec, res)
    return _cache["gemm"]


def _gemm_form(dev, form):
    """(run, reference) of one epilogue form on the matrix GEMM; run() writes a sentinel-prefilled buffer."""
    from imagdressing_b200 import ops

    a, w, bias, rowvec, res = _gemm_inputs(dev)
    key = ("gemm", form)
    fp32 = form == "fp32_residual"
    kw = dict(bias=bias, residual=res) if fp32 else dict(bias=bias, rowvec=rowvec, rows_per_group=GRPG, residual=res,
                                                          alpha=0.75)
    if key not in _cache:
        _cache[key] = R.gemm(a, w, act=ACTS[form], out_fp32=fp32, **{k: v for k, v in kw.items()})
    act = {"none": ops.ACT_NONE, "silu": ops.ACT_SILU, "gelu": ops.ACT_GELU, "quick_gelu": ops.ACT_QUICK_GELU}[ACTS[form]]

    def run():
        out = R.sentinel_buffer((GM, GN), torch.float32 if fp32 else BF, dev)
        return ops.gemm(a, w, out=out, act=act, out_fp32=fp32, **kw)

    return run, _cache[key]


def _conv_inputs(dev):
    if "conv" not in _cache:
        NB, H, W, Cin, Cout = CONV
        x = _rand((NB, H, W, Cin), dev, 6).to(BF)
        wp = _rand((Cout, 9 * Cin), dev, 7, (9 * Cin) ** -0.5).to(BF)
        bias, temb = _rand((Cout,), dev, 8), _rand((NB, Cout), dev, 9)
        res = _rand((NB, H, W, Cout), dev, 10).to(BF)
        _cache["conv"] = (x, wp, bias, temb, res)
    return _cache["conv"]


def _conv_form(dev, form):
    from imagdressing_b200 import ops

    x, wp, bias, temb, res = _conv_inputs(dev)
    key = ("conv", form)
    if key not in _cache:
        _cache[key] = R.conv3x3(x, wp, bias=bias, rowvec=temb, residual=res, act=ACTS[form])
    act = {"none": ops.ACT_NONE, "silu": ops.ACT_SILU, "gelu": ops.ACT_GELU, "quick_gelu": ops.ACT_QUICK_GELU}[ACTS[form]]

    def run():
        out = R.sentinel_buffer(x.shape[:3] + (wp.shape[0],), BF, dev)
        return ops.conv3x3(x, wp, out=out, bias=bias, rowvec=temb, residual=res, act=act)

    return run, _cache[key]


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("splits", SPLITS, ids=lambda s: f"splits{s}")
@pytest.mark.parametrize("variant", VARIANTS, ids=_vid)
def test_matrix_gemm(cuda_device, variant, splits, form):
    run, ref = _gemm_form(cuda_device, form)
    with forced(*variant, splits):
        out, cfg, line = launch(run)
    check_cfg(cfg, variant, splits, -(-GK // 64))
    R.check(f"gemm {_vid(variant)} splits {splits} {form}", out, ref, bn=variant[0], cfg=line, family="a. matrix")


@pytest.mark.parametrize("form", [f for f in FORMS if f != "fp32_residual"])
@pytest.mark.parametrize("splits", SPLITS, ids=lambda s: f"splits{s}")
@pytest.mark.parametrize("variant", VARIANTS, ids=_vid)
def test_matrix_conv(cuda_device, variant, splits, form):
    run, ref = _conv_form(cuda_device, form)
    with forced(*variant, splits):
        out, cfg, line = launch(run)
    NB, H, W, Cin, _ = CONV
    check_cfg(cfg, variant, splits, 9 * Cin // 64)
    R.check(f"conv {_vid(variant)} splits {splits} {form}", out, ref, bn=variant[0], geom=R.Geom(NB, H, W), cfg=line,
            family="a. matrix")


@pytest.mark.parametrize("splits", SPLITS, ids=lambda s: f"splits{s}")
@pytest.mark.parametrize("variant", [(128, 3), (128, 6), (64, 8), (256, 4)], ids=_vid)
def test_matrix_geglu(cuda_device, variant, splits):
    """GEGLU runs on the 128 tile whatever is forced, and never splits K."""
    from imagdressing_b200 import ops

    a = _rand((GM, GK), cuda_device, 11).to(BF)
    wp = _rand((512, GK), cuda_device, 12, GK ** -0.5).to(BF)
    bias = _rand((512,), cuda_device, 13, 0.3)
    with forced(*variant, splits):
        out, cfg, line = launch(lambda: ops.gemm(a, wp, bias=bias, act=ops.ACT_GEGLU, alpha=0.75,
                                                 out=R.sentinel_buffer((GM, 256), BF, cuda_device)))
    assert cfg["bn"] == 128 and cfg["splits"] == 1 and cfg["geglu"] == 1, line
    if variant[0] == 128:
        assert cfg["stages"] == variant[1]
    R.check(f"geglu {_vid(variant)} splits {splits}", out, R.geglu(a, wp, alpha=0.75, bias=bias), bn=64, cfg=line,
            family="a. matrix")


@pytest.mark.parametrize("op,form", [("gemm", f) for f in FORMS] + [("conv", f) for f in FORMS if f != "fp32_residual"])
def test_matrix_cross_variant_bitwise(cuda_device, op, form):
    """At splits 1 each output element sums the same k16 products in the same order whatever the wgmma N width and
    ring depth, so the eight kernels agree bit for bit."""
    run, _ = (_gemm_form if op == "gemm" else _conv_form)(cuda_device, form)
    outs = []
    for v in VARIANTS:
        with forced(*v, 1):
            outs.append(run())
    same = [torch.equal(outs[0], o) for o in outs]
    _BITWISE[f"{op} {form}"] = "identical" if all(same) else "differ: " + ",".join(
        _vid(v) for v, s in zip(VARIANTS, same) if not s)
    assert all(same), _BITWISE[f"{op} {form}"]


# ================================================================================= b. pixel-box and row-group geometry
# (NB, H, W) -> the box the rule gives, and whether the row vector of a tile is staged (<= 4 samples per tile)
GEOMETRY = [
    ((2, 1, 200), (128, 1, 1), "staged"),    # W >= 128: long rows, ragged in x, two samples
    ((1, 3, 130), (32, 4, 1), "staged"),
    ((1, 64, 64), (64, 2, 1), "staged"),
    ((1, 80, 64), (64, 2, 1), "staged"),     # 640 x 512 latent
    ((1, 64, 80), (16, 8, 1), "staged"),
    ((3, 12, 9), (2, 16, 4), "staged"),      # 768 x 576 deepest level, odd batch
    ((3, 9, 12), (16, 2, 4), "staged"),
    ((1, 20, 16), (16, 8, 1), "staged"),
    ((1, 200, 1), (1, 128, 1), "staged"),
    ((300, 1, 1), (1, 1, 128), "unstaged"),  # a tile spans 128 samples
    ((16, 4, 4), (4, 2, 16), "unstaged"),
    ((7, 3, 5), (8, 2, 8), "unstaged"),
]


def _gid(g):
    (NB, H, W), _, st = g
    return f"{NB}x{H}x{W}-{st}"


@pytest.mark.parametrize("variant", [(0, 0, 0), (160, 3, 2)], ids=["auto", "bn160-shallow-splits2"])
@pytest.mark.parametrize("geom", GEOMETRY, ids=_gid)
def test_geometry_conv(cuda_device, geom, variant):
    from imagdressing_b200 import ops

    (NB, H, W), box, staged = geom
    Cin, Cout = 64, 200
    G = R.Geom(NB, H, W)
    assert G.box() == box
    assert ("staged" if min(box[2], NB) <= 4 else "unstaged") == staged
    x = _rand((NB, H, W, Cin), cuda_device, 20).to(BF)
    wp = _rand((Cout, 9 * Cin), cuda_device, 21, (9 * Cin) ** -0.5).to(BF)
    bias, temb = _rand((Cout,), cuda_device, 22), _rand((NB, Cout), cuda_device, 23)
    res = _rand((NB, H, W, Cout), cuda_device, 24).to(BF)
    with forced(*variant):
        out, cfg, line = launch(lambda: ops.conv3x3(x, wp, out=R.sentinel_buffer((NB, H, W, Cout), BF, cuda_device),
                                                    bias=bias, rowvec=temb, residual=res))
    assert cfg["m_tiles"] == G.m_tiles(), (line, box)
    R.check(f"conv {NB}x{H}x{W}", out, R.conv3x3(x, wp, bias=bias, rowvec=temb, residual=res), bn=cfg["bn"], geom=G,
            cfg=line, family="b. geometry")


@pytest.mark.parametrize("variant", [(0, 0, 0), (64, 8, 3)], ids=["auto", "bn64-deep-splits3"])
@pytest.mark.parametrize("rpg", [16, 77, 128, 1000])
def test_geometry_gemm_row_groups(cuda_device, rpg, variant):
    """rows_per_group 16: a 128-row tile spans 8 groups (row vector read from global memory); 77 / 128 / 1000: staged."""
    from imagdressing_b200 import ops

    M, N, K = 1000, 200, 320
    a = _rand((M, K), cuda_device, 25).to(BF)
    w = _rand((N, K), cuda_device, 26, K ** -0.5).to(BF)
    rowvec = _rand((-(-M // rpg), N), cuda_device, 27)
    with forced(*variant):
        out, cfg, line = launch(lambda: ops.gemm(a, w, rowvec=rowvec, rows_per_group=rpg, act=ops.ACT_SILU,
                                                 out=R.sentinel_buffer((M, N), BF, cuda_device)))
    R.check(f"gemm rows_per_group {rpg}", out, R.gemm(a, w, rowvec=rowvec, rows_per_group=rpg, act="silu"),
            bn=cfg["bn"], cfg=line, family="b. geometry")


# ================================================================================= c. degenerate extents
DEGENERATE = [(1, 8, 8), (129, 64, 64), (200, 8, 320), (300, 136, 72)]


@pytest.mark.parametrize("variant", [(0, 0, 0), (256, 4, 1), (64, 8, 3)], ids=["auto", "bn256-deep", "bn64-deep-splits3"])
@pytest.mark.parametrize("M,N,K", DEGENERATE, ids=lambda v: str(v))
def test_degenerate_extents(cuda_device, M, N, K, variant):
    from imagdressing_b200 import ops

    a = _rand((M, K), cuda_device, 30).to(BF)
    w = _rand((N, K), cuda_device, 31, K ** -0.5).to(BF)
    bias, res = _rand((N,), cuda_device, 32), _rand((M, N), cuda_device, 33).to(BF)
    buf = R.sentinel_buffer((M + 2, N + 16), BF, cuda_device)
    view = buf[1:M + 1, 8:N + 8]
    with forced(*variant):
        _, cfg, line = launch(lambda: ops.gemm(a, w, out=view, bias=bias, residual=res))
    R.check(f"gemm {M}x{N}x{K}", view, R.gemm(a, w, bias=bias, residual=res), bn=cfg["bn"], cfg=line,
            family="c. degenerate")
    R.assert_outside_untouched(f"gemm {M}x{N}x{K}", buf, (slice(1, M + 1), slice(8, N + 8)))


# ================================================================================= d. strided operands
@pytest.mark.parametrize("variant", [(0, 0, 0), (128, 3, 3), (256, 2, 1)], ids=["auto", "bn128-shallow-splits3",
                                                                                 "bn256-shallow"])
@pytest.mark.parametrize("out_kind", ["column_slice", "row_block"])
def test_strided_gemm(cuda_device, variant, out_kind):
    """A and W as column slices (lda, ldw > K), residual with ldr != N, rowvec with rowvec_ld > N, and the output as a
    column slice or as rows [r0, r0 + M) of a taller, wider buffer."""
    from imagdressing_b200 import ops

    M, N, K, rpg = 300, 328, 200, 128
    dev = cuda_device
    a = _rand((M, K + 40), dev, 40).to(BF)[:, 24:24 + K]
    w = _rand((N, K + 16), dev, 41, K ** -0.5).to(BF)[:, 8:8 + K]
    res = _rand((M, N + 24), dev, 42).to(BF)[:, 16:16 + N]
    rowvec = _rand((3, N + 12), dev, 43)[:, 8:8 + N]
    bias = _rand((N,), dev, 44)
    assert a.stride(0) > K and w.stride(0) > K and res.stride(0) != N and rowvec.stride(0) > N
    if out_kind == "column_slice":
        buf, index = R.sentinel_buffer((M, N + 40), BF, dev), (slice(None), slice(32, 32 + N))
    else:
        buf, index = R.sentinel_buffer((M + 77, N + 8), BF, dev), (slice(40, 40 + M), slice(0, N))
    view = buf[index]
    with forced(*variant):
        _, cfg, line = launch(lambda: ops.gemm(a, w, out=view, bias=bias, rowvec=rowvec, rows_per_group=rpg,
                                               residual=res, alpha=1.5))
    ref = R.gemm(a, w, bias=bias, rowvec=rowvec, rows_per_group=rpg, residual=res, alpha=1.5)
    R.check(f"strided gemm ({out_kind})", view, ref, bn=cfg["bn"], cfg=line, family="d. strided")
    R.assert_outside_untouched(f"strided gemm ({out_kind})", buf, index)


@pytest.mark.parametrize("sliced", ["out", "x-out-residual"])
@pytest.mark.parametrize("variant", [(0, 0, 0), (64, 4, 2)], ids=["auto", "bn64-shallow-splits2"])
def test_conv_into_a_channel_slice_of_a_wider_buffer(cuda_device, variant, sliced):
    """Regression: ops.conv3x3 passed out.shape[-1] as the output's pixel stride, so writing into channels
    [64, 64 + Cout) of a wider NHWC buffer (an up block's concat buffer) put every pixel but the first in the wrong
    place, over the neighbouring channels. Also the input and the residual as channel slices (ldx > Cin, ldr > Cout)."""
    from imagdressing_b200 import ops

    NB, H, W, Cin, Cout = 2, 10, 7, 64, 136
    dev = cuda_device
    x = _rand((NB, H, W, Cin + 128), dev, 50).to(BF)[..., 64:64 + Cin]
    res = _rand((NB, H, W, Cout + 16), dev, 51).to(BF)[..., 8:8 + Cout]
    if sliced == "out":
        x, res = x.contiguous(), res.contiguous()
    wp = _rand((Cout, 9 * Cin), dev, 52, (9 * Cin) ** -0.5).to(BF)
    bias, temb = _rand((Cout,), dev, 53), _rand((NB + 1, Cout + 24), dev, 54)[:, 8:8 + Cout]
    buf = R.sentinel_buffer((NB, H, W, 64 + Cout + 32), BF, dev)
    index = (Ellipsis, slice(64, 64 + Cout))
    with forced(*variant):
        _, cfg, line = launch(lambda: ops.conv3x3(x, wp, out=buf[index], bias=bias, rowvec=temb, residual=res))
    R.check("conv into a channel slice", buf[index], R.conv3x3(x, wp, bias=bias, rowvec=temb, residual=res),
            bn=cfg["bn"], geom=R.Geom(NB, H, W), cfg=line, family="d. strided")
    R.assert_outside_untouched("conv into a channel slice", buf, index)


def test_upconv_into_a_channel_slice_of_a_wider_buffer(cuda_device):
    from imagdressing_b200 import modeling, ops

    NB, H, W, Cin, Cout = 3, 5, 4, 64, 72
    dev = cuda_device
    x = _rand((NB, H, W, Cin + 64), dev, 55).to(BF)[..., 32:32 + Cin]
    wph = modeling.pack_upconv3x3(_rand((Cout, Cin, 3, 3), dev, 56, (9 * Cin) ** -0.5).to(BF))
    b = _rand((Cout,), dev, 57)
    buf = R.sentinel_buffer((NB, 2 * H, 2 * W, Cout + 40), BF, dev)
    index = (Ellipsis, slice(16, 16 + Cout))
    _, cfg, line = launch(lambda: ops.upconv3x3(x, wph, bias=b, out=buf[index]))
    R.check("upconv into a channel slice", buf[index], R.upconv3x3(x, wph, bias=b), bn=cfg["bn"],
            geom=R.Geom(NB, H, W, ups=True), cfg=line, family="d. strided")
    R.assert_outside_untouched("upconv into a channel slice", buf, index)


def test_geglu_rejects_epilogue_terms_it_does_not_apply(cuda_device):
    """The GEGLU epilogue applies bias and alpha only: a row vector, a residual or an fp32 output used to be accepted
    and silently ignored (the fp32 output was never written)."""
    from imagdressing_b200 import _lib, ops

    a = _rand((128, 64), cuda_device, 60).to(BF)
    wp = _rand((128, 64), cuda_device, 61, 0.125).to(BF)
    for kw in (dict(rowvec=torch.zeros(1, 128, device=cuda_device), rows_per_group=128),
               dict(residual=torch.zeros(128, 64, device=cuda_device, dtype=BF)), dict(out_fp32=True)):
        with pytest.raises(_lib.ImagdError, match="GEGLU epilogue takes bias and alpha only"):
            ops.gemm(a, wp, act=ops.ACT_GEGLU, **kw)


# ================================================================================= e. product and training shapes
STEP_CONV = [(2, 64, 64, 320, 320), (2, 32, 32, 640, 640), (2, 16, 16, 1280, 1280), (2, 16, 16, 2560, 1280),
             (2, 32, 32, 1920, 640), (2, 8, 8, 1280, 1280)]
STEP_GEMM = [(8192, 320, 320), (8192, 320, 1280), (2048, 640, 640), (2048, 640, 1920), (512, 1280, 5120),
             (512, 3840, 1280), (128, 1280, 5120)]


@pytest.mark.parametrize("NB,H,W,Cin,Cout", STEP_CONV, ids=lambda v: str(v))
def test_product_conv(cuda_device, NB, H, W, Cin, Cout):
    from imagdressing_b200 import ops

    x = _rand((NB, H, W, Cin), cuda_device, 70).to(BF)
    wp = _rand((Cout, 9 * Cin), cuda_device, 71, (9 * Cin) ** -0.5).to(BF)
    bias, temb = _rand((Cout,), cuda_device, 72), _rand((NB, Cout), cuda_device, 73)
    res = _rand((NB, H, W, Cout), cuda_device, 74).to(BF)
    out, cfg, line = launch(lambda: ops.conv3x3(x, wp, bias=bias, rowvec=temb, residual=res))
    R.check(f"step conv {NB}x{H}x{W} {Cin}->{Cout}", out, R.conv3x3(x, wp, bias=bias, rowvec=temb, residual=res),
            bn=cfg["bn"], geom=R.Geom(NB, H, W), cfg=line, family="e. step")


@pytest.mark.parametrize("M,N,K", STEP_GEMM, ids=lambda v: str(v))
def test_product_gemm(cuda_device, M, N, K):
    from imagdressing_b200 import ops

    a = _rand((M, K), cuda_device, 75).to(BF)
    w = _rand((N, K), cuda_device, 76, K ** -0.5).to(BF)
    bias, res = _rand((N,), cuda_device, 77), _rand((M, N), cuda_device, 78).to(BF)
    out, cfg, line = launch(lambda: ops.gemm(a, w, bias=bias, residual=res))
    R.check(f"step gemm {M}x{N}x{K}", out, R.gemm(a, w, bias=bias, residual=res), bn=cfg["bn"], cfg=line,
            family="e. step")


@pytest.mark.parametrize("M,C", [(8192, 320), (512, 1280)])
def test_product_geglu(cuda_device, M, C):
    from imagdressing_b200 import ops

    a = _rand((M, C), cuda_device, 79).to(BF)
    wp = _rand((8 * C, C), cuda_device, 80, C ** -0.5).to(BF)
    bias = _rand((8 * C,), cuda_device, 81, 0.1)
    out, cfg, line = launch(lambda: ops.gemm(a, wp, bias=bias, act=ops.ACT_GEGLU))
    R.check(f"step geglu {M}x{C}", out, R.geglu(a, wp, bias=bias), bn=64, cfg=line, family="e. step")


@pytest.mark.parametrize("NB,H,W,C", [(2, 16, 16, 1280), (2, 32, 32, 640)])
def test_product_upconv(cuda_device, NB, H, W, C):
    from imagdressing_b200 import modeling, ops

    x = _rand((NB, H, W, C), cuda_device, 82).to(BF)
    wph = modeling.pack_upconv3x3(_rand((C, C, 3, 3), cuda_device, 83, (9 * C) ** -0.5).to(BF))
    b = _rand((C,), cuda_device, 84)
    out, cfg, line = launch(lambda: ops.upconv3x3(x, wph, bias=b))
    R.check(f"step upconv {NB}x{H}x{W}x{C}", out, R.upconv3x3(x, wph, bias=b), bn=cfg["bn"],
            geom=R.Geom(NB, H, W, ups=True), cfg=line, family="e. step")


@pytest.mark.parametrize("level,NB,H,W,Cin,Cout", [(0, 2, 64, 64, 320, 320), (3, 2, 8, 8, 1280, 1280)],
                         ids=["level0", "level3"])
def test_training_wgrad(cuda_device, level, NB, H, W, Cin, Cout):
    """The training step's weight gradients: linear gemm(transpose(dY), transpose(X)) and conv
    gemm(transpose(dY), im2col3x3_t(X)), K = the (padded) token count; checked from the operands the GEMM read, after
    checking that those are exact transposes / patches."""
    from imagdressing_b200 import ops

    dev = cuda_device
    T = NB * H * W
    x = _rand((NB, H, W, Cin), dev, 85).to(BF)
    dy = _rand((NB, H, W, Cout), dev, 86, 1e-3).to(BF)
    dy2, x2 = dy.view(T, Cout), x.view(T, Cin)
    dyt, xt = ops.transpose(dy2), ops.transpose(x2)
    assert torch.equal(dyt[:, :T], dy2.t()) and torch.equal(xt[:, :T], x2.t())
    dw, cfg, line = launch(lambda: ops.gemm(dyt, xt))
    R.check(f"linear wgrad level {level} (K {T})", dw, R.gemm(dyt, xt), bn=cfg["bn"], cfg=line,
            family="e. training wgrad")
    cols = ops.im2col3x3_t(x)
    patches = torch.nn.functional.unfold(x.permute(0, 3, 1, 2).float(), 3, padding=1)  # [NB, Cin * 9, HW], c-major
    patches = patches.view(NB, Cin, 9, H * W).permute(2, 1, 0, 3).reshape(9 * Cin, T)  # tap-major rows
    assert torch.equal(cols[:9 * Cin, :T].float(), patches)
    dwc, cfg, line = launch(lambda: ops.gemm(dyt, cols))
    R.check(f"conv wgrad level {level} (K {T}, N {cols.shape[0]})", dwc, R.gemm(dyt, cols), bn=cfg["bn"], cfg=line,
            family="e. training wgrad")


def test_training_conv_dgrad(cuda_device):
    from imagdressing_b200 import ops

    NB, H, W, Cin, Cout = 2, 32, 32, 640, 640
    dev = cuda_device
    wp = _rand((Cout, 9 * Cin), dev, 87, (9 * Cin) ** -0.5).to(BF)
    wf = ops.conv_weight_flip(wp, Cin)
    assert torch.equal(wf.view(Cin, 9, Cout), wp.view(Cout, 9, Cin).permute(2, 1, 0).flip(1))
    dy = _rand((NB, H, W, Cout), dev, 88).to(BF)
    dx, cfg, line = launch(lambda: ops.conv3x3(dy, wf))
    R.check("conv dgrad", dx, R.conv3x3(dy, wf), bn=cfg["bn"], geom=R.Geom(NB, H, W), cfg=line,
            family="e. training dgrad")


def test_vae_attention_products(cuda_device):
    """The VAE mid-block attention at a 640 x 512 image (80 x 64 latent, 5120 tokens, C 512): S = Q K^T to fp32
    (K 512), then P V (K 5120) on the bf16 probabilities softmax_rows wrote."""
    from imagdressing_b200 import ops

    L, C = 5120, 512
    dev = cuda_device
    q, k = _rand((L, C), dev, 89).to(BF), _rand((L, C), dev, 90).to(BF)
    vt = _rand((C, L), dev, 91).to(BF)
    s, cfg, line = launch(lambda: ops.gemm(q, k, out_fp32=True))
    R.check("vae S = Q K^T", s, R.gemm(q, k, out_fp32=True), bn=cfg["bn"], cfg=line, family="e. vae fp32 S")
    prob = ops.softmax_rows(s, 1.0 / math.sqrt(C))
    o, cfg, line = launch(lambda: ops.gemm(prob, vt))
    R.check("vae P V", o, R.gemm(prob, vt), bn=cfg["bn"], cfg=line, family="e. vae P V")


# ================================================================================= f. split-K state
def test_splitk_counters_rearm_across_launches(cuda_device):
    """Two split-K launches with different tile counts, then a third identical to the first: the per-tile arrival
    counters must be back at zero after each launch, or the third one reduces early or never."""
    from imagdressing_b200 import ops

    dev = cuda_device
    a1, w1 = _rand((300, 1000), dev, 92).to(BF), _rand((648, 1000), dev, 93, 0.03).to(BF)
    a2, w2 = _rand((1000, 2000), dev, 94).to(BF), _rand((200, 2000), dev, 95, 0.02).to(BF)
    with forced(128, 6, 3):
        first, c1, _ = launch(lambda: ops.gemm(a1, w1))
        second, c2, _ = launch(lambda: ops.gemm(a2, w2))
        third = ops.gemm(a1, w1)
        repeats = [ops.gemm(a2, w2) for _ in range(3)]
    assert c1["splits"] == 3 and c2["splits"] == 3 and c1["m_tiles"] != c2["m_tiles"]
    assert torch.equal(first, third)
    assert all(torch.equal(second, r) for r in repeats)
    R.check("split-K first", first, R.gemm(a1, w1), family="f. split-K")
    R.check("split-K second", second, R.gemm(a2, w2), family="f. split-K")


def test_auto_splitk_repeat_runs_are_bitwise_equal(cuda_device):
    from imagdressing_b200 import ops

    a, w = _rand((128, 5120), cuda_device, 96).to(BF), _rand((1280, 5120), cuda_device, 97, 0.014).to(BF)
    out, cfg, _ = launch(lambda: ops.gemm(a, w))
    assert cfg["splits"] > 1, cfg  # the automatic choice splits this shape (few tiles, long K)
    assert all(torch.equal(out, ops.gemm(a, w)) for _ in range(3))


# ================================================================================= g. LayerNorm fold under forced N tiles
LN_M, LN_C = 300, 648


@pytest.mark.parametrize("splits", [1, 3], ids=lambda s: f"splits{s}")
@pytest.mark.parametrize("bn", [64, 128, 160, 256], ids=lambda b: f"bn{b}")
def test_ln_producer_slots(cuda_device, bn, splits):
    """One statistics slot per N tile of the launch, each the sum / sum of squares of the kernel's own rounded outputs
    over that tile's columns (the last slot over the ragged remainder)."""
    from imagdressing_b200 import ops

    dev = cuda_device
    M, N, K = LN_M, LN_C, 320
    a, w = _rand((M, K), dev, 100).to(BF), _rand((N, K), dev, 101, K ** -0.5).to(BF)
    bias, res = _rand((N,), dev, 102), _rand((M, N), dev, 103, 1.0, 1.5).to(BF)
    with forced(bn, 0, splits):
        parts = ops.gemm_tile_count_n(M, N, K)
        assert parts == -(-N // bn)
        stats = torch.full((M, parts + 1, 2), float("nan"), device=dev)
        y, cfg, line = launch(lambda: ops.gemm(a, w, bias=bias, residual=res, stats_out=stats))
    assert cfg["bn"] == bn
    R.check(f"ln producer bn {bn}", y, R.gemm(a, w, bias=bias, residual=res), bn=bn, cfg=line, family="g. ln fold")
    assert torch.isnan(stats[:, parts]).all()  # the slot past the launch's tiles stays untouched
    yd = y.double()
    for j in range(parts):
        blk = yd[:, j * bn:(j + 1) * bn]
        for q, (want, mag) in enumerate(((blk.sum(1), blk.abs().sum(1)), (blk.square().sum(1), blk.square().sum(1)))):
            got = stats[:, j, q].double()
            lim = 256 * 2.0 ** -24 * mag + 1e-30  # fp32 summation of <= 256 terms
            assert bool(((got - want).abs() <= lim).all()), (bn, j, q, float(((got - want).abs() - lim).max()))


@pytest.mark.parametrize("splits", [1, 3], ids=lambda s: f"splits{s}")
@pytest.mark.parametrize("bn,act", [(64, "none"), (128, "none"), (160, "none"), (256, "none"), (128, "geglu")],
                         ids=lambda v: str(v))
def test_ln_consumer(cuda_device, bn, act, splits):
    from imagdressing_b200 import ops

    dev = cuda_device
    M, C = LN_M, 640
    a0, w0 = _rand((M, C), dev, 104).to(BF), _rand((C, C), dev, 105, C ** -0.5).to(BF)
    res = _rand((M, C), dev, 106, 1.0, 1.5).to(BF)
    parts = ops.gemm_tile_count_n(M, C, C)
    stats = torch.zeros(M, parts, 2, device=dev)
    x = ops.gemm(a0, w0, residual=res, stats_out=stats)  # the raw residual stream and its statistics (automatic tiles)
    N = 1280 if act == "geglu" else 648
    wp = _rand((N, C), dev, 107, C ** -0.5).to(BF)
    bias = _rand((N,), dev, 108, 0.1)
    colsum = wp.double().sum(1).float()
    ln = ops.LnFold(stats, parts, C, 1e-5, colsum)
    with forced(bn, 0, splits):
        out, cfg, line = launch(lambda: ops.gemm(x, wp, bias=bias, ln=ln, alpha=0.5,
                                                 act=ops.ACT_GEGLU if act == "geglu" else ops.ACT_NONE))
    assert cfg["bn"] == bn
    ref = R.ln_consumer(x, wp, stats, C, 1e-5, colsum, bias, alpha=0.5, act=act)
    R.check(f"ln consumer bn {bn} {act}", out, ref, bn=64 if act == "geglu" else bn, cfg=line, family="g. ln fold")


# ================================================================================= h. upsample-phase conv
@pytest.mark.parametrize("NB,H,W", [(3, 10, 8), (1, 12, 9), (3, 5, 3)], ids=lambda v: str(v))
@pytest.mark.parametrize("variant", VARIANTS, ids=_vid)
def test_upconv_variants(cuda_device, variant, NB, H, W):
    from imagdressing_b200 import modeling, ops

    Cin, Cout = 128, 200
    dev = cuda_device
    x = _rand((NB, H, W, Cin), dev, 110).to(BF)
    wph = modeling.pack_upconv3x3(_rand((Cout, Cin, 3, 3), dev, 111, (9 * Cin) ** -0.5).to(BF))
    b = _rand((Cout,), dev, 112)
    with forced(*variant, 3):
        out, cfg, line = launch(lambda: ops.upconv3x3(x, wph, bias=b,
                                                      out=R.sentinel_buffer((NB, 2 * H, 2 * W, Cout), BF, dev)))
    assert (cfg["bn"], cfg["stages"], cfg["splits"]) == (variant[0], variant[1], 1), line
    R.check(f"upconv {_vid(variant)} {NB}x{H}x{W}", out, R.upconv3x3(x, wph, bias=b), bn=variant[0],
            geom=R.Geom(NB, H, W, ups=True), cfg=line, family="h. upconv")
