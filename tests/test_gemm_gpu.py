"""GPU parity: wgmma GEMM / implicit-GEMM conv3x3 (through the C ABI) vs the fp32 oracle ops.

Tolerance: bf16 inputs, fp32 accumulation, bf16 output -> rel-L2 <= 1e-2 (SURVEY.md §8c); typical is ~3e-3
(one bf16 rounding of the output).
"""
import pytest
import torch

from conftest import rel_l2
from oracle import ops_ref

pytestmark = pytest.mark.gpu
TOL = 1e-2


def _rand(shape, dev, seed, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dev)


@pytest.mark.parametrize(
    "M,N,K",
    [
        (128, 64, 64),      # one tile, one k-block
        (128, 128, 320),    # k tail (320 = 5 x 64)
        (4096, 320, 320),   # level-0 linear
        (4096, 960, 320),   # fused QKV
        (1024, 640, 640),
        (256, 1280, 1280),
        (64, 1280, 1280),   # M < tile (level 3 at batch 1)
        (77, 640, 768),     # text K/V projection: ragged M, 768-wide context
        (200, 328, 72),     # ragged everything (N % 8 == 0, K % 8 == 0)
        (8192, 1280, 5120), # FF out projection at batch 2
    ],
)
def test_gemm_plain(cuda_device, M, N, K):
    from imagdressing_b200 import ops

    a = _rand((M, K), cuda_device, 1).bfloat16()
    w = _rand((N, K), cuda_device, 2, K ** -0.5).bfloat16()
    out = ops.gemm(a, w)
    ref = ops_ref.gemm_ref(a, w)
    assert out.shape == (M, N) and out.dtype == torch.bfloat16
    assert rel_l2(out, ref) < TOL


def test_gemm_epilogue_bias_residual_rowvec(cuda_device):
    from imagdressing_b200 import ops

    M, N, K, rpg = 2 * 1024, 640, 320, 1024
    a = _rand((M, K), cuda_device, 3).bfloat16()
    w = _rand((N, K), cuda_device, 4, K ** -0.5).bfloat16()
    bias = _rand((N,), cuda_device, 5)
    rowvec = _rand((M // rpg, N), cuda_device, 6)
    res = _rand((M, N), cuda_device, 7).bfloat16()
    out = ops.gemm(a, w, bias=bias, rowvec=rowvec, rows_per_group=rpg, residual=res)
    ref = ops_ref.gemm_ref(a, w, bias, rowvec, rpg, res)
    assert rel_l2(out, ref) < TOL
    out32 = ops.gemm(a, w, bias=bias, out_fp32=True)
    assert out32.dtype == torch.float32
    assert rel_l2(out32, ops_ref.gemm_ref(a, w, bias)) < 2e-3  # no output rounding
    outs = ops.gemm(a, w, bias=bias, act=ops.ACT_SILU, alpha=0.5)
    assert rel_l2(outs, ops_ref.gemm_ref(a, w, bias, act="silu", alpha=0.5)) < TOL
    outg = ops.gemm(a, w, act=ops.ACT_GELU)
    assert rel_l2(outg, ops_ref.gemm_ref(a, w, act="gelu")) < TOL


def test_gemm_strided_views(cuda_device):
    """A and D as column slices of wider buffers (the fused-QKV / concat use)."""
    from imagdressing_b200 import ops

    M, K, N = 512, 320, 320
    big_a = _rand((M, 3 * K), cuda_device, 8).bfloat16()
    a = big_a[:, K:2 * K]
    w = _rand((N, K), cuda_device, 9, K ** -0.5).bfloat16()
    big_out = torch.zeros(M, 2 * N, device=cuda_device, dtype=torch.bfloat16)
    ops.gemm(a, w, out=big_out[:, N:])
    assert rel_l2(big_out[:, N:], ops_ref.gemm_ref(a, w)) < TOL
    assert float(big_out[:, :N].abs().max()) == 0.0


@pytest.mark.parametrize("M,C", [(4096, 320), (1024, 640), (64, 1280)])
def test_gemm_geglu(cuda_device, M, C):
    from imagdressing_b200 import ops

    a = _rand((M, C), cuda_device, 10).bfloat16()
    w = _rand((8 * C, C), cuda_device, 11, C ** -0.5).bfloat16()
    b = _rand((8 * C,), cuda_device, 12, 0.1)
    wp, bp = ops_ref.geglu_pack(w, b)
    out = ops.gemm(a, wp, bias=bp, act=ops.ACT_GEGLU)
    assert out.shape == (M, 4 * C)
    assert rel_l2(out, ops_ref.geglu_ref(a, w, b)) < TOL


@pytest.mark.parametrize(
    "NB,H,W,Cin,Cout",
    [
        (1, 64, 64, 320, 320),
        (2, 32, 32, 640, 640),
        (1, 16, 16, 1280, 1280),
        (1, 8, 8, 1280, 1280),     # one tile spans two images' worth of rows
        (3, 8, 8, 2560, 1280),     # up-block conv on a concat input, odd batch
        (1, 80, 64, 320, 320),     # 640x512 default resolution
        (1, 20, 16, 64, 64),       # H not a multiple of the row box
        (1, 12, 9, 64, 128),       # 768x576 deepest level (W = 9)
        (2, 24, 18, 128, 64),
    ],
)
def test_conv3x3(cuda_device, NB, H, W, Cin, Cout):
    from imagdressing_b200 import ops

    x = _rand((NB, H, W, Cin), cuda_device, 13).bfloat16()
    w = _rand((Cout, Cin, 3, 3), cuda_device, 14, (9 * Cin) ** -0.5).bfloat16()
    bias = _rand((Cout,), cuda_device, 15)
    temb = _rand((NB, Cout), cuda_device, 16)
    res = _rand((NB, H, W, Cout), cuda_device, 17).bfloat16()
    out = ops.conv3x3(x, ops_ref.conv3x3_pack(w), bias=bias, rowvec=temb, residual=res)
    ref = ops_ref.conv3x3_ref(x, w, bias, temb, res)
    assert out.shape == (NB, H, W, Cout)
    assert rel_l2(out, ref) < TOL


def test_conv3x3_linearity_full_size(cuda_device):
    """Size-independent property at the bench shape: conv(a + b) == conv(a) + conv(b) (bias-free)."""
    from imagdressing_b200 import ops

    x1 = _rand((2, 64, 64, 320), cuda_device, 18).bfloat16()
    x2 = _rand((2, 64, 64, 320), cuda_device, 19).bfloat16()
    w = ops_ref.conv3x3_pack(_rand((320, 320, 3, 3), cuda_device, 20, 2880 ** -0.5).bfloat16())
    xs = (x1.float() + x2.float()).bfloat16()
    lhs = ops.conv3x3(xs, w).float()
    rhs = ops.conv3x3(x1, w).float() + ops.conv3x3(x2, w).float()
    assert rel_l2(lhs, rhs) < 2e-2


@pytest.mark.parametrize("bn,stages,splits", [(64, 4, 1), (128, 3, 1), (160, 3, 1), (256, 2, 1), (64, 8, 1), (128, 6, 1),
                                              (160, 5, 1), (256, 4, 1), (64, 8, 4), (128, 6, 3), (160, 3, 2),
                                              (256, 4, 8), (64, 4, 24)])
def test_gemm_tile_and_splitk_variants(cuda_device, bn, stages, splits):
    """Every N-tile / split-K kernel variant (forced through the test hook) on a ragged GEMM and a conv."""
    from imagdressing_b200 import _lib, ops

    lib = _lib.load()
    try:
        assert lib.imagd_gemm_debug_force(bn, stages, splits) == 0
        M, N, K = 300, 648, 1024
        a = _rand((M, K), cuda_device, 31).bfloat16()
        w = _rand((N, K), cuda_device, 32, K ** -0.5).bfloat16()
        bias = _rand((N,), cuda_device, 33)
        res = _rand((M, N), cuda_device, 34).bfloat16()
        out = ops.gemm(a, w, bias=bias, residual=res)
        assert rel_l2(out, ops_ref.gemm_ref(a, w, bias, residual=res)) < TOL
        out2 = ops.gemm(a, w, bias=bias, residual=res)
        assert torch.equal(out, out2)  # split-K reduction order is fixed -> bit-reproducible
        x = _rand((2, 8, 8, 256), cuda_device, 35).bfloat16()
        wc = _rand((328, 256, 3, 3), cuda_device, 36, (9 * 256) ** -0.5).bfloat16()
        temb = _rand((2, 328), cuda_device, 37)
        y = ops.conv3x3(x, ops_ref.conv3x3_pack(wc), rowvec=temb)
        assert rel_l2(y, ops_ref.conv3x3_ref(x, wc, None, temb)) < TOL
    finally:
        lib.imagd_gemm_debug_force(0, 0, 0)


def test_gemm_auto_config_deep_level_shapes(cuda_device):
    """The shapes where the automatic choice picks split-K (few output tiles, long K)."""
    from imagdressing_b200 import ops

    for (NB, H, W, Cin, Cout) in [(2, 8, 8, 2560, 1280), (2, 16, 16, 1280, 1280), (2, 8, 8, 1280, 1280)]:
        x = _rand((NB, H, W, Cin), cuda_device, 41).bfloat16()
        w = _rand((Cout, Cin, 3, 3), cuda_device, 42, (9 * Cin) ** -0.5).bfloat16()
        b = _rand((Cout,), cuda_device, 43)
        assert rel_l2(ops.conv3x3(x, ops_ref.conv3x3_pack(w), bias=b), ops_ref.conv3x3_ref(x, w, b)) < TOL
