"""GPU: the automatic GEMM / conv configuration at shapes of the batch-1 denoising step, against the fp32 oracle.

The tile rule picks the deep operand ring and, for long K on few output tiles, split-K with the wider N tiles; these
are the configurations the step now runs, checked here at the step's own shapes (the configuration that ran is read
back from imagd_gemm_debug_log)."""
import pytest
import torch

from conftest import rel_l2
from oracle import ops_ref

pytestmark = pytest.mark.gpu
TOL = 1e-2
DEEP = {64: 8, 128: 6, 160: 5, 256: 4}


def _rand(shape, dev, seed, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dev)


def _ran(lib, fn):
    """Run fn once with the launch log on; return (block_n, stages, splits) of its single launch."""
    lib.imagd_gemm_debug_log(1, None, 0)
    try:
        out = fn()
    finally:
        lib.imagd_gemm_debug_log(0, None, 0)
    buf = bytes(1024)
    assert lib.imagd_gemm_debug_log(-1, buf, len(buf)) == 1
    return out, [int(v) for v in buf.split(b"\0", 1)[0].decode().split("|")[1].split()]


@pytest.mark.parametrize("NB,H,W,Cin,Cout", [(2, 64, 64, 320, 320), (2, 32, 32, 640, 640), (2, 16, 16, 1280, 1280),
                                             (2, 16, 16, 2560, 1280), (2, 32, 32, 1920, 640), (2, 8, 8, 1280, 1280)])
def test_conv3x3_step_shapes(cuda_device, NB, H, W, Cin, Cout):
    from imagdressing_b200 import _lib, ops

    lib = _lib.load()
    x = _rand((NB, H, W, Cin), cuda_device, 1).bfloat16()
    w = _rand((Cout, Cin, 3, 3), cuda_device, 2, (9 * Cin) ** -0.5).bfloat16()
    bias, temb = _rand((Cout,), cuda_device, 3), _rand((NB, Cout), cuda_device, 4)
    res = _rand((NB, H, W, Cout), cuda_device, 5).bfloat16()
    wp = ops_ref.conv3x3_pack(w)
    out, (bn, stages, splits) = _ran(lib, lambda: ops.conv3x3(x, wp, bias=bias, rowvec=temb, residual=res))
    assert stages == DEEP[bn]
    assert rel_l2(out, ops_ref.conv3x3_ref(x, w, bias, temb, res)) < TOL
    assert torch.equal(out, ops.conv3x3(x, wp, bias=bias, rowvec=temb, residual=res))  # fixed split-K order


@pytest.mark.parametrize("M,N,K", [(8192, 320, 320), (8192, 320, 1280), (2048, 640, 640), (2048, 640, 1920),
                                   (512, 1280, 5120), (512, 3840, 1280), (128, 1280, 5120)])
def test_gemm_step_shapes(cuda_device, M, N, K):
    from imagdressing_b200 import _lib, ops

    lib = _lib.load()
    a = _rand((M, K), cuda_device, 6).bfloat16()
    w = _rand((N, K), cuda_device, 7, K ** -0.5).bfloat16()
    bias, res = _rand((N,), cuda_device, 8), _rand((M, N), cuda_device, 9).bfloat16()
    out, (bn, stages, splits) = _ran(lib, lambda: ops.gemm(a, w, bias=bias, residual=res))
    assert stages == DEEP[bn]
    assert rel_l2(out, ops_ref.gemm_ref(a, w, bias, residual=res)) < TOL
    assert ops.gemm_tile_count_n(M, N, K) == (N + bn - 1) // bn  # what LayerNorm-fold producers size their slots by


@pytest.mark.parametrize("M,C", [(8192, 320), (512, 1280)])
def test_geglu_step_shapes(cuda_device, M, C):
    from imagdressing_b200 import _lib, ops

    lib = _lib.load()
    a = _rand((M, C), cuda_device, 10).bfloat16()
    w = _rand((8 * C, C), cuda_device, 11, C ** -0.5).bfloat16()
    b = _rand((8 * C,), cuda_device, 12, 0.1)
    wp, bp = ops_ref.geglu_pack(w, b)
    out, (bn, stages, splits) = _ran(lib, lambda: ops.gemm(a, wp, bias=bp, act=ops.ACT_GEGLU))
    assert (bn, stages, splits) == (128, DEEP[128], 1)
    assert rel_l2(out, ops_ref.geglu_ref(a, w, b)) < TOL


@pytest.mark.parametrize("NB,H,W,C", [(2, 16, 16, 1280), (2, 32, 32, 640)])
def test_upconv_step_shapes(cuda_device, NB, H, W, C):
    from imagdressing_b200 import _lib, modeling, ops

    lib = _lib.load()
    x = _rand((NB, H, W, C), cuda_device, 13).bfloat16()
    w = _rand((C, C, 3, 3), cuda_device, 14, (9 * C) ** -0.5).bfloat16()
    b = _rand((C,), cuda_device, 15)
    out, (bn, stages, splits) = _ran(lib, lambda: ops.upconv3x3(x, modeling.pack_upconv3x3(w), bias=b))
    assert stages == DEEP[bn] and splits == 1
    up = x.repeat_interleave(2, 1).repeat_interleave(2, 2).contiguous()
    assert rel_l2(out, ops_ref.conv3x3_ref(up, w, b)) < TOL
