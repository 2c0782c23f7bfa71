"""GPU: GEMM / conv kernels on multi-wave problems (many times the 132 SMs) with every LINEAR epilogue ingredient — the
grids where the bulk-store epilogue is selected."""
import pytest
import torch

from conftest import rel_l2
from oracle import ops_ref

pytestmark = pytest.mark.gpu
BF = torch.bfloat16


def _rand(shape, dev, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dev)


@pytest.mark.parametrize("M,N,K", [(65536, 320, 320), (65536, 960, 320), (16384, 640, 2560), (40000, 328, 72),
                                   (70000, 64, 640), (33000, 136, 128)])
def test_persistent_gemm(cuda_device, M, N, K):
    from imagdressing_b200 import ops

    a, w = _rand((M, K), cuda_device, 1).to(BF), _rand((N, K), cuda_device, 2, K ** -0.5).to(BF)
    b, res = _rand((N,), cuda_device, 3), _rand((M, N), cuda_device, 4).to(BF)
    out = ops.gemm(a, w, bias=b, residual=res)
    assert rel_l2(out, ops_ref.gemm_ref(a, w, b, residual=res)) < 1e-2
    assert torch.equal(out, ops.gemm(a, w, bias=b, residual=res))
    plain = ops.gemm(a, w)
    assert rel_l2(plain, ops_ref.gemm_ref(a, w)) < 1e-2


@pytest.mark.parametrize("NB,H,W,Cin,Cout", [(16, 64, 64, 320, 320), (16, 32, 32, 640, 640), (16, 16, 16, 1280, 1280),
                                             (5, 80, 64, 320, 320), (9, 24, 18, 128, 64)])
def test_persistent_conv3x3(cuda_device, NB, H, W, Cin, Cout):
    from imagdressing_b200 import ops

    x = _rand((NB, H, W, Cin), cuda_device, 13).to(BF)
    w = _rand((Cout, Cin, 3, 3), cuda_device, 14, (9 * Cin) ** -0.5).to(BF)
    bias, temb = _rand((Cout,), cuda_device, 15), _rand((NB, Cout), cuda_device, 16)
    res = _rand((NB, H, W, Cout), cuda_device, 17).to(BF)
    out = ops.conv3x3(x, ops_ref.conv3x3_pack(w), bias=bias, rowvec=temb, residual=res)
    assert rel_l2(out, ops_ref.conv3x3_ref(x, w, bias, temb, res)) < 1e-2
