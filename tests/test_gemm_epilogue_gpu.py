"""GPU parity of the wgmma GEMM / conv epilogue forms against fp32 torch, for every N tile with and without split-K
(forced through imagd_gemm_debug_force): the register epilogue with TMA residual loads and TMA tile stores.

Also covered: ragged M / N at the tile edges, output into a column slice of a wider buffer (neighbouring columns must stay
untouched), a residual whose row stride differs from N, and 8x8-latent conv tiles that span two samples with a
per-sample row vector.
"""
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_l2
from oracle import ops_ref

pytestmark = pytest.mark.gpu
TOL = 1e-2
DEEP = {64: 8, 128: 6, 160: 5, 256: 4}


def _rand(shape, dev, seed, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dev)


class _Forced:
    def __init__(self, bn, splits):
        from imagdressing_b200 import _lib

        self.lib, self.cfg = _lib.load(), (bn, DEEP[bn], splits)

    def __enter__(self):
        assert self.lib.imagd_gemm_debug_force(*self.cfg) == 0

    def __exit__(self, *exc):
        self.lib.imagd_gemm_debug_force(0, 0, 0)


def _ref_act(y, form):
    if form == "silu":
        return F.silu(y)
    if form == "gelu":
        return F.gelu(y)
    if form == "quick_gelu":
        return y * torch.sigmoid(1.702 * y)
    return y


@pytest.mark.parametrize("splits", [1, 3])
@pytest.mark.parametrize("bn", [64, 128, 160, 256])
@pytest.mark.parametrize("form", ["linear", "silu", "gelu", "quick_gelu", "fp32", "geglu"])
def test_epilogue_forms(cuda_device, form, bn, splits):
    """M and N ragged at the tile edges (M = 300, N = 648 / GEGLU 640), K long enough for split-K."""
    from imagdressing_b200 import ops

    M, K = 300, 1024 * 2
    N = 640 if form == "geglu" else 648
    a = _rand((M, K), cuda_device, 1).bfloat16()
    w = _rand((N, K), cuda_device, 2, K ** -0.5).bfloat16()
    bias = _rand((N,), cuda_device, 3)
    act = {"silu": ops.ACT_SILU, "gelu": ops.ACT_GELU, "quick_gelu": ops.ACT_QUICK_GELU, "geglu": ops.ACT_GEGLU}.get(
        form, ops.ACT_NONE)
    with _Forced(bn, splits):
        if form == "geglu":
            out = ops.gemm(a, w, bias=bias, act=act)
            y = a.float() @ w.float().t() + bias
            y = y.view(M, N // 128, 2, 64)
            ref = (y[:, :, 0] * F.gelu(y[:, :, 1])).reshape(M, N // 2)
        else:
            res = _rand((M, N), cuda_device, 4).bfloat16()
            out = ops.gemm(a, w, bias=bias, residual=res, act=act, out_fp32=form == "fp32")
            ref = _ref_act(a.float() @ w.float().t() + bias, form) + res.float()
            assert out.dtype == (torch.float32 if form == "fp32" else torch.bfloat16)
    assert rel_l2(out, ref) < TOL


@pytest.mark.parametrize("bn", [64, 128, 160, 256])
def test_column_slice_and_strided_residual(cuda_device, bn):
    """out is columns [64, 64 + N) of a wider buffer whose other columns hold sentinels; the residual is a column
    slice of a wider tensor too (ldr != N)."""
    from imagdressing_b200 import ops

    M, N, K, wide = 200, 328, 320, 520
    a = _rand((M, K), cuda_device, 5).bfloat16()
    w = _rand((N, K), cuda_device, 6, K ** -0.5).bfloat16()
    bias = _rand((N,), cuda_device, 7)
    res_full = _rand((M, 400), cuda_device, 8).bfloat16()
    res = res_full[:, 8:8 + N]
    buf = torch.full((M, wide), 7.0, device=cuda_device, dtype=torch.bfloat16)
    with _Forced(bn, 1):
        ops.gemm(a, w, out=buf[:, 64:64 + N], bias=bias, residual=res)
    assert rel_l2(buf[:, 64:64 + N], ops_ref.gemm_ref(a, w, bias, residual=res)) < TOL
    assert bool((buf[:, :64] == 7.0).all()) and bool((buf[:, 64 + N:] == 7.0).all())


@pytest.mark.parametrize("bn", [64, 128, 160, 256])
def test_conv_tiles_spanning_samples_rowvec(cuda_device, bn):
    """8x8 latents: a 128-pixel tile covers two samples, each with its own time-embedding row vector."""
    from imagdressing_b200 import ops

    NB, H, W, Cin, Cout = 4, 8, 8, 128, 328
    x = _rand((NB, H, W, Cin), cuda_device, 9).bfloat16()
    w = _rand((Cout, Cin, 3, 3), cuda_device, 10, (9 * Cin) ** -0.5).bfloat16()
    bias = _rand((Cout,), cuda_device, 11)
    temb = _rand((NB, Cout), cuda_device, 12)
    res = _rand((NB, H, W, Cout), cuda_device, 13).bfloat16()
    with _Forced(bn, 1):
        out = ops.conv3x3(x, ops_ref.conv3x3_pack(w), bias=bias, rowvec=temb, residual=res)
    assert rel_l2(out, ops_ref.conv3x3_ref(x, w, bias, temb, res)) < TOL
