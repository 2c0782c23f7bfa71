"""GPU parity of every GroupNorm plan the library can run (forced through imagd_groupnorm_debug_force): the rendezvous kernel
and the cluster kernel at each cluster size x each legal slice width, against the fp32 reference; the automatic plan is
bit-reproducible from launch to launch."""
import ctypes

import pytest
import torch

from conftest import rel_l2
from oracle import ops_ref

pytestmark = pytest.mark.gpu

CLUSTER_SIZES = (2, 4, 8, 16)


def _plans(lib, NB, HW, C, groups):
    """Every distinct plan the forced-variant hook can select at this shape (the library decides what is legal)."""
    cpg = C // groups
    forced = [(1, 0, 0)] + [(2, cs, gps * cpg) for cs in CLUSTER_SIZES for gps in range(1, groups + 1)
                            if groups % gps == 0 and gps * cpg % 8 == 0]
    out = (ctypes.c_int * 5)()
    for f in forced:
        assert lib.imagd_groupnorm_debug_force(*f) == 0
        if lib.imagd_groupnorm_plan(NB, HW, C, groups, None, out) == 0:
            assert (out[0], out[1], out[2]) == f
            yield f


@pytest.fixture
def lib():
    from imagdressing_b200 import _lib

    lib = _lib.load()
    yield lib
    lib.imagd_groupnorm_debug_force(0, 0, 0)


# the step's level-0 / level-1 / mid / up-block shapes at batch 1, level 0 at batch 8 (512 x 512 and 768 x 576), a VAE shape
# with 4-channel groups, and HW smaller than every cluster size but 2 and 4
@pytest.mark.parametrize("NB,H,W,C", [(2, 64, 64, 320), (2, 32, 32, 640), (2, 8, 8, 1280), (2, 16, 16, 2560), (16, 64, 64, 320),
                                      (16, 96, 72, 320), (1, 64, 64, 128), (2, 1, 5, 640)])
def test_every_plan_matches_reference(cuda_device, lib, NB, H, W, C):
    from imagdressing_b200 import ops

    g = torch.Generator().manual_seed(5)
    x = (torch.randn(NB, H, W, C, generator=g) * 1.5 + 0.3).to(cuda_device).bfloat16()
    gamma = (1.0 + 0.1 * torch.randn(C, generator=g)).to(cuda_device)
    beta = (0.1 * torch.randn(C, generator=g)).to(cuda_device)
    ref = ops_ref.groupnorm_ref(x, gamma, beta, 32, 1e-5, True)
    xg = x.float().reshape(NB, H * W, 32, C // 32)
    mean, rstd = xg.mean(dim=(1, 3)), torch.rsqrt(xg.var(dim=(1, 3), unbiased=False) + 1e-5)
    seen = 0
    for f in _plans(lib, NB, H * W, C, 32):
        stats = torch.empty(NB, 32, 2, device=cuda_device, dtype=torch.float32)
        out = ops.groupnorm(x, gamma, beta, 32, 1e-5, silu=True, stats_out=stats)
        assert rel_l2(out, ref) < 5e-3, f
        assert torch.allclose(stats[..., 0], mean, atol=2e-4, rtol=1e-4), f
        assert torch.allclose(stats[..., 1], rstd, rtol=1e-3), f
        seen += 1
    assert seen >= 3  # the rendezvous kernel and at least two cluster plans
    lib.imagd_groupnorm_debug_force(0, 0, 0)
    a = ops.groupnorm(x, gamma, beta, 32, 1e-5, silu=True)
    assert rel_l2(a, ref) < 5e-3
    assert torch.equal(a, ops.groupnorm(x, gamma, beta, 32, 1e-5, silu=True))


def test_every_plan_leaves_the_columns_beyond_c_alone(cuda_device, lib):
    """A strided output (ldy > C): the sentinel columns after the C written ones keep their value."""
    from imagdressing_b200 import _lib, ops

    NB, HW, C, pad = 2, 256, 640, 16
    g = torch.Generator().manual_seed(6)
    x = torch.randn(NB, HW, C, generator=g).to(cuda_device).bfloat16()
    gamma = (1.0 + 0.1 * torch.randn(C, generator=g)).to(cuda_device)
    beta = (0.1 * torch.randn(C, generator=g)).to(cuda_device)
    ref = ops_ref.groupnorm_ref(x, gamma, beta, 32, 1e-5, False)
    ws = ops._gn_workspace(x.device, lib.imagd_groupnorm_ws_bytes(NB, HW, C, 32))
    for f in _plans(lib, NB, HW, C, 32):
        y = torch.full((NB, HW, C + pad), 7.0, device=cuda_device, dtype=torch.bfloat16)
        rc = lib.imagd_groupnorm_bf16(x.data_ptr(), C, y.data_ptr(), C + pad, NB, HW, C, 32, gamma.data_ptr(), beta.data_ptr(),
                                      1e-5, 0, ws.data_ptr(), torch.cuda.current_stream().cuda_stream)
        _lib.check(rc, "imagd_groupnorm_bf16")
        assert rel_l2(y[..., :C], ref) < 5e-3, f
        assert bool((y[..., C:] == 7.0).all()), f
