"""CPU check of the GroupNorm plan rule (imagd_groupnorm_plan with the cluster capacity given, so no device is needed): at
every GroupNorm shape of the UNet step the plan meets the cluster kernel's own preconditions, and every forced plan the
library accepts does too (cluster sizes and slice widths the kernel cannot run are refused, not launched)."""
import ctypes

import pytest

# co-resident clusters of size 2 / 4 / 8 / 16 at one and at two CTAs per SM, as cudaOccupancyMaxActiveClusters reports them
# for the cluster kernel on an H100 80GB HBM3 SXM (132 SMs; a cluster must sit inside one GPC)
H100_CAPACITY = (66, 132, 30, 62, 15, 30, 7, 14)
# (latent side relative to a 64 x 64 level 0, C) of the step's GroupNorm launches (tools/gn_bench.py)
SHAPES = [(64, 320), (32, 320), (32, 640), (16, 640), (16, 1280), (8, 1280), (8, 2560), (16, 2560), (16, 1920), (32, 1920),
          (32, 1280), (32, 960), (64, 960), (64, 640)]
WORKLOADS = [(1, 64, 64), (8, 64, 64), (32, 64, 64), (8, 96, 72)]  # batch, level-0 latent H, W
STATIC_SMEM, CTA_SMEM_LIMIT = 33792, 227 * 1024


def _check(plan, NB, HW, C, groups=32):
    kernel, cs, sc, smem, waves = plan
    assert kernel in (1, 2) and waves >= 1
    if kernel == 1:
        return
    cpg = C // groups
    assert cs in (2, 4, 8, 16)
    assert sc % 8 == 0 and sc % cpg == 0 and C % sc == 0 and sc // 8 <= 512
    rows = -(-HW // cs)  # rows per CTA; the last CTAs of a cluster may own none when HW < cs * rows
    assert smem >= rows * sc * 2 + 3 * sc * 4
    assert smem + STATIC_SMEM <= CTA_SMEM_LIMIT
    index = (2, 4, 8, 16).index(cs)
    clusters = NB * (C // sc)
    assert waves == -(-clusters // max(H100_CAPACITY[2 * index + 1], 1)) or waves == -(-clusters // H100_CAPACITY[2 * index])


@pytest.fixture
def lib():
    from imagdressing_b200 import _lib

    lib = _lib.load()
    yield lib
    lib.imagd_groupnorm_debug_force(0, 0, 0)


def _plan(lib, NB, HW, C, groups=32):
    cap = (ctypes.c_int * 8)(*H100_CAPACITY)
    out = (ctypes.c_int * 5)()
    return list(out) if lib.imagd_groupnorm_plan(NB, HW, C, groups, cap, out) == 0 else None


@pytest.mark.parametrize("batch,H0,W0", WORKLOADS)
def test_automatic_plan_is_legal_and_one_wave(lib, batch, H0, W0):
    for side, C in SHAPES:
        NB, HW = 2 * batch, (H0 * side // 64) * (W0 * side // 64)
        plan = _plan(lib, NB, HW, C)
        assert plan is not None
        _check(plan, NB, HW, C)
        assert plan[4] == 1  # the cluster kernel is only chosen when all its clusters are co-resident


def test_batch_1_step_reads_x_once_below_level_0(lib):
    """Every batch-1 launch under 15 MB of traffic runs the cluster kernel (x read once, no global rendezvous)."""
    for side, C in SHAPES:
        if 4 * 2 * side * side * C < 15e6 and (side, C) != (64, 320):
            assert _plan(lib, 2, side * side, C)[0] == 2, (side, C)


def test_forced_plans_are_legal_or_refused(lib):
    for NB, HW, C in [(2, 4096, 320), (16, 6912, 320), (2, 5, 640), (1, 4096, 128), (2, 64, 2560)]:
        cpg = C // 32
        accepted = 0
        for cs in (2, 4, 8, 16):
            for gps in (1, 2, 4, 8, 16, 32):
                if gps * cpg % 8:
                    assert lib.imagd_groupnorm_debug_force(2, cs, gps * cpg) != 0  # not a multiple of 8 channels
                    continue
                assert lib.imagd_groupnorm_debug_force(2, cs, gps * cpg) == 0
                plan = _plan(lib, NB, HW, C)
                if plan is not None:
                    assert plan[:3] == [2, cs, gps * cpg]
                    _check(plan, NB, HW, C)
                    accepted += 1
        assert accepted >= 4
        assert lib.imagd_groupnorm_debug_force(1, 0, 0) == 0
        assert _plan(lib, NB, HW, C)[0] == 1
    assert lib.imagd_groupnorm_debug_force(2, 3, 0) != 0  # not a cluster size
    assert lib.imagd_groupnorm_debug_force(1, 8, 0) != 0  # a cluster size on the rendezvous kernel
