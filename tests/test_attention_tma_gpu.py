"""GPU checks of the attention forward's memory behaviour: the output is written only inside its head slice and below
Lq, padding rows of a K / V sample are never read, and repeated launches agree bit for bit.

Head_dim 40 / 80 calls with >= 1024 keys in stream 0 run the TMA / wgmma kernel; the lengths used for it here are not
multiples of the key block (the last block of each stream is masked) and Lq is not a multiple of the 128-row tile.
The short-key and head_dim 160 cases run the mma.sync kernel."""
import pytest
import torch

from conftest import rel_l2
from oracle import ops_ref

pytestmark = pytest.mark.gpu
TOL = 1e-2


def _rand(shape, dev, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return torch.randn(shape, generator=g).to(dev).bfloat16()


def _flat(t):
    B, L, C = t.shape
    return t.as_strided((B * L, C), (t.stride(1), 1), t.storage_offset())


@pytest.mark.parametrize("hd,Lq,L", [(40, 1000, 1100), (80, 1000, 1100), (160, 200, 200)])
def test_output_stays_in_head_slice(cuda_device, hd, Lq, L):
    """Output as a column slice of a wider buffer (one head's width of columns before it, 16 spare columns after it),
    with rows past B * Lq: every element outside [rows < B * Lq] x [columns of the computed heads] keeps its sentinel."""
    from imagdressing_b200 import ops

    B, heads = 2, 3
    C = heads * hd
    q = _rand((B, Lq, C), cuda_device, 1)
    k, v = (_rand((B, L, C), cuda_device, s) for s in (2, 3))
    ld = C + hd + 16
    buf = torch.full((B * Lq + 64, ld), 7.0, device=cuda_device, dtype=torch.bfloat16)
    col0 = hd
    out = buf[: B * Lq, col0:col0 + C]
    ops.attention(_flat(q), B, Lq, heads, hd, ops.kv_stream(_flat(k), _flat(v), L), out=out)
    ref = ops_ref.sdpa_ref(q, k, v, heads)
    assert rel_l2(out.reshape(B, Lq, C), ref) < TOL
    mask = torch.ones_like(buf, dtype=torch.bool)
    mask[: B * Lq, col0:col0 + C] = False
    assert (buf[mask] == 7.0).all()


@pytest.mark.parametrize("hd,Lq,L0,L1", [(40, 1000, 1100, 1090), (80, 1000, 1100, 1090), (40, 300, 200, 70)])
def test_padding_rows_are_not_read(cuda_device, hd, Lq, L0, L1):
    """Each sample of both streams spans `rows` rows of which the first L0 / L1 are keys; the rest hold NaN. The result
    stays finite and equal to the oracle over the keys. Stream 1 applies to the first two of three query samples."""
    from imagdressing_b200 import ops

    B, heads, n1 = 3, 8, 2
    rows = max(L0, L1) + 64
    C = heads * hd
    q = _rand((B, Lq, C), cuda_device, 4)
    kv0 = _rand((B, rows, 2 * C), cuda_device, 5)
    kv1 = _rand((n1, rows, 2 * C), cuda_device, 6)
    kv0[:, L0:] = float("nan")
    kv1[:, L1:] = float("nan")
    s0 = ops.kv_stream(_flat(kv0[..., :C]), _flat(kv0[..., C:]), L0, sample_rows=rows)
    s1 = ops.kv_stream(_flat(kv1[..., :C]), _flat(kv1[..., C:]), L1, sample_rows=rows, n_query_samples=n1,
                       out_scale=0.7)
    out = ops.attention(_flat(q), B, Lq, heads, hd, s0, s1).view(B, Lq, C)
    ref = ops_ref.hybrid_attention_ref(q, kv0[:, :L0, :C], kv0[:, :L0, C:], heads, kv1[:, :L1, :C], kv1[:, :L1, C:],
                                       1.0, 0.7, n1)
    assert torch.isfinite(out).all()
    assert rel_l2(out, ref) < TOL


@pytest.mark.parametrize("hd", [40, 80])
def test_repeated_launches_bitwise_equal(cuda_device, hd):
    from imagdressing_b200 import ops

    B, L, heads = 2, 1100, 8
    C = heads * hd
    qkv = _rand((B, L, 3 * C), cuda_device, 7)
    kv1 = _rand((1, L, 2 * C), cuda_device, 8)
    s0 = ops.kv_stream(_flat(qkv[..., C:2 * C]), _flat(qkv[..., 2 * C:]), L)
    s1 = ops.kv_stream(_flat(kv1[..., :C]), _flat(kv1[..., C:]), L, n_query_samples=1)
    a = ops.attention(_flat(qkv[..., :C]), B, L, heads, hd, s0, s1)
    b = ops.attention(_flat(qkv[..., :C]), B, L, heads, hd, s0, s1)
    assert torch.equal(a, b)
