"""GPU parity: two-stream attention (through the C ABI) vs the fp32 oracle.

Tolerance rel-L2 <= 1e-2: bf16 Q/K/V, fp32 scores and softmax statistics, P rounded to bf16 before P.V
(as FlashAttention does), bf16 output.
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


def _run(dev, B, Lq, heads, hd, L0, L1=0, n1=None, bcast1=False, w0=1.0, w1=1.0, fused=True, seed=0):
    from imagdressing_b200 import ops

    C = heads * hd
    if fused:  # Q, K, V as column slices of one fused projection output (row stride 3C)
        qkv = _rand((B, Lq, 3 * C), dev, seed + 1).bfloat16()
        q = qkv[..., :C]
        if L0 == Lq:
            k0, v0 = qkv[..., C:2 * C], qkv[..., 2 * C:]
        else:
            kv = _rand((B, L0, 2 * C), dev, seed + 2).bfloat16()
            k0, v0 = kv[..., :C], kv[..., C:]
    else:
        q = _rand((B, Lq, C), dev, seed + 1).bfloat16()
        k0 = _rand((B, L0, C), dev, seed + 2).bfloat16()
        v0 = _rand((B, L0, C), dev, seed + 3).bfloat16()
    s0 = ops.kv_stream(_flat(k0), _flat(v0), L0, out_scale=w0)
    s1 = None
    k1 = v1 = None
    if L1:
        nb1 = 1 if bcast1 else (n1 or B)
        kv1 = _rand((nb1, L1, 2 * C), dev, seed + 4).bfloat16()
        k1, v1 = kv1[..., :C], kv1[..., C:]
        s1 = ops.kv_stream(_flat(k1), _flat(v1), L1, broadcast=bcast1, n_query_samples=n1 or B, out_scale=w1)
    out = ops.attention(_flat(q), B, Lq, heads, hd, s0, s1)
    ref = ops_ref.hybrid_attention_ref(q, k0, v0, heads, k1, v1, w0, w1, n1)
    return out.view(B, Lq, C), ref


def _flat(t):
    """[B, L, C] view with uniform row stride -> 2-D [B*L, C] view sharing storage."""
    B, L, C = t.shape
    assert t.stride(0) == L * t.stride(1)
    return t.as_strided((B * L, C), (t.stride(1), 1), t.storage_offset())


@pytest.mark.parametrize(
    "B,L,heads,hd",
    [(1, 4096, 8, 40), (2, 1024, 8, 80), (2, 256, 8, 160), (1, 64, 8, 160), (1, 5120, 8, 40), (1, 432, 8, 160)],
)
def test_self_attention_levels(cuda_device, B, L, heads, hd):
    out, ref = _run(cuda_device, B, L, heads, hd, L)
    assert rel_l2(out, ref) < TOL


@pytest.mark.parametrize("B,L,hd", [(2, 4096, 40), (2, 1024, 80), (2, 256, 160), (2, 64, 160)])
def test_hybrid_cfg_batch(cuda_device, B, L, hd):
    """Sample 0 = conditional (self + garment stream, scale 0.9), sample 1 = unconditional (self only)."""
    out, ref = _run(cuda_device, B, L, 8, hd, L, L1=L, n1=1, w1=0.9)
    assert rel_l2(out[0], ref[0]) < TOL
    assert rel_l2(out[1], ref[1]) < TOL


def test_hybrid_ref_length_differs_and_broadcast(cuda_device):
    """Garment at another resolution (L_ref != L) and one garment broadcast over a batch of 3."""
    out, ref = _run(cuda_device, 3, 1024, 8, 80, 1024, L1=1280, n1=3, bcast1=True, w1=1.0)
    assert rel_l2(out, ref) < TOL


@pytest.mark.parametrize("L,hd", [(4096, 40), (1024, 80), (256, 160), (64, 160)])
def test_text_cross_attention_77(cuda_device, L, hd):
    out, ref = _run(cuda_device, 2, L, 8, hd, 77, fused=False)
    assert rel_l2(out, ref) < TOL


def test_text_plus_ip_tokens(cuda_device):
    """LoRAIPAttnProcessor2_0: 77 text tokens + 4 IP tokens as a second softmax, scale 0.9 (:833-856)."""
    out, ref = _run(cuda_device, 2, 1024, 8, 80, 77, L1=4, w1=0.9, fused=False)
    assert rel_l2(out, ref) < TOL


def test_perceiver_shape(cuda_device):
    """Resampler attention: 16 latent queries, 257+16 keys, 12 heads x 64 (adapter/resampler.py:62-78)."""
    out, ref = _run(cuda_device, 2, 16, 12, 64, 273, fused=False)
    assert rel_l2(out, ref) < TOL


def test_softmax_extreme_scores(cuda_device):
    """Rows whose max moves block to block (forces the O rescale) and large logits (no overflow)."""
    from imagdressing_b200 import ops

    dev = cuda_device
    B, L, heads, hd = 1, 512, 8, 40
    C = heads * hd
    q = _rand((B, L, C), dev, 50, 4.0).bfloat16()
    k = _rand((B, L, C), dev, 51, 4.0).bfloat16()
    k[:, 384:] *= 3.0  # later blocks dominate
    v = _rand((B, L, C), dev, 52).bfloat16()
    out = ops.attention(_flat(q), B, L, heads, hd, ops.kv_stream(_flat(k), _flat(v), L))
    ref = ops_ref.sdpa_ref(q, k, v, heads)
    assert torch.isfinite(out).all()
    assert rel_l2(out.view(B, L, C), ref) < 2e-2
