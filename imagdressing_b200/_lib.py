"""ctypes binding of libimagd_b200.so (the C ABI declared in include/imagd_b200.h).

The library is the product: there is no CPU or PyTorch fallback. Importing this module never needs a GPU (the
build check and the symbol test run on a CPU box); calling a kernel without the library or without an H100 (sm_90) raises.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, Structure, c_char_p, c_float, c_int, c_int32, c_int64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libimagd_b200.so")

IMAGD_OK = 0
ACT_NONE, ACT_GEGLU, ACT_SILU, ACT_GELU, ACT_QUICK_GELU, ACT_RELU = 0, 1, 2, 3, 4, 5


class Epilogue(Structure):
    """struct imagd_epilogue (include/imagd_b200.h)."""

    _fields_ = [
        ("bias", c_void_p),
        ("rowvec", c_void_p),
        ("rowvec_ld", c_int64),
        ("rows_per_group", c_int32),
        ("act", c_int32),
        ("residual", c_void_p),
        ("ldr", c_int64),
        ("alpha", c_float),
        ("out_fp32", c_int32),
        ("row_stats_out", c_void_p),
        ("stats_ld", c_int64),
        ("row_stats_in", c_void_p),
        ("stats_in_ld", c_int64),
        ("stats_parts", c_int32),
        ("ln_dim", c_int32),
        ("ln_eps", c_float),
        ("colsum", c_void_p),
        ("scale_table", c_void_p),
        ("scale_step", c_void_p),
        ("scale_ld", c_int64),
    ]


class AttnTrain(Structure):
    """struct imagd_attn_train (include/imagd_b200.h)."""

    _fields_ = [("lse", c_void_p), ("out_s0", c_void_p), ("out_s1", c_void_p), ("ld_s", c_int64), ("lq_pad", c_int32)]


class KVStream(Structure):
    """struct imagd_kv_stream (include/imagd_b200.h)."""

    _fields_ = [
        ("k", c_void_p),
        ("v", c_void_p),
        ("ld", c_int64),
        ("len", c_int32),
        ("sample_rows", c_int32),
        ("broadcast", c_int32),
        ("n_query_samples", c_int32),
        ("out_scale", c_float),
    ]


# name -> (restype, argtypes); mirrors include/imagd_b200.h one to one (tests/test_abi.py checks the header).
SIGNATURES = {
    "imagd_version": (c_int, []),
    "imagd_last_error": (c_char_p, []),
    "imagd_device_check": (c_int, []),
    "imagd_gemm_bf16": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_int64, c_int, c_int, c_int,
                                POINTER(Epilogue), c_void_p]),
    "imagd_gemm_debug_force": (c_int, [c_int, c_int, c_int]),
    "imagd_gemm_debug_log": (c_int, [c_int, c_char_p, c_int]),
    "imagd_gemm_debug_timeline": (c_int, [c_void_p]),
    "imagd_gemm_tile_count_n": (c_int, [c_int, c_int, c_int]),
    "imagd_conv3x3_bf16": (c_int, [c_void_p, c_int64, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int64, c_int,
                                   POINTER(Epilogue), c_void_p]),
    "imagd_upconv3x3_bf16": (c_int, [c_void_p, c_int64, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int64, c_int,
                                     POINTER(Epilogue), c_void_p]),
    "imagd_attention_bf16": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_int, c_int, c_int, c_int,
                                     POINTER(KVStream), POINTER(KVStream), c_float, c_void_p]),
    "imagd_attention_causal_bf16": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_int, c_int, c_int, c_int,
                                            POINTER(KVStream), c_float, c_void_p]),
    "imagd_attention_debug_force": (c_int, [c_int]),
    "imagd_groupnorm_ws_bytes": (c_int64, [c_int, c_int, c_int, c_int]),
    "imagd_groupnorm_plan": (c_int, [c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "imagd_groupnorm_cluster_capacity": (c_int, [c_void_p]),
    "imagd_groupnorm_debug_force": (c_int, [c_int, c_int, c_int]),
    "imagd_groupnorm_debug_log": (c_int, [c_int, c_char_p, c_int]),
    "imagd_groupnorm_bf16": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_int, c_int, c_int, c_int, c_void_p,
                                     c_void_p, c_float, c_int, c_void_p, c_void_p]),
    "imagd_layernorm_bf16": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p, c_float,
                                     c_void_p]),
    "imagd_concat_add_bf16": (c_int, [c_void_p, c_int64, c_int, c_void_p, c_int64, c_void_p, c_int64, c_int, c_void_p,
                                      c_int64, c_void_p, c_int64, c_int64, c_void_p]),
    "imagd_upsample2x_bf16": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "imagd_im2col3x3_s2_bf16": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "imagd_im2col3x3_s2_pad_bf16": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "imagd_embed_tokens_bf16": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "imagd_patchify_bf16": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "imagd_broadcast_row_bf16": (c_int, [c_void_p, c_void_p, c_int, c_int64, c_int, c_int, c_void_p]),
    "imagd_softmax_rows": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_int64, c_int, c_float, c_void_p]),
    "imagd_conv3x3_direct_bf16": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int,
                                          c_int, c_int, c_int, c_void_p, c_void_p]),
    "imagd_nchw_f32_to_nhwc_bf16": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "imagd_timestep_embedding": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "imagd_linear_small_m": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_void_p, c_int64, c_int, c_int,
                                     c_int, c_int, c_int, c_void_p]),
    "imagd_cfg_ddim_step": (c_int, [c_void_p, c_void_p, c_float, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                    c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "imagd_nchw_f32_to_nhwc_bf16_scaled": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p,
                                                   c_void_p, c_void_p]),
    "imagd_cfg_sampler_step": (c_int, [c_void_p, c_void_p, c_float, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                       c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "imagd_cfg_sampler_pc_step": (c_int, [c_void_p, c_void_p, c_float, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                          c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    # ---- T2I-Adapter
    "imagd_pixel_unshuffle8_bf16": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "imagd_avgpool2x2_bf16": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "imagd_scaled_add_bcast_bf16": (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_int, c_int, c_int64, c_int, c_void_p]),
    # ---- training step (row a13)
    "imagd_attention_train_fwd_bf16": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_int, c_int, c_int, c_int,
                                               POINTER(KVStream), POINTER(KVStream), c_float, POINTER(AttnTrain), c_void_p]),
    "imagd_attention_bwd_prep": (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_int64, c_float, c_float, c_void_p, c_int,
                                         c_int, c_int, c_int, c_int, c_void_p]),
    "imagd_attention_bwd_bf16": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_int, c_int, c_int, c_int, POINTER(KVStream),
                                         POINTER(KVStream), c_float, c_void_p, c_void_p, c_int, c_void_p, c_int64, c_void_p,
                                         c_void_p, c_int64, c_void_p, c_void_p, c_int64, c_void_p]),
    "imagd_transpose_bf16": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_int, c_int, c_int, c_void_p]),
    "imagd_conv_weight_layout_bf16": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "imagd_conv_weight_flip_bf16": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "imagd_im2col3x3_t_bf16": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_int, c_void_p]),
    "imagd_col2im3x3_s2_bf16": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "imagd_downsum2x_bf16": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "imagd_colreduce_ws_bytes": (c_int64, [c_int, c_int, c_int]),
    "imagd_colsum_bf16": (c_int, [c_void_p, c_int64, c_int, c_int, c_int, c_void_p, c_int, c_void_p, c_void_p]),
    "imagd_layernorm_bwd_bf16": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_int64, c_int, c_int, c_void_p,
                                         c_float, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "imagd_groupnorm_stats_bf16": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_int, c_int, c_int, c_int, c_void_p,
                                           c_void_p, c_float, c_int, c_void_p, c_void_p, c_void_p]),
    "imagd_groupnorm_bwd_ws_bytes": (c_int64, [c_int, c_int, c_int, c_int]),
    "imagd_groupnorm_bwd_bf16": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                                         c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    "imagd_act_bf16": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_void_p]),
    "imagd_geglu_bf16": (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_int64, c_int64, c_int, c_void_p]),
    "imagd_mse_loss_grad": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_float, c_void_p, c_void_p]),
    "imagd_adamw_step": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_float, c_float, c_float,
                                 c_float, c_float, c_int, c_float, c_void_p]),
    "imagd_adamw_step_dev": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_float, c_float, c_float,
                                     c_void_p, c_void_p]),
    "imagd_grad_norm_ws_bytes": (c_int64, [c_int64]),
    "imagd_grad_norm_clip": (c_int, [c_void_p, c_int64, c_float, c_void_p, c_void_p, c_void_p, c_void_p]),
    "imagd_adamw_step_clip": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_float, c_float, c_float,
                                      c_void_p, c_void_p, c_void_p]),
}

_lib = None


class ImagdError(RuntimeError):
    pass


def load() -> ctypes.CDLL:
    """dlopen the in-tree library and attach signatures. Raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImagdError(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(or `make -C imagdressing_b200/csrc`). There is no fallback path."
        )
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError here == ABI drift, fail loudly
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


# kernels launched through the C ABI (bench.py reports it as gpu_launches); graph replays add their node count
LAUNCHES = {"imagd_gemm_bf16": 1, "imagd_conv3x3_bf16": 1, "imagd_upconv3x3_bf16": 1, "imagd_attention_bf16": 1, "imagd_attention_causal_bf16": 1, "imagd_groupnorm_bf16": 1,
            "imagd_layernorm_bf16": 1, "imagd_concat_add_bf16": 1, "imagd_upsample2x_bf16": 1,
            "imagd_im2col3x3_s2_bf16": 1, "imagd_im2col3x3_s2_pad_bf16": 1, "imagd_softmax_rows": 1, "imagd_embed_tokens_bf16": 1, "imagd_patchify_bf16": 1, "imagd_broadcast_row_bf16": 1, "imagd_conv3x3_direct_bf16": 1, "imagd_nchw_f32_to_nhwc_bf16": 1,
            "imagd_timestep_embedding": 1, "imagd_linear_small_m": 1, "imagd_cfg_ddim_step": 1,
            "imagd_nchw_f32_to_nhwc_bf16_scaled": 1, "imagd_cfg_sampler_step": 1,
            "imagd_cfg_sampler_pc_step": 1,
            "imagd_pixel_unshuffle8_bf16": 1, "imagd_avgpool2x2_bf16": 1, "imagd_scaled_add_bcast_bf16": 1,
            "imagd_attention_train_fwd_bf16": 1, "imagd_attention_bwd_prep": 1, "imagd_attention_bwd_bf16": 3,
            "imagd_transpose_bf16": 1, "imagd_conv_weight_layout_bf16": 1, "imagd_conv_weight_flip_bf16": 1, "imagd_im2col3x3_t_bf16": 1, "imagd_col2im3x3_s2_bf16": 1, "imagd_downsum2x_bf16": 1,
            "imagd_colsum_bf16": 2, "imagd_layernorm_bwd_bf16": 3, "imagd_groupnorm_bwd_bf16": 4, "imagd_groupnorm_stats_bf16": 1, "imagd_act_bf16": 1,
            "imagd_geglu_bf16": 1, "imagd_mse_loss_grad": 2, "imagd_adamw_step": 1, "imagd_adamw_step_dev": 1,
            "imagd_grad_norm_clip": 1, "imagd_adamw_step_clip": 1}
launch_count = 0


def check(rc: int, what: str) -> None:
    global launch_count
    launch_count += LAUNCHES.get(what, 0)
    if rc != IMAGD_OK:
        msg = load().imagd_last_error()
        raise ImagdError(f"{what} failed ({rc}): {msg.decode() if msg else '?'}")


class _ProfiledLib:
    """Proxy over the loaded library that brackets every launching C-ABI call with CUDA events on the current stream
    (bench.py's live per-kernel step shares; never active on a production path). Keys = symbol + small integer
    arguments (shapes), so launches group by kernel and problem size."""

    def __init__(self, lib, records):
        self._lib, self._records = lib, records

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if name not in LAUNCHES:
            return fn
        import torch

        def wrapped(*args):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            rc = fn(*args)
            e1.record()
            key = name + "(" + ",".join(str(a) for a in args if isinstance(a, int) and 0 <= a < 1000000) + ")"
            self._records.append((key, e0, e1))
            return rc

        return wrapped


class profile_launches:
    """with profile_launches() as rec: ...eager kernels...  -> rec.by_key() = {key: (launches, total_ms)}."""

    def __enter__(self):
        global _lib
        self._saved = load()
        self._records = []
        _lib = _ProfiledLib(self._saved, self._records)
        return self

    def __exit__(self, *exc):
        global _lib
        _lib = self._saved
        return False

    def by_key(self):
        import torch

        torch.cuda.synchronize()
        out = {}
        for key, e0, e1 in self._records:
            n, ms = out.get(key, (0, 0.0))
            out[key] = (n + 1, ms + e0.elapsed_time(e1))
        return out


def require_b200() -> None:
    rc = load().imagd_device_check()
    if rc < 0:
        msg = load().imagd_last_error()
        raise ImagdError(f"imagd_b200 needs an sm_90 (H100) GPU: {msg.decode() if msg else rc}")
