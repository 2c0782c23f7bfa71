// Shared pieces of the attention forward / backward kernels (sm_90a): row-tile loads into padded shared memory and the
// warp-level MMA fragment helpers.
#pragma once
#include "ptx.cuh"

namespace imagd {

// one key / value stream of an attention call, in the caller's token-major layout
struct AttnKV {
    const __nv_bfloat16* k;
    const __nv_bfloat16* v;
    int64_t ld;
    int len;          // keys per sample
    int sample_rows;  // rows between samples
    int bcast;        // every query sample reads sample 0
};

// shared-memory row of a head tile: HDP (head_dim rounded up to 16) bf16 + 16 bytes, so that the eight 16-byte rows
// of an ldmatrix phase land on eight different bank groups
__host__ __device__ constexpr int attn_row_bytes(int hdp) { return (hdp + 8) * 2; }

// rows [r0, r0 + nrows) of one head (columns [0, hd) of rows base + r * ld) -> shared memory; rows >= valid and columns
// >= hd are zero-filled. Issued by the whole CTA as cp.async; the caller commits / waits.
template <int HDP>
__device__ __forceinline__ void attn_load_rows(uint32_t sdst, const __nv_bfloat16* base, int64_t ld, int hd, int r0,
                                               int valid, int nrows) {
    constexpr int kChunks = HDP / 8;
    for (int idx = threadIdx.x; idx < nrows * kChunks; idx += blockDim.x) {
        const int rr = idx / kChunks, c = idx - rr * kChunks;
        const int row = r0 + rr;
        const bool ok = row < valid && c * 8 < hd;
        const __nv_bfloat16* src = ok ? base + static_cast<int64_t>(row) * ld + c * 8 : base;
        cp_async16(sdst + rr * attn_row_bytes(HDP) + c * 16, src, ok ? 16u : 0u);
    }
}

__device__ __forceinline__ float quad_max(float v) {
    v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
    return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// A 16 x (8 NT) accumulator fragment (rows row0 / row0 + 8, scaled by u0 / u1) -> bf16 columns [0, hd) of head h in a
// token-major [rows, ld] tensor, at rows row_base + row for row < valid
template <int NT>
__device__ __forceinline__ void attn_store_frag(const float (&o)[NT][4], float u0, float u1, __nv_bfloat16* out,
                                                int64_t ld, int64_t row_base, int valid, int h, int hd, int row0, int t) {
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
        const int row = row0 + hr * 8;
        if (row >= valid) continue;
        const float u = hr ? u1 : u0;
        uint32_t* dst = reinterpret_cast<uint32_t*>(out + (row_base + row) * ld + h * hd);
#pragma unroll
        for (int n = 0; n < NT; ++n) {
            const int col = n * 8 + 2 * t;
            if (col < hd) dst[col / 2] = pack_bf16x2(o[n][2 * hr] * u, o[n][2 * hr + 1] * u);
        }
    }
}

}  // namespace imagd
