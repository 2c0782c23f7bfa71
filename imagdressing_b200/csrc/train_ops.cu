// Backward / training-step kernels that are NOT tensor-core work (SURVEY.md section 8 row a13; reference train.py:573-609 gets
// all of this from torch autograd + DeepSpeed's fused Adam): layout transposes that feed the wgmma GEMM its dgrad / wgrad
// operands, GroupNorm / LayerNorm / activation backward, column reductions (bias and time-embedding gradients), the
// stride-2 col2im and 2x-upsample adjoints, the MSE loss + its gradient, AdamW. All HBM / L2-bound: 128-bit accesses where
// the layout allows, fp32 accumulation, fixed-order (bit-reproducible) reductions — no atomics on data.
#include <cstdlib>

#include "common.cuh"
#include "ptx.cuh"

namespace imagd {

// ------------------------------------------------------------------------------------------------ transposes
// 64 x 64 tiles through shared memory, 128-bit global accesses on both sides: rows are staged as they are (16-byte shared
// stores), every output vector gathers 8 elements of one column with 2-byte shared loads (row pitch 66 elements = 33 words:
// the 8 rows of a gather and the 32 lanes of a warp fall into distinct banks or share a word). `load_row` abstracts where a
// tile row comes from, so the plain transpose and the transposed im2col share the body.
template <typename LoadRow>
__device__ __forceinline__ void transpose_tile_body(LoadRow load_row, __nv_bfloat16* __restrict__ y, int64_t ldy, int r0, int c0,
                                                    int cols, int rows_pad, bool vec_ok) {
    __shared__ __align__(16) __nv_bfloat16 tile[64][72];  // pitch 72 elements = 144 B: 16-byte aligned rows, 36-word stride
    // stage: 64 rows x 8 vectors of 8 elements = 512 vectors, two per thread
#pragma unroll
    for (int it = 0; it < 2; ++it) {
        const int v = threadIdx.x + it * 256;
        const int rr = v >> 3, cv = v & 7;
        uint4 val = load_row(r0 + rr, c0 + cv * 8);
        *reinterpret_cast<uint4*>(&tile[rr][cv * 8]) = val;
    }
    __syncthreads();
    // emit: 64 output rows (source columns) x 8 vectors of 8 source rows
#pragma unroll
    for (int it = 0; it < 2; ++it) {
        const int v = threadIdx.x + it * 256;
        const int cc = v & 63, rv = v >> 6;  // consecutive lanes -> consecutive source columns (distinct banks), same row group
        const int c = c0 + cc, r = r0 + rv * 8;
        if (c >= cols || r >= rows_pad) continue;
        __nv_bfloat16 e[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) e[k] = tile[rv * 8 + k][cc];
        __nv_bfloat16* dst = y + static_cast<int64_t>(c) * ldy + r;
        if (vec_ok && r + 8 <= rows_pad) {
            *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(e);
        } else {
#pragma unroll
            for (int k = 0; k < 8; ++k)
                if (r + k < rows_pad) dst[k] = e[k];
        }
    }
}

// y[c, r] = x[r, c] for r < rows, 0 for rows <= r < rows_pad  (y: [cols, ldy], ldy >= rows_pad).
__global__ void __launch_bounds__(256) transpose_bf16_kernel(const __nv_bfloat16* __restrict__ x, int64_t ldx,
                                                             __nv_bfloat16* __restrict__ y, int64_t ldy, int rows, int cols,
                                                             int rows_pad) {
    const bool in_vec = (ldx % 8 == 0) && ((reinterpret_cast<uintptr_t>(x) & 15) == 0);
    const bool out_vec = (ldy % 8 == 0) && ((reinterpret_cast<uintptr_t>(y) & 15) == 0);
    auto load_row = [&](int r, int c) -> uint4 {
        uint4 val = make_uint4(0u, 0u, 0u, 0u);
        if (r < rows && c < cols) {
            const __nv_bfloat16* src = x + static_cast<int64_t>(r) * ldx + c;
            if (in_vec && c + 8 <= cols) {
                val = __ldg(reinterpret_cast<const uint4*>(src));
            } else {
                __nv_bfloat16 e[8];
#pragma unroll
                for (int k = 0; k < 8; ++k) e[k] = c + k < cols ? src[k] : __float2bfloat16(0.f);
                val = *reinterpret_cast<const uint4*>(e);
            }
        }
        return val;
    };
    transpose_tile_body(load_row, y, ldy, blockIdx.y * 64, blockIdx.x * 64, cols, rows_pad, out_vec);
}

// Transposed im2col of a stride-1 pad-1 3x3 conv input: out[(tap * C + c), p] = x[n, y + ky - 1, x + kx - 1, c] (0 outside),
// p = (n * H + y) * W + x, zero for P <= p < ldo. The B operand [9 Cin, P] of the conv weight-gradient GEMM
// dW[Cout, 9 Cin] = dY^T[Cout, P] . col^T (K = P contiguous). grid (C tiles, P tiles, 9 taps).
__global__ void __launch_bounds__(256) im2col3x3_t_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ out,
                                                          int64_t ldo, int NB, int H, int W, int C) {
    const int tap = blockIdx.z, ky = tap / 3, kx = tap % 3;
    const int P = NB * H * W;
    const bool in_vec = (C % 8 == 0) && ((reinterpret_cast<uintptr_t>(x) & 15) == 0);
    const bool out_vec = (ldo % 8 == 0) && ((reinterpret_cast<uintptr_t>(out) & 15) == 0);
    auto load_row = [&](int p, int c) -> uint4 {
        uint4 val = make_uint4(0u, 0u, 0u, 0u);
        if (p < P && c < C) {
            const int xx = p % W, yy = (p / W) % H, n = p / (W * H);
            const int sy = yy + ky - 1, sx = xx + kx - 1;
            if (sy >= 0 && sy < H && sx >= 0 && sx < W) {
                const __nv_bfloat16* src = x + ((static_cast<int64_t>(n) * H + sy) * W + sx) * C + c;
                if (in_vec && c + 8 <= C) {
                    val = __ldg(reinterpret_cast<const uint4*>(src));
                } else {
                    __nv_bfloat16 e[8];
#pragma unroll
                    for (int k = 0; k < 8; ++k) e[k] = c + k < C ? src[k] : __float2bfloat16(0.f);
                    val = *reinterpret_cast<const uint4*>(e);
                }
            }
        }
        return val;
    };
    transpose_tile_body(load_row, out + static_cast<int64_t>(tap) * C * ldo, ldo, blockIdx.y * 64, blockIdx.x * 64, C,
                        static_cast<int>(ldo), out_vec);
}

// 3x3 conv weight layouts, one CTA per output channel (the row of Cin * 9 values is staged in shared memory, both global
// sides contiguous): mode 0 packs diffusers' [Cout, Cin, 3, 3] into the kernels' tap-major [Cout, 9, Cin]; mode 1 is the
// inverse (a packed weight GRADIENT back to the parameter's layout).
__global__ void __launch_bounds__(256) conv_weight_layout_kernel(const __nv_bfloat16* __restrict__ src,
                                                                 __nv_bfloat16* __restrict__ dst, int Cin, int mode) {
    extern __shared__ __nv_bfloat16 wrow[];
    const int n = Cin * 9;
    const int64_t base = static_cast<int64_t>(blockIdx.x) * n;
    for (int i = threadIdx.x; i < n; i += 256) wrow[i] = src[base + i];
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += 256) {
        int j;
        if (mode == 0) {
            const int t = i / Cin, ci = i - t * Cin;  // dst[t][ci] = src[ci][t]
            j = ci * 9 + t;
        } else {
            const int ci = i / 9, t = i - ci * 9;  // dst[ci][t] = src[t][ci]
            j = t * Cin + ci;
        }
        dst[base + i] = wrow[j];
    }
}

// Packed forward weight [Cout, 9, Cin] -> the data-gradient weight [Cin, 9, Cout] with the taps reversed:
// dst[ci, 8 - t, co] = src[co, t, ci] — nine [Cout, Cin] -> [Cin, Cout] tile transposes, blockIdx.z = tap.
__global__ void __launch_bounds__(256) conv_weight_flip_kernel(const __nv_bfloat16* __restrict__ src, __nv_bfloat16* __restrict__ dst,
                                                               int Cout, int Cin) {
    const int t = blockIdx.z;
    const __nv_bfloat16* x = src + static_cast<int64_t>(t) * Cin;        // rows = co (stride 9 Cin), cols = ci
    __nv_bfloat16* y = dst + static_cast<int64_t>(8 - t) * Cout;          // rows = ci (stride 9 Cout), cols = co
    const int64_t ldx = static_cast<int64_t>(9) * Cin, ldy = static_cast<int64_t>(9) * Cout;
    const bool in_vec = (Cin % 8 == 0) && ((reinterpret_cast<uintptr_t>(src) & 15) == 0);
    const bool out_vec = (Cout % 8 == 0) && ((reinterpret_cast<uintptr_t>(dst) & 15) == 0);
    auto load_row = [&](int r, int c) -> uint4 {
        uint4 val = make_uint4(0u, 0u, 0u, 0u);
        if (r < Cout && c < Cin) {
            const __nv_bfloat16* p = x + static_cast<int64_t>(r) * ldx + c;
            if (in_vec && c + 8 <= Cin) {
                val = __ldg(reinterpret_cast<const uint4*>(p));
            } else {
                __nv_bfloat16 e[8];
#pragma unroll
                for (int k = 0; k < 8; ++k) e[k] = c + k < Cin ? p[k] : __float2bfloat16(0.f);
                val = *reinterpret_cast<const uint4*>(e);
            }
        }
        return val;
    };
    transpose_tile_body(load_row, y, ldy, blockIdx.y * 64, blockIdx.x * 64, Cin, Cout, out_vec);
}

// Adjoint of im2col3x3_s2 (pad 1, stride 2): dx[n, y, x, c] = sum over taps with 2 oy + ky - 1 == y, 2 ox + kx - 1 == x of
// dcol[n, oy, ox, (ky * 3 + kx) * C + c].  One thread per 8 channels of an input pixel.
__global__ void col2im3x3_s2_kernel(const __nv_bfloat16* __restrict__ dcol, __nv_bfloat16* __restrict__ dx, int NB, int H,
                                    int W, int C) {
    const int CV = C / 8;
    const int64_t idx = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    const int64_t total = static_cast<int64_t>(NB) * H * W * CV;
    if (idx >= total) return;
    const int cv = static_cast<int>(idx % CV);
    const int64_t pix = idx / CV;
    const int xx = static_cast<int>(pix % W), yy = static_cast<int>((pix / W) % H), n = static_cast<int>(pix / (static_cast<int64_t>(W) * H));
    const int Ho = H / 2, Wo = W / 2;
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;
    for (int ky = 0; ky < 3; ++ky) {
        const int ty = yy + 1 - ky;
        if (ty < 0 || (ty & 1)) continue;
        const int oy = ty >> 1;
        if (oy >= Ho) continue;
        for (int kx = 0; kx < 3; ++kx) {
            const int tx = xx + 1 - kx;
            if (tx < 0 || (tx & 1)) continue;
            const int ox = tx >> 1;
            if (ox >= Wo) continue;
            const uint4 v = __ldg(reinterpret_cast<const uint4*>(
                dcol + ((static_cast<int64_t>(n) * Ho + oy) * Wo + ox) * (9 * C) + (ky * 3 + kx) * C + cv * 8));
            const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                acc[2 * k] += bf16lo(u[k]);
                acc[2 * k + 1] += bf16hi(u[k]);
            }
        }
    }
    *reinterpret_cast<uint4*>(dx + pix * C + cv * 8) = make_uint4(pack_bf16x2(acc[0], acc[1]), pack_bf16x2(acc[2], acc[3]),
                                                                  pack_bf16x2(acc[4], acc[5]), pack_bf16x2(acc[6], acc[7]));
}

// Adjoint of the nearest-neighbour 2x upsample: dx[n, y, x, :] = sum of the 2x2 block of dy.
__global__ void downsum2x_kernel(const __nv_bfloat16* __restrict__ dy, __nv_bfloat16* __restrict__ dx, int NB, int H, int W,
                                 int C) {
    const int CV = C / 8;
    const int64_t idx = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    const int64_t total = static_cast<int64_t>(NB) * H * W * CV;
    if (idx >= total) return;
    const int cv = static_cast<int>(idx % CV);
    const int64_t pix = idx / CV;
    const int xx = static_cast<int>(pix % W), yy = static_cast<int>((pix / W) % H), n = static_cast<int>(pix / (static_cast<int64_t>(W) * H));
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;
#pragma unroll
    for (int t = 0; t < 4; ++t) {
        const int sy = 2 * yy + (t >> 1), sx = 2 * xx + (t & 1);
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(dy + ((static_cast<int64_t>(n) * 2 * H + sy) * 2 * W + sx) * C + cv * 8));
        const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            acc[2 * k] += bf16lo(u[k]);
            acc[2 * k + 1] += bf16hi(u[k]);
        }
    }
    *reinterpret_cast<uint4*>(dx + pix * C + cv * 8) = make_uint4(pack_bf16x2(acc[0], acc[1]), pack_bf16x2(acc[2], acc[3]),
                                                                  pack_bf16x2(acc[4], acc[5]), pack_bf16x2(acc[6], acc[7]));
}

// ------------------------------------------------------------------------------------------------ column reductions
// Stage 1: block (column slab of 64, group g, row split s) adds rows [s * span, (s+1) * span) of its group in a fixed order
// -> part[s][g][c]; stage 2 folds the splits. MODE 0: sum of x.  MODE 1 (LayerNorm backward): a = dy * xhat, b = dy with
// xhat = (x - mean[r]) * rstd[r]; two outputs.
template <int MODE>
__global__ void __launch_bounds__(256) colreduce_kernel(const __nv_bfloat16* __restrict__ x, int64_t ldx,
                                                        const __nv_bfloat16* __restrict__ dy, int64_t lddy,
                                                        const float* __restrict__ rowstat, float* __restrict__ part, int C,
                                                        int rows_per_group, int groups, int splits) {
    __shared__ float sa[8][64], sb[8][64];
    const int c = blockIdx.x * 64 + (threadIdx.x & 31) * 2;
    const int g = blockIdx.y, s = blockIdx.z;
    const int lane_r = threadIdx.x >> 5;
    const int span = (rows_per_group + splits - 1) / splits;
    const int r_begin = s * span, r_end = min(rows_per_group, r_begin + span);
    float a0 = 0.f, a1 = 0.f, b0 = 0.f, b1 = 0.f;
    if (c < C) {
        for (int r = r_begin + lane_r; r < r_end; r += 8) {
            const int64_t row = static_cast<int64_t>(g) * rows_per_group + r;
            float x0 = __bfloat162float(x[row * ldx + c]);
            float x1 = c + 1 < C ? __bfloat162float(x[row * ldx + c + 1]) : 0.f;
            if (MODE == 0) {
                a0 += x0;
                a1 += x1;
            } else {
                const float mean = rowstat[2 * row], rstd = rowstat[2 * row + 1];
                const float d0 = __bfloat162float(dy[row * lddy + c]);
                const float d1 = c + 1 < C ? __bfloat162float(dy[row * lddy + c + 1]) : 0.f;
                a0 += d0 * (x0 - mean) * rstd;
                a1 += d1 * (x1 - mean) * rstd;
                b0 += d0;
                b1 += d1;
            }
        }
    }
    sa[lane_r][(threadIdx.x & 31) * 2] = a0;
    sa[lane_r][(threadIdx.x & 31) * 2 + 1] = a1;
    sb[lane_r][(threadIdx.x & 31) * 2] = b0;
    sb[lane_r][(threadIdx.x & 31) * 2 + 1] = b1;
    __syncthreads();
    if (threadIdx.x < 64) {
        const int cc = blockIdx.x * 64 + threadIdx.x;
        if (cc < C) {
            float a = 0.f, b = 0.f;
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                a += sa[k][threadIdx.x];
                b += sb[k][threadIdx.x];
            }
            const int64_t o = (static_cast<int64_t>(s) * groups + g) * C + cc;
            part[o] = a;
            if (MODE == 1) part[static_cast<int64_t>(splits) * groups * C + o] = b;
        }
    }
}

// out[k][g][c] = sum_s part[k][s][g][c]   (k < nout)
__global__ void colreduce_fold_kernel(const float* __restrict__ part, void* __restrict__ out0, void* __restrict__ out1, int C,
                                      int groups, int splits, int out_bf16) {
    const int64_t idx = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    const int64_t n = static_cast<int64_t>(groups) * C;
    if (idx >= n) return;
    float a = 0.f, b = 0.f;
    for (int s = 0; s < splits; ++s) {
        a += part[static_cast<int64_t>(s) * n + idx];
        if (out1) b += part[(static_cast<int64_t>(splits) + s) * n + idx];
    }
    if (out_bf16) {  // parameter gradients of a bf16 model: written in the parameter's dtype, no conversion launch
        static_cast<__nv_bfloat16*>(out0)[idx] = __float2bfloat16(a);
        if (out1) static_cast<__nv_bfloat16*>(out1)[idx] = __float2bfloat16(b);
    } else {
        static_cast<float*>(out0)[idx] = a;
        if (out1) static_cast<float*>(out1)[idx] = b;
    }
}

// ------------------------------------------------------------------------------------------------ LayerNorm backward
// One warp per row, VPL 128-bit vectors per lane (C <= VPL * 256): recompute mean / rstd (two-pass on the registers),
// dx = rstd * (g - mean(g) - xhat * mean(g xhat)) with g = dy * gamma; writes {mean, rstd} per row for the column reduction that
// produces dgamma / dbeta.
template <int VPL>
__global__ void __launch_bounds__(256) layernorm_bwd_kernel(const __nv_bfloat16* __restrict__ x, int64_t ldx,
                                                            const __nv_bfloat16* __restrict__ dy, int64_t lddy,
                                                            __nv_bfloat16* __restrict__ dx, int64_t lddx,
                                                            const float* __restrict__ gamma, float* __restrict__ rowstat,
                                                            int rows, int C, float eps) {
    const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    const int CV = C / 8;
    float xv[VPL][8], gv[VPL][8];
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
        const int cv = lane + 32 * i;
#pragma unroll
        for (int k = 0; k < 8; ++k) xv[i][k] = gv[i][k] = 0.f;
        if (cv < CV) {
            const uint4 a = __ldg(reinterpret_cast<const uint4*>(x + static_cast<int64_t>(row) * ldx + cv * 8));
            const uint4 d = __ldg(reinterpret_cast<const uint4*>(dy + static_cast<int64_t>(row) * lddy + cv * 8));
            const uint32_t au[4] = {a.x, a.y, a.z, a.w}, du[4] = {d.x, d.y, d.z, d.w};
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                xv[i][2 * k] = bf16lo(au[k]);
                xv[i][2 * k + 1] = bf16hi(au[k]);
                gv[i][2 * k] = bf16lo(du[k]) * (gamma ? __ldg(gamma + cv * 8 + 2 * k) : 1.f);
                gv[i][2 * k + 1] = bf16hi(du[k]) * (gamma ? __ldg(gamma + cv * 8 + 2 * k + 1) : 1.f);
            }
#pragma unroll
            for (int k = 0; k < 8; ++k) sum += xv[i][k];
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float mean = sum / C;
    float var = 0.f;
#pragma unroll
    for (int i = 0; i < VPL; ++i)
        if (lane + 32 * i < CV) {
#pragma unroll
            for (int k = 0; k < 8; ++k) var += (xv[i][k] - mean) * (xv[i][k] - mean);
        }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) var += __shfl_xor_sync(0xffffffffu, var, o);
    const float rstd = rsqrtf(var / C + eps);
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < VPL; ++i)
        if (lane + 32 * i < CV) {
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                xv[i][k] = (xv[i][k] - mean) * rstd;  // xhat from here on
                s1 += gv[i][k];
                s2 += gv[i][k] * xv[i][k];
            }
        }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        s1 += __shfl_xor_sync(0xffffffffu, s1, o);
        s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    }
    s1 /= C;
    s2 /= C;
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
        const int cv = lane + 32 * i;
        if (cv < CV) {
            float o[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) o[k] = rstd * (gv[i][k] - s1 - xv[i][k] * s2);
            *reinterpret_cast<uint4*>(dx + static_cast<int64_t>(row) * lddx + cv * 8) =
                make_uint4(pack_bf16x2(o[0], o[1]), pack_bf16x2(o[2], o[3]), pack_bf16x2(o[4], o[5]), pack_bf16x2(o[6], o[7]));
        }
    }
    if (lane == 0) {
        rowstat[2 * row] = mean;
        rowstat[2 * row + 1] = rstd;
    }
}

// ------------------------------------------------------------------------------------------------ GroupNorm backward
__device__ __forceinline__ float silu_grad(float z) {
    const float s = 1.f / (1.f + __expf(-z));
    return s * (1.f + z * (1.f - s));
}

// Forward-pass statistics (mean, rstd per sample and group; imagd_groupnorm_stats_bf16) come in as `fstat`. Two steps, both
// with the forward kernel's coalesced layout (thread = (pixel row slot, 8-channel vector), 128-bit loads):
//   groupnorm_bwd_partial_kernel  grid (chunks, NB): per channel of its pixel chunk  a = sum dz xhat,  b = sum dz
//                                 (dz = dy * act'(z), z = xhat gamma + beta) -> part[n][chunk][{a, b}][C]
//   groupnorm_bwd_fold_kernel     grid (NB): chunks -> sample in a fixed order -> pc[{a, b}][n][c] (these fold over n into
//                                 dgamma / dbeta) and per group S1 = sum_c gamma_c b_c, S2 = sum_c gamma_c a_c ->
//                                 stat[n][g] = {mean, rstd, S1 / m, S2 / m}
constexpr int kGbThreads = 512;
__global__ void __launch_bounds__(kGbThreads) groupnorm_bwd_partial_kernel(
    const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dy, int HW, int C, int groups, int chunks,
    const float* __restrict__ gamma, const float* __restrict__ beta, int fuse_silu, const float* __restrict__ fstat,
    float* __restrict__ part) {
    extern __shared__ float sm[];  // [rows][C] a | [rows][C] b  (rows = kGbThreads / CV row slots)
    const int n = blockIdx.y, chunk = blockIdx.x;
    const int CV = C / 8;
    const int rows = kGbThreads / CV;
    const int cpg = C / groups;
    const int ppc = (HW + chunks - 1) / chunks;
    const int p_begin = chunk * ppc, p_end = min(HW, p_begin + ppc);
    const int cv = threadIdx.x % CV, prow = threadIdx.x / CV;
    float* sa = sm;
    float* sb = sm + rows * C;
    if (prow < rows) {
        float a[8], b[8], sc[8], sh[8], ga[8], be[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int c = cv * 8 + k;
            const float* st = fstat + (static_cast<int64_t>(n) * groups + c / cpg) * 2;
            sc[k] = st[1];
            sh[k] = -st[0] * st[1];
            ga[k] = gamma ? gamma[c] : 1.f;
            be[k] = beta ? beta[c] : 0.f;
            a[k] = b[k] = 0.f;
        }
        const int64_t base = static_cast<int64_t>(n) * HW * C + cv * 8;
        for (int p = p_begin + prow; p < p_end; p += rows) {
            const uint4 xv = __ldg(reinterpret_cast<const uint4*>(x + base + static_cast<int64_t>(p) * C));
            const uint4 dv = __ldg(reinterpret_cast<const uint4*>(dy + base + static_cast<int64_t>(p) * C));
            const uint32_t xu[4] = {xv.x, xv.y, xv.z, xv.w}, du[4] = {dv.x, dv.y, dv.z, dv.w};
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const float xe = (k & 1) ? bf16hi(xu[k >> 1]) : bf16lo(xu[k >> 1]);
                float dz = (k & 1) ? bf16hi(du[k >> 1]) : bf16lo(du[k >> 1]);
                const float xh = fmaf(xe, sc[k], sh[k]);
                if (fuse_silu) dz *= silu_grad(fmaf(xh, ga[k], be[k]));
                a[k] = fmaf(dz, xh, a[k]);
                b[k] += dz;
            }
        }
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            sa[prow * C + cv * 8 + k] = a[k];
            sb[prow * C + cv * 8 + k] = b[k];
        }
    }
    __syncthreads();
    float* dst = part + (static_cast<int64_t>(n) * chunks + chunk) * 2 * C;
    for (int c = threadIdx.x; c < C; c += kGbThreads) {
        float fa = 0.f, fb = 0.f;
        for (int r = 0; r < rows; ++r) {
            fa += sa[r * C + c];
            fb += sb[r * C + c];
        }
        dst[c] = fa;
        dst[C + c] = fb;
    }
}

// grid (group blocks, NB): a CTA owns `gpb` whole groups (<= 128 channels) of one sample; 4 chunk lanes per channel add the
// chunk partials in a fixed order, the lanes meet in shared memory, then one thread per group folds its channels.
__global__ void __launch_bounds__(kGbThreads) groupnorm_bwd_fold_kernel(const float* __restrict__ part, int HW, int C, int groups,
                                                                        int chunks, const float* __restrict__ gamma,
                                                                        const float* __restrict__ fstat,
                                                                        float* __restrict__ stat, float* __restrict__ pc,
                                                                        int NB, int gpb) {
    __shared__ float sa[4][128], sb[4][128];
    const int n = blockIdx.y;
    const int cpg = C / groups;
    const int g0 = blockIdx.x * gpb;
    const int ng = min(gpb, groups - g0);
    const int nch = ng * cpg;                       // channels of this CTA (<= 128)
    const int cl = threadIdx.x & 127, lane = threadIdx.x >> 7;  // 128 channel slots x 4 chunk lanes
    float a = 0.f, b = 0.f;
    if (cl < nch) {
        const int c = g0 * cpg + cl;
        const float* src = part + static_cast<int64_t>(n) * chunks * 2 * C + c;
        for (int k = lane; k < chunks; k += 4) {
            a += src[static_cast<int64_t>(k) * 2 * C];
            b += src[static_cast<int64_t>(k) * 2 * C + C];
        }
    }
    sa[lane][cl] = a;
    sb[lane][cl] = b;
    __syncthreads();
    if (lane == 0 && cl < nch) {
        const int c = g0 * cpg + cl;
        a = (sa[0][cl] + sa[1][cl]) + (sa[2][cl] + sa[3][cl]);
        b = (sb[0][cl] + sb[1][cl]) + (sb[2][cl] + sb[3][cl]);
        pc[static_cast<int64_t>(n) * C + c] = a;
        pc[static_cast<int64_t>(NB) * C + static_cast<int64_t>(n) * C + c] = b;
        const float ga = gamma ? gamma[c] : 1.f;
        sa[0][cl] = ga * a;
        sb[0][cl] = ga * b;
    }
    __syncthreads();
    if (threadIdx.x < ng) {
        const int g = g0 + threadIdx.x;
        const float m = static_cast<float>(HW) * cpg;
        float s2 = 0.f, s1 = 0.f;
        for (int k = threadIdx.x * cpg; k < (threadIdx.x + 1) * cpg; ++k) {
            s2 += sa[0][k];
            s1 += sb[0][k];
        }
        float* o = stat + (static_cast<int64_t>(n) * groups + g) * 4;
        o[0] = fstat[(static_cast<int64_t>(n) * groups + g) * 2];
        o[1] = fstat[(static_cast<int64_t>(n) * groups + g) * 2 + 1];
        o[2] = s1 / m;
        o[3] = s2 / m;
    }
}

// dx = rstd * (dz gamma - S1/m - xhat S2/m), elementwise over [NB, HW, C] (8 channels per thread).
__global__ void groupnorm_bwd_apply_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dy,
                                           __nv_bfloat16* __restrict__ dx, int HW, int C, int groups,
                                           const float* __restrict__ gamma, const float* __restrict__ beta, int fuse_silu,
                                           const float* __restrict__ stat, int64_t total_vec) {
    const int64_t idx = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= total_vec) return;
    const int CV = C / 8;
    const int cv = static_cast<int>(idx % CV);
    const int64_t pix = idx / CV;
    const int n = static_cast<int>(pix / HW);
    const int cpg = C / groups;
    const uint4 xv = __ldg(reinterpret_cast<const uint4*>(x + pix * C + cv * 8));
    const uint4 dv = __ldg(reinterpret_cast<const uint4*>(dy + pix * C + cv * 8));
    const uint32_t xu[4] = {xv.x, xv.y, xv.z, xv.w}, du[4] = {dv.x, dv.y, dv.z, dv.w};
    float o[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int c = cv * 8 + k;
        const float* st = stat + (static_cast<int64_t>(n) * groups + c / cpg) * 4;
        const float xe = (k & 1) ? bf16hi(xu[k >> 1]) : bf16lo(xu[k >> 1]);
        const float de = (k & 1) ? bf16hi(du[k >> 1]) : bf16lo(du[k >> 1]);
        const float ga = gamma ? gamma[c] : 1.f, be = beta ? beta[c] : 0.f;
        const float xh = (xe - st[0]) * st[1];
        float dz = de;
        if (fuse_silu) dz *= silu_grad(fmaf(xh, ga, be));
        o[k] = st[1] * (dz * ga - st[2] - xh * st[3]);
    }
    *reinterpret_cast<uint4*>(dx + pix * C + cv * 8) =
        make_uint4(pack_bf16x2(o[0], o[1]), pack_bf16x2(o[2], o[3]), pack_bf16x2(o[4], o[5]), pack_bf16x2(o[6], o[7]));
}

// ------------------------------------------------------------------------------------------------ activations
__device__ __forceinline__ float gelu_grad(float x) {
    const float cdf = 0.5f * (1.0f + erf_fast(x * 0.70710678118654752f));
    return cdf + x * 0.3989422804014327f * __expf(-0.5f * x * x);
}

// mode 2 SiLU, 3 GELU(erf). dy == nullptr: y = act(x); else y = dy * act'(x). Element pairs.
__global__ void act_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dy,
                           __nv_bfloat16* __restrict__ y, int64_t n, int mode) {
    const int64_t i = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) * 2;
    if (i >= n) return;
    auto f = [&](float v, float g, bool bwd) {
        if (!bwd) return mode == 2 ? silu(v) : gelu_erf(v);
        return g * (mode == 2 ? silu_grad(v) : gelu_grad(v));
    };
    if (i + 1 < n) {
        const __nv_bfloat162 xv = *reinterpret_cast<const __nv_bfloat162*>(x + i);
        __nv_bfloat162 gv = xv;
        if (dy) gv = *reinterpret_cast<const __nv_bfloat162*>(dy + i);
        __nv_bfloat162 o;
        o.x = __float2bfloat16(f(__bfloat162float(xv.x), __bfloat162float(gv.x), dy != nullptr));
        o.y = __float2bfloat16(f(__bfloat162float(xv.y), __bfloat162float(gv.y), dy != nullptr));
        *reinterpret_cast<__nv_bfloat162*>(y + i) = o;
    } else {
        y[i] = __float2bfloat16(f(__bfloat162float(x[i]), dy ? __bfloat162float(dy[i]) : 0.f, dy != nullptr));
    }
}

// GEGLU on an un-fused projection h = [value | gate] ([M, 2F], diffusers-0.24 GEGLU: hidden, gate = proj(x).chunk(2)):
// forward out = value * gelu(gate); backward dh = [dout * gelu(gate) | dout * value * gelu'(gate)].
__global__ void geglu_kernel(const __nv_bfloat16* __restrict__ h, int64_t ldh, const __nv_bfloat16* __restrict__ dout,
                             __nv_bfloat16* __restrict__ out, int64_t ldo, int64_t M, int F) {
    const int64_t idx = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    const int FV = F / 2;
    if (idx >= M * FV) return;
    const int64_t r = idx / FV;
    const int c = static_cast<int>(idx % FV) * 2;
    const __nv_bfloat162 v = *reinterpret_cast<const __nv_bfloat162*>(h + r * ldh + c);
    const __nv_bfloat162 g = *reinterpret_cast<const __nv_bfloat162*>(h + r * ldh + F + c);
    const float v0 = __bfloat162float(v.x), v1 = __bfloat162float(v.y), g0 = __bfloat162float(g.x), g1 = __bfloat162float(g.y);
    if (dout == nullptr) {
        __nv_bfloat162 o;
        o.x = __float2bfloat16(v0 * gelu_erf(g0));
        o.y = __float2bfloat16(v1 * gelu_erf(g1));
        *reinterpret_cast<__nv_bfloat162*>(out + r * ldo + c) = o;
    } else {  // out = dh [M, 2F] (ldo), dout [M, F] contiguous
        const __nv_bfloat162 d = *reinterpret_cast<const __nv_bfloat162*>(dout + r * F + c);
        const float d0 = __bfloat162float(d.x), d1 = __bfloat162float(d.y);
        __nv_bfloat162 dv, dg;
        dv.x = __float2bfloat16(d0 * gelu_erf(g0));
        dv.y = __float2bfloat16(d1 * gelu_erf(g1));
        dg.x = __float2bfloat16(d0 * v0 * gelu_grad(g0));
        dg.y = __float2bfloat16(d1 * v1 * gelu_grad(g1));
        *reinterpret_cast<__nv_bfloat162*>(out + r * ldo + c) = dv;
        *reinterpret_cast<__nv_bfloat162*>(out + r * ldo + F + c) = dg;
    }
}

// ------------------------------------------------------------------------------------------------ loss
// MSE(pred, target) (reference train.py:577, F.mse_loss(..., reduction="mean")) + its gradient 2 (pred - target) / n, one pass.
// part[blockIdx.x] = block partial; mse_fold_kernel adds the partials in order.
__global__ void __launch_bounds__(256) mse_kernel(const float* __restrict__ pred, const float* __restrict__ target,
                                                  float* __restrict__ grad, float* __restrict__ part, int64_t n, float gscale) {
    __shared__ float red[256];
    float s = 0.f;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
         i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const float d = pred[i] - target[i];
        s += d * d;
        grad[i] = gscale * d;
    }
    red[threadIdx.x] = s;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) part[blockIdx.x] = red[0];
}
__global__ void mse_fold_kernel(const float* __restrict__ part, int nparts, float inv_n, float* __restrict__ loss) {
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        float s = 0.f;
        for (int i = 0; i < nparts; ++i) s += part[i];
        loss[0] = s * inv_n;
    }
}

// ------------------------------------------------------------------------------------------------ optimizer
// AdamW (decoupled weight decay; reference train.py:386-398 torch.optim.AdamW, run by DeepSpeed in bf16 mode with fp32 master
// weights): fp32 master / moments, bf16 gradient in, bf16 working copy out. bc1 = 1 - beta1^t, bc2 = 1 - beta2^t.
__global__ void adamw_kernel(float* __restrict__ master, __nv_bfloat16* __restrict__ param, const __nv_bfloat16* __restrict__ grad,
                             float* __restrict__ m, float* __restrict__ v, int64_t n, float lr, float b1, float b2, float eps,
                             float wd, float bc1, float bc2, float gscale) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float g = __bfloat162float(grad[i]) * gscale;
    const float mi = b1 * m[i] + (1.f - b1) * g;
    const float vi = b2 * v[i] + (1.f - b2) * g * g;
    m[i] = mi;
    v[i] = vi;
    float w = master[i];
    w -= lr * wd * w;
    w -= lr * (mi / bc1) / (sqrtf(vi / bc2) + eps);
    master[i] = w;
    param[i] = __float2bfloat16(w);
}

// The same with the step-dependent scalars in DEVICE memory — hyper = {lr, weight_decay, step (1-based, as float), grad_scale} —
// so that a captured CUDA graph of the whole training step replays with a moving step count and learning-rate schedule.
// CLIP: the update also reads the global-norm state grad_norm_clip_kernel wrote, clip = {norm, coef, finite, skipped}: a
// non-finite gradient leaves every buffer untouched, otherwise the gradient scale is grad_scale * coef.
template <bool CLIP>
__global__ void adamw_dev_kernel(float* __restrict__ master, __nv_bfloat16* __restrict__ param,
                                 const __nv_bfloat16* __restrict__ grad, float* __restrict__ m, float* __restrict__ v, int64_t n,
                                 float b1, float b2, float eps, const float* __restrict__ hyper, const double* __restrict__ clip) {
    if (CLIP && clip[2] == 0.0) return;  // uniform over the grid: the skipped update
    __shared__ float bc[2];
    if (threadIdx.x == 0) {  // the two powf calls once per CTA, not per element
        bc[0] = 1.f - powf(b1, hyper[2]);
        bc[1] = 1.f - powf(b2, hyper[2]);
    }
    __syncthreads();
    const float lr = hyper[0], wd = hyper[1], gscale = CLIP ? hyper[3] * static_cast<float>(clip[1]) : hyper[3];
    const float bc1 = bc[0], bc2 = bc[1];
    const int64_t i4 = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) * 4;  // four elements per thread, 128-bit accesses
    if (i4 >= n) return;
    if (i4 + 4 <= n) {
        float4 w4 = *reinterpret_cast<const float4*>(master + i4);
        float4 m4 = *reinterpret_cast<const float4*>(m + i4);
        float4 v4 = *reinterpret_cast<const float4*>(v + i4);
        const uint2 g2 = *reinterpret_cast<const uint2*>(grad + i4);
        const float g[4] = {bf16lo(g2.x) * gscale, bf16hi(g2.x) * gscale, bf16lo(g2.y) * gscale, bf16hi(g2.y) * gscale};
        float* w = reinterpret_cast<float*>(&w4);
        float* mm = reinterpret_cast<float*>(&m4);
        float* vv = reinterpret_cast<float*>(&v4);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            mm[k] = b1 * mm[k] + (1.f - b1) * g[k];
            vv[k] = b2 * vv[k] + (1.f - b2) * g[k] * g[k];
            w[k] -= lr * wd * w[k];
            w[k] -= lr * (mm[k] / bc1) / (sqrtf(vv[k] / bc2) + eps);
        }
        *reinterpret_cast<float4*>(master + i4) = w4;
        *reinterpret_cast<float4*>(m + i4) = m4;
        *reinterpret_cast<float4*>(v + i4) = v4;
        *reinterpret_cast<uint2*>(param + i4) = make_uint2(pack_bf16x2(w[0], w[1]), pack_bf16x2(w[2], w[3]));
    } else {
        for (int64_t i = i4; i < n; ++i) {
            const float g = __bfloat162float(grad[i]) * gscale;
            const float mi = b1 * m[i] + (1.f - b1) * g;
            const float vi = b2 * v[i] + (1.f - b2) * g * g;
            m[i] = mi;
            v[i] = vi;
            float w = master[i];
            w -= lr * wd * w;
            w -= lr * (mi / bc1) / (sqrtf(vi / bc2) + eps);
            master[i] = w;
            param[i] = __float2bfloat16(w);
        }
    }
}

// ------------------------------------------------------------------------------------------------ global gradient norm
// Gradient clipping of the reference's DeepSpeed config ("gradient_clipping": 1.0): the L2 norm of the averaged gradient
// scale * grad, coef = min(1, max_norm / (norm + 1e-6)), and a finite flag (a non-finite gradient skips the update). Squares
// add up in fp64: the largest finite bf16 squared is ~1.2e77, so no finite input overflows the sum, and the sum is non-finite
// exactly when an element is Inf / NaN. Deterministic: one partial per block into `part`, the last block to arrive folds them
// in a fixed order and resets the arrival counter (graph replays find it at zero). The grid depends on n only.
constexpr int kNormThreads = 256;
constexpr int kNormUnroll = 4;  // 128-bit loads in flight per thread

__device__ __forceinline__ double sumsq_bf16x8(const uint4 u, double acc) {
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const double lo = bf16lo(w[k]), hi = bf16hi(w[k]);
        acc = fma(lo, lo, acc);
        acc = fma(hi, hi, acc);
    }
    return acc;
}

// state = {norm, coef, finite (1 / 0), skipped updates}; hyper[2] (the AdamW step count) advances on a finite norm only.
__global__ void __launch_bounds__(kNormThreads) grad_norm_clip_kernel(const __nv_bfloat16* __restrict__ grad, int64_t n,
                                                                      float max_norm, float* __restrict__ hyper,
                                                                      double* __restrict__ state, unsigned int* __restrict__ counter,
                                                                      double* __restrict__ part) {
    __shared__ double red[kNormThreads / 32];
    __shared__ bool last;
    const int64_t nvec = n / 8;
    const uint4* g8 = reinterpret_cast<const uint4*>(grad);
    const int64_t stride = static_cast<int64_t>(gridDim.x) * kNormThreads;
    int64_t i = static_cast<int64_t>(blockIdx.x) * kNormThreads + threadIdx.x;
    double acc = 0.0;
    for (; i + (kNormUnroll - 1) * stride < nvec; i += kNormUnroll * stride) {
        uint4 u[kNormUnroll];
#pragma unroll
        for (int k = 0; k < kNormUnroll; ++k) u[k] = __ldg(g8 + i + k * stride);
#pragma unroll
        for (int k = 0; k < kNormUnroll; ++k) acc = sumsq_bf16x8(u[k], acc);
    }
    for (; i < nvec; i += stride) acc = sumsq_bf16x8(__ldg(g8 + i), acc);
    if (blockIdx.x == 0 && threadIdx.x < n - nvec * 8) {  // the < 8 trailing elements
        const double e = __bfloat162float(grad[nvec * 8 + threadIdx.x]);
        acc = fma(e, e, acc);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
#pragma unroll
        for (int w = 0; w < kNormThreads / 32; ++w) s += red[w];
        part[blockIdx.x] = s;
        __threadfence();
        last = atomicAdd(counter, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!last || threadIdx.x >= 32) return;
    __threadfence();
    double s = 0.0;
    for (unsigned b = threadIdx.x; b < gridDim.x; b += 32) s += __ldcg(part + b);  // L2: the other blocks' partials
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (threadIdx.x == 0) {
        const bool finite = isfinite(s);
        const double norm = sqrt(s) * static_cast<double>(hyper[3]);
        state[0] = norm;
        state[1] = finite ? fmin(1.0, static_cast<double>(max_norm) / (norm + 1e-6)) : 0.0;
        state[2] = finite ? 1.0 : 0.0;
        if (finite) hyper[2] += 1.f;
        else state[3] += 1.0;
        *counter = 0u;
    }
}

static int grad_norm_blocks(int64_t n) {
    const int64_t per_block = static_cast<int64_t>(kNormThreads) * kNormUnroll * 8;
    const int64_t b = (n + per_block - 1) / per_block;
    return static_cast<int>(b < 1 ? 1 : (b > kNumSms * 4 ? kNumSms * 4 : b));
}

static inline unsigned blocks_for(int64_t n, int threads) { return static_cast<unsigned>((n + threads - 1) / threads); }

}  // namespace imagd

using namespace imagd;
#define BF(p) static_cast<const __nv_bfloat16*>(p)
#define BFW(p) static_cast<__nv_bfloat16*>(p)
#define ST(s) static_cast<cudaStream_t>(s)

extern "C" int imagd_transpose_bf16(const void* x, int64_t ldx, void* y, int64_t ldy, int rows, int cols, int rows_pad,
                                    imagd_stream stream) {
    IMAGD_CHECK_ARG(x && y && rows > 0 && cols > 0 && rows_pad >= rows && ldy >= rows_pad && ldx >= cols, "transpose: bad argument");
    dim3 grid((cols + 63) / 64, (rows_pad + 63) / 64);
    transpose_bf16_kernel<<<grid, 256, 0, ST(stream)>>>(BF(x), ldx, BFW(y), ldy, rows, cols, rows_pad);
    IMAGD_LAUNCH_CHECK("transpose_bf16_kernel");
    return IMAGD_OK;
}

extern "C" int imagd_conv_weight_layout_bf16(const void* src, void* dst, int Cout, int Cin, int mode, imagd_stream stream) {
    IMAGD_CHECK_ARG(src && dst && Cout > 0 && Cin > 0 && Cin * 9 * 2 <= 48 * 1024 && (mode == 0 || mode == 1),
                    "conv_weight_layout: bad argument");
    conv_weight_layout_kernel<<<Cout, 256, static_cast<size_t>(Cin) * 9 * 2, ST(stream)>>>(BF(src), BFW(dst), Cin, mode);
    IMAGD_LAUNCH_CHECK("conv_weight_layout_kernel");
    return IMAGD_OK;
}

extern "C" int imagd_conv_weight_flip_bf16(const void* src, void* dst, int Cout, int Cin, imagd_stream stream) {
    IMAGD_CHECK_ARG(src && dst && Cout > 0 && Cin > 0, "conv_weight_flip: bad argument");
    dim3 grid((Cin + 63) / 64, (Cout + 63) / 64, 9);
    conv_weight_flip_kernel<<<grid, 256, 0, ST(stream)>>>(BF(src), BFW(dst), Cout, Cin);
    IMAGD_LAUNCH_CHECK("conv_weight_flip_kernel");
    return IMAGD_OK;
}

extern "C" int imagd_im2col3x3_t_bf16(const void* x, void* out, int64_t ldo, int NB, int H, int W, int C, imagd_stream stream) {
    IMAGD_CHECK_ARG(x && out && NB > 0 && H > 0 && W > 0 && C > 0 && ldo >= static_cast<int64_t>(NB) * H * W, "im2col3x3_t: bad argument");
    dim3 grid((C + 63) / 64, static_cast<unsigned>((ldo + 63) / 64), 9);
    im2col3x3_t_kernel<<<grid, 256, 0, ST(stream)>>>(BF(x), BFW(out), ldo, NB, H, W, C);
    IMAGD_LAUNCH_CHECK("im2col3x3_t_kernel");
    return IMAGD_OK;
}

extern "C" int imagd_col2im3x3_s2_bf16(const void* dcol, void* dx, int NB, int H, int W, int C, imagd_stream stream) {
    IMAGD_CHECK_ARG(dcol && dx && C % 8 == 0 && H % 2 == 0 && W % 2 == 0, "col2im3x3_s2: bad argument");
    const int64_t total = static_cast<int64_t>(NB) * H * W * (C / 8);
    col2im3x3_s2_kernel<<<blocks_for(total, 256), 256, 0, ST(stream)>>>(BF(dcol), BFW(dx), NB, H, W, C);
    IMAGD_LAUNCH_CHECK("col2im3x3_s2_kernel");
    return IMAGD_OK;
}

extern "C" int imagd_downsum2x_bf16(const void* dy, void* dx, int NB, int H, int W, int C, imagd_stream stream) {
    IMAGD_CHECK_ARG(dy && dx && C % 8 == 0, "downsum2x: bad argument");
    const int64_t total = static_cast<int64_t>(NB) * H * W * (C / 8);
    downsum2x_kernel<<<blocks_for(total, 256), 256, 0, ST(stream)>>>(BF(dy), BFW(dx), NB, H, W, C);
    IMAGD_LAUNCH_CHECK("downsum2x_kernel");
    return IMAGD_OK;
}

static int colreduce_splits(int rows_per_group, int groups, int C) {
    const int slabs = (C + 63) / 64;
    int s = (kNumSms * 2) / (slabs * groups > 0 ? slabs * groups : 1);
    const int by_rows = (rows_per_group + 63) / 64;  // at least 64 rows per split
    if (s > by_rows) s = by_rows;
    if (s > 64) s = 64;
    return s < 1 ? 1 : s;
}

extern "C" int64_t imagd_colreduce_ws_bytes(int rows_per_group, int groups, int C) {
    return static_cast<int64_t>(2) * colreduce_splits(rows_per_group, groups, C) * groups * C * 4;
}

extern "C" int imagd_colsum_bf16(const void* x, int64_t ldx, int rows_per_group, int groups, int C, void* out, int out_bf16,
                                 void* ws, imagd_stream stream) {
    IMAGD_CHECK_ARG(x && out && ws && rows_per_group > 0 && groups > 0 && C > 0, "colsum: bad argument");
    const int splits = colreduce_splits(rows_per_group, groups, C);
    dim3 grid((C + 63) / 64, groups, splits);
    colreduce_kernel<0><<<grid, 256, 0, ST(stream)>>>(BF(x), ldx, nullptr, 0, nullptr, static_cast<float*>(ws), C,
                                                      rows_per_group, groups, splits);
    IMAGD_LAUNCH_CHECK("colreduce_kernel<0>");
    colreduce_fold_kernel<<<blocks_for(static_cast<int64_t>(groups) * C, 256), 256, 0, ST(stream)>>>(
        static_cast<const float*>(ws), out, nullptr, C, groups, splits, out_bf16);
    IMAGD_LAUNCH_CHECK("colreduce_fold_kernel");
    return IMAGD_OK;
}

extern "C" int imagd_layernorm_bwd_bf16(const void* x, int64_t ldx, const void* dy, int64_t lddy, void* dx, int64_t lddx,
                                        int rows, int C, const float* gamma, float eps, void* dgamma, void* dbeta,
                                        int out_bf16, float* rowstat, void* ws, imagd_stream stream) {
    IMAGD_CHECK_ARG(x && dy && dx && rowstat && rows > 0 && C > 0 && C % 2 == 0 && C <= 2048, "layernorm_bwd: bad argument");
    IMAGD_CHECK_ARG(ldx % 2 == 0 && lddy % 2 == 0 && lddx % 2 == 0, "layernorm_bwd: odd row stride");
    IMAGD_CHECK_ARG(C % 8 == 0 && ldx % 8 == 0 && lddy % 8 == 0 && lddx % 8 == 0 && imagd::aligned16(x) && imagd::aligned16(dy) &&
                        imagd::aligned16(dx), "layernorm_bwd: C / strides must be multiples of 8, pointers 16-byte aligned");
#define IMAGD_LNB(V) layernorm_bwd_kernel<V><<<(rows + 7) / 8, 256, 0, ST(stream)>>>(BF(x), ldx, BF(dy), lddy, BFW(dx), lddx, gamma, rowstat, rows, C, eps)
    if (C <= 512) IMAGD_LNB(2);
    else if (C <= 768) IMAGD_LNB(3);
    else if (C <= 1280) IMAGD_LNB(5);
    else IMAGD_LNB(8);
#undef IMAGD_LNB
    IMAGD_LAUNCH_CHECK("layernorm_bwd_kernel");
    if (dgamma != nullptr) {
        IMAGD_CHECK_ARG(dbeta && ws, "layernorm_bwd: dbeta / ws");
        const int splits = colreduce_splits(rows, 1, C);
        dim3 grid((C + 63) / 64, 1, splits);
        colreduce_kernel<1><<<grid, 256, 0, ST(stream)>>>(BF(x), ldx, BF(dy), lddy, rowstat, static_cast<float*>(ws), C, rows, 1,
                                                          splits);
        IMAGD_LAUNCH_CHECK("colreduce_kernel<1>");
        colreduce_fold_kernel<<<blocks_for(C, 256), 256, 0, ST(stream)>>>(static_cast<const float*>(ws), dgamma, dbeta, C, 1,
                                                                         splits, out_bf16);
        IMAGD_LAUNCH_CHECK("colreduce_fold_kernel");
    }
    return IMAGD_OK;
}

static int gn_bwd_chunks(int HW, int NB) {
    int c = (HW + 15) / 16;
    const int cap = (kNumSms * 2) / (NB > 0 ? NB : 1);
    if (c > 64) c = 64;
    if (c > cap) c = cap;
    return c < 1 ? 1 : c;
}

extern "C" int64_t imagd_groupnorm_bwd_ws_bytes(int NB, int HW, int C, int groups) {
    // stat [NB * groups * 4] | pc [2 * NB * C] | part [NB * chunks * 2 * C]
    return (static_cast<int64_t>(NB) * groups * 4 + static_cast<int64_t>(2) * NB * C +
            static_cast<int64_t>(NB) * gn_bwd_chunks(HW, NB) * 2 * C) * 4;
}

extern "C" int imagd_groupnorm_bwd_bf16(const void* x, const void* dy, void* dx, int NB, int HW, int C, int groups,
                                        const float* gamma, const float* beta, const float* fwd_stats, int fuse_silu,
                                        void* dgamma, void* dbeta, int out_bf16, void* ws, imagd_stream stream) {
    IMAGD_CHECK_ARG(x && dy && dx && ws && fwd_stats && NB > 0 && HW > 0 && C % 8 == 0 && C <= 2560 && groups > 0 && C % groups == 0,
                    "groupnorm_bwd: bad argument");
    float* stat = static_cast<float*>(ws);
    float* pc = stat + static_cast<int64_t>(NB) * groups * 4;
    float* part = pc + static_cast<int64_t>(2) * NB * C;
    const int chunks = gn_bwd_chunks(HW, NB);
    const int rows = kGbThreads / (C / 8);
    const size_t smem1 = static_cast<size_t>(2) * rows * C * 4;  // <= 2 * 512 * 8 * 4 = 32 KB
    groupnorm_bwd_partial_kernel<<<dim3(chunks, NB), kGbThreads, smem1, ST(stream)>>>(BF(x), BF(dy), HW, C, groups, chunks, gamma,
                                                                                      beta, fuse_silu, fwd_stats, part);
    IMAGD_LAUNCH_CHECK("groupnorm_bwd_partial_kernel");
    const int cpg = C / groups;
    IMAGD_CHECK_ARG(cpg <= 128, "groupnorm_bwd: more than 128 channels per group");
    const int gpb = 128 / cpg;  // whole groups per fold CTA
    groupnorm_bwd_fold_kernel<<<dim3((groups + gpb - 1) / gpb, NB), kGbThreads, 0, ST(stream)>>>(part, HW, C, groups, chunks,
                                                                                                gamma, fwd_stats, stat, pc, NB,
                                                                                                gpb);
    IMAGD_LAUNCH_CHECK("groupnorm_bwd_fold_kernel");
    const int64_t total = static_cast<int64_t>(NB) * HW * (C / 8);
    groupnorm_bwd_apply_kernel<<<blocks_for(total, 256), 256, 0, ST(stream)>>>(BF(x), BF(dy), BFW(dx), HW, C, groups, gamma, beta,
                                                                              fuse_silu, stat, total);
    IMAGD_LAUNCH_CHECK("groupnorm_bwd_apply_kernel");
    if (dgamma != nullptr) {
        IMAGD_CHECK_ARG(dbeta, "groupnorm_bwd: dbeta");
        // fold the per-sample partials: pc is [2][NB][C] = the colreduce part layout with splits = NB, groups = 1
        colreduce_fold_kernel<<<blocks_for(C, 256), 256, 0, ST(stream)>>>(pc, dgamma, dbeta, C, 1, NB, out_bf16);
        IMAGD_LAUNCH_CHECK("colreduce_fold_kernel");
    }
    return IMAGD_OK;
}

extern "C" int imagd_act_bf16(const void* x, const void* dy, void* y, int64_t n, int mode, imagd_stream stream) {
    IMAGD_CHECK_ARG(x && y && n > 0 && (mode == IMAGD_ACT_SILU || mode == IMAGD_ACT_GELU), "act: bad argument");
    IMAGD_CHECK_ARG((reinterpret_cast<uintptr_t>(x) & 3) == 0 && (reinterpret_cast<uintptr_t>(y) & 3) == 0, "act: alignment");
    act_kernel<<<blocks_for((n + 1) / 2, 256), 256, 0, ST(stream)>>>(BF(x), BF(dy), BFW(y), n, mode);
    IMAGD_LAUNCH_CHECK("act_kernel");
    return IMAGD_OK;
}

extern "C" int imagd_geglu_bf16(const void* h, int64_t ldh, const void* dout, void* out, int64_t ldo, int64_t M, int F,
                                imagd_stream stream) {
    IMAGD_CHECK_ARG(h && out && M > 0 && F > 0 && F % 2 == 0 && ldh % 2 == 0 && ldo % 2 == 0, "geglu: bad argument");
    geglu_kernel<<<blocks_for(M * (F / 2), 256), 256, 0, ST(stream)>>>(BF(h), ldh, BF(dout), BFW(out), ldo, M, F);
    IMAGD_LAUNCH_CHECK("geglu_kernel");
    return IMAGD_OK;
}

extern "C" int imagd_mse_loss_grad(const float* pred, const float* target, float* grad, float* loss, int64_t n, float grad_scale,
                                   void* ws, imagd_stream stream) {
    IMAGD_CHECK_ARG(pred && target && grad && loss && ws && n > 0, "mse: bad argument");
    const int blocks = static_cast<int>(n / 1024 < 1 ? 1 : (n / 1024 > 296 ? 296 : n / 1024));
    mse_kernel<<<blocks, 256, 0, ST(stream)>>>(pred, target, grad, static_cast<float*>(ws), n, grad_scale * 2.f / static_cast<float>(n));
    IMAGD_LAUNCH_CHECK("mse_kernel");
    mse_fold_kernel<<<1, 32, 0, ST(stream)>>>(static_cast<const float*>(ws), blocks, 1.f / static_cast<float>(n), loss);
    IMAGD_LAUNCH_CHECK("mse_fold_kernel");
    return IMAGD_OK;
}

extern "C" int imagd_adamw_step(float* master, void* param, const void* grad, float* m, float* v, int64_t n, float lr, float beta1,
                                float beta2, float eps, float weight_decay, int step, float grad_scale, imagd_stream stream) {
    IMAGD_CHECK_ARG(master && param && grad && m && v && n > 0 && step >= 1, "adamw: bad argument");
    const float bc1 = 1.f - powf(beta1, static_cast<float>(step)), bc2 = 1.f - powf(beta2, static_cast<float>(step));
    adamw_kernel<<<blocks_for(n, 256), 256, 0, ST(stream)>>>(master, BFW(param), BF(grad), m, v, n, lr, beta1, beta2, eps,
                                                            weight_decay, bc1, bc2, grad_scale);
    IMAGD_LAUNCH_CHECK("adamw_kernel");
    return IMAGD_OK;
}

extern "C" int imagd_adamw_step_dev(float* master, void* param, const void* grad, float* m, float* v, int64_t n, float beta1,
                                    float beta2, float eps, const float* hyper, imagd_stream stream) {
    IMAGD_CHECK_ARG(master && param && grad && m && v && hyper && n > 0, "adamw_dev: bad argument");
    IMAGD_CHECK_ARG(imagd::aligned16(master) && imagd::aligned16(m) && imagd::aligned16(v) &&
                        (reinterpret_cast<uintptr_t>(param) & 7) == 0 && (reinterpret_cast<uintptr_t>(grad) & 7) == 0,
                    "adamw_dev: buffers must be 16-byte (fp32) / 8-byte (bf16) aligned");
    adamw_dev_kernel<false><<<blocks_for((n + 3) / 4, 256), 256, 0, ST(stream)>>>(master, BFW(param), BF(grad), m, v, n, beta1, beta2,
                                                                                 eps, hyper, nullptr);
    IMAGD_LAUNCH_CHECK("adamw_dev_kernel");
    return IMAGD_OK;
}

extern "C" int64_t imagd_grad_norm_ws_bytes(int64_t n) { return 16 + static_cast<int64_t>(8) * grad_norm_blocks(n); }

extern "C" int imagd_grad_norm_clip(const void* grad, int64_t n, float max_norm, float* hyper, double* state, void* ws,
                                    imagd_stream stream) {
    IMAGD_CHECK_ARG(grad && hyper && state && ws && n > 0 && max_norm > 0.f, "grad_norm_clip: bad argument");
    IMAGD_CHECK_ARG(imagd::aligned16(grad) && imagd::aligned16(ws) && (reinterpret_cast<uintptr_t>(state) & 7) == 0,
                    "grad_norm_clip: grad / ws must be 16-byte aligned, state 8-byte aligned");
    grad_norm_clip_kernel<<<grad_norm_blocks(n), kNormThreads, 0, ST(stream)>>>(
        BF(grad), n, max_norm, hyper, state, static_cast<unsigned int*>(ws),
        reinterpret_cast<double*>(static_cast<char*>(ws) + 16));
    IMAGD_LAUNCH_CHECK("grad_norm_clip_kernel");
    return IMAGD_OK;
}

extern "C" int imagd_adamw_step_clip(float* master, void* param, const void* grad, float* m, float* v, int64_t n, float beta1,
                                     float beta2, float eps, const float* hyper, const double* clip_state, imagd_stream stream) {
    IMAGD_CHECK_ARG(master && param && grad && m && v && hyper && clip_state && n > 0, "adamw_clip: bad argument");
    IMAGD_CHECK_ARG(imagd::aligned16(master) && imagd::aligned16(m) && imagd::aligned16(v) &&
                        (reinterpret_cast<uintptr_t>(param) & 7) == 0 && (reinterpret_cast<uintptr_t>(grad) & 7) == 0,
                    "adamw_clip: buffers must be 16-byte (fp32) / 8-byte (bf16) aligned");
    adamw_dev_kernel<true><<<blocks_for((n + 3) / 4, 256), 256, 0, ST(stream)>>>(master, BFW(param), BF(grad), m, v, n, beta1, beta2,
                                                                                eps, hyper, clip_state);
    IMAGD_LAUNCH_CHECK("adamw_dev_kernel<clip>");
    return IMAGD_OK;
}
