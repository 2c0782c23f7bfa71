// HBM-/latency-bound glue kernels of the denoising step: skip concat (+ControlNet residual), nearest-2x upsample,
// stride-2 im2col, thin direct 3x3 convs (conv_in / conv_out / ControlNet conditioning embedding), layout
// conversion at the pipeline boundary, timestep embedding, small-M linears, and the fused CFG + DDIM step.
#include <algorithm>

#include "common.cuh"
#include "ptx.cuh"

namespace imagd {

__device__ __forceinline__ uint4 add_bf16x8(uint4 a, uint4 b) {
    const uint32_t ua[4] = {a.x, a.y, a.z, a.w}, ub[4] = {b.x, b.y, b.z, b.w};
    uint32_t r[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) r[k] = pack_bf16x2(bf16lo(ua[k]) + bf16lo(ub[k]), bf16hi(ua[k]) + bf16hi(ub[k]));
    return make_uint4(r[0], r[1], r[2], r[3]);
}

__global__ void concat_add_kernel(const __nv_bfloat16* __restrict__ a, int64_t lda, int Ca,
                                  const __nv_bfloat16* __restrict__ ra, int64_t ldra,
                                  const __nv_bfloat16* __restrict__ b, int64_t ldb, int Cb,
                                  const __nv_bfloat16* __restrict__ rb, int64_t ldrb, __nv_bfloat16* __restrict__ out,
                                  int64_t ldo, int64_t rows) {
    pdl_launch_dependents();
    pdl_wait();
    const int CV = (Ca + Cb) / 8, CVa = Ca / 8;
    const int64_t total = rows * CV;
    for (int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; idx < total;
         idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int64_t row = idx / CV;
        const int cv = static_cast<int>(idx % CV);
        uint4 v;
        if (cv < CVa) {
            v = __ldg(reinterpret_cast<const uint4*>(a + row * lda + cv * 8));
            if (ra) v = add_bf16x8(v, __ldg(reinterpret_cast<const uint4*>(ra + row * ldra + cv * 8)));
        } else {
            const int c = (cv - CVa) * 8;
            v = __ldg(reinterpret_cast<const uint4*>(b + row * ldb + c));
            if (rb) v = add_bf16x8(v, __ldg(reinterpret_cast<const uint4*>(rb + row * ldrb + c)));
        }
        *reinterpret_cast<uint4*>(out + row * ldo + cv * 8) = v;
    }
}

__global__ void upsample2x_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, int NB, int H,
                                  int W, int C) {
    pdl_launch_dependents();
    pdl_wait();
    const int CV = C / 8;
    const int64_t total = static_cast<int64_t>(NB) * 4 * H * W * CV;
    for (int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; idx < total;
         idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int cv = static_cast<int>(idx % CV);
        int64_t pix = idx / CV;
        const int xo = static_cast<int>(pix % (2 * W));
        pix /= 2 * W;
        const int yo = static_cast<int>(pix % (2 * H));
        const int n = static_cast<int>(pix / (2 * H));
        const int64_t src = ((static_cast<int64_t>(n) * H + yo / 2) * W + xo / 2) * C + cv * 8;
        *reinterpret_cast<uint4*>(y + (idx / CV) * C + cv * 8) = __ldg(reinterpret_cast<const uint4*>(x + src));
    }
}

__global__ void im2col3x3_s2_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ col, int NB, int H,
                                    int W, int C, int pad_lo) {
    pdl_launch_dependents();
    pdl_wait();
    const int Ho = H / 2, Wo = W / 2, CV = C / 8;
    const int64_t total = static_cast<int64_t>(NB) * Ho * Wo * 9 * CV;
    for (int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; idx < total;
         idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int cv = static_cast<int>(idx % CV);
        int64_t t = idx / CV;
        const int tap = static_cast<int>(t % 9);
        t /= 9;
        const int xo = static_cast<int>(t % Wo);
        t /= Wo;
        const int yo = static_cast<int>(t % Ho);
        const int n = static_cast<int>(t / Ho);
        const int yi = 2 * yo + tap / 3 - pad_lo, xi = 2 * xo + tap % 3 - pad_lo;
        uint4 v = make_uint4(0, 0, 0, 0);
        if (yi >= 0 && yi < H && xi >= 0 && xi < W)
            v = __ldg(reinterpret_cast<const uint4*>(x + ((static_cast<int64_t>(n) * H + yi) * W + xi) * C + cv * 8));
        *reinterpret_cast<uint4*>(col + idx * 8) = v;
    }
}

// Row softmax of an fp32 score matrix into bf16 probabilities: P[r, :] = softmax(scale * S[r, :]). One CTA per row, the
// row lives in registers (<= 64 values per thread = 16384 columns), fp32 statistics, fixed-order block reductions. Serves
// the single-head, head-dim-512 attention of the VAE mid block (AutoencoderKL, diffusers-0.24: 4096..6912 tokens at
// 512x512..768x576), whose 512-wide head does not fit the register budget of the flash kernel: S = Q K^T and O = P V run
// as plain GEMMs around this HBM-bound pass (2 x rows x cols x 4 B read, 2 B written per element).
__global__ void __launch_bounds__(256) softmax_rows_kernel(const float* __restrict__ s, int64_t lds,
                                                           __nv_bfloat16* __restrict__ p, int64_t ldp, int cols,
                                                           float scale_log2) {
    pdl_launch_dependents();
    pdl_wait();
    __shared__ float red[8];
    const float* row = s + static_cast<int64_t>(blockIdx.x) * lds;
    __nv_bfloat16* out = p + static_cast<int64_t>(blockIdx.x) * ldp;
    const int nvec = cols / 4;
    float4 v[16];
    float mx = -INFINITY;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
        const int c = threadIdx.x + i * 256;
        v[i] = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
        if (c < nvec) v[i] = __ldg(reinterpret_cast<const float4*>(row) + c);
        mx = fmaxf(mx, fmaxf(fmaxf(v[i].x, v[i].y), fmaxf(v[i].z, v[i].w)));
    }
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
    __syncthreads();
    mx = red[0];
#pragma unroll
    for (int w = 1; w < 8; ++w) mx = fmaxf(mx, red[w]);
    __syncthreads();
    const float m = mx * scale_log2;
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
        v[i].x = ex2_approx(v[i].x * scale_log2 - m);
        v[i].y = ex2_approx(v[i].y * scale_log2 - m);
        v[i].z = ex2_approx(v[i].z * scale_log2 - m);
        v[i].w = ex2_approx(v[i].w * scale_log2 - m);
        sum += (v[i].x + v[i].y) + (v[i].z + v[i].w);  // -inf padding contributes exp2(-inf) = 0
    }
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
    __syncthreads();
    sum = red[0];
#pragma unroll
    for (int w = 1; w < 8; ++w) sum += red[w];
    const float inv = 1.0f / sum;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
        const int c = threadIdx.x + i * 256;
        if (c < nvec)
            *reinterpret_cast<uint2*>(out + c * 4) =
                make_uint2(pack_bf16x2(v[i].x * inv, v[i].y * inv), pack_bf16x2(v[i].z * inv, v[i].w * inv));
    }
}

// ---- CLIP encoder front ends (SURVEY.md 8f row 3): gathers and layout only, the arithmetic is the GEMM / LN / attention
// out[b*T + t, :] = tok[ids[b*T + t], :] + pos[t, :]   (CLIPTextEmbeddings: token + position embedding)
__global__ void embed_tokens_kernel(const int64_t* __restrict__ ids, const __nv_bfloat16* __restrict__ tok,
                                    const __nv_bfloat16* __restrict__ pos, __nv_bfloat16* __restrict__ out, int rows, int T,
                                    int C, int vocab) {
    pdl_launch_dependents();
    pdl_wait();
    const int CV = C / 8;
    for (int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; idx < static_cast<int64_t>(rows) * CV;
         idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int row = static_cast<int>(idx / CV), cv = static_cast<int>(idx % CV);
        int64_t id = ids[row];
        id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
        const uint4 a = __ldg(reinterpret_cast<const uint4*>(tok + id * C + cv * 8));
        const uint4 b = __ldg(reinterpret_cast<const uint4*>(pos + static_cast<int64_t>(row % T) * C + cv * 8));
        const uint32_t ua[4] = {a.x, a.y, a.z, a.w}, ub[4] = {b.x, b.y, b.z, b.w};
        uint32_t o[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) o[k] = pack_bf16x2(bf16lo(ua[k]) + bf16lo(ub[k]), bf16hi(ua[k]) + bf16hi(ub[k]));
        *reinterpret_cast<uint4*>(out + static_cast<int64_t>(row) * C + cv * 8) = make_uint4(o[0], o[1], o[2], o[3]);
    }
}

// Non-overlapping patches of an fp32 NCHW image as GEMM rows (CLIPVisionEmbeddings.patch_embedding = conv with
// kernel = stride = patch): out[(b*Py + py)*Px + px, (c*patch + iy)*patch + ix] = x[b, c, py*patch + iy, px*patch + ix];
// columns [3*patch*patch, Kpad) are zero (K is padded to a multiple of 8 for the tensor-core GEMM).
__global__ void patchify_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ out, int B, int H, int W, int patch,
                                int Kpad) {
    pdl_launch_dependents();
    pdl_wait();
    const int Py = H / patch, Px = W / patch, K = 3 * patch * patch;
    const int64_t total = static_cast<int64_t>(B) * Py * Px * Kpad;
    for (int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; idx < total;
         idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int k = static_cast<int>(idx % Kpad);
        int64_t t = idx / Kpad;
        const int px = static_cast<int>(t % Px);
        t /= Px;
        const int py = static_cast<int>(t % Py);
        const int b = static_cast<int>(t / Py);
        float v = 0.f;
        if (k < K) {
            const int c = k / (patch * patch), iy = (k / patch) % patch, ix = k % patch;
            v = __ldg(x + ((static_cast<int64_t>(b) * 3 + c) * H + py * patch + iy) * W + px * patch + ix);
        }
        out[idx] = __float2bfloat16_rn(v);
    }
}

// out[b * rows_per_sample + row, :] = vec  for every sample b (the ViT class-token row: class_embedding + position[0])
__global__ void broadcast_row_kernel(const __nv_bfloat16* __restrict__ vec, __nv_bfloat16* __restrict__ out, int B,
                                     int64_t rows_per_sample, int row, int C) {
    pdl_launch_dependents();
    pdl_wait();
    for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < B * C; idx += gridDim.x * blockDim.x)
        out[(static_cast<int64_t>(idx / C) * rows_per_sample + row) * C + idx % C] = vec[idx % C];
}

// thread per (output pixel, cout): thin convs where 9*Cin is small or the call happens once per image
__global__ void conv3x3_direct_thread_kernel(const __nv_bfloat16* __restrict__ x, int NB, int H, int W, int Cin,
                                             const __nv_bfloat16* __restrict__ w, const float* __restrict__ bias,
                                             void* __restrict__ y, int Cout, int stride, int act, int out_nchw_f32,
                                             const __nv_bfloat16* __restrict__ add) {
    pdl_launch_dependents();
    pdl_wait();
    const int Ho = (H + stride - 1) / stride, Wo = (W + stride - 1) / stride;
    const int64_t total = static_cast<int64_t>(NB) * Ho * Wo * Cout;
    for (int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; idx < total;
         idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int co = static_cast<int>(idx % Cout);
        int64_t t = idx / Cout;
        const int xo = static_cast<int>(t % Wo);
        t /= Wo;
        const int yo = static_cast<int>(t % Ho);
        const int n = static_cast<int>(t / Ho);
        float acc = bias ? bias[co] : 0.f;
        const __nv_bfloat16* wr = w + static_cast<int64_t>(co) * 9 * Cin;
        for (int tap = 0; tap < 9; ++tap) {
            const int yi = yo * stride + tap / 3 - 1, xi = xo * stride + tap % 3 - 1;
            if (yi < 0 || yi >= H || xi < 0 || xi >= W) continue;
            const __nv_bfloat16* xr = x + ((static_cast<int64_t>(n) * H + yi) * W + xi) * Cin;
            const __nv_bfloat16* wt = wr + tap * Cin;
            for (int c = 0; c < Cin; ++c) acc += __bfloat162float(xr[c]) * __bfloat162float(wt[c]);
        }
        if (act == IMAGD_ACT_SILU) acc = silu(acc);
        const int64_t opix = (static_cast<int64_t>(n) * Ho + yo) * Wo + xo;
        if (add) acc += __bfloat162float(add[opix * Cout + co]);
        if (out_nchw_f32)
            reinterpret_cast<float*>(y)[((static_cast<int64_t>(n) * Cout + co) * Ho + yo) * Wo + xo] = acc;
        else
            reinterpret_cast<__nv_bfloat16*>(y)[opix * Cout + co] = __float2bfloat16(acc);
    }
}

// conv_in (Cin = 4): 8 threads per output pixel, each keeps the 3x3x4 patch in registers and produces Cout/8 channels
// from weights staged in shared memory; stores are 16-byte vectors.
__global__ void __launch_bounds__(256) conv3x3_cin4_kernel(const __nv_bfloat16* __restrict__ x, int NB, int H, int W,
                                                           const __nv_bfloat16* __restrict__ w,
                                                           const float* __restrict__ bias,
                                                           __nv_bfloat16* __restrict__ y, int Cout,
                                                           const __nv_bfloat16* __restrict__ add) {
    pdl_launch_dependents();
    pdl_wait();
    extern __shared__ float s_w[];  // [Cout][37] (row padded: fewer bank conflicts) + [Cout] bias
    for (int i = threadIdx.x; i < Cout * 36; i += blockDim.x) s_w[(i / 36) * 37 + i % 36] = __bfloat162float(w[i]);
    float* s_b = s_w + Cout * 37;
    for (int i = threadIdx.x; i < Cout; i += blockDim.x) s_b[i] = bias ? bias[i] : 0.f;
    __syncthreads();
    const int64_t pix = blockIdx.x * static_cast<int64_t>(blockDim.x / 8) + (threadIdx.x >> 3);
    const int part = threadIdx.x & 7;
    if (pix >= static_cast<int64_t>(NB) * H * W) return;
    const int xo = static_cast<int>(pix % W);
    const int yo = static_cast<int>((pix / W) % H);
    const int n = static_cast<int>(pix / (static_cast<int64_t>(W) * H));
    float patch[36];
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
        const int yi = yo + tap / 3 - 1, xi = xo + tap % 3 - 1;
        uint2 v = make_uint2(0u, 0u);
        if (yi >= 0 && yi < H && xi >= 0 && xi < W)
            v = __ldg(reinterpret_cast<const uint2*>(x + ((static_cast<int64_t>(n) * H + yi) * W + xi) * 4));
        patch[tap * 4 + 0] = bf16lo(v.x);
        patch[tap * 4 + 1] = bf16hi(v.x);
        patch[tap * 4 + 2] = bf16lo(v.y);
        patch[tap * 4 + 3] = bf16hi(v.y);
    }
    const int per = Cout / 8;  // channels per thread (multiple of 8)
    for (int c0 = part * per; c0 < (part + 1) * per; c0 += 8) {
        float acc[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const float* wr = s_w + (c0 + k) * 37;
            float a = s_b[c0 + k];
#pragma unroll
            for (int t = 0; t < 36; ++t) a += patch[t] * wr[t];
            acc[k] = a;
        }
        if (add) {
            const uint4 av = __ldg(reinterpret_cast<const uint4*>(add + pix * Cout + c0));
            acc[0] += bf16lo(av.x); acc[1] += bf16hi(av.x); acc[2] += bf16lo(av.y); acc[3] += bf16hi(av.y);
            acc[4] += bf16lo(av.z); acc[5] += bf16hi(av.z); acc[6] += bf16lo(av.w); acc[7] += bf16hi(av.w);
        }
        *reinterpret_cast<uint4*>(y + pix * Cout + c0) = make_uint4(pack_bf16x2(acc[0], acc[1]), pack_bf16x2(acc[2], acc[3]),
                                                                   pack_bf16x2(acc[4], acc[5]), pack_bf16x2(acc[6], acc[7]));
    }
}

// warp per output pixel, COUT <= 8, Cin % 8 == 0: conv_out (320 -> 4). Lanes split the 9*Cin reduction.
template <int COUT>
__global__ void __launch_bounds__(256) conv3x3_direct_warp_kernel(const __nv_bfloat16* __restrict__ x, int NB, int H,
                                                                  int W, int Cin, const __nv_bfloat16* __restrict__ w,
                                                                  const float* __restrict__ bias, void* __restrict__ y,
                                                                  int act, int out_nchw_f32) {
    pdl_launch_dependents();
    pdl_wait();
    constexpr int Cout = COUT;
    const int64_t pix = blockIdx.x * static_cast<int64_t>(blockDim.x / 32) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (pix >= static_cast<int64_t>(NB) * H * W) return;
    const int xo = static_cast<int>(pix % W);
    const int yo = static_cast<int>((pix / W) % H);
    const int n = static_cast<int>(pix / (static_cast<int64_t>(W) * H));
    float acc[COUT];
#pragma unroll
    for (int k = 0; k < COUT; ++k) acc[k] = 0.f;
    const int CV = Cin / 8;
    for (int tap = 0; tap < 9; ++tap) {
        const int yi = yo + tap / 3 - 1, xi = xo + tap % 3 - 1;
        if (yi < 0 || yi >= H || xi < 0 || xi >= W) continue;
        const __nv_bfloat16* xr = x + ((static_cast<int64_t>(n) * H + yi) * W + xi) * Cin;
        for (int cv = lane; cv < CV; cv += 32) {
            const uint4 xv = __ldg(reinterpret_cast<const uint4*>(xr + cv * 8));
            const uint32_t xu[4] = {xv.x, xv.y, xv.z, xv.w};
#pragma unroll
            for (int co = 0; co < COUT; ++co) {
                const uint4 wv =
                    __ldg(reinterpret_cast<const uint4*>(w + (static_cast<int64_t>(co) * 9 + tap) * Cin + cv * 8));
                const uint32_t wu[4] = {wv.x, wv.y, wv.z, wv.w};
#pragma unroll
                for (int k = 0; k < 4; ++k)
                    acc[co] += bf16lo(xu[k]) * bf16lo(wu[k]) + bf16hi(xu[k]) * bf16hi(wu[k]);
            }
        }
    }
#pragma unroll
    for (int k = 0; k < COUT; ++k)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc[k] += __shfl_xor_sync(0xffffffffu, acc[k], o);
    if (lane < Cout) {
        float v = acc[0];
#pragma unroll
        for (int k = 1; k < COUT; ++k)
            if (lane == k) v = acc[k];
        v += bias ? bias[lane] : 0.f;
        if (act == IMAGD_ACT_SILU) v = silu(v);
        if (out_nchw_f32)
            reinterpret_cast<float*>(y)[((static_cast<int64_t>(n) * Cout + lane) * H + yo) * W + xo] = v;
        else
            reinterpret_cast<__nv_bfloat16*>(y)[pix * Cout + lane] = __float2bfloat16(v);
    }
}

__global__ void nchw_f32_to_nhwc_bf16_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ y, int NB, int C,
                                             int H, int W, int Cpad, int repeat) {
    pdl_launch_dependents();
    pdl_wait();
    const int64_t total = static_cast<int64_t>(NB) * repeat * H * W * Cpad;
    for (int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; idx < total;
         idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int c = static_cast<int>(idx % Cpad);
        const int64_t pix = idx / Cpad;
        const int64_t hw = pix % (static_cast<int64_t>(H) * W);
        const int64_t n = (pix / (static_cast<int64_t>(H) * W)) % NB;
        const float v = c < C ? x[(n * C + c) * H * W + hw] : 0.f;
        y[idx] = __float2bfloat16(v);
    }
}

__global__ void timestep_embedding_kernel(const float* __restrict__ timesteps, const int32_t* __restrict__ step_ptr,
                                          float* __restrict__ out, int NB, int dim) {
    pdl_launch_dependents();
    pdl_wait();
    const int half = dim / 2;
    const float t = timesteps[step_ptr ? *step_ptr : 0];
    for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < NB * dim; idx += gridDim.x * blockDim.x) {
        const int i = idx % dim;
        const int k = i < half ? i : i - half;
        const float freq = expf(-9.210340371976184f * static_cast<float>(k) / static_cast<float>(half));
        const float a = t * freq;
        out[idx] = i < half ? cosf(a) : sinf(a);
    }
}

// warp per output feature; M tiled by 8
__global__ void __launch_bounds__(256) linear_small_m_kernel(const float* __restrict__ x, int64_t ldx,
                                                             const __nv_bfloat16* __restrict__ W, int64_t ldw,
                                                             const float* __restrict__ bias, float* __restrict__ out,
                                                             int64_t ldo, int M, int N, int K, int act_in, int act_out) {
    pdl_launch_dependents();
    pdl_wait();
    const int n = blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (n >= N) return;
    const __nv_bfloat16* wr = W + static_cast<int64_t>(n) * ldw;
    for (int m0 = 0; m0 < M; m0 += 8) {
        float acc[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] = 0.f;
        for (int k0 = lane * 8; k0 < K; k0 += 256) {
            const uint4 wv = __ldg(reinterpret_cast<const uint4*>(wr + k0));
            const uint32_t wu[4] = {wv.x, wv.y, wv.z, wv.w};
            float wf[8];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                wf[2 * k] = bf16lo(wu[k]);
                wf[2 * k + 1] = bf16hi(wu[k]);
            }
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                if (m0 + i < M) {
                    const float* xr = x + static_cast<int64_t>(m0 + i) * ldx + k0;
                    const float4 a = __ldg(reinterpret_cast<const float4*>(xr));
                    const float4 b = __ldg(reinterpret_cast<const float4*>(xr + 4));
                    float xv[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
                    for (int k = 0; k < 8; ++k) {
                        const float xa = act_in == IMAGD_ACT_SILU ? silu(xv[k]) : xv[k];
                        acc[i] += xa * wf[k];
                    }
                }
            }
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], o);
        }
        if (lane == 0) {
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                if (m0 + i < M) {
                    float v = acc[i] + (bias ? bias[n] : 0.f);
                    if (act_out == IMAGD_ACT_SILU) v = silu(v);
                    else if (act_out == IMAGD_ACT_GELU) v = gelu_erf(v);
                    out[static_cast<int64_t>(m0 + i) * ldo + n] = v;
                }
            }
        }
    }
}

__global__ void cfg_ddim_step_kernel(const float* __restrict__ eps_c, const float* __restrict__ eps_u, float g,
                                     float* __restrict__ lat, const float* __restrict__ coef,
                                     int32_t* __restrict__ step_ptr, const float* __restrict__ mask,
                                     const float* __restrict__ img, const float* __restrict__ noise,
                                     const float* __restrict__ blend_coef, int NB, int C, int HW) {
    pdl_launch_dependents();
    pdl_wait();
    unsigned int* done_counter = reinterpret_cast<unsigned int*>(step_ptr + 1);
    const int step = *step_ptr;
    const float sa_t = coef[step * 4 + 0], sb_t = coef[step * 4 + 1], sa_p = coef[step * 4 + 2],
                sb_p = coef[step * 4 + 3];
    float bn_a = 1.f, bn_b = 0.f;
    if (mask) {
        bn_a = blend_coef[step * 2 + 0];
        bn_b = blend_coef[step * 2 + 1];
    }
    const int64_t total = static_cast<int64_t>(NB) * C * HW;
    for (int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; idx < total;
         idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const float u = eps_u ? eps_u[idx] : 0.f;
        const float c = eps_c[idx];
        const float eps = eps_u ? u + g * (c - u) : c;
        const float xt = lat[idx];
        const float x0 = (xt - sb_t * eps) / sa_t;
        float xn = sa_p * x0 + sb_p * eps;
        if (mask) {
            const int64_t n = idx / (static_cast<int64_t>(C) * HW);
            const float m = mask[n * HW + idx % HW];
            const float proper = bn_a * img[idx] + bn_b * noise[idx];
            xn = (1.f - m) * proper + m * xn;
        }
        lat[idx] = xn;
    }
    // the last block to finish advances the device-side step counter (graph replays then see the next step)
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned int prev = atomicAdd(done_counter, 1u);
        if (prev == gridDim.x - 1) {
            *done_counter = 0u;
            *step_ptr = step + 1;
        }
    }
}

static inline int grid_for(int64_t total, int threads) {
    int64_t g = (total + threads - 1) / threads;
    if (g > kNumSms * 16) g = kNumSms * 16;
    if (g < 1) g = 1;
    return static_cast<int>(g);
}

}  // namespace imagd

extern "C" {

int imagd_concat_add_bf16(const void* a, int64_t lda, int Ca, const void* res_a, int64_t ld_ra, const void* b,
                          int64_t ldb, int Cb, const void* res_b, int64_t ld_rb, void* out, int64_t ldo, int64_t rows,
                          imagd_stream stream) {
    using namespace imagd;
    IMAGD_CHECK_ARG(a && out && rows > 0, "concat_add: null pointer / rows");
    if (!b) Cb = 0;
    IMAGD_CHECK_ARG(Ca % 8 == 0 && Cb % 8 == 0 && lda % 8 == 0 && ldo % 8 == 0 && (Cb == 0 || ldb % 8 == 0),
                    "concat_add: channel counts / strides must be multiples of 8");
    IMAGD_CHECK_ARG((!res_a || ld_ra % 8 == 0) && (!res_b || ld_rb % 8 == 0), "concat_add: residual stride");
    const int64_t total = rows * ((Ca + Cb) / 8);
    IMAGD_CUDA(launch_pdl(concat_add_kernel, dim3(grid_for(total, 256)), dim3(256), 0, static_cast<cudaStream_t>(stream), 
        reinterpret_cast<const __nv_bfloat16*>(a), lda, Ca, reinterpret_cast<const __nv_bfloat16*>(res_a), ld_ra,
        reinterpret_cast<const __nv_bfloat16*>(b), ldb, Cb, reinterpret_cast<const __nv_bfloat16*>(res_b), ld_rb,
        reinterpret_cast<__nv_bfloat16*>(out), ldo, rows));
    return IMAGD_OK;
}

int imagd_upsample2x_bf16(const void* x, void* y, int NB, int H, int W, int C, imagd_stream stream) {
    using namespace imagd;
    IMAGD_CHECK_ARG(x && y && NB > 0 && H > 0 && W > 0 && C % 8 == 0, "upsample2x: bad args");
    const int64_t total = static_cast<int64_t>(NB) * 4 * H * W * (C / 8);
    IMAGD_CUDA(launch_pdl(upsample2x_kernel, dim3(grid_for(total, 256)), dim3(256), 0, static_cast<cudaStream_t>(stream), 
        reinterpret_cast<const __nv_bfloat16*>(x), reinterpret_cast<__nv_bfloat16*>(y), NB, H, W, C));
    return IMAGD_OK;
}

static int im2col_s2(const void* x, void* col, int NB, int H, int W, int C, int pad_lo, imagd_stream stream) {
    using namespace imagd;
    IMAGD_CHECK_ARG(x && col && NB > 0 && H % 2 == 0 && W % 2 == 0 && C % 8 == 0, "im2col_s2: bad args");
    IMAGD_CHECK_ARG(pad_lo == 0 || pad_lo == 1, "im2col_s2: pad_lo %d", pad_lo);
    const int64_t total = static_cast<int64_t>(NB) * (H / 2) * (W / 2) * 9 * (C / 8);
    IMAGD_CUDA(launch_pdl(im2col3x3_s2_kernel, dim3(grid_for(total, 256)), dim3(256), 0, static_cast<cudaStream_t>(stream), 
        reinterpret_cast<const __nv_bfloat16*>(x), reinterpret_cast<__nv_bfloat16*>(col), NB, H, W, C, pad_lo));
    return IMAGD_OK;
}

int imagd_im2col3x3_s2_bf16(const void* x, void* col, int NB, int H, int W, int C, imagd_stream stream) {
    return im2col_s2(x, col, NB, H, W, C, 1, stream);
}

int imagd_im2col3x3_s2_pad_bf16(const void* x, void* col, int NB, int H, int W, int C, int pad_lo, imagd_stream stream) {
    return im2col_s2(x, col, NB, H, W, C, pad_lo, stream);
}

int imagd_embed_tokens_bf16(const int64_t* ids, const void* tok, const void* pos, void* out, int rows, int T, int C, int vocab,
                            imagd_stream stream) {
    using namespace imagd;
    IMAGD_CHECK_ARG(ids && tok && pos && out && rows > 0 && T > 0 && C % 8 == 0 && vocab > 0, "embed_tokens: bad args");
    IMAGD_CUDA(launch_pdl(embed_tokens_kernel, dim3(grid_for(static_cast<int64_t>(rows) * (C / 8), 256)), dim3(256), 0,
                          static_cast<cudaStream_t>(stream), ids, reinterpret_cast<const __nv_bfloat16*>(tok),
                          reinterpret_cast<const __nv_bfloat16*>(pos), reinterpret_cast<__nv_bfloat16*>(out), rows, T, C, vocab));
    return IMAGD_OK;
}

int imagd_patchify_bf16(const float* x, void* out, int B, int H, int W, int patch, int Kpad, imagd_stream stream) {
    using namespace imagd;
    IMAGD_CHECK_ARG(x && out && B > 0 && patch > 0 && H % patch == 0 && W % patch == 0 && Kpad >= 3 * patch * patch &&
                        Kpad % 8 == 0, "patchify: bad args");
    const int64_t total = static_cast<int64_t>(B) * (H / patch) * (W / patch) * Kpad;
    IMAGD_CUDA(launch_pdl(patchify_kernel, dim3(grid_for(total, 256)), dim3(256), 0, static_cast<cudaStream_t>(stream), x,
                          reinterpret_cast<__nv_bfloat16*>(out), B, H, W, patch, Kpad));
    return IMAGD_OK;
}

int imagd_broadcast_row_bf16(const void* vec, void* out, int B, int64_t rows_per_sample, int row, int C, imagd_stream stream) {
    using namespace imagd;
    IMAGD_CHECK_ARG(vec && out && B > 0 && C > 0 && row >= 0 && row < rows_per_sample, "broadcast_row: bad args");
    IMAGD_CUDA(launch_pdl(broadcast_row_kernel, dim3(grid_for(static_cast<int64_t>(B) * C, 256)), dim3(256), 0,
                          static_cast<cudaStream_t>(stream), reinterpret_cast<const __nv_bfloat16*>(vec),
                          reinterpret_cast<__nv_bfloat16*>(out), B, rows_per_sample, row, C));
    return IMAGD_OK;
}

int imagd_softmax_rows(const float* s, int64_t lds, void* p, int64_t ldp, int64_t rows, int cols, float scale,
                       imagd_stream stream) {
    using namespace imagd;
    IMAGD_CHECK_ARG(s && p && rows > 0 && cols > 0 && cols <= 256 * 64, "softmax_rows: rows=%lld cols=%d unsupported",
                    (long long)rows, cols);
    IMAGD_CHECK_ARG(cols % 4 == 0 && lds % 4 == 0 && ldp % 4 == 0 && aligned16(s) && (reinterpret_cast<uintptr_t>(p) & 7u) == 0,
                    "softmax_rows: alignment");
    IMAGD_CHECK_ARG(rows < (1ll << 31), "softmax_rows: too many rows");
    IMAGD_CUDA(launch_pdl(softmax_rows_kernel, dim3(static_cast<unsigned>(rows)), dim3(256), 0, static_cast<cudaStream_t>(stream),
                          s, lds, reinterpret_cast<__nv_bfloat16*>(p), ldp, cols, scale * 1.4426950408889634f));
    return IMAGD_OK;
}

int imagd_conv3x3_direct_bf16(const void* x, int NB, int H, int W, int Cin, const void* w, const float* bias, void* y,
                              int Cout, int stride, int act, int out_nchw_f32, const void* add_nhwc,
                              imagd_stream stream) {
    using namespace imagd;
    IMAGD_CHECK_ARG(x && w && y && NB > 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0, "conv3x3_direct: bad args");
    IMAGD_CHECK_ARG(stride == 1 || stride == 2, "conv3x3_direct: stride %d", stride);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (Cout == 4 && Cin % 8 == 0 && Cin >= 64 && stride == 1 && !add_nhwc) {
        const int64_t pixels = static_cast<int64_t>(NB) * H * W;
        IMAGD_CUDA(launch_pdl(conv3x3_direct_warp_kernel<4>, dim3(static_cast<int>((pixels + 7) / 8)), dim3(256), 0, st, 
            reinterpret_cast<const __nv_bfloat16*>(x), NB, H, W, Cin, reinterpret_cast<const __nv_bfloat16*>(w), bias, y,
            act, out_nchw_f32));
        return IMAGD_OK;
    }
    if (Cin == 4 && Cout % 64 == 0 && Cout <= 640 && stride == 1 && act == IMAGD_ACT_NONE && !out_nchw_f32) {
        const int64_t pixels = static_cast<int64_t>(NB) * H * W;
        const size_t smem = static_cast<size_t>(Cout) * 38 * sizeof(float);
        IMAGD_SET_MAX_SMEM(conv3x3_cin4_kernel, 640 * 38 * 4);
        IMAGD_CUDA(launch_pdl(conv3x3_cin4_kernel, dim3(static_cast<int>((pixels + 31) / 32)), dim3(256), smem, st, 
            reinterpret_cast<const __nv_bfloat16*>(x), NB, H, W, reinterpret_cast<const __nv_bfloat16*>(w), bias,
            reinterpret_cast<__nv_bfloat16*>(y), Cout, reinterpret_cast<const __nv_bfloat16*>(add_nhwc)));
        return IMAGD_OK;
    }
    const int Ho = (H + stride - 1) / stride, Wo = (W + stride - 1) / stride;
    const int64_t total = static_cast<int64_t>(NB) * Ho * Wo * Cout;
    const int tgrid = std::min(grid_for(total, 256) * 4, kNumSms * 64);
    IMAGD_CUDA(launch_pdl(conv3x3_direct_thread_kernel, dim3(tgrid), dim3(256), 0, st, reinterpret_cast<const __nv_bfloat16*>(x), NB, H, W, Cin,
                                         reinterpret_cast<const __nv_bfloat16*>(w), bias, y, Cout, stride, act,
                                         out_nchw_f32, reinterpret_cast<const __nv_bfloat16*>(add_nhwc)));
    return IMAGD_OK;
}

int imagd_nchw_f32_to_nhwc_bf16(const float* x, void* y, int NB, int C, int H, int W, int Cpad, int repeat,
                                imagd_stream stream) {
    using namespace imagd;
    IMAGD_CHECK_ARG(x && y && NB > 0 && C > 0 && Cpad >= C && repeat >= 1, "nchw_to_nhwc: bad args");
    const int64_t total = static_cast<int64_t>(NB) * repeat * H * W * Cpad;
    IMAGD_CUDA(launch_pdl(nchw_f32_to_nhwc_bf16_kernel, dim3(grid_for(total, 256)), dim3(256), 0, static_cast<cudaStream_t>(stream), 
        x, reinterpret_cast<__nv_bfloat16*>(y), NB, C, H, W, Cpad, repeat));
    return IMAGD_OK;
}

int imagd_timestep_embedding(const float* timesteps, const int32_t* step_ptr, float* out, int NB, int dim,
                             imagd_stream stream) {
    using namespace imagd;
    IMAGD_CHECK_ARG(timesteps && out && NB > 0 && dim > 0 && dim % 2 == 0, "timestep_embedding: bad args");
    IMAGD_CUDA(launch_pdl(timestep_embedding_kernel, dim3(grid_for(static_cast<int64_t>(NB) * dim, 256)), dim3(256), 0, static_cast<cudaStream_t>(stream), timesteps, step_ptr, out, NB, dim));
    return IMAGD_OK;
}

int imagd_linear_small_m(const float* x, int64_t ldx, const void* W, int64_t ldw, const float* bias, float* out,
                         int64_t ldo, int M, int N, int K, int act_in, int act_out, imagd_stream stream) {
    using namespace imagd;
    IMAGD_CHECK_ARG(x && W && out && M > 0 && N > 0 && K > 0, "linear_small_m: bad args");
    IMAGD_CHECK_ARG(K % 8 == 0 && ldx % 4 == 0 && ldw % 8 == 0 && aligned16(x) && aligned16(W),
                    "linear_small_m: K / stride alignment");
    IMAGD_CUDA(launch_pdl(linear_small_m_kernel, dim3((N + 7) / 8), dim3(256), 0, static_cast<cudaStream_t>(stream), 
        x, ldx, reinterpret_cast<const __nv_bfloat16*>(W), ldw, bias, out, ldo, M, N, K, act_in, act_out));
    return IMAGD_OK;
}

int imagd_cfg_ddim_step(const float* eps_cond, const float* eps_uncond, float guidance, float* latents,
                        const float* coef, int32_t* step_ptr, const float* mask, const float* image_latents,
                        const float* noise, const float* blend_coef, int NB, int C, int HW, imagd_stream stream) {
    using namespace imagd;
    IMAGD_CHECK_ARG(eps_cond && latents && coef && step_ptr && NB > 0 && C > 0 && HW > 0, "cfg_ddim_step: bad args");
    IMAGD_CHECK_ARG(!mask || (image_latents && noise && blend_coef), "cfg_ddim_step: inpaint blend needs all operands");
    const int64_t total = static_cast<int64_t>(NB) * C * HW;
    int grid = grid_for(total, 256);
    if (grid > kNumSms) grid = kNumSms;
    IMAGD_CUDA(launch_pdl(cfg_ddim_step_kernel, dim3(grid), dim3(256), 0, static_cast<cudaStream_t>(stream), 
        eps_cond, eps_uncond, guidance, latents, coef, step_ptr, mask, image_latents, noise, blend_coef, NB, C, HW));
    return IMAGD_OK;
}

}  // extern "C"
