// Backward of the two-stream ("hybrid") attention for sm_90a — the training step of SURVEY.md section 8 row
// a13 (reference train.py:255-281,573-605: loss -> frozen denoising UNet -> to_k_ref / to_v_ref and the garment taps ->
// garment UNet; the reference gets this from torch autograd over F.scaled_dot_product_attention,
// adapter/attention_processor.py:589-612).
//
//   O = w0 softmax(Q K0^T s) V0 + w1 softmax(Q K1^T s) V1          (forward, attention_tc.cu)
//   per stream:  P = exp2(S s log2e - lse2),  dP = w dO V^T,  D = rowsum(P o dP) = w rowsum(dO o O_s),
//                dS = P o (dP - D),  dQ += s dS K,  dK = s dS^T Q,  dV = w P^T dO
//
// Recompute-S flash style, two kernels, no atomics, deterministic (attn_bwd_dq_kernel: dQ over both streams;
// attn_bwd_dkv_kernel: dK / dV of one stream), on mma.sync m16n8k16 tensor-core tiles fed from padded shared memory.
// lse2 / D rows arrive as fp32 vectors [2 streams][B][heads][lq_pad]; lse2 of padding rows is +inf (P = 0).
#include <cstdlib>

#include "common.cuh"
#include "ptx.cuh"
#include "attention_common.cuh"

namespace imagd {

struct AttnBwdParams {
    int B, Lq, heads, hd;
    float scale_log2;  // sm_scale * log2(e)
    float sm_scale;
    const __nv_bfloat16* q;
    int64_t q_ld;
    const __nv_bfloat16* d_out;
    int64_t do_ld;
    AttnKV kv[2];    // kv[1].len = 0: one stream
    float w0, w1;    // out_scale of the streams
    int lq_pad;
    const float* lse;   // [2][B][heads][lq_pad]
    const float* dsum;  // [2][B][heads][lq_pad]   D = w * rowsum(dO o O_s)
    // dq kernel
    void* dq;
    int64_t dq_ld;
    // dkv kernel (one stream per launch)
    int stream;  // 0 / 1
    void* dk;
    void* dv;
    int64_t dkv_ld;
    int kv_sample_rows;  // rows between samples in dk / dv
};

// ------------------------------------------------------------------------------------------------ dQ kernel
// CTA = 128 queries of one (sample, head), 8 warps of 16 rows; K / V blocks of 64 keys of both streams stream through
// a two-stage ring. Per block: S = Q K^T and dP = dO V^T (mma.sync), P = exp2(S s log2e - lse2), dS = P o (w dP - D),
// dQ += dS K with dS kept in registers as the A fragment.
template <int HDP>
struct BwdDqSmem {
    static constexpr int kQBytes = 128 * attn_row_bytes(HDP);
    static constexpr int kKVBytes = 64 * attn_row_bytes(HDP);
    static constexpr int kDoOff = kQBytes;
    static constexpr int kKOff = 2 * kQBytes;
    static constexpr int kVOff = kKOff + 2 * kKVBytes;
    static constexpr int kTotal = kVOff + 2 * kKVBytes;
};

// 16 x 64 product of a 16-row A tile (rows arow.. of sA) and 64 B rows (brow.. of sB), K = HDP, both row-major in smem
template <int HDP>
__device__ __forceinline__ void bwd_mma_abt(float (&c)[8][4], uint32_t sA, int arow, uint32_t sB, int lane) {
    constexpr int kRow = attn_row_bytes(HDP);
#pragma unroll
    for (int n = 0; n < 8; ++n) c[n][0] = c[n][1] = c[n][2] = c[n][3] = 0.f;
#pragma unroll
    for (int ks = 0; ks < HDP / 16; ++ks) {
        uint32_t a[4];
        ldmatrix_x4(a, sA + (arow + (lane & 15)) * kRow + (ks * 16 + (lane >> 4) * 8) * 2);
#pragma unroll
        for (int np = 0; np < 4; ++np) {
            uint32_t bb[4];
            ldmatrix_x4(bb, sB + (np * 16 + (lane & 7) + (lane >> 4) * 8) * kRow + (ks * 16 + ((lane >> 3) & 1) * 8) * 2);
            mma_bf16_16816(c[2 * np], a, bb[0], bb[1]);
            mma_bf16_16816(c[2 * np + 1], a, bb[2], bb[3]);
        }
    }
}

// acc[16 x HDP] += A[16 x 64] (bf16 fragments a[kk], kk = 16-column step) * B[64 x HDP] (rows of sB, row-major in smem)
template <int HDP>
__device__ __forceinline__ void bwd_mma_ab(float (&acc)[HDP / 8][4], const uint32_t (&a)[4][4], uint32_t sB, int lane) {
    constexpr int kRow = attn_row_bytes(HDP);
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
        for (int np = 0; np < HDP / 16; ++np) {
            uint32_t bb[4];
            ldmatrix_x4_trans(bb, sB + (kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * kRow + (np * 16 + (lane >> 4) * 8) * 2);
            mma_bf16_16816(acc[2 * np], a[kk], bb[0], bb[1]);
            mma_bf16_16816(acc[2 * np + 1], a[kk], bb[2], bb[3]);
        }
    }
}

// C fragments of a 16 x 64 tile -> bf16 A fragments of the same tile
__device__ __forceinline__ void bwd_pack_a(const float (&c)[8][4], uint32_t (&a)[4][4]) {
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
        a[kk][0] = pack_bf16x2(c[2 * kk][0], c[2 * kk][1]);
        a[kk][1] = pack_bf16x2(c[2 * kk][2], c[2 * kk][3]);
        a[kk][2] = pack_bf16x2(c[2 * kk + 1][0], c[2 * kk + 1][1]);
        a[kk][3] = pack_bf16x2(c[2 * kk + 1][2], c[2 * kk + 1][3]);
    }
}

template <int HDP>
__global__ void __launch_bounds__(256, 1) attn_bwd_dq_kernel(const AttnBwdParams p) {
    using C = BwdDqSmem<HDP>;
    constexpr int NT = HDP / 8;
    extern __shared__ __align__(128) uint8_t smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int g = lane >> 2, t = lane & 3;
    const int q0 = blockIdx.x * 128, h = blockIdx.y, b = blockIdx.z;
    const uint32_t sQ = smem_u32(smem), sDo = sQ + C::kDoOff, sK = sQ + C::kKOff, sV = sQ + C::kVOff;
    const int nb0 = (p.kv[0].len + 63) / 64;
    const int nb1 = p.kv[1].len > 0 ? (p.kv[1].len + 63) / 64 : 0;
    const int T = nb0 + nb1;

    attn_load_rows<HDP>(sQ, p.q + static_cast<int64_t>(b) * p.Lq * p.q_ld + h * p.hd, p.q_ld, p.hd, q0, p.Lq, 128);
    attn_load_rows<HDP>(sDo, p.d_out + static_cast<int64_t>(b) * p.Lq * p.do_ld + h * p.hd, p.do_ld, p.hd, q0, p.Lq, 128);
    auto load_kv = [&](int i) {
        const int s = i < nb0 ? 0 : 1;
        const int j = s ? i - nb0 : i;
        const AttnKV& kv = p.kv[s];
        const int64_t base = static_cast<int64_t>(b) * kv.sample_rows * kv.ld + h * p.hd;
        attn_load_rows<HDP>(sK + (i & 1) * C::kKVBytes, kv.k + base, kv.ld, p.hd, j * 64, kv.len, 64);
        attn_load_rows<HDP>(sV + (i & 1) * C::kKVBytes, kv.v + base, kv.ld, p.hd, j * 64, kv.len, 64);
    };
    load_kv(0);
    cp_async_commit();

    const int row0 = q0 + warp * 16 + g;
    float dq[NT][4];
#pragma unroll
    for (int n = 0; n < NT; ++n) dq[n][0] = dq[n][1] = dq[n][2] = dq[n][3] = 0.f;
    for (int i = 0; i < T; ++i) {
        const int s = i < nb0 ? 0 : 1;
        const int j = s ? i - nb0 : i;
        const float w = s ? p.w1 : p.w0;
        float lse[2], dd[2];
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
            const int q = row0 + hr * 8;
            const int64_t idx = ((static_cast<int64_t>(s) * p.B + b) * p.heads + h) * p.lq_pad + q;
            lse[hr] = q < p.Lq ? __ldg(p.lse + idx) : INFINITY;
            dd[hr] = q < p.Lq ? __ldg(p.dsum + idx) : 0.f;
        }
        cp_async_wait<0>();
        __syncthreads();
        if (i + 1 < T) load_kv(i + 1);
        cp_async_commit();
        const uint32_t kb = sK + (i & 1) * C::kKVBytes, vb = sV + (i & 1) * C::kKVBytes;
        float sc[8][4], dp[8][4];
        bwd_mma_abt<HDP>(sc, sQ, warp * 16, kb, lane);
        bwd_mma_abt<HDP>(dp, sDo, warp * 16, vb, lane);
        const int len = p.kv[s].len;
#pragma unroll
        for (int n = 0; n < 8; ++n) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int key = j * 64 + n * 8 + 2 * t + (e & 1);
                const float pr = key < len ? ex2_approx(sc[n][e] * p.scale_log2 - lse[e >> 1]) : 0.f;
                sc[n][e] = pr * (w * dp[n][e] - dd[e >> 1]);
            }
        }
        uint32_t a[4][4];
        bwd_pack_a(sc, a);
        bwd_mma_ab<HDP>(dq, a, kb, lane);
    }
    attn_store_frag<NT>(dq, p.sm_scale, p.sm_scale, reinterpret_cast<__nv_bfloat16*>(p.dq), p.dq_ld,
                        static_cast<int64_t>(b) * p.Lq, p.Lq, h, p.hd, row0, t);
}

// ------------------------------------------------------------------------------------------------ dK / dV kernel
// CTA = 128 keys of one (sample, head) of ONE stream, 8 warps of 16 keys; Q / dO blocks of 64 queries stream through a
// two-stage ring. The products are taken transposed (row = key): S^T = K Q^T, dP^T = V dO^T, P^T = exp2(S^T s log2e -
// lse2[q]), dS^T = P^T o (w dP^T - D[q]), then dV += P^T dO and dK += dS^T Q with P^T / dS^T as register A fragments.
template <int HDP>
struct BwdDkvSmem {
    static constexpr int kKBytes = 128 * attn_row_bytes(HDP);
    static constexpr int kQBytes = 64 * attn_row_bytes(HDP);
    static constexpr int kVOff = kKBytes;
    static constexpr int kQOff = 2 * kKBytes;
    static constexpr int kDoOff = kQOff + 2 * kQBytes;
    static constexpr int kVecOff = kDoOff + 2 * kQBytes;  // [2 stages][lse2 | D][64] fp32
    static constexpr int kTotal = kVecOff + 2 * 2 * 64 * 4;
};

template <int HDP>
__global__ void __launch_bounds__(256, 1) attn_bwd_dkv_kernel(const AttnBwdParams p) {
    using C = BwdDkvSmem<HDP>;
    constexpr int NT = HDP / 8;
    extern __shared__ __align__(128) uint8_t smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int g = lane >> 2, t = lane & 3;
    const int k0 = blockIdx.x * 128, h = blockIdx.y, b = blockIdx.z;
    const uint32_t sK = smem_u32(smem), sV = sK + C::kVOff, sQ = sK + C::kQOff, sDo = sK + C::kDoOff;
    float* s_vec = reinterpret_cast<float*>(smem + C::kVecOff);
    const AttnKV& kv = p.kv[p.stream];
    const float w = p.stream ? p.w1 : p.w0;
    const int T = (p.Lq + 63) / 64;

    const int64_t kbase = static_cast<int64_t>(b) * kv.sample_rows * kv.ld + h * p.hd;
    attn_load_rows<HDP>(sK, kv.k + kbase, kv.ld, p.hd, k0, kv.len, 128);
    attn_load_rows<HDP>(sV, kv.v + kbase, kv.ld, p.hd, k0, kv.len, 128);
    const int64_t vec_base = ((static_cast<int64_t>(p.stream) * p.B + b) * p.heads + h) * p.lq_pad;
    auto load_q = [&](int i) {
        attn_load_rows<HDP>(sQ + (i & 1) * C::kQBytes, p.q + static_cast<int64_t>(b) * p.Lq * p.q_ld + h * p.hd, p.q_ld,
                            p.hd, i * 64, p.Lq, 64);
        attn_load_rows<HDP>(sDo + (i & 1) * C::kQBytes, p.d_out + static_cast<int64_t>(b) * p.Lq * p.do_ld + h * p.hd,
                            p.do_ld, p.hd, i * 64, p.Lq, 64);
        if (threadIdx.x < 128) {
            const int qq = i * 64 + (threadIdx.x & 63);
            const bool ok = qq < p.Lq;
            float* dst = s_vec + (i & 1) * 128 + threadIdx.x;
            if (threadIdx.x < 64) *dst = ok ? __ldg(p.lse + vec_base + qq) : INFINITY;
            else *dst = ok ? __ldg(p.dsum + vec_base + qq) : 0.f;
        }
    };
    load_q(0);
    cp_async_commit();

    float dk[NT][4], dv[NT][4];
#pragma unroll
    for (int n = 0; n < NT; ++n) {
        dk[n][0] = dk[n][1] = dk[n][2] = dk[n][3] = 0.f;
        dv[n][0] = dv[n][1] = dv[n][2] = dv[n][3] = 0.f;
    }
    for (int i = 0; i < T; ++i) {
        cp_async_wait<0>();
        __syncthreads();
        if (i + 1 < T) load_q(i + 1);
        cp_async_commit();
        const uint32_t qb = sQ + (i & 1) * C::kQBytes, dob = sDo + (i & 1) * C::kQBytes;
        const float* lse = s_vec + (i & 1) * 128;
        const float* dd = lse + 64;
        float sc[8][4], dp[8][4];
        bwd_mma_abt<HDP>(sc, sK, warp * 16, qb, lane);
        bwd_mma_abt<HDP>(dp, sV, warp * 16, dob, lane);
        uint32_t a[4][4];
#pragma unroll
        for (int n = 0; n < 8; ++n) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int qc = n * 8 + 2 * t + (e & 1);  // query column within the block
                const float pr = ex2_approx(sc[n][e] * p.scale_log2 - lse[qc]);
                sc[n][e] = pr;
                dp[n][e] = pr * (w * dp[n][e] - dd[qc]);
            }
        }
        bwd_pack_a(sc, a);
        bwd_mma_ab<HDP>(dv, a, dob, lane);
        bwd_pack_a(dp, a);
        bwd_mma_ab<HDP>(dk, a, qb, lane);
    }
    const int key0 = k0 + warp * 16 + g;
    const int64_t rb = static_cast<int64_t>(b) * p.kv_sample_rows;
    attn_store_frag<NT>(dv, w, w, reinterpret_cast<__nv_bfloat16*>(p.dv), p.dkv_ld, rb, kv.len, h, p.hd, key0, t);
    attn_store_frag<NT>(dk, p.sm_scale, p.sm_scale, reinterpret_cast<__nv_bfloat16*>(p.dk), p.dkv_ld, rb, kv.len, h, p.hd,
                        key0, t);
}

// ------------------------------------------------------------------------------------------------ D = w * rowsum(dO o O_s)
// One warp per (row, head); padding rows of dsum are left as the caller initialised them (0).
__global__ void attn_bwd_prep_kernel(const __nv_bfloat16* __restrict__ d_out, int64_t do_ld,
                                     const __nv_bfloat16* __restrict__ o0, const __nv_bfloat16* __restrict__ o1, int64_t ld_s,
                                     float w0, float w1, float* __restrict__ dsum, int B, int Lq, int heads, int hd,
                                     int lq_pad) {
    const int64_t gw = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    const int64_t total = static_cast<int64_t>(B) * Lq * heads;
    if (gw >= total) return;
    const int h = static_cast<int>(gw % heads);
    const int64_t row = gw / heads;
    const int b = static_cast<int>(row / Lq), q = static_cast<int>(row % Lq);
    const __nv_bfloat16* g = d_out + row * do_ld + h * hd;
    const __nv_bfloat16* a0 = o0 + row * ld_s + h * hd;
    const __nv_bfloat16* a1 = o1 ? o1 + row * ld_s + h * hd : nullptr;
    float s0 = 0.f, s1 = 0.f;
    for (int d = lane; d < hd; d += 32) {
        const float gv = __bfloat162float(g[d]);
        s0 += gv * __bfloat162float(a0[d]);
        if (a1) s1 += gv * __bfloat162float(a1[d]);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        s0 += __shfl_xor_sync(0xffffffffu, s0, o);
        s1 += __shfl_xor_sync(0xffffffffu, s1, o);
    }
    if (lane == 0) {
        const int64_t idx = (static_cast<int64_t>(b) * heads + h) * lq_pad + q;
        dsum[idx] = w0 * s0;
        if (a1) dsum[static_cast<int64_t>(B) * heads * lq_pad + idx] = w1 * s1;
    }
}

// ------------------------------------------------------------------------------------------------ host side
template <int HDP>
static int launch_dq(const AttnBwdParams& p, cudaStream_t stream) {
    using C = BwdDqSmem<HDP>;
    IMAGD_SET_MAX_SMEM(attn_bwd_dq_kernel<HDP>, C::kTotal);
    dim3 grid((p.Lq + 127) / 128, p.heads, p.B);
    attn_bwd_dq_kernel<HDP><<<grid, 256, C::kTotal, stream>>>(p);
    IMAGD_LAUNCH_CHECK("attn_bwd_dq_kernel");
    return IMAGD_OK;
}

template <int HDP>
static int launch_dkv(const AttnBwdParams& p, int len, cudaStream_t stream) {
    using C = BwdDkvSmem<HDP>;
    IMAGD_SET_MAX_SMEM(attn_bwd_dkv_kernel<HDP>, C::kTotal);
    dim3 grid((len + 127) / 128, p.heads, p.B);
    attn_bwd_dkv_kernel<HDP><<<grid, 256, C::kTotal, stream>>>(p);
    IMAGD_LAUNCH_CHECK("attn_bwd_dkv_kernel");
    return IMAGD_OK;
}

template <int HDP>
static int launch_bwd(AttnBwdParams p, void* dk0, void* dv0, int64_t dkv0_ld, void* dk1, void* dv1, int64_t dkv1_ld,
                      cudaStream_t stream) {
    if (p.dq != nullptr) {
        const int rc = launch_dq<HDP>(p, stream);
        if (rc != IMAGD_OK) return rc;
    }
    for (int s = 0; s < 2; ++s) {
        void* dk = s ? dk1 : dk0;
        if (dk == nullptr) continue;
        p.stream = s;
        p.dk = dk;
        p.dv = s ? dv1 : dv0;
        p.dkv_ld = s ? dkv1_ld : dkv0_ld;
        p.kv_sample_rows = p.kv[s].sample_rows;
        const int rc = launch_dkv<HDP>(p, p.kv[s].len, stream);
        if (rc != IMAGD_OK) return rc;
    }
    return IMAGD_OK;
}

}  // namespace imagd

extern "C" int imagd_attention_bwd_prep(const void* d_out, int64_t do_ld, const void* o0, const void* o1, int64_t ld_s,
                                        float w0, float w1, float* dsum, int B, int Lq, int heads, int head_dim, int lq_pad,
                                        imagd_stream stream) {
    using namespace imagd;
    IMAGD_CHECK_ARG(d_out && o0 && dsum && B > 0 && Lq > 0 && heads > 0 && lq_pad >= Lq, "attention_bwd_prep: bad argument");
    const int64_t warps = static_cast<int64_t>(B) * Lq * heads;
    const int threads = 256;
    const int64_t blocks = (warps * 32 + threads - 1) / threads;
    attn_bwd_prep_kernel<<<static_cast<unsigned>(blocks), threads, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const __nv_bfloat16*>(d_out), do_ld, static_cast<const __nv_bfloat16*>(o0),
        static_cast<const __nv_bfloat16*>(o1), ld_s, w0, w1, dsum, B, Lq, heads, head_dim, lq_pad);
    IMAGD_LAUNCH_CHECK("attn_bwd_prep_kernel");
    return IMAGD_OK;
}

extern "C" int imagd_attention_bwd_bf16(const void* q, int64_t q_ld, const void* d_out, int64_t do_ld, int B, int Lq,
                                        int heads, int head_dim, const imagd_kv_stream* s0, const imagd_kv_stream* s1,
                                        float sm_scale, const float* lse, const float* dsum, int lq_pad, void* dq,
                                        int64_t dq_ld, void* dk0, void* dv0, int64_t dkv0_ld, void* dk1, void* dv1,
                                        int64_t dkv1_ld, imagd_stream stream) {
    using namespace imagd;
    IMAGD_CHECK_ARG(q && d_out && s0 && s0->k && s0->v && lse && dsum, "attention_bwd: null pointer");
    IMAGD_CHECK_ARG(B > 0 && Lq > 0 && heads > 0, "attention_bwd: bad shape");
    IMAGD_CHECK_ARG(head_dim == 40 || head_dim == 64 || head_dim == 80 || head_dim == 160,
                    "attention_bwd: head_dim %d not in {40, 64, 80, 160}", head_dim);
    IMAGD_CHECK_ARG(lq_pad >= Lq && lq_pad % 128 == 0, "attention_bwd: lq_pad must be a multiple of 128 >= Lq");
    const bool has1 = s1 != nullptr && s1->k != nullptr && s1->len > 0;
    IMAGD_CHECK_ARG(!s0->broadcast && s0->n_query_samples >= B && (!has1 || (!s1->broadcast && s1->n_query_samples >= B)),
                    "attention_bwd: every query sample must own its keys in both streams (no broadcast / partial streams)");
    IMAGD_CHECK_ARG((dq == nullptr || (dq_ld % 8 == 0 && aligned16(dq))) &&
                        ((dk0 == nullptr) == (dv0 == nullptr)) && ((dk1 == nullptr) == (dv1 == nullptr)),
                    "attention_bwd: output pointers");
    IMAGD_CHECK_ARG((!dk0 || (dkv0_ld % 8 == 0 && aligned16(dk0) && aligned16(dv0))) &&
                        (!dk1 || (has1 && dkv1_ld % 8 == 0 && aligned16(dk1) && aligned16(dv1))),
                    "attention_bwd: dk / dv alignment");

    AttnBwdParams p{};
    p.B = B;
    p.Lq = Lq;
    p.heads = heads;
    p.hd = head_dim;
    p.sm_scale = sm_scale;
    p.scale_log2 = sm_scale * 1.4426950408889634f;
    p.q = static_cast<const __nv_bfloat16*>(q);
    p.q_ld = q_ld;
    p.d_out = static_cast<const __nv_bfloat16*>(d_out);
    p.do_ld = do_ld;
    IMAGD_CHECK_ARG(q_ld % 8 == 0 && do_ld % 8 == 0 && aligned16(q) && aligned16(d_out), "attention_bwd: Q / dO alignment");
    for (int s = 0; s < 2; ++s) {
        const imagd_kv_stream* ks = s ? s1 : s0;
        if (s == 1 && !has1) break;
        IMAGD_CHECK_ARG(ks->ld % 8 == 0 && aligned16(ks->k) && aligned16(ks->v), "attention_bwd: K / V alignment");
        p.kv[s].k = static_cast<const __nv_bfloat16*>(ks->k);
        p.kv[s].v = static_cast<const __nv_bfloat16*>(ks->v);
        p.kv[s].ld = ks->ld;
        p.kv[s].len = ks->len;
        p.kv[s].sample_rows = ks->sample_rows > 0 ? ks->sample_rows : ks->len;
    }
    p.w0 = s0->out_scale;
    p.w1 = has1 ? s1->out_scale : 0.f;
    p.lq_pad = lq_pad;
    p.lse = lse;
    p.dsum = dsum;
    p.dq = dq;
    p.dq_ld = dq_ld;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    switch (head_dim) {
        case 40: return launch_bwd<48>(p, dk0, dv0, dkv0_ld, dk1, dv1, dkv1_ld, st);
        case 64: return launch_bwd<64>(p, dk0, dv0, dkv0_ld, dk1, dv1, dkv1_ld, st);
        case 80: return launch_bwd<80>(p, dk0, dv0, dkv0_ld, dk1, dv1, dkv1_ld, st);
        default: return launch_bwd<160>(p, dk0, dv0, dkv0_ld, dk1, dv1, dkv1_ld, st);
    }
}
