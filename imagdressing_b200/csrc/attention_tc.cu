// Two-stream ("hybrid") FlashAttention-style kernel for sm_90a.
//
//   out = w0 * softmax(Q K0^T * s) V0  +  w1 * softmax(Q K1^T * s) V1
//
// The two softmaxes are independent (separate running max / sum and separate O accumulators) but share one
// resident Q tile, exactly the arithmetic of RefSAttnProcessor2_0 (reference adapter/attention_processor.py:
// 589-612: self SDPA, garment SDPA on the same query, scale-add) and of LoRAIPAttnProcessor2_0's text + IP
// pair (:833-856). With w1 unused it is plain SDPA (cross-attention, the garment UNet's cached self-attention,
// the Perceiver resampler).
//
// Q/K/V stay in the projection GEMM's natural token-major output [rows, ld] (heads side by side in the channel dim);
// columns beyond head_dim and rows beyond a stream's length are zero-filled on the way into shared memory, so no padded
// copies exist in HBM. Online softmax in the log2 domain; when the first stream is done its weighted output w0 O0 / l0
// waits in shared memory (fp32) for the second. CTA = 128 queries of one (sample, head). Two kernels:
//
// attention_fwd_wgmma_kernel (head_dim 40 / 80, non-causal, streams of >= kAttnWgmmaMinKeys keys: the hybrid
// self-attention of UNet levels 0 and 1). 384 threads:
//   warps 0-3  consumer warpgroup 0: query rows 0-63     warps 4-7  consumer warpgroup 1: query rows 64-127
//   warps 8-11 producer warpgroup; one lane issues TMA: the Q tile once, then the 128-key K / V blocks of stream 0 and
//              stream 1 through a ring of full / empty mbarriers. Both consumer warpgroups read every stage, so a block
//              crosses L2 once per 128 query rows.
//   Each operand is read through one 4-D TMA map (head_dim, heads, rows of a sample, samples) in 128B-swizzled boxes 64
//   columns wide; out-of-bounds fill zeroes the columns >= head_dim and the rows >= the stream's length. Per key block
//   each warpgroup runs S = Q K^T (wgmma, both operands in shared memory, K-major) and O += P V (wgmma, P from registers:
//   the S accumulator packed to bf16; V in shared memory, MN-major). The next block's Q K^T and this block's P V are in
//   flight while the warpgroup computes the softmax, so the exp2 / FP32 work of one block overlaps the tensor work of
//   its neighbours, with no CTA-wide barrier per block. The softmax scale folds into one FFMA with the running max; the
//   length mask runs only on a stream's last block.
//
// attention_fwd_mma_kernel (everything else: text / IP cross-attention, head_dim 64 / 160, causal, short streams).
//   8 warps of 16 query rows; 64-key K / V blocks arrive by cp.async into a two-stage ring of padded rows; S = Q K^T
//   and O += P V on mma.sync.m16n8k16 with P kept in registers. With one or two key blocks per CTA the work is
//   dominated by load latency, which this kernel hides with up to three resident CTAs per SM; the wgmma kernel holds
//   an SM alone (its consumers take 232 registers per thread).
#include <cstdlib>

#include "common.cuh"
#include "ptx.cuh"
#include "attention_common.cuh"

namespace imagd {

struct AttnParams {
    int B, Lq, heads, hd;
    float scale_log2;  // sm_scale * log2(e)
    const __nv_bfloat16* q;
    int64_t q_ld;
    AttnKV kv[2];      // stream 0 / 1
    int nq1;           // stream 1 applies to samples [0, nq1)
    float oscale0, oscale1;
    int causal;        // stream 0 only: query q sees keys 0..q
    void* out;
    int64_t out_ld;
    // training-mode extras (imagd_attention_train_fwd_bf16; all null / 0 on the inference path): per-row log-sum-exp of
    // each stream in the log2 domain, [2][B][heads][lq_pad] fp32, and the un-weighted per-stream outputs O_s / l_s
    float* lse;
    void* out_s0;
    void* out_s1;
    int64_t ld_s;
    int lq_pad;
};

template <int HDP>
struct AttnSmem {
    static constexpr int kQBytes = 128 * attn_row_bytes(HDP);
    static constexpr int kKVBytes = 64 * attn_row_bytes(HDP);  // one K or V block
    static constexpr int kKOff = kQBytes;
    static constexpr int kVOff = kKOff + 2 * kKVBytes;
    static constexpr int kOutOff = kVOff + 2 * kKVBytes;       // fp32 w0 O0 / l0 of the first stream, [HDP / 2][256 threads]
    static constexpr int kTotal = kOutOff + HDP / 2 * 256 * 4;
};

template <int HDP>
__global__ void __launch_bounds__(256, 1) attention_fwd_mma_kernel(const AttnParams p) {
    using C = AttnSmem<HDP>;
    constexpr int kRow = attn_row_bytes(HDP);
    constexpr int NT = HDP / 8;  // n8 tiles of O
    extern __shared__ __align__(1024) uint8_t smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int q0 = blockIdx.x * 128;
    const int h = blockIdx.y;
    const int b = blockIdx.z;
    const uint32_t sQ = smem_u32(smem), sK = sQ + C::kKOff, sV = sQ + C::kVOff;
    float* s_out = reinterpret_cast<float*>(smem + C::kOutOff);

    const int nb0 = (p.kv[0].len + 63) / 64;
    const int nb1 = (b < p.nq1) ? (p.kv[1].len + 63) / 64 : 0;
    const int T = nb0 + nb1;

    pdl_launch_dependents();
    pdl_wait();
    attn_load_rows<HDP>(sQ, p.q + (static_cast<int64_t>(b) * p.Lq) * p.q_ld + h * p.hd, p.q_ld, p.hd, q0, p.Lq, 128);
    auto load_kv = [&](int i) {
        const int s = i < nb0 ? 0 : 1;
        const int j = s ? i - nb0 : i;
        const AttnKV& kv = p.kv[s];
        const int64_t base = static_cast<int64_t>(kv.bcast ? 0 : b) * kv.sample_rows * kv.ld + h * p.hd;
        attn_load_rows<HDP>(sK + (i & 1) * C::kKVBytes, kv.k + base, kv.ld, p.hd, j * 64, kv.len, 64);
        attn_load_rows<HDP>(sV + (i & 1) * C::kKVBytes, kv.v + base, kv.ld, p.hd, j * 64, kv.len, 64);
    };
    load_kv(0);
    cp_async_commit();

    const int g = lane >> 2, t = lane & 3;
    const int row0 = q0 + warp * 16 + g;  // this thread's query rows: row0, row0 + 8
    float o[NT][4];
#pragma unroll
    for (int n = 0; n < NT; ++n) o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    float m_first[2] = {0.f, 0.f}, l_first[2] = {0.f, 0.f};

    for (int i = 0; i < T; ++i) {
        const int s = i < nb0 ? 0 : 1;
        const int j = s ? i - nb0 : i;
        if (j == 0 && i > 0) {
            // first stream done: park w0 * O0 / l0 (and the per-stream output of a training forward), restart for stream 1
#pragma unroll
            for (int hr = 0; hr < 2; ++hr) {
                l_run[hr] = quad_sum(l_run[hr]);
                m_first[hr] = m_run[hr];
                l_first[hr] = l_run[hr];
            }
            const float u0 = 1.f / l_run[0], u1 = 1.f / l_run[1];
#pragma unroll
            for (int n = 0; n < NT; ++n) {
                s_out[(n * 4 + 0) * 256 + threadIdx.x] = p.oscale0 * o[n][0] * u0;
                s_out[(n * 4 + 1) * 256 + threadIdx.x] = p.oscale0 * o[n][1] * u0;
                s_out[(n * 4 + 2) * 256 + threadIdx.x] = p.oscale0 * o[n][2] * u1;
                s_out[(n * 4 + 3) * 256 + threadIdx.x] = p.oscale0 * o[n][3] * u1;
            }
            if (p.out_s0 != nullptr)
                attn_store_frag<NT>(o, u0, u1, reinterpret_cast<__nv_bfloat16*>(p.out_s0), p.ld_s, static_cast<int64_t>(b) * p.Lq, p.Lq, h, p.hd, row0, t);
#pragma unroll
            for (int n = 0; n < NT; ++n) o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f;
            m_run[0] = m_run[1] = -INFINITY;
            l_run[0] = l_run[1] = 0.f;
        }
        cp_async_wait<0>();
        __syncthreads();  // block i landed for every thread; every warp is done with block i - 1's stage
        if (i + 1 < T) load_kv(i + 1);
        cp_async_commit();

        // S = Q K^T: 16 rows x 64 keys per warp
        float sc[8][4];
#pragma unroll
        for (int n = 0; n < 8; ++n) sc[n][0] = sc[n][1] = sc[n][2] = sc[n][3] = 0.f;
        const uint32_t kb = sK + (i & 1) * C::kKVBytes;
#pragma unroll
        for (int ks = 0; ks < HDP / 16; ++ks) {
            uint32_t a[4];
            ldmatrix_x4(a, sQ + (warp * 16 + (lane & 15)) * kRow + (ks * 16 + (lane >> 4) * 8) * 2);
#pragma unroll
            for (int np = 0; np < 4; ++np) {
                uint32_t bb[4];
                ldmatrix_x4(bb, kb + (np * 16 + (lane & 7) + (lane >> 4) * 8) * kRow + (ks * 16 + ((lane >> 3) & 1) * 8) * 2);
                mma_bf16_16816(sc[2 * np], a, bb[0], bb[1]);
                mma_bf16_16816(sc[2 * np + 1], a, bb[2], bb[3]);
            }
        }
        // mask + block row max (the four threads of a quad share a row)
        const int len = p.kv[s].len;
        float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int n = 0; n < 8; ++n) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int key = j * 64 + n * 8 + 2 * t + (e & 1);
                const int qrow = row0 + (e >> 1) * 8;
                bool ok = key < len;
                if (s == 0 && p.causal) ok = ok && key <= qrow;
                sc[n][e] = ok ? sc[n][e] * p.scale_log2 : -INFINITY;
                mx[e >> 1] = fmaxf(mx[e >> 1], sc[n][e]);
            }
        }
        float alpha[2];
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
            const float m_new = fmaxf(m_run[hr], quad_max(mx[hr]));
            alpha[hr] = ex2_approx(m_run[hr] - m_new);  // 0 on a stream's first block
            m_run[hr] = m_new;
            l_run[hr] *= alpha[hr];
        }
#pragma unroll
        for (int n = 0; n < NT; ++n) {
            o[n][0] *= alpha[0];
            o[n][1] *= alpha[0];
            o[n][2] *= alpha[1];
            o[n][3] *= alpha[1];
        }
        // P = exp2(S - m) -> bf16 A fragments (keys 16 kk .. 16 kk + 15), O += P V
        const uint32_t vb = sV + (i & 1) * C::kKVBytes;
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
            uint32_t a[4];
#pragma unroll
            for (int hf = 0; hf < 2; ++hf) {
                float* c = sc[2 * kk + hf];
                const float e0 = ex2_approx(c[0] - m_run[0]), e1 = ex2_approx(c[1] - m_run[0]);
                const float e2 = ex2_approx(c[2] - m_run[1]), e3 = ex2_approx(c[3] - m_run[1]);
                l_run[0] += e0 + e1;
                l_run[1] += e2 + e3;
                a[2 * hf] = pack_bf16x2(e0, e1);
                a[2 * hf + 1] = pack_bf16x2(e2, e3);
            }
#pragma unroll
            for (int np = 0; np < NT / 2; ++np) {
                uint32_t bb[4];
                ldmatrix_x4_trans(bb, vb + (kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * kRow + (np * 16 + (lane >> 4) * 8) * 2);
                mma_bf16_16816(o[2 * np], a, bb[0], bb[1]);
                mma_bf16_16816(o[2 * np + 1], a, bb[2], bb[3]);
            }
        }
    }

    // ---- epilogue: out = w0 * O0 / l0 + w1 * O1 / l1
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) l_run[hr] = quad_sum(l_run[hr]);
    const float u0 = 1.f / l_run[0], u1 = 1.f / l_run[1];
    if (p.lse != nullptr && t == 0) {  // training: log2-domain log-sum-exp per stream (m + log2 l)
        const int64_t per = static_cast<int64_t>(p.B) * p.heads * p.lq_pad;
        float* lp = p.lse + (static_cast<int64_t>(b) * p.heads + h) * p.lq_pad;
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
            const int q = row0 + hr * 8;
            if (q >= p.Lq) continue;
            if (nb1 > 0) {
                lp[q] = m_first[hr] + __log2f(l_first[hr]);
                lp[per + q] = m_run[hr] + __log2f(l_run[hr]);
            } else {
                lp[q] = m_run[hr] + __log2f(l_run[hr]);
            }
        }
    }
    if (nb1 > 0 && p.out_s1 != nullptr)
        attn_store_frag<NT>(o, u0, u1, reinterpret_cast<__nv_bfloat16*>(p.out_s1), p.ld_s, static_cast<int64_t>(b) * p.Lq, p.Lq, h, p.hd, row0, t);
    const float w = nb1 > 0 ? p.oscale1 : p.oscale0;
#pragma unroll
    for (int n = 0; n < NT; ++n) {
        float f[4] = {w * o[n][0] * u0, w * o[n][1] * u0, w * o[n][2] * u1, w * o[n][3] * u1};
        if (nb1 > 0) {
#pragma unroll
            for (int e = 0; e < 4; ++e) f[e] += s_out[(n * 4 + e) * 256 + threadIdx.x];
        }
        o[n][0] = f[0];
        o[n][1] = f[1];
        o[n][2] = f[2];
        o[n][3] = f[3];
    }
    attn_store_frag<NT>(o, 1.f, 1.f, reinterpret_cast<__nv_bfloat16*>(p.out), p.out_ld, static_cast<int64_t>(b) * p.Lq, p.Lq, h, p.hd, row0, t);
}

// Stream-0 length from which the wgmma kernel runs: measured on H100, it is faster from 8 key blocks per CTA on (UNet
// levels 0 and 1, 4096 and 1024 keys) and slower on the 77 text tokens.
constexpr int kAttnWgmmaMinKeys = 1024;
// two consumer warpgroups + one producer warpgroup: at 384 threads each SM sub-partition holds one warp of each, so the
// producer's registers (40 of the 168 the launch grants) can go to the consumers (232), which hold S, P and O
constexpr int kAttnThreads = 384;
constexpr int kAttnBox = 64;  // TMA box width in head-dim columns: one 128-byte swizzle row

// Key block and ring depth. Head_dim 80 (two boxes per row, 40 O accumulators) takes 64-key blocks: with 128 the S, P
// and O registers of a consumer thread do not fit without spilling inside the key loop.
template <int HD>
struct AttnCfg {
    static_assert(HD == 40 || HD == 80, "wgmma attention: head_dim 40 or 80");
    static constexpr int kBN = HD == 40 ? 128 : 64;
    static constexpr int kStages = 3;
    static constexpr int kBoxes = (HD + kAttnBox - 1) / kAttnBox;
    static constexpr int kKSteps = (HD + 15) / 16;                  // Q K^T k-steps: head_dim padded to 16
    static constexpr int kQBytes = kBoxes * 128 * 128;
    static constexpr int kKVBoxBytes = kBN * 128;                  // one 64-column box of a K or V block
    static constexpr int kStageBytes = 2 * kBoxes * kKVBoxBytes;   // K | V
    static constexpr int kRingOff = kQBytes;
    static constexpr int kParkOff = kRingOff + kStages * kStageBytes;  // fp32 w0 O0 / l0: [HD / 2][256 threads]
    static constexpr int kBarOff = kParkOff + HD / 2 * 256 * 4;
    static constexpr int kTotal = kBarOff + (1 + 2 * kStages) * 8;
    // every TMA destination (Q box, K / V box) starts on a 1024-byte swizzle atom
    static_assert(kRingOff % 1024 == 0 && kKVBoxBytes % 1024 == 0 && kStageBytes % 1024 == 0, "swizzle alignment");
    static_assert(kTotal <= 227 * 1024, "shared memory");
};

template <int BN>
__device__ __forceinline__ void wgmma_qk(float (&d)[BN / 2], uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
    if constexpr (BN == 64) wgmma_m64n64k16(d, a_desc, b_desc, scale_d);
    else wgmma_m64n128k16(d, a_desc, b_desc, scale_d);
}
template <int HD>
__device__ __forceinline__ void wgmma_pv(float (&d)[HD / 2], const uint32_t (&a)[4], uint64_t b_desc) {
    if constexpr (HD == 40) wgmma_m64n40k16_rs(d, a, b_desc, 1u);
    else wgmma_m64n80k16_rs(d, a, b_desc, 1u);
}

template <int HD>
__global__ void __launch_bounds__(kAttnThreads, 1)
attention_fwd_wgmma_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK0,
                     const __grid_constant__ CUtensorMap tmV0, const __grid_constant__ CUtensorMap tmK1,
                     const __grid_constant__ CUtensorMap tmV1, const AttnParams p) {
    using C = AttnCfg<HD>;
    constexpr int BN = C::kBN, S = C::kStages, NT = HD / 8;
    extern __shared__ __align__(1024) uint8_t smem[];  // SWIZZLE_128B tiles need 1024-byte alignment
    uint64_t* q_bar = reinterpret_cast<uint64_t*>(smem + C::kBarOff);
    uint64_t* full_bar = q_bar + 1;
    uint64_t* empty_bar = full_bar + S;
    float* s_park = reinterpret_cast<float*>(smem + C::kParkOff);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int q0 = blockIdx.x * 128;
    const int h = blockIdx.y;
    const int b = blockIdx.z;
    const int nb0 = (p.kv[0].len + BN - 1) / BN;
    const int nb1 = (b < p.nq1) ? (p.kv[1].len + BN - 1) / BN : 0;
    const int T = nb0 + nb1;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmQ);
        tma_prefetch_desc(&tmK0);
        tma_prefetch_desc(&tmV0);
        tma_prefetch_desc(&tmK1);
        tma_prefetch_desc(&tmV1);
        mbar_init(q_bar, 1);
        for (int i = 0; i < S; ++i) {
            mbar_init(&full_bar[i], 1);
            mbar_init(&empty_bar[i], 2);  // one arrival per consumer warpgroup
        }
        fence_barrier_init();
    }
    __syncthreads();
    pdl_launch_dependents();
    pdl_wait();

    if (warp >= 8) {
        setmaxnreg_dec<40>();
        if (warp == 8 && elect_one()) {
            mbar_arrive_expect_tx(q_bar, C::kQBytes);
            for (int x = 0; x < C::kBoxes; ++x) tma_load_4d(smem + x * 128 * 128, &tmQ, q_bar, x * kAttnBox, h, q0, b);
            for (int i = 0; i < T; ++i) {
                const int stage = i % S;
                mbar_wait_quiet(&empty_bar[stage], ((i / S) & 1) ^ 1);
                mbar_arrive_expect_tx(&full_bar[stage], C::kStageBytes);
                const int s = i < nb0 ? 0 : 1;
                const int r0 = (s ? i - nb0 : i) * BN;
                const CUtensorMap* tk = s ? &tmK1 : &tmK0;
                const CUtensorMap* tv = s ? &tmV1 : &tmV0;
                uint8_t* sk = smem + C::kRingOff + stage * C::kStageBytes;
                uint8_t* sv = sk + C::kBoxes * C::kKVBoxBytes;
                const int smp = (s ? p.kv[1].bcast : p.kv[0].bcast) ? 0 : b;
                for (int x = 0; x < C::kBoxes; ++x) {
                    tma_load_4d(sk + x * C::kKVBoxBytes, tk, &full_bar[stage], x * kAttnBox, h, r0, smp);
                    tma_load_4d(sv + x * C::kKVBoxBytes, tv, &full_bar[stage], x * kAttnBox, h, r0, smp);
                }
            }
        }
        return;
    }

    setmaxnreg_inc<232>();
    const int wg = warp >> 2;
    const int g = lane >> 2, t = lane & 3;
    const int row0 = q0 + wg * 64 + (warp & 3) * 16 + g;  // this thread's query rows: row0, row0 + 8
    const bool leader = (threadIdx.x & 127) == 0;
    const uint32_t sq = smem_u32(smem) + wg * 64 * 128;
    const uint32_t ring = smem_u32(smem + C::kRingOff);

    float o[HD / 2];
#pragma unroll
    for (int n = 0; n < HD / 2; ++n) o[n] = 0.f;
    float sc[BN / 2];
    uint32_t pa[BN / 16][4];
    // m: running row max of the raw scores; ms = m * scale_log2; l: this thread's share of the running row sum
    float m_run[2] = {-INFINITY, -INFINITY}, ms_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    float ms_first[2] = {0.f, 0.f}, l_first[2] = {0.f, 0.f};
    float alpha[2] = {0.f, 0.f};

    auto issue_qk = [&](int i) __attribute__((always_inline)) {
        const uint32_t kb = ring + (i % S) * C::kStageBytes;
        wgmma_fence_regs(sc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < C::kKSteps; ++k) {
            wgmma_qk<BN>(sc, wgmma_desc_sw128(sq + (k / 4) * 128 * 128 + (k % 4) * 32),
                         wgmma_desc_sw128(kb + (k / 4) * C::kKVBoxBytes + (k % 4) * 32), k > 0 ? 1u : 0u);
        }
        wgmma_commit();
    };
    auto issue_pv = [&](int i) __attribute__((always_inline)) {
        const uint32_t vb = ring + (i % S) * C::kStageBytes + C::kBoxes * C::kKVBoxBytes;
#pragma unroll
        for (int n = 0; n < HD / 8; ++n) {
            o[4 * n + 0] *= alpha[0];
            o[4 * n + 1] *= alpha[0];
            o[4 * n + 2] *= alpha[1];
            o[4 * n + 3] *= alpha[1];
        }
        wgmma_fence_regs(o);
        wgmma_fence_regs(pa);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < BN / 16; ++kk)
            wgmma_pv<HD>(o, pa[kk], wgmma_desc_sw128_mn(vb + kk * 16 * 128, C::kKVBoxBytes));
        wgmma_commit();
    };
    // S of block i (landed in sc) -> exp2 values in sc, running max / sum, alpha for the O rescale
    auto softmax = [&](int i) __attribute__((always_inline)) {
        const int s = i < nb0 ? 0 : 1;
        const int j = s ? i - nb0 : i;
        const int len = s ? p.kv[1].len : p.kv[0].len;
        if ((j + 1) * BN > len) {
#pragma unroll
            for (int n = 0; n < BN / 8; ++n) {
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    if (j * BN + n * 8 + 2 * t + (e & 1) >= len) sc[4 * n + e] = -INFINITY;
                }
            }
        }
        float mx[2] = {m_run[0], m_run[1]};
#pragma unroll
        for (int n = 0; n < BN / 8; ++n) {
            mx[0] = fmaxf(mx[0], fmaxf(sc[4 * n + 0], sc[4 * n + 1]));
            mx[1] = fmaxf(mx[1], fmaxf(sc[4 * n + 2], sc[4 * n + 3]));
        }
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
            m_run[hr] = quad_max(mx[hr]);
            const float ms = m_run[hr] * p.scale_log2;
            alpha[hr] = ex2_approx(ms_run[hr] - ms);  // 0 on a stream's first block
            ms_run[hr] = ms;
            l_run[hr] *= alpha[hr];
        }
#pragma unroll
        for (int n = 0; n < BN / 8; ++n) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float v = ex2_approx(fmaf(sc[4 * n + e], p.scale_log2, -ms_run[e >> 1]));
                sc[4 * n + e] = v;
                l_run[e >> 1] += v;
            }
        }
    };
    // exp2 values -> bf16 A fragments of P V (keys 16 kk .. 16 kk + 15)
    auto pack_p = [&]() __attribute__((always_inline)) {
#pragma unroll
        for (int kk = 0; kk < BN / 16; ++kk) {
            pa[kk][0] = pack_bf16x2(sc[8 * kk + 0], sc[8 * kk + 1]);
            pa[kk][1] = pack_bf16x2(sc[8 * kk + 2], sc[8 * kk + 3]);
            pa[kk][2] = pack_bf16x2(sc[8 * kk + 4], sc[8 * kk + 5]);
            pa[kk][3] = pack_bf16x2(sc[8 * kk + 6], sc[8 * kk + 7]);
        }
    };
    float o4[NT][4];
    auto view_o4 = [&]() __attribute__((always_inline)) {
#pragma unroll
        for (int n = 0; n < NT; ++n)
#pragma unroll
            for (int e = 0; e < 4; ++e) o4[n][e] = o[4 * n + e];
    };

    mbar_wait_quiet(q_bar, 0);
    mbar_wait_quiet(&full_bar[0], 0);
    issue_qk(0);
    wgmma_wait<0>();
    wgmma_fence_regs(sc);
    softmax(0);
    pack_p();
    for (int i = 1; i < T; ++i) {
        mbar_wait_quiet(&full_bar[i % S], (i / S) & 1);
        issue_qk(i);       // S_i = Q K_i^T ...
        issue_pv(i - 1);   // ... and O = alpha O + P_{i-1} V_{i-1} in flight together
        wgmma_wait<1>();
        wgmma_fence_regs(sc);
        const bool switch1 = i == nb0;
        if (switch1) {     // first block of stream 1: stream 0's statistics are final
#pragma unroll
            for (int hr = 0; hr < 2; ++hr) {
                ms_first[hr] = ms_run[hr];
                l_first[hr] = quad_sum(l_run[hr]);
                m_run[hr] = ms_run[hr] = -INFINITY;
                l_run[hr] = 0.f;
            }
        }
        softmax(i);
        wgmma_wait<0>();
        wgmma_fence_regs(o);
        wgmma_fence_regs(pa);
        if (leader) mbar_arrive(&empty_bar[(i - 1) % S]);
        pack_p();
        if (switch1) {
            // stream 0 done: park w0 * O0 / l0 (and the per-stream output of a training forward), restart for stream 1
            const float u0 = 1.f / l_first[0], u1 = 1.f / l_first[1];
            view_o4();
#pragma unroll
            for (int n = 0; n < NT; ++n) {
                s_park[(n * 4 + 0) * 256 + threadIdx.x] = p.oscale0 * o4[n][0] * u0;
                s_park[(n * 4 + 1) * 256 + threadIdx.x] = p.oscale0 * o4[n][1] * u0;
                s_park[(n * 4 + 2) * 256 + threadIdx.x] = p.oscale0 * o4[n][2] * u1;
                s_park[(n * 4 + 3) * 256 + threadIdx.x] = p.oscale0 * o4[n][3] * u1;
            }
            if (p.out_s0 != nullptr)
                attn_store_frag<NT>(o4, u0, u1, reinterpret_cast<__nv_bfloat16*>(p.out_s0), p.ld_s,
                                    static_cast<int64_t>(b) * p.Lq, p.Lq, h, p.hd, row0, t);
#pragma unroll
            for (int n = 0; n < HD / 2; ++n) o[n] = 0.f;
        }
    }
    issue_pv(T - 1);
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    wgmma_fence_regs(pa);

    // ---- epilogue: out = w0 * O0 / l0 + w1 * O1 / l1
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) l_run[hr] = quad_sum(l_run[hr]);
    const float u0 = 1.f / l_run[0], u1 = 1.f / l_run[1];
    view_o4();
    if (p.lse != nullptr && t == 0) {  // training: log2-domain log-sum-exp per stream (m + log2 l)
        const int64_t per = static_cast<int64_t>(p.B) * p.heads * p.lq_pad;
        float* lp = p.lse + (static_cast<int64_t>(b) * p.heads + h) * p.lq_pad;
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
            const int q = row0 + hr * 8;
            if (q >= p.Lq) continue;
            if (nb1 > 0) {
                lp[q] = ms_first[hr] + __log2f(l_first[hr]);
                lp[per + q] = ms_run[hr] + __log2f(l_run[hr]);
            } else {
                lp[q] = ms_run[hr] + __log2f(l_run[hr]);
            }
        }
    }
    if (nb1 > 0 && p.out_s1 != nullptr)
        attn_store_frag<NT>(o4, u0, u1, reinterpret_cast<__nv_bfloat16*>(p.out_s1), p.ld_s, static_cast<int64_t>(b) * p.Lq,
                            p.Lq, h, p.hd, row0, t);
    const float w = nb1 > 0 ? p.oscale1 : p.oscale0;
#pragma unroll
    for (int n = 0; n < NT; ++n) {
        float f[4] = {w * o4[n][0] * u0, w * o4[n][1] * u0, w * o4[n][2] * u1, w * o4[n][3] * u1};
        if (nb1 > 0) {
#pragma unroll
            for (int e = 0; e < 4; ++e) f[e] += s_park[(n * 4 + e) * 256 + threadIdx.x];
        }
        o4[n][0] = f[0];
        o4[n][1] = f[1];
        o4[n][2] = f[2];
        o4[n][3] = f[3];
    }
    attn_store_frag<NT>(o4, 1.f, 1.f, reinterpret_cast<__nv_bfloat16*>(p.out), p.out_ld, static_cast<int64_t>(b) * p.Lq,
                        p.Lq, h, p.hd, row0, t);
}

// ------------------------------------------------------------------------------------------------ host side

// One head-sliced operand as a 4-D map (head_dim, heads, rows, samples), box 64 columns x `rows_box` rows of one head
static int make_head_tmap(CUtensorMap* m, const void* base, int hd, int heads, int64_t ld, int rows, int64_t sample_rows,
                          int samples, int rows_box) {
    const uint64_t dims[4] = {static_cast<uint64_t>(hd), static_cast<uint64_t>(heads), static_cast<uint64_t>(rows),
                              static_cast<uint64_t>(samples)};
    const uint64_t strides[3] = {static_cast<uint64_t>(hd) * 2, static_cast<uint64_t>(ld) * 2,
                                 static_cast<uint64_t>(sample_rows) * ld * 2};
    const uint32_t box[4] = {kAttnBox, 1, static_cast<uint32_t>(rows_box), 1};
    return make_tmap_bf16(m, base, 4, dims, strides, box);
}

// ss[1] == nullptr: no second stream (its maps repeat stream 0's, which the kernel never reads then)
template <int HD>
static int launch_attn_wgmma(const AttnParams& p, const imagd_kv_stream* const (&ss)[2],
                       cudaStream_t stream) {
    using C = AttnCfg<HD>;
    CUtensorMap tm[5];
    int rc = make_head_tmap(&tm[0], p.q, HD, p.heads, p.q_ld, p.Lq, p.Lq, p.B, 128);
    for (int s = 0; s < 2 && rc == IMAGD_OK; ++s) {
        if (ss[s] == nullptr) {
            tm[3] = tm[1];
            tm[4] = tm[2];
            break;
        }
        const imagd_kv_stream* kv = ss[s];
        const int64_t sample_rows = kv->sample_rows > 0 ? kv->sample_rows : kv->len;
        const int samples = kv->broadcast ? 1 : (s == 0 ? p.B : p.nq1);
        rc = make_head_tmap(&tm[1 + 2 * s], kv->k, HD, p.heads, kv->ld, kv->len, sample_rows, samples, C::kBN);
        if (rc == IMAGD_OK)
            rc = make_head_tmap(&tm[2 + 2 * s], kv->v, HD, p.heads, kv->ld, kv->len, sample_rows, samples, C::kBN);
    }
    if (rc != IMAGD_OK) return rc;
    IMAGD_SET_MAX_SMEM(attention_fwd_wgmma_kernel<HD>, C::kTotal);
    dim3 grid((p.Lq + 127) / 128, p.heads, p.B);
    IMAGD_CUDA(launch_pdl(attention_fwd_wgmma_kernel<HD>, grid, dim3(kAttnThreads), C::kTotal, stream, tm[0], tm[1], tm[2], tm[3],
                          tm[4], p));
    return IMAGD_OK;
}

template <int HDP>
static int launch_attn_mma(const AttnParams& p, cudaStream_t stream) {
    using C = AttnSmem<HDP>;
    IMAGD_SET_MAX_SMEM(attention_fwd_mma_kernel<HDP>, C::kTotal);
    dim3 grid((p.Lq + 127) / 128, p.heads, p.B);
    IMAGD_CUDA(launch_pdl(attention_fwd_mma_kernel<HDP>, grid, dim3(256), C::kTotal, stream, p));
    return IMAGD_OK;
}

// Test hook (imagd_attention_debug_force): 0 automatic, 1 the mma.sync kernel, 2 the wgmma kernel
constexpr int kAttnForceMma = 1, kAttnForceWgmma = 2;
static int g_attn_force = 0;

}  // namespace imagd

extern "C" int imagd_attention_debug_force(int kernel) {
    using namespace imagd;
    IMAGD_CHECK_ARG(kernel == 0 || kernel == kAttnForceMma || kernel == kAttnForceWgmma, "attention_debug_force: kernel %d",
                    kernel);
    g_attn_force = kernel;
    return IMAGD_OK;
}

static int attention_impl(const void* q, int64_t q_ld, void* out, int64_t out_ld, int B, int Lq, int heads, int head_dim,
                          const imagd_kv_stream* s0, const imagd_kv_stream* s1, float sm_scale, int causal,
                          imagd_stream stream, const imagd_attn_train* aux = nullptr);

extern "C" int imagd_attention_train_fwd_bf16(const void* q, int64_t q_ld, void* out, int64_t out_ld, int B, int Lq, int heads,
                                              int head_dim, const imagd_kv_stream* s0, const imagd_kv_stream* s1,
                                              float sm_scale, const imagd_attn_train* aux, imagd_stream stream) {
    IMAGD_CHECK_ARG(aux != nullptr, "attention(train): aux is null");
    return attention_impl(q, q_ld, out, out_ld, B, Lq, heads, head_dim, s0, s1, sm_scale, 0, stream, aux);
}

extern "C" int imagd_attention_bf16(const void* q, int64_t q_ld, void* out, int64_t out_ld, int B, int Lq, int heads,
                                    int head_dim, const imagd_kv_stream* s0, const imagd_kv_stream* s1, float sm_scale,
                                    imagd_stream stream) {
    return attention_impl(q, q_ld, out, out_ld, B, Lq, heads, head_dim, s0, s1, sm_scale, 0, stream);
}

extern "C" int imagd_attention_causal_bf16(const void* q, int64_t q_ld, void* out, int64_t out_ld, int B, int Lq, int heads,
                                           int head_dim, const imagd_kv_stream* s0, float sm_scale, imagd_stream stream) {
    return attention_impl(q, q_ld, out, out_ld, B, Lq, heads, head_dim, s0, nullptr, sm_scale, 1, stream);
}

static int attention_impl(const void* q, int64_t q_ld, void* out, int64_t out_ld, int B, int Lq, int heads, int head_dim,
                          const imagd_kv_stream* s0, const imagd_kv_stream* s1, float sm_scale, int causal,
                          imagd_stream stream, const imagd_attn_train* aux) {
    using namespace imagd;
    IMAGD_CHECK_ARG(q && out && s0 && s0->k && s0->v, "attention: null pointer");
    IMAGD_CHECK_ARG(B > 0 && Lq > 0 && heads > 0, "attention: bad shape");
    IMAGD_CHECK_ARG(head_dim == 40 || head_dim == 64 || head_dim == 80 || head_dim == 160,
                    "attention: head_dim %d not in {40, 64, 80, 160}", head_dim);
    IMAGD_CHECK_ARG(s0->len > 0 && s0->n_query_samples >= B, "attention: stream 0 must cover every query sample");
    IMAGD_CHECK_ARG(out_ld % 8 == 0 && aligned16(out), "attention: output alignment");
    IMAGD_CHECK_ARG(s0->sample_rows == 0 || s0->sample_rows >= s0->len, "attention: sample_rows < len");
    const bool has1 = s1 != nullptr && s1->k != nullptr && s1->len > 0 && s1->n_query_samples > 0;

    AttnParams p{};
    p.B = B;
    p.Lq = Lq;
    p.heads = heads;
    p.hd = head_dim;
    p.scale_log2 = sm_scale * 1.4426950408889634f;
    p.q = static_cast<const __nv_bfloat16*>(q);
    p.q_ld = q_ld;
    const imagd_kv_stream* ss[2] = {s0, has1 ? s1 : s0};
    for (int s = 0; s < 2; ++s) {
        p.kv[s].k = static_cast<const __nv_bfloat16*>(ss[s]->k);
        p.kv[s].v = static_cast<const __nv_bfloat16*>(ss[s]->v);
        p.kv[s].ld = ss[s]->ld;
        p.kv[s].len = ss[s]->len;
        p.kv[s].sample_rows = ss[s]->sample_rows > 0 ? ss[s]->sample_rows : ss[s]->len;
        p.kv[s].bcast = ss[s]->broadcast;
        IMAGD_CHECK_ARG(ss[s]->ld % 8 == 0 && aligned16(ss[s]->k) && aligned16(ss[s]->v), "attention: K / V alignment");
    }
    IMAGD_CHECK_ARG(q_ld % 8 == 0 && aligned16(q), "attention: Q alignment");
    p.nq1 = has1 ? (s1->n_query_samples < B ? s1->n_query_samples : B) : 0;
    p.oscale0 = s0->out_scale;
    p.oscale1 = has1 ? s1->out_scale : 0.f;
    p.causal = causal;
    p.out = out;
    p.out_ld = out_ld;
    p.lse = aux ? aux->lse : nullptr;
    p.out_s0 = aux ? aux->out_s0 : nullptr;
    p.out_s1 = aux ? aux->out_s1 : nullptr;
    p.ld_s = aux ? aux->ld_s : 0;
    p.lq_pad = aux ? aux->lq_pad : 0;
    if (aux) {
        IMAGD_CHECK_ARG(aux->lse && aux->lq_pad >= Lq && aux->lq_pad % 128 == 0, "attention(train): lse / lq_pad");
        IMAGD_CHECK_ARG(!has1 || (aux->out_s0 && aux->out_s1 && aux->ld_s % 8 == 0 && aligned16(aux->out_s0) &&
                                  aligned16(aux->out_s1)),
                        "attention(train): two streams need out_s0 / out_s1");
        // out_s0 is stored when stream 1 starts, so a sample that skips stream 1 would leave its O_0 rows unwritten;
        // the backward needs every query sample in both streams anyway
        IMAGD_CHECK_ARG(!has1 || s1->n_query_samples >= B,
                        "attention(train): stream 1 must cover every query sample (n_query_samples %d < B %d)",
                        s1->n_query_samples, B);
        IMAGD_CHECK_ARG(!causal, "attention(train): causal not supported");
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const bool wgmma_ok = (head_dim == 40 || head_dim == 80) && !causal;
    const int force = g_attn_force;
    IMAGD_CHECK_ARG(force != kAttnForceWgmma || wgmma_ok,
                    "attention: the wgmma kernel was forced but serves head_dim 40 / 80 non-causal only (head_dim %d%s)",
                    head_dim, causal ? ", causal" : "");
    const bool use_wgmma = force == kAttnForceWgmma || (force == 0 && wgmma_ok && s0->len >= kAttnWgmmaMinKeys);
    if (use_wgmma) {
        const imagd_kv_stream* ws[2] = {s0, has1 ? s1 : nullptr};
        return head_dim == 40 ? launch_attn_wgmma<40>(p, ws, st) : launch_attn_wgmma<80>(p, ws, st);
    }
    switch (head_dim) {
        case 40: return launch_attn_mma<48>(p, st);
        case 64: return launch_attn_mma<64>(p, st);
        case 80: return launch_attn_mma<80>(p, st);
        default: return launch_attn_mma<160>(p, st);
    }
}
