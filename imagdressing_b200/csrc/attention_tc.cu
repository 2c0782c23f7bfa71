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
// Data layout: Q/K/V stay in the projection GEMM's natural token-major output [rows, ld] (heads side by side in
// the channel dim). Tiles are copied to shared memory with cp.async in 16-byte pieces; the head-dim columns
// beyond hd (40 -> 48) and the rows beyond a stream's length are zero-filled, so no padded copies exist in HBM.
//
// CTA = 128 queries of one (sample, head), 8 warps of 16 query rows each. Key blocks of 64 rows stream through a
// two-stage K / V ring; S = Q K^T and O += P V run on the tensor cores (mma.sync m16n8k16, bf16 -> fp32) with the
// probabilities kept in registers (the S accumulator fragment is the P operand fragment). Online softmax in the log2
// domain; when the first stream is done its weighted output w0 O0 / l0 waits in shared memory (fp32) for the second.
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
__global__ void __launch_bounds__(256, 1) attention_fwd_kernel(const AttnParams p) {
    using C = AttnSmem<HDP>;
    constexpr int kRow = attn_row_bytes(HDP);
    constexpr int NT = HDP / 8;  // n8 tiles of O
    extern __shared__ __align__(128) uint8_t smem[];
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

// ------------------------------------------------------------------------------------------------ host side

template <int HDP>
static int launch_attn(const AttnParams& p, cudaStream_t stream) {
    using C = AttnSmem<HDP>;
    IMAGD_SET_MAX_SMEM(attention_fwd_kernel<HDP>, C::kTotal);
    dim3 grid((p.Lq + 127) / 128, p.heads, p.B);
    IMAGD_CUDA(launch_pdl(attention_fwd_kernel<HDP>, grid, dim3(256), C::kTotal, stream, p));
    return IMAGD_OK;
}

}  // namespace imagd

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
        IMAGD_CHECK_ARG(!causal, "attention(train): causal not supported");
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    switch (head_dim) {
        case 40: return launch_attn<48>(p, st);
        case 64: return launch_attn<64>(p, st);
        case 80: return launch_attn<80>(p, st);
        default: return launch_attn<160>(p, st);
    }
}
