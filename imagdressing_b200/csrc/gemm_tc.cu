// wgmma GEMM / implicit-GEMM 3x3 convolution for sm_90a.
//
//   D[p, c] = epilogue( sum_{tap, k} A_tap[p, k] * W[c, tap*Cin + k] )
//
// A is a token-major bf16 activation [NB, H, W, ld]; for the 3x3 convolution the nine taps are nine shifted
// views of the same tensor, fetched by TMA as 4-D boxes (channels, x, y, image) whose out-of-bounds part the
// hardware zero-fills — that is the conv's zero padding, with no im2col buffer. A plain GEMM is the same
// kernel with one tap and a [K, M, 1, 1] view.
//
// CTA = 128 output pixels x BLOCK_N output channels: a TMA producer warp feeds a STAGES-deep ring of 128B-swizzled
// A / B tiles, two warpgroups accumulate 64 rows each with wgmma in registers, and the accumulator tile is handed to
// the epilogue through shared memory (bias / time-embedding row vector / activation / residual -> bf16 stores).
// One CTA runs per SM (288 threads, up to 168 registers each, 96-200 KB of shared memory).
#include <algorithm>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "common.cuh"
#include "ptx.cuh"

namespace imagd {

struct GemmParams {
    // K loop
    int taps;          // 1 or 9
    int kb_per_tap;    // ceil(Cin / 64)
    int cin;           // K per tap (weight column offset between taps)
    // pixel-tile geometry: a tile is bw x bh x bn pixels (product 128)
    int bw, bh, bn;
    int tiles_x, tiles_y;
    int W, H, NB;
    // output
    int N;             // logical output columns of the GEMM (before GEGLU halving)
    void* out;
    int64_t ldd;
    imagd_epilogue ep;
    // split-K: gridDim.z CTAs share one output tile; fp32 partials meet in `ws`, the last arriver reduces them in
    // a fixed order (deterministic) and runs the epilogue
    int splits;
    int kb_per_split;
    float* ws;
    unsigned int* counters;
    // debug: when non-null, every CTA records its timeline (imagd_gemm_debug_timeline; tools/gemm_timeline.py)
    unsigned long long* dbg;
    int ups_n_tiles;  // LNM == 3: N tiles per phase (gridDim.y = 4 * ups_n_tiles)
    int pdl_late;     // 1: release the dependent kernel when the accumulator is complete instead of at kernel entry
};

__device__ __forceinline__ void dbg_mark(const GemmParams& p, int slot) {
    if (p.dbg != nullptr) {
        const int64_t cta = (static_cast<int64_t>(blockIdx.z) * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
        p.dbg[cta * 8 + slot] = static_cast<unsigned long long>(clock64());
    }
}

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;
constexpr int kABytes = kBlockM * kBlockK * 2;  // 16 KB
constexpr int kGemmThreads = 288;               // two consumer warpgroups + one producer warp

template <int BLOCK_N, int STAGES>
struct GemmSmem {
    static constexpr int kBBytes = BLOCK_N * kBlockK * 2;
    static constexpr int kStageBytes = kABytes + kBBytes;
    static constexpr int kRing = STAGES * kStageBytes;
    // after the mainloop the fp32 accumulator tile is staged row by row over the idle operand ring: one row per epilogue
    // thread, +16 bytes so that the float4 reads of eight consecutive rows hit eight bank groups
    static constexpr int kAccRowBytes = BLOCK_N * 4 + 16;
    static constexpr int kAccBytes = kBlockM * kAccRowBytes;
    static constexpr int kBarOffset = (kRing > kAccBytes ? kRing : kAccBytes);
    static constexpr int kVecOffset = (kBarOffset + (2 * STAGES) * 8 + 16 + 15) & ~15;  // float4 reads
    // epilogue vectors staged once per CTA: bias[BLOCK_N] | row vector[BLOCK_N] (when the tile lies in one row group)
    static constexpr int kTotal = kVecOffset + 2 * BLOCK_N * 4;
};

// LINEAR = the epilogue has no activation and writes bf16 (every conv and most linears of the UNet): straight-line,
// branch-free column loop. !LINEAR = the generic epilogue (SiLU / GELU / GEGLU / fp32 output).
// EPI: 0 generic, 1 LINEAR, 2 LINEAR with the output row staged in shared memory (in the thread's own accumulator row,
// behind the columns it has already read) and written by one bulk copy per row instead of 16-byte stores.
// LNM: LayerNorm folding (see include/imagd_b200.h): 0 off, 1 producer (emit per-row {sum, sum of squares} of the rounded
// outputs, one slot per N tile), 2 consumer (apply rstd * (alpha * acc - mean * colsum) + bias).
//
// CTA = 128 output pixels x BLOCK_N output channels, 288 threads:
//   warps 0-3  warpgroup 0: wgmma on accumulator rows 0-63, then the epilogue (thread = tile row)
//   warps 4-7  warpgroup 1: wgmma on accumulator rows 64-127
//   warp 8     TMA producer (one elected lane; STAGES-deep smem ring, full / empty mbarriers)
template <int BLOCK_N, int STAGES, int EPI, int LNM>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmParams p) {
    using L = GemmSmem<BLOCK_N, STAGES>;
    constexpr bool LINEAR = EPI != 0;
    constexpr bool BULK = EPI == 2;
    constexpr bool LN_PRODUCE = LNM == 1;
    constexpr bool LN_CONSUME = LNM == 2;
    // LNM == 3: nearest-2x upsample + 3x3 conv as four 2x2 "phase" convs on the LOW-resolution input (2.25x fewer MACs,
    // no upsampled tensor): blockIdx.y = phase * n_tiles + n_blk, phase = py * 2 + px; tap t = ty * 2 + tx reads input
    // pixel (y + py - 1 + ty, x + px - 1 + tx); the weight matrix is [4 * N, 4 * Cin] (phase-major rows, tap-major
    // columns); output pixel (2y + py, 2x + px) of a [NB, 2H, 2W, N] tensor.
    constexpr bool UPS = LNM == 3;
    static_assert(!LN_PRODUCE || LINEAR, "row statistics are emitted by the LINEAR epilogue only");
    static_assert(BLOCK_N % 64 == 0 || BLOCK_N == 160, "wgmma N tile");
    extern __shared__ __align__(1024) uint8_t smem[];  // SWIZZLE_128B tiles need 1024-byte alignment
    if (threadIdx.x == 0 && (smem_u32(smem) & 1023u) != 0) __trap();  // (no printf: see mbar_wait_quiet)
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::kBarOffset);
    uint64_t* empty_bar = full_bar + STAGES;
    uint32_t* flag_slot = reinterpret_cast<uint32_t*>(empty_bar + STAGES);
    float* s_bias = reinterpret_cast<float*>(smem + L::kVecOffset);
    float* s_rowvec = s_bias + BLOCK_N;

    if (!p.pdl_late) pdl_launch_dependents();
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    if (threadIdx.x == 0 && p.dbg != nullptr) {
        dbg_mark(p, 0);
        unsigned long long gt;
        unsigned int smid;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(gt));
        asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
        const int64_t cta = (static_cast<int64_t>(blockIdx.z) * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
        p.dbg[cta * 8 + 6] = gt;
        p.dbg[cta * 8 + 7] = smid;
    }

    // tile coordinates
    const int m_blk = blockIdx.x;
    const int ups_phase = UPS ? static_cast<int>(blockIdx.y) / p.ups_n_tiles : 0;
    const int n_blk = UPS ? static_cast<int>(blockIdx.y) % p.ups_n_tiles : static_cast<int>(blockIdx.y);
    const int tx = m_blk % p.tiles_x;
    const int ty = (m_blk / p.tiles_x) % p.tiles_y;
    const int tn = m_blk / (p.tiles_x * p.tiles_y);
    const int x0 = tx * p.bw, y0 = ty * p.bh, n0 = tn * p.bn;
    const int total_kb = p.taps * p.kb_per_tap;
    const int kb_begin = blockIdx.z * p.kb_per_split;
    const int nk = min(total_kb, kb_begin + p.kb_per_split) - kb_begin;  // >= 1 (host guarantees)

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        for (int i = 0; i < STAGES; ++i) {
            mbar_init(&full_bar[i], 1);
            mbar_init(&empty_bar[i], 2);  // one arrival per consumer warpgroup
        }
        fence_barrier_init();
    }
    __syncthreads();
    if (threadIdx.x == 0) dbg_mark(p, 1);
    pdl_wait();  // predecessor's output (our A operand / residual) and our output buffer are safe from here on

    if (warp == 8) {
        if (elect_one()) {
            for (int i = 0; i < nk; ++i) {
                const int kb = kb_begin + i;
                const int stage = i % STAGES;
                const uint32_t phase = (i / STAGES) & 1;
                mbar_wait_quiet(&empty_bar[stage], phase ^ 1);
                mbar_arrive_expect_tx(&full_bar[stage], L::kStageBytes);
                const int tap = kb / p.kb_per_tap;
                const int kc = kb - tap * p.kb_per_tap;
                int dx = 0, dy = 0;
                if constexpr (UPS) {
                    dy = (ups_phase >> 1) - 1 + (tap >> 1);
                    dx = (ups_phase & 1) - 1 + (tap & 1);
                } else if (p.taps == 9) {
                    dy = tap / 3 - 1;
                    dx = tap % 3 - 1;
                }
                uint8_t* sa = smem + stage * L::kStageBytes;
                uint8_t* sb = sa + kABytes;
                tma_load_4d(sa, &tmA, &full_bar[stage], kc * kBlockK, x0 + dx, y0 + dy, n0);
                tma_load_2d(sb, &tmB, &full_bar[stage], tap * p.cin + kc * kBlockK,
                            (UPS ? ups_phase * p.N : 0) + n_blk * BLOCK_N);
            }
        }
        return;
    }

    const int wg = warp >> 2;  // consumer warpgroup: accumulator rows [64 wg, 64 wg + 64)
    const imagd_epilogue& ep = p.ep;
    const int col_base = n_blk * BLOCK_N;
    // ---- epilogue preparation (warpgroup 0, before the mainloop): stage the per-column vectors in shared memory (every
    // row of the tile reads the same bias; the row vector too when the whole tile lies in one row group, i.e. one sample)
    const int r = threadIdx.x;  // warpgroup 0: tile-local pixel
    const int x = x0 + r % p.bw;
    const int y = y0 + (r / p.bw) % p.bh;
    const int n = n0 + r / (p.bw * p.bh);
    const bool row_ok = (x < p.W) && (y < p.H) && (n < p.NB);
    const int64_t pix = UPS ? (static_cast<int64_t>(n) * (2 * p.H) + (2 * y + (ups_phase >> 1))) * (2 * p.W) +
                                  (2 * x + (ups_phase & 1))
                            : (static_cast<int64_t>(n) * p.H + y) * p.W + x;
    const float* rowvec = nullptr;  // per-thread global fallback (tile spans several row groups)
    bool rowvec_shared = false;
    float ln_mean = 0.f, ln_rstd = 0.f;
    if (wg == 0) {
        if (ep.rowvec != nullptr) {
            const int xl = min(x0 + p.bw, p.W) - 1, yl = min(y0 + p.bh, p.H) - 1, nl = min(n0 + p.bn, p.NB) - 1;
            const int64_t pix_first = (static_cast<int64_t>(n0) * p.H + y0) * p.W + x0;
            const int64_t pix_last = (static_cast<int64_t>(nl) * p.H + yl) * p.W + xl;
            const int64_t g_first = pix_first / ep.rows_per_group;
            rowvec_shared = g_first == pix_last / ep.rows_per_group;
            if (rowvec_shared) {
                const float* src = ep.rowvec + g_first * ep.rowvec_ld;
                for (int c = threadIdx.x; c < BLOCK_N; c += 128)
                    s_rowvec[c] = (col_base + c < p.N) ? __ldg(src + col_base + c) : 0.f;
            } else if (row_ok) {
                rowvec = ep.rowvec + (pix / ep.rows_per_group) * ep.rowvec_ld;
            }
        }
        if constexpr (LN_CONSUME) {  // the row-vector slot carries the folded weight's column sums instead
            for (int c = threadIdx.x; c < BLOCK_N; c += 128)
                s_rowvec[c] = (col_base + c < p.N) ? __ldg(ep.colsum + col_base + c) : 0.f;
        } else if (LINEAR && !rowvec_shared) {  // the straight-line loop always adds the staged vectors: absent = zeros
            for (int c = threadIdx.x; c < BLOCK_N; c += 128) s_rowvec[c] = 0.f;
        }
        if (ep.bias != nullptr) {
            for (int c = threadIdx.x; c < BLOCK_N; c += 128)
                s_bias[c] = (col_base + c < p.N) ? __ldg(ep.bias + col_base + c) : 0.f;
        } else if (LINEAR) {
            for (int c = threadIdx.x; c < BLOCK_N; c += 128) s_bias[c] = 0.f;
        }
        if constexpr (LN_CONSUME) {
            if (row_ok) {  // fixed-order fold of the producer's per-tile partials -> mean / rstd of my row of A
                const float2* sp = reinterpret_cast<const float2*>(ep.row_stats_in) + pix * ep.stats_in_ld;
                float s1 = 0.f, s2 = 0.f;
                for (int i = 0; i < ep.stats_parts; ++i) {
                    const float2 t = __ldg(sp + i);
                    s1 += t.x;
                    s2 += t.y;
                }
                const float inv = 1.0f / static_cast<float>(ep.ln_dim);
                ln_mean = s1 * inv;
                ln_rstd = rsqrtf(fmaxf(fmaf(-ln_mean, ln_mean, s2 * inv), 0.f) + ep.ln_eps);
            }
        }
    }

    // ---- mainloop: each warpgroup multiplies its 64 rows of A by the whole B tile; the previous stage is released once
    // the MMAs that read it have retired (wait_group 1 keeps one group in flight)
    {
        float acc[BLOCK_N / 2];
#pragma unroll
        for (int j = 0; j < BLOCK_N / 2; ++j) acc[j] = 0.f;
        const bool leader = (threadIdx.x & 127) == 0;
        for (int i = 0; i < nk; ++i) {
            const int stage = i % STAGES;
            mbar_wait_quiet(&full_bar[stage], (i / STAGES) & 1);
            if (i == 0 && threadIdx.x == 0) dbg_mark(p, 2);
            const uint32_t sa = smem_u32(smem + stage * L::kStageBytes) + wg * (64 * 128);
            const uint32_t sb = smem_u32(smem + stage * L::kStageBytes) + kABytes;
            wgmma_fence_regs(acc);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < kBlockK / 16; ++k) {
                const uint64_t ad = wgmma_desc_sw128(sa + k * 32), bd = wgmma_desc_sw128(sb + k * 32);
                if constexpr (BLOCK_N == 64) wgmma_m64n64k16(acc, ad, bd, 1u);
                else if constexpr (BLOCK_N == 128) wgmma_m64n128k16(acc, ad, bd, 1u);
                else if constexpr (BLOCK_N == 160) wgmma_m64n160k16(acc, ad, bd, 1u);
                else wgmma_m64n256k16(acc, ad, bd, 1u);
            }
            wgmma_commit();
            wgmma_wait<1>();
            wgmma_fence_regs(acc);
            if (i > 0 && leader) mbar_arrive(&empty_bar[(i - 1) % STAGES]);
        }
        wgmma_wait<0>();
        wgmma_fence_regs(acc);
        // every MMA of the CTA has to retire before the ring is overwritten by the accumulator rows
        asm volatile("bar.sync 1, 256;" ::: "memory");
        if (threadIdx.x == 0) dbg_mark(p, 3);
        if (p.pdl_late) pdl_launch_dependents();  // mainloop done: the next kernel's prologue may overlap this epilogue
        // wgmma m64nN accumulator layout: warp w of the warpgroup holds rows 16 w + lane / 4 (+ 8), columns 8 j + 2 (lane % 4)
        const int wrow = wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j) {
            const int col = j * 8 + 2 * (lane & 3);
            *reinterpret_cast<float2*>(smem + wrow * L::kAccRowBytes + col * 4) = make_float2(acc[4 * j], acc[4 * j + 1]);
            *reinterpret_cast<float2*>(smem + (wrow + 8) * L::kAccRowBytes + col * 4) =
                make_float2(acc[4 * j + 2], acc[4 * j + 3]);
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");
    }
    if (wg != 0) return;

    {
        // ---------------- epilogue (warpgroup 0, thread = tile row) ----------------
        const float alpha = ep.alpha;
        const __nv_bfloat16* res = nullptr;
        if (ep.residual != nullptr && row_ok)
            res = reinterpret_cast<const __nv_bfloat16*>(ep.residual) + pix * ep.ldr;
        const bool split = p.splits > 1;
        uint8_t* acc_row = smem + r * L::kAccRowBytes;
        uint4 rcur[4];
        auto load_res = [&](int c0, uint4(&rv)[4]) {
#pragma unroll
            for (int g = 0; g < 4; ++g) {
                const int cg = col_base + c0 + g * 8;
                rv[g] = (res != nullptr && cg < p.N) ? __ldg(reinterpret_cast<const uint4*>(res + cg))
                                                     : make_uint4(0u, 0u, 0u, 0u);
            }
        };
        if (!split) load_res(0, rcur);
        float st1 = 0.f, st2 = 0.f;  // producer: my row's statistics over this tile's columns
        if (threadIdx.x == 0) dbg_mark(p, 4);

        // ---- split-K rendezvous
        const int64_t tile_elems = static_cast<int64_t>(kBlockM) * BLOCK_N;
        const int64_t tile_id = static_cast<int64_t>(blockIdx.y) * gridDim.x + blockIdx.x;
        const int64_t n_tiles_total = static_cast<int64_t>(gridDim.x) * gridDim.y;
        if (split) {
            float* mine = p.ws + (static_cast<int64_t>(blockIdx.z) * n_tiles_total + tile_id) * tile_elems +
                          static_cast<int64_t>(r) * BLOCK_N;
#pragma unroll 1
            for (int c0 = 0; c0 < BLOCK_N; c0 += 4)
                __stcg(reinterpret_cast<float4*>(mine + c0), *reinterpret_cast<const float4*>(acc_row + c0 * 4));
            __threadfence();
            asm volatile("bar.sync 2, 128;" ::: "memory");
            if (threadIdx.x == 0) {
                const unsigned int old = atomicAdd(&p.counters[tile_id], 1u);
                *flag_slot = (old == static_cast<unsigned int>(p.splits - 1)) ? 1u : 0u;
                if (old == static_cast<unsigned int>(p.splits - 1)) p.counters[tile_id] = 0u;  // re-arm for next launch
            }
            asm volatile("bar.sync 2, 128;" ::: "memory");
            const bool last = *reinterpret_cast<volatile uint32_t*>(flag_slot) != 0u;
            if (!last) {
                if (threadIdx.x == 0) dbg_mark(p, 5);
                return;
            }
            __threadfence();
            load_res(0, rcur);
        }
        // accumulator chunk loader: my staged row (single CTA per tile) or the fixed-order sum of the split partials
        auto load_acc = [&](int c0, uint32_t(&v)[32]) {
            if (!split) {
#pragma unroll
                for (int j = 0; j < 32; j += 4) {
                    const uint4 t = *reinterpret_cast<const uint4*>(acc_row + (c0 + j) * 4);
                    v[j] = t.x; v[j + 1] = t.y; v[j + 2] = t.z; v[j + 3] = t.w;
                }
            } else {
                float acc[32];
#pragma unroll
                for (int j = 0; j < 32; ++j) acc[j] = 0.f;
                for (int sidx = 0; sidx < p.splits; ++sidx) {
                    const float* src = p.ws + (static_cast<int64_t>(sidx) * n_tiles_total + tile_id) * tile_elems +
                                       static_cast<int64_t>(r) * BLOCK_N + c0;
#pragma unroll
                    for (int j = 0; j < 32; j += 4) {
                        const float4 t = __ldcg(reinterpret_cast<const float4*>(src + j));
                        acc[j] += t.x; acc[j + 1] += t.y; acc[j + 2] += t.z; acc[j + 3] += t.w;
                    }
                }
#pragma unroll
                for (int j = 0; j < 32; ++j) v[j] = __float_as_uint(acc[j]);
            }
        };

        if constexpr (LINEAR) {
            constexpr int NCH = BLOCK_N / 32;
            __nv_bfloat16* orow = reinterpret_cast<__nv_bfloat16*>(p.out) + pix * p.ldd + col_base;
#pragma unroll
            for (int ch = 0; ch < NCH; ++ch) {
                const int c0 = ch * 32;
                uint32_t vc[32];
                load_acc(c0, vc);
                uint4 rnext[4];
                if (ch + 1 < NCH) load_res(c0 + 32, rnext);
                if (row_ok && col_base + c0 < p.N) {
#pragma unroll
                    for (int g = 0; g < 4; ++g) {
                        const int cl = c0 + g * 8;  // tile-local column
                        float f[8];
#pragma unroll
                        for (int j = 0; j < 8; ++j) f[j] = alpha * __uint_as_float(vc[g * 8 + j]);
                        if constexpr (LN_CONSUME) {
                            const float4 b0 = *reinterpret_cast<const float4*>(s_bias + cl);
                            const float4 b1 = *reinterpret_cast<const float4*>(s_bias + cl + 4);
                            const float4 c0v = *reinterpret_cast<const float4*>(s_rowvec + cl);
                            const float4 c1v = *reinterpret_cast<const float4*>(s_rowvec + cl + 4);
                            const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
                            const float cs[8] = {c0v.x, c0v.y, c0v.z, c0v.w, c1v.x, c1v.y, c1v.z, c1v.w};
#pragma unroll
                            for (int j = 0; j < 8; ++j) f[j] = fmaf(ln_rstd, fmaf(-ln_mean, cs[j], f[j]), bb[j]);
                        } else {
                            const float4 b0 = *reinterpret_cast<const float4*>(s_bias + cl);
                            const float4 b1 = *reinterpret_cast<const float4*>(s_bias + cl + 4);
                            f[0] += b0.x; f[1] += b0.y; f[2] += b0.z; f[3] += b0.w;
                            f[4] += b1.x; f[5] += b1.y; f[6] += b1.z; f[7] += b1.w;
                            const float4 r0 = *reinterpret_cast<const float4*>(s_rowvec + cl);
                            const float4 r1 = *reinterpret_cast<const float4*>(s_rowvec + cl + 4);
                            f[0] += r0.x; f[1] += r0.y; f[2] += r0.z; f[3] += r0.w;
                            f[4] += r1.x; f[5] += r1.y; f[6] += r1.z; f[7] += r1.w;
                        }
                        if (!LN_CONSUME && rowvec && col_base + cl < p.N) {  // rare: the tile spans several samples (deep levels)
                            const float4 b0 = __ldg(reinterpret_cast<const float4*>(rowvec + col_base + cl));
                            const float4 b1 = __ldg(reinterpret_cast<const float4*>(rowvec + col_base + cl + 4));
                            f[0] += b0.x; f[1] += b0.y; f[2] += b0.z; f[3] += b0.w;
                            f[4] += b1.x; f[5] += b1.y; f[6] += b1.z; f[7] += b1.w;
                        }
                        const uint4 rv = rcur[g];  // zeros when there is no residual
                        f[0] += bf16lo(rv.x); f[1] += bf16hi(rv.x); f[2] += bf16lo(rv.y); f[3] += bf16hi(rv.y);
                        f[4] += bf16lo(rv.z); f[5] += bf16hi(rv.z); f[6] += bf16lo(rv.w); f[7] += bf16hi(rv.w);
                        const uint4 o = make_uint4(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]),
                                                   pack_bf16x2(f[4], f[5]), pack_bf16x2(f[6], f[7]));
                        if constexpr (LN_PRODUCE) {  // statistics of what the consumer will READ: the rounded values
                            if (col_base + cl < p.N) {
                                const uint32_t ow[4] = {o.x, o.y, o.z, o.w};
#pragma unroll
                                for (int j = 0; j < 4; ++j) {
                                    const float lo = bf16lo(ow[j]), hi = bf16hi(ow[j]);
                                    st1 += lo + hi;
                                    st2 = fmaf(lo, lo, fmaf(hi, hi, st2));
                                }
                            }
                        }
                        if constexpr (BULK) {
                            // bytes [2 cl, 2 cl + 16) of my row: accumulator columns this thread has already read
                            *reinterpret_cast<uint4*>(acc_row + cl * 2) = o;
                        } else {
                            if (col_base + cl < p.N) *reinterpret_cast<uint4*>(orow + cl) = o;
                        }
                    }
                }
#pragma unroll
                for (int g = 0; g < 4; ++g) rcur[g] = rnext[g];
            }
            if constexpr (BULK) {
                // each thread ships its own row: generic-proxy writes -> async-proxy read needs the proxy fence only
                fence_proxy_async_smem();
                const int valid = min(BLOCK_N, p.N - col_base);
                if (row_ok && valid > 0) bulk_store_s2g(orow, smem_u32(acc_row), static_cast<uint32_t>(valid) * 2u);
                bulk_commit();
                bulk_wait_read0();  // the staging bytes must stay valid until the copy engine has read them
            }
            if constexpr (LN_PRODUCE) {
                if (row_ok)
                    reinterpret_cast<float2*>(ep.row_stats_out)[pix * ep.stats_ld + n_blk] = make_float2(st1, st2);
            }
        } else if (ep.act == IMAGD_ACT_GEGLU) {
            // tile = [64 value | 64 gate]; output columns n_blk*64 + [0, 64)
            if constexpr (BLOCK_N == 128) {
#pragma unroll 1
                for (int c0 = 0; c0 < 64; c0 += 32) {
                    uint32_t va[32], vg[32];
                    load_acc(c0, va);
                    load_acc(64 + c0, vg);
                    const int pcol = n_blk * 128 + c0;  // packed column of value; gate at +64
                    const int ocol = n_blk * 64 + c0;
                    if (row_ok && pcol < p.N) {
                        uint32_t packed[16];
#pragma unroll
                        for (int j = 0; j < 32; j += 2) {
                            float a0 = alpha * __uint_as_float(va[j]), a1 = alpha * __uint_as_float(va[j + 1]);
                            float g0 = alpha * __uint_as_float(vg[j]), g1 = alpha * __uint_as_float(vg[j + 1]);
                            if constexpr (LN_CONSUME) {  // bias (folded) is mandatory here: s_bias always staged
                                const float2 ba = *reinterpret_cast<const float2*>(s_bias + c0 + j);
                                const float2 bg = *reinterpret_cast<const float2*>(s_bias + 64 + c0 + j);
                                const float2 ca = *reinterpret_cast<const float2*>(s_rowvec + c0 + j);
                                const float2 cg = *reinterpret_cast<const float2*>(s_rowvec + 64 + c0 + j);
                                a0 = fmaf(ln_rstd, fmaf(-ln_mean, ca.x, a0), ba.x);
                                a1 = fmaf(ln_rstd, fmaf(-ln_mean, ca.y, a1), ba.y);
                                g0 = fmaf(ln_rstd, fmaf(-ln_mean, cg.x, g0), bg.x);
                                g1 = fmaf(ln_rstd, fmaf(-ln_mean, cg.y, g1), bg.y);
                            } else if (ep.bias) {
                                const float2 ba = *reinterpret_cast<const float2*>(s_bias + c0 + j);
                                const float2 bg = *reinterpret_cast<const float2*>(s_bias + 64 + c0 + j);
                                a0 += ba.x;
                                a1 += ba.y;
                                g0 += bg.x;
                                g1 += bg.y;
                            }
                            packed[j / 2] = pack_bf16x2(a0 * gelu_erf(g0), a1 * gelu_erf(g1));
                        }
                        uint4* dst = reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(p.out) + pix * p.ldd + ocol);
#pragma unroll
                        for (int q = 0; q < 4; ++q)
                            dst[q] = make_uint4(packed[4 * q], packed[4 * q + 1], packed[4 * q + 2], packed[4 * q + 3]);
                    }
                }
            }
        } else {
#pragma unroll 1
            for (int c0 = 0; c0 < BLOCK_N; c0 += 32) {
                uint32_t v[32];
                load_acc(c0, v);
                uint4 rnext[4];
                if (c0 + 32 < BLOCK_N) load_res(c0 + 32, rnext);  // in flight while this chunk is processed
                const int col = col_base + c0;
                if (row_ok && col < p.N) {
                // row vector fallback (tile spans several samples): all of the chunk's loads issued together
                float4 rvv[8];
                if (rowvec) {
#pragma unroll
                    for (int q = 0; q < 8; ++q)
                        rvv[q] = (col + q * 4 < p.N) ? __ldg(reinterpret_cast<const float4*>(rowvec + col + q * 4))
                                                     : make_float4(0.f, 0.f, 0.f, 0.f);
                }
                // columns are handled in groups of 8 (N % 8 == 0 is enforced on the host)
#pragma unroll
                for (int g = 0; g < 4; ++g) {
                    const int cg = col + g * 8;
                    if (cg >= p.N) break;
                    float f[8];
#pragma unroll
                    for (int j = 0; j < 8; ++j) f[j] = alpha * __uint_as_float(v[g * 8 + j]);
                    if (ep.bias) {
                        const float4 b0 = *reinterpret_cast<const float4*>(s_bias + c0 + g * 8);
                        const float4 b1 = *reinterpret_cast<const float4*>(s_bias + c0 + g * 8 + 4);
                        f[0] += b0.x; f[1] += b0.y; f[2] += b0.z; f[3] += b0.w;
                        f[4] += b1.x; f[5] += b1.y; f[6] += b1.z; f[7] += b1.w;
                    }
                    if (rowvec_shared) {
                        const float4 b0 = *reinterpret_cast<const float4*>(s_rowvec + c0 + g * 8);
                        const float4 b1 = *reinterpret_cast<const float4*>(s_rowvec + c0 + g * 8 + 4);
                        f[0] += b0.x; f[1] += b0.y; f[2] += b0.z; f[3] += b0.w;
                        f[4] += b1.x; f[5] += b1.y; f[6] += b1.z; f[7] += b1.w;
                    } else if (rowvec) {
                        const float4 b0 = rvv[2 * g], b1 = rvv[2 * g + 1];
                        f[0] += b0.x; f[1] += b0.y; f[2] += b0.z; f[3] += b0.w;
                        f[4] += b1.x; f[5] += b1.y; f[6] += b1.z; f[7] += b1.w;
                    }
                    if (ep.act == IMAGD_ACT_SILU) {
#pragma unroll
                        for (int j = 0; j < 8; ++j) f[j] = silu(f[j]);
                    } else if (ep.act == IMAGD_ACT_GELU) {
#pragma unroll
                        for (int j = 0; j < 8; ++j) f[j] = gelu_erf(f[j]);
                    } else if (ep.act == IMAGD_ACT_QUICK_GELU) {  // x * sigmoid(1.702 x): CLIP text MLP (quick_gelu)
#pragma unroll
                        for (int j = 0; j < 8; ++j) f[j] = __fdividef(f[j], 1.0f + __expf(-1.702f * f[j]));
                    }
                    if (res) {
                        const uint4 rv = rcur[g];
                        f[0] += bf16lo(rv.x); f[1] += bf16hi(rv.x); f[2] += bf16lo(rv.y); f[3] += bf16hi(rv.y);
                        f[4] += bf16lo(rv.z); f[5] += bf16hi(rv.z); f[6] += bf16lo(rv.w); f[7] += bf16hi(rv.w);
                    }
                    if (ep.out_fp32) {
                        float4* dst = reinterpret_cast<float4*>(reinterpret_cast<float*>(p.out) + pix * p.ldd + cg);
                        dst[0] = make_float4(f[0], f[1], f[2], f[3]);
                        dst[1] = make_float4(f[4], f[5], f[6], f[7]);
                    } else {
                        uint4* dst = reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(p.out) + pix * p.ldd + cg);
                        *dst = make_uint4(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]), pack_bf16x2(f[4], f[5]),
                                          pack_bf16x2(f[6], f[7]));
                    }
                }
                }
#pragma unroll
                for (int g = 0; g < 4; ++g) rcur[g] = rnext[g];
            }
        }
    }
    if (threadIdx.x == 0) dbg_mark(p, 5);
}

// ------------------------------------------------------------------------------------------------ host side

// Split 128 pixels into a (bw, bh, bn) box of powers of two that wastes the fewest tile slots.
static void choose_pixel_box(int W, int H, int NB, int* bw, int* bh, int* bn) {
    double best = -1.0;
    for (int w = 1; w <= 128; w *= 2) {
        for (int h = 1; w * h <= 128; h *= 2) {
            const int n = 128 / (w * h);
            const int64_t tiles = static_cast<int64_t>((W + w - 1) / w) * ((H + h - 1) / h) * ((NB + n - 1) / n);
            const double eff = static_cast<double>(static_cast<int64_t>(W) * H * NB) / (tiles * 128.0);
            // prefer wider boxes on ties (longer contiguous TMA rows)
            if (eff > best + 1e-9 || (eff > best - 1e-9 && w > *bw)) {
                best = eff;
                *bw = w;
                *bh = h;
                *bn = n;
            }
        }
    }
}

// ---- split-K scratch: fp32 partial tiles + per-tile arrival counters, one set per device, allocated on first use
// (outside any stream capture: the engine's eager warm-up step comes first). Kernels on one stream serialise, so
// one scratch area per device suffices; concurrent streams must not share a device.
constexpr size_t kWsBytes = size_t(96) << 20;
constexpr int kMaxTilesSplit = 1 << 16;
static float* g_ws[16] = {nullptr};
static unsigned int* g_counters[16] = {nullptr};

static std::mutex g_scratch_mu;

// Library-owned split-K scratch, one per device, allocated on first use. It is shared by every split-K launch on
// that device: callers must not run split-K GEMMs concurrently on several streams of one device (documented in
// include/imagd_b200.h). The first use must not happen inside a stream capture (cudaMalloc is illegal there).
static int ensure_scratch(float** ws, unsigned int** counters, cudaStream_t stream) {
    int dev = 0;
    IMAGD_CUDA(cudaGetDevice(&dev));
    IMAGD_CHECK_ARG(dev >= 0 && dev < 16, "gemm: device index %d out of range", dev);
    std::lock_guard<std::mutex> lock(g_scratch_mu);
    if (!g_ws[dev]) {
        cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
        IMAGD_CUDA(cudaStreamIsCapturing(stream, &st));
        if (st != cudaStreamCaptureStatusNone) {
            set_error("gemm: the split-K scratch is allocated on first use, which cannot happen inside a CUDA graph "
                      "capture; run the same call once eagerly before capturing");
            return IMAGD_ERR_CUDA;
        }
        IMAGD_CUDA(cudaMalloc(&g_ws[dev], kWsBytes));
        IMAGD_CUDA(cudaMalloc(&g_counters[dev], kMaxTilesSplit * sizeof(unsigned int)));
        IMAGD_CUDA(cudaMemset(g_counters[dev], 0, kMaxTilesSplit * sizeof(unsigned int)));
        IMAGD_CUDA(cudaDeviceSynchronize());
    }
    *ws = g_ws[dev];
    *counters = g_counters[dev];
    return IMAGD_OK;
}

// ---- tile / pipeline-depth / split-K choice --------------------------------------------------------------------
// Variants: N tile 64 / 128 / 160 / 256 with a "shallow" (2-4 stages) or "deep" (4-8 stages, ~190 KB) operand ring. Every
// variant runs one CTA per SM; the shared-memory footprint is max(ring, 128 x (4 BN + 16) bytes of accumulator staging)
// plus the epilogue vectors (about 96-200 KB). Deep rings keep more bytes in flight for grids of at most one wave, where
// each CTA is bound by the latency of its own TMA ring; split-K serves the deep UNet levels whose output has only a
// handful of tiles. The thresholds below are a rule of thumb in units of the 132 SMs, not tuned by measurement on H100.
struct GemmCfg {
    int bn, stages, splits;
};

static int shallow_stages(int bn) { return bn == 64 ? 4 : (bn == 256 ? 2 : 3); }
static int deep_stages(int bn) { return bn == 64 ? 8 : (bn == 128 ? 6 : (bn == 160 ? 5 : 4)); }

static GemmCfg choose_cfg(int m_tiles, int N, int kb_total, bool geglu) {
    auto ctas = [&](int bn) { return static_cast<int64_t>(m_tiles) * ((N + bn - 1) / bn); };
    if (geglu) return {128, ctas(128) > kNumSms ? 3 : 6, 1};
    if (ctas(160) >= 3 * kNumSms) return {160, 3, 1};  // many waves: widest 2-CTA/SM tile
    int bn = 64;
    if (ctas(160) >= kNumSms && ctas(160) <= 2 * kNumSms && (N % 160 == 0 || N > 640)) bn = 160;
    else if (ctas(128) >= kNumSms) bn = 128;
    int splits = 1;
    if (ctas(bn) < kNumSms * 2 / 3 && kb_total >= 60) {
        splits = static_cast<int>((kNumSms + ctas(bn) - 1) / ctas(bn));
        splits = std::min(splits, std::min(6, kb_total / 30));
        splits = std::max(splits, 1);
    }
    const bool deep = ctas(bn) * splits <= kNumSms;
    return {bn, deep ? deep_stages(bn) : shallow_stages(bn), splits};
}

template <int BLOCK_N, int STAGES, int EPI, int LNM = 0>
static int launch_gemm_impl(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParams& p, int m_tiles,
                            cudaStream_t stream) {
    using L = GemmSmem<BLOCK_N, STAGES>;
    constexpr int kSmem = L::kTotal;
    IMAGD_SET_MAX_SMEM((gemm_tc_kernel<BLOCK_N, STAGES, EPI, LNM>), kSmem);
    const int n_tiles = (p.N + BLOCK_N - 1) / BLOCK_N;
    dim3 grid(m_tiles, LNM == 3 ? 4 * n_tiles : n_tiles, p.splits);
    IMAGD_CUDA(launch_pdl(gemm_tc_kernel<BLOCK_N, STAGES, EPI, LNM>, grid, dim3(kGemmThreads), kSmem, stream, tmA, tmB, p));
    return IMAGD_OK;
}

template <int BLOCK_N, int STAGES>
static int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParams& p, int m_tiles,
                       cudaStream_t stream) {
    const bool linear = p.ep.act == IMAGD_ACT_NONE && !p.ep.out_fp32;
    if (p.ups_n_tiles > 0) {  // upsample-phase conv: plain bf16 epilogue (bias only), validated by the caller
        GemmParams q = p;
        q.ups_n_tiles = (p.N + BLOCK_N - 1) / BLOCK_N;
        return launch_gemm_impl<BLOCK_N, STAGES, 1, 3>(tmA, tmB, q, m_tiles, stream);
    }
    // LayerNorm folding variants (plain stores only for now; the bulk-store combination comes after validation)
    if (p.ep.row_stats_out != nullptr) return launch_gemm_impl<BLOCK_N, STAGES, 1, 1>(tmA, tmB, p, m_tiles, stream);
    if (p.ep.row_stats_in != nullptr) {
        if (linear) return launch_gemm_impl<BLOCK_N, STAGES, 1, 2>(tmA, tmB, p, m_tiles, stream);
        if constexpr (BLOCK_N == 128) return launch_gemm_impl<BLOCK_N, STAGES, 0, 2>(tmA, tmB, p, m_tiles, stream);
        set_error("gemm: LayerNorm-folded generic epilogue exists for the GEGLU tile (128) only");
        return IMAGD_ERR_ARG;
    }
    // Bulk row stores: for grids that cover the chip more than twice. IMAGD_GEMM_BULK_STORE = 0 / 1 forces them off / on.
    static int bulk_env = -2;
    if (bulk_env == -2) {
        const char* e = getenv("IMAGD_GEMM_BULK_STORE");
        bulk_env = e ? (e[0] == '1' ? 1 : 0) : -1;
    }
    const int64_t ctas = static_cast<int64_t>(m_tiles) * ((p.N + BLOCK_N - 1) / BLOCK_N) * p.splits;
    const bool bulk = bulk_env >= 0 ? bulk_env == 1 : ctas > 2 * kNumSms;
    if (!linear) return launch_gemm_impl<BLOCK_N, STAGES, 0>(tmA, tmB, p, m_tiles, stream);
    if (!bulk) return launch_gemm_impl<BLOCK_N, STAGES, 1>(tmA, tmB, p, m_tiles, stream);
    return launch_gemm_impl<BLOCK_N, STAGES, 2>(tmA, tmB, p, m_tiles, stream);
}


static int g_force_bn = 0, g_force_stages = 0, g_force_splits = 0;  // test hooks (imagd_gemm_debug_force)
static int g_log_on = 0;
static unsigned long long* g_dbg_timeline = nullptr;  // imagd_gemm_debug_timeline
static std::vector<std::string> g_log;  // unique problem keys seen while logging (tools/gemm_sweep.py)

static int run_gemm_like(const void* A, int64_t lda, int NB, int H, int W, int Cin, int taps, const void* Wt,
                         int64_t ldw, void* D, int64_t ldd, int N, const imagd_epilogue* ep_in, cudaStream_t stream,
                         bool ups_mode = false) {
    imagd_epilogue ep;
    if (ep_in) {
        ep = *ep_in;
    } else {
        memset(&ep, 0, sizeof(ep));
        ep.alpha = 1.0f;
    }
    IMAGD_CHECK_ARG(A && Wt && D, "gemm: null pointer");
    IMAGD_CHECK_ARG(Cin % 8 == 0 && lda % 8 == 0 && ldw % 8 == 0, "gemm: K=%d lda=%lld ldw=%lld must be multiples of 8",
                    Cin, (long long)lda, (long long)ldw);
    IMAGD_CHECK_ARG(N % 8 == 0, "gemm: N=%d must be a multiple of 8", N);
    IMAGD_CHECK_ARG(taps == 1 || Cin % 64 == 0, "conv3x3: Cin=%d must be a multiple of 64", Cin);
    const bool geglu = ep.act == IMAGD_ACT_GEGLU;
    IMAGD_CHECK_ARG(!geglu || N % 128 == 0, "gemm: GEGLU needs packed N %% 128 == 0 (N=%d)", N);
    IMAGD_CHECK_ARG(ldd % 8 == 0 && aligned16(D), "gemm: output ld=%lld / pointer must be 16-byte aligned", (long long)ldd);
    IMAGD_CHECK_ARG(!ep.residual || (ep.ldr % 8 == 0 && aligned16(ep.residual)), "gemm: residual alignment");
    IMAGD_CHECK_ARG(!ep.bias || aligned16(ep.bias), "gemm: bias alignment");
    IMAGD_CHECK_ARG(!ep.rowvec || (aligned16(ep.rowvec) && ep.rowvec_ld % 4 == 0 && ep.rows_per_group > 0),
                    "gemm: rowvec alignment / rows_per_group");
    IMAGD_CHECK_ARG(!(ep.row_stats_out && ep.row_stats_in), "gemm: a launch is either a statistics producer or a consumer");
    IMAGD_CHECK_ARG(!ep.row_stats_out || (ep.act == IMAGD_ACT_NONE && !ep.out_fp32 && ep.stats_ld > 0 &&
                                          (reinterpret_cast<uintptr_t>(ep.row_stats_out) & 7u) == 0),
                    "gemm: row_stats_out needs a plain bf16 epilogue, stats_ld > 0 and 8-byte alignment");
    IMAGD_CHECK_ARG(!ep.row_stats_in ||
                        (ep.colsum && ep.bias && ep.stats_parts > 0 && ep.stats_in_ld >= ep.stats_parts && ep.ln_dim == Cin &&
                         taps == 1 && !ep.rowvec && !ep.residual && !ep.out_fp32 &&
                         (ep.act == IMAGD_ACT_NONE || ep.act == IMAGD_ACT_GEGLU) &&
                         (reinterpret_cast<uintptr_t>(ep.row_stats_in) & 7u) == 0),
                    "gemm: LayerNorm-folded consumer needs colsum + folded bias, stats_parts, ln_dim == K, no rowvec / "
                    "residual / fp32 output, act NONE or GEGLU");

    GemmParams p;
    p.taps = taps;
    p.kb_per_tap = (Cin + kBlockK - 1) / kBlockK;
    p.cin = Cin;
    p.bw = p.bh = p.bn = 1;
    choose_pixel_box(W, H, NB, &p.bw, &p.bh, &p.bn);
    p.tiles_x = (W + p.bw - 1) / p.bw;
    p.tiles_y = (H + p.bh - 1) / p.bh;
    const int tiles_n = (NB + p.bn - 1) / p.bn;
    p.W = W;
    p.H = H;
    p.NB = NB;
    p.N = N;
    p.out = D;
    p.ldd = ldd;
    p.ep = ep;
    const int64_t m_tiles64 = static_cast<int64_t>(p.tiles_x) * p.tiles_y * tiles_n;
    IMAGD_CHECK_ARG(m_tiles64 > 0 && m_tiles64 < (1 << 30), "gemm: bad tile count");
    const int m_tiles = static_cast<int>(m_tiles64);
    const int kb_total = taps * p.kb_per_tap;

    GemmCfg cfg = choose_cfg(m_tiles, N, kb_total, geglu);
    if (g_force_bn) {
        cfg.bn = geglu ? 128 : g_force_bn;
        cfg.stages = g_force_stages ? g_force_stages : shallow_stages(cfg.bn);
        if (cfg.stages != shallow_stages(cfg.bn) && cfg.stages != deep_stages(cfg.bn)) cfg.stages = shallow_stages(cfg.bn);
    }
    if (g_force_splits && !geglu) cfg.splits = std::min(g_force_splits, kb_total);
    if (g_log_on) {
        char key[160];
        snprintf(key, sizeof(key), "%d %d %d %d %d %d %d %d %d %d", taps, NB, H, W, Cin, N, geglu ? 1 : 0, m_tiles,
                 kb_total, ep.out_fp32);
        if (std::find(g_log.begin(), g_log.end(), key) == g_log.end()) g_log.push_back(key);
    }
    IMAGD_CHECK_ARG(!ep.row_stats_out || ep.stats_ld >= (N + cfg.bn - 1) / cfg.bn,
                    "gemm: stats_ld=%lld is smaller than the %d N tiles of this launch (imagd_gemm_tile_count_n)",
                    (long long)ep.stats_ld, (N + cfg.bn - 1) / cfg.bn);
    if (ups_mode) cfg.splits = 1;  // (the split-K scratch is sized for one phase)
    p.ups_n_tiles = ups_mode ? 1 : 0;  // the launcher fills in the real tile count
    p.pdl_late = pdl_mode() == 2 ? 1 : 0;
    p.splits = cfg.splits;
    p.kb_per_split = (kb_total + cfg.splits - 1) / cfg.splits;
    p.splits = (kb_total + p.kb_per_split - 1) / p.kb_per_split;  // no empty splits
    p.ws = nullptr;
    p.counters = nullptr;
    p.dbg = g_dbg_timeline;
    if (p.splits > 1) {
        int rc = ensure_scratch(&p.ws, &p.counters, stream);
        if (rc != IMAGD_OK) return rc;
        const int64_t n_tiles = (N + cfg.bn - 1) / cfg.bn;
        IMAGD_CHECK_ARG(m_tiles64 * n_tiles <= kMaxTilesSplit &&
                            static_cast<size_t>(m_tiles64 * n_tiles * p.splits) * 128 * cfg.bn * 4 <= kWsBytes,
                        "gemm: split-K scratch too small");
    }

    // A: [NB, H, W, lda] viewed (c, x, y, n)
    CUtensorMap tmA, tmB;
    {
        uint64_t dims[4] = {static_cast<uint64_t>(Cin), static_cast<uint64_t>(W), static_cast<uint64_t>(H),
                            static_cast<uint64_t>(NB)};
        uint64_t strides[3] = {static_cast<uint64_t>(lda) * 2, static_cast<uint64_t>(lda) * 2 * W,
                               static_cast<uint64_t>(lda) * 2 * W * H};
        uint32_t box[4] = {kBlockK, static_cast<uint32_t>(p.bw), static_cast<uint32_t>(p.bh), static_cast<uint32_t>(p.bn)};
        int rc = make_tmap_bf16(&tmA, A, 4, dims, strides, box);
        if (rc != IMAGD_OK) return rc;
    }
    {
        uint64_t dims[2] = {static_cast<uint64_t>(taps) * Cin, static_cast<uint64_t>(N) * (ups_mode ? 4 : 1)};
        uint64_t strides[1] = {static_cast<uint64_t>(ldw) * 2};
        uint32_t box[2] = {kBlockK, static_cast<uint32_t>(cfg.bn)};
        int rc = make_tmap_bf16(&tmB, Wt, 2, dims, strides, box);
        if (rc != IMAGD_OK) return rc;
    }
    switch (cfg.bn * 100 + cfg.stages) {
        case 6404: return launch_gemm<64, 4>(tmA, tmB, p, m_tiles, stream);
        case 6408: return launch_gemm<64, 8>(tmA, tmB, p, m_tiles, stream);
        case 12803: return launch_gemm<128, 3>(tmA, tmB, p, m_tiles, stream);
        case 12806: return launch_gemm<128, 6>(tmA, tmB, p, m_tiles, stream);
        case 16003: return launch_gemm<160, 3>(tmA, tmB, p, m_tiles, stream);
        case 16005: return launch_gemm<160, 5>(tmA, tmB, p, m_tiles, stream);
        case 25602: return launch_gemm<256, 2>(tmA, tmB, p, m_tiles, stream);
        case 25604: return launch_gemm<256, 4>(tmA, tmB, p, m_tiles, stream);
        default:
            set_error("gemm: no kernel variant for N tile %d with %d stages", cfg.bn, cfg.stages);
            return IMAGD_ERR_ARG;
    }
}

}  // namespace imagd

extern "C" {

int imagd_gemm_bf16(const void* A, int64_t lda, const void* W, int64_t ldw, void* D, int64_t ldd, int M, int N, int K,
                    const imagd_epilogue* ep, imagd_stream stream) {
    IMAGD_CHECK_ARG(M > 0 && N > 0 && K > 0, "gemm: bad shape M=%d N=%d K=%d", M, N, K);
    return imagd::run_gemm_like(A, lda, 1, 1, M, K, 1, W, ldw, D, ldd, N, ep, static_cast<cudaStream_t>(stream));
}

int imagd_gemm_debug_force(int block_n, int stages, int splits) {
    IMAGD_CHECK_ARG(block_n == 0 || block_n == 64 || block_n == 128 || block_n == 160 || block_n == 256,
                    "debug_force: block_n %d", block_n);
    imagd::g_force_bn = block_n;
    imagd::g_force_stages = stages;
    imagd::g_force_splits = splits;
    return IMAGD_OK;
}

int imagd_gemm_debug_log(int enable, char* out, int out_bytes) {
    if (enable >= 0) {
        imagd::g_log_on = enable;
        if (enable) imagd::g_log.clear();
    }
    if (out && out_bytes > 0) {
        std::string all;
        for (const auto& k : imagd::g_log) all += k + "\n";
        IMAGD_CHECK_ARG(static_cast<int>(all.size()) < out_bytes, "debug_log: buffer too small (%d needed)",
                        static_cast<int>(all.size()) + 1);
        memcpy(out, all.c_str(), all.size() + 1);
    }
    return static_cast<int>(imagd::g_log.size());
}

int imagd_upconv3x3_bf16(const void* X, int64_t ldx, int NB, int H, int W, int Cin, const void* Wt, void* Y, int64_t ldy,
                         int Cout, const imagd_epilogue* ep, imagd_stream stream) {
    IMAGD_CHECK_ARG(NB > 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0 && Cin % 64 == 0, "upconv3x3: bad shape");
    IMAGD_CHECK_ARG(!ep || (!ep->rowvec && !ep->residual && ep->act == IMAGD_ACT_NONE && !ep->out_fp32 &&
                            !ep->row_stats_out && !ep->row_stats_in),
                    "upconv3x3: bias-only epilogue");
    return imagd::run_gemm_like(X, ldx, NB, H, W, Cin, 4, Wt, static_cast<int64_t>(4) * Cin, Y, ldy, Cout, ep,
                                static_cast<cudaStream_t>(stream), true);
}

int imagd_gemm_tile_count_n(int M, int N, int K) {
    using namespace imagd;
    IMAGD_CHECK_ARG(M > 0 && N > 0 && K > 0, "tile_count_n: bad shape");
    int bw = 1, bh = 1, bn = 1;
    choose_pixel_box(M, 1, 1, &bw, &bh, &bn);
    const int m_tiles = ((M + bw - 1) / bw);
    GemmCfg cfg = choose_cfg(m_tiles, N, (K + kBlockK - 1) / kBlockK, false);
    if (g_force_bn) cfg.bn = g_force_bn;
    return (N + cfg.bn - 1) / cfg.bn;
}

int imagd_gemm_debug_timeline(void* device_buf) {
    imagd::g_dbg_timeline = static_cast<unsigned long long*>(device_buf);
    return IMAGD_OK;
}

int imagd_conv3x3_bf16(const void* X, int64_t ldx, int NB, int H, int W, int Cin, const void* Wt, void* Y, int64_t ldy,
                       int Cout, const imagd_epilogue* ep, imagd_stream stream) {
    IMAGD_CHECK_ARG(NB > 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0, "conv3x3: bad shape");
    return imagd::run_gemm_like(X, ldx, NB, H, W, Cin, 9, Wt, static_cast<int64_t>(9) * Cin, Y, ldy, Cout, ep,
                                static_cast<cudaStream_t>(stream));
}

}  // extern "C"
