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
// A / B tiles (then the residual tile), two warpgroups accumulate 64 rows each with wgmma in registers and apply the
// epilogue (bias / time-embedding row vector / activation / residual) to their own fragments; the bf16 tile leaves by
// TMA stores. One CTA runs per SM (288 threads, 96-200 KB of shared memory).
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
    int res_tma;      // 1: the residual is read through tmR (any epilogue but GEGLU)
    int store_tma;    // 1: the bf16 output is written through tmD (all but fp32 outputs and the upsample-phase conv)
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
// The bf16 residual (in) and the bf16 output (out) tiles pass through shared memory in chunks of 32 columns x 128 rows:
// TMA boxes of (32 channels, bw, bh, bn) pixels, 64-byte rows in the 64-byte swizzle (conflict-free fragment-order access)
constexpr int kEpiCols = 32;
constexpr int kEpiChunkBytes = kBlockM * kEpiCols * 2;  // 8 KB
constexpr int kRowGroups = 4;  // row-vector groups (samples) one tile may span with its row vector staged in shared memory

template <int BLOCK_N, int STAGES>
struct GemmSmem {
    static constexpr int kBBytes = BLOCK_N * kBlockK * 2;
    static constexpr int kStageBytes = kABytes + kBBytes;
    static constexpr int kRing = STAGES * kStageBytes;
    // epilogue chunk c lives in the ring stage that producer iteration nk + c / kChunksPerStage would fill
    static constexpr int kChunksPerStage = kStageBytes / kEpiChunkBytes;
    static_assert(BLOCK_N / kEpiCols <= STAGES * kChunksPerStage, "epilogue tile does not fit the ring");
    static constexpr int kBarOffset = kRing;
    // full[STAGES] | empty[STAGES] | residual | split-K flag
    static constexpr int kVecOffset = (kBarOffset + (2 * STAGES + 1) * 8 + 16 + 15) & ~15;
    // epilogue vectors staged once per CTA: bias[BLOCK_N] | row vector[kRowGroups][BLOCK_N] (LayerNorm consumer: column sums)
    static constexpr int kTotal = kVecOffset + (1 + kRowGroups) * BLOCK_N * 4;
};

// Byte offset of (tile row r, even chunk column cl) in an epilogue chunk: rows of 64 bytes, TMA SWIZZLE_64B (16-byte unit
// bits [4, 6) XOR address bits [7, 9)). The eight rows a warp touches per access land in eight distinct 16-byte units.
__device__ __forceinline__ int epi_offset(int r, int cl) { return r * 64 + ((cl * 2) ^ (((r >> 1) & 3) << 4)); }

// LINEAR = the epilogue has no activation and writes bf16 (every conv and most linears of the UNet); !LINEAR = the
// generic epilogue (SiLU / GELU / quick-GELU / GEGLU / fp32 output).
// LNM: LayerNorm folding (see include/imagd_b200.h): 0 off, 1 producer (emit per-row {sum, sum of squares} of the rounded
// outputs, one slot per N tile), 2 consumer (apply rstd * (alpha * acc - mean * colsum) + bias), 3 upsample-phase conv.
//
// CTA = 128 output pixels x BLOCK_N output channels, 288 threads:
//   warps 0-3  warpgroup 0: wgmma on accumulator rows 0-63, then the epilogue of those rows from registers
//   warps 4-7  warpgroup 1: the same for rows 64-127
//   warp 8     TMA producer (one elected lane; STAGES-deep smem ring, full / empty mbarriers; then the residual tile)
// The epilogue applies bias / row vector / activation / residual to the accumulator fragments, stages the bf16 tile over
// the idle ring and writes it with TMA tile stores (the tensor map clips ragged M / N edges). fp32 outputs and the
// upsample-phase conv store straight from the fragments.
template <int BLOCK_N, int STAGES, bool LINEAR, int LNM>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               const __grid_constant__ CUtensorMap tmR, const __grid_constant__ CUtensorMap tmD, const GemmParams p) {
    using L = GemmSmem<BLOCK_N, STAGES>;
    constexpr bool LN_PRODUCE = LNM == 1;
    constexpr bool LN_CONSUME = LNM == 2;
    // LNM == 3: nearest-2x upsample + 3x3 conv as four 2x2 "phase" convs on the LOW-resolution input (2.25x fewer MACs,
    // no upsampled tensor): blockIdx.y = phase * n_tiles + n_blk, phase = py * 2 + px; tap t = ty * 2 + tx reads input
    // pixel (y + py - 1 + ty, x + px - 1 + tx); the weight matrix is [4 * N, 4 * Cin] (phase-major rows, tap-major
    // columns); output pixel (2y + py, 2x + px) of a [NB, 2H, 2W, N] tensor.
    constexpr bool UPS = LNM == 3;
    constexpr int kResChunks = BLOCK_N / kEpiCols;
    static_assert(!LN_PRODUCE || LINEAR, "row statistics are emitted by the LINEAR epilogue only");
    static_assert(BLOCK_N % 64 == 0 || BLOCK_N == 160, "wgmma N tile");
    extern __shared__ __align__(1024) uint8_t smem[];  // SWIZZLE_128B tiles need 1024-byte alignment
    if (threadIdx.x == 0 && (smem_u32(smem) & 1023u) != 0) __trap();  // (no printf: see mbar_wait_quiet)
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::kBarOffset);
    uint64_t* empty_bar = full_bar + STAGES;
    uint64_t* res_bar = empty_bar + STAGES;
    uint32_t* flag_slot = reinterpret_cast<uint32_t*>(res_bar + 1);
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
    const int col_base = n_blk * BLOCK_N;
    auto epi_chunk = [&](int c) {
        return smem + ((nk + c / L::kChunksPerStage) % STAGES) * L::kStageBytes + (c % L::kChunksPerStage) * kEpiChunkBytes;
    };
    auto load_residual = [&]() {  // one elected thread; completes on res_bar
        mbar_arrive_expect_tx(res_bar, kResChunks * kEpiChunkBytes);
#pragma unroll 1
        for (int c = 0; c < kResChunks; ++c) tma_load_4d(epi_chunk(c), &tmR, res_bar, col_base + c * kEpiCols, x0, y0, n0);
    };

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        for (int i = 0; i < STAGES; ++i) {
            mbar_init(&full_bar[i], 1);
            mbar_init(&empty_bar[i], 2);  // one arrival per consumer warpgroup
        }
        mbar_init(res_bar, 1);
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
            // the residual tile goes to the stages of iterations nk, nk + 1, ...: free from the start when nk < STAGES,
            // otherwise as soon as the consumers release them at the end of the K loop. (Split-K: the last arriver loads it.)
            if (p.res_tma && p.splits == 1) {
                for (int c = 0; c < kResChunks; c += L::kChunksPerStage) {
                    const int v = nk + c / L::kChunksPerStage;
                    mbar_wait_quiet(&empty_bar[v % STAGES], ((v / STAGES) & 1) ^ 1);
                }
                load_residual();
            }
        }
        return;
    }

    const int wg = warp >> 2;  // consumer warpgroup: accumulator rows [64 wg, 64 wg + 64)
    const int ct = threadIdx.x;  // consumer thread 0..255
    const imagd_epilogue& ep = p.ep;
    // wgmma m64nN accumulator layout: warp w of the warpgroup holds rows 16 w + lane / 4 (+ 8), columns 8 j + 2 (lane % 4)
    // (+ 1); acc[4 j + 2 h + e] is (row frow + 8 h, column 8 j + 2 (lane % 4) + e)
    const int quad = lane & 3;
    const int frow = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    auto row_at = [&](int h, int64_t& pix) {  // output pixel of fragment row h; false outside the image
        const int r = frow + 8 * h;
        const int x = x0 + r % p.bw;
        const int y = y0 + (r / p.bw) % p.bh;
        const int n = n0 + r / (p.bw * p.bh);
        pix = UPS ? (static_cast<int64_t>(n) * (2 * p.H) + (2 * y + (ups_phase >> 1))) * (2 * p.W) + (2 * x + (ups_phase & 1))
                  : (static_cast<int64_t>(n) * p.H + y) * p.W + x;
        return (x < p.W) && (y < p.H) && (n < p.NB);
    };
    int64_t pix[2];
    bool row_ok[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) row_ok[h] = row_at(h, pix[h]);
    // ---- epilogue preparation (before the mainloop): stage the per-column vectors in shared memory. The row vector is
    // staged per row group (sample) when the tile spans at most kRowGroups of them; otherwise each row reads it from
    // global memory. Without a row vector the LINEAR epilogue adds the zeroed slot, as it always adds bias and row vector.
    const float* rowvec[2] = {s_rowvec, s_rowvec};
    float ln_mean[2] = {0.f, 0.f}, ln_rstd[2] = {0.f, 0.f};
    if (LN_CONSUME) {  // the row-vector slot carries the folded weight's column sums instead
        for (int c = ct; c < BLOCK_N; c += 256) s_rowvec[c] = (col_base + c < p.N) ? __ldg(ep.colsum + col_base + c) : 0.f;
    } else if (ep.rowvec != nullptr) {
        const int xl = min(x0 + p.bw, p.W) - 1, yl = min(y0 + p.bh, p.H) - 1, nl = min(n0 + p.bn, p.NB) - 1;
        const int64_t g_first = ((static_cast<int64_t>(n0) * p.H + y0) * p.W + x0) / ep.rows_per_group;
        const int64_t g_last = ((static_cast<int64_t>(nl) * p.H + yl) * p.W + xl) / ep.rows_per_group;
        const bool staged = g_last - g_first < kRowGroups;
        if (staged) {
            for (int i = ct; i < (g_last - g_first + 1) * BLOCK_N; i += 256) {
                const int c = i % BLOCK_N;
                s_rowvec[i] = (col_base + c < p.N) ? __ldg(ep.rowvec + (g_first + i / BLOCK_N) * ep.rowvec_ld + col_base + c)
                                                   : 0.f;
            }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int64_t g = pix[h] / ep.rows_per_group;
            if (row_ok[h]) rowvec[h] = staged ? s_rowvec + (g - g_first) * BLOCK_N : ep.rowvec + g * ep.rowvec_ld + col_base;
        }
    } else if (LINEAR) {
        for (int c = ct; c < BLOCK_N; c += 256) s_rowvec[c] = 0.f;
    }
    for (int c = ct; c < BLOCK_N; c += 256)
        s_bias[c] = (ep.bias != nullptr && col_base + c < p.N) ? __ldg(ep.bias + col_base + c) : 0.f;
    if constexpr (LN_CONSUME) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            if (row_ok[h]) {  // fixed-order fold of the producer's per-tile partials -> mean / rstd of the row of A
                const float2* sp = reinterpret_cast<const float2*>(ep.row_stats_in) + pix[h] * ep.stats_in_ld;
                float s1 = 0.f, s2 = 0.f;
                for (int i = 0; i < ep.stats_parts; ++i) {
                    const float2 t = __ldg(sp + i);
                    s1 += t.x;
                    s2 += t.y;
                }
                const float inv = 1.0f / static_cast<float>(ep.ln_dim);
                ln_mean[h] = s1 * inv;
                ln_rstd[h] = rsqrtf(fmaxf(fmaf(-ln_mean[h], ln_mean[h], s2 * inv), 0.f) + ep.ln_eps);
            }
        }
    }

    // ---- mainloop: each warpgroup multiplies its 64 rows of A by the whole B tile; the previous stage is released once
    // the MMAs that read it have retired (wait_group 1 keeps one group in flight)
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
    if (leader) mbar_arrive(&empty_bar[(nk - 1) % STAGES]);  // the residual tile may go to this stage
    // every MMA of the CTA has to retire before the ring is overwritten by the output tile
    asm volatile("bar.sync 1, 256;" ::: "memory");
    if (threadIdx.x == 0) dbg_mark(p, 3);
    if (p.pdl_late) pdl_launch_dependents();  // mainloop done: the next kernel's prologue may overlap this epilogue

    // ---- split-K rendezvous: partials in fragment order (float4 q of consumer thread ct at [q][ct]), the last arriver
    // sums them in split order
    if (p.splits > 1) {
        const int64_t tile_elems = static_cast<int64_t>(kBlockM) * BLOCK_N;
        const int64_t tile_id = static_cast<int64_t>(blockIdx.y) * gridDim.x + blockIdx.x;
        const int64_t n_tiles_total = static_cast<int64_t>(gridDim.x) * gridDim.y;
        float4* mine = reinterpret_cast<float4*>(p.ws + (static_cast<int64_t>(blockIdx.z) * n_tiles_total + tile_id) * tile_elems);
#pragma unroll
        for (int q = 0; q < BLOCK_N / 8; ++q)
            __stcg(mine + q * 256 + ct, make_float4(acc[4 * q], acc[4 * q + 1], acc[4 * q + 2], acc[4 * q + 3]));
        __threadfence();
        asm volatile("bar.sync 2, 256;" ::: "memory");
        if (ct == 0) {
            const unsigned int old = atomicAdd(&p.counters[tile_id], 1u);
            *flag_slot = (old == static_cast<unsigned int>(p.splits - 1)) ? 1u : 0u;
            if (old == static_cast<unsigned int>(p.splits - 1)) p.counters[tile_id] = 0u;  // re-arm for next launch
        }
        asm volatile("bar.sync 2, 256;" ::: "memory");
        const bool last = *reinterpret_cast<volatile uint32_t*>(flag_slot) != 0u;
        if (!last) {
            if (ct == 0) dbg_mark(p, 5);
            return;
        }
        __threadfence();
        if (p.res_tma && ct == 0) load_residual();  // the ring is idle: no stage to wait for
#pragma unroll
        for (int j = 0; j < BLOCK_N / 2; ++j) acc[j] = 0.f;
        for (int s = 0; s < p.splits; ++s) {
            const float4* src = reinterpret_cast<const float4*>(p.ws + (static_cast<int64_t>(s) * n_tiles_total + tile_id) * tile_elems);
#pragma unroll
            for (int q = 0; q < BLOCK_N / 8; ++q) {
                const float4 t = __ldcg(src + q * 256 + ct);
                acc[4 * q] += t.x; acc[4 * q + 1] += t.y; acc[4 * q + 2] += t.z; acc[4 * q + 3] += t.w;
            }
        }
    }
    if (p.res_tma) mbar_wait_quiet(res_bar, 0);
    if (threadIdx.x == 0) dbg_mark(p, 4);

    // ---- epilogue from registers. Per element, in this order: alpha * acc, + bias, + row vector, activation, + residual,
    // round. The LINEAR form always adds bias, row vector and residual (zeros when absent).
    const float alpha = ep.alpha;
    const bool geglu = !LINEAR && ep.act == IMAGD_ACT_GEGLU;
    const int n_out = geglu ? p.N / 2 : p.N;
    if (geglu) {
        // tile = [64 value | 64 gate] columns; output columns n_blk * 64 + [0, 64): value j and gate j + 8 are both mine
        if constexpr (BLOCK_N == 128) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int cl = 8 * j + 2 * quad;
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    float o[2];
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        float a = alpha * acc[4 * j + 2 * h + e], g = alpha * acc[4 * (j + 8) + 2 * h + e];
                        if constexpr (LN_CONSUME) {  // bias (folded) is mandatory here: s_bias always staged
                            a = fmaf(ln_rstd[h], fmaf(-ln_mean[h], s_rowvec[cl + e], a), s_bias[cl + e]);
                            g = fmaf(ln_rstd[h], fmaf(-ln_mean[h], s_rowvec[64 + cl + e], g), s_bias[64 + cl + e]);
                        } else if (ep.bias) {
                            a += s_bias[cl + e];
                            g += s_bias[64 + cl + e];
                        }
                        o[e] = a * gelu_erf(g);
                    }
                    const int r = frow + 8 * h;
                    *reinterpret_cast<uint32_t*>(epi_chunk(cl / kEpiCols) + epi_offset(r, cl % kEpiCols)) =
                        pack_bf16x2(o[0], o[1]);
                }
            }
        }
    } else {
        const bool add_bias = LINEAR || ep.bias != nullptr;
        const bool add_rowvec = LINEAR || ep.rowvec != nullptr;
        const bool add_res = LINEAR || p.res_tma;
        const int act = LINEAR ? IMAGD_ACT_NONE : ep.act;
        float st1[2] = {0.f, 0.f}, st2[2] = {0.f, 0.f};  // LayerNorm producer: my rows' statistics over this tile
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j) {
            const int cl = 8 * j + 2 * quad;  // tile-local column of element e = 0
            const bool col_ok = col_base + cl < p.N;  // (N % 8 == 0: both elements or neither)
            uint8_t* chunk = epi_chunk(cl / kEpiCols);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = frow + 8 * h;
                float f[2];
#pragma unroll
                for (int e = 0; e < 2; ++e) f[e] = alpha * acc[4 * j + 2 * h + e];
                if constexpr (LN_CONSUME) {
#pragma unroll
                    for (int e = 0; e < 2; ++e)
                        f[e] = fmaf(ln_rstd[h], fmaf(-ln_mean[h], s_rowvec[cl + e], f[e]), s_bias[cl + e]);
                } else {
                    if (add_bias) {
                        f[0] += s_bias[cl];
                        f[1] += s_bias[cl + 1];
                    }
                    if (add_rowvec) {
                        const float2 v = col_ok ? *reinterpret_cast<const float2*>(rowvec[h] + cl) : make_float2(0.f, 0.f);
                        f[0] += v.x;
                        f[1] += v.y;
                    }
                }
                if (act == IMAGD_ACT_SILU) {
                    f[0] = silu(f[0]);
                    f[1] = silu(f[1]);
                } else if (act == IMAGD_ACT_GELU) {
                    f[0] = gelu_erf(f[0]);
                    f[1] = gelu_erf(f[1]);
                } else if (act == IMAGD_ACT_QUICK_GELU) {  // x * sigmoid(1.702 x): CLIP text MLP (quick_gelu)
                    f[0] = __fdividef(f[0], 1.0f + __expf(-1.702f * f[0]));
                    f[1] = __fdividef(f[1], 1.0f + __expf(-1.702f * f[1]));
                }
                uint32_t* slot = reinterpret_cast<uint32_t*>(chunk + epi_offset(r, cl % kEpiCols));
                if (add_res) {  // the residual tile is staged where the output goes (zeros beyond N)
                    const uint32_t rv = p.res_tma ? *slot : 0u;
                    f[0] += bf16lo(rv);
                    f[1] += bf16hi(rv);
                }
                if (!LINEAR && ep.out_fp32) {
                    if (row_ok[h] && col_ok)
                        *reinterpret_cast<float2*>(reinterpret_cast<float*>(p.out) + pix[h] * p.ldd + col_base + cl) =
                            make_float2(f[0], f[1]);
                    continue;
                }
                const uint32_t o = pack_bf16x2(f[0], f[1]);
                if constexpr (LN_PRODUCE) {  // statistics of what the consumer will READ: the rounded values
                    if (col_ok) {
                        const float lo = bf16lo(o), hi = bf16hi(o);
                        st1[h] += lo + hi;
                        st2[h] = fmaf(lo, lo, fmaf(hi, hi, st2[h]));
                    }
                }
                if constexpr (UPS) {
                    if (row_ok[h] && col_ok)
                        *reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(p.out) + pix[h] * p.ldd + col_base + cl) = o;
                } else {
                    *slot = o;
                }
            }
        }
        if constexpr (LN_PRODUCE) {  // the quad holds the row's columns: reduce, one write per row and N tile
#pragma unroll
            for (int h = 0; h < 2; ++h) {
#pragma unroll
                for (int m = 1; m < 4; m <<= 1) {
                    st1[h] += __shfl_xor_sync(0xffffffffu, st1[h], m);
                    st2[h] += __shfl_xor_sync(0xffffffffu, st2[h], m);
                }
                int64_t px;  // (recomputed: keeping the pixel index live through the loop costs registers at BLOCK_N 256)
                if (quad == 0 && row_at(h, px))
                    reinterpret_cast<float2*>(ep.row_stats_out)[px * ep.stats_ld + n_blk] = make_float2(st1[h], st2[h]);
            }
        }
    }
    if (p.store_tma) {
        fence_proxy_async_smem();  // generic-proxy writes -> async-proxy reads
        asm volatile("bar.sync 1, 256;" ::: "memory");
        if (ct == 0) {
            const int oc0 = geglu ? n_blk * 64 : col_base;
            const int chunks = geglu ? 64 / kEpiCols : BLOCK_N / kEpiCols;
            for (int c = 0; c < chunks && oc0 + c * kEpiCols < n_out; ++c)
                tma_store_4d(&tmD, epi_chunk(c), oc0 + c * kEpiCols, x0, y0, n0);
            bulk_commit();
            bulk_wait_read0();  // the staged tile must stay valid until the copy engine has read it
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
// variant runs one CTA per SM (the register file allows no second one); the shared-memory footprint is the ring plus the
// epilogue vectors (about 96-200 KB): the residual / output tiles of the epilogue reuse the ring.
//
// Measured on an H100 80GB HBM3 (SXM, 400 W power limit, 1980 MHz max SM clock) with tools/gemm_bench.py over the 92
// launch keys of a denoising step at batch 1 and 8, every variant timed in isolation:
//   - the deep ring is faster than the shallow one for nearly every key, one wave or many;
//   - a CTA spends about a constant time per k-block that grows with the operand bytes of the k-block (16 KB of A plus
//     BN x 128 B of B), roughly 75 GB/s per SM: 0.32 / 0.45 / 0.50 / 0.65 us for BN = 64 / 128 / 160 / 256;
//   - the chip-wide rate is not the limit: variants reach 6.6-7.8 TB/s of modelled L2 -> shared-memory operand
//     traffic, and the slow launches of the old rule (~4-5 TB/s) lost their time to partly filled last waves.
// So the rule minimises  waves x (t_wave(BN) + k-blocks per CTA x t_kb(BN)) + t_split x (MB of split-K partials)  with
// waves = ceil(CTAs / 132), t_kb / t_wave (prologue + epilogue) fitted by least squares to those timings. With it the
// step's GEMM + conv launches take 4.6 ms instead of 6.2 ms at batch 1 and 28.4 ms instead of 32.7 ms at batch 8
// (sum of the isolated launch times, same card). The constants were fitted with the earlier epilogue, which staged the
// fp32 accumulator tile through shared memory; the register epilogue lowers t_wave, and they have not been re-fitted.
struct GemmCfg {
    int bn, stages, splits;
};

static int shallow_stages(int bn) { return bn == 64 ? 4 : (bn == 256 ? 2 : 3); }
static int deep_stages(int bn) { return bn == 64 ? 8 : (bn == 128 ? 6 : (bn == 160 ? 5 : 4)); }

static GemmCfg choose_cfg(int m_tiles, int N, int kb_total, bool geglu, bool allow_split) {
    constexpr int kBn[4] = {64, 128, 160, 256};
    constexpr double kWaveUs[4] = {3.76, 5.31, 7.34, 10.18};  // per wave: prologue, pipeline fill, epilogue
    constexpr double kKbUs[4] = {0.324, 0.454, 0.496, 0.648};  // per k-block of one CTA, deep ring
    constexpr double kSplitUsPerMB = 1.94;                     // fp32 partials written and reduced
    GemmCfg best{128, deep_stages(128), 1};
    double best_us = 1e30;
    for (int i = 0; i < 4; ++i) {
        const int bn = kBn[i];
        if (geglu && bn != 128) continue;  // the GEGLU epilogue pairs the value / gate halves of a 128-wide tile
        const int64_t tiles = static_cast<int64_t>(m_tiles) * ((N + bn - 1) / bn);
        for (int splits = 1; splits <= 6; ++splits) {
            // split-K for long K only (>= 30 k-blocks per split) and within the scratch (kWsBytes, kMaxTilesSplit)
            if (splits > 1 && (!allow_split || kb_total / splits < 30 || tiles > kMaxTilesSplit ||
                               static_cast<size_t>(tiles * splits) * 128 * bn * 4 > kWsBytes))
                continue;
            const int64_t waves = (tiles * splits + kNumSms - 1) / kNumSms;
            const int kb = (kb_total + splits - 1) / splits;
            const double part_mb = splits > 1 ? static_cast<double>(tiles * splits) * 128 * bn * 4 / 1e6 : 0.0;
            const double us = static_cast<double>(waves) * (kWaveUs[i] + kb * kKbUs[i]) + kSplitUsPerMB * part_mb;
            if (us < best_us) {
                best_us = us;
                best = {bn, deep_stages(bn), splits};
            }
        }
    }
    return best;
}

template <int BLOCK_N, int STAGES, bool LINEAR, int LNM = 0>
static int launch_gemm_impl(const CUtensorMap (&tm)[4], const GemmParams& p, int m_tiles, cudaStream_t stream) {
    using L = GemmSmem<BLOCK_N, STAGES>;
    constexpr int kSmem = L::kTotal;
    IMAGD_SET_MAX_SMEM((gemm_tc_kernel<BLOCK_N, STAGES, LINEAR, LNM>), kSmem);
    const int n_tiles = (p.N + BLOCK_N - 1) / BLOCK_N;
    dim3 grid(m_tiles, LNM == 3 ? 4 * n_tiles : n_tiles, p.splits);
    IMAGD_CUDA(launch_pdl(gemm_tc_kernel<BLOCK_N, STAGES, LINEAR, LNM>, grid, dim3(kGemmThreads), kSmem, stream, tm[0], tm[1],
                          tm[2], tm[3], p));
    return IMAGD_OK;
}

// tm = {A, B, residual, output}
template <int BLOCK_N, int STAGES>
static int launch_gemm(const CUtensorMap (&tm)[4], const GemmParams& p, int m_tiles, cudaStream_t stream) {
    const bool linear = p.ep.act == IMAGD_ACT_NONE && !p.ep.out_fp32;
    if (p.ups_n_tiles > 0) {  // upsample-phase conv: plain bf16 epilogue (bias only), validated by the caller
        GemmParams q = p;
        q.ups_n_tiles = (p.N + BLOCK_N - 1) / BLOCK_N;
        return launch_gemm_impl<BLOCK_N, STAGES, true, 3>(tm, q, m_tiles, stream);
    }
    if (p.ep.row_stats_out != nullptr) return launch_gemm_impl<BLOCK_N, STAGES, true, 1>(tm, p, m_tiles, stream);
    if (p.ep.row_stats_in != nullptr) {
        if (linear) return launch_gemm_impl<BLOCK_N, STAGES, true, 2>(tm, p, m_tiles, stream);
        if constexpr (BLOCK_N == 128) return launch_gemm_impl<BLOCK_N, STAGES, false, 2>(tm, p, m_tiles, stream);
        set_error("gemm: LayerNorm-folded generic epilogue exists for the GEGLU tile (128) only");
        return IMAGD_ERR_ARG;
    }
    if (linear) return launch_gemm_impl<BLOCK_N, STAGES, true>(tm, p, m_tiles, stream);
    return launch_gemm_impl<BLOCK_N, STAGES, false>(tm, p, m_tiles, stream);
}


static int g_force_bn = 0, g_force_stages = 0, g_force_splits = 0;  // test hooks (imagd_gemm_debug_force)
static int g_log_on = 0;
static unsigned long long* g_dbg_timeline = nullptr;  // imagd_gemm_debug_timeline
static std::vector<std::pair<std::string, int>> g_log;  // unique keys seen while logging, launch counts (tools/gemm_bench.py)

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
    IMAGD_CHECK_ARG(!geglu || (!ep.rowvec && !ep.residual && !ep.out_fp32),
                    "gemm: the GEGLU epilogue takes bias and alpha only (no row vector, residual or fp32 output)");
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

    GemmCfg cfg = choose_cfg(m_tiles, N, kb_total, geglu, !ups_mode);
    if (g_force_bn) {
        cfg.bn = geglu ? 128 : g_force_bn;
        cfg.stages = g_force_stages ? g_force_stages : shallow_stages(cfg.bn);
        if (cfg.stages != shallow_stages(cfg.bn) && cfg.stages != deep_stages(cfg.bn)) cfg.stages = shallow_stages(cfg.bn);
    }
    if (g_force_splits && !geglu) cfg.splits = std::min(g_force_splits, kb_total);
    IMAGD_CHECK_ARG(!ep.row_stats_out || ep.stats_ld >= (N + cfg.bn - 1) / cfg.bn,
                    "gemm: stats_ld=%lld is smaller than the %d N tiles of this launch (imagd_gemm_tile_count_n)",
                    (long long)ep.stats_ld, (N + cfg.bn - 1) / cfg.bn);
    if (ups_mode) cfg.splits = 1;  // (the split-K scratch is sized for one phase)
    p.ups_n_tiles = ups_mode ? 1 : 0;  // the launcher fills in the real tile count
    p.pdl_late = pdl_mode() == 2 ? 1 : 0;
    p.splits = cfg.splits;
    p.kb_per_split = (kb_total + cfg.splits - 1) / cfg.splits;
    p.splits = (kb_total + p.kb_per_split - 1) / p.kb_per_split;  // no empty splits
    if (g_log_on) {  // problem key | the configuration this launch runs
        char key[192];
        snprintf(key, sizeof(key), "%d %d %d %d %d %d %d %d %d %d | %d %d %d", taps, NB, H, W, Cin, N, geglu ? 1 : 0,
                 m_tiles, kb_total, ep.out_fp32, cfg.bn, cfg.stages, p.splits);
        auto it = std::find_if(g_log.begin(), g_log.end(), [&](const auto& e) { return e.first == key; });
        if (it == g_log.end()) g_log.emplace_back(key, 1);
        else ++it->second;
    }
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
    CUtensorMap tm[4];  // A, B, residual, output
    {
        uint64_t dims[4] = {static_cast<uint64_t>(Cin), static_cast<uint64_t>(W), static_cast<uint64_t>(H),
                            static_cast<uint64_t>(NB)};
        uint64_t strides[3] = {static_cast<uint64_t>(lda) * 2, static_cast<uint64_t>(lda) * 2 * W,
                               static_cast<uint64_t>(lda) * 2 * W * H};
        uint32_t box[4] = {kBlockK, static_cast<uint32_t>(p.bw), static_cast<uint32_t>(p.bh), static_cast<uint32_t>(p.bn)};
        int rc = make_tmap_bf16(&tm[0], A, 4, dims, strides, box);
        if (rc != IMAGD_OK) return rc;
    }
    {
        uint64_t dims[2] = {static_cast<uint64_t>(taps) * Cin, static_cast<uint64_t>(N) * (ups_mode ? 4 : 1)};
        uint64_t strides[1] = {static_cast<uint64_t>(ldw) * 2};
        uint32_t box[2] = {kBlockK, static_cast<uint32_t>(cfg.bn)};
        int rc = make_tmap_bf16(&tm[1], Wt, 2, dims, strides, box);
        if (rc != IMAGD_OK) return rc;
    }
    // residual and output: the same (c, x, y, n) pixel geometry with the logical column count, in 32-column boxes; the
    // extents clip ragged tiles, so a launch writing a column slice of a wider buffer leaves the other columns alone
    auto pixel_map = [&](CUtensorMap* m, const void* base, int64_t ld, int cols) {
        uint64_t dims[4] = {static_cast<uint64_t>(cols), static_cast<uint64_t>(W), static_cast<uint64_t>(H),
                            static_cast<uint64_t>(NB)};
        uint64_t strides[3] = {static_cast<uint64_t>(ld) * 2, static_cast<uint64_t>(ld) * 2 * W,
                               static_cast<uint64_t>(ld) * 2 * W * H};
        uint32_t box[4] = {kEpiCols, static_cast<uint32_t>(p.bw), static_cast<uint32_t>(p.bh), static_cast<uint32_t>(p.bn)};
        return make_tmap_bf16(m, base, 4, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_64B);
    };
    p.res_tma = ep.residual != nullptr && !geglu;
    p.store_tma = !ep.out_fp32 && !ups_mode;
    tm[2] = tm[3] = tm[0];
    if (p.res_tma) {
        int rc = pixel_map(&tm[2], ep.residual, ep.ldr, N);
        if (rc != IMAGD_OK) return rc;
    }
    if (p.store_tma) {
        int rc = pixel_map(&tm[3], D, ldd, geglu ? N / 2 : N);
        if (rc != IMAGD_OK) return rc;
    }
    switch (cfg.bn * 100 + cfg.stages) {
        case 6404: return launch_gemm<64, 4>(tm, p, m_tiles, stream);
        case 6408: return launch_gemm<64, 8>(tm, p, m_tiles, stream);
        case 12803: return launch_gemm<128, 3>(tm, p, m_tiles, stream);
        case 12806: return launch_gemm<128, 6>(tm, p, m_tiles, stream);
        case 16003: return launch_gemm<160, 3>(tm, p, m_tiles, stream);
        case 16005: return launch_gemm<160, 5>(tm, p, m_tiles, stream);
        case 25602: return launch_gemm<256, 2>(tm, p, m_tiles, stream);
        case 25604: return launch_gemm<256, 4>(tm, p, m_tiles, stream);
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
        for (const auto& k : imagd::g_log) all += k.first + " | " + std::to_string(k.second) + "\n";
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
    GemmCfg cfg = choose_cfg(m_tiles, N, (K + kBlockK - 1) / kBlockK, false, true);
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
