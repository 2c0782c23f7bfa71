/*
 * imagd_b200.h — C ABI of libimagd_b200.so: the sm_90a kernels behind the IMAGDressing-v1 denoising hot path.
 *
 * Boundary contract (SURVEY.md §8b, "C-ABI extension"): plain pointers + sizes, no torch types; the caller
 * owns every buffer (kernels never allocate), every launch goes to the caller's stream (so the whole step is
 * CUDA-graph capturable), every entry point returns 0 or a negative imagd_status and records a message that
 * imagd_last_error() returns.  All activations are bf16, token-major ("NHWC" / [rows, channels]) with an explicit
 * row stride `ld*` in ELEMENTS; weights are bf16 [out_features, in_features] (torch nn.Linear layout; 3x3 conv
 * weights repacked tap-major to [Cout, 3*3*Cin]); biases / norm affine / time-embedding vectors are fp32.
 *
 * Each entry point cites the reference code (relative to /root/reference) whose arithmetic it replaces.
 * "diffusers-0.24" marks third-party code the reference calls (SURVEY.md §2a, Appendix A).
 */
#ifndef IMAGD_B200_H
#define IMAGD_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* imagd_stream; /* cudaStream_t */

enum imagd_status {
    IMAGD_OK = 0,
    IMAGD_ERR_ARG = -1,  /* bad shape / alignment / null pointer */
    IMAGD_ERR_CUDA = -2, /* CUDA runtime / driver error */
    IMAGD_ERR_ARCH = -3  /* device is not sm_90 */
};

enum imagd_act { IMAGD_ACT_NONE = 0, IMAGD_ACT_GEGLU = 1, IMAGD_ACT_SILU = 2, IMAGD_ACT_GELU = 3,
                 IMAGD_ACT_QUICK_GELU = 4 /* x * sigmoid(1.702 x): the CLIP text encoder's MLP */,
                 IMAGD_ACT_RELU = 5 /* max(x, 0): T2I-Adapter AdapterResnetBlock */ };

/* ---- library ---- */
int imagd_version(void);
const char* imagd_last_error(void);
/* Returns 90 on an H100 (cc 9.0); IMAGD_ERR_ARCH on anything else; IMAGD_ERR_CUDA with no device. */
int imagd_device_check(void);

/* ---- fused GEMM / conv epilogue ----
 * out[r, c] = act( alpha * acc[r, c] + bias[c] + rowvec[r / rows_per_group, c] ) + residual[r, c]
 * IMAGD_ACT_GEGLU: the packed weight interleaves, per 128 output rows, 64 "value" rows then their 64 "gate"
 * rows; out has N/2 columns: value * gelu_erf(gate)   (diffusers-0.24 GEGLU in BasicTransformerBlock.ff). It takes
 * bias and alpha only: a row vector, a residual or an fp32 output is rejected (IMAGD_ERR_ARG). */
typedef struct imagd_epilogue {
    const float* bias;     /* [N] or NULL */
    const float* rowvec;   /* [groups, rowvec_ld] or NULL (ResnetBlock2D time-embedding add) */
    int64_t rowvec_ld;
    int32_t rows_per_group; /* rows (pixels) per sample */
    int32_t act;            /* enum imagd_act */
    const void* residual;   /* bf16 [M, ldr] or NULL */
    int64_t ldr;
    float alpha;            /* 1.0f for plain */
    int32_t out_fp32;       /* 0: bf16 output, 1: fp32 output */
    /* ---- LayerNorm folding (r2-prep; DESIGN.md section 8 item 1). The GEMM that WRITES the residual stream emits, per
     * output row and per N tile of that launch, {sum, sum of squares} of its bf16-rounded outputs (producer); the GEMM
     * that follows the LayerNorm reads the raw stream and applies  rstd * (alpha * acc - mean * colsum[c]) + bias[c]
     * (consumer), with W' = W * diag(gamma) as its weight, colsum[c] = sum_k W'[c, k] and bias = b + W beta. */
    float* row_stats_out;       /* producer: [M, stats_ld] float2 (slot = N-tile index); NULL = off. act NONE, bf16 out only */
    int64_t stats_ld;           /* in float2 units, >= imagd_gemm_tile_count_n(...) of the producing launch */
    const float* row_stats_in;  /* consumer: [M, stats_in_ld] float2 partials of the A operand's rows; NULL = off */
    int64_t stats_in_ld;
    int32_t stats_parts;        /* partials per row to add up (the producer's N-tile count) */
    int32_t ln_dim;             /* C of the folded LayerNorm (= K of this GEMM) */
    float ln_eps;
    const float* colsum;        /* consumer: [N] fp32 */
    /* ---- per-step scale (the ControlNet zero convs of a multi-ControlNet step). When scale_table is non-NULL the kernel
     * reads s = scale_table[scale_step[0] * scale_ld] on the device (row 0 when scale_step is NULL) and computes
     *   out[r, c] = s * acc[r, c] + s * bias[c] + residual[r, c]
     * with s * bias[c] rounded to fp32 on its own; alpha is ignored. For the same s this is bitwise the launch with
     * alpha = s and bias = fp32(s * bias). A captured CUDA graph replays with whatever the table holds, and walks its
     * rows as the step counter advances. imagd_gemm_bf16 only, with a plain bf16 epilogue: an activation, a row vector,
     * a LayerNorm fold (either side), row statistics or an fp32 output is rejected, and so is a table passed to
     * imagd_conv3x3_bf16 / imagd_upconv3x3_bf16 (IMAGD_ERR_ARG). Zero-initialise all three when unused. */
    const float* scale_table;   /* fp32, 4-byte aligned; column k of an [S, K] table: base + k, scale_ld = K */
    const int32_t* scale_step;  /* device step counter (the sampler's step_ptr) or NULL */
    int64_t scale_ld;           /* row stride in floats, > 0 */
} imagd_epilogue;

/* D[M,N] = A[M,K] * W[N,K]^T (+ epilogue).  wgmma tensor cores, TMA-fed, fp32 accumulation.
 * Replaces every nn.Linear / 1x1 conv on the path: attn.to_q/to_k/to_v/to_out, to_k_ref/to_v_ref
 * (adapter/attention_processor.py:568-615,598-601), to_k_ip/to_v_ip (:841-842), Transformer2DModel proj_in/out,
 * FeedForward (diffusers-0.24), Resampler linears (adapter/resampler.py:13-20,45-47,186-188).
 * K % 8 == 0, lda/ldw % 8 == 0, pointers 16-byte aligned.
 * Threading: every call only enqueues work on `stream`; it is safe from several host threads. One exception: problems
 * with few output tiles and a long K run as a deterministic split-K whose fp32 partials live in a library-owned,
 * per-device scratch (96 MB, allocated at the first such call - which therefore must not happen inside a stream
 * capture; run the call once eagerly first). Split-K launches of ONE device must be ordered on one stream. */
int imagd_gemm_bf16(const void* A, int64_t lda, const void* W, int64_t ldw, void* D, int64_t ldd, int M, int N,
                    int K, const imagd_epilogue* ep, imagd_stream stream);

/* Test / tuning hooks. debug_force: force the N tile (0 = automatic; 64 / 128 / 160 / 256), the TMA ring depth
 * (0 = the shallow two-CTAs-per-SM variant) and the split-K factor (0 = automatic) of the next imagd_gemm_bf16 /
 * imagd_conv3x3_bf16 calls, so the parity tests cover every kernel variant. debug_log: enable = 1 starts recording
 * the distinct launches issued ("taps NB H W Cin N geglu m_tiles kb_total out_fp32 | block_n stages splits | count"
 * per line: the problem, the configuration it ran with, how many times), 0 stops, -1 leaves the state; when `out` is
 * given the recorded lines are copied there. Returns the number of lines. */
int imagd_gemm_debug_force(int block_n, int stages, int splits);
/* r2-prep: Upsample2D (nearest 2x) + its 3x3 conv in one implicit GEMM over the LOW-resolution input: four 2x2 "phase"
 * convolutions (output pixel (2y+py, 2x+px) sees input rows {y+py-1, y+py} and columns {x+px-1, x+px}); Wt is the
 * phase weight matrix [4*Cout, 4*Cin]: row = phase*Cout + co (phase = py*2+px), column = tap*Cin + ci (tap = ty*2+tx),
 * value = sum of the 3x3 taps (ky, kx) that land on that input pixel. X: [NB,H,W,ldx] -> Y: [NB,2H,2W,ldy]. Bias only. */
int imagd_upconv3x3_bf16(const void* X, int64_t ldx, int NB, int H, int W, int Cin, const void* Wt, void* Y, int64_t ldy,
                         int Cout, const imagd_epilogue* ep, imagd_stream stream);
/* Number of N tiles imagd_gemm_bf16 will use for an [M, K] x [N, K]^T problem with a plain (LINEAR) epilogue - the
 * number of row-statistics partials a producer launch writes per row (depends on the table-driven tile choice). */
int imagd_gemm_tile_count_n(int M, int N, int K);
int imagd_gemm_debug_log(int enable, char* out, int out_bytes);
/* Profiling hook: while `device_buf` is non-NULL every GEMM/conv CTA writes 8 x u64 at device_buf[cta_linear * 8]:
 * clock64 at {kernel entry, prologue done, first operand tile landed, last MMA issued, accumulator ready, epilogue done},
 * then %globaltimer at entry and %smid. The caller sizes the buffer for the largest grid. NULL switches it off. */
int imagd_gemm_debug_timeline(void* device_buf);

/* Y[n,y,x,:] = sum_{ky,kx} X[n,y+ky-1,x+kx-1,:] * Wt[:, (ky*3+kx)*Cin : +Cin]^T  (stride 1, zero pad 1) as an
 * implicit GEMM on wgmma: the 9 shifted activation views are fetched by TMA with out-of-bounds zero fill.
 * Replaces ResnetBlock2D.conv1/conv2 and Upsample2D.conv (diffusers-0.24; SURVEY.md Appendix A.2).
 * Cin % 64 == 0.  X: [NB,H,W,ldx], Y: [NB,H,W,ldy]. */
int imagd_conv3x3_bf16(const void* X, int64_t ldx, int NB, int H, int W, int Cin, const void* Wt, void* Y,
                       int64_t ldy, int Cout, const imagd_epilogue* ep, imagd_stream stream);

/* ---- attention ----
 * One KV stream of the two-stream ("hybrid") attention.  k and v are [n_kv_samples * len, ld] bf16 with head h at
 * columns [h*head_dim, (h+1)*head_dim).  The stream applies to query samples [0, n_query_samples); later samples
 * skip it (the unconditional half of a CFG batch has no garment stream:
 * dressing_sd/pipelines/IMAGDressing_v1_pipeline.py:511-518, adapter/attention_processor.py:597). */
typedef struct imagd_kv_stream {
    const void* k;
    const void* v;
    int64_t ld;
    int32_t len;             /* keys per sample */
    int32_t sample_rows;     /* rows between consecutive samples in k / v (0: = len); > len lets a stream visit a
                                prefix or suffix window of a longer per-sample context (text vs IP tokens) */
    int32_t broadcast;       /* 1: one KV sample shared by all query samples (garment dressed on a batch) */
    int32_t n_query_samples; /* query samples [0, n) use this stream */
    float out_scale;         /* weight of this stream's softmax output */
} imagd_kv_stream;

/* out = s0.out_scale * softmax(q k0^T * sm_scale) v0 + s1.out_scale * softmax(q k1^T * sm_scale) v1
 * — two independent softmaxes sharing one Q tile (FlashAttention-style, S/O accumulators in registers).
 * Replaces the two F.scaled_dot_product_attention calls + scale-add of RefSAttnProcessor2_0
 * (adapter/attention_processor.py:589-612), the text+IP pair of LoRAIPAttnProcessor2_0 (:833-856), the single
 * SDPA of CAttnProcessor2_0 / CacheAttnProcessor2_0 (:80, :270), and PerceiverAttention's fp32 softmax
 * (adapter/resampler.py:71-74).  q: [B*Lq, q_ld], out: [B*Lq, out_ld].  head_dim in {40, 64, 80, 160}. s1 may be
 * NULL. */
int imagd_attention_bf16(const void* q, int64_t q_ld, void* out, int64_t out_ld, int B, int Lq, int heads,
                         int head_dim, const imagd_kv_stream* s0, const imagd_kv_stream* s1, float sm_scale,
                         imagd_stream stream);
/* The same with a causal mask on stream 0 (query i sees keys 0..i; s1 must be NULL): the CLIP text encoder's
 * self-attention (transformers CLIPTextModel, reference call sites inference_IMAGdressing.py:44-46,
 * IMAGDressing_v1_pipeline.py:396-405 encode_prompt). */
int imagd_attention_causal_bf16(const void* q, int64_t q_ld, void* out, int64_t out_ld, int B, int Lq, int heads,
                                int head_dim, const imagd_kv_stream* s0, float sm_scale, imagd_stream stream);
/* Test hook, as for the GEMM: the forward kernel of the next imagd_attention_bf16 / imagd_attention_causal_bf16 /
 * imagd_attention_train_fwd_bf16 calls (0 automatic, 1 mma.sync, 2 wgmma). A call the forced kernel cannot serve
 * (wgmma: head_dim 64 / 160 or causal) fails without launching; other values are rejected. */
int imagd_attention_debug_force(int kernel);

/* ---- normalisation ---- */
/* GroupNorm over [NB, HW, C] (token-major) with optional fused SiLU, one launch. When the launch fits the device as one
 * wave of CTA clusters, each cluster keeps a (sample, channel slice) in shared memory: x is read once and the partial
 * statistics meet in distributed shared memory. Larger launches run a chunked kernel whose CTAs rendezvous through the
 * workspace ws (imagd_groupnorm_ws_bytes; its first 4 KB are arrival counters that the caller zero-initialises ONCE, the
 * rest holds per-chunk partial sums; grid <= 2 CTAs per SM, so all are co-resident).
 * Replaces ResnetBlock2D.norm1/norm2 + nonlinearity, Transformer2DModel.norm, conv_norm_out (diffusers-0.24). */
int64_t imagd_groupnorm_ws_bytes(int NB, int HW, int C, int groups);
int imagd_groupnorm_bf16(const void* x, int64_t ldx, void* y, int64_t ldy, int NB, int HW, int C, int groups,
                         const float* gamma, const float* beta, float eps, int fuse_silu, void* ws,
                         imagd_stream stream);
/* The plan imagd_groupnorm_bf16 runs for a shape: out[5] = {kernel (1 chunked rendezvous, 2 cluster), cluster size,
 * channels per slice, dynamic shared memory per CTA, waves}. cluster_capacity: co-resident clusters per cluster size
 * 2 / 4 / 8 / 16 at one and at two CTAs per SM ({c2x1, c2x2, c4x1, c4x2, c8x1, c8x2, c16x1, c16x2}, 0 = size not
 * launchable), or NULL for the current device's (imagd_groupnorm_cluster_capacity). Host-only when the capacity is given. */
int imagd_groupnorm_plan(int NB, int HW, int C, int groups, const int* cluster_capacity, int* out);
int imagd_groupnorm_cluster_capacity(int* out);
/* Test / tuning hooks, as for the GEMM. debug_force: kernel (0 automatic, 1 rendezvous, 2 cluster), cluster size
 * (0 automatic) and channels per slice (0 automatic) of the next GroupNorm calls; a launch with no legal plan under the
 * forced values fails. debug_log: "NB HW C groups | kernel cluster slice smem waves | count" per distinct launch. */
int imagd_groupnorm_debug_force(int kernel, int cluster_size, int slice_channels);
int imagd_groupnorm_debug_log(int enable, char* out, int out_bytes);
/* LayerNorm over the last dim of [rows, C]; BasicTransformerBlock.norm1-3 (diffusers-0.24),
 * adapter/resampler.py:16,43-44,187. gamma/beta may be NULL. */
int imagd_layernorm_bf16(const void* x, int64_t ldx, void* y, int64_t ldy, int rows, int C, const float* gamma,
                         const float* beta, float eps, imagd_stream stream);

/* ---- data movement / small convs ---- */
/* out[:, :Ca] = a ; out[:, Ca:Ca+Cb] = b (+ res_b) ; also a += res_a when given — the up-block skip concat
 * (torch.cat([hidden, skip], 1), diffusers-0.24 unet_2d_blocks) with the ControlNet residual add folded in
 * (UNet2DConditionModel.forward down_block_additional_residuals). b may be NULL (plain add/copy). */
int imagd_concat_add_bf16(const void* a, int64_t lda, int Ca, const void* res_a, int64_t ld_ra, const void* b,
                          int64_t ldb, int Cb, const void* res_b, int64_t ld_rb, void* out, int64_t ldo,
                          int64_t rows, imagd_stream stream);
/* Nearest-neighbour 2x upsample of [NB,H,W,C] -> [NB,2H,2W,C] (Upsample2D, diffusers-0.24). */
int imagd_upsample2x_bf16(const void* x, void* y, int NB, int H, int W, int C, imagd_stream stream);
/* im2col for the stride-2 pad-1 3x3 Downsample2D conv: [NB,H,W,C] -> [NB*(H/2)*(W/2), 9*C] tap-major. */
int imagd_im2col3x3_s2_bf16(const void* x, void* col, int NB, int H, int W, int C, imagd_stream stream);
/* The same with a selectable leading pad: pad_lo = 1 is the UNet's Downsample2D (padding 1); pad_lo = 0 is the VAE
 * encoder's Downsample2D, which pads (0,1,0,1) — right / bottom only — and convolves with padding 0 (diffusers-0.24
 * Downsample2D with padding=0; AutoencoderKL encoder, reference call site IMAGDressing_v1_pipeline.py:457). */
int imagd_im2col3x3_s2_pad_bf16(const void* x, void* col, int NB, int H, int W, int C, int pad_lo, imagd_stream stream);
/* P[r, :] = softmax(scale * S[r, :]): fp32 scores [rows, lds] -> bf16 probabilities [rows, ldp]; cols % 4 == 0,
 * cols <= 16384. The softmax of the VAE mid-block attention (one head of width 512: AutoencoderKL, diffusers-0.24
 * Attention with upcast_softmax; reference call sites IMAGDressing_v1_pipeline.py:457,544), between two GEMMs. */
int imagd_softmax_rows(const float* s, int64_t lds, void* p, int64_t ldp, int64_t rows, int cols, float scale,
                       imagd_stream stream);
/* Direct (SIMT) 3x3 conv, pad 1, stride 1 or 2, for the thin ends of the network where a tensor-core tile would
 * be empty: conv_in (4->320), conv_out (320->4), ControlNet conditioning embedding (3->16->...->320).
 * x: bf16 [NB,H,W,Cin]; w: bf16 [Cout, 9*Cin] tap-major; bias fp32; act in {NONE, SILU}.
 * out_nchw_f32 != 0 writes fp32 NCHW (the latent layout of the pipeline API) instead of bf16 NHWC. */
int imagd_conv3x3_direct_bf16(const void* x, int NB, int H, int W, int Cin, const void* w, const float* bias,
                              void* y, int Cout, int stride, int act, int out_nchw_f32, const void* add_nhwc,
                              imagd_stream stream);
/* fp32 NCHW latents -> bf16 NHWC (channels zero-padded to Cpad). The output batch is NB * repeat (sample i reads
 * source i % NB): repeat = 2 builds the CFG-duplicated model input (torch.cat([latents] * 2),
 * dressing_sd/pipelines/IMAGDressing_v1_pipeline.py:483-485) in the same pass. */
int imagd_nchw_f32_to_nhwc_bf16(const float* x, void* y, int NB, int C, int H, int W, int Cpad, int repeat,
                                imagd_stream stream);
/* The same layout with every value multiplied by scale_table[step_ptr ? *step_ptr : 0]: the model-input scaling
 * x / sqrt(sigma_i^2 + 1) of the sigma-space samplers (EulerDiscreteScheduler.scale_model_input, diffusers-0.24),
 * read on the device so a captured step graph walks the table. */
int imagd_nchw_f32_to_nhwc_bf16_scaled(const float* x, void* y, int NB, int C, int H, int W, int Cpad, int repeat,
                                       const float* scale_table, const int32_t* step_ptr, imagd_stream stream);

/* ---- T2I-Adapter (diffusers-0.24 models/adapter.py T2IAdapter "full_adapter"; UNet2DConditionModel.forward
 * down_intrablock_additional_residuals) ---- */
/* fp32 NCHW image [NB, C, H, W] -> bf16 NHWC [NB, H/8, W/8, C*64] in torch.nn.PixelUnshuffle(8) channel order: output
 * channel c*64 + i*8 + j holds x[n, c, 8h+i, 8w+j]. H % 8 == W % 8 == 0. The input of the adapter's conv_in. */
int imagd_pixel_unshuffle8_bf16(const float* x, void* y, int NB, int C, int H, int W, imagd_stream stream);
/* 2x2 average pool, stride 2: [NB, H, W, C] -> [NB, H/2, W/2, C], summed in fp32, rounded once (AvgPool2d(2, 2,
 * ceil_mode=True) for even H and W; odd H or W is rejected). C % 8 == 0. AdapterBlock's downsample. */
int imagd_avgpool2x2_bf16(const void* x, void* y, int NB, int H, int W, int C, imagd_stream stream);
/* In place: x[s, r, :C] += scale[0] * f[s % n_src, r, :C] for s < NB, r < rows, in fp32 with one bf16 rounding.
 * x: [NB, rows] pixels of row stride ldx; f: contiguous [n_src, rows, C]. scale: device fp32 scalar, so a captured
 * step graph replays with a new adapter_conditioning_scale. C, ldx % 8 == 0, pointers 16-byte aligned. */
int imagd_scaled_add_bcast_bf16(void* x, int64_t ldx, const void* f, const float* scale, int NB, int n_src, int64_t rows,
                                int C, imagd_stream stream);

/* ---- CLIP encoder front ends (SURVEY.md 8f row 3; transformers CLIPTextModel / CLIPVisionModelWithProjection, reference
 * call sites inference_IMAGdressing.py:44-49, IMAGDressing_v1_pipeline.py:396-415) ---- */
/* out[r, :] = tok[ids[r], :] + pos[r % T, :]  (token + position embedding; ids int64, clamped to the vocabulary). */
int imagd_embed_tokens_bf16(const int64_t* ids, const void* tok, const void* pos, void* out, int rows, int T, int C, int vocab,
                            imagd_stream stream);
/* fp32 NCHW image -> bf16 patch rows [B*(H/patch)*(W/patch), Kpad], column = (c*patch + iy)*patch + ix, zero padded:
 * the A operand of the patch-embedding GEMM (a conv with kernel = stride = patch). */
int imagd_patchify_bf16(const float* x, void* out, int B, int H, int W, int patch, int Kpad, imagd_stream stream);
/* out[b*rows_per_sample + row, :] = vec for every sample (the ViT class-token row). */
int imagd_broadcast_row_bf16(const void* vec, void* out, int B, int64_t rows_per_sample, int row, int C, imagd_stream stream);

/* ---- time conditioning ---- */
/* Sinusoidal timestep embedding, flip_sin_to_cos=True, freq_shift=0: out[b] = [cos | sin] (dim/2 each), fp32.
 * t = timesteps[step_ptr ? *step_ptr : 0] broadcast to all NB rows when per_sample == 0. diffusers-0.24
 * get_timestep_embedding (SURVEY.md A.2). */
int imagd_timestep_embedding(const float* timesteps, const int32_t* step_ptr, float* out, int NB, int dim,
                             imagd_stream stream);
/* out[m, n] = act_out( sum_k act_in(x[m,k]) * W[n,k] + bias[n] ), fp32 activations, bf16 weights, for the
 * M <= 64 "one row per sample" linears: TimestepEmbedding.linear_1/2 and every ResnetBlock2D.time_emb_proj
 * (batched into one call by concatenating the weights). act: 0 none, 2 SiLU. */
int imagd_linear_small_m(const float* x, int64_t ldx, const void* W, int64_t ldw, const float* bias, float* out,
                         int64_t ldo, int M, int N, int K, int act_in, int act_out, imagd_stream stream);

/* ---- sampler ---- */
/* Classifier-free guidance + DDIM (eta = 0) step, optionally + the inpainting blend, in one pass over the
 * latents (dressing_sd/pipelines/IMAGDressing_v1_pipeline.py:521-532; DDIMScheduler.step, diffusers-0.24;
 * IMAGDressing_v1_pipeline_controlnet_inpainting.py:487-500).
 *   eps  = eps_uncond + g * (eps_cond - eps_uncond)
 *   x0   = (x - sqrt(1-a_t) eps) / sqrt(a_t) ;  x' = sqrt(a_p) x0 + sqrt(1-a_p) eps
 *   if mask: x' = (1-mask) * (sqrt(a_n) img + sqrt(1-a_n) noise) + mask * x'       (a_n: alpha-bar at t_{i+1})
 * coef: device array [n_steps, 4] = {sqrt(a_t), sqrt(1-a_t), sqrt(a_p), sqrt(1-a_p)}; blend_coef [n_steps, 2]
 * = {sqrt(a_n), sqrt(1-a_n)} (last row {1, 0}).  step_ptr points at TWO device int32: [0] the step index, read
 * on the device and incremented by the kernel (so one captured CUDA graph replays all steps), [1] a scratch
 * counter the caller zero-initialises once.  All tensors fp32 NCHW [NB,4,h,w];
 * mask is [NB,1,h,w]. */
int imagd_cfg_ddim_step(const float* eps_cond, const float* eps_uncond, float guidance, float* latents,
                        const float* coef, int32_t* step_ptr, const float* mask, const float* image_latents,
                        const float* noise, const float* blend_coef, int NB, int C, int HW,
                        imagd_stream stream);
/* Classifier-free guidance + one step of a multistep sampler (DPMSolverMultistepScheduler dpmsolver++ order 1/2,
 * EulerDiscreteScheduler, EulerAncestralDiscreteScheduler; diffusers-0.24), optionally + the inpainting blend.
 * coef: device array [n_steps, 6], row = {dx, de, cx, ce, ch, cz}; per element, with eps the CFG-combined output:
 *   D  = dx x + de eps                         (the data prediction of this step)
 *   x' = cx x + ce eps + ch H + cz z[step]     (H: history, the previous step's D; z: this step's noise)
 *   if history: H = D (after reading it)
 *   if mask: x' = (1-mask) * (blend[0] img + blend[1] noise) + mask * x'
 * history: fp32 [NB,C,h,w] or NULL; step_noise: fp32 [n_steps,NB,C,h,w] or NULL. A zero ch / cz skips reading its
 * operand. step_ptr and blend_coef as for imagd_cfg_ddim_step (the kernel advances the step counter). */
int imagd_cfg_sampler_step(const float* eps_cond, const float* eps_uncond, float guidance, float* latents,
                           float* history, const float* step_noise, const float* coef, int32_t* step_ptr,
                           const float* mask, const float* image_latents, const float* noise, const float* blend_coef,
                           int NB, int C, int HW, imagd_stream stream);
/* Classifier-free guidance + one predictor-corrector multistep step (UniPCMultistepScheduler bh1 / bh2, orders 1-3,
 * predict_x0; diffusers-0.24), optionally + the inpainting blend. bank: fp32 [4,NB,C,h,w], four caller-owned slots H[k]
 * (the host decides which slot holds the stash of the previous corrected sample and which the previous data
 * predictions). coef: device array [n_steps, 16], row = {dx, de, ax, am, a0..a3, bc, bm, b0..b3, w_m, w_c}; per
 * element, with eps the CFG-combined output:
 *   m  = dx x + de eps                          (this step's data prediction)
 *   c  = ax x + am m + sum_k a_k H[k]           (the corrected sample; ax = 1, the rest 0 without a corrector)
 *   x' = bc c + bm m + sum_k b_k H[k]           (the predictor)
 *   H[w_m] = m ; H[w_c] = c                     (slot indices 0..3 stored as floats, written after every read)
 *   if mask: x' = (1-mask) * (blend[0] img + blend[1] noise) + mask * x'    (c, the stash, is the pre-blend value)
 * A slot whose a_k and b_k are both zero is not read (an unwritten slot may hold NaN). step_ptr and blend_coef as for
 * imagd_cfg_ddim_step (the kernel advances the step counter). */
int imagd_cfg_sampler_pc_step(const float* eps_cond, const float* eps_uncond, float guidance, float* latents,
                              float* bank, const float* coef, int32_t* step_ptr, const float* mask,
                              const float* image_latents, const float* noise, const float* blend_coef, int NB, int C,
                              int HW, imagd_stream stream);

/* ================================================================================================================
 * Training step (SURVEY.md 8 row a13; reference train.py:255-281 SDModel.forward, :573-605 loss + backward, :386-398 AdamW).
 * The reference obtains every gradient from torch autograd over the diffusers modules; these entry points are the backward
 * kernels a torch.autograd.Function per operator calls (imagdressing_b200/autograd.py).
 * ================================================================================================================ */

/* Extra outputs of a training-mode attention forward. lse: [2, B, heads, lq_pad] fp32, the per-row log-sum-exp of each
 * stream in the log2 domain (m + log2 l); the caller pre-fills it with +inf (padding rows then give P = 0 in the backward);
 * lq_pad = a multiple of 128 >= Lq. out_s0 / out_s1: the un-weighted per-stream outputs softmax(q k_s^T) v_s, bf16
 * [B*Lq, ld_s] (needed for D_s = w_s rowsum(dO o O_s)); may be NULL when there is one stream (then D = rowsum(dO o out)). */
typedef struct imagd_attn_train {
    float* lse;
    void* out_s0;
    void* out_s1;
    int64_t ld_s;
    int32_t lq_pad;
} imagd_attn_train;

/* imagd_attention_bf16 + the imagd_attn_train outputs (adapter/attention_processor.py:589-612 under autograd). A second
 * stream must apply to every query sample (n_query_samples >= B), as the backward requires. */
int imagd_attention_train_fwd_bf16(const void* q, int64_t q_ld, void* out, int64_t out_ld, int B, int Lq, int heads,
                                   int head_dim, const imagd_kv_stream* s0, const imagd_kv_stream* s1, float sm_scale,
                                   const imagd_attn_train* aux, imagd_stream stream);
/* dsum[s, b, h, q] = w_s * sum_d d_out[b, q, h, d] * o_s[b, q, h, d]  (o1 NULL: one stream); padding rows are left as the
 * caller initialised them (0). */
int imagd_attention_bwd_prep(const void* d_out, int64_t do_ld, const void* o0, const void* o1, int64_t ld_s, float w0, float w1,
                             float* dsum, int B, int Lq, int heads, int head_dim, int lq_pad, imagd_stream stream);
/* Backward of the two-stream attention (recompute-S flash style, deterministic, no atomics):
 *   dq [B*Lq, dq_ld]           += over both streams   (NULL: skipped)
 *   dk_s / dv_s                 same layout as the stream's k / v (row stride dkv_s_ld, sample stride = the stream's
 *                               sample_rows or len)      (NULL pair: that stream's key / value gradients are skipped)
 * Every query sample must own its keys in both streams (no broadcast, n_query_samples >= B): the training layout
 * (train.py:266-268 keeps every cache row). */
int imagd_attention_bwd_bf16(const void* q, int64_t q_ld, const void* d_out, int64_t do_ld, int B, int Lq, int heads,
                             int head_dim, const imagd_kv_stream* s0, const imagd_kv_stream* s1, float sm_scale,
                             const float* lse, const float* dsum, int lq_pad, void* dq, int64_t dq_ld, void* dk0, void* dv0,
                             int64_t dkv0_ld, void* dk1, void* dv1, int64_t dkv1_ld, imagd_stream stream);

/* y[c, r] = x[r, c] (r < rows), 0 for rows <= r < rows_pad; y: [cols, ldy]. Builds the K-contiguous operands of the
 * dgrad / wgrad GEMMs (dX = dY W, dW = dY^T X) for imagd_gemm_bf16. */
int imagd_transpose_bf16(const void* x, int64_t ldx, void* y, int64_t ldy, int rows, int cols, int rows_pad,
                         imagd_stream stream);
/* 3x3 conv weight layouts: mode 0 packs [Cout, Cin, 3, 3] (diffusers) into tap-major [Cout, 9*Cin] (pack_conv3x3 of the
 * trainable garment UNet, every step); mode 1 is the inverse, applied to the packed weight gradient. */
int imagd_conv_weight_layout_bf16(const void* src, void* dst, int Cout, int Cin, int mode, imagd_stream stream);
/* Packed forward weight [Cout, 9*Cin] -> the conv data-gradient weight [Cin, 9*Cout]: dst[ci, 8 - tap, co] = src[co, tap, ci]
 * (dX = conv3x3 of dY with the taps reversed and the channel roles swapped). */
int imagd_conv_weight_flip_bf16(const void* src, void* dst, int Cout, int Cin, imagd_stream stream);
/* Transposed im2col of a stride-1 pad-1 3x3 conv input: out[tap*C + c, p] = x[n, y+ky-1, x+kx-1, c], p = (n*H + y)*W + x,
 * zero for p >= NB*H*W; out: [9*C, ldo]. The B operand of the conv weight-gradient GEMM dW[Cout, 9 Cin] = dY^T col^T. */
int imagd_im2col3x3_t_bf16(const void* x, void* out, int64_t ldo, int NB, int H, int W, int C, imagd_stream stream);
/* Adjoint of imagd_im2col3x3_s2_bf16: dcol [NB, H/2, W/2, 9*C] -> dx [NB, H, W, C]. */
int imagd_col2im3x3_s2_bf16(const void* dcol, void* dx, int NB, int H, int W, int C, imagd_stream stream);
/* Adjoint of imagd_upsample2x_bf16: dy [NB, 2H, 2W, C] -> dx [NB, H, W, C] (sum of each 2x2 block). */
int imagd_downsum2x_bf16(const void* dy, void* dx, int NB, int H, int W, int C, imagd_stream stream);
/* out[g, c] = sum over the rows of group g of x[r, c] (fp32; bias gradients: groups = 1; ResnetBlock2D time-embedding
 * gradients: one group per sample). out: fp32, or bf16 when out_bf16 != 0 (a parameter gradient in the parameter's dtype).
 * Fixed-order two-stage reduction; ws >= imagd_colreduce_ws_bytes. */
int64_t imagd_colreduce_ws_bytes(int rows_per_group, int groups, int C);
int imagd_colsum_bf16(const void* x, int64_t ldx, int rows_per_group, int groups, int C, void* out, int out_bf16, void* ws,
                      imagd_stream stream);
/* LayerNorm backward: dx, and (dgamma non-NULL) dgamma / dbeta [C] (fp32, or bf16 when out_bf16 != 0). rowstat: [rows, 2] fp32 scratch (mean, rstd). */
int imagd_layernorm_bwd_bf16(const void* x, int64_t ldx, const void* dy, int64_t lddy, void* dx, int64_t lddx, int rows, int C,
                             const float* gamma, float eps, void* dgamma, void* dbeta, int out_bf16, float* rowstat, void* ws,
                             imagd_stream stream);
/* imagd_groupnorm_bf16 that also writes {mean, rstd} of every (sample, group) to stats_out [NB, groups, 2] fp32 (may be NULL):
 * the training-mode forward; the backward reuses the statistics instead of recomputing them. */
int imagd_groupnorm_stats_bf16(const void* x, int64_t ldx, void* y, int64_t ldy, int NB, int HW, int C, int groups,
                               const float* gamma, const float* beta, float eps, int fuse_silu, void* ws, float* stats_out,
                               imagd_stream stream);
/* GroupNorm (+SiLU) backward over contiguous [NB, HW, C] given the forward statistics fwd_stats [NB, groups, 2]: dx, and
 * (dgamma non-NULL) dgamma / dbeta [C] (fp32, or bf16 when out_bf16 != 0). Three coalesced passes (per-chunk channel partials, fixed-order fold, apply). */
int64_t imagd_groupnorm_bwd_ws_bytes(int NB, int HW, int C, int groups);
int imagd_groupnorm_bwd_bf16(const void* x, const void* dy, void* dx, int NB, int HW, int C, int groups, const float* gamma,
                             const float* beta, const float* fwd_stats, int fuse_silu, void* dgamma, void* dbeta, int out_bf16,
                             void* ws, imagd_stream stream);
/* Elementwise activation (mode IMAGD_ACT_SILU / IMAGD_ACT_GELU): dy NULL: y = act(x); else y = dy * act'(x). */
int imagd_act_bf16(const void* x, const void* dy, void* y, int64_t n, int mode, imagd_stream stream);
/* GEGLU on an un-fused projection h = [value | gate], [M, 2F]: dout NULL: out [M, F] = value * gelu(gate);
 * else out [M, 2F] = [dout * gelu(gate) | dout * value * gelu'(gate)] (dout contiguous [M, F]). */
int imagd_geglu_bf16(const void* h, int64_t ldh, const void* dout, void* out, int64_t ldo, int64_t M, int F,
                     imagd_stream stream);
/* loss[0] = mean((pred - target)^2) (train.py:577) and grad = grad_scale * 2 (pred - target) / n, fp32; ws >= 2 KB. */
int imagd_mse_loss_grad(const float* pred, const float* target, float* grad, float* loss, int64_t n, float grad_scale, void* ws,
                        imagd_stream stream);
/* AdamW, decoupled weight decay (train.py:386-398), fp32 master weights + moments, bf16 gradient in, bf16 working copy out. */
int imagd_adamw_step(float* master, void* param, const void* grad, float* m, float* v, int64_t n, float lr, float beta1,
                     float beta2, float eps, float weight_decay, int step, float grad_scale, imagd_stream stream);
/* The same with the step-dependent scalars read from DEVICE memory: hyper = {lr, weight_decay, step (1-based, as float),
 * grad_scale}. A CUDA graph of the whole training step (forward, backward, update) then replays with a moving step count and
 * learning-rate schedule — the host only rewrites these four floats. */
int imagd_adamw_step_dev(float* master, void* param, const void* grad, float* m, float* v, int64_t n, float beta1, float beta2,
                         float eps, const float* hyper, imagd_stream stream);
/* Global-norm gradient clipping (the reference's DeepSpeed "gradient_clipping"): one deterministic pass over the flat bf16
 * gradient grad[0:n] writes state (4 doubles) = {norm, coef, finite, skipped}:
 *   norm = || hyper[3] * grad ||_2 (squares summed in fp64: no finite input overflows), coef = min(1, max_norm / (norm + 1e-6)),
 *   finite = 1 / 0, skipped += 1 when not finite; hyper[2] (the AdamW step count) += 1 only when finite.
 * ws: >= imagd_grad_norm_ws_bytes(n) bytes, 16-byte aligned, zeroed once by the caller (an arrival counter the kernel resets
 * itself, then per-block partials); reused by every call, so one captured CUDA graph replays it. */
int64_t imagd_grad_norm_ws_bytes(int64_t n);
int imagd_grad_norm_clip(const void* grad, int64_t n, float max_norm, float* hyper, double* state, void* ws, imagd_stream stream);
/* imagd_adamw_step_dev reading that state: finite == 0 leaves master, param, m and v untouched; otherwise the update runs
 * with gradient scale hyper[3] * (float)coef (coef == 1: bitwise the imagd_adamw_step_dev result). */
int imagd_adamw_step_clip(float* master, void* param, const void* grad, float* m, float* v, int64_t n, float beta1, float beta2,
                          float eps, const float* hyper, const double* clip_state, imagd_stream stream);

#ifdef __cplusplus
}
#endif
#endif /* IMAGD_B200_H */
