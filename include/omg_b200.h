/*
 * omg_b200 — C ABI of the H100-native (sm_90a) OMG denoising hot path.
 *
 * The reference (kongzhecn/OMG) is pure Python on diffusers and has no FFI of its own; the
 * "interface each entry point replaces" is therefore the torch / diffusers / xformers library call
 * the reference makes at the cited line.  Ownership: the caller owns every buffer; the library only
 * borrows raw device pointers for the duration of the call and keeps no state besides a per-process
 * error string.  Every function returns 0 on success, non-zero on failure (omg_last_error() gives
 * the message); nothing throws across the boundary.  All kernels are launched on the CUstream /
 * cudaStream_t handle passed as `stream` (void*), never synchronise the host, and are CUDA-graph
 * capturable.  fp16 storage, fp32 accumulation; omg_gemm (dtype = OMG_DTYPE_BF16), omg_groupnorm_bf16 and
 * omg_softmax_rows_bf16 also take bf16 storage (the VAE decoder's path).  Activations are channels-last:
 * (B, H, W, C) == (B, H*W tokens, C).
 */
#ifndef OMG_B200_H
#define OMG_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define OMG_MAX_A 4
#define OMG_MAX_SEGS 12

/* Strided channels-last view: element (b,h,w,c) lives at ptr + b*sb + h*sh + w*sw + c (in elements). */
typedef struct {
    const void* ptr;
    int32_t C, W, H, B;
    int64_t sw, sh, sb;
} omg_view4;

/* One K-segment of a (implicit) GEMM: A operand = view a[a_idx] shifted by (dx,dy) pixels (out-of-range
 * pixels read as zero = conv padding), channels [a_c0, a_c0+k_len); weight columns [b_k0, b_k0+k_len). */
typedef struct {
    int32_t a_idx, dx, dy, a_c0, k_len, b_k0;
    int32_t b_idx; /* 0: columns of w, 1: columns of w2 (e.g. the LoRA up-projection B, kept un-merged) */
} omg_seg;

/* Storage type of a descriptor's 16-bit operands (omg_gemm_desc.dtype). */
enum { OMG_DTYPE_F16 = 0, OMG_DTYPE_BF16 = 1 };

enum { OMG_EPI_NONE = 0, OMG_EPI_GEGLU = 1, OMG_EPI_SILU = 2, OMG_EPI_QUICK_GELU = 3, OMG_EPI_GELU = 4, OMG_EPI_GELU_TANH = 5,
       OMG_EPI_RELU = 6 };

/*
 * out[pix, n] = epi( sum_seg sum_k A_seg[pix+(dx,dy), k] * W[n, b_k0+k] + bias[n] + rowvec[b, n] ) + residual[pix, n]
 *
 * Replaces: torch.nn.Linear / Conv2d(3x3 | 1x1, stride 1 | 2) / peft LoRA delta / GEGLU inside
 * diffusers UNet2DConditionModel.forward, reference call sites src/pipelines/lora_pipeline.py:546-566,592-599
 * (cuBLAS / cuDNN in the reference).  wgmma tensor cores, TMA-staged operands.
 * OMG_EPI_GEGLU: W rows (and bias) are interleaved (value_j, gate_j) pairs; out has N/2 channels,
 * out_j = value_j * gelu_erf(gate_j).   OMG_EPI_SILU: epi(x) = x * sigmoid(x) (time-embedding MLPs).
 * OMG_EPI_QUICK_GELU: x * sigmoid(1.702 x), OMG_EPI_GELU: erf-gelu (the fc1 activations of the two CLIP text towers,
 * transformers CLIPMLP [3P], reached from src/pipelines/lora_pipeline.py:315-347).  OMG_EPI_RELU: max(x, 0) (the MLP,
 * hypernetwork and IoU-head layers of the SAM mask decoder, segment_anything MaskDecoder / TwoWayTransformer [3P]).
 */
typedef struct {
    omg_view4 a[OMG_MAX_A];
    int32_t n_a;
    omg_seg segs[OMG_MAX_SEGS];
    int32_t n_segs;
    const void* w;      /* [N, Ktot] row-major fp16 */
    int32_t N, Ktot;
    const void* w2;     /* optional second weight matrix [N, K2tot] (segments with b_idx == 1) or NULL */
    int32_t K2tot;
    omg_view4 d;        /* output view; d.W/H/B define the pixel grid the tiles walk */
    const void* bias;   /* [N] fp16 or NULL */
    const void* rowvec; /* [B, rowvec_ld] fp16 or NULL: per-image additive vector (time-embedding projection) */
    int32_t rowvec_ld;
    const void* residual; /* contiguous [B*H*W, residual_ld] fp16 or NULL, added after the epilogue */
    int32_t residual_ld;
    int32_t epilogue;
    int32_t block_n;    /* 0 = auto; else 64 | 128 | 160 | 256 | 320 */
    /* LayerNorm folded into a GEMM pair (BasicTransformerBlock norm1/2/3 [3P] followed by to_q|k|v / ff.net.0.proj):
     * the GEMM that PRODUCES the hidden state h writes per-row partial (sum, sum of squares) of its output, one
     * partial per n-tile, to row_stats_out [n_tiles][rows][2] fp32; the GEMM that CONSUMES LayerNorm(h) runs on raw h
     * with gamma folded into its weights and finishes  out = rstd * (acc - mean * c1[n]) + c2[n]  in the epilogue,
     * c1 = row sums of the folded fp16 weights, c2 = W beta + bias (fp32 [N]).  No LayerNorm kernel, no normalised
     * copy of h.  ln_dim = channels of h; row_stats_parts = n-tiles of the producer (omg_gemm_plan). */
    void* row_stats_out;
    const void* row_stats_in;
    int32_t row_stats_parts;
    int64_t row_stats_stride; /* rows per partial plane (0 = rows of this GEMM); lets a row-sliced GEMM index the full buffer */
    int32_t ln_dim;
    float ln_eps;
    const void* col_c1;
    const void* col_c2;
    /* multi-stream launches: streams (row groups) with different LoRA sets have different c1/c2; then col_c1/col_c2
     * are [n_col_groups][N] and rows [col_group_end[g-1], col_group_end[g]) use plane g (boundaries as for
     * w_group_planes below). */
    int32_t n_col_groups;
    int64_t col_group_end[8];
    int32_t w_group_planes; /* 0: one weight matrix for all rows; else == n_col_groups: w is [planes][N][Ktot] and row
                             * group g multiplies with plane g (per-stream weights, e.g. W + s B_g A_g merged per concept).
                             * Every segment reads plane g (all taps of a conv, the conv2 | shortcut concatenation); bias,
                             * rowvec, column statistics and the fp32 twins do not depend on the plane.  Not with w2.
                             * No tile may mix two groups: on a token grid (d.H == 1) every col_group_end is a multiple
                             * of 128 rows; on a spatial grid (d.H > 1: convs) a tile lies inside one image, so every
                             * col_group_end is a multiple of d.W * d.H pixels (whole images), whatever the image size.
                             * Tall tiles pair two consecutive m-tiles; where a boundary would fall inside a pair the
                             * launch uses single tiles instead. */
    int32_t cta_pair;   /* 0 = auto, 1 = single 128-row tiles, 2 = not available (rejected),
                         * 3 = tall tiles (one CTA, 256 x 160: two 128-row sub-tiles share each weight tile; block_n 160) */
    /* GroupNorm statistics out of the producing GEMM / conv (ResnetBlock2D norm1/norm2, Transformer2DModel.norm,
     * conv_norm_out [3P]): per image and per 32-pixel block of the output, the per-channel (sum, sum of squares) of the
     * fp16-ROUNDED output values, written as float2 to col_stats_out [B][col_stats_rb_total][N]; this launch fills the
     * blocks [col_stats_rb0, col_stats_rb0 + omg_gemm_colstats_blocks(W, H)) of every image.  The consuming
     * omg_groupnorm_apply reduces them to (mean, rstd) per group - for any grouping, also over the channel
     * concatenation of two producers - so GroupNorm never re-reads its input for statistics.  Not with GEGLU. */
    void* col_stats_out;
    int32_t col_stats_rb0, col_stats_rb_total;
    /* fp32 master copy of the residual trunk (x <- x + f(x) through ~70 transformer blocks and the ResBlocks): the addend
     * is read from residual_f32 [pixels, residual_f32_ld] instead of the fp16 `residual`, and the result is ALSO written as
     * fp32 to out_f32 [pixels, out_f32_ld] (the fp16 output stays what the next GEMM / norm reads), so rounding to fp16
     * no longer accumulates along the chain.  Either may be NULL.  Contiguous output view, N % 32 == 0, not with GEGLU. */
    const void* residual_f32;
    int64_t residual_f32_ld;
    void* out_f32;
    int64_t out_f32_ld;
    /* Storage type of the A views, w, bias, residual and the output: OMG_DTYPE_F16 (0, so a zeroed descriptor is fp16)
     * or OMG_DTYPE_BF16.  bf16 covers what the VAE decoder needs - OMG_EPI_NONE with bias and residual, every block_n
     * and tall tiles - and rejects GEGLU, activation epilogues, rowvec, w2, weight planes, the folded LayerNorm, row and
     * column statistics and the fp32 twins.  Accumulation is fp32 either way. */
    int32_t dtype;
} omg_gemm_desc;

int omg_gemm(const omg_gemm_desc* desc, void* stream);

/* Tile plan omg_gemm will use for an output grid (W, H, B) with N channels: block_n and the number of row-statistics
 * partial planes this GEMM emits (= row_stats_parts for the consumer; two per n-tile). */
int omg_gemm_plan(int N, int epilogue, int W, int H, int B, int* block_n, int* stats_parts);

/* Number of 32-pixel column-statistics blocks one omg_gemm launch over an output grid (W, H) writes per image. */
int omg_gemm_colstats_blocks(int W, int H);

#define OMG_ATTN_MAX_ITEMS 16

/*
 * Flash attention, head_dim 64, fp32 softmax, probabilities never materialised:
 *   out[out_b[i], :, h] = (accumulate ? out : 0) + out_weight * softmax(scale * Q[q_b[i],:,h] K[k_b[i],:,h]^T) V[v_b[i],:,h]
 * for every item i and head h.  Q/K/V are row-major [batch, tokens, ld] fp16 with the head's 64 columns at
 * col0 + 64*h.
 *
 * Replaces: attn.get_attention_scores + controller(probs) + torch.bmm in RegionControlNet_AttnProcessor
 * (src/pipelines/lora_pipeline.py:114-116) with the prompt-to-prompt edit of src/prompt_attention/p2p_attention.py:
 * 124-138 folded into the (q_b, k_b, v_b) remap; xformers.ops.memory_efficient_attention / F.scaled_dot_product_
 * attention of the concept UNet (src/ip_adapter/attention_processor.py:197-204,383-401); and the decoupled
 * text + scale*ip sum (attention_processor.py:370-409) via accumulate/out_weight.
 */
typedef struct {
    const void* q; int32_t q_ld; int64_t q_bs; int32_t q_col0;
    const void* k; int32_t k_ld; int64_t k_bs; int32_t k_col0;
    const void* v; int32_t v_ld; int64_t v_bs; int32_t v_col0;
    void* out;     int32_t out_ld; int64_t out_bs; int32_t out_col0;
    int32_t n_q, n_kv, heads, head_dim;
    int32_t n_items;
    int32_t out_b[OMG_ATTN_MAX_ITEMS], q_b[OMG_ATTN_MAX_ITEMS], k_b[OMG_ATTN_MAX_ITEMS], v_b[OMG_ATTN_MAX_ITEMS];
    float scale;      /* softmax scale, head_dim^-0.5 */
    float out_weight; /* weight of this term */
    int32_t accumulate;
    int32_t causal;   /* 1: key j attends only to queries i >= j (CLIP text towers); n_kv <= 128 only */
} omg_attn_desc;

int omg_attention(const omg_attn_desc* desc, void* stream);

/*
 * GroupNorm(32 groups) over channels-last fp16, optional SiLU, input = channel-concatenation of (x1 | x2).
 * y[B, HW, C1+C2].  stats_ws: OMG_GN_WS_FLOATS(B) floats of scratch.  Deterministic: no atomics, results do not depend
 * on the batch position of an image.  x1, x2, y and stats_ws 16 B aligned.  Replaces torch GroupNorm + SiLU + torch.cat
 * inside diffusers ResnetBlock2D / Transformer2DModel / UNet up-blocks [3P] (call site
 * src/pipelines/lora_pipeline.py:546-566).
 */
#define OMG_GN_MAX_SPLITS 256
#define OMG_GN_WS_FLOATS(B) ((B) * (2 * 2 * 2560 + 64 * OMG_GN_MAX_SPLITS))
int omg_groupnorm(const void* x1, int C1, const void* x2, int C2, int B, int HW, const void* gamma, const void* beta,
                  float eps, int silu, void* stats_ws, void* y, void* stream);
/* omg_groupnorm over bf16 x1 / x2 / gamma / beta / y: same arguments, limits, fp32 statistics and summation order. */
int omg_groupnorm_bf16(const void* x1, int C1, const void* x2, int C2, int B, int HW, const void* gamma, const void* beta,
                       float eps, int silu, void* stats_ws, void* y, void* stream);

/* Per-channel (sum, sum of squares) partials of a stored channels-last tensor x [B, HW, C], one float2 per channel per
 * 32-row block: out [B][ceil(HW/32)][C] - the layout omg_gemm's col_stats_out produces (for tensors that were modified
 * after their producing GEMM, e.g. skip connections that received ControlNet residuals).  x 4 B, out 16 B aligned. */
int omg_colstats(const void* x, int C, int B, int HW, void* out, void* stream);

/* GroupNorm(32) [+ SiLU] of cat(x1 | x2) from per-channel partials (omg_gemm col_stats_out / omg_colstats): one tiny
 * reduction launch (partials -> mean, rstd per image and group, fixed summation order) and one apply pass.
 * part1 [B][rb1][C1] float2, part2 [B][rb2][C2] float2 (NULL when C2 == 0), 8 B aligned; stats_ws: OMG_GN_WS_FLOATS(B)
 * floats.  x1, x2, y and stats_ws 16 B aligned. */
int omg_groupnorm_apply(const void* x1, int C1, const void* part1, int rb1, const void* x2, int C2, const void* part2,
                        int rb2, int B, int HW, const void* gamma, const void* beta, float eps, int silu, void* stats_ws,
                        void* y, void* stream);

/* LayerNorm over the last dim of [rows, C] fp16 (BasicTransformerBlock norm1/2/3 [3P]).  x, gamma, beta and y 16 B
 * aligned. */
int omg_layernorm(const void* x, const void* gamma, const void* beta, void* y, long long rows, int C, float eps,
                  void* stream);

#define OMG_MAX_CONCEPTS 8

/*
 * One denoising-step tail in a single launch: region noise fusion, classifier-free guidance, Euler-discrete step,
 * and the next step's scaled model inputs.  Replaces src/pipelines/lora_pipeline.py:568-615 and :491-492,583-585
 * (src/pipelines/instantid_pipeline.py:618-690).
 *   noise_main [4, HW, 8] fp16 rows (uncond0, uncond1, cond0, cond1), channels 0..3 used;
 *   noise_concept[k] [2, HW, 8] rows (uncond, cond); mask[k] [HW] float {0,1} or NULL (concept skipped);
 *   image-1 rows: eps = (1 - U) * eps_main + sum_k M_k * eps_k with U = OR_k M_k;
 *   eps = eps_u + guidance * (eps_c - eps_u);  latents += eps * (sigma_next - sigma)   (fp32 state [2, HW, 4]);
 *   next_main_in [4, HW, 8] = latents / sqrt(sigma_next^2 + 1) in row order (img0, img1, img0, img1);
 *   next_concept_in [2, HW, 8] = scaled image-1 latent twice; latents_f16 optional fp16 copy [2, HW, 4].
 * Alignment: noise_main and noise_concept 8 B; latents, next_main_in and next_concept_in 16 B; latents_f16 4 B.
 */
typedef struct {
    const void* noise_main;
    const void* noise_concept[OMG_MAX_CONCEPTS];
    const void* mask[OMG_MAX_CONCEPTS];
    int32_t n_concepts;
    float guidance, sigma, sigma_next;
    void* latents;
    void* next_main_in;
    void* next_concept_in;
    void* latents_f16;
    int32_t HW;
} omg_fuse_desc;

int omg_fuse_step(const omg_fuse_desc* desc, void* stream);

/*
 * omg_fuse_step with a general one-step sampler update in place of Euler's, in a single launch: the scheduler step
 * of diffusers' EulerDiscreteScheduler (any prediction type), EulerAncestralDiscreteScheduler and
 * DPMSolverMultistepScheduler (dpmsolver++ / sde-dpmsolver++, orders 1 and 2) in coefficient form [3P]
 * (lora_pipeline.py:615 `self.scheduler.step`).  Per element of each image, with eps the fused, guided prediction:
 *   x0 = c_x * x + c_eps * eps;   x' = a * x + b * x0 + c * h + d * z;   latents = x';
 *   next inputs = x' * input_scale (same rows as omg_fuse_step); latents_f16 as omg_fuse_step.
 *   h = history [2, HW, 4] fp32, read when c != 0, then overwritten with x0 when store_x0 != 0;
 *   z = noise, fp16 in NCHW [2, 4, HW] (the layout torch.randn((2, 4, h, w)) draws), read when d != 0.
 * fuse.sigma / fuse.sigma_next are unused.  Alignment: as omg_fuse_step; history 16 B, noise 2 B.
 */
typedef struct {
    omg_fuse_desc fuse;
    float c_x, c_eps;
    float a, b, c, d;
    float input_scale;
    void* history;
    const void* noise;
    int32_t store_x0;
} omg_solver_desc;

int omg_solver_step(const omg_solver_desc* desc, void* stream);

/*
 * out[b, w, :] = sum_n coef[w, n] * ctx[b, n, :]  (fp16 ctx/out [B, L, C], fp32 coef [L, L]).  Builds the
 * prompt-to-prompt edited context  M diag(alpha) ctx  /  diag(1-alpha) ctx  so that the cross-attention edit
 * P0 M * alpha + (1-alpha) P1  (src/prompt_attention/p2p_attention.py:131-134,146-147) becomes two plain attention
 * terms over projected V.
 */
int omg_ctx_mix(const void* ctx, const void* coef, void* out, int B, int L, int C, void* stream);

/* y = a + alpha * b over n fp16 elements (n % 8 == 0; a, b, y 16 B aligned): ControlNet residual injection
 * (down_block_additional_residuals / mid_block_additional_residual, src/pipelines/lora_pipeline.py:546-556). */
int omg_axpy(const void* a, const void* b, float alpha, void* y, long long n, void* stream);

/* In-place row softmax: x[r, :cols] = softmax(scale * x[r, :cols]) for an fp16 matrix with row stride ld (elements),
 * fp32 arithmetic; cols % 8 == 0, cols <= 32768, scale > 0, x 16 B aligned.  The VAE decoder's mid-block attention
 * (one head of 512 channels: `Attention(heads=1)` inside diffusers' AutoencoderKL, reached from
 * src/pipelines/lora_pipeline.py:649) materialises its scores with omg_gemm, normalises them here and applies them with
 * a second omg_gemm. */
int omg_softmax_rows(void* x, long long rows, int cols, long long ld, float scale, void* stream);
/* omg_softmax_rows over a bf16 matrix: same arguments and limits, fp32 arithmetic. */
int omg_softmax_rows_bf16(void* x, long long rows, int cols, long long ld, float scale, void* stream);

/*
 * EfficientViT-SAM image encoder (the segmentation model between the two stages; SURVEY 8f-4), the ops that are not
 * GEMM-shaped.  Channels-last fp16, fp32 arithmetic.  Dense convolutions of the encoder go through omg_gemm (BatchNorm
 * folded into the weights, OMG_EPI_GELU_TANH), LayerNorm2d through omg_layernorm.
 *   omg_dwconv: depthwise k x k (3 | 5) convolution, stride 1 | 2, "same" padding, + bias, act 1 = tanh-GELU; w is
 *     tap-major [k*k, C]; x / y rows of ldx / ldy elements (MBConv.depth_conv, LiteMLA.aggreg[.][0];
 *     src/efficientvit/models/nn/ops.py:196-241,371-392).
 *   omg_group1x1: grouped 1x1 convolution with square groups of 32 channels, w [C, 32] (LiteMLA.aggreg[.][1]).
 *   omg_relu_linear_attention: LiteMLA.relu_linear_att (ops.py:404-440): per head (q | k | v, dim 32)
 *     out = relu(q) (relu(k)^T [v | 1]) normalised by its last column + eps; qkv [B, N, heads*96] -> out [B, N, heads*32].
 *   omg_resize_bicubic: F.interpolate(mode="bicubic", align_corners=False) (SamNeck inputs, sam.py:117-123).
 * The fp16 tensors these read and write 8 channels at a time - x, w, bias and y of omg_dwconv, x and y of omg_group1x1 and
 * omg_resize_bicubic - must be 16 B aligned.
 */
int omg_dwconv(const void* x, const void* w, const void* bias, void* y, int B, int H, int W, int C, int ldx, int ldy, int ksize,
               int stride, int act, void* stream);
int omg_group1x1(const void* x, const void* w, void* y, long long pixels, int C, int ldx, int ldy, int group, void* stream);
int omg_relu_linear_attention(const void* qkv, void* out, int B, int N, int heads, int dim, float eps, void* stream);
int omg_resize_bicubic(const void* x, void* y, int B, int H, int W, int C, int Ho, int Wo, void* stream);

/*
 * EfficientViT-SAM prompt-to-mask path (SURVEY 8f-4): segment_anything's MaskDecoder / TwoWayTransformer [3P] as the
 * reference builds them (src/efficientvit/models/efficientvit/sam.py:520-544) and EfficientViTSam.postprocess_masks
 * (sam.py:224-241).  Projections, MLPs, hypernetworks and the IoU head run on omg_gemm, LayerNorm on omg_layernorm.
 *
 * omg_attention_small: softmax(scale Q K^T) V per head for head_dim 16 | 32 when one side is short, fp32 softmax.  The
 *   descriptor is omg_attn_desc (items remap batches; out_weight must be 1, accumulate and causal 0; q / out rows 16 B
 *   aligned).  n_kv <= 64 (image -> token, token self-attention): K/V of the item and head live in shared memory, any
 *   n_q.  Otherwise n_q <= 64 (token -> image): the keys are split over CTAs of 128, and `ws` must hold
 *   OMG_ATTN_SMALL_WS_FLOATS(n_items, heads, n_q, n_kv) floats for the (acc, max, sum) partials that a second launch
 *   combines.
 */
#define OMG_ATTN_SMALL_WS_FLOATS(items, heads, n_q, n_kv) \
    ((long long)(items) * (heads) * (n_q) * (((n_kv) + 127) / 128) * 36)
int omg_attention_small(const omg_attn_desc* desc, void* ws, void* stream);

/*
 * omg_sam_mask_head: MaskDecoder.output_upscaling after its first ConvTranspose2d, fused with the hypernetwork product:
 *   out[b, m, 2Y+ey, 2X+ex] = sum_o hyper[b, m, o] gelu(b2[o] + sum_c gelu(LN2d(up1[b, Y, X, :]))[c] w2[ey, ex, c, o])
 * up1: fp16 [B, 64, 64, 2, 2, 64] = ConvTranspose2d(256 -> 64, k2, s2) as omg_gemm writes it with weight rows
 * (dy, dx, channel): element (b, 2y + dy, 2x + dx, c) of the 128 x 128 map.  ln_w / ln_b fp32 [64] (LayerNorm2d, eps);
 * w2 fp32 [2][2][64][32] (ConvTranspose2d(64 -> 32) weight [c, o, ey, ex] permuted), b2 fp32 [32]; hyper fp16,
 * element (b, m, o) at hyper + b * hyper_bs + m * hyper_ms + o; M <= 4 masks.  out fp32 [B, M, 256, 256] low-res logits.
 *
 * omg_sam_postprocess: bilinear (align_corners = False) low x low -> mid x mid, crop to [h_in, w_in], bilinear -> H x W,
 * evaluated as one composite per output pixel of lowres fp32 [BM, low, low].  mask (uint8 / bool [BM, H, W]) gets
 * value > threshold, logits (fp32 [BM, H, W]) the value; either may be NULL.
 */
int omg_sam_mask_head(const void* up1, const void* ln_w, const void* ln_b, const void* w2, const void* b2, const void* hyper,
                      long long hyper_bs, long long hyper_ms, int B, int M, float eps, void* out, void* stream);
int omg_sam_postprocess(const void* lowres, int BM, int low, int mid, int h_in, int w_in, int H, int W, float threshold,
                        void* mask, void* logits, void* stream);

/*
 * omg_attention_relpos: segment_anything's ViT image-encoder attention with decomposed relative-position bias
 * (Attention.forward with use_rel_pos = True, add_decomposed_rel_pos / get_rel_pos [3P]; the original SAM ViT-B/L/H that
 * the reference's `--segment_type GroundingDINO` branch prompts, inference_lora.py:91-126,191-198), fp32 softmax,
 * probabilities never materialised:
 *   S[q, k] = scale q.k + q.Rh[qh - kh + Sh - 1] + q.Rw[qw - kw + Sw - 1]     (the rel-pos terms use the UNSCALED q)
 *   out = softmax(S) V                                                      per image, head and attention group.
 * qkv: fp16 [B, H*W, ld] rows in token order (row-major H x W grid) - the qkv Linear's output, head h's q / k / v at
 * columns q_col0 / k_col0 / v_col0 + head_dim * h.  out: fp16 [B, H*W, out_ld], head h at out_col0 + head_dim * h (what
 * proj consumes).  head_dim 64 | 80.  rel_pos_h [rel_h_len, head_dim], rel_pos_w [rel_w_len, head_dim] fp16, contiguous.
 *   window == 0: global attention over the H x W grid (H, W <= 64); rel_h_len = 2H - 1, rel_w_len = 2W - 1.
 *   window  > 0: window_partition / window_unpartition: the grid is padded at the bottom and right to multiples of the
 *     window and attention runs inside each window x window group (window <= 64); rel_h_len = rel_w_len = 2 window - 1.
 *     The reference pads the normalised input before qkv, so a padded key / value is the qkv bias: k_bias / v_bias
 *     (fp16 [heads * head_dim], head h at head_dim * h) are required when H or W is not a multiple of the window.
 *     Outputs of padded queries are not written.
 * No interpolation of the tables (get_rel_pos with unequal sizes) and no batch remapping.
 */
typedef struct {
    const void* qkv; int32_t ld; int64_t bs; int32_t q_col0, k_col0, v_col0;
    void* out;       int32_t out_ld; int64_t out_bs; int32_t out_col0;
    int32_t B, H, W, heads, head_dim, window;
    const void* rel_pos_h; int32_t rel_h_len;
    const void* rel_pos_w; int32_t rel_w_len;
    const void* k_bias;
    const void* v_bias;
    float scale;      /* head_dim^-0.5 */
} omg_attn_relpos_desc;

int omg_attention_relpos(const omg_attn_relpos_desc* desc, void* stream);

/*
 * Face analysis (insightface FaceAnalysis('antelopev2'): an SCRFD detector and an ArcFace IResNet recogniser).  Their
 * convolutions and the recogniser's FC run on omg_gemm; these are the ops that are not GEMM-shaped.
 *
 * omg_channel_op: channels-last fp16, fp32 arithmetic, over B x H x W pixels of C channels (x / y rows of ldx / ldy
 *   elements):  v = x[p, c] * scale[c] + shift[c];  y[p, c] = act(v) + a  (act_after_add = 0) or act(v + a) (= 1), where
 *   a = addend[b, y / add_scale, x / add_scale, c] (rows of ld_add elements, grid H / add_scale x W / add_scale: the
 *   nearest x2 up-sampling of an FPN top-down path when add_scale = 2) or 0 without an addend (add_scale 0).  x may be
 *   NULL (read as 0: a nearest up-sampling on its own), scale / shift NULL (1 / 0).  act: OMG_CH_ACT_*; PReLU reads
 *   slope[c].  scale, shift and slope are fp32 [C].  y may alias x; it must not overlap the addend.
 * omg_pool2d: max (is_max = 1) or average pooling, k x k window (1 <= k <= 3), stride 1 | 2, symmetric pad < k, with
 *   ONNX / PyTorch ceil_mode and count_include_pad.  x [B, H, W, C] and y [B, Ho, Wo, C] contiguous and 16 B aligned,
 *   C % 8 == 0.
 * omg_scrfd_detect: SCRFD.detect after the network, in one CTA: anchors with score >= det_thresh (strides' row-major
 *   grids, num_anchors consecutive anchors per cell, centre (x, y) * stride), distance2bbox / distance2kps of the
 *   predictions times the stride, / det_scale, a descending sort of the scores (ties: lower anchor index first) and
 *   greedy NMS with the +1 pixel area convention (suppress when IoU > nms_thresh), all in fp32 with no contraction.
 *   Writes rows [x1, y1, x2, y2, score, kx0, ky0, .., kx4, ky4] to out (fp32, capacity max_out rows) and the row count
 *   to *count (device int).  Every anchor of the levels must fit the CTA's shared memory (13 B each, at most
 *   OMG_SCRFD_MAX_ANCHORS: 640 x 640 with strides 8 / 16 / 32 and two anchors is 16 800); max_out must be at least the
 *   number of anchors, so no face can be dropped.
 */
#define OMG_CH_ACT_NONE 0
#define OMG_CH_ACT_RELU 1
#define OMG_CH_ACT_PRELU 2
#define OMG_CH_ACT_SIGMOID 3
int omg_channel_op(const void* x, long long ldx, void* y, long long ldy, const float* scale, const float* shift,
                   const float* slope, const void* addend, long long ld_add, int add_scale, int B, int H, int W, int C,
                   int act, int act_after_add, void* stream);
int omg_pool2d(const void* x, void* y, int B, int H, int W, int C, int k, int stride, int pad, int ceil_mode,
               int count_include_pad, int is_max, void* stream);

#define OMG_SCRFD_MAX_LEVELS 5
#define OMG_SCRFD_MAX_ANCHORS 17800
typedef struct {
    const float* scores[OMG_SCRFD_MAX_LEVELS];  /* [fh * fw * num_anchors] per level */
    const float* boxes[OMG_SCRFD_MAX_LEVELS];   /* [fh * fw * num_anchors, 4] distances in units of the stride */
    const float* kps[OMG_SCRFD_MAX_LEVELS];     /* [fh * fw * num_anchors, 10], or NULL everywhere (no key-points) */
    int32_t stride[OMG_SCRFD_MAX_LEVELS];
    int32_t fh[OMG_SCRFD_MAX_LEVELS], fw[OMG_SCRFD_MAX_LEVELS];
    int32_t n_levels, num_anchors;
    float det_thresh, nms_thresh, det_scale;
    float* out;       /* [max_out, 15] */
    int32_t max_out;
    int32_t* count;   /* device */
} omg_scrfd_desc;

int omg_scrfd_detect(const omg_scrfd_desc* desc, void* stream);

/*
 * YOLO-World (ultralytics WorldModel: the open-vocabulary detector whose boxes prompt SAM between OMG's two stages).
 * Its convolutions and linears run on omg_gemm, SPPF's max-pool on omg_pool2d, up-sampling on omg_channel_op,
 * LayerNorm on omg_layernorm and the pooling attention on omg_attention_small; these are the ops that are not.
 *
 * omg_text_gate: MaxSigmoidAttnBlock after its convs, fp32 arithmetic, per image b and pixel of a B x HW grid:
 *   gate[h] = sigmoid(max_k <embed[b, pix, h*hc : (h+1)*hc], guide[b, k, h*hc : (h+1)*hc]> / sqrt(hc) + bias[h])
 *             * scale[h]                                        (hc = Ce / nh; scale NULL = 1)
 *   out[b, pix, c] = p[b, pix, c] * gate[c / (C2 / nh)]
 * embed fp16 rows of ld_e elements (Ce channels), guide fp32 [B, n, Ce] contiguous (gl(text) of each image, so images
 * with different prompts share one launch), bias / scale fp32 [nh], p (proj_conv's output) and out fp16 rows of ld_p /
 * ld_o elements (C2 channels; out may alias p - the gated slice of C2fAttn's concat buffer).  n >= 1, hc 16 | 32 | 64,
 * C2 % nh == 0, C2 and every row stride a multiple of 8, embed / p / out 16 B aligned; the guide of one image
 * (n * Ce floats) must fit in shared memory.
 * omg_adaptive_maxpool: AdaptiveMaxPool2d((k, k)) of x [B, H, W, C] (rows of ldx elements) with PyTorch's windows
 *   [floor(i H / k), ceil((i + 1) H / k)) (overlapping when k does not divide H); patch i * k + j of image b goes to
 *   out + b * out_bs + (row0 + i * k + j) * out_ld (fp16, C channels): ImagePoolingAttn's 3 levels x 9 patches fill
 *   rows 0..26 of its key buffer.  C, ldx, out_ld and out_bs multiples of 8, x / out 16 B aligned.
 * omg_yolo_detect: WorldDetect + non_max_suppression + scale_boxes for one image, in up to two launches.
 *   (a) one warp per anchor over the levels (row-major grids, anchor centre (x + 0.5, y + 0.5) * stride):
 *       logit_k = <x', text[k]> * cls_scale[l] + cls_bias[l] with x' = x / max(|x|, 1e-12) when normalize_x (the
 *       plain ContrastiveHead; BNContrastiveHead's BatchNorm is folded into the embedding conv instead and
 *       normalize_x = 0), text [nc, E] fp32 already L2-normalised, cls_scale = exp(logit_scale); score = max_k
 *       sigmoid(logit_k), cls = its first argmax; DFL (softmax expectation over 16 bins of each side's box logits) and
 *       dist2bbox -> xywh -> xyxy in letterbox pixels.  rows [T, 6] fp32 = [x0, y0, x1, y1, score, cls] per anchor.
 *   (b) skipped when out is NULL; otherwise one CTA: anchors with score > conf (strict), a descending sort (ties: lower
 *       anchor index first), greedy NMS on boxes offset by cls * max_wh (0 when agnostic) that suppresses IoU > iou
 *       (torchvision's IoU, no +1), at most max_det rows, then (box - pad) / gain clipped to [0, clip_w] x [0, clip_h],
 *       all fp32 without contraction.  out [max_out, 6] rows [x0, y0, x1, y1, score, cls]; *count (device int).
 *   box: fp16 rows of box_ld elements, the 4 x 16 DFL logits (l, t, r, b); emb: fp16 rows of emb_ld elements, E channels.
 *   At most OMG_YOLO_MAX_ANCHORS anchors (640 x 640 at strides 8 / 16 / 32 is 8 400) and OMG_YOLO_MAX_CLASSES classes.
 *   Cost of (b): the rank of each of the n candidates is a count over all n (n^2 shared-memory reads over 1024
 *   threads), then one barrier per kept row.  ultralytics' max_nms (30 000) never binds below the anchor cap, so n is
 *   every anchor above conf: at most 17 800 (about 310 000 reads per thread).
 */
int omg_text_gate(const void* embed, long long ld_e, int Ce, const float* guide, int n, const float* bias,
                  const float* scale, int nh, const void* p, long long ld_p, void* out, long long ld_o, int C2, int B,
                  int HW, void* stream);
int omg_adaptive_maxpool(const void* x, long long ldx, int B, int H, int W, int C, int k, void* out, long long out_bs,
                         long long out_ld, int row0, void* stream);

#define OMG_YOLO_MAX_LEVELS 4
#define OMG_YOLO_MAX_ANCHORS 17800
#define OMG_YOLO_MAX_CLASSES 1024
#define OMG_YOLO_REG_MAX 16
typedef struct {
    const void* box[OMG_YOLO_MAX_LEVELS];
    const void* emb[OMG_YOLO_MAX_LEVELS];
    int64_t box_ld[OMG_YOLO_MAX_LEVELS], emb_ld[OMG_YOLO_MAX_LEVELS];
    float cls_scale[OMG_YOLO_MAX_LEVELS], cls_bias[OMG_YOLO_MAX_LEVELS];
    int32_t stride[OMG_YOLO_MAX_LEVELS], fh[OMG_YOLO_MAX_LEVELS], fw[OMG_YOLO_MAX_LEVELS];
    int32_t n_levels, nc, E, normalize_x;
    const float* text;   /* [nc, E] */
    float* rows;         /* [anchors, 6] */
    float conf, iou, max_wh;
    int32_t agnostic, max_det;
    float gain, pad_x, pad_y, clip_w, clip_h;
    float* out;          /* [max_out, 6], or NULL: pass (a) only */
    int32_t max_out;
    int32_t* count;      /* device */
} omg_yolo_desc;

int omg_yolo_detect(const omg_yolo_desc* desc, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Launch plans: a forward as a handle.  The reference drives one UNet forward as a Python call
 * (`self.unet(latent_model_input, t, ...)`, src/pipelines/lora_pipeline.py:558-567, 588-606); a host that is not Python -
 * or does not want ~720 descriptor builds per forward - records that call once and replays it through this handle:
 *
 *   omg_plan* fwd = omg_plan_create();
 *   omg_plan_record_begin(fwd);  ... one eager forward: omg_gemm / omg_attention / omg_groupnorm_apply / ... ;
 *   omg_plan_record_end(fwd);
 *   for every step:  (write the sample and the step's time embedding into their buffers)  omg_plan_run(fwd, stream);
 *
 * While a thread records, every entry point above that launched successfully also appends a copy of its call - the
 * descriptor by value, so every pointer in it must stay valid for as long as the plan is run (the executor's persistent
 * workspace does) - and omg_plan_run re-issues the calls in order on `stream` with no further host work than the launches.
 * Replay validates each descriptor and encodes its tensor maps again (a plan holds descriptors, not encoded launches), so a
 * plan is valid exactly as long as the buffers its descriptors point to.
 * One recording per thread at a time; a plan may be run from any thread once recording has ended.
 */
typedef struct omg_plan omg_plan;
omg_plan* omg_plan_create(void);
void omg_plan_destroy(omg_plan* plan);
int omg_plan_record_begin(omg_plan* plan);
int omg_plan_record_end(omg_plan* plan);
int omg_plan_length(const omg_plan* plan);     /* number of recorded launches; -1 for NULL */
int omg_plan_clear(omg_plan* plan);
int omg_plan_run(const omg_plan* plan, void* stream);

/* Error string of the last failing call on this thread (never NULL). */
const char* omg_last_error(void);
/* Library / build identification: returns e.g. "omg_b200 0.1 sm_90a". */
const char* omg_version(void);
/* Number of kernel launches issued by this library since process start (bench.py's gpu_launches). */
uint64_t omg_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif
