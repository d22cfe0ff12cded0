// Kernels of the EfficientViT-SAM prompt-to-mask path (SURVEY section 8, row f-4): what the mask decoder
// (segment_anything MaskDecoder / TwoWayTransformer [3P], configured by reference sam.py:520-544) and the predictor's
// postprocess (EfficientViTSam.postprocess_masks, sam.py:224-241) need besides omg_gemm / omg_layernorm:
//   * attention with head dims 16 / 32 where one side has few tokens (<= 64 prompt tokens) and the other side up to
//     4096 image tokens per prompt: the short side's K/V in shared memory (image -> token, token self-attention), or the
//     long key side split over CTAs with (max, sum, acc) partials and a combine pass (token -> image);
//   * the mask head: LayerNorm2d + GELU of the first transposed conv's output, the second 2x2 / stride 2 transposed
//     conv, GELU and the hypernetwork dot products in one pass (the 32-channel upscaled tensor is never stored);
//   * the two bilinear resizes + crop + threshold of postprocess_masks as one composite per output pixel.
// Everything here is tiny in FLOPs (~2 GFLOP per prompt); the decoder is bound by launch count, so each kernel is a
// plain fp32 CUDA-core kernel and the launch count is what the design minimises.
#include <cuda_fp16.h>

#include "../../include/omg_b200.h"
#include "host_common.h"
#include "ptx.cuh"

namespace omg {

constexpr int SA_SHORT = 64;     // max tokens of the short side
constexpr int SA_CHUNK = 128;    // keys per CTA of the split-key path
constexpr int SA_WS_ROW = 36;    // floats per (split, query) partial: acc[<= 32], max, sum

template <int D>
__device__ __forceinline__ void load_row(const __half* src, float scale, float (&dst)[D]) {
#pragma unroll
    for (int v = 0; v < D / 8; ++v) {
        const uint4 raw = *reinterpret_cast<const uint4*>(src + 8 * v);
        const __half2* h = reinterpret_cast<const __half2*>(&raw);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float2 f = __half22float2(h[e]);
            dst[8 * v + 2 * e] = f.x * scale;
            dst[8 * v + 2 * e + 1] = f.y * scale;
        }
    }
}

template <int D>
__device__ __forceinline__ void store_row(__half* dst, const float (&src)[D], float mul) {
#pragma unroll
    for (int v = 0; v < D / 8; ++v) {
        uint4 raw;
        __half2* h = reinterpret_cast<__half2*>(&raw);
#pragma unroll
        for (int e = 0; e < 4; ++e) h[e] = __floats2half2_rn(src[8 * v + 2 * e] * mul, src[8 * v + 2 * e + 1] * mul);
        *reinterpret_cast<uint4*>(dst + 8 * v) = raw;
    }
}

// Short key side (n_kv <= 64): the (item, head)'s K and V sit in shared memory, one thread per query, online softmax.
// grid (ceil(n_q / 128), heads, items).
template <int D>
__global__ void __launch_bounds__(128) attn_small_kv_kernel(const __grid_constant__ omg_attn_desc p) {
    griddep_launch_dependents();
    griddep_wait();
    __shared__ float ks[SA_SHORT][D + 1];
    __shared__ float vs[SA_SHORT][D + 1];
    const int item = blockIdx.z, h = blockIdx.y;
    const __half* kb = static_cast<const __half*>(p.k) + (size_t)p.k_b[item] * p.k_bs + p.k_col0 + h * D;
    const __half* vb = static_cast<const __half*>(p.v) + (size_t)p.v_b[item] * p.v_bs + p.v_col0 + h * D;
    for (int e = threadIdx.x; e < p.n_kv * D; e += blockDim.x) {
        const int j = e / D, c = e % D;
        ks[j][c] = __half2float(kb[(size_t)j * p.k_ld + c]);
        vs[j][c] = __half2float(vb[(size_t)j * p.v_ld + c]);
    }
    __syncthreads();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.n_q) return;
    float q[D], acc[D];
    load_row<D>(static_cast<const __half*>(p.q) + (size_t)p.q_b[item] * p.q_bs + (size_t)i * p.q_ld + p.q_col0 + h * D, p.scale, q);
#pragma unroll
    for (int c = 0; c < D; ++c) acc[c] = 0.f;
    float m = -INFINITY, l = 0.f;
    for (int j = 0; j < p.n_kv; ++j) {
        float s = 0.f;
#pragma unroll
        for (int c = 0; c < D; ++c) s = fmaf(q[c], ks[j][c], s);
        const float mn = fmaxf(m, s);
        const float corr = __expf(m - mn), pj = __expf(s - mn);
        l = fmaf(l, corr, pj);
#pragma unroll
        for (int c = 0; c < D; ++c) acc[c] = fmaf(acc[c], corr, pj * vs[j][c]);
        m = mn;
    }
    store_row<D>(static_cast<__half*>(p.out) + (size_t)p.out_b[item] * p.out_bs + (size_t)i * p.out_ld + p.out_col0 + h * D, acc,
                 1.0f / l);
}

// Long key side (n_q <= 64, n_kv > 64): CTA (split, head, item) scores its 128 keys against every query - one warp per
// query, a lane per 4 keys - and writes the unnormalised partial (acc, max, sum) of each query to ws.
template <int D>
__global__ void __launch_bounds__(256) attn_small_split_kernel(const __grid_constant__ omg_attn_desc p, float* __restrict__ ws,
                                                               int n_split) {
    griddep_launch_dependents();
    griddep_wait();
    __shared__ float qs[SA_SHORT][D + 1];
    __shared__ float ks[SA_CHUNK][D + 1];
    __shared__ float vs[SA_CHUNK][D + 1];
    __shared__ float ps[8][SA_CHUNK];
    const int split = blockIdx.x, h = blockIdx.y, item = blockIdx.z;
    const int j0 = split * SA_CHUNK, nk = min(SA_CHUNK, p.n_kv - j0);
    const __half* qb = static_cast<const __half*>(p.q) + (size_t)p.q_b[item] * p.q_bs + p.q_col0 + h * D;
    const __half* kb = static_cast<const __half*>(p.k) + (size_t)p.k_b[item] * p.k_bs + (size_t)j0 * p.k_ld + p.k_col0 + h * D;
    const __half* vb = static_cast<const __half*>(p.v) + (size_t)p.v_b[item] * p.v_bs + (size_t)j0 * p.v_ld + p.v_col0 + h * D;
    for (int e = threadIdx.x; e < p.n_q * D; e += blockDim.x) {
        const int i = e / D, c = e % D;
        qs[i][c] = __half2float(qb[(size_t)i * p.q_ld + c]) * p.scale;
    }
    for (int e = threadIdx.x; e < SA_CHUNK * D; e += blockDim.x) {
        const int j = e / D, c = e % D;
        const bool ok = j < nk;
        ks[j][c] = ok ? __half2float(kb[(size_t)j * p.k_ld + c]) : 0.f;
        vs[j][c] = ok ? __half2float(vb[(size_t)j * p.v_ld + c]) : 0.f;
    }
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    constexpr int KPL = SA_CHUNK / 32;  // keys per lane
    for (int i = warp; i < p.n_q; i += 8) {
        float s[KPL];
        float m = -INFINITY;
#pragma unroll
        for (int t = 0; t < KPL; ++t) {
            const int j = lane + 32 * t;
            float a = 0.f;
#pragma unroll
            for (int c = 0; c < D; ++c) a = fmaf(qs[i][c], ks[j][c], a);
            s[t] = j < nk ? a : -INFINITY;
            m = fmaxf(m, s[t]);
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, off));
        float l = 0.f;
#pragma unroll
        for (int t = 0; t < KPL; ++t) {
            const float e = __expf(s[t] - m);  // exp(-inf) = 0 for keys past the end
            ps[warp][lane + 32 * t] = e;
            l += e;
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) l += __shfl_xor_sync(0xffffffffu, l, off);
        __syncwarp();
        // P.V: lane = (key parity, channel) for D = 16, channel for D = 32
        constexpr int JS = 32 / D;
        const int c = lane % D, jp = lane / D;
        float a = 0.f;
        for (int j = jp; j < SA_CHUNK; j += JS) a = fmaf(ps[warp][j], vs[j][c], a);
        if constexpr (JS == 2) a += __shfl_down_sync(0xffffffffu, a, 16);
        float* row = ws + ((((size_t)item * p.heads + h) * p.n_q + i) * n_split + split) * SA_WS_ROW;
        if (lane < D) row[c] = a;
        if (lane == 0) {
            row[D] = m;
            row[D + 1] = l;
        }
        __syncwarp();
    }
}

// Combine of the split-key partials: thread = (item, head, query, channel).
template <int D>
__global__ void attn_small_combine_kernel(const __grid_constant__ omg_attn_desc p, const float* __restrict__ ws, int n_split) {
    griddep_launch_dependents();
    griddep_wait();
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)p.n_items * p.heads * p.n_q * D) return;
    const int c = (int)(idx % D);
    const long long r = idx / D;  // ((item * heads) + h) * n_q + i
    const int i = (int)(r % p.n_q);
    const int h = (int)((r / p.n_q) % p.heads);
    const int item = (int)(r / ((long long)p.n_q * p.heads));
    const float* rows = ws + (size_t)r * n_split * SA_WS_ROW;
    float m = -INFINITY;
    for (int s = 0; s < n_split; ++s) m = fmaxf(m, rows[(size_t)s * SA_WS_ROW + D]);
    float l = 0.f, a = 0.f;
    for (int s = 0; s < n_split; ++s) {
        const float* row = rows + (size_t)s * SA_WS_ROW;
        const float w = __expf(row[D] - m);
        l = fmaf(row[D + 1], w, l);
        a = fmaf(row[c], w, a);
    }
    static_cast<__half*>(p.out)[(size_t)p.out_b[item] * p.out_bs + (size_t)i * p.out_ld + p.out_col0 + h * D + c] =
        __float2half_rn(a / l);
}

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f)); }

// Mask head. up1 = ConvTranspose2d #1 output as the GEMM stores it: [B][64][64][dy][dx][64] fp16, i.e. the 128 x 128 map
// at (2y + dy, 2x + dx).  Thread = one 128-grid position x one of the 2 x 2 output sub-pixels of ConvTranspose2d #2:
//   v = gelu(LayerNorm2d(up1[Y, X, :]));  u[o] = gelu(b2[o] + sum_c v[c] w2[ey, ex, c, o]);
//   out[b, m, 2Y + ey, 2X + ex] = sum_o hyper[b, m, o] u[o]
constexpr int MH_C = 64, MH_O = 32, MH_MAX_M = 4, MH_WSUB = MH_C * MH_O + 1;  // +1: the 4 sub-pixels on distinct banks
__global__ void __launch_bounds__(256) sam_mask_head_kernel(const __half* __restrict__ up1, const float* __restrict__ ln_w,
                                                            const float* __restrict__ ln_b, const float* __restrict__ w2,
                                                            const float* __restrict__ b2, const __half* __restrict__ hyper,
                                                            long long hyper_bs, long long hyper_ms, int M, float eps,
                                                            float* __restrict__ out) {
    griddep_launch_dependents();
    griddep_wait();
    __shared__ float ws[4 * MH_WSUB];
    __shared__ float hs[MH_MAX_M][MH_O];
    __shared__ float lw[MH_C], lb[MH_C], bs[MH_O];
    const int b = blockIdx.y;
    for (int e = threadIdx.x; e < 4 * MH_C * MH_O; e += blockDim.x) ws[(e / (MH_C * MH_O)) * MH_WSUB + e % (MH_C * MH_O)] = w2[e];
    for (int e = threadIdx.x; e < M * MH_O; e += blockDim.x)
        hs[e / MH_O][e % MH_O] = __half2float(hyper[(size_t)b * hyper_bs + (size_t)(e / MH_O) * hyper_ms + e % MH_O]);
    if (threadIdx.x < MH_C) {
        lw[threadIdx.x] = ln_w[threadIdx.x];
        lb[threadIdx.x] = ln_b[threadIdx.x];
    }
    if (threadIdx.x < MH_O) bs[threadIdx.x] = b2[threadIdx.x];
    __syncthreads();
    const int pos = blockIdx.x * (blockDim.x / 4) + (threadIdx.x >> 2), sub = threadIdx.x & 3;
    const int Y = pos >> 7, X = pos & 127;
    const __half* src = up1 + ((((size_t)b * 64 + (Y >> 1)) * 64 + (X >> 1)) * 4 + (Y & 1) * 2 + (X & 1)) * MH_C;
    float v[MH_C];
    load_row<MH_C>(src, 1.0f, v);
    float mu = 0.f;
#pragma unroll
    for (int c = 0; c < MH_C; ++c) mu += v[c];
    mu *= 1.0f / MH_C;
    float var = 0.f;
#pragma unroll
    for (int c = 0; c < MH_C; ++c) var = fmaf(v[c] - mu, v[c] - mu, var);
    const float rstd = rsqrtf(var * (1.0f / MH_C) + eps);
#pragma unroll
    for (int c = 0; c < MH_C; ++c) v[c] = gelu_erf(fmaf((v[c] - mu) * rstd, lw[c], lb[c]));
    float u[MH_O];
#pragma unroll
    for (int o = 0; o < MH_O; ++o) u[o] = bs[o];
    const float* wsub = ws + sub * MH_WSUB;
#pragma unroll 4
    for (int c = 0; c < MH_C; ++c) {
#pragma unroll
        for (int o = 0; o < MH_O; ++o) u[o] = fmaf(v[c], wsub[c * MH_O + o], u[o]);
    }
#pragma unroll
    for (int o = 0; o < MH_O; ++o) u[o] = gelu_erf(u[o]);
    const int P = 2 * Y + (sub >> 1), Q = 2 * X + (sub & 1);
    for (int m = 0; m < M; ++m) {
        float a = 0.f;
#pragma unroll
        for (int o = 0; o < MH_O; ++o) a = fmaf(hs[m][o], u[o], a);
        out[(((size_t)b * M + m) * 256 + P) * 256 + Q] = a;
    }
}

// postprocess_masks: F.interpolate(bilinear, align_corners=False) low x low -> mid x mid, crop to (h_in, w_in),
// F.interpolate(bilinear) -> (H, W), > threshold; both resizes evaluated per output pixel with PyTorch's source-index rule
// (src = max(scale * (dst + 0.5) - 0.5, 0), scale = in / out, upper tap clamped).
struct Taps {
    int i0, i1;
    float l0, l1;
};
__device__ __forceinline__ Taps bilinear_taps(int dst, float scale, int in_size) {
    const float s = fmaxf(scale * ((float)dst + 0.5f) - 0.5f, 0.f);
    Taps t;
    t.i0 = (int)s;
    t.i1 = t.i0 + ((t.i0 < in_size - 1) ? 1 : 0);
    t.l1 = s - (float)t.i0;
    t.l0 = 1.0f - t.l1;
    return t;
}

__device__ __forceinline__ float mid_value(const float* __restrict__ plane, int low, float s_low, int Y, int X) {
    const Taps ty = bilinear_taps(Y, s_low, low), tx = bilinear_taps(X, s_low, low);
    const float* r0 = plane + (size_t)ty.i0 * low;
    const float* r1 = plane + (size_t)ty.i1 * low;
    return ty.l0 * (tx.l0 * __ldg(r0 + tx.i0) + tx.l1 * __ldg(r0 + tx.i1)) + ty.l1 * (tx.l0 * __ldg(r1 + tx.i0) + tx.l1 * __ldg(r1 + tx.i1));
}

__global__ void sam_postprocess_kernel(const float* __restrict__ lowres, int low, int mid, int h_in, int w_in, int H, int W,
                                       float threshold, uint8_t* __restrict__ mask, float* __restrict__ logits) {
    griddep_launch_dependents();
    griddep_wait();
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)H * W) return;
    const int bm = blockIdx.y;
    const int i = (int)(idx / W), j = (int)(idx % W);
    const float* plane = lowres + (size_t)bm * low * low;
    const float s_low = (float)low / (float)mid;
    const Taps ty = bilinear_taps(i, (float)h_in / (float)H, h_in), tx = bilinear_taps(j, (float)w_in / (float)W, w_in);
    const float v = ty.l0 * (tx.l0 * mid_value(plane, low, s_low, ty.i0, tx.i0) + tx.l1 * mid_value(plane, low, s_low, ty.i0, tx.i1)) +
                    ty.l1 * (tx.l0 * mid_value(plane, low, s_low, ty.i1, tx.i0) + tx.l1 * mid_value(plane, low, s_low, ty.i1, tx.i1));
    const size_t o = (size_t)bm * H * W + idx;
    if (mask != nullptr) mask[o] = v > threshold ? 1 : 0;
    if (logits != nullptr) logits[o] = v;
}

}  // namespace omg

using namespace omg;

static int attention_small_impl(const omg_attn_desc* d, void* ws, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    OMG_CHECK(d != nullptr && d->q && d->k && d->v && d->out, "omg_attention_small: null pointer");
    OMG_CHECK(d->head_dim == 16 || d->head_dim == 32, "omg_attention_small: head_dim %d (16 or 32)", d->head_dim);
    OMG_CHECK(d->n_items >= 1 && d->n_items <= OMG_ATTN_MAX_ITEMS && d->heads >= 1 && d->n_q >= 1 && d->n_kv >= 1,
              "omg_attention_small: bad shape");
    OMG_CHECK(d->out_weight == 1.0f && !d->accumulate && !d->causal, "omg_attention_small: plain attention only");
    OMG_CHECK(d->q_ld % 8 == 0 && d->out_ld % 8 == 0 && d->q_col0 % 8 == 0 && d->out_col0 % 8 == 0 && d->q_bs % 8 == 0 &&
                  d->out_bs % 8 == 0 && ((uintptr_t)d->q & 15) == 0 && ((uintptr_t)d->out & 15) == 0,
              "omg_attention_small: q / out rows must be 16 B aligned (ld, col0, batch stride multiples of 8)");
    if (check_head_windows("omg_attention_small", d->heads, d->head_dim, {d->q_col0, d->k_col0, d->v_col0, d->out_col0},
                           {d->q_ld, d->k_ld, d->v_ld, d->out_ld}))
        return 1;
    const omg_attn_desc p = *d;
    const bool d16 = d->head_dim == 16;
    if (d->n_kv <= SA_SHORT) {
        const dim3 grid((unsigned)((d->n_q + 127) / 128), d->heads, d->n_items);
        if (d16) OMG_CUDA(launch_pdl(attn_small_kv_kernel<16>, grid, dim3(128), 0, stream, p));
        else OMG_CUDA(launch_pdl(attn_small_kv_kernel<32>, grid, dim3(128), 0, stream, p));
        return check_launch("attn_small_kv_kernel");
    }
    OMG_CHECK(d->n_q <= SA_SHORT, "omg_attention_small: one side must have <= %d tokens (n_q %d, n_kv %d)", SA_SHORT, d->n_q,
              d->n_kv);
    OMG_CHECK(ws != nullptr, "omg_attention_small: %d keys need the split-key workspace", d->n_kv);
    const int n_split = (d->n_kv + SA_CHUNK - 1) / SA_CHUNK;
    const dim3 grid(n_split, d->heads, d->n_items);
    float* w = static_cast<float*>(ws);
    if (d16) OMG_CUDA(launch_pdl(attn_small_split_kernel<16>, grid, dim3(256), 0, stream, p, w, n_split));
    else OMG_CUDA(launch_pdl(attn_small_split_kernel<32>, grid, dim3(256), 0, stream, p, w, n_split));
    if (check_launch("attn_small_split_kernel")) return 1;
    const long long total = (long long)d->n_items * d->heads * d->n_q * d->head_dim;
    const dim3 cgrid((unsigned)((total + 255) / 256));
    if (d16) OMG_CUDA(launch_pdl(attn_small_combine_kernel<16>, cgrid, dim3(256), 0, stream, p, (const float*)w, n_split));
    else OMG_CUDA(launch_pdl(attn_small_combine_kernel<32>, cgrid, dim3(256), 0, stream, p, (const float*)w, n_split));
    return check_launch("attn_small_combine_kernel");
}

static int sam_mask_head_impl(const void* up1, const void* ln_w, const void* ln_b, const void* w2, const void* b2,
                              const void* hyper, long long hyper_bs, long long hyper_ms, int B, int M, float eps, void* out,
                              void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    OMG_CHECK(up1 && ln_w && ln_b && w2 && b2 && hyper && out, "omg_sam_mask_head: null pointer");
    OMG_CHECK(B >= 1 && M >= 1 && M <= MH_MAX_M, "omg_sam_mask_head: B >= 1, 1 <= M <= 4");
    OMG_CHECK(((uintptr_t)up1 & 15) == 0, "omg_sam_mask_head: up1 must be 16 B aligned");
    OMG_CUDA(launch_pdl(sam_mask_head_kernel, dim3(128 * 128 / 64, B), dim3(256), 0, stream, static_cast<const __half*>(up1),
                        static_cast<const float*>(ln_w), static_cast<const float*>(ln_b), static_cast<const float*>(w2),
                        static_cast<const float*>(b2), static_cast<const __half*>(hyper), hyper_bs, hyper_ms, M, eps,
                        static_cast<float*>(out)));
    return check_launch("sam_mask_head_kernel");
}

static int sam_postprocess_impl(const void* lowres, int BM, int low, int mid, int h_in, int w_in, int H, int W, float threshold,
                                void* mask, void* logits, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    OMG_CHECK(lowres && (mask || logits), "omg_sam_postprocess: null pointer");
    OMG_CHECK(BM >= 1 && low >= 1 && mid >= 1 && h_in >= 1 && w_in >= 1 && h_in <= mid && w_in <= mid && H >= 1 && W >= 1,
              "omg_sam_postprocess: bad shape");
    const long long total = (long long)H * W;
    OMG_CUDA(launch_pdl(sam_postprocess_kernel, dim3((unsigned)((total + 255) / 256), BM), dim3(256), 0, stream,
                        static_cast<const float*>(lowres), low, mid, h_in, w_in, H, W, threshold, static_cast<uint8_t*>(mask),
                        static_cast<float*>(logits)));
    return check_launch("sam_postprocess_kernel");
}

// C-ABI entry points: launch, and - while this thread records a launch plan (omg_plan_record_begin) - remember the call
extern "C" int omg_attention_small(const omg_attn_desc* desc, void* ws, void* stream_) {
    const int rc = attention_small_impl(desc, ws, stream_);
    if (rc == 0 && ::omg::plan_recording()) {
        const omg_attn_desc d = *desc;
        ::omg::plan_note([=](void* s) { return attention_small_impl(&d, ws, s); });
    }
    return rc;
}

extern "C" int omg_sam_mask_head(const void* up1, const void* ln_w, const void* ln_b, const void* w2, const void* b2,
                                 const void* hyper, long long hyper_bs, long long hyper_ms, int B, int M, float eps, void* out,
                                 void* stream_) {
    const int rc = sam_mask_head_impl(up1, ln_w, ln_b, w2, b2, hyper, hyper_bs, hyper_ms, B, M, eps, out, stream_);
    if (rc == 0 && ::omg::plan_recording())
        ::omg::plan_note([=](void* s) { return sam_mask_head_impl(up1, ln_w, ln_b, w2, b2, hyper, hyper_bs, hyper_ms, B, M, eps, out, s); });
    return rc;
}

extern "C" int omg_sam_postprocess(const void* lowres, int BM, int low, int mid, int h_in, int w_in, int H, int W, float threshold,
                                   void* mask, void* logits, void* stream_) {
    const int rc = sam_postprocess_impl(lowres, BM, low, mid, h_in, w_in, H, W, threshold, mask, logits, stream_);
    if (rc == 0 && ::omg::plan_recording())
        ::omg::plan_note([=](void* s) { return sam_postprocess_impl(lowres, BM, low, mid, h_in, w_in, H, W, threshold, mask, logits, s); });
    return rc;
}
