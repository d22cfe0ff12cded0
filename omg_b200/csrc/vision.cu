// Kernels of the EfficientViT-SAM image encoder (SURVEY section 8, row f-4: the segmentation model between the two
// stages, reference src/efficientvit/models/nn/ops.py + models/efficientvit/sam.py) that are not GEMM-shaped:
// depthwise convolutions (MBConv, the multi-scale aggregation of LiteMLA), the grouped 1x1 convolution of that
// aggregation, the ReLU linear attention core of LiteMLA, and the bicubic resize of the SAM neck.  Dense 3x3 / 1x1
// convolutions (BatchNorm folded, tanh-GELU in the epilogue), LayerNorm2d and residual adds run on gemm_tc.cu / norm.cu.
// All of these are HBM- / latency-bound (a few MAC per byte) and run once per image: plain coalesced kernels,
// channels-last fp16 storage, fp32 arithmetic.
#include <cuda_fp16.h>

#include "../../include/omg_b200.h"
#include "host_common.h"
#include "ptx.cuh"

namespace omg {

__device__ __forceinline__ float gelu_tanh(float x) {
    // nn.GELU(approximate="tanh"): 0.5 x (1 + tanh(sqrt(2/pi) (x + 0.044715 x^3))); tanh(u) = 1 - 2 / (1 + e^(2u))
    const float u = 0.7978845608028654f * fmaf(0.044715f * x * x, x, x);
    const float t = 1.0f - __fdividef(2.0f, 1.0f + __expf(2.0f * u));
    return 0.5f * x * (1.0f + t);
}

// Depthwise k x k convolution, stride 1 | 2, "same" padding, + bias, + optional tanh-GELU.
// x [B, H, W, C], w [k*k, C] (tap-major so that a thread's 8 channels are one 16 B load per tap), y [B, Ho, Wo, C].
// thread = 8 channels of one output pixel.
template <int K>
__global__ void dwconv_kernel(const __half* __restrict__ x, const __half* __restrict__ w, const __half* __restrict__ bias,
                              __half* __restrict__ y, int H, int W, int C, int ldx, int ldy, int Ho, int Wo, int stride, int act) {
    griddep_launch_dependents();
    griddep_wait();
    const int vpr = C / 8;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)Ho * Wo * vpr;
    if (idx >= total) return;
    const int b = blockIdx.y;
    const int c0 = (int)(idx % vpr) * 8;
    const int pix = (int)(idx / vpr);
    const int oy = pix / Wo, ox = pix - oy * Wo;
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
    constexpr int P = K / 2;
#pragma unroll
    for (int ky = 0; ky < K; ++ky) {
        const int iy = oy * stride + ky - P;
        if (iy < 0 || iy >= H) continue;
#pragma unroll
        for (int kx = 0; kx < K; ++kx) {
            const int ix = ox * stride + kx - P;
            if (ix < 0 || ix >= W) continue;
            const uint4 xv = *reinterpret_cast<const uint4*>(x + (((size_t)b * H + iy) * W + ix) * ldx + c0);
            const uint4 wv = __ldg(reinterpret_cast<const uint4*>(w + (size_t)(ky * K + kx) * C + c0));
            const __half2* xh = reinterpret_cast<const __half2*>(&xv);
            const __half2* wh = reinterpret_cast<const __half2*>(&wv);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float2 xf = __half22float2(xh[i]), wf = __half22float2(wh[i]);
                acc[2 * i] = fmaf(xf.x, wf.x, acc[2 * i]);
                acc[2 * i + 1] = fmaf(xf.y, wf.y, acc[2 * i + 1]);
            }
        }
    }
    if (bias != nullptr) {
        const uint4 bv = __ldg(reinterpret_cast<const uint4*>(bias + c0));
        const __half2* bh = reinterpret_cast<const __half2*>(&bv);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float2 bf = __half22float2(bh[i]);
            acc[2 * i] += bf.x;
            acc[2 * i + 1] += bf.y;
        }
    }
    if (act == 1) {
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] = gelu_tanh(acc[i]);
    }
    uint4 o;
    __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
    for (int i = 0; i < 4; ++i) oh[i] = __floats2half2_rn(acc[2 * i], acc[2 * i + 1]);
    *reinterpret_cast<uint4*>(y + (((size_t)b * Ho + oy) * Wo + ox) * ldy + c0) = o;
}

// Grouped 1x1 convolution with square groups of G channels (LiteMLA aggregation: G = head dim 32, groups = 3 * heads):
// y[p, g*G + o] = sum_i w[g*G + o, i] * x[p, g*G + i].  block = one group x 64 pixels; the group's weights sit in smem
// transposed ([i][o]) so that a thread's 8 outputs are contiguous.
template <int G>
__global__ void group1x1_kernel(const __half* __restrict__ x, const __half* __restrict__ w, __half* __restrict__ y,
                                long long pixels, int ldx, int ldy) {
    griddep_launch_dependents();
    griddep_wait();
    __shared__ float wt[G][G + 1];
    const int g = blockIdx.y;
    for (int t = threadIdx.x; t < G * G; t += blockDim.x) {
        const int o = t / G, i = t % G;
        wt[i][o] = __half2float(w[(size_t)(g * G + o) * G + i]);
    }
    __syncthreads();
    constexpr int OV = G / 8;  // 8-channel output vectors per pixel and group
    const long long p = (long long)blockIdx.x * (blockDim.x / OV) + threadIdx.x / OV;
    if (p >= pixels) return;
    const int o0 = (threadIdx.x % OV) * 8;
    const __half* xp = x + (size_t)p * ldx + g * G;
    float acc[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] = 0.f;
#pragma unroll
    for (int iv = 0; iv < G / 8; ++iv) {
        const uint4 xv = *reinterpret_cast<const uint4*>(xp + iv * 8);
        const __half* xh = reinterpret_cast<const __half*>(&xv);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const float xf = __half2float(xh[k]);
#pragma unroll
            for (int e = 0; e < 8; ++e) acc[e] = fmaf(xf, wt[iv * 8 + k][o0 + e], acc[e]);
        }
    }
    uint4 o;
    __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
    for (int e = 0; e < 4; ++e) oh[e] = __floats2half2_rn(acc[2 * e], acc[2 * e + 1]);
    *reinterpret_cast<uint4*>(y + (size_t)p * ldy + g * G + o0) = o;
}

// ReLU linear attention of LiteMLA (ops.py:404-440), head dim D = 32, fp32 like the reference (autocast disabled):
//   kv = relu(K)^T [V | 1]  (D x (D+1));   out = relu(Q) kv;   out = out[:, :D] / (out[:, D] + eps)
// qkv [B, N, heads * 3D] with a head's channels laid out (q | k | v); out [B, N, heads * D].
// One CTA per (batch, head): phase 1 streams the tokens through shared memory and accumulates kv in registers
// (thread (j, r): column j of V, rows 4r..4r+3 of K), phase 2 applies it to every token.
template <int D>
__global__ void __launch_bounds__(256) relu_linear_attn_kernel(const __half* __restrict__ qkv, __half* __restrict__ out, int N,
                                                              int heads, float eps) {
    griddep_launch_dependents();
    griddep_wait();
    constexpr int CH = 64;  // tokens per shared-memory chunk
    __shared__ float ks[CH][D + 1];
    __shared__ float vs[CH][D + 1];
    __shared__ float kv[D][D + 2];  // column D = sum_t relu(k_t)
    const int h = blockIdx.x, b = blockIdx.y;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
    const size_t ld = (size_t)heads * 3 * D;
    const __half* base = qkv + (size_t)b * N * ld + (size_t)h * 3 * D;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    float ksum = 0.f;  // threads with ty == 0 .. : tx < D -> sum of relu(k)[tx]
    for (int t0 = 0; t0 < N; t0 += CH) {
        const int nt = min(CH, N - t0);
        for (int e = threadIdx.x; e < CH * D; e += 256) {
            const int t = e / D, c = e % D;
            float kf = 0.f, vf = 0.f;
            if (t < nt) {
                kf = fmaxf(__half2float(base[(size_t)(t0 + t) * ld + D + c]), 0.f);
                vf = __half2float(base[(size_t)(t0 + t) * ld + 2 * D + c]);
            }
            ks[t][c] = kf;
            vs[t][c] = vf;
        }
        __syncthreads();
        for (int t = 0; t < nt; ++t) {
            const float vj = vs[t][tx];
#pragma unroll
            for (int r = 0; r < 4; ++r) acc[r] = fmaf(ks[t][ty * 4 + r], vj, acc[r]);
            if (ty == 0) ksum += ks[t][tx];
        }
        __syncthreads();
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) kv[ty * 4 + r][tx] = acc[r];
    if (ty == 0) kv[tx][D] = ksum;
    __syncthreads();
    // phase 2: 8 tokens in flight (one per warp), lane = output channel
    __half* ob = out + (size_t)b * N * heads * D + (size_t)h * D;
    for (int t = ty; t < N; t += 8) {
        const float qf = fmaxf(__half2float(base[(size_t)t * ld + tx]), 0.f);
        float o = 0.f, den = 0.f;
#pragma unroll
        for (int i = 0; i < D; ++i) {
            const float qi = __shfl_sync(0xffffffffu, qf, i);
            o = fmaf(qi, kv[i][tx], o);
            den = fmaf(qi, kv[i][D], den);
        }
        ob[(size_t)t * heads * D + tx] = __float2half_rn(o / (den + eps));
    }
}

// F.interpolate(mode="bicubic", align_corners=False) (the SAM neck resizes its three inputs to 64 x 64, sam.py:117-123):
// PyTorch's kernel - A = -0.75, source index (dst + 0.5) * scale - 0.5, taps clamped to the border.
__device__ __forceinline__ void cubic_coeffs(float t, float (&c)[4]) {
    const float A = -0.75f;
    const float x0 = t + 1.0f, x1 = t, x2 = 1.0f - t, x3 = 2.0f - t;
    c[0] = ((A * x0 - 5.0f * A) * x0 + 8.0f * A) * x0 - 4.0f * A;
    c[1] = ((A + 2.0f) * x1 - (A + 3.0f)) * x1 * x1 + 1.0f;
    c[2] = ((A + 2.0f) * x2 - (A + 3.0f)) * x2 * x2 + 1.0f;
    c[3] = ((A * x3 - 5.0f * A) * x3 + 8.0f * A) * x3 - 4.0f * A;
}

__global__ void resize_bicubic_kernel(const __half* __restrict__ x, __half* __restrict__ y, int H, int W, int C, int Ho, int Wo,
                                      float sy, float sx) {
    griddep_launch_dependents();
    griddep_wait();
    const int vpr = C / 8;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)Ho * Wo * vpr) return;
    const int b = blockIdx.y;
    const int c0 = (int)(idx % vpr) * 8;
    const int pix = (int)(idx / vpr);
    const int oy = pix / Wo, ox = pix - oy * Wo;
    const float fy = (oy + 0.5f) * sy - 0.5f, fx = (ox + 0.5f) * sx - 0.5f;
    const int iy = (int)floorf(fy), ix = (int)floorf(fx);
    float cy[4], cx[4];
    cubic_coeffs(fy - iy, cy);
    cubic_coeffs(fx - ix, cx);
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
#pragma unroll
    for (int a = 0; a < 4; ++a) {
        const int yy = min(max(iy - 1 + a, 0), H - 1);
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const int xx = min(max(ix - 1 + c, 0), W - 1);
            const float wgt = cy[a] * cx[c];
            const uint4 v = *reinterpret_cast<const uint4*>(x + (((size_t)b * H + yy) * W + xx) * C + c0);
            const __half2* vh = reinterpret_cast<const __half2*>(&v);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float2 f = __half22float2(vh[i]);
                acc[2 * i] = fmaf(wgt, f.x, acc[2 * i]);
                acc[2 * i + 1] = fmaf(wgt, f.y, acc[2 * i + 1]);
            }
        }
    }
    uint4 o;
    __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
    for (int i = 0; i < 4; ++i) oh[i] = __floats2half2_rn(acc[2 * i], acc[2 * i + 1]);
    *reinterpret_cast<uint4*>(y + (((size_t)b * Ho + oy) * Wo + ox) * C + c0) = o;
}

}  // namespace omg

using namespace omg;

static int dwconv_impl(const void* x, const void* w, const void* bias, void* y, int B, int H, int W, int C, int ldx, int ldy,
                          int ksize, int stride, int act, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    OMG_CHECK(x && w && y, "omg_dwconv: null pointer");
    if (check_aligned("omg_dwconv", 16, {{"x", x}, {"w", w}, {"bias", bias}, {"y", y}})) return 1;
    OMG_CHECK(B >= 1 && H >= 1 && W >= 1 && C >= 8 && C % 8 == 0, "omg_dwconv: bad shape (C must be a multiple of 8)");
    OMG_CHECK(ldx >= C && ldy >= C && ldx % 8 == 0 && ldy % 8 == 0, "omg_dwconv: row strides must be >= C and multiples of 8");
    OMG_CHECK((ksize == 3 || ksize == 5) && (stride == 1 || stride == 2) && (act == 0 || act == 1), "omg_dwconv: kernel 3|5, stride 1|2, act 0|1");
    const int Ho = (H + stride - 1) / stride, Wo = (W + stride - 1) / stride;  // "same" padding: ceil(H / stride)
    const long long total = (long long)Ho * Wo * (C / 8);
    const dim3 grid((unsigned)((total + 255) / 256), B);
    const __half *xp = static_cast<const __half*>(x), *wp = static_cast<const __half*>(w), *bp = static_cast<const __half*>(bias);
    __half* yp = static_cast<__half*>(y);
    if (ksize == 3)
        OMG_CUDA(launch_pdl(dwconv_kernel<3>, grid, dim3(256), 0, stream, xp, wp, bp, yp, H, W, C, ldx, ldy, Ho, Wo, stride, act));
    else
        OMG_CUDA(launch_pdl(dwconv_kernel<5>, grid, dim3(256), 0, stream, xp, wp, bp, yp, H, W, C, ldx, ldy, Ho, Wo, stride, act));
    return check_launch("dwconv_kernel");
}

static int group1x1_impl(const void* x, const void* w, void* y, long long pixels, int C, int ldx, int ldy, int group,
                            void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    OMG_CHECK(x && w && y, "omg_group1x1: null pointer");
    if (check_aligned("omg_group1x1", 16, {{"x", x}, {"y", y}})) return 1;
    OMG_CHECK(group == 32 && C >= 32 && C % 32 == 0 && pixels >= 1, "omg_group1x1: group size 32, C a multiple of 32");
    OMG_CHECK(ldx >= C && ldy >= C && ldx % 8 == 0 && ldy % 8 == 0, "omg_group1x1: row strides must be >= C and multiples of 8");
    const dim3 grid((unsigned)((pixels + 63) / 64), C / 32);
    OMG_CUDA(launch_pdl(group1x1_kernel<32>, grid, dim3(256), 0, stream, static_cast<const __half*>(x), static_cast<const __half*>(w),
                        static_cast<__half*>(y), pixels, ldx, ldy));
    return check_launch("group1x1_kernel");
}

static int relu_linear_attention_impl(const void* qkv, void* out, int B, int N, int heads, int dim, float eps, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    OMG_CHECK(qkv && out, "omg_relu_linear_attention: null pointer");
    OMG_CHECK(dim == 32 && B >= 1 && N >= 1 && heads >= 1, "omg_relu_linear_attention: head dim 32 only (EfficientViT-SAM)");
    OMG_CUDA(launch_pdl(relu_linear_attn_kernel<32>, dim3(heads, B), dim3(256), 0, stream, static_cast<const __half*>(qkv),
                        static_cast<__half*>(out), N, heads, eps));
    return check_launch("relu_linear_attn_kernel");
}

static int resize_bicubic_impl(const void* x, void* y, int B, int H, int W, int C, int Ho, int Wo, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    OMG_CHECK(x && y, "omg_resize_bicubic: null pointer");
    if (check_aligned("omg_resize_bicubic", 16, {{"x", x}, {"y", y}})) return 1;
    OMG_CHECK(B >= 1 && H >= 1 && W >= 1 && Ho >= 1 && Wo >= 1 && C >= 8 && C % 8 == 0, "omg_resize_bicubic: bad shape");
    const long long total = (long long)Ho * Wo * (C / 8);
    OMG_CUDA(launch_pdl(resize_bicubic_kernel, dim3((unsigned)((total + 255) / 256), B), dim3(256), 0, stream,
                        static_cast<const __half*>(x), static_cast<__half*>(y), H, W, C, Ho, Wo, (float)H / (float)Ho,
                        (float)W / (float)Wo));
    return check_launch("resize_bicubic_kernel");
}

// C-ABI entry points: launch, and - while this thread records a launch plan (omg_plan_record_begin) - remember the call
extern "C" int omg_dwconv(const void* x, const void* w, const void* bias, void* y, int B, int H, int W, int C, int ldx, int ldy,
                          int ksize, int stride, int act, void* stream_) {
    const int rc = dwconv_impl(x, w, bias, y, B, H, W, C, ldx, ldy, ksize, stride, act, stream_);
    if (rc == 0 && ::omg::plan_recording()) ::omg::plan_note([=](void* s) { return dwconv_impl(x, w, bias, y, B, H, W, C, ldx, ldy, ksize, stride, act, s); });
    return rc;
}

extern "C" int omg_group1x1(const void* x, const void* w, void* y, long long pixels, int C, int ldx, int ldy, int group,
                            void* stream_) {
    const int rc = group1x1_impl(x, w, y, pixels, C, ldx, ldy, group, stream_);
    if (rc == 0 && ::omg::plan_recording()) ::omg::plan_note([=](void* s) { return group1x1_impl(x, w, y, pixels, C, ldx, ldy, group, s); });
    return rc;
}

extern "C" int omg_relu_linear_attention(const void* qkv, void* out, int B, int N, int heads, int dim, float eps, void* stream_) {
    const int rc = relu_linear_attention_impl(qkv, out, B, N, heads, dim, eps, stream_);
    if (rc == 0 && ::omg::plan_recording()) ::omg::plan_note([=](void* s) { return relu_linear_attention_impl(qkv, out, B, N, heads, dim, eps, s); });
    return rc;
}

extern "C" int omg_resize_bicubic(const void* x, void* y, int B, int H, int W, int C, int Ho, int Wo, void* stream_) {
    const int rc = resize_bicubic_impl(x, y, B, H, W, C, Ho, Wo, stream_);
    if (rc == 0 && ::omg::plan_recording()) ::omg::plan_note([=](void* s) { return resize_bicubic_impl(x, y, B, H, W, C, Ho, Wo, s); });
    return rc;
}
