// Kernels of face analysis (insightface FaceAnalysis('antelopev2'), the identity and key-point source of the InstantID
// flow, reference inference_instantid.py:226-228,353-354) that are not GEMM-shaped.  The SCRFD detector's and the
// IResNet recogniser's convolutions run on gemm_tc.cu (BatchNorm folded where it is exact, ReLU and residual adds in the
// epilogue where they can be); what is left is
//   - channel_op: a per-channel affine + activation + (up-sampled) addend: the BatchNorm that precedes a padded conv,
//     PReLU, the score sigmoid, the FPN top-down nearest-x2 + add, and residual adds the GEMM epilogue cannot take;
//   - pool2d: the detector stem's max-pool and the average-pool of its avg-down shortcuts;
//   - scrfd_detect: threshold, anchor decode, sort and greedy NMS of SCRFD.detect in one CTA.
// Channels-last fp16 storage, fp32 arithmetic.  All of these are memory- or latency-bound and run once per image.
#include <cuda_fp16.h>

#include "../../include/omg_b200.h"
#include "host_common.h"
#include "ptx.cuh"

namespace omg {

__device__ __forceinline__ float channel_act(float v, int act, float slope) {
    if (act == OMG_CH_ACT_RELU) return fmaxf(v, 0.f);
    if (act == OMG_CH_ACT_PRELU) return v >= 0.f ? v : v * slope;
    if (act == OMG_CH_ACT_SIGMOID) return 1.f / (1.f + __expf(-v));
    return v;
}

// thread = V consecutive channels of one pixel (V = 8: 16 B accesses; V = 1 for channel counts or row strides that
// are not multiples of 8, e.g. a score map flattened to one channel)
template <int V>
__global__ void channel_op_kernel(const __half* x, long long ldx, __half* y, long long ldy,
                                  const float* __restrict__ scale, const float* __restrict__ shift,
                                  const float* __restrict__ slope, const __half* __restrict__ addend, long long ld_add,
                                  int add_scale, int H, int W, int C, int act, int act_after_add, long long total) {
    griddep_launch_dependents();
    griddep_wait();
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const int vpr = C / V;
    const int c0 = (int)(idx % vpr) * V;
    const long long pix = idx / vpr;  // b * H * W + yy * W + xx
    float v[V], a[V];
    if (x != nullptr) {
        const __half* xp = x + pix * ldx + c0;
        if constexpr (V == 8) {
            const uint4 u = *reinterpret_cast<const uint4*>(xp);
            const __half* h = reinterpret_cast<const __half*>(&u);
#pragma unroll
            for (int i = 0; i < 8; ++i) v[i] = __half2float(h[i]);
        } else {
            v[0] = __half2float(*xp);
        }
    } else {
#pragma unroll
        for (int i = 0; i < V; ++i) v[i] = 0.f;
    }
#pragma unroll
    for (int i = 0; i < V; ++i) {
        a[i] = 0.f;
        if (scale != nullptr) v[i] *= scale[c0 + i];
        if (shift != nullptr) v[i] += shift[c0 + i];
    }
    if (add_scale > 0) {
        const long long hw = (long long)H * W;
        const long long b = pix / hw;
        const int r = (int)(pix - b * hw);
        const int yy = r / W, xx = r - yy * W;
        const int Ha = H / add_scale, Wa = W / add_scale;
        const __half* ap = addend + ((b * Ha + yy / add_scale) * Wa + xx / add_scale) * ld_add + c0;
        if constexpr (V == 8) {
            const uint4 u = *reinterpret_cast<const uint4*>(ap);
            const __half* h = reinterpret_cast<const __half*>(&u);
#pragma unroll
            for (int i = 0; i < 8; ++i) a[i] = __half2float(h[i]);
        } else {
            a[0] = __half2float(*ap);
        }
    }
    float o[V];
#pragma unroll
    for (int i = 0; i < V; ++i) {
        const float s = (act == OMG_CH_ACT_PRELU) ? slope[c0 + i] : 0.f;
        o[i] = act_after_add ? channel_act(v[i] + a[i], act, s) : channel_act(v[i], act, s) + a[i];
    }
    __half* yp = y + pix * ldy + c0;
    if constexpr (V == 8) {
        uint4 u;
        __half2* h = reinterpret_cast<__half2*>(&u);
#pragma unroll
        for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(o[2 * i], o[2 * i + 1]);
        *reinterpret_cast<uint4*>(yp) = u;
    } else {
        *yp = __float2half_rn(o[0]);
    }
}

// PyTorch's pooling windows: start = o * stride - pad, end = min(start + k, H + pad) (the divisor of count_include_pad),
// then clipped to the image.  thread = 8 channels of one output pixel.
__global__ void pool2d_kernel(const __half* __restrict__ x, __half* __restrict__ y, int H, int W, int C, int Ho, int Wo, int k,
                              int stride, int pad, int count_include_pad, int is_max, long long total) {
    griddep_launch_dependents();
    griddep_wait();
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const int vpr = C / 8;
    const int c0 = (int)(idx % vpr) * 8;
    long long pix = idx / vpr;
    const int ox = (int)(pix % Wo);
    pix /= Wo;
    const int oy = (int)(pix % Ho);
    const long long b = pix / Ho;
    const int hs = oy * stride - pad, ws = ox * stride - pad;
    const int he = min(hs + k, H + pad), we = min(ws + k, W + pad);
    const int pool_size = (he - hs) * (we - ws);
    const int h0 = max(hs, 0), w0 = max(ws, 0), h1 = min(he, H), w1 = min(we, W);
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = is_max ? -INFINITY : 0.f;
    for (int iy = h0; iy < h1; ++iy)
        for (int ix = w0; ix < w1; ++ix) {
            const uint4 u = *reinterpret_cast<const uint4*>(x + ((b * H + iy) * W + ix) * C + c0);
            const __half* h = reinterpret_cast<const __half*>(&u);
#pragma unroll
            for (int i = 0; i < 8; ++i) acc[i] = is_max ? fmaxf(acc[i], __half2float(h[i])) : acc[i] + __half2float(h[i]);
        }
    if (!is_max) {
        const float div = (float)(count_include_pad ? pool_size : (h1 - h0) * (w1 - w0));
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] /= div;
    }
    uint4 u;
    __half2* h = reinterpret_cast<__half2*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(acc[2 * i], acc[2 * i + 1]);
    *reinterpret_cast<uint4*>(y + ((b * Ho + oy) * Wo + ox) * C + c0) = u;
}

struct ScrfdLevels {
    const float* scores[OMG_SCRFD_MAX_LEVELS];
    const float* boxes[OMG_SCRFD_MAX_LEVELS];
    const float* kps[OMG_SCRFD_MAX_LEVELS];
    int stride[OMG_SCRFD_MAX_LEVELS], fw[OMG_SCRFD_MAX_LEVELS], first[OMG_SCRFD_MAX_LEVELS + 1];
    int n_levels, num_anchors;
};

// candidate g (index into the concatenation of the levels) -> level, anchor within it, anchor centre
__device__ __forceinline__ int scrfd_locate(const ScrfdLevels& L, int g, int& a, float& cx, float& cy) {
    int l = 0;
    while (g >= L.first[l + 1]) ++l;
    a = g - L.first[l];
    const int cell = a / L.num_anchors;
    const int s = L.stride[l];
    cx = (float)((cell % L.fw[l]) * s);
    cy = (float)((cell / L.fw[l]) * s);
    return l;
}

// box of candidate g exactly as insightface computes it in fp32: (centre -/+ pred * stride) / det_scale
__device__ __forceinline__ void scrfd_box(const ScrfdLevels& L, int g, float det_scale, float (&bx)[4]) {
    int a;
    float cx, cy;
    const int l = scrfd_locate(L, g, a, cx, cy);
    const float sf = (float)L.stride[l];
    const float* d = L.boxes[l] + (size_t)a * 4;
    bx[0] = __fdiv_rn(__fsub_rn(cx, __fmul_rn(d[0], sf)), det_scale);
    bx[1] = __fdiv_rn(__fsub_rn(cy, __fmul_rn(d[1], sf)), det_scale);
    bx[2] = __fdiv_rn(__fadd_rn(cx, __fmul_rn(d[2], sf)), det_scale);
    bx[3] = __fdiv_rn(__fadd_rn(cy, __fmul_rn(d[3], sf)), det_scale);
}

__device__ __forceinline__ float box_area1(const float (&b)[4]) {
    return __fmul_rn(__fadd_rn(__fsub_rn(b[2], b[0]), 1.f), __fadd_rn(__fsub_rn(b[3], b[1]), 1.f));
}

__global__ void __launch_bounds__(1024) scrfd_detect_kernel(ScrfdLevels L, float det_thresh, float nms_thresh,
                                                            float det_scale, float* __restrict__ out, int* __restrict__ count) {
    griddep_launch_dependents();
    griddep_wait();
    extern __shared__ __align__(16) unsigned char smem[];
    const int T = L.first[L.n_levels];
    float* key = reinterpret_cast<float*>(smem);            // score of compacted candidate i
    int* gid = reinterpret_cast<int*>(key + T);             // its anchor index in the concatenation
    int* order = gid + T;                                   // anchor index of rank r
    unsigned char* supp = reinterpret_cast<unsigned char*>(order + T);
    __shared__ int n_cand, n_keep;
    if (threadIdx.x == 0) n_cand = n_keep = 0;
    __syncthreads();
    // 1. threshold + compaction (slot order is arbitrary; the sort key includes the anchor index)
    for (int g = threadIdx.x; g < T; g += blockDim.x) {
        int l = 0;
        while (g >= L.first[l + 1]) ++l;
        const float s = L.scores[l][g - L.first[l]];
        if (s >= det_thresh) {
            const int slot = atomicAdd(&n_cand, 1);
            key[slot] = s;
            gid[slot] = g;
        }
    }
    __syncthreads();
    const int n = n_cand;
    // 2. rank sort: descending score, ties by ascending anchor index (a total order, so ranks are a permutation)
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const float si = key[i];
        const int gi = gid[i];
        int rank = 0;
        for (int j = 0; j < n; ++j) {
            const float sj = key[j];
            rank += (sj > si) || (sj == si && gid[j] < gi);
        }
        order[rank] = gi;
    }
    for (int i = threadIdx.x; i < n; i += blockDim.x) supp[i] = 0;
    __syncthreads();
    // 3. greedy NMS in rank order; supp[p] is final once the loop reaches p (only kept candidates suppress, and each
    //    kept iteration ends with a barrier), so a suppressed p is skipped by every thread alike
    for (int p = 0; p < n; ++p) {
        if (supp[p]) continue;
        const int gp = order[p];
        float bp[4];
        scrfd_box(L, gp, det_scale, bp);
        const float ap = box_area1(bp);
        if (threadIdx.x == 0) {
            float* row = out + (size_t)n_keep * 15;
            int a;
            float cx, cy;
            const int l = scrfd_locate(L, gp, a, cx, cy);
#pragma unroll
            for (int i = 0; i < 4; ++i) row[i] = bp[i];
            row[4] = L.scores[l][a];
            const float sf = (float)L.stride[l];
            for (int i = 0; i < 10; ++i) {
                const float c = (i % 2 == 0) ? cx : cy;
                row[5 + i] = L.kps[l] ? __fdiv_rn(__fadd_rn(c, __fmul_rn(L.kps[l][(size_t)a * 10 + i], sf)), det_scale) : 0.f;
            }
            ++n_keep;
        }
        for (int q = p + 1 + threadIdx.x; q < n; q += blockDim.x) {
            if (supp[q]) continue;
            float bq[4];
            scrfd_box(L, order[q], det_scale, bq);
            const float xx1 = fmaxf(bp[0], bq[0]), yy1 = fmaxf(bp[1], bq[1]);
            const float xx2 = fminf(bp[2], bq[2]), yy2 = fminf(bp[3], bq[3]);
            const float w = fmaxf(0.f, __fadd_rn(__fsub_rn(xx2, xx1), 1.f));
            const float h = fmaxf(0.f, __fadd_rn(__fsub_rn(yy2, yy1), 1.f));
            const float inter = __fmul_rn(w, h);
            const float ovr = __fdiv_rn(inter, __fsub_rn(__fadd_rn(ap, box_area1(bq)), inter));
            if (ovr > nms_thresh) supp[q] = 1;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) *count = n_keep;
}

}  // namespace omg

using namespace omg;

static int channel_op_impl(const void* x, long long ldx, void* y, long long ldy, const float* scale, const float* shift,
                           const float* slope, const void* addend, long long ld_add, int add_scale, int B, int H, int W,
                           int C, int act, int act_after_add, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    OMG_CHECK(y != nullptr, "omg_channel_op: null output");
    OMG_CHECK(B >= 1 && H >= 1 && W >= 1 && C >= 1, "omg_channel_op: bad shape B=%d H=%d W=%d C=%d", B, H, W, C);
    OMG_CHECK(act >= OMG_CH_ACT_NONE && act <= OMG_CH_ACT_SIGMOID, "omg_channel_op: unknown activation %d", act);
    OMG_CHECK(act != OMG_CH_ACT_PRELU || slope != nullptr, "omg_channel_op: PReLU needs a slope vector");
    OMG_CHECK(add_scale == 0 || add_scale == 1 || add_scale == 2, "omg_channel_op: add_scale %d (0, 1 or 2)", add_scale);
    OMG_CHECK((add_scale == 0) == (addend == nullptr), "omg_channel_op: an addend needs add_scale 1 | 2, and add_scale one");
    OMG_CHECK(add_scale != 2 || (H % 2 == 0 && W % 2 == 0), "omg_channel_op: a x2 addend needs even H and W (%d x %d)", H, W);
    OMG_CHECK(x != nullptr || add_scale != 0, "omg_channel_op: x and addend both NULL");
    OMG_CHECK((x == nullptr || ldx >= C) && ldy >= C && (addend == nullptr || ld_add >= C),
              "omg_channel_op: row strides must be >= C");
    const bool vec = C % 8 == 0 && (x == nullptr || ldx % 8 == 0) && ldy % 8 == 0 && (addend == nullptr || ld_add % 8 == 0) &&
                     ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y) | reinterpret_cast<uintptr_t>(addend)) & 15) == 0;
    const long long total = (long long)B * H * W * (vec ? C / 8 : C);
    const dim3 grid((unsigned)((total + 255) / 256));
    auto k = vec ? channel_op_kernel<8> : channel_op_kernel<1>;
    OMG_CUDA(launch_pdl(k, grid, dim3(256), 0, stream, static_cast<const __half*>(x), ldx, static_cast<__half*>(y), ldy,
                        scale, shift, slope, static_cast<const __half*>(addend), ld_add, add_scale, H, W, C, act,
                        act_after_add ? 1 : 0, total));
    return check_launch("channel_op_kernel");
}

static int pool2d_impl(const void* x, void* y, int B, int H, int W, int C, int k, int stride, int pad, int ceil_mode,
                       int count_include_pad, int is_max, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    OMG_CHECK(x && y, "omg_pool2d: null pointer");
    if (check_aligned("omg_pool2d", 16, {{"x", x}, {"y", y}})) return 1;
    OMG_CHECK(B >= 1 && H >= 1 && W >= 1 && C >= 8 && C % 8 == 0, "omg_pool2d: bad shape (C=%d must be a multiple of 8)", C);
    OMG_CHECK(k >= 1 && k <= 3 && (stride == 1 || stride == 2) && pad >= 0 && 2 * pad <= k,
              "omg_pool2d: kernel %d, stride %d, pad %d unsupported (k <= 3, stride 1 | 2, pad <= k / 2)", k, stride, pad);
    OMG_CHECK(H + 2 * pad >= k && W + 2 * pad >= k, "omg_pool2d: window %d larger than the padded input", k);
    int Ho = (H + 2 * pad - k + (ceil_mode ? stride - 1 : 0)) / stride + 1;
    int Wo = (W + 2 * pad - k + (ceil_mode ? stride - 1 : 0)) / stride + 1;
    if (ceil_mode && (Ho - 1) * stride >= H + pad) --Ho;  // the last window must start inside the image or its left pad
    if (ceil_mode && (Wo - 1) * stride >= W + pad) --Wo;
    const long long total = (long long)B * Ho * Wo * (C / 8);
    OMG_CUDA(launch_pdl(pool2d_kernel, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, stream,
                        static_cast<const __half*>(x), static_cast<__half*>(y), H, W, C, Ho, Wo, k, stride, pad,
                        count_include_pad ? 1 : 0, is_max ? 1 : 0, total));
    return check_launch("pool2d_kernel");
}

static constexpr int kScrfdSmemLimit = 232448;  // sm_90 opt-in shared memory per block (227 KB)

static int scrfd_detect_impl(const omg_scrfd_desc d, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    OMG_CHECK(d.n_levels >= 1 && d.n_levels <= OMG_SCRFD_MAX_LEVELS, "omg_scrfd_detect: n_levels=%d out of range", d.n_levels);
    OMG_CHECK(d.num_anchors >= 1 && d.num_anchors <= 4, "omg_scrfd_detect: num_anchors=%d out of range", d.num_anchors);
    OMG_CHECK(d.out && d.count, "omg_scrfd_detect: null output");
    OMG_CHECK(d.det_scale > 0.f && d.nms_thresh >= 0.f, "omg_scrfd_detect: det_scale must be positive, nms_thresh >= 0");
    ScrfdLevels L;
    L.n_levels = d.n_levels;
    L.num_anchors = d.num_anchors;
    L.first[0] = 0;
    const bool with_kps = d.kps[0] != nullptr;
    for (int l = 0; l < d.n_levels; ++l) {
        OMG_CHECK(d.scores[l] && d.boxes[l], "omg_scrfd_detect: level %d has a null score or box pointer", l);
        OMG_CHECK((d.kps[l] != nullptr) == with_kps, "omg_scrfd_detect: key-points on some levels only");
        OMG_CHECK(d.stride[l] >= 1 && d.fh[l] >= 1 && d.fw[l] >= 1, "omg_scrfd_detect: level %d: bad stride or grid", l);
        const long long n = (long long)d.fh[l] * d.fw[l] * d.num_anchors;
        OMG_CHECK(L.first[l] + n <= OMG_SCRFD_MAX_ANCHORS,
                  "omg_scrfd_detect: %lld anchors exceed the %d one CTA can sort in shared memory", L.first[l] + n,
                  OMG_SCRFD_MAX_ANCHORS);
        L.scores[l] = d.scores[l];
        L.boxes[l] = d.boxes[l];
        L.kps[l] = d.kps[l];
        L.stride[l] = d.stride[l];
        L.fw[l] = d.fw[l];
        L.first[l + 1] = L.first[l] + (int)n;
    }
    const int T = L.first[d.n_levels];
    OMG_CHECK(d.max_out >= T, "omg_scrfd_detect: max_out=%d is below the %d anchors", d.max_out, T);
    const size_t smem = ((size_t)T * 13 + 15) / 16 * 16;
    static_assert((size_t)OMG_SCRFD_MAX_ANCHORS * 13 + 16 <= (size_t)kScrfdSmemLimit, "anchor cap exceeds shared memory");
    OMG_CUDA(cudaFuncSetAttribute(scrfd_detect_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    OMG_CUDA(launch_pdl(scrfd_detect_kernel, dim3(1), dim3(1024), smem, stream, L, d.det_thresh, d.nms_thresh, d.det_scale,
                        d.out, d.count));
    return check_launch("scrfd_detect_kernel");
}

// C-ABI entry points: launch, and - while this thread records a launch plan (omg_plan_record_begin) - remember the call
extern "C" int omg_channel_op(const void* x, long long ldx, void* y, long long ldy, const float* scale, const float* shift,
                              const float* slope, const void* addend, long long ld_add, int add_scale, int B, int H, int W,
                              int C, int act, int act_after_add, void* stream_) {
    const int rc = channel_op_impl(x, ldx, y, ldy, scale, shift, slope, addend, ld_add, add_scale, B, H, W, C, act,
                                   act_after_add, stream_);
    if (rc == 0 && ::omg::plan_recording())
        ::omg::plan_note([=](void* s) {
            return channel_op_impl(x, ldx, y, ldy, scale, shift, slope, addend, ld_add, add_scale, B, H, W, C, act,
                                   act_after_add, s);
        });
    return rc;
}

extern "C" int omg_pool2d(const void* x, void* y, int B, int H, int W, int C, int k, int stride, int pad, int ceil_mode,
                          int count_include_pad, int is_max, void* stream_) {
    const int rc = pool2d_impl(x, y, B, H, W, C, k, stride, pad, ceil_mode, count_include_pad, is_max, stream_);
    if (rc == 0 && ::omg::plan_recording())
        ::omg::plan_note([=](void* s) {
            return pool2d_impl(x, y, B, H, W, C, k, stride, pad, ceil_mode, count_include_pad, is_max, s);
        });
    return rc;
}

extern "C" int omg_scrfd_detect(const omg_scrfd_desc* desc, void* stream_) {
    OMG_CHECK(desc != nullptr, "omg_scrfd_detect: null descriptor");
    const omg_scrfd_desc d = *desc;
    const int rc = scrfd_detect_impl(d, stream_);
    if (rc == 0 && ::omg::plan_recording()) ::omg::plan_note([=](void* s) { return scrfd_detect_impl(d, s); });
    return rc;
}
