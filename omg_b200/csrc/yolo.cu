// Kernels of the YOLO-World open-vocabulary detector (ultralytics WorldModel, the `--segment_type yoloworld` box source
// of both OMG CLIs, reference inference_lora.py:91-126) that are not GEMM-shaped.  Its convolutions, linears and the
// pooling attention's 27-key attention run on gemm_tc.cu / attn_tc.cu; what is left is
//   - text_gate: MaxSigmoidAttnBlock after its convs - the per-head max over the class prompts of the image-text
//     similarity, sigmoid, and the gating of proj_conv's output;
//   - adaptive_maxpool: ImagePoolingAttn's AdaptiveMaxPool2d((k, k)) into the rows of its key buffer;
//   - yolo_detect: WorldDetect's contrastive class scores, DFL and box decode per anchor, then threshold, sort,
//     greedy NMS and the letterbox-to-image rescale of ultralytics' non_max_suppression / scale_boxes in one CTA.
// Channels-last fp16 storage, fp32 arithmetic.  All of these are memory- or latency-bound and run once per image.
#include <cuda_fp16.h>

#include "../../include/omg_b200.h"
#include "host_common.h"
#include "ptx.cuh"

namespace omg {

// ------------------------------------------------------------------------------------------------------ text_gate
// block = up to 256 threads over P = 256 / nh pixels of one image (blockIdx.y).  The image's guide lives in shared
// memory as [n][hc][nh] so the nh threads of one pixel read consecutive words.  Phase 1: thread (pixel, head) takes the
// max over the n prompts of <embed_h, guide_h>, then / sqrt(hc), + bias, sigmoid, * scale.  Phase 2: out = p * gate.
template <int HC>
__global__ void __launch_bounds__(256) text_gate_kernel(const __half* __restrict__ embed, long long ld_e,
                                                        const float* __restrict__ guide, int n,
                                                        const float* __restrict__ bias, const float* __restrict__ scale,
                                                        int nh, const __half* p, long long ld_p, __half* out,
                                                        long long ld_o, int C2, int HW, float inv_sqrt_hc) {
    griddep_launch_dependents();
    griddep_wait();
    extern __shared__ __align__(16) float gsm[];        // [n][HC][nh], then gate[P][nh]
    const int Ce = HC * nh;
    const int b = blockIdx.y;
    const int P = 256 / nh;
    float* gate = gsm + (size_t)n * Ce;
    const float* g = guide + (size_t)b * n * Ce;
    for (int i = threadIdx.x; i < n * Ce; i += blockDim.x) {
        const int k = i / Ce, c = i - k * Ce;
        const int h = c / HC, j = c - h * HC;
        gsm[((size_t)k * HC + j) * nh + h] = g[i];
    }
    __syncthreads();
    const int pix0 = blockIdx.x * P;
    {
        const int lp = threadIdx.x / nh, h = threadIdx.x - lp * nh;
        const int pix = pix0 + lp;
        if (lp < P && pix < HW) {
            float e[HC];
            const __half* ep = embed + ((size_t)b * HW + pix) * ld_e + h * HC;
#pragma unroll
            for (int v = 0; v < HC / 8; ++v) {
                const uint4 u = *reinterpret_cast<const uint4*>(ep + v * 8);
                const __half* hh = reinterpret_cast<const __half*>(&u);
#pragma unroll
                for (int i = 0; i < 8; ++i) e[v * 8 + i] = __half2float(hh[i]);
            }
            float best = -INFINITY;
            for (int k = 0; k < n; ++k) {
                const float* gk = gsm + (size_t)k * HC * nh + h;
                float s = 0.f;
#pragma unroll
                for (int j = 0; j < HC; ++j) s = fmaf(e[j], gk[j * nh], s);
                best = fmaxf(best, s);
            }
            const float a = best * inv_sqrt_hc + bias[h];
            float gv = 1.f / (1.f + expf(-a));
            if (scale != nullptr) gv *= scale[h];
            gate[lp * nh + h] = gv;
        }
    }
    __syncthreads();
    const int vpr = C2 / 8, grp = C2 / nh;
    for (int i = threadIdx.x; i < P * vpr; i += blockDim.x) {
        const int lp = i / vpr, c0 = (i - lp * vpr) * 8;
        const int pix = pix0 + lp;
        if (pix >= HW) break;
        const size_t row = (size_t)b * HW + pix;
        const uint4 u = *reinterpret_cast<const uint4*>(p + row * ld_p + c0);
        const __half* hh = reinterpret_cast<const __half*>(&u);
        uint4 o;
        __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float g0 = gate[lp * nh + (c0 + 2 * j) / grp], g1 = gate[lp * nh + (c0 + 2 * j + 1) / grp];
            oh[j] = __floats2half2_rn(__half2float(hh[2 * j]) * g0, __half2float(hh[2 * j + 1]) * g1);
        }
        *reinterpret_cast<uint4*>(out + row * ld_o + c0) = o;
    }
}

// ------------------------------------------------------------------------------------------------ adaptive_maxpool
// PyTorch's adaptive windows: rows [floor(i H / k), ceil((i + 1) H / k)), likewise for columns.  thread = 8 channels
// of one (image, patch); patch i * k + j goes to row row0 + i * k + j of the image's [patches, C] block.
__global__ void adaptive_maxpool_kernel(const __half* __restrict__ x, long long ldx, int H, int W, int C, int k,
                                        __half* __restrict__ out, long long out_bs, long long out_ld, int row0,
                                        long long total) {
    griddep_launch_dependents();
    griddep_wait();
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const int vpr = C / 8;
    const int c0 = (int)(idx % vpr) * 8;
    const long long r = idx / vpr;
    const int patch = (int)(r % (k * k));
    const long long b = r / (k * k);
    const int pi = patch / k, pj = patch - pi * k;
    const int h0 = pi * H / k, h1 = ((pi + 1) * H + k - 1) / k;
    const int w0 = pj * W / k, w1 = ((pj + 1) * W + k - 1) / k;
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = -INFINITY;
    for (int iy = h0; iy < h1; ++iy)
        for (int ix = w0; ix < w1; ++ix) {
            const uint4 u = *reinterpret_cast<const uint4*>(x + ((b * H + iy) * W + ix) * ldx + c0);
            const __half* h = reinterpret_cast<const __half*>(&u);
#pragma unroll
            for (int i = 0; i < 8; ++i) acc[i] = fmaxf(acc[i], __half2float(h[i]));
        }
    uint4 u;
    __half2* h = reinterpret_cast<__half2*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(acc[2 * i], acc[2 * i + 1]);
    *reinterpret_cast<uint4*>(out + b * out_bs + (long long)(row0 + patch) * out_ld + c0) = u;
}

// ------------------------------------------------------------------------------------------------------ yolo_detect
struct YoloLevels {
    const __half* box[OMG_YOLO_MAX_LEVELS];
    const __half* emb[OMG_YOLO_MAX_LEVELS];
    long long box_ld[OMG_YOLO_MAX_LEVELS], emb_ld[OMG_YOLO_MAX_LEVELS];
    float cls_scale[OMG_YOLO_MAX_LEVELS], cls_bias[OMG_YOLO_MAX_LEVELS];
    int stride[OMG_YOLO_MAX_LEVELS], fw[OMG_YOLO_MAX_LEVELS], first[OMG_YOLO_MAX_LEVELS + 1];
    int n_levels;
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// pass (a): one warp per anchor.  rows[g] = [x0, y0, x1, y1 (letterbox pixels), max sigmoid score, argmax class].
__global__ void __launch_bounds__(256) yolo_anchor_kernel(YoloLevels L, const float* __restrict__ text, int nc, int E,
                                                          int normalize_x, float* __restrict__ rows) {
    griddep_launch_dependents();
    griddep_wait();
    extern __shared__ __align__(16) float xs[];    // [warps][E]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int g = blockIdx.x * (blockDim.x >> 5) + warp;
    const int T = L.first[L.n_levels];
    if (g >= T) return;
    int l = 0;
    while (g >= L.first[l + 1]) ++l;
    const int a = g - L.first[l];
    float* x = xs + (size_t)warp * E;
    const __half* ep = L.emb[l] + (size_t)a * L.emb_ld[l];
    float ss = 0.f;
    for (int c = lane; c < E; c += 32) {
        const float v = __half2float(ep[c]);
        x[c] = v;
        ss = fmaf(v, v, ss);
    }
    __syncwarp();
    float inv = 1.f;
    if (normalize_x) inv = 1.f / fmaxf(sqrtf(warp_sum(ss)), 1e-12f);   // F.normalize(x, dim=1)
    float best = -1.f;
    int best_k = 0;
    for (int k = 0; k < nc; ++k) {
        const float* t = text + (size_t)k * E;
        float s = 0.f;
        for (int c = lane; c < E; c += 32) s = fmaf(x[c], t[c], s);
        s = warp_sum(s);
        const float logit = (s * inv) * L.cls_scale[l] + L.cls_bias[l];
        const float p = 1.f / (1.f + expf(-logit));
        if (p > best) {       // the first class of the largest score
            best = p;
            best_k = k;
        }
    }
    // DFL: lane i < 4 takes side i (l, t, r, b): softmax over 16 bins, expectation of the bin index
    float d = 0.f;
    if (lane < 4) {
        const __half* bp = L.box[l] + (size_t)a * L.box_ld[l] + lane * 16;
        float v[16], m = -INFINITY;
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            v[i] = __half2float(bp[i]);
            m = fmaxf(m, v[i]);
        }
        float s0 = 0.f, s1 = 0.f;
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            const float e = expf(v[i] - m);
            s0 += e;
            s1 = fmaf(e, (float)i, s1);
        }
        d = s1 / s0;
    }
    const float dl = __shfl_sync(0xffffffffu, d, 0), dt = __shfl_sync(0xffffffffu, d, 1);
    const float dr = __shfl_sync(0xffffffffu, d, 2), db = __shfl_sync(0xffffffffu, d, 3);
    if (lane == 0) {
        const int cell = a, fw = L.fw[l];
        const float ax = (float)(cell % fw) + 0.5f, ay = (float)(cell / fw) + 0.5f;
        const float sf = (float)L.stride[l];
        // dist2bbox(xywh=True) * stride, then xywh2xyxy, as ultralytics computes them in fp32
        const float x1 = __fsub_rn(ax, dl), y1 = __fsub_rn(ay, dt), x2 = __fadd_rn(ax, dr), y2 = __fadd_rn(ay, db);
        const float cx = __fmul_rn(__fmul_rn(__fadd_rn(x1, x2), 0.5f), sf);
        const float cy = __fmul_rn(__fmul_rn(__fadd_rn(y1, y2), 0.5f), sf);
        const float w = __fmul_rn(__fsub_rn(x2, x1), sf), h = __fmul_rn(__fsub_rn(y2, y1), sf);
        float* r = rows + (size_t)g * 6;
        r[0] = __fsub_rn(cx, __fmul_rn(w, 0.5f));
        r[1] = __fsub_rn(cy, __fmul_rn(h, 0.5f));
        r[2] = __fadd_rn(cx, __fmul_rn(w, 0.5f));
        r[3] = __fadd_rn(cy, __fmul_rn(h, 0.5f));
        r[4] = best;
        r[5] = (float)best_k;
    }
}

struct YoloNms {
    float conf, iou, max_wh, gain, pad_x, pad_y, clip_w, clip_h;
    int agnostic, max_det, T;
};

__device__ __forceinline__ void nms_box(const float* rows, int g, float off, float (&b)[4]) {
#pragma unroll
    for (int i = 0; i < 4; ++i) b[i] = __fadd_rn(rows[(size_t)g * 6 + i], off);
}

__device__ __forceinline__ float box_area(const float (&b)[4]) {
    return __fmul_rn(__fsub_rn(b[2], b[0]), __fsub_rn(b[3], b[1]));
}

// pass (b), one CTA: score > conf, rank sort (descending score, ties: lower anchor index first), greedy NMS on boxes
// offset by class * max_wh (0 when agnostic; torchvision IoU, suppress when IoU > iou), at most max_det rows, then
// scale_boxes: (box - pad) / gain clipped to the image.
__global__ void __launch_bounds__(1024) yolo_nms_kernel(const float* __restrict__ rows, YoloNms P,
                                                        float* __restrict__ out, int* __restrict__ count) {
    griddep_launch_dependents();
    griddep_wait();
    extern __shared__ __align__(16) unsigned char smem[];
    const int T = P.T;
    float* key = reinterpret_cast<float*>(smem);
    int* gid = reinterpret_cast<int*>(key + T);
    int* order = gid + T;
    unsigned char* supp = reinterpret_cast<unsigned char*>(order + T);
    __shared__ int n_cand, n_keep;
    if (threadIdx.x == 0) n_cand = n_keep = 0;
    __syncthreads();
    for (int g = threadIdx.x; g < T; g += blockDim.x) {
        const float s = rows[(size_t)g * 6 + 4];
        if (s > P.conf) {
            const int slot = atomicAdd(&n_cand, 1);
            key[slot] = s;
            gid[slot] = g;
        }
    }
    __syncthreads();
    const int n = n_cand;
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
    for (int p = 0; p < n && n_keep < P.max_det; ++p) {   // n_keep changes only before the barrier that ends an iteration
        if (supp[p]) continue;
        const int gp = order[p];
        const float cls_p = rows[(size_t)gp * 6 + 5];
        float bp[4];
        nms_box(rows, gp, P.agnostic ? 0.f : __fmul_rn(cls_p, P.max_wh), bp);
        const float ap = box_area(bp);
        __syncthreads();    // every thread has read n_keep for this iteration's loop test
        if (threadIdx.x == 0) {
            float* o = out + (size_t)n_keep * 6;
            const float* r = rows + (size_t)gp * 6;
            const float px[4] = {P.pad_x, P.pad_y, P.pad_x, P.pad_y};
            const float lim[4] = {P.clip_w, P.clip_h, P.clip_w, P.clip_h};
#pragma unroll
            for (int i = 0; i < 4; ++i) o[i] = fminf(fmaxf(__fdiv_rn(__fsub_rn(r[i], px[i]), P.gain), 0.f), lim[i]);
            o[4] = r[4];
            o[5] = cls_p;
            ++n_keep;
        }
        for (int q = p + 1 + threadIdx.x; q < n; q += blockDim.x) {
            if (supp[q]) continue;
            const int gq = order[q];
            float bq[4];
            nms_box(rows, gq, P.agnostic ? 0.f : __fmul_rn(rows[(size_t)gq * 6 + 5], P.max_wh), bq);
            const float xx1 = fmaxf(bp[0], bq[0]), yy1 = fmaxf(bp[1], bq[1]);
            const float xx2 = fminf(bp[2], bq[2]), yy2 = fminf(bp[3], bq[3]);
            const float inter = __fmul_rn(fmaxf(0.f, __fsub_rn(xx2, xx1)), fmaxf(0.f, __fsub_rn(yy2, yy1)));
            const float iou = __fdiv_rn(inter, __fsub_rn(__fadd_rn(ap, box_area(bq)), inter));
            if (iou > P.iou) supp[q] = 1;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) *count = n_keep;
}

}  // namespace omg

using namespace omg;

static constexpr int kSmemLimit = 232448;  // sm_90 opt-in shared memory per block (227 KB)

static int text_gate_impl(const void* embed, long long ld_e, int Ce, const float* guide, int n, const float* bias,
                          const float* scale, int nh, const void* p, long long ld_p, void* out, long long ld_o, int C2,
                          int B, int HW, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    OMG_CHECK(B >= 1 && HW >= 1 && n >= 1, "omg_text_gate: bad shape B=%d HW=%d n=%d (n >= 1 prompts)", B, HW, n);
    OMG_CHECK(embed && guide && bias && p && out, "omg_text_gate: null pointer");
    OMG_CHECK(nh >= 1 && nh <= 256, "omg_text_gate: nh=%d out of range (1..256)", nh);
    OMG_CHECK(Ce % nh == 0 && C2 % nh == 0, "omg_text_gate: Ce=%d and C2=%d must be multiples of nh=%d", Ce, C2, nh);
    const int hc = Ce / nh;
    OMG_CHECK(hc == 16 || hc == 32 || hc == 64, "omg_text_gate: head channels Ce / nh = %d (16, 32 or 64)", hc);
    OMG_CHECK(C2 % 8 == 0 && ld_e % 8 == 0 && ld_p % 8 == 0 && ld_o % 8 == 0 && ld_e >= Ce && ld_p >= C2 && ld_o >= C2,
              "omg_text_gate: C2 and the row strides must be multiples of 8 and cover the rows");
    if (check_aligned("omg_text_gate", 16, {{"embed", embed}, {"p", p}, {"out", out}})) return 1;
    const int P = 256 / nh;
    const size_t smem = ((size_t)n * Ce + (size_t)P * nh) * sizeof(float);
    OMG_CHECK(smem <= (size_t)kSmemLimit, "omg_text_gate: n * Ce = %lld guide floats exceed shared memory",
              (long long)n * Ce);
    auto k = hc == 16 ? text_gate_kernel<16> : hc == 32 ? text_gate_kernel<32> : text_gate_kernel<64>;
    OMG_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const dim3 grid((unsigned)((HW + P - 1) / P), (unsigned)B);
    OMG_CUDA(launch_pdl(k, grid, dim3(256), smem, stream, static_cast<const __half*>(embed), ld_e, guide, n, bias, scale,
                        nh, static_cast<const __half*>(p), ld_p, static_cast<__half*>(out), ld_o, C2, HW,
                        1.f / sqrtf((float)hc)));
    return check_launch("text_gate_kernel");
}

static int adaptive_maxpool_impl(const void* x, long long ldx, int B, int H, int W, int C, int k, void* out,
                                 long long out_bs, long long out_ld, int row0, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    OMG_CHECK(x && out, "omg_adaptive_maxpool: null pointer");
    if (check_aligned("omg_adaptive_maxpool", 16, {{"x", x}, {"out", out}})) return 1;
    OMG_CHECK(B >= 1 && H >= 1 && W >= 1 && k >= 1 && C >= 8 && C % 8 == 0,
              "omg_adaptive_maxpool: bad shape (B=%d H=%d W=%d k=%d, C=%d a multiple of 8)", B, H, W, k, C);
    OMG_CHECK(ldx % 8 == 0 && ldx >= C && out_ld % 8 == 0 && out_ld >= C && out_bs % 8 == 0 && row0 >= 0 &&
                  out_bs >= (long long)(row0 + k * k) * out_ld,
              "omg_adaptive_maxpool: row strides must be multiples of 8 that hold the rows");
    const long long total = (long long)B * k * k * (C / 8);
    OMG_CUDA(launch_pdl(adaptive_maxpool_kernel, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, stream,
                        static_cast<const __half*>(x), ldx, H, W, C, k, static_cast<__half*>(out), out_bs, out_ld, row0,
                        total));
    return check_launch("adaptive_maxpool_kernel");
}

static int yolo_detect_impl(const omg_yolo_desc d, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    OMG_CHECK(d.n_levels >= 1 && d.n_levels <= OMG_YOLO_MAX_LEVELS, "omg_yolo_detect: n_levels=%d out of range", d.n_levels);
    OMG_CHECK(d.nc >= 1 && d.nc <= OMG_YOLO_MAX_CLASSES, "omg_yolo_detect: nc=%d out of range (1..%d)", d.nc,
              OMG_YOLO_MAX_CLASSES);
    OMG_CHECK(d.text && d.rows, "omg_yolo_detect: null text or rows");
    OMG_CHECK(d.E >= 32 && d.E <= 1024 && d.E % 8 == 0, "omg_yolo_detect: E=%d (32..1024, a multiple of 8)", d.E);
    YoloLevels L;
    L.n_levels = d.n_levels;
    L.first[0] = 0;
    for (int l = 0; l < d.n_levels; ++l) {
        OMG_CHECK(d.box[l] && d.emb[l], "omg_yolo_detect: level %d has a null box or embedding pointer", l);
        OMG_CHECK(d.stride[l] >= 1 && d.fh[l] >= 1 && d.fw[l] >= 1, "omg_yolo_detect: level %d: bad stride or grid", l);
        OMG_CHECK(d.box_ld[l] >= 4 * OMG_YOLO_REG_MAX && d.emb_ld[l] >= d.E,
                  "omg_yolo_detect: level %d: row strides below 64 box / E embedding channels", l);
        const long long n = (long long)d.fh[l] * d.fw[l];
        OMG_CHECK(L.first[l] + n <= OMG_YOLO_MAX_ANCHORS,
                  "omg_yolo_detect: %lld anchors exceed the %d one CTA can sort in shared memory", L.first[l] + n,
                  OMG_YOLO_MAX_ANCHORS);
        L.box[l] = static_cast<const __half*>(d.box[l]);
        L.emb[l] = static_cast<const __half*>(d.emb[l]);
        L.box_ld[l] = d.box_ld[l];
        L.emb_ld[l] = d.emb_ld[l];
        L.cls_scale[l] = d.cls_scale[l];
        L.cls_bias[l] = d.cls_bias[l];
        L.stride[l] = d.stride[l];
        L.fw[l] = d.fw[l];
        L.first[l + 1] = L.first[l] + (int)n;
    }
    const int T = L.first[d.n_levels];
    const int warps = 8;
    OMG_CUDA(launch_pdl(yolo_anchor_kernel, dim3((unsigned)((T + warps - 1) / warps)), dim3(32 * warps),
                        (size_t)warps * d.E * sizeof(float), stream, L, d.text, d.nc, d.E, d.normalize_x ? 1 : 0, d.rows));
    if (check_launch("yolo_anchor_kernel")) return 1;
    if (d.out == nullptr) return 0;   // pass (a) only
    OMG_CHECK(d.count, "omg_yolo_detect: null count");
    OMG_CHECK(d.max_det >= 0 && d.max_out >= d.max_det, "omg_yolo_detect: max_out=%d below max_det=%d", d.max_out, d.max_det);
    OMG_CHECK(d.gain > 0.f && d.iou >= 0.f && d.clip_w > 0.f && d.clip_h > 0.f,
              "omg_yolo_detect: gain and the clip extent must be positive, iou >= 0");
    YoloNms P{d.conf, d.iou, d.max_wh, d.gain, d.pad_x, d.pad_y, d.clip_w, d.clip_h, d.agnostic ? 1 : 0, d.max_det, T};
    const size_t smem = ((size_t)T * 13 + 15) / 16 * 16;
    static_assert((size_t)OMG_YOLO_MAX_ANCHORS * 13 + 16 <= (size_t)kSmemLimit, "anchor cap exceeds shared memory");
    OMG_CUDA(cudaFuncSetAttribute(yolo_nms_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    OMG_CUDA(launch_pdl(yolo_nms_kernel, dim3(1), dim3(1024), smem, stream, (const float*)d.rows, P, d.out, d.count));
    return check_launch("yolo_nms_kernel");
}

// C-ABI entry points: launch, and - while this thread records a launch plan (omg_plan_record_begin) - remember the call
extern "C" int omg_text_gate(const void* embed, long long ld_e, int Ce, const float* guide, int n, const float* bias,
                             const float* scale, int nh, const void* p, long long ld_p, void* out, long long ld_o, int C2,
                             int B, int HW, void* stream_) {
    const int rc = text_gate_impl(embed, ld_e, Ce, guide, n, bias, scale, nh, p, ld_p, out, ld_o, C2, B, HW, stream_);
    if (rc == 0 && ::omg::plan_recording())
        ::omg::plan_note([=](void* s) {
            return text_gate_impl(embed, ld_e, Ce, guide, n, bias, scale, nh, p, ld_p, out, ld_o, C2, B, HW, s);
        });
    return rc;
}

extern "C" int omg_adaptive_maxpool(const void* x, long long ldx, int B, int H, int W, int C, int k, void* out,
                                    long long out_bs, long long out_ld, int row0, void* stream_) {
    const int rc = adaptive_maxpool_impl(x, ldx, B, H, W, C, k, out, out_bs, out_ld, row0, stream_);
    if (rc == 0 && ::omg::plan_recording())
        ::omg::plan_note([=](void* s) { return adaptive_maxpool_impl(x, ldx, B, H, W, C, k, out, out_bs, out_ld, row0, s); });
    return rc;
}

extern "C" int omg_yolo_detect(const omg_yolo_desc* desc, void* stream_) {
    OMG_CHECK(desc != nullptr, "omg_yolo_detect: null descriptor");
    const omg_yolo_desc d = *desc;
    const int rc = yolo_detect_impl(d, stream_);
    if (rc == 0 && ::omg::plan_recording()) ::omg::plan_note([=](void* s) { return yolo_detect_impl(d, s); });
    return rc;
}
