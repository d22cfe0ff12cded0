// Attention with decomposed relative-position bias for SAM's ViT image encoder (segment_anything Attention with
// use_rel_pos, add_decomposed_rel_pos, window_partition / window_unpartition [3P]): global attention over the 64 x 64
// token grid and 14 x 14 window attention, head_dim 64 (ViT-B/L) and 80 (ViT-H), read straight from the qkv GEMM output.
//
// CTA = one (attention group, 128-query tile, head, image), 256 threads; warpgroups 0 and 1 each own 64 query rows, as in
// attn_tc.cu.  The group is the whole grid (global) or one window; its tokens are a rectangle of the row-major grid, so Q
// and each K / V block are one 4-D TMA box (columns, x, y, image) of `Ww` x `by` tokens.  Boxes past the grid's bottom or
// right edge read zeros: those are the window padding.  An 80-column head is 160 B per row, more than one 128-B swizzle
// span, so every operand is two tiles: columns 0..63 with SWIZZLE_128B and 64..79 with SWIZZLE_32B; Q.K^T takes a fifth
// k-step from the 32-B tiles and P.V a second, 16-wide wgmma.
//
// Bias: before the key loop, each warpgroup multiplies its Q rows with both fp16 tables (Q Rh^T, Q Rw^T, wgmma, fp32
// accumulators) and scatters the products into per-row fp32 shared-memory tables bias_h[row][kh] and bias_w[row][kw]
// (get_rel_pos with equal sizes is the gather idx = q - k + S - 1).  The key loop adds bias_h + bias_w to each logit.
//
// Window padding: the reference pads the normalised input before qkv, so a padded key is k_bias and a padded value
// v_bias.  Their TMA rows are zero, so the kernel adds scale q.k_bias to a padded key's logit and, at the end,
// (sum of padded probabilities) * v_bias to the output: the same softmax, evaluated in fp32.
#include <cuda_fp16.h>

#include <algorithm>
#include <math.h>
#include <string.h>

#include "../../include/omg_b200.h"
#include "host_common.h"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace omg {

constexpr int RP_BQ = 128;      // query rows per CTA (tile slots; a window tile uses Ww * byq of them)
constexpr int RP_BKV = 64;      // key slots per block
constexpr int RP_TROWS = 128;   // table rows staged (2 * 64 - 1 at most)
constexpr int RP_STAGES = 3;
constexpr int RP_THREADS = 256;
constexpr float RP_LOG2E = 1.4426950408889634f;

template <int D>
struct RpLayout {
    static constexpr bool X = D > 64;                              // the 16 columns past the 128-B span
    static constexpr int Q64 = RP_BQ * 128;                        // Q: [128][64] sw128 | [128][16] sw32
    static constexpr int Q_BYTES = Q64 + (X ? RP_BQ * 32 : 0);
    static constexpr int K64 = RP_BKV * 128, K16 = RP_BKV * 32;
    static constexpr int STAGE = 2 * K64 + (X ? 2 * K16 : 0);     // K64 | V64 | K16 | V16
    static constexpr int T64 = RP_TROWS * 128, T16 = RP_TROWS * 32;  // tables, staged in the K/V ring before the loop:
    static constexpr int T_BYTES = 2 * T64 + (X ? 2 * T16 : 0);   // Rh64 | Rw64 | Rh16 | Rw16
    static_assert(T_BYTES <= RP_STAGES * STAGE, "tables must fit the K/V ring");
    static constexpr int FIXED = 1024 + Q_BYTES + RP_STAGES * STAGE + 8 * (2 + 2 * RP_STAGES) + 4 * RP_BKV + 4 * RP_BQ;
};

struct alignas(64) RelposParams {
    CUtensorMap q64, q16, kv64, kv16;  // 4-D (columns, x, y, image) over qkv; q: box (64 | 16, Ww, byq), kv: (.., Ww, byk)
    CUtensorMap th64, th16, tw64, tw16;  // 2-D (columns, rows) over the tables, box (64 | 16, 128)
    const __half* qkv;
    const __half* kb;
    const __half* vb;
    __half* out;
    long long bs, out_bs;
    int ld, out_ld, out_col0;
    int q_col0, k_col0, v_col0;
    int H, W, Wh, Ww;          // grid; attention group (window, or the grid itself)
    int nwx, ntiles, byq, byk, nkb;
    int sh_stride, sw_stride;  // row strides (floats) of bias_h / bias_w in shared memory
    int has_pad;
    float scale_log2;
};

static inline int rp_bias_stride(int S) {  // >= S and = 8 mod 16, so the 8 rows a warp reads at once spread over the banks
    int s = (S + 7) / 8 * 8;
    return s % 16 == 0 ? s + 8 : s;
}

template <int D>
__global__ void __launch_bounds__(RP_THREADS, 1) attn_relpos_kernel(const __grid_constant__ RelposParams p) {
    using Lt = RpLayout<D>;
    constexpr bool X = Lt::X;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* q_smem = smem;
    uint8_t* kv_smem = q_smem + Lt::Q_BYTES;
    uint64_t* q_full = reinterpret_cast<uint64_t*>(kv_smem + RP_STAGES * Lt::STAGE);
    uint64_t* t_full = q_full + 1;
    uint64_t* kv_full = q_full + 2;                 // [stage]
    uint64_t* kv_empty = kv_full + RP_STAGES;       // [stage] both warpgroups' MMAs on the stage have completed
    int* kmap = reinterpret_cast<int*>(kv_empty + RP_STAGES);  // key slot -> (row in block << 8 | x), -1 = no key
    float* qkb = reinterpret_cast<float*>(kmap + RP_BKV);      // per query row: scale log2(e) q.k_bias
    float* bias_h = qkb + RP_BQ;                                // [128][sh_stride]  log2(e) q.Rh[qh - kh + Wh - 1]
    float* bias_w = bias_h + RP_BQ * p.sh_stride;               // [128][sw_stride]  log2(e) q.Rw[qw - kw + Ww - 1]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tile = blockIdx.x % p.ntiles, grp = blockIdx.x / p.ntiles;
    const int y0 = (grp / p.nwx) * p.Wh, x0 = (grp % p.nwx) * p.Ww;  // group origin in the grid
    const int head = blockIdx.y, img = blockIdx.z;
    const int nq_box = p.Ww * p.byq, nk_box = p.Ww * p.byk;
    const int qc = p.q_col0 + head * D, kc = p.k_col0 + head * D, vc = p.v_col0 + head * D;
    const int qy_base = tile * p.byq;

    // Query slots past the box are never written by TMA: zero them so every row of the tile is finite.
    for (int i = threadIdx.x; i < (RP_BQ - nq_box) * 8; i += RP_THREADS)
        reinterpret_cast<uint4*>(q_smem + nq_box * 128)[i] = make_uint4(0, 0, 0, 0);
    if (X)
        for (int i = threadIdx.x; i < (RP_BQ - nq_box) * 2; i += RP_THREADS)
            reinterpret_cast<uint4*>(q_smem + Lt::Q64 + nq_box * 32)[i] = make_uint4(0, 0, 0, 0);
    if (threadIdx.x == 0) {
        tma_prefetch_desc(&p.q64);
        tma_prefetch_desc(&p.kv64);
        mbar_init(q_full, 1);
        mbar_init(t_full, 1);
        for (int i = 0; i < RP_STAGES; ++i) {
            mbar_init(&kv_full[i], 1);
            mbar_init(&kv_empty[i], 2);
        }
        fence_barrier_init();
    }
    if (threadIdx.x < RP_BKV) {
        const int kr = threadIdx.x;
        kmap[kr] = kr < nk_box ? ((kr / p.Ww) << 8) | (kr % p.Ww) : -1;
    }
    fence_proxy_async_smem();
    __syncthreads();
    griddep_launch_dependents();
    griddep_wait();
    if (threadIdx.x == 0) {
        mbar_arrive_expect_tx(q_full, nq_box * D * 2);
        tma_load_4d(q_smem, &p.q64, q_full, qc, x0, y0 + qy_base, img);
        if (X) tma_load_4d(q_smem + Lt::Q64, &p.q16, q_full, qc + 64, x0, y0 + qy_base, img);
        mbar_arrive_expect_tx(t_full, 2 * RP_TROWS * D * 2);
        tma_load_2d(kv_smem, &p.th64, t_full, 0, 0);
        tma_load_2d(kv_smem + Lt::T64, &p.tw64, t_full, 0, 0);
        if (X) {
            tma_load_2d(kv_smem + 2 * Lt::T64, &p.th16, t_full, 64, 0);
            tma_load_2d(kv_smem + 2 * Lt::T64 + Lt::T16, &p.tw16, t_full, 64, 0);
        }
    }
    // scale log2(e) q.k_bias for the padded keys (fp32, from the fp16 q row in global memory)
    if (p.has_pad && threadIdx.x < RP_BQ) {
        const int r = threadIdx.x;
        const int gy = y0 + qy_base + r / p.Ww, gx = x0 + r % p.Ww;
        float acc = 0.f;
        if (r < nq_box && gy < p.H && gx < p.W) {
            const __half* q = p.qkv + img * p.bs + (long long)(gy * p.W + gx) * p.ld + qc;
            const __half* kb = p.kb + head * D;
#pragma unroll 8
            for (int d = 0; d < D; ++d) acc = fmaf(__half2float(q[d]), __half2float(kb[d]), acc);
        }
        qkb[r] = acc * p.scale_log2;
    }

    const int wg = warp >> 2, wi = warp & 3;
    const int g = lane >> 2, c = lane & 3;
    const int row0 = wg * 64 + wi * 16 + g;  // this thread's rows: row0 and row0 + 8 (accumulator layout, see wgmma.cuh)
    const uint32_t q_addr = smem_u32(q_smem) + wg * (64 * 128);
    const uint32_t q16_addr = smem_u32(q_smem + Lt::Q64) + wg * (64 * 32);
    mbar_wait(q_full, 0);
    mbar_wait(t_full, 0);
    // bias tables: Q (64 rows per warpgroup) x table^T in 64-row chunks, scattered by qpos - k + S - 1 = table row
#pragma unroll 1
    for (int t = 0; t < 2; ++t) {
        const int S = t ? p.Ww : p.Wh;
        float* bias = t ? bias_w : bias_h;
        const int stride = t ? p.sw_stride : p.sh_stride;
        const uint32_t t_addr = smem_u32(kv_smem) + t * Lt::T64;
        const uint32_t t16_addr = smem_u32(kv_smem) + 2 * Lt::T64 + t * Lt::T16;
        int qpos[2];
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            const int r = row0 + 8 * hh;
            qpos[hh] = t ? r % p.Ww : min(qy_base + r / p.Ww, p.Wh - 1);  // slots outside the group: any in-range row
        }
#pragma unroll 1
        for (int ch = 0; ch * 64 < 2 * S - 1; ++ch) {
            float acc[32];
#pragma unroll
            for (int i = 0; i < 32; ++i) acc[i] = 0.f;
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k)
                wgmma_ss_n64(acc, gmma_desc_sw128(q_addr + k * 32, 1024, 16),
                             gmma_desc_sw128(t_addr + ch * 8192 + k * 32, 1024, 16), 1u);
            if (X) wgmma_ss_n64(acc, gmma_desc_sw32(q16_addr), gmma_desc_sw32(t16_addr + ch * 2048), 1u);
            wgmma_commit();
            wgmma_wait<0>();
            reg_fence(acc);
#pragma unroll
            for (int J = 0; J < 8; ++J)
#pragma unroll
                for (int hh = 0; hh < 2; ++hh)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int k = qpos[hh] + S - 1 - (ch * 64 + 8 * J + 2 * c + e);
                        if (k >= 0 && k < S) bias[(row0 + 8 * hh) * stride + k] = acc[4 * J + 2 * hh + e] * RP_LOG2E;
                    }
        }
    }
    __syncthreads();  // tables consumed: the ring is free.  Key slots past the box are never loaded: zero K and V there.
    for (int st = 0; st < RP_STAGES; ++st) {
        uint8_t* sd = kv_smem + st * Lt::STAGE;
        for (int i = threadIdx.x; i < (RP_BKV - nk_box) * 8; i += RP_THREADS) {
            reinterpret_cast<uint4*>(sd + nk_box * 128)[i] = make_uint4(0, 0, 0, 0);
            reinterpret_cast<uint4*>(sd + Lt::K64 + nk_box * 128)[i] = make_uint4(0, 0, 0, 0);
        }
        if (X)
            for (int i = threadIdx.x; i < (RP_BKV - nk_box) * 2; i += RP_THREADS) {
                reinterpret_cast<uint4*>(sd + 2 * Lt::K64 + nk_box * 32)[i] = make_uint4(0, 0, 0, 0);
                reinterpret_cast<uint4*>(sd + 2 * Lt::K64 + Lt::K16 + nk_box * 32)[i] = make_uint4(0, 0, 0, 0);
            }
    }
    fence_proxy_async_smem();
    __syncthreads();

    auto load_kv = [&](int jb) {  // thread 0: block jb into its stage, once both warpgroups have released the stage
        const int st = jb % RP_STAGES;
        mbar_wait(&kv_empty[st], ((jb / RP_STAGES) & 1) ^ 1);
        uint8_t* sd = kv_smem + st * Lt::STAGE;
        const int y = y0 + jb * p.byk;
        mbar_arrive_expect_tx(&kv_full[st], 2 * nk_box * D * 2);
        tma_load_4d(sd, &p.kv64, &kv_full[st], kc, x0, y, img);
        tma_load_4d(sd + Lt::K64, &p.kv64, &kv_full[st], vc, x0, y, img);
        if (X) {
            tma_load_4d(sd + 2 * Lt::K64, &p.kv16, &kv_full[st], kc + 64, x0, y, img);
            tma_load_4d(sd + 2 * Lt::K64 + Lt::K16, &p.kv16, &kv_full[st], vc + 64, x0, y, img);
        }
    };
    if (threadIdx.x == 0)
        for (int jb = 0; jb < RP_STAGES && jb < p.nkb; ++jb) load_kv(jb);

    const float* bh[2] = {bias_h + row0 * p.sh_stride, bias_h + (row0 + 8) * p.sh_stride};
    const float* bw[2] = {bias_w + row0 * p.sw_stride, bias_w + (row0 + 8) * p.sw_stride};
    const float qk[2] = {p.has_pad ? qkb[row0] : 0.f, p.has_pad ? qkb[row0 + 8] : 0.f};
    float o[32], o16[8];
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) o16[i] = 0.f;
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f}, lp[2] = {0.f, 0.f};  // lp: probability mass of padded keys
    for (int j = 0; j < p.nkb; ++j) {
        const int st = j % RP_STAGES;
        mbar_wait(&kv_full[st], (j / RP_STAGES) & 1);
        const uint32_t k_addr = smem_u32(kv_smem + st * Lt::STAGE);
        float s[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) s[i] = 0.f;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k)
            wgmma_ss_n64(s, gmma_desc_sw128(q_addr + k * 32, 1024, 16), gmma_desc_sw128(k_addr + k * 32, 1024, 16), 1u);
        if (X) wgmma_ss_n64(s, gmma_desc_sw32(q16_addr), gmma_desc_sw32(k_addr + 2 * Lt::K64), 1u);
        wgmma_commit();
        if (threadIdx.x == 0 && j >= 1 && j - 1 + RP_STAGES < p.nkb) load_kv(j - 1 + RP_STAGES);
        __syncwarp();
        wgmma_wait<0>();
        reg_fence(s);
        // logits in the log2 domain: scale q.k + bias_h + bias_w (+ scale q.k_bias for a padded key); no key -> -inf
        uint32_t padbits = 0;
#pragma unroll
        for (int J = 0; J < 8; ++J)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int km = kmap[8 * J + 2 * c + e];
                const int ky = j * p.byk + (km >> 8), kx = km & 255;
                const bool valid = km >= 0 && ky < p.Wh;
                const bool pad = valid && (y0 + ky >= p.H || x0 + kx >= p.W);
                padbits |= (uint32_t)pad << (2 * J + e);
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    float& v = s[4 * J + 2 * hh + e];
                    v = valid ? fmaf(v, p.scale_log2, bh[hh][ky] + bw[hh][kx] + (pad ? qk[hh] : 0.f)) : -INFINITY;
                }
            }
        float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int J = 0; J < 8; ++J)
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) mx[hh] = fmaxf(mx[hh], fmaxf(s[4 * J + 2 * hh], s[4 * J + 2 * hh + 1]));
        float corr[2];
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 1));
            mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 2));
            const float m_new = fmaxf(m[hh], mx[hh]);
            corr[hh] = fast_exp2(m[hh] - m_new);  // 0 on the first block (m = -inf)
            m[hh] = m_new;
            l[hh] *= corr[hh];
            lp[hh] *= corr[hh];
        }
#pragma unroll
        for (int J = 0; J < 8; ++J)
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
                o[4 * J + 2 * hh] *= corr[hh];
                o[4 * J + 2 * hh + 1] *= corr[hh];
            }
#pragma unroll
        for (int J = 0; J < 2; ++J)
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
                o16[4 * J + 2 * hh] *= corr[hh];
                o16[4 * J + 2 * hh + 1] *= corr[hh];
            }
        // P = exp2(logit - m) as fp16 A fragments of P.V: keys 16kk .. 16kk + 15 are accumulator chunks 2kk, 2kk + 1
        uint32_t pa[4][4];
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
#pragma unroll
            for (int t = 0; t < 4; ++t) {  // t: (row g | g + 8) x (keys 2c | 8 + 2c)
                const int hh = t & 1, J = 2 * kk + (t >> 1), i0 = 4 * J + 2 * hh;
                const float p0 = fast_exp2(s[i0] - m[hh]);
                const float p1 = fast_exp2(s[i0 + 1] - m[hh]);
                l[hh] += p0 + p1;
                if (padbits >> (2 * J) & 1u) lp[hh] += p0;
                if (padbits >> (2 * J + 1) & 1u) lp[hh] += p1;
                pa[kk][t] = pack_half2(p0, p1);
            }
        const uint32_t v_addr = k_addr + Lt::K64;
        const uint32_t v16_addr = k_addr + 2 * Lt::K64 + Lt::K16;
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {  // V: 16 key rows per K step, MN-major (2 KB of the 64-column tile, 512 B of the 16)
            wgmma_rs_n64_tb(o, pa[kk], gmma_desc_sw128(v_addr + kk * 2048, 1024, 1024), 1u);
            if (X) wgmma_rs_n16_tb(o16, pa[kk], gmma_desc_sw32(v16_addr + kk * 512), 1u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        reg_fence(o);
        if constexpr (X) reg_fence(o16);
        if ((threadIdx.x & 127) == 0) mbar_arrive(&kv_empty[st]);
    }

    // out = (O + lp v_bias) / l for the group's real tokens
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 1);
        l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 2);
        lp[hh] += __shfl_xor_sync(0xffffffffu, lp[hh], 1);
        lp[hh] += __shfl_xor_sync(0xffffffffu, lp[hh], 2);
        const int r = row0 + 8 * hh;
        const int qy = qy_base + r / p.Ww, qx = r % p.Ww;
        const int gy = y0 + qy, gx = x0 + qx;
        if (r >= nq_box || qy >= p.Wh || gy >= p.H || gx >= p.W) continue;
        const float inv = 1.f / l[hh];
        __half* op = p.out + img * p.out_bs + (long long)(gy * p.W + gx) * p.out_ld + p.out_col0 + head * D + 2 * c;
        const __half* vb = p.has_pad ? p.vb + head * D + 2 * c : nullptr;
#pragma unroll
        for (int J = 0; J < 8; ++J) {
            float v0 = o[4 * J + 2 * hh], v1 = o[4 * J + 2 * hh + 1];
            if (vb) {
                v0 = fmaf(lp[hh], __half2float(vb[8 * J]), v0);
                v1 = fmaf(lp[hh], __half2float(vb[8 * J + 1]), v1);
            }
            *reinterpret_cast<__half2*>(op + 8 * J) = __floats2half2_rn(v0 * inv, v1 * inv);
        }
        if (X)
#pragma unroll
            for (int J = 0; J < 2; ++J) {
                float v0 = o16[4 * J + 2 * hh], v1 = o16[4 * J + 2 * hh + 1];
                if (vb) {
                    v0 = fmaf(lp[hh], __half2float(vb[64 + 8 * J]), v0);
                    v1 = fmaf(lp[hh], __half2float(vb[64 + 8 * J + 1]), v1);
                }
                *reinterpret_cast<__half2*>(op + 64 + 8 * J) = __floats2half2_rn(v0 * inv, v1 * inv);
            }
    }
}

static size_t rp_smem_bytes(int D, int Wh, int Ww) {
    const size_t fixed = D > 64 ? RpLayout<80>::FIXED : RpLayout<64>::FIXED;
    return fixed + (size_t)4 * RP_BQ * (rp_bias_stride(Wh) + rp_bias_stride(Ww));
}

template <int D>
static int launch_relpos(RelposParams& p, dim3 grid, size_t smem, cudaStream_t stream) {
    static bool configured = false;
    if (!configured) {
        OMG_CUDA(cudaFuncSetAttribute(attn_relpos_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)rp_smem_bytes(D, 64, 64)));
        configured = true;
    }
    OMG_CUDA(launch_pdl(attn_relpos_kernel<D>, grid, dim3(RP_THREADS), smem, stream, p));
    return check_launch(D > 64 ? "attn_relpos_kernel<80>" : "attn_relpos_kernel<64>");
}

}  // namespace omg

using namespace omg;

static int relpos_impl(const omg_attn_relpos_desc* d, void* stream_) {
    static const char* who = "omg_attention_relpos";
    OMG_CHECK(d != nullptr, "%s: null descriptor", who);
    OMG_CHECK(d->head_dim == 64 || d->head_dim == 80, "%s: head_dim %d unsupported (SAM ViT-B/L use 64, ViT-H 80)", who,
              d->head_dim);
    OMG_CHECK(d->B >= 1 && d->H >= 1 && d->W >= 1 && d->heads >= 1, "%s: empty problem", who);
    OMG_CHECK(d->window >= 0 && d->window <= 64, "%s: window %d out of range [0, 64]", who, d->window);
    OMG_CHECK(d->window > 0 || (d->H <= 64 && d->W <= 64), "%s: global attention over a %d x %d grid (at most 64 x 64)",
              who, d->H, d->W);
    const int Wh = d->window ? d->window : d->H, Ww = d->window ? d->window : d->W;
    OMG_CHECK(d->rel_h_len == 2 * Wh - 1, "%s: rel_pos_h has %d rows, expected 2 * %d - 1 = %d (no interpolation)", who,
              d->rel_h_len, Wh, 2 * Wh - 1);
    OMG_CHECK(d->rel_w_len == 2 * Ww - 1, "%s: rel_pos_w has %d rows, expected 2 * %d - 1 = %d (no interpolation)", who,
              d->rel_w_len, Ww, 2 * Ww - 1);
    OMG_CHECK(d->qkv && d->out && d->rel_pos_h && d->rel_pos_w, "%s: null pointer", who);
    const bool pad = d->window > 0 && (d->H % d->window || d->W % d->window);
    OMG_CHECK(!pad || (d->k_bias && d->v_bias),
              "%s: a %d x %d grid in windows of %d is padded: k_bias and v_bias (the padded tokens' key and value) are "
              "required", who, d->H, d->W, d->window);
    OMG_CHECK(((uintptr_t)d->qkv & 15) == 0 && d->ld % 8 == 0 && d->bs % 8 == 0,
              "%s: qkv rows must be 16 B aligned (pointer, ld, bs)", who);
    OMG_CHECK(((uintptr_t)d->rel_pos_h & 15) == 0 && ((uintptr_t)d->rel_pos_w & 15) == 0,
              "%s: rel-pos tables must be 16 B aligned", who);
    OMG_CHECK(((uintptr_t)d->out & 15) == 0 && d->out_ld % 8 == 0 && d->out_col0 % 8 == 0 && d->out_bs % 8 == 0,
              "%s: output must be 16 B aligned per row", who);
    if (check_head_windows(who, d->heads, d->head_dim, {d->q_col0, d->k_col0, d->v_col0, d->out_col0},
                           {d->ld, d->ld, d->ld, d->out_ld}))
        return 1;

    const int D = d->head_dim;
    RelposParams p;
    memset(&p, 0, sizeof(p));
    const int byq = std::min(RP_BQ / Ww, Wh), byk = std::min(RP_BKV / Ww, Wh);
    const uint64_t dims[4] = {(uint64_t)d->ld, (uint64_t)d->W, (uint64_t)d->H, (uint64_t)d->B};
    const uint64_t strides[4] = {1, (uint64_t)d->ld, (uint64_t)d->ld * d->W, (uint64_t)d->bs};
    const uint32_t bq64[4] = {64, (uint32_t)Ww, (uint32_t)byq, 1}, bq16[4] = {16, (uint32_t)Ww, (uint32_t)byq, 1};
    const uint32_t bk64[4] = {64, (uint32_t)Ww, (uint32_t)byk, 1}, bk16[4] = {16, (uint32_t)Ww, (uint32_t)byk, 1};
    const auto F16 = CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
    if (make_tmap(&p.q64, F16, d->qkv, 4, dims, strides, bq64, CU_TENSOR_MAP_SWIZZLE_128B)) return 1;
    if (make_tmap(&p.kv64, F16, d->qkv, 4, dims, strides, bk64, CU_TENSOR_MAP_SWIZZLE_128B)) return 1;
    const uint64_t th_dims[2] = {(uint64_t)D, (uint64_t)d->rel_h_len}, tw_dims[2] = {(uint64_t)D, (uint64_t)d->rel_w_len};
    const uint64_t t_str[2] = {1, (uint64_t)D};
    const uint32_t bt64[2] = {64, RP_TROWS}, bt16[2] = {16, RP_TROWS};
    if (make_tmap(&p.th64, F16, d->rel_pos_h, 2, th_dims, t_str, bt64, CU_TENSOR_MAP_SWIZZLE_128B)) return 1;
    if (make_tmap(&p.tw64, F16, d->rel_pos_w, 2, tw_dims, t_str, bt64, CU_TENSOR_MAP_SWIZZLE_128B)) return 1;
    if (D > 64) {
        if (make_tmap(&p.q16, F16, d->qkv, 4, dims, strides, bq16, CU_TENSOR_MAP_SWIZZLE_32B)) return 1;
        if (make_tmap(&p.kv16, F16, d->qkv, 4, dims, strides, bk16, CU_TENSOR_MAP_SWIZZLE_32B)) return 1;
        if (make_tmap(&p.th16, F16, d->rel_pos_h, 2, th_dims, t_str, bt16, CU_TENSOR_MAP_SWIZZLE_32B)) return 1;
        if (make_tmap(&p.tw16, F16, d->rel_pos_w, 2, tw_dims, t_str, bt16, CU_TENSOR_MAP_SWIZZLE_32B)) return 1;
    }
    p.qkv = static_cast<const __half*>(d->qkv);
    p.kb = static_cast<const __half*>(d->k_bias);
    p.vb = static_cast<const __half*>(d->v_bias);
    p.out = static_cast<__half*>(d->out);
    p.bs = d->bs;
    p.out_bs = d->out_bs;
    p.ld = d->ld;
    p.out_ld = d->out_ld;
    p.out_col0 = d->out_col0;
    p.q_col0 = d->q_col0;
    p.k_col0 = d->k_col0;
    p.v_col0 = d->v_col0;
    p.H = d->H;
    p.W = d->W;
    p.Wh = Wh;
    p.Ww = Ww;
    p.nwx = (d->W + Ww - 1) / Ww;
    p.byq = byq;
    p.byk = byk;
    p.ntiles = (Wh + byq - 1) / byq;
    p.nkb = (Wh + byk - 1) / byk;
    p.sh_stride = rp_bias_stride(Wh);
    p.sw_stride = rp_bias_stride(Ww);
    p.has_pad = pad;
    p.scale_log2 = d->scale * RP_LOG2E;
    const int nwy = (d->H + Wh - 1) / Wh;
    const dim3 grid(nwy * p.nwx * p.ntiles, d->heads, d->B);
    const size_t smem = rp_smem_bytes(D, Wh, Ww);
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    return D > 64 ? launch_relpos<80>(p, grid, smem, stream) : launch_relpos<64>(p, grid, smem, stream);
}

extern "C" int omg_attention_relpos(const omg_attn_relpos_desc* d, void* stream_) {
    const int rc = relpos_impl(d, stream_);
    if (rc == 0 && ::omg::plan_recording()) {
        const omg_attn_relpos_desc c = *d;  // by value: a plan outlives the caller's descriptor
        ::omg::plan_note([c](void* s) { return relpos_impl(&c, s); });
    }
    return rc;
}
