// Persistent wgmma implicit-GEMM for every Linear / Conv2d / LoRA / GEGLU of the SDXL UNet.
//
//   out[pix, n] = epi( sum_seg sum_k A_seg[pix + (dx,dy), k] * W[n, b_k0 + k] + bias[n] + rowvec[b, n] ) + residual
//
// * Activations are channels-last, so a 3x3 conv is 9 K-segments whose A tiles are the SAME tensor read
//   through TMA at shifted pixel coordinates (hardware zero-fill = padding); no im2col buffer exists.
//   Stride-2 convs and nearest-2x-upsample convs use strided "phase" views of the tensor as A / D maps.
//   A ResBlock's 1x1 shortcut and a LoRA delta  s*B(Ax)  are just more K-segments of the same accumulator.
// * One CTA per SM, 384 threads: warps 0..7 are two consumer warpgroups (wgmma issue, then the epilogue straight
//   from the register accumulators), one thread of warpgroup 2 is the TMA producer (setmaxnreg moves that
//   warpgroup's registers to the consumers: the 128 x 256 accumulator is 128 registers per thread).  The producer runs ahead through a ring of shared-
//   memory stages, also into the next tile while the consumers are in the epilogue of the current one.
// * Tile 128 (pixels) x BN (channels) x 64 (K); warpgroup w owns rows 64w..64w+63.  MT = 2 ("tall tile") stacks two
//   128-row m-tiles that share every weight tile: warpgroup w then owns m-tile w (two m64 blocks).  Operands land in
//   shared memory in the 128B-swizzled K-major layout the GMMA descriptors expect.
//
// Roofline: tensor-bound; algorithmic FLOPs per launch = 2 * pixels * N * sum(k_len).
#include <cuda_fp16.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>

#include "../../include/omg_b200.h"
#include "host_common.h"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace omg {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int GEMM_THREADS = 384;  // warpgroups 0, 1: MMA + epilogue; warpgroup 2: TMA (one thread)

struct SegDev {
    int a_map, dx, dy, a_c0, k_blocks, b_k0, b_map;
};

struct alignas(64) GemmParams {
    CUtensorMap a_maps[OMG_MAX_A];
    CUtensorMap b_maps[2];
    SegDev segs[OMG_MAX_SEGS];
    int n_segs;
    int m_tiles, n_tiles;
    int tw, th, tiles_w, tiles_h;
    int img_w, img_h, img_b;
    int N, N_out;
    __half* out;               // output view (channels-last, element strides)
    long long out_sw, out_sh, out_sb;
    const __half* bias;
    const __half* rowvec;
    int rowvec_ld;
    const __half* residual;
    int residual_ld;
    int act_silu;
    // LayerNorm folded into the GEMM pair (see omg_gemm_desc): statistics written by the producer's epilogue ...
    float* stats_out;          // [n_tiles][rows][2] partial (sum, sum of squares) of this GEMM's output rows, or null
    // ... and consumed by the next GEMM's epilogue: out = rstd * (acc - mean * c1[n]) + c2[n]
    const float* stats_in;     // [stats_parts][rows][2] or null
    int stats_parts;
    long long stats_rows;      // rows per part (both directions)
    float ln_inv_dim, ln_eps;
    const float* col_c1;       // [N] fp32: row sums of the gamma-folded weights
    const float* col_c2;       // [N] fp32: W beta + bias
    int n_col_groups;          // c1/c2 are [n_col_groups][N]; row group g = rows [col_group_end[g-1], col_group_end[g])
    long long col_group_end[8];
    int w_group_rows;          // > 0: the weight matrix holds one [N, K] plane per row group (per-stream merged LoRA)
    // fp32 master copy of the residual trunk: the addend is read from / the result also written to fp32 twins, so the
    // chain h <- h + f(h) accumulates in fp32 while every GEMM / norm input stays the fp16 copy
    const float* residual_f32;
    long long residual_f32_ld;
    float* out_f32;
    long long out_f32_ld;
    float4* col_stats;         // GroupNorm statistics of the output: [B][cs_rb_total][N] float2 (sum, sumsq), or null
    int cs_rb0, cs_rb_total;
};

// BN = 320: two N = 160 wgmmas per K step into one 320-column accumulator (wgmma N <= 256).
// MT = 2: a 256 x BN work unit of two 128-row m-tiles; each consumer warpgroup holds the accumulator of one of them.
// CS: the epilogue can emit GroupNorm column statistics (FEAT >= 1); only then is their exchange buffer reserved, so the
// lean instantiations keep that shared memory for pipeline stages.
template <int BN, int MT, bool CS>
struct GemmCfg {
    static constexpr int WN = BN > 256 ? BN / 2 : BN;  // N of one wgmma
    static constexpr int NW = BN / WN;                  // wgmmas per m64 block and K = 16 step
    static constexpr int ACC = MT * BN / 2;             // fp32 accumulators per thread
    static constexpr int A_BYTES = MT * BM * BK * 2;
    static constexpr int B_BYTES = BN * BK * 2;
    static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
    static constexpr int VEC_BYTES = 2 * MT * BN * 4;     // per-column epilogue vectors (bias | c1), one plane per m-tile
    static constexpr int CS_BYTES = CS ? 8 * MT * BN * 8 : 0;  // column-statistics exchange: one float4 per column pair and warp
    static constexpr int BARS_BYTES = 256;
    static constexpr int BUDGET = 227 * 1024 - 1024 /*alignment slack*/ - VEC_BYTES - CS_BYTES - BARS_BYTES;
    static constexpr int STAGES_RAW = BUDGET / STAGE_BYTES;
    static constexpr int STAGES = STAGES_RAW > 8 ? 8 : STAGES_RAW;
    static constexpr int SMEM_BYTES = 1024 + STAGES * STAGE_BYTES + VEC_BYTES + CS_BYTES + BARS_BYTES;
    static_assert(STAGES >= 2, "shared memory budget");
};

// GEGLU / erf-GELU use libdevice's erff.
__device__ __forceinline__ float gelu_exact(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f)); }

template <int WN>
__device__ __forceinline__ void wgmma_ss(float* d, uint64_t da, uint64_t db) {
    if constexpr (WN == 64) wgmma_ss_n64(*reinterpret_cast<float(*)[32]>(d), da, db, 1u);
    else if constexpr (WN == 128) wgmma_ss_n128(*reinterpret_cast<float(*)[64]>(d), da, db, 1u);
    else if constexpr (WN == 160) wgmma_ss_n160(*reinterpret_cast<float(*)[80]>(d), da, db, 1u);
    else wgmma_ss_n256(*reinterpret_cast<float(*)[128]>(d), da, db, 1u);
}

// FEAT selects what the epilogue carries besides bias / time-embedding vector / residual / LayerNorm fold / row statistics:
//   0  nothing else (the linears of the transformer blocks)
//   1  + GroupNorm column statistics (convs, proj_out)
//   2  + activations (SiLU, quick-GELU, erf / tanh GELU) and the fp32 residual-trunk twins (once-per-call MLPs, CLIP / SAM
//      towers, OMG_TRUNK_F32)
template <int BN, int EPI, int MT, int FEAT>
__global__ void __launch_bounds__(GEMM_THREADS, 1) gemm_tc_kernel(const __grid_constant__ GemmParams p) {
    constexpr bool kStats = FEAT >= 1, kExtra = FEAT >= 2;
    static_assert(EPI != OMG_EPI_GEGLU || (BN <= 256 && MT == 1), "GEGLU runs on single 128-row tiles");
    using Cfg = GemmCfg<BN, MT, kStats>;
    constexpr int STAGES = Cfg::STAGES;
    constexpr int NJ = BN / 8;  // 8-column chunks of the accumulator
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    float* s_bias = reinterpret_cast<float*>(smem + STAGES * Cfg::STAGE_BYTES);
    float* s_c1 = s_bias + MT * BN;
    float4* s_cs = reinterpret_cast<float4*>(s_c1 + MT * BN);
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(s_cs) + Cfg::CS_BYTES);
    uint64_t* empty_bar = full_bar + STAGES;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int total_tiles = ((p.m_tiles + MT - 1) / MT) * p.n_tiles;
    const int tiles_per_img = p.tiles_w * p.tiles_h;

    if (warp == 8 && lane == 0) {
        for (int i = 0; i < OMG_MAX_A; ++i) tma_prefetch_desc(&p.a_maps[i]);
        tma_prefetch_desc(&p.b_maps[0]);
        tma_prefetch_desc(&p.b_maps[1]);
        for (int i = 0; i < STAGES; ++i) {
            mbar_init(&full_bar[i], 1);
            mbar_init(&empty_bar[i], 2);  // one arrival per consumer warpgroup
        }
        fence_barrier_init();
    }
    __syncthreads();
    griddep_launch_dependents();  // the prologue above overlaps the previous kernel's tail
    griddep_wait();               // operands / residual / output buffers belong to earlier kernels until here

    if (warp >= 8) {
        // ------------------------------------------------------------- TMA producer
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (warp == 8 && lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
                const int m_tile = (tile / p.n_tiles) * MT, n_tile = tile % p.n_tiles;
                const int b = m_tile / tiles_per_img;
                const int rem = m_tile % tiles_per_img;
                const int h0 = (rem / p.tiles_w) * p.th, w0 = (rem % p.tiles_w) * p.tw;
                // second 128-row m-tile of a tall tile (the next m-tile in (w, h, image) order; past the last image for
                // an odd m-tile count: TMA zero-fills)
                const int b1 = (m_tile + 1) / tiles_per_img, rem1 = (m_tile + 1) % tiles_per_img;
                const int h1 = (rem1 / p.tiles_w) * p.th, w1 = (rem1 % p.tiles_w) * p.tw;
                int n0 = n_tile * BN;
                if (p.w_group_rows > 0) {  // multi-stream launch: this tile's stream selects the weight plane
                    const long long tile_pix0 = ((long long)b * p.img_h + h0) * p.img_w + w0;
                    for (int g2 = 0; g2 + 1 < p.n_col_groups; ++g2)
                        if (tile_pix0 >= p.col_group_end[g2]) n0 += p.w_group_rows;
                }
                for (int s = 0; s < p.n_segs; ++s) {
                    const SegDev sg = p.segs[s];
                    for (int kb = 0; kb < sg.k_blocks; ++kb) {
                        mbar_wait(&empty_bar[stage], phase ^ 1);
                        uint8_t* a_dst = smem + stage * Cfg::STAGE_BYTES;
                        uint8_t* b_dst = a_dst + Cfg::A_BYTES;
                        mbar_arrive_expect_tx(&full_bar[stage], Cfg::STAGE_BYTES);
                        tma_load_4d(a_dst, &p.a_maps[sg.a_map], &full_bar[stage], sg.a_c0 + kb * BK, w0 + sg.dx, h0 + sg.dy, b);
                        if constexpr (MT == 2)
                            tma_load_4d(a_dst + BM * BK * 2, &p.a_maps[sg.a_map], &full_bar[stage], sg.a_c0 + kb * BK,
                                        w1 + sg.dx, h1 + sg.dy, b1);
#pragma unroll
                        for (int nw = 0; nw < Cfg::NW; ++nw)
                            tma_load_2d(b_dst + nw * Cfg::WN * BK * 2, &p.b_maps[sg.b_map], &full_bar[stage],
                                        sg.b_k0 + kb * BK, n0 + nw * Cfg::WN);
                        if (++stage == STAGES) {
                            stage = 0;
                            phase ^= 1;
                        }
                    }
                }
            }
        }
        return;
    }

    // ----------------------------------------------------------------- consumer warpgroups
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int wg = warp >> 2;         // warpgroup 0 | 1
    const int wi = warp & 3;          // warp within the warpgroup: rows 16 wi .. 16 wi + 15 of each m64 block
    const int g = lane >> 2, c = lane & 3;
    const int ctid = threadIdx.x;     // 0..255
    int stage = 0;
    uint32_t phase = 0;
    float acc[Cfg::ACC];

    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int unit_m = (tile / p.n_tiles) * MT, n_tile = tile % p.n_tiles;
        const int n0 = n_tile * BN;
        const bool ln = p.stats_in != nullptr;

        // per-column vectors of every m-tile of the unit (tall tiles: the two m-tiles may belong to different images /
        // streams); the barrier in front also tells that the previous tile's epilogue is done with them
        named_bar_sync(1, 256);
        for (int sub = 0; sub < MT; ++sub) {
            const int mt = unit_m + sub;
            const int b = mt / tiles_per_img, rem = mt % tiles_per_img;
            size_t cg = 0;  // tiles never straddle row groups (host guarantees 128-row alignment): this tile's c1/c2 plane
            if (ln && p.n_col_groups > 1) {
                const long long tile_pix0 = ((long long)b * p.img_h + (rem / p.tiles_w) * p.th) * p.img_w + (rem % p.tiles_w) * p.tw;
                for (int g2 = 0; g2 + 1 < p.n_col_groups; ++g2)
                    if (tile_pix0 >= p.col_group_end[g2]) cg = g2 + 1;
                cg *= (size_t)p.N;
            }
            for (int j = ctid; j < BN; j += 256) {
                float v = 0.f, c1 = 0.f;
                const int n = n0 + j;
                if (n < p.N) {
                    if (ln) {
                        v = p.col_c2[cg + n];
                        c1 = p.col_c1[cg + n];
                    } else {
                        if (p.bias) v += __half2float(p.bias[n]);
                        if (p.rowvec && b < p.img_b) v += __half2float(p.rowvec[(size_t)b * p.rowvec_ld + n]);
                    }
                }
                s_bias[sub * BN + j] = v;
                s_c1[sub * BN + j] = c1;
            }
        }
        named_bar_sync(1, 256);

        // ------------------------------------------------------------- main loop
#pragma unroll
        for (int i = 0; i < Cfg::ACC; ++i) acc[i] = 0.f;
        int prev_stage = -1;
        for (int s = 0; s < p.n_segs; ++s) {
            const int kbs = p.segs[s].k_blocks;
            for (int kb = 0; kb < kbs; ++kb) {
                mbar_wait(&full_bar[stage], phase);
                const uint32_t a_addr = smem_u32(smem + stage * Cfg::STAGE_BYTES) + (uint32_t)(wg * MT) * (64 * BK * 2);
                const uint32_t b_addr = smem_u32(smem + stage * Cfg::STAGE_BYTES + Cfg::A_BYTES);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < BK / 16; ++k) {
#pragma unroll
                    for (int i = 0; i < MT; ++i) {
                        const uint64_t a_desc = gmma_desc_sw128(a_addr + i * (64 * BK * 2) + k * 32, 1024, 16);
#pragma unroll
                        for (int nw = 0; nw < Cfg::NW; ++nw) {
                            const uint64_t b_desc = gmma_desc_sw128(b_addr + nw * (Cfg::WN * BK * 2) + k * 32, 1024, 16);
                            wgmma_ss<Cfg::WN>(acc + i * (BN / 2) + nw * (Cfg::WN / 2), a_desc, b_desc);
                        }
                    }
                }
                wgmma_commit();
                wgmma_wait<1>();  // the previous stage's wgmmas have completed: hand that stage back to the producer
                if (prev_stage >= 0 && (ctid & 127) == 0) mbar_arrive(&empty_bar[prev_stage]);
                prev_stage = stage;
                if (++stage == STAGES) {
                    stage = 0;
                    phase ^= 1;
                }
            }
        }
        wgmma_wait<0>();
        reg_fence(acc);
        if ((ctid & 127) == 0) mbar_arrive(&empty_bar[prev_stage]);

        // ------------------------------------------------------------- epilogue from the accumulator registers
#pragma unroll
        for (int i = 0; i < MT; ++i) {
            const int blk = wg * MT + i;        // m64 block of the unit
            const int sub = blk >> 1;           // m-tile of the unit
            const int m_tile = unit_m + sub;
            const int b = m_tile / tiles_per_img;
            const int rem = m_tile % tiles_per_img;
            const int h0 = (rem / p.tiles_w) * p.th, w0 = (rem % p.tiles_w) * p.tw;
            const float* sb = s_bias + sub * BN;
            const float* sc = s_c1 + sub * BN;
            float* a = acc + i * (BN / 2);
            float row_sum[2] = {0.f, 0.f}, row_sq[2] = {0.f, 0.f};
            bool valid[2];
            size_t pix[2];
            __half* orow[2];
            float ln_a[2] = {1.f, 1.f}, ln_k[2] = {0.f, 0.f};
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int et = (blk & 1) * 64 + wi * 16 + g + 8 * h;  // row of the 128-row m-tile
                const int ph = h0 + et / p.tw, pw = w0 + et % p.tw;
                valid[h] = (ph < p.img_h) && (pw < p.img_w) && (b < p.img_b);
                pix[h] = ((size_t)b * p.img_h + ph) * p.img_w + pw;
                orow[h] = p.out + (long long)b * p.out_sb + (long long)ph * p.out_sh + (long long)pw * p.out_sw;
                // folded LayerNorm: this row's mean / rstd from the producer's partial sums;
                // out = ln_a * acc + (ln_k * c1 + c2), ln_k = -rstd * mean
                if (ln && valid[h]) {
                    float sa = 0.f, sq = 0.f;
                    for (int t = 0; t < p.stats_parts; ++t) {
                        const float2 st = __ldg(reinterpret_cast<const float2*>(p.stats_in) + (size_t)t * p.stats_rows + pix[h]);
                        sa += st.x;
                        sq += st.y;
                    }
                    const float mu = sa * p.ln_inv_dim;
                    ln_a[h] = rsqrtf(fmaxf(sq * p.ln_inv_dim - mu * mu, 0.f) + p.ln_eps);
                    ln_k[h] = -ln_a[h] * mu;
                }
            }
            // column statistics: this warp's 16 rows go to its slot of the exchange buffer, (sum, sumsq) per column pair
            float4* cs_slot = s_cs + (size_t)(blk * 4 + wi) * (BN / 2);
#pragma unroll
            for (int J = 0; J < NJ; ++J) {
                const int col = 8 * J + 2 * c;  // within the tile
                const int n = n0 + col;
                float x[2][2];
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const float v = a[4 * J + 2 * h + e];
                        x[h][e] = ln ? fmaf(ln_a[h], v, fmaf(ln_k[h], sc[col + e], sb[col + e])) : v + sb[col + e];
                    }
                if constexpr (EPI == OMG_EPI_GEGLU) {
                    // columns (2i, 2i + 1) are (value, gate) pairs: one output column per pair, two per lane pair
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const float o = x[h][0] * gelu_exact(x[h][1]);
                        const float o_nb = __shfl_down_sync(0xffffffffu, o, 1);
                        if ((c & 1) == 0 && valid[h] && n < p.N)
                            *reinterpret_cast<__half2*>(orow[h] + (n >> 1)) = __floats2half2_rn(o, o_nb);
                    }
                } else {
                    if constexpr (kExtra) {
#pragma unroll
                        for (int h = 0; h < 2; ++h)
#pragma unroll
                            for (int e = 0; e < 2; ++e) {
                                float v = x[h][e];
                                if (p.act_silu == 1) {
                                    v = v / (1.0f + __expf(-v));
                                } else if (p.act_silu == 2) {  // quick_gelu
                                    v = v / (1.0f + __expf(-1.702f * v));
                                } else if (p.act_silu == 3) {  // erf-gelu
                                    v = gelu_exact(v);
                                } else if (p.act_silu == 4) {  // tanh-gelu (EfficientViT-SAM): 0.5 x (1 + tanh(sqrt(2/pi)(x + 0.044715 x^3)))
                                    const float u = 0.7978845608028654f * fmaf(0.044715f * v * v, v, v);
                                    v = 0.5f * v * (2.0f - __fdividef(2.0f, 1.0f + __expf(2.0f * u)));
                                }
                                x[h][e] = v;
                            }
                    }
                    float4 cs = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const bool ok = valid[h] && n < p.N;
                        if (ok && p.residual != nullptr) {
                            const float2 r = __half22float2(*reinterpret_cast<const __half2*>(p.residual + pix[h] * (size_t)p.residual_ld + n));
                            x[h][0] += r.x;
                            x[h][1] += r.y;
                        }
                        if constexpr (kExtra) {
                            if (ok && p.residual_f32 != nullptr) {
                                const float2 r = *reinterpret_cast<const float2*>(p.residual_f32 + pix[h] * (size_t)p.residual_f32_ld + n);
                                x[h][0] += r.x;
                                x[h][1] += r.y;
                            }
                            if (ok && p.out_f32 != nullptr)
                                *reinterpret_cast<float2*>(p.out_f32 + pix[h] * (size_t)p.out_f32_ld + n) = make_float2(x[h][0], x[h][1]);
                        }
                        if (ok) {
                            row_sum[h] += x[h][0] + x[h][1];
                            row_sq[h] = fmaf(x[h][0], x[h][0], fmaf(x[h][1], x[h][1], row_sq[h]));
                        }
                        const __half2 o = __floats2half2_rn(x[h][0], x[h][1]);
                        if (ok) *reinterpret_cast<__half2*>(orow[h] + n) = o;
                        if constexpr (kStats) {  // of the fp16-rounded values the consumer GroupNorm will see; rows outside the image count as zeros
                            const float2 f = valid[h] ? __half22float2(o) : make_float2(0.f, 0.f);
                            cs.x += f.x;
                            cs.y = fmaf(f.x, f.x, cs.y);
                            cs.z += f.y;
                            cs.w = fmaf(f.y, f.y, cs.w);
                        }
                    }
                    if constexpr (kStats) {
                        if (p.col_stats != nullptr) {  // sum over the 8 row groups of the warp (lanes with the same c)
#pragma unroll
                            for (int off = 4; off < 32; off <<= 1) {
                                cs.x += __shfl_xor_sync(0xffffffffu, cs.x, off);
                                cs.y += __shfl_xor_sync(0xffffffffu, cs.y, off);
                                cs.z += __shfl_xor_sync(0xffffffffu, cs.z, off);
                                cs.w += __shfl_xor_sync(0xffffffffu, cs.w, off);
                            }
                            if (g == 0) cs_slot[4 * J + c] = cs;
                        }
                    }
                }
            }
            if constexpr (EPI != OMG_EPI_GEGLU) {
                if (p.stats_out != nullptr) {  // per-row partials of this tile: the four lanes of a row hold its columns
                    float2* so = reinterpret_cast<float2*>(p.stats_out);
                    constexpr int PLANES = BN > 256 ? 4 : 2;  // as many partial planes as two 160-wide tiles would emit
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        float s = row_sum[h], q = row_sq[h];
                        s += __shfl_xor_sync(0xffffffffu, s, 1);
                        q += __shfl_xor_sync(0xffffffffu, q, 1);
                        s += __shfl_xor_sync(0xffffffffu, s, 2);
                        q += __shfl_xor_sync(0xffffffffu, q, 2);
                        if (c == 0 && valid[h]) {
                            so[(size_t)(n_tile * PLANES) * p.stats_rows + pix[h]] = make_float2(s, q);
                            for (int t = 1; t < PLANES; ++t) so[(size_t)(n_tile * PLANES + t) * p.stats_rows + pix[h]] = make_float2(0.f, 0.f);
                        }
                    }
                }
            }
            if constexpr (EPI != OMG_EPI_GEGLU && kStats) {
                if (p.col_stats != nullptr) {  // the two warps of a 32-row block add their slots
                    named_bar_sync(2 + wg * 2 + (wi >> 1), 64);
                    const int q = (blk & 1) * 2 + (wi >> 1);  // 32-row quarter of the m-tile
                    const float4* s0 = s_cs + (size_t)(blk * 4 + (wi & 2)) * (BN / 2);
                    const float4* s1 = s0 + BN / 2;
                    if (b < p.img_b) {
                        const size_t rb = (size_t)b * p.cs_rb_total + p.cs_rb0 + (size_t)rem * 4 + q;
                        for (int cp = (wi & 1) * 32 + lane; cp < BN / 2; cp += 64) {
                            const int col = n0 + 2 * cp;
                            if (col < p.N) {
                                const float4 u = s0[cp], w = s1[cp];
                                p.col_stats[(rb * p.N + col) >> 1] = make_float4(u.x + w.x, u.y + w.y, u.z + w.z, u.w + w.w);
                            }
                        }
                    }
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------ host
static int view_to_tmap(CUtensorMap* m, const omg_view4& v, uint32_t box_c, uint32_t box_w, uint32_t box_h,
                        CUtensorMapSwizzle sw) {
    const uint64_t dims[4] = {(uint64_t)v.C, (uint64_t)v.W, (uint64_t)v.H, (uint64_t)v.B};
    const uint64_t strides[4] = {1, (uint64_t)v.sw, (uint64_t)v.sh, (uint64_t)v.sb};
    const uint32_t box[4] = {box_c, box_w, box_h, 1};
    return make_tmap_f16(m, v.ptr, 4, dims, strides, box, sw);
}

template <int BN, int EPI, int MT, int FEAT>
static int launch_gemm_f(const GemmParams& p, cudaStream_t stream) {
    using Cfg = GemmCfg<BN, MT, (FEAT >= 1)>;
    static bool configured = false;
    static int num_sms = 0;
    if (!configured) {
        OMG_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<BN, EPI, MT, FEAT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      Cfg::SMEM_BYTES));
        int dev = 0;
        OMG_CUDA(cudaGetDevice(&dev));
        OMG_CUDA(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev));
        configured = true;
    }
    const int units = ((p.m_tiles + MT - 1) / MT) * p.n_tiles;
    const int grid = std::min(units, num_sms);
    OMG_CUDA(launch_pdl(gemm_tc_kernel<BN, EPI, MT, FEAT>, dim3(grid), dim3(GEMM_THREADS), Cfg::SMEM_BYTES, stream, p));
    return check_launch("gemm_tc_kernel");
}

// FEAT dispatch: 0 lean, 1 + GroupNorm column statistics, 2 + activations / fp32 twins (GEGLU launches are always lean)
template <int BN, int EPI, int MT = 1>
static int launch_gemm(const GemmParams& p, cudaStream_t stream) {
    if constexpr (EPI == OMG_EPI_GEGLU) {
        return launch_gemm_f<BN, EPI, MT, 0>(p, stream);
    } else {
        if (p.act_silu != 0 || p.residual_f32 != nullptr || p.out_f32 != nullptr) return launch_gemm_f<BN, EPI, MT, 2>(p, stream);
        if (p.col_stats != nullptr) return launch_gemm_f<BN, EPI, MT, 1>(p, stream);
        return launch_gemm_f<BN, EPI, MT, 0>(p, stream);
    }
}

// Tile-shape cost model: time ~ waves * per-tile cost, a tile's cost being its output columns per 128 rows plus a fixed
// overhead worth 48 columns (prologue, pipeline fill, epilogue tail).  It is a model, not a calibration: it runs on the
// host without a GPU (omg_gemm_plan) and uses the SM count of an H100 SXM.
constexpr int PLAN_SMS = 132;
constexpr double TILE_OVERHEAD = 48.0;
static double tile_time(long tiles, double cols) {
    return (double)((tiles + PLAN_SMS - 1) / PLAN_SMS) * (cols + TILE_OVERHEAD);
}

// tall tiles (256 x 160): half as many work units, each sharing its weight tiles between two m-tiles
static bool use_tall_tiles(long m_tiles, long n_tiles, long k_blocks) {
    if (m_tiles < 2 || k_blocks < 16) return false;
    return tile_time(((m_tiles + 1) / 2) * n_tiles, 320.0) < tile_time(m_tiles * n_tiles, 160.0);
}

// k_plan: K blocks the choice is made for; k_blocks: K blocks of this launch.  Row-statistics producers of one consumer
// must all emit the same number of partials (= 2 * n_tiles), so they - and omg_gemm_plan - choose with k_plan = "long"
// whatever their own K; whether a 160-wide choice then runs as tall or as 128-row tiles does not change n_tiles.
constexpr long K_PLAN_LONG = 1000;
static int pick_block_n(int N, int epilogue, long m_tiles, long k_plan, long k_blocks, bool* prefer_tall) {
    if (prefer_tall) *prefer_tall = false;
    if (epilogue == OMG_EPI_GEGLU) return 256;
    const int cands[5] = {256, 160, 128, 64, 160};
    int best = 256;
    double best_t = 1e30;
    for (int i = 0; i < 5; ++i) {
        const bool tall = i == 4;
        if (tall && (k_plan < 16 || m_tiles < 2)) continue;
        const long nt = (N + cands[i] - 1) / cands[i];
        const long mt = tall ? (m_tiles + 1) / 2 : m_tiles;
        const double t = tile_time(nt * mt, tall ? 2.0 * cands[i] : cands[i]);
        if (t < best_t - 1e-9) {
            best_t = t;
            best = cands[i];
            if (prefer_tall) *prefer_tall = tall && k_blocks >= 16;
        }
    }
    return best;
}

}  // namespace omg

using namespace omg;

extern "C" int omg_gemm_plan(int N, int epilogue, int W, int H, int B, int* block_n, int* n_tiles) {
    OMG_CHECK(N >= 8 && W >= 1 && H >= 1 && B >= 1, "omg_gemm_plan: bad arguments");
    int tw = 128;
    while (tw / 2 >= W && tw > 1) tw /= 2;
    const int th = 128 / tw;
    const long m_tiles = (long)((W + tw - 1) / tw) * ((H + th - 1) / th) * B;
    const int bn = pick_block_n(N, epilogue, m_tiles, K_PLAN_LONG, 0, nullptr);
    if (block_n) *block_n = bn;
    if (n_tiles) *n_tiles = 2 * ((N + bn - 1) / bn);  // row-statistics partials: one per (n-tile, chunk parity)
    return 0;
}

extern "C" int omg_gemm_colstats_blocks(int W, int H) {
    if (W < 1 || H < 1) return 0;
    int tw = 128;
    while (tw / 2 >= W && tw > 1) tw /= 2;
    const int th = 128 / tw;
    return ((W + tw - 1) / tw) * ((H + th - 1) / th) * 4;
}

static int gemm_impl(const omg_gemm_desc* d, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    OMG_CHECK(d != nullptr, "omg_gemm: null descriptor");
    OMG_CHECK(d->n_a >= 1 && d->n_a <= OMG_MAX_A, "omg_gemm: n_a=%d out of range", d->n_a);
    OMG_CHECK(d->n_segs >= 1 && d->n_segs <= OMG_MAX_SEGS, "omg_gemm: n_segs=%d out of range", d->n_segs);
    OMG_CHECK(d->w && d->d.ptr, "omg_gemm: null weight/output pointer");
    OMG_CHECK(d->N >= 8 && d->N % 8 == 0, "omg_gemm: N=%d must be a positive multiple of 8", d->N);
    OMG_CHECK(d->Ktot % 8 == 0, "omg_gemm: Ktot=%d must be a multiple of 8", d->Ktot);
    const bool geglu = d->epilogue == OMG_EPI_GEGLU;
    const bool silu = d->epilogue == OMG_EPI_SILU;
    const int act = silu ? 1 : (d->epilogue == OMG_EPI_QUICK_GELU ? 2 : (d->epilogue == OMG_EPI_GELU ? 3 : (d->epilogue == OMG_EPI_GELU_TANH ? 4 : 0)));
    OMG_CHECK(d->epilogue == OMG_EPI_NONE || geglu || act, "omg_gemm: unknown epilogue %d", d->epilogue);
    const int N_out = geglu ? d->N / 2 : d->N;
    OMG_CHECK(d->d.C == N_out, "omg_gemm: output view has %d channels, expected %d", d->d.C, N_out);
    OMG_CHECK(!geglu || (d->N % 64 == 0 && !d->residual && !d->rowvec),
              "omg_gemm: GEGLU needs N %% 64 == 0 and no residual/rowvec");
    OMG_CHECK(!d->residual || (N_out % 32 == 0 && d->residual_ld % 8 == 0),
              "omg_gemm: residual needs N %% 32 == 0 and ld %% 8 == 0");

    GemmParams p;
    memset(&p, 0, sizeof(p));
    const int W = d->d.W, H = d->d.H, B = d->d.B;
    OMG_CHECK(W >= 1 && H >= 1 && B >= 1, "omg_gemm: empty output grid");
    int tw = 128;
    while (tw / 2 >= W && tw > 1) tw /= 2;  // smallest power of two >= W, capped at 128
    const int th = 128 / tw;
    p.tw = tw;
    p.th = th;
    p.tiles_w = (W + tw - 1) / tw;
    p.tiles_h = (H + th - 1) / th;
    p.img_w = W;
    p.img_h = H;
    p.img_b = B;
    p.m_tiles = p.tiles_w * p.tiles_h * B;
    p.N = d->N;
    p.N_out = N_out;
    bool prefer_tall = false;
    const long k_blocks_hint = (long)(d->Ktot + (d->w2 ? d->K2tot : 0)) / 64;
    int bn = d->block_n ? d->block_n
                        : pick_block_n(d->N, d->epilogue, p.m_tiles, d->row_stats_out ? K_PLAN_LONG : k_blocks_hint,
                                       k_blocks_hint, &prefer_tall);
    OMG_CHECK(bn == 64 || bn == 128 || bn == 160 || bn == 256 || bn == 320, "omg_gemm: block_n=%d unsupported", bn);
    OMG_CHECK(bn != 320 || (!geglu && d->N % 320 == 0), "omg_gemm: block_n=320 needs N %% 320 == 0 and no GEGLU");
    // cta_pair: 0 automatic, 1 single 128-row tiles, 3 tall 256 x 160 tiles; 2 (CTA pairs) has no Hopper counterpart
    OMG_CHECK(d->cta_pair == 0 || d->cta_pair == 1 || d->cta_pair == 3, "omg_gemm: cta_pair=%d unsupported (0, 1 or 3)",
              d->cta_pair);
    if (geglu) bn = 256;
    p.n_tiles = (d->N + bn - 1) / bn;
    p.bias = static_cast<const __half*>(d->bias);
    p.rowvec = static_cast<const __half*>(d->rowvec);
    p.rowvec_ld = d->rowvec_ld;
    p.residual = static_cast<const __half*>(d->residual);
    p.residual_ld = d->residual_ld;
    p.act_silu = act;  // 0 none, 1 SiLU, 2 quick_gelu, 3 erf-gelu, 4 tanh-gelu
    p.stats_out = static_cast<float*>(d->row_stats_out);
    p.stats_in = static_cast<const float*>(d->row_stats_in);
    p.stats_parts = d->row_stats_parts;
    p.stats_rows = d->row_stats_stride > 0 ? d->row_stats_stride : (long long)W * H * B;
    p.ln_inv_dim = d->ln_dim > 0 ? 1.0f / (float)d->ln_dim : 0.f;
    p.ln_eps = d->ln_eps;
    p.col_c1 = static_cast<const float*>(d->col_c1);
    p.col_c2 = static_cast<const float*>(d->col_c2);
    p.n_col_groups = d->n_col_groups > 0 ? d->n_col_groups : 1;
    p.w_group_rows = d->w_group_planes > 0 ? d->N : 0;
    OMG_CHECK(d->w_group_planes == 0 || d->w_group_planes == p.n_col_groups, "omg_gemm: w_group_planes must equal n_col_groups");
    OMG_CHECK(p.n_col_groups <= 8, "omg_gemm: at most 8 column-vector row groups");
    for (int i = 0; i < 8; ++i) {
        p.col_group_end[i] = d->col_group_end[i];
        OMG_CHECK(i + 1 >= p.n_col_groups || d->col_group_end[i] % 128 == 0,
                  "omg_gemm: row-group boundary %lld is not a multiple of the 128-row tile", (long long)d->col_group_end[i]);
    }
    OMG_CHECK(!p.stats_in || (p.col_c1 && p.col_c2 && d->ln_dim > 0 && d->row_stats_parts >= 1 && !d->rowvec),
              "omg_gemm: folded LayerNorm needs col_c1, col_c2, ln_dim, row_stats_parts and no rowvec");
    OMG_CHECK(!p.stats_out || !geglu, "omg_gemm: row statistics cannot be emitted by the GEGLU epilogue");
    p.residual_f32 = static_cast<const float*>(d->residual_f32);
    p.residual_f32_ld = d->residual_f32_ld;
    p.out_f32 = static_cast<float*>(d->out_f32);
    p.out_f32_ld = d->out_f32_ld;
    OMG_CHECK((!p.residual_f32 && !p.out_f32) || (!geglu && d->N % 32 == 0 && !(d->residual && d->residual_f32)),
              "omg_gemm: fp32 residual / output twins need a non-GEGLU epilogue, N %% 32 == 0, and replace the fp16 residual");
    OMG_CHECK((!p.residual_f32 || d->residual_f32_ld % 4 == 0) && (!p.out_f32 || d->out_f32_ld % 4 == 0),
              "omg_gemm: fp32 twin row strides must be multiples of 4");
    OMG_CHECK((!p.residual_f32 && !p.out_f32) || (d->d.sw == d->d.C && d->d.sh == (int64_t)d->d.sw * W && d->d.sb == d->d.sh * H),
              "omg_gemm: fp32 twins need a contiguous output view (rows are indexed by pixel)");
    p.col_stats = static_cast<float4*>(d->col_stats_out);
    p.cs_rb0 = d->col_stats_rb0;
    p.cs_rb_total = d->col_stats_rb_total;
    OMG_CHECK(!p.col_stats || (!geglu && d->N % 32 == 0 && d->col_stats_rb0 >= 0 &&
                               d->col_stats_rb0 + p.tiles_w * p.tiles_h * 4 <= d->col_stats_rb_total),
              "omg_gemm: column statistics need a non-GEGLU epilogue, N %% 32 == 0 and rb0 + blocks <= rb_total");
    OMG_CHECK((!p.stats_out && !p.stats_in) || (d->d.sw == d->d.C && d->d.sh == (int64_t)d->d.sw * W && d->d.sb == d->d.sh * H),
              "omg_gemm: row statistics need a contiguous output view");

    for (int i = 0; i < d->n_a; ++i) {
        OMG_CHECK(d->a[i].ptr != nullptr, "omg_gemm: A view %d is null", i);
        if (view_to_tmap(&p.a_maps[i], d->a[i], BK, tw, th, CU_TENSOR_MAP_SWIZZLE_128B)) return 1;
    }
    for (int i = d->n_a; i < OMG_MAX_A; ++i) p.a_maps[i] = p.a_maps[0];
    {
        const uint64_t planes = d->w_group_planes > 0 ? (uint64_t)d->w_group_planes : 1;
        const uint64_t dims[2] = {(uint64_t)d->Ktot, (uint64_t)d->N * planes};
        const uint64_t strides[2] = {1, (uint64_t)d->Ktot};
        const uint32_t box[2] = {BK, (uint32_t)(bn > 256 ? bn / 2 : bn)};
        if (make_tmap_f16(&p.b_maps[0], d->w, 2, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B)) return 1;
        p.b_maps[1] = p.b_maps[0];
    }
    if (d->w2 != nullptr) {
        OMG_CHECK(d->K2tot >= 8 && d->K2tot % 8 == 0, "omg_gemm: K2tot=%d must be a positive multiple of 8", d->K2tot);
        const uint64_t dims[2] = {(uint64_t)d->K2tot, (uint64_t)d->N};
        const uint64_t strides[2] = {1, (uint64_t)d->K2tot};
        const uint32_t box[2] = {BK, (uint32_t)(bn > 256 ? bn / 2 : bn)};
        if (make_tmap_f16(&p.b_maps[1], d->w2, 2, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B)) return 1;
    }
    OMG_CHECK(d->d.sw % 2 == 0 && d->d.sh % 2 == 0 && d->d.sb % 2 == 0 && (reinterpret_cast<uintptr_t>(d->d.ptr) & 3) == 0,
              "omg_gemm: output view must be 4 B aligned per pixel");
    p.out = static_cast<__half*>(const_cast<void*>(d->d.ptr));
    p.out_sw = d->d.sw;
    p.out_sh = d->d.sh;
    p.out_sb = d->d.sb;

    p.n_segs = d->n_segs;
    for (int s = 0; s < d->n_segs; ++s) {
        const omg_seg& sg = d->segs[s];
        OMG_CHECK(sg.a_idx >= 0 && sg.a_idx < d->n_a, "omg_gemm: segment %d references A view %d", s, sg.a_idx);
        OMG_CHECK(sg.k_len > 0 && sg.a_c0 >= 0 && sg.b_k0 >= 0 && sg.a_c0 + sg.k_len <= d->a[sg.a_idx].C,
                  "omg_gemm: segment %d has a bad K range", s);
        OMG_CHECK(sg.b_idx == 0 || (sg.b_idx == 1 && d->w2 != nullptr), "omg_gemm: segment %d has a bad b_idx", s);
        const int ktot_s = sg.b_idx ? d->K2tot : d->Ktot;
        OMG_CHECK(sg.b_k0 + sg.k_len <= ktot_s, "omg_gemm: segment %d exceeds weight K (%d + %d > %d)", s, sg.b_k0,
                  sg.k_len, ktot_s);
        // A K-tail (k_len % 64 != 0) is only legal when the over-read of A is zero-filled, i.e. the segment ends
        // at the end of the A view's channel range.
        OMG_CHECK(sg.k_len % BK == 0 || sg.a_c0 + sg.k_len == d->a[sg.a_idx].C,
                  "omg_gemm: segment %d: K tail must end at the A view's last channel", s);
        p.segs[s] = SegDev{sg.a_idx, sg.dx, sg.dy, sg.a_c0, (sg.k_len + BK - 1) / BK, sg.b_k0, sg.b_idx};
    }

    long k_blocks = 0;
    for (int i = 0; i < p.n_segs; ++i) k_blocks += p.segs[i].k_blocks;
    bool pair_ok = true;  // both m-tiles of a tall tile must belong to the same stream
    for (int i = 0; i + 1 < p.n_col_groups; ++i) pair_ok = pair_ok && (p.col_group_end[i] % 256 == 0);
    if (bn == 320) return launch_gemm<320, OMG_EPI_NONE>(p, stream);
    // tall tiles (256 x 160 per CTA): the narrow-N, long-enough-K GEMMs
    const bool tall = bn == 160 && !geglu && pair_ok &&
                      (d->cta_pair == 3 ||
                       (d->cta_pair == 0 && (prefer_tall || use_tall_tiles(p.m_tiles, p.n_tiles, k_blocks))));
    if (tall) return launch_gemm<160, OMG_EPI_NONE, 2>(p, stream);
    if (geglu) return launch_gemm<256, OMG_EPI_GEGLU>(p, stream);
    switch (bn) {
        case 64: return launch_gemm<64, OMG_EPI_NONE>(p, stream);
        case 128: return launch_gemm<128, OMG_EPI_NONE>(p, stream);
        case 160: return launch_gemm<160, OMG_EPI_NONE>(p, stream);
        default: return launch_gemm<256, OMG_EPI_NONE>(p, stream);
    }
}

// C-ABI entry points: launch, and - while this thread records a launch plan (omg_plan_record_begin) - remember the call
extern "C" int omg_gemm(const omg_gemm_desc* d, void* stream_) {
    const int rc = gemm_impl(d, stream_);
    if (rc == 0 && ::omg::plan_recording()) {
        const omg_gemm_desc c = *d;  // by value: a plan outlives the caller's descriptor
        ::omg::plan_note([c](void* s) { return gemm_impl(&c, s); });
    }
    return rc;
}
