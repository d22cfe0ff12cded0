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
//   warpgroup's registers to the consumers: a 128 x 160 unit is 160 accumulators per thread).  The producer runs ahead
//   through a ring of shared-memory stages in the CTA's unit order.
// * Ping-pong: the work is cut into units of 128 (pixels) x UN (channels, 64 | 128 | 160), K in steps of 64.  Unit j
//   of a CTA belongs to consumer warpgroup j % 2, which owns it whole (both m64 blocks).  The two warpgroups take turns
//   on the tensor cores: a warpgroup waits for its turn before its first wgmma of a unit and hands the turn over as
//   soon as its last wgmma is issued, so one unit's epilogue (and the next unit's per-column vectors) runs while the
//   other warpgroup's MMAs keep the tensor cores busy.  An fp16 residual that a tensor map can describe is staged per
//   unit in shared memory by a second TMA thread of warpgroup 2, so the epilogue reads it there instead of waiting on
//   global loads that the aliased output stores keep in order.  A logical tile wider than a unit (block_n 256 / 320) runs as
//   two units of half its width; GEGLU runs on 160-wide units.  Operands land in shared memory in the 128B-swizzled K-major layout the GMMA
//   descriptors expect.
//
// Roofline: tensor-bound; algorithmic FLOPs per launch = 2 * pixels * N * sum(k_len).
#include <cuda_fp16.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <type_traits>

#include "../../include/omg_b200.h"
#include "elem.cuh"
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
    int units;                 // m_tiles * n_units work units of 128 x UN
    int n_units;               // units across N: (logical n-tiles) x (units per logical tile)
    int tw, th, tiles_w, tiles_h;
    int img_w, img_h, img_b;
    int N, N_out;
    // 16-bit operands in the kernel's storage type (fp16 | bf16, omg_gemm_desc.dtype)
    void* out;                 // output view (channels-last, element strides)
    long long out_sw, out_sh, out_sb;
    const void* bias;
    const void* rowvec;
    int rowvec_ld;
    const void* residual;
    int residual_ld;
    int act_silu;
    // LayerNorm folded into the GEMM pair (see omg_gemm_desc): statistics written by the producer's epilogue ...
    float* stats_out;          // [planes][rows][2] partial (sum, sum of squares) of this GEMM's output rows, or null
    int stats_unit_planes;     // k partial planes per unit: unit column nu writes planes nu*k .. nu*k + k-1 (k = 1 for block_n 256)
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
    // the residual over the output grid (N, W, H, B), boxes of 32 columns x one tw x th patch, 64B-swizzled (RES kernels)
    CUtensorMap res_map;
};

// A unit is 128 rows x UN columns, owned by one consumer warpgroup (two m64 blocks of UN / 2 accumulators each).
// CS: the epilogue can emit GroupNorm column statistics (FEAT >= 1); only then is their exchange buffer reserved, so the
// lean instantiations keep that shared memory for pipeline stages.
// RES: the residual is staged by TMA into one buffer of UN / 32 boxes of 128 rows x 32 columns, shared by both
// warpgroups (their epilogues take turns, as their MMAs do).  Stages: 8 / 5 / 5 for UN 64 / 128 / 160 (8 / 5 / 4 with
// CS), against 8 / 7 / 6 (8 / 6 / 5) without; a buffer per warpgroup would leave 8 / 4 / 3 (7 / 4 / 3).
constexpr int RES_BOX_BYTES = BM * 32 * 2;
template <int UN, bool CS, bool RES = false>
struct GemmCfg {
    static constexpr int ACC = UN;                        // fp32 accumulators per thread
    static constexpr int A_BYTES = BM * BK * 2;
    static constexpr int B_BYTES = UN * BK * 2;
    static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
    static constexpr int VEC_BYTES = 2 * 2 * UN * 4;      // per warpgroup: the unit's per-column vectors (bias | c1)
    static constexpr int CS_BYTES = CS ? 2 * 8 * (UN / 2) * 16 : 0;  // per warpgroup: a float4 per column pair and warp of each m64 block
    static constexpr int RES_BYTES = RES ? (UN / 32) * RES_BOX_BYTES : 0;
    static constexpr int BARS_BYTES = 256;
    static constexpr int BUDGET = 227 * 1024 - 1024 /*alignment slack*/ - RES_BYTES - VEC_BYTES - CS_BYTES - BARS_BYTES;
    static constexpr int STAGES_RAW = BUDGET / STAGE_BYTES;
    static constexpr int STAGES = STAGES_RAW > 8 ? 8 : STAGES_RAW;
    static constexpr int SMEM_BYTES = 1024 + STAGES * STAGE_BYTES + RES_BYTES + VEC_BYTES + CS_BYTES + BARS_BYTES;
    static_assert(STAGES >= 2, "shared memory budget");
    static_assert(STAGE_BYTES % 1024 == 0, "the residual buffer follows the stages on a 1024 B boundary");
    static_assert((2 * STAGES + 5) * 8 <= BARS_BYTES, "barrier space");
};

// GEGLU / erf-GELU use libdevice's erff.
__device__ __forceinline__ float gelu_exact(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f)); }

template <typename T, int WN>
__device__ __forceinline__ void wgmma_ss(float* d, uint64_t da, uint64_t db) {
    if constexpr (std::is_same_v<T, __nv_bfloat16>) {
        if constexpr (WN == 64) wgmma_ss_n64_bf16(*reinterpret_cast<float(*)[32]>(d), da, db, 1u);
        else if constexpr (WN == 128) wgmma_ss_n128_bf16(*reinterpret_cast<float(*)[64]>(d), da, db, 1u);
        else wgmma_ss_n160_bf16(*reinterpret_cast<float(*)[80]>(d), da, db, 1u);
    } else {
        if constexpr (WN == 64) wgmma_ss_n64(*reinterpret_cast<float(*)[32]>(d), da, db, 1u);
        else if constexpr (WN == 128) wgmma_ss_n128(*reinterpret_cast<float(*)[64]>(d), da, db, 1u);
        else wgmma_ss_n160(*reinterpret_cast<float(*)[80]>(d), da, db, 1u);
    }
}

// moves a ring position (stage, phase) on by n k-blocks
template <int STAGES>
__device__ __forceinline__ void ring_advance(int& stage, uint32_t& phase, int n) {
    stage += n;
    const int wraps = stage / STAGES;
    stage -= wraps * STAGES;
    phase ^= (uint32_t)wraps & 1u;
}

// FEAT selects what the epilogue carries besides bias / time-embedding vector / residual / LayerNorm fold / row statistics:
//   0  nothing else (the linears of the transformer blocks)
//   1  + GroupNorm column statistics (convs, proj_out)
//   2  + activations (SiLU, quick-GELU, erf / tanh GELU) and the fp32 residual-trunk twins (once-per-call MLPs, CLIP / SAM
//      towers, OMG_TRUNK_F32)
// T is the storage type of A, W, bias, rowvec, residual and the output (__half, or __nv_bfloat16 for the lean
// OMG_EPI_NONE instantiations the VAE decoder uses).
// RES (fp16, FEAT 0 / 1): the residual comes from shared memory, staged per unit by a second TMA thread, instead of one
// dependent global load per 8-column chunk in the epilogue (the output may alias the residual, so those loads cannot be
// hoisted above the stores).
template <typename T, int UN, int EPI, int FEAT, bool RES = false>
__global__ void __launch_bounds__(GEMM_THREADS, 1) gemm_tc_kernel(const __grid_constant__ GemmParams p) {
    using T2 = pair_t<T>;
    constexpr bool kStats = FEAT >= 1, kExtra = FEAT >= 2;
    static_assert(EPI != OMG_EPI_GEGLU || UN == 160, "GEGLU runs on 160-wide units");
    static_assert(!RES || (std::is_same_v<T, __half> && EPI == OMG_EPI_NONE && FEAT <= 1), "staged residual: fp16, FEAT 0 / 1");
    using Cfg = GemmCfg<UN, kStats, RES>;
    constexpr int STAGES = Cfg::STAGES;
    constexpr int NJ = UN / 8;  // 8-column chunks of an m64 block's accumulator
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* s_res = smem + STAGES * Cfg::STAGE_BYTES;
    float* s_vec = reinterpret_cast<float*>(s_res + Cfg::RES_BYTES);
    float4* s_cs_all = reinterpret_cast<float4*>(s_vec + 2 * 2 * UN);
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(s_cs_all) + Cfg::CS_BYTES);
    uint64_t* empty_bar = full_bar + STAGES;
    uint64_t* turn_bar = empty_bar + STAGES;  // turn_bar[w]: warpgroup w may issue its next unit's wgmmas
    uint64_t* res_full = turn_bar + 2;        // res_full[w]: the residual of warpgroup w's next unit has landed
    uint64_t* res_empty = res_full + 2;       // the owner of the buffered residual has read it (one arrival per warp)

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int tiles_per_img = p.tiles_w * p.tiles_h;

    if (warp == 8 && lane == 0) {
        for (int i = 0; i < OMG_MAX_A; ++i) tma_prefetch_desc(&p.a_maps[i]);
        tma_prefetch_desc(&p.b_maps[0]);
        tma_prefetch_desc(&p.b_maps[1]);
        for (int i = 0; i < STAGES; ++i) {
            mbar_init(&full_bar[i], 1);
            mbar_init(&empty_bar[i], 1);  // released by the warpgroup that owns the stage's unit
        }
        mbar_init(&turn_bar[0], 1);
        mbar_init(&turn_bar[1], 1);
        if constexpr (RES) {
            tma_prefetch_desc(&p.res_map);
            mbar_init(&res_full[0], 1);
            mbar_init(&res_full[1], 1);
            mbar_init(res_empty, 4);
        }
        fence_barrier_init();
    }
    __syncthreads();
    griddep_launch_dependents();  // the prologue above overlaps the previous kernel's tail
    griddep_wait();               // operands / residual / output buffers belong to earlier kernels until here

    if (warp >= 8) {
        // ------------------------------------------------------------- TMA producer: every unit of the CTA, in order
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (warp == 8 && lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int u = blockIdx.x; u < p.units; u += gridDim.x) {
                const int m_tile = u / p.n_units, nu = u % p.n_units;
                const int b = m_tile / tiles_per_img;
                const int rem = m_tile % tiles_per_img;
                const int h0 = (rem / p.tiles_w) * p.th, w0 = (rem % p.tiles_w) * p.tw;
                int n0 = nu * UN;
                if (p.w_group_rows > 0) {  // multi-stream launch: this unit's stream selects the weight plane
                    const long long tile_pix0 = ((long long)b * p.img_h + h0) * p.img_w + w0;
                    for (int g2 = 0; g2 + 1 < p.n_col_groups; ++g2)
                        if (tile_pix0 >= p.col_group_end[g2]) n0 += p.w_group_rows;
                }
                for (int s = 0; s < p.n_segs; ++s) {
                    const SegDev sg = p.segs[s];
                    for (int kb = 0; kb < sg.k_blocks; ++kb) {
                        mbar_wait_nocall(&empty_bar[stage], phase ^ 1);
                        uint8_t* a_dst = smem + stage * Cfg::STAGE_BYTES;
                        uint8_t* b_dst = a_dst + Cfg::A_BYTES;
                        mbar_arrive_expect_tx(&full_bar[stage], Cfg::STAGE_BYTES);
                        tma_load_4d(a_dst, &p.a_maps[sg.a_map], &full_bar[stage], sg.a_c0 + kb * BK, w0 + sg.dx, h0 + sg.dy, b);
                        tma_load_2d(b_dst, &p.b_maps[sg.b_map], &full_bar[stage], sg.b_k0 + kb * BK, n0);
                        if (++stage == STAGES) {
                            stage = 0;
                            phase ^= 1;
                        }
                    }
                }
            }
        }
        if constexpr (RES) {
            // residual producer: the same units in the same order, one at a time through the shared buffer.  A thread of
            // its own, so that waiting for the buffer never holds up the operand ring.  The residual's columns are the
            // output's (no weight-plane offset).
            if (warp == 9 && lane == 0) {
                int j = 0;  // unit of the CTA: warpgroup j % 2 reads it
                for (int u = blockIdx.x; u < p.units; u += gridDim.x, ++j) {
                    const int m_tile = u / p.n_units, nu = u % p.n_units;
                    const int b = m_tile / tiles_per_img;
                    const int rem = m_tile % tiles_per_img;
                    const int h0 = (rem / p.tiles_w) * p.th, w0 = (rem % p.tiles_w) * p.tw;
                    mbar_wait_nocall(res_empty, (j & 1) ^ 1);  // unit j - 1's epilogue has read the buffer
                    mbar_arrive_expect_tx(&res_full[j & 1], Cfg::RES_BYTES);
#pragma unroll
                    for (int i = 0; i < UN / 32; ++i)
                        tma_load_4d(s_res + i * RES_BOX_BYTES, &p.res_map, &res_full[j & 1], nu * UN + 32 * i, w0, h0, b);
                }
            }
        }
        return;
    }

    // ----------------------------------------------------------------- consumer warpgroups (ping-pong)
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int wg = warp >> 2;         // warpgroup 0 | 1: units j of the CTA with j % 2 == wg
    const int wi = warp & 3;          // warp within the warpgroup: rows 16 wi .. 16 wi + 15 of each m64 block
    const int g = lane >> 2, c = lane & 3;
    const int wtid = threadIdx.x & 127;
    float* s_bias = s_vec + wg * (2 * UN);
    float* s_c1 = s_bias + UN;
    float4* s_cs = s_cs_all + wg * (8 * (UN / 2));
    int unit_kb = 0;  // every unit of a launch runs the same K blocks
    for (int s = 0; s < p.n_segs; ++s) unit_kb += p.segs[s].k_blocks;
    int stage = 0;
    uint32_t phase = 0;
    if (wg == 1) ring_advance<STAGES>(stage, phase, unit_kb);  // past the CTA's unit 0
    // warpgroup 0 goes first: parity 1 of a fresh mbarrier reads as a completed phase
    uint32_t turn_phase = wg == 0 ? 1u : 0u;
    float acc[Cfg::ACC];

    for (int u = blockIdx.x + wg * gridDim.x; u < p.units; u += 2 * gridDim.x) {
        const int m_tile = u / p.n_units, nu = u % p.n_units;
        const int n0 = nu * UN;
        const int b = m_tile / tiles_per_img;
        const int rem = m_tile % tiles_per_img;
        const int h0 = (rem / p.tiles_w) * p.th, w0 = (rem % p.tiles_w) * p.tw;
        const bool ln = p.stats_in != nullptr;

        // per-column vectors of the unit, in this warpgroup's own time; the barrier in front also tells that the
        // previous unit's epilogue is done with them (and with the column-statistics slots)
        named_bar_sync(1 + wg, 128);
        {
            size_t cg = 0;  // units never straddle row groups (host guarantees 128-row alignment): this unit's c1/c2 plane
            if (ln && p.n_col_groups > 1) {
                const long long tile_pix0 = ((long long)b * p.img_h + h0) * p.img_w + w0;
                for (int g2 = 0; g2 + 1 < p.n_col_groups; ++g2)
                    if (tile_pix0 >= p.col_group_end[g2]) cg = g2 + 1;
                cg *= (size_t)p.N;
            }
            for (int j = wtid; j < UN; j += 128) {
                float v = 0.f, c1 = 0.f;
                const int n = n0 + j;
                if (n < p.N) {
                    if (ln) {
                        v = p.col_c2[cg + n];
                        c1 = p.col_c1[cg + n];
                    } else {
                        if (p.bias) v += to_f32(static_cast<const T*>(p.bias)[n]);
                        if (p.rowvec && b < p.img_b) v += to_f32(static_cast<const T*>(p.rowvec)[(size_t)b * p.rowvec_ld + n]);
                    }
                }
                s_bias[j] = v;
                s_c1[j] = c1;
            }
        }
        named_bar_sync(1 + wg, 128);

        // ------------------------------------------------------------- main loop, on this warpgroup's turn
#pragma unroll
        for (int i = 0; i < Cfg::ACC; ++i) acc[i] = 0.f;
        mbar_wait_nocall(&turn_bar[wg], turn_phase);
        turn_phase ^= 1;
        int prev_stage = -1;
        for (int s = 0; s < p.n_segs; ++s) {
            const int kbs = p.segs[s].k_blocks;
            for (int kb = 0; kb < kbs; ++kb) {
                mbar_wait_nocall(&full_bar[stage], phase);
                const uint32_t a_addr = smem_u32(smem + stage * Cfg::STAGE_BYTES);
                const uint32_t b_addr = a_addr + Cfg::A_BYTES;
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < BK / 16; ++k) {
                    const uint64_t b_desc = gmma_desc_sw128(b_addr + k * 32, 1024, 16);
#pragma unroll
                    for (int i = 0; i < 2; ++i)
                        wgmma_ss<T, UN>(acc + i * (UN / 2), gmma_desc_sw128(a_addr + i * (64 * BK * 2) + k * 32, 1024, 16), b_desc);
                }
                wgmma_commit();
                wgmma_wait<1>();  // the previous stage's wgmmas have completed: hand that stage back to the producer
                if (prev_stage >= 0 && wtid == 0) mbar_arrive(&empty_bar[prev_stage]);
                prev_stage = stage;
                if (++stage == STAGES) {
                    stage = 0;
                    phase ^= 1;
                }
            }
        }
        // every wgmma of the unit is issued: the other warpgroup's unit may start while these complete
        if (wtid == 0) mbar_arrive(&turn_bar[wg ^ 1]);
        wgmma_wait<0>();
        reg_fence(acc);
        if (wtid == 0) mbar_arrive(&empty_bar[prev_stage]);
        ring_advance<STAGES>(stage, phase, unit_kb);  // past the other warpgroup's next unit

        // ------------------------------------------------------------- epilogue from the accumulator registers
        // staged residual of row et = blk * 64 + wi * 16 + g + 8 h, columns 8 J + 2 c, 2 c + 1: box J / 4, 64-byte row et,
        // 16-byte chunk J % 4 under the 64B swizzle (chunk ^= (et >> 1) & 3 = g >> 1, as et - g is a multiple of 8).  A
        // warp's read of one (J, h) falls on 32-bit bank 16 (g & 1) + 4 ((J % 4) ^ (g >> 1)) + c: a different bank per lane.
        // (s_res is 1024 B aligned and bits 4, 5 of (wi * 16 + g) * 64 + 4 c are clear, so the chunk is XORed into them)
        const uint32_t res_row = (smem_u32(s_res) + (wi * 16 + g) * 64 + 4 * c) | ((g >> 1) << 4);
        if constexpr (RES) mbar_wait_nocall(&res_full[wg], turn_phase ^ wg);  // this warpgroup's k-th unit: parity k % 2
#pragma unroll
        for (int blk = 0; blk < 2; ++blk) {  // m64 block of the unit
            float* a = acc + blk * (UN / 2);
            float row_sum[2] = {0.f, 0.f}, row_sq[2] = {0.f, 0.f};
            bool valid[2];
            size_t pix[2];
            T* orow[2];
            float ln_a[2] = {1.f, 1.f}, ln_k[2] = {0.f, 0.f};
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int et = blk * 64 + wi * 16 + g + 8 * h;  // row of the 128-row m-tile
                const int ph = h0 + et / p.tw, pw = w0 + et % p.tw;
                valid[h] = (ph < p.img_h) && (pw < p.img_w) && (b < p.img_b);
                pix[h] = ((size_t)b * p.img_h + ph) * p.img_w + pw;
                orow[h] = static_cast<T*>(p.out) + (long long)b * p.out_sb + (long long)ph * p.out_sh + (long long)pw * p.out_sw;
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
            float4* cs_slot = s_cs + (size_t)(blk * 4 + wi) * (UN / 2);
#pragma unroll
            for (int J = 0; J < NJ; ++J) {
                const int col = 8 * J + 2 * c;  // within the unit
                const int n = n0 + col;
                float x[2][2];
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const float v = a[4 * J + 2 * h + e];
                        x[h][e] = ln ? fmaf(ln_a[h], v, fmaf(ln_k[h], s_c1[col + e], s_bias[col + e])) : v + s_bias[col + e];
                    }
                if constexpr (EPI == OMG_EPI_GEGLU) {
                    // columns (2i, 2i + 1) are (value, gate) pairs: one output column per pair, two per lane pair
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const float o = x[h][0] * gelu_exact(x[h][1]);
                        const float o_nb = __shfl_down_sync(0xffffffffu, o, 1);
                        if ((c & 1) == 0 && valid[h] && n < p.N)
                            *reinterpret_cast<T2*>(orow[h] + (n >> 1)) = from_f32x2<T>(o, o_nb);
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
                                } else if (p.act_silu == 5) {  // ReLU (SAM mask decoder MLPs)
                                    v = fmaxf(v, 0.f);
                                }
                                x[h][e] = v;
                            }
                    }
                    float4 cs = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const bool ok = valid[h] && n < p.N;
                        if constexpr (RES) {
                            const uint32_t rb = ld_shared_b32((res_row ^ ((J & 3) << 4)) + (J >> 2) * RES_BOX_BYTES + blk * 64 * 64 + h * 8 * 64);
                            const T2 rv = *reinterpret_cast<const T2*>(&rb);
                            if (ok) {
                                const float2 r = to_f32x2(rv);
                                x[h][0] += r.x;
                                x[h][1] += r.y;
                            }
                        } else if (ok && p.residual != nullptr) {
                            const float2 r = to_f32x2(*reinterpret_cast<const T2*>(static_cast<const T*>(p.residual) + pix[h] * (size_t)p.residual_ld + n));
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
                        const T2 o = from_f32x2<T>(x[h][0], x[h][1]);
                        if (ok) *reinterpret_cast<T2*>(orow[h] + n) = o;
                        if constexpr (kStats) {  // of the fp16-rounded values the consumer GroupNorm will see; rows outside the image count as zeros
                            const float2 f = valid[h] ? to_f32x2(o) : make_float2(0.f, 0.f);
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
            if constexpr (RES) {
                if (blk == 1) {  // the last read of the buffer: the residual thread may refill it for the next unit
                    __syncwarp();
                    if (elect_one()) mbar_arrive(res_empty);
                }
            }
            if constexpr (EPI != OMG_EPI_GEGLU) {
                if (p.stats_out != nullptr) {  // per-row partials of this unit: the four lanes of a row hold its columns
                    float2* so = reinterpret_cast<float2*>(p.stats_out);
                    const int kp = p.stats_unit_planes, plane0 = nu * kp;
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        float s = row_sum[h], q = row_sq[h];
                        s += __shfl_xor_sync(0xffffffffu, s, 1);
                        q += __shfl_xor_sync(0xffffffffu, q, 1);
                        s += __shfl_xor_sync(0xffffffffu, s, 2);
                        q += __shfl_xor_sync(0xffffffffu, q, 2);
                        if (c == 0 && valid[h]) {
                            so[(size_t)plane0 * p.stats_rows + pix[h]] = make_float2(s, q);
                            for (int t = 1; t < kp; ++t) so[(size_t)(plane0 + t) * p.stats_rows + pix[h]] = make_float2(0.f, 0.f);
                        }
                    }
                }
            }
            if constexpr (EPI != OMG_EPI_GEGLU && kStats) {
                if (p.col_stats != nullptr) {  // the two warps of a 32-row block add their slots
                    named_bar_sync(3 + wg * 2 + (wi >> 1), 64);
                    const int q = blk * 2 + (wi >> 1);  // 32-row quarter of the m-tile
                    const float4* s0 = s_cs + (size_t)(blk * 4 + (wi & 2)) * (UN / 2);
                    const float4* s1 = s0 + UN / 2;
                    if (b < p.img_b) {
                        const size_t rb = (size_t)b * p.cs_rb_total + p.cs_rb0 + (size_t)rem * 4 + q;
                        for (int cp = (wi & 1) * 32 + lane; cp < UN / 2; cp += 64) {
                            const int col = n0 + 2 * cp;
                            if (col < p.N) {
                                const float4 u4 = s0[cp], w4 = s1[cp];
                                p.col_stats[(rb * p.N + col) >> 1] = make_float4(u4.x + w4.x, u4.y + w4.y, u4.z + w4.z, u4.w + w4.w);
                            }
                        }
                    }
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------ host
static int view_to_tmap(CUtensorMap* m, const omg_view4& v, CUtensorMapDataType dt, uint32_t box_c, uint32_t box_w,
                        uint32_t box_h, CUtensorMapSwizzle sw) {
    const uint64_t dims[4] = {(uint64_t)v.C, (uint64_t)v.W, (uint64_t)v.H, (uint64_t)v.B};
    const uint64_t strides[4] = {1, (uint64_t)v.sw, (uint64_t)v.sh, (uint64_t)v.sb};
    const uint32_t box[4] = {box_c, box_w, box_h, 1};
    return make_tmap(m, dt, v.ptr, 4, dims, strides, box, sw);
}

template <typename T, int UN, int EPI, int FEAT, bool RES = false>
static int launch_gemm_f(const GemmParams& p, cudaStream_t stream) {
    using Cfg = GemmCfg<UN, (FEAT >= 1), RES>;
    static bool configured = false;
    static int num_sms = 0;
    if (!configured) {
        OMG_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<T, UN, EPI, FEAT, RES>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      Cfg::SMEM_BYTES));
        int dev = 0;
        OMG_CUDA(cudaGetDevice(&dev));
        OMG_CUDA(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev));
        configured = true;
    }
    const int grid = std::min(p.units, num_sms);
    OMG_CUDA(launch_pdl(gemm_tc_kernel<T, UN, EPI, FEAT, RES>, dim3(grid), dim3(GEMM_THREADS), Cfg::SMEM_BYTES, stream, p));
    return check_launch("gemm_tc_kernel");
}

// FEAT dispatch: 0 lean, 1 + GroupNorm column statistics, 2 + activations / fp32 twins (GEGLU launches are always lean).
// res_staged: p.res_map describes the residual, so FEAT 0 / 1 launches stage it by TMA.
template <int UN, int EPI>
static int launch_gemm(const GemmParams& p, bool res_staged, cudaStream_t stream) {
    if constexpr (EPI == OMG_EPI_GEGLU) {
        return launch_gemm_f<__half, UN, EPI, 0>(p, stream);
    } else {
        if (p.act_silu != 0 || p.residual_f32 != nullptr || p.out_f32 != nullptr) return launch_gemm_f<__half, UN, EPI, 2>(p, stream);
        if (p.col_stats != nullptr)
            return res_staged ? launch_gemm_f<__half, UN, EPI, 1, true>(p, stream) : launch_gemm_f<__half, UN, EPI, 1>(p, stream);
        return res_staged ? launch_gemm_f<__half, UN, EPI, 0, true>(p, stream) : launch_gemm_f<__half, UN, EPI, 0>(p, stream);
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

// k_plan: K blocks the choice is made for.  Row-statistics producers of one consumer must all emit the same number of
// partials (= 2 * n_tiles), so they - and omg_gemm_plan - choose with k_plan = "long" whatever their own K.  The fifth
// candidate prices 160-wide tiles two m-tiles at a time (half the fixed overhead per m-tile) for long enough K.
constexpr long K_PLAN_LONG = 1000;
static int pick_block_n(int N, int epilogue, long m_tiles, long k_plan) {
    if (epilogue == OMG_EPI_GEGLU) return 256;
    const int cands[5] = {256, 160, 128, 64, 160};
    int best = 256;
    double best_t = 1e30;
    for (int i = 0; i < 5; ++i) {
        const bool pair = i == 4;
        if (pair && (k_plan < 16 || m_tiles < 2)) continue;
        const long nt = (N + cands[i] - 1) / cands[i];
        const long mt = pair ? (m_tiles + 1) / 2 : m_tiles;
        const double t = tile_time(nt * mt, pair ? 2.0 * cands[i] : cands[i]);
        if (t < best_t - 1e-9) {
            best_t = t;
            best = cands[i];
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
    const int bn = pick_block_n(N, epilogue, m_tiles, K_PLAN_LONG);
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
    OMG_CHECK(d->dtype == OMG_DTYPE_F16 || d->dtype == OMG_DTYPE_BF16, "omg_gemm: dtype=%d unsupported (0 fp16, 1 bf16)",
              d->dtype);
    const bool bf16 = d->dtype == OMG_DTYPE_BF16;
    if (bf16) {  // the bf16 instantiations are the lean ones: bias and residual, no other epilogue feature
        OMG_CHECK(d->epilogue == OMG_EPI_NONE, "omg_gemm: bf16 supports only OMG_EPI_NONE (epilogue %d)", d->epilogue);
        OMG_CHECK(!d->rowvec, "omg_gemm: bf16 does not support rowvec");
        OMG_CHECK(!d->w2, "omg_gemm: bf16 does not support a second weight matrix (w2)");
        OMG_CHECK(d->w_group_planes == 0, "omg_gemm: bf16 does not support weight planes");
        OMG_CHECK(!d->row_stats_in, "omg_gemm: bf16 does not support the folded LayerNorm");
        OMG_CHECK(!d->row_stats_out, "omg_gemm: bf16 does not support row statistics");
        OMG_CHECK(!d->col_stats_out, "omg_gemm: bf16 does not support column statistics");
        OMG_CHECK(!d->residual_f32 && !d->out_f32, "omg_gemm: bf16 does not support fp32 twins");
    }
    const CUtensorMapDataType tdt = bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
    const bool geglu = d->epilogue == OMG_EPI_GEGLU;
    const bool silu = d->epilogue == OMG_EPI_SILU;
    const int act = silu ? 1 : (d->epilogue == OMG_EPI_QUICK_GELU ? 2 : (d->epilogue == OMG_EPI_GELU ? 3 : (d->epilogue == OMG_EPI_GELU_TANH ? 4 :
                    (d->epilogue == OMG_EPI_RELU ? 5 : 0))));
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
    const int m_tiles = p.tiles_w * p.tiles_h * B;
    p.N = d->N;
    p.N_out = N_out;
    const long k_blocks_hint = (long)(d->Ktot + (d->w2 ? d->K2tot : 0)) / 64;
    int bn = d->block_n ? d->block_n
                        : pick_block_n(d->N, d->epilogue, m_tiles, d->row_stats_out ? K_PLAN_LONG : k_blocks_hint);
    OMG_CHECK(bn == 64 || bn == 128 || bn == 160 || bn == 256 || bn == 320, "omg_gemm: block_n=%d unsupported", bn);
    OMG_CHECK(bn != 320 || (!geglu && d->N % 320 == 0), "omg_gemm: block_n=320 needs N %% 320 == 0 and no GEGLU");
    // cta_pair: 0, 1 and 3 (the former tall 256 x 160 tiles) all run the same units; 2 (CTA pairs) has no Hopper counterpart
    OMG_CHECK(d->cta_pair == 0 || d->cta_pair == 1 || d->cta_pair == 3, "omg_gemm: cta_pair=%d unsupported (0, 1 or 3)",
              d->cta_pair);
    if (geglu) bn = 256;
    // a logical tile wider than 160 runs as two units of half its width; each unit writes its share of the tile's
    // row-statistics partial planes (2 per tile, 4 for block_n 320), so every plane is written exactly once per row
    // GEGLU (no row statistics, so no planes to share out) runs on the widest unit: more MMA per unit and per staged byte
    const int unit_n = geglu ? 160 : (bn > 160 ? bn / 2 : bn);
    const int tile_units = geglu ? 1 : bn / unit_n;
    p.n_units = geglu ? (d->N + 159) / 160 : (d->N + bn - 1) / bn * tile_units;
    p.units = m_tiles * p.n_units;
    p.stats_unit_planes = (bn == 320 ? 4 : 2) / tile_units;
    p.bias = d->bias;
    p.rowvec = d->rowvec;
    p.rowvec_ld = d->rowvec_ld;
    p.residual = d->residual;
    p.residual_ld = d->residual_ld;
    p.act_silu = act;  // 0 none, 1 SiLU, 2 quick_gelu, 3 erf-gelu, 4 tanh-gelu, 5 ReLU
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
    OMG_CHECK(d->w_group_planes == 0 || !d->w2, "omg_gemm: weight planes do not extend to the second weight matrix (w2)");
    // A tile must not mix two row groups (the producer picks the weight plane, the epilogue the c1 / c2 plane, from the
    // tile's first pixel).  Token GEMMs (H == 1) walk 128 consecutive rows per tile: boundaries are multiples of 128.
    // On a spatial grid a tile is a tw x th patch of ONE image, so boundaries are whole numbers of images.
    const long long img_pix = (long long)W * H;
    for (int i = 0; i < 8; ++i) {
        p.col_group_end[i] = d->col_group_end[i];
        if (i + 1 >= p.n_col_groups) continue;
        if (H > 1)
            OMG_CHECK(d->col_group_end[i] % img_pix == 0,
                      "omg_gemm: row-group boundary %lld is inside an image of the %d x %d output grid (boundaries are "
                      "multiples of %lld pixels)", (long long)d->col_group_end[i], W, H, img_pix);
        else
            OMG_CHECK(d->col_group_end[i] % 128 == 0, "omg_gemm: row-group boundary %lld is not a multiple of the 128-row tile",
                      (long long)d->col_group_end[i]);
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
        if (view_to_tmap(&p.a_maps[i], d->a[i], tdt, BK, tw, th, CU_TENSOR_MAP_SWIZZLE_128B)) return 1;
    }
    for (int i = d->n_a; i < OMG_MAX_A; ++i) p.a_maps[i] = p.a_maps[0];
    {
        const uint64_t planes = d->w_group_planes > 0 ? (uint64_t)d->w_group_planes : 1;
        const uint64_t dims[2] = {(uint64_t)d->Ktot, (uint64_t)d->N * planes};
        const uint64_t strides[2] = {1, (uint64_t)d->Ktot};
        const uint32_t box[2] = {BK, (uint32_t)unit_n};
        if (make_tmap(&p.b_maps[0], tdt, d->w, 2, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B)) return 1;
        p.b_maps[1] = p.b_maps[0];
    }
    if (d->w2 != nullptr) {
        OMG_CHECK(d->K2tot >= 8 && d->K2tot % 8 == 0, "omg_gemm: K2tot=%d must be a positive multiple of 8", d->K2tot);
        const uint64_t dims[2] = {(uint64_t)d->K2tot, (uint64_t)d->N};
        const uint64_t strides[2] = {1, (uint64_t)d->K2tot};
        const uint32_t box[2] = {BK, (uint32_t)unit_n};
        if (make_tmap(&p.b_maps[1], tdt, d->w2, 2, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B)) return 1;
    }
    OMG_CHECK(d->d.sw % 2 == 0 && d->d.sh % 2 == 0 && d->d.sb % 2 == 0 && (reinterpret_cast<uintptr_t>(d->d.ptr) & 3) == 0,
              "omg_gemm: output view must be 4 B aligned per pixel");
    p.out = const_cast<void*>(d->d.ptr);
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

    if (bf16) {  // lean (FEAT 0) OMG_EPI_NONE units only: every other feature was rejected above
        switch (unit_n) {
            case 64: return launch_gemm_f<__nv_bfloat16, 64, OMG_EPI_NONE, 0>(p, stream);
            case 128: return launch_gemm_f<__nv_bfloat16, 128, OMG_EPI_NONE, 0>(p, stream);
            default: return launch_gemm_f<__nv_bfloat16, 160, OMG_EPI_NONE, 0>(p, stream);
        }
    }
    if (geglu) return launch_gemm<160, OMG_EPI_GEGLU>(p, false, stream);
    // The residual is staged by TMA when a tensor map can describe it: 16 B aligned base (ld % 8 == 0 is checked above).
    // Otherwise the epilogue reads it from global memory as before.  Boxes clip at N and at the grid's edges, so columns
    // past N and pixels outside the image are zero-filled, never read.
    bool res_staged = false;
    if (d->residual != nullptr && (reinterpret_cast<uintptr_t>(d->residual) & 15) == 0) {
        const uint64_t ld = (uint64_t)d->residual_ld;
        const uint64_t dims[4] = {(uint64_t)N_out, (uint64_t)W, (uint64_t)H, (uint64_t)B};
        const uint64_t strides[4] = {1, ld, ld * W, ld * W * H};
        const uint32_t box[4] = {32, (uint32_t)tw, (uint32_t)th, 1};
        res_staged = make_tmap(&p.res_map, tdt, d->residual, 4, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_64B) == 0;
    }
    switch (unit_n) {
        case 64: return launch_gemm<64, OMG_EPI_NONE>(p, res_staged, stream);
        case 128: return launch_gemm<128, OMG_EPI_NONE>(p, res_staged, stream);
        default: return launch_gemm<160, OMG_EPI_NONE>(p, res_staged, stream);
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
