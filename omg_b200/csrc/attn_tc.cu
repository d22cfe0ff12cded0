// Flash attention on wgmma for the SDXL transformer blocks (head_dim 64): self-attention (N = 1024 / 4096 keys)
// and cross-attention (77 text keys, 16 IP-adapter keys), never materialising the probability matrix.
//
// Prompt-to-prompt control and decoupled (IP-adapter) attention are expressed through the descriptor instead of
// through a probability callback (reference: src/pipelines/lora_pipeline.py:114-116 + src/prompt_attention/
// p2p_attention.py:124-138, src/ip_adapter/attention_processor.py:370-409):
//   * every output batch row names the batch rows its Q, K and V come from  -> "replace self-attention"
//     out_1 = softmax(Q_0 K_0^T) V_1 is a pointer remap;
//   * `accumulate` + `out_weight` add a second separately-normalised term    -> txt + scale * ip, and the general
//     cross-attention edit  P_0 (M diag(a) V_1) + P_1 (diag(1-a) V_1).
//
// CTA = one (item, head, 128-query tile), two CTAs per SM, 256 threads: warpgroups 0 and 1 each own 64 query rows
// (S = Q K^T and O += P V on wgmma, softmax in registers).  Thread 0 streams Q and the K / V blocks (64 keys) through
// a ring of shared-memory stages with TMA: it refills the stage of block j - 1 once block j's Q.K^T is issued, so
// the loads run ATT_KV_STAGES - 1 blocks ahead and no registers are spent on a producer warpgroup.  P never touches shared memory: the S accumulator is
// converted in registers into the A operand of the P.V wgmma.  The softmax is the online (running maximum) form;
// keys beyond n_kv (zero-filled by TMA) and, for causal masking, keys after the query are excluded.
#include <cuda_fp16.h>

#include <algorithm>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/omg_b200.h"
#include "host_common.h"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace omg {

constexpr int ATT_BQ = 128;       // query rows per CTA
constexpr int ATT_BKV = 64;       // keys per block
constexpr int ATT_D = 64;
constexpr int ATT_Q_BYTES = ATT_BQ * ATT_D * 2;    // 16 KB
constexpr int ATT_K_BYTES = ATT_BKV * ATT_D * 2;   // 8 KB (K) ; V same
constexpr int ATT_KV_STAGES = 4;
constexpr int ATT_THREADS = 256;
constexpr int ATT_SMEM = 1024 + ATT_Q_BYTES + ATT_KV_STAGES * 2 * ATT_K_BYTES + 256;

struct alignas(64) AttnParams {
    CUtensorMap q_map, k_map, v_map;  // 3D (cols, tokens, batch), box (64, 128 | 64, 1), SWIZZLE_128B
    __half* out;
    int out_ld;
    long long out_bs;
    int n_q, n_kv, heads;
    int q_col0, k_col0, v_col0, out_col0;
    int n_items;
    int out_b[OMG_ATTN_MAX_ITEMS], q_b[OMG_ATTN_MAX_ITEMS], k_b[OMG_ATTN_MAX_ITEMS], v_b[OMG_ATTN_MAX_ITEMS];
    float scale_log2;  // softmax scale * log2(e)
    float out_weight;
    int accumulate;
    int causal;        // key index > query index is masked
};

__global__ void __launch_bounds__(ATT_THREADS, 2) attn_tc_kernel(const __grid_constant__ AttnParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* q_smem = smem;
    uint8_t* kv_smem = q_smem + ATT_Q_BYTES;  // stages x (K 8 KB | V 8 KB)
    uint64_t* q_full = reinterpret_cast<uint64_t*>(kv_smem + ATT_KV_STAGES * 2 * ATT_K_BYTES);
    uint64_t* kv_full = q_full + 1;               // [stage]
    uint64_t* kv_empty = kv_full + ATT_KV_STAGES;  // [stage] both warpgroups' MMAs on the stage have completed

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int slab = blockIdx.x, head = blockIdx.y, item = blockIdx.z;
    const int nkv = (p.n_kv + ATT_BKV - 1) / ATT_BKV;

    const int kb = p.k_b[item], vb = p.v_b[item];
    auto load_kv = [&](int jb) {  // thread 0: block jb into its stage, once both warpgroups have released the stage
        const int st = jb % ATT_KV_STAGES;
        mbar_wait_nocall(&kv_empty[st], ((jb / ATT_KV_STAGES) & 1) ^ 1);
        uint8_t* kd = kv_smem + st * 2 * ATT_K_BYTES;
        mbar_arrive_expect_tx(&kv_full[st], 2 * ATT_K_BYTES);
        tma_load_3d(kd, &p.k_map, &kv_full[st], p.k_col0 + head * ATT_D, jb * ATT_BKV, kb);
        tma_load_3d(kd + ATT_K_BYTES, &p.v_map, &kv_full[st], p.v_col0 + head * ATT_D, jb * ATT_BKV, vb);
    };
    if (threadIdx.x == 0) {
        tma_prefetch_desc(&p.q_map);
        tma_prefetch_desc(&p.k_map);
        tma_prefetch_desc(&p.v_map);
        mbar_init(q_full, 1);
        for (int i = 0; i < ATT_KV_STAGES; ++i) {
            mbar_init(&kv_full[i], 1);
            mbar_init(&kv_empty[i], 2);
        }
        fence_barrier_init();
    }
    __syncthreads();
    griddep_launch_dependents();
    griddep_wait();
    if (threadIdx.x == 0) {
        mbar_arrive_expect_tx(q_full, ATT_Q_BYTES);
        tma_load_3d(q_smem, &p.q_map, q_full, p.q_col0 + head * ATT_D, slab * ATT_BQ, p.q_b[item]);
        for (int jb = 0; jb < ATT_KV_STAGES && jb < nkv; ++jb) load_kv(jb);
    }

    const int wg = warp >> 2, wi = warp & 3;
    const int g = lane >> 2, c = lane & 3;
    // rows of this thread: r0 = g and r1 = g + 8 of the warp's 16 (accumulator layout, see wgmma.cuh)
    const int qrow0 = slab * ATT_BQ + wg * 64 + wi * 16 + g;
    const uint32_t q_addr = smem_u32(q_smem) + wg * (64 * 128);
    float o[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
    mbar_wait_nocall(q_full, 0);
    for (int j = 0; j < nkv; ++j) {
        const int st = j % ATT_KV_STAGES;
        mbar_wait_nocall(&kv_full[st], (j / ATT_KV_STAGES) & 1);
        const uint32_t k_addr = smem_u32(kv_smem + st * 2 * ATT_K_BYTES);
        float s[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) s[i] = 0.f;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < ATT_D / 16; ++k)
            wgmma_ss_n64(s, gmma_desc_sw128(q_addr + k * 32, 1024, 16), gmma_desc_sw128(k_addr + k * 32, 1024, 16), 1u);
        wgmma_commit();
        if (threadIdx.x == 0 && j >= 1 && j - 1 + ATT_KV_STAGES < nkv) load_kv(j - 1 + ATT_KV_STAGES);
        __syncwarp();
        wgmma_wait<0>();
        reg_fence(s);
        // mask: keys beyond n_kv (partial last block) and, causal, keys after the query
        const int key0 = j * ATT_BKV + 2 * c;
        if ((j + 1) * ATT_BKV > p.n_kv || p.causal) {  // a block with keys past n_kv, for every lane alike
#pragma unroll
            for (int J = 0; J < 8; ++J)
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int key = key0 + 8 * J + e;
                        if (key >= p.n_kv || (p.causal && key > qrow0 + 8 * h)) s[4 * J + 2 * h + e] = -INFINITY;
                    }
        }
        float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int J = 0; J < 8; ++J)
#pragma unroll
            for (int h = 0; h < 2; ++h) mx[h] = fmaxf(mx[h], fmaxf(s[4 * J + 2 * h], s[4 * J + 2 * h + 1]));
        float corr[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
            mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
            const float m_new = fmaxf(m[h], mx[h] * p.scale_log2);
            corr[h] = fast_exp2(m[h] - m_new);  // 0 on the first block (m = -inf)
            m[h] = m_new;
            l[h] *= corr[h];
        }
#pragma unroll
        for (int J = 0; J < 8; ++J)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                o[4 * J + 2 * h] *= corr[h];
                o[4 * J + 2 * h + 1] *= corr[h];
            }
        // P = exp2(S * scale - m) as fp16 A fragments of P.V: keys 16kk .. 16kk + 15 are accumulator chunks 2kk, 2kk + 1
        uint32_t pa[4][4];
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
#pragma unroll
            for (int t = 0; t < 4; ++t) {  // t: (row g | g + 8) x (keys 2c | 8 + 2c)
                const int h = t & 1, i0 = 8 * kk + 4 * (t >> 1) + 2 * h;
                const float p0 = fast_exp2(fmaf(s[i0], p.scale_log2, -m[h]));
                const float p1 = fast_exp2(fmaf(s[i0 + 1], p.scale_log2, -m[h]));
                l[h] += p0 + p1;
                pa[kk][t] = pack_half2(p0, p1);
            }
        const uint32_t v_addr = k_addr + ATT_K_BYTES;
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)  // V: 16 key rows (2 KB) per K step, MN-major
            wgmma_rs_n64_tb(o, pa[kk], gmma_desc_sw128(v_addr + kk * 2048, 1024, 1024), 1u);
        wgmma_commit();
        wgmma_wait<0>();
        reg_fence(o);
        if ((threadIdx.x & 127) == 0) mbar_arrive(&kv_empty[st]);
    }

    // finalise: out = (accumulate ? out : 0) + w * O / l
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        l[h] += __shfl_xor_sync(0xffffffffu, l[h], 1);
        l[h] += __shfl_xor_sync(0xffffffffu, l[h], 2);
        const int qrow = qrow0 + 8 * h;
        if (qrow < p.n_q) {
            const float inv = p.out_weight / l[h];
            __half* op = p.out + (long long)p.out_b[item] * p.out_bs + (long long)qrow * p.out_ld + p.out_col0 +
                         head * ATT_D + 2 * c;
#pragma unroll
            for (int J = 0; J < 8; ++J) {
                float v0 = o[4 * J + 2 * h] * inv, v1 = o[4 * J + 2 * h + 1] * inv;
                __half2* dst = reinterpret_cast<__half2*>(op + 8 * J);
                if (p.accumulate) {
                    const float2 f = __half22float2(*dst);
                    v0 += f.x;
                    v1 += f.y;
                }
                *dst = __floats2half2_rn(v0, v1);
            }
        }
    }
}

static int make_attn_map(CUtensorMap* m, const void* ptr, int cols, int ld, int tokens, long long bs, int nb,
                         uint32_t box_rows) {
    const uint64_t dims[3] = {(uint64_t)cols, (uint64_t)tokens, (uint64_t)nb};
    const uint64_t strides[3] = {1, (uint64_t)ld, (uint64_t)bs};
    const uint32_t box[3] = {64, box_rows, 1};
    return make_tmap(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, ptr, 3, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
}

}  // namespace omg

using namespace omg;

static int attention_impl(const omg_attn_desc* d, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    OMG_CHECK(d != nullptr, "omg_attention: null descriptor");
    OMG_CHECK(d->head_dim == 64, "omg_attention: head_dim %d unsupported (SDXL uses 64)", d->head_dim);
    OMG_CHECK(d->n_items >= 1 && d->n_items <= OMG_ATTN_MAX_ITEMS, "omg_attention: n_items=%d out of range",
              d->n_items);
    OMG_CHECK(d->n_q >= 1 && d->n_kv >= 1 && d->heads >= 1, "omg_attention: empty problem");
    OMG_CHECK(d->q && d->k && d->v && d->out, "omg_attention: null pointer");
    OMG_CHECK(d->out_ld % 8 == 0 && d->out_col0 % 8 == 0 && d->out_bs % 8 == 0,
              "omg_attention: output must be 16 B aligned per row");
    if (check_head_windows("omg_attention", d->heads, d->head_dim, {d->q_col0, d->k_col0, d->v_col0, d->out_col0},
                           {d->q_ld, d->k_ld, d->v_ld, d->out_ld}))
        return 1;
    OMG_CHECK(!d->causal || (d->n_kv <= 128 && d->n_q <= 128), "omg_attention: causal masking is available for sequences of <= 128 tokens");
    static bool configured = false;
    if (!configured) {
        OMG_CUDA(cudaFuncSetAttribute(attn_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ATT_SMEM));
        configured = true;
    }
    AttnParams p;
    memset(&p, 0, sizeof(p));
    int max_qb = 0, max_kb = 0, max_vb = 0;
    for (int i = 0; i < d->n_items; ++i) {
        p.out_b[i] = d->out_b[i];
        p.q_b[i] = d->q_b[i];
        p.k_b[i] = d->k_b[i];
        p.v_b[i] = d->v_b[i];
        max_qb = d->q_b[i] > max_qb ? d->q_b[i] : max_qb;
        max_kb = d->k_b[i] > max_kb ? d->k_b[i] : max_kb;
        max_vb = d->v_b[i] > max_vb ? d->v_b[i] : max_vb;
        OMG_CHECK(d->out_b[i] >= 0 && d->q_b[i] >= 0 && d->k_b[i] >= 0 && d->v_b[i] >= 0,
                  "omg_attention: negative batch index in item %d", i);
    }
    const int cols = d->heads * 64;
    if (make_attn_map(&p.q_map, d->q, d->q_col0 + cols, d->q_ld, d->n_q, d->q_bs, max_qb + 1, ATT_BQ)) return 1;
    if (make_attn_map(&p.k_map, d->k, d->k_col0 + cols, d->k_ld, d->n_kv, d->k_bs, max_kb + 1, ATT_BKV)) return 1;
    if (make_attn_map(&p.v_map, d->v, d->v_col0 + cols, d->v_ld, d->n_kv, d->v_bs, max_vb + 1, ATT_BKV)) return 1;
    p.out = static_cast<__half*>(d->out);
    p.out_ld = d->out_ld;
    p.out_bs = d->out_bs;
    p.n_q = d->n_q;
    p.n_kv = d->n_kv;
    p.heads = d->heads;
    p.q_col0 = d->q_col0;
    p.k_col0 = d->k_col0;
    p.v_col0 = d->v_col0;
    p.out_col0 = d->out_col0;
    p.n_items = d->n_items;
    p.scale_log2 = d->scale * 1.4426950408889634f;
    p.out_weight = d->out_weight;
    p.accumulate = d->accumulate;
    p.causal = d->causal;
    dim3 grid((d->n_q + ATT_BQ - 1) / ATT_BQ, d->heads, d->n_items);
    OMG_CUDA(launch_pdl(attn_tc_kernel, grid, dim3(ATT_THREADS), ATT_SMEM, stream, p));
    return check_launch("attn_tc_kernel");
}

// C-ABI entry points: launch, and - while this thread records a launch plan (omg_plan_record_begin) - remember the call
extern "C" int omg_attention(const omg_attn_desc* d, void* stream_) {
    const int rc = attention_impl(d, stream_);
    if (rc == 0 && ::omg::plan_recording()) {
        const omg_attn_desc c = *d;  // by value: a plan outlives the caller's descriptor
        ::omg::plan_note([c](void* s) { return attention_impl(&c, s); });
    }
    return rc;
}
