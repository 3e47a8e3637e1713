// wgmma flash attention for prefill / ViT (sm_90a): S = Q·K^T and O += P·V on the Hopper tensor cores with fp32
// accumulators in registers, TMA-fed operands, fp32 online softmax on the accumulator fragment.
//
// Replaces the eager attention of the reference's HF path, which materialises the [B,H,S,S] score matrix
// (transformers modeling_llama.py:199-221 eager_attention_forward; modeling_clip.py:261-279).
//
// CTA = one (batch, head, 128-query tile); 288 threads:
//   warp 8 / lane 0 : TMA producer — Q once, then K_j / V_j tiles (128 keys) into separate two-stage rings
//                     (4-D tensor maps over the strided [b, t, h, d] views: the same kernel reads the fused qkv
//                     activation buffer of the ViT and the [B, H, Smax, 128] KV cache of the decoder)
//   warps 0..7      : two consumer warpgroups of 64 query rows each:
//                     S = Q K_j^T   (wgmma m64n128k16, both operands K-major in shared memory, SWIZZLE_128B)
//                     softmax on the fragment: a query row lives in the four threads of a quad (scale/mask, running max /
//                     sum, O rescaled in registers), P = exp2(s - m) packed to bf16 IS the A-operand fragment of the next MMA
//                     O += P_j V_j  (wgmma m64nDk16, P from registers, V straight from its [keys, d] tile as an MN-major
//                     operand — no transpose pass), finally O / l -> global.
// mbarriers: q_full, k_full[2], k_empty[2], v_full[2], v_empty[2].
#include <cuda.h>
#include <math.h>
#include <stdlib.h>

#include "common.cuh"
#include "kernels.h"

namespace b2 {
namespace {

constexpr int TC_BM = 128;  // queries per CTA
constexpr int TC_BN = 128;  // keys per tile
constexpr int TC_THREADS = 288;
constexpr int TC_CONSUMER_WARPS = 8;

__device__ __forceinline__ void tma_load_4d(void* smem_dst, const void* tmap, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}
// MUFU.EX2 without exp2f's denormal-range fix-up (inputs here are <= 0, results feed a bf16 / an fp32 sum)
__device__ __forceinline__ float ex2_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

struct FlashTcParams {
    const int32_t* seq_lens;
    const int32_t* pos0;  // OFFSET only: absolute position of query row 0 of each sample (keys 0 .. pos0 + t are attended)
    __nv_bfloat16* o;
    int64_t o_bs, o_ts, o_hs;
    int S;
    float scale_log2;
};

template <int D>
struct TcCfg {
    static constexpr int SMEM = 5 * TC_BN * D * 2 + 1024 /*align*/ + 128 /*barriers*/;  // Q + 2 K stages + 2 V stages
};

// OFFSET: the queries of sample b are a chunk appended at cache position pos0[b] (query row t sits at absolute position
// pos0[b] + t) and K / V are the whole cache [B][H][Smax][D]. Key tiles stay aligned to absolute position 0; masks compare
// absolute positions. OFFSET == false is the position-0 kernel (qpos0 folds to 0).
template <int D, bool CAUSAL, bool OFFSET>
__global__ void __launch_bounds__(TC_THREADS, 1)
flash_wgmma_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_k,
                   const __grid_constant__ CUtensorMap tm_v, FlashTcParams p) {
    constexpr int SLABS = D / 64;                 // 64-wide (128 B) slabs of the head dim
    constexpr int TILE_BYTES = TC_BN * D * 2;     // one Q / K / V tile
    constexpr int SLAB_BYTES = TC_BN * 128;       // [128 rows x 128 B]

    extern __shared__ uint8_t tc_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(tc_raw) + 1023) & ~static_cast<uintptr_t>(1023));
    uint8_t* sQ = smem;
    uint8_t* sK = sQ + TILE_BYTES;            // [2][TILE_BYTES]
    uint8_t* sV = sK + 2 * TILE_BYTES;        // [2][TILE_BYTES]
    uint64_t* bars = reinterpret_cast<uint64_t*>(sV + 2 * TILE_BYTES);
    uint64_t* q_full = bars;
    uint64_t* k_full = bars + 1;    // [2]
    uint64_t* k_empty = bars + 3;   // [2]
    uint64_t* v_full = bars + 5;    // [2]
    uint64_t* v_empty = bars + 7;   // [2]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int q0 = blockIdx.x * TC_BM;
    const int head = blockIdx.y, b = blockIdx.z;
    pdl_trigger();
    pdl_wait();  // q/k/v (and seq_lens) are outputs of upstream kernels (programmatic dependent launch)
    const int len = p.seq_lens != nullptr ? p.seq_lens[b] : p.S;
    const int qpos0 = OFFSET ? p.pos0[b] : 0;
    const int kv_len = qpos0 + len;  // keys of this sample: [0, kv_len)
    const int kv_end = CAUSAL ? min(kv_len, qpos0 + q0 + TC_BM) : kv_len;
    const int n_tiles = (kv_end + TC_BN - 1) / TC_BN;  // >= 1 (len >= 1)

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tm_q);
        tma_prefetch_desc(&tm_k);
        tma_prefetch_desc(&tm_v);
        mbar_init(q_full, 1);
        for (int s = 0; s < 2; ++s) {
            mbar_init(&k_full[s], 1); mbar_init(&k_empty[s], TC_CONSUMER_WARPS);
            mbar_init(&v_full[s], 1); mbar_init(&v_empty[s], TC_CONSUMER_WARPS);
        }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == TC_CONSUMER_WARPS) {
        if (lane == 0) {
            // ---------------- TMA producer ----------------
            mbar_arrive_expect_tx(q_full, TILE_BYTES);
            for (int sl = 0; sl < SLABS; ++sl) tma_load_4d(sQ + sl * SLAB_BYTES, &tm_q, q_full, sl * 64, q0, head, b);
            for (int j = 0; j < n_tiles; ++j) {
                const int s = j & 1;
                const uint32_t ph = (j >> 1) & 1;
                mbar_wait(&k_empty[s], ph ^ 1);
                mbar_arrive_expect_tx(&k_full[s], TILE_BYTES);
                for (int sl = 0; sl < SLABS; ++sl)
                    tma_load_4d(sK + s * TILE_BYTES + sl * SLAB_BYTES, &tm_k, &k_full[s], sl * 64, j * TC_BN, head, b);
                mbar_wait(&v_empty[s], ph ^ 1);
                mbar_arrive_expect_tx(&v_full[s], TILE_BYTES);
                for (int sl = 0; sl < SLABS; ++sl)
                    tma_load_4d(sV + s * TILE_BYTES + sl * SLAB_BYTES, &tm_v, &v_full[s], sl * 64, j * TC_BN, head, b);
            }
        }
    } else {
        // ---------------- consumer warpgroups: 64 query rows each; a row lives in the 4 threads of a quad ----------------
        const int wg = warp >> 2;
        const int tid = threadIdx.x & 127;
        const int c2 = 2 * (lane & 3);
        int rows[2];   // the two query rows of this thread's fragment, relative to q0
        rows[0] = 64 * wg + 16 * (warp & 3) + (lane >> 2);
        rows[1] = rows[0] + 8;
        float o[D / 2];
#pragma unroll
        for (int i = 0; i < D / 2; ++i) o[i] = 0.f;
        float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
        const uint32_t q_addr = smem_u32(sQ) + wg * (64 * 128);
        mbar_wait(q_full, 0);
        for (int j = 0; j < n_tiles; ++j) {
            const int s = j & 1;
            const uint32_t ph = (j >> 1) & 1;
            const int key0 = j * TC_BN;
            float sc[TC_BN / 2];  // RAW scores (masked -> -inf); the softmax scale is folded into the exponent's FMA below
            mbar_wait(&k_full[s], ph);
            wgmma_fence();
            // S = Q K_j^T : K-loop over the head dim in steps of 16 (32 B inside a 128 B swizzle row; slabs of 64)
#pragma unroll
            for (int k = 0; k < D / 16; ++k) {
                const uint32_t off = (k >> 2) * SLAB_BYTES + (k & 3) * 32;
                wgmma_bf16_ss<TC_BN>(sc, make_sw128_kmajor_desc(q_addr + off),
                                     make_sw128_kmajor_desc(smem_u32(sK + s * TILE_BYTES) + off), k != 0 ? 1u : 0u);
            }
            wgmma_commit();
            wgmma_wait<0>();
            if (lane == 0) mbar_arrive(&k_empty[s]);  // K_j consumed
            // interior tiles need no per-key mask (CTA-uniform test: every key valid for every query row of this CTA)
            const bool full_tile = (key0 + TC_BN <= kv_len) && (!CAUSAL || key0 + TC_BN - 1 <= qpos0 + q0);
            float mx[2] = {-INFINITY, -INFINITY};
            if (!full_tile) {
#pragma unroll
                for (int i = 0; i < TC_BN / 2; ++i) {
                    const int key = key0 + frag_col(tid, i);
                    bool ok = key < kv_len;
                    if (CAUSAL) ok = ok && (key <= qpos0 + q0 + rows[(i >> 1) & 1]);
                    if (!ok) sc[i] = -INFINITY;
                }
            }
#pragma unroll
            for (int i = 0; i < TC_BN / 2; ++i) mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], sc[i]);
            float m_use[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
                mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
                mx[h] *= p.scale_log2;  // scale > 0: max commutes with the scaling (-inf stays -inf)
                const float m_new = fmaxf(m_run[h], mx[h]);
                m_use[h] = (m_new == -INFINITY) ? 0.f : m_new;
                const float corr = exp2f(m_run[h] - m_use[h]);  // m_run = -inf -> 0
                m_run[h] = m_new;
                l_run[h] *= corr;
#pragma unroll
                for (int i = 0; i < D / 2; ++i)
                    if (((i >> 1) & 1) == h) o[i] *= corr;
            }
            // P = exp2(s - m) as bf16: fragment elements (8kk .. 8kk+7) are exactly the A operand of k-step kk
            uint32_t pa[TC_BN / 4];
#pragma unroll
            for (int i = 0; i < TC_BN / 2; i += 2) {
                const int h = (i >> 1) & 1;
                const float p0 = ex2_approx(fmaf(sc[i], p.scale_log2, -m_use[h]));      // -inf -> +0
                const float p1 = ex2_approx(fmaf(sc[i + 1], p.scale_log2, -m_use[h]));
                l_run[h] += p0 + p1;
                pa[i >> 1] = pack_bf16(p0, p1);
            }
            mbar_wait(&v_full[s], ph);
            wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < TC_BN / 16; ++kk) {
                const uint32_t a[4] = {pa[4 * kk], pa[4 * kk + 1], pa[4 * kk + 2], pa[4 * kk + 3]};
                // V: MN-major, 16 key rows per step
                wgmma_bf16_rs_tb<D>(o, a, make_sw128_mnmajor_desc(smem_u32(sV + s * TILE_BYTES) + kk * 16 * 128, SLAB_BYTES));
            }
            wgmma_commit();
            wgmma_wait<0>();
            if (lane == 0) mbar_arrive(&v_empty[s]);  // V_j consumed
        }
        // ---- epilogue: O / l (each thread summed its own columns of the row: finish the sum over the quad) ----
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            float l = l_run[h];
            l += __shfl_xor_sync(0xffffffffu, l, 1);
            l += __shfl_xor_sync(0xffffffffu, l, 2);
            const float inv = l > 0.f ? 1.f / l : 0.f;
            const int qrow = q0 + rows[h];
            if (qrow >= p.S) continue;
            __nv_bfloat16* orow = p.o + b * p.o_bs + (int64_t)qrow * p.o_ts + head * p.o_hs;
#pragma unroll
            for (int jj = 0; jj < D / 8; ++jj)
                *reinterpret_cast<uint32_t*>(orow + 8 * jj + c2) = pack_bf16(o[4 * jj + 2 * h] * inv, o[4 * jj + 2 * h + 1] * inv);
        }
    }
}

// ------------------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                    CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                    CUtensorMapFloatOOBfill);

// 4-D view (d, t, h, b) of a bf16 tensor with element strides (1, ts, hs, bs); box = [64, 128, 1, 1], SWIZZLE_128B
int make_tmap_4d(CUtensorMap* map, const void* ptr, int D, int S, int H, int B, int64_t ts, int64_t hs, int64_t bs) {
    static PFN_encodeTiled fn = nullptr;
    if (fn == nullptr) {
        void* f = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &qres) != cudaSuccess ||
            qres != cudaDriverEntryPointSuccess || f == nullptr) {
            set_error("cuTensorMapEncodeTiled entry point unavailable");
            return -2;
        }
        fn = reinterpret_cast<PFN_encodeTiled>(f);
    }
    if ((reinterpret_cast<uintptr_t>(ptr) & 15) != 0 || (ts * 2) % 16 != 0 || (hs * 2) % 16 != 0 || (bs * 2) % 16 != 0) {
        set_error("flash_attn: operands must be 16B aligned with 16B-multiple strides");
        return -1;
    }
    cuuint64_t dims[4] = {(cuuint64_t)D, (cuuint64_t)S, (cuuint64_t)H, (cuuint64_t)B};
    cuuint64_t strides[3] = {(cuuint64_t)(ts * 2), (cuuint64_t)(hs * 2), (cuuint64_t)(bs * 2)};
    cuuint32_t box[4] = {64, (cuuint32_t)TC_BN, 1, 1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(ptr), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled(4d) failed (%d): D=%d S=%d H=%d B=%d ts=%lld hs=%lld bs=%lld", (int)r, D, S, H,
                  B, (long long)ts, (long long)hs, (long long)bs);
        return -2;
    }
    return 0;
}

template <int D, bool CAUSAL, bool OFFSET>
int launch_tc(const FlashArgs& a, cudaStream_t stream) {
    const int skv = OFFSET ? a.Skv : a.S;  // rows of the K / V views
    CUtensorMap tq, tk, tv;
    B2_TRY(make_tmap_4d(&tq, a.q, D, a.S, a.H, a.B, a.q_ts, a.q_hs, a.q_bs));
    B2_TRY(make_tmap_4d(&tk, a.k, D, skv, a.H, a.B, a.k_ts, a.k_hs, a.k_bs));
    B2_TRY(make_tmap_4d(&tv, a.v, D, skv, a.H, a.B, a.v_ts, a.v_hs, a.v_bs));
    FlashTcParams p;
    p.seq_lens = a.seq_lens;
    p.pos0 = a.pos0;
    p.o = reinterpret_cast<__nv_bfloat16*>(a.o);
    p.o_bs = a.o_bs; p.o_ts = a.o_ts; p.o_hs = a.o_hs;
    p.S = a.S;
    p.scale_log2 = a.scale * 1.4426950408889634f;
    constexpr int smem = TcCfg<D>::SMEM;
    static bool attr_set = false;
    auto kern = flash_wgmma_kernel<D, CAUSAL, OFFSET>;
    if (!attr_set) {
        B2_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        attr_set = true;
    }
    dim3 grid((a.S + TC_BM - 1) / TC_BM, a.H, a.B);
    B2_CUDA_CHECK(launch_pdl(kern, grid, dim3(TC_THREADS), (size_t)smem, stream, tq, tk, tv, p));
    B2_LAUNCH_CHECK();
    return 0;
}

}  // namespace

int flash_attn_bf16(const FlashArgs& a, cudaStream_t stream) {
    B2_CHECK_ARG(a.D == 64 || a.D == 128, "flash_attn: head_dim must be 64 or 128 (got %d)", a.D);
    B2_CHECK_ARG(a.B > 0 && a.H > 0 && a.S > 0, "flash_attn: empty problem");
    B2_CHECK_ARG((a.o_ts % 8) == 0 && (a.o_hs % 8) == 0 && (a.o_bs % 8) == 0 && (reinterpret_cast<uintptr_t>(a.o) & 15) == 0,
                 "flash_attn: output must be 16B aligned with 16B-multiple strides");
    if (a.pos0 != nullptr) {
        // chunk against a cache: causal, head_dim 128 (the decoder's attention) only
        B2_CHECK_ARG(a.D == 128 && a.causal && a.Skv >= 1, "flash_attn: offset queries need D=128, causal, Skv >= 1 (D=%d causal=%d Skv=%d)",
                     a.D, a.causal, a.Skv);
        return launch_tc<128, true, true>(a, stream);
    }
    if (a.D == 64) return a.causal ? launch_tc<64, true, false>(a, stream) : launch_tc<64, false, false>(a, stream);
    return a.causal ? launch_tc<128, true, false>(a, stream) : launch_tc<128, false, false>(a, stream);
}

}  // namespace b2
