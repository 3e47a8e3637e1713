// Persistent warp-specialised bf16 GEMM for sm_90a:  C[M,N] = epilogue(A[M,K] · W[N,K]^T)
//
//   * A (activations, row-major, K contiguous) and W (nn.Linear weight [out,in], K contiguous) are both
//     "K-major" operands: TMA (cp.async.bulk.tensor.2d, SWIZZLE_128B) stages 128x64 / BNx64 bf16 tiles
//     into shared memory; two consumer warpgroups issue wgmma.mma_async (m64 x n x k16, fp32 accumulators in
//     registers) for 64 rows each straight out of shared memory and apply the fused epilogue from the fragment.
//   * One pipeline: smem full/empty mbarrier ring (TMA producer warp <-> consumer warpgroups); the producer runs ahead
//     into the next tile while the consumers are in their epilogue. Static persistent tile scheduler (grid = #SMs)
//     with grouped rasterisation for L2 reuse.
//   * CTA-pair variant for the big-M launches (ViT at large batch, LLaMA prefill): clusters of two CTAs share a 256x256
//     tile and fetch each W tile once, by TMA multicast. It also carries the fused RoPE + KV-cache-write epilogue.
//   * Fused epilogues replace the separate bias / activation / residual / silu*mul kernels of the
//     reference's HF path (transformers modeling_clip.py:347-351 CLIPMLP, modeling_llama.py:182-184
//     LlamaMLP, :303-332 residual adds; llava/model/multimodal_projector/builder.py:42-46).
#include <cuda.h>
#include <math.h>
#include <stdlib.h>

#include "common.cuh"
#include "kernels.h"

namespace b2 {

static int g_num_sms = 0;
int num_sms() {
    if (g_num_sms == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
        if (g_num_sms <= 0) g_num_sms = 132;
    }
    return g_num_sms;
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                    CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                    CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode_fn() {
    static PFN_encodeTiled fn = nullptr;
    if (fn == nullptr) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
        if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || p == nullptr) return nullptr;
        fn = reinterpret_cast<PFN_encodeTiled>(p);
    }
    return fn;
}

// 2D bf16 row-major [rows, cols] with leading dimension ld (elements); box = [box_rows, 64]. Shared with gemm_skinny.cu.
int make_tmap_bf16(CUtensorMap* map, const void* ptr, int64_t rows, int64_t cols, int64_t ld, int box_rows) {
    PFN_encodeTiled fn = get_encode_fn();
    if (fn == nullptr) {
        set_error("cuTensorMapEncodeTiled entry point unavailable");
        return -2;
    }
    if ((reinterpret_cast<uintptr_t>(ptr) & 15) != 0 || (ld * 2) % 16 != 0) {
        set_error("TMA operand must be 16B aligned with a 16B-multiple row pitch (ptr=%p ld=%lld)", ptr,
                  (long long)ld);
        return -1;
    }
    cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)(ld * 2)};
    cuuint32_t box[2] = {64u /* bf16 = one 128 B swizzle row */, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                    CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled failed (%d) rows=%lld cols=%lld ld=%lld", (int)r, (long long)rows,
                  (long long)cols, (long long)ld);
        return -2;
    }
    return 0;
}

// 2D byte tensor (fp8 operands) row-major [rows, cols] with row pitch ld bytes; box = [box_rows, 128 B]. gemm_skinny.cu.
int make_tmap_u8(CUtensorMap* map, const void* ptr, int64_t rows, int64_t cols, int64_t ld, int box_rows) {
    PFN_encodeTiled fn = get_encode_fn();
    if (fn == nullptr) {
        set_error("cuTensorMapEncodeTiled entry point unavailable");
        return -2;
    }
    if ((reinterpret_cast<uintptr_t>(ptr) & 15) != 0 || ld % 16 != 0) {
        set_error("TMA operand must be 16B aligned with a 16B-multiple row pitch (ptr=%p ld=%lld)", ptr, (long long)ld);
        return -1;
    }
    cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)ld};
    cuuint32_t box[2] = {128u, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                    CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled(u8) failed (%d) rows=%lld cols=%lld ld=%lld", (int)r, (long long)rows,
                  (long long)cols, (long long)ld);
        return -2;
    }
    return 0;
}

namespace {

constexpr int BM = 128;            // rows of A per CTA: two consumer warpgroups of 64 rows each
constexpr int BK = 64;             // 64 bf16 = 128 B = one swizzle row
constexpr int kNumThreads = 384;   // warpgroup 0: TMA producer (one thread), warpgroups 1..2: wgmma + epilogue
constexpr int kConsumerWarps = 8;
constexpr int A_TILE_BYTES = BM * BK * 2;

template <int BN>
struct GemmCfg {
    static constexpr int CH = BN == 192 ? 64 : (BN > 128 ? 128 : BN);  // columns per wgmma instruction (m64 x CH x 16)
    static constexpr int NCH = BN / CH;
    static constexpr int B_TILE_BYTES = BN * BK * 2;
    static constexpr int STAGE_BYTES = A_TILE_BYTES + B_TILE_BYTES;
    static constexpr int STAGES = (BN == 256) ? 4 : (BN == 192 ? 5 : (BN == 128 ? 6 : 8));  // 192-200 KB of the 227 KB a block may use
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
};

struct EpiParams {
    const __nv_bfloat16* bias;      // [N] or nullptr
    const __nv_bfloat16* residual;  // [M, ld_res] or nullptr (may alias out)
    void* out;                      // bf16 [M, ld_out] or fp32 [M, ld_out]
    int ld_out, ld_res, out_fp32;
    // ACT_ROPE_QKV
    const uint32_t* rope_tab;
    const int32_t* rope_pos0;
    __nv_bfloat16* kcache;
    __nv_bfloat16* vcache;
    int rope_S, rope_H, rope_Smax;
};

__device__ __forceinline__ float act_quick_gelu(float x) { return __fdividef(x, 1.0f + __expf(-1.702f * x)); }
__device__ __forceinline__ float act_gelu_erf(float x) {
    return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f));
}
__device__ __forceinline__ float act_silu(float x) { return __fdividef(x, 1.0f + __expf(-x)); }
// q*cos + rotate_half(q)*sin with bf16 rounding of each product and of the sum (attention.cu rope_apply: same expression)
__device__ __forceinline__ float act_rope(float x, float partner_signed, float c, float s) {
    return round_bf16(round_bf16(x * c) + round_bf16(partner_signed * s));
}

// ---- thread-block cluster helpers (the CTA-pair variant) ----
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// shared::cluster address of `local_smem_addr` (a shared::cta address of THIS CTA) in CTA `rank` of the cluster
__device__ __forceinline__ uint32_t mapa_rank(uint32_t local_smem_addr, uint32_t rank) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_smem_addr), "r"(rank));
    return r;
}
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t cluster_addr) {
    asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(cluster_addr) : "memory");
}
// TMA load whose tile lands at the same shared-memory offset in every CTA of `mask`, completing bytes on the mbarrier at the
// same offset in each of them
__device__ __forceinline__ void tma_load_2d_mcast(void* smem_dst, const void* tmap, uint64_t* bar, int32_t c0, int32_t c1, uint16_t mask) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
        " [%0], [%1, {%3, %4}], [%2], %5;"
        ::"r"(smem_u32(smem_dst)), "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(mask)
        : "memory");
}
// register budget: the producer warpgroup gives registers back, the consumers hold up to 128 accumulators per thread
__device__ __forceinline__ void reg_dealloc_producer() { asm volatile("setmaxnreg.dec.sync.aligned.u32 40;"); }
__device__ __forceinline__ void reg_alloc_consumer() { asm volatile("setmaxnreg.inc.sync.aligned.u32 232;"); }

// One warp of a consumer warpgroup hands a ring slot back to the producer(s) that fill it. wgmma.wait_group is warp-aligned,
// so the warp is converged here and every lane's view of "the MMAs that read this slot have retired" is the same.
template <int CL>
__device__ __forceinline__ void release_stage(uint64_t* bar, int lane) {
    if (lane == 0) {
        if constexpr (CL == 1) {
            mbar_arrive(bar);
        } else {
            const uint32_t a = smem_u32(bar);
#pragma unroll
            for (uint32_t r = 0; r < (uint32_t)CL; ++r) mbar_arrive_cluster(mapa_rank(a, r));
        }
    }
}

// acc = A[64 rows of this warpgroup, nkb k-blocks] · B[BN rows]^T out of the shared-memory ring
template <int BN, int CL>
__device__ __forceinline__ void mma_tile(float (&acc)[GemmCfg<BN>::NCH][GemmCfg<BN>::CH / 2], uint8_t* smem, uint64_t* full_bar,
                                         uint64_t* empty_bar, int& stage, uint32_t& phase, int nkb, int cw, int lane) {
    using Cfg = GemmCfg<BN>;
    int prev = -1;
    for (int kb = 0; kb < nkb; ++kb) {
        mbar_wait(&full_bar[stage], phase);  // TMA bytes have landed
        wgmma_fence();
        const uint32_t sa = smem_u32(smem + stage * Cfg::STAGE_BYTES) + cw * (64 * 128);
        const uint32_t sb = smem_u32(smem + stage * Cfg::STAGE_BYTES) + A_TILE_BYTES;
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) {
            // advance 16 bf16 = 32 B along K inside the 128 B swizzle atom: +2 in the descriptor's address field
            const uint64_t da = make_sw128_kmajor_desc(sa) + 2 * k;
#pragma unroll
            for (int ch = 0; ch < Cfg::NCH; ++ch)
                wgmma_bf16_ss<Cfg::CH>(acc[ch], da, make_sw128_kmajor_desc(sb + ch * (Cfg::CH * 128)) + 2 * k, (kb | k) != 0 ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<1>();  // the previous k-block's MMAs have retired: its slot is reusable
        if (prev >= 0) release_stage<CL>(&empty_bar[prev], lane);
        prev = stage;
        if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    release_stage<CL>(&empty_bar[prev], lane);
}

// bias -> activation -> residual -> store for two adjacent columns of one row
template <int ACT>
__device__ __forceinline__ void epi_store2(const EpiParams& ep, int row, int col, float x0, float x1) {
    if (ep.bias != nullptr) {
        const uint32_t b = *reinterpret_cast<const uint32_t*>(ep.bias + col);
        x0 += bf16_lo(b); x1 += bf16_hi(b);
    }
    if constexpr (ACT == ACT_QUICK_GELU) { x0 = act_quick_gelu(x0); x1 = act_quick_gelu(x1); }
    else if constexpr (ACT == ACT_GELU_ERF) { x0 = act_gelu_erf(x0); x1 = act_gelu_erf(x1); }
    if (ep.residual != nullptr) {
        const uint32_t r = *reinterpret_cast<const uint32_t*>(ep.residual + (size_t)row * ep.ld_res + col);
        x0 += bf16_lo(r); x1 += bf16_hi(r);
    }
    if (ep.out_fp32) *reinterpret_cast<float2*>(reinterpret_cast<float*>(ep.out) + (size_t)row * ep.ld_out + col) = make_float2(x0, x1);
    else *reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(ep.out) + (size_t)row * ep.ld_out + col) = pack_bf16(x0, x1);
}

// Fused epilogue straight out of the wgmma accumulator fragment (common.cuh): this thread holds rows row_lo and row_lo + 8,
// and in every group of 8 columns the two adjacent columns 2 * (lane % 4), + 1. N % 8 == 0 is enforced on the host.
template <int BN, int ACT>
__device__ __forceinline__ void epilogue_tile(const float (&acc)[GemmCfg<BN>::NCH][GemmCfg<BN>::CH / 2], const EpiParams& ep, int row_lo,
                                              int n0, int M, int N, int lane) {
    using Cfg = GemmCfg<BN>;
    const int c2 = 2 * (lane & 3);
#pragma unroll
    for (int ch = 0; ch < Cfg::NCH; ++ch) {
        const int col_base = n0 + ch * Cfg::CH;
        if constexpr (ACT == ACT_SWIGLU) {
            // W rows are block-interleaved: within each 128-col group, cols [0,64) = gate, [64,128) = up for the same 64 output
            // channels (fragment element i + 32 is column + 64 of the same row). out is [M, N/2].
            static_assert(Cfg::CH == 128, "swiglu needs 128-column chunks");
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int ocol = col_base / 2 + 8 * j + c2;
                if (ocol >= N / 2) continue;
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    const int row = row_lo + 8 * hh;
                    if (row >= M) continue;
                    const float g0 = acc[ch][4 * j + 2 * hh], g1 = acc[ch][4 * j + 2 * hh + 1];
                    const float u0 = acc[ch][32 + 4 * j + 2 * hh], u1 = acc[ch][32 + 4 * j + 2 * hh + 1];
                    *reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(ep.out) + (size_t)row * ep.ld_out + ocol) =
                        pack_bf16(act_silu(g0) * u0, act_silu(g1) * u1);
                }
            }
        } else if constexpr (ACT == ACT_ROPE_QKV) {
            // This 128-column chunk is ONE head of q, k or v (hidden % 256 == 0, head_dim 128). Element i of the head rotates
            // with element i + 64, which the same thread holds 32 fragment elements further on.
            static_assert(Cfg::CH == 128, "rope_qkv needs 128-column chunks");
            if (col_base >= N) continue;
            const int hdim = ep.rope_H * 128;
            const int part = col_base / hdim;  // 0 = q, 1 = k, 2 = v
            const int head = (col_base - part * hdim) >> 7;
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
                const int row = row_lo + 8 * hh;
                if (row >= M) continue;
                const int b = row / ep.rope_S;
                int tpos = row - b * ep.rope_S;
                if (ep.rope_pos0 != nullptr) {
                    // chunk at a cache offset: padding rows beyond the cache keep a finite q (last table row), store no k / v
                    tpos += ep.rope_pos0[b];
                    if (tpos >= ep.rope_Smax) {
                        if (part != 0) continue;
                        tpos = ep.rope_Smax - 1;
                    }
                }
                __nv_bfloat16* dst;
                if (part == 0) dst = reinterpret_cast<__nv_bfloat16*>(ep.out) + (size_t)row * ep.ld_out + col_base;
                else dst = (part == 1 ? ep.kcache : ep.vcache) + (((size_t)b * ep.rope_H + head) * ep.rope_Smax + tpos) * 128;
                const uint32_t* tab = ep.rope_tab + (size_t)tpos * 64;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int i0 = 8 * j + c2;
                    float ol[2], oh[2];
                    uint2 cs = make_uint2(0u, 0u);
                    if (part < 2) cs = __ldg(reinterpret_cast<const uint2*>(tab + i0));
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const float xl = round_bf16(acc[ch][4 * j + 2 * hh + e]);  // the projection as bf16, like the unfused path
                        const float xh = round_bf16(acc[ch][32 + 4 * j + 2 * hh + e]);
                        if (part < 2) {
                            const uint32_t w = e == 0 ? cs.x : cs.y;
                            ol[e] = act_rope(xl, -xh, bf16_lo(w), bf16_hi(w));
                            oh[e] = act_rope(xh, xl, bf16_lo(w), bf16_hi(w));
                        } else {
                            ol[e] = xl; oh[e] = xh;
                        }
                    }
                    *reinterpret_cast<uint32_t*>(dst + i0) = pack_bf16(ol[0], ol[1]);
                    *reinterpret_cast<uint32_t*>(dst + 64 + i0) = pack_bf16(oh[0], oh[1]);
                }
            }
        } else {
#pragma unroll
            for (int j = 0; j < Cfg::CH / 8; ++j) {
                const int col = col_base + 8 * j + c2;
                if (col >= N) continue;
                if (row_lo < M) epi_store2<ACT>(ep, row_lo, col, acc[ch][4 * j], acc[ch][4 * j + 1]);
                if (row_lo + 8 < M) epi_store2<ACT>(ep, row_lo + 8, col, acc[ch][4 * j + 2], acc[ch][4 * j + 3]);
            }
        }
    }
}

// CL = 1: one 128 x BN tile per CTA. CL = 2 (BN = 256): a cluster of two CTAs owns a 256 x 256 tile; each CTA computes its own
// 128 rows against the whole 256-row W tile, of which it fetches only HALF: the half is multicast by TMA into both shared
// memories, so W crosses L2 -> SM once per pair instead of once per CTA.
template <int BN, int ACT, int CL>
__global__ void __launch_bounds__(kNumThreads, 1)
gemm_bf16_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a,
                       const __grid_constant__ CUtensorMap tmap_b, int M, int N, int K,
                       EpiParams ep) {
    using Cfg = GemmCfg<BN>;
    constexpr int STAGES = Cfg::STAGES;
    static_assert(CL == 1 || BN == 256, "the CTA-pair variant uses 256 x 256 pair tiles");

    extern __shared__ uint8_t smem_raw[];
    // SWIZZLE_128B tiles need 1024-byte alignment
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                               ~static_cast<uintptr_t>(1023));
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * Cfg::STAGE_BYTES);
    uint64_t* full_bar = bars;                    // [STAGES]
    uint64_t* empty_bar = bars + STAGES;          // [STAGES]

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int wg = warp >> 2;
    const int rank = CL == 1 ? 0 : (int)cluster_ctarank();
    const int unit = blockIdx.x / CL, num_units = gridDim.x / CL;  // CTA (or CTA pair) index in the persistent schedule

    constexpr int TM = BM * CL;
    const int num_m = (M + TM - 1) / TM;
    const int num_n = (N + BN - 1) / BN;
    const int num_tiles = num_m * num_n;
    const int num_kb = (K + BK - 1) / BK;
    constexpr int GM = 8 / CL;  // m-blocks per raster group

    auto tile_coords = [&](int t, int& m_blk, int& n_blk) {
        const int tiles_per_group = GM * num_n;
        const int group = t / tiles_per_group;
        const int first_m = group * GM;
        const int gsize = min(GM, num_m - first_m);
        const int within = t - group * tiles_per_group;
        m_blk = first_m + within % gsize;
        n_blk = within / gsize;
    };

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmap_a);
        tma_prefetch_desc(&tmap_b);
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], kConsumerWarps * CL);  // every consumer warp of every CTA the slot's loads write into
        }
        fence_barrier_init();
    }
    if constexpr (CL == 1) __syncthreads();
    else cluster_sync_all();  // barriers initialised in both CTAs before anyone signals across

    pdl_trigger();
    if (wg == 0) {
        reg_dealloc_producer();
        // ===================== TMA producer (one thread) =====================
        if (warp == 0 && lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            int pre_n = 0;
            if constexpr (CL == 1) {
                // Programmatic dependent launch: the WEIGHT halves of the first ring-full of stages are requested before the
                // upstream kernel (which produces A) is known to have finished; the A halves follow after pdl_wait().
                if (unit < num_tiles) {
                    int m_blk, n_blk;
                    tile_coords(unit, m_blk, n_blk);
                    for (int kb = 0; kb < num_kb && pre_n < STAGES; ++kb, ++pre_n) {
                        uint8_t* sb = smem + pre_n * Cfg::STAGE_BYTES + A_TILE_BYTES;
                        mbar_arrive_expect_tx(&full_bar[pre_n], Cfg::STAGE_BYTES);
                        tma_load_2d(sb, &tmap_b, &full_bar[pre_n], kb * BK, n_blk * BN, kEvictNormal);
                    }
                }
            }
            pdl_wait();
            int seen = 0;
            for (int t = unit; t < num_tiles; t += num_units) {
                int m_blk, n_blk;
                tile_coords(t, m_blk, n_blk);
                for (int kb = 0; kb < num_kb; ++kb, ++seen) {
                    uint8_t* sa = smem + stage * Cfg::STAGE_BYTES;
                    uint8_t* sb = sa + A_TILE_BYTES;
                    if (seen >= pre_n) {
                        mbar_wait(&empty_bar[stage], phase ^ 1);
                        mbar_arrive_expect_tx(&full_bar[stage], Cfg::STAGE_BYTES);
                        if constexpr (CL == 1) {
                            tma_load_2d(sb, &tmap_b, &full_bar[stage], kb * BK, n_blk * BN, kEvictNormal);
                        } else {
                            // this CTA's half of the W tile, delivered to both CTAs of the pair
                            tma_load_2d_mcast(sb + rank * (BM * 128), &tmap_b, &full_bar[stage], kb * BK, n_blk * BN + rank * BM,
                                              (uint16_t)((1u << CL) - 1));
                        }
                    }
                    tma_load_2d(sa, &tmap_a, &full_bar[stage], kb * BK, m_blk * TM + rank * BM, kEvictNormal);
                    if (++stage == STAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
    } else {
        reg_alloc_consumer();
        // ===================== consumer warpgroups: wgmma main loop, then the fused epilogue from registers =====================
        pdl_wait();  // residual / out may be read or written by the upstream kernel
        const int cw = wg - 1;
        float acc[Cfg::NCH][Cfg::CH / 2];
        int stage = 0;
        uint32_t phase = 0;
        for (int t = unit; t < num_tiles; t += num_units) {
            int m_blk, n_blk;
            tile_coords(t, m_blk, n_blk);
            mma_tile<BN, CL>(acc, smem, full_bar, empty_bar, stage, phase, num_kb, cw, lane);
            const int row_lo = m_blk * TM + rank * BM + cw * 64 + 16 * (warp & 3) + (lane >> 2);
            epilogue_tile<BN, ACT>(acc, ep, row_lo, n_blk * BN, M, N, lane);
        }
    }
    if constexpr (CL > 1) {
        __syncwarp();
        cluster_sync_all();  // no CTA may exit while its partner can still signal or multicast into its shared memory
    }
}

// ---------------------------------------------------------------------------------------------
// mm_projector as ONE kernel: out = (gelu_erf(X·W1^T + b1))·W2^T + b2   (reference: nn.Sequential(Linear, GELU, Linear),
// llava/model/multimodal_projector/builder.py:39-46)
// ---------------------------------------------------------------------------------------------
// Same warp-specialised pipeline as gemm_bf16_wgmma_kernel, but the persistent tile loop walks the tiles of BOTH GEMMs in
// one dependency-ordered sequence:  P1(g0) P1(g1) P2(g0) P1(g2) P2(g1) ... P2(gLast)   (g = group of FP_GM row blocks).
// A phase-2 tile of row block m needs the whole 128 x N1 slab of the intermediate H, i.e. all N1/BN phase-1 tiles of m: their
// consumer warps publish completion with st.global -> __threadfence -> red.release(row_done[m]); the phase-2 TMA producer
// acquires the counter, crosses from the generic to the async proxy (fence.proxy.async) and only then issues its loads.
// Every dependency points backwards in the sequence and every CTA walks it in increasing order, so the spin cannot
// deadlock (grid <= #SMs, one CTA per SM: all CTAs are resident). H never needs a second launch to become visible and, for
// batches of images, is consumed one group (1024 rows = 8 MB) behind its production, out of L2.
constexpr int FP_GM = 8;

struct FusedProjParams {
    int M, N1, K1, N2;       // K2 == N1
    EpiParams ep1, ep2;      // ep1.out = H (bf16 [M, N1]); ep2.out = result
    int* row_done;           // [ceil(M/128)] completion counters, zeroed (stream-ordered) before the launch
    int target;              // value row_done[m] reaches when every consumer warp of every phase-1 tile of row block m has arrived
};

struct FpTile { int phase, m_blk, n_blk; };

__device__ __forceinline__ FpTile fp_tile(int t, int num_m, int nn1, int nn2) {
    // sequence: P1(0) | P1(1) P2(0) | P1(2) P2(1) | ... | P2(G-1)
    const int G = (num_m + FP_GM - 1) / FP_GM;
    FpTile r;
    for (int slot = 0; slot < 2 * G; ++slot) {
        int phase, g;
        if (slot == 0) { phase = 1; g = 0; }
        else if (slot == 2 * G - 1) { phase = 2; g = G - 1; }
        else { phase = (slot & 1) ? 1 : 2; g = (slot & 1) ? (slot + 1) / 2 : slot / 2 - 1; }
        const int gs = min(FP_GM, num_m - g * FP_GM);
        const int n = gs * (phase == 1 ? nn1 : nn2);
        if (t < n) {
            r.phase = phase;
            r.m_blk = g * FP_GM + t % gs;
            r.n_blk = t / gs;
            return r;
        }
        t -= n;
    }
    r.phase = 0; r.m_blk = 0; r.n_blk = 0;
    return r;
}

template <int BN>
__global__ void __launch_bounds__(kNumThreads, 1)
projector_fused_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_w1,
                       const __grid_constant__ CUtensorMap tmap_h, const __grid_constant__ CUtensorMap tmap_w2,
                       FusedProjParams P) {
    using Cfg = GemmCfg<BN>;
    constexpr int STAGES = Cfg::STAGES;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * Cfg::STAGE_BYTES);
    uint64_t* full_bar = bars;
    uint64_t* empty_bar = bars + STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;
    const int num_m = (P.M + BM - 1) / BM;
    const int nn1 = (P.N1 + BN - 1) / BN, nn2 = (P.N2 + BN - 1) / BN;
    const int total_tiles = num_m * (nn1 + nn2);
    const int nkb1 = (P.K1 + BK - 1) / BK, nkb2 = (P.N1 + BK - 1) / BK;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmap_x); tma_prefetch_desc(&tmap_w1); tma_prefetch_desc(&tmap_h); tma_prefetch_desc(&tmap_w2);
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], kConsumerWarps); }
        fence_barrier_init();
    }
    __syncthreads();

    if (wg == 0) {
        reg_dealloc_producer();
        if (warp == 0 && lane == 0) {  // ===== TMA producer =====
            pdl_wait();   // X comes from the vision tower's last kernel
            int stage = 0; uint32_t phase = 0;
            for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
                const FpTile tl = fp_tile(t, num_m, nn1, nn2);
                if (tl.phase == 2) {
                    // all phase-1 tiles of this row block have been stored and fenced by their CTAs
                    unsigned int spins = 0;
                    int seen;
                    do {
                        asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(seen) : "l"(P.row_done + tl.m_blk) : "memory");
                        if (++spins > (1u << 26)) asm volatile("trap;");
                    } while (seen - P.target < 0);
                    asm volatile("fence.proxy.async;" ::: "memory");  // generic-proxy stores of H -> async-proxy (TMA) reads
                }
                const CUtensorMap* ta = tl.phase == 1 ? &tmap_x : &tmap_h;
                const CUtensorMap* tb = tl.phase == 1 ? &tmap_w1 : &tmap_w2;
                const int nkb = tl.phase == 1 ? nkb1 : nkb2;
                for (int kb = 0; kb < nkb; ++kb) {
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    uint8_t* sa = smem + stage * Cfg::STAGE_BYTES;
                    mbar_arrive_expect_tx(&full_bar[stage], Cfg::STAGE_BYTES);
                    tma_load_2d(sa, ta, &full_bar[stage], kb * BK, tl.m_blk * BM, kEvictNormal);
                    tma_load_2d(sa + A_TILE_BYTES, tb, &full_bar[stage], kb * BK, tl.n_blk * BN, kEvictNormal);
                    if (++stage == STAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
    } else {
        reg_alloc_consumer();
        // ===== consumer warpgroups: bias (+ erf-GELU in phase 1), bf16 stores; phase 1 publishes the row block =====
        pdl_wait();
        const int cw = wg - 1;
        float acc[Cfg::NCH][Cfg::CH / 2];
        int stage = 0; uint32_t phase = 0;
        for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
            const FpTile tl = fp_tile(t, num_m, nn1, nn2);
            mma_tile<BN, 1>(acc, smem, full_bar, empty_bar, stage, phase, tl.phase == 1 ? nkb1 : nkb2, cw, lane);
            const int row_lo = tl.m_blk * BM + cw * 64 + 16 * (warp & 3) + (lane >> 2);
            if (tl.phase == 1) {
                epilogue_tile<BN, ACT_GELU_ERF>(acc, P.ep1, row_lo, tl.n_blk * BN, P.M, P.N1, lane);
                __threadfence();  // this lane's H stores are visible device-wide before the warp's arrival below
                asm volatile("fence.proxy.async;" ::: "memory");
                __syncwarp();
                if (lane == 0) asm volatile("red.release.gpu.global.add.s32 [%0], 1;" ::"l"(P.row_done + tl.m_blk) : "memory");
            } else {
                epilogue_tile<BN, ACT_NONE>(acc, P.ep2, row_lo, tl.n_blk * BN, P.M, P.N2, lane);
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
// programmatic dependent launch, plus a cluster dimension for the CTA-pair variant
template <typename... KArgs, typename... Args>
cudaError_t launch_cluster_pdl(void (*kernel)(KArgs...), int grid, int cluster, size_t smem, cudaStream_t stream, Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid); cfg.blockDim = dim3(kNumThreads); cfg.dynamicSmemBytes = smem; cfg.stream = stream;
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    attr[1].id = cudaLaunchAttributeClusterDimension;
    attr[1].val.clusterDim.x = cluster; attr[1].val.clusterDim.y = 1; attr[1].val.clusterDim.z = 1;
    cfg.attrs = attr; cfg.numAttrs = cluster > 1 ? 2 : 1;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

template <int BN, int ACT, int CL>
int launch_gemm(const CUtensorMap& ta, const CUtensorMap& tb, int M, int N, int K, const EpiParams& ep,
                cudaStream_t stream) {
    using Cfg = GemmCfg<BN>;
    static bool attr_set = false;
    auto kern = gemm_bf16_wgmma_kernel<BN, ACT, CL>;
    if (!attr_set) {
        B2_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
        attr_set = true;
    }
    const int num_tiles = ((M + BM * CL - 1) / (BM * CL)) * ((N + BN - 1) / BN);
    const int slots = num_sms() / CL;
    const int units = num_tiles < slots ? num_tiles : slots;
    B2_CUDA_CHECK(launch_cluster_pdl(kern, units * CL, CL, (size_t)Cfg::SMEM_BYTES, stream, ta, tb, M, N, K, ep));
    B2_LAUNCH_CHECK();
    return 0;
}

template <int BN>
int dispatch_act(int act, const CUtensorMap& ta, const CUtensorMap& tb, int M, int N, int K,
                 const EpiParams& ep, cudaStream_t stream) {
    switch (act) {
        case ACT_NONE: return launch_gemm<BN, ACT_NONE, 1>(ta, tb, M, N, K, ep, stream);
        case ACT_QUICK_GELU: return launch_gemm<BN, ACT_QUICK_GELU, 1>(ta, tb, M, N, K, ep, stream);
        case ACT_GELU_ERF: return launch_gemm<BN, ACT_GELU_ERF, 1>(ta, tb, M, N, K, ep, stream);
        default: break;
    }
    set_error("gemm: unsupported activation %d", act);
    return -1;
}

template <int BN>
int launch_fused_projector(const CUtensorMap& tx, const CUtensorMap& tw1, const CUtensorMap& th, const CUtensorMap& tw2,
                           const FusedProjParams& P, cudaStream_t stream) {
    using Cfg = GemmCfg<BN>;
    static bool attr_set = false;
    auto kern = projector_fused_kernel<BN>;
    if (!attr_set) {
        B2_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
        attr_set = true;
    }
    const int num_m = (P.M + BM - 1) / BM;
    const int tiles = num_m * ((P.N1 + BN - 1) / BN + (P.N2 + BN - 1) / BN);
    const int grid = tiles < num_sms() ? tiles : num_sms();  // <= #SMs, 1 CTA/SM: every CTA is resident (the spin needs it)
    B2_CUDA_CHECK(launch_cluster_pdl(kern, grid, 1, (size_t)Cfg::SMEM_BYTES, stream, tx, tw1, th, tw2, P));
    B2_LAUNCH_CHECK();
    return 0;
}

EpiParams make_epi(const GemmArgs& g) {
    EpiParams ep;
    ep.bias = reinterpret_cast<const __nv_bfloat16*>(g.bias);
    ep.residual = reinterpret_cast<const __nv_bfloat16*>(g.residual);
    ep.out = g.out; ep.ld_out = g.ld_out; ep.ld_res = g.ld_res; ep.out_fp32 = g.out_fp32;
    ep.rope_tab = reinterpret_cast<const uint32_t*>(g.rope.table);
    ep.kcache = reinterpret_cast<__nv_bfloat16*>(g.rope.kcache); ep.vcache = reinterpret_cast<__nv_bfloat16*>(g.rope.vcache);
    ep.rope_S = g.rope.S; ep.rope_H = g.rope.H; ep.rope_Smax = g.rope.Smax;
    ep.rope_pos0 = g.rope.pos0;
    return ep;
}

}  // namespace

// out[M,N2] = (gelu_erf(X[M,K1]·W1[N1,K1]^T + b1))·W2[N2,N1]^T + b2 in one launch; H [M,N1] bf16 is the caller's scratch,
// row_done the caller's int[ceil(M/128)] scratch (zeroed here, on the stream).
int projector_fused_bf16(const void* X, int ldx, const void* W1, const void* b1, const void* W2, const void* b2, void* H,
                         void* out, int ld_out, int M, int K1, int N1, int N2, int* row_done, cudaStream_t stream) {
    B2_CHECK_ARG(M > 0 && K1 % 8 == 0 && N1 % 8 == 0 && N2 % 8 == 0 && b1 && b2 && row_done,
                 "projector_fused: bad problem M=%d K1=%d N1=%d N2=%d", M, K1, N1, N2);
    const int num_m = (M + BM - 1) / BM;
    // tile width: 192-wide tiles while each GEMM of the pair still fits one wave (a single image: 5 row blocks x 22 = 110
    // tiles on 132 SMs), 256 otherwise
    const int bn = (num_m * ((N1 + 191) / 192) <= num_sms()) ? 192 : 256;
    CUtensorMap tx, tw1, th, tw2;
    B2_TRY(make_tmap_bf16(&tx, X, M, K1, ldx, BM));
    B2_TRY(make_tmap_bf16(&tw1, W1, N1, K1, K1, bn));
    B2_TRY(make_tmap_bf16(&th, H, M, N1, N1, BM));
    B2_TRY(make_tmap_bf16(&tw2, W2, N2, N1, N1, bn));
    FusedProjParams P;
    P.M = M; P.N1 = N1; P.K1 = K1; P.N2 = N2;
    GemmArgs g1, g2;
    g1.bias = b1; g1.out = H; g1.ld_out = N1;
    g2.bias = b2; g2.out = out; g2.ld_out = ld_out;
    P.ep1 = make_epi(g1);
    P.ep2 = make_epi(g2);
    P.row_done = row_done;
    P.target = ((N1 + bn - 1) / bn) * kConsumerWarps;
    B2_CUDA_CHECK(cudaMemsetAsync(row_done, 0, (size_t)num_m * sizeof(int), stream));
    if (bn == 192) return launch_fused_projector<192>(tx, tw1, th, tw2, P, stream);
    return launch_fused_projector<256>(tx, tw1, th, tw2, P, stream);
}

// CTA-pair variant (clusters of two, 256 x 256 pair tiles, W multicast). Same contract as gemm_bf16 (kernels.h).
int gemm_bf16_2cta(const GemmArgs& g, cudaStream_t stream) {
    B2_CHECK_ARG(g.M > 0 && g.N > 0 && g.K > 0, "gemm_2cta: empty problem M=%d N=%d K=%d", g.M, g.N, g.K);
    B2_CHECK_ARG(g.K % 8 == 0 && g.N % 8 == 0, "gemm_2cta: K and N must be multiples of 8 (K=%d N=%d)", g.K, g.N);
    B2_CHECK_ARG(g.act != ACT_SWIGLU || (g.N % 128 == 0 && !g.out_fp32 && g.bias == nullptr && g.residual == nullptr),
                 "gemm_2cta: swiglu needs N %% 128 == 0, no bias/residual, bf16 output");
    B2_CHECK_ARG((reinterpret_cast<uintptr_t>(g.out) & 15) == 0 && (g.ld_out % 8) == 0, "gemm_2cta: out alignment");
    B2_CHECK_ARG(g.residual == nullptr || ((reinterpret_cast<uintptr_t>(g.residual) & 15) == 0 && (g.ld_res % 8) == 0),
                 "gemm_2cta: residual alignment");
    CUtensorMap ta, tb;
    B2_TRY(make_tmap_bf16(&ta, g.A, g.M, g.K, g.lda, BM));
    B2_TRY(make_tmap_bf16(&tb, g.W, g.N, g.K, g.ldw, BM));  // each CTA of a pair fetches 128 of the tile's 256 W rows
    const EpiParams ep = make_epi(g);
    if (g.act == ACT_ROPE_QKV) {
        B2_CHECK_ARG(g.rope.table && g.rope.kcache && g.rope.vcache && g.rope.S > 0 && g.rope.H > 0 &&
                         (g.rope.pos0 != nullptr || g.rope.Smax >= g.rope.S),
                     "gemm_2cta(rope_qkv): rope arguments missing");
        B2_CHECK_ARG(g.N == 3 * g.rope.H * 128 && (g.rope.H * 128) % 256 == 0 && g.M % g.rope.S == 0 && !g.out_fp32 &&
                         g.bias == nullptr && g.residual == nullptr,
                     "gemm_2cta(rope_qkv): needs N = 3*H*128 with H*128 %% 256 == 0, M = B*S, bf16 output, no bias/residual");
    }
    switch (g.act) {
        case ACT_NONE: return launch_gemm<256, ACT_NONE, 2>(ta, tb, g.M, g.N, g.K, ep, stream);
        case ACT_QUICK_GELU: return launch_gemm<256, ACT_QUICK_GELU, 2>(ta, tb, g.M, g.N, g.K, ep, stream);
        case ACT_GELU_ERF: return launch_gemm<256, ACT_GELU_ERF, 2>(ta, tb, g.M, g.N, g.K, ep, stream);
        case ACT_SWIGLU: return launch_gemm<256, ACT_SWIGLU, 2>(ta, tb, g.M, g.N, g.K, ep, stream);
        case ACT_ROPE_QKV: return launch_gemm<256, ACT_ROPE_QKV, 2>(ta, tb, g.M, g.N, g.K, ep, stream);
        default: break;
    }
    set_error("gemm_2cta: unsupported activation %d", g.act);
    return -1;
}

// C[M, N(/2 for swiglu)] = epi(A[M,K](lda) · W[N,K](ldw)^T). See kernels.h for the contract.
int gemm_bf16(const GemmArgs& g, cudaStream_t stream) {
    B2_CHECK_ARG(g.M > 0 && g.N > 0 && g.K > 0, "gemm: empty problem M=%d N=%d K=%d", g.M, g.N, g.K);
    B2_CHECK_ARG(g.K % 8 == 0 && g.N % 8 == 0, "gemm: K and N must be multiples of 8 (K=%d N=%d)", g.K, g.N);
    B2_CHECK_ARG(g.act != ACT_SWIGLU || g.N % 128 == 0, "gemm: swiglu needs N %% 128 == 0 (N=%d)", g.N);
    B2_CHECK_ARG(g.act != ACT_SWIGLU || (!g.out_fp32 && g.bias == nullptr && g.residual == nullptr),
                 "gemm: swiglu epilogue takes no bias/residual and writes bf16");
    B2_CHECK_ARG((reinterpret_cast<uintptr_t>(g.out) & 15) == 0 && (g.ld_out % 8) == 0,
                 "gemm: out must be 16B aligned with ld_out %% 8 == 0");
    B2_CHECK_ARG(g.residual == nullptr ||
                     ((reinterpret_cast<uintptr_t>(g.residual) & 15) == 0 && (g.ld_res % 8) == 0),
                 "gemm: residual must be 16B aligned with ld_res %% 8 == 0");

    if (g.bn_override == 2) return gemm_bf16_2cta(g, stream);  // CTA-pair kernel

    // Tile-N choice: the launch takes ceil(tiles / #SMs) waves and a tile costs ~BN plus a fixed part (pipeline fill, epilogue),
    // so the widest tile wins unless a narrower one saves a wave. BN=64 re-reads A most often per unit of work and is
    // charged for it. BN=192 exists for the N=4096 projections of a B=1 prefill (M=704): 96 tiles of 256 leave a quarter of
    // the 132 SMs idle, 132 tiles of 192 fill exactly one wave. The CTA-pair kernel competes as a fifth shape: per SM a pair
    // tile is the work of a 128x256 tile with half the L2 -> SM traffic for W, so it is preferred wherever it needs no more
    // waves of SM pairs than the 1-CTA kernel needs of SMs.
    const int num_m = (g.M + BM - 1) / BM;
    int bn = 64;
    {
        const int cand[4] = {256, 192, 128, 64};
        const float rel[4] = {1.00f, 1.00f, 1.00f, 0.80f};
        float best = 0.f;
        for (int i = 0; i < 4; ++i) {
            if (g.act == ACT_SWIGLU && cand[i] % 128 != 0) continue;
            const long long tiles = (long long)num_m * ((g.N + cand[i] - 1) / cand[i]);
            const long long waves = (tiles + num_sms() - 1) / num_sms();
            const float cost = (float)waves * ((float)cand[i] / rel[i] + 24.f /*per-tile fixed cost*/);
            if (best == 0.f || cost < best) { best = cost; bn = cand[i]; }
        }
        if (g.bn_override == 0 && g.M >= 512 && g.N >= 256) {
            const long long pairs = (long long)((g.M + 255) / 256) * ((g.N + 255) / 256);
            const long long pair_slots = num_sms() / 2;
            const long long waves = (pairs + pair_slots - 1) / pair_slots;
            const float cost = (float)waves * (256.f + 24.f);
            if (cost <= best) return gemm_bf16_2cta(g, stream);
        }
    }
    if (g.bn_override == 64 || g.bn_override == 128 || g.bn_override == 192 || g.bn_override == 256) bn = g.bn_override;
    if (g.act == ACT_SWIGLU && bn % 128 != 0) bn = 128;

    CUtensorMap ta, tb;
    B2_TRY(make_tmap_bf16(&ta, g.A, g.M, g.K, g.lda, BM));
    B2_TRY(make_tmap_bf16(&tb, g.W, g.N, g.K, g.ldw, bn));
    const EpiParams ep = make_epi(g);

    if (g.act == ACT_SWIGLU) {
        if (bn == 256) return launch_gemm<256, ACT_SWIGLU, 1>(ta, tb, g.M, g.N, g.K, ep, stream);
        return launch_gemm<128, ACT_SWIGLU, 1>(ta, tb, g.M, g.N, g.K, ep, stream);
    }
    if (bn == 64) return dispatch_act<64>(g.act, ta, tb, g.M, g.N, g.K, ep, stream);
    if (bn == 192) return dispatch_act<192>(g.act, ta, tb, g.M, g.N, g.K, ep, stream);
    if (bn == 256) return dispatch_act<256>(g.act, ta, tb, g.M, g.N, g.K, ep, stream);
    return dispatch_act<128>(g.act, ta, tb, g.M, g.N, g.K, ep, stream);
}

}  // namespace b2
