// Weight-streaming "skinny" GEMM for decode at batch 9..128 on sm_90a (swap-AB + stream-K):
//
//     out[b, n] = sum_k x[b, k] * W[n, k]   (+ residual[b, n])          b < B <= 128,  n < N
//     out[b, c] = silu(gate_c . x_b) * (up_c . x_b)                     (ACT_SWIGLU, W rows block-64 interleaved)
//
// A decode step at these batch sizes is still a pure weight stream (every weight byte is used by <= 128 tokens),
// so the kernel is organised around HBM, not around the tensor pipe:
//   * swap-AB: the WEIGHT tile is the M operand of wgmma (two m64 x BN x k16 blocks, fp32 accumulators in registers),
//     the activations are the narrow N operand (BN = 32/64/128 >= B, rows >= B zero-filled by TMA) — no M padding
//     of the batch to 128 and no wasted weight re-reads.
//   * stream-K: the (weight tile, k-block) space is cut into gridDim.x contiguous ranges that differ by at most one
//     16 KB k-block, so every SM streams the same number of weight bytes whatever N and K are (N = 4096 gives only
//     32 tiles for 132 SMs). A tile that is shared by several CTAs is reduced through an fp32 workspace by the LAST
//     CTA to arrive, in fixed slot order (deterministic), which then runs the fused epilogue.
//   * warp-specialised: 1 TMA producer thread (deep smem ring), one consumer warpgroup that issues the wgmma and then
//     runs the epilogue: the fragment goes through shared memory once, transposed, so that lane = weight row and the
//     stores are coalesced (consecutive lanes = consecutive n).
//   * FP8 variant (template flag): e4m3 weights (per-output-channel fp32 scale) x e4m3 activations (per-token fp32 scale),
//     wgmma e4m3 (K = 32 per instruction, 128 elements per 128-byte swizzle row), dequantisation
//     acc * w_scale[n] * x_scale[b] in the epilogue — BASELINE configs[4] ("fp8-weight path"): halves the weight
//     stream. Same pipeline, same stream-K reduction.
// Replaces, for B > 8, the HF one-token Linear calls (transformers modeling_llama.py:251-289 q/k/v/o_proj, :182-184
// LlamaMLP, :486-487 lm_head) behind the reference's decode branch (llava/model/llava_arch.py:103-112).
#include <cuda.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>

#include <string>
#include <vector>

#include "common.cuh"
#include "kernels.h"

namespace b2 {

int make_tmap_bf16(CUtensorMap* map, const void* ptr, int64_t rows, int64_t cols, int64_t ld, int box_rows);
int make_tmap_u8(CUtensorMap* map, const void* ptr, int64_t rows, int64_t cols, int64_t ld, int box_rows);

namespace {

constexpr int SK_BM = 128;          // weight rows per tile (two m64 wgmma blocks)
constexpr int SK_BK = 64;           // bf16: 64 elements = one 128 B swizzle row (fp8: 128 elements, same bytes)
constexpr int SK_THREADS = 160;     // warps 0..3: consumer warpgroup (wgmma + epilogue), warp 4: TMA producer
constexpr int SK_ACC_LD = 132;      // row pitch (floats) of the accumulator staging tile: conflict-free fragment writes and row reads
constexpr int SK_W_TILE = SK_BM * SK_BK * 2;

template <int BN>
struct SkCfg {
    static constexpr int X_TILE = BN * SK_BK * 2;
    static constexpr int STAGE = SK_W_TILE + X_TILE;
    // Ring depth: what fits beside the fp32 staging tile (ACC_BYTES). With it the CTA asks for 186 KB (BN = 32) to 204 KB
    // (BN = 128) of the 227 KB a block may use, so two of these CTAs never share an SM and the weight prefetch of the next
    // launch (programmatic dependent launch) starts only as CTAs of this one exit. Neither the depths nor that overlap have
    // been measured on the H100.
    static constexpr int STAGES = BN == 32 ? 8 : (BN == 64 ? 6 : 4);
    static constexpr int ACC_BYTES = BN * SK_ACC_LD * 4;  // the tile's fp32 accumulator, out of the wgmma fragment
    static constexpr int UP_BYTES = 64 * 33 * 4;  // SwiGLU staging of the tile's up rows, one 32-column chunk
    static constexpr int SMEM = STAGES * STAGE + ACC_BYTES + UP_BYTES + 1024 /*align*/ + 256 /*barriers*/;
};

struct SkEpi {
    const __nv_bfloat16* residual;  // [B, ld_res] or nullptr (may alias out)
    void* out;                      // bf16 / fp32 [B, ld_out]
    float* partial;                 // stream-K workspace: [tile][maxseg][BN][128] fp32
    int* counters;                  // [tiles], zero-initialised, self-resetting
    int ld_out, ld_res, out_fp32, maxseg;
    const float* w_scale;           // fp8 only: [N] per weight row (physical row order of W)
    const float* x_scale;           // fp8 only: [B] per token
    int stages;                     // ring depth: SkCfg<BN>::STAGES (set by sk_launch)
    unsigned long long* trace;      // debug (B2_SKINNY_TRACE=<file>): 16 slots (8 %globaltimer stamps + tiles finalised) per CTA of this launch, else nullptr
};

__device__ __forceinline__ unsigned long long sk_now() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
#define SK_STAMP(slot) do { if (ep.trace != nullptr) ep.trace[(size_t)blockIdx.x * 16 + (slot)] = sk_now(); } while (0)

// 1-D bulk copy global -> shared, completion (bytes) on an mbarrier
__device__ __forceinline__ void sk_bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
                 "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

__device__ __forceinline__ void epi_sync() { asm volatile("bar.sync 2, 128;" ::: "memory"); }

// CTA that owns global k-block unit u when `total` units are cut into `grid` ranges [total*c/grid, total*(c+1)/grid)
__device__ __forceinline__ int sk_cta_of(long long u, long long total, int grid) {
    int c = (int)((u * grid) / total);
    while (c + 1 < grid && (total * (c + 1)) / grid <= u) ++c;
    while (c > 0 && (total * c) / grid > u) --c;
    return c;
}

template <int BN, int ACT, bool FP8>
__global__ void __launch_bounds__(SK_THREADS, 1)
gemm_skinny_kernel(const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_x, int N, int K,
                   int B, SkEpi ep) {
    using Cfg = SkCfg<BN>;
    const int STAGES = ep.stages;
    extern __shared__ uint8_t sk_smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(sk_smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
    float* s_acc = reinterpret_cast<float*>(smem + STAGES * Cfg::STAGE);  // [BN][SK_ACC_LD]: the tile's accumulator, batch-major
    float* s_up = reinterpret_cast<float*>(smem + STAGES * Cfg::STAGE + Cfg::ACC_BYTES);
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * Cfg::STAGE + Cfg::ACC_BYTES + Cfg::UP_BYTES);
    uint64_t* full_bar = bars;
    uint64_t* empty_bar = bars + STAGES;
    uint64_t* fix_bar = bars + 2 * STAGES;  // fix-up staging: the tile's partials, bulk-copied into the drained ring
    int* s_flag = reinterpret_cast<int*>(bars + 2 * STAGES + 1);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int num_m = (N + SK_BM - 1) / SK_BM;
    constexpr int BKE = FP8 ? 2 * SK_BK : SK_BK;  // elements per 128-byte k-block
    const int nkb = (K + BKE - 1) / BKE;
    const long long total = (long long)num_m * nkb;
    const int grid = gridDim.x;
    const long long u0 = (total * blockIdx.x) / grid;
    const long long u1 = (total * (blockIdx.x + 1)) / grid;
    const int t_first = (int)(u0 / nkb), t_last = (int)((u1 - 1) / nkb);  // u1 > u0: the host keeps grid <= total

    if (threadIdx.x == 0) {
        SK_STAMP(0);  // entry
        tma_prefetch_desc(&tmap_w);
        tma_prefetch_desc(&tmap_x);
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 4); }
        mbar_init(fix_bar, 1);
        fence_barrier_init();
    }
    __syncthreads();

    if (threadIdx.x == 0) SK_STAMP(1);  // set-up done (barriers)
    pdl_trigger();  // the next kernel of the step may start its own weight prefetch as soon as it finds room on an SM
    if (warp == 4) {
        if (lane == 0) {  // ===== TMA producer: weights are read exactly once -> evict-first; activations stay in L2 =====
            // Programmatic dependent launch: this CTA may be running while the kernel that PRODUCES x is still finishing.
            // Weights depend on nothing, so the first ring-full of W tiles is requested right away; the activation half of
            // those stages follows once the upstream grid has completed (pdl_wait), everything after that runs as usual.
            int stage = 0; uint32_t phase = 0;
            int pre_n = 0;                      // stages whose W half is already in flight
            {
                int t = t_first;
                int kb = (int)(u0 - (long long)t * nkb);
                long long u = u0;
                while (u < u1 && pre_n < STAGES) {
                    uint8_t* sw = smem + pre_n * Cfg::STAGE;
                    mbar_arrive_expect_tx(&full_bar[pre_n], Cfg::STAGE);
                    tma_load_2d(sw, &tmap_w, &full_bar[pre_n], kb * BKE, t * SK_BM, kEvictFirst);
                    ++pre_n; ++u;
                    if (++kb == nkb) { kb = 0; ++t; }
                }
            }
            pdl_wait();
            SK_STAMP(2);  // upstream grid complete
            int seen = 0;
            for (int t = t_first; t <= t_last; ++t) {
                const int kb0 = (int)(max(u0, (long long)t * nkb) - (long long)t * nkb);
                const int kb1 = (int)(min(u1, (long long)(t + 1) * nkb) - (long long)t * nkb);
                for (int kb = kb0; kb < kb1; ++kb, ++seen) {
                    uint8_t* sw = smem + stage * Cfg::STAGE;
                    if (seen >= pre_n) {
                        mbar_wait(&empty_bar[stage], phase ^ 1);
                        mbar_arrive_expect_tx(&full_bar[stage], Cfg::STAGE);
                        tma_load_2d(sw, &tmap_w, &full_bar[stage], kb * BKE, t * SK_BM, kEvictFirst);
                    }
                    tma_load_2d(sw + SK_W_TILE, &tmap_x, &full_bar[stage], kb * BKE, 0, kEvictLast);
                    if (++stage == STAGES) { stage = 0; phase ^= 1; }
                }
            }
            SK_STAMP(3);  // last load issued
        }
    } else {
        // ===== consumer warpgroup (warps 0..3): wgmma main loop, then the tile's epilogue with thread = weight row =====
        pdl_wait();                           // residual / out / the stream-K workspace are shared with upstream kernels
        const int q = warp;                   // 32-row quarter of the tile this warp's epilogue threads own
        const int row_in_tile = q * 32 + lane;
        const int et = threadIdx.x;           // 0..127
        int n_final = 0;
        int stage = 0; uint32_t phase = 0;
        for (int t = t_first; t <= t_last; ++t) {
            const int kb0 = (int)(max(u0, (long long)t * nkb) - (long long)t * nkb);
            const int kb1 = (int)(min(u1, (long long)(t + 1) * nkb) - (long long)t * nkb);
            {
                float facc[2][BN / 2];  // two m64 blocks: weight rows [0,64) and [64,128) of the tile
                int prev = -1;
                if constexpr (FP8) {
#pragma unroll
                    for (int mb = 0; mb < 2; ++mb)
#pragma unroll
                        for (int i = 0; i < BN / 2; ++i) facc[mb][i] = 0.f;
                }
                for (int kb = kb0; kb < kb1; ++kb) {
                    mbar_wait(&full_bar[stage], phase);
                    const uint32_t sw = smem_u32(smem + stage * Cfg::STAGE);
                    if constexpr (FP8) {
                        // The e4m3 wgmma keeps fewer mantissa bits than fp32 while it accumulates, so a sum over K = 4096..13824
                        // drifts. Each k-block (128 elements) is therefore summed by the tensor core into a fresh fragment and
                        // added to the running fp32 accumulator by the CUDA cores. The kernel is HBM-bound: the serialisation
                        // of MMA and add is hidden behind the weight stream.
#pragma unroll
                        for (int mb = 0; mb < 2; ++mb) {
                            float part[BN / 2];
                            wgmma_fence();
#pragma unroll
                            for (int k = 0; k < 4; ++k)  // 32 bytes of K per instruction: 32 e4m3
                                wgmma_e4m3_ss<BN>(part, make_sw128_kmajor_desc(sw + mb * (64 * 128)) + 2 * k,
                                                  make_sw128_kmajor_desc(sw + SK_W_TILE) + 2 * k, k > 0 ? 1u : 0u);
                            wgmma_commit();
                            wgmma_wait<0>();
#pragma unroll
                            for (int i = 0; i < BN / 2; ++i) facc[mb][i] += part[i];
                        }
                        if (lane == 0) mbar_arrive(&empty_bar[stage]);
                    } else {
                        wgmma_fence();
#pragma unroll
                        for (int k = 0; k < 4; ++k) {  // 32 bytes of K per instruction: 16 bf16
                            const uint64_t db = make_sw128_kmajor_desc(sw + SK_W_TILE) + 2 * k;
                            const uint32_t accum = (kb > kb0 || k > 0) ? 1u : 0u;
#pragma unroll
                            for (int mb = 0; mb < 2; ++mb)
                                wgmma_bf16_ss<BN>(facc[mb], make_sw128_kmajor_desc(sw + mb * (64 * 128)) + 2 * k, db, accum);
                        }
                        wgmma_commit();
                        wgmma_wait<1>();  // the previous k-block's MMAs have retired: hand its slot back
                        if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
                        prev = stage;
                    }
                    if (++stage == STAGES) { stage = 0; phase ^= 1; }
                }
                if constexpr (!FP8) {
                    wgmma_wait<0>();
                    if (lane == 0) mbar_arrive(&empty_bar[prev]);
                }
                if (et == 0 && t == t_last) SK_STAMP(4);  // last MMA retired
                // fragment -> shared memory, transposed: afterwards thread r reads weight row r for every batch column
#pragma unroll
                for (int mb = 0; mb < 2; ++mb)
#pragma unroll
                    for (int i = 0; i < BN / 2; ++i)
                        s_acc[frag_col(et, i) * SK_ACC_LD + 64 * mb + frag_row(et, i)] = facc[mb][i];
            }
            epi_sync();
            if (et == 0 && t == t_last) SK_STAMP(5);  // accumulator of the last tile complete
            const float* acc_row = s_acc + row_in_tile;
            const int first = sk_cta_of((long long)t * nkb, total, grid);
            const int last = sk_cta_of((long long)(t + 1) * nkb - 1, total, grid);
            const int nseg = last - first + 1;
            const int seg = (int)blockIdx.x - first;
            float* slot0 = ep.partial + (size_t)t * ep.maxseg * (BN * SK_BM);
            bool finalize = true, staged = false;
            if (nseg > 1) {
                float* mine = slot0 + (size_t)seg * (BN * SK_BM);
#pragma unroll 1
                for (int c = 0; c < BN / 32; ++c) {
#pragma unroll
                    for (int j = 0; j < 32; ++j) mine[(size_t)(c * 32 + j) * SK_BM + row_in_tile] = acc_row[(c * 32 + j) * SK_ACC_LD];
                }
                __threadfence();
                epi_sync();
                if (et == 0) *s_flag = (atomicAdd(&ep.counters[t], 1) == nseg - 1) ? 1 : 0;
                epi_sync();
                finalize = *s_flag != 0;
                if (finalize) __threadfence();
                // Fix-up through shared memory: when the tile being finalised is this CTA's LAST one, the ring is drained (every
                // load consumed, every MMA complete), so the nseg partials are fetched with ONE round of 1-D bulk copies into it
                // instead of nseg x 32 L2 loads per thread in dependent rounds.
                staged = finalize && t == t_last && (size_t)nseg * (BN * SK_BM * 4) <= (size_t)STAGES * Cfg::STAGE;
                if (staged && et == 0) {
                    asm volatile("fence.proxy.async;" ::: "memory");  // other CTAs' generic-proxy stores -> async-proxy reads
                    mbar_arrive_expect_tx(fix_bar, (uint32_t)nseg * (BN * SK_BM * 4));
                    for (int sidx = 0; sidx < nseg; ++sidx)
                        sk_bulk_g2s(smem + (size_t)sidx * (BN * SK_BM * 4), slot0 + (size_t)sidx * (BN * SK_BM), BN * SK_BM * 4, fix_bar);
                }
                if (et == 0 && t == t_last) SK_STAMP(6);  // partial published / finaliser elected
                if (et == 0 && finalize) ++n_final;
            }
#pragma unroll 1
            for (int c = 0; c < BN / 32; ++c) {
                if (!finalize) break;  // CTA-uniform: the last CTA to arrive owns the tile's epilogue
                float acc[32];
                float resv[32];  // residual values of this chunk, requested before the accumulator / partial loads are waited for
                if constexpr (ACT != ACT_SWIGLU) {
                    const int n = t * SK_BM + row_in_tile;
#pragma unroll
                    for (int j = 0; j < 32; ++j) {
                        const int b = c * 32 + j;
                        resv[j] = (ep.residual != nullptr && n < N && b < B) ? __bfloat162float(ep.residual[(size_t)b * ep.ld_res + n]) : 0.f;
                    }
                }
                if (nseg == 1) {
#pragma unroll
                    for (int j = 0; j < 32; ++j) acc[j] = acc_row[(c * 32 + j) * SK_ACC_LD];
                } else if (staged) {
                    if (c == 0) mbar_wait(fix_bar, 0);  // at most one staged fix-up per CTA (its last tile): phase 0
                    if (c == 0 && et == 0) SK_STAMP(9);  // partials landed in shared memory
                    const float* sp = reinterpret_cast<const float*>(smem) + (size_t)(c * 32) * SK_BM + row_in_tile;
#pragma unroll
                    for (int j = 0; j < 32; ++j) acc[j] = 0.f;
                    for (int sidx = 0; sidx < nseg; ++sidx) {  // segment order, as in the register path: bit-identical sums
#pragma unroll
                        for (int j = 0; j < 32; ++j) acc[j] += sp[(size_t)sidx * (BN * SK_BM) + (size_t)j * SK_BM];
                    }
                } else if (finalize) {
                    // Fix-up. The partials are summed in segment order (deterministic whatever CTA arrives last), but all of a
                    // half chunk's loads — up to 6 segments x 8 columns — are issued before the first add: otherwise the finaliser of an N = 4096 GEMM waits for six
                    // dependent L2 round trips in a row. Absent segments contribute +0.0f, which leaves the sum bit-identical.
#pragma unroll
                    for (int j = 0; j < 32; ++j) acc[j] = 0.f;
                    constexpr int SEG_U = 6, HC = 8;
                    for (int s0 = 0; s0 < nseg; s0 += SEG_U) {
#pragma unroll
                        for (int hh = 0; hh < 32 / HC; ++hh) {
                            float pv[SEG_U][HC];
#pragma unroll
                            for (int u = 0; u < SEG_U; ++u) {
                                const bool on = s0 + u < nseg;
                                const float* ps = slot0 + (size_t)(on ? s0 + u : s0) * (BN * SK_BM) + (size_t)(c * 32 + hh * HC) * SK_BM +
                                                  row_in_tile;
#pragma unroll
                                for (int j = 0; j < HC; ++j) pv[u][j] = on ? __ldcg(ps + (size_t)j * SK_BM) : 0.f;
                            }
#pragma unroll
                            for (int u = 0; u < SEG_U; ++u)
#pragma unroll
                                for (int j = 0; j < HC; ++j) acc[hh * HC + j] += pv[u][j];
                        }
                    }
                }
                if constexpr (FP8) {  // dequantise: per weight row (this thread's row) x per token (column)
                    const int nrow = t * SK_BM + row_in_tile;
                    const float ws = (finalize && nrow < N) ? __ldg(ep.w_scale + nrow) : 0.f;
#pragma unroll
                    for (int j = 0; j < 32; ++j) {
                        const int b = c * 32 + j;
                        acc[j] *= ws * (b < B ? __ldg(ep.x_scale + b) : 0.f);
                    }
                }
                if constexpr (ACT == ACT_SWIGLU) {
                    // tile rows [0,64) = gate, [64,128) = up of channels t*64 + (0..63): up rows go through smem
                    if (finalize && q >= 2) {
#pragma unroll
                        for (int j = 0; j < 32; ++j) s_up[((q - 2) * 32 + lane) * 33 + j] = acc[j];
                    }
                    epi_sync();
                    if (finalize && q < 2) {
                        const int ch = t * 64 + q * 32 + lane;
                        if (ch < N / 2) {
#pragma unroll
                            for (int j = 0; j < 32; ++j) {
                                const int b = c * 32 + j;
                                if (b < B) {
                                    const float g = acc[j], u = s_up[(q * 32 + lane) * 33 + j];
                                    reinterpret_cast<__nv_bfloat16*>(ep.out)[(size_t)b * ep.ld_out + ch] =
                                        __float2bfloat16_rn(__fdividef(g, 1.0f + __expf(-g)) * u);
                                }
                            }
                        }
                    }
                    epi_sync();
                } else {
                    const int n = t * SK_BM + row_in_tile;
                    if (n < N) {
#pragma unroll
                        for (int j = 0; j < 32; ++j) {
                            const int b = c * 32 + j;
                            if (b < B) {
                                float y = acc[j];
                                if (ep.residual != nullptr) y += resv[j];
                                if (ep.out_fp32) reinterpret_cast<float*>(ep.out)[(size_t)b * ep.ld_out + n] = y;
                                else reinterpret_cast<__nv_bfloat16*>(ep.out)[(size_t)b * ep.ld_out + n] = __float2bfloat16_rn(y);
                            }
                        }
                    }
                }
            }
            if (nseg > 1 && finalize && et == 0) ep.counters[t] = 0;  // ready for the next launch
            if (finalize && et == 0 && t == t_last) SK_STAMP(10);  // epilogue stores issued
            epi_sync();  // s_acc is rewritten by the next tile
        }
        if (et == 0 && ep.trace != nullptr) ep.trace[(size_t)blockIdx.x * 16 + 8] = (unsigned long long)n_final;  // tiles finalised here
    }

    __syncthreads();
    if (threadIdx.x == 0) SK_STAMP(7);  // exit
}

struct SkPlan { int bn, num_m, nkb, grid, maxseg; long long total; };

SkPlan sk_plan(int B, int N, int K, bool fp8 = false) {
    SkPlan p;
    const int bke = fp8 ? 2 * SK_BK : SK_BK;
    p.bn = B <= 32 ? 32 : (B <= 64 ? 64 : 128);
    p.num_m = (N + SK_BM - 1) / SK_BM;
    p.nkb = (K + bke - 1) / bke;
    p.total = (long long)p.num_m * p.nkb;
    p.grid = (long long)num_sms() < p.total ? num_sms() : (int)p.total;
    const long long per_min = p.total / p.grid;  // >= 1
    p.maxseg = (int)((p.nkb + per_min - 1) / per_min) + 1;
    return p;
}

template <int BN, int ACT, bool FP8>
int sk_launch(const CUtensorMap& tw, const CUtensorMap& tx, const SkPlan& pl, int N, int K, int B, SkEpi ep,
              cudaStream_t st) {
    using Cfg = SkCfg<BN>;
    static bool attr_set = false;
    auto kern = gemm_skinny_kernel<BN, ACT, FP8>;
    if (!attr_set) {
        B2_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM));
        attr_set = true;
    }
    ep.stages = Cfg::STAGES;
    B2_CUDA_CHECK(launch_pdl(kern, dim3(pl.grid), dim3(SK_THREADS), (size_t)Cfg::SMEM, st, tw, tx, N, K, B, ep));
    B2_LAUNCH_CHECK();
    return 0;
}

}  // namespace

// scratch that satisfies BOTH element types (the fp8 plan has half the k-blocks per tile and can need one slot more)
size_t gemm_skinny_workspace_bytes(int B, int N, int K) {
    const SkPlan p = sk_plan(B, N, K, false), q = sk_plan(B, N, K, true);
    const int maxseg = p.maxseg > q.maxseg ? p.maxseg : q.maxseg;
    return (size_t)p.num_m * maxseg * p.bn * SK_BM * sizeof(float);
}
size_t gemm_skinny_counter_bytes(int N) { return (size_t)((N + SK_BM - 1) / SK_BM) * sizeof(int); }

// ---- debug trace (B2_SKINNY_TRACE=<file>): per-CTA phase stamps of the last kTraceLaunches launches, dumped at exit ----
constexpr int kTraceLaunches = 512;
constexpr int kTraceCtas = 132;  // CTAs per launch the trace has room for (grid <= #SMs)
struct SkTrace {
    unsigned long long* dev = nullptr;
    std::vector<int> shape;  // per launch: N, K, B, grid
    long long launches = 0;
    std::string path;
};
static SkTrace g_sk_trace;
static void sk_trace_dump() {
    SkTrace& t = g_sk_trace;
    if (t.dev == nullptr) return;
    const size_t per = (size_t)kTraceCtas * 16;
    std::vector<unsigned long long> host(per * kTraceLaunches);
    if (cudaDeviceSynchronize() != cudaSuccess) return;
    if (cudaMemcpy(host.data(), t.dev, host.size() * 8, cudaMemcpyDeviceToHost) != cudaSuccess) return;
    FILE* f = fopen(t.path.c_str(), "w");
    if (f == nullptr) return;
    const long long first = t.launches > kTraceLaunches ? t.launches - kTraceLaunches : 0;
    for (long long l = first; l < t.launches; ++l) {
        const int slot = (int)(l % kTraceLaunches);
        const int* sh = &t.shape[(size_t)slot * 4];
        fprintf(f, "launch %lld N %d K %d B %d grid %d\n", l, sh[0], sh[1], sh[2], sh[3]);
        for (int c = 0; c < sh[3] && c < kTraceCtas; ++c) {
            const unsigned long long* r = &host[(size_t)slot * per + (size_t)c * 16];
            fprintf(f, "%d %llu %llu %llu %llu %llu %llu %llu %llu %llu %llu %llu\n", c, r[0], r[1], r[2], r[3], r[4], r[5], r[6], r[7],
                    r[8], r[9], r[10]);
        }
    }
    fclose(f);
}
static unsigned long long* sk_trace_slot(int N, int K, int B, int grid, cudaStream_t stream) {
    static int enabled = -1;
    SkTrace& t = g_sk_trace;
    if (enabled < 0) {
        const char* e = getenv("B2_SKINNY_TRACE");
        enabled = (e != nullptr && e[0] != 0) ? 1 : 0;
        if (enabled) {
            t.path = e;
            if (cudaMalloc(&t.dev, (size_t)kTraceCtas * 16 * 8 * kTraceLaunches) != cudaSuccess) { enabled = 0; t.dev = nullptr; }
            else { cudaMemset(t.dev, 0, (size_t)kTraceCtas * 16 * 8 * kTraceLaunches); t.shape.assign((size_t)kTraceLaunches * 4, 0); atexit(sk_trace_dump); }
        }
    }
    if (!enabled) return nullptr;
    const int slot = (int)(t.launches++ % kTraceLaunches);
    int* sh = &t.shape[(size_t)slot * 4];
    sh[0] = N; sh[1] = K; sh[2] = B; sh[3] = grid;
    (void)stream;
    return t.dev + (size_t)slot * kTraceCtas * 16;
}

template <bool FP8>
static int gemm_skinny_any(const SkinnyArgs& g, cudaStream_t stream) {
    B2_CHECK_ARG(g.B >= 1 && g.B <= 128 && g.N > 0 && g.K > 0, "gemm_skinny: bad problem B=%d N=%d K=%d", g.B, g.N, g.K);
    B2_CHECK_ARG(g.K % (FP8 ? 16 : 8) == 0, "gemm_skinny: K must be a multiple of %d (K=%d)", FP8 ? 16 : 8, g.K);
    B2_CHECK_ARG(g.act == ACT_NONE || g.act == ACT_SWIGLU, "gemm_skinny: unsupported activation %d", g.act);
    B2_CHECK_ARG(g.act != ACT_SWIGLU || (g.N % 128 == 0 && !g.out_fp32 && g.residual == nullptr),
                 "gemm_skinny: swiglu needs N %% 128 == 0, bf16 output, no residual (N=%d)", g.N);
    B2_CHECK_ARG(g.partial != nullptr && g.counters != nullptr, "gemm_skinny: workspace missing");
    B2_CHECK_ARG(!FP8 || (g.w_scale != nullptr && g.x_scale != nullptr), "gemm_skinny(fp8): scale vectors missing");
    const SkPlan pl = sk_plan(g.B, g.N, g.K, FP8);
    B2_CHECK_ARG(g.partial_bytes >= (size_t)pl.num_m * pl.maxseg * pl.bn * SK_BM * sizeof(float),
                 "gemm_skinny: workspace too small (%zu bytes)", g.partial_bytes);
    CUtensorMap tw, tx;
    if (FP8) {
        B2_TRY(make_tmap_u8(&tw, g.W, g.N, g.K, g.ldw, SK_BM));
        B2_TRY(make_tmap_u8(&tx, g.x, g.B, g.K, g.ldx, pl.bn));
    } else {
        B2_TRY(make_tmap_bf16(&tw, g.W, g.N, g.K, g.ldw, SK_BM));
        B2_TRY(make_tmap_bf16(&tx, g.x, g.B, g.K, g.ldx, pl.bn));
    }
    SkEpi ep;
    ep.residual = reinterpret_cast<const __nv_bfloat16*>(g.residual);
    ep.out = g.out; ep.partial = g.partial; ep.counters = g.counters;
    ep.ld_out = g.ld_out; ep.ld_res = g.ld_res; ep.out_fp32 = g.out_fp32; ep.maxseg = pl.maxseg;
    ep.w_scale = g.w_scale; ep.x_scale = g.x_scale;
    ep.trace = sk_trace_slot(g.N, g.K, g.B, pl.grid, stream);
    const bool sw = g.act == ACT_SWIGLU;
    switch (pl.bn) {
        case 32: return sw ? sk_launch<32, ACT_SWIGLU, FP8>(tw, tx, pl, g.N, g.K, g.B, ep, stream)
                           : sk_launch<32, ACT_NONE, FP8>(tw, tx, pl, g.N, g.K, g.B, ep, stream);
        case 64: return sw ? sk_launch<64, ACT_SWIGLU, FP8>(tw, tx, pl, g.N, g.K, g.B, ep, stream)
                           : sk_launch<64, ACT_NONE, FP8>(tw, tx, pl, g.N, g.K, g.B, ep, stream);
        default: return sw ? sk_launch<128, ACT_SWIGLU, FP8>(tw, tx, pl, g.N, g.K, g.B, ep, stream)
                           : sk_launch<128, ACT_NONE, FP8>(tw, tx, pl, g.N, g.K, g.B, ep, stream);
    }
}

int gemm_skinny_bf16(const SkinnyArgs& g, cudaStream_t stream) { return gemm_skinny_any<false>(g, stream); }
// x and W hold e4m3 bytes (ldx / ldw in elements = bytes); w_scale [N], x_scale [B] fp32
int gemm_skinny_fp8(const SkinnyArgs& g, cudaStream_t stream) { return gemm_skinny_any<true>(g, stream); }

}  // namespace b2
