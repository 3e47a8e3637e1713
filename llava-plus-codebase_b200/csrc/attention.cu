// Attention kernels besides the prefill / ViT flash attention (attention_wgmma.cu).
//   rope_kv_write    : RoPE (modeling_llama.py:124-168, half-split rotate_half) on q,k of a prefill chunk and
//                      the KV-cache write (modeling_llama.py:269-270 cache update).
//   decode_attn_bf16 : one-token decode: RoPE + cache append + split-KV attention with coalesced 16-byte
//                      cache reads and an in-kernel last-CTA merge (HBM-bound: reads each K/V row once).
//   kv_quantize_e4m3 : prefill's roped bf16 K/V staging slab -> e4m3 cache rows + one fp32 scale per head-token.
//   decode_attn_e4m3 : decode_attn_bf16 over an e4m3 cache (128-byte rows, scales folded into score and p).
#include <cuda_fp16.h>
#include <cuda_fp8.h>
#include <math.h>

#include "common.cuh"
#include "kernels.h"

namespace b2 {
namespace {

// ------------------------------------------------------------------------------------------------
// helpers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void cp_async_16(void* smem_dst, const void* gsrc, bool valid) {
    const uint32_t d = smem_u32(smem_dst);
    const int sz = valid ? 16 : 0;  // src-size 0 => zero fill
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(gsrc), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], const void* smem_ptr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
                 : "r"(smem_u32(smem_ptr)));
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t (&r)[4], const void* smem_ptr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
                 : "r"(smem_u32(smem_ptr)));
}
__device__ __forceinline__ void mma_bf16_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
        "{%0,%1,%2,%3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// ------------------------------------------------------------------------------------------------
// RoPE helpers (HF semantics: cos/sin computed in fp32, cast to bf16, products rounded to bf16)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void rope_cos_sin(int pos, int i /*0..D/2*/, int D, float theta, float& c, float& s) {
    // inv_freq = theta^(-2i/D)
    const float inv_freq = exp2f(-(2.0f * i / D) * log2f(theta));
    const float ang = pos * inv_freq;
    float sv, cv;
    sincosf(ang, &sv, &cv);
    c = round_bf16(cv);
    s = round_bf16(sv);
}
__device__ __forceinline__ float rope_apply(float x, float partner_signed, float c, float s) {
    // q*cos + rotate_half(q)*sin with bf16 rounding of each product and of the sum
    return round_bf16(round_bf16(x * c) + round_bf16(partner_signed * s));
}

// the same (cos, sin) values as a table [Smax][D/2] of bf16 pairs (cos | sin << 16) for the QKV GEMM's fused RoPE epilogue
// (gemm_wgmma.cu, ACT_ROPE_QKV)
__global__ void rope_table_kernel(uint32_t* __restrict__ table, int Smax, int D, float theta) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    const int half = D / 2;
    if (idx >= Smax * half) return;
    float c, s;
    rope_cos_sin(idx / half, idx % half, D, theta, c, s);
    table[idx] = pack_bf16(c, s);  // both are bf16-rounded already: the packing is exact
}

// grid: (B*S) tokens, 256 threads. The D/2 (cos, sin) pairs of the token's position are tabulated once in shared
// memory (they are the same for every head); every thread then moves 16-byte vectors: one (head, 8-lane chunk) item
// = q/k/v elements [c*8, c*8+8) and their rotation partners [D/2 + c*8, ...), six loads and six stores of 16 B.
__global__ void __launch_bounds__(256)
rope_kv_write_kernel(__nv_bfloat16* __restrict__ qkv, __nv_bfloat16* __restrict__ kcache,
                     __nv_bfloat16* __restrict__ vcache, const int32_t* __restrict__ pos0, int S, int H, int D, int Smax,
                     float theta) {
    __shared__ float s_c[128], s_s[128];  // D/2 <= 128
    pdl_trigger();
    pdl_wait();  // inputs are outputs of the upstream kernel (programmatic dependent launch)
    const int row = blockIdx.x;  // b*S + t
    const int b = row / S;
    // absolute position of the token: its RoPE angle and its cache row. With an offset, padding rows of a chunk may lie
    // beyond the cache: they are rotated (q stays finite) but not stored.
    const int t = row % S + (pos0 != nullptr ? pos0[b] : 0);
    const bool store = t < Smax;
    const int hd = H * D;
    const int half = D / 2;
    for (int i = threadIdx.x; i < half; i += blockDim.x) rope_cos_sin(t, i, D, theta, s_c[i], s_s[i]);
    __syncthreads();
    __nv_bfloat16* q = qkv + (size_t)row * 3 * hd;
    __nv_bfloat16* k = q + hd;
    const __nv_bfloat16* v = q + 2 * hd;
    const int cpd = half / 8;  // 8-element chunks per half head
    for (int idx = threadIdx.x; idx < H * cpd; idx += blockDim.x) {
        const int h = idx / cpd, c = idx % cpd;
        const int o1 = h * D + c * 8, o2 = o1 + half;
        const uint4 q1 = *reinterpret_cast<const uint4*>(q + o1), q2 = *reinterpret_cast<const uint4*>(q + o2);
        const uint4 k1 = *reinterpret_cast<const uint4*>(k + o1), k2 = *reinterpret_cast<const uint4*>(k + o2);
        const uint4 v1 = *reinterpret_cast<const uint4*>(v + o1), v2 = *reinterpret_cast<const uint4*>(v + o2);
        const uint32_t qa[4] = {q1.x, q1.y, q1.z, q1.w}, qb[4] = {q2.x, q2.y, q2.z, q2.w};
        const uint32_t ka[4] = {k1.x, k1.y, k1.z, k1.w}, kb[4] = {k2.x, k2.y, k2.z, k2.w};
        uint32_t oq1[4], oq2[4], ok1[4], ok2[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float c0 = s_c[c * 8 + 2 * e], s0 = s_s[c * 8 + 2 * e];
            const float c1 = s_c[c * 8 + 2 * e + 1], s1 = s_s[c * 8 + 2 * e + 1];
            const float qa0 = bf16_lo(qa[e]), qa1 = bf16_hi(qa[e]), qb0 = bf16_lo(qb[e]), qb1 = bf16_hi(qb[e]);
            const float ka0 = bf16_lo(ka[e]), ka1 = bf16_hi(ka[e]), kb0 = bf16_lo(kb[e]), kb1 = bf16_hi(kb[e]);
            oq1[e] = pack_bf16(rope_apply(qa0, -qb0, c0, s0), rope_apply(qa1, -qb1, c1, s1));
            oq2[e] = pack_bf16(rope_apply(qb0, qa0, c0, s0), rope_apply(qb1, qa1, c1, s1));
            ok1[e] = pack_bf16(rope_apply(ka0, -kb0, c0, s0), rope_apply(ka1, -kb1, c1, s1));
            ok2[e] = pack_bf16(rope_apply(kb0, ka0, c0, s0), rope_apply(kb1, ka1, c1, s1));
        }
        *reinterpret_cast<uint4*>(q + o1) = make_uint4(oq1[0], oq1[1], oq1[2], oq1[3]);
        *reinterpret_cast<uint4*>(q + o2) = make_uint4(oq2[0], oq2[1], oq2[2], oq2[3]);
        if (!store) continue;
        const size_t co = (((size_t)b * H + h) * Smax + t) * D + c * 8;
        *reinterpret_cast<uint4*>(kcache + co) = make_uint4(ok1[0], ok1[1], ok1[2], ok1[3]);
        *reinterpret_cast<uint4*>(kcache + co + half) = make_uint4(ok2[0], ok2[1], ok2[2], ok2[3]);
        *reinterpret_cast<uint4*>(vcache + co) = v1;
        *reinterpret_cast<uint4*>(vcache + co + half) = v2;
    }
}

// ------------------------------------------------------------------------------------------------
// decode attention: grid (nsplit, H, B), 128 threads. D = 128 fixed: a half-warp (16 lanes x 8 elems)
// covers one K/V row with one 16-byte load per lane.
// ------------------------------------------------------------------------------------------------
constexpr int DA_D = 128;
constexpr int DA_THREADS = 128;
constexpr int DA_UNROLL = 4;

struct DecodeAttnParams {
    const __nv_bfloat16* qkv;
    __nv_bfloat16* kcache;
    __nv_bfloat16* vcache;
    const int32_t* cur_len;
    __nv_bfloat16* out;
    float* partial;
    int32_t* counters;
    int H, Smax, nsplit;
    float theta, scale_log2;
};

// One CTA of decode attention for sample b, head `head`: RoPE of q and of the new k at pos, the append of the new K / V row when
// this split's range holds pos, and the half-warp attention over keys [key_lo + split * chunk, ...) of [key_lo, pos] in b's slab;
// this CTA's partial (o[128], m, l) goes to slot part_off + split of the part_stride slots of (b, head). decode_attn_kernel runs it over [0, pos], the shared-prefix
// kernel over a row's suffix [P, pos]: both append bit-identical rows.
__device__ __forceinline__ void decode_attn_cta(const __nv_bfloat16* qkv, __nv_bfloat16* kcache, __nv_bfloat16* vcache, int b,
                                                int head, int split, int nsplit, int pos, int key_lo, int H, int Smax, float theta,
                                                float scale_log2, float* partial, int part_stride, int part_off, float* s_q, float* s_knew, float* s_m, float* s_l,
                                                float (*s_o)[DA_D]) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int hw = (warp << 1) | (lane >> 4);  // half-warp id 0..7
    const int c = lane & 15;                   // 8-element chunk of the head dim
    const int total = pos + 1;
    const int hd = H * DA_D;

    // ---- RoPE on q and the new k (every CTA: 128 threads, one element each) ----
    {
        const __nv_bfloat16* qrow = qkv + (size_t)b * 3 * hd + head * DA_D;
        const __nv_bfloat16* krow = qrow + hd;
        const int i = tid & 63;
        float cs, sn;
        rope_cos_sin(pos, i, DA_D, theta, cs, sn);
        const float q1 = __bfloat162float(qrow[i]), q2 = __bfloat162float(qrow[i + 64]);
        const float k1 = __bfloat162float(krow[i]), k2 = __bfloat162float(krow[i + 64]);
        if (tid < 64) {
            s_q[i] = rope_apply(q1, -q2, cs, sn);
            s_knew[i] = rope_apply(k1, -k2, cs, sn);
        } else {
            s_q[i + 64] = rope_apply(q2, q1, cs, sn);
            s_knew[i + 64] = rope_apply(k2, k1, cs, sn);
        }
    }
    __syncthreads();

    // key range of this split (device-side: the launch grid is fixed so the step can live in a CUDA graph)
    const int chunk = (total - key_lo + nsplit - 1) / nsplit;
    const int k_begin = key_lo + split * chunk;
    const int k_end = min(k_begin + chunk, total);
    const bool owns_new = (pos >= k_begin) && (pos < k_end);

    const size_t cbase = ((size_t)b * H + head) * Smax * DA_D;
    if (owns_new) {
        // append the new token's k (roped) and v to the cache; exactly one CTA per (b, head) does this
        const __nv_bfloat16* vrow = qkv + (size_t)b * 3 * hd + 2 * hd + head * DA_D;
        kcache[cbase + (size_t)pos * DA_D + tid] = __float2bfloat16_rn(s_knew[tid]);
        vcache[cbase + (size_t)pos * DA_D + tid] = vrow[tid];
    }

    float qreg[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) qreg[e] = s_q[c * 8 + e];

    float m_run = -INFINITY, l_run = 0.f;
    float acc[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] = 0.f;

    const __nv_bfloat16* kb = kcache + cbase + c * 8;
    const __nv_bfloat16* vb = vcache + cbase + c * 8;
    const __nv_bfloat16* vnew = qkv + (size_t)b * 3 * hd + 2 * hd + head * DA_D + c * 8;
    // each half-warp walks keys k_begin + hw, +8, ...; DA_UNROLL keys (2*DA_UNROLL 16B loads) in flight
    // (trip count is CTA-uniform: the shuffles below use the full warp mask)
    for (int kbase = k_begin; kbase < k_end; kbase += 8 * DA_UNROLL) {
        const int k0 = kbase + hw;
        uint4 kraw[DA_UNROLL], vraw[DA_UNROLL];
#pragma unroll
        for (int u = 0; u < DA_UNROLL; ++u) {
            const int key = k0 + u * 8;
            if (key < k_end && key != pos) {
                kraw[u] = ld_stream_16(kb + (size_t)key * DA_D);
                vraw[u] = ld_stream_16(vb + (size_t)key * DA_D);
            } else {
                kraw[u] = make_uint4(0, 0, 0, 0);
                vraw[u] = make_uint4(0, 0, 0, 0);
            }
        }
#pragma unroll
        for (int u = 0; u < DA_UNROLL; ++u) {
            const int key = k0 + u * 8;
            const bool valid = key < k_end;  // uniform across the half-warp
            float kf[8], vf[8];
            if (key == pos) {
                // the new token: k from smem (already roped, bf16-rounded), v straight from qkv
#pragma unroll
                for (int e = 0; e < 8; ++e) kf[e] = round_bf16(s_knew[c * 8 + e]);
                const uint4 vv = *reinterpret_cast<const uint4*>(vnew);
                vf[0] = bf16_lo(vv.x); vf[1] = bf16_hi(vv.x); vf[2] = bf16_lo(vv.y); vf[3] = bf16_hi(vv.y);
                vf[4] = bf16_lo(vv.z); vf[5] = bf16_hi(vv.z); vf[6] = bf16_lo(vv.w); vf[7] = bf16_hi(vv.w);
            } else {
                kf[0] = bf16_lo(kraw[u].x); kf[1] = bf16_hi(kraw[u].x); kf[2] = bf16_lo(kraw[u].y);
                kf[3] = bf16_hi(kraw[u].y); kf[4] = bf16_lo(kraw[u].z); kf[5] = bf16_hi(kraw[u].z);
                kf[6] = bf16_lo(kraw[u].w); kf[7] = bf16_hi(kraw[u].w);
                vf[0] = bf16_lo(vraw[u].x); vf[1] = bf16_hi(vraw[u].x); vf[2] = bf16_lo(vraw[u].y);
                vf[3] = bf16_hi(vraw[u].y); vf[4] = bf16_lo(vraw[u].z); vf[5] = bf16_hi(vraw[u].z);
                vf[6] = bf16_lo(vraw[u].w); vf[7] = bf16_hi(vraw[u].w);
            }
            float dot = 0.f;
#pragma unroll
            for (int e = 0; e < 8; ++e) dot += qreg[e] * kf[e];
            // reduce over the 16 lanes of the half-warp (xor 8,4,2,1 stays inside the half)
            dot += __shfl_xor_sync(0xffffffffu, dot, 8);
            dot += __shfl_xor_sync(0xffffffffu, dot, 4);
            dot += __shfl_xor_sync(0xffffffffu, dot, 2);
            dot += __shfl_xor_sync(0xffffffffu, dot, 1);
            if (valid) {
                const float sc = dot * scale_log2;
                const float m_new = fmaxf(m_run, sc);
                const float corr = exp2f(m_run - m_new);
                const float pr = exp2f(sc - m_new);
                l_run = l_run * corr + pr;
#pragma unroll
                for (int e = 0; e < 8; ++e) acc[e] = acc[e] * corr + pr * vf[e];
                m_run = m_new;
            }
        }
    }

    // ---- merge the 8 half-warps of this CTA ----
    if (c == 0) { s_m[hw] = m_run; s_l[hw] = l_run; }
#pragma unroll
    for (int e = 0; e < 8; ++e) s_o[hw][c * 8 + e] = acc[e];
    __syncthreads();
    float m_cta = -INFINITY;
#pragma unroll
    for (int i = 0; i < 8; ++i) m_cta = fmaxf(m_cta, s_m[i]);
    float l_cta = 0.f, o_cta = 0.f;  // thread tid owns output element tid
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const float w = (s_m[i] == -INFINITY) ? 0.f : exp2f(s_m[i] - m_cta);
        l_cta += s_l[i] * w;
        o_cta += s_o[i][tid] * w;
    }
    const int bh = b * H + head;
    float* part = partial + ((size_t)bh * part_stride + part_off + split) * (DA_D + 2);
    part[tid] = o_cta;
    if (tid == 0) { part[DA_D] = m_cta; part[DA_D + 1] = l_cta; }
}

__global__ void __launch_bounds__(DA_THREADS) decode_attn_kernel(DecodeAttnParams p) {
    const int split = blockIdx.x, head = blockIdx.y, b = blockIdx.z;
    const int tid = threadIdx.x;
    pdl_trigger();
    pdl_wait();                                // qkv (previous GEMM) and cur_len (previous step) are upstream outputs
    const int pos = p.cur_len[b];              // position of the new token == number of cached keys
    const int hd = p.H * DA_D;

    __shared__ float s_q[DA_D];
    __shared__ float s_knew[DA_D];
    __shared__ float s_m[8], s_l[8];
    __shared__ float s_o[8][DA_D];
    __shared__ int s_last;

    decode_attn_cta(p.qkv, p.kcache, p.vcache, b, head, split, p.nsplit, pos, 0, p.H, p.Smax, p.theta, p.scale_log2, p.partial,
                    p.nsplit, 0, s_q, s_knew, s_m, s_l, s_o);
    const int bh = b * p.H + head;

    // ---- last CTA of this (b, head) merges the splits ----
    __threadfence();
    __syncthreads();
    if (tid == 0) {
        const int prev = atomicAdd(&p.counters[bh], 1);
        s_last = (prev == p.nsplit - 1) ? 1 : 0;
    }
    __syncthreads();
    if (s_last) {
        __threadfence();
        const float* pb = p.partial + (size_t)bh * p.nsplit * (DA_D + 2);
        float m_all = -INFINITY;
#pragma unroll 8
        for (int s = 0; s < p.nsplit; ++s) m_all = fmaxf(m_all, __ldcg(pb + (size_t)s * (DA_D + 2) + DA_D));
        float l_all = 0.f, o_all = 0.f;
#pragma unroll 8
        for (int s = 0; s < p.nsplit; ++s) {  // independent loads: unrolled so they overlap instead of chaining
            const float ms = __ldcg(pb + (size_t)s * (DA_D + 2) + DA_D);
            const float w = (ms == -INFINITY) ? 0.f : exp2f(ms - m_all);
            l_all += __ldcg(pb + (size_t)s * (DA_D + 2) + DA_D + 1) * w;
            o_all += __ldcg(pb + (size_t)s * (DA_D + 2) + tid) * w;
        }
        p.out[(size_t)b * hd + head * DA_D + tid] = __float2bfloat16_rn(o_all / l_all);
        if (tid == 0) p.counters[bh] = 0;  // self-reset for the next launch
    }
}

// ------------------------------------------------------------------------------------------------
// multi-query decode attention (the prompt-lookup verify step): R <= 16 query rows of one sample, row j at position
// len + j attending cache rows 0 .. len + j. The rows' own K / V are already in the cache and q is roped in place in qkv
// (rope_kv_write at pos0 = cur_len). grid (nsplit, H, B), 128 threads. Each 64-key tile of the split's range is loaded
// once (cp.async, double-buffered) and serves every query row: the 16 rows are one mma.sync m16n8k16 A tile for QK^T and
// for PV, warp w takes keys [16w, 16w + 16) of each tile with its own fp32 online softmax. The four warps merge in shared
// memory, and the last CTA of a (b, head) merges the splits in split order, as decode_attn_kernel does.
// ------------------------------------------------------------------------------------------------
constexpr int MQ_ROWS = 16;
constexpr int MQ_BN = 64;
constexpr int MQ_LD = DA_D + 8;  // padded smem row: conflict-free ldmatrix
constexpr size_t MQ_SMEM = (size_t)(MQ_ROWS + 4 * MQ_BN) * MQ_LD * sizeof(__nv_bfloat16);

struct DecodeAttnMqParams {
    const __nv_bfloat16* qkv;  // [B*R, 3*H*128], q roped
    const __nv_bfloat16* kcache;
    const __nv_bfloat16* vcache;
    const int32_t* cur_len;    // [B]: position of row 0
    __nv_bfloat16* out;        // [B*R, H*128]
    float* partial;            // [B*H*nsplit][16][128 + 2]
    int32_t* counters;         // [B*H]
    int R, H, Smax, nsplit;
    float scale_log2;
};

__global__ void __launch_bounds__(128) decode_attn_mq_kernel(DecodeAttnMqParams p) {
    extern __shared__ __align__(16) uint8_t mq_smem[];
    __nv_bfloat16* sQ = reinterpret_cast<__nv_bfloat16*>(mq_smem);  // [16][LD]
    __nv_bfloat16* sK = sQ + MQ_ROWS * MQ_LD;                         // [2][64][LD]
    __nv_bfloat16* sV = sK + 2 * MQ_BN * MQ_LD;                       // [2][64][LD]
    __shared__ int s_last;
    const int split = blockIdx.x, head = blockIdx.y, b = blockIdx.z;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    pdl_trigger();
    pdl_wait();  // qkv (rope_kv_write) and cur_len are upstream outputs
    const int R = p.R, len = p.cur_len[b];
    const int total = len + R;  // keys the last row attends
    const int hd = p.H * DA_D;
    const int chunk = (total + p.nsplit - 1) / p.nsplit;
    const int k_begin = min(split * chunk, total), k_end = min(k_begin + chunk, total);
    const int n_tiles = (k_end - k_begin + MQ_BN - 1) / MQ_BN;

    const size_t cbase = ((size_t)b * p.H + head) * p.Smax * DA_D;
    const __nv_bfloat16* kg = p.kcache + cbase;
    const __nv_bfloat16* vg = p.vcache + cbase;
    const __nv_bfloat16* qg = p.qkv + (size_t)b * R * 3 * hd + head * DA_D;
    constexpr int CH = DA_D / 8;  // 16-byte chunks per row
    for (int i = tid; i < MQ_ROWS * CH; i += 128) {
        const int r = i / CH, c = i % CH;
        cp_async_16(sQ + r * MQ_LD + c * 8, qg + (size_t)min(r, R - 1) * 3 * hd + c * 8, r < R);  // rows >= R are zero
    }
    auto load_kv = [&](int tile, int buf) {
        for (int i = tid; i < MQ_BN * CH; i += 128) {
            const int r = i / CH, c = i % CH;
            const int t = k_begin + tile * MQ_BN + r;
            const bool ok = t < k_end;
            const size_t off = (size_t)(ok ? t : 0) * DA_D + c * 8;
            cp_async_16(sK + (buf * MQ_BN + r) * MQ_LD + c * 8, kg + off, ok);
            cp_async_16(sV + (buf * MQ_BN + r) * MQ_LD + c * 8, vg + off, ok);
        }
    };
    if (n_tiles > 0) load_kv(0, 0);
    cp_async_commit();

    uint32_t qf[DA_D / 16][4];
    float oacc[DA_D / 8][4];
#pragma unroll
    for (int i = 0; i < DA_D / 8; ++i) oacc[i][0] = oacc[i][1] = oacc[i][2] = oacc[i][3] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY};
    float l_run[2] = {0.f, 0.f};
    const int g = lane >> 2, tq = lane & 3;  // this thread's query rows: g and g + 8

    for (int j = 0; j < n_tiles; ++j) {
        if (j + 1 < n_tiles) load_kv(j + 1, (j + 1) & 1);
        cp_async_commit();
        cp_async_wait<1>();
        __syncthreads();
        if (j == 0) {
#pragma unroll
            for (int kk = 0; kk < DA_D / 16; ++kk)
                ldmatrix_x4(qf[kk], sQ + ((lane & 7) + ((lane >> 3) & 1) * 8) * MQ_LD + kk * 16 + (lane >> 4) * 8);
        }
        const __nv_bfloat16* tK = sK + ((j & 1) * MQ_BN + warp * 16) * MQ_LD;
        const __nv_bfloat16* tV = sV + ((j & 1) * MQ_BN + warp * 16) * MQ_LD;

        // ---- S = Q K^T over this warp's 16 keys ----
        float s[2][4];
#pragma unroll
        for (int nt = 0; nt < 2; ++nt) s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
#pragma unroll
        for (int kk = 0; kk < DA_D / 16; ++kk) {
            uint32_t bfr[4];
            ldmatrix_x4(bfr, tK + ((lane & 7) + (lane >> 4) * 8) * MQ_LD + kk * 16 + ((lane >> 3) & 1) * 8);
            mma_bf16_16816(s[0], qf[kk], bfr[0], bfr[1]);
            mma_bf16_16816(s[1], qf[kk], bfr[2], bfr[3]);
        }

        // ---- scale, per-row causal limit, online softmax (fp32, log2 domain) ----
        const int key0 = k_begin + j * MQ_BN + warp * 16;
        float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int nt = 0; nt < 2; ++nt) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int key = key0 + nt * 8 + tq * 2 + (e & 1);
                const int row = g + (e >> 1) * 8;
                const bool ok = key < k_end && key <= len + row;
                const float val = ok ? s[nt][e] * p.scale_log2 : -INFINITY;
                s[nt][e] = val;
                mx[e >> 1] = fmaxf(mx[e >> 1], val);
            }
        }
        float corr[2], m_use[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
            mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
            const float m_new = fmaxf(m_run[h], mx[h]);
            m_use[h] = (m_new == -INFINITY) ? 0.f : m_new;
            corr[h] = exp2f(m_run[h] - m_use[h]);
            m_run[h] = m_new;
            l_run[h] *= corr[h];
        }
#pragma unroll
        for (int nt = 0; nt < 2; ++nt) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float pv = exp2f(s[nt][e] - m_use[e >> 1]);
                s[nt][e] = pv;
                l_run[e >> 1] += pv;
            }
        }
#pragma unroll
        for (int i = 0; i < DA_D / 8; ++i) {
            oacc[i][0] *= corr[0]; oacc[i][1] *= corr[0];
            oacc[i][2] *= corr[1]; oacc[i][3] *= corr[1];
        }

        // ---- O += P V, with P = hi + lo as two bf16 operands: p keeps ~16 significant bits, close to decode_attn's fp32 p ----
        uint32_t pa[4], pl[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float x0 = s[i >> 1][(i & 1) * 2], x1 = s[i >> 1][(i & 1) * 2 + 1];
            pa[i] = pack_bf16(x0, x1);
            pl[i] = pack_bf16(x0 - bf16_lo(pa[i]), x1 - bf16_hi(pa[i]));
        }
#pragma unroll
        for (int dp = 0; dp < DA_D / 16; ++dp) {
            uint32_t bfr[4];
            ldmatrix_x4_trans(bfr, tV + ((lane & 7) + ((lane >> 3) & 1) * 8) * MQ_LD + dp * 16 + (lane >> 4) * 8);
            mma_bf16_16816(oacc[2 * dp], pa, bfr[0], bfr[1]);
            mma_bf16_16816(oacc[2 * dp + 1], pa, bfr[2], bfr[3]);
            mma_bf16_16816(oacc[2 * dp], pl, bfr[0], bfr[1]);
            mma_bf16_16816(oacc[2 * dp + 1], pl, bfr[2], bfr[3]);
        }
        __syncthreads();  // buffer (j & 1) is refilled at iteration j + 1
    }
    cp_async_wait<0>();
    __syncthreads();

    // ---- merge the four warps (the K tiles' shared memory is free now) ----
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 1);
        l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 2);
    }
    float* s_o = reinterpret_cast<float*>(sK);   // [4][16][128]
    float* s_ml = reinterpret_cast<float*>(sV);  // [4][16][2]
#pragma unroll
    for (int i = 0; i < DA_D / 8; ++i)
#pragma unroll
        for (int e = 0; e < 4; ++e)
            s_o[(warp * MQ_ROWS + g + (e >> 1) * 8) * DA_D + i * 8 + tq * 2 + (e & 1)] = oacc[i][e];
    if (tq == 0)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            s_ml[(warp * MQ_ROWS + g + h * 8) * 2] = m_run[h];
            s_ml[(warp * MQ_ROWS + g + h * 8) * 2 + 1] = l_run[h];
        }
    __syncthreads();
    const int bh = b * p.H + head;
    for (int r = 0; r < R; ++r) {  // thread tid owns output column tid
        float m_cta = -INFINITY;
#pragma unroll
        for (int w = 0; w < 4; ++w) m_cta = fmaxf(m_cta, s_ml[(w * MQ_ROWS + r) * 2]);
        float l_cta = 0.f, o_cta = 0.f;
#pragma unroll
        for (int w = 0; w < 4; ++w) {
            const float mw = s_ml[(w * MQ_ROWS + r) * 2];
            const float wt = (mw == -INFINITY) ? 0.f : exp2f(mw - m_cta);
            l_cta += s_ml[(w * MQ_ROWS + r) * 2 + 1] * wt;
            o_cta += s_o[(w * MQ_ROWS + r) * DA_D + tid] * wt;
        }
        float* part = p.partial + (((size_t)bh * p.nsplit + split) * MQ_ROWS + r) * (DA_D + 2);
        part[tid] = o_cta;
        if (tid == 0) { part[DA_D] = m_cta; part[DA_D + 1] = l_cta; }
    }

    // ---- last CTA of this (b, head) merges the splits ----
    __threadfence();
    __syncthreads();
    if (tid == 0) {
        const int prev = atomicAdd(&p.counters[bh], 1);
        s_last = (prev == p.nsplit - 1) ? 1 : 0;
    }
    __syncthreads();
    if (s_last) {
        __threadfence();
        for (int r = 0; r < R; ++r) {
            const float* pb = p.partial + ((size_t)bh * p.nsplit * MQ_ROWS + r) * (DA_D + 2);
            const size_t stride = (size_t)MQ_ROWS * (DA_D + 2);
            float m_all = -INFINITY;
            for (int s = 0; s < p.nsplit; ++s) m_all = fmaxf(m_all, __ldcg(pb + s * stride + DA_D));
            float l_all = 0.f, o_all = 0.f;
#pragma unroll 4
            for (int s = 0; s < p.nsplit; ++s) {
                const float ms = __ldcg(pb + s * stride + DA_D);
                const float wt = (ms == -INFINITY) ? 0.f : exp2f(ms - m_all);
                l_all += __ldcg(pb + s * stride + DA_D + 1) * wt;
                o_all += __ldcg(pb + s * stride + tid) * wt;
            }
            p.out[((size_t)b * R + r) * hd + head * DA_D + tid] = __float2bfloat16_rn(o_all / l_all);
        }
        if (tid == 0) p.counters[bh] = 0;  // self-reset for the next launch
    }
}

// ------------------------------------------------------------------------------------------------
// shared-prefix decode attention: the result of decode_attn_kernel for every row b at pos = cur_len[b], for a batch whose rows
// come in groups that share a prompt. Keys [0, P_g) of group g's rows are read from the group's source slot (the rows' own
// copies of them are never read); keys [P_g, pos] of a row come from its own slot, and a row outside every group attends its
// own slot only. grid (nsplit, H, G + B), 128 threads:
//   z <  G : group z's prefix, split nsplit ways. Each 64-key tile of the split's range is loaded once (cp.async, double-
//            buffered) and scores all (<= 16) rows of the group as one mma.sync m16n8k16 A tile, as decode_attn_mq_kernel
//            does; the CTA ropes the rows' q itself. Partial (o, m, l) of row r -> slot `split` of (r, head).
//   z >= G : row z - G, decode_attn_cta over its suffix [P, pos] (RoPE, the append of the new row, half-warp attention), split
//            nsplit ways. Partial -> slot nsplit + split.
// The last CTA of a (row, head) merges its 2 * nsplit partials (nsplit for a row outside every group) in slot order and resets
// the counter.
// ------------------------------------------------------------------------------------------------
constexpr size_t SH_SMEM = MQ_SMEM;

struct DecodeAttnSharedParams {
    const __nv_bfloat16* qkv;  // [B, 3*H*128], not roped
    __nv_bfloat16* kcache;
    __nv_bfloat16* vcache;
    const int32_t* cur_len;    // [B]
    const PrefixGroup* groups; // [G]
    const int32_t* row_prefix; // [B]: P of the row's group, 0 outside every group
    __nv_bfloat16* out;        // [B, H*128]
    float* partial;            // [B*H][2*nsplit][128 + 2]
    int32_t* counters;         // [B*H]
    int G, H, Smax, nsplit;
    float theta, scale_log2;
};

// the merge of row b's partials (slots [s0, 2 * nsplit) of (b, head)) by the CTA that completed them
__device__ __forceinline__ void shared_merge(const DecodeAttnSharedParams& p, int b, int head, int s0) {
    const int tid = threadIdx.x;
    const int bh = b * p.H + head;
    const float* pb = p.partial + (size_t)bh * 2 * p.nsplit * (DA_D + 2);
    float m_all = -INFINITY;
    for (int s = s0; s < 2 * p.nsplit; ++s) m_all = fmaxf(m_all, __ldcg(pb + (size_t)s * (DA_D + 2) + DA_D));
    float l_all = 0.f, o_all = 0.f;
#pragma unroll 4
    for (int s = s0; s < 2 * p.nsplit; ++s) {
        const float ms = __ldcg(pb + (size_t)s * (DA_D + 2) + DA_D);
        const float w = (ms == -INFINITY) ? 0.f : exp2f(ms - m_all);
        l_all += __ldcg(pb + (size_t)s * (DA_D + 2) + DA_D + 1) * w;
        o_all += __ldcg(pb + (size_t)s * (DA_D + 2) + tid) * w;
    }
    p.out[(size_t)b * p.H * DA_D + head * DA_D + tid] = __float2bfloat16_rn(o_all / l_all);
    if (tid == 0) p.counters[bh] = 0;  // self-reset for the next launch
}

__global__ void __launch_bounds__(128) decode_attn_shared_kernel(DecodeAttnSharedParams p) {
    extern __shared__ __align__(16) uint8_t sh_smem[];
    __shared__ int s_rows[MQ_ROWS];
    __shared__ int s_last[MQ_ROWS];
    const int split = blockIdx.x, head = blockIdx.y, z = blockIdx.z;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    pdl_trigger();
    pdl_wait();  // qkv (previous GEMM) and cur_len (previous step) are upstream outputs
    const int hd = p.H * DA_D;

    if (z >= p.G) {  // ---- a row's suffix ----
        const int b = z - p.G;
        const int pos = p.cur_len[b], P = p.row_prefix[b];
        float* s_q = reinterpret_cast<float*>(sh_smem);
        float* s_knew = s_q + DA_D;
        float* s_m = s_knew + DA_D;
        float* s_l = s_m + 8;
        float (*s_o)[DA_D] = reinterpret_cast<float (*)[DA_D]>(s_l + 8);
        const int bh = b * p.H + head;
        decode_attn_cta(p.qkv, p.kcache, p.vcache, b, head, split, p.nsplit, pos, P, p.H, p.Smax, p.theta, p.scale_log2, p.partial,
                        2 * p.nsplit, p.nsplit, s_q, s_knew, s_m, s_l, s_o);
        __threadfence();
        __syncthreads();
        if (tid == 0) {
            const int prev = atomicAdd(&p.counters[bh], 1);
            s_last[0] = (prev == (P > 0 ? 2 : 1) * p.nsplit - 1) ? 1 : 0;
        }
        __syncthreads();
        if (s_last[0]) {
            __threadfence();
            shared_merge(p, b, head, P > 0 ? 0 : p.nsplit);
        }
        return;
    }

    // ---- a group's prefix ----
    __nv_bfloat16* sQ = reinterpret_cast<__nv_bfloat16*>(sh_smem);  // [16][LD]
    __nv_bfloat16* sK = sQ + MQ_ROWS * MQ_LD;                         // [2][64][LD]
    __nv_bfloat16* sV = sK + 2 * MQ_BN * MQ_LD;                       // [2][64][LD]
    const PrefixGroup& gr = p.groups[z];
    const int n = gr.n_rows, P = gr.prefix_len;
    if (tid < MQ_ROWS) s_rows[tid] = tid < n ? gr.rows[tid] : 0;
    const int chunk = (P + p.nsplit - 1) / p.nsplit;
    const int k_begin = min(split * chunk, P), k_end = min(k_begin + chunk, P);
    const int n_tiles = (k_end - k_begin + MQ_BN - 1) / MQ_BN;
    const size_t cbase = ((size_t)gr.src_slot * p.H + head) * p.Smax * DA_D;
    const __nv_bfloat16* kg = p.kcache + cbase;
    const __nv_bfloat16* vg = p.vcache + cbase;
    constexpr int CH = DA_D / 8;
    auto load_kv = [&](int tile, int buf) {
        for (int i = tid; i < MQ_BN * CH; i += 128) {
            const int r = i / CH, c = i % CH;
            const int t = k_begin + tile * MQ_BN + r;
            const bool ok = t < k_end;
            const size_t off = (size_t)(ok ? t : 0) * DA_D + c * 8;
            cp_async_16(sK + (buf * MQ_BN + r) * MQ_LD + c * 8, kg + off, ok);
            cp_async_16(sV + (buf * MQ_BN + r) * MQ_LD + c * 8, vg + off, ok);
        }
    };
    if (n_tiles > 0) load_kv(0, 0);
    cp_async_commit();
    __syncthreads();  // s_rows
    // q of every row, roped at the row's own position exactly as decode_attn_cta ropes it (bf16 values: exact as an mma operand);
    // rows >= n are zero
    for (int i = tid; i < MQ_ROWS * 64; i += 128) {
        const int r = i >> 6, e = i & 63;
        float lo = 0.f, hi = 0.f;
        if (r < n) {
            const int row = s_rows[r];
            const __nv_bfloat16* qrow = p.qkv + (size_t)row * 3 * hd + head * DA_D;
            float cs, sn;
            rope_cos_sin(p.cur_len[row], e, DA_D, p.theta, cs, sn);
            const float q1 = __bfloat162float(qrow[e]), q2 = __bfloat162float(qrow[e + 64]);
            lo = rope_apply(q1, -q2, cs, sn);
            hi = rope_apply(q2, q1, cs, sn);
        }
        sQ[r * MQ_LD + e] = __float2bfloat16_rn(lo);
        sQ[r * MQ_LD + e + 64] = __float2bfloat16_rn(hi);
    }

    uint32_t qf[DA_D / 16][4];
    float oacc[DA_D / 8][4];
#pragma unroll
    for (int i = 0; i < DA_D / 8; ++i) oacc[i][0] = oacc[i][1] = oacc[i][2] = oacc[i][3] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY};
    float l_run[2] = {0.f, 0.f};
    const int g = lane >> 2, tq = lane & 3;  // this thread's rows: g and g + 8

    for (int j = 0; j < n_tiles; ++j) {
        if (j + 1 < n_tiles) load_kv(j + 1, (j + 1) & 1);
        cp_async_commit();
        cp_async_wait<1>();
        __syncthreads();
        if (j == 0) {
#pragma unroll
            for (int kk = 0; kk < DA_D / 16; ++kk)
                ldmatrix_x4(qf[kk], sQ + ((lane & 7) + ((lane >> 3) & 1) * 8) * MQ_LD + kk * 16 + (lane >> 4) * 8);
        }
        const __nv_bfloat16* tK = sK + ((j & 1) * MQ_BN + warp * 16) * MQ_LD;
        const __nv_bfloat16* tV = sV + ((j & 1) * MQ_BN + warp * 16) * MQ_LD;

        float s[2][4];
#pragma unroll
        for (int nt = 0; nt < 2; ++nt) s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
#pragma unroll
        for (int kk = 0; kk < DA_D / 16; ++kk) {
            uint32_t bfr[4];
            ldmatrix_x4(bfr, tK + ((lane & 7) + (lane >> 4) * 8) * MQ_LD + kk * 16 + ((lane >> 3) & 1) * 8);
            mma_bf16_16816(s[0], qf[kk], bfr[0], bfr[1]);
            mma_bf16_16816(s[1], qf[kk], bfr[2], bfr[3]);
        }

        // every row's position is >= P: the only limit is the end of the split's range
        const int key0 = k_begin + j * MQ_BN + warp * 16;
        float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int nt = 0; nt < 2; ++nt) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int key = key0 + nt * 8 + tq * 2 + (e & 1);
                const float val = key < k_end ? s[nt][e] * p.scale_log2 : -INFINITY;
                s[nt][e] = val;
                mx[e >> 1] = fmaxf(mx[e >> 1], val);
            }
        }
        float corr[2], m_use[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
            mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
            const float m_new = fmaxf(m_run[h], mx[h]);
            m_use[h] = (m_new == -INFINITY) ? 0.f : m_new;
            corr[h] = exp2f(m_run[h] - m_use[h]);
            m_run[h] = m_new;
            l_run[h] *= corr[h];
        }
#pragma unroll
        for (int nt = 0; nt < 2; ++nt) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float pv = exp2f(s[nt][e] - m_use[e >> 1]);
                s[nt][e] = pv;
                l_run[e >> 1] += pv;
            }
        }
#pragma unroll
        for (int i = 0; i < DA_D / 8; ++i) {
            oacc[i][0] *= corr[0]; oacc[i][1] *= corr[0];
            oacc[i][2] *= corr[1]; oacc[i][3] *= corr[1];
        }
        // O += P V with P = hi + lo bf16 operands
        uint32_t pa[4], pl[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float x0 = s[i >> 1][(i & 1) * 2], x1 = s[i >> 1][(i & 1) * 2 + 1];
            pa[i] = pack_bf16(x0, x1);
            pl[i] = pack_bf16(x0 - bf16_lo(pa[i]), x1 - bf16_hi(pa[i]));
        }
#pragma unroll
        for (int dp = 0; dp < DA_D / 16; ++dp) {
            uint32_t bfr[4];
            ldmatrix_x4_trans(bfr, tV + ((lane & 7) + ((lane >> 3) & 1) * 8) * MQ_LD + dp * 16 + (lane >> 4) * 8);
            mma_bf16_16816(oacc[2 * dp], pa, bfr[0], bfr[1]);
            mma_bf16_16816(oacc[2 * dp + 1], pa, bfr[2], bfr[3]);
            mma_bf16_16816(oacc[2 * dp], pl, bfr[0], bfr[1]);
            mma_bf16_16816(oacc[2 * dp + 1], pl, bfr[2], bfr[3]);
        }
        __syncthreads();  // buffer (j & 1) is refilled at iteration j + 1
    }
    cp_async_wait<0>();
    __syncthreads();

    // ---- merge the four warps, one partial per row of the group ----
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 1);
        l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 2);
    }
    float* s_o = reinterpret_cast<float*>(sK);   // [4][16][128]
    float* s_ml = reinterpret_cast<float*>(sV);  // [4][16][2]
#pragma unroll
    for (int i = 0; i < DA_D / 8; ++i)
#pragma unroll
        for (int e = 0; e < 4; ++e)
            s_o[(warp * MQ_ROWS + g + (e >> 1) * 8) * DA_D + i * 8 + tq * 2 + (e & 1)] = oacc[i][e];
    if (tq == 0)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            s_ml[(warp * MQ_ROWS + g + h * 8) * 2] = m_run[h];
            s_ml[(warp * MQ_ROWS + g + h * 8) * 2 + 1] = l_run[h];
        }
    __syncthreads();
    for (int r = 0; r < n; ++r) {  // thread tid owns output column tid
        float m_cta = -INFINITY;
#pragma unroll
        for (int w = 0; w < 4; ++w) m_cta = fmaxf(m_cta, s_ml[(w * MQ_ROWS + r) * 2]);
        float l_cta = 0.f, o_cta = 0.f;
#pragma unroll
        for (int w = 0; w < 4; ++w) {
            const float mw = s_ml[(w * MQ_ROWS + r) * 2];
            const float wt = (mw == -INFINITY) ? 0.f : exp2f(mw - m_cta);
            l_cta += s_ml[(w * MQ_ROWS + r) * 2 + 1] * wt;
            o_cta += s_o[(w * MQ_ROWS + r) * DA_D + tid] * wt;
        }
        float* part = p.partial + (((size_t)s_rows[r] * p.H + head) * 2 * p.nsplit + split) * (DA_D + 2);
        part[tid] = o_cta;
        if (tid == 0) { part[DA_D] = m_cta; part[DA_D + 1] = l_cta; }
    }

    // ---- the last CTA of a (row, head) merges that row ----
    __threadfence();
    __syncthreads();
    if (tid < n) {
        const int prev = atomicAdd(&p.counters[s_rows[tid] * p.H + head], 1);
        s_last[tid] = (prev == 2 * p.nsplit - 1) ? 1 : 0;
    }
    __syncthreads();
    for (int r = 0; r < n; ++r) {
        if (!s_last[r]) continue;  // CTA-uniform
        __threadfence();
        shared_merge(p, s_rows[r], head, 0);
    }
}

// ------------------------------------------------------------------------------------------------
// e4m3 KV cache. A cache row is one head of one token: 128 e4m3 bytes + one fp32 scale (amax / 448, 1 for a zero row;
// the rule of quant_fp8.cu over the 128 elements of the row). K is quantised after RoPE.
// ------------------------------------------------------------------------------------------------
constexpr float kE4M3Max = 448.0f;

__device__ __forceinline__ uint32_t pack4_e4m3(float a, float b, float c, float d) {
    const uint32_t lo = __nv_cvt_float2_to_fp8x2(make_float2(a, b), __NV_SATFINITE, __NV_E4M3);
    const uint32_t hi = __nv_cvt_float2_to_fp8x2(make_float2(c, d), __NV_SATFINITE, __NV_E4M3);
    return lo | (hi << 16);
}
// 4 e4m3 bytes -> 4 floats through the packed e4m3x2 -> f16x2 conversion (exact: every e4m3 value is an f16 value)
__device__ __forceinline__ void unpack4_e4m3(uint32_t w, float* f) {
    uint32_t h01, h23;
    asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(h01) : "h"(static_cast<unsigned short>(w & 0xffffu)));
    asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(h23) : "h"(static_cast<unsigned short>(w >> 16)));
    const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&h01));
    const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&h23));
    f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y;
}
__device__ __forceinline__ void unpack16_e4m3(const uint4& u, float (&f)[16]) {
    unpack4_e4m3(u.x, f); unpack4_e4m3(u.y, f + 4); unpack4_e4m3(u.z, f + 8); unpack4_e4m3(u.w, f + 12);
}

// Prefill cache write. src [B][H][S][128] bf16 (K and V staging slabs of one layer) -> dst rows [b][h][t < len[b]] of
// [B][H][Smax][128] bytes and [B][H][Smax] scales. grid (ceil(S / 64), H, B), 256 threads: a half-warp owns one row (16 lanes
// x 16-byte loads), amax over its 16 lanes, one 8-byte store per lane; 4 rows of K and of V in flight per half-warp.
constexpr int KQ_TILE = 64;

__global__ void __launch_bounds__(256)
kv_quantize_e4m3_kernel(const __nv_bfloat16* __restrict__ ksrc, const __nv_bfloat16* __restrict__ vsrc,
                        uint8_t* __restrict__ k8, uint8_t* __restrict__ v8, float* __restrict__ kscale,
                        float* __restrict__ vscale, const int32_t* __restrict__ seq_lens, const int32_t* __restrict__ pos0,
                        int S, int S_src, int H, int Smax) {
    pdl_trigger();
    pdl_wait();  // the slabs are written by the upstream kernels, seq_lens by an earlier one
    const int head = blockIdx.y, b = blockIdx.z;
    const int hw = threadIdx.x >> 4, c = threadIdx.x & 15;
    // chunk rows t < len, stored at row p0 + t of the slab and of the cache (rows outside either are never touched)
    const int p0 = pos0 != nullptr ? pos0[b] : 0;
    const int len = min(seq_lens != nullptr ? min(seq_lens[b], S) : S, min(S_src, Smax) - p0);
    const int t0 = blockIdx.x * KQ_TILE + hw;
    const size_t src_row0 = ((size_t)b * H + head) * S_src + p0, dst_row0 = ((size_t)b * H + head) * Smax + p0;
    uint4 raw[2][4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
        const int t = t0 + u * 16;
        if (t < len) {
            raw[0][u] = ld_stream_16(ksrc + (src_row0 + t) * DA_D + c * 8);
            raw[1][u] = ld_stream_16(vsrc + (src_row0 + t) * DA_D + c * 8);
        }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
        const int t = t0 + u * 16;
        if (t >= len) continue;  // uniform across the half-warp (the shuffles below stay inside it)
#pragma unroll
        for (int kv = 0; kv < 2; ++kv) {
            const uint4 r = raw[kv][u];
            const float f[8] = {bf16_lo(r.x), bf16_hi(r.x), bf16_lo(r.y), bf16_hi(r.y),
                                bf16_lo(r.z), bf16_hi(r.z), bf16_lo(r.w), bf16_hi(r.w)};
            float amax = 0.f;
#pragma unroll
            for (int e = 0; e < 8; ++e) amax = fmaxf(amax, fabsf(f[e]));
            const unsigned mask = 0xffffu << (threadIdx.x & 16);
#pragma unroll
            for (int o = 8; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(mask, amax, o));
            const float inv = amax > 0.f ? kE4M3Max / amax : 1.0f;
            const uint2 q = make_uint2(pack4_e4m3(f[0] * inv, f[1] * inv, f[2] * inv, f[3] * inv),
                                       pack4_e4m3(f[4] * inv, f[5] * inv, f[6] * inv, f[7] * inv));
            *reinterpret_cast<uint2*>((kv == 0 ? k8 : v8) + (dst_row0 + t) * DA_D + c * 8) = q;
            if (c == 0) (kv == 0 ? kscale : vscale)[dst_row0 + t] = amax > 0.f ? amax / kE4M3Max : 1.0f;
        }
    }
}

// The stored prefix of a cache as bf16, for a prefill chunk that attends over it: rows t < pos0[b] of k8 / v8 [B][H][Smax][128]
// -> bf16(float(q) * scale) at row t of dst [B][H][S_dst][128]. grid (ceil(S_dst / 64), H, B), 256 threads: 16 lanes per
// row, 8 bytes in and 16 bytes out per lane.
__global__ void __launch_bounds__(256)
kv_dequantize_e4m3_kernel(const uint8_t* __restrict__ k8, const uint8_t* __restrict__ v8, const float* __restrict__ kscale,
                          const float* __restrict__ vscale, const int32_t* __restrict__ pos0, __nv_bfloat16* __restrict__ kdst,
                          __nv_bfloat16* __restrict__ vdst, int H, int Smax, int S_dst) {
    pdl_trigger();
    pdl_wait();
    const int head = blockIdx.y, b = blockIdx.z;
    const int hw = threadIdx.x >> 4, c = threadIdx.x & 15;
    const int n = min(pos0[b], min(Smax, S_dst));
    const size_t src_row0 = ((size_t)b * H + head) * Smax, dst_row0 = ((size_t)b * H + head) * S_dst;
#pragma unroll
    for (int u = 0; u < KQ_TILE / 16; ++u) {
        const int t = blockIdx.x * KQ_TILE + hw + u * 16;
        if (t >= n) break;
#pragma unroll
        for (int kv = 0; kv < 2; ++kv) {
            const uint2 q = *reinterpret_cast<const uint2*>((kv == 0 ? k8 : v8) + (src_row0 + t) * DA_D + c * 8);
            const float sc = (kv == 0 ? kscale : vscale)[src_row0 + t];
            float f[8];
            unpack4_e4m3(q.x, f);
            unpack4_e4m3(q.y, f + 4);
            *reinterpret_cast<uint4*>((kv == 0 ? kdst : vdst) + (dst_row0 + t) * DA_D + c * 8) =
                make_uint4(pack_bf16(f[0] * sc, f[1] * sc), pack_bf16(f[2] * sc, f[3] * sc),
                           pack_bf16(f[4] * sc, f[5] * sc), pack_bf16(f[6] * sc, f[7] * sc));
        }
    }
}

// Decode attention over an e4m3 cache: the contract of decode_attn_kernel (grid (nsplit, H, B), fixed grid, RoPE on q and
// the new k in-kernel, one CTA per (b, head) appends, self-resetting counters, same partial / merge scratch). A row is
// 128 bytes, so 8 lanes x 16-byte loads cover a key and the CTA's 16 lane groups take 4 consecutive keys each per pass
// (64 keys per pass); the 4 scales of a group are one 16-byte load. k_scale multiplies the score after the lane
// reduction and v_scale is folded into p: dequantisation costs one multiply per key. The appended row is quantised
// first and the step attends over the stored (dequantised) values, like every later step will.
constexpr int DA8_KEYS = 4;  // consecutive keys per lane group and pass

struct DecodeAttnE4m3Params {
    const __nv_bfloat16* qkv;
    uint8_t* k8;
    uint8_t* v8;
    float* kscale;
    float* vscale;
    const int32_t* cur_len;
    __nv_bfloat16* out;
    float* partial;
    int32_t* counters;
    int H, Smax, nsplit;
    float theta, scale_log2;
};

__global__ void __launch_bounds__(DA_THREADS) decode_attn_e4m3_kernel(DecodeAttnE4m3Params p) {
    const int split = blockIdx.x, head = blockIdx.y, b = blockIdx.z;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int grp = (warp << 2) | (lane >> 3);  // lane group 0..15
    const int c = lane & 7;                     // 16-element chunk of the head dim
    pdl_trigger();
    pdl_wait();                                 // qkv (previous GEMM) and cur_len (previous step) are upstream outputs
    const int pos = p.cur_len[b];
    const int total = pos + 1;
    const int hd = p.H * DA_D;

    __shared__ float s_q[DA_D];
    __shared__ float s_knew[DA_D];
    __shared__ __align__(16) uint8_t s_new8[2][DA_D];  // the appended row as stored: k bytes, v bytes
    __shared__ float s_newscale[2];
    __shared__ float s_red[2][4];
    __shared__ float s_m[16], s_l[16];
    __shared__ float s_o[16][DA_D];
    __shared__ int s_last;

    // key range of this split; multiples of DA8_KEYS so that a group's scale vector is 16-byte aligned
    int chunk = (total + p.nsplit - 1) / p.nsplit;
    chunk = (chunk + DA8_KEYS - 1) / DA8_KEYS * DA8_KEYS;
    const int k_begin = split * chunk;
    const int k_end = min(k_begin + chunk, total);
    const bool owns_new = (pos >= k_begin) && (pos < k_end);

    const __nv_bfloat16* qrow = p.qkv + (size_t)b * 3 * hd + head * DA_D;
    {   // RoPE on q (every CTA) and on the new k (the CTA that appends it)
        const __nv_bfloat16* krow = qrow + hd;
        const int i = tid & 63;
        float cs, sn;
        rope_cos_sin(pos, i, DA_D, p.theta, cs, sn);
        const float q1 = __bfloat162float(qrow[i]), q2 = __bfloat162float(qrow[i + 64]);
        if (tid < 64) s_q[i] = rope_apply(q1, -q2, cs, sn); else s_q[i + 64] = rope_apply(q2, q1, cs, sn);
        if (owns_new) {
            const float k1 = __bfloat162float(krow[i]), k2 = __bfloat162float(krow[i + 64]);
            if (tid < 64) s_knew[i] = rope_apply(k1, -k2, cs, sn); else s_knew[i + 64] = rope_apply(k2, k1, cs, sn);
        }
    }
    __syncthreads();

    const size_t rbase = ((size_t)b * p.H + head) * p.Smax;  // first row of this (b, head) slab
    if (owns_new) {
        // quantise and append the new token's k (roped) and v: thread tid owns element tid of both rows
        const float kx = s_knew[tid], vx = __bfloat162float(qrow[2 * hd + tid]);
        const float ka = warp_max(fabsf(kx)), va = warp_max(fabsf(vx));
        if (lane == 0) { s_red[0][warp] = ka; s_red[1][warp] = va; }
        __syncthreads();
        const float kamax = fmaxf(fmaxf(s_red[0][0], s_red[0][1]), fmaxf(s_red[0][2], s_red[0][3]));
        const float vamax = fmaxf(fmaxf(s_red[1][0], s_red[1][1]), fmaxf(s_red[1][2], s_red[1][3]));
        const float kinv = kamax > 0.f ? kE4M3Max / kamax : 1.0f, vinv = vamax > 0.f ? kE4M3Max / vamax : 1.0f;
        const uint8_t kq = (uint8_t)__nv_cvt_float_to_fp8(kx * kinv, __NV_SATFINITE, __NV_E4M3);
        const uint8_t vq = (uint8_t)__nv_cvt_float_to_fp8(vx * vinv, __NV_SATFINITE, __NV_E4M3);
        s_new8[0][tid] = kq; s_new8[1][tid] = vq;
        p.k8[(rbase + pos) * DA_D + tid] = kq;
        p.v8[(rbase + pos) * DA_D + tid] = vq;
        if (tid == 0) {
            const float ks = kamax > 0.f ? kamax / kE4M3Max : 1.0f, vs = vamax > 0.f ? vamax / kE4M3Max : 1.0f;
            s_newscale[0] = ks; s_newscale[1] = vs;
            p.kscale[rbase + pos] = ks; p.vscale[rbase + pos] = vs;
        }
        __syncthreads();
    }

    float qreg[16];
#pragma unroll
    for (int e = 0; e < 16; ++e) qreg[e] = s_q[c * 16 + e];

    float m_run = -INFINITY, l_run = 0.f;
    float acc[16];
#pragma unroll
    for (int e = 0; e < 16; ++e) acc[e] = 0.f;

    const uint8_t* kb = p.k8 + rbase * DA_D + c * 16;
    const uint8_t* vb = p.v8 + rbase * DA_D + c * 16;

    // trip count is CTA-uniform: the shuffles below use the full warp mask
    for (int kbase = k_begin; kbase < k_end; kbase += 16 * DA8_KEYS) {
        const int k0 = kbase + grp * DA8_KEYS;
        uint4 kraw[DA8_KEYS], vraw[DA8_KEYS];
        float4 ks4 = make_float4(0.f, 0.f, 0.f, 0.f), vs4 = ks4;
        if (k0 < k_end) {  // k0 % 4 == 0 and Smax % 4 == 0: aligned, and k0 + 3 stays inside the slab's Smax scales
            ks4 = __ldg(reinterpret_cast<const float4*>(p.kscale + rbase + k0));
            vs4 = __ldg(reinterpret_cast<const float4*>(p.vscale + rbase + k0));
        }
#pragma unroll
        for (int u = 0; u < DA8_KEYS; ++u) {
            const int key = k0 + u;
            if (key < k_end && key != pos) {
                kraw[u] = ld_stream_16(kb + (size_t)key * DA_D);
                vraw[u] = ld_stream_16(vb + (size_t)key * DA_D);
            } else {
                kraw[u] = make_uint4(0, 0, 0, 0);
                vraw[u] = make_uint4(0, 0, 0, 0);
            }
        }
        float ksc[DA8_KEYS] = {ks4.x, ks4.y, ks4.z, ks4.w}, vsc[DA8_KEYS] = {vs4.x, vs4.y, vs4.z, vs4.w};
        float sc[DA8_KEYS];
        float m_new = m_run;
#pragma unroll
        for (int u = 0; u < DA8_KEYS; ++u) {
            const int key = k0 + u;
            if (key >= k_end) { ksc[u] = 0.f; vsc[u] = 0.f; }  // whatever lies behind the range never reaches p * v_scale
            if (key == pos && owns_new) {  // the row appended above: bytes and scales from shared memory
                kraw[u] = *reinterpret_cast<const uint4*>(&s_new8[0][c * 16]);
                vraw[u] = *reinterpret_cast<const uint4*>(&s_new8[1][c * 16]);
                ksc[u] = s_newscale[0]; vsc[u] = s_newscale[1];
            }
            float kf[16];
            unpack16_e4m3(kraw[u], kf);
            float dot = 0.f;
#pragma unroll
            for (int e = 0; e < 16; ++e) dot += qreg[e] * kf[e];
            dot += __shfl_xor_sync(0xffffffffu, dot, 4);
            dot += __shfl_xor_sync(0xffffffffu, dot, 2);
            dot += __shfl_xor_sync(0xffffffffu, dot, 1);
            sc[u] = key < k_end ? dot * ksc[u] * p.scale_log2 : -INFINITY;
            m_new = fmaxf(m_new, sc[u]);
        }
        // one rescale of the accumulators per pass (4 keys)
        const float m_use = (m_new == -INFINITY) ? 0.f : m_new;
        const float corr = exp2f(m_run - m_use);  // m_run = -inf -> 0
        m_run = m_new;
        l_run *= corr;
#pragma unroll
        for (int e = 0; e < 16; ++e) acc[e] *= corr;
#pragma unroll
        for (int u = 0; u < DA8_KEYS; ++u) {
            const float pr = exp2f(sc[u] - m_use);  // invalid key: exp2(-inf) = 0
            l_run += pr;
            const float pv = pr * vsc[u];
            float vf[16];
            unpack16_e4m3(vraw[u], vf);
#pragma unroll
            for (int e = 0; e < 16; ++e) acc[e] += pv * vf[e];
        }
    }

    // ---- merge the 16 lane groups of this CTA ----
    if (c == 0) { s_m[grp] = m_run; s_l[grp] = l_run; }
#pragma unroll
    for (int e = 0; e < 16; ++e) s_o[grp][c * 16 + e] = acc[e];
    __syncthreads();
    float m_cta = -INFINITY;
#pragma unroll
    for (int i = 0; i < 16; ++i) m_cta = fmaxf(m_cta, s_m[i]);
    float l_cta = 0.f, o_cta = 0.f;  // thread tid owns output element tid
#pragma unroll
    for (int i = 0; i < 16; ++i) {
        const float w = (s_m[i] == -INFINITY) ? 0.f : exp2f(s_m[i] - m_cta);
        l_cta += s_l[i] * w;
        o_cta += s_o[i][tid] * w;
    }
    const int bh = b * p.H + head;
    float* part = p.partial + ((size_t)bh * p.nsplit + split) * (DA_D + 2);
    part[tid] = o_cta;
    if (tid == 0) { part[DA_D] = m_cta; part[DA_D + 1] = l_cta; }

    // ---- last CTA of this (b, head) merges the splits ----
    __threadfence();
    __syncthreads();
    if (tid == 0) {
        const int prev = atomicAdd(&p.counters[bh], 1);
        s_last = (prev == p.nsplit - 1) ? 1 : 0;
    }
    __syncthreads();
    if (s_last) {
        __threadfence();
        const float* pb = p.partial + (size_t)bh * p.nsplit * (DA_D + 2);
        float m_all = -INFINITY;
#pragma unroll 8
        for (int s = 0; s < p.nsplit; ++s) m_all = fmaxf(m_all, __ldcg(pb + (size_t)s * (DA_D + 2) + DA_D));
        float l_all = 0.f, o_all = 0.f;
#pragma unroll 8
        for (int s = 0; s < p.nsplit; ++s) {
            const float ms = __ldcg(pb + (size_t)s * (DA_D + 2) + DA_D);
            const float w = (ms == -INFINITY) ? 0.f : exp2f(ms - m_all);
            l_all += __ldcg(pb + (size_t)s * (DA_D + 2) + DA_D + 1) * w;
            o_all += __ldcg(pb + (size_t)s * (DA_D + 2) + tid) * w;
        }
        p.out[(size_t)b * hd + head * DA_D + tid] = __float2bfloat16_rn(o_all / l_all);
        if (tid == 0) p.counters[bh] = 0;  // self-reset for the next launch
    }
}

}  // namespace

int rope_table_build(void* table, int Smax, int D, float theta, cudaStream_t stream) {
    B2_CHECK_ARG(table != nullptr && Smax > 0 && D > 0 && D % 2 == 0, "rope_table_build: bad argument");
    const int n = Smax * (D / 2);
    rope_table_kernel<<<(n + 255) / 256, 256, 0, stream>>>(reinterpret_cast<uint32_t*>(table), Smax, D, theta);
    B2_LAUNCH_CHECK();
    return 0;
}

int rope_kv_write(void* qkv, void* kcache, void* vcache, int B, int S, int H, int D, int Smax, float theta,
                  cudaStream_t stream, const int32_t* pos0) {
    B2_CHECK_ARG(pos0 != nullptr || S <= Smax, "rope_kv_write: S=%d exceeds cache capacity %d", S, Smax);
    B2_CHECK_ARG(D % 16 == 0 && D <= 256, "rope_kv_write: head_dim must be a multiple of 16, <= 256 (got %d)", D);
    B2_CHECK_ARG(((reinterpret_cast<uintptr_t>(qkv) | reinterpret_cast<uintptr_t>(kcache) |
                   reinterpret_cast<uintptr_t>(vcache)) & 15) == 0, "rope_kv_write: buffers must be 16-byte aligned");
    B2_CUDA_CHECK(launch_pdl(rope_kv_write_kernel, dim3(B * S), dim3(256), 0, stream, reinterpret_cast<__nv_bfloat16*>(qkv),
                             reinterpret_cast<__nv_bfloat16*>(kcache), reinterpret_cast<__nv_bfloat16*>(vcache), pos0, S, H, D, Smax, theta));
    B2_LAUNCH_CHECK();
    return 0;
}

// resident CTAs of decode_attn_kernel per SM (register-limited: 79 registers x 128 threads -> 6), for the split heuristic
int decode_attn_ctas_per_sm() {
    static int occ = 0;
    if (occ == 0) {
        int n = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, decode_attn_kernel, DA_THREADS, 0) != cudaSuccess || n < 1) n = 6;
        occ = n;
    }
    return occ;
}

int decode_attn_bf16(const DecodeAttnArgs& a, cudaStream_t stream) {
    B2_CHECK_ARG(a.D == DA_D, "decode_attn: head_dim must be 128 (got %d)", a.D);
    B2_CHECK_ARG(a.nsplit >= 1 && a.B > 0 && a.H > 0, "decode_attn: bad launch shape");
    DecodeAttnParams p;
    p.qkv = reinterpret_cast<const __nv_bfloat16*>(a.qkv);
    p.kcache = reinterpret_cast<__nv_bfloat16*>(a.kcache);
    p.vcache = reinterpret_cast<__nv_bfloat16*>(a.vcache);
    p.cur_len = a.cur_len;
    p.out = reinterpret_cast<__nv_bfloat16*>(a.out);
    p.partial = a.partial;
    p.counters = a.counters;
    p.H = a.H; p.Smax = a.Smax; p.nsplit = a.nsplit;
    p.theta = a.theta;
    p.scale_log2 = a.scale * 1.4426950408889634f;
    dim3 grid(a.nsplit, a.H, a.B);
    B2_CUDA_CHECK(launch_pdl(decode_attn_kernel, grid, dim3(DA_THREADS), 0, stream, p));
    B2_LAUNCH_CHECK();
    return 0;
}

// resident CTAs of decode_attn_mq_kernel per SM (shared-memory-limited: 74 KB of K / V tiles per CTA), for the split heuristic
int decode_attn_mq_ctas_per_sm() {
    static int occ = 0;
    if (occ == 0) {
        int n = 0;
        if (cudaFuncSetAttribute(decode_attn_mq_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)MQ_SMEM) != cudaSuccess ||
            cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, decode_attn_mq_kernel, 128, MQ_SMEM) != cudaSuccess || n < 1) {
            cudaGetLastError();
            n = 3;
        }
        occ = n;
    }
    return occ;
}

size_t decode_attn_mq_scratch_bytes(int B, int H, int nsplit) {
    return (size_t)B * H * nsplit * MQ_ROWS * (DA_D + 2) * sizeof(float) + (size_t)B * H * sizeof(int32_t);
}

int decode_attn_mq_bf16(const DecodeAttnArgs& a, cudaStream_t stream) {
    B2_CHECK_ARG(a.D == DA_D, "decode_attn_mq: head_dim must be 128 (got %d)", a.D);
    B2_CHECK_ARG(a.R >= 1 && a.R <= MQ_ROWS, "decode_attn_mq: %d query rows (1..%d)", a.R, MQ_ROWS);
    B2_CHECK_ARG(a.nsplit >= 1 && a.B > 0 && a.H > 0, "decode_attn_mq: bad launch shape");
    B2_CHECK_ARG(((reinterpret_cast<uintptr_t>(a.qkv) | reinterpret_cast<uintptr_t>(a.kcache) |
                   reinterpret_cast<uintptr_t>(a.vcache)) & 15) == 0, "decode_attn_mq: buffers must be 16-byte aligned");
    decode_attn_mq_ctas_per_sm();  // sets the dynamic shared-memory attribute
    DecodeAttnMqParams p;
    p.qkv = reinterpret_cast<const __nv_bfloat16*>(a.qkv);
    p.kcache = reinterpret_cast<const __nv_bfloat16*>(a.kcache);
    p.vcache = reinterpret_cast<const __nv_bfloat16*>(a.vcache);
    p.cur_len = a.cur_len;
    p.out = reinterpret_cast<__nv_bfloat16*>(a.out);
    p.partial = a.partial;
    p.counters = a.counters;
    p.R = a.R; p.H = a.H; p.Smax = a.Smax; p.nsplit = a.nsplit;
    p.scale_log2 = a.scale * 1.4426950408889634f;
    B2_CUDA_CHECK(launch_pdl(decode_attn_mq_kernel, dim3(a.nsplit, a.H, a.B), dim3(128), MQ_SMEM, stream, p));
    B2_LAUNCH_CHECK();
    return 0;
}

// resident CTAs of decode_attn_shared_kernel per SM (shared-memory-limited like decode_attn_mq_kernel), for the split heuristic
int decode_attn_shared_ctas_per_sm() {
    static int occ = 0;
    if (occ == 0) {
        int n = 0;
        if (cudaFuncSetAttribute(decode_attn_shared_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SH_SMEM) != cudaSuccess ||
            cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, decode_attn_shared_kernel, 128, SH_SMEM) != cudaSuccess || n < 1) {
            cudaGetLastError();
            n = 3;
        }
        occ = n;
    }
    return occ;
}

size_t decode_attn_shared_scratch_bytes(int B, int H, int nsplit) {
    return (size_t)B * H * 2 * nsplit * (DA_D + 2) * sizeof(float) + (size_t)B * H * sizeof(int32_t);
}

int decode_attn_shared_bf16(const DecodeAttnArgs& a, const PrefixGroup* groups, const int32_t* row_prefix, int G,
                            cudaStream_t stream) {
    B2_CHECK_ARG(a.D == DA_D, "decode_attn_shared: head_dim must be 128 (got %d)", a.D);
    B2_CHECK_ARG(a.nsplit >= 1 && a.B > 0 && a.H > 0 && G >= 0 && G <= a.B, "decode_attn_shared: bad launch shape");
    B2_CHECK_ARG(G == 0 || (groups != nullptr && row_prefix != nullptr), "decode_attn_shared: null group table");
    B2_CHECK_ARG(((reinterpret_cast<uintptr_t>(a.qkv) | reinterpret_cast<uintptr_t>(a.kcache) |
                   reinterpret_cast<uintptr_t>(a.vcache)) & 15) == 0, "decode_attn_shared: buffers must be 16-byte aligned");
    decode_attn_shared_ctas_per_sm();  // sets the dynamic shared-memory attribute
    DecodeAttnSharedParams p;
    p.qkv = reinterpret_cast<const __nv_bfloat16*>(a.qkv);
    p.kcache = reinterpret_cast<__nv_bfloat16*>(a.kcache);
    p.vcache = reinterpret_cast<__nv_bfloat16*>(a.vcache);
    p.cur_len = a.cur_len;
    p.groups = groups;
    p.row_prefix = row_prefix;
    p.out = reinterpret_cast<__nv_bfloat16*>(a.out);
    p.partial = a.partial;
    p.counters = a.counters;
    p.G = G; p.H = a.H; p.Smax = a.Smax; p.nsplit = a.nsplit;
    p.theta = a.theta;
    p.scale_log2 = a.scale * 1.4426950408889634f;
    B2_CUDA_CHECK(launch_pdl(decode_attn_shared_kernel, dim3(a.nsplit, a.H, G + a.B), dim3(128), SH_SMEM, stream, p));
    B2_LAUNCH_CHECK();
    return 0;
}

int decode_attn_e4m3_ctas_per_sm() {
    static int occ = 0;
    if (occ == 0) {
        int n = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, decode_attn_e4m3_kernel, DA_THREADS, 0) != cudaSuccess || n < 1) n = 4;
        occ = n;
    }
    return occ;
}

int decode_attn_e4m3(const DecodeAttnArgs& a, cudaStream_t stream) {
    B2_CHECK_ARG(a.D == DA_D, "decode_attn_e4m3: head_dim must be 128 (got %d)", a.D);
    B2_CHECK_ARG(a.nsplit >= 1 && a.B > 0 && a.H > 0, "decode_attn_e4m3: bad launch shape");
    B2_CHECK_ARG(a.kscale != nullptr && a.vscale != nullptr, "decode_attn_e4m3: null scale array");
    B2_CHECK_ARG(a.Smax > 0 && a.Smax % DA8_KEYS == 0, "decode_attn_e4m3: Smax must be a multiple of %d (got %d)", DA8_KEYS, a.Smax);
    B2_CHECK_ARG(((reinterpret_cast<uintptr_t>(a.kcache) | reinterpret_cast<uintptr_t>(a.vcache) |
                   reinterpret_cast<uintptr_t>(a.kscale) | reinterpret_cast<uintptr_t>(a.vscale)) & 15) == 0,
                 "decode_attn_e4m3: caches and scales must be 16-byte aligned");
    DecodeAttnE4m3Params p;
    p.qkv = reinterpret_cast<const __nv_bfloat16*>(a.qkv);
    p.k8 = reinterpret_cast<uint8_t*>(a.kcache);
    p.v8 = reinterpret_cast<uint8_t*>(a.vcache);
    p.kscale = a.kscale; p.vscale = a.vscale;
    p.cur_len = a.cur_len;
    p.out = reinterpret_cast<__nv_bfloat16*>(a.out);
    p.partial = a.partial;
    p.counters = a.counters;
    p.H = a.H; p.Smax = a.Smax; p.nsplit = a.nsplit;
    p.theta = a.theta;
    p.scale_log2 = a.scale * 1.4426950408889634f;
    dim3 grid(a.nsplit, a.H, a.B);
    B2_CUDA_CHECK(launch_pdl(decode_attn_e4m3_kernel, grid, dim3(DA_THREADS), 0, stream, p));
    B2_LAUNCH_CHECK();
    return 0;
}

int kv_quantize_e4m3(const void* ksrc, const void* vsrc, void* k8, void* v8, float* kscale, float* vscale,
                     const int32_t* seq_lens, int B, int S, int H, int D, int Smax, cudaStream_t stream, const int32_t* pos0,
                     int S_src) {
    if (S_src == 0) S_src = S;
    B2_CHECK_ARG(D == DA_D, "kv_quantize_e4m3: head_dim must be 128 (got %d)", D);
    B2_CHECK_ARG(B > 0 && H > 0 && S > 0 && (pos0 != nullptr || (S <= Smax && S_src == S)),
                 "kv_quantize_e4m3: B=%d H=%d S=%d S_src=%d Smax=%d", B, H, S, S_src, Smax);
    B2_CHECK_ARG(((reinterpret_cast<uintptr_t>(ksrc) | reinterpret_cast<uintptr_t>(vsrc)) & 15) == 0 &&
                 ((reinterpret_cast<uintptr_t>(k8) | reinterpret_cast<uintptr_t>(v8)) & 7) == 0,
                 "kv_quantize_e4m3: slabs must be 16-byte and caches 8-byte aligned");
    dim3 grid((S + KQ_TILE - 1) / KQ_TILE, H, B);
    B2_CUDA_CHECK(launch_pdl(kv_quantize_e4m3_kernel, grid, dim3(256), 0, stream, reinterpret_cast<const __nv_bfloat16*>(ksrc),
                             reinterpret_cast<const __nv_bfloat16*>(vsrc), reinterpret_cast<uint8_t*>(k8),
                             reinterpret_cast<uint8_t*>(v8), kscale, vscale, seq_lens, pos0, S, S_src, H, Smax));
    B2_LAUNCH_CHECK();
    return 0;
}

int kv_dequantize_e4m3(const void* k8, const void* v8, const float* kscale, const float* vscale, const int32_t* pos0, void* kdst,
                       void* vdst, int B, int H, int Smax, int S_dst, cudaStream_t stream) {
    B2_CHECK_ARG(k8 && v8 && kscale && vscale && pos0 && kdst && vdst, "kv_dequantize_e4m3: null argument");
    B2_CHECK_ARG(B > 0 && H > 0 && Smax > 0 && S_dst > 0, "kv_dequantize_e4m3: B=%d H=%d Smax=%d S_dst=%d", B, H, Smax, S_dst);
    B2_CHECK_ARG(((reinterpret_cast<uintptr_t>(k8) | reinterpret_cast<uintptr_t>(v8)) & 7) == 0 &&
                 ((reinterpret_cast<uintptr_t>(kdst) | reinterpret_cast<uintptr_t>(vdst)) & 15) == 0,
                 "kv_dequantize_e4m3: caches must be 8-byte and slabs 16-byte aligned");
    dim3 grid((S_dst + KQ_TILE - 1) / KQ_TILE, H, B);
    B2_CUDA_CHECK(launch_pdl(kv_dequantize_e4m3_kernel, grid, dim3(256), 0, stream, reinterpret_cast<const uint8_t*>(k8),
                             reinterpret_cast<const uint8_t*>(v8), kscale, vscale, pos0, reinterpret_cast<__nv_bfloat16*>(kdst),
                             reinterpret_cast<__nv_bfloat16*>(vdst), H, Smax, S_dst));
    B2_LAUNCH_CHECK();
    return 0;
}

}  // namespace b2
