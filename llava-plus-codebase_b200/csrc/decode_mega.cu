// Persistent decode-step megakernel (batch <= 2): ONE cooperative launch per generated token.
//
// The one-token decode step of LLaVA/LLaMA (reference: the HF one-token forward behind
// llava/model/llava_arch.py:103-112; transformers modeling_llama.py:303-332 per layer) is a pure weight
// stream: 13.2 GB (7B) read once per token, through 5 dependent phases per layer
//     embed -> L x { QKV gemv (+RMSNorm) | RoPE + KV append + split-KV attention | o_proj gemv (+res) |
//                    gate/up gemv (+RMSNorm, SwiGLU) | down gemv (+res) } -> lm_head gemv (+RMSNorm) -> argmax.
// Every phase boundary is an all-to-all dependency (each SM needs the whole activation vector), i.e. a grid
// barrier plus a short prologue/epilogue: ~7 us of latency 161 times per token if the memory pipe drains there
// Weights, however, do not depend on activations. So each CTA
// runs a decoupled PRODUCER warp that walks the weight tiles of ALL phases in order and streams them with TMA
// bulk copies (cp.async.bulk + mbarrier complete_tx) into a ~170 KB shared-memory ring, never waiting for a
// barrier — only for a free ring slot. The 16 CONSUMER warps do the dependent work (activation staging + fused
// RMSNorm, tensor-core dot products straight out of the ring, reductions, epilogues, attention, grid barriers);
// while they sit in a dependency the producer keeps HBM busy filling the ring for the next phase.
//
// Consumer math: mma.sync.m16n8k16 (bf16 x bf16 -> fp32) with the activations as the A operand (rows = batch,
// zero padded to 16) and 8 weight rows as the B operand; one 16-byte LDS per lane feeds two MMAs without any
// unpacking because the k index is permuted consistently on both operands (a dot product does not care).
// Activations that cross a grid barrier are read with ld.global.cg (L1 is not coherent between SMs).
#include <limits.h>
#include <math.h>

#include "common.cuh"
#include "kernels.h"

namespace b2 {
namespace {

constexpr int MK_CONS_WARPS = 16;
constexpr int MK_CONS = MK_CONS_WARPS * 32;   // 512 consumer threads
constexpr int MK_PROD_WARPS = 4;              // TMA issue is per-thread work: tiles are dealt round-robin to 4 producer warps
constexpr int MK_THREADS = MK_CONS + 32 * MK_PROD_WARPS;
constexpr int MK_D = 128;
constexpr int MK_U = 4;                       // keys per half-warp per attention iteration
constexpr int MK_KT = 2048;                   // K elements per weight tile (8 rows x 2048 bf16 = 32 KB): per-tile mbarrier
                                              // wait/arrive overhead of the 16 consumer warps is amortised over 4 k32 slices each
constexpr int MK_ROW_PAD = 64;                // bytes of padding per tile row -> conflict-free 16 B fragment loads
constexpr int MK_ROW_STRIDE = MK_KT * 2 + MK_ROW_PAD;
constexpr int MK_TILE_BYTES = 8 * MK_ROW_STRIDE;
constexpr int MK_MAXNB = 32;                  // max 8-row blocks per CTA per phase (host-checked)
constexpr int MK_MAXL = 48;                   // decoder layers whose weight-pointer table is cached in smem
constexpr int MK_MAX_STAGES = 12;

__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
    f[0] = bf16_lo(u.x); f[1] = bf16_hi(u.x); f[2] = bf16_lo(u.y); f[3] = bf16_hi(u.y);
    f[4] = bf16_lo(u.z); f[5] = bf16_hi(u.z); f[6] = bf16_lo(u.w); f[7] = bf16_hi(u.w);
}
__device__ __forceinline__ uint4 ldcg16(const void* p) { return __ldcg(reinterpret_cast<const uint4*>(p)); }

// consumer-only CTA barrier (the producer warp never joins it)
__device__ __forceinline__ void cons_sync() { asm volatile("bar.sync 1, %0;" ::"n"(MK_CONS) : "memory"); }

// Grid barrier over the consumer halves of all CTAs (co-resident: cooperative launch, grid = #SMs). One
// monotonically increasing counter: fire-and-forget red.release (+1), then ld.acquire polling until the value
// implied by the host-provided launch sequence number is reached. Signed compare survives 32-bit wrap-around.
__device__ __forceinline__ void grid_sync(unsigned int* counter, unsigned int target) {
    cons_sync();
    if (threadIdx.x == 0) {
        asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(counter) : "memory");
        unsigned int cur, spins = 0;
        do {
            asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(cur) : "l"(counter) : "memory");
            if (++spins > (1u << 26)) asm volatile("trap;");  // protocol bug -> CUDA error, not a hang
        } while ((int)(cur - target) < 0);
    }
    cons_sync();
}

// 1-D TMA bulk copy global -> shared, completion (bytes) signalled on an mbarrier
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// One GEMV phase as seen by a CTA. Output units (rows; SwiGLU: channels = a gate row + its up row) are cut into
// gridDim.x contiguous ranges that differ by at most ONE unit, so every SM streams the same number of bytes to
// within 1-4% (a split in whole 8-row blocks left +-1 block = 6-16% skew per phase in front of every grid barrier:
// The range is walked in MMA-sized blocks of 8 rows (SwiGLU: 4 gate rows +
// the 4 up rows of the same channels); the last block may be partial — its missing rows are simply not fetched.
struct GemvCtx {
    const __nv_bfloat16* W;
    int K, act;
    int u_lo, nu;   // first output unit (row / channel) and number of units owned by this CTA
    int nb;         // blocks: ceil(nu / 8) (SwiGLU: ceil(nu / 4))
    int nchunk;     // K tiles per block
};
// cold per-phase I/O, recomputed from the phase index where needed (prologue, epilogue)
struct PhaseIO {
    const __nv_bfloat16* xin;
    const __nv_bfloat16* gamma;
    const __nv_bfloat16* residual;
    void* out;
    int ld_out, out_fp32;
};

// physical weight row of lane-group g (0..7) of the CTA's local block `rb`; `valid` = the row exists in this CTA's range
__device__ __forceinline__ int mk_phys_row(const GemvCtx& c, int rb, int g, bool& valid) {
    if (c.act == ACT_SWIGLU) {  // block-64 interleaved gate/up: g<4 -> gate of local channel 4*rb+g, g>=4 -> its up row
        const int lc = rb * 4 + (g & 3);
        valid = lc < c.nu;
        const int ch = c.u_lo + lc;
        return (ch >> 6) * 128 + (ch & 63) + ((g >> 2) ? 64 : 0);
    }
    const int lr = rb * 8 + g;
    valid = lr < c.nu;
    return c.u_lo + lr;
}

// rows actually fetched for local block rb (8, or fewer for the partial last block)
__device__ __forceinline__ int mk_rows_in_block(const GemvCtx& c, int rb) {
    if (c.act == ACT_SWIGLU) return 2 * min(4, c.nu - rb * 4);
    return min(8, c.nu - rb * 8);
}

// phase k of layer l (k: 0 = QKV, 1 = attention, 2 = o_proj, 3 = gate/up, 4 = down); index 5L = lm_head
__device__ __forceinline__ bool mk_is_attention(const MegaParams& p, int ph) { return ph % 5 == 1 && ph < 5 * p.L; }

__device__ __forceinline__ PhaseIO mk_phase_io(const MegaParams& p, const MegaLayer* layers, int ph) {
    PhaseIO c;
    const int l = ph / 5, k = ph % 5;
    c.gamma = nullptr; c.residual = nullptr; c.out_fp32 = 0;
    if (l >= p.L) { c.xin = p.x; c.gamma = p.final_norm; c.out = p.logits; c.ld_out = p.V; c.out_fp32 = 1; }
    else if (k <= 1) { c.xin = p.x; c.gamma = layers[l].ln1; c.out = p.qkv; c.ld_out = 3 * p.h; }
    else if (k == 2) { c.xin = p.attn; c.residual = p.x; c.out = p.x; c.ld_out = p.h; }
    else if (k == 3) { c.xin = p.x; c.gamma = layers[l].ln2; c.out = p.act; c.ld_out = p.I; }
    else { c.xin = p.act; c.residual = p.x; c.out = p.x; c.ld_out = p.h; }
    return c;
}
__device__ __forceinline__ GemvCtx mk_phase_ctx(const MegaParams& p, const MegaLayer* layers, int ph) {
    GemvCtx c;
    const int l = ph / 5, k = ph % 5;
    int N;
    c.act = ACT_NONE;
    if (l >= p.L) { c.W = p.lm_head; N = p.V; c.K = p.h; }
    else if (k <= 1) { c.W = layers[l].wqkv; N = 3 * p.h; c.K = p.h; }
    else if (k == 2) { c.W = layers[l].wo; N = p.h; c.K = p.h; }
    else if (k == 3) { c.W = layers[l].wgu; N = 2 * p.I; c.K = p.h; c.act = ACT_SWIGLU; }
    else { c.W = layers[l].wd; N = p.h; c.K = p.I; }
    const long long units = c.act == ACT_SWIGLU ? (N >> 1) : N;
    c.u_lo = (int)((units * blockIdx.x) / gridDim.x);
    c.nu = (int)((units * (blockIdx.x + 1)) / gridDim.x) - c.u_lo;
    c.nb = c.act == ACT_SWIGLU ? (c.nu + 3) >> 2 : (c.nu + 7) >> 3;
    c.nchunk = (c.K + MK_KT - 1) / MK_KT;
    return c;
}

// x -> smem (bf16), optional RMSNorm (HF semantics: gamma * bf16(x * rstd)); consumer threads only
template <int NB>
__device__ __forceinline__ void mk_prologue(const PhaseIO& c, int K, int B, float eps, int tid, int lane, int warp,
                                            __nv_bfloat16* xs, float (*s_red)[NB], float* s_rstd,
                                            const __nv_bfloat16* gamma_smem) {
    const int nvec = K >> 3;
    float ss[NB];
#pragma unroll
    for (int b = 0; b < NB; ++b) ss[b] = 0.f;
    for (int i = tid; i < nvec; i += MK_CONS) {
#pragma unroll
        for (int b = 0; b < NB; ++b) {
            uint4 u = make_uint4(0, 0, 0, 0);
            if (b < B) u = ldcg16(c.xin + (size_t)b * K + i * 8);
            *reinterpret_cast<uint4*>(xs + (size_t)b * K + i * 8) = u;
            if (c.gamma != nullptr) {
                float f[8];
                unpack8(u, f);
#pragma unroll
                for (int e = 0; e < 8; ++e) ss[b] += f[e] * f[e];
            }
        }
    }
    if (c.gamma != nullptr) {
#pragma unroll
        for (int b = 0; b < NB; ++b) {
            const float v = warp_sum(ss[b]);
            if (lane == 0) s_red[warp][b] = v;
        }
        cons_sync();
        if (tid < NB) {
            float t = 0.f;
            for (int i = 0; i < MK_CONS_WARPS; ++i) t += s_red[i][tid];
            s_rstd[tid] = rsqrtf(t / K + eps);
        }
        cons_sync();
        // staged copy: thread t copied exactly the 16-byte chunks t, t + 512, ... it reads below, so its own wait is enough
        if (gamma_smem != nullptr) asm volatile("cp.async.wait_all;" ::: "memory");
        const __nv_bfloat16* gsrc = gamma_smem != nullptr ? gamma_smem : c.gamma;
        for (int i = tid; i < nvec; i += MK_CONS) {
            float gf[8];
            unpack8(*reinterpret_cast<const uint4*>(gsrc + i * 8), gf);
#pragma unroll
            for (int b = 0; b < NB; ++b) {
                uint4* px = reinterpret_cast<uint4*>(xs + (size_t)b * K + i * 8);
                float f[8], o[8];
                unpack8(*px, f);
                const float rstd = s_rstd[b];
#pragma unroll
                for (int e = 0; e < 8; ++e) o[e] = gf[e] * round_bf16(f[e] * rstd);
                *px = make_uint4(pack_bf16(o[0], o[1]), pack_bf16(o[2], o[3]), pack_bf16(o[4], o[5]),
                                 pack_bf16(o[6], o[7]));
            }
        }
    }
    cons_sync();
}

__device__ __forceinline__ void mk_mma(float (&c)[4], uint32_t a0, uint32_t a2, uint32_t b0, uint32_t b1) {
    // A rows 8..15 (a1, a3) are the zero padding of the batch dimension
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a0), "r"(0u), "r"(a2), "r"(0u), "r"(b0), "r"(b1));
}

// s_gpart layout: [warp][block][b][8 rows] fp32 (each consumer warp owns interleaved 32-element K slices)
template <int NB>
__device__ __forceinline__ float mk_row_value(const float* s_gpart, int rb, int b, int r) {
    float v = 0.f;
#pragma unroll
    for (int ww = 0; ww < MK_CONS_WARPS; ++ww) v += s_gpart[(((size_t)ww * MK_MAXNB + rb) * NB + b) * 8 + r];  // fixed order
    return v;
}

// after the streaming loop: reduce the 16 K-slices, apply the epilogue, coalesced global writes
template <int NB>
__device__ __forceinline__ void mk_epilogue(const MegaParams& p, const MegaLayer* layers, int ph, const GemvCtx& c,
                                            int B, int tid, const float* s_gpart, float res_pref, bool have_res_pref) {
    const PhaseIO io = mk_phase_io(p, layers, ph);
    if (c.act == ACT_SWIGLU) {
        const int nch = c.nu;
        for (int idx = tid; idx < nch * B; idx += MK_CONS) {
            const int b = idx / nch, r = idx - b * nch;
            const int rb = r >> 2, q = r & 3;
            const float gt = mk_row_value<NB>(s_gpart, rb, b, q);
            const float up = mk_row_value<NB>(s_gpart, rb, b, q + 4);
            reinterpret_cast<__nv_bfloat16*>(io.out)[(size_t)b * io.ld_out + (size_t)c.u_lo + r] =
                __float2bfloat16_rn(gt / (1.0f + __expf(-gt)) * up);
        }
    } else {
        const int nr = c.nu;
        for (int idx = tid; idx < nr * B; idx += MK_CONS) {
            const int b = idx / nr, r = idx - b * nr;
            float y = mk_row_value<NB>(s_gpart, r >> 3, b, r & 7);
            const size_t o = (size_t)b * io.ld_out + (size_t)c.u_lo + r;
            if (io.residual != nullptr) y += have_res_pref ? res_pref : __bfloat162float(__ldcg(io.residual + o));
            if (io.out_fp32) reinterpret_cast<float*>(io.out)[o] = y;
            else reinterpret_cast<__nv_bfloat16*>(io.out)[o] = __float2bfloat16_rn(y);
        }
    }
}

// RoPE + cache append + split-KV attention (consumer warps).
// (b, head) pairs are spread over the grid: with pairs <= #CTAs, G = #CTAs / pairs CTAs share one pair (split-KV
// across CTAs, merged by the last CTA to arrive — only G partials, G = 4 at B = 1); otherwise each CTA walks
// pairs one after the other. Inside a CTA the 16 warps split the key range (half-warp per 256 B K/V row,
// online softmax in registers) and merge through shared memory, so no long serial merge sits on the critical path.
__device__ __forceinline__ void mk_attention(const MegaParams& p, const MegaLayer& Lw, int tid, int lane, int warp,
                                             float (*s_part)[MK_D + 2], int* s_flag, const float* s_cos,
                                             const float* s_sin) {
    const int h = p.h, H = p.H;
    const int pairs = p.B * H;
    const int grid = gridDim.x;
    const int G = pairs <= grid ? grid / pairs : 1;
    const int hw = lane >> 4, c = lane & 15;
    const int split = pairs <= grid ? (int)blockIdx.x % G : 0;
    for (int pair = pairs <= grid ? (int)blockIdx.x / G : (int)blockIdx.x; pair < pairs;
         pair += (pairs <= grid ? pairs : grid)) {  // CTA-uniform loop
        const int head = pair % H, b = pair / H;
        const int pos = p.cur_len[b];
        const int total = pos + 1;
        const int cchunk = (total + G - 1) / G;
        const int cb = split * cchunk;
        const int ce = min(cb + cchunk, total);
        const int wchunk = (max(ce - cb, 0) + MK_CONS_WARPS - 1) / MK_CONS_WARPS;
        const int k_begin = cb + warp * wchunk;
        const int k_end = min(k_begin + wchunk, ce);
        const __nv_bfloat16* qrow = p.qkv + (size_t)b * 3 * h + head * MK_D;
        float qreg[8], knew[8], vnew[8];
        {
            // RoPE: element i pairs with i+64 -> chunk c pairs with chunk c^8
            float qa[8], qb[8], ka[8], kb[8];
            unpack8(ldcg16(qrow + c * 8), qa);
            unpack8(ldcg16(qrow + (c ^ 8) * 8), qb);
            unpack8(ldcg16(qrow + h + c * 8), ka);
            unpack8(ldcg16(qrow + h + (c ^ 8) * 8), kb);
            unpack8(ldcg16(qrow + 2 * h + c * 8), vnew);
            const float sign = (c < 8) ? -1.f : 1.f;
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const int i = ((c & 7) * 8 + e);  // frequency index 0..63; cos/sin(pos_b * inv_freq_i) tabulated once per step
                const float cbf = s_cos[b * 64 + i], sbf = s_sin[b * 64 + i];
                qreg[e] = round_bf16(round_bf16(qa[e] * cbf) + round_bf16(sign * qb[e] * sbf));
                knew[e] = round_bf16(round_bf16(ka[e] * cbf) + round_bf16(sign * kb[e] * sbf));
            }
        }
        const size_t cbase = ((size_t)b * H + head) * p.Smax * MK_D;
        if (pos >= k_begin && pos < k_end && hw == 0) {  // append (one half-warp writes the 256 B rows)
            *reinterpret_cast<uint4*>(Lw.kcache + cbase + (size_t)pos * MK_D + c * 8) =
                make_uint4(pack_bf16(knew[0], knew[1]), pack_bf16(knew[2], knew[3]),
                           pack_bf16(knew[4], knew[5]), pack_bf16(knew[6], knew[7]));
            *reinterpret_cast<uint4*>(Lw.vcache + cbase + (size_t)pos * MK_D + c * 8) =
                make_uint4(pack_bf16(vnew[0], vnew[1]), pack_bf16(vnew[2], vnew[3]),
                           pack_bf16(vnew[4], vnew[5]), pack_bf16(vnew[6], vnew[7]));
        }
        float m_run = -INFINITY, l_run = 0.f, av[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) av[e] = 0.f;
        const __nv_bfloat16* kb_ = Lw.kcache + cbase + c * 8;
        const __nv_bfloat16* vb_ = Lw.vcache + cbase + c * 8;
        for (int kbase = k_begin; kbase < k_end; kbase += 2 * MK_U) {  // warp-uniform trip count
            uint4 kraw[MK_U], vraw[MK_U];
#pragma unroll
            for (int u = 0; u < MK_U; ++u) {
                const int key = kbase + hw + 2 * u;
                if (key < k_end && key != pos) {
                    kraw[u] = ld_stream_16(kb_ + (size_t)key * MK_D);
                    vraw[u] = ld_stream_16(vb_ + (size_t)key * MK_D);
                } else {
                    kraw[u] = make_uint4(0, 0, 0, 0);
                    vraw[u] = make_uint4(0, 0, 0, 0);
                }
            }
#pragma unroll
            for (int u = 0; u < MK_U; ++u) {
                const int key = kbase + hw + 2 * u;
                float kf[8], vf[8];
                unpack8(kraw[u], kf);
                unpack8(vraw[u], vf);
                if (key == pos) {
#pragma unroll
                    for (int e = 0; e < 8; ++e) { kf[e] = knew[e]; vf[e] = vnew[e]; }
                }
                float dot = 0.f;
#pragma unroll
                for (int e = 0; e < 8; ++e) dot += qreg[e] * kf[e];
                dot += __shfl_xor_sync(0xffffffffu, dot, 8);
                dot += __shfl_xor_sync(0xffffffffu, dot, 4);
                dot += __shfl_xor_sync(0xffffffffu, dot, 2);
                dot += __shfl_xor_sync(0xffffffffu, dot, 1);
                if (key < k_end) {
                    const float sc = dot * p.scale_log2;
                    const float m_new = fmaxf(m_run, sc);
                    const float corr = exp2f(m_run - m_new);
                    const float pr = exp2f(sc - m_new);
                    l_run = l_run * corr + pr;
#pragma unroll
                    for (int e = 0; e < 8; ++e) av[e] = av[e] * corr + pr * vf[e];
                    m_run = m_new;
                }
            }
        }
        {   // merge the two half-warps
            const float m_o = __shfl_xor_sync(0xffffffffu, m_run, 16);
            const float l_o = __shfl_xor_sync(0xffffffffu, l_run, 16);
            const float m_c = fmaxf(m_run, m_o);
            const float w_s = (m_run == -INFINITY) ? 0.f : exp2f(m_run - m_c);
            const float w_o = (m_o == -INFINITY) ? 0.f : exp2f(m_o - m_c);
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const float a_o = __shfl_xor_sync(0xffffffffu, av[e], 16);
                av[e] = av[e] * w_s + a_o * w_o;
            }
            l_run = l_run * w_s + l_o * w_o;
            m_run = m_c;
        }
        if (hw == 0) {
#pragma unroll
            for (int e = 0; e < 8; ++e) s_part[warp][c * 8 + e] = av[e];
            if (c == 0) { s_part[warp][MK_D] = m_run; s_part[warp][MK_D + 1] = l_run; }
        }
        cons_sync();
        // ---- merge the 16 warps of this CTA (thread d owns output element d) ----
        float m_cta = -INFINITY, l_cta = 0.f, o_cta = 0.f;
        if (tid < MK_D) {
#pragma unroll
            for (int i = 0; i < MK_CONS_WARPS; ++i) m_cta = fmaxf(m_cta, s_part[i][MK_D]);
#pragma unroll
            for (int i = 0; i < MK_CONS_WARPS; ++i) {
                const float ms = s_part[i][MK_D];
                const float wgt = (ms == -INFINITY) ? 0.f : exp2f(ms - m_cta);
                l_cta += s_part[i][MK_D + 1] * wgt;
                o_cta += s_part[i][tid] * wgt;
            }
        }
        if (G == 1) {
            if (tid < MK_D) p.attn[(size_t)b * h + head * MK_D + tid] = __float2bfloat16_rn(o_cta / l_cta);
        } else {
            float* part = p.attn_partial + ((size_t)pair * G + split) * (MK_D + 2);
            if (tid < MK_D) {
                part[tid] = o_cta;
                if (tid == 0) { part[MK_D] = m_cta; part[MK_D + 1] = l_cta; }
            }
            __threadfence();
            cons_sync();
            if (tid == 0) *s_flag = (atomicAdd(&p.attn_counters[pair], 1) == G - 1) ? 1 : 0;
            cons_sync();
            if (*s_flag) {  // last CTA of this (b, head): merge the G partials
                __threadfence();
                if (tid < MK_D) {
                    const float* pb = p.attn_partial + (size_t)pair * G * (MK_D + 2);
                    float m_all = -INFINITY;
                    for (int sidx = 0; sidx < G; ++sidx) m_all = fmaxf(m_all, __ldcg(pb + (size_t)sidx * (MK_D + 2) + MK_D));
                    float l_all = 0.f, o_all = 0.f;
                    for (int sidx = 0; sidx < G; ++sidx) {
                        const float ms = __ldcg(pb + (size_t)sidx * (MK_D + 2) + MK_D);
                        const float wgt = (ms == -INFINITY) ? 0.f : exp2f(ms - m_all);
                        l_all += __ldcg(pb + (size_t)sidx * (MK_D + 2) + MK_D + 1) * wgt;
                        o_all += __ldcg(pb + (size_t)sidx * (MK_D + 2) + tid) * wgt;
                    }
                    p.attn[(size_t)b * h + head * MK_D + tid] = __float2bfloat16_rn(o_all / l_all);
                    if (tid == 0) p.attn_counters[pair] = 0;
                }
            }
        }
        cons_sync();  // s_part / s_flag are reused by the next pair
    }
}

// position in the CTA's tile sequence over all GEMV phases (phase -> 8-row block -> K tile)
struct TileCursor {
    GemvCtx c;
    int ph, rb, kc;
    uint32_t tile;
    bool valid;
};
__device__ __forceinline__ void cursor_seek(TileCursor& t, const MegaParams& p, const MegaLayer* layers, int n_phases) {
    // move to the first phase at or after t.ph that is a GEMV phase with work for this CTA
    while (t.ph < n_phases) {
        if (!mk_is_attention(p, t.ph)) {
            t.c = mk_phase_ctx(p, layers, t.ph);
            if (t.c.nb > 0) { t.rb = 0; t.kc = 0; t.valid = true; return; }
        }
        ++t.ph;
    }
    t.valid = false;
}
__device__ __forceinline__ void cursor_begin(TileCursor& t, const MegaParams& p, const MegaLayer* layers, int n_phases) {
    t.ph = 0; t.tile = 0; t.rb = 0; t.kc = 0;
    cursor_seek(t, p, layers, n_phases);
}
__device__ __forceinline__ void cursor_next(TileCursor& t, const MegaParams& p, const MegaLayer* layers, int n_phases) {
    ++t.tile;
    if (++t.kc < t.c.nchunk) return;
    t.kc = 0;
    if (++t.rb < t.c.nb) return;
    ++t.ph;
    cursor_seek(t, p, layers, n_phases);
}
template <int NB>
__global__ void __launch_bounds__(MK_THREADS, 1) decode_mega_kernel(MegaParams p, int n_stages) {
    extern __shared__ __align__(128) uint8_t mk_smem[];
    // dynamic smem: [ring: n_stages x MK_TILE_BYTES][xs: NB x Kmax bf16][s_gpart: 16 x MAXNB x NB x 8 fp32][mbarriers]
    uint8_t* ring = mk_smem;
    __nv_bfloat16* xs = reinterpret_cast<__nv_bfloat16*>(ring + (size_t)n_stages * MK_TILE_BYTES);
    float* s_gpart = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(xs) + (size_t)NB * (p.h > p.I ? p.h : p.I) * 2);
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(s_gpart + (size_t)MK_CONS_WARPS * MK_MAXNB * NB * 8);
    uint64_t* empty_bar = full_bar + MK_MAX_STAGES;
    __shared__ float s_red[MK_CONS_WARPS][NB];
    __shared__ float s_rstd[NB];
    __shared__ float s_av[MK_CONS_WARPS];
    __shared__ int s_ai[MK_CONS_WARPS];
    __shared__ float s_part[MK_CONS_WARPS][MK_D + 2];
    __shared__ int s_flag;
    __shared__ float s_cos[NB * 64], s_sin[NB * 64];  // RoPE table of this step (HF: cos/sin cast to bf16)
    __shared__ __align__(16) MegaLayer s_layers[MK_MAXL];           // weight-pointer table: no dependent global load per phase

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int B = p.B;
    const int n_phases = 5 * p.L + 1;

    // ---- one-time setup (all warps) ----
    {
        const uint4* src = reinterpret_cast<const uint4*>(p.layers);
        uint4* dst = reinterpret_cast<uint4*>(s_layers);
        for (int i = tid; i < p.L * (int)(sizeof(MegaLayer) / 16); i += MK_THREADS) dst[i] = src[i];
        if (tid == 0) {
            for (int s = 0; s < n_stages; ++s) {
                mbar_init(&full_bar[s], 1);               // producer's arrive.expect_tx (+ TMA bytes)
                mbar_init(&empty_bar[s], MK_CONS_WARPS);  // one arrive per consumer warp
            }
            fence_barrier_init();
        }
        __syncthreads();
    }

    if (warp >= MK_CONS_WARPS) {
        // =========================== PRODUCERS: stream every phase's weight tiles, in order ===========================
        // `cp` feeds the shared-memory ring with TMA bulk copies, throttled by free ring slots
        const uint32_t pw = (uint32_t)(warp - MK_CONS_WARPS);
        TileCursor cp;
        cursor_begin(cp, p, s_layers, n_phases);
        while (cp.valid) {
            if (cp.tile % (uint32_t)MK_PROD_WARPS == pw) {
                const uint32_t stage = cp.tile % (uint32_t)n_stages;
                const uint32_t parity = (cp.tile / (uint32_t)n_stages) & 1u;
                const uint32_t row_bytes = (uint32_t)min(MK_KT, cp.c.K - cp.kc * MK_KT) * 2u;
                if (lane == 0) {
                    mbar_wait(&empty_bar[stage], parity ^ 1u);  // slot drained by all consumer warps
                    mbar_arrive_expect_tx(&full_bar[stage], (uint32_t)mk_rows_in_block(cp.c, cp.rb) * row_bytes);
                }
                __syncwarp();
                bool row_valid;
                const int prow = mk_phys_row(cp.c, cp.rb, lane & 7, row_valid);
                if (lane < 8 && row_valid)
                    bulk_g2s(ring + (size_t)stage * MK_TILE_BYTES + (size_t)lane * MK_ROW_STRIDE,
                             cp.c.W + (size_t)prow * cp.c.K + (size_t)cp.kc * MK_KT, row_bytes, &full_bar[stage]);
            }
            cursor_next(cp, p, s_layers, n_phases);
        }
        return;
    }

    // =========================== CONSUMERS (16 warps) ===========================
    // ---- phase "-1": RoPE table, x = embed_tokens[tok] ----
    for (int i = tid; i < B * 64; i += MK_CONS) {
        const int b = i >> 6, f = i & 63;
        const float inv_freq = exp2f(-(2.0f * f / MK_D) * log2f(p.theta));
        float sv, cv;
        sincosf((float)p.cur_len[b] * inv_freq, &sv, &cv);
        s_cos[i] = round_bf16(cv);
        s_sin[i] = round_bf16(sv);
    }
    if (blockIdx.x < B) {
        int t = p.tok[blockIdx.x];
        t = t < 0 ? 0 : (t >= p.V ? p.V - 1 : t);
        const uint4* src = reinterpret_cast<const uint4*>(p.embed + (size_t)t * p.h);
        uint4* dst = reinterpret_cast<uint4*>(p.x + (size_t)blockIdx.x * p.h);
        for (int i = tid; i < p.h / 8; i += MK_CONS) dst[i] = src[i];
    }
    // The RMSNorm weights of the NEXT phase are copied (cp.async, no registers held) into the part of the
    // activation tile that a K = h phase leaves unused, in front of the grid barrier; the prologue then finds them in shared
    // memory instead of paying an L2/HBM round trip between its two passes.
    __nv_bfloat16* gsm = xs + (size_t)NB * p.h;
    const bool gsm_fits = (size_t)(NB + 1) * p.h <= (size_t)NB * (p.h > p.I ? p.h : p.I);
    auto gamma_prefetch = [&](int ph) -> bool {
        if (!gsm_fits || ph >= n_phases || mk_is_attention(p, ph)) return false;
        const PhaseIO io = mk_phase_io(p, s_layers, ph);
        if (io.gamma == nullptr) return false;
        for (int i = tid; i < (p.h >> 3); i += MK_CONS)
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(gsm + i * 8)), "l"(io.gamma + i * 8) : "memory");
        asm volatile("cp.async.commit_group;" ::: "memory");
        return true;
    };
    bool gsm_ok = gamma_prefetch(0);
    unsigned int bar_target = p.bar_base + gridDim.x;
    grid_sync(p.bar_count, bar_target);

    const bool tracing = p.trace != nullptr && blockIdx.x == 0 && tid == 0;
    const int g = lane >> 2, t4 = lane & 3;
    uint32_t tile = 0;
#pragma unroll 1
    for (int ph = 0; ph < n_phases; ++ph) {
        if (tracing) p.trace[ph * 4 + 0] = clock64();
        if (mk_is_attention(p, ph)) {
            mk_attention(p, s_layers[ph / 5], tid, lane, warp, s_part, &s_flag, s_cos, s_sin);
        } else {
            const GemvCtx c = mk_phase_ctx(p, s_layers, ph);
            const PhaseIO io = mk_phase_io(p, s_layers, ph);
            // residual of the (<= 512) outputs this CTA writes: fetched now, consumed after the weight stream
            const bool have_res = io.residual != nullptr && c.nu * B <= MK_CONS;
            float res_pref = 0.f;
            if (have_res && tid < c.nu * B) {
                const int b = tid / c.nu, r = tid - b * c.nu;
                res_pref = __bfloat162float(__ldcg(io.residual + (size_t)b * io.ld_out + (size_t)c.u_lo + r));
            }
            mk_prologue<NB>(io, c.K, B, p.eps, tid, lane, warp, xs, s_red, s_rstd, gsm_ok ? gsm : nullptr);
            if (tracing) p.trace[ph * 4 + 1] = clock64();
#pragma unroll 1
            for (int rb = 0; rb < c.nb; ++rb) {
                float acc[4] = {0.f, 0.f, 0.f, 0.f}, acc2[4] = {0.f, 0.f, 0.f, 0.f};  // two independent MMA chains
#pragma unroll 1
                for (int kc = 0; kc < c.nchunk; ++kc, ++tile) {
                    const uint32_t stage = tile % (uint32_t)n_stages;
                    const uint32_t parity = (tile / (uint32_t)n_stages) & 1u;
                    const int nk32 = min(MK_KT, c.K - kc * MK_KT) >> 5;
                    mbar_wait(&full_bar[stage], parity);  // TMA bytes of this tile have landed
                    const uint8_t* trow = ring + (size_t)stage * MK_TILE_BYTES + (size_t)g * MK_ROW_STRIDE + t4 * 16;
                    const __nv_bfloat16* xrow = xs + (size_t)g * c.K + (size_t)kc * MK_KT + t4 * 8;
#pragma unroll 4
                    for (int k32 = warp; k32 < nk32; k32 += MK_CONS_WARPS) {
                        const uint4 wv = *reinterpret_cast<const uint4*>(trow + k32 * 64);
                        uint4 xv = make_uint4(0, 0, 0, 0);
                        if (g < B) xv = *reinterpret_cast<const uint4*>(xrow + k32 * 32);
                        mk_mma(acc, xv.x, xv.y, wv.x, wv.y);
                        mk_mma(acc2, xv.z, xv.w, wv.z, wv.w);
                    }
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&empty_bar[stage]);  // this warp is done reading the slot
                }
                // acc[0], acc[1] = D[batch g][weight rows 2*t4, 2*t4+1] over this warp's K slices
                if (g < NB)
                    *reinterpret_cast<float2*>(s_gpart + (((size_t)warp * MK_MAXNB + rb) * NB + g) * 8 + t4 * 2) =
                        make_float2(acc[0] + acc2[0], acc[1] + acc2[1]);
            }
            cons_sync();
            if (tracing) p.trace[ph * 4 + 2] = clock64();
            mk_epilogue<NB>(p, s_layers, ph, c, B, tid, s_gpart, res_pref, have_res);
        }
        if (tracing) p.trace[ph * 4 + 3] = clock64();
        gsm_ok = gamma_prefetch(ph + 1);
        bar_target += gridDim.x;
        grid_sync(p.bar_count, bar_target);
    }
    if (tracing) p.trace[n_phases * 4] = clock64();

    // ---------------- greedy argmax (first occurrence), token store, counters ----------------
    if (blockIdx.x < B) {
        const int b = blockIdx.x;
        const float* row = p.logits + (size_t)b * p.V;
        float best = -INFINITY;
        int bi = INT_MAX;
        for (int i = tid; i < p.V; i += MK_CONS) {
            const float v = __ldcg(row + i);
            if (v == v && (bi == INT_MAX || v > best)) { best = v; bi = i; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, best, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
        }
        if (lane == 0) { s_av[warp] = best; s_ai[warp] = bi; }
        cons_sync();
        if (warp == 0) {
            best = lane < MK_CONS_WARPS ? s_av[lane] : -INFINITY;
            bi = lane < MK_CONS_WARPS ? s_ai[lane] : INT_MAX;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const float ov = __shfl_xor_sync(0xffffffffu, best, o);
                const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
                if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
            }
            if (lane == 0) {
                const int tk = bi == INT_MAX ? 0 : bi;
                p.tok[b] = tk;
                p.out_tokens[(size_t)(*p.step_counter) * B + b] = tk;
                if (p.rows == nullptr || p.rows[b].active) p.cur_len[b] += 1;  // every attention phase of this launch is behind the last barrier
                if (p.ring != nullptr) {  // streaming generate(): the host reads the token from mapped pinned memory
                    const int pub = p.sstate->pub_counter, tag0 = p.sstate->tag;
                    if (tag0 != 0) {
                        const int tag = 1 + (tag0 - 1 + pub / p.ring_cap) % 2047;  // advances when the ring wraps (sampling.cu)
                        reinterpret_cast<volatile int32_t*>(p.ring)[(size_t)(pub % p.ring_cap) * B + b] = (tag << 20) | (tk & 0xFFFFF);
                        __threadfence_system();
                    }
                }
            }
        }
    }
    // step counter: bumped by the last CTA to get here (after all token stores read it)
    cons_sync();
    if (tid == 0) {
        __threadfence();
        if (atomicAdd(p.done_count, 1u) == gridDim.x - 1) {
            *p.done_count = 0u;
            *p.step_counter += 1;
            if (p.ring != nullptr) p.sstate->pub_counter += 1;
        }
    }
}

// dynamic smem carve-up (must match the kernel): ring, activation tile, K-slice partial sums, mbarriers
size_t mega_fixed_bytes(int NB, int h, int I) {
    return (size_t)NB * (h > I ? h : I) * 2 + (size_t)MK_CONS_WARPS * MK_MAXNB * NB * 8 * 4 + 2 * MK_MAX_STAGES * 8;
}
size_t mega_static_bytes(int NB) {
    return (size_t)(MK_CONS_WARPS + 1) * NB * 4 + MK_CONS_WARPS * (MK_D + 2 + 2) * 4 + NB * 512 +
           MK_MAXL * sizeof(MegaLayer) + 1024;
}
int mega_stages(int NB, int h, int I) {
    const long long avail = 227 * 1024 - (long long)mega_fixed_bytes(NB, h, I) - (long long)mega_static_bytes(NB);
    long long s = avail / MK_TILE_BYTES;
    return (int)(s > MK_MAX_STAGES ? MK_MAX_STAGES : s);
}

}  // namespace

bool decode_mega_fits(int B, int h, int I) {
    if (B < 1 || B > 2) return false;
    return mega_stages(B, h, I) >= 4;
}

int decode_mega(const MegaParams& p, cudaStream_t stream) {
    B2_CHECK_ARG(p.B >= 1 && p.B <= 2, "decode_mega: batch must be 1..2");
    B2_CHECK_ARG(p.L <= MK_MAXL, "decode_mega: %d layers exceed the shared layer table (%d)", p.L, MK_MAXL);
    B2_CHECK_ARG(p.h % 256 == 0 && p.I % 256 == 0 && p.V % 8 == 0 && p.h / p.H == MK_D,
                 "decode_mega: unsupported dims h=%d I=%d V=%d H=%d", p.h, p.I, p.V, p.H);
    {
        const int grid = num_sms();
        const int nmax = p.V > 3 * p.h ? (p.V > 2 * p.I ? p.V : 2 * p.I) : (3 * p.h > 2 * p.I ? 3 * p.h : 2 * p.I);
        B2_CHECK_ARG((nmax / 8 + grid - 1) / grid + 1 <= MK_MAXNB,
                     "decode_mega: %d output rows per CTA exceed the shared-memory block table", nmax / grid);
    }
    const int NB = p.B;
    const int stages = mega_stages(NB, p.h, p.I);
    B2_CHECK_ARG(stages >= 4, "decode_mega: shared memory too small for the weight ring (B=%d h=%d I=%d)", p.B, p.h, p.I);
    const size_t smem = (size_t)stages * MK_TILE_BYTES + mega_fixed_bytes(NB, p.h, p.I);
    void* fn = NB == 1 ? (void*)decode_mega_kernel<1> : (void*)decode_mega_kernel<2>;
    static size_t attr_smem[3] = {0, 0, 0};
    if (smem > attr_smem[NB]) {
        B2_CUDA_CHECK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr_smem[NB] = smem;
    }
    MegaParams pp = p;
    int n_stages = stages;
    void* args[] = {&pp, &n_stages};
    // cooperative launch: the grid barrier needs every CTA resident (grid = #SMs, 1 CTA/SM)
    B2_CUDA_CHECK(cudaLaunchCooperativeKernel(fn, dim3(num_sms()), dim3(MK_THREADS), args, smem, stream));
    B2_LAUNCH_CHECK();
    return 0;
}

}  // namespace b2
