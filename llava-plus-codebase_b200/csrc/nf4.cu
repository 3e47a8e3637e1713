// NF4 decoder weights (load_4bit; reference llava/model/builder.py:26-41, bitsandbytes `bnb_4bit_quant_type='nf4'`).
// Format (DESIGN.md §2-3):
//   * per output row, every block of 64 consecutive K elements: absmax = fp32 max |w|, x = w / absmax (IEEE division),
//     code = number of fp32 midpoints of the 16-entry NF4 table that x lies strictly above (a tie takes the lower code, as
//     in bitsandbytes' dQuantizeNF4); an all-zero block stores absmax 0 and code 7;
//   * w_hat = bf16_rn(fp32(table[code]) * absmax);
//   * codes [N, K/2] bytes, element 2j in the high nibble of byte j ("canonical"); absmax [N, K/64] fp32.
// The engine keeps the codes in "GEMV order": within each 128-element chunk of a row (64 bytes), the 16-bit word holding
// elements 4G .. 4G+3 (G = 4m + t) moves from word G to word 8t + m. One 16-byte load of lane t then holds, for each
// m = 0..7, the four elements 16m + 4t .. +3: exactly what lane t contributes to the m-th mma.sync k16 step, and the four
// lanes of an mma step cover 16 consecutive elements, which lie in ONE absmax block. That lets gemv_nf4 multiply raw
// (unscaled) codebook values on the tensor cores and apply the block's absmax to the fp32 partial sum.
#include "common.cuh"
#include "kernels.h"

namespace b2 {
namespace {

__constant__ float c_nf4[16] = {
    -1.0f, -0.6961928009986877f, -0.5250730514526367f, -0.39491748809814453f, -0.28444138169288635f,
    -0.18477343022823334f, -0.09105003625154495f, 0.0f, 0.07958029955625534f, 0.16093020141124725f,
    0.24611230194568634f, 0.33791524171829224f, 0.44070982933044434f, 0.5626170039176941f, 0.7229568362236023f, 1.0f};

__device__ __forceinline__ uint32_t nf4_code(float x) {
    uint32_t q = 0;
#pragma unroll
    for (int i = 0; i < 15; ++i) q += x > __fmul_rn(__fadd_rn(c_nf4[i], c_nf4[i + 1]), 0.5f) ? 1u : 0u;
    return q;
}

// byte offset inside a row of the byte that holds canonical byte j (j = 2 * element index, high nibble first)
__device__ __forceinline__ int64_t nf4_byte_pos(int64_t j, int gemv_order) {
    if (!gemv_order) return j;
    const int64_t chunk = j >> 6;
    const int cb = (int)(j & 63), G = cb >> 1;
    return chunk * 64 + 2 * (8 * (G & 3) + (G >> 2)) + (cb & 1);
}

// one warp per 64-element block; lane l quantises elements 2l, 2l+1 into one byte
__global__ void quantize_nf4_kernel(const __nv_bfloat16* __restrict__ w, int64_t ldw, uint8_t* __restrict__ q,
                                    float* __restrict__ absmax, int N, int K, int gemv_order) {
    const int lane = threadIdx.x & 31;
    const int64_t nblk_row = K / 64, nblk = (int64_t)N * nblk_row;
    const int64_t warps = (int64_t)gridDim.x * (blockDim.x / 32);
    for (int64_t blk = (int64_t)blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5); blk < nblk; blk += warps) {
        const int64_t row = blk / nblk_row, kb = blk - row * nblk_row;
        const uint32_t pair = *reinterpret_cast<const uint32_t*>(w + row * ldw + kb * 64 + lane * 2);
        const float w0 = bf16_lo(pair), w1 = bf16_hi(pair);
        const float a = warp_max(fmaxf(fabsf(w0), fabsf(w1)));
        uint32_t hi = 7, lo = 7;
        if (a > 0.f) {
            hi = nf4_code(__fdiv_rn(w0, a));
            lo = nf4_code(__fdiv_rn(w1, a));
        }
        q[row * (K / 2) + nf4_byte_pos(kb * 32 + lane, gemv_order)] = (uint8_t)(hi << 4 | lo);
        if (lane == 0) absmax[blk] = a;
    }
}

struct Nf4Mats {
    const uint8_t* q[4];
    const float* absmax[4];
    __nv_bfloat16* out[4];
    int N[4], K[4];
    int gemv_order;
};

// w_hat of the two elements of a code byte (element 2j in the high nibble) as a bf16x2 value (low half = element 2j). `tab`
// is the table in shared memory: 16 words in 16 banks, so lanes looking up different codes never conflict (the constant
// cache would serialise them)
__device__ __forceinline__ uint32_t nf4_pair(const float* tab, uint32_t byte, float a) {
    return pack_bf16(__fmul_rn(tab[byte >> 4], a), __fmul_rn(tab[byte & 15], a));
}

// blockIdx.y = matrix; a thread dequantises one 16-byte piece of codes (32 elements): one 16-byte load, four 16-byte stores
// (canonical order: 32 consecutive elements of one absmax block) or eight 8-byte stores (GEMV order: piece t of a 128-element
// chunk holds elements 16m + 4t .. +3, m = 0..7, the first four in the chunk's first block; the four pieces of a chunk write
// whole 32-byte sectors together)
__global__ void dequantize_nf4_kernel(Nf4Mats p) {
    __shared__ float tab[16];
    if (threadIdx.x < 16) tab[threadIdx.x] = c_nf4[threadIdx.x];
    __syncthreads();
    const int mi = blockIdx.y;
    const int K = p.K[mi], ppr = K / 32;  // pieces per row
    const int pieces = p.N[mi] * ppr;
    const uint8_t* __restrict__ q = p.q[mi];
    const float* __restrict__ am = p.absmax[mi];
    __nv_bfloat16* __restrict__ out = p.out[mi];
    for (int u = blockIdx.x * blockDim.x + threadIdx.x; u < pieces; u += gridDim.x * blockDim.x) {
        const int row = u / ppr, pp = u - row * ppr;
        const uint4 v = ld_stream_16(q + (size_t)u * 16);
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
        __nv_bfloat16* orow = out + (size_t)row * K;
        const float* arow = am + (size_t)row * (K / 64);
        if (!p.gemv_order) {
            const float a = arow[pp >> 1];
#pragma unroll
            for (int j = 0; j < 4; ++j)
                *reinterpret_cast<uint4*>(orow + pp * 32 + j * 8) =
                    make_uint4(nf4_pair(tab, w[j] & 0xff, a), nf4_pair(tab, (w[j] >> 8) & 0xff, a),
                               nf4_pair(tab, (w[j] >> 16) & 0xff, a), nf4_pair(tab, w[j] >> 24, a));
        } else {
            const int chunk = pp >> 2, t = pp & 3;
            const float2 a2 = *reinterpret_cast<const float2*>(arow + chunk * 2);
#pragma unroll
            for (int m = 0; m < 8; ++m) {
                const float a = m < 4 ? a2.x : a2.y;
                const uint32_t h = (w[m >> 1] >> ((m & 1) * 16)) & 0xffff;
                *reinterpret_cast<uint2*>(orow + chunk * 128 + 16 * m + 4 * t) = make_uint2(nf4_pair(tab, h & 0xff, a), nf4_pair(tab, h >> 8, a));
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------------------------------
// gemv_nf4: out[B, N] = (RMSNorm(x) | x)[B, K] · w_hat[N, K]^T (+ residual), or the fused SwiGLU variant; B <= 8.
// Same skeleton as gemv_bf16 (gemv.cu): persistent grid of one 512-thread CTA per SM, contiguous output ranges per CTA,
// 16 warps splitting K, 16-byte L1-bypassing weight loads issued before the activation prologue, fixed-order reduction of
// the 16 partial sums through shared memory. The tensor-core step is mma.sync.m16n8k16 with the WEIGHTS as the A operand
// (16 weight rows) and the activations as B (8 batch columns, zero beyond B): a lane holds rows g and g + 8 of a 16-row
// block, one 16-byte load per row per 128-element chunk = 8 k16 steps. Every weight enters the MMA as exactly w_hat =
// bf16_rn(table[code] * absmax), the value the dequantiser writes: the fp32 code comes from a 16-entry shared-memory table
// (16 words in 16 banks, so any access pattern is conflict-free), is multiplied by its block's absmax (__fmul_rn) and
// rounded in pairs to bf16x2 operands. The product therefore equals a dense bf16 GEMV over w_hat up to the order of the
// fp32 accumulation.
constexpr int Q4_THREADS = 512;
constexpr int Q4_WARPS = Q4_THREADS / 32;
constexpr int Q4_NU = 2;  // 128-element units per pipeline batch (two 16-byte weight loads + two absmax pairs each)

struct Nf4GemvParams {
    const __nv_bfloat16* x; int64_t ldx;
    const uint8_t* q; const float* absmax;
    const __nv_bfloat16* gamma; float eps;
    const __nv_bfloat16* residual; int ld_res;
    __nv_bfloat16* out; int ld_out;
    int B, N, K, act;
    int nb_max;
};

struct Q4Ctx {
    int u_lo, nu, nb;   // output units (rows / SwiGLU channels), blocks of 16 rows
    int ks_lo, ks_len;  // this warp's K slice in 128-element chunks
};

// physical row of A-row r (0..15) of local block rb
__device__ __forceinline__ int q4_phys_row(const Nf4GemvParams& p, const Q4Ctx& c, int rb, int r, bool& valid) {
    if (p.act == ACT_SWIGLU) {  // rows 0..7 = gate of channels 8rb .. 8rb+7, rows 8..15 = their up rows
        const int lc = rb * 8 + (r & 7);
        valid = lc < c.nu;
        const int ch = c.u_lo + lc;
        return (ch >> 6) * 128 + (ch & 63) + (r >= 8 ? 64 : 0);
    }
    const int lr = rb * 16 + r;
    valid = lr < c.nu;
    return c.u_lo + lr;
}

struct Q4Buf {
    uint4 w[2 * Q4_NU];    // [unit][row g, row g+8]
    float2 s[2 * Q4_NU];   // absmax of the chunk's two blocks, same order
};

__device__ __forceinline__ void q4_issue(const Nf4GemvParams& p, const Q4Ctx& c, int bt, int lane, Q4Buf& buf) {
    const int U = c.nb * c.ks_len;
    const int g = lane >> 2, t = lane & 3;
    const int64_t qpitch = p.K / 2, spitch = p.K / 64;
#pragma unroll
    for (int j = 0; j < Q4_NU; ++j) {
        const int u = bt * Q4_NU + j;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            buf.w[2 * j + h] = make_uint4(0, 0, 0, 0);
            buf.s[2 * j + h] = make_float2(0.f, 0.f);
        }
        if (u < U) {
            const int rb = u / c.ks_len, kc = c.ks_lo + (u - rb * c.ks_len);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                bool valid;
                const int row = q4_phys_row(p, c, rb, g + 8 * h, valid);
                if (valid) {
                    buf.w[2 * j + h] = ld_stream_16(p.q + (int64_t)row * qpitch + (int64_t)kc * 64 + t * 16);
                    buf.s[2 * j + h] = __ldg(reinterpret_cast<const float2*>(p.absmax + (int64_t)row * spitch + kc * 2));
                }
            }
        }
    }
}

__device__ __forceinline__ void q4_mma(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0,
                                       uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

__device__ __forceinline__ uint32_t u4_word(const uint4& v, int i) {
    return i == 0 ? v.x : (i == 1 ? v.y : (i == 2 ? v.z : v.w));
}

// position of element k of a row in the permuted activation tile (lane t's 32 elements of a chunk are contiguous)
__device__ __forceinline__ int q4_xpos(int k) {
    return (k & ~127) | (((k >> 2) & 3) << 5) | (((k >> 4) & 7) << 2) | (k & 3);
}

template <int NB>
__global__ void __launch_bounds__(Q4_THREADS, 1) gemv_nf4_kernel(Nf4GemvParams p) {
    extern __shared__ __align__(16) uint8_t q4_smem[];
    __nv_bfloat16* xs = reinterpret_cast<__nv_bfloat16*>(q4_smem);                                  // [NB][K] permuted
    float* s_part = reinterpret_cast<float*>(q4_smem + (size_t)NB * p.K * 2);                      // [16][nb_max][16][NB]
    __shared__ float s_code[16];
    __shared__ float s_red[Q4_WARPS][NB];
    __shared__ float s_rstd[NB];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int K = p.K;
    Q4Ctx c;
    {
        const long long units = p.act == ACT_SWIGLU ? (p.N >> 1) : p.N;
        c.u_lo = (int)((units * blockIdx.x) / gridDim.x);
        c.nu = (int)((units * (blockIdx.x + 1)) / gridDim.x) - c.u_lo;
        c.nb = p.act == ACT_SWIGLU ? (c.nu + 7) >> 3 : (c.nu + 15) >> 4;
        const int nk = K >> 7;
        c.ks_lo = (nk * warp) / Q4_WARPS;
        c.ks_len = (nk * (warp + 1)) / Q4_WARPS - c.ks_lo;
    }

    Q4Buf bufA, bufB;
    q4_issue(p, c, 0, lane, bufA);  // weights do not depend on x: get HBM requests in flight before the prologue
    q4_issue(p, c, 1, lane, bufB);

    // ---------------- prologue: code table, x -> smem (bf16, permuted), optional fused RMSNorm ----------------
    if (tid < 16) s_code[tid] = c_nf4[tid];
    {
        const int nvec = K >> 3;
        float ss[NB];
#pragma unroll
        for (int b = 0; b < NB; ++b) ss[b] = 0.f;
        for (int i = tid; i < nvec; i += Q4_THREADS) {
            const int p0 = q4_xpos(i * 8), p1 = q4_xpos(i * 8 + 4);
#pragma unroll
            for (int b = 0; b < NB; ++b) {
                uint4 u = make_uint4(0, 0, 0, 0);
                if (b < p.B) u = *reinterpret_cast<const uint4*>(p.x + (size_t)b * p.ldx + i * 8);
                *reinterpret_cast<uint2*>(xs + (size_t)b * K + p0) = make_uint2(u.x, u.y);
                *reinterpret_cast<uint2*>(xs + (size_t)b * K + p1) = make_uint2(u.z, u.w);
                if (p.gamma != nullptr) {
                    const uint32_t wv[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
                    for (int e = 0; e < 4; ++e) ss[b] += bf16_lo(wv[e]) * bf16_lo(wv[e]) + bf16_hi(wv[e]) * bf16_hi(wv[e]);
                }
            }
        }
        if (p.gamma != nullptr) {
#pragma unroll
            for (int b = 0; b < NB; ++b) {
                const float v = warp_sum(ss[b]);
                if (lane == 0) s_red[warp][b] = v;
            }
            __syncthreads();
            if (tid < NB) {
                float t = 0.f;
                for (int w = 0; w < Q4_WARPS; ++w) t += s_red[w][tid];
                s_rstd[tid] = rsqrtf(t / K + p.eps);
            }
            __syncthreads();
            for (int i = tid; i < nvec; i += Q4_THREADS) {
                const uint4 gv = *reinterpret_cast<const uint4*>(p.gamma + i * 8);
                const uint32_t gw[4] = {gv.x, gv.y, gv.z, gv.w};
                const int p0 = q4_xpos(i * 8), p1 = q4_xpos(i * 8 + 4);
#pragma unroll
                for (int b = 0; b < NB; ++b) {
                    uint2* x0 = reinterpret_cast<uint2*>(xs + (size_t)b * K + p0);
                    uint2* x1 = reinterpret_cast<uint2*>(xs + (size_t)b * K + p1);
                    const uint2 v0 = *x0, v1 = *x1;
                    const uint32_t xw[4] = {v0.x, v0.y, v1.x, v1.y};
                    uint32_t o[4];
                    const float rstd = s_rstd[b];
                    // HF LlamaRMSNorm: weight * (x * rstd).to(bf16), result in bf16
#pragma unroll
                    for (int e = 0; e < 4; ++e)
                        o[e] = pack_bf16(bf16_lo(gw[e]) * round_bf16(bf16_lo(xw[e]) * rstd),
                                         bf16_hi(gw[e]) * round_bf16(bf16_hi(xw[e]) * rstd));
                    *x0 = make_uint2(o[0], o[1]);
                    *x1 = make_uint2(o[2], o[3]);
                }
            }
        }
        __syncthreads();
    }

    // ---------------- main loop ----------------
    {
        const int g = lane >> 2, t = lane & 3;
        const int U = c.nb * c.ks_len;
        const int n_batches = (U + Q4_NU - 1) / Q4_NU;
        const __nv_bfloat16* xrow = xs + (size_t)(g < NB ? g : 0) * K + t * 32;
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
        int rb = 0, kk = 0;
        auto compute = [&](int bt, const Q4Buf& buf) {
#pragma unroll
            for (int j = 0; j < Q4_NU; ++j) {
                if (bt * Q4_NU + j < U) {  // warp-uniform
                    const uint4 w0 = buf.w[2 * j], w1 = buf.w[2 * j + 1];
                    const float2 s0 = buf.s[2 * j], s1 = buf.s[2 * j + 1];
                    const __nv_bfloat16* xc = xrow + (size_t)(c.ks_lo + kk) * 128;
#pragma unroll
                    for (int h = 0; h < 2; ++h) {  // the chunk's two 64-element absmax blocks
                        const float sa = h ? s0.y : s0.x, sb = h ? s1.y : s1.x;  // rows g and g + 8
#pragma unroll
                        for (int jj = 0; jj < 2; ++jj) {  // two 16-byte activation loads = four k16 steps
                            uint4 xv = make_uint4(0, 0, 0, 0);
                            if (g < p.B) xv = *reinterpret_cast<const uint4*>(xc + (h * 2 + jj) * 8);
                            const uint32_t r0 = u4_word(w0, h * 2 + jj), r1 = u4_word(w1, h * 2 + jj);
                            q4_mma(acc, nf4_pair(s_code, r0 & 0xff, sa), nf4_pair(s_code, r1 & 0xff, sb),
                                   nf4_pair(s_code, (r0 >> 8) & 0xff, sa), nf4_pair(s_code, (r1 >> 8) & 0xff, sb), xv.x, xv.y);
                            q4_mma(acc, nf4_pair(s_code, (r0 >> 16) & 0xff, sa), nf4_pair(s_code, (r1 >> 16) & 0xff, sb),
                                   nf4_pair(s_code, r0 >> 24, sa), nf4_pair(s_code, r1 >> 24, sb), xv.z, xv.w);
                        }
                    }
                    if (++kk == c.ks_len) {
                        // acc = D[rows g, g+8][batches 2t, 2t+1] of block rb over this warp's K slice
                        float* sp = s_part + ((size_t)warp * p.nb_max + rb) * 16 * NB;
                        if (2 * t < NB) {
                            sp[g * NB + 2 * t] = acc[0];
                            sp[(g + 8) * NB + 2 * t] = acc[2];
                        }
                        if (2 * t + 1 < NB) {
                            sp[g * NB + 2 * t + 1] = acc[1];
                            sp[(g + 8) * NB + 2 * t + 1] = acc[3];
                        }
                        acc[0] = acc[1] = acc[2] = acc[3] = 0.f;
                        kk = 0;
                        ++rb;
                    }
                }
            }
        };
#pragma unroll 1
        for (int bt = 0; bt < n_batches; bt += 2) {
            compute(bt, bufA);
            q4_issue(p, c, bt + 2, lane, bufA);
            compute(bt + 1, bufB);
            q4_issue(p, c, bt + 3, lane, bufB);
        }
    }
    __syncthreads();

    // ---------------- reduce the 16 K slices (fixed order), epilogue ----------------
    {
        const int nk = K >> 7;
        auto row_value = [&](int rbl, int b, int r) {
            float v = 0.f;
#pragma unroll
            for (int ww = 0; ww < Q4_WARPS; ++ww) {
                const bool has = (nk * (ww + 1)) / Q4_WARPS > (nk * ww) / Q4_WARPS;  // K < 2048: empty slices
                if (has) v += s_part[(((size_t)ww * p.nb_max + rbl) * 16 + r) * NB + b];
            }
            return v;
        };
        if (p.act == ACT_SWIGLU) {
            for (int idx = tid; idx < c.nu * p.B; idx += Q4_THREADS) {
                const int b = idx / c.nu, r = idx - b * c.nu;
                const float gt = row_value(r >> 3, b, r & 7);
                const float up = row_value(r >> 3, b, (r & 7) + 8);
                p.out[(size_t)b * p.ld_out + c.u_lo + r] = __float2bfloat16_rn(gt / (1.0f + __expf(-gt)) * up);
            }
        } else {
            for (int idx = tid; idx < c.nu * p.B; idx += Q4_THREADS) {
                const int b = idx / c.nu, r = idx - b * c.nu;
                float y = row_value(r >> 4, b, r & 15);
                const int row = c.u_lo + r;
                if (p.residual != nullptr) y += __bfloat162float(p.residual[(size_t)b * p.ld_res + row]);
                p.out[(size_t)b * p.ld_out + row] = __float2bfloat16_rn(y);
            }
        }
    }
}

int q4_nb(int B) { return B == 1 ? 1 : (B == 2 ? 2 : (B <= 4 ? 4 : 8)); }

int q4_nb_max(int N, int act) {
    const int grid = num_sms();
    const long long units = act == ACT_SWIGLU ? (N >> 1) : N;
    const int nu_max = (int)((units + grid - 1) / grid);
    return act == ACT_SWIGLU ? (nu_max + 7) / 8 : (nu_max + 15) / 16;
}

size_t q4_smem_bytes(int B, int N, int K, int act) {
    const int NB = q4_nb(B);
    return (size_t)NB * K * 2 + (size_t)Q4_WARPS * q4_nb_max(N, act) * 16 * NB * 4;
}

constexpr size_t kQ4SmemMax = 226 * 1024;

template <int NB>
int launch_gemv_nf4(Nf4GemvParams p, cudaStream_t stream) {
    p.nb_max = q4_nb_max(p.N, p.act);
    const size_t smem = q4_smem_bytes(p.B, p.N, p.K, p.act);
    B2_CHECK_ARG(smem <= kQ4SmemMax, "gemv_nf4: activation tile + partial table do not fit shared memory (B=%d K=%d N=%d)",
                 p.B, p.K, p.N);
    static size_t attr_smem = 0;
    if (smem > attr_smem) {
        B2_CUDA_CHECK(cudaFuncSetAttribute(gemv_nf4_kernel<NB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr_smem = smem;
    }
    gemv_nf4_kernel<NB><<<num_sms(), Q4_THREADS, smem, stream>>>(p);
    B2_LAUNCH_CHECK();
    return 0;
}

}  // namespace

int quantize_nf4(const void* w, int64_t ldw, int N, int K, void* q, float* absmax, int gemv_order, cudaStream_t stream) {
    B2_CHECK_ARG(w && q && absmax, "quantize_nf4: null argument");
    B2_CHECK_ARG(N > 0 && K > 0 && K % 64 == 0 && ldw >= K && ldw % 2 == 0, "quantize_nf4: need N > 0, K a positive multiple of 64, "
                 "ldw >= K and even (N=%d K=%d ldw=%lld)", N, K, (long long)ldw);
    B2_CHECK_ARG(!gemv_order || K % 128 == 0, "quantize_nf4: GEMV order needs K %% 128 == 0 (K=%d)", K);
    B2_CHECK_ARG((reinterpret_cast<uintptr_t>(w) & 3) == 0, "quantize_nf4: w must be 4-byte aligned");
    const int64_t blocks = (int64_t)N * (K / 64);
    const int64_t ctas = (blocks + 7) / 8;
    quantize_nf4_kernel<<<(unsigned)(ctas < 65535 * 16 ? ctas : 65535 * 16), 256, 0, stream>>>(
        reinterpret_cast<const __nv_bfloat16*>(w), ldw, reinterpret_cast<uint8_t*>(q), absmax, N, K, gemv_order);
    B2_LAUNCH_CHECK();
    return 0;
}

int dequantize_nf4(const Nf4Matrix* mats, int n, int gemv_order, cudaStream_t stream) {
    B2_CHECK_ARG(mats && n >= 1 && n <= 4, "dequantize_nf4: 1..4 matrices per launch (got %d)", n);
    Nf4Mats p;
    int64_t most = 0;
    for (int i = 0; i < n; ++i) {
        const Nf4Matrix& m = mats[i];
        B2_CHECK_ARG(m.q && m.absmax && m.out && m.N > 0 && m.K > 0 && m.K % 64 == 0,
                     "dequantize_nf4: matrix %d: null pointer or K not a positive multiple of 64 (N=%d K=%d)", i, m.N, m.K);
        B2_CHECK_ARG(!gemv_order || m.K % 128 == 0, "dequantize_nf4: GEMV order needs K %% 128 == 0 (K=%d)", m.K);
        B2_CHECK_ARG((int64_t)m.N * m.K / 32 < INT32_MAX, "dequantize_nf4: matrix %d too large (N=%d K=%d)", i, m.N, m.K);
        B2_CHECK_ARG((reinterpret_cast<uintptr_t>(m.out) & 15) == 0 && (reinterpret_cast<uintptr_t>(m.q) & 15) == 0 &&
                         (reinterpret_cast<uintptr_t>(m.absmax) & 7) == 0,
                     "dequantize_nf4: out and codes must be 16-byte, absmax 8-byte aligned");
        p.q[i] = reinterpret_cast<const uint8_t*>(m.q);
        p.absmax[i] = m.absmax;
        p.out[i] = reinterpret_cast<__nv_bfloat16*>(m.out);
        p.N[i] = m.N;
        p.K[i] = m.K;
        most = (int64_t)m.N * m.K / 32 > most ? (int64_t)m.N * m.K / 32 : most;
    }
    p.gemv_order = gemv_order;
    const int64_t ctas = (most + 255) / 256;
    const int64_t cap = (int64_t)num_sms() * 8;
    dequantize_nf4_kernel<<<dim3((unsigned)(ctas < cap ? ctas : cap), (unsigned)n), 256, 0, stream>>>(p);
    B2_LAUNCH_CHECK();
    return 0;
}

bool gemv_nf4_fits(int B, int N, int K, int act) {
    return B >= 1 && B <= 8 && K % 128 == 0 && q4_smem_bytes(B, N, K, act) <= kQ4SmemMax;
}

int gemv_nf4(const GemvArgs& g, const void* q, const float* absmax, cudaStream_t stream) {
    B2_CHECK_ARG(g.B >= 1 && g.B <= 8, "gemv_nf4: batch must be 1..8 (got %d)", g.B);
    B2_CHECK_ARG(g.K % 128 == 0 && g.K > 0, "gemv_nf4: K must be a positive multiple of 128 (K=%d)", g.K);
    B2_CHECK_ARG(g.N % 2 == 0 && g.N > 0, "gemv_nf4: N must be even (N=%d)", g.N);
    B2_CHECK_ARG(g.act == ACT_NONE || g.act == ACT_SWIGLU, "gemv_nf4: unsupported activation %d", g.act);
    B2_CHECK_ARG(!g.out_fp32, "gemv_nf4: bf16 output only");
    B2_CHECK_ARG(g.act != ACT_SWIGLU || (g.N % 128 == 0 && g.residual == nullptr),
                 "gemv_nf4: swiglu needs N %% 128 == 0 and no residual");
    B2_CHECK_ARG(q && absmax && (reinterpret_cast<uintptr_t>(q) & 15) == 0 && (reinterpret_cast<uintptr_t>(absmax) & 7) == 0,
                 "gemv_nf4: codes must be 16-byte and absmax 8-byte aligned");
    B2_CHECK_ARG((reinterpret_cast<uintptr_t>(g.x) & 15) == 0 && g.ldx % 8 == 0, "gemv_nf4: x must be 16B aligned with a 16B-multiple row pitch");
    Nf4GemvParams p;
    p.x = reinterpret_cast<const __nv_bfloat16*>(g.x); p.ldx = g.ldx;
    p.q = reinterpret_cast<const uint8_t*>(q); p.absmax = absmax;
    p.gamma = reinterpret_cast<const __nv_bfloat16*>(g.norm_gamma); p.eps = g.eps;
    p.residual = reinterpret_cast<const __nv_bfloat16*>(g.residual); p.ld_res = g.ld_res;
    p.out = reinterpret_cast<__nv_bfloat16*>(g.out); p.ld_out = g.ld_out;
    p.B = g.B; p.N = g.N; p.K = g.K; p.act = g.act; p.nb_max = 0;
    if (g.B == 1) return launch_gemv_nf4<1>(p, stream);
    if (g.B == 2) return launch_gemv_nf4<2>(p, stream);
    if (g.B <= 4) return launch_gemv_nf4<4>(p, stream);
    return launch_gemv_nf4<8>(p, stream);
}

}  // namespace b2
