// Selection primitives shared by token selection (sampling.cu) and beam-candidate selection (beam.cu): the counter-based
// Philox4x32-10 draw, a fixed-order block sum, and a radix descent over 32-bit keys of a row. Each caller brings its own
// key function, so the two files keep their own treatment of NaN (sampling.cu orders NaN by its bits, beam.cu below -inf).
#pragma once
#include <stdint.h>

namespace b2 {

__device__ __forceinline__ void philox_round(uint32_t (&c)[4], uint32_t k0, uint32_t k1) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c[0]), lo0 = 0xD2511F53u * c[0];
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c[2]), lo1 = 0xCD9E8D57u * c[2];
    const uint32_t n0 = hi1 ^ c[1] ^ k0, n1 = lo1, n2 = hi0 ^ c[3] ^ k1, n3 = lo0;
    c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
}
// Philox4x32-10 with counter (index, row, 0, 0) and the seed as key; returns (c0 << 32) | c1
__device__ __forceinline__ unsigned long long philox_u64(unsigned long long seed, uint32_t index, uint32_t row) {
    uint32_t c[4] = {index, row, 0u, 0u};
    uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        philox_round(c, k0, k1);
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    return ((unsigned long long)c[0] << 32) | c[1];
}

// probability mass in 2^-40 fixed point: integer sums of it are exact and independent of the order of the adds
__device__ __forceinline__ unsigned long long mass_of(float e) {
    return e > 0.f ? __float2ull_rz(e * 1099511627776.0f) : 0ull;  // NaN / -inf survivors carry no mass
}

template <int THREADS, typename T>
__device__ __forceinline__ T block_sum(T v, T* s_w, int tid) {  // fixed order: warp shuffle tree, then warp sums in order
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((tid & 31) == 0) s_w[tid >> 5] = v;
    __syncthreads();
    T t = 0;
    for (int i = 0; i < THREADS / 32; ++i) t += s_w[i];
    return t;
}

// Radix descent over key_of(i), i in [0, V), 8 bits per level from the top. Level state lives in shared memory (s_prefix /
// s_above); every thread of the block calls it. On return *s_above holds the weight strictly above the selected key.
//   COUNT mode (MASS = false): weight of an element = 1; selects the key of the limit-th largest element. A warp adds its
//     elements with one shared atomic per distinct digit: keys of a row crowd into a few digits (at level 0 nearly all share
//     sign and exponent), and one atomic per element would serialise on the crowded bin.
//   MASS mode: weight = weight_of(i); selects the smallest key whose strictly-above weight is < limit.
// Integer adds only, so the result does not depend on the thread schedule.
template <int THREADS, bool MASS, typename KeyOf, typename WeightOf>
__device__ __forceinline__ uint32_t radix_select(int V, unsigned long long limit, int tid, KeyOf key_of, WeightOf weight_of,
                                                 unsigned long long* s_hist, uint32_t* s_prefix, unsigned long long* s_above) {
    if (tid == 0) { *s_prefix = 0u; *s_above = 0ull; }
    for (int level = 0; level < 4; ++level) {
        const int shift = 24 - 8 * level;
        if (tid < 256) s_hist[tid] = 0ull;
        __syncthreads();
        const uint32_t prefix = *s_prefix;
        if (MASS) {
            for (int i = tid; i < V; i += THREADS) {
                const uint32_t key = key_of(i);
                if (level == 0 || (key >> (shift + 8)) == prefix) {
                    const unsigned long long w = weight_of(i);
                    if (w) atomicAdd(&s_hist[(key >> shift) & 255u], w);
                }
            }
        } else {
            for (int base = 0; base < V; base += THREADS) {  // uniform trip count: the whole warp reaches the match
                const int i = base + tid;
                const uint32_t key = i < V ? key_of(i) : 0u;
                const bool take = i < V && (level == 0 || (key >> (shift + 8)) == prefix);
                const uint32_t digit = take ? ((key >> shift) & 255u) : 256u;
                const unsigned peers = __match_any_sync(0xffffffffu, digit);
                if (take && (tid & 31) == __ffs(peers) - 1) atomicAdd(&s_hist[digit], (unsigned long long)__popc(peers));
            }
        }
        __syncthreads();
        if (tid == 0) {
            unsigned long long acc = *s_above;
            int pick = 255;
            if (MASS) {
                // smallest digit d whose strictly-above mass acc_d is still < limit (acc_255 = above < limit by construction)
                for (int d = 255; d >= 0; --d) {
                    if (acc >= limit) break;
                    pick = d;
                    *s_above = acc;
                    acc += s_hist[d];
                }
            } else {
                // digit holding the limit-th largest element: walk down until the running count reaches it
                pick = 0;
                for (int d = 255; d >= 0; --d) {
                    if (acc + s_hist[d] >= limit) { pick = d; *s_above = acc; break; }
                    acc += s_hist[d];
                }
            }
            *s_prefix = (prefix << 8) | (uint32_t)pick;
        }
        __syncthreads();
    }
    return *s_prefix;
}

}  // namespace b2
