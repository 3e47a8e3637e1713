// Small HBM-bound data-movement kernels of the multimodal path:
//   splice_embed  : the GPU half of prepare_inputs_labels_for_multimodal (llava/model/llava_arch.py:150-225):
//                   embed_tokens gather for text positions, image-feature rows for the <image> span, zero rows
//                   for padding — one pass, 16-byte vectors, driven by a host-built source-row index.
//   embed_tokens  : embedding lookup for the decode token (modeling_llama.py embed_tokens).
//   argmax_f32    : greedy sampling on the last-position logits (HF GenerationMixin greedy_search argmax;
//                   ties resolve to the lowest index like torch.argmax).
//   convert / interleave: weight ingestion (dtype cast, gate||up block-64 interleave for the fused SwiGLU epilogue).
#include <cuda_fp16.h>
#include <limits.h>

#include "common.cuh"
#include "kernels.h"

namespace b2 {
namespace {

// err_flag points at int[8] in mapped host memory: slot log2(code) is set to 1 with a plain store (no PCIe atomics needed)
__device__ __forceinline__ void report_err(int* err_flag, int code) {
    reinterpret_cast<volatile int*>(err_flag)[31 - __clz(code)] = 1;
}

// An index outside the embedding table / the image-feature rows (tokenizer larger than the table, a leftover
// IMAGE_TOKEN_INDEX with no images, ...) must neither read out of bounds nor kill the context: the row becomes zeros and the
// code is flagged in err_flag[] (mapped host memory), which the host turns into a ValueError at its next sync point.
__global__ void splice_embed_kernel(const int32_t* __restrict__ src_index, const uint4* __restrict__ table,
                                    const uint4* __restrict__ feats, uint4* __restrict__ out, int vec_per_row, int vocab,
                                    int n_feat_rows, int* err_flag) {
    const int row = blockIdx.x;
    const int32_t s = src_index[row];
    uint4* o = out + (size_t)row * vec_per_row;
    const uint4* src = nullptr;
    if (s >= 0) {
        if (s < vocab) src = table + (size_t)s * vec_per_row;
        else if (threadIdx.x == 0 && err_flag) report_err(err_flag, B2_ERR_TOKEN_RANGE);
    } else if (s != INT_MIN) {
        const int64_t f = -(int64_t)s - 1;
        if (feats != nullptr && f < n_feat_rows) src = feats + (size_t)f * vec_per_row;
        else if (threadIdx.x == 0 && err_flag) report_err(err_flag, feats == nullptr ? B2_ERR_TOKEN_RANGE : B2_ERR_IMAGE_ROW_RANGE);
    }
    if (src == nullptr) {
        for (int c = threadIdx.x; c < vec_per_row; c += blockDim.x) o[c] = make_uint4(0, 0, 0, 0);
    } else {
        for (int c = threadIdx.x; c < vec_per_row; c += blockDim.x) o[c] = src[c];
    }
}

__global__ void embed_tokens_kernel(const int32_t* __restrict__ tokens, const uint4* __restrict__ table,
                                    uint4* __restrict__ out, int vec_per_row, int vocab, int* err_flag) {
    const int row = blockIdx.x;
    pdl_trigger();
    pdl_wait();  // tokens come from the previous step's selection kernel
    int32_t t = tokens[row];
    if ((t < 0 || t >= vocab) && threadIdx.x == 0 && err_flag) report_err(err_flag, B2_ERR_TOKEN_RANGE);
    t = t < 0 ? 0 : (t >= vocab ? vocab - 1 : t);  // never read out of bounds
    const uint4* src = table + (size_t)t * vec_per_row;
    uint4* o = out + (size_t)row * vec_per_row;
    for (int c = threadIdx.x; c < vec_per_row; c += blockDim.x) o[c] = src[c];
}

// one CTA per row; (value desc, index asc) ordering == torch.argmax first-occurrence semantics
__global__ void __launch_bounds__(1024) argmax_kernel(const float* __restrict__ logits, int V,
                                                      int32_t* __restrict__ out) {
    const float* row = logits + (size_t)blockIdx.x * V;
    float best = -INFINITY;
    int bi = INT_MAX;
    for (int i = threadIdx.x; i < V; i += blockDim.x) {
        const float v = row[i];
        // indices are visited in increasing order per thread: strict > keeps the first occurrence; NaN skipped
        if (v == v && (bi == INT_MAX || v > best)) { best = v; bi = i; }
    }
    __shared__ float sv[32];
    __shared__ int si[32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) { sv[warp] = best; si[warp] = bi; }
    __syncthreads();
    if (warp == 0) {
        const int nw = blockDim.x >> 5;
        best = lane < nw ? sv[lane] : -INFINITY;
        bi = lane < nw ? si[lane] : INT_MAX;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, best, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
        }
        if (lane == 0) out[blockIdx.x] = bi == INT_MAX ? 0 : bi;
    }
}

template <typename T>
__device__ __forceinline__ float to_f32(T v);
template <>
__device__ __forceinline__ float to_f32<float>(float v) { return v; }
template <>
__device__ __forceinline__ float to_f32<__half>(__half v) { return __half2float(v); }

template <typename T>
__global__ void convert_kernel(const T* __restrict__ src, __nv_bfloat16* __restrict__ dst, int64_t n) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
        dst[i] = __float2bfloat16_rn(to_f32<T>(src[i]));
}

__global__ void interleave_gate_up_kernel(const uint4* __restrict__ gate, const uint4* __restrict__ up,
                                          uint4* __restrict__ out, int I, int vec_per_row) {
    const int orow = blockIdx.x;  // 0 .. 2I
    const int grp = orow >> 7, r = orow & 127;
    const uint4* src = (r < 64) ? gate + (size_t)(grp * 64 + r) * vec_per_row
                                : up + (size_t)(grp * 64 + r - 64) * vec_per_row;
    uint4* o = out + (size_t)orow * vec_per_row;
    for (int c = threadIdx.x; c < vec_per_row; c += blockDim.x) o[c] = src[c];
}

// Device half of the splice INDEX (llava/model/llava_arch.py:143-187 of the reference, equal-length unpadded rows): one CTA
// per prompt row scans the ids for IMAGE_TOKEN_INDEX with a block-wide prefix count and writes, for every output position
// of the row, the source row that splice_embed_kernel gathers: token id for text, -(feature row)-1 for the image span.
// Image slots are consumed in row-major order (row b owns slots b*k .. b*k+k-1, k = placeholders per row as the caller
// expects them: a different count is reported through err_flag[B2_ERR_SPLICE_SLOTS] and the host redoes the splice on its
// exact path). Output positions beyond S (cannot happen when the count matches) are dropped; nothing is written out of bounds.
__global__ void __launch_bounds__(256)
splice_index_kernel(const long long* __restrict__ ids, int Lt, int k_expected, I32Pack feat_off, int image_token, int S,
                    int32_t* __restrict__ src_index, int* err_flag) {
    __shared__ int s_warp[8];
    __shared__ int s_total;
    const int b = blockIdx.x, tid = threadIdx.x;
    const long long* row = ids + (size_t)b * Lt;
    const int chunk = (Lt + 255) / 256;
    const int lo = min(tid * chunk, Lt), hi = min(lo + chunk, Lt);
    int mine = 0;
    for (int i = lo; i < hi; ++i) mine += row[i] == (long long)image_token;
    int incl = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int up = __shfl_up_sync(0xffffffffu, incl, o);
        if ((tid & 31) >= o) incl += up;
    }
    if ((tid & 31) == 31) s_warp[tid >> 5] = incl;
    __syncthreads();
    int base = 0;
    for (int w = 0; w < (tid >> 5); ++w) base += s_warp[w];
    if (tid == 255) s_total = base + incl;
    int c = base + incl - mine;  // placeholders before position lo
    const int slot0 = b * k_expected;
    int32_t* out = src_index + (size_t)b * S;
    // positions the row does not cover are zero rows (INT32_MIN): only reachable when the placeholder count is wrong
    for (int i = tid; i < S; i += 256) out[i] = INT_MIN;
    __syncthreads();
    for (int i = lo; i < hi; ++i) {
        const long long id = row[i];
        const int cc = min(c, k_expected);
        const int pos = (i - c) + (feat_off.v[slot0 + cc] - feat_off.v[slot0]);
        if (id == (long long)image_token) {
            if (c < k_expected) {
                const int f0 = feat_off.v[slot0 + c], f1 = feat_off.v[slot0 + c + 1];
                for (int f = f0; f < f1; ++f)
                    if (pos + (f - f0) < S) out[pos + (f - f0)] = -f - 1;
            }
            ++c;
        } else if (pos < S) {
            // ids that do not fit an int32 can only be invalid: map them to an out-of-range index (reported by the gather)
            out[pos] = (id >= 0 && id < 0x7fffffffLL) ? (int32_t)id : 0x7fffffff;
        }
    }
    __syncthreads();
    if (tid == 0 && s_total != k_expected && err_flag) report_err(err_flag, B2_ERR_SPLICE_SLOTS);
}

// dst_a[off + i] = a.v[i], dst_b[off + i] = b.v[i]: small host vectors travel as kernel parameters (no pinned staging
// buffer whose lifetime would force a stream sync in the caller)
__global__ void set_i32_pairs_kernel(int32_t* dst_a, int32_t* dst_b, I32Pack a, I32Pack b, int n, int off) {
    const int i = threadIdx.x;
    if (i < n) { dst_a[off + i] = a.v[i]; if (dst_b) dst_b[off + i] = b.v[i]; }
}

}  // namespace

int set_i32_pairs(int32_t* dst_a, const int32_t* a_host, int32_t* dst_b, const int32_t* b_host, int n, cudaStream_t stream) {
    for (int off = 0; off < n; off += 128) {
        const int c = n - off < 128 ? n - off : 128;
        I32Pack pa, pb;
        for (int i = 0; i < c; ++i) { pa.v[i] = a_host[off + i]; pb.v[i] = b_host ? b_host[off + i] : 0; }
        set_i32_pairs_kernel<<<1, 128, 0, stream>>>(dst_a, dst_b, pa, pb, c, off);
        B2_LAUNCH_CHECK();
    }
    return 0;
}

int splice_index(const long long* ids, int B, int Lt, int k_per_row, const int32_t* feat_offsets_host, int n_img, int image_token,
                 int S, int32_t* src_index, int* err_flag, cudaStream_t stream) {
    B2_CHECK_ARG(B >= 1 && Lt >= 1 && S >= 1 && k_per_row >= 0 && n_img == B * k_per_row && n_img + 1 <= 128,
                 "splice_index: bad arguments B=%d Lt=%d S=%d k=%d n_img=%d (at most 127 image slots)", B, Lt, S, k_per_row, n_img);
    I32Pack off;
    for (int i = 0; i <= n_img; ++i) off.v[i] = feat_offsets_host[i];
    splice_index_kernel<<<B, 256, 0, stream>>>(ids, Lt, k_per_row, off, image_token, S, src_index, err_flag);
    B2_LAUNCH_CHECK();
    return 0;
}

int splice_embed(const int32_t* src_index, const void* table, const void* feats, void* out, int rows, int h, int vocab,
                 int n_feat_rows, int* err_flag, cudaStream_t stream) {
    B2_CHECK_ARG(h % 8 == 0 && rows > 0, "splice_embed: bad shape rows=%d h=%d", rows, h);
    splice_embed_kernel<<<rows, 128, 0, stream>>>(src_index, reinterpret_cast<const uint4*>(table),
                                                  reinterpret_cast<const uint4*>(feats),
                                                  reinterpret_cast<uint4*>(out), h / 8, vocab, n_feat_rows, err_flag);
    B2_LAUNCH_CHECK();
    return 0;
}

int embed_tokens(const int32_t* tokens, const void* table, void* out, int rows, int h, int vocab, int* err_flag,
                 cudaStream_t stream) {
    B2_CHECK_ARG(h % 8 == 0 && rows > 0, "embed_tokens: bad shape rows=%d h=%d", rows, h);
    B2_CUDA_CHECK(launch_pdl(embed_tokens_kernel, dim3(rows), dim3(128), 0, stream, tokens, reinterpret_cast<const uint4*>(table),
                             reinterpret_cast<uint4*>(out), h / 8, vocab, err_flag));
    B2_LAUNCH_CHECK();
    return 0;
}

int argmax_f32(const float* logits, int B, int V, int32_t* out, cudaStream_t stream) {
    B2_CHECK_ARG(B > 0 && V > 0, "argmax: empty input");
    argmax_kernel<<<B, 1024, 0, stream>>>(logits, V, out);
    B2_LAUNCH_CHECK();
    return 0;
}

int convert_to_bf16(const void* src, int src_dtype, void* dst, int64_t n, cudaStream_t stream) {
    if (n == 0) return 0;
    if (src_dtype == DT_BF16) {
        B2_CUDA_CHECK(cudaMemcpyAsync(dst, src, (size_t)n * 2, cudaMemcpyDefault, stream));
        return 0;
    }
    const int grid = (int)((n + 255) / 256 < 4096 ? (n + 255) / 256 : 4096);
    if (src_dtype == DT_F32) {
        convert_kernel<float><<<grid, 256, 0, stream>>>(reinterpret_cast<const float*>(src),
                                                        reinterpret_cast<__nv_bfloat16*>(dst), n);
    } else if (src_dtype == DT_F16) {
        convert_kernel<__half><<<grid, 256, 0, stream>>>(reinterpret_cast<const __half*>(src),
                                                         reinterpret_cast<__nv_bfloat16*>(dst), n);
    } else {
        set_error("convert_to_bf16: unsupported dtype %d", src_dtype);
        return -1;
    }
    B2_LAUNCH_CHECK();
    return 0;
}

int interleave_gate_up(const void* gate, const void* up, void* out, int I, int h, cudaStream_t stream) {
    B2_CHECK_ARG(I % 64 == 0 && h % 8 == 0, "interleave_gate_up: I %% 64 and h %% 8 must be 0 (I=%d h=%d)", I, h);
    interleave_gate_up_kernel<<<2 * I, 128, 0, stream>>>(reinterpret_cast<const uint4*>(gate),
                                                         reinterpret_cast<const uint4*>(up),
                                                         reinterpret_cast<uint4*>(out), I, h / 8);
    B2_LAUNCH_CHECK();
    return 0;
}

}  // namespace b2
