// Beam search on the device (generate(num_beams > 1), llava/_b2/beam.py holds the host half):
//
//   * beam_topk: per sample, the K best continuations among its nb beams x V tokens of
//     score = log_softmax(logits[row_of_beam[beam]]) + beam_scores[beam] (fp32, torch's rounding order: (x - max) - log(sum)),
//     sorted by score descending; ties go to the lower flat index beam * V + token. NaN logits are never preferred to a
//     number (they rank below -inf); -inf is an ordinary value. Two launches: one CTA per beam row stages the row in shared
//     memory, turns it into scores in place, radix-selects the row's K-th best key and compacts the row's top K in index
//     order; a second launch merges the nb sorted lists of each sample by rank (binary search in every list).
//     A candidate is one 64-bit key: order_key(score) << 32 | ~flat, so "larger key" is exactly the ranking rule above.
//   * beam_sample (generate(do_sample=True, num_beams > 1)): the same two launches, but the row kernel warps the log-softmax
//     row (temperature, top-k, top-p with at least min_keep survivors, HF 5.5's warpers on log-probabilities) and ranks each
//     finite survivor by the Gumbel-perturbed key fp32(acc + g), g = -log(-log u), u from Philox(seed; step, global flat index).
//     The K largest keys in order are HF's torch.multinomial(softmax(acc), K) draw order (multinomial without replacement is
//     top-K of p / Exp(1) there). Warped-away tokens (-inf) rank below every finite key by index, NaN logits below those. The
//     merge carries each candidate's unperturbed score acc beside its key.
//   * with logits processors (BeamProc, b2_beam_step_proc / b2_op_beam_select_proc): both row kernels turn the staged row into
//     log-probabilities, run HF's processors over them against the history of the row's cache slot (logits_proc.cuh's
//     process_row, after appending the token the step fed to that slot), and rank on processed + running score; under beam
//     sampling the warpers follow the processors. Instantiated separately (PROC = true), so the unprocessed kernels are unchanged.
//   * kv_copy_slots: cache slot dst := rows [row_begin, end) of slot src for every layer, head, K and V (and the fp32 scale
//     rows of an e4m3 cache); one (layer, head, K|V) slab of one slot is contiguous, so each CTA streams 64 rows with
//     16-byte vectors. The caller guarantees that no dst is also a src (b2_kv_copy_slots checks it), so pairs are independent.
#include <limits.h>
#include <math.h>

#include "common.cuh"
#include "kernels.h"
#include "logits_proc.cuh"
#include "select.cuh"

namespace b2 {
namespace {

constexpr int BT_THREADS = 1024;
constexpr int BM_THREADS = 256;
constexpr int CP_THREADS = 256;
constexpr int CP_ROWS = 64;  // cache rows per copy CTA (16 KiB of a bf16 slab)

__device__ __forceinline__ uint32_t order_key(float x) {  // monotone float -> uint; NaN -> 0 (below -inf)
    if (x != x) return 0u;
    const uint32_t u = __float_as_uint(x);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_float(uint32_t k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k);
}

// fixed-order block reduction (warp shuffle tree, then the warp partials in order): the same bits on every run
template <bool MAX>
__device__ __forceinline__ float block_reduce(float v, float* s_w, int tid) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float w = __shfl_xor_sync(0xffffffffu, v, o);
        v = MAX ? fmaxf(v, w) : v + w;
    }
    __syncthreads();
    if ((tid & 31) == 0) s_w[tid >> 5] = v;
    __syncthreads();
    float t = s_w[0];
    for (int i = 1; i < BT_THREADS / 32; ++i) t = MAX ? fmaxf(t, s_w[i]) : t + s_w[i];
    return t;
}

// Shared state of one row CTA's candidate selection
struct RowSmem {
    float w[BT_THREADS / 32];
    int wa[BT_THREADS / 32];
    unsigned long long wsum[BT_THREADS / 32];
    unsigned long long hist[256];
    unsigned long long above;
    uint32_t prefix;
    int gt;
    unsigned long long cand[128];
};

// The row's Kr best 64-bit candidates order_key(s_x[i]) << 32 | ~(flat0 + i) into sm.cand[0, Kr), unordered: a radix select
// of the Kr-th largest key, then compaction in index order, 1024 consecutive elements per pass (a warp reads 32 consecutive
// words: no bank conflicts): every element above the Kr-th key, then the lowest-index elements equal to it until Kr are taken.
__device__ __forceinline__ void row_top_candidates(const float* s_x, int V, int Kr, unsigned long long flat0, int tid, RowSmem& sm) {
    const uint32_t kth = radix_select<BT_THREADS, false>(
        V, (unsigned long long)Kr, tid, [&](int i) { return order_key(s_x[i]); }, [](int) { return 1ull; }, sm.hist, &sm.prefix,
        &sm.above);
    const int n_gt = (int)sm.above, need_eq = Kr - n_gt;
    const int lane = tid & 31, warp = tid >> 5;
    if (tid == 0) sm.gt = 0;
    __syncthreads();
    int eq_seen = 0;  // uniform: elements equal to kth in the passes before this one
    for (int base = 0; base < V; base += BT_THREADS) {
        const int i = base + tid;
        const uint32_t key = i < V ? order_key(s_x[i]) : 0u;
        const unsigned long long cand = ((unsigned long long)key << 32) | (uint32_t)(0xFFFFFFFFu - (uint32_t)(flat0 + i));
        if (i < V && key > kth) sm.cand[atomicAdd(&sm.gt, 1)] = cand;
        const bool eq = i < V && key == kth;
        const unsigned bal = __ballot_sync(0xffffffffu, eq);
        if (lane == 0) sm.wa[warp] = __popc(bal);
        __syncthreads();
        int before = 0, total = 0;
        for (int w = 0; w < BT_THREADS / 32; ++w) {
            before += w < warp ? sm.wa[w] : 0;
            total += sm.wa[w];
        }
        if (eq) {
            const int r = eq_seen + before + __popc(bal & ((1u << lane) - 1u));
            if (r < need_eq) sm.cand[n_gt + r] = cand;
        }
        eq_seen += total;
        // sm.gt is final for this pass after the barrier above; read it before the next one, after which a faster warp may
        // already add to it in the next pass, so that every thread tests the same value
        const int gt = sm.gt;
        __syncthreads();
        if (eq_seen >= need_eq && gt == n_gt) break;  // uniform: both parts complete
    }
    __syncthreads();
}

// Stages logits row `row` in s_x and returns its max (NaN skipped) and log-sum-exp: torch's log_softmax is (x - mx) - lse
__device__ __forceinline__ void stage_row(const float* __restrict__ x, float* s_x, int V, int tid, RowSmem& sm, float& mx, float& lse) {
    mx = -INFINITY;
    for (int i = tid; i < V; i += BT_THREADS) {
        const float v = x[i];
        s_x[i] = v;
        if (v > mx) mx = v;  // NaN never compares greater
    }
    mx = block_reduce<true>(mx, sm.w, tid);
    float part = 0.f;
    for (int i = tid; i < V; i += BT_THREADS) {
        const float v = s_x[i];
        if (v == v) part += expf(v - mx);
    }
    lse = logf(block_reduce<false>(part, sm.w, tid));
}

// Processing of beam row `beam` (logits row `row`) against history `row`: the token the step fed to that slot joins the history
// first (each slot is read by exactly one beam row when `append` is given). Returns whether the row's processors are on.
__device__ __forceinline__ bool beam_proc_begin(const BeamProc& bp, int beam, int row, int V, int tid) {
    ProcRow& pr = bp.proc.rows[row];
    const bool on = pr.on != 0;
    if (on && bp.append != nullptr && tid == 0) {
        const int t = bp.append[beam], n = pr.hist_len;
        if (n < bp.proc.cap) {
            bp.proc.hist[(size_t)row * bp.proc.cap + n] = t;
            pr.hist_len = n + 1;
        }
        if (t >= 0 && t < V) bp.proc.bits[(size_t)row * bp.proc.words + (t >> 5)] |= 1u << (t & 31);
    }
    __syncthreads();  // the history and its length are final for process_row
    return on;
}

template <bool PROC>
__global__ void __launch_bounds__(BT_THREADS, 1)
beam_row_topk_kernel(const float* __restrict__ logits, const int32_t* __restrict__ row_of_beam, const float* __restrict__ beam_scores,
                     int nb, int V, int K, unsigned long long* __restrict__ keys_out, BeamRowsOut ro, BeamProc bp) {
    extern __shared__ __align__(16) uint8_t bt_smem[];
    float* s_x = reinterpret_cast<float*>(bt_smem);
    __shared__ RowSmem sm;

    const int tid = threadIdx.x, j = blockIdx.x, b = blockIdx.y;
    const int beam = b * nb + j;
    const int row = row_of_beam ? row_of_beam[beam] : beam;
    const int Kr = K < V ? K : V;  // candidates this row can supply

    float mx, lse;
    stage_row(logits + (size_t)row * V, s_x, V, tid, sm, mx, lse);
    const float run = beam_scores[beam];
    const size_t out0 = (size_t)beam * ro.fan * V;
    if constexpr (PROC) {
        // the log-probabilities, processed in place; the output score row is the processed row
        for (int i = tid; i < V; i += BT_THREADS) {
            const float x = s_x[i];
            s_x[i] = (x - mx) - lse;
            if (ro.logits != nullptr)
                for (int r = 0; r < ro.fan; ++r) ro.logits[out0 + (size_t)r * V + i] = x;
        }
        if (beam_proc_begin(bp, beam, row, V, tid)) process_row<BT_THREADS>(s_x, V, bp.proc, row, tid);
        __syncthreads();
        for (int i = tid; i < V; i += BT_THREADS) {
            const float ls = s_x[i];
            s_x[i] = ls + run;
            if (ro.scores != nullptr)
                for (int r = 0; r < ro.fan; ++r) ro.scores[out0 + (size_t)r * V + i] = ls;
        }
    } else {
        for (int i = tid; i < V; i += BT_THREADS) {
            const float x = s_x[i], ls = (x - mx) - lse;
            s_x[i] = ls + run;
            for (int r = 0; r < ro.fan; ++r) {  // output rows: the log-softmax row and the raw row, once per running beam it feeds
                if (ro.scores != nullptr) ro.scores[out0 + (size_t)r * V + i] = ls;
                if (ro.logits != nullptr) ro.logits[out0 + (size_t)r * V + i] = x;
            }
        }
    }
    __syncthreads();
    row_top_candidates(s_x, V, Kr, (unsigned long long)j * V, tid, sm);

    // sort the row's Kr candidates (descending key) by rank; pad the list with 0 (below every real candidate)
    unsigned long long* out = keys_out + (size_t)beam * K;
    if (tid < Kr) {
        const unsigned long long me = sm.cand[tid];
        int rank = 0;
        for (int c = 0; c < Kr; ++c) rank += sm.cand[c] > me;
        out[rank] = me;
    } else if (tid < K) {
        out[tid] = 0ull;
    }
}

// Beam sampling (HF _beam_search with do_sample): per beam row, the warped scores w = ((x - max) - lse) / T with top-k and
// top-p survivors (at least min_keep of each), the accumulated score acc = w + running score, and for every finite survivor
// the Gumbel-perturbed key fp32(acc + g), g = -log(-log u) in fp64, u from Philox(seed; step, global flat index). The row's K
// largest keys are selected as in beam_row_topk_kernel (warped-away tokens are -inf and rank by index below every finite key,
// NaN logits below them); the candidate's score is its unperturbed acc, written beside its key. With PROC the processors run on
// the log-probabilities before the division by T.
template <bool PROC>
__global__ void __launch_bounds__(BT_THREADS, 1)
beam_row_sample_kernel(const float* __restrict__ logits, const int32_t* __restrict__ row_of_beam, const float* __restrict__ beam_scores,
                       int nb, int V, int K, BeamSampleParams sp, unsigned long long* __restrict__ keys_out,
                       float* __restrict__ scores_out, BeamRowsOut ro, BeamProc bp) {
    extern __shared__ __align__(16) uint8_t bt_smem[];
    float* s_x = reinterpret_cast<float*>(bt_smem);
    __shared__ RowSmem sm;

    const int tid = threadIdx.x, j = blockIdx.x, b = blockIdx.y;
    const int beam = b * nb + j;
    const int row = row_of_beam ? row_of_beam[beam] : beam;
    const int Kr = K < V ? K : V;
    const float* x = logits + (size_t)row * V;
    const float T = sp.temperature;
    auto key_of = [&](int i) { return order_key(s_x[i]); };

    float mx, lse;
    stage_row(x, s_x, V, tid, sm, mx, lse);
    const size_t out0 = (size_t)beam * V;  // beam sampling reads one row per running beam: fan is 1
    for (int i = tid; i < V; i += BT_THREADS) {
        if (ro.logits != nullptr) ro.logits[out0 + i] = s_x[i];
        s_x[i] = PROC ? (s_x[i] - mx) - lse : __fdiv_rn((s_x[i] - mx) - lse, T);
    }
    if constexpr (PROC) {  // HF's order: processors, then temperature
        if (beam_proc_begin(bp, beam, row, V, tid)) process_row<BT_THREADS>(s_x, V, bp.proc, row, tid);
        __syncthreads();
        for (int i = tid; i < V; i += BT_THREADS) s_x[i] = __fdiv_rn(s_x[i], T);
    }
    __syncthreads();

    // top-k: keep w >= the k-th largest w (ties kept), k = max(top_k, min_keep)
    const int k = sp.top_k > 0 ? max(sp.top_k, sp.min_keep) : 0;
    if (k > 0 && k < V) {
        const uint32_t kth = radix_select<BT_THREADS, false>(V, (unsigned long long)k, tid, key_of, [](int) { return 1ull; }, sm.hist,
                                                             &sm.prefix, &sm.above);
        for (int i = tid; i < V; i += BT_THREADS)
            if (order_key(s_x[i]) < kth && s_x[i] == s_x[i]) s_x[i] = -INFINITY;  // NaN stays NaN: it ranks below -inf
        __syncthreads();
    }
    // top-p over fixed-point masses of e_i = exp(w_i - max w) (the rule of sample_publish_kernel); the min_keep largest w survive
    if (sp.top_p < 1.0f) {
        float m = -INFINITY;
        for (int i = tid; i < V; i += BT_THREADS) m = fmaxf(m, s_x[i] == s_x[i] ? s_x[i] : -INFINITY);
        const float wmax = block_reduce<true>(m, sm.w, tid);
        auto e_of = [&](int i) {
            const float w = s_x[i];
            return (w == w && w > -INFINITY) ? expf(w - wmax) : 0.f;
        };
        auto mass = [&](int i) { return mass_of(e_of(i)); };
        unsigned long long part = 0ull;
        for (int i = tid; i < V; i += BT_THREADS) part += mass(i);
        const unsigned long long total = block_sum<BT_THREADS, unsigned long long>(part, sm.wsum, tid);
        unsigned long long limit = (unsigned long long)((double)total * (double)sp.top_p);
        if (limit < 1ull) limit = 1ull;
        const uint32_t thr = radix_select<BT_THREADS, true>(V, limit, tid, [&](int i) { return __float_as_uint(e_of(i)); }, mass, sm.hist,
                                                            &sm.prefix, &sm.above);
        uint32_t kmin = 0xFFFFFFFFu;
        __syncthreads();  // every thread has read the last level's prefix before the next descent resets it
        if (sp.min_keep > 1)
            kmin = radix_select<BT_THREADS, false>(V, (unsigned long long)sp.min_keep, tid, key_of, [](int) { return 1ull; }, sm.hist,
                                                   &sm.prefix, &sm.above);
        __syncthreads();
        for (int i = tid; i < V; i += BT_THREADS) {
            const bool keep = __float_as_uint(e_of(i)) >= thr || order_key(s_x[i]) >= kmin;
            if (!keep && s_x[i] == s_x[i]) s_x[i] = -INFINITY;  // e_of reads only element i: in-place is safe per thread
        }
        __syncthreads();
    }
    // perturbed keys of the finite survivors
    const float run = beam_scores[beam];
    const uint32_t flat_base = (uint32_t)beam * (uint32_t)V;
    for (int i = tid; i < V; i += BT_THREADS) {
        const float w = s_x[i];
        if (ro.scores != nullptr) ro.scores[out0 + i] = w;  // the warped row, -inf outside the survivors
        if (w == w && w > -INFINITY) {
            const float acc = w + run;
            const unsigned long long r = philox_u64(sp.seed, sp.step, flat_base + (uint32_t)i);
            const double u = ((double)(r >> 11) + 0.5) * 0x1.0p-53;  // (0, 1)
            s_x[i] = (float)((double)acc - log(-log(u)));
        }
    }
    __syncthreads();
    row_top_candidates(s_x, V, Kr, (unsigned long long)j * V, tid, sm);

    unsigned long long* out = keys_out + (size_t)beam * K;
    float* out_s = scores_out + (size_t)beam * K;
    if (tid < Kr) {
        const unsigned long long me = sm.cand[tid];
        int rank = 0;
        for (int c = 0; c < Kr; ++c) rank += sm.cand[c] > me;
        const int i = (int)(0xFFFFFFFFu - (uint32_t)(me & 0xFFFFFFFFull) - (uint32_t)(j * V));
        const float kx = s_x[i];
        // a finite key is a survivor: its score is acc, recomputed with the same operations; -inf and NaN carry themselves. A
        // survivor was not banned by a processor, so of the processors only the repetition penalty can have changed it
        float w = (x[i] - mx) - lse;
        if constexpr (PROC) {
            const ProcRow& pr = bp.proc.rows[row];
            if (pr.on && pr.penalty != 1.0f && ((bp.proc.bits[(size_t)row * bp.proc.words + (i >> 5)] >> (i & 31)) & 1u))
                w = repetition_penalised(w, pr.penalty);
        }
        out[rank] = me;
        out_s[rank] = (kx == kx && kx > -INFINITY) ? __fdiv_rn(w, T) + run : kx;
    } else if (tid < K) {
        out[tid] = 0ull;
        out_s[tid] = -INFINITY;
    }
}

__global__ void __launch_bounds__(BM_THREADS)
beam_merge_kernel(const unsigned long long* __restrict__ keys, const float* __restrict__ scores, int nb, int K, int V,
                  float* __restrict__ out_scores, int32_t* __restrict__ out_tokens, int32_t* __restrict__ out_beams) {
    const int b = blockIdx.x;
    const unsigned long long* lists = keys + (size_t)b * nb * K;
    for (int c = threadIdx.x; c < nb * K; c += BM_THREADS) {
        const unsigned long long me = lists[c];
        if (me == 0ull) continue;
        int rank = 0;
        for (int r = 0; r < nb && rank < K; ++r) {  // elements of sorted list r above me: binary search
            const unsigned long long* l = lists + (size_t)r * K;
            int a = 0, z = K;
            while (a < z) {
                const int mid = (a + z) >> 1;
                if (l[mid] > me) a = mid + 1; else z = mid;
            }
            rank += a;
        }
        if (rank < K) {
            const uint32_t flat = 0xFFFFFFFFu - (uint32_t)(me & 0xFFFFFFFFull);
            // a sampled list carries each candidate's score beside its key; a greedy key is the score itself
            out_scores[(size_t)b * K + rank] = scores ? scores[(size_t)b * nb * K + c] : key_float((uint32_t)(me >> 32));
            out_tokens[(size_t)b * K + rank] = (int32_t)(flat % (uint32_t)V);
            out_beams[(size_t)b * K + rank] = (int32_t)(flat / (uint32_t)V);
        }
    }
}

__global__ void __launch_bounds__(CP_THREADS)
kv_copy_slots_kernel(uint8_t* __restrict__ k, uint8_t* __restrict__ v, float* __restrict__ ks, float* __restrict__ vs, KvCopyPairs p,
                     int row_begin, int H, int max_batch, int pitch, int row_bytes, int32_t* __restrict__ len_dev) {
    const int pair = blockIdx.z, lh = blockIdx.y >> 1, is_v = blockIdx.y & 1;
    const int l = lh / H, h = lh % H;
    const int src = p.src[pair], dst = p.dst[pair], end = p.end[pair];
    if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) len_dev[dst] = end;
    const int r0 = row_begin + blockIdx.x * CP_ROWS;
    const int r1 = min(r0 + CP_ROWS, end);
    if (r0 >= r1) return;
    const size_t slab_src = ((size_t)l * max_batch + src) * H + h, slab_dst = ((size_t)l * max_batch + dst) * H + h;
    uint8_t* base = is_v ? v : k;
    const uint4* from = reinterpret_cast<const uint4*>(base + (slab_src * pitch + r0) * row_bytes);
    uint4* to = reinterpret_cast<uint4*>(base + (slab_dst * pitch + r0) * row_bytes);
    const int n16 = (r1 - r0) * row_bytes / 16;
    for (int i = threadIdx.x; i < n16; i += CP_THREADS) to[i] = from[i];
    if (ks != nullptr) {
        float* sc = is_v ? vs : ks;
        for (int i = threadIdx.x; i < r1 - r0; i += CP_THREADS) sc[slab_dst * pitch + r0 + i] = sc[slab_src * pitch + r0 + i];
    }
}

__global__ void __launch_bounds__(CP_THREADS) proc_copy_slots_kernel(ProcState proc, KvCopyPairs p) {
    const int src = p.src[blockIdx.x], dst = p.dst[blockIdx.x];
    const int n = min(proc.rows[src].hist_len, proc.cap);
    const int32_t* hs = proc.hist + (size_t)src * proc.cap;
    int32_t* hd = proc.hist + (size_t)dst * proc.cap;
    for (int i = threadIdx.x; i < n; i += CP_THREADS) hd[i] = hs[i];
    const uint32_t* bs = proc.bits + (size_t)src * proc.words;
    uint32_t* bd = proc.bits + (size_t)dst * proc.words;
    for (int i = threadIdx.x; i < proc.words; i += CP_THREADS) bd[i] = bs[i];
    if (threadIdx.x == 0) proc.rows[dst] = proc.rows[src];
}

}  // namespace

size_t beam_topk_workspace_bytes(int B, int nb, int K) { return (size_t)B * nb * K * sizeof(unsigned long long); }

int beam_topk(const float* logits, const int32_t* row_of_beam, const float* beam_scores, int B, int nb, int V, int K,
              void* workspace, float* out_scores, int32_t* out_tokens, int32_t* out_beams, cudaStream_t stream,
              const BeamRowsOut& rows_out, const BeamProc& proc) {
    B2_CHECK_ARG(logits && beam_scores && workspace && out_scores && out_tokens && out_beams, "beam_topk: null argument");
    B2_CHECK_ARG(rows_out.fan >= 1, "beam_topk: %d output rows per beam", rows_out.fan);
    B2_CHECK_ARG(B >= 1 && nb >= 1 && nb <= 32, "beam_topk: B=%d nb=%d (1 <= nb <= 32)", B, nb);
    B2_CHECK_ARG(K >= 1 && K <= 128 && (long long)K <= (long long)nb * V, "beam_topk: K=%d outside [1, min(128, nb*V=%lld)]", K,
                 (long long)nb * V);
    const size_t smem = (size_t)V * sizeof(float);
    B2_CHECK_ARG(V >= 1 && smem <= 200 * 1024 && (long long)nb * V < 0xFFFFFFFFll,
                 "beam_topk: vocab %d exceeds the shared-memory staging of the kernel", V);
    const bool on = proc.proc.rows != nullptr;
    auto* kernel = on ? beam_row_topk_kernel<true> : beam_row_topk_kernel<false>;
    static size_t attr[2] = {0, 0};
    if (smem > attr[on]) {
        B2_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr[on] = smem;
    }
    auto* keys = reinterpret_cast<unsigned long long*>(workspace);
    kernel<<<dim3(nb, B), BT_THREADS, smem, stream>>>(logits, row_of_beam, beam_scores, nb, V, K, keys, rows_out, proc);
    B2_LAUNCH_CHECK();
    beam_merge_kernel<<<B, BM_THREADS, 0, stream>>>(keys, nullptr, nb, K, V, out_scores, out_tokens, out_beams);
    B2_LAUNCH_CHECK();
    return 0;
}

size_t beam_sample_workspace_bytes(int B, int nb, int K) {
    return (size_t)B * nb * K * (sizeof(unsigned long long) + sizeof(float));
}

int beam_sample(const float* logits, const int32_t* row_of_beam, const float* beam_scores, int B, int nb, int V, int K,
                const BeamSampleParams& sp, void* workspace, float* out_scores, int32_t* out_tokens, int32_t* out_beams,
                cudaStream_t stream, const BeamRowsOut& rows_out, const BeamProc& proc) {
    B2_CHECK_ARG(logits && beam_scores && workspace && out_scores && out_tokens && out_beams, "beam_sample: null argument");
    B2_CHECK_ARG(rows_out.fan == 1, "beam_sample: output rows are written once per beam row (fan %d)", rows_out.fan);
    B2_CHECK_ARG(B >= 1 && nb >= 1 && nb <= 32, "beam_sample: B=%d nb=%d (1 <= nb <= 32)", B, nb);
    B2_CHECK_ARG(K >= 1 && K <= 128 && (long long)K <= (long long)nb * V, "beam_sample: K=%d outside [1, min(128, nb*V=%lld)]", K,
                 (long long)nb * V);
    const size_t smem = (size_t)V * sizeof(float);
    B2_CHECK_ARG(V >= 1 && smem <= 200 * 1024 && (long long)B * nb * V <= 0xFFFFFFFFll,
                 "beam_sample: vocab %d exceeds the shared-memory staging of the kernel or B*nb*V the 32-bit Philox row", V);
    B2_CHECK_ARG(sp.temperature > 0.f, "beam_sample: temperature %g must be > 0", (double)sp.temperature);
    B2_CHECK_ARG(sp.top_p > 0.f && sp.top_p <= 1.f, "beam_sample: top_p %g outside (0, 1]", (double)sp.top_p);
    B2_CHECK_ARG(sp.top_k >= 0, "beam_sample: top_k %d must be >= 0", sp.top_k);
    B2_CHECK_ARG(sp.min_keep >= 1 && sp.min_keep <= K, "beam_sample: min_keep %d outside [1, K=%d]", sp.min_keep, K);
    const bool on = proc.proc.rows != nullptr;
    auto* kernel = on ? beam_row_sample_kernel<true> : beam_row_sample_kernel<false>;
    static size_t attr[2] = {0, 0};
    if (smem > attr[on]) {
        B2_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr[on] = smem;
    }
    auto* keys = reinterpret_cast<unsigned long long*>(workspace);
    float* scores = reinterpret_cast<float*>(keys + (size_t)B * nb * K);
    kernel<<<dim3(nb, B), BT_THREADS, smem, stream>>>(logits, row_of_beam, beam_scores, nb, V, K, sp, keys, scores, rows_out, proc);
    B2_LAUNCH_CHECK();
    beam_merge_kernel<<<B, BM_THREADS, 0, stream>>>(keys, scores, nb, K, V, out_scores, out_tokens, out_beams);
    B2_LAUNCH_CHECK();
    return 0;
}

int kv_copy_slots(void* k, void* v, float* kscale, float* vscale, const int32_t* src, const int32_t* dst, const int32_t* end, int n,
                  int row_begin, int L, int H, int max_batch, int pitch, int row_bytes, int32_t* len_dev, cudaStream_t stream) {
    B2_CHECK_ARG(row_bytes % 16 == 0 && row_begin >= 0, "kv_copy_slots: bad layout");
    for (int off = 0; off < n; off += KvCopyPairs::kMax) {
        const int c = n - off < KvCopyPairs::kMax ? n - off : KvCopyPairs::kMax;
        KvCopyPairs p;
        int rows = 1;
        for (int i = 0; i < c; ++i) {
            p.src[i] = src[off + i]; p.dst[i] = dst[off + i]; p.end[i] = end[off + i];
            rows = end[off + i] - row_begin > rows ? end[off + i] - row_begin : rows;
        }
        const dim3 grid((rows + CP_ROWS - 1) / CP_ROWS, L * H * 2, c);
        kv_copy_slots_kernel<<<grid, CP_THREADS, 0, stream>>>(reinterpret_cast<uint8_t*>(k), reinterpret_cast<uint8_t*>(v), kscale, vscale,
                                                               p, row_begin, H, max_batch, pitch, row_bytes, len_dev);
        B2_LAUNCH_CHECK();
    }
    return 0;
}

int proc_copy_slots(const ProcState& proc, const int32_t* src, const int32_t* dst, int n, cudaStream_t stream) {
    B2_CHECK_ARG(proc.rows != nullptr && n >= 0, "proc_copy_slots: bad argument");
    for (int off = 0; off < n; off += KvCopyPairs::kMax) {
        const int c = n - off < KvCopyPairs::kMax ? n - off : KvCopyPairs::kMax;
        KvCopyPairs p;
        for (int i = 0; i < c; ++i) { p.src[i] = src[off + i]; p.dst[i] = dst[off + i]; p.end[i] = 0; }
        proc_copy_slots_kernel<<<c, CP_THREADS, 0, stream>>>(proc, p);
        B2_LAUNCH_CHECK();
    }
    return 0;
}

}  // namespace b2
