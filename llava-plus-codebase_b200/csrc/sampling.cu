// Token selection + publication for the decode loop (one CTA per sample):
//
//   * greedy: argmax over the fp32 last-position logits (first occurrence wins, like torch.argmax) — the HF
//     GenerationMixin greedy_search step the reference's callers use with do_sample=False
//     (llava/eval/model_vqa_loader.py:98-106, llava/serve/model_worker.py:161 when temperature <= 0.001);
//   * sampling: HF's warper chain for do_sample=True as invoked by llava/serve/model_worker.py:155-185
//     (temperature, top_p; top_k from the GenerationConfig default): logits / T -> keep the k largest (ties kept) ->
//     softmax over the survivors -> nucleus: keep token i iff the probability mass STRICTLY above it is < top_p
//     (== TopPLogitsWarper's "remove where ascending cumsum <= 1 - top_p", at least one token kept) -> draw from the
//     renormalised survivors with a counter-based Philox4x32-10 stream keyed by (seed; token index, row).
//     Everything after exp() is integer arithmetic (probabilities as 2^-40 fixed point, radix select over float bit
//     patterns, integer prefix sums), so a draw is reproducible bit for bit from (logits, seed, index) whatever the
//     thread schedule (the test suite carries a numpy restatement).
//   * publication: the chosen token goes to kv->tok (next step's input, stays on the device), to the step's slot
//     in out_tokens, and — tagged with the generation's epoch — into a ring in MAPPED PINNED HOST memory, so the host
//     loop of generate() (streamer / stopping criteria, llava/serve/model_worker.py:166-188) reads token t while the
//     device is already running step t+k: no D2H copy, no stream sync per token.
#include <limits.h>
#include <math.h>

#include "common.cuh"
#include "kernels.h"
#include "logits_proc.cuh"
#include "select.cuh"

namespace b2 {
namespace {

constexpr int SP_THREADS = 1024;

__device__ __forceinline__ uint32_t order_key(float x) {  // monotone float -> uint (x < y  <=>  key(x) < key(y))
    const uint32_t u = __float_as_uint(x);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// argmax with torch.argmax tie-breaking (value desc, index asc), NaN skipped; result valid in every thread
__device__ __forceinline__ int block_argmax(const float* row, int V, int tid, float* s_v, int* s_i, float* max_out) {
    float best = -INFINITY;
    int bi = INT_MAX;
    for (int i = tid; i < V; i += SP_THREADS) {
        const float v = row[i];
        if (v == v && (bi == INT_MAX || v > best)) { best = v; bi = i; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
    }
    __syncthreads();
    if ((tid & 31) == 0) { s_v[tid >> 5] = best; s_i[tid >> 5] = bi; }
    __syncthreads();
    best = s_v[0]; bi = s_i[0];
    for (int w = 1; w < SP_THREADS / 32; ++w) {
        const float ov = s_v[w];
        const int oi = s_i[w];
        if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
    }
    if (max_out) *max_out = best;
    return bi == INT_MAX ? 0 : bi;
}

// HF 5.5 assisted decoding's acceptance (generation/utils.py, n_matches): the draft's leading tokens that equal the tokens
// selected at the rows before them are kept, plus the token selected after the last match; a draft that reaches max_length
// gives up its last match. Runs in the last CTA of the step, after every row's selection is in spec->sel.
__device__ void spec_accept(SpecState* spec, SampleState* st, int pub, int32_t* tok, int32_t* cur_len, int32_t* hist,
                            volatile int32_t* ring, int ring_cap) {
    const int d = spec->draft_len;
    const volatile int32_t* sel = spec->sel;
    int n = 0;  // a step queued after the generation published its max_new tokens changes nothing
    if (pub < spec->max_new) {
        int m = 0;
        while (m < d && sel[m] == spec->rows[1 + m]) ++m;
        const int L = spec->hist_len + 1;  // history length with the pending token
        if (d > 0 && m == d && L + d >= spec->prompt_len + spec->max_new) m -= 1;  // is_done_candidate
        n = min(m + 1, spec->max_new - pub);
        for (int i = 0; i + 1 < n; ++i) hist[L + i] = sel[i];
        tok[0] = sel[n - 1];
        spec->hist_len += n;
        cur_len[0] += n;
        st->pub_counter = pub + n;
        spec->steps += 1;
        spec->drafted += d;
        spec->accepted += n - 1;
    }
    spec->retired += 1;
    // the mirror before the ring: a host that has read token t finds published > t and the steps retired up to it there
    if (spec->mirror != nullptr) {
        volatile int* mr = spec->mirror;
        mr[0] = spec->steps; mr[1] = spec->drafted; mr[2] = spec->accepted; mr[3] = cur_len[0]; mr[4] = spec->retired;
        __threadfence_system();
        mr[5] = pub + n;
        __threadfence_system();
    }
    for (int i = 0; i < n; ++i) {
        if (ring != nullptr && st->tag != 0) {
            const int t = pub + i;
            const int tag = 1 + (st->tag - 1 + t / ring_cap) % 2047;
            ring[t % ring_cap] = (tag << 20) | (sel[i] & 0xFFFFF);
        }
    }
    __threadfence_system();
}

__global__ void __launch_bounds__(SP_THREADS, 1)
sample_publish_kernel(const float* __restrict__ logits, int V, int B, SampleState* st, RowState* rows, int32_t* tok, int32_t* out_tokens,
                      int32_t* step_counter, int32_t* cur_len, volatile int32_t* ring, int ring_cap, int flags,
                      int step_offset, ProcState proc, float* processed_out, SpecState* spec) {
    extern __shared__ __align__(16) uint8_t sp_smem[];
    float* s_x = reinterpret_cast<float*>(sp_smem);
    __shared__ unsigned long long s_hist[256];
    __shared__ unsigned long long s_wsum[SP_THREADS / 32];
    __shared__ unsigned long long s_above, s_target;
    __shared__ uint32_t s_prefix;
    __shared__ float s_v[SP_THREADS / 32];
    __shared__ int s_i[SP_THREADS / 32];
    __shared__ int s_choice;

    const int tid = threadIdx.x, b = blockIdx.x;
    pdl_trigger();
    pdl_wait();  // logits / tok / the selection state are outputs of earlier kernels in the stream
    const bool per_row = st->per_row != 0;
    const bool active = !per_row || rows[b].active != 0;
    const int do_sample = per_row ? rows[b].do_sample : st->do_sample;
    const float temperature = per_row ? rows[b].temperature : st->temperature;
    const float top_p = per_row ? rows[b].top_p : st->top_p;
    const int top_k = per_row ? rows[b].top_k : st->top_k;
    const unsigned long long seed = per_row ? rows[b].seed : st->seed;
    const int pub = st->pub_counter;
    // multi-row acceptance: row b is token pub + b of the generation; rows past the draft (and every row once the generation
    // has published its max_new tokens) are not selected
    const int draw = per_row ? rows[b].index : pub + (spec ? b : 0);
    const uint32_t draw_row = spec ? 0u : (uint32_t)b;
    const bool spec_idle = spec != nullptr && (b > spec->draft_len || pub >= spec->max_new);
    const bool select = active && (flags & SP_SELECT) && !spec_idle;
    const bool proc_on = spec == nullptr && proc.rows != nullptr && proc.rows[b].on != 0 && active;
    int choice = 0;
    const float* row = logits + (size_t)b * V;
    // output rows of token `pub` (generate(output_scores / output_logits)); a multi-row acceptance or an idle slot writes none
    float* srow = nullptr;
    if (select && spec == nullptr && !per_row && pub < st->out_cap) {
        const size_t off = ((size_t)pub * B + b) * V;
        if (st->out_scores != nullptr) srow = st->out_scores + off;
        if (st->out_logits != nullptr)
            for (int i = tid; i < V; i += SP_THREADS) st->out_logits[off + i] = row[i];
    }
    if (select && (proc_on || processed_out != nullptr)) {
        // stage the row and run the processors in HF's order over it; selection below reads the staged row
        for (int i = tid; i < V; i += SP_THREADS) s_x[i] = row[i];
        if (proc_on) process_row<SP_THREADS>(s_x, V, proc, b, tid);
        __syncthreads();
        if (processed_out != nullptr)
            for (int i = tid; i < V; i += SP_THREADS) processed_out[(size_t)b * V + i] = s_x[i];
        row = s_x;
    }

    if (!active) {
        choice = tok[b];  // an idle slot keeps its token; nothing is selected or counted for it
    } else if (spec_idle) {
        choice = 0;
    } else if (!(flags & SP_SELECT)) {
        choice = tok[b];  // already chosen by the producer of `tok` (decode megakernel's fused argmax)
    } else if (!do_sample) {
        if (srow != nullptr)  // greedy: the score row is the processed row the argmax reads
            for (int i = tid; i < V; i += SP_THREADS) srow[i] = row[i];
        choice = block_argmax(row, V, tid, s_v, s_i, nullptr);
    } else {
        // the score row is HF's x / T (IEEE division, TemperatureLogitsWarper); the draw keeps multiplying by 1 / T. Tokens the
        // filters below remove become -inf in it where the draw's own rule removes them
        if (srow != nullptr)
            for (int i = tid; i < V; i += SP_THREADS) srow[i] = __fdiv_rn(row[i], temperature);
        const float inv_t = 1.0f / temperature;
        for (int i = tid; i < V; i += SP_THREADS) s_x[i] = row[i] * inv_t;  // in place when staged: each thread its own i
        __syncthreads();
        // ---- top-k: keep everything >= the k-th largest scaled logit (ties kept, like TopKLogitsWarper) ----
        const int k = top_k;
        if (k > 0 && k < V) {
            const uint32_t kth = radix_select<SP_THREADS, false>(
                V, (unsigned long long)k, tid, [&](int i) { return order_key(s_x[i]); }, [](int) { return 1ull; }, s_hist,
                &s_prefix, &s_above);
            for (int i = tid; i < V; i += SP_THREADS)
                if (order_key(s_x[i]) < kth) {
                    s_x[i] = -INFINITY;
                    if (srow != nullptr) srow[i] = -INFINITY;
                }
            __syncthreads();
        }
        // ---- softmax numerators over the survivors: e_i = exp(x_i - max) (max itself always survives) ----
        float mx;
        block_argmax(s_x, V, tid, s_v, s_i, &mx);
        for (int i = tid; i < V; i += SP_THREADS) {
            const float x = s_x[i];
            s_x[i] = (x == x && x > -INFINITY) ? expf(x - mx) : 0.f;
        }
        __syncthreads();
        // ---- top-p over the fixed-point masses ----
        if (top_p < 1.0f) {
            unsigned long long part = 0ull;
            for (int i = tid; i < V; i += SP_THREADS) part += mass_of(s_x[i]);
            const unsigned long long total = block_sum<SP_THREADS, unsigned long long>(part, s_wsum, tid);
            unsigned long long limit = (unsigned long long)((double)total * (double)(top_p > 0.f ? top_p : 0.f));
            if (limit < 1ull) limit = 1ull;  // min_tokens_to_keep = 1: the largest probability always survives
            const uint32_t thr = radix_select<SP_THREADS, true>(
                V, limit, tid, [&](int i) { const float x = s_x[i]; return __float_as_uint(x > 0.f ? x : 0.f); },
                [&](int i) { return mass_of(s_x[i]); }, s_hist, &s_prefix, &s_above);
            for (int i = tid; i < V; i += SP_THREADS) {
                const float x = s_x[i];
                if (__float_as_uint(x > 0.f ? x : 0.f) < thr) {
                    s_x[i] = 0.f;
                    if (srow != nullptr) srow[i] = -INFINITY;
                }
            }
            __syncthreads();
        }
        // ---- inverse CDF in index order: thread t owns the contiguous chunk [t*C, (t+1)*C) ----
        const int C = ((V + SP_THREADS - 1) / SP_THREADS) | 1;  // odd stride: conflict-free shared-memory walks
        const int lo = tid * C, hi = min(lo + C, V);
        unsigned long long mine = 0ull;
        for (int i = lo; i < hi; ++i) mine += mass_of(s_x[i]);
        // exclusive prefix over threads: warp scan + scan of the 32 warp totals
        unsigned long long incl = mine;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long up = __shfl_up_sync(0xffffffffu, incl, o);
            if ((tid & 31) >= o) incl += up;
        }
        if ((tid & 31) == 31) s_wsum[tid >> 5] = incl;
        __syncthreads();
        unsigned long long warp_base = 0ull, total = 0ull;
        for (int w = 0; w < SP_THREADS / 32; ++w) {
            if (w < (tid >> 5)) warp_base += s_wsum[w];
            total += s_wsum[w];
        }
        const unsigned long long excl = warp_base + incl - mine;
        if (tid == 0) {
            s_target = total ? __umul64hi(total, philox_u64(seed, (uint32_t)draw, draw_row)) : 0ull;
            s_choice = 0;
        }
        __syncthreads();
        const unsigned long long target = s_target;
        if (mine != 0ull && target >= excl && target < excl + mine) {  // exactly one thread
            unsigned long long run = excl;
            int pick = lo;
            for (int i = lo; i < hi; ++i) {
                const unsigned long long m = mass_of(s_x[i]);
                if (m != 0ull && target < run + m) { pick = i; break; }
                run += m;
            }
            s_choice = pick;
        }
        __syncthreads();
        choice = s_choice;
    }

    if (tid == 0 && spec != nullptr) {
        spec->sel[b] = choice;
        __threadfence();
        if (atomicAdd(&st->done, 1u) == (unsigned)B - 1u) {  // last row of the step: accept
            st->done = 0u;
            spec_accept(spec, st, pub, tok, cur_len, proc.hist, ring, ring_cap);
        }
    } else if (tid == 0) {
        if ((flags & SP_SELECT) && active) tok[b] = choice;
        if (per_row && active) rows[b].index = draw + 1;
        if (proc_on) {  // the chosen token joins the row's history
            ProcRow& pr = proc.rows[b];
            const int n = pr.hist_len;
            if (n < proc.cap) {
                proc.hist[(size_t)b * proc.cap + n] = choice;
                pr.hist_len = n + 1;
            }
            if (choice >= 0 && choice < V) proc.bits[(size_t)b * proc.words + (choice >> 5)] |= 1u << (choice & 31);
        }
        if (flags & SP_WRITE_OUT) out_tokens[(size_t)(*step_counter + step_offset) * B + b] = choice;
        if (ring != nullptr && st->tag != 0) {
            // the tag advances every time the ring wraps, so an entry left from ring_cap steps ago is never taken for a new one
            const int tag = 1 + (st->tag - 1 + pub / ring_cap) % 2047;
            ring[(size_t)(pub % ring_cap) * B + b] = (tag << 20) | (choice & 0xFFFFF);
            __threadfence_system();
        }
        __threadfence();
        if (atomicAdd(&st->done, 1u) == (unsigned)B - 1u) {  // last row of this step: advance the counters
            st->done = 0u;
            st->pub_counter = pub + 1;
            if (flags & SP_BUMP) {
                *step_counter += 1;
                for (int i = 0; i < B; ++i)
                    if (!per_row || rows[i].active) cur_len[i] += 1;
            }
        }
    }
}

// HF 5.5 PromptLookupCandidateGenerator.get_candidates over hist[0, L) (the pending token appended at hist_len): n-gram sizes
// min(ngram, L - 1) .. 1; for each, the leftmost earlier occurrence of the last n ids with a continuation wins; the draft is
// hist[start, min(start + K, L, max_length)), cut before the first eos id and (unlike HF, which would feed the -200 image
// placeholder to the model) before the first id outside [0, V)
constexpr int LK_THREADS = 256;
__global__ void __launch_bounds__(LK_THREADS)
prompt_lookup_kernel(int32_t* hist, SpecState* spec, const SampleState* st, const int32_t* tok, int V, int R) {
    __shared__ int s_start;
    const int tid = threadIdx.x;
    pdl_trigger();
    pdl_wait();  // tok, the history and the counters are written by the previous step's acceptance
    const int h0 = spec->hist_len, K = spec->K;
    const int L = h0 + 1;
    const int pending = tok[0];
    const int max_length = spec->prompt_len + spec->max_new;
    if (tid == 0) hist[h0] = pending;
    __syncthreads();
    int start = -1, end = -1;
    if (st->pub_counter < spec->max_new && max_length != L + 1) {
        const int lim = min(L, max_length);  // a match must start its continuation before lim
        for (int n = min(spec->ngram, L - 1); n >= 1; --n) {
            if (tid == 0) s_start = INT_MAX;
            __syncthreads();
            const int32_t* tail = hist + (L - n);
            for (int s = tid; s + n < lim; s += LK_THREADS) {
                bool match = true;
                for (int i = 0; i < n && match; ++i) match = hist[s + i] == tail[i];
                if (match) atomicMin(&s_start, s);
            }
            __syncthreads();
            const int s0 = s_start;
            __syncthreads();
            if (s0 != INT_MAX) {
                start = s0 + n;
                end = min(start + K, lim);
                break;
            }
        }
    }
    if (tid == 0) {
        int d = 0;
        for (int i = start; start >= 0 && i < end; ++i) {
            const int id = hist[i];
            bool stop = id < 0 || id >= V;
            for (int e = 0; e < spec->n_eos; ++e) stop = stop || id == spec->eos[e];
            if (stop) break;
            spec->rows[1 + d++] = id;
        }
        spec->rows[0] = pending;
        for (int j = 1 + d; j < R; ++j) spec->rows[j] = pending;
        spec->draft_len = d;
    }
}

__global__ void __launch_bounds__(SP_THREADS, 1)
proc_seed_kernel(ProcState proc, int row, ProcRow v, const int64_t* __restrict__ ids, int len, int first_token, int V) {
    uint32_t* bits = proc.bits + (size_t)row * proc.words;
    int32_t* hist = proc.hist + (size_t)row * proc.cap;
    const int tid = threadIdx.x;
    for (int i = tid; i < proc.words; i += SP_THREADS) bits[i] = 0u;
    __syncthreads();
    for (int i = tid; i <= len; i += SP_THREADS) {
        const long long id = i < len ? ids[i] : (long long)first_token;
        if (i == len && first_token < 0) break;
        hist[i] = (int32_t)id;
        if (id >= 0 && id < V) atomicOr(&bits[id >> 5], 1u << (id & 31));
    }
    if (tid == 0) proc.rows[row] = v;
}

// the output rows of a token the megakernel's fused argmax chose and published: grid (chunks, B), 256 threads
constexpr int PR_THREADS = 256, PR_CHUNKS = 16;
__global__ void __launch_bounds__(PR_THREADS)
publish_rows_kernel(const float* __restrict__ logits, int V, int B, const SampleState* st) {
    pdl_trigger();
    pdl_wait();  // the logits and the publication counter are written by the megakernel before this launch
    const int t = st->pub_counter - 1, b = blockIdx.y;
    if (t < 0 || t >= st->out_cap) return;
    const float* row = logits + (size_t)b * V;
    const size_t off = ((size_t)t * B + b) * V;
    float* s = st->out_scores;
    float* l = st->out_logits;
    for (int i = blockIdx.x * PR_THREADS + threadIdx.x; i < V; i += PR_CHUNKS * PR_THREADS) {
        const float x = row[i];
        if (s != nullptr) s[off + i] = x;
        if (l != nullptr) l[off + i] = x;
    }
}

__global__ void sample_state_set_kernel(SampleState* st, SampleState v) {
    if (threadIdx.x == 0) *st = v;
}
__global__ void row_state_set_kernel(RowState* row, RowState v, int32_t* tok, int token) {
    if (threadIdx.x == 0) {
        *row = v;
        if (tok != nullptr) *tok = token;
    }
}

}  // namespace

size_t sample_smem_bytes(int V) { return (size_t)V * sizeof(float); }

int sample_state_set(SampleState* st_dev, const SampleState& v, cudaStream_t stream) {
    sample_state_set_kernel<<<1, 32, 0, stream>>>(st_dev, v);
    B2_LAUNCH_CHECK();
    return 0;
}

int publish_rows(const float* logits, int V, int B, const SampleState* st_dev, cudaStream_t stream) {
    B2_CHECK_ARG(logits != nullptr && st_dev != nullptr && B >= 1 && V >= 1, "publish_rows: bad argument");
    B2_CUDA_CHECK(launch_pdl(publish_rows_kernel, dim3(PR_CHUNKS, B), dim3(PR_THREADS), 0, stream, logits, V, B, st_dev));
    B2_LAUNCH_CHECK();
    return 0;
}

int row_state_set(RowState* row_dev, const RowState& v, int32_t* tok_dev, int token, cudaStream_t stream) {
    row_state_set_kernel<<<1, 32, 0, stream>>>(row_dev, v, tok_dev, token);
    B2_LAUNCH_CHECK();
    return 0;
}

int proc_seed(const ProcState& proc, int row, const ProcRow& v, const int64_t* ids, int len, int first_token, int V,
              cudaStream_t stream) {
    B2_CHECK_ARG(proc.rows != nullptr && len >= 0 && (len == 0 || ids != nullptr), "proc_seed: bad argument");
    B2_CHECK_ARG(len + (first_token >= 0 ? 1 : 0) <= proc.cap, "proc_seed: history of %d ids exceeds its capacity %d", len, proc.cap);
    proc_seed_kernel<<<1, SP_THREADS, 0, stream>>>(proc, row, v, ids, len, first_token, V);
    B2_LAUNCH_CHECK();
    return 0;
}

int prompt_lookup(int32_t* hist, SpecState* spec, const SampleState* st, const int32_t* tok, int V, int R, cudaStream_t stream) {
    B2_CHECK_ARG(hist != nullptr && spec != nullptr && st != nullptr && tok != nullptr && R >= 2 && R <= kSpecMaxRows,
                 "prompt_lookup: bad argument");
    B2_CUDA_CHECK(launch_pdl(prompt_lookup_kernel, dim3(1), dim3(LK_THREADS), 0, stream, hist, spec, st, tok, V, R));
    B2_LAUNCH_CHECK();
    return 0;
}

int sample_publish(const float* logits, int V, int B, SampleState* st_dev, RowState* rows_dev, int32_t* tok, int32_t* out_tokens,
                   int32_t* step_counter, int32_t* cur_len, int32_t* ring_dev, int ring_cap, int flags, int step_offset,
                   const ProcState& proc, float* processed_out, cudaStream_t stream, SpecState* spec) {
    B2_CHECK_ARG(B >= 1 && V >= 1 && st_dev != nullptr && tok != nullptr, "sample_publish: bad argument");
    B2_CHECK_ARG(spec == nullptr || (B <= kSpecMaxRows && flags == SP_SELECT && proc.hist != nullptr && rows_dev == nullptr),
                 "sample_publish: bad multi-row acceptance");
    B2_CHECK_ARG(V < (1 << 20), "sample_publish: vocab %d does not fit the 20-bit token field of the host ring", V);
    const size_t smem = sample_smem_bytes(V);
    B2_CHECK_ARG(smem <= 200 * 1024, "sample_publish: vocab %d exceeds the shared-memory staging of the sampling kernel", V);
    static size_t attr = 0;
    if (smem > attr) {
        B2_CUDA_CHECK(cudaFuncSetAttribute(sample_publish_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr = smem;
    }
    B2_CUDA_CHECK(launch_pdl(sample_publish_kernel, dim3(B), dim3(SP_THREADS), smem, stream, logits, V, B, st_dev, rows_dev, tok,
                             out_tokens, step_counter, cur_len, ring_dev, ring_cap, flags, step_offset, proc, processed_out, spec));
    B2_LAUNCH_CHECK();
    return 0;
}

}  // namespace b2
