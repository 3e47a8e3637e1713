// HF's history-aware logits processors over one row staged in shared memory, shared by token selection (sampling.cu, over
// logits) and beam-candidate selection (beam.cu, over log-probabilities, as HF's _beam_search applies them).
#pragma once
#include <stdint.h>

#include "kernels.h"

namespace b2 {

// RepetitionPenaltyLogitsProcessor on one score of a history id: IEEE fp32
__device__ __forceinline__ float repetition_penalised(float x, float p) { return x < 0.f ? __fmul_rn(x, p) : __fdiv_rn(x, p); }

// HF's processors over the staged row s_x against history row b of `proc`, in transformers' order (repetition -> no-repeat-ngram
// -> min_length / min_new_tokens). Ids of the history outside [0, V) (IMAGE_TOKEN_INDEX placeholders) are never penalised or
// banned. Every thread of the block calls it; the row's ProcRow and history must be final before the call.
template <int THREADS>
__device__ __forceinline__ void process_row(float* s_x, int V, const ProcState& proc, int b, int tid) {
    const ProcRow& pr = proc.rows[b];
    const int L = pr.hist_len, n = pr.ngram;
    const float p = pr.penalty;
    const int32_t* hist = proc.hist + (size_t)b * proc.cap;
    const uint32_t* bits = proc.bits + (size_t)b * proc.words;
    __syncthreads();  // the staged row is complete
    if (p != 1.0f) {  // once per distinct id of the history
        for (int i = tid; i < V; i += THREADS)
            if ((bits[i >> 5] >> (i & 31)) & 1u) s_x[i] = repetition_penalised(s_x[i], p);
        __syncthreads();
    }
    if (n > 0 && L + 1 >= n) {  // NoRepeatNGramLogitsProcessor: every n-gram whose first n-1 ids equal the last n-1 ids
        const int32_t* tail = hist + (L - n + 1);
        for (int s = tid; s <= L - n; s += THREADS) {
            bool match = true;
            for (int j = 0; j < n - 1 && match; ++j) match = hist[s + j] == tail[j];
            const int t = hist[s + n - 1];
            if (match && t >= 0 && t < V) s_x[t] = -INFINITY;  // idempotent: threads may ban the same id
        }
    }
    if (L - pr.prompt_len < pr.min_gen && tid < pr.n_eos) {  // MinLength / MinNewTokensLength
        const int e = pr.eos[tid];
        if (e >= 0 && e < V) s_x[e] = -INFINITY;
    }
}

}  // namespace b2
