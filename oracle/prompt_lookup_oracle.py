"""Prompt-lookup speculative decoding in numpy: the draft rule of csrc/sampling.cu's prompt_lookup_kernel and the acceptance rule
of sample_publish's multi-row mode.

draft(): HF 5.5 PromptLookupCandidateGenerator.get_candidates (generation/candidate_generator.py) over one history row, with one
deliberate difference: the draft also ends before the first id outside [0, V) (an IMAGE_TOKEN_INDEX placeholder, which HF would
feed to the model). HF's fake-logits filter for logits processors is not reproduced (processors are not combined with lookup).

accept(): HF's n_matches rule (generation/utils.py, assisted decoding without candidate logits), capped so that a generation
never publishes more than max_new_tokens tokens."""
import numpy as np


def draft(hist, K, max_ngram, max_length, eos_ids=(), vocab=None):
    """hist: the history (prompt ids, then every published token; the last one is the pending token). Returns the draft list."""
    hist = [int(t) for t in hist]
    L = len(hist)
    if max_length == L + 1:
        return []
    for n in range(min(max_ngram, L - 1), 0, -1):
        tail = hist[L - n:]
        for s in range(0, L - n + 1):
            if hist[s:s + n] != tail:
                continue
            start = s + n
            end = min(start + K, L, max_length)
            if start < end:
                out = []
                for t in hist[start:end]:
                    if t in eos_ids or (vocab is not None and not 0 <= t < vocab):
                        break
                    out.append(t)
                return out
    return []


def accept(drafted, selected, hist_len, max_length, published, max_new_tokens):
    """Tokens a step publishes. drafted: the step's draft (d tokens); selected: the token chosen from each of its d + 1 rows;
    hist_len: history length with the pending token; published: tokens of the generation published before the step."""
    d = len(drafted)
    m = 0
    while m < d and int(selected[m]) == int(drafted[m]):
        m += 1
    if d > 0 and m == d and hist_len + d >= max_length:  # is_done_candidate
        m -= 1
    n = min(m + 1, max_new_tokens - published)
    return [int(t) for t in selected[:n]]


def hf_n_matches(candidate_new_tokens, selected_tokens, is_done_candidate):
    """HF's formula, verbatim in numpy, for comparison with accept()."""
    c = np.asarray(candidate_new_tokens)[None, :]
    s = np.asarray(selected_tokens)[None, :]
    n = int(((~(c == s[:, :-1])).cumsum(axis=-1) < 1).sum())
    if is_done_candidate and n == c.shape[1]:
        n -= 1
    return n
