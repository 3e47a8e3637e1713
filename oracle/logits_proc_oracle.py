"""CPU restatement (numpy) of the history-aware logits processing of the decode loop — TEST INFRASTRUCTURE ONLY (never imported
by the product; tests/ are the only callers).

What it restates: the HF processors `generate()` builds for repetition_penalty, no_repeat_ngram_size, min_length and
min_new_tokens, in the order of transformers 5.5 `GenerationMixin._get_logits_processor`:
  RepetitionPenaltyLogitsProcessor   every distinct id of the history: x < 0 ? x * p : x / p
  NoRepeatNGramLogitsProcessor       every n-gram of the history whose first n-1 ids equal the last n-1 ids bans its last id;
                                     nothing is banned while len(history) + 1 < n
  MinLengthLogitsProcessor           eos ids get -inf while len(history) < min_length
  MinNewTokensLengthLogitsProcessor  eos ids get -inf while generated < min_new_tokens
followed by the warpers that `sampling_oracle.kept_mask` / `sample_row` restate (temperature -> top-k -> top-p).

The history is the caller's prompt row as passed, then the generated tokens. Two deliberate differences from HF, both about ids
outside [0, V) (the IMAGE_TOKEN_INDEX = -200 placeholders of a LLaVA prompt):
  1. the repetition penalty skips them (HF's torch.gather raises on them);
  2. an n-gram ban that would fall on one is dropped (HF's scores[i, [-200]] = -inf bans id V - 200 by negative indexing).
Placeholders still take part in n-gram matching. `hf_processed` runs the installed processors for histories without them.
"""
import numpy as np

from . import sampling_oracle as so


def min_generated(min_new_tokens=0, min_length=0, prompt_len=0):
    """The one threshold the device keeps for both eos processors: eos is banned while generated < this."""
    return max(int(min_new_tokens or 0), int(min_length or 0) - int(prompt_len))


def process(scores, history, prompt_len, repetition_penalty=1.0, no_repeat_ngram_size=0, min_gen=0, eos_ids=()):
    """One row's processed scores (float32 [V]) for `history` (ints; prompt row then generated tokens)."""
    x = np.array(scores, dtype=np.float32, copy=True)
    V = x.shape[0]
    hist = [int(t) for t in history]
    p = np.float32(repetition_penalty)
    if p != np.float32(1.0):
        ids = np.unique(np.asarray([t for t in hist if 0 <= t < V], dtype=np.int64))
        v = x[ids]
        x[ids] = np.where(v < 0, v * p, v / p).astype(np.float32)
    n = int(no_repeat_ngram_size or 0)
    L = len(hist)
    if n > 0 and L + 1 >= n:
        tail = hist[L - n + 1:] if n > 1 else []
        for s in range(L - n + 1):
            if hist[s:s + n - 1] == tail and 0 <= hist[s + n - 1] < V:
                x[hist[s + n - 1]] = -np.inf
    if eos_ids and L - prompt_len < min_gen:
        for e in eos_ids:
            if 0 <= e < V:
                x[e] = -np.inf
    return x


def select(processed, do_sample=False, temperature=1.0, top_k=0, top_p=1.0, seed=0, index=0, row=0):
    """The token the device picks from processed scores: argmax, or the Philox draw of sampling_oracle."""
    if not do_sample:
        return so.greedy(processed), None
    return so.sample_row(processed, temperature, top_k, top_p, seed, index, row)


def hf_processed(scores, history, prompt_len, repetition_penalty=1.0, no_repeat_ngram_size=0, min_new_tokens=None,
                 min_length=0, eos_ids=()):
    """The same scores through the INSTALLED transformers processors, composed in HF's order (ids must be in [0, V))."""
    import torch
    from transformers.generation.logits_process import (MinLengthLogitsProcessor, MinNewTokensLengthLogitsProcessor,
                                                        NoRepeatNGramLogitsProcessor, RepetitionPenaltyLogitsProcessor)

    ids = torch.tensor([list(history)], dtype=torch.long)
    s = torch.tensor(np.asarray(scores, dtype=np.float32))[None].clone()
    if repetition_penalty is not None and repetition_penalty != 1.0:
        s = RepetitionPenaltyLogitsProcessor(float(repetition_penalty))(ids, s)
    if no_repeat_ngram_size:
        s = NoRepeatNGramLogitsProcessor(int(no_repeat_ngram_size))(ids, s)
    eos = list(eos_ids)
    if eos and min_length:
        s = MinLengthLogitsProcessor(int(min_length), eos)(ids, s)
    if eos and min_new_tokens:
        s = MinNewTokensLengthLogitsProcessor(int(prompt_len), int(min_new_tokens), eos)(ids, s)
    return s[0].numpy()
