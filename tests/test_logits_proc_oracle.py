"""CPU: pins oracle/logits_proc_oracle.py — the four history-aware processors against the INSTALLED transformers processors and
warpers composed in HF's order, the two placeholder rules on hand-built cases, and generate()'s argument handling of the
opt-in (config.b2_logits_processors)."""
import types

import numpy as np
import pytest
import torch

from oracle import logits_proc_oracle as P
from oracle import sampling_oracle as S


def _case(rng, V):
    L = int(rng.integers(1, 40))
    if rng.random() < 0.5:  # with repeats: ids from a small pool
        hist = rng.integers(0, min(V, 6), size=L).tolist()
    else:
        hist = rng.choice(V, size=min(L, V), replace=False).tolist()
    prompt_len = int(rng.integers(0, len(hist) + 1))
    x = (rng.standard_normal(V) * rng.uniform(0.5, 6)).astype(np.float32)
    x[rng.integers(0, V, size=3)] = 0.0  # exact zeros take the divide branch, like HF
    pen = float(rng.choice([0.5, 0.8, 1.0, 1.2, 1.7]))
    n = int(rng.integers(0, 5))
    eos = rng.choice(V, size=int(rng.integers(0, 3)), replace=False).tolist()
    mnt = int(rng.integers(0, 4))
    ml = int(rng.integers(0, len(hist) + 3))
    return x, hist, prompt_len, pen, n, eos, mnt, ml


@pytest.mark.parametrize("V", [50, 32000])
@pytest.mark.parametrize("seed", range(5))
def test_processed_scores_and_survivors_equal_hf(V, seed):
    rng = np.random.default_rng(1000 * seed + V)
    for _ in range(24):  # 2 V x 5 seeds x 24 = 240 random cases
        x, hist, plen, pen, n, eos, mnt, ml = _case(rng, V)
        mg = P.min_generated(mnt, ml, plen)
        ours = P.process(x, hist, plen, pen, n, mg, eos)
        hf = P.hf_processed(x, hist, plen, pen, n, mnt, ml, eos)
        assert np.array_equal(ours.view(np.uint32), hf.astype(np.float32).view(np.uint32)), (V, hist, plen, pen, n, eos, mnt, ml)
        # selection over the processed row: greedy, and every warper setting through sampling_oracle
        assert P.select(ours)[0] == S.greedy(hf)
        if np.isfinite(ours).any():
            T = float(rng.choice([0.3, 0.7, 1.0, 1.5]))
            k = int(rng.choice([0, 1, 5, 50]))
            p = float(rng.choice([0.3, 0.9, 1.0]))
            keep, _ = S.kept_mask(ours, T, k, p)
            keep &= np.isfinite(ours)  # a banned id can sit in the top-k set, but it carries no mass and is never drawn
            assert np.array_equal(keep, S.kept_set_hf(hf, T, k, p))


def test_ngram_rules_by_hand():
    x = np.zeros(10, dtype=np.float32)
    # bigram: history 1 2 3 1 -> the last id 1 was followed by 2 once: 2 is banned, nothing else
    out = P.process(x, [1, 2, 3, 1], 0, no_repeat_ngram_size=2)
    assert np.isneginf(out).nonzero()[0].tolist() == [2]
    # n = 1 bans every id of the history
    assert np.isneginf(P.process(x, [4, 4, 7], 0, no_repeat_ngram_size=1)).nonzero()[0].tolist() == [4, 7]
    # too short a history bans nothing: len + 1 < n
    assert not np.isneginf(P.process(x, [1, 1], 0, no_repeat_ngram_size=4)).any()
    # min_new_tokens / min_length count from the unspliced prompt length
    assert np.isneginf(P.process(x, [5, 6, 7], 2, min_gen=P.min_generated(2, 0, 2), eos_ids=[9]))[9]
    assert not np.isneginf(P.process(x, [5, 6, 7, 8], 2, min_gen=P.min_generated(2, 0, 2), eos_ids=[9])).any()
    assert P.min_generated(0, 7, 5) == 2 and P.min_generated(3, 7, 5) == 3


def test_placeholder_rules():
    V = 300
    x = np.linspace(-3, 3, V).astype(np.float32)
    # 1. the repetition penalty skips ids outside [0, V) (HF raises on -200) and still penalises the rest
    out = P.process(x, [-200, 5, -200, 290], 3, repetition_penalty=2.0)
    changed = np.nonzero(out != x)[0].tolist()
    assert changed == [5, 290]
    assert out[5] == np.float32(x[5] * np.float32(2.0)) and out[290] == np.float32(x[290] / np.float32(2.0))
    # 2. a ban that would fall on a placeholder is dropped (HF bans V - 200 by negative indexing) ...
    out = P.process(x, [7, -200, 8, 7], 4, no_repeat_ngram_size=2)
    assert np.isneginf(out).nonzero()[0].tolist() == []
    assert not np.isneginf(out[V - 200])
    # ... while placeholders still match one another: -200 -200 11, then -200 -200 -> 11 is banned
    out = P.process(x, [-200, -200, 11, 3, -200, -200], 6, no_repeat_ngram_size=3)
    assert np.isneginf(out).nonzero()[0].tolist() == [11]


def _stub(opt_in):
    """A model-shaped object with generate()'s argument handling (the methods need only `config`)."""
    from llava.model.language_model.llava_llama import LlavaLlamaForCausalLM as M

    stub = types.SimpleNamespace(config=types.SimpleNamespace(b2_logits_processors=opt_in))
    stub._LOGITS_PROCESSOR_ARGS = M._LOGITS_PROCESSOR_ARGS
    stub._logits_processors_on = types.MethodType(M._logits_processors_on, stub)
    return types.MethodType(M._logits_processor_arguments, stub)


def test_generate_arguments_with_and_without_opt_in(monkeypatch):
    monkeypatch.delenv("B2_LOGITS_PROCESSORS", raising=False)
    off = _stub(None)
    kw = {"repetition_penalty": 1.2, "no_repeat_ngram_size": 3}
    assert off(kw) == {} and kw == {"repetition_penalty": 1.2, "no_repeat_ngram_size": 3}  # left for the NotImplementedError
    monkeypatch.setenv("B2_LOGITS_PROCESSORS", "1")
    on_env = _stub(None)
    assert on_env({"repetition_penalty": 1.2})["repetition_penalty"] == 1.2
    on = _stub(True)
    kw = {"repetition_penalty": 1.2, "no_repeat_ngram_size": 3, "min_new_tokens": 4, "min_length": 9, "top_k": 5}
    got = on(kw)
    assert got == {"repetition_penalty": 1.2, "no_repeat_ngram_size": 3, "min_new_tokens": 4, "min_length": 9}
    assert kw == {"top_k": 5}
    assert on({"repetition_penalty": 1.0, "no_repeat_ngram_size": 0, "min_new_tokens": None, "min_length": 0}) == {}
    with pytest.raises(ValueError):
        on({"repetition_penalty": 0.0})
    with pytest.raises(ValueError):
        on({"no_repeat_ngram_size": -1})


def test_make_logits_proc_off_values_and_eos_limit():
    from llava._b2 import make_logits_proc

    ids = torch.zeros(3, dtype=torch.int64)  # never dereferenced for the off / error cases below
    assert make_logits_proc(ids) is None
    assert make_logits_proc(ids, min_generated=5, eos_ids=()) is None  # min_length / min_new_tokens without eos: no-op, as HF
    with pytest.raises(ValueError):
        make_logits_proc(ids, repetition_penalty=1.2, eos_ids=range(9))
    with pytest.raises(ValueError):  # the history must live on the device
        make_logits_proc(ids, repetition_penalty=1.2)


def test_beam_search_with_processors_is_refused(monkeypatch):
    """generate(num_beams > 1) with a processor raises NotImplementedError before any engine exists."""
    from llava.model.language_model.llava_llama import LlavaLlamaForCausalLM as M

    class Stub:
        config = types.SimpleNamespace(b2_logits_processors=True, b2_beam_search=4)
        _LOGITS_PROCESSOR_ARGS = M._LOGITS_PROCESSOR_ARGS
        _logits_processors_on = M._logits_processors_on
        _logits_processor_arguments = M._logits_processor_arguments
        _beam_search_cap = M._beam_search_cap

        def _ensure_engine(self):
            raise AssertionError("no engine should be built")

    with pytest.raises(NotImplementedError):
        M.generate.__wrapped__(Stub(), torch.ones(1, 4, dtype=torch.long), num_beams=2, no_repeat_ngram_size=3)
