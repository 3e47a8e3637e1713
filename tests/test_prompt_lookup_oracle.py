"""CPU: prompt-lookup speculative decoding. The numpy draft and acceptance rules (oracle/prompt_lookup_oracle.py) against the
installed transformers' PromptLookupCandidateGenerator and n_matches formula, generate()'s argument handling, and the host loop
(`_stream_decode`) over a stand-in engine whose steps publish several tokens each."""
import random
import types

import pytest
import torch

from oracle import prompt_lookup_oracle as PL

transformers_cg = pytest.importorskip("transformers.generation.candidate_generator")


def _hf_draft(hist, K, ngram, max_length, eos):
    gen = transformers_cg.PromptLookupCandidateGenerator(
        eos_token_id=torch.tensor(sorted(eos) if eos else [-12345]), num_output_tokens=K, max_matching_ngram_size=ngram,
        max_length=max_length)
    ids = torch.tensor([hist], dtype=torch.long)
    out, _ = gen.get_candidates(ids)
    return out[0, len(hist):].tolist()


@pytest.mark.parametrize("seed", range(6))
def test_draft_equals_hf(seed):
    rng = random.Random(seed)
    for _ in range(60):
        V = rng.choice([4, 8, 30])  # small vocabularies: many repeated n-grams
        L = rng.randint(1, 60)
        hist = [rng.randrange(V) for _ in range(L)]
        K, ngram = rng.randint(1, 15), rng.randint(1, 4)
        eos = set(rng.sample(range(V), rng.randint(0, 2)))
        max_length = rng.choice([L + 1, L + 2, L + rng.randint(1, 40), max(1, L - rng.randint(0, 5))])
        got = PL.draft(hist, K, ngram, max_length, eos, vocab=V)
        assert got == _hf_draft(hist, K, ngram, max_length, eos), (hist, K, ngram, max_length, eos)


def test_draft_by_hand_and_placeholders():
    #        0  1  2  3  4  5  6  7
    hist = [5, 6, 7, 8, 9, 5, 6]
    assert PL.draft(hist, 3, 2, 100) == [7, 8, 9]          # the 2-gram (5, 6) recurs at 0
    assert PL.draft(hist, 10, 2, 100) == [7, 8, 9, 5, 6]   # clamped at the history's end
    assert PL.draft(hist, 3, 2, 100, eos_ids={8}) == [7]   # cut before the eos id
    assert PL.draft(hist, 3, 2, 8) == []                   # max_length == len + 1: no draft
    assert PL.draft([1, 2, 3], 3, 2, 100) == []             # no earlier occurrence
    # an IMAGE_TOKEN_INDEX placeholder ends a draft (HF would propose it); the match itself may sit next to it
    img = [5, 6, -200, 7, 5, 6]
    assert PL.draft(img, 4, 2, 100, vocab=30) == []
    assert _hf_draft(img, 4, 2, 100, set()) == [-200, 7, 5, 6]
    assert PL.draft([-200, 4, 9, 1, 4], 3, 2, 100, vocab=30) == [9, 1, 4]


def test_accept_equals_hf_n_matches():
    rng = random.Random(7)
    for _ in range(400):
        d = rng.randint(0, 15)
        drafted = [rng.randrange(3) for _ in range(d)]
        selected = [rng.randrange(3) for _ in range(d + 1)]
        hist_len = rng.randint(1, 50)
        max_length = hist_len + rng.randint(1, 20)
        done = d > 0 and hist_len + d >= max_length
        n = PL.hf_n_matches(drafted, selected, done) if d > 0 else 0
        got = PL.accept(drafted, selected, hist_len, max_length, 0, 10 ** 6)
        assert got == selected[:n + 1]
        # the budget caps what a step publishes
        published = rng.randint(0, 5)
        capped = PL.accept(drafted, selected, hist_len, max_length, published, published + 2)
        assert capped == selected[:min(n + 1, 2)]


def _stub(cap, **cfg):
    from llava.model.language_model.llava_llama import LlavaLlamaForCausalLM as M

    stub = types.SimpleNamespace(config=types.SimpleNamespace(b2_prompt_lookup=cap, **cfg))
    stub._prompt_lookup_cap = types.MethodType(M._prompt_lookup_cap, stub)
    return types.MethodType(M._prompt_lookup_arguments, stub)


def test_generate_arguments(monkeypatch):
    monkeypatch.delenv("B2_PROMPT_LOOKUP", raising=False)
    monkeypatch.delenv("B2_KV_DTYPE", raising=False)
    kw = {"prompt_lookup_num_tokens": 4}
    assert _stub(None)(kw, 1, 1, False) == {} and kw == {"prompt_lookup_num_tokens": 4}  # off: left for NotImplementedError
    on = _stub(8)
    kw = {"prompt_lookup_num_tokens": 4, "top_k": 3}
    assert on(kw, 1, 1, False) == {"num_tokens": 4, "max_ngram": 2} and kw == {"top_k": 3}
    assert on({"prompt_lookup_num_tokens": 12, "max_matching_ngram_size": 3}, 1, 1, False) == {"num_tokens": 8, "max_ngram": 3}
    assert on({}, 1, 1, False) == {"num_tokens": 8, "max_ngram": 2}       # batch 1 without the argument: K
    assert on({}, 2, 1, False) == {} and on({}, 1, 2, False) == {} and on({}, 1, 1, True) == {}
    with pytest.raises(ValueError, match="batch_size = 1"):
        on({"prompt_lookup_num_tokens": 4}, 2, 1, False)
    for B, beams, procs in ((1, 2, False), (1, 1, True)):
        with pytest.raises(NotImplementedError):
            on({"prompt_lookup_num_tokens": 4}, B, beams, procs)
    with pytest.raises(NotImplementedError):
        _stub(8, b2_continuous_batching=4)({"prompt_lookup_num_tokens": 4}, 1, 1, False)
    with pytest.raises(NotImplementedError):
        _stub(8, b2_kv_dtype="e4m3")({"prompt_lookup_num_tokens": 4}, 1, 1, False)
    assert _stub(8, b2_kv_dtype="e4m3")({}, 1, 1, False) == {}
    with pytest.raises(ValueError):
        on({"prompt_lookup_num_tokens": 4, "max_matching_ngram_size": 0}, 1, 1, False)
    with pytest.raises(ValueError):
        _stub(16)({}, 1, 1, False)
    monkeypatch.setenv("B2_PROMPT_LOOKUP", "3")
    assert _stub(None)({}, 1, 1, False) == {"num_tokens": 3, "max_ngram": 2}


def test_generate_without_opt_in_raises_as_before(monkeypatch):
    from llava.model.language_model.llava_llama import LlavaLlamaForCausalLM as M

    monkeypatch.delenv("B2_PROMPT_LOOKUP", raising=False)

    class Stub:
        config = types.SimpleNamespace()
        _LOGITS_PROCESSOR_ARGS = M._LOGITS_PROCESSOR_ARGS
        _UNSUPPORTED_GENERATION_ARGS = M._UNSUPPORTED_GENERATION_ARGS
        _IGNORED_GENERATION_ARGS = M._IGNORED_GENERATION_ARGS
        _logits_processors_on = M._logits_processors_on
        _logits_processor_arguments = M._logits_processor_arguments
        _prompt_lookup_cap = M._prompt_lookup_cap
        _prompt_lookup_arguments = M._prompt_lookup_arguments

        def _ensure_engine(self):
            raise AssertionError("no engine should be built")

    with pytest.raises(NotImplementedError, match="unsupported argument 'prompt_lookup_num_tokens'"):
        M.generate.__wrapped__(Stub(), torch.ones(1, 4, dtype=torch.long), prompt_lookup_num_tokens=4)


# ------------------------------------------------------------------------------------------------ the host loop
def _next(tok):
    return (tok * 7 + 3) % 23


class LookupEngine:
    """The lookup streaming contract of include/b2llava.h, with a device that runs behind the host: stream_enqueue(n) tops the
    verify steps in flight (queued, not retired) up to n and queues none once max_new tokens are published; a step publishes
    1..K+1 tokens (a fixed pattern here) when it retires; stream_wait(index) retires queued steps until token `index` is out
    and is legal only for index < published + steps in flight, as the engine checks."""

    def __init__(self, first, max_new, per_step):
        self.tokens = [int(first)]
        self.max_new, self.per_step = max_new, per_step
        self.queued = self.retired = 0
        self.useful = 0  # retired steps that published tokens

    def stream_enqueue(self, kv, n):
        assert n >= 1
        if len(self.tokens) < self.max_new and self.queued - self.retired < n:
            self.queued += n - (self.queued - self.retired)

    def _retire(self):
        k = self.per_step[self.retired % len(self.per_step)]
        self.retired += 1
        if len(self.tokens) < self.max_new:
            self.useful += 1
            for _ in range(min(k, self.max_new - len(self.tokens))):
                self.tokens.append(int(_next(self.tokens[-1])))

    def stream_wait(self, kv, index, B, timeout_ms=0):
        assert index < min(self.max_new, len(self.tokens) + self.queued - self.retired), "token not guaranteed"
        while index >= len(self.tokens):
            self._retire()
        return [self.tokens[index]]


def test_host_loop_reads_token_by_token():
    from llava.model.language_model.llava_llama import _LOOKUP_STEPS_IN_FLIGHT, _stream_decode

    for per_step in ([1], [4], [1, 5, 2], [16]):
        for max_new in (1, 3, 9, 40):
            for eos in (set(), {int(_next(_next(5)))}):
                eng = LookupEngine(5, max_new, per_step)
                seen = []

                class Streamer:
                    def put(self, t):
                        seen.append(t.tolist())

                crit_calls = []

                def crit(ids, scores):
                    crit_calls.append(ids.shape[1])
                    return ids.shape[1] >= 3 + 7

                prompt = torch.arange(3).reshape(1, 3)
                out = _stream_decode(eng, None, None, None, 1, max_new, eos, 0, prompt, Streamer(), [crit], run_ahead=4,
                                     begun=True, lookup_steps=_LOOKUP_STEPS_IN_FLIGHT)
                want, t = [], 5
                for _ in range(max_new):
                    want.append(t)
                    if t in eos or len(want) >= 7:
                        break
                    t = int(_next(t))
                assert out[0].tolist() == want, (per_step, max_new, eos)
                assert [s[0] for s in seen] == want  # one streamer call per token
                assert crit_calls == [3 + i + 1 for i in range(len(want))]  # criteria see cat(prompt, tokens) per token
                # steps are scheduled against what the device retired: at most the in-flight window runs past the useful ones
                assert eng.queued <= eng.useful + _LOOKUP_STEPS_IN_FLIGHT, (per_step, max_new, eng.queued, eng.useful)
