"""CPU: logits processors in beam search and beam sampling. tests/beam_proc_ref.py against the installed transformers'
generate(num_beams=..., repetition_penalty / no_repeat_ngram_size / min_new_tokens / min_length) on a tiny CPU Llama, and
generate() over a CPU stand-in of the engine's processed beam entry points: the opt-in matrix, the arguments the stand-in
receives, ids against the reference and score rows against transformers'."""
import itertools
import types

import numpy as np
import pytest
import torch

import beam_proc_ref as BPR
import beam_sampling_ref as BSR
from oracle import beam_oracle as BO
from oracle import logits_proc_oracle as P
from test_beam_sample_host import SampleEngine, _hf_model, _logits_fn

V = 64
PROC = dict(repetition_penalty=1.3, no_repeat_ngram_size=2)
EOS = {"none": None, "one": [5], "two": [5, 6]}
CASES = list(itertools.product([1, 2], [2, 4], ["none", "one", "two"], [False, True, "never"]))


def _hf_kw(nb, eos, es, i):
    kw = dict(num_beams=nb, max_new_tokens=9, early_stopping=es, num_return_sequences=[1, nb][i % 2], use_cache=False,
              **PROC)
    if eos is not None:
        kw["eos_token_id"] = eos
        kw["min_new_tokens" if i % 2 else "min_length"] = 3 if i % 2 else 5 + 4
    return kw


def _ref_kw(kw):
    return {k: kw[k] for k in ("repetition_penalty", "no_repeat_ngram_size", "min_new_tokens", "min_length") if k in kw}


@pytest.mark.parametrize("B,nb,eos,es", CASES)
def test_reference_equals_transformers_beam_search(B, nb, eos, es):
    i = CASES.index((B, nb, eos, es))
    m = _hf_model(seed=100 + i)
    p = torch.randint(8, V, (B, 5), generator=torch.Generator().manual_seed(i))
    kw = _hf_kw(nb, EOS[eos], es, i)
    with torch.no_grad():
        hf = m.generate(p, attention_mask=torch.ones_like(p), do_sample=False, output_scores=True, return_dict_in_generate=True, **kw)
        seq, sc, rows = BPR.beam_search(_logits_fn(m), p, nb, 9, EOS[eos], None, 1.0, es, kw["num_return_sequences"],
                                        return_rows=True, **_ref_kw(kw))
        plain = BO.beam_search(_logits_fn(m), p, nb, 9, EOS[eos], None, 1.0, es, kw["num_return_sequences"])[0]
    assert torch.equal(seq, hf.sequences), (seq, hf.sequences)
    torch.testing.assert_close(sc, hf.sequences_scores.float(), atol=1e-5, rtol=0)
    assert len(rows) == len(hf.scores)
    for got, want in zip(rows, hf.scores):
        torch.testing.assert_close(got, want.float(), atol=1e-5, rtol=0)
    assert not torch.equal(seq, plain) or not torch.equal(rows[1], torch.log_softmax(rows[1], -1))  # the processors acted


def test_reference_without_processors_is_the_plain_reference():
    m = _hf_model(seed=7)
    p = torch.randint(8, V, (2, 5), generator=torch.Generator().manual_seed(7))
    with torch.no_grad():
        a = BPR.beam_search(_logits_fn(m), p, 3, 8, [5])
        b = BO.beam_search(_logits_fn(m), p, 3, 8, [5])
        c = BPR.beam_search(_logits_fn(m), p, 3, 8, [5], do_sample=True, temperature=0.7, sampler="philox", seed=9)
        d = BSR.beam_search(_logits_fn(m), p, 3, 8, [5], do_sample=True, temperature=0.7, sampler="philox", seed=9)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and torch.equal(c[0], d[0]) and torch.equal(c[1], d[1])


@pytest.mark.parametrize("B,nb,eos", [(1, 2, None), (2, 3, [5]), (1, 4, [5, 6])])
def test_torch_sampler_equals_transformers_beam_sampling(B, nb, eos):
    m = _hf_model(seed=B * 10 + nb)
    p = torch.randint(8, V, (B, 5), generator=torch.Generator().manual_seed(nb))
    kw = dict(num_beams=nb, max_new_tokens=8, temperature=0.8, top_k=20, top_p=0.9, num_return_sequences=nb, **PROC)
    if eos is not None:
        kw["eos_token_id"] = eos
        kw["min_new_tokens"] = 3
    with torch.no_grad():
        torch.manual_seed(31)
        hf = m.generate(p, attention_mask=torch.ones_like(p), do_sample=True, use_cache=False, **kw)
        torch.manual_seed(31)
        got = BPR.beam_search(_logits_fn(m), p, nb, 8, eos, None, 1.0, False, nb, do_sample=True, temperature=0.8, top_k=20,
                              top_p=0.9, sampler="torch", **_ref_kw(kw))[0]
    assert torch.equal(got, hf), (got, hf)


# ------------------------------------------------------------------------------------------------------- generate()
class ProcEngine(SampleEngine):
    """SampleEngine with the processed entry points: histories per slot as the device keeps them (prompt, then every token fed
    to the slot, carried along the copies), and each selected row processed against its history."""

    def __init__(self, fn, vocab):
        super().__init__(fn, vocab)
        self.armed = None

    def _rows(self, logits, hists, sampling):
        if sampling is None:
            ls = torch.log_softmax(logits.float(), -1)
        else:
            ls = torch.from_numpy(np.stack([BSR.log_softmax32(r) for r in logits.float().numpy()]))
        out = []
        for r, (h, pr) in enumerate(hists):
            x = ls[r].numpy()
            if pr is not None:
                x = P.process(x, h, pr.prompt_len, pr.repetition_penalty, pr.no_repeat_ngram_size, pr.min_generated,
                              tuple(pr.eos_ids))
            if sampling is not None:
                w = (x / np.float32(sampling.temperature)).astype(np.float32)
                x = np.where(BSR.kept_mask(w, sampling.top_k, sampling.top_p, sampling.min_keep) | np.isnan(w), w, -np.inf)
            out.append(torch.from_numpy(np.asarray(x, dtype=np.float32)))
        return torch.stack(out)

    def _pick(self, w, run, nb, K, sampling, step):
        B = run.numel() // nb
        if sampling is None:
            s, i = BO.select_candidates((w + run.view(-1, 1)).view(B, nb * V), K)
            return s, i % V, i // V
        acc = (w.numpy().reshape(B, nb, V) + run.numpy().reshape(B, nb, 1).astype(np.float32)).astype(np.float32).reshape(B, nb * V)
        s, i, _, _ = BSR.philox_select(acc, sampling.seed, step, nb, K)
        i = torch.from_numpy(i.astype(np.int64))
        return torch.from_numpy(s.astype(np.float32)), i % V, i // V

    def beam_select_proc(self, logits, scores, nb, K, procs, row_scores=None, row_logits=None, sampling=None, step=0,
                         row_of_beam=None, fan=1):
        self.calls.append(("select_proc", tuple(procs), fan))
        rows = list(range(logits.shape[0])) if row_of_beam is None else list(row_of_beam)
        w = self._rows(logits, [(pr.ids.tolist() if pr is not None else [], pr) for pr in procs], sampling)
        w, lg = w[rows].repeat_interleave(fan, 0), logits[rows].float().repeat_interleave(fan, 0)
        if row_scores is not None:
            row_scores.copy_(w)
        if row_logits is not None:
            row_logits.copy_(lg)
        return self._pick(w[::fan] if fan > 1 else w, scores.float(), nb, K, sampling, step)

    def beam_begin_proc(self, kv, procs):
        self.calls.append(("begin_proc", tuple(procs)))
        self.armed = {b: pr for b, pr in enumerate(procs)}

    def beam_step_proc(self, kv, copies, row_begin, tokens, slot_of, scores, nb, K, sampling=None, step=0, row_scores=None,
                       row_logits=None):
        self.calls.append(("step_proc", step))
        armed = dict(self.armed)
        new = dict(self.hist)
        for s, d in copies:
            new[d] = self.hist[s][:]
            armed[d] = self.armed.get(s)
        for t, s in zip(tokens, slot_of):
            new[s] = new[s] + [int(t)]
        self.hist, self.armed = new, armed
        logits = self.fn(torch.tensor([self.hist[s] for s in slot_of]))
        # the history of slot s is its prompt row then its tokens: here the stand-in's token list itself
        w = self._rows(logits, [(self.hist[s], self.armed.get(s)) for s in slot_of], sampling)
        if row_scores is not None:
            row_scores.copy_(w)
        if row_logits is not None:
            row_logits.copy_(logits.float())
        return self._pick(w, torch.tensor(scores), nb, K, sampling, step)


def _fake_logits_proc(prompt_row, repetition_penalty=1.0, no_repeat_ngram_size=0, min_generated=0, eos_ids=()):
    """make_logits_proc's values on a CPU prompt row (the real struct wants a device pointer)."""
    eos = sorted(set(int(e) for e in eos_ids))
    mg = int(min_generated or 0) if eos else 0
    if repetition_penalty == 1.0 and not no_repeat_ngram_size and mg <= 0:
        return None
    return types.SimpleNamespace(repetition_penalty=float(repetition_penalty), no_repeat_ngram_size=int(no_repeat_ngram_size),
                                 min_generated=max(mg, 0), eos_ids=eos, prompt_len=int(prompt_row.numel()), ids=prompt_row)


def _stub(fn, monkeypatch, **cfg):
    from llava.model.language_model import llava_llama as LL
    M = LL.LlavaLlamaForCausalLM

    monkeypatch.setattr(LL, "make_logits_proc", _fake_logits_proc)
    eng = ProcEngine(fn, V)

    class Pool:
        def acquire(self):
            return types.SimpleNamespace(reset=lambda: None)

        def release(self, kv):
            pass

    class Stub:
        config = types.SimpleNamespace(b2_beam_search=4, eos_token_id=None, **cfg)
        _LOGITS_PROCESSOR_ARGS = M._LOGITS_PROCESSOR_ARGS
        _UNSUPPORTED_GENERATION_ARGS = M._UNSUPPORTED_GENERATION_ARGS
        _IGNORED_GENERATION_ARGS = M._IGNORED_GENERATION_ARGS
        _logits_processors_on = M._logits_processors_on
        _logits_processor_arguments = M._logits_processor_arguments
        _prompt_lookup_cap = M._prompt_lookup_cap
        _prompt_lookup_arguments = M._prompt_lookup_arguments
        _beam_search_cap = M._beam_search_cap
        _beam_sample_on = M._beam_sample_on
        _beam_arguments = M._beam_arguments
        _beam_generate = M._beam_generate
        _pool = Pool()

        def _ensure_engine(self):
            return eng

        def _prompt_embeds(self, engine, prompt, attention_mask, images, force_host):
            return prompt, [prompt.shape[1]] * prompt.shape[0], False

        def _check_limits(self, engine, n, length):
            pass

    stub = Stub()
    return (lambda *a, **k: M.generate.__wrapped__(stub, *a, **k)), eng


@pytest.fixture
def no_env(monkeypatch):
    for k in ("B2_BEAM_SAMPLE", "B2_BEAM_SEARCH", "B2_PROMPT_LOOKUP", "B2_LOGITS_PROCESSORS", "B2_BEAM_LOGITS_PROCESSORS"):
        monkeypatch.delenv(k, raising=False)


def test_opt_in_matrix_and_arguments(no_env, monkeypatch):
    m = _hf_model(seed=3)
    fn = _logits_fn(m)
    p = torch.randint(8, V, (1, 5), generator=torch.Generator().manual_seed(3))
    for cfg in ({}, {"b2_logits_processors": True}, {"b2_beam_logits_processors": True}):
        gen, eng = _stub(fn, monkeypatch, **cfg)
        with pytest.raises(NotImplementedError):
            gen(p, num_beams=2, max_new_tokens=3, no_repeat_ngram_size=2)
        assert not eng.calls
    gen, eng = _stub(fn, monkeypatch, b2_logits_processors=True, b2_beam_logits_processors=True)
    with pytest.raises(NotImplementedError, match="beam sampling"):        # beam sampling keeps its own opt-in
        gen(p, num_beams=2, do_sample=True, max_new_tokens=3, repetition_penalty=1.2)
    with pytest.raises(ValueError, match="repetition_penalty"):
        gen(p, num_beams=2, max_new_tokens=3, repetition_penalty=0.0)
    with pytest.raises(ValueError, match="no_repeat_ngram_size"):
        gen(p, num_beams=2, max_new_tokens=3, no_repeat_ngram_size=-1)
    with torch.no_grad():
        gen(p, num_beams=2, max_new_tokens=3, eos_token_id=[5], repetition_penalty=1.2, no_repeat_ngram_size=3, min_length=7,
            min_new_tokens=1)
    first, begin = eng.calls[0], eng.calls[1]
    assert first[0] == "select_proc" and first[2] == 2 and begin[0] == "begin_proc"
    pr = first[1][0]
    assert (pr.repetition_penalty, pr.no_repeat_ngram_size, pr.min_generated, pr.eos_ids) == (1.2, 3, 2, [5])
    assert begin[1] == first[1] and all(c[0] == "step_proc" for c in eng.calls[2:])
    eng.calls.clear()
    with torch.no_grad():                                                  # every processor at its off value: plain beam search
        gen(p, num_beams=2, max_new_tokens=3, repetition_penalty=1.0)
    assert eng.calls[0] == "topk" and not any(isinstance(c, tuple) and c[0].endswith("proc") for c in eng.calls)
    monkeypatch.setenv("B2_LOGITS_PROCESSORS", "1")
    monkeypatch.setenv("B2_BEAM_LOGITS_PROCESSORS", "1")                   # the environment switches
    gen_env, eng = _stub(fn, monkeypatch)
    with torch.no_grad():
        gen_env(p, num_beams=2, max_new_tokens=3, no_repeat_ngram_size=2)
    assert eng.calls[0][0] == "select_proc"


@pytest.mark.parametrize("B,nb,eos", [(1, 2, None), (2, 3, [5]), (2, 4, [5, 6])])
def test_generate_equals_transformers_with_score_rows(no_env, monkeypatch, B, nb, eos):
    """ids, sequences_scores and every score row against the installed transformers; compute_transition_scores over them."""
    from llava.model.language_model.llava_llama import LlavaLlamaForCausalLM as M

    m = _hf_model(seed=50 + nb)
    fn = _logits_fn(m)
    p = torch.randint(8, V, (B, 5), generator=torch.Generator().manual_seed(nb))
    kw = dict(num_beams=nb, max_new_tokens=8, num_return_sequences=nb, repetition_penalty=1.3, no_repeat_ngram_size=2)
    if eos is not None:
        kw.update(eos_token_id=eos, min_new_tokens=2)
    gen, _ = _stub(fn, monkeypatch, b2_logits_processors=True, b2_beam_logits_processors=True)
    with torch.no_grad():
        hf = m.generate(p, attention_mask=torch.ones_like(p), do_sample=False, use_cache=False, output_scores=True,
                        return_dict_in_generate=True, **kw)
        got = gen(p, output_scores=True, output_logits=True, return_dict_in_generate=True, **kw)
    assert torch.equal(got.sequences, hf.sequences)
    torch.testing.assert_close(got.sequences_scores, hf.sequences_scores.float(), atol=1e-5, rtol=0)
    assert len(got.scores) == len(hf.scores)
    for a, b in zip(got.scores, hf.scores):
        torch.testing.assert_close(a, b.float(), atol=1e-5, rtol=0)
    ts = M.compute_transition_scores(types.SimpleNamespace(config=m.config), got.sequences, got.scores, got.beam_indices)
    ts_hf = m.compute_transition_scores(hf.sequences, hf.scores, hf.beam_indices)
    torch.testing.assert_close(ts, ts_hf.float(), atol=1e-5, rtol=0)


@pytest.mark.parametrize("B,nb,eos", [(1, 3, [5]), (2, 2, None)])
def test_generate_beam_sampling_equals_the_philox_reference(no_env, monkeypatch, B, nb, eos):
    m = _hf_model(seed=60 + nb)
    fn = _logits_fn(m)
    p = torch.randint(8, V, (B, 5), generator=torch.Generator().manual_seed(nb))
    gen, eng = _stub(fn, monkeypatch, b2_logits_processors=True, b2_beam_logits_processors=True, b2_beam_sample=True)
    kw = dict(num_beams=nb, do_sample=True, temperature=0.8, top_k=20, top_p=0.9, max_new_tokens=8, num_return_sequences=nb,
              repetition_penalty=1.3, no_repeat_ngram_size=2)
    if eos is not None:
        kw.update(eos_token_id=eos, min_new_tokens=2)
    with torch.no_grad():
        torch.manual_seed(5)
        got = gen(p, **kw)
        torch.manual_seed(5)
        seed = int(torch.randint(0, 2**62, (1,), dtype=torch.int64).item())
        want = BPR.beam_search(fn, p, nb, 8, eos, None, 1.0, False, nb, do_sample=True, temperature=0.8, top_k=20, top_p=0.9,
                               sampler="philox", seed=seed, repetition_penalty=1.3, no_repeat_ngram_size=2,
                               min_new_tokens=2 if eos else 0)[0]
    assert torch.equal(got, want), (got, want)
    assert eng.calls[0][0] == "select_proc" and eng.calls[0][2] == 1
