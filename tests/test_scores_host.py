"""CPU: generate(return_dict_in_generate=True, output_scores / output_logits). Argument handling (what returns ids, what raises
before an engine exists), and the beam bookkeeping behind GenerateBeamDecoderOnlyOutput: BeamSearch's beam_indices and
sequences_scores against the installed transformers' over the cases of tests/test_beam_host.py, driven through the CPU stand-in
of b2_beam_step, and compute_transition_scores over the stand-in's score rows reconstructing sequences_scores."""
import types

import pytest
import torch

from llava._b2 import beam as BM
from llava.model.language_model.llava_llama import LlavaLlamaForCausalLM as M
from test_beam_host import CASES, EOS, V, KeywordBool, RowTail, SlotStandIn, _hf_model, _logits_fn
from test_beam_sample_host import _stub


@pytest.fixture
def no_env(monkeypatch):
    for k in ("B2_BEAM_SAMPLE", "B2_BEAM_SEARCH", "B2_PROMPT_LOOKUP", "B2_LOGITS_PROCESSORS", "B2_KV_DTYPE"):
        monkeypatch.delenv(k, raising=False)


def _no_engine_stub(**cfg):
    class Stub:
        config = types.SimpleNamespace(eos_token_id=None, **cfg)
        _LOGITS_PROCESSOR_ARGS = M._LOGITS_PROCESSOR_ARGS
        _UNSUPPORTED_GENERATION_ARGS = M._UNSUPPORTED_GENERATION_ARGS
        _IGNORED_GENERATION_ARGS = M._IGNORED_GENERATION_ARGS
        _logits_processors_on = M._logits_processors_on
        _logits_processor_arguments = M._logits_processor_arguments
        _prompt_lookup_cap = M._prompt_lookup_cap
        _prompt_lookup_arguments = M._prompt_lookup_arguments
        _beam_search_cap = M._beam_search_cap

        def _ensure_engine(self):
            raise AssertionError("an engine was created before the arguments were refused")

    stub = Stub()
    return lambda *a, **k: M.generate.__wrapped__(stub, *a, **k)


def test_ids_without_return_dict(no_env):
    m = _hf_model(seed=1)
    gen, _ = _stub(_logits_fn(m))
    p = torch.randint(8, V, (2, 5), generator=torch.Generator().manual_seed(1))
    plain = gen(p, num_beams=2, max_new_tokens=4)
    for kw in (dict(output_scores=True), dict(output_logits=True), dict(output_scores=True, output_logits=True)):
        out = gen(p, num_beams=2, max_new_tokens=4, return_dict_in_generate=False, **kw)
        assert torch.is_tensor(out) and torch.equal(out, plain)


@pytest.mark.parametrize("cfg,match", [
    (dict(b2_prompt_lookup=4), "prompt-lookup path"),
    (dict(b2_continuous_batching=4), "continuous batcher"),
])
def test_refused_combinations_raise_before_an_engine(no_env, cfg, match):
    gen = _no_engine_stub(**cfg)
    p = torch.randint(8, V, (1, 5), generator=torch.Generator().manual_seed(2))
    for kw in (dict(output_scores=True), dict(output_logits=True)):
        with pytest.raises(NotImplementedError, match=match):
            gen(p, max_new_tokens=4, return_dict_in_generate=True, **kw)


@pytest.mark.parametrize("flag", ["output_attentions", "output_hidden_states"])
def test_attentions_and_hidden_states_raise(no_env, flag):
    gen = _no_engine_stub()
    p = torch.randint(8, V, (1, 5), generator=torch.Generator().manual_seed(3))
    with pytest.raises(NotImplementedError, match=flag):
        gen(p, max_new_tokens=4, return_dict_in_generate=True, **{flag: True})


def test_output_logits_is_an_accepted_argument(no_env):
    m = _hf_model(seed=4)
    gen, _ = _stub(_logits_fn(m))
    p = torch.randint(8, V, (1, 5), generator=torch.Generator().manual_seed(4))
    assert torch.is_tensor(gen(p, num_beams=2, max_new_tokens=3, output_logits=True))


def _run_host(m, prompt, nb, eos, lp, es, nrs, crit):
    """BeamSearch over the CPU stand-in of b2_beam_step; returns (search, per-step score rows [B * nb, V] in running-beam
    order, as the device writes them: log_softmax of each running beam's logits, step 0 fanned out from the prefill row)."""
    fn = _logits_fn(m)
    B = prompt.shape[0]
    search = BM.BeamSearch(prompt, nb, 9, eos, lp, es, nrs, None, crit)
    eng = SlotStandIn(fn, prompt, B * nb)
    planner = BM.SlotPlanner(B, nb)
    first = fn(prompt)
    rows = [torch.log_softmax(first.float(), -1).repeat_interleave(nb, dim=0)]
    cand, row_begin = eng.first(B, search.K), 0
    while not search.step(*cand):
        copies = planner.plan(search.parents)
        cand = eng.step(copies, row_begin, search.next_tokens().tolist(), planner.flat(),
                        search.running_scores.reshape(-1).tolist(), nb, search.K)
        slots = planner.flat()
        rows.append(torch.log_softmax(fn(torch.tensor([eng.hist[s] for s in slots])).float(), -1))
        row_begin = prompt.shape[1]
    return search, tuple(rows)


@pytest.mark.parametrize("nb,B,es,eos", CASES[1::2])
def test_beam_indices_and_sequence_scores_equal_transformers(no_env, nb, B, es, eos):
    from transformers import LlamaConfig, StoppingCriteriaList

    i = CASES.index((nb, B, es, eos))
    lp = [1.0, 0.0, -0.5, 2.0][i % 4]
    nrs = [1, nb][(i // 4) % 2]
    crit = [None, [KeywordBool(7)], [RowTail()]][i % 3]
    m = _hf_model(seed=i)
    prompt = torch.randint(8, V, (B, 5), generator=torch.Generator().manual_seed(i))
    kw = dict(num_beams=nb, do_sample=False, max_new_tokens=9, length_penalty=lp, early_stopping=es, num_return_sequences=nrs,
              use_cache=False, output_scores=True, return_dict_in_generate=True)
    if EOS[eos] is not None:
        kw["eos_token_id"] = EOS[eos]
    if crit:
        kw["stopping_criteria"] = StoppingCriteriaList(crit)
    with torch.no_grad():
        hf = m.generate(prompt, attention_mask=torch.ones_like(prompt), **kw)
        search, rows = _run_host(m, prompt, nb, EOS[eos], lp, es, nrs, crit)
    seq, seq_scores = search.output()
    bi = search.output_beam_indices()
    assert torch.equal(seq, hf.sequences)
    assert torch.equal(bi, hf.beam_indices.to(bi.dtype)) and bi.shape == hf.beam_indices.shape
    torch.testing.assert_close(seq_scores, hf.sequences_scores.float(), atol=1e-5, rtol=0)
    assert len(rows) == len(hf.scores)
    for got, want in zip(rows, hf.scores):
        torch.testing.assert_close(got, want.float(), atol=1e-5, rtol=0)

    # HF's documented identity: the generated tokens' transition scores, summed and length-normalised, are sequences_scores
    stub = types.SimpleNamespace(config=LlamaConfig(vocab_size=V))
    ts = M.compute_transition_scores(stub, seq, rows, bi, normalize_logits=False)
    length = (bi >= 0).sum(dim=1)
    recon = ts.sum(dim=1) / (length.float() ** lp)
    torch.testing.assert_close(recon, seq_scores, atol=1e-5, rtol=1e-5)
    ts_hf = m.compute_transition_scores(hf.sequences, hf.scores, hf.beam_indices, normalize_logits=False)
    torch.testing.assert_close(ts, ts_hf.float(), atol=1e-5, rtol=0)
