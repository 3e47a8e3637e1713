"""GPU: generate(return_dict_in_generate=True, output_scores=True, output_logits=True).

- The ids equal the plain call's on every path: the megakernel (B = 1), the GEMV graph (B = 4) and stream-K (B = 12), seeded
  sampling, logits processors, prefix reuse, an e4m3 KV cache, beam search and beam sampling.
- logits[t] is step t's: it matches the fp32 oracle's forward over the prompt and the generated ids at that position, with the
  default run-ahead, so a stale or overwritten row would fail.
- scores[t] is transformers' own processing of logits[t] (its LogitsProcessorList in HF's order, over the ids so far): finite
  entries bit-equal, -inf masks equal away from the top-k / top-p thresholds, the chosen token finite. A low temperature puts
  top-k survivors whose exp underflows in the rows. Beam rows are log_softmax(logits[t]), warped under beam sampling.
- Rows that end at different steps, and the launch counts: unchanged with the outputs off, one more per step at batch <= 8
  greedy with them on."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from helpers import make_model, rel_err  # noqa: E402
from llava import _b2  # noqa: E402
from oracle import llava_oracle as O  # noqa: E402

DEV = "cuda"
CFG = O.CONFIGS["tiny"]
W = None
ON = dict(return_dict_in_generate=True, output_scores=True, output_logits=True)
SAMPLED = dict(do_sample=True, temperature=0.7, top_p=0.9, top_k=50)
PRM = dict(repetition_penalty=1.3, no_repeat_ngram_size=3, min_new_tokens=4)


def _weights():
    global W
    if W is None:
        W = O.make_weights(CFG, seed=0)
    return W


def _model(**extra):
    return make_model(CFG, _weights(), max_batch=16, max_seq=160, **extra)


def _prompt(B, seed, Lt=12):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(3, CFG["vocab"], (B, Lt), generator=g)
    ids[:, 0] = 1
    return ids.to(DEV)


def _run(model, ids, seed, **kw):
    torch.manual_seed(seed)
    return model.generate(ids, eos_token_id=kw.pop("eos_token_id", []), **kw)


def _hf_processors(kw, Lt, eos):
    from transformers import (LogitsProcessorList, MinNewTokensLengthLogitsProcessor, NoRepeatNGramLogitsProcessor,
                              RepetitionPenaltyLogitsProcessor, TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper)

    lp = LogitsProcessorList()
    if kw.get("repetition_penalty", 1.0) != 1.0:
        lp.append(RepetitionPenaltyLogitsProcessor(kw["repetition_penalty"]))
    if kw.get("no_repeat_ngram_size", 0):
        lp.append(NoRepeatNGramLogitsProcessor(kw["no_repeat_ngram_size"]))
    if kw.get("min_new_tokens", 0) and eos:
        lp.append(MinNewTokensLengthLogitsProcessor(Lt, kw["min_new_tokens"], eos))
    if kw.get("do_sample"):
        lp.append(TemperatureLogitsWarper(kw["temperature"]))
        lp.append(TopKLogitsWarper(kw["top_k"]))
        if kw["top_p"] < 1.0:
            lp.append(TopPLogitsWarper(kw["top_p"]))
    return lp


def _check_scores(out, Lt, kw, eos):
    """scores[t] of every row up to its eos = HF's processors over logits[t] and the ids before it, run on the CPU, where
    TemperatureLogitsWarper's x / T is an IEEE division (on a CUDA tensor torch multiplies by 1 / T instead)."""
    seq = out.sequences.cpu()
    lp = _hf_processors(kw, Lt, eos)
    ended = torch.zeros(seq.shape[0], dtype=torch.bool)
    for t, (s, l) in enumerate(zip(out.scores, out.logits)):
        s, l = s.cpu(), l.cpu()
        want = lp(seq[:, :Lt + t].clone(), l.clone())
        tok = seq[:, Lt + t]
        for b in range(seq.shape[0]):
            if ended[b]:
                continue
            g, w = s[b], want[b]
            assert torch.isfinite(g[tok[b]]), (t, b)
            fin = torch.isfinite(g) & torch.isfinite(w)
            if kw.get("do_sample"):  # within one ulp
                inf = torch.tensor(float("inf"))
                assert bool(((g[fin] == w[fin]) | (g[fin] == torch.nextafter(w[fin], inf))
                             | (g[fin] == torch.nextafter(w[fin], -inf))).all()), (t, b, (g[fin] - w[fin]).abs().max())
            else:
                assert torch.equal(g[fin], w[fin]), (t, b, (g[fin] - w[fin]).abs().max())
            diff = (torch.isfinite(g) != torch.isfinite(w)).nonzero().flatten()
            if diff.numel():
                assert kw.get("do_sample"), ("greedy masks differ", t, b, diff)
                x = l[b] / kw["temperature"]
                kth = torch.topk(x, kw["top_k"])[0][-1]
                p = torch.softmax(torch.where(x >= kth, x, -float("inf")), -1)
                srt, idx = torch.sort(p)
                cum = torch.cumsum(srt, 0)
                edge = cum[torch.argsort(idx)]
                for i in diff.tolist():  # within an ulp of the top-k value, or at the top-p boundary
                    near_k = abs(float(x[i] - kth)) <= float(torch.finfo(torch.float32).eps * kth.abs() * 2)
                    near_p = abs(float(edge[i]) - (1 - kw["top_p"])) < 1e-5
                    assert near_k or near_p, (t, b, i)
        if eos:
            ended |= torch.isin(tok, torch.tensor(eos, dtype=tok.dtype))


def _check_logits(out, Lt, ends=None):
    """logits[t] of row b (t up to its eos) = the oracle's fp32 forward over sequences[b, :Lt + t] at its last position."""
    w = _weights()
    seq = out.sequences.cpu()
    emb = w["model.embed_tokens.weight"].float()
    for b in range(seq.shape[0]):
        n = len(out.logits) if ends is None else ends[b] + 1
        ref, _ = O.llama_forward(w, emb[seq[b:b + 1, :Lt + n - 1]], CFG)
        got = torch.stack([out.logits[t][b] for t in range(n)])
        mx, mn = rel_err(got, ref[0, Lt - 1:Lt - 1 + n])
        assert mx < 0.05 and mn < 0.01, (b, mx, mn)


@pytest.mark.parametrize("B", [1, 4, 12])
@pytest.mark.parametrize("kind", ["greedy", "sampled", "processors"])
def test_same_ids_and_rows_are_hf(B, kind):
    model = _model(b2_logits_processors=True)
    ids = _prompt(B, seed=B)
    kw = dict(max_new_tokens=20)
    kw.update({"greedy": {}, "sampled": SAMPLED, "processors": PRM}[kind])
    eos = [9] if kind == "processors" else []
    plain = _run(model, ids, 7, eos_token_id=eos, **kw)
    out = _run(model, ids, 7, eos_token_id=eos, **kw, **ON)
    assert torch.equal(out.sequences, plain)
    n = plain.shape[1] - ids.shape[1]
    assert len(out.scores) == len(out.logits) == n
    assert all(s.shape == (B, CFG["vocab"]) and s.dtype == torch.float32 and s.device.type == "cuda" for s in out.scores)
    assert out.past_key_values is None and out.attentions is None and out.hidden_states is None
    _check_scores(out, ids.shape[1], kw, eos)
    _check_logits(out, ids.shape[1])
    only = _run(model, ids, 7, eos_token_id=eos, return_dict_in_generate=True, output_logits=True, **kw)
    assert only.scores is None and torch.equal(only.sequences, plain)
    assert all(torch.equal(a, b) for a, b in zip(only.logits, out.logits))
    model.invalidate_engine()


def test_underflowing_top_k_survivors_keep_finite_scores():
    """T = 0.01 spreads the logits so far that most of the 50 top-k survivors' exp underflows: with top_p = 1 HF keeps all of
    them finite, and so do the written rows."""
    model = _model()
    ids = _prompt(2, seed=11)
    kw = dict(max_new_tokens=8, do_sample=True, temperature=0.01, top_k=50, top_p=1.0)
    plain = _run(model, ids, 3, **kw)
    out = _run(model, ids, 3, **kw, **ON)
    assert torch.equal(out.sequences, plain)
    for s, l in zip(out.scores, out.logits):
        x = l / 0.01
        assert (torch.isfinite(s).sum(-1) >= 50).all()
        under = torch.exp(x - x.max(-1, keepdim=True)[0]) == 0
        assert (torch.isfinite(s) & under).any()  # survivors whose exp underflows
    _check_scores(out, ids.shape[1], dict(kw), [])
    model.invalidate_engine()


def test_rows_that_end_at_different_steps():
    model = _model()
    ids = _prompt(4, seed=21)
    free = _run(model, ids, 0, max_new_tokens=24)[:, ids.shape[1]:].cpu()
    eos = int(free[1, 5])  # row 1 ends at step 5 at the latest; the others where (and if) the id recurs
    plain = _run(model, ids, 0, max_new_tokens=24, eos_token_id=[eos])
    out = _run(model, ids, 0, max_new_tokens=24, eos_token_id=[eos], **ON)
    assert torch.equal(out.sequences, plain)
    new = plain[:, ids.shape[1]:].cpu()
    assert len(out.scores) == new.shape[1]
    ends = [int((new[b] == eos).nonzero()[0]) if (new[b] == eos).any() else new.shape[1] - 1 for b in range(4)]
    assert len(set(ends)) > 1, ends
    # up to its eos a row is HF's: the finished rows' later ids are pad (= eos), so compare each row on its own prefix
    for b in range(4):
        sub = type(out)(sequences=out.sequences[b:b + 1, :ids.shape[1] + ends[b] + 1],
                        scores=tuple(s[b:b + 1] for s in out.scores[:ends[b] + 1]),
                        logits=tuple(l[b:b + 1] for l in out.logits[:ends[b] + 1]))
        _check_scores(sub, ids.shape[1], {}, [])
        _check_logits(sub, ids.shape[1])
    model.invalidate_engine()


@pytest.mark.parametrize("extra", [dict(b2_kv_dtype="e4m3"), dict(b2_prefix_cache=True)])
def test_same_ids_on_e4m3_and_prefix_reuse(extra):
    model = make_model(CFG, _weights(), max_batch=4, max_seq=160, **extra)
    B = 1 if "b2_prefix_cache" in extra else 4
    ids = _prompt(B, seed=31)
    for kw in ({}, SAMPLED):
        _run(model, ids, 5, max_new_tokens=16, **kw)  # with the prefix cache: the later calls reuse this one's prompt rows
        plain = _run(model, ids, 5, max_new_tokens=16, **kw)
        out = _run(model, ids, 5, max_new_tokens=16, **kw, **ON)
        assert torch.equal(out.sequences, plain)
        assert len(out.scores) == plain.shape[1] - ids.shape[1]
        _check_scores(out, ids.shape[1], dict(kw), [])
        if "b2_prefix_cache" in extra:  # rows that were never written would pass the check above if they happened to agree
            _check_logits(out, ids.shape[1])
    model.invalidate_engine()


@pytest.mark.parametrize("sampled", [False, True])
def test_beam_rows_and_ids(sampled):
    model = _model(b2_beam_search=4, b2_beam_sample=True)
    ids = _prompt(2, seed=41)
    kw = dict(num_beams=4, max_new_tokens=10, length_penalty=1.0)
    if sampled:
        kw.update(do_sample=True, temperature=0.8, top_k=20, top_p=0.9)
    plain = _run(model, ids, 9, **kw)
    out = _run(model, ids, 9, **kw, **ON)
    assert torch.equal(out.sequences, plain)
    assert len(out.scores) == len(out.logits) and out.scores[0].shape == (2 * 4, CFG["vocab"])
    for t, (s, l) in enumerate(zip(out.scores, out.logits)):
        want = torch.log_softmax(l, -1)
        if sampled:
            from transformers import LogitsProcessorList, TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper

            warp = LogitsProcessorList([TemperatureLogitsWarper(0.8), TopKLogitsWarper(20, min_tokens_to_keep=1),
                                        TopPLogitsWarper(0.9, min_tokens_to_keep=1)])
            want = warp(None, want)
            fin = torch.isfinite(s) & torch.isfinite(want)
            assert (torch.isfinite(s) != torch.isfinite(want)).sum() <= 2 * s.shape[0], t
            torch.testing.assert_close(s[fin], want[fin], atol=1e-5, rtol=0)
        else:
            torch.testing.assert_close(s, want, atol=1e-5, rtol=0)
        if t == 0:  # the nb running rows of a sample all come from its one prefill row
            assert torch.equal(l[0], l[3]) and torch.equal(s[4], s[7])
    # sequences_scores = the transition scores summed and length-normalised (HF's identity)
    ts = model.compute_transition_scores(out.sequences, out.scores, out.beam_indices)
    length = (out.beam_indices >= 0).sum(-1)
    torch.testing.assert_close(ts.sum(-1) / length.float(), out.sequences_scores, atol=1e-4, rtol=1e-5)
    model.invalidate_engine()


def test_launch_counts():
    model = _model()
    ids = _prompt(1, seed=51)
    _run(model, ids, 0, max_new_tokens=4, **ON)  # warm

    def count(n, **kw):
        before = _b2.launch_count()
        _run(model, ids, 0, max_new_tokens=n, **kw)
        torch.cuda.synchronize()
        return _b2.launch_count() - before

    off = count(24)
    assert count(24, return_dict_in_generate=True) == off  # the output object alone changes nothing
    assert count(24, output_scores=True, output_logits=True) == off  # ignored without return_dict_in_generate
    assert count(24, **ON) - off == 23  # one rows launch after each of the 23 megakernel steps
    model.invalidate_engine()
