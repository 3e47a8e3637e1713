"""CPU: beam search semantics. oracle/beam_oracle.py against the installed transformers' generate(num_beams=...), the host half
of the engine's beam search (llava/_b2/beam.py: bookkeeping + slot planner) against the oracle through a CPU stand-in for
b2_beam_step that keeps real per-slot histories, and the slot planner's copy rules."""
import itertools
import random

import pytest
import torch

from llava._b2 import beam as BM
from oracle import beam_oracle as BO
from oracle import llava_oracle as O

V = 64


def _hf_model(seed=0):
    from transformers import LlamaConfig, LlamaForCausalLM

    torch.manual_seed(seed)
    cfg = LlamaConfig(vocab_size=V, hidden_size=32, intermediate_size=64, num_hidden_layers=2, num_attention_heads=2,
                      num_key_value_heads=2, max_position_embeddings=128, bos_token_id=None, eos_token_id=None,
                      pad_token_id=None, attn_implementation="eager")
    m = LlamaForCausalLM(cfg).float().eval()
    with torch.no_grad():
        m.lm_head.weight.mul_(8.0)
        m.lm_head.weight[[5, 6]] += 0.3 * m.model.norm.weight  # eos ids 5 / 6 are likely: beams finish early
    m.generation_config.eos_token_id = m.generation_config.pad_token_id = m.generation_config.bos_token_id = None
    return m


def _logits_fn(m):
    return lambda seqs: m(input_ids=seqs, use_cache=False).logits[:, -1].float()


class KeywordBool:
    """Like the reference's KeywordsStoppingCriteria (llava/mm_utils.py:109-114): one plain bool for the whole batch."""

    def __init__(self, tok):
        self.tok = tok

    def __call__(self, ids, scores, **kw):
        return bool((ids[:, -1] == self.tok).any())


class RowTail:
    """Per-row tensor criterion: the last two tokens are equal."""

    def __call__(self, ids, scores, **kw):
        return (ids[:, -1] == ids[:, -2]) if ids.shape[1] >= 2 else torch.zeros(ids.shape[0], dtype=torch.bool)


EOS = {"none": None, "one": [5], "two": [5, 6]}
CASES = list(itertools.product([2, 3, 5], [1, 3], [False, True, "never"], ["none", "one", "two"]))


@pytest.mark.parametrize("nb,B,es,eos", CASES)
def test_oracle_equals_transformers_beam_search(nb, B, es, eos):
    from transformers import StoppingCriteriaList

    i = CASES.index((nb, B, es, eos))
    lp = [1.0, 0.0, -0.5, 2.0][i % 4]
    nrs = [1, nb][(i // 4) % 2]
    crit = [None, [KeywordBool(7)], [RowTail()]][i % 3]
    m = _hf_model(seed=i)
    g = torch.Generator().manual_seed(i)
    prompt = torch.randint(8, V, (B, 5), generator=g)
    kw = dict(num_beams=nb, do_sample=False, max_new_tokens=9, length_penalty=lp, early_stopping=es, num_return_sequences=nrs,
              use_cache=False, output_scores=True, return_dict_in_generate=True)
    if EOS[eos] is not None:
        kw["eos_token_id"] = EOS[eos]
    if crit:
        kw["stopping_criteria"] = StoppingCriteriaList(crit)
    with torch.no_grad():
        hf = m.generate(prompt, attention_mask=torch.ones_like(prompt), **kw)
        seq, scores = BO.beam_search(_logits_fn(m), prompt, nb, 9, EOS[eos], None, lp, es, nrs, crit)
    assert torch.equal(seq, hf.sequences), (seq, hf.sequences)
    torch.testing.assert_close(scores, hf.sequences_scores.float(), atol=1e-5, rtol=0)


class SlotStandIn:
    """CPU stand-in for the engine's cache and b2_beam_step: slot histories are real token lists, copies follow the C ABI's
    rules, logits of beam i come from the history of slot slot_of_beam[i]."""

    def __init__(self, logits_fn, prompt, n_slots):
        self.fn = logits_fn
        self.hist = [list(map(int, prompt[b])) if b < prompt.shape[0] else [] for b in range(n_slots)]

    def _topk(self, logits, scores, nb, K):
        lp = torch.log_softmax(logits.float(), -1)
        B = scores.numel() // nb
        Vv = lp.shape[-1]
        allc = (lp + scores.view(-1, 1)).view(B, nb * Vv)
        s, idx = BO.select_candidates(allc, K)
        return s, idx % Vv, idx // Vv

    def first(self, B, K):
        logits = self.fn(torch.tensor([self.hist[b] for b in range(B)]))
        return self._topk(logits, torch.zeros(B), 1, K)

    def step(self, copies, row_begin, tokens, slot_of, scores, nb, K):
        srcs = {s for s, _ in copies}
        assert not any(d in srcs for _, d in copies) and len({d for _, d in copies}) == len(copies)
        for s, d in copies:
            assert len(self.hist[s]) >= row_begin and self.hist[d][:row_begin] == self.hist[s][:row_begin]
            self.hist[d] = self.hist[d][:row_begin] + self.hist[s][row_begin:]
        for t, s in zip(tokens, slot_of):
            self.hist[s] = self.hist[s] + [int(t)]
        logits = self.fn(torch.tensor([self.hist[s] for s in slot_of]))
        return self._topk(logits, torch.tensor(scores), nb, K)


@pytest.mark.parametrize("nb,B,es,eos", CASES[::2])
def test_host_half_equals_oracle(nb, B, es, eos):
    i = CASES.index((nb, B, es, eos))
    lp = [1.0, 0.0, -0.5, 2.0][i % 4]
    nrs = [1, nb][(i // 4) % 2]
    crit = [None, [KeywordBool(7)], [RowTail()]][i % 3]
    m = _hf_model(seed=i)
    fn = _logits_fn(m)
    g = torch.Generator().manual_seed(i)
    prompt = torch.randint(8, V, (B, 5), generator=g)
    with torch.no_grad():
        want = BO.beam_search(fn, prompt, nb, 9, EOS[eos], None, lp, es, nrs, crit)
        search = BM.BeamSearch(prompt, nb, 9, EOS[eos], lp, es, nrs, None, crit)
        eng = SlotStandIn(fn, prompt, B * nb)
        planner = BM.SlotPlanner(B, nb)
        cand, row_begin = eng.first(B, search.K), 0
        while not search.step(*cand):
            copies = planner.plan(search.parents)
            cand = eng.step(copies, row_begin, search.next_tokens().tolist(), planner.flat(),
                            search.running_scores.reshape(-1).tolist(), nb, search.K)
            row_begin = prompt.shape[1]
        got = search.output()
    assert torch.equal(got[0], want[0])
    assert torch.equal(got[1], want[1])


def _simulate(B, nb, parent_steps):
    planner = BM.SlotPlanner(B, nb)
    slot_hist = {s: [("prompt", b)] for b in range(B) for s in [planner.slot_of[b][0]]}
    beam_hist = [[[("prompt", b)] for _ in range(nb)] for b in range(B)]
    for t, parents in enumerate(parent_steps):
        before = [list(r) for r in planner.slot_of]
        copies = planner.plan(parents)
        srcs, dsts = [s for s, _ in copies], [d for _, d in copies]
        assert not set(srcs) & set(dsts) and len(set(dsts)) == len(dsts)
        distinct = sum(len(set(int(p) for p in parents[b])) for b in range(B))
        assert len(copies) == B * nb - distinct                           # minimal: one copy per extra child
        for s, d in copies:
            slot_hist[d] = list(slot_hist[s])
        new_hist = []
        for b in range(B):
            row = []
            for j in range(nb):
                h = beam_hist[b][int(parents[b][j])] + [(t, b, j)]
                row.append(h)
                slot_hist[planner.slot_of[b][j]] = slot_hist[planner.slot_of[b][j]] + [(t, b, j)]
            new_hist.append(row)
        beam_hist = new_hist
        for b in range(B):
            for j in range(nb):
                assert slot_hist[planner.slot_of[b][j]] == beam_hist[b][j], (t, b, j, before)
        assert sorted(planner.flat()) == list(range(B * nb))


@pytest.mark.parametrize("nb", [1, 2, 3, 4, 8])
def test_slot_planner(nb):
    B = 3
    fixed = [[0] * nb,                                   # all children of one parent (the prompt fork)
             list(range(nb)),                            # identity
             [1, 0] + list(range(2, nb)) if nb >= 2 else [0],   # swap
             ([1, 2, 0] + list(range(3, nb))) if nb >= 3 else [0] * nb,  # 3-cycle
             [nb - 1] * nb]
    rng = random.Random(nb)
    steps = [[row] * B for row in fixed]
    steps += [[[rng.randrange(nb) for _ in range(nb)] for _ in range(B)] for _ in range(30)]
    _simulate(B, nb, steps)


def test_output_fill_and_crop():
    """eos finishes beam 0 after one token; returned rows are cropped to the longest and padded with HF's fill value."""
    prompt = torch.tensor([[9, 9, 9]])
    s = BM.BeamSearch(prompt, 2, 4, [5], num_return_sequences=2, pad_token_id=0)
    assert s.fill == 5                                   # a pad id of 0 falls through to eos
    assert BM.BeamSearch(prompt, 2, 4, None, pad_token_id=3).fill == -1
    with pytest.raises(ValueError):
        BM.BeamSearch(prompt, 2, 4, [5], num_return_sequences=3)


@pytest.mark.parametrize("shape", ["tiny", "7b2"])
def test_condition_weights_beam_separates_beams_in_bf16(shape):
    """fp32 and bf16 oracle runs pick the same beams on condition_weights_beam weights (the strict-greedy argument of
    condition_weights, extended to beam search)."""
    cfg = O.CONFIGS["tiny"] if shape == "tiny" else dict(O.CONFIGS["llava-1.5-7b"], layers=2)
    w = BO.condition_weights_beam(O.make_weights(cfg, seed=3) if shape == "tiny" else _lm_weights(cfg), cfg, seed=3)
    g = torch.Generator().manual_seed(4)
    prompt = torch.randint(3, cfg["vocab"], (1, 6), generator=g)

    def fn(dtype):
        def f(seqs):
            emb = w["model.embed_tokens.weight"][seqs].to(dtype)
            return O.llama_forward(w, emb, cfg, dtype=dtype, last_only=True)[0][:, -1]
        return f

    with torch.no_grad():
        a = BO.beam_search(fn(torch.float32), prompt, 4, 5, None)
        b = BO.beam_search(fn(torch.bfloat16), prompt, 4, 5, None)
    assert torch.equal(a[0], b[0])


def _lm_weights(cfg):
    """Decoder-only weights at cfg's shapes (the vision tower is not needed for a text-only beam search)."""
    g = torch.Generator().manual_seed(3)
    w = {}
    for key, shape, kind in O.weight_shapes(dict(cfg, vit_layers=0)):
        if key.startswith(O.VT) or "mm_projector" in key:
            continue
        t = torch.randn(*shape, generator=g) * O.init_std(kind, shape)
        w[key] = (t + 1.0 if kind == "g" else t).to(torch.bfloat16).float()
    return w
