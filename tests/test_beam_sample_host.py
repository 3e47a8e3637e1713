"""CPU: beam sampling semantics (generate(do_sample=True, num_beams > 1)).

- torch.multinomial without replacement is top-K of p / Exp(1) in the installed torch: HF's candidate list is in draw order.
- tests/beam_sampling_ref.beam_search(sampler="torch") equals the installed transformers' beam sampling under the same seed.
- The device's warper survivors (beam_sampling_ref.kept_mask) equal HF's Temperature -> TopK -> TopP on log_softmax rows.
- The Philox rule draws ordered K-tuples with the Plackett-Luce probabilities of softmax(acc) (chi-square), and includes tokens
  as often as torch.multinomial does.
- generate() argument handling and the host loop of beam sampling over a stand-in engine that applies the Philox rule."""
import itertools
import types

import numpy as np
import pytest
import torch
from scipy import stats

import beam_sampling_ref as BSR
from llava import _b2
from llava._b2 import beam as BM

V = 64


def _hf_model(seed=0):
    from transformers import LlamaConfig, LlamaForCausalLM

    torch.manual_seed(seed)
    cfg = LlamaConfig(vocab_size=V, hidden_size=32, intermediate_size=64, num_hidden_layers=2, num_attention_heads=2,
                      num_key_value_heads=2, max_position_embeddings=128, bos_token_id=None, eos_token_id=None,
                      pad_token_id=None, attn_implementation="eager")
    m = LlamaForCausalLM(cfg).float().eval()
    with torch.no_grad():
        m.lm_head.weight.mul_(4.0)
        m.lm_head.weight[[5, 6]] += 0.3 * m.model.norm.weight  # eos ids 5 / 6 are likely: beams finish early
    m.generation_config.eos_token_id = m.generation_config.pad_token_id = m.generation_config.bos_token_id = None
    return m


def _logits_fn(m):
    return lambda seqs: m(input_ids=seqs, use_cache=False).logits[:, -1].float()


# ------------------------------------------------------------------------------------------------ draw order of torch
@pytest.mark.parametrize("seed", range(20))
def test_multinomial_is_topk_of_p_over_exponential_noise(seed):
    g = torch.Generator().manual_seed(1000 + seed)
    n, k = [(3, 8), (2, 64), (4, 300)][seed % 3]
    p = torch.softmax(torch.randn(n, k * 5, generator=g) * 3, -1)
    p[0, :k] = 0.0                                                # zero-probability entries, as warped-away tokens give
    K = k
    torch.manual_seed(seed)
    a = torch.multinomial(p, K, replacement=False)
    torch.manual_seed(seed)
    q = torch.empty_like(p).exponential_(1)
    b = torch.topk(p / q, K).indices
    assert torch.equal(a[:, :k // 2], b[:, :k // 2])              # positive-probability draws: same ids, same order
    pos = (p > 0).sum(-1)
    for r in range(n):
        m = min(int(pos[r]), K)
        assert torch.equal(a[r, :m], b[r, :m]), r


# ---------------------------------------------------------------------------------- reference against transformers
EOS = {"none": None, "one": [5], "two": [5, 6]}
CASES = list(itertools.product([2, 3, 5], [1, 3], [False, True, "never"], ["none", "one", "two"]))
TEMPS, TOPK, TOPP = [0.2, 0.7, 1.0, 1.5], [0, 5, 50], [1.0, 0.9, 0.5]


@pytest.mark.parametrize("nb,B,es,eos", CASES)
def test_reference_equals_transformers_beam_sampling(nb, B, es, eos):
    i = CASES.index((nb, B, es, eos))
    T, tk, tp = TEMPS[i % 4], TOPK[(i // 4) % 3], TOPP[(i // 2) % 3]
    lp = [1.0, 0.0, -0.5, 2.0][(i // 3) % 4]
    nrs = [1, nb][i % 2]
    m = _hf_model(seed=i)
    g = torch.Generator().manual_seed(i)
    prompt = torch.randint(8, V, (B, 5), generator=g)
    kw = dict(num_beams=nb, do_sample=True, temperature=T, top_k=tk, top_p=tp, max_new_tokens=9, length_penalty=lp,
              early_stopping=es, num_return_sequences=nrs, use_cache=False, output_scores=True, return_dict_in_generate=True)
    if EOS[eos] is not None:
        kw["eos_token_id"] = EOS[eos]
    drawn = []
    real = torch.multinomial

    def recording(*a, **k):                                       # every draw of HF's run, replayed into the reference
        out = real(*a, **k)
        drawn.append(out)
        return out

    with torch.no_grad():
        torch.multinomial = recording
        try:
            hf = m.generate(prompt, attention_mask=torch.ones_like(prompt), **kw)
        finally:
            torch.multinomial = real
        replay = iter(drawn)

        def replaying(p, num_samples, **k):
            out = next(replay)
            assert out.shape == (p.shape[0], num_samples)
            assert bool((torch.gather(p, 1, out)[:, 0] > 0).all())   # the recorded first draw is possible under our p
            return out

        torch.multinomial = replaying
        try:
            seq, scores = BSR.beam_search(_logits_fn(m), prompt, nb, 9, EOS[eos], None, lp, es, nrs, do_sample=True,
                                          temperature=T, top_k=tk, top_p=tp, sampler="torch")
        finally:
            torch.multinomial = real
        assert next(replay, None) is None                         # one draw per step, as many steps as HF
        # and without the replay: the same seed gives the same run (HF draws from torch's generator nowhere else)
        torch.manual_seed(77 + i)
        hf2 = m.generate(prompt, attention_mask=torch.ones_like(prompt), **kw)
        torch.manual_seed(77 + i)
        seq2, _ = BSR.beam_search(_logits_fn(m), prompt, nb, 9, EOS[eos], None, lp, es, nrs, do_sample=True, temperature=T,
                                  top_k=tk, top_p=tp, sampler="torch")
    assert torch.equal(seq, hf.sequences), (seq, hf.sequences)
    torch.testing.assert_close(scores, hf.sequences_scores.float(), atol=1e-5, rtol=0)
    assert torch.equal(seq2, hf2.sequences)


# ------------------------------------------------------------------------------------------------------ warper survivors
@pytest.mark.parametrize("V_", [50, 32000])
@pytest.mark.parametrize("min_keep", [1, 2, 3])
def test_warper_survivors_equal_transformers(V_, min_keep):
    rng = np.random.default_rng(V_ + min_keep)
    n = 0
    for case in range(40):
        x = (rng.standard_normal(V_) * rng.choice([0.5, 2.0, 6.0])).astype(np.float32)
        if case % 5 == 0:
            x[rng.choice(V_, V_ // 4, replace=False)] = -np.inf
        T = float(rng.choice([0.2, 0.7, 1.0, 1.5]))
        tk = int(rng.choice([0, 1, 5, 50]))
        tp = float(rng.choice([1.0, 0.95, 0.5, 0.05, 1e-6]))
        ours = np.isfinite(BSR.device_warp(x, T, tk, tp, min_keep))
        lp = torch.log_softmax(torch.from_numpy(x)[None], -1)
        hf = torch.isfinite(BSR.hf_warp_installed(lp, T, tk, tp, min_keep))[0].numpy()
        assert np.array_equal(ours, hf), (case, T, tk, tp, np.flatnonzero(ours != hf))
        assert torch.equal(torch.isfinite(BSR.hf_warp(lp, T, tk, tp, min_keep)), torch.isfinite(BSR.hf_warp_installed(lp, T, tk, tp, min_keep)))
        assert ours.sum() >= min(min_keep, np.isfinite(x).sum())
        n += 1
    assert n == 40


def test_philox_vectorised_equals_the_scalar_oracle():
    from oracle import sampling_oracle as SO

    rows = np.array([0, 1, 31999, 2**31 + 5, 2**32 - 1], dtype=np.uint64)
    for seed, step in [(0, 0), (12345678901234, 7), (2**62 - 1, 2**32 - 1)]:
        got = BSR.philox_u64_np(seed, step, rows)
        assert [int(v) for v in got] == [SO.philox_u64(seed, step, int(r)) for r in rows]


# ------------------------------------------------------------------------------------------------- the Philox rule's law
def _pl_prob(p, tup):
    q, left = 1.0, 1.0
    for t in tup:
        q *= p[t] / left
        left -= p[t]
    return q


def test_philox_rule_draws_plackett_luce_tuples():
    """Ordered 2-tuples of 2 beams x 3 tokens (K = 2) over 30000 draws: chi-square against the exact Plackett-Luce law of
    softmax(acc), and inclusion counts against torch.multinomial's (contingency chi-square)."""
    nb, Vs, K, N = 2, 3, 2, 30000
    acc = np.array([[-0.3, -1.2, -2.0, -0.9, -1.6, -0.7]], dtype=np.float32)
    p = np.exp(acc[0].astype(np.float64))
    p /= p.sum()
    counts = {}
    incl = np.zeros(nb * Vs)
    for t in range(N):
        _, idx, _, _ = BSR.philox_select(acc, 424242, t, nb, K)
        tup = tuple(int(v) for v in idx[0])
        counts[tup] = counts.get(tup, 0) + 1
        incl[list(tup)] += 1
    tuples = list(itertools.permutations(range(nb * Vs), K))
    obs = np.array([counts.get(t, 0) for t in tuples], dtype=np.float64)
    exp = np.array([_pl_prob(p, t) for t in tuples]) * N
    assert abs(exp.sum() - N) < 1e-6 * N
    chi = stats.chisquare(obs, exp)
    print(f"ordered tuples: chi2 {chi.statistic:.1f} over {len(tuples) - 1} dof, p = {chi.pvalue:.3f}")
    assert chi.pvalue > 1e-3
    g = torch.Generator().manual_seed(5)
    tm = torch.multinomial(torch.from_numpy(p).float().expand(N, -1).contiguous(), K, generator=g)
    incl_t = np.bincount(tm.reshape(-1).numpy(), minlength=nb * Vs)
    ct = stats.chi2_contingency(np.stack([incl, incl_t]))
    print(f"inclusion vs torch.multinomial: p = {ct.pvalue:.3f}")
    assert ct.pvalue > 1e-3


def test_philox_rule_fill_order():
    """Fewer finite candidates than K: finite by key, then -inf by flat index, then NaN by flat index."""
    acc = np.array([[-np.inf, 0.5, np.nan, -np.inf, -1e9, -np.inf]], dtype=np.float32)
    s, idx, _, _ = BSR.philox_select(acc, 1, 0, 2, 6)
    assert set(idx[0, :2].tolist()) == {1, 4} and idx[0, 0] == 1      # -1e9 + g cannot beat 0.5 + g
    assert idx[0, 2:].tolist() == [0, 3, 5, 2]
    assert np.isnan(s[0, -1]) and np.isinf(s[0, 2])
    # NaN logits stay NaN through every warper (top-k, top-p with min_keep): they rank below -inf, not among it
    x = np.array([np.nan, 2.0, 1.0, np.nan, -1.0, 0.5], dtype=np.float32)
    for tk, tp, mk in [(2, 1.0, 1), (0, 1e-6, 1), (2, 0.5, 2), (50, 0.9, 3)]:
        w = BSR.device_warp(x, 0.7, tk, tp, mk)
        assert np.isnan(w[[0, 3]]).all() and np.isfinite(w[1]) and not np.isnan(w[[1, 2, 4, 5]]).any(), (tk, tp, mk, w)


# ------------------------------------------------------------------------------------------------------- generate()
class SampleEngine:
    """Stand-in for the engine's beam entry points on the CPU: per-slot token histories, logits from `fn`, candidates by the
    Philox rule (beam_sampling_ref.philox_select) or, without sampling, best first (oracle select_candidates)."""

    def __init__(self, fn, vocab):
        self.fn, self.vocab, self.hist, self.calls = fn, vocab, {}, []
        self.device = "cpu"

    def prefill(self, kv, embeds, lens, mode):
        for b in range(embeds.shape[0]):
            self.hist[b] = [int(t) for t in embeds[b]]
        return self.fn(embeds)

    def _select(self, logits, run, nb, K, sampling, step, rows=None):
        logits = logits if rows is None else logits[torch.as_tensor(rows)]
        Vv = logits.shape[-1]
        B = run.numel() // nb
        if sampling is None:
            from oracle import beam_oracle as BO
            s, i = BO.select_candidates((torch.log_softmax(logits.float(), -1) + run.view(-1, 1)).view(B, nb * Vv), K)
            return s, i % Vv, i // Vv
        w = np.stack([BSR.device_warp(r, sampling.temperature, sampling.top_k, sampling.top_p, sampling.min_keep)
                      for r in logits.float().numpy()])
        acc = (w.reshape(B, nb, Vv) + run.numpy().reshape(B, nb, 1).astype(np.float32)).astype(np.float32).reshape(B, nb * Vv)
        s, i, _, _ = BSR.philox_select(acc, sampling.seed, step, nb, K)
        i = torch.from_numpy(i.astype(np.int64))
        return torch.from_numpy(s.astype(np.float32)), i % Vv, i // Vv

    def beam_topk(self, logits, scores, nb, K, row_of_beam=None):
        self.calls.append("topk")
        return self._select(logits, scores.float(), nb, K, None, 0, row_of_beam)

    def beam_sample(self, logits, scores, nb, K, sampling, step, row_of_beam=None):
        self.calls.append(("sample", step, tuple(row_of_beam or ()), tuple(scores.tolist())))
        return self._select(logits, scores.float(), nb, K, sampling, step, row_of_beam)

    def beam_step(self, kv, copies, row_begin, tokens, slot_of, scores, nb, K, sampling=None, step=0):
        self.calls.append(("step", step, sampling is not None))
        new = dict(self.hist)
        for s, d in copies:
            new[d] = self.hist[s][:]
        for t, s in zip(tokens, slot_of):
            new[s] = new[s] + [int(t)]
        self.hist = new
        logits = self.fn(torch.tensor([self.hist[s] for s in slot_of]))
        return self._select(logits, torch.tensor(scores), nb, K, sampling, step)

    def take_async_error(self):
        return 0

    def check_async_error(self):
        pass


def _stub(fn, cap=4, **cfg):
    from llava.model.language_model.llava_llama import LlavaLlamaForCausalLM as M

    eng = SampleEngine(fn, V)

    class Pool:
        def acquire(self):
            return types.SimpleNamespace(reset=lambda: None)

        def release(self, kv):
            pass

    class Stub:
        config = types.SimpleNamespace(b2_beam_search=cap, eos_token_id=None, **cfg)
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
    for k in ("B2_BEAM_SAMPLE", "B2_BEAM_SEARCH", "B2_PROMPT_LOOKUP", "B2_LOGITS_PROCESSORS"):
        monkeypatch.delenv(k, raising=False)


def test_generate_arguments(no_env, monkeypatch):
    m = _hf_model(seed=3)
    fn = _logits_fn(m)
    p = torch.randint(8, V, (1, 5), generator=torch.Generator().manual_seed(3))
    off, _ = _stub(fn)
    with pytest.raises(NotImplementedError, match="beam sampling"):           # the off switch raises as before
        off(p, num_beams=2, do_sample=True, temperature=0.7, max_new_tokens=3)
    gen, eng = _stub(fn, b2_beam_sample=True)
    with pytest.raises(ValueError, match="num_beams"):
        gen(p, num_beams=5, do_sample=True, max_new_tokens=3)              # the cap of b2_beam_search still applies
    with pytest.raises(ValueError, match="streamer"):
        gen(p, num_beams=2, do_sample=True, max_new_tokens=3, streamer=object())
    for bad in (0.0, 1.5, -0.1):
        with pytest.raises(ValueError, match="top_p"):
            gen(p, num_beams=2, do_sample=True, top_p=bad, max_new_tokens=3)
    with pytest.raises(NotImplementedError):
        gen(p, num_beams=2, do_sample=True, max_new_tokens=3, num_beam_groups=2)
    with pytest.raises(NotImplementedError):
        gen(p, num_beams=2, do_sample=True, max_new_tokens=3, repetition_penalty=1.2)
    # temperature <= 1e-5 is beam search, with or without do_sample
    with torch.no_grad():
        a = gen(p, num_beams=2, do_sample=True, temperature=0.0, max_new_tokens=4, eos_token_id=[5])
    assert eng.calls[0] == "topk" and not any(isinstance(c, tuple) and c[0] == "sample" for c in eng.calls)
    from oracle import beam_oracle as BO
    with torch.no_grad():
        assert torch.equal(a, BO.beam_search(fn, p, 2, 4, [5])[0])
    monkeypatch.setenv("B2_BEAM_SAMPLE", "1")                              # the environment switch
    gen_env, _ = _stub(fn)
    with torch.no_grad():
        gen_env(p, num_beams=2, do_sample=True, max_new_tokens=2)


@pytest.mark.parametrize("B,nb,eos,T,tk,tp", [(1, 2, None, 0.7, 50, 1.0), (3, 3, [5], 0.2, 50, 1.0), (2, 4, [5, 6], 1.0, 0, 0.9),
                                               (1, 3, [], 1.5, 5, 0.5)])
def test_generate_host_loop_equals_the_philox_reference(no_env, B, nb, eos, T, tk, tp):
    """generate() over the stand-in: the seed from torch's generator, draw index t at step t, the first draw over all nb rows
    mapped to the prefill row with scores [0, -1e9, ...], and min_keep = 1 + n_eos (2 without eos ids)."""
    m = _hf_model(seed=B * 10 + nb)
    fn = _logits_fn(m)
    p = torch.randint(8, V, (B, 5), generator=torch.Generator().manual_seed(nb))
    gen, eng = _stub(fn, b2_beam_sample=True)
    kw = dict(num_beams=nb, do_sample=True, temperature=T, top_k=tk, top_p=tp, max_new_tokens=8, num_return_sequences=nb)
    if eos is not None:
        kw["eos_token_id"] = eos
    with torch.no_grad():
        torch.manual_seed(123)
        got = gen(p, **kw)
        torch.manual_seed(123)
        seed = int(torch.randint(0, 2**62, (1,), dtype=torch.int64).item())
        want = BSR.beam_search(fn, p, nb, 8, eos, None, 1.0, False, nb, do_sample=True, temperature=T, top_k=tk, top_p=tp,
                               sampler="philox", seed=seed)[0]
        torch.manual_seed(123)
        again = gen(p, **kw)
    assert torch.equal(got, want), (got, want)
    assert torch.equal(again, got)
    first = next(c for c in eng.calls if isinstance(c, tuple) and c[0] == "sample")
    assert first[1] == 0 and first[2] == tuple(b for b in range(B) for _ in range(nb))
    assert first[3] == tuple(([0.0] + [-1e9] * (nb - 1)) * B)
    steps = [c[1] for c in eng.calls if isinstance(c, tuple) and c[0] == "step"]
    assert all(s for c in eng.calls if isinstance(c, tuple) and c[0] == "step" for s in [c[2]])
    assert steps[:len(steps) // 2] == list(range(1, len(steps) // 2 + 1))


def test_beam_sampling_struct_defaults():
    s = _b2.make_beam_sampling(0.2, None, None, 3, 2**64 + 5)
    assert (s.top_k, s.top_p, s.min_keep, s.seed) == (0, 1.0, 3, 5)
    assert abs(s.temperature - 0.2) < 1e-7
    assert BM.BeamSearch(torch.zeros(1, 2, dtype=torch.long), 3, 4, [1, 2]).K == 9 and BSR.min_keep_of([1, 2]) == 3
    assert BSR.min_keep_of(None) == 2 and BSR.min_keep_of([]) == 1
