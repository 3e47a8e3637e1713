"""CPU: generate(do_sample=True, num_return_sequences=n) without a GPU.

- ForkPlan: leader and follower slots, the one copy call, the group table (n > 16, unequal prompt lengths) and the slot <-> HF
  row permutation.
- generate() over a CPU stand-in of the streaming engine that keeps the device's slot order: the result [B * n, Lt + new] in
  repeat_interleave order, score rows permuted to HF's rows, eos / pad per row, stopping criteria and the streamer seeing
  HF-ordered ids, one prefill of B rows.
- The argument matrix: greedy raises transformers' own GenerationConfig.validate error, a list of images, the continuous
  batcher and an explicit prompt_lookup_num_tokens raise, beams keep their handling.
- The mutated references of the shared-prefix kernel test (reading the row's own prefix, the source past P, P off by one) each
  leave the attention bound."""
import types

import pytest
import torch

from llava._b2.fork import GROUP_ROWS, ForkPlan
from llava.model.language_model.llava_llama import LlavaLlamaForCausalLM as M
from test_attention_numerics_gpu import attend, bound, rope_rows_cpu
from test_num_return_gpu import KERNEL_CASES, _kid, build_shared, shared_problems

V = 23


# ------------------------------------------------------------------------------------------------------ planner
def test_plan_slots_copies_and_permutation():
    p = ForkPlan([5, 7, 3], 4)
    assert [p.slot(b, 0) for b in range(3)] == [0, 1, 2]
    assert [p.slot(1, j) for j in range(4)] == [1, 6, 7, 8]
    src, dst = p.copies()
    assert src == [0, 0, 0, 1, 1, 1, 2, 2, 2] and dst == list(range(3, 12))
    assert not set(src) & set(dst) and len(set(dst)) == len(dst)
    sor = p.slot_of_row
    assert sorted(sor) == list(range(12))
    assert [p.prompt_of_slot[s] for s in sor] == [r // 4 for r in range(12)]  # row b * n + j belongs to prompt b
    assert p.groups() == [(0, 5, [0, 3, 4, 5]), (1, 7, [1, 6, 7, 8]), (2, 3, [2, 9, 10, 11])]


@pytest.mark.parametrize("n", [1, 2, 16, 17, 33])
def test_groups_split_past_sixteen_rows(n):
    p = ForkPlan([9, 4], n)
    gs = p.groups()
    assert all(1 <= len(r) <= GROUP_ROWS for _, _, r in gs)
    assert len(gs) == 2 * -(-n // GROUP_ROWS)
    for b, plen in ((0, 9), (1, 4)):
        mine = [g for g in gs if g[0] == b]
        assert all(g[1] == plen for g in mine)
        assert sorted(r for g in mine for r in g[2]) == sorted(p.slot(b, j) for j in range(n))
    if n == 1:
        assert p.copies() == ([], [])


# ------------------------------------------------------------------------------------------------------ generate()
def _next(tok, slot):
    return (tok * 7 + 3 + slot) % V


class ForkEngine:
    """The streaming half of the engine in slot order: token t of slot s = f(token t - 1 of s, s), token 0 from the prefill
    row of the slot's prompt (its argmax), so siblings differ from step 1 on. Score / logits rows get [slot, t] markers."""
    vocab = V
    device = torch.device("cpu")

    def __init__(self):
        self.prefills, self.copies, self.groups, self.B = [], [], None, 0

    def prefill(self, kv, embeds, lens, mode):
        self.prefills.append(embeds.shape[0])
        logits = torch.zeros(embeds.shape[0], V)
        for b in range(embeds.shape[0]):
            logits[b, int(embeds[b, -1]) % V] = 1.0
        return logits

    def kv_copy_slots(self, kv, src, dst, row_begin=0):
        self.copies.append((list(src), list(dst)))

    def stream_begin(self, kv, logits, sampling, procs=None, out_scores=None, out_logits=None, groups=None, share_prefix=True):
        self.B, self.groups, self.rows = logits.shape[0], groups, (out_scores, out_logits)
        self.tokens = [[int(x) for x in logits.argmax(-1)]]
        self._mark(0)

    def _mark(self, t):
        for buf in self.rows:
            if buf is not None and t < buf.shape[0]:
                for s in range(self.B):
                    buf[t, s] = 0.0
                    buf[t, s, :2] = torch.tensor([float(s), float(t)])

    def stream_enqueue(self, kv, n):
        for _ in range(n):
            self.tokens.append([_next(tok, s) for s, tok in enumerate(self.tokens[-1])])
            self._mark(len(self.tokens) - 1)

    def stream_wait(self, kv, index, B, timeout_ms=0):
        assert B == self.B
        return list(self.tokens[index])

    def take_async_error(self):
        return 0

    def check_async_error(self):
        pass


def _stub(**cfg):
    eng = ForkEngine()

    class Pool:
        def acquire(self):
            return types.SimpleNamespace(reset=lambda: None)

        def release(self, kv, record=None):
            pass

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
        _prefix_cache_on = lambda self: False  # noqa: E731
        _pool = Pool()

        def _ensure_engine(self):
            return eng

        def _get_batcher(self, engine):
            return None

        def _prompt_embeds(self, engine, prompt, attention_mask, images, force_host):
            return prompt, [prompt.shape[1]] * prompt.shape[0], False

        def _check_limits(self, engine, n, length):
            pass

    stub = Stub()
    return (lambda *a, **k: M.generate.__wrapped__(stub, *a, **k)), eng


@pytest.fixture
def no_env(monkeypatch):
    for k in ("B2_BEAM_SAMPLE", "B2_BEAM_SEARCH", "B2_PROMPT_LOOKUP", "B2_LOGITS_PROCESSORS", "B2_KV_DTYPE"):
        monkeypatch.delenv(k, raising=False)


def _expected(prompt, n, steps, eos=(), pad=0):
    """What the stand-in generates, in HF's row order, with finished rows showing pad."""
    B = prompt.shape[0]
    plan = ForkPlan([prompt.shape[1]] * B, n)
    cur = {plan.slot(b, j): int(prompt[b, -1]) % V for b in range(B) for j in range(n)}
    cols, done = [], [False] * (B * n)
    for _ in range(steps):
        col = []
        for r, s in enumerate(plan.slot_of_row):
            col.append(pad if done[r] else cur[s])
        for r in range(B * n):
            done[r] = done[r] or col[r] in eos
        cols.append(col)
        if eos and all(done):
            break
        cur = {s: _next(t, s) for s, t in cur.items()}
    return torch.tensor(cols).t()


@pytest.mark.parametrize("B,n", [(1, 3), (2, 4), (3, 17)])
def test_result_rows_in_repeat_interleave_order(no_env, B, n):
    gen, eng = _stub()
    prompt = torch.randint(1, V, (B, 5), generator=torch.Generator().manual_seed(B * n))
    out = gen(prompt, do_sample=True, num_return_sequences=n, max_new_tokens=6)
    assert out.shape == (B * n, 5 + 6)
    assert torch.equal(out[:, :5], prompt.repeat_interleave(n, 0))
    assert torch.equal(out[:, 5:], _expected(prompt, n, 6))
    plan = ForkPlan([5] * B, n)
    assert eng.prefills == [B] and eng.copies == [plan.copies()] and eng.groups == plan.groups()


def test_score_rows_follow_hf_rows(no_env):
    gen, _ = _stub()
    prompt = torch.randint(1, V, (2, 4), generator=torch.Generator().manual_seed(1))
    out = gen(prompt, do_sample=True, num_return_sequences=3, max_new_tokens=4, return_dict_in_generate=True, output_scores=True,
              output_logits=True)
    slot = ForkPlan([4, 4], 3).slot_of_row
    for rows in (out.scores, out.logits):
        assert len(rows) == 4
        for t, row in enumerate(rows):
            assert row.shape == (6, V)
            assert row[:, 0].tolist() == [float(s) for s in slot] and row[:, 1].tolist() == [float(t)] * 6


def test_eos_pad_and_stopping_criteria_see_hf_rows(no_env):
    prompt = torch.tensor([[3, 9], [4, 11]])
    free = _expected(prompt, 3, 12)
    eos = {int(free[1, 2]), int(free[4, 5])}
    gen, _ = _stub()
    seen = []

    def crit(ids, scores):
        seen.append(ids.clone())
        return False

    out = gen(prompt, do_sample=True, num_return_sequences=3, max_new_tokens=12, eos_token_id=list(eos), pad_token_id=0,
              stopping_criteria=[crit])
    want = _expected(prompt, 3, 12, eos, 0)
    assert torch.equal(out[:, 2:], want)
    assert torch.equal(seen[-1], out)  # the criteria saw the HF-ordered rows, prompt included


def test_streamer_gets_the_expanded_rows(no_env):
    class Rec:
        def __init__(self):
            self.got = []

        def put(self, v):
            self.got.append(v.clone())

        def end(self):
            pass

    gen, _ = _stub()
    prompt = torch.tensor([[3, 9]])
    st = Rec()
    out = gen(prompt, do_sample=True, num_return_sequences=2, max_new_tokens=3, streamer=st)
    assert torch.equal(st.got[0], prompt.repeat_interleave(2, 0))
    assert torch.equal(torch.stack(st.got[1:], 1), out[:, 2:])


def test_greedy_like_temperature_is_greedy(no_env):
    gen, eng = _stub()
    prompt = torch.tensor([[3, 9]])
    gen(prompt, do_sample=True, temperature=1e-6, num_return_sequences=2, max_new_tokens=2)
    assert eng.groups == ForkPlan([2], 2).groups()


# ------------------------------------------------------------------------------------------------------ arguments
def test_greedy_raises_transformers_error(no_env):
    from transformers import GenerationConfig

    with pytest.raises(ValueError) as hf:
        GenerationConfig(num_return_sequences=2).validate()
    gen, _ = _stub()
    with pytest.raises(ValueError) as ours:
        gen(torch.tensor([[3, 9]]), do_sample=False, num_return_sequences=2, max_new_tokens=2)
    assert str(ours.value) == str(hf.value)


@pytest.mark.parametrize("cfg,kw,exc,match", [
    (dict(), dict(images=[torch.zeros(3, 4, 4)]), NotImplementedError, "list of images"),
    (dict(b2_continuous_batching=4), dict(), NotImplementedError, "continuous batcher"),
    (dict(b2_prompt_lookup=4), dict(prompt_lookup_num_tokens=3), ValueError, "num_return_sequences has to be 1 when doing assisted"),
    (dict(), dict(prompt_lookup_num_tokens=3), ValueError, "num_return_sequences has to be 1 when doing assisted"),
])
def test_refused_combinations(no_env, cfg, kw, exc, match):
    gen, eng = _stub(**cfg)
    with pytest.raises(exc, match=match):
        gen(torch.tensor([[3, 9]]), do_sample=True, num_return_sequences=2, max_new_tokens=2, **kw)
    assert eng.prefills == []


def test_prompt_lookup_opt_in_is_not_used_for_forks(no_env):
    gen, eng = _stub(b2_prompt_lookup=4)
    out = gen(torch.tensor([[3, 9]]), do_sample=True, num_return_sequences=2, max_new_tokens=3)
    assert out.shape == (2, 5) and eng.groups is not None


def test_beams_keep_their_handling(no_env):
    from test_beam_host import _hf_model, _logits_fn
    from test_beam_sample_host import _stub as beam_stub

    gen, _ = beam_stub(_logits_fn(_hf_model(seed=3)))
    p = torch.randint(8, 40, (1, 5), generator=torch.Generator().manual_seed(3))
    out = gen(p, num_beams=3, num_return_sequences=2, max_new_tokens=4)
    assert out.shape[0] == 2


# ------------------------------------------------------------------------------------------------------ kernel references
def test_mutated_references_violate_the_bound():
    """Reading the row's own prefix, reading the source past P, or P off by one each leave the bound on the kernel test's
    inputs (built here for 3 splits; the GPU test builds them for the device's split factor)."""
    H = 2
    for c in KERNEL_CASES[1:]:
        inp = build_shared(c["Ps"], c["ns"], c["suffix"], H, seed=5, nsplit=3)
        q, k_new = rope_rows_cpu(inp["qkv"], inp["lens"], H)
        good = {(r, h): pr for r, h, pr in shared_problems(inp, q, k_new, H)}
        for name, kw in [("own prefix", dict(own_prefix=True)), ("source past P", dict(src_past=2)), ("P - 1", dict(p_shift=-1)),
                         ("P + 1", dict(p_shift=1))]:
            if kw.get("src_past") and c["suffix"] == 0:
                continue
            worst = 0.0
            for r, h, bad in shared_problems(inp, q, k_new, H, **kw):
                pr = good[(r, h)]
                ref, p = attend(pr)
                got, _ = attend(bad)
                worst = max(worst, float(((got - ref).abs() / bound(pr, ref, p)).max()))
            assert worst > 1.0, f"{_kid(c)}: the {name} mutation stays inside the bound ({worst:.3f})"
