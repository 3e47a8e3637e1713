"""GPU: prompt-lookup speculative decoding (b2_stream_begin_lookup, b2_decode_rows).

- decode_attn_mq against an fp32 reference for R = 1..16 (contexts that are not multiples of the 64-key tile, H = 32 / 40), and
  against decode_attn at R = 1.
- b2_op_prompt_lookup equal to oracle/prompt_lookup_oracle.py.
- b2_decode_rows logits against R teacher-forced decode steps on bf16 and NF4 weights (GEMV rows), and against the oracle
  forward at GEMV and stream-K row counts.
- Streaming with guaranteed acceptance: tokens equal to the plain stream's, accepted drafts counted; a sampled stream checked token
  by token against the oracle selection over the verify logits.
- generate() with and without config.b2_prompt_lookup: the same ids and streamer output."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from helpers import make_engine, make_model, synth_inputs  # noqa: E402
from llava import _b2  # noqa: E402
from oracle import llava_oracle as O  # noqa: E402
from oracle import prompt_lookup_oracle as PL  # noqa: E402
from oracle import sampling_oracle as S  # noqa: E402
from test_nf4_gpu import CFG2, dev_weights, rnd  # noqa: E402

DEV = "cuda"
BF = torch.bfloat16
P = _b2.ptr
MAX_SEQ, PROMPT = 192, 40


def _stream():
    return _b2.stream_ptr()


# ------------------------------------------------------------------------------------------------ decode_attn_mq
def _mq(qkv, kc, vc, lens, R, H, nsplit):
    B = len(lens)
    lib = _b2.load_library()
    scratch = torch.zeros(lib.b2_op_decode_attn_mq_scratch_bytes(B, H, nsplit), device=DEV, dtype=torch.uint8)
    cur = torch.tensor(lens, device=DEV, dtype=torch.int32)
    out = torch.empty(B * R, H * 128, device=DEV, dtype=BF)
    for _ in range(2):  # the second launch checks the self-resetting counters
        _b2.check(lib.b2_op_decode_attn_mq(P(qkv), P(kc), P(vc), P(cur), P(out), P(scratch), B, R, H, kc.shape[2], nsplit,
                                           1 / math.sqrt(128), _stream()), "b2_op_decode_attn_mq")
    return out


@pytest.mark.parametrize("H,lens,nsplit", [(32, [703], 12), (40, [129], 5), (32, [1, 64], 3), (40, [1000], 16)])
def test_decode_attn_mq_equals_fp32_reference(H, lens, nsplit):
    D = 128
    for R in range(1, 17):
        B = len(lens)
        Smax = max(lens) + 16
        qkv = rnd(B * R, 3 * H * D, seed=R)
        kc, vc = rnd(B, H, Smax, D, seed=100 + R), rnd(B, H, Smax, D, seed=200 + R)
        out = _mq(qkv, kc, vc, lens, R, H, nsplit).float()
        q = qkv.view(B, R, 3, H, D)[:, :, 0].float()
        for b in range(B):
            for j in range(R):
                n = lens[b] + j + 1
                s = torch.einsum("hd,hnd->hn", q[b, j], kc[b, :, :n].float()) / math.sqrt(D)
                want = torch.einsum("hn,hnd->hd", torch.softmax(s, -1), vc[b, :, :n].float()).reshape(-1)
                torch.testing.assert_close(out[b * R + j], want, rtol=2e-2, atol=2e-2)


def test_decode_attn_mq_at_one_row_agrees_with_decode_attn():
    """R = 1 over the cache decode_attn appends to: the same attention output within bf16 rounding."""
    B, H, D, n = 1, 32, 128, 517
    Smax = n + 8
    lib = _b2.load_library()
    qkv = rnd(1, 3 * H * D, seed=5)
    kc, vc = rnd(B, H, Smax, D, seed=6), rnd(B, H, Smax, D, seed=7)
    cur = torch.tensor([n], device=DEV, dtype=torch.int32)
    scratch = torch.zeros(lib.b2_op_decode_attn_scratch_bytes(B, H, 4), device=DEV, dtype=torch.uint8)
    ref = torch.empty(1, H * D, device=DEV, dtype=BF)
    _b2.check(lib.b2_op_decode_attn(P(qkv.clone()), P(kc), P(vc), P(cur), P(ref), P(scratch), B, H, Smax, 4, 10000.0,
                                    1 / math.sqrt(D), _stream()))
    # the same step as the verify forward does it: rope + cache write at pos0 = n, then decode_attn_mq over n + 1 keys
    q2 = qkv.clone()
    _b2.check(lib.b2_op_rope_kv_write_at(P(q2), P(kc), P(vc), P(cur), 1, 1, H, D, Smax, 10000.0, _stream()))
    got = _mq(q2, kc, vc, [n], 1, H, 7)
    torch.testing.assert_close(got.float(), ref.float(), rtol=2e-2, atol=2e-2)


# ------------------------------------------------------------------------------------------------ prompt_lookup
def test_op_prompt_lookup_equals_oracle():
    lib = _b2.load_library()
    rng = np.random.default_rng(3)
    V = 32
    out = torch.empty(16, device=DEV, dtype=torch.int32)
    dl = torch.empty(1, device=DEV, dtype=torch.int32)
    for case in range(300):
        L = int(rng.integers(1, 120))
        hist = rng.integers(0, 6 if case % 2 else V, L).astype(np.int32)
        if case % 5 == 0:
            hist[rng.integers(0, L)] = -200
        hist[-1] = abs(hist[-1])
        K, ngram = int(rng.integers(1, 16)), int(rng.integers(1, 5))
        eos = sorted(set(rng.integers(0, 6, int(rng.integers(0, 3))).tolist()))
        max_length = int(rng.choice([L + 1, L + int(rng.integers(2, 30)), max(1, L - 2)]))
        h = torch.from_numpy(hist).to(DEV)
        e = (torch.tensor(eos, dtype=torch.int32) if eos else torch.zeros(1, dtype=torch.int32)).numpy()
        _b2.check(lib.b2_op_prompt_lookup(P(h), L, K, ngram, max_length, e.ctypes.data_as(_b2.ctypes.POINTER(_b2.ctypes.c_int32)),
                                          len(eos), V, P(out), P(dl), _stream()), "b2_op_prompt_lookup")
        want = PL.draft(hist.tolist(), K, ngram, max_length, set(eos), vocab=V)
        d = int(dl.item())
        rows = out[:K + 1].tolist()
        assert d == len(want) and rows[1:1 + d] == want, (case, rows, d, want)
        assert rows[0] == int(hist[-1]) and all(t == rows[0] for t in rows[1 + d:])


# ------------------------------------------------------------------------------------------------ the verify forward
@pytest.fixture(scope="module")
def engines():
    built = {}

    def get(fmt):
        if fmt not in built:
            eng = make_engine(CFG2, dev_weights(CFG2, seed=3), max_batch=12, max_seq=MAX_SEQ, max_images=1)
            if fmt == "nf4":
                eng.enable_nf4()
            built[fmt] = eng
        return built[fmt]

    yield get
    for eng in built.values():
        eng.close()


def _rel(a, b, std):
    d = (a.float() - b.float()).abs()
    return float(d.max()) / std, float(d.mean()) / std


def _steps(eng, emb, toks):
    """Logits of len(toks) teacher-forced batch-1 decode steps after a prefill of `emb` (the megakernel on bf16 weights, gemv_nf4
    on NF4)."""
    kv = eng.new_kv(1, MAX_SEQ)
    eng.prefill(kv, emb, None, _b2.LOGITS_LAST)
    out = torch.stack([eng.decode_step(kv, toks[j:j + 1].to(DEV))[0].cpu() for j in range(len(toks))])
    kv.close()
    return out


def _batch_steps(eng, emb, toks, B=12):
    """The same teacher-forced steps through the multi-kernel decode step at batch B (every slot the same sample; slot 0's
    logits): the stream-K GEMM over the bf16 (or dequantised NF4) weights, another engine path over the same inputs."""
    kv = eng.new_kv(B, MAX_SEQ)
    eng.prefill(kv, emb.expand(B, -1, -1).contiguous(), None, _b2.LOGITS_LAST)
    out = torch.stack([eng.decode_step(kv, toks[j:j + 1].expand(B).contiguous().to(DEV))[0].cpu() for j in range(len(toks))])
    kv.close()
    return out


# The verify forward's Linears run on the GEMV kernels up to 6 rows and on the stream-K GEMM from 7 (decode_plan); the teacher-
# forced steps run on the megakernel (bf16) or gemv_nf4 (NF4). Two engine paths differ by rounding order: the bound is the issue's
# 2 % / 0.3 % of the logit std, or 1.5x what the engine's own batch-12 decode step differs from the same steps by on the same
# inputs, whichever is larger (at 7B width the stream-K step itself differs by about 0.02 / 0.003; DESIGN §4.1).
@pytest.mark.parametrize("fmt", ["bf16", "nf4"])
@pytest.mark.parametrize("R", [4, 6, 8, 12])
def test_decode_rows_equals_teacher_forced_steps(engines, fmt, R):
    eng = engines(fmt)
    emb = rnd(1, PROMPT, CFG2["hidden"], seed=11)
    toks = torch.randint(0, CFG2["vocab"], (R,), generator=torch.Generator().manual_seed(R), dtype=torch.int32)
    kv = eng.new_kv(1, MAX_SEQ)
    eng.prefill(kv, emb, None, _b2.LOGITS_LAST)
    rows = eng.decode_rows(kv, toks).cpu()
    assert kv.lengths(1)[0] == PROMPT + R
    kv.close()
    steps = _steps(eng, emb, toks)
    std = float(steps.std())
    mx, mean = _rel(rows, steps, std)
    g_mx, g_mean = _rel(_batch_steps(eng, emb, toks), steps, std)
    assert mx <= max(0.02, 1.5 * g_mx) and mean <= max(0.003, 1.5 * g_mean), (mx, mean, g_mx, g_mean)


@pytest.mark.parametrize("R", [3, 9, 16])
def test_decode_rows_equals_oracle_forward(engines, R):
    eng = engines("bf16")
    w = dev_weights(CFG2, seed=3)
    emb = rnd(1, PROMPT, CFG2["hidden"], seed=12)
    toks = torch.randint(0, CFG2["vocab"], (R,), generator=torch.Generator().manual_seed(R), dtype=torch.int32)
    kv = eng.new_kv(1, MAX_SEQ)
    eng.prefill(kv, emb, None, _b2.LOGITS_LAST)
    got = eng.decode_rows(kv, toks).cpu()
    kv.close()
    w = {k: v.float().cpu() for k, v in w.items() if k.startswith(("model.embed", "model.layers", "model.norm", "lm_head"))}
    full = torch.cat([emb.float().cpu(), w["model.embed_tokens.weight"][toks.long()][None]], 1)
    ref = O.llama_forward(w, full, CFG2)[0][0, PROMPT:].float()
    mx, mean = _rel(got, ref, float(ref.std()))
    assert mx <= 0.05 and mean <= 0.01, (mx, mean)


# ------------------------------------------------------------------------------------------------ streaming
def _plain(eng, kv, emb, n, sampling):
    logits = eng.prefill(kv, emb, None, _b2.LOGITS_LAST)
    eng.stream_begin(kv, logits, sampling)
    eng.stream_enqueue(kv, n - 1)
    return [eng.stream_wait(kv, t, 1)[0] for t in range(n)]


def _lookup(eng, kv, emb, ids, K, n, sampling, max_new):
    logits = eng.prefill(kv, emb, None, _b2.LOGITS_LAST)
    lk = _b2.make_prompt_lookup(ids.to(DEV), K, 2, max_new)
    eng.stream_begin_lookup(kv, logits, sampling, lk)
    eng.stream_enqueue(kv, n - 1)
    toks = [eng.stream_wait(kv, t, 1)[0] for t in range(n)]
    torch.cuda.synchronize()
    return toks, eng.lookup_stats(kv)


def test_stream_with_guaranteed_acceptance(engines):
    """Prompt ids [.., z, T0 .. T20, .., z] where T is the plain greedy stream of the same embeds: token 0 completes the 2-gram
    (z, T0), and every draft is a true continuation."""
    eng = engines("bf16")
    N = 22
    kv = eng.new_kv(1, MAX_SEQ)
    # the first prompt whose plain stream has no near tie: every step's top-1 minus top-2 logit exceeds the logit error between
    # the two paths, so that equal tokens are a fair requirement
    for seed in range(21, 41):
        emb = rnd(1, PROMPT, CFG2["hidden"], seed=seed)
        plain = _plain(eng, kv, emb, N, _b2.make_sampling())
        ref = eng.new_kv(1, MAX_SEQ)
        lg = [eng.prefill(ref, emb, None, _b2.LOGITS_LAST)[0].cpu()]
        for t in range(N - 1):
            lg.append(eng.decode_step(ref, torch.tensor([plain[t]], dtype=torch.int32, device=DEV))[0].cpu())
        ref.close()
        margins = [float(x.topk(2).values[0] - x.topk(2).values[1]) for x in lg]
        if min(margins) > 0.02 * float(torch.stack(lg).std()):
            break
    else:
        pytest.skip("every prompt tried has a near tie in its plain stream")
    z = CFG2["vocab"] - 7
    ids = torch.tensor([3, 9, z] + plain[:21] + [5, z], dtype=torch.int64)
    K = 3  # R = 4 rows: the GEMV path, whose captured step launches lookup, embed, 6 per layer, lm_head and acceptance
    logits = eng.prefill(kv, emb, None, _b2.LOGITS_LAST)
    eng.stream_begin_lookup(kv, logits, _b2.make_sampling(), _b2.make_prompt_lookup(ids.to(DEV), K, 2, N))
    # one verify step at a time: the published count and the counters after each
    per_step, launches = [], []
    published = 1
    while published < N:
        before = _b2.launch_count()
        eng.stream_enqueue(kv, 1)
        launches.append(_b2.launch_count() - before)
        torch.cuda.synchronize()
        steps, drafted, accepted = eng.lookup_stats(kv)
        per_step.append((steps, drafted, accepted))
        published = 1 + steps + accepted
    eng.stream_enqueue(kv, 1)  # queues nothing: the generation is complete
    toks = [eng.stream_wait(kv, t, 1)[0] for t in range(N)]
    kv.close()
    assert toks == plain
    assert per_step[-1][2] > 0 and len(per_step) < N - 1, per_step
    assert all(n == 4 + 6 * CFG2["layers"] for n in launches[2:]), launches  # graph replays from the third step on
    # host re-derivation of every step: the oracle draft over the history, the verify rows' argmax from b2_decode_rows over the
    # same cache contents, the oracle acceptance
    ref = eng.new_kv(1, MAX_SEQ)
    prev = (0, 0, 0)
    for steps, drafted, accepted in per_step:
        P0 = 1 + prev[0] + prev[2]
        hist = ids.tolist() + toks[:P0]
        draft = PL.draft(hist, K, 2, len(ids) + N, (), vocab=CFG2["vocab"])
        eng.prefill(ref, emb, None, _b2.LOGITS_LAST)
        done = toks[:P0 - 1]
        for c in range(0, len(done), 16):
            eng.decode_rows(ref, done[c:c + 16])
        sel = eng.decode_rows(ref, [toks[P0 - 1]] + draft).argmax(-1).tolist()
        want = PL.accept(draft, sel, len(hist), len(ids) + N, P0, N)
        assert drafted - prev[1] == len(draft), (P0, draft)
        assert toks[P0:P0 + len(want)] == want and 1 + steps + accepted == P0 + len(want), (P0, draft, sel, want)
        prev = (steps, drafted, accepted)
    ref.close()


def test_sampled_stream_equals_oracle_selection(engines):
    """do_sample: every token is the oracle draw over the logits of the row that produced it (draw index = token index, Philox
    row 0), replayed through b2_decode_rows from the same prefill."""
    eng = engines("bf16")
    emb = rnd(1, PROMPT, CFG2["hidden"], seed=31)
    sp = dict(do_sample=True, temperature=0.7, top_p=0.9, top_k=20, seed=0xACE)
    N = 16
    kv = eng.new_kv(1, MAX_SEQ)
    plain = _plain(eng, kv, emb, N, _b2.make_sampling(**sp))
    z = CFG2["vocab"] - 3
    ids = torch.tensor([z] + plain[:12] + [z], dtype=torch.int64)
    toks, stats = _lookup(eng, kv, emb, ids, 4, N, _b2.make_sampling(**sp), N)
    kv.close()
    # replay: the logits of token t's row are those of the forward over the tokens before it
    ref = eng.new_kv(1, MAX_SEQ)
    raw = eng.prefill(ref, emb, None, _b2.LOGITS_LAST)[0].cpu().numpy()
    for t in range(N):
        want, info = S.sample_row(raw, sp["temperature"], sp["top_k"], sp["top_p"], sp["seed"], t, 0)
        if toks[t] != want:
            slack = 1e-6 * info["total"]
            assert info["lo"][toks[t]] - slack <= info["target"] <= info["hi"][toks[t]] + slack, (t, toks[t], want)
        if t + 1 < N:
            raw = eng.decode_rows(ref, [toks[t]])[0].cpu().numpy()
    ref.close()


# ------------------------------------------------------------------------------------------------ generate()
class _Keywords:
    """KeywordsStoppingCriteria-style (llava/mm_utils.py): stop once the ids end with the keyword ids."""

    def __init__(self, kw):
        self.kw = list(kw)

    def __call__(self, ids, scores):
        return ids.shape[1] >= len(self.kw) and ids[0, -len(self.kw):].tolist() == self.kw


def test_generate_with_and_without_prompt_lookup(monkeypatch):
    """Image and text prompts: ids and streamer output equal to plain decoding's, speculation ran and drafted (the text prompt
    holds every id of the vocabulary, so every pending token has an earlier occurrence), and eos / a keyword criterion stop at the
    same token."""
    cfg = O.CONFIGS["tiny"]
    w = O.make_weights(cfg, seed=0)
    began = []
    real_begin = _b2.Engine.stream_begin_lookup

    def spy(self, kv, logits, sampling, lookup):
        began.append((self, kv, lookup.num_tokens))
        return real_begin(self, kv, logits, sampling, lookup)

    monkeypatch.setattr(_b2.Engine, "stream_begin_lookup", spy)
    outs = {}
    stats = []
    for k in (0, 5):
        model = make_model(cfg, w, max_batch=1, max_seq=1200, b2_prompt_lookup=k)
        input_ids, images = synth_inputs(cfg, 1, 24, seed=4)
        text = torch.cat([torch.tensor([[1]]), torch.randperm(cfg["vocab"], generator=torch.Generator().manual_seed(2))[None]], 1)
        cases = {"image": (images, input_ids), "text": (None, text)}
        for name, (imgs, ids) in cases.items():
            seen = []

            class Streamer:
                def put(self, t):
                    seen.append(t.tolist())

                def end(self):
                    pass

            began.clear()
            out = model.generate(ids, images=imgs, max_new_tokens=24, streamer=Streamer())
            outs[(k, name)] = (out.tolist(), seen)
            assert len(began) == (1 if k else 0)
            if k:
                torch.cuda.synchronize()
                stats.append(began[0][0].lookup_stats(began[0][1]))
        # eos and a keyword criterion stop at the same token as without speculation
        gen = outs[(k, "text")][0][0][text.shape[1]:]
        eos = gen[6]
        cut = gen.index(eos) + 1
        out = model.generate(text, max_new_tokens=24, eos_token_id=eos)
        assert out[0, text.shape[1]:].tolist() == gen[:cut]
        out = model.generate(text, max_new_tokens=24, stopping_criteria=[_Keywords(gen[9:11])])
        assert out[0, text.shape[1]:].tolist()[-2:] == gen[9:11] and out.shape[1] <= text.shape[1] + 11
        outs[(k, "stops")] = out.tolist()
        model.invalidate_engine()
    for name in ("image", "text", "stops"):
        assert outs[(5, name)] == outs[(0, name)], name
    assert all(steps > 0 for steps, _, _ in stats), stats
    assert stats[1][1] > 0, stats  # the text prompt: drafts were proposed
