"""GPU: history-aware logits processing (repetition_penalty, no_repeat_ngram_size, min_length / min_new_tokens) in the token
selection kernel (csrc/sampling.cu) against oracle/logits_proc_oracle.py.

- b2_op_sample_ex: processed logits bit-equal to the oracle, greedy tokens equal, sampled tokens in the oracle's CDF interval.
- Teacher-forced streams on every decode path: the device's token at every step equals the oracle's selection from that step's
  raw logits, which a second cache replays through decode_step (the step logits are bit-equal between the two).
- Properties and generate() with config.b2_logits_processors: image and text prompts, the continuous batcher, the prefix cache,
  and the off values, which must change neither tokens nor launch counts."""
import os
import subprocess
import sys
import threading

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from helpers import make_engine, make_model, synth_inputs  # noqa: E402
from llava import _b2  # noqa: E402
from oracle import llava_oracle as O  # noqa: E402
from oracle import logits_proc_oracle as P  # noqa: E402
from oracle import sampling_oracle as S  # noqa: E402
from test_nf4_gpu import CFG2, dev_weights, rnd  # noqa: E402

DEV = "cuda"
V7 = CFG2["vocab"]
MAX_SEQ, PROMPT, STEPS = 128, 40, 24
SAMPLED = dict(do_sample=True, temperature=0.8, top_p=0.9, top_k=50, seed=0x5EED)


def _sampling(kind):
    return _b2.make_sampling(**SAMPLED) if kind == "sampled" else _b2.make_sampling()


def _check_token(tok, processed, kind, index, row):
    """greedy: the oracle's argmax exactly. sampled: the token whose CDF interval holds the Philox target (GPU expf and numpy
    exp may differ in the last ulp: a slack of 1e-6 of the total mass on the interval ends)."""
    if kind == "greedy":
        assert tok == S.greedy(processed), (tok, S.greedy(processed), index, row)
        return
    s = SAMPLED
    want, info = S.sample_row(processed, s["temperature"], s["top_k"], s["top_p"], s["seed"], index, row)
    if tok != want:
        slack = 1e-6 * info["total"]
        assert info["lo"][tok] - slack <= info["target"] <= info["hi"][tok] + slack, (tok, want, index, row)
    assert np.isfinite(processed[tok]), (tok, index, row)  # a banned id is never drawn


def _histories(B, L, logits0, seed):
    """Prompt rows (int64 [B, L]) that hold the rows' top prefill tokens, repeats and (row 0) an image placeholder, so that
    every processor changes what is chosen."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, V7, (B, L), generator=g)
    top = logits0.float().topk(6, dim=-1).indices.cpu()
    for b in range(B):
        ids[b, L - 8:L - 2] = top[b]
        ids[b, 3:9] = top[b]  # an n-gram of the prompt that recurs: its continuation is banned
    ids[0, 1] = O.IMAGE_TOKEN_INDEX
    return ids


def _params(logits0):
    eos = logits0[0].float().topk(2).indices.cpu().tolist()
    return dict(repetition_penalty=1.3, no_repeat_ngram_size=3, min_generated=4, eos_ids=eos)


def _procs(ids_dev, prm):
    return [_b2.make_logits_proc(ids_dev[b], **prm) for b in range(ids_dev.shape[0])]


def _oracle(raw, hist, plen, prm):
    return P.process(raw, hist, plen, prm["repetition_penalty"], prm["no_repeat_ngram_size"], prm["min_generated"], prm["eos_ids"])


# ---------------------------------------------------------------------------------------------------- the selection op
@pytest.fixture(scope="module")
def tiny_engine():
    cfg = O.CONFIGS["tiny"]
    eng = make_engine(cfg, O.make_weights(cfg, seed=0), max_batch=16, max_seq=160, max_images=4)
    yield eng
    eng.close()


@pytest.mark.parametrize("B", [1, 4, 12])
def test_op_sample_ex_equals_oracle(tiny_engine, B):
    eng = tiny_engine
    g = torch.Generator().manual_seed(B)
    logits = torch.randn(B, V7, generator=g) * 3
    ids = _histories(B, 30, logits, seed=B)
    ids[:, -1] = ids[:, 5]  # the tail ngram (ids[-2], ids[-1]) occurs at 4..5 for n = 2
    ids_dev = ids.to(DEV)
    cases = [dict(repetition_penalty=1.2, no_repeat_ngram_size=0, min_generated=0, eos_ids=()),
             dict(repetition_penalty=0.7, no_repeat_ngram_size=2, min_generated=1, eos_ids=(5, 77)),
             dict(repetition_penalty=1.0, no_repeat_ngram_size=1, min_generated=0, eos_ids=()),
             _params(logits)]
    for prm in cases:
        procs = _procs(ids_dev, prm)
        for kind in ("greedy", "sampled"):
            for index in (0, 5):
                tok, processed = eng.sample(logits.to(DEV), _sampling(kind), index=index, procs=procs, want_processed=True)
                tok, processed = tok.cpu().tolist(), processed.cpu().numpy()
                for b in range(B):
                    want = _oracle(logits[b].numpy(), ids[b].tolist(), 30, prm)
                    assert np.array_equal(processed[b].view(np.uint32), want.view(np.uint32)), (prm, b)
                    _check_token(tok[b], want, kind, index, b)
    # rows with every processor off select from their raw logits; bad arguments are refused
    procs = _procs(ids_dev, cases[0])
    procs[0] = None
    tok, processed = eng.sample(logits.to(DEV), _b2.make_sampling(), procs=procs, want_processed=True)
    assert torch.equal(processed[0].cpu(), logits[0]) and tok[0].item() == S.greedy(logits[0].numpy())
    bad = _b2.make_logits_proc(ids_dev[0], repetition_penalty=1.2)
    bad.repetition_penalty = -1.0
    with pytest.raises(ValueError):
        eng.sample(logits.to(DEV), _b2.make_sampling(), procs=[bad] + [None] * (B - 1))


# ------------------------------------------------------------------------------------------------ teacher-forced streams
# id: (weights, kv dtype, B): megakernel, the GEMV graph on an e4m3 cache (which takes the multi-kernel step at every batch) and
# on a bf16 cache, stream-K, NF4. A bf16 cache at batch 4 takes the megakernel unless B2_DECODE_MEGA=0, which is read once per
# process, so "gemv-bf16-b4" runs in a process of its own (test_gemv_graph_on_a_bf16_cache)
PATHS = {"mega-b1": ("bf16", "bf16", 1), "gemv-e4m3kv-b4": ("bf16", "e4m3", 4), "gemv-bf16-b4": ("bf16", "bf16", 4),
         "streamk-b12": ("bf16", "bf16", 12), "nf4-b1": ("nf4", "bf16", 1)}
GEMV_STEP_LAUNCHES = 1 + CFG2["layers"] * 5 + 1 + 1  # embed, 5 per layer, lm_head, sample_publish


@pytest.fixture(scope="module")
def engines():
    built = {}

    def get(fmt):
        if fmt not in built:
            eng = make_engine(CFG2, dev_weights(CFG2, seed=3), max_batch=16, max_seq=MAX_SEQ, max_images=1)
            if fmt == "nf4":
                eng.enable_nf4()
            built[fmt] = eng
        return built[fmt]

    yield get
    for eng in built.values():
        eng.close()


def _stream(eng, kv, logits, B, sampling, procs, n):
    eng.stream_begin(kv, logits, sampling, procs)
    eng.stream_enqueue(kv, n - 1)
    return [eng.stream_wait(kv, t, B) for t in range(n)]


@pytest.mark.parametrize("kind", ["greedy", "sampled"])
@pytest.mark.parametrize("path", list(PATHS))
def test_teacher_forced_stream_equals_oracle(engines, path, kind):
    fmt, kv_dtype, B = PATHS[path]
    if path == "gemv-bf16-b4" and os.environ.get("B2_DECODE_MEGA") != "0":
        pytest.skip("runs in a process without the megakernel: test_gemv_graph_on_a_bf16_cache")
    eng = engines(fmt)
    emb = rnd(B, PROMPT, CFG2["hidden"], seed=80 + B)
    kv = eng.new_kv(B, MAX_SEQ, dtype=kv_dtype)
    logits0 = eng.prefill(kv, emb, None, _b2.LOGITS_LAST).clone()
    plain = _stream(eng, kv, logits0, B, _sampling(kind), None, 6)  # a decode graph captured before the state exists
    kv.reset()
    eng.prefill(kv, emb, None, _b2.LOGITS_LAST)
    ids = _histories(B, PROMPT, logits0, seed=B)
    ids_dev = ids.to(DEV)
    prm = _params(logits0)
    toks = np.asarray(_stream(eng, kv, logits0, B, _sampling(kind), _procs(ids_dev, prm), STEPS))  # [STEPS, B]
    kv.close()
    assert toks[0].tolist() != plain[0] or kind == "sampled"  # the prompt history changed token 0
    # replay: the raw logits of every step from a second cache fed the same tokens
    ref = eng.new_kv(B, MAX_SEQ, dtype=kv_dtype)
    raw = eng.prefill(ref, emb, None, _b2.LOGITS_LAST).cpu().numpy()
    for t in range(STEPS):
        for b in range(B):
            hist = ids[b].tolist() + toks[:t, b].tolist()
            _check_token(int(toks[t, b]), _oracle(raw[b], hist, PROMPT, prm), kind, t, b)
        if t + 1 < STEPS:
            before = _b2.launch_count()
            raw = eng.decode_step(ref, torch.tensor(toks[t], dtype=torch.int32, device=DEV)).cpu().numpy()
            if path.startswith("gemv") and t == 2:  # the step really is the GEMV graph, not the megakernel
                assert _b2.launch_count() - before == GEMV_STEP_LAUNCHES
    ref.close()


def test_gemv_graph_on_a_bf16_cache(repo_root):
    """The teacher-forced cases of the bf16 GEMV graph at batch 4, in a process started with B2_DECODE_MEGA=0."""
    env = dict(os.environ, B2_DECODE_MEGA="0")
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", os.path.abspath(__file__),
                        "-k", "test_teacher_forced_stream_equals_oracle and gemv-bf16-b4"],
                       cwd=repo_root, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "2 passed" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]


def test_off_values_keep_tokens_and_launch_counts(engines):
    """Every processor at its off value: the plain path, including the megakernel's one launch per greedy token."""
    eng = engines("bf16")
    emb = rnd(1, PROMPT, CFG2["hidden"], seed=91)
    kv = eng.new_kv(1, MAX_SEQ)
    ids_dev = torch.arange(PROMPT, device=DEV, dtype=torch.int64)
    off = _b2.make_logits_proc(ids_dev, repetition_penalty=1.0, no_repeat_ngram_size=0, min_generated=3, eos_ids=())
    assert off is None
    runs = []
    for procs in (None, [off], [_b2.make_logits_proc(ids_dev, no_repeat_ngram_size=2)], None):
        logits = eng.prefill(kv, emb, None, _b2.LOGITS_LAST)
        _stream(eng, kv, logits, 1, None, procs, 3)  # warm
        kv.reset()
        logits = eng.prefill(kv, emb, None, _b2.LOGITS_LAST)
        torch.cuda.synchronize()
        before = _b2.launch_count()
        toks = _stream(eng, kv, logits, 1, None, procs, 17)
        runs.append((toks, _b2.launch_count() - before))
        kv.reset()
    kv.close()
    assert runs[0] == runs[1] == runs[3]
    assert runs[0][1] == 2 + 16          # selection-state upload and token 0, then one megakernel launch per token
    assert runs[2][1] == 3 + 2 * 16      # ... plus the history seeding, and sample_publish after every megakernel launch


def test_generate_off_values_keep_tokens_and_launch_counts():
    """generate() with the opt-in set and every processor at its off value: the same ids and the same kernel launches as
    without the opt-in (batch 1 on a bf16 cache: the megakernel, one launch per greedy token)."""
    cfg, model = _tiny_model()
    ids, images = synth_inputs(cfg, B=1, Lt=12, seed=21)
    ids, images = ids.to(DEV), images.to(DEV)
    off = dict(repetition_penalty=1.0, no_repeat_ngram_size=0, min_new_tokens=0, min_length=0)

    def run(opt_in, kw, n):
        model.config.b2_logits_processors = opt_in
        torch.cuda.synchronize()
        before = _b2.launch_count()
        out = model.generate(ids, images=images, max_new_tokens=n, eos_token_id=[], **kw)
        torch.cuda.synchronize()
        return out.cpu(), _b2.launch_count() - before

    run(False, {}, 16)  # warm: caches, function attributes
    plain, plain_short = run(False, {}, 16), run(False, {}, 8)
    assert plain[1] - plain_short[1] == 8  # one megakernel launch per further greedy token
    for _ in range(2):
        got = run(True, off, 16)
        assert torch.equal(got[0], plain[0]) and got[1] == plain[1], (got[1], plain[1])
    with_proc = run(True, dict(no_repeat_ngram_size=2), 16)
    assert with_proc[1] > plain[1]  # processors on: a selection launch follows each megakernel launch
    model.invalidate_engine()


# ----------------------------------------------------------------------------------------------------------- properties
def _tiny_model(**extra):
    cfg = O.CONFIGS["tiny"]
    return cfg, make_model(cfg, O.make_weights(cfg, seed=0), max_batch=2, max_seq=160, b2_logits_processors=True, **extra)


def test_no_repeated_bigram_and_min_new_tokens():
    cfg, model = _tiny_model()
    ids = torch.randperm(cfg["vocab"] - 3, generator=torch.Generator().manual_seed(2))[:10].add(3)[None].to(DEV)
    out = model.generate(ids, max_new_tokens=64, no_repeat_ngram_size=2, eos_token_id=[])[0].tolist()
    assert len(out) == 10 + 64
    bigrams = list(zip(out, out[1:]))
    assert len(bigrams) == len(set(bigrams))
    g0 = int(model.generate(ids, max_new_tokens=1, eos_token_id=[])[0, -1])
    out = model.generate(ids, max_new_tokens=12, min_new_tokens=5, eos_token_id=[g0])[0, 10:].tolist()
    assert g0 not in out[:5] and len(out) >= 5
    model.invalidate_engine()


# ------------------------------------------------------------------------------------------------------------ generate()
def _teacher_forced(model, prompt_dev, images, out, prm, eos):
    """Every generated token of `out` (up to its row's first eos) equals the oracle's greedy selection from raw logits replayed
    on a fresh cache of the model's engine."""
    engine = model._ensure_engine()
    B, Lt = prompt_dev.shape
    embeds, lens, _ = model._prompt_embeds(engine, prompt_dev, None, images, False)
    prompt = prompt_dev.cpu()
    kv = engine.new_kv(B, 160)
    raw = engine.prefill(kv, embeds, lens, _b2.LOGITS_LAST).cpu().numpy()
    new = out[:, Lt:].cpu()
    mg = P.min_generated(prm.get("min_new_tokens", 0), prm.get("min_length", 0), Lt)
    done = [False] * B
    for t in range(new.shape[1]):
        for b in range(B):
            if done[b]:
                continue
            hist = prompt[b].tolist() + new[b, :t].tolist()
            want = P.process(raw[b], hist, Lt, prm.get("repetition_penalty", 1.0), prm.get("no_repeat_ngram_size", 0), mg, eos)
            assert int(new[b, t]) == S.greedy(want), (b, t)
            done[b] = int(new[b, t]) in eos
        if t + 1 < new.shape[1]:
            raw = engine.decode_step(kv, new[:, t].to(torch.int32).to(DEV)).cpu().numpy()
    kv.close()


PRM = dict(repetition_penalty=1.3, no_repeat_ngram_size=3, min_new_tokens=4)


@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("image", [True, False])
def test_generate_equals_teacher_forced_oracle(B, image):
    cfg, model = _tiny_model()
    ids, images = synth_inputs(cfg, B=B, Lt=12, seed=30 + B)
    if not image:
        images = None
        ids[:, 5] = 7
    ids, images = ids.to(DEV), (images.to(DEV) if image else None)
    eos = [int(model.generate(ids, images=images, max_new_tokens=1, eos_token_id=[])[0, -1])]
    out = model.generate(ids, images=images, max_new_tokens=24, eos_token_id=eos, **PRM)
    _teacher_forced(model, ids, images, out, PRM, eos)
    model.invalidate_engine()


def test_continuous_batcher_and_prefix_cache_equal_the_pool_path():
    """Two threads with different settings through config.b2_continuous_batching = 2 (a slot retired and refilled), and a
    second turn through config.b2_prefix_cache: tokens equal the pool path, which equals the teacher-forced oracle."""
    cfg = O.CONFIGS["tiny"]
    wc = O.condition_weights(O.make_weights(cfg, seed=0), cfg, seed=0)
    solo = make_model(cfg, wc, max_batch=1, max_seq=160, b2_logits_processors=True)
    batched = make_model(cfg, wc, max_batch=2, max_seq=160, b2_logits_processors=True, b2_continuous_batching=2)
    jobs = []
    settings = [dict(repetition_penalty=1.5, no_repeat_ngram_size=2), dict(no_repeat_ngram_size=1), dict(min_new_tokens=6)]
    for i, s in enumerate(settings):
        ids, images = synth_inputs(cfg, B=1, Lt=9 + 3 * i, seed=50 + i)
        jobs.append(dict(ids=ids.to(DEV), images=images.to(DEV), kw=dict(s, max_new_tokens=14 + 4 * i, eos_token_id=[])))
    jobs[2]["kw"]["eos_token_id"] = [int(solo.generate(jobs[2]["ids"], images=jobs[2]["images"], max_new_tokens=1)[0, -1])]
    want = [solo.generate(j["ids"], images=j["images"], **j["kw"]) for j in jobs]
    for j, w in zip(jobs, want):
        _teacher_forced(solo, j["ids"], j["images"], w, j["kw"], j["kw"]["eos_token_id"])
    got, errors = [None] * 3, []

    def work(order):
        try:
            for i in order:
                got[i] = batched.generate(jobs[i]["ids"], images=jobs[i]["images"], **jobs[i]["kw"])
        except Exception as e:  # pragma: no cover
            errors.append(e)

    threads = [threading.Thread(target=work, args=(o,)) for o in ([0, 2], [1])]
    [t.start() for t in threads]
    [t.join() for t in threads]
    assert not errors, errors
    for i in range(3):
        assert torch.equal(got[i].cpu(), want[i].cpu()), i
    assert batched._batcher.stats["admitted"] == 3
    batched.invalidate_engine()

    # prefix cache: a second turn that extends the first one's prompt and answer reuses its rows
    prefix = make_model(cfg, wc, max_batch=1, max_seq=160, b2_logits_processors=True, b2_prefix_cache=True)
    text = torch.randint(3, cfg["vocab"], (1, 12), generator=torch.Generator().manual_seed(7)).to(DEV)
    kw = dict(repetition_penalty=1.5, no_repeat_ngram_size=2, max_new_tokens=12, eos_token_id=[])
    first = prefix.generate(text, **kw)
    turn2 = torch.cat([first, text[:, :5]], dim=1)
    second = prefix.generate(turn2, **kw)
    assert prefix._pool.reused_positions > 0
    assert torch.equal(second.cpu(), solo.generate(turn2, **kw).cpu())
    _teacher_forced(solo, turn2, None, second, kw, [])
    prefix.invalidate_engine()
    solo.invalidate_engine()
