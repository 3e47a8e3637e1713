"""GPU: logits processors in beam search and beam sampling. b2_op_beam_select_proc against logits_proc_oracle.process over the
device's own log-softmax rows (bit for bit) and the candidate rules of beam_oracle / beam_sampling_ref; the engine's processed
beam search (b2_beam_begin_proc + b2_beam_step_proc: histories carried along the slot copies) against tests/beam_proc_ref.py on
every decode path, bf16 and e4m3 caches and at 7B width; generate() with the opt-ins; state hygiene of a pooled cache, launch
counts, and a concurrent greedy thread."""
import threading

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import beam_proc_ref as BPR  # noqa: E402
import beam_sampling_ref as BSR  # noqa: E402
from helpers import make_engine, make_model  # noqa: E402
from llava import _b2  # noqa: E402
from llava._b2 import beam as BM  # noqa: E402
from oracle import beam_oracle as BO  # noqa: E402
from oracle import llava_oracle as O  # noqa: E402
from oracle import logits_proc_oracle as P  # noqa: E402
from test_beam_gpu import CFG7, _decoder_weights_on_device, _device_logits_fn, _text_logits_fn  # noqa: E402

DEV = "cuda"


@pytest.fixture(scope="module", autouse=True)
def _init():
    _b2.init(0)


_ENG = {}


def _tiny():
    if "tiny" not in _ENG:
        cfg = O.CONFIGS["tiny"]
        w = BO.condition_weights_beam(O.make_weights(cfg, seed=5), cfg, seed=5)
        _ENG["tiny"] = (cfg, w, make_engine(cfg, w, max_batch=16, max_seq=96))
    return _ENG["tiny"]


def _same(a, b):
    """bitwise equality of fp32 arrays, NaN equal to NaN"""
    a, b = np.asarray(a, dtype=np.float32), np.asarray(b, dtype=np.float32)
    return a.shape == b.shape and bool(np.array_equal(a.view(np.uint32), b.view(np.uint32)) or
                                       (np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(a[~np.isnan(a)], b[~np.isnan(b)])))


# ------------------------------------------------------------------------------------------------------------ op level
@pytest.mark.parametrize("V", [1000, 32000])
@pytest.mark.parametrize("mode", ["greedy", "greedy_fan", "sampled"])
def test_op_select_proc_against_the_oracle(V, mode):
    eng = _tiny()[2]
    g = torch.Generator().manual_seed(V + len(mode))
    B, nb = 2, 3
    rows = B if mode != "greedy" else B * nb
    logits = torch.randn(rows, V, generator=g) * 4
    logits[0, 7] = float("nan")                                   # a NaN logit
    logits[rows - 1, : V // 3] = float("-inf")                    # -inf entries
    hist = [torch.randint(0, V, (30,), generator=g) for _ in range(rows)]
    for h in hist:
        h[[3, 11]] = -200                                          # placeholders: never penalised or banned, still matched
        h[20:22] = h[-1:].repeat(2)                                # a repeated tail: the n-gram ban has matches
    eos = [int(hist[0][5]), 1]
    ids = [h.to(DEV) for h in hist]
    procs = [_b2.make_logits_proc(ids[r], 1.3, [2, 3][r % 2], 2, eos) for r in range(rows)]
    procs[1] = None                                                # an unprocessed row beside processed ones
    K = 2 * nb
    nbk, fan, rob = {"greedy": (nb, 1, None), "greedy_fan": (1, nb, None),
                     "sampled": (nb, 1, [b for b in range(B) for _ in range(nb)])}[mode]
    run = torch.randn(B * nbk, generator=g)
    bs = _b2.make_beam_sampling(0.8, 40, 0.9, 3, 1234) if mode == "sampled" else None
    ld = logits.to(DEV)
    rs = torch.empty(B * nbk * fan, V, device=DEV)
    s, t, b = (x.cpu() for x in eng.beam_select_proc(ld, run, nbk, K, procs, rs, None, sampling=bs, step=3, row_of_beam=rob, fan=fan))
    # the device's own unprocessed log-softmax rows (greedy b2_op_beam_select_out over every logits row)
    ls = torch.empty(rows, V, device=DEV)
    eng.beam_select_out(ld, torch.zeros(rows), 1, 2, ls, None)
    ls = ls.cpu().numpy()
    proc_rows = [P.process(ls[r], hist[r].tolist(), 30, 1.3, [2, 3][r % 2], 2, eos) if procs[r] is not None else ls[r]
                 for r in range(rows)]
    beam_row = rob if rob is not None else (list(range(rows)) if fan == 1 else [r for r in range(rows) for _ in range(fan)])
    if bs is None:
        want_rows = np.stack([proc_rows[r] for r in beam_row])
        sel = torch.from_numpy(np.stack([proc_rows[r] for r in (beam_row if fan == 1 else range(rows))])).view(B, -1)
        # the device ranks NaN below -inf; the K best of these rows are finite
        ws, wi = BO.select_candidates(torch.nan_to_num(sel, nan=float("-inf")) + run.view(B, nbk).repeat_interleave(V, 1), K)
        assert torch.equal(s, ws) and torch.equal((b * V + t).long(), wi), (s, ws)
    else:
        w = [(proc_rows[r] / np.float32(0.8)).astype(np.float32) for r in beam_row]
        want_rows = np.stack([np.where(BSR.kept_mask(x, 40, 0.9, 3) | np.isnan(x), x, -np.inf).astype(np.float32) for x in w])
        acc = (want_rows.reshape(B, nb, V) + run.numpy().reshape(B, nb, 1).astype(np.float32)).astype(np.float32).reshape(B, nb * V)
        ws, wi, _, _ = BSR.philox_select(acc, 1234, 3, nb, K)
        assert _same(s.numpy(), ws) and np.array_equal((b * V + t).numpy(), wi), (s, ws)
    assert _same(rs.cpu().numpy(), want_rows)


def test_op_select_proc_with_every_processor_off_is_select_out():
    eng = _tiny()[2]
    g = torch.Generator().manual_seed(2)
    V, B, nb = 1000, 2, 3
    ld = (torch.randn(B * nb, V, generator=g) * 3).to(DEV)
    run = torch.randn(B * nb, generator=g)
    ids = torch.arange(10, device=DEV)
    off = [_b2.LogitsProc(1.0, 0, 5, 0) for _ in range(B * nb)]   # min_generated without eos: off, as HF
    for p in off:
        p.prompt_ids, p.prompt_len = ids.data_ptr(), 10
    for bs in (None, _b2.make_beam_sampling(0.7, 50, 1.0, 2, 9)):
        r1, r2 = torch.empty(B * nb, V, device=DEV), torch.empty(B * nb, V, device=DEV)
        a = [x.cpu() for x in eng.beam_select_proc(ld, run, nb, 2 * nb, off, r1, None, sampling=bs, step=1)]
        c = [x.cpu() for x in eng.beam_select_out(ld, run, nb, 2 * nb, r2, None, sampling=bs, step=1)]
        assert all(torch.equal(x, y) for x, y in zip(a, c)) and torch.equal(r1, r2)


def test_op_select_proc_rejects_bad_arguments():
    eng = _tiny()[2]
    ld = torch.zeros(4, 100, device=DEV)
    ids = torch.arange(5, device=DEV)
    for kw in (dict(repetition_penalty=0.0), dict(no_repeat_ngram_size=-1)):
        p = _b2.LogitsProc(kw.get("repetition_penalty", 1.0), kw.get("no_repeat_ngram_size", 0), 0, 0)
        p.prompt_ids, p.prompt_len = ids.data_ptr(), 5
        with pytest.raises(ValueError):
            eng.beam_select_proc(ld, torch.zeros(4), 2, 4, [p] * 4)


# ------------------------------------------------------------------------------------------------- engine beam search
def engine_beam_proc(eng, kv, prompt, nb, max_new, proc, eos=None, nrs=1, sampling=None, counts=None):
    """generate()'s processed beam loop over the engine; `counts` collects (copies, launches) of every step."""
    B, Lt = prompt.shape
    s = BM.BeamSearch(prompt, nb, max_new, eos, 1.0, False, nrs)
    emb = eng.splice(prompt.to(torch.int32).reshape(-1).to(DEV), None, B, Lt)
    kv.reset()
    logits = eng.prefill(kv, emb, None, _b2.LOGITS_LAST)
    pd = prompt.to(DEV)
    procs = None if proc is None else [_b2.make_logits_proc(pd[b], proc.get("repetition_penalty", 1.0), proc.get("no_repeat_ngram_size", 0),
                                                              proc.get("min_new_tokens", 0), eos or ()) for b in range(B)]
    if procs is None:
        cand = [t.cpu() for t in (eng.beam_topk(logits, torch.zeros(B), 1, s.K) if sampling is None else
                                  eng.beam_sample(logits, s.running_scores.reshape(-1), nb, s.K, sampling, 0,
                                                  row_of_beam=[b for b in range(B) for _ in range(nb)]))]
    else:
        cand = [t.cpu() for t in (eng.beam_select_proc(logits, torch.zeros(B), 1, s.K, procs, fan=nb) if sampling is None else
                                  eng.beam_select_proc(logits, s.running_scores.reshape(-1), nb, s.K, procs, sampling=sampling, step=0,
                                                       row_of_beam=[b for b in range(B) for _ in range(nb)]))]
        eng.beam_begin_proc(kv, procs)
    if sampling is not None:
        cand[2].zero_()
    step_fn = eng.beam_step if procs is None else eng.beam_step_proc
    plan, rb, step = BM.SlotPlanner(B, nb), 0, 0
    while not s.step(*cand):
        step += 1
        copies = plan.plan(s.parents)
        before = _b2.launch_count()
        cand = step_fn(kv, copies, rb, s.next_tokens().tolist(), plan.flat(), s.running_scores.reshape(-1).tolist(), nb, s.K,
                       sampling=sampling, step=step)
        if counts is not None:
            counts.append((len(copies), _b2.launch_count() - before))
        rb = Lt
    return s.output()


PROC = dict(repetition_penalty=1.2, no_repeat_ngram_size=2)


@pytest.mark.parametrize("B,nb,kv_dtype", [(1, 2, "bf16"), (1, 4, "bf16"), (3, 4, "bf16"), (2, 4, "e4m3"), (1, 3, "e4m3")])
def test_engine_beam_search_with_processors_equals_the_reference(B, nb, kv_dtype):
    """condition_weights_beam weights: continuations repeat, so forked beams ban tokens their parents generated. Decode paths on a
    bf16 cache: 2 rows the megakernel, 4 rows the GEMV graph, 12 rows the stream-K GEMM; an e4m3 cache the multi-kernel step."""
    cfg, w, eng = _tiny()
    kv = eng.new_kv(16, 96, dtype=kv_dtype)
    fn = _text_logits_fn(w, cfg)
    prompt = torch.randint(3, cfg["vocab"], (B, 9), generator=torch.Generator().manual_seed(B * 10 + nb))
    # these weights continue mostly from the token fed: the prompt starts with the 3rd and 4th tokens its plain best beam would
    # generate, so that bigram is banned and the search has to leave the plain path
    best = BO.beam_search(fn, prompt, nb, 12, None)[0][:, 9:]
    prompt[:, :2] = best[:, 2:4]
    changed = 0
    for eos, nrs in [(None, 1), ([int(prompt[0, 3])], nb)]:
        kw = dict(PROC, min_new_tokens=3) if eos else PROC
        got = engine_beam_proc(eng, kv, prompt, nb, 12, kw, eos, nrs)
        want, want_scores, margins = BPR.beam_search(fn, prompt, nb, 12, eos, None, 1.0, False, nrs, return_margins=True, **kw)
        plain = BO.beam_search(fn, prompt, nb, 12, eos, None, 1.0, False, nrs)[0]
        print(f"B={B} nb={nb} {kv_dtype} eos={eos}: min margin {min(margins):.3e}, processors change the ids {not torch.equal(want, plain)}")
        assert torch.equal(got[0][::nrs], want[::nrs]), (got[0], want)   # each sample's best hypothesis, strictly
        # the returned hypotheses of a sample as a set: finished hypotheses whose normalised scores are closer than the cache's
        # rounding may swap places (the margins above cover the candidate and running selections, not that order)
        for b in range(B):
            g_rows, w_rows = got[0][b * nrs:(b + 1) * nrs], want[b * nrs:(b + 1) * nrs]
            assert sorted(map(tuple, g_rows.tolist())) == sorted(map(tuple, w_rows.tolist())), (g_rows, w_rows)
            for i, row in enumerate(g_rows):
                j = next(j for j, r in enumerate(w_rows) if torch.equal(r, row))
                # an e4m3 cache's logit error, which the repetition penalty scales by p on penalised tokens, is about twice bf16's
                torch.testing.assert_close(got[1][b * nrs + i], want_scores[b * nrs + j], atol=0.1 if kv_dtype == "e4m3" else 0.05,
                                           rtol=0.01)
        changed += not torch.equal(want, plain)
    assert changed == 2
    kv.close()


def test_engine_beam_search_with_processors_at_7b_width():
    cfg = CFG7
    w = BO.condition_weights_beam(_decoder_weights_on_device(cfg, 3), cfg, seed=3)
    eng = make_engine(cfg, w, max_batch=8, max_seq=64, max_images=1)
    kv = eng.new_kv(8, 64)
    fn = _device_logits_fn(w, cfg)
    p = torch.randint(3, cfg["vocab"], (2, 9), generator=torch.Generator().manual_seed(4))
    got = engine_beam_proc(eng, kv, p, 4, 8, PROC)
    want, _, margins = BPR.beam_search(fn, p, 4, 8, None, return_margins=True, **PROC)
    print(f"7B width, 2 layers: min margin {min(margins):.3e}")
    assert torch.equal(got[0], want), (got[0], want)
    kv.close()
    eng.close()


@pytest.mark.parametrize("B,nb,eos", [(1, 3, None), (2, 4, [7])])
def test_engine_beam_sampling_with_processors_equals_the_philox_reference(B, nb, eos):
    cfg, w, eng = _tiny()
    kv = eng.new_kv(16, 96)
    fn = _text_logits_fn(w, cfg)
    p = torch.randint(3, cfg["vocab"], (B, 9), generator=torch.Generator().manual_seed(nb))
    kw = dict(PROC, min_new_tokens=2) if eos else PROC
    mk = BSR.min_keep_of(eos)
    bs = _b2.make_beam_sampling(0.9, 30, 0.95, mk, 77)
    got = engine_beam_proc(eng, kv, p, nb, 10, kw, eos, nb, sampling=bs)
    want, _, margins = BPR.beam_search(fn, p, nb, 10, eos, None, 1.0, False, nb, return_margins=True, do_sample=True,
                                       temperature=0.9, top_k=30, top_p=0.95, sampler="philox", seed=77, **kw)
    print(f"beam sampling B={B} nb={nb}: min key margin {min(margins):.3e}")
    assert torch.equal(got[0], want), (got[0], want)
    kv.close()


def test_launch_counts_and_state_hygiene():
    """A processors-off step launches what b2_beam_step_out launches; a processed step one kernel more (the tokens to the device)
    and one more again when it copies slots (the histories). A processed search leaves nothing behind: plain beam search and
    plain streaming on the same cache afterwards give what they gave before, and b2_beam_step_proc is disarmed."""
    cfg, w, eng = _tiny()
    kv = eng.new_kv(16, 96)
    p = torch.randint(3, cfg["vocab"], (2, 9), generator=torch.Generator().manual_seed(21))
    engine_beam_proc(eng, kv, p, 4, 6, None)                                   # warm every shape
    engine_beam_proc(eng, kv, p, 4, 6, PROC)
    plain_counts, proc_counts = [], []
    plain = engine_beam_proc(eng, kv, p, 4, 12, None, counts=plain_counts)
    engine_beam_proc(eng, kv, p, 4, 12, PROC, counts=proc_counts)
    base = {c > 0: n for c, n in plain_counts}
    print(f"launches per step: plain {plain_counts}, processed {proc_counts}")
    assert len(set((c > 0, n) for c, n in plain_counts)) == len(base)          # one count per kind of step
    for c, n in proc_counts:
        if (c > 0) in base:
            assert n == base[c > 0] + 1 + (1 if c > 0 else 0), (c, n, base)
    again = engine_beam_proc(eng, kv, p, 4, 12, None)
    assert torch.equal(again[0], plain[0]) and torch.equal(again[1], plain[1])
    with pytest.raises(ValueError):                                           # a plain step disarmed the processing
        eng.beam_step_proc(kv, [], 9, [1] * 8, list(range(8)), [0.0] * 8, 4, 8)
    # streaming after a processed search equals streaming on a fresh cache
    emb = eng.splice(p.to(torch.int32).reshape(-1).to(DEV), None, 2, 9)
    outs = []
    fresh = eng.new_kv(16, 96)
    for k in (kv, fresh):
        engine_beam_proc(eng, kv, p, 4, 6, PROC)
        k.reset()
        logits = eng.prefill(k, emb, None, _b2.LOGITS_LAST)
        eng.stream_begin(k, logits, _b2.make_sampling())
        eng.stream_enqueue(k, 7)
        outs.append([eng.stream_wait(k, i, 2) for i in range(8)])
    assert outs[0] == outs[1]
    kv.close()
    fresh.close()


# ------------------------------------------------------------------------------------------------------------ generate()
def _model(**extra):
    cfg, w, _ = _tiny()
    return cfg, w, make_model(cfg, w, max_batch=8, max_seq=96, b2_beam_search=4, b2_logits_processors=True,
                              b2_beam_logits_processors=True, **extra)


def test_generate_with_the_opt_ins():
    cfg, w, model = _model(b2_beam_sample=True)
    fn = _text_logits_fn({k: v.float() for k, v in w.items()}, cfg)
    p = torch.randint(3, cfg["vocab"], (2, 9), generator=torch.Generator().manual_seed(8))
    pd = p.to(DEV)
    out = model.generate(pd, num_beams=3, no_repeat_ngram_size=3, max_new_tokens=10, eos_token_id=[]).cpu()  # the eval call
    assert torch.equal(out, BPR.beam_search(fn, p, 3, 10, [], no_repeat_ngram_size=3)[0])
    kw = dict(num_beams=3, max_new_tokens=10, eos_token_id=[int(out[0, 12])], repetition_penalty=1.2, no_repeat_ngram_size=2,
              min_new_tokens=4, num_return_sequences=3)
    r = model.generate(pd, output_scores=True, output_logits=True, return_dict_in_generate=True, **kw)
    want = BPR.beam_search(fn, p, 3, 10, kw["eos_token_id"], None, 1.0, False, 3, repetition_penalty=1.2, no_repeat_ngram_size=2,
                           min_new_tokens=4)
    assert torch.equal(r.sequences.cpu(), want[0])
    # step 0: every beam's score row is its sample's prefill row processed over the prompt, bit for bit
    ls = torch.empty(2, cfg["vocab"], device=DEV)
    model._engine.beam_select_out(r.logits[0][::3].contiguous(), torch.zeros(2), 1, 2, ls, None)
    for i in range(6):
        want0 = P.process(ls[i // 3].cpu().numpy(), p[i // 3].tolist(), 9, 1.2, 2, 4, tuple(kw["eos_token_id"]))
        assert _same(r.scores[0][i].cpu().numpy(), want0)
    # HF's identity: the generated tokens' transition scores, summed over the length, are sequences_scores
    ts = model.compute_transition_scores(r.sequences, r.scores, r.beam_indices)
    length = (r.beam_indices >= 0).sum(dim=1)
    torch.testing.assert_close(ts.sum(dim=1).cpu() / length.float().cpu(), r.sequences_scores.cpu(), atol=1e-4, rtol=1e-5)
    # beam sampling with processors runs, and repeats under the same torch seed
    torch.manual_seed(3)
    a = model.generate(pd, num_beams=3, do_sample=True, temperature=0.7, max_new_tokens=6, no_repeat_ngram_size=2)
    torch.manual_seed(3)
    b = model.generate(pd, num_beams=3, do_sample=True, temperature=0.7, max_new_tokens=6, no_repeat_ngram_size=2)
    assert torch.equal(a, b)
    model.invalidate_engine()


def test_concurrent_processed_beam_and_greedy_threads_equal_serial():
    cfg, w, model = _model()
    p = [torch.randint(3, cfg["vocab"], (1, 9 + i), generator=torch.Generator().manual_seed(40 + i)).to(DEV) for i in range(3)]
    calls = [dict(num_beams=4, no_repeat_ngram_size=2, repetition_penalty=1.2), dict(num_beams=3), dict()]
    run = lambda i: model.generate(p[i], max_new_tokens=16, eos_token_id=[], **calls[i]).cpu()
    serial = [run(i) for i in range(3)]
    res, errs = [None] * 3, []

    def work(i):
        try:
            res[i] = run(i)
        except Exception as e:  # pragma: no cover
            errs.append(e)

    th = [threading.Thread(target=work, args=(i,)) for i in range(3)]
    [t.start() for t in th]
    [t.join() for t in th]
    assert not errs, errs
    for i in range(3):
        assert torch.equal(res[i], serial[i]), i
    model.invalidate_engine()
