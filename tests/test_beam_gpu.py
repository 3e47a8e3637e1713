"""GPU: beam search. b2_op_beam_topk against a float64 restatement, b2_kv_copy_slots on bf16 and e4m3 caches at 7B layer shapes,
the engine's beam search (b2_beam_step + llava/_b2/beam.py) against oracle/beam_oracle.py on every decode path, score
self-consistency against a fresh prefill, and generate(num_beams > 1)."""
import threading

import pytest
import torch

pytestmark = pytest.mark.gpu

from helpers import make_engine, make_model, synth_inputs  # noqa: E402
from llava import _b2  # noqa: E402
from llava._b2 import beam as BM  # noqa: E402
from oracle import beam_oracle as BO  # noqa: E402
from oracle import llava_oracle as O  # noqa: E402
from test_dropin_cpu import _KeywordStop, _Tok  # noqa: E402  (restated reference KeywordsStoppingCriteria, pinned to tests/golden)

DEV = "cuda"


@pytest.fixture(scope="module", autouse=True)
def _init():
    _b2.init(0)


# ------------------------------------------------------------------------------------------------------------- beam_topk
@pytest.mark.parametrize("V", [32000, 1000, 40])
@pytest.mark.parametrize("nb", [1, 2, 4, 8])
@pytest.mark.parametrize("kmul", [2, 3])
def test_beam_topk_against_float64(V, nb, kmul):
    eng = _tiny_engine()
    B, K = 3, kmul * nb
    g = torch.Generator().manual_seed(V + nb * 7 + kmul)
    logits = torch.randn(B * nb, V, generator=g) * 3
    logits[0, : V // 4] = float("-inf")                            # a row with -inf entries
    logits[(B - 1) * nb, 5:9] = logits[(B - 1) * nb, 4]             # exact ties inside a row
    if nb > 1:
        logits[1] = logits[0]                                       # two beams with identical rows
    scores = torch.randn(B * nb, generator=g)
    scores.view(B, nb)[:, 1:] = -1e9                                # running scores of -1e9 (HF's initial beams)
    s, t, b = (x.cpu() for x in eng.beam_topk(logits.to(DEV), scores, nb, K))
    ref = (torch.log_softmax(logits.double(), -1) + scores.double()[:, None]).view(B, nb * V)
    rs, ri = torch.sort(ref, dim=1, descending=True, stable=True)
    rs, ri = rs[:, :K], ri[:, :K]
    assert (s.double() - rs).abs().max() <= 2e-5
    flat = (b * V + t).long()
    full = torch.sort(ref, dim=1, descending=True)[0][:, : K + 1]
    for bb in range(B):
        for r in range(K):
            gap = min(full[bb, r - 1] - full[bb, r] if r else float("inf"), full[bb, r] - full[bb, r + 1])
            if gap > 1e-4:
                assert int(flat[bb, r]) == int(ri[bb, r]), (bb, r)
        for r in range(K - 1):                                      # equal fp32 scores: lower flat index first
            if float(s[bb, r]) == float(s[bb, r + 1]):
                assert int(flat[bb, r]) < int(flat[bb, r + 1])
        assert bool((s[bb, :-1] >= s[bb, 1:]).all())


def test_beam_topk_rejects_out_of_range_arguments():
    lib = _b2.load_library()
    t = torch.zeros(64, 1024, device=DEV)
    P, S = _b2.ptr, _b2.stream_ptr
    for B, nb, V, K in [(1, 33, 8, 2), (1, 2, 1024, 129), (1, 2, 3, 7), (0, 1, 8, 1)]:
        assert lib.b2_op_beam_topk(P(t), None, P(t), B, nb, V, K, P(t), P(t), P(t), S()) == -1


# --------------------------------------------------------------------------------------------------------- kv_copy_slots
_ENGINES = {}


def _tiny_engine():
    if "tiny" not in _ENGINES:
        cfg = O.CONFIGS["tiny"]
        _ENGINES["tiny"] = make_engine(cfg, O.make_weights(cfg, seed=0), max_batch=16, max_seq=160)
    return _ENGINES["tiny"]


CFG7 = O.make_config(layers=2, vit_hidden=256, vit_inter=512, vit_layers=3, vit_heads=4, image_size=56)


def _engine7():
    if "7b" not in _ENGINES:
        _ENGINES.pop("tiny", None)
        _ENGINES["7b"] = make_engine(CFG7, O.make_weights(CFG7, seed=1), max_batch=12, max_seq=320)
    return _ENGINES["7b"]


@pytest.mark.parametrize("kv_dtype", ["bf16", "e4m3"])
def test_kv_copy_slots_at_7b_layer_shapes(kv_dtype):
    """After a copy, feeding the same token to src and dst gives the same logit row on each decode path the batch sizes reach
    (4 rows: the GEMV graph; 8 and 12 rows: the stream-K GEMM; an e4m3 cache: the multi-kernel step); the other slots decode
    exactly as on a cache without the copy; rows below row_begin of the destination are kept."""
    eng = _engine7()
    g = torch.Generator().manual_seed(3)
    for n in (4, 8, 12):
        lens = [200 + 7 * i for i in range(n)]
        emb = (torch.randn(n, max(lens), CFG7["hidden"], generator=g) * 0.5).to(torch.bfloat16).to(DEV)
        lens[2] = 150                                                # slot 2: 150 rows of its own
        kvs = [eng.new_kv(12, 320, dtype=kv_dtype) for _ in range(3)]
        for kv in kvs:
            eng.prefill(kv, emb, lens, _b2.LOGITS_NONE)
        eng.kv_copy_slots(kvs[0], [0], [n - 1], row_begin=0)          # whole rows
        eng.kv_copy_slots(kvs[0], [1], [2], row_begin=150)            # rows [150, len(1)) only
        eng.kv_copy_slots(kvs[2], [1], [2], row_begin=0)              # the same copy from row 0
        assert kvs[0].lengths(n)[n - 1] == lens[0] and kvs[0].lengths(n)[2] == lens[1]
        tok = torch.randint(0, CFG7["vocab"], (n,), generator=g, dtype=torch.int32)
        tok[n - 1], tok[2] = tok[0], tok[1]
        a, b, c = (eng.decode_step(kv, tok).cpu() for kv in kvs)
        assert torch.equal(a[n - 1], a[0]), (n, float((a[n - 1] - a[0]).abs().max()))
        assert torch.equal(c[2], c[1]) and torch.equal(c[1], a[1])    # a whole copy decodes as its source
        assert not torch.equal(a[2], a[1])                            # slot 2 kept its own rows below 150
        assert not torch.equal(a[2], b[2])                            # ... and holds slot 1's rows from 150 on
        for r in range(n):
            if r not in (2, n - 1):
                assert torch.equal(a[r], b[r]), (n, r)
        for kv in kvs:
            kv.close()


def test_kv_copy_slots_rejects_hazards_and_ranges():
    eng = _tiny_engine()
    kv = eng.new_kv(6, 64)
    emb = torch.zeros(4, 10, 256, dtype=torch.bfloat16, device=DEV)
    eng.prefill(kv, emb, None, _b2.LOGITS_NONE)
    for src, dst, rb in [([0, 1], [1, 2], 0),        # dst 1 is also a src
                         ([0, 1], [2, 2], 0),        # repeated dst
                         ([0], [6], 0), ([-1], [2], 0),  # out of range
                         ([0], [2], 11)]:            # row_begin beyond len(src)
        with pytest.raises(ValueError):
            eng.kv_copy_slots(kv, src, dst, row_begin=rb)
    assert kv.lengths(4) == [10] * 4
    eng.kv_copy_slots(kv, [0], [4], row_begin=10)
    assert kv.lengths(6)[4] == 10
    kv.close()


# --------------------------------------------------------------------------------------------------- engine beam search
def engine_beam(eng, kv, prompt, nb, max_new, eos=None, lp=1.0, es=False, nrs=1):
    B, Lt = prompt.shape
    s = BM.BeamSearch(prompt, nb, max_new, eos, lp, es, nrs)
    emb = eng.splice(prompt.to(torch.int32).reshape(-1).to(DEV), None, B, Lt)
    kv.reset()
    logits = eng.prefill(kv, emb, None, _b2.LOGITS_LAST)
    cand = [t.cpu() for t in eng.beam_topk(logits, torch.zeros(B), 1, s.K)]
    plan, rb = BM.SlotPlanner(B, nb), 0
    while not s.step(*cand):
        cand = eng.beam_step(kv, plan.plan(s.parents), rb, s.next_tokens().tolist(), plan.flat(),
                             s.running_scores.reshape(-1).tolist(), nb, s.K)
        rb = Lt
    return s.output()


def _text_logits_fn(w, cfg):
    return lambda seqs: O.llama_forward(w, w["model.embed_tokens.weight"][seqs], cfg, last_only=True)[0][:, -1]


@pytest.mark.parametrize("B,nb,kv_dtype", [(1, 2, "bf16"), (1, 4, "bf16"), (2, 4, "bf16"), (3, 4, "bf16"), (1, 4, "e4m3"),
                                            (3, 4, "e4m3"), (2, 3, "bf16")])
def test_engine_beam_search_equals_oracle_strict_ids(B, nb, kv_dtype):
    """condition_weights_beam weights: every decision is far above bf16 noise, so ids must match exactly. Decode paths on a
    bf16 cache: 2 rows the megakernel, 4 and 6 rows the GEMV graph, 8 and 12 rows the stream-K GEMM; an e4m3 cache takes the
    multi-kernel step at every batch size."""
    cfg = O.CONFIGS["tiny"]
    w = BO.condition_weights_beam(O.make_weights(cfg, seed=5), cfg, seed=5)
    eng = make_engine(cfg, w, max_batch=16, max_seq=96)
    kv = eng.new_kv(16, 96, dtype=kv_dtype)
    g = torch.Generator().manual_seed(B * 10 + nb)
    prompt = torch.randint(3, cfg["vocab"], (B, 9), generator=g)
    for eos, nrs in [(None, 1), ([int(prompt[0, 3])], nb)]:
        got = engine_beam(eng, kv, prompt, nb, 12, eos=eos, nrs=nrs)
        want = BO.beam_search(_text_logits_fn(w, cfg), prompt, nb, 12, eos, None, 1.0, False, nrs)
        assert torch.equal(got[0], want[0]), (got[0], want[0])
        torch.testing.assert_close(got[1], want[1], atol=0.05, rtol=0.01)
    kv.close()
    eng.close()


def test_engine_beam_scores_match_a_fresh_prefill():
    """Self-consistency on random weights (catches a wrong reorder): a returned beam's score equals the sum of log_softmax of
    its tokens under a B2_LOGITS_ALL prefill of prompt + continuation, over its length. The bound is derived from a replay of
    the returned sequences through decode steps at the same batch size: with d the largest |decode - prefill| logit difference
    of that replay, a log-probability moves by at most 2 d (the logit and the log-sum-exp), and so does their mean."""
    cfg = O.CONFIGS["tiny"]
    eng = _tiny_engine()
    kv = eng.new_kv(16, 160)
    g = torch.Generator().manual_seed(11)
    prompt = torch.randint(3, cfg["vocab"], (2, 10), generator=g)
    nb, n_new = 4, 16
    seqs, scores = engine_beam(eng, kv, prompt, nb, n_new, nrs=nb)
    Lt, N, L = prompt.shape[1], seqs.shape[0], seqs.shape[1]
    assert L == Lt + n_new                                          # no eos: every returned beam has the full length
    full = eng.prefill(kv, eng.splice(seqs.to(torch.int32).reshape(-1).to(DEV), None, N, L), None, _b2.LOGITS_ALL).double().cpu()
    kv3 = eng.new_kv(16, 160)
    dec = [eng.prefill(kv3, eng.splice(seqs[:, :Lt].to(torch.int32).reshape(-1).to(DEV), None, N, Lt), None, _b2.LOGITS_LAST)]
    for t in range(Lt, L - 1):
        dec.append(eng.decode_step(kv3, seqs[:, t].to(torch.int32)))
    dec = torch.stack([x.double().cpu() for x in dec], 1)           # [N, n_new, V]: logits at positions Lt-1 .. L-2
    d = float((dec - full[:, Lt - 1:L - 1]).abs().max())
    lp = torch.log_softmax(full, -1)
    want = torch.stack([lp[i, torch.arange(Lt - 1, L - 1), seqs[i, Lt:]].sum() / n_new for i in range(N)])
    worst = float((want - scores.double()).abs().max())
    bound = 2 * d + 1e-4
    print(f"beam score vs fresh prefill: max |diff| = {worst:.3e}; decode-vs-prefill logit difference d = {d:.3e}, bound {bound:.3e}")
    assert worst <= bound
    kv.close()
    kv3.close()


def test_one_beam_through_the_beam_machinery_is_greedy():
    cfg = O.CONFIGS["tiny"]
    eng = _tiny_engine()
    kv = eng.new_kv(16, 160)
    g = torch.Generator().manual_seed(12)
    prompt = torch.randint(3, cfg["vocab"], (3, 8), generator=g)
    got = engine_beam(eng, kv, prompt, 1, 20)[0]
    emb = eng.splice(prompt.to(torch.int32).reshape(-1).to(DEV), None, 3, 8)
    kv.reset()
    logits = eng.prefill(kv, emb, None, _b2.LOGITS_LAST)
    first = eng.argmax(logits)
    rest = eng.decode_greedy(kv, first, 19).cpu().t()
    want = torch.cat([prompt, first.cpu()[:, None].long(), rest.long()], 1)
    assert torch.equal(got, want)
    kv.close()


# ------------------------------------------------------------------------------------------------------------ generate()
def _beam_model(max_batch=2, **extra):
    cfg = O.CONFIGS["tiny"]
    w = BO.condition_weights_beam(O.make_weights(cfg, seed=0), cfg, seed=0)
    return cfg, w, make_model(cfg, w, max_batch=max_batch, max_seq=160, **extra)


def test_generate_beam_search():
    cfg, w, model = _beam_model(max_batch=8, b2_beam_search=4)
    ids, images = synth_inputs(cfg, B=2, Lt=12, seed=3)
    ids_d, img_d = ids.to(DEV), images.to(DEV)
    out = model.generate(ids_d, images=img_d, num_beams=4, max_new_tokens=10, eos_token_id=[], num_return_sequences=3)
    assert out.shape[0] == 6 and (out[:, :12].cpu() == ids.repeat_interleave(3, 0)).all()   # prompt echoed, image token too
    assert model._engine.desc.max_batch == 8
    best = model.generate(ids_d, images=img_d, num_beams=4, max_new_tokens=10, eos_token_id=[])
    assert torch.equal(best.cpu(), out[::3].cpu())
    # text-only prompt against the oracle on the same weights: an early eos finish, and the restated reference keyword criterion
    fn = _text_logits_fn({k: v.float() for k, v in w.items()}, cfg)
    p = torch.randint(3, cfg["vocab"], (1, 9), generator=torch.Generator().manual_seed(8))
    free = model.generate(p.to(DEV), num_beams=4, max_new_tokens=10, eos_token_id=[]).cpu()
    eos = int(free[0, 11])                                          # the third token of the best beam
    e = model.generate(p.to(DEV), num_beams=4, max_new_tokens=10, eos_token_id=eos, early_stopping=True).cpu()
    assert torch.equal(e, BO.beam_search(fn, p, 4, 10, [eos], None, 1.0, True)[0])
    assert e.shape[1] < 9 + 10                                      # eos finished the search before the length limit
    tok = _Tok()
    keyword = tok.batch_decode([free[0, 12:14]])[0]                 # text of the best beam's 4th and 5th tokens
    crit = lambda: [_KeywordStop([keyword], tok, p)]
    k = model.generate(p.to(DEV), num_beams=4, max_new_tokens=10, eos_token_id=[], stopping_criteria=crit()).cpu()
    assert torch.equal(k, BO.beam_search(fn, p, 4, 10, [], None, 1.0, False, 1, crit())[0])
    # errors
    with pytest.raises(ValueError):
        model.generate(ids_d, images=img_d, num_beams=4, max_new_tokens=4, streamer=object())
    with pytest.raises(NotImplementedError):
        model.generate(ids_d, images=img_d, num_beams=4, do_sample=True, temperature=0.7, max_new_tokens=4)
    with pytest.raises(ValueError):
        model.generate(ids_d.repeat(3, 1), images=img_d.repeat(3, 1, 1, 1), num_beams=4, max_new_tokens=4)  # 12 beams > 8 slots
    model.invalidate_engine()


def test_beam_search_is_off_without_the_knob():
    cfg, w, model = _beam_model()
    ids, images = synth_inputs(cfg, B=1, Lt=10, seed=1)
    with pytest.raises(NotImplementedError):
        model.generate(ids.to(DEV), images=images.to(DEV), num_beams=4, max_new_tokens=2)
    model.invalidate_engine()


def test_concurrent_beam_and_greedy_threads_equal_serial():
    cfg, w, model = _beam_model(b2_beam_search=4)
    p = [synth_inputs(cfg, B=1, Lt=10 + i, seed=30 + i) for i in range(3)]
    calls = [dict(num_beams=4), dict(num_beams=3), dict()]
    run = lambda i: model.generate(p[i][0].to(DEV), images=p[i][1].to(DEV), max_new_tokens=16, eos_token_id=[], **calls[i]).cpu()
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


# ------------------------------------------------------------------------------------------ random weights, margin-gated
@pytest.mark.parametrize("shape", ["tiny", "7b2"])
def test_engine_beam_search_on_random_weights_where_the_oracle_decides_clearly(shape):
    """Random weights: the engine's ids equal the oracle's for every seed whose decision margins (beam_oracle return_margins:
    candidate ranks K / K+1 and nb / nb+1 at every step) exceed 8x the engine's logit error, measured per seed as
    max |engine - oracle| over the prompt's last-position logits. Prints how many seeds qualify; at these shapes random
    logits put neighbouring candidates 1e-3..1e-1 apart, so few do, and the strict-id tests above carry the id check."""
    cfg = O.CONFIGS["tiny"] if shape == "tiny" else CFG7
    qualified = 0
    for seed in range(6):
        w = O.make_weights(cfg, seed=40 + seed) if shape == "tiny" else _decoder_weights_on_device(cfg, 40 + seed)
        eng = make_engine(cfg, w, max_batch=4, max_seq=64)
        kv = eng.new_kv(4, 64)
        p = torch.randint(3, cfg["vocab"], (1, 9), generator=torch.Generator().manual_seed(seed))
        fn = _device_logits_fn(w, cfg) if shape == "7b2" else _text_logits_fn(w, cfg)
        ref = fn(p).float().cpu()
        err = float((eng.prefill(kv, eng.splice(p.to(torch.int32).reshape(-1).to(DEV), None, 1, 9), None, _b2.LOGITS_LAST).cpu()
                     - ref).abs().max())
        want, _, margins = BO.beam_search(fn, p, 2, 4, None, return_margins=True)
        got = engine_beam(eng, kv, p, 2, 4)[0]
        ok = min(margins) > 8 * err
        print(f"{shape} seed {seed}: min margin {min(margins):.3e}, logit error {err:.3e}, qualifies {ok}, equal {torch.equal(got, want)}")
        if ok:
            qualified += 1
            assert torch.equal(got, want), (seed, got, want)
        kv.close()
        eng.close()
    print(f"{shape}: {qualified} of 6 seeds qualify")


def _decoder_weights_on_device(cfg, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    w = {}
    for key, shape, kind in O.weight_shapes(cfg):
        t = torch.randn(*shape, generator=g, device=DEV) * O.init_std(kind, shape)
        w[key] = (t + 1.0 if kind == "g" else t).to(torch.bfloat16)
    return w


def _device_logits_fn(w, cfg):
    """fp32 oracle forward on the device (the 7B weights stay there as bf16, converted per matmul)."""
    def fn(seqs):
        with torch.device(DEV):
            emb = w["model.embed_tokens.weight"][seqs.to(DEV)].float()
            return O.llama_forward(w, emb, cfg, last_only=True)[0][:, -1]
    return fn


# ------------------------------------------------------------------------------------------------- 7B, 32 layers, strict
def test_7b_full_depth_strict_ids():
    """condition_weights_beam at LLaVA-1.5-7B decoder shapes and depth (32 layers, V = 32000; a small vision tower, unused by
    text prompts): engine ids equal the fp32 oracle's (run on the device) for (B, nb) = (1, 2) megakernel, (1, 4) GEMV graph,
    (2, 4) and (3, 4) stream-K on a bf16 cache, and (1, 4), (3, 4) on an e4m3 cache."""
    cfg = dict(O.CONFIGS["llava-1.5-7b"], vit_hidden=256, vit_inter=512, vit_layers=3, vit_heads=4, image_size=56)
    w = BO.condition_weights_beam(_decoder_weights_on_device(cfg, 7), cfg, seed=7)
    eng = make_engine(cfg, w, max_batch=12, max_seq=64, max_images=1)
    fn = _device_logits_fn(w, cfg)
    for B, nb, kv_dtype in [(1, 2, "bf16"), (1, 4, "bf16"), (2, 4, "bf16"), (3, 4, "bf16"), (1, 4, "e4m3"), (3, 4, "e4m3")]:
        kv = eng.new_kv(12, 64, dtype=kv_dtype)
        p = torch.randint(3, cfg["vocab"], (B, 9), generator=torch.Generator().manual_seed(B * 10 + nb))
        got = engine_beam(eng, kv, p, nb, 8)
        want, _, margins = BO.beam_search(fn, p, nb, 8, None, return_margins=True)
        print(f"7b32 B={B} nb={nb} {kv_dtype}: min margin {min(margins):.3f}, equal {torch.equal(got[0], want)}")
        assert torch.equal(got[0], want), (B, nb, kv_dtype, got[0], want)
        kv.close()
    eng.close()
