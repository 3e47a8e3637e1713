"""GPU: beam sampling. b2_op_beam_sample against the Philox rule restated in numpy (tests/beam_sampling_ref.py), its argument
checks and its law (chi-square), the engine's beam sampling (b2_beam_step_ex + llava/_b2/beam.py) against
beam_sampling_ref.beam_search(sampler="philox"), generate(do_sample=True, num_beams > 1) with config.b2_beam_sample, and the
launch count of a sampled step."""
import itertools
import threading

import numpy as np
import pytest
import torch
from scipy import stats

pytestmark = pytest.mark.gpu

import beam_sampling_ref as BSR  # noqa: E402
from helpers import make_engine, make_model, synth_inputs  # noqa: E402
from llava import _b2  # noqa: E402
from llava._b2 import beam as BM  # noqa: E402
from oracle import beam_oracle as BO  # noqa: E402
from oracle import llava_oracle as O  # noqa: E402
from test_dropin_cpu import _KeywordStop, _Tok  # noqa: E402

DEV = "cuda"
_ENGINES = {}


@pytest.fixture(scope="module", autouse=True)
def _init():
    _b2.init(0)


def _tiny_engine():
    if "tiny" not in _ENGINES:
        cfg = O.CONFIGS["tiny"]
        _ENGINES["tiny"] = make_engine(cfg, O.make_weights(cfg, seed=0), max_batch=16, max_seq=160)
    return _ENGINES["tiny"]


# ------------------------------------------------------------------------------------------------------ b2_op_beam_sample
PARAMS = [(0.2, 50, 1.0), (0.7, 0, 0.9), (1.0, 5, 1.0), (1.5, 0, 1.0), (1.0, 0, 1e-6), (0.7, 50, 0.5)]


def _f32(a):
    return np.asarray(a, dtype=np.float64).astype(np.float32).astype(np.float64)


def _ulp(a):
    return np.spacing(np.abs(np.asarray(a, dtype=np.float32))).astype(np.float64)


@pytest.mark.parametrize("V", [32000, 1000, 40])
@pytest.mark.parametrize("nb", [1, 2, 4, 8])
@pytest.mark.parametrize("kmul", [2, 3])
def test_beam_sample_against_the_philox_rule(V, nb, kmul):
    """Three samples. Sample 0 has a row with -inf logits. Sample 2 fills its list: every row is NaN except two finite
    tokens, so at most 2 nb candidates are finite (fewer than K = 3 nb, and with top_p 1e-6 and min_keep 1 only nb), the
    warped-away ones are -inf and the NaN logits rank last; top-k or top-p is on in every case but one. Half the cases run
    beams at -1e9 (HF's initial beams), whose finite keys all round to the same fp32 values. Rows are read through a
    permutation.

    Bound: the device's w = fp32(((x - max) - lse) / T) differs from the fp32 restatement only through lse = log(sum), the
    sum of up to 32000 terms in [0, 1] in a different fp32 order (32 sequential adds per thread and a tree on the device,
    pairwise in numpy): its relative error, and so the absolute error of lse, stays below 2^-18; the log, the subtraction and
    the division round within 2^-20 of |lse| and |w|: |dw| <= tol_w = (2^-18 + 2^-20 |lse|) / T + 2^-20 |w|. Where fp32(w + run) rounds the same way for every w within
    tol_w (checked in fp64), the device's acc equals the restatement's bit for bit; elsewhere they differ by at most
    tol_w + ulp(acc). The key fp32(acc + g) then moves by that much (g itself agrees to ~1e-15). A candidate whose key is that
    far from every fp32 rounding boundary has the same fp32 key on both sides, so ties between such keys (the -1e9 beams,
    the -inf and NaN fill) are compared exactly. A rank is compared when its candidate and both neighbours in the
    restatement's full order have certain keys, or are further apart than both uncertainties plus an ulp each. Every
    decided rank must hold the same candidate; every score must equal the restatement's acc (exactly where certain) and
    the fp64 acc within tol_w + ulp(acc)."""
    eng = _tiny_engine()
    case = [32000, 1000, 40].index(V) * 8 + [1, 2, 4, 8].index(nb) * 2 + kmul - 2
    T, tk, tp = PARAMS[case % len(PARAMS)]
    B, K = 3, kmul * nb
    mk = 1 if tp < 1e-3 else min([1, 2, 3][case % 3], K)
    g = torch.Generator().manual_seed(case)
    logits = torch.randn(B * nb, V, generator=g) * 3
    perm = torch.randperm(B * nb, generator=g)
    logits[int(perm[0]), : V // 4] = float("-inf")
    for j in range(nb):                                             # sample 2: NaN but for two tokens per row
        r = int(perm[2 * nb + j])
        logits[r] = float("nan")
        logits[r, [j % V, (5 * j + 3) % V]] = torch.randn(2, generator=g) * 3
    scores = torch.randn(B * nb, generator=g)
    if case % 2 == 0:
        scores.view(B, nb)[:, 1:] = -1e9
    seed, step = 1234567 + case, 3 + case
    bs = _b2.make_beam_sampling(T, tk, tp, mk, seed)
    s, t, b = (x.cpu() for x in eng.beam_sample(logits.to(DEV), scores, nb, K, bs, step, row_of_beam=perm.tolist()))
    s = s.double().numpy()
    flat = (b * V + t).long().numpy()
    x = logits[perm].numpy()
    w = np.stack([BSR.device_warp(r, T, tk, tp, mk) for r in x])              # [B * nb, V]
    run = scores.numpy().astype(np.float32)
    acc = (w + run[:, None]).astype(np.float32)
    _, _, _, allk = BSR.philox_select(acc.reshape(B, nb * V), seed, step, nb, K)
    lp64 = torch.log_softmax(torch.nan_to_num(logits[perm].double(), nan=-np.inf), -1).numpy()
    with np.errstate(over="ignore"):
        acc64 = (lp64 / T + scores.double().numpy()[:, None]).reshape(B, nb * V)
    lse = np.log(np.exp(x.astype(np.float64) - np.nanmax(x, 1, keepdims=True)).sum(1, where=~np.isnan(x)))
    with np.errstate(invalid="ignore"):
        tol_w = (2.0 ** -18 + 2.0 ** -20 * np.abs(lse)[:, None]) / T + 2.0 ** -20 * np.abs(w)   # [B * nb, V]
        a64 = w.astype(np.float64) + run.astype(np.float64)[:, None]                   # exact in fp64
        sure_acc = _f32(a64 - tol_w) == _f32(a64 + tol_w)
        dk = np.where(sure_acc, 1e-9, tol_w + _ulp(acc) + 1e-9).reshape(B, nb * V)
        sure_acc = sure_acc.reshape(B, nb * V)
        tol_s = (tol_w + _ulp(acc)).reshape(B, nb * V)
    acc = acc.reshape(B, nb * V)
    decided = fill = 0
    for bb in range(B):
        fin = np.isfinite(acc[bb])
        k64 = allk[bb]
        with np.errstate(invalid="ignore"):
            sure_key = ~fin | (_f32(k64 - dk[bb]) == _f32(k64 + dk[bb]))
        k32 = np.where(fin, _f32(k64), 0.0)
        cls = np.where(fin, 0, np.where(np.isnan(acc[bb]), 2, 1))
        order = np.lexsort((np.arange(nb * V), -k32, cls))                        # the restatement's full order
        fin_dev = np.isfinite(s[bb])
        assert fin_dev.sum() == min(K, fin.sum()), (bb, fin_dev.sum(), fin.sum())  # survivor counts agree
        assert fin[flat[bb][fin_dev]].all(), "a finite device candidate is not a survivor"

        def apart(c, n):  # the device orders c and n as the restatement does
            if not (fin[c] and fin[n]) or (sure_key[c] and sure_key[n]):
                return True   # different classes, ties of -inf / NaN by index, or the same fp32 keys on both sides
            return abs(k64[c] - k64[n]) > dk[bb, c] + dk[bb, n] + _ulp(k64[c]) + _ulp(k64[n])

        for r in range(K):
            c = int(order[r])
            nbrs = [int(order[q]) for q in (r - 1, r + 1) if 0 <= q < nb * V]
            if all(apart(c, n) for n in nbrs):
                assert flat[bb, r] == c, (bb, r, flat[bb], order[:K])
                decided += 1
                fill += not fin[c]
            if flat[bb, r] == c:
                if not fin[c]:
                    assert (np.isnan(s[bb, r]) and np.isnan(acc[bb, c])) or s[bb, r] == acc[bb, c] == -np.inf, (bb, r)
                else:
                    if sure_acc[bb, c]:
                        assert s[bb, r] == acc[bb, c], (bb, r, s[bb, r], acc[bb, c])
                    assert abs(s[bb, r] - acc64[bb, c]) <= tol_s[bb, c], (bb, r, s[bb, r], acc64[bb, c])
    nan_listed = int(np.isnan(s).sum())
    print(f"V={V} nb={nb} K={K} T={T} top_k={tk} top_p={tp} min_keep={mk}: {decided} of {B * K} ranks decided, "
          f"{fill} from the -inf / NaN fill, {nan_listed} NaN")
    assert decided >= B * K // 2
    if kmul == 3:
        assert nan_listed >= 1 and fill >= 1                       # sample 2's list reaches the NaN logits


def test_beam_sample_rejects_bad_arguments():
    lib = _b2.load_library()
    t = torch.zeros(64, 1024, device=DEV)
    P, S = _b2.ptr, _b2.stream_ptr
    good = dict(temperature=0.7, top_k=50, top_p=0.9, min_keep=2)
    for bad in [dict(temperature=0.0), dict(temperature=-1.0), dict(top_p=0.0), dict(top_p=1.5), dict(top_k=-1),
                dict(min_keep=0), dict(min_keep=5)]:
        bs = _b2.make_beam_sampling(**dict(good, **bad))
        assert lib.b2_op_beam_sample(P(t), None, P(t), 1, 2, 1024, 4, bs, 0, P(t), P(t), P(t), S()) == -1, bad
    bs = _b2.make_beam_sampling(**good)
    for B, nb, V, K in [(1, 33, 8, 2), (1, 2, 1024, 129), (1, 2, 3, 7), (0, 1, 8, 1)]:
        assert lib.b2_op_beam_sample(P(t), None, P(t), B, nb, V, K, bs, 0, P(t), P(t), P(t), S()) == -1
    assert lib.b2_op_beam_sample(P(t), None, P(t), 1, 2, 1024, 4, None, 0, P(t), P(t), P(t), S()) == -1


def test_device_draws_follow_plackett_luce():
    """3 tokens x 2 beams, K = 2, 6000 draws (steps): ordered pairs against the exact Plackett-Luce law (chi-square) and
    inclusion counts against torch.multinomial's (contingency chi-square)."""
    eng = _tiny_engine()
    nb, Vs, K, N = 2, 3, 2, 6000
    logits = torch.tensor([[0.4, -0.5, -1.3], [0.1, -0.6, 0.7]])
    run = torch.tensor([0.0, -0.5])
    bs = _b2.make_beam_sampling(1.0, 0, 1.0, 2, 99)
    acc = (torch.log_softmax(logits.double(), -1) + run.double()[:, None]).reshape(-1)
    p = torch.softmax(acc, 0).numpy()
    counts = {}
    incl = np.zeros(nb * Vs)
    ld = logits.to(DEV)
    outs = [eng.beam_sample(ld, run, nb, K, bs, st) for st in range(N)]
    for _, tt, bb in outs:
        f = (bb.cpu() * Vs + tt.cpu()).reshape(-1).tolist()
        counts[tuple(f)] = counts.get(tuple(f), 0) + 1
        incl[f] += 1
    tuples = list(itertools.permutations(range(nb * Vs), K))
    exp = np.array([p[a] * p[c] / (1 - p[a]) for a, c in tuples]) * N
    chi = stats.chisquare(np.array([counts.get(u, 0) for u in tuples], dtype=np.float64), exp)
    tm = torch.multinomial(torch.from_numpy(p).float().expand(N, -1).contiguous(), K, generator=torch.Generator().manual_seed(1))
    ct = stats.chi2_contingency(np.stack([incl, np.bincount(tm.reshape(-1).numpy(), minlength=nb * Vs)]))
    print(f"device ordered pairs: p = {chi.pvalue:.3f}; inclusion vs torch.multinomial: p = {ct.pvalue:.3f}")
    assert chi.pvalue > 1e-3 and ct.pvalue > 1e-3


# --------------------------------------------------------------------------------------------------- engine beam sampling
def engine_beam_sample(eng, kv, prompt, nb, max_new, bs, eos=None, nrs=1):
    B, Lt = prompt.shape
    s = BM.BeamSearch(prompt, nb, max_new, eos, 1.0, False, nrs)
    emb = eng.splice(prompt.to(torch.int32).reshape(-1).to(DEV), None, B, Lt)
    kv.reset()
    logits = eng.prefill(kv, emb, None, _b2.LOGITS_LAST)
    cand = [t.cpu() for t in eng.beam_sample(logits, s.running_scores.reshape(-1), nb, s.K, bs, 0,
                                              row_of_beam=[b for b in range(B) for _ in range(nb)])]
    cand[2].zero_()
    plan, rb, step = BM.SlotPlanner(B, nb), 0, 0
    while not s.step(*cand):
        step += 1
        cand = eng.beam_step(kv, plan.plan(s.parents), rb, s.next_tokens().tolist(), plan.flat(),
                             s.running_scores.reshape(-1).tolist(), nb, s.K, sampling=bs, step=step)
        rb = Lt
    return s.output()


def _text_logits_fn(w, cfg):
    return lambda seqs: O.llama_forward(w, w["model.embed_tokens.weight"][seqs], cfg, last_only=True)[0][:, -1]


NEED, SEED_CAP = 3, 40


def _run_against_oracle(eng, kv, fn, cfg, B, nb, T, tk, tp, seed0, max_new=4, eos=None):
    """Engine vs the Philox reference over seeds seed0, seed0 + 1, ... until NEED seeds qualify (at most SEED_CAP tried);
    returns the number that qualified, each with equal ids.

    A seed qualifies when every decision of the reference (key margins at ranks nb / nb+1 and K / K+1, and the running
    selection's score gaps) exceeds 4 err / T, and the prompt's top-k boundary (the gap between the tk-th and (tk+1)-th
    log-probability of every row) exceeds 2 err. err = max |engine - oracle| of the prompt's last-position log-probabilities
    over each row's tk + 1 largest: a key is acc + g with acc a sum of such log-probabilities over T, so a step moves it by
    about err / T, and four times that covers the running score's accumulation over the steps. A small top_k (2 here) keeps
    the candidates to the tokens that condition_weights_beam separates; with top_k 50 the keys of the tail crowd within the
    bf16 error and hardly a seed qualifies."""
    qualified = tried = 0
    mk = BSR.min_keep_of(eos)
    for seed in range(seed0, seed0 + SEED_CAP):
        tried += 1
        p = torch.randint(3, cfg["vocab"], (B, 9), generator=torch.Generator().manual_seed(seed))
        ref = torch.log_softmax(fn(p).float().cpu(), -1)
        got_lp = torch.log_softmax(eng.prefill(kv, eng.splice(p.to(torch.int32).reshape(-1).to(DEV), None, B, 9), None,
                                               _b2.LOGITS_LAST).float().cpu(), -1)
        top, idx = torch.topk(ref, tk + 1, dim=-1)
        err = float((got_lp.gather(1, idx) - top).abs().max())
        boundary = float((top[:, tk - 1] - top[:, tk]).min())
        want, want_s, margins = BSR.beam_search(fn, p, nb, max_new, eos, None, 1.0, False, 1, return_margins=True, do_sample=True,
                                                temperature=T, top_k=tk, top_p=tp, sampler="philox", seed=seed)
        got = engine_beam_sample(eng, kv, p, nb, max_new, _b2.make_beam_sampling(T, tk, tp, mk, seed), eos=eos)
        ok = min(margins) > 4 * err / T and boundary > 2 * err
        print(f"B={B} nb={nb} T={T} top_k={tk} top_p={tp} seed {seed}: min margin {min(margins):.3e}, top-k gap {boundary:.3e}, "
              f"log-prob error {err:.3e}, qualifies {ok}, equal {torch.equal(got[0], want)}")
        if ok:
            qualified += 1
            assert torch.equal(got[0], want), (seed, got[0], want)
            torch.testing.assert_close(got[1], want_s, atol=0.05, rtol=0.01)
            if qualified == NEED:
                break
    print(f"B={B} nb={nb} T={T} top_k={tk} top_p={tp}: {qualified} of {tried} seeds qualify")
    return qualified


@pytest.mark.parametrize("B,nb,kv_dtype", [(1, 2, "bf16"), (1, 4, "bf16"), (2, 4, "bf16"), (3, 4, "bf16"), (2, 2, "bf16"),
                                            (1, 4, "e4m3"), (3, 4, "e4m3")])
def test_engine_beam_sampling_equals_the_philox_reference(B, nb, kv_dtype):
    """condition_weights_beam weights; for each of two settings (T 1.0 / top_k 2, no eos; T 0.7 / top_k 2 / top_p 0.9 with an
    eos id, whose K = 4 nb candidates include the -inf fill) NEED seeds must qualify and give equal ids."""
    cfg = O.CONFIGS["tiny"]
    w = BO.condition_weights_beam(O.make_weights(cfg, seed=5), cfg, seed=5)
    eng = make_engine(cfg, w, max_batch=16, max_seq=96)
    kv = eng.new_kv(16, 96, dtype=kv_dtype)
    fn = _text_logits_fn(w, cfg)
    assert _run_against_oracle(eng, kv, fn, cfg, B, nb, 1.0, 2, 1.0, B * 1000 + nb * 100) >= NEED
    assert _run_against_oracle(eng, kv, fn, cfg, B, nb, 0.7, 2, 0.9, B * 1000 + nb * 100 + 50, eos=[7]) >= NEED
    kv.close()
    eng.close()


def test_engine_beam_sampling_at_7b_width():
    """LLaVA-1.5-7B decoder width (hidden 4096, V = 32000), 2 layers, condition_weights_beam weights, B = 2, nb = 4."""
    cfg = O.make_config(layers=2, vit_hidden=256, vit_inter=512, vit_layers=3, vit_heads=4, image_size=56)
    g = torch.Generator(device=DEV).manual_seed(9)
    w = {}
    for key, shape, kind in O.weight_shapes(cfg):
        t = torch.randn(*shape, generator=g, device=DEV) * O.init_std(kind, shape)
        w[key] = (t + 1.0 if kind == "g" else t).to(torch.bfloat16)
    w = BO.condition_weights_beam(w, cfg, seed=9)
    eng = make_engine(cfg, w, max_batch=8, max_seq=64)
    kv = eng.new_kv(8, 64)

    def fn(seqs):
        with torch.device(DEV):
            emb = w["model.embed_tokens.weight"][seqs.to(DEV)].float()
            return O.llama_forward(w, emb, cfg, last_only=True)[0][:, -1]

    assert _run_against_oracle(eng, kv, fn, cfg, 2, 4, 1.0, 2, 1.0, 0) >= NEED
    kv.close()
    eng.close()


def test_sampled_step_makes_as_many_launches_as_a_greedy_step():
    eng = _tiny_engine()
    kv = eng.new_kv(16, 160)
    cfg = O.CONFIGS["tiny"]
    lib = _b2.load_library()
    p = torch.randint(3, cfg["vocab"], (2, 9), generator=torch.Generator().manual_seed(1))
    emb = eng.splice(p.to(torch.int32).reshape(-1).to(DEV), None, 2, 9)
    counts = []
    for sampling in (None, None, _b2.make_beam_sampling(0.7, 50, 0.9, 2, 3), None, _b2.make_beam_sampling(0.2, 50, 1.0, 2, 3)):
        eng.prefill(kv, emb, None, _b2.LOGITS_NONE)
        eng.kv_copy_slots(kv, [0, 1], [2, 3])
        n0 = lib.b2_launch_count()
        eng.beam_step(kv, [], 0, [5, 6, 7, 8], [0, 2, 1, 3], [0.0, -1.0, 0.0, -2.0], 2, 4, sampling=sampling, step=1)
        counts.append(lib.b2_launch_count() - n0)
    counts = counts[1:]  # the first step at a batch size also captures its decode graph
    print(f"launches per beam step: greedy {counts[0]}, sampled {counts[1]}")
    assert counts[0] == counts[1] == counts[2] == counts[3]
    kv.close()


# ------------------------------------------------------------------------------------------------------------ generate()
def _beam_model(max_batch=8, weights=None, **extra):
    cfg = O.CONFIGS["tiny"]
    w = weights if weights is not None else BO.condition_weights_beam(O.make_weights(cfg, seed=0), cfg, seed=0)
    return cfg, w, make_model(cfg, w, max_batch=max_batch, max_seq=160, **extra)


def test_generate_beam_sampling():
    cfg, w, model = _beam_model(b2_beam_search=4, b2_beam_sample=True)
    ids, images = synth_inputs(cfg, B=2, Lt=12, seed=3)
    ids_d, img_d = ids.to(DEV), images.to(DEV)
    kw = dict(num_beams=4, do_sample=True, temperature=0.7, top_p=0.9, max_new_tokens=10, eos_token_id=[])
    torch.manual_seed(5)
    a = model.generate(ids_d, images=img_d, num_return_sequences=3, **kw).cpu()
    torch.manual_seed(5)
    b = model.generate(ids_d, images=img_d, num_return_sequences=3, **kw).cpu()
    assert torch.equal(a, b)                                        # same seed, same ids
    assert a.shape[0] == 6 and (a[:, :12] == ids.repeat_interleave(3, 0)).all()   # prompt echoed, image token too
    # conditioned weights make a few continuations dominate; on plain random weights different seeds draw different ids
    _, _, flat = _beam_model(b2_beam_search=4, b2_beam_sample=True, weights=O.make_weights(cfg, seed=1))
    runs = []
    for s in (5, 5, 6, 7, 8):
        torch.manual_seed(s)
        runs.append(flat.generate(ids_d, images=img_d, **dict(kw, temperature=1.0)).cpu())
    assert torch.equal(runs[0], runs[1])
    assert any(not torch.equal(o, runs[0]) for o in runs[2:])        # different seeds, different ids at least once
    flat.invalidate_engine()
    # text prompt against the Philox reference: eos and keyword stops
    fn = _text_logits_fn({k: v.float() for k, v in w.items()}, cfg)
    p = torch.randint(3, cfg["vocab"], (1, 9), generator=torch.Generator().manual_seed(8))
    torch.manual_seed(3)
    free = model.generate(p.to(DEV), **kw).cpu()
    eos = int(free[0, 11])
    kwe = dict(kw, eos_token_id=eos)
    torch.manual_seed(3)
    seed = int(torch.randint(0, 2**62, (1,), dtype=torch.int64).item())
    torch.manual_seed(3)
    e = model.generate(p.to(DEV), **kwe).cpu()
    want_e = BSR.beam_search(fn, p, 4, 10, [eos], None, do_sample=True, temperature=0.7, top_k=50, top_p=0.9, sampler="philox",
                             seed=seed)[0]
    assert torch.equal(e, want_e), (e, want_e)
    tok = _Tok()
    keyword = tok.batch_decode([free[0, 12:14]])[0]
    crit = lambda: [_KeywordStop([keyword], tok, p)]
    torch.manual_seed(3)
    k = model.generate(p.to(DEV), stopping_criteria=crit(), **kw).cpu()
    want_k = BSR.beam_search(fn, p, 4, 10, [], None, 1.0, False, 1, crit(), do_sample=True, temperature=0.7, top_k=50, top_p=0.9,
                             sampler="philox", seed=seed)[0]
    assert torch.equal(k, want_k), (k, want_k)
    # errors and the plain beam search below temperature 1e-5
    with pytest.raises(ValueError):
        model.generate(ids_d, images=img_d, num_beams=4, do_sample=True, max_new_tokens=4, streamer=object())
    with pytest.raises(ValueError):
        model.generate(ids_d, images=img_d, num_beams=4, do_sample=True, top_p=0.0, max_new_tokens=4)
    g0 = model.generate(p.to(DEV), num_beams=4, do_sample=True, temperature=0.0, max_new_tokens=6, eos_token_id=[]).cpu()
    assert torch.equal(g0, model.generate(p.to(DEV), num_beams=4, max_new_tokens=6, eos_token_id=[]).cpu())
    model.invalidate_engine()


def test_concurrent_beam_sampling_and_greedy_threads_equal_serial():
    """A beam-sampling thread next to a beam-search and a greedy thread (neither draws from torch's generator, so the sampling
    thread's seed is the one torch.manual_seed fixes before the threads start)."""
    cfg, w, model = _beam_model(max_batch=4, b2_beam_search=4, b2_beam_sample=True)
    p = [synth_inputs(cfg, B=1, Lt=10 + i, seed=30 + i) for i in range(3)]
    calls = [dict(num_beams=4, do_sample=True, temperature=0.7, top_p=0.9), dict(num_beams=3), dict()]
    run = lambda i: model.generate(p[i][0].to(DEV), images=p[i][1].to(DEV), max_new_tokens=16, eos_token_id=[], **calls[i]).cpu()
    torch.manual_seed(100)
    serial = [run(i) for i in range(3)]
    res, errs = [None] * 3, []

    def work(i):
        try:
            res[i] = run(i)
        except Exception as e:  # pragma: no cover
            errs.append(e)

    torch.manual_seed(100)
    th = [threading.Thread(target=work, args=(i,)) for i in range(3)]
    [t.start() for t in th]
    [t.join() for t in th]
    assert not errs, errs
    for i in range(3):
        assert torch.equal(res[i], serial[i]), i
    model.invalidate_engine()
