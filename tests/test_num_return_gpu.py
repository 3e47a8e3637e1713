"""GPU: generate(do_sample=True, num_return_sequences=n) and the shared-prefix decode attention behind it.

- b2_op_decode_attn_shared against an fp64 reference under the bound of tests/test_attention_numerics_gpu.py, with follower
  slots poisoned in [0, P) and the source slot poisoned past P (a wrong indirection attends +-1e3 values); needles at P - 1,
  P, the split edges and the new token; one to four groups of 1, 2, 15 and 16 rows at different P; suffixes 0, 1, 63, 64, 65.
  The appended K / V rows are bit-identical to b2_op_decode_attn's on the same qkv, and the split counters end at zero.
- Forked generations at B * n = 2 (megakernel), 4 and 8 (GEMV graph), 12 and 32 (stream-K): every draw, token 0 included, is the
  one the Philox target of (seed, index, slot) selects from the returned raw logits row; greedy-like temperature gives every
  sibling the batch-B greedy ids.
- The shared step against the same forked generation on decode_attn (share_prefix=False): the first decode step's logits rows
  within 2 % max / 0.3 % mean of the std, the same launches per step. An e4m3 cache (which reads every row's own copy) within
  ENGINE_LOGIT_TOL of the bf16 cache. Processors on forked rows match logits_proc_oracle.
- A plain generation after a forked one on the same pooled cache equals the same generation on a fresh model; a forked call
  prefills once."""

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from helpers import make_model, rel_err  # noqa: E402
from llava import _b2  # noqa: E402
from llava._b2.fork import ForkPlan  # noqa: E402
from oracle import llava_oracle as O  # noqa: E402
from oracle import logits_proc_oracle as LP  # noqa: E402
from oracle import sampling_oracle as S  # noqa: E402
from test_attention_numerics_gpu import F64, KAPPA, T_NEEDLE, attend, bound, rope_rows_cpu  # noqa: E402
from test_kv_fp8_oracle import ENGINE_LOGIT_TOL  # noqa: E402

DEV, BF = "cuda", torch.bfloat16
CFG = O.CONFIGS["tiny"]
W = None

def _weights():
    global W
    if W is None:
        W = O.make_weights(CFG, seed=0)
    return W

def _P(t):
    return _b2.ptr(t)

@pytest.fixture(scope="module")
def lib():
    _b2.init(0)
    return _b2.load_library()

# ------------------------------------------------------------------------------------------------------ kernel
def shared_splits(lo, hi, nsplit):
    chunk = (hi - lo + nsplit - 1) // nsplit
    return [(min(lo + s * chunk, hi), min(lo + s * chunk + chunk, hi)) for s in range(nsplit)]

def build_shared(Ps, ns, suffix, H, seed, nsplit):
    """Slot 0 .. G-1: the groups' sources (rows outside every group at pos = P_g, so their keys past P_g are never theirs);
    then the groups' rows, at pos = P_g + suffix. Follower rows hold poison in [0, P_g) and the sources poison past P_g, aimed
    at the rows that must not see it. Returns the inputs and, per (row, head), the keys / values the row must attend."""
    G = len(Ps)
    B = G + sum(ns)
    D, scale = 128, 128 ** -0.5
    Smax = max(Ps) + suffix + 4
    Smax = (Smax + 63) // 64 * 64
    g = torch.Generator().manual_seed(seed)
    groups, lens, member = [], [], {}
    r = G
    for gi, (P, n) in enumerate(zip(Ps, ns)):
        groups.append((gi, P, list(range(r, r + n))))
        for row in range(r, r + n):
            member[row] = gi
        r += n
    lens = [Ps[gi] for gi in range(G)] + [Ps[member[row]] + suffix for row in range(G, B)]
    qkv = torch.randn(B, 3, H, D, generator=g, dtype=F64)
    qkv = qkv.to(BF).to(F64)
    kc = torch.randn(B, H, Smax, D, generator=g, dtype=F64)
    vc = torch.randn(B, H, Smax, D, generator=g, dtype=F64)
    q_roped, _ = rope_rows_cpu(qkv.reshape(B, -1).to(BF), lens, H)
    poison_v = lambda: 1e3 * (torch.randint(0, 2, (D,), generator=g) * 2 - 1).to(F64)  # noqa: E731
    for row in range(G, B):
        gi = member[row]
        P, src, pos = Ps[gi], gi, lens[row]
        for h in range(H):
            q = q_roped[row, h].to(F64)
            aim = q / (scale * (q * q).sum())
            for key in {P - 1, P - 2} & set(range(P)):  # this row's own (stale) copy of the prompt: never read
                kc[row, h, key] = (T_NEEDLE + 2) * aim
                vc[row, h, key] = poison_v()
            for key in range(P, min(P + 2, Smax)):      # the source past P: never read by a member
                if row == groups[gi][2][0]:
                    kc[src, h, key] = (T_NEEDLE + 2) * aim
                    vc[src, h, key] = poison_v()
            if row == groups[gi][2][0]:
                edges = {e - 1 for s, e in shared_splits(0, P, nsplit) if e > s}
                for i, key in enumerate(sorted(edges | {P - 1})):
                    kc[src, h, key] = (T_NEEDLE - (i % 3)) * aim
                    vc[src, h, key] = 8.0 * torch.nn.functional.one_hot(torch.tensor((key * 37) % D), D).to(F64)
                if pos > P:
                    kc[row, h, P] = (T_NEEDLE - 1) * aim
            qp = qkv[row, 0, h]
            qkv[row, 1, h] = (T_NEEDLE - 0.5) * qp / (scale * (qp * qp).sum())
    qkv = qkv.reshape(B, -1).to(BF)
    kc, vc = kc.to(BF), vc.to(BF)
    return dict(qkv=qkv, kc=kc, vc=vc, lens=lens, groups=groups, member=member, Smax=Smax, B=B, G=G)

def shared_problems(inp, q_roped, k_new, H, own_prefix=False, src_past=0, p_shift=0):
    """(row, head, problem) of every grouped row: keys [0, P) from the source, [P, pos) from the row, the new token at pos.
    The keyword arguments build the mutated references (own prefix, source read `src_past` keys past P, P moved)."""
    out = []
    v3 = inp["qkv"].view(inp["B"], 3, H, 128)
    for row, gi in inp["member"].items():
        src, P, _ = inp["groups"][gi]
        P = P + p_shift
        pos = inp["lens"][row]
        for h in range(H):
            k = inp["kc"][row, h, :pos + 1].clone()
            v = inp["vc"][row, h, :pos + 1].clone()
            if not own_prefix:
                k[:P], v[:P] = inp["kc"][src, h, :P], inp["vc"][src, h, :P]
            if src_past:
                e = min(P + src_past, pos)
                k[P:e], v[P:e] = inp["kc"][src, h, P:e], inp["vc"][src, h, P:e]
            k[pos], v[pos] = k_new[row, h], v3[row, 2, h]
            pr = dict(q=q_roped[row, h].to(F64)[None], k=k.to(F64), v=v.to(F64), lim=torch.tensor([pos]),
                      rows=torch.tensor([True]), scale=128 ** -0.5)
            out.append((row, h, pr))
    return out

KERNEL_CASES = [
    dict(Ps=[63], ns=[1], suffix=0), dict(Ps=[65], ns=[2], suffix=1), dict(Ps=[127], ns=[15], suffix=63),
    dict(Ps=[129], ns=[16], suffix=64), dict(Ps=[64, 193], ns=[2, 16], suffix=65),
    dict(Ps=[191, 63, 129], ns=[15, 1, 2], suffix=1), dict(Ps=[65, 127, 255, 63], ns=[16, 2, 1, 15], suffix=64),
]

def _kid(c):
    return f"P{'-'.join(map(str, c['Ps']))}_n{'-'.join(map(str, c['ns']))}_s{c['suffix']}"

def _device_rope(lib, qkv, lens, H, Smax):
    B = qkv.shape[0]
    x = qkv.clone().to(DEV)
    kd = torch.zeros(B, H, Smax, 128, device=DEV, dtype=BF)
    vd = torch.zeros_like(kd)
    pos = torch.tensor(lens, device=DEV, dtype=torch.int32)
    _b2.check(lib.b2_op_rope_kv_write_at(_P(x), _P(kd), _P(vd), _P(pos), B, 1, H, 128, Smax, 10000.0, _b2.stream_ptr()))
    return x.view(B, 3, H, 128)[:, 0].cpu(), torch.stack([kd[b, :, lens[b]] for b in range(B)]).cpu()

@pytest.mark.parametrize("case", KERNEL_CASES, ids=[_kid(c) for c in KERNEL_CASES])
def test_shared_kernel_vs_fp64(lib, case):
    H = 2
    inp = build_shared(case["Ps"], case["ns"], case["suffix"], H, seed=3, nsplit=1)
    B, Smax = inp["B"], inp["Smax"]
    nsplit = int(lib.b2_op_decode_attn_shared_nsplit(B, H, Smax))
    inp = build_shared(case["Ps"], case["ns"], case["suffix"], H, seed=3, nsplit=nsplit)
    q_roped, k_new = _device_rope(lib, inp["qkv"], inp["lens"], H, Smax)
    groups = _b2._group_array(inp["groups"])
    qkv = inp["qkv"].to(DEV)
    cur = torch.tensor(inp["lens"], device=DEV, dtype=torch.int32)
    scratch = torch.zeros(int(lib.b2_op_decode_attn_shared_scratch_bytes(B, H, nsplit)), device=DEV, dtype=torch.uint8)
    out = torch.full((B, H * 128), float("nan"), device=DEV, dtype=BF)
    for _ in range(2):  # the second launch runs on the counters the first one left behind
        kc, vc = inp["kc"].to(DEV), inp["vc"].to(DEV)
        _b2.check(lib.b2_op_decode_attn_shared(_P(qkv), _P(kc), _P(vc), _P(cur), groups, inp["G"], _P(out), _P(scratch), B, H, Smax,
                                               nsplit, 10000.0, 128 ** -0.5, _b2.stream_ptr()), "b2_op_decode_attn_shared")
    attn = int(lib.b2_op_decode_attn_shared_scratch_bytes(B, H, nsplit)) - B * (19 * 4 + 4)
    assert int(scratch[attn - B * H * 4: attn].view(torch.int32).abs().sum()) == 0, "counters must be left at zero"
    o = out.view(B, H, 128).cpu().to(F64)
    worst = 0.0
    for row, h, pr in shared_problems(inp, q_roped, k_new, H):
        ref, p = attend(pr)
        assert torch.isfinite(o[row, h]).all()
        r = float(((o[row, h][None] - ref).abs() / bound(pr, ref, p)).max())
        worst = max(worst, r)
        assert r <= 1.0, f"row {row} head {h}: err/bound {r:.3f} (> 1 at kappa = {KAPPA})"
    print(f"\n[num-return] decode_attn_shared {_kid(case)} nsplit {nsplit}: worst err/bound {worst:.4f}")
    # the appended rows: bit-identical to decode_attn's on the same qkv
    kd, vd = inp["kc"].to(DEV), inp["vc"].to(DEV)
    sd = torch.zeros(int(lib.b2_op_decode_attn_scratch_bytes(B, H, 4)), device=DEV, dtype=torch.uint8)
    od = torch.empty_like(out)
    _b2.check(lib.b2_op_decode_attn(_P(qkv), _P(kd), _P(vd), _P(cur), _P(od), _P(sd), B, H, Smax, 4, 10000.0, 128 ** -0.5,
                                    _b2.stream_ptr()))
    for b, pos in enumerate(inp["lens"]):
        assert torch.equal(kc[b, :, pos], kd[b, :, pos]) and torch.equal(vc[b, :, pos], vd[b, :, pos]), b
    assert torch.equal(kc, kd) and torch.equal(vc, vd)

# ------------------------------------------------------------------------------------------------------ engine
def _model(**extra):
    return make_model(CFG, _weights(), max_batch=32, max_seq=160, **extra)

@pytest.fixture(scope="module")
def model():
    return _model()

def _prompt(B, seed, Lt=12):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(3, CFG["vocab"], (B, Lt), generator=g)
    ids[:, 0] = 1
    return ids.to(DEV)

def _check_draw(row, tok, T, k, p, seed, index, slot):
    want, info = S.sample_row(row, T, k, p, seed, index, slot)
    if tok == want:
        return
    slack = 1e-6 * info["total"]
    assert info["lo"][tok] - slack <= info["target"] <= info["hi"][tok] + slack, (tok, want, index, slot)

@pytest.mark.parametrize("B,n", [(1, 2), (1, 4), (3, 4), (2, 16), (4, 8), (2, 4)], ids=["mega-1x2", "gemv-1x4", "sk-3x4", "sk-2x16", "sk-4x8", "gemv-2x4"])
def test_forked_draws_follow_the_philox_targets(model, B, n):
    ids = _prompt(B, seed=10 + B * n)
    kw = dict(do_sample=True, temperature=0.8, top_k=40, top_p=0.95)
    torch.manual_seed(7)
    seed = int(torch.randint(0, 2**62, (1,), dtype=torch.int64).item())
    torch.manual_seed(7)
    out = model.generate(ids, num_return_sequences=n, max_new_tokens=6, eos_token_id=[], return_dict_in_generate=True,
                         output_logits=True, **kw)
    assert out.sequences.shape == (B * n, ids.shape[1] + 6)
    assert torch.equal(out.sequences[:, :ids.shape[1]].cpu(), ids.cpu().repeat_interleave(n, 0))
    slot = ForkPlan([ids.shape[1]] * B, n).slot_of_row
    for t, lg in enumerate(out.logits):
        assert lg.shape == (B * n, CFG["vocab"])
        for r in range(B * n):
            _check_draw(lg[r].cpu().numpy(), int(out.sequences[r, ids.shape[1] + t]), 0.8, 40, 0.95, seed, t, slot[r])
    # siblings of a prompt start from the same prefill row
    for b in range(B):
        for j in range(1, n):
            assert torch.equal(out.logits[0][b * n], out.logits[0][b * n + j])

@pytest.mark.parametrize("B,n", [(1, 2), (1, 4), (3, 4), (4, 8)])
def test_greedy_like_temperature_gives_equal_siblings(model, B, n):
    ids = _prompt(B, seed=30 + B)
    greedy = model.generate(ids, do_sample=False, max_new_tokens=8, eos_token_id=[])
    out = model.generate(ids, do_sample=True, temperature=1e-6, num_return_sequences=n, max_new_tokens=8, eos_token_id=[])
    assert torch.equal(out.cpu(), greedy.cpu().repeat_interleave(n, 0))

def _forked_logits(model, ids, n, steps, share, kv_model=None):
    """A forked greedy generation driven through the engine: (ids [slots, steps], raw logits [steps, slots, V]), launches/step."""
    m = kv_model or model
    eng = m._ensure_engine()
    B, Lt = ids.shape
    plan = ForkPlan([Lt] * B, n)
    kv = m._pool.acquire()
    try:
        kv.reset()
        emb = eng.splice(ids.to(torch.int32).reshape(-1), None, B, Lt)
        logits = eng.prefill(kv, emb, [Lt] * B, _b2.LOGITS_LAST)
        eng.kv_copy_slots(kv, *plan.copies())
        logits = logits.index_select(0, torch.tensor(plan.prompt_of_slot, device=DEV))
        rows = torch.empty(steps, B * n, CFG["vocab"], dtype=torch.float32, device=DEV)
        eng.stream_begin(kv, logits, None, None, None, rows, groups=plan.groups(), share_prefix=share)
        eng.stream_wait(kv, 0, B * n)
        eng.stream_enqueue(kv, 2)
        eng.stream_wait(kv, 2, B * n)
        torch.cuda.synchronize()
        c0 = _b2.launch_count()
        eng.stream_enqueue(kv, steps - 3)
        toks = [eng.stream_wait(kv, t, B * n) for t in range(steps)]
        torch.cuda.synchronize()
        per_step = (_b2.launch_count() - c0) / (steps - 3)
    finally:
        m._pool.release(kv, None)
    return torch.tensor(toks).t(), rows.cpu(), per_step

@pytest.mark.parametrize("B,n", [(3, 4), (4, 8), (1, 4), (1, 2)], ids=["sk-12", "sk-32", "gemv-4", "mega-2"])
def test_shared_step_matches_decode_attn(model, B, n):
    ids = _prompt(B, seed=50 + B)
    steps = 12
    t1, l1, c1 = _forked_logits(model, ids, n, steps, share=True)
    t0, l0, c0 = _forked_logits(model, ids, n, steps, share=False)
    assert c1 == c0, (c1, c0)
    # step 1 is the first decode step, and the one whose inputs are the same on both paths (the prefilled and copied rows, token
    # 0): later steps attend rows each path appended from its own, slightly different, hidden states
    assert torch.equal(t1[:, :2], t0[:, :2])
    for s in range(B * n):
        mx, mn = rel_err(l1[1, s], l0[1, s])
        assert mx < 0.02 and mn < 0.003, (s, mx, mn)

def test_e4m3_fork_within_engine_tolerance():
    ids = _prompt(3, seed=71)
    bf = _model()
    e4 = _model(b2_kv_dtype="e4m3")
    t1, l1, _ = _forked_logits(bf, ids, 4, 8, share=True)
    t0, l0, _ = _forked_logits(e4, ids, 4, 8, share=True)
    for s in range(12):
        same = int((t1[s] != t0[s]).nonzero()[0, 0]) if bool((t1[s] != t0[s]).any()) else 8
        for t in range(min(same + 1, 8)):
            mx, mn = rel_err(l0[t, s], l1[t, s])
            assert mx < ENGINE_LOGIT_TOL[0] and mn < ENGINE_LOGIT_TOL[1], (s, t, mx, mn)

def test_processors_on_forked_rows_match_the_oracle():
    m = _model(b2_logits_processors=True)
    ids = _prompt(2, seed=81)
    n = 6
    kw = dict(repetition_penalty=1.4, no_repeat_ngram_size=2)
    out = m.generate(ids, do_sample=True, temperature=0.9, top_k=0, num_return_sequences=n, max_new_tokens=8, eos_token_id=[],
                     return_dict_in_generate=True, output_logits=True, output_scores=True, **kw)
    seq = out.sequences.cpu()
    Lt = ids.shape[1]
    for t in range(len(out.scores)):
        for r in range(2 * n):
            hist = seq[r, :Lt + t].tolist()
            want = LP.process(out.logits[t][r].cpu().numpy(), hist, Lt, kw["repetition_penalty"], kw["no_repeat_ngram_size"], 0, [])
            got = out.scores[t][r].cpu().numpy() * 0.9
            fin = np.isfinite(want)
            assert np.array_equal(np.isfinite(got), fin), (t, r)
            np.testing.assert_allclose(got[fin], want[fin], rtol=1e-5, atol=1e-5)

def test_plain_generation_after_a_fork_on_the_pooled_cache():
    ids = _prompt(3, seed=91)
    m = _model()
    m.generate(ids, do_sample=True, num_return_sequences=8, max_new_tokens=6, eos_token_id=[])
    after = m.generate(ids, do_sample=False, max_new_tokens=10, eos_token_id=[])
    fresh = _model().generate(ids, do_sample=False, max_new_tokens=10, eos_token_id=[])
    assert torch.equal(after.cpu(), fresh.cpu())

def test_one_prefill_for_b_prompts(monkeypatch):
    m = _model()
    eng = m._ensure_engine()
    calls = []
    real = eng.prefill
    monkeypatch.setattr(eng, "prefill", lambda kv, emb, *a, **k: calls.append(emb.shape[0]) or real(kv, emb, *a, **k))
    m.generate(_prompt(3, seed=95), do_sample=True, num_return_sequences=5, max_new_tokens=3, eos_token_id=[])
    assert calls == [3]
