"""GPU: the e4m3 KV cache (b2_kv_create_ex(B2_KV_E4M3)) against oracle/kv_fp8_oracle.py, through the C ABI and the Python
surface: the quantising prefill cache write, the fp8 split-KV decode attention, the engine on both weight formats, strict
greedy ids on the well-conditioned weight set (plain and continuously batched), generate(), and the error paths."""
import ctypes
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from helpers import make_engine, make_model, rel_err, synth_inputs  # noqa: E402
from llava import _b2  # noqa: E402
from oracle import kv_fp8_oracle as KV  # noqa: E402
from oracle import llava_oracle as O  # noqa: E402
from test_kv_fp8_oracle import ENGINE_LOGIT_TOL  # noqa: E402

DEV, BF, D = "cuda", torch.bfloat16, 128
P, S = _b2.ptr, _b2.stream_ptr
KERNEL_TOL = (0.08, 0.015)   # engine vs the restated step over the same quantised cache: bf16 rounding of the rest of the layer


@pytest.fixture(scope="module", autouse=True)
def _init():
    _b2.init(0)
    torch.manual_seed(0)


def u8(t):
    return t.view(torch.uint8)


# ---------------------------------------------------------------------------------------------- prefill cache write
@pytest.mark.parametrize("B,S_,lens,slot0", [(2, 128, None, 0), (3, 203, [203, 1, 77], 1), (1, 64, [64], 2), (2, 70, [5, 70], 0)])
def test_kv_quantize_bit_exact(B, S_, lens, slot0):
    """7B head geometry (32 heads of 128): bytes and scales equal the oracle bit for bit; S on and off the 64-token tile,
    ragged lengths, a non-zero slot offset; rows beyond seq_lens and other slots keep what they held."""
    H, Smax, Bmax = 32, 256, 4
    g = torch.Generator().manual_seed(S_)
    k = (torch.randn(B, H, S_, D, generator=g) * torch.logspace(-2, 1, S_)[:, None]).to(BF)
    v = torch.randn(B, H, S_, D, generator=g).to(BF)
    k[0, 0, 0] = 0                                           # a zero row: scale 1
    k8 = torch.full((Bmax, H, Smax, D), 0x5A, device=DEV, dtype=torch.uint8)
    v8 = torch.full_like(k8, 0x5A)
    ks = torch.full((Bmax, H, Smax), -7.0, device=DEV)
    vs = torch.full_like(ks, -7.0)
    lens_d = None if lens is None else torch.tensor(lens, device=DEV, dtype=torch.int32)
    kd, vd = k.to(DEV), v.to(DEV)
    _b2.check(_b2.load_library().b2_op_kv_quantize_e4m3(P(kd), P(vd), P(k8[slot0:]), P(v8[slot0:]), P(ks[slot0:]), P(vs[slot0:]),
                                                        P(lens_d), B, S_, H, Smax, S()), "kv_quantize")
    want = dict(k8=torch.full((Bmax, H, Smax, D), 0x5A, dtype=torch.uint8).view(torch.float8_e4m3fn),
                v8=torch.full((Bmax, H, Smax, D), 0x5A, dtype=torch.uint8).view(torch.float8_e4m3fn),
                ks=torch.full((Bmax, H, Smax), -7.0), vs=torch.full((Bmax, H, Smax), -7.0))
    KV.store_rows(want, k, v, lens, slot0=slot0)
    assert torch.equal(ks.cpu(), want["ks"]) and torch.equal(vs.cpu(), want["vs"])
    for got, ref in ((k8, want["k8"]), (v8, want["v8"])):
        bad = (got.cpu() != u8(ref)).nonzero()
        assert len(bad) == 0, f"{len(bad)} codes differ, first at {bad[0].tolist()}"
    assert float(ks[slot0, 0, 0]) == 1.0


# ---------------------------------------------------------------------------------------------- decode attention
LENGTHS = [0, 1, 7, 127, 128, 703, 711]   # Smax - 1 = 711


def _attn_case(B, H, lens, nsplit):
    Smax = 712
    lib = _b2.load_library()
    g = torch.Generator().manual_seed(B * 1000 + H)
    qkv = torch.randn(B, 3 * H * D, generator=g).to(BF)
    cache = KV.empty_cache(B, H, Smax)
    nmax = max(lens)
    if nmax:
        KV.store_rows(cache, torch.randn(B, H, nmax, D, generator=g), torch.randn(B, H, nmax, D, generator=g), lens)
    dev = {k: t.to(DEV) for k, t in cache.items()}
    cur = torch.tensor(lens, device=DEV, dtype=torch.int32)
    qkv_d = qkv.to(DEV)
    if nsplit == 0:
        nsplit = lib.b2_op_decode_attn_nsplit(B, H, Smax, _b2.KV_E4M3)
        assert 1 <= nsplit <= 32
    # the roped k row exactly as the bf16 kernel stores it (same RoPE code; torch's sin / cos can differ in the last bf16 bit)
    kc, vc = torch.zeros(B, H, Smax, D, device=DEV, dtype=BF), torch.zeros(B, H, Smax, D, device=DEV, dtype=BF)
    scratch = torch.zeros(lib.b2_op_decode_attn_scratch_bytes(B, H, nsplit), device=DEV, dtype=torch.uint8)
    out = torch.empty(B, H * D, device=DEV, dtype=BF)
    _b2.check(lib.b2_op_decode_attn(P(qkv_d), P(kc), P(vc), P(cur), P(out), P(scratch), B, H, Smax, nsplit, 10000.0,
                                    1 / math.sqrt(D), S()), "decode_attn")
    k_roped = torch.stack([kc[b, :, lens[b]] for b in range(B)]).cpu()
    out.zero_()
    for _ in range(2):  # the second launch runs on the counters the first one left behind
        _b2.check(lib.b2_op_decode_attn_e4m3(P(qkv_d), P(dev["k8"]), P(dev["v8"]), P(dev["ks"]), P(dev["vs"]), P(cur), P(out),
                                             P(scratch), B, H, Smax, nsplit, 10000.0, 1 / math.sqrt(D), S()), "decode_attn_e4m3")
    want = KV.decode_attn_call(qkv, cache, lens, H, k_roped=k_roped)   # appends to `cache` on the CPU
    torch.testing.assert_close(out.float().cpu(), want, rtol=2 ** -7, atol=5e-4)
    # the cache after the call: the appended row bit-exact, every other byte and scale untouched
    for name in ("k8", "v8"):
        assert torch.equal(u8(dev[name]).cpu(), u8(cache[name])), name
    for name in ("ks", "vs"):
        assert torch.equal(dev[name].cpu(), cache[name]), name
    assert int(scratch[: B * H * 4].view(torch.int32).abs().sum()) == 0


@pytest.mark.parametrize("nsplit", [1, 4, 0])   # 0: the engine's heuristic
@pytest.mark.parametrize("n", [0, 128, 711])
def test_decode_attn_e4m3_single_sample(n, nsplit):
    _attn_case(1, 32, [n], nsplit)


@pytest.mark.parametrize("nsplit", [1, 4, 0])
@pytest.mark.parametrize("B,H", [(12, 32), (64, 4)])
def test_decode_attn_e4m3_batched_ragged(B, H, nsplit):
    _attn_case(B, H, [LENGTHS[(b * 3 + 1) % len(LENGTHS)] for b in range(B)], nsplit)


def test_decode_attn_e4m3_rejects_bad_shapes():
    lib = _b2.load_library()
    t = torch.zeros(4096, device=DEV, dtype=torch.uint8)
    rc = lib.b2_op_decode_attn_e4m3(P(t), P(t), P(t), P(t), P(t), P(t), P(t), P(t), 1, 1, 7, 1, 10000.0, 1.0, S())
    assert rc == -1 and "multiple of 4" in _b2.last_error()
    assert lib.b2_op_decode_attn_nsplit(1, 32, 128, 2) == -1


# ---------------------------------------------------------------------------------------------- engine
@pytest.fixture(scope="module")
def tiny_engine():
    cfg = O.CONFIGS["tiny"]
    w = O.make_weights(cfg, seed=0)
    eng = make_engine(cfg, w, max_batch=4, max_seq=320, max_images=1)
    yield cfg, w, eng
    eng.close()


@pytest.mark.parametrize("B,S_,lens", [(2, 100, None), (2, 300, None), (3, 200, [200, 33, 150])])
def test_prefill_logits_do_not_depend_on_the_cache_format(tiny_engine, B, S_, lens):
    """Prefill attends over its own unquantised K / V: bit-identical logits, below and above the 512-row threshold where the
    QKV GEMM's fused RoPE epilogue replaces rope_kv_write as the producer of the roped K."""
    cfg, w, eng = tiny_engine
    g = torch.Generator().manual_seed(S_)
    embeds = (torch.randn(B, S_, cfg["hidden"], generator=g) * 0.5).to(BF).to(DEV)
    kvs = [eng.new_kv(B, 320), eng.new_kv(B, 320, dtype="e4m3")]
    assert [kv.dtype for kv in kvs] == ["bf16", "e4m3"]
    assert eng.lib.b2_kv_dtype(kvs[0].handle) == _b2.KV_BF16 and eng.lib.b2_kv_dtype(kvs[1].handle) == _b2.KV_E4M3
    a, b = (eng.prefill(kv, embeds, lens, _b2.LOGITS_LAST) for kv in kvs)
    assert torch.equal(a, b)
    assert kvs[1].lengths(B) == (lens or [S_] * B)
    assert kvs[1].nbytes * 512 == kvs[0].nbytes * 264            # max_seq is a multiple of 4: exactly 264 / 512
    [kv.close() for kv in kvs]


@pytest.mark.parametrize("fp8_weights", [False, True])
def test_engine_decode_logits_7b_shapes(fp8_weights):
    """7B layer shapes, 2 layers, B = 16, 8 teacher-forced steps on one engine with a bf16 and an e4m3 cache: within
    ENGINE_LOGIT_TOL (derived in tests/test_kv_fp8_oracle.py) of each other; with bf16 weights also within KERNEL_TOL of the
    oracle's restated step over the quantised cache."""
    cfg = O.make_config(hidden=4096, inter=11008, layers=2, heads=32, vit_layers=2)
    w = O.make_weights(cfg, seed=13)
    g = torch.Generator().manual_seed(6)
    B, S_, steps = 16, 64, 8
    embeds = (torch.randn(B, S_, 4096, generator=g) * 0.5).to(BF)
    eng = make_engine(cfg, w, max_batch=B, max_seq=128, max_images=1)
    if fp8_weights:
        eng.enable_fp8_decode()
    kv16, kv8 = eng.new_kv(B, 128), eng.new_kv(B, 128, dtype="e4m3")
    last = eng.prefill(kv16, embeds.to(DEV), None, _b2.LOGITS_LAST)
    assert torch.equal(last, eng.prefill(kv8, embeds.to(DEV), None, _b2.LOGITS_LAST))
    if not fp8_weights:
        _, caches = KV.prefill_cache(w, embeds.float(), cfg, Smax=128, last_only=True)
    tok = last.argmax(-1).to(torch.int32)
    lens = [S_] * B
    worst, worst_k = (0.0, 0.0), (0.0, 0.0)
    for _ in range(steps):
        l16, l8 = eng.decode_step(kv16, tok).cpu(), eng.decode_step(kv8, tok).cpu()
        worst = tuple(max(a, b) for a, b in zip(worst, rel_err(l8, l16)))
        if not fp8_weights:
            want = KV.decode_step(w, tok.cpu().long(), cfg, caches, lens)
            worst_k = tuple(max(a, b) for a, b in zip(worst_k, rel_err(l8, want)))
            lens = [n + 1 for n in lens]
        tok = l16.argmax(-1).to(torch.int32)              # teacher-forced with the bf16-cache tokens
    print(f"e4m3 vs bf16 cache (fp8 weights {fp8_weights}): max {worst[0]:.4f} mean {worst[1]:.4f} of std; "
          f"vs restated step: max {worst_k[0]:.4f} mean {worst_k[1]:.4f}")
    assert kv8.lengths(B) == [S_ + steps] * B
    # e4m3 weights re-quantise every activation row: a perturbation d of an element flips its code (a step of ~6 %) with
    # probability d / step, so the cache's error passes each W8A8 Linear amplified (RMS sqrt(d * step) > d): twice the bound
    slack = 2.0 if fp8_weights else 1.0
    assert worst[0] < slack * ENGINE_LOGIT_TOL[0] and worst[1] < slack * ENGINE_LOGIT_TOL[1], worst
    assert worst[1] > 0, "the e4m3 cache must change the decode numerics"
    assert worst_k[0] < KERNEL_TOL[0] and worst_k[1] < KERNEL_TOL[1], worst_k
    kv16.close(), kv8.close(), eng.close()


# ---------------------------------------------------------------------------------------------- strict greedy ids
@pytest.fixture(scope="module")
def conditioned():
    cfg = O.CONFIGS["tiny"]
    wc = O.condition_weights(O.make_weights(cfg, seed=0), cfg, seed=0)
    eng = make_engine(cfg, wc, max_batch=12, max_seq=128, max_images=1)
    yield cfg, wc, eng
    eng.close()


def _prompts(cfg, n, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(3, cfg["vocab"], (1, 20 + 3 * i), generator=g) for i in range(n)]


def _oracle_ids(wc, cfg, prompt, n):
    return KV.greedy_generate(wc, wc["model.embed_tokens.weight"].float()[prompt], cfg, n, Smax=128)[0].tolist()


@pytest.mark.parametrize("B", [1, 4, 12])
def test_greedy_ids_on_conditioned_weights(conditioned, B):
    """Plumbing: slots, offsets, scale arrays, token feedback. All three batch sizes take the multi-kernel step on an e4m3
    cache (GEMV graph at B <= 6, stream-K GEMM above); rows carry different prompts of one length."""
    cfg, wc, eng = conditioned
    g = torch.Generator().manual_seed(50 + B)
    prompts = torch.randint(3, cfg["vocab"], (B, 24), generator=g)
    want = KV.greedy_generate(wc, wc["model.embed_tokens.weight"].float()[prompts], cfg, 16, Smax=128).tolist()
    kv = eng.new_kv(B, 128, dtype="e4m3")
    launches = _b2.launch_count()
    lg = eng.prefill(kv, eng.splice(prompts.to(torch.int32).reshape(-1).to(DEV), None, B, 24), None, _b2.LOGITS_LAST)
    first = eng.argmax(lg)
    rest = eng.decode_greedy(kv, first, 15).cpu()
    got = torch.cat([first.cpu()[None], rest]).t().tolist()
    assert got == want
    assert _b2.launch_count() - launches > 15 * 5, "one launch per step would be the bf16-only megakernel"
    kv.close()


def test_continuous_batching_slots_on_an_e4m3_cache(conditioned):
    """Three slots, requests of different lengths; slot 0 is freed mid-run and refilled with a new request while slot 1 keeps
    decoding. Every request must reproduce the ids the oracle gets for it alone over a quantised cache."""
    cfg, wc, eng = conditioned
    pa, pb, pc = _prompts(cfg, 3, seed=77)
    want = {"a": _oracle_ids(wc, cfg, pa, 6), "b": _oracle_ids(wc, cfg, pb, 14), "c": _oracle_ids(wc, cfg, pc, 7)}
    kv = eng.new_kv(3, 128, dtype="e4m3")
    eng.batch_begin(kv, 3)
    got, state = {"a": [], "b": [], "c": []}, {"step": 0}

    def admit(slot, name, prompt):
        n = prompt.shape[1]
        lg = eng.prefill(kv, eng.splice(prompt.to(torch.int32).reshape(-1).to(DEV), None, 1, n), [n], _b2.LOGITS_LAST, slot0=slot)
        first = int(lg.argmax(-1))
        eng.batch_set_row(kv, slot, True, None, first)
        got[name].append(first)

    def step(rows):
        eng.stream_enqueue(kv, 1)
        toks = eng.stream_wait(kv, state["step"], 3)
        state["step"] += 1
        for slot, name in rows.items():
            got[name].append(int(toks[slot]))

    admit(0, "a", pa)
    admit(1, "b", pb)
    for _ in range(5):
        step({0: "a", 1: "b"})
    eng.batch_set_row(kv, 0, False)          # a is done: its slot goes back to the pool ...
    step({1: "b"})
    admit(0, "c", pc)                        # ... and is refilled while b keeps its context
    for _ in range(6):
        step({0: "c", 1: "b"})
    step({1: "b"})
    assert got == want, (got, want)
    kv.close()


# ---------------------------------------------------------------------------------------------- Python surface
class _ListStreamer:
    def __init__(self):
        self.values, self.ended = [], False

    def put(self, value):
        self.values.append(value)

    def end(self):
        self.ended = True


class _StopAfter:
    """Keyword-style criterion: stops once the new tokens end with `keyword` (a list of ids)."""

    def __init__(self, keyword, start_len):
        self.keyword, self.start_len = keyword, start_len

    def __call__(self, output_ids, scores, **kw):
        return output_ids[0, self.start_len:][-len(self.keyword):].tolist() == self.keyword


def test_generate_with_config_kv_dtype_e4m3(monkeypatch):
    monkeypatch.delenv("B2_KV_DTYPE", raising=False)
    cfg = O.CONFIGS["tiny"]
    wc = O.condition_weights(O.make_weights(cfg, seed=0), cfg, seed=0)
    model = make_model(cfg, wc, max_batch=2, max_seq=160, b2_kv_dtype="e4m3")
    ids, images = synth_inputs(cfg, B=1, Lt=12, seed=9)
    ids_d, img_d = ids.to(DEV), images.to(DEV)
    ref = model.generate(ids_d, images=img_d, do_sample=False, max_new_tokens=20, eos_token_id=[])
    assert ref.shape == (1, ids.shape[1] + 20) and torch.equal(ref[:, : ids.shape[1]].cpu(), ids)
    new = ref[0, ids.shape[1]:].tolist()
    keyword = new[8:10]
    hit = next(i for i in range(2, 21) if new[i - 2:i] == keyword)
    streamer = _ListStreamer()
    out = model.generate(inputs=ids_d, images=img_d, do_sample=False, max_new_tokens=20, streamer=streamer,
                         stopping_criteria=[_StopAfter(keyword, ids.shape[1])], use_cache=True, eos_token_id=[])
    assert out.shape == (1, ids.shape[1] + hit) and torch.equal(out.cpu(), ref[:, : out.shape[1]].cpu())
    assert streamer.ended and len(streamer.values) >= hit
    eng = model._ensure_engine()
    kv8 = model._pool.acquire()
    assert kv8.dtype == "e4m3"
    kv16 = eng.new_kv(kv8.max_batch, kv8.max_seq)
    assert 0 < kv8.nbytes <= 0.52 * kv16.nbytes
    kv16.close()
    model._pool.release(kv8)
    # forward(use_cache=True) leases follow the same knob
    fwd = model(input_ids=ids_d, images=img_d, use_cache=True)
    assert fwd.past_key_values.kv.dtype == "e4m3"
    model.invalidate_engine()


def test_env_knob_selects_the_format(monkeypatch):
    monkeypatch.setenv("B2_KV_DTYPE", "e4m3")
    cfg = O.CONFIGS["tiny"]
    model = make_model(cfg, O.make_weights(cfg, seed=0), max_batch=1, max_seq=96)
    ids, images = synth_inputs(cfg, B=1, Lt=12, seed=3)
    out = model.generate(ids.to(DEV), images=images.to(DEV), do_sample=False, max_new_tokens=4, eos_token_id=[])
    assert out.shape == (1, ids.shape[1] + 4)
    kv = model._pool.acquire()
    assert kv.dtype == "e4m3"
    model._pool.release(kv)
    model.invalidate_engine()


# ---------------------------------------------------------------------------------------------- errors
def test_unknown_dtype_raises_and_allocates_nothing(tiny_engine, monkeypatch):
    """The dtype is checked before anything is created: no handle comes back and no engine is built."""
    cfg, w, eng = tiny_engine
    h = ctypes.c_void_p()
    rc = eng.lib.b2_kv_create_ex(eng.handle, 2, 64, 7, ctypes.byref(h))
    assert rc == -1 and not h.value and "kv_dtype" in _b2.last_error()
    with pytest.raises(ValueError):
        eng.new_kv(2, 64, dtype="fp8")
    with pytest.raises(ValueError):
        eng.new_kv(2, 64, dtype="int8")
    monkeypatch.delenv("B2_KV_DTYPE", raising=False)
    model = make_model(cfg, w, max_batch=1, max_seq=96, b2_kv_dtype="e5m2")
    ids, images = synth_inputs(cfg, B=1, Lt=12, seed=3)
    with pytest.raises(ValueError, match="e5m2"):
        model.generate(ids.to(DEV), images=images.to(DEV), do_sample=False, max_new_tokens=2)
    assert model._engine is None
