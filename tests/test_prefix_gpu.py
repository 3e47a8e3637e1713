"""GPU: prefill of a chunk at an offset into a live KV cache (b2_prefill_at and its kernels) and conversation prefix reuse in
generate() (config.b2_prefix_cache): kernels against PyTorch / the oracles, the engine split at the image / text boundary
against an unsplit prefill and the oracle, strict greedy ids at full 7B depth, and the Python surface."""
import math
import os
import threading

import pytest
import torch

pytestmark = pytest.mark.gpu

from helpers import make_engine, make_model, rel_err, synth_inputs  # noqa: E402
from llava import _b2  # noqa: E402
from oracle import kv_fp8_oracle as KV  # noqa: E402
from oracle import kv_prefix_oracle as KP  # noqa: E402
from oracle import llava_oracle as O  # noqa: E402

DEV, BF, D = "cuda", torch.bfloat16, 128
P, S = _b2.ptr, _b2.stream_ptr
SPLIT_TOL = (0.02, 0.003)    # split vs unsplit prefill, as fused vs standalone RoPE (tests/test_model_gpu.py)
ORACLE_TOL = (0.05, 0.01)    # 2-3 layers against the fp32 oracle (tests/test_model_gpu.py)
KERNEL_TOL = (0.08, 0.015)   # e4m3 engine vs the restated step over the same quantised cache (tests/test_kv_fp8_gpu.py)


@pytest.fixture(scope="module", autouse=True)
def _init():
    _b2.init(0)


def i32(x):
    return torch.tensor(x, device=DEV, dtype=torch.int32)


# ------------------------------------------------------------------------------------------------------------- kernels
POS0 = [0, 1, 127, 128, 576, 1000]


@pytest.mark.parametrize("n", [1, 17, 128, 129, 300])
def test_flash_attn_kv_against_offset_causal_attention(n):
    lib = _b2.load_library()
    B, H = len(POS0), 32
    Smax = (max(POS0) + n + 15) // 16 * 16
    g = torch.Generator(device=DEV).manual_seed(n)
    q = torch.randn(B, n, H, D, device=DEV, generator=g).to(BF)
    kc = torch.randn(B, H, Smax, D, device=DEV, generator=g).to(BF)
    vc = torch.randn(B, H, Smax, D, device=DEV, generator=g).to(BF)
    lens = [n if b % 2 == 0 else max(1, n - 5) for b in range(B)]
    o = torch.zeros(B, n, H, D, device=DEV, dtype=BF)
    scale = 1 / math.sqrt(D)
    pos_d, lens_d = i32(POS0), i32(lens)   # kept alive until the kernel has run (a freed block is handed to the next tensor)
    _b2.check(lib.b2_op_flash_attn_kv(P(q), P(kc), P(vc), P(o), P(pos_d), P(lens_d), B, n, H, Smax, scale, S()), "flash_kv")
    for b in range(B):
        p, L = POS0[b], lens[b]
        qf = q[b, :L].float().transpose(0, 1)                          # [H, L, D]
        s = qf @ kc[b, :, :p + L].float().transpose(1, 2) * scale      # [H, L, p + L]
        mask = torch.arange(p + L, device=DEV)[None, :] <= (p + torch.arange(L, device=DEV))[:, None]
        want = torch.softmax(s.masked_fill(~mask, float("-inf")), -1) @ vc[b, :, :p + L].float()
        torch.testing.assert_close(o[b, :L].float().transpose(0, 1), want, rtol=2e-2, atol=2e-2)


@pytest.mark.parametrize("n", [17, 300])
def test_flash_attn_kv_at_position_zero_is_the_plain_kernel(n):
    lib = _b2.load_library()
    B, H, Smax = 3, 32, 512
    g = torch.Generator(device=DEV).manual_seed(100 + n)
    q, k, v = (torch.randn(B, n, H, D, device=DEV, generator=g).to(BF) for _ in range(3))
    lens = i32([n, max(1, n - 3), n])
    kc = torch.randn(B, H, Smax, D, device=DEV, generator=g).to(BF)
    vc = torch.randn(B, H, Smax, D, device=DEV, generator=g).to(BF)
    kc[:, :, :n], vc[:, :, :n] = k.transpose(1, 2), v.transpose(1, 2)
    o1, o2 = torch.zeros_like(q), torch.zeros_like(q)
    scale = 1 / math.sqrt(D)
    _b2.check(lib.b2_op_flash_attn(P(q), P(k), P(v), P(o1), P(lens), B, n, H, D, 1, scale, S()), "flash")
    zeros = i32([0] * B)
    _b2.check(lib.b2_op_flash_attn_kv(P(q), P(kc), P(vc), P(o2), P(zeros), P(lens), B, n, H, Smax, scale, S()), "flash_kv")
    for b in range(B):
        L = int(lens[b])
        assert torch.equal(o1[b, :L], o2[b, :L]), b


def test_rope_kv_write_at_equals_whole_sequence_rows():
    lib = _b2.load_library()
    B, H, n, Smax = 3, 32, 77, 1024
    starts = [0, 130, 600]
    L = max(starts) + n
    g = torch.Generator(device=DEV).manual_seed(7)
    qkv = torch.randn(B, L, 3 * H * D, device=DEV, generator=g).to(BF)
    whole = qkv.clone()
    kw, vw = (torch.zeros(B, H, Smax, D, device=DEV, dtype=BF) for _ in range(2))
    _b2.check(lib.b2_op_rope_kv_write(P(whole), P(kw), P(vw), B, L, H, D, Smax, 10000.0, S()), "rope")
    chunk = torch.stack([qkv[b, starts[b]:starts[b] + n] for b in range(B)]).contiguous()
    kc, vc = (torch.zeros(B, H, Smax, D, device=DEV, dtype=BF) for _ in range(2))
    starts_d = i32(starts)
    _b2.check(lib.b2_op_rope_kv_write_at(P(chunk), P(kc), P(vc), P(starts_d), B, n, H, D, Smax, 10000.0, S()), "rope_at")
    for b in range(B):
        r = slice(starts[b], starts[b] + n)
        assert torch.equal(kc[b, :, r], kw[b, :, r]) and torch.equal(vc[b, :, r], vw[b, :, r])
        assert torch.equal(chunk[b], whole[b, r])                                          # q rows, roped in place
        assert int(kc[b, :, :starts[b]].abs().sum()) == 0 and int(kc[b, :, starts[b] + n:].abs().sum()) == 0


def test_kv_dequantize_and_offset_quantize_bit_exact():
    lib = _b2.load_library()
    B, H, Smax, Sdst = 3, 32, 256, 200
    g = torch.Generator().manual_seed(9)
    cache = KV.empty_cache(B, H, Smax)
    KV.store_rows(cache, (torch.randn(B, H, Smax, D, generator=g) * 3).to(BF), torch.randn(B, H, Smax, D, generator=g).to(BF))
    dev = {k: t.to(DEV) for k, t in cache.items()}
    pos0 = [0, 64, 130]
    kd, vd = (torch.full((B, H, Sdst, D), 7.0, device=DEV, dtype=BF) for _ in range(2))
    pos_d = i32(pos0)
    _b2.check(lib.b2_op_kv_dequantize_e4m3(P(dev["k8"]), P(dev["v8"]), P(dev["ks"]), P(dev["vs"]), P(pos_d), P(kd), P(vd),
                                           B, H, Smax, Sdst, S()), "dequant")
    for b in range(B):
        k_ref, v_ref = KP.stage_prefix(cache, b, pos0[b])
        assert torch.equal(kd[b:b + 1, :, :pos0[b]].cpu(), k_ref) and torch.equal(vd[b:b + 1, :, :pos0[b]].cpu(), v_ref)
        assert bool((kd[b, :, pos0[b]:] == 7.0).all())                                       # nothing past the prefix
    # offset quantisation: slab rows [pos0, pos0 + len) -> the same cache rows; everything else keeps its bytes
    n, lens = 60, [60, 1, 45]
    slab_k = torch.randn(B, H, Sdst, D, device=DEV).to(BF)
    slab_v = torch.randn(B, H, Sdst, D, device=DEV).to(BF)
    before = {k: t.clone() for k, t in dev.items()}
    lens_d = i32(lens)
    _b2.check(lib.b2_op_kv_quantize_e4m3_at(P(slab_k), P(slab_v), P(dev["k8"]), P(dev["v8"]), P(dev["ks"]), P(dev["vs"]),
                                            P(pos_d), P(lens_d), B, n, Sdst, H, Smax, S()), "quant_at")
    for b in range(B):
        r = slice(pos0[b], pos0[b] + lens[b])
        for src, q8, sc in ((slab_k, "k8", "ks"), (slab_v, "v8", "vs")):
            q, s = KV.quantize_kv(src[b, :, r].cpu())
            assert torch.equal(dev[q8][b, :, r].view(torch.uint8).cpu(), q.view(torch.uint8))
            assert torch.equal(dev[sc][b, :, r].cpu(), s)
            keep = torch.ones(Smax, dtype=torch.bool, device=DEV)
            keep[r] = False
            assert torch.equal(dev[q8][b, :, keep].view(torch.uint8), before[q8][b, :, keep].view(torch.uint8))
            assert torch.equal(dev[sc][b, :, keep], before[sc][b, :, keep])


# ------------------------------------------------------------------------------------------------------------- engine
@pytest.fixture(scope="module")
def eng7():
    """7B layer shapes, 2 layers; one sequence of S = 704 per row (576 image-feature-sized rows + 128 text rows)."""
    torch.set_num_threads(min(32, os.cpu_count() or 1))
    cfg = O.make_config(layers=2, vit_layers=2)
    w = O.make_weights(cfg, seed=41)
    eng = make_engine(cfg, w, max_batch=3, max_seq=768, max_images=1)
    g = torch.Generator().manual_seed(42)
    E = (torch.randn(3, 704, cfg["hidden"], generator=g) * 0.5).to(BF)
    ref, _ = O.llama_forward(w, E.float(), cfg, last_only=True)
    yield cfg, w, eng, E, ref[:, -1]
    eng.close()


# first prefill: row 0 stops at the image / text boundary, row 1 runs past its later start (the chunk rewinds it), row 2
# holds 100 rows; "big" restarts row 2 at 0 (704-row chunk: B*S >= 512, the fused RoPE epilogue), "small" at 640 (128 rows)
CASES = {"big": [576, 650, 0], "small": [576, 650, 640]}
_E4M3_ORACLE = {}


@pytest.mark.parametrize("dtype", ["bf16", "e4m3"])
@pytest.mark.parametrize("case,fused", [("big", "1"), ("big", "0"), ("small", "1")])
def test_engine_split_prefill(eng7, monkeypatch, dtype, case, fused):
    cfg, w, eng, E, ref = eng7
    monkeypatch.setenv("B2_ROPE_FUSED", fused)
    starts = CASES[case]
    first_lens = [576, 700, 100 if case == "big" else 640]
    full_kv = eng.new_kv(3, 768, dtype=dtype)
    full = eng.prefill(full_kv, E.to(DEV), None, _b2.LOGITS_LAST).cpu()
    kv = eng.new_kv(3, 768, dtype=dtype)
    eng.prefill(kv, E[:, :700].to(DEV), first_lens, _b2.LOGITS_NONE)
    lens = [704 - s for s in starts]
    chunk = torch.zeros(3, max(lens), cfg["hidden"], dtype=BF)
    for b in range(3):
        chunk[b, :lens[b]] = E[b, starts[b]:]
    got = eng.prefill(kv, chunk.to(DEV), lens, _b2.LOGITS_LAST, start=starts).cpu()
    assert kv.lengths(3) == [704] * 3
    assert torch.isfinite(got).all()
    mx, mn = rel_err(got, full)
    print(f"{dtype} {case} fused={fused}: split vs unsplit max {mx:.4f} mean {mn:.4f}")
    if dtype == "bf16":
        assert mx <= SPLIT_TOL[0] and mn <= SPLIT_TOL[1], (mx, mn)
        for name, x in (("split", got), ("unsplit", full)):
            e = rel_err(x, ref)
            assert e[0] <= ORACLE_TOL[0] and e[1] <= ORACLE_TOL[1], (name, e)
    else:
        if case not in _E4M3_ORACLE:
            _, caches = KV.prefill_cache(w, E[:, :700].float(), cfg, Smax=768, seq_lens=first_lens)
            _E4M3_ORACLE[case] = KP.prefill_chunk(w, chunk.float(), cfg, caches, starts, seq_lens=lens, last_only=True)
        e = rel_err(got, _E4M3_ORACLE[case])
        print(f"  vs restated chunk prefill max {e[0]:.4f} mean {e[1]:.4f}")
        assert e[0] <= KERNEL_TOL[0] and e[1] <= KERNEL_TOL[1], e
    kv.close(), full_kv.close()


def test_prefill_at_argument_checks(eng7):
    cfg, w, eng, E, ref = eng7
    kv = eng.new_kv(3, 768)
    x = E[:1, :10].to(DEV)
    with pytest.raises(ValueError, match="current length"):
        eng.prefill(kv, x, None, _b2.LOGITS_LAST, start=[5])             # the slot is empty
    eng.prefill(kv, E[:1, :700].to(DEV), None, _b2.LOGITS_NONE)
    with pytest.raises(ValueError, match="max_seq"):
        eng.prefill(kv, E[:1, :100].to(DEV), None, _b2.LOGITS_LAST, start=[700])
    eng.prefill(kv, x, None, _b2.LOGITS_LAST, start=[700])
    assert kv.lengths(1) == [710]
    kv.close()


def test_strict_greedy_ids_after_a_continued_prefill_7b_full_depth():
    """32 layers of 7B on the well-conditioned weight set: the ids after prefill(20) + rewind to 10 + prefill_at(14) equal those
    after one prefill(24), on every decode path (megakernel B=1, GEMV graph B=4, stream-K GEMM B=12)."""
    cfg = O.CONFIGS["llava-1.5-7b"]
    g = torch.Generator(device=DEV).manual_seed(0)
    w = {}
    for key, shape, kind in O.weight_shapes(cfg):
        t = torch.randn(*shape, generator=g, device=DEV) * O.init_std(kind, shape)
        w[key] = (t + 1.0 if kind == "g" else t).to(BF)
    w = O.condition_weights(w, cfg, seed=0)
    eng = make_engine(cfg, w, max_batch=12, max_seq=128, max_images=1)
    del w
    prompt = torch.randint(3, cfg["vocab"], (1, 24), generator=torch.Generator().manual_seed(5))
    for B in (1, 4, 12):
        emb = eng.splice(prompt.repeat(B, 1).to(torch.int32).reshape(-1).to(DEV), None, B, 24)
        ids = []
        for split in (False, True):
            kv = eng.new_kv(B, 128)
            if split:
                eng.prefill(kv, emb[:, :20], None, _b2.LOGITS_NONE)
                lg = eng.prefill(kv, emb[:, 10:], None, _b2.LOGITS_LAST, start=[10] * B)
            else:
                lg = eng.prefill(kv, emb, None, _b2.LOGITS_LAST)
            first = eng.argmax(lg)
            rest = eng.decode_greedy(kv, first, 15).cpu()
            ids.append(torch.cat([first.cpu()[None], rest]).t().tolist())
            kv.close()
        assert ids[0] == ids[1], (B, ids)
        assert all(r == ids[0][0] for r in ids[0])
    eng.close()


# ------------------------------------------------------------------------------------------------------------- Python
@pytest.fixture(scope="module")
def tiny():
    cfg = O.CONFIGS["tiny"]
    return cfg, O.condition_weights(O.make_weights(cfg, seed=0), cfg, seed=0)


def test_forward_continuation_against_oracle(tiny):
    cfg = O.CONFIGS["tiny"]
    w = O.make_weights(cfg, seed=2)
    model = make_model(cfg, w, max_batch=2, max_seq=256)
    ids1, img1 = synth_inputs(cfg, B=1, Lt=12, seed=3)
    _, img2 = synth_inputs(cfg, B=1, Lt=12, seed=4)
    g = torch.Generator().manual_seed(5)
    ids2 = torch.randint(3, cfg["vocab"], (1, 6), generator=g)
    ids3 = torch.randint(3, cfg["vocab"], (1, 5), generator=g)
    ids3[0, 2] = O.IMAGE_TOKEN_INDEX
    out1 = model(input_ids=ids1.to(DEV), images=img1.to(DEV), use_cache=True)
    lease = out1.past_key_values
    out2 = model(input_ids=ids2.to(DEV), past_key_values=lease)
    assert out2.past_key_values is lease and out2.logits.shape == (1, 6, cfg["vocab"])
    out3 = model(input_ids=ids3.to(DEV), past_key_values=lease, images=img2.to(DEV))
    Pn = (cfg["image_size"] // cfg["patch_size"]) ** 2
    assert out3.logits.shape == (1, 4 + Pn, cfg["vocab"])
    full_ids = torch.cat([ids1, ids2, ids3], dim=1)
    embeds, _, _, _ = O.prepare_multimodal(w, full_ids, torch.cat([img1, img2]).to(BF).float(), cfg)
    ref, _ = O.llama_forward(w, embeds, cfg)
    n1 = out1.logits.shape[1]
    for got, want in ((out2.logits, ref[:, n1:n1 + 6]), (out3.logits, ref[:, n1 + 6:])):
        e = rel_err(got, want)
        assert e[0] <= ORACLE_TOL[0] and e[1] <= ORACLE_TOL[1], e
    assert lease.get_seq_length() == ref.shape[1]
    with pytest.raises(NotImplementedError):
        model(input_ids=ids2.to(DEV), past_key_values=lease, attention_mask=torch.tensor([[1, 1, 1, 0, 1, 1]], device=DEV))
    model(input_ids=ids1.to(DEV), images=img1.to(DEV), use_cache=True)
    model(input_ids=ids1.to(DEV), images=img1.to(DEV), use_cache=True)   # recycles the first lease
    with pytest.raises(RuntimeError, match="recycled"):
        model(input_ids=ids2.to(DEV), past_key_values=lease)
    model.invalidate_engine()


def _conversation(model, ids, image, seed, turns=3, sample=False, edit=None):
    """A chat: every turn sends the whole history (previous prompt + answer + a new question) with the same image."""
    g = torch.Generator().manual_seed(seed)
    outs, prompt = [], ids
    for t in range(turns):
        if t:
            q = torch.randint(3, model.config.vocab_size, (1, 7), generator=g)
            prompt = torch.cat([outs[-1], q], dim=1)
            if edit is not None:
                prompt, image = edit(t, prompt, image)
        torch.manual_seed(1000 * seed + t)
        kw = dict(do_sample=True, temperature=0.7, top_p=0.9) if sample else dict(do_sample=False)
        outs.append(model.generate(prompt.to(DEV), images=image.to(DEV), max_new_tokens=9, eos_token_id=[], **kw).cpu())
    return outs


@pytest.mark.parametrize("kv_dtype", ["bf16", "e4m3"])
@pytest.mark.parametrize("sample", [False, True])
def test_generate_conversation_reuse_equals_fresh(tiny, monkeypatch, kv_dtype, sample):
    monkeypatch.delenv("B2_PREFIX_CACHE", raising=False)
    cfg, wc = tiny
    model = make_model(cfg, wc, max_batch=1, max_seq=256, b2_kv_dtype=kv_dtype)
    ids, image = synth_inputs(cfg, B=1, Lt=12, seed=11)
    model.config.b2_prefix_cache = False
    off = _conversation(model, ids, image, seed=1, sample=sample)
    pool = model._pool
    assert pool.reused_positions == 0 and pool.skipped_encodes == 0
    model.config.b2_prefix_cache = True
    counters = []
    g = torch.Generator().manual_seed(1)
    outs, prompt = [], ids
    for t in range(3):
        if t:
            prompt = torch.cat([outs[-1], torch.randint(3, cfg["vocab"], (1, 7), generator=g)], dim=1)
        torch.manual_seed(1000 + t)
        kw = dict(do_sample=True, temperature=0.7, top_p=0.9) if sample else dict(do_sample=False)
        outs.append(model.generate(prompt.to(DEV), images=image.to(DEV), max_new_tokens=9, eos_token_id=[], **kw).cpu())
        counters.append((pool.reused_positions, pool.skipped_encodes))
    for a, b in zip(off, outs):
        assert torch.equal(a, b)
    Pn = (cfg["image_size"] // cfg["patch_size"]) ** 2
    # turn 2 reuses turn 1's spliced prompt and its answer but the last token; turn 3 likewise on top of turn 2
    assert counters[0] == (0, 0)
    assert counters[1] == (12 - 1 + Pn + 8, 1)
    assert counters[2] == (counters[1][0] + 12 - 1 + Pn + 9 + 7 + 8, 2)
    model.invalidate_engine()
    assert model._pool is None


def test_changed_image_or_history_reuses_only_the_true_prefix(tiny, monkeypatch):
    monkeypatch.delenv("B2_PREFIX_CACHE", raising=False)
    cfg, wc = tiny
    model = make_model(cfg, wc, max_batch=1, max_seq=256, b2_prefix_cache=True)
    ids, image = synth_inputs(cfg, B=1, Lt=12, seed=12)
    _, other = synth_inputs(cfg, B=1, Lt=12, seed=13)
    first = model.generate(ids.to(DEV), images=image.to(DEV), do_sample=False, max_new_tokens=6, eos_token_id=[]).cpu()
    nxt = torch.cat([first, torch.tensor([[5, 6, 7]])], dim=1)
    pool = model._pool
    r0 = pool.reused_positions
    model.generate(nxt.to(DEV), images=other.to(DEV), do_sample=False, max_new_tokens=4, eos_token_id=[])
    assert pool.reused_positions - r0 == 5 and pool.skipped_encodes == 0       # the 5 tokens in front of the image
    edited = nxt.clone()
    edited[0, 3] = 4 if int(edited[0, 3]) != 4 else 9
    r1 = pool.reused_positions
    out = model.generate(edited.to(DEV), images=image.to(DEV), do_sample=False, max_new_tokens=4, eos_token_id=[]).cpu()
    assert pool.reused_positions - r1 == 3 and pool.skipped_encodes == 0
    model.config.b2_prefix_cache = False
    fresh = model.generate(edited.to(DEV), images=image.to(DEV), do_sample=False, max_new_tokens=4, eos_token_id=[]).cpu()
    assert torch.equal(out, fresh)
    model.invalidate_engine()


def test_four_threads_four_conversations_give_the_serial_results(tiny, monkeypatch):
    monkeypatch.delenv("B2_PREFIX_CACHE", raising=False)
    cfg, wc = tiny
    model = make_model(cfg, wc, max_batch=1, max_seq=256)
    convs = [synth_inputs(cfg, B=1, Lt=12, seed=20 + i) for i in range(4)]
    model.config.b2_prefix_cache = False
    serial = [_conversation(model, ids, img, seed=30 + i, turns=2) for i, (ids, img) in enumerate(convs)]
    model.config.b2_prefix_cache = True
    got, errors = [None] * 4, []

    def run(i):
        try:
            got[i] = _conversation(model, convs[i][0], convs[i][1], seed=30 + i, turns=2)
        except Exception as e:  # pragma: no cover - reported below
            errors.append(e)

    threads = [threading.Thread(target=run, args=(i,)) for i in range(4)]
    [t.start() for t in threads]
    [t.join() for t in threads]
    assert not errors, errors
    for a, b in zip(serial, got):
        assert all(torch.equal(x, y) for x, y in zip(a, b))
    assert model._pool.reused_positions > 0 and model._pool.skipped_encodes > 0
    model.invalidate_engine()


def test_continuous_batching_keeps_the_prefix_cache_out(tiny, monkeypatch):
    monkeypatch.delenv("B2_PREFIX_CACHE", raising=False)
    cfg, wc = tiny
    model = make_model(cfg, wc, max_batch=2, max_seq=256, b2_continuous_batching=2)
    ids, image = synth_inputs(cfg, B=1, Lt=12, seed=40)
    model.config.b2_prefix_cache = False
    off = _conversation(model, ids, image, seed=41, turns=2)
    model.config.b2_prefix_cache = True
    on = _conversation(model, ids, image, seed=41, turns=2)
    assert all(torch.equal(a, b) for a, b in zip(off, on))
    assert model._pool.reused_positions == 0 and model._pool.skipped_encodes == 0
    model.invalidate_engine()
