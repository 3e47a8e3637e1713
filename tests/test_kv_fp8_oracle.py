"""CPU: pins the e4m3 KV-cache oracle (oracle/kv_fp8_oracle.py) and derives the tolerances tests/test_kv_fp8_gpu.py uses."""
import math

import torch

from oracle import kv_fp8_oracle as KV
from oracle import llava_oracle as O

BF = torch.bfloat16

# Engine tolerance, e4m3 cache vs bf16 cache, decode logits as a share of the logit std (max, mean). The oracle pair below
# (2 layers, unit-gain random weights, 6 steps) measures 0.058 / 0.010; the bound leaves room for the bf16 rounding noise of
# the two engines being compared (0.05 / 0.01 each, tests/test_model_gpu.py) on top of it.
ENGINE_LOGIT_TOL = (0.25, 0.05)


def test_row_quantiser_round_trip_at_head_width():
    g = torch.Generator().manual_seed(0)
    x = (torch.randn(4, 32, 77, KV.D, generator=g) * torch.logspace(-3, 2, 77)[:, None]).to(BF)
    x[0, 0, 0] = 0                                                    # zero row: scale 1, codes 0
    x[0, 0, 1, 1:] = 0                                                # one element: it is the amax, stored exactly
    q, s = KV.quantize_kv(x)
    assert q.dtype == torch.float8_e4m3fn and s.dtype == torch.float32 and s.shape == x.shape[:-1]
    assert float(s[0, 0, 0]) == 1.0 and int(q[0, 0, 0].view(torch.uint8).max()) == 0
    amax = x.float().abs().amax(-1)
    assert torch.equal(s[amax > 0], (amax / 448.0)[amax > 0])
    deq = KV.dequantize_kv(q, s)
    assert float(deq[0, 0, 1, 0]) == float(x[0, 0, 1, 0])
    err = (deq - x.float()).abs()
    bound = torch.maximum(KV.ROW_REL_ERROR_MAX * x.float().abs(), KV.ROW_ABS_ERROR_FLOOR * amax[..., None]) * (1 + 1e-6)
    assert bool((err <= bound).all()), float((err / bound.clamp_min(1e-30)).max())
    rel_rms = float((err.pow(2).sum(-1) / x.float().pow(2).sum(-1).clamp_min(1e-30)).sqrt().mean())
    assert 0.02 < rel_rms < 2.0 ** -4 / math.sqrt(3) * 1.15, rel_rms  # ~3.6 % of the row's RMS


def _bf16_attention(q, K, V):
    s = torch.einsum("bhd,bhnd->bhn", q.float(), K.float()) * KV.D ** -0.5
    return torch.einsum("bhn,bhnd->bhd", torch.softmax(s, -1), V.float())


def test_attention_over_quantised_cache_close_to_bf16_cache():
    g = torch.Generator().manual_seed(1)
    B, H = 3, 4
    for n in (1, 7, 128, 703):
        K, V = torch.randn(B, H, n + 1, KV.D, generator=g).to(BF), torch.randn(B, H, n + 1, KV.D, generator=g).to(BF)
        q = torch.randn(B, H, KV.D, generator=g).to(BF)
        cache = KV.empty_cache(B, H, n + 8)
        KV.store_rows(cache, K[:, :, :n], V[:, :, :n])
        got = KV.decode_attention(q, K[:, :, n], V[:, :, n], cache, [n] * B)
        want = _bf16_attention(q, K, V)
        rel = float((got - want).pow(2).mean().sqrt() / want.pow(2).mean().sqrt())
        assert rel < 1.3 * KV.expected_attention_error(), (n, rel)
        # the appended row is stored, and attended over, quantised
        qk, sk = KV.quantize_kv(K[:, :, n])
        assert torch.equal(cache["k8"][:, :, n].view(torch.uint8), qk.view(torch.uint8)) and torch.equal(cache["ks"][:, :, n], sk)
        assert int(cache["k8"][:, :, n + 1:].view(torch.uint8).max()) == 0


def test_decode_attn_call_ropes_then_quantises():
    g = torch.Generator().manual_seed(2)
    B, H, lens = 2, 2, [5, 0]
    qkv = torch.randn(B, 3 * H * KV.D, generator=g).to(BF)
    cache = KV.empty_cache(B, H, 8)
    KV.store_rows(cache, torch.randn(B, H, 5, KV.D, generator=g), torch.randn(B, H, 5, KV.D, generator=g), seq_lens=lens)
    out = KV.decode_attn_call(qkv, cache, lens, H)
    v3 = qkv.view(B, 3, H, KV.D)
    k = KV.rope_bf16(v3[:, 1], torch.tensor(lens))
    for b in range(B):
        qk, sk = KV.quantize_kv(k[b])
        assert torch.equal(cache["k8"][b, :, lens[b]].view(torch.uint8), qk.view(torch.uint8))
        assert torch.equal(cache["ks"][b, :, lens[b]], sk)
    # a single key: softmax is 1, the output is the dequantised new v row
    qv, sv = KV.quantize_kv(v3[1, 2])
    torch.testing.assert_close(out[1].view(H, KV.D), KV.dequantize_kv(qv, sv), rtol=1e-6, atol=0)
    assert torch.equal(KV.rope_bf16(v3[:, 1], torch.tensor([0, 0]))[1], v3[1, 1])  # position 0 is the identity


def test_engine_level_step_and_tolerance():
    """Prefill logits do not depend on the cache format; decode logits over the quantised cache stay within
    ENGINE_LOGIT_TOL of the bf16-cache oracle (what the GPU engine test then asserts between the two engines)."""
    cfg = O.make_config(hidden=256, inter=512, layers=2, heads=2, vocab=1024, vit_hidden=256, vit_inter=512, vit_layers=3,
                        vit_heads=4, image_size=56)
    w = O.make_weights(cfg, seed=3)
    g = torch.Generator().manual_seed(4)
    B, S = 4, 48
    embeds = (torch.randn(B, S, cfg["hidden"], generator=g) * 0.5).to(BF).float()
    logits, caches = KV.prefill_cache(w, embeds, cfg, Smax=64)
    ref, kv = O.llama_forward(w, embeds, cfg)
    assert torch.equal(logits, ref)
    tok = logits[:, -1].argmax(-1)
    lens = [S] * B
    worst = (0.0, 0.0)
    for _ in range(6):
        got = KV.decode_step(w, tok, cfg, caches, lens)
        e = w["model.embed_tokens.weight"][tok][:, None]
        want, kv = O.llama_forward(w, e, cfg, kv=kv, last_only=True)
        want = want[:, -1]
        d = (got - want).abs() / float(want.std())
        worst = (max(worst[0], float(d.max())), max(worst[1], float(d.mean())))
        tok, lens = want.argmax(-1), [n + 1 for n in lens]
    assert worst[0] < ENGINE_LOGIT_TOL[0] and worst[1] < ENGINE_LOGIT_TOL[1], worst
    assert worst[1] > 1e-4, "the quantised cache must actually be in the path"
    assert int(caches[0]["k8"][:, :, S + 5].view(torch.uint8).max()) > 0 and float(caches[1]["vs"][:, :, S + 5].min()) > 0


def test_bytes_per_token():
    assert KV.BYTES_PER_HEAD_TOKEN == 264 and KV.BYTES_PER_HEAD_TOKEN_BF16 == 512
    assert 32 * 32 * KV.BYTES_PER_HEAD_TOKEN == 270336 and 32 * 32 * KV.BYTES_PER_HEAD_TOKEN_BF16 == 524288  # 7B, per token and sample
