"""CPU: the matching rule of conversation prefix reuse (llava/_b2/prefix.py) and the restated prefill of a chunk appended to
an e4m3 cache (oracle/kv_prefix_oracle.py)."""
import numpy as np
import torch

from llava._b2 import INT32_MIN
from llava._b2 import prefix as PX
from oracle import kv_fp8_oracle as KV
from oracle import kv_prefix_oracle as KP
from oracle import llava_oracle as O

P = 4  # feature rows per image in these cases


def _img(seed, shape=(3, 8, 8), dtype=torch.float32):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)).to(dtype)


def test_placeholders_match_only_on_equal_pixels():
    a = _img(0)
    cached = [1, 2, a, 3, 4]
    assert PX.match_rows(cached, [1, 2, a.clone(), 3, 4, 9], P) == 2 + P + 2      # equal pixels, a different object
    assert PX.match_rows(cached, [1, 2, _img(1), 3, 4], P) == 2                    # other pixels: stop at the placeholder
    assert PX.match_rows(cached, [1, 2, a.to(torch.float16), 3], P) == 2          # same values, other dtype
    assert PX.match_rows(cached, [1, 2, a[None], 3], P) == 2                      # other shape
    assert PX.match_rows(cached, [1, 2, 7, 3], P) == 2                             # token against placeholder
    two = torch.stack([a, _img(2)])                                                # one slot holding two images
    assert PX.item_rows(two, P) == 2 * P
    assert PX.match_rows([1, two, 5], [1, two.clone(), 5, 6], P) == 1 + 2 * P + 1


def test_divergence_mid_text():
    a = _img(3)
    cached = [1, a, 10, 11, 12, 13]
    assert PX.match_rows(cached, [1, a, 10, 11, 99, 13, 14], P) == 1 + P + 2
    assert PX.match_rows(cached, [5, a, 10], P) == 0


def test_strict_prefix_is_capped_one_below_the_new_length():
    a = _img(4)
    cached = [1, a, 10, 11, 12, 13, 14]
    new = [1, a, 10, 11]                                  # "regenerate": the prompt is a prefix of what the cache holds
    assert PX.match_rows(cached, new, P) == 1 + P + 2
    assert PX.reusable_rows(cached, new, P) == 1 + P + 2 - 1
    assert PX.reusable_rows(cached, list(cached), P) == 1 + P + 5 - 1
    assert PX.reusable_rows(cached, [1, a], P) == P       # the cap can fall inside an image: its rows are spliced again


def test_valid_rows_after_eos_and_keyword_stops():
    prompt = [1, _img(5), 10]
    eos = 2
    # eos stop: the eos token was returned but never fed; rows of steps queued past it are not part of the record
    assert PX.record_after_generation(prompt, [7, 8, eos])[3:] == [7, 8]
    # keyword stop: the answer ends with the keyword's last token, which was not fed either
    assert PX.record_after_generation(prompt, torch.tensor([7, 8, 30, 31]).tolist())[3:] == [7, 8, 30]
    assert PX.record_after_generation(prompt, [7]) == prompt
    # the next turn's prompt repeats the answer: reuse reaches the end of the valid rows, not beyond
    rec = PX.record_after_generation(prompt, [7, 8, eos])
    nxt = prompt + [7, 8, eos, 40, 41]
    assert PX.reusable_rows(rec, nxt, P) == 1 + P + 1 + 2


def test_select_prefers_longest_match_then_least_recently_used():
    a, b = _img(6), _img(7)
    recs = [[1, a, 10], None, [1, b, 10, 11, 12], [1, b, 10]]
    assert PX.select(recs, [1, b, 10, 11, 12, 13], P) == (2, 1 + P + 3)
    assert PX.select(recs, [1, a, 10, 20], P) == (0, 1 + P + 1)
    assert PX.select(recs, [9, 9], P) == (0, 0)                  # miss: the least recently released cache is evicted
    assert PX.select([None, None], [1, 2], P) == (0, 0)


def test_chunk_source_index_shifts_feature_rows_of_skipped_images():
    src = np.array([5, -1, -2, -3, -4, 6, -5, -6, -7, -8, 7, INT32_MIN], dtype=np.int64)
    out = PX.chunk_source_index(src, 5, 4, INT32_MIN)            # the first image (4 rows) lies inside the reused rows
    assert out.tolist() == [6, -1, -2, -3, -4, 7, INT32_MIN]


# ------------------------------------------------------------------------------------------------ oracle
CFG = O.make_config(hidden=256, inter=512, layers=2, heads=2, vocab=1024, vit_hidden=256, vit_inter=512, vit_layers=3,
                    vit_heads=4, image_size=56)


def test_prefill_chunk_at_zero_is_prefill_cache():
    w = O.make_weights(CFG, seed=3)
    g = torch.Generator().manual_seed(4)
    embeds = (torch.randn(2, 40, CFG["hidden"], generator=g) * 0.5).to(torch.bfloat16).float()
    want, want_caches = KV.prefill_cache(w, embeds, CFG, Smax=64)
    caches = [KV.empty_cache(2, CFG["heads"], 64) for _ in range(CFG["layers"])]
    got = KP.prefill_chunk(w, embeds, CFG, caches, [0, 0])
    assert torch.equal(got, want)
    for c, wc in zip(caches, want_caches):
        for k in ("k8", "v8"):
            assert torch.equal(c[k].view(torch.uint8), wc[k].view(torch.uint8))
        for k in ("ks", "vs"):
            assert torch.equal(c[k], wc[k])


def test_prefill_chunk_error_against_bf16_oracle():
    """A chunk over a stored e4m3 prefix: its attention sees the prefix with the e4m3 rounding, so its logits move away from
    the bf16-cache continuation by no more than the attention error the e4m3 cache is specified with (5.1 % of the RMS)
    carried through the rest of the layer; the chunk's own rows are stored as a whole-sequence prefill would store them."""
    w = O.make_weights(CFG, seed=5)
    g = torch.Generator().manual_seed(6)
    S, p = 48, 30
    embeds = (torch.randn(1, S, CFG["hidden"], generator=g) * 0.5).to(torch.bfloat16).float()
    ref, _ = O.llama_forward(w, embeds, CFG)
    _, caches = KV.prefill_cache(w, embeds[:, :p], CFG, Smax=64)
    got = KP.prefill_chunk(w, embeds[:, p:], CFG, caches, [p])
    want = ref[:, p:]
    rel = float((got - want).pow(2).mean().sqrt() / want.pow(2).mean().sqrt())
    assert 1e-5 < rel < KV.expected_attention_error(), rel
    _, full = KV.prefill_cache(w, embeds, CFG, Smax=64)
    # stored chunk rows: each is within one e4m3 step of the whole-sequence prefill's (its K / V came through a perturbed prefix)
    for c, f in zip(caches, full):
        d = (KV.dequantize_kv(c["v8"][:, :, :S], c["vs"][:, :, :S]) - KV.dequantize_kv(f["v8"][:, :, :S], f["vs"][:, :, :S]))
        assert float(d[:, :, :p].abs().max()) == 0.0
        assert float(d.pow(2).mean().sqrt()) < 0.1 * float(KV.dequantize_kv(f["v8"], f["vs"]).pow(2).mean().sqrt())
