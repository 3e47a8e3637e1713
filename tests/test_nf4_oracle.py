"""CPU: the NF4 oracle (oracle/nf4_oracle.py) and the load_4bit argument handling of the Python surface."""
import json

import pytest
import torch

from oracle import llava_oracle as O
from oracle import nf4_oracle as Q

# the largest gap between neighbouring table entries is at the negative end, -1 .. -0.6961928 (the positive end's
# 1 - 0.7229568 is smaller): half of it bounds the error of the nearest-entry rule
LARGEST_GAP = 1.0 - 0.6961928


def test_table_equals_the_normal_map_construction():
    assert Q.NF4_TABLE.shape == (16,) and float(Q.NF4_TABLE[7]) == 0.0
    assert float((Q.normal_map() - Q.NF4_TABLE).abs().max()) <= 1e-7
    gaps = Q.NF4_TABLE[1:] - Q.NF4_TABLE[:-1]
    assert float(gaps.max()) == pytest.approx(LARGEST_GAP, abs=1e-7)


def _nearest_lower_on_tie(x):
    """Brute force: the nearest table entry, ties (x exactly on an fp32 midpoint) to the lower code."""
    mids = Q.midpoints()
    return (x[..., None] > mids).sum(-1)


def test_quantiser_rule_random_blocks():
    g = torch.Generator().manual_seed(0)
    w = (torch.randn(64, 512, generator=g) * torch.rand(64, 1, generator=g) * 3).to(torch.bfloat16).float()
    q, a = Q.quantize_nf4(w)
    assert torch.equal(a, w.view(64, 8, 64).abs().amax(-1))
    x = w.view(64, 8, 64) / a[..., None]
    d = (x[..., None] - Q.NF4_TABLE).abs()
    best = d.min(-1, keepdim=True).values
    # the code is a nearest entry, and where two entries are equally near, the lower one
    first_nearest = (d == best).float().argmax(-1)
    assert torch.equal(q.view(64, 8, 64).long(), first_nearest)
    assert torch.equal(q.view(64, 8, 64).long(), _nearest_lower_on_tie(x))
    assert int(q.max()) == 15 and int(q.min()) == 0


def test_all_zero_block_and_values_on_midpoints():
    w = torch.zeros(2, 128)
    w[1, 64] = 1.0  # absmax 1: x equals w exactly
    mids = Q.midpoints()
    w[1, 65:80] = mids
    w[1, 80:95] = torch.nextafter(mids, torch.full_like(mids, 2.0))  # just above: the upper code
    q, a = Q.quantize_nf4(w)
    assert float(a[0, 0]) == 0.0 and float(a[0, 1]) == 0.0 and float(a[1, 1]) == 1.0
    assert bool((q[0] == 7).all()) and bool((q[1, :64] == 7).all())
    assert q[1, 65:80].tolist() == list(range(15))       # on the midpoint: the lower code
    assert q[1, 80:95].tolist() == list(range(1, 16))
    assert bool((Q.dequantize_nf4(q, a)[0] == 0).all())


def test_invariant_to_scale_and_sign():
    g = torch.Generator().manual_seed(1)
    w = torch.randn(16, 256, generator=g).to(torch.bfloat16).float()
    q, a = Q.quantize_nf4(w)
    for s in (2.0 ** -9, 0.5, 8.0, 2.0 ** 20):  # exact scalings: x = w / absmax does not change
        qs, as_ = Q.quantize_nf4(w * s)
        assert torch.equal(qs, q) and torch.equal(as_, a * s)
    qn, an = Q.quantize_nf4(-w)
    assert torch.equal(an, a)
    x = -w.view(16, 4, 64) / a[..., None]
    assert torch.equal(qn.view(16, 4, 64).long(), _nearest_lower_on_tie(x))


def test_round_trip_error_bound():
    g = torch.Generator().manual_seed(2)
    w = (torch.randn(32, 1024, generator=g) * 0.02).to(torch.bfloat16).float()
    q, a = Q.quantize_nf4(w)
    wh = Q.dequantize_nf4(q, a).float()
    amax = a.repeat_interleave(64, dim=1)
    bound = LARGEST_GAP / 2 * amax + 2.0 ** -8 * wh.abs()  # nearest-entry error + the bf16 rounding of w_hat
    assert bool(((wh - w).abs() <= bound).all())
    exact = Q.NF4_TABLE[q.long()] * amax
    assert torch.equal(wh, exact.to(torch.bfloat16).float())


@pytest.mark.parametrize("order", ["canonical", "gemv"])
def test_pack_and_unpack_are_inverses(order):
    g = torch.Generator().manual_seed(3)
    q = torch.randint(0, 16, (24, 768), generator=g, dtype=torch.uint8)
    p = Q.pack_nf4(q, order)
    assert p.shape == (24, 384) and torch.equal(Q.unpack_nf4(p, order), q)
    if order == "canonical":
        assert int(p[0, 0]) == int(q[0, 0]) << 4 | int(q[0, 1])  # element 2j in the high nibble
    else:  # word 8t + m of a 128-element chunk holds elements 16m + 4t .. + 3
        words = p.view(24, 6, 32, 2)
        for t, m in ((1, 2), (3, 7)):
            w16 = words[0, 1, 8 * t + m]
            k = 128 + 16 * m + 4 * t
            assert int(w16[0]) == int(q[0, k]) << 4 | int(q[0, k + 1]) and int(w16[1]) == int(q[0, k + 2]) << 4 | int(q[0, k + 3])


def _lm_weights(cfg, seed):
    g = torch.Generator().manual_seed(seed)
    w = {}
    for key, shape, kind in O.weight_shapes(dict(cfg, vit_layers=0)):
        if key.startswith(O.VT):
            continue
        t = torch.randn(*shape, generator=g) * O.init_std(kind, shape)
        w[key] = (t + 1.0 if kind == "g" else t).to(torch.bfloat16).float()
    return w


def test_nf4_weights_replace_exactly_the_quantised_tensors():
    cfg = O.CONFIGS["tiny"]
    w = O.make_weights(cfg, seed=0)
    wq = Q.nf4_weights(w, cfg)
    changed = {k for k in w if wq[k] is not w[k]}
    want = {f"model.layers.{i}.{k}" for i in range(cfg["layers"]) for k in Q.DECODER_LINEARS} | set(Q.PROJECTOR_WEIGHTS)
    assert changed == want
    for k in want:
        assert torch.equal(wq[k], Q.w_hat(w[k]).float())


def test_strict_id_margins_survive_quantisation_7b_shapes():
    """nf4_weights(condition_weights(w)) through the fp32 and the bf16 oracle: identical greedy ids (7B shapes, 2 layers)."""
    torch.set_num_threads(min(16, torch.get_num_threads()))
    cfg = dict(O.CONFIGS["llava-1.5-7b"], layers=2)
    wc = Q.nf4_weights(O.condition_weights(_lm_weights(cfg, seed=0), cfg, seed=0), cfg)
    prompt = torch.randint(3, cfg["vocab"], (1, 8), generator=torch.Generator().manual_seed(4))

    def ids(dtype):
        with torch.no_grad():
            logits, kv = O.llama_forward(wc, wc["model.embed_tokens.weight"][prompt], cfg, dtype=dtype, last_only=True)
            out = []
            for _ in range(8):
                nxt = logits[:, -1].argmax(-1)
                out.append(int(nxt))
                logits, kv = O.llama_forward(wc, wc["model.embed_tokens.weight"][nxt][:, None], cfg, kv=kv, dtype=dtype,
                                             last_only=True)
        return out

    assert ids(torch.float32) == ids(torch.bfloat16)


# ---------------------------------------------------------------------------------------------- argument handling
def test_quantization_arguments():
    from transformers import BitsAndBytesConfig
    from llava.model.language_model.llava_llama import _nf4_requested

    assert _nf4_requested({}) is False
    assert _nf4_requested({"load_in_4bit": True}) is True
    bnb = BitsAndBytesConfig(load_in_4bit=True, bnb_4bit_compute_dtype=torch.float16, bnb_4bit_use_double_quant=True,
                             bnb_4bit_quant_type="nf4")
    assert _nf4_requested({"quantization_config": bnb}) is True
    assert _nf4_requested({"quantization_config": {"load_in_4bit": True, "bnb_4bit_quant_type": "nf4"}}) is True
    for bad in ({"load_in_8bit": True}, {"quantization_config": BitsAndBytesConfig(load_in_8bit=True)},
                {"quantization_config": BitsAndBytesConfig(load_in_4bit=True, bnb_4bit_quant_type="fp4")},
                {"quantization_config": {"load_in_4bit": True, "bnb_4bit_quant_type": "fp4"}},
                {"quantization_config": {"load_in_4bit": True}}):  # bitsandbytes' default quant type is fp4
        with pytest.raises(NotImplementedError):
            _nf4_requested(bad)


def _config_dir(tmp_path, **extra):
    cfg = O.CONFIGS["tiny"]
    d = tmp_path / "ck"
    d.mkdir()
    (d / "config.json").write_text(json.dumps(dict(
        model_type="llava", vocab_size=cfg["vocab"], hidden_size=cfg["hidden"], intermediate_size=cfg["inter"],
        num_hidden_layers=cfg["layers"], num_attention_heads=cfg["heads"], num_key_value_heads=cfg["heads"], **extra)))
    return str(d)


def test_from_pretrained_nf4_with_fp8_decode_is_a_value_error(tmp_path, monkeypatch):
    from llava.model import LlavaLlamaForCausalLM

    monkeypatch.delenv("B2_FP8_DECODE", raising=False)
    path = _config_dir(tmp_path, b2_fp8_decode=True)
    with pytest.raises(ValueError, match="b2_fp8_decode"):
        LlavaLlamaForCausalLM.from_pretrained(path, load_in_4bit=True)
    with pytest.raises(ValueError, match="b2_fp8_decode"):
        LlavaLlamaForCausalLM.from_pretrained(path, quantization_config={"load_in_4bit": True, "bnb_4bit_quant_type": "nf4"})
    with pytest.raises(NotImplementedError):
        LlavaLlamaForCausalLM.from_pretrained(path, quantization_config={"load_in_4bit": True, "bnb_4bit_quant_type": "fp4"})


def test_load_pretrained_model_8bit_still_raises(tmp_path):
    from llava.model.builder import load_pretrained_model

    with pytest.raises(NotImplementedError):
        load_pretrained_model(str(tmp_path), None, "llava-v1.5-7b", load_8bit=True)
