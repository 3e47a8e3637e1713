"""GPU: the whole hot path (CLIP ViT -> mm_projector -> splice -> LLaMA prefill -> KV-cache decode) through the
C ABI and through the reference-facing Python surface, against
  (1) the committed golden outputs of the UNMODIFIED reference (tests/golden/*.npz), and
  (2) the fp32 oracle (oracle/llava_oracle.py) on the same seeded inputs,
plus size-independent properties at the LLaVA-1.5-7B layer shapes.

Floating-point tolerance (stated, as north_star asks): the engine computes in bf16 with fp32 accumulation.
Errors are measured as max|x - ref| / std(ref) against the fp32 reference and must stay within
TOL_MAX (5%) / TOL_MEAN (1%) of the logit standard deviation AND within 2x the error of the reference's OWN
bf16 path (the oracle run in bf16, which mirrors HF's bf16 rounding points) on the same inputs. Greedy token
ids must be identical wherever the reference's top-1/top-2 margin exceeds twice the measured logit error.
"""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from helpers import make_engine, make_model, rel_err, synth_inputs  # noqa: E402
from llava import _b2  # noqa: E402
from oracle import llava_oracle as O  # noqa: E402

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
DEV = "cuda"
TOL_MAX, TOL_MEAN = 0.05, 0.01


def _gold(name):
    return np.load(os.path.join(GOLD, name))


@pytest.fixture(scope="module")
def tiny():
    cfg = O.CONFIGS["tiny"]
    w = O.make_weights(cfg, seed=0)
    eng = make_engine(cfg, w, max_batch=4, max_seq=128, max_images=4)
    yield cfg, w, eng
    eng.close()


def _check(name, got, ref, bf16_ref=None, tol_max=TOL_MAX, tol_mean=TOL_MEAN):
    mx, mn = rel_err(got, ref)
    msg = f"{name}: max {mx:.4f} mean {mn:.4f} (of std)"
    if bf16_ref is not None:
        bmx, bmn = rel_err(bf16_ref, ref)
        msg += f"; reference-bf16 noise max {bmx:.4f} mean {bmn:.4f}"
        assert mn <= 2.0 * bmn + 2e-3, msg
    print(msg)
    assert mx <= tol_max and mn <= tol_mean, msg


def _assert_tokens(got, ref_tokens, ref_step_logits, err_abs):
    """ids equal wherever the reference margin > 2*err; after a (justified) divergence the contexts differ."""
    got, ref_tokens = np.asarray(got), np.asarray(ref_tokens)
    for b in range(ref_tokens.shape[0]):
        for i in range(ref_tokens.shape[1]):
            if got[b, i] == ref_tokens[b, i]:
                continue
            top2 = np.sort(np.asarray(ref_step_logits[i][b]))[-2:]
            margin = float(top2[1] - top2[0])
            assert margin <= 2 * err_abs, f"sample {b} step {i}: token {got[b, i]} != {ref_tokens[b, i]} at margin {margin:.4f} (err {err_abs:.4f})"
            break


# ------------------------------------------------------------------------------------------ golden fixtures
def test_encode_images_vs_reference_golden(tiny):
    cfg, w, eng = tiny
    g = _gold("tiny_prefill_decode.npz")
    images = torch.from_numpy(g["images"])
    bf = O.clip_vit_features(w, images, cfg, dtype=torch.bfloat16)
    _check("vit", eng.vit_encode(images.to(DEV)), torch.from_numpy(g["tower_features"]), bf)
    bf = O.encode_images(w, images, cfg, dtype=torch.bfloat16)
    _check("encode_images", eng.encode_images(images.to(DEV)), torch.from_numpy(g["image_features"]), bf)


def test_prefill_and_greedy_vs_reference_golden(tiny):
    cfg, w, eng = tiny
    g = _gold("tiny_prefill_decode.npz")
    embeds = torch.from_numpy(g["inputs_embeds"])
    B, S_ = embeds.shape[:2]
    kv = eng.new_kv(B, 128)
    logits = eng.prefill(kv, embeds.to(DEV), None, _b2.LOGITS_ALL)
    ref = torch.from_numpy(g["logits"])
    bf, _ = O.llama_forward(w, embeds, cfg, dtype=torch.bfloat16)
    _check("prefill logits", logits, ref, bf)
    assert kv.lengths(B) == [S_] * B
    # greedy decode from the engine's own prefill, device-resident loop
    last = eng.prefill(kv, embeds.to(DEV), None, _b2.LOGITS_LAST)
    torch.testing.assert_close(last, logits[:, -1], rtol=2e-2, atol=2e-2 * float(ref.std()))
    first = eng.argmax(last)
    n = g["greedy_tokens"].shape[1]
    rest = eng.decode_greedy(kv, first, n - 1)
    toks = torch.cat([first[None], rest]).t().cpu().numpy()
    err_abs = rel_err(logits, ref)[0] * float(ref.std())
    _assert_tokens(toks, g["greedy_tokens"], g["step_logits"], err_abs)
    assert kv.lengths(B) == [S_ + n - 1] * B
    kv.close()


def test_decode_step_logits_vs_reference_golden(tiny):
    cfg, w, eng = tiny
    g = _gold("tiny_prefill_decode.npz")
    embeds = torch.from_numpy(g["inputs_embeds"]).to(DEV)
    B = embeds.shape[0]
    kv = eng.new_kv(B, 128)
    eng.prefill(kv, embeds, None, _b2.LOGITS_NONE)
    ref_steps, ref_toks = torch.from_numpy(g["step_logits"]), torch.from_numpy(g["greedy_tokens"])
    # teacher-forced with the REFERENCE tokens so every step is comparable even after a near-tie
    for i in range(1, ref_toks.shape[1]):
        logits = eng.decode_step(kv, ref_toks[:, i - 1].to(torch.int32))
        _check(f"decode step {i}", logits, ref_steps[i], tol_max=0.06)
    kv.close()


def test_python_surface_splice_vs_reference_golden():
    cfg = O.CONFIGS["tiny"]
    w = O.make_weights(cfg, seed=0)
    g = _gold("tiny_splice_edges.npz")
    ids, mask = torch.from_numpy(g["input_ids"]), torch.from_numpy(g["attention_mask"])
    labels, images = torch.from_numpy(g["labels"]), torch.from_numpy(g["images"])
    Lt = ids.shape[1]
    for case, extra in (("right", {}), ("left", {"tokenizer_padding_side": "left"}), ("trunc", {"tokenizer_model_max_length": 20})):
        model = make_model(cfg, w, max_batch=4, max_seq=128, **extra)
        r = model.prepare_inputs_labels_for_multimodal(ids.to(DEV), torch.arange(Lt)[None].expand(3, Lt).to(DEV),
                                                       mask.to(DEV), None, labels.to(DEV), images.to(DEV))
        assert r[0] is None and r[3] is None
        assert (r[2].cpu().numpy().astype(bool) == g[f"{case}_mask"].astype(bool)).all()
        assert (r[1].cpu().numpy() == g[f"{case}_pos"]).all()
        assert (r[5].cpu().numpy() == g[f"{case}_labels"]).all()
        m = torch.from_numpy(g[f"{case}_mask"].astype(bool))
        got, ref = r[4].float().cpu(), torch.from_numpy(g[f"{case}_embeds"])
        assert (got[~m] == 0).all()  # zero embeddings in the padding
        _check(f"splice {case}", got[m], ref[m])
        model.invalidate_engine()
    # None-mirroring + 5-D images flattened into one slot
    model = make_model(cfg, w, max_batch=4, max_seq=128)
    r = model.prepare_inputs_labels_for_multimodal(torch.from_numpy(g["ids5"]).to(DEV), None, None, None, None,
                                                   torch.from_numpy(g["images5"]).to(DEV))
    assert r[0] is None and r[1] is None and r[2] is None and r[5] is None
    _check("splice 5-D", r[4], torch.from_numpy(g["embeds5"]))


# ------------------------------------------------------------------------------------------ oracle, larger config
def test_small_config_end_to_end_vs_oracle():
    cfg = O.CONFIGS["small"]
    w = O.make_weights(cfg, seed=11)
    ids, images = synth_inputs(cfg, B=3, Lt=20, seed=4)
    n = 8
    ref_toks, ref_steps = O.greedy_generate(w, ids, images, cfg, n, return_logits=True)
    embeds, _, _, _ = O.prepare_multimodal(w, ids, images, cfg)
    ref_logits, _ = O.llama_forward(w, embeds, cfg)
    bf_logits, _ = O.llama_forward(w, O.prepare_multimodal(w, ids, images, cfg, dtype=torch.bfloat16)[0], cfg, dtype=torch.bfloat16)
    model = make_model(cfg, w, max_batch=4, max_seq=256)
    out = model(input_ids=ids.to(DEV), images=images.to(DEV), use_cache=True)
    _check("small forward logits", out.logits, ref_logits, bf_logits)
    err_abs = rel_err(out.logits, ref_logits)[0] * float(ref_logits.std())
    full = model.generate(ids.to(DEV), images=images.to(DEV), do_sample=False, max_new_tokens=n, use_cache=True)
    assert full.shape == (3, ids.shape[1] + n) and (full[:, : ids.shape[1]].cpu() == ids).all()  # prompt echoed
    _assert_tokens(full[:, ids.shape[1]:].cpu().numpy(), ref_toks.numpy(), ref_steps.numpy(), err_abs)


def test_generate_protocols_streamer_stopping_eos():
    cfg = O.CONFIGS["tiny"]
    w = O.make_weights(cfg, seed=0)
    model = make_model(cfg, w, max_batch=2, max_seq=128)
    ids, images = synth_inputs(cfg, B=1, Lt=12, seed=9)
    ref = model.generate(ids.to(DEV), images=images.to(DEV), do_sample=False, max_new_tokens=6)

    class Streamer:
        def __init__(self):
            self.chunks, self.ended = [], False

        def put(self, v):
            assert v.device.type == "cpu"
            self.chunks.append(v.clone())

        def end(self):
            self.ended = True

    class StopAfter:  # plain-bool criterion like the reference's KeywordsStoppingCriteria (mm_utils.py:109-114)
        def __init__(self, start_len, n):
            self.start_len, self.n, self.calls = start_len, n, 0

        def __call__(self, output_ids, scores, **kw):
            self.calls += 1
            assert output_ids.shape[1] - self.start_len == self.calls  # cat(prompt ids with -200, new tokens)
            return output_ids.shape[1] - self.start_len >= self.n

    st, crit = Streamer(), StopAfter(ids.shape[1], 3)
    out = model.generate(inputs=ids.to(DEV), images=images.to(DEV), do_sample=False, max_new_tokens=6,
                         streamer=st, stopping_criteria=[crit], use_cache=True)
    assert out.shape[1] == ids.shape[1] + 3 and st.ended
    assert torch.equal(st.chunks[0], ids) and len(st.chunks) == 1 + 3
    assert torch.equal(out.cpu(), ref[:, : ids.shape[1] + 3].cpu())  # step loop == graph-replay loop
    # eos stops generation
    eos = int(ref[0, ids.shape[1] + 1])
    out = model.generate(ids.to(DEV), images=images.to(DEV), do_sample=False, max_new_tokens=6, eos_token_id=eos)
    assert int(out[0, -1]) == eos and out.shape[1] <= ids.shape[1] + 2
    # sampling path runs and echoes the prompt
    torch.manual_seed(0)
    out = model.generate(ids.to(DEV), images=images.to(DEV), do_sample=True, temperature=0.7, top_p=0.9, max_new_tokens=4)
    assert out.shape[1] == ids.shape[1] + 4 and (out[:, : ids.shape[1]].cpu() == ids).all()
    with pytest.raises(NotImplementedError):
        model.generate(ids.to(DEV), images=images.to(DEV), num_beams=4, max_new_tokens=2)
    with pytest.raises(ValueError):
        model.generate(ids.to(DEV), images=images.to(DEV), max_new_tokens=4096)  # exceeds engine limits


def test_forward_incremental_decode_and_loss():
    cfg = O.CONFIGS["tiny"]
    w = O.make_weights(cfg, seed=2)
    model = make_model(cfg, w, max_batch=2, max_seq=128)
    ids, images = synth_inputs(cfg, B=2, Lt=10, seed=3)
    labels = ids.clone()
    out = model(input_ids=ids.to(DEV), images=images.to(DEV), labels=labels.to(DEV), use_cache=True)
    embeds, _, _, new_labels = O.prepare_multimodal(w, ids, images, cfg, labels=labels)
    ref_logits, _ = O.llama_forward(w, embeds, cfg)
    ref_loss = torch.nn.functional.cross_entropy(ref_logits[:, :-1].reshape(-1, cfg["vocab"]), new_labels[:, 1:].reshape(-1), ignore_index=-100)
    assert abs(float(out.loss) - float(ref_loss)) <= 0.03 * abs(float(ref_loss))
    nxt = out.logits[:, -1].argmax(-1, keepdim=True)
    step = model(input_ids=nxt, past_key_values=out.past_key_values, use_cache=True)
    e = w["model.embed_tokens.weight"][nxt.cpu()]
    ref2, _ = O.llama_forward(w, torch.cat([embeds, e], 1), cfg)
    _check("incremental decode", step.logits[:, 0], ref2[:, -1], tol_max=0.06)


def test_left_padded_batch_matches_right_padded():
    cfg = O.CONFIGS["tiny"]
    w = O.make_weights(cfg, seed=0)
    g = _gold("tiny_splice_edges.npz")
    ids, mask, images = (torch.from_numpy(g[k]) for k in ("input_ids", "attention_mask", "images"))
    outs = {}
    for side in ("right", "left"):
        model = make_model(cfg, w, max_batch=4, max_seq=128, tokenizer_padding_side=side)
        r = model(input_ids=ids.to(DEV), attention_mask=mask.to(DEV), images=images.to(DEV))
        outs[side] = r.logits.float().cpu()
        model.invalidate_engine()
    mr, ml = g["right_mask"].astype(bool), g["left_mask"].astype(bool)
    for b in range(ids.shape[0]):
        torch.testing.assert_close(outs["left"][b][torch.from_numpy(ml[b])], outs["right"][b][torch.from_numpy(mr[b])],
                                   rtol=1e-3, atol=1e-3)


# ------------------------------------------------------------------------------------------ full-size properties
def test_7b_layer_shapes_prefill_decode_consistency():
    """LLaVA-1.5-7B layer shapes (h=4096, I=11008, 32 heads, V=32000; 2 decoder layers and 2 live ViT layers so
    the fp32 oracle finishes in seconds): engine vs oracle, and decode-step logits == prefill-recompute logits
    (GEMV/split-KV decode path vs wgmma/flash prefill path on the same cache)."""
    cfg = O.make_config(layers=2, vit_layers=3)
    w = O.make_weights(cfg, seed=5)
    eng = make_engine(cfg, w, max_batch=2, max_seq=1024, max_images=2)
    B, Lt = 2, 40
    ids, images = synth_inputs(cfg, B=B, Lt=Lt, seed=6)
    feats = eng.encode_images(images.to(DEV))
    ref_feats = O.encode_images(w, images, cfg)
    _check("7B-shape encode_images", feats, ref_feats)
    embeds, _, _, _ = O.prepare_multimodal(w, ids, images, cfg, image_features=list(ref_feats))
    S_ = embeds.shape[1]
    assert S_ == Lt - 1 + 576
    kv = eng.new_kv(B, 1024)
    last = eng.prefill(kv, embeds.to(DEV), None, _b2.LOGITS_LAST)
    ref_logits, _ = O.llama_forward(w, embeds, cfg, last_only=True)
    _check("7B-shape prefill last logits", last, ref_logits[:, 0])
    tok = last.argmax(-1).to(torch.int32)
    step1 = eng.decode_step(kv, tok)
    ext = torch.cat([embeds, w["model.embed_tokens.weight"][tok.cpu().long()][:, None]], 1)
    kv2 = eng.new_kv(B, 1024)
    re_last = eng.prefill(kv2, ext.to(DEV), None, _b2.LOGITS_LAST)
    _check("decode step vs prefill recompute", step1, re_last, tol_max=0.03, tol_mean=0.006)
    ref2, _ = O.llama_forward(w, ext, cfg, last_only=True)
    _check("7B-shape decode logits vs oracle", step1, ref2[:, 0])
    # batch invariance: sample 0 alone == sample 0 in the batch
    kv3 = eng.new_kv(1, 1024)
    solo = eng.prefill(kv3, embeds[:1].to(DEV), None, _b2.LOGITS_LAST)
    torch.testing.assert_close(solo[0], last[0], rtol=1e-3, atol=1e-3)
    for k in (kv, kv2, kv3):
        k.close()
    eng.close()


@pytest.mark.parametrize("B", [1, 2, 4])
def test_13b_layer_shapes_decode_equals_prefill_recompute(B):
    """LLaVA-1.5-13B layer shapes (h=5120, I=13824, 40 heads; 2 layers): size-independent property at BASELINE
    config-4 dims — the logits of a decode step (B<=2: persistent megakernel with its 5-stage TMA ring; B=4: GEMV
    kernels from a CUDA graph) must equal the logits of a prefill over the extended sequence (wgmma GEMM + flash)."""
    cfg = O.make_config(hidden=5120, inter=13824, layers=2, heads=40, vit_layers=2)
    w = O.make_weights(cfg, seed=7)
    eng = make_engine(cfg, w, max_batch=4, max_seq=256, max_images=1)
    g = torch.Generator().manual_seed(3)
    S_ = 150
    embeds = (torch.randn(B, S_, cfg["hidden"], generator=g) * 0.5).to(torch.bfloat16)
    kv = eng.new_kv(B, 256)
    last = eng.prefill(kv, embeds.to(DEV), None, _b2.LOGITS_LAST)
    toks = last.argmax(-1).to(torch.int32)
    ext = embeds
    for step in range(3):
        lg = eng.decode_step(kv, toks)
        ext = torch.cat([ext, w["model.embed_tokens.weight"][toks.cpu().long()][:, None].to(torch.bfloat16)], 1)
        kv2 = eng.new_kv(B, 256)
        ref = eng.prefill(kv2, ext.to(DEV), None, _b2.LOGITS_LAST)
        _check(f"13B-shape decode step {step} vs prefill recompute (B={B})", lg, ref, tol_max=0.03, tol_mean=0.006)
        kv2.close()
        toks = lg.argmax(-1).to(torch.int32)
    assert kv.lengths(B) == [S_ + 3] * B
    kv.close()
    eng.close()


@pytest.mark.parametrize("B,dims", [(12, (4096, 11008, 32)), (32, (4096, 11008, 32)), (32, (5120, 13824, 40))])
def test_batched_decode_skinny_gemm_equals_prefill_recompute(B, dims):
    """BASELINE bs=32 decode at LLaVA-1.5-7B / 13B layer shapes (2 layers): every Linear of the step runs through the
    swap-AB stream-K wgmma GEMM (csrc/gemm_skinny.cu: stream-K splits, SwiGLU epilogue, fp32 logits) replayed from a
    CUDA graph; its logits must equal a prefill (tile GEMM + flash attention) over the extended sequence."""
    h, I, H = dims
    cfg = O.make_config(hidden=h, inter=I, layers=2, heads=H, vit_layers=2)
    w = O.make_weights(cfg, seed=11)
    eng = make_engine(cfg, w, max_batch=B, max_seq=160, max_images=1)
    g = torch.Generator().manual_seed(5)
    S_ = 100
    embeds = (torch.randn(B, S_, h, generator=g) * 0.5).to(torch.bfloat16)
    kv = eng.new_kv(B, 160)
    last = eng.prefill(kv, embeds.to(DEV), None, _b2.LOGITS_LAST)
    toks = last.argmax(-1).to(torch.int32)
    ext = embeds
    for step in range(3):  # step 0 runs eagerly, steps 1-2 replay the captured graph
        lg = eng.decode_step(kv, toks)
        ext = torch.cat([ext, w["model.embed_tokens.weight"][toks.cpu().long()][:, None].to(torch.bfloat16)], 1)
        kv2 = eng.new_kv(B, 160)
        ref = eng.prefill(kv2, ext.to(DEV), None, _b2.LOGITS_LAST)
        _check(f"batched decode step {step} vs prefill recompute (B={B}, h={h})", lg, ref, tol_max=0.03, tol_mean=0.006)
        kv2.close()
        toks = lg.argmax(-1).to(torch.int32)
    assert kv.lengths(B) == [S_ + 3] * B
    kv.close()
    eng.close()


def test_decode_batch_above_8_uses_gemm_path_and_matches_oracle():
    """B > 8 decode runs the swap-AB stream-K wgmma GEMM path (+ CUDA-graph replay); B <= 8 the GEMV kernels / the
    persistent megakernel (B <= 2).
    Both must agree with the oracle and with each other on the shared samples."""
    cfg = O.CONFIGS["tiny"]
    w = O.make_weights(cfg, seed=0)
    eng = make_engine(cfg, w, max_batch=12, max_seq=96, max_images=4)
    B, Lt, n = 10, 9, 5
    ids, images = synth_inputs(cfg, B=B, Lt=Lt, seed=21, image_pos=2)
    ref_toks, ref_steps = O.greedy_generate(w, ids, images, cfg, n, return_logits=True)
    embeds, _, _, _ = O.prepare_multimodal(w, ids, images, cfg)
    ref_logits, _ = O.llama_forward(w, embeds, cfg)
    out = {}
    for nb in (B, 4):
        kv = eng.new_kv(nb, 96)
        last = eng.prefill(kv, embeds[:nb].to(DEV), None, _b2.LOGITS_LAST)
        _check(f"prefill last (B={nb})", last, ref_logits[:nb, -1])
        first = eng.argmax(last)
        rest = eng.decode_greedy(kv, first, n - 1)
        out[nb] = torch.cat([first[None], rest]).t().cpu()
        # teacher-forced step logits through the same path
        kv.reset()
        eng.prefill(kv, embeds[:nb].to(DEV), None, _b2.LOGITS_NONE)
        for i in range(1, n):
            lg = eng.decode_step(kv, ref_toks[:nb, i - 1].to(torch.int32))
            _check(f"decode step {i} (B={nb})", lg, ref_steps[i][:nb], tol_max=0.06)
        kv.close()
    err_abs = 0.05 * float(ref_logits.std())
    _assert_tokens(out[B].numpy(), ref_toks.numpy(), ref_steps.numpy(), err_abs)
    _assert_tokens(out[4].numpy(), ref_toks[:4].numpy(), ref_steps[:, :4].numpy(), err_abs)
    eng.close()


def test_error_convention():
    cfg = O.CONFIGS["tiny"]
    w = O.make_weights(cfg, seed=0)
    from llava._b2 import Engine
    from helpers import desc_from_cfg

    eng = Engine(desc_from_cfg(cfg), DEV)
    with pytest.raises(ValueError):
        eng.set_weight("model.not_a_key", torch.zeros(4, device=DEV))
    with pytest.raises(ValueError):
        eng.set_weight("model.norm.weight", torch.zeros(7, device=DEV))  # wrong shape
    with pytest.raises(RuntimeError):
        eng.finalize()  # missing weights
    eng.close()
    eng = make_engine(cfg, w, max_batch=1, max_seq=32, max_images=1)
    kv = eng.new_kv(1, 32)
    with pytest.raises(ValueError):
        eng.prefill(kv, torch.zeros(1, 64, cfg["hidden"], device=DEV), None, _b2.LOGITS_LAST)  # S > capacity
    with pytest.raises(ValueError):
        eng.decode_step(kv, torch.zeros(1, dtype=torch.int32))  # empty cache
    eng.close()


def test_rope_fused_into_qkv_gemm_equals_the_standalone_pass():
    """Judge row N3: RoPE + KV-cache write in the QKV GEMM's epilogue (CTA-pair kernel, M >= 512) against the standalone
    rope_kv_write pass (B2_ROPE_FUSED=0) at the 7B layer shape: prefill logits, and the logits of a decode step that reads the
    K/V rows the epilogue wrote — ragged lengths, cache slots 1..2 of 3 (prefill_slots), so batch / position / slot indexing of
    the epilogue are all exercised. The two paths may run different GEMM tile kernels (<= 1 bf16 ulp apart on q, k, v)."""
    cfg = O.make_config(layers=2, vit_layers=2)
    w = O.make_weights(cfg, seed=31)
    eng = make_engine(cfg, w, max_batch=3, max_seq=640, max_images=2)
    g = torch.Generator().manual_seed(32)
    B, S = 2, 600
    embeds = (torch.randn(B, S, cfg["hidden"], generator=g) * 0.5).to(torch.bfloat16)
    lens = [600, 433]
    out = {}
    try:
        for mode in ("0", "1"):
            os.environ["B2_ROPE_FUSED"] = mode
            kv = eng.new_kv(3, 640)
            eng.prefill(kv, embeds[:1, :8].to(DEV), None, _b2.LOGITS_LAST, slot0=0)   # slot 0: a short context (standalone pass)
            last = eng.prefill(kv, embeds.to(DEV), lens, _b2.LOGITS_LAST, slot0=1)
            tok = last.argmax(-1).to(torch.int32)
            full = torch.zeros(3, dtype=torch.int32, device=DEV)
            full[1:] = tok
            step = eng.decode_step(kv, full)
            out[mode] = (last.float().cpu(), step.float().cpu()[1:])
            kv.close()
    finally:
        os.environ.pop("B2_ROPE_FUSED", None)
    for a, b, what in ((out["1"][0], out["0"][0], "prefill logits"), (out["1"][1], out["0"][1], "decode-step logits")):
        assert torch.isfinite(a).all()
        err = (a - b).abs()
        assert err.max() <= 0.02 * b.std() and err.mean() <= 0.003 * b.std(), (what, float(err.max()), float(b.std()))
    ref, _ = O.llama_forward(w, embeds[:1].float(), cfg, last_only=True)
    _check("rope-fused prefill vs oracle (row 0)", out["1"][0][:1], ref[:, 0])
    eng.close()


def _two_gemm_projector(w, feats):
    """mm_projector as two b2_op_gemm launches (bias + erf GELU into a bf16 H, then bias): the GEMM the fused kernel runs."""
    lib = _b2.load_library()
    x = feats.reshape(-1, feats.shape[-1]).to(DEV)
    W1, b1, W2, b2 = (w[f"model.mm_projector.{k}"].to(DEV, torch.bfloat16) for k in ("0.weight", "0.bias", "2.weight", "2.bias"))
    (M, K), N = x.shape, W1.shape[0]
    mid, out = (torch.empty(M, N, device=DEV, dtype=torch.bfloat16) for _ in range(2))
    st = _b2.stream_ptr()
    _b2.check(lib.b2_op_gemm(_b2.ptr(x), K, _b2.ptr(W1), K, _b2.ptr(b1), None, 0, _b2.ptr(mid), N, 0, M, N, K, _b2.ACT_GELU_ERF,
                             0, st), "b2_op_gemm")
    _b2.check(lib.b2_op_gemm(_b2.ptr(mid), N, _b2.ptr(W2), N, _b2.ptr(b2), None, 0, _b2.ptr(out), N, 0, M, N, N, _b2.ACT_NONE,
                             0, st), "b2_op_gemm")
    return out.reshape(*feats.shape[:-1], N)


@pytest.mark.parametrize("n_img", [1, 3, 20])
def test_fused_projector_kernel_equals_the_two_gemm_form(n_img):
    """north_star: "mm_projector as one fused GEMM->GELU->GEMM kernel". The single-launch kernel (phase-2 tiles gated on
    per-row-block completion counters) against the two-launch form of the same GEMM (two b2_op_gemm calls) and the oracle,
    at the 7B projector shape; 20 images = 90 row blocks = 12 dependency groups, repeated to catch a stale read of H."""
    cfg = O.make_config(hidden=4096, inter=11008, layers=1, heads=32, vit_layers=2)
    w = O.make_weights(cfg, seed=21)
    eng = make_engine(cfg, w, max_batch=1, max_seq=32, max_images=n_img)
    g = torch.Generator().manual_seed(n_img)
    feats = (torch.randn(n_img, 576, 1024, generator=g)).to(torch.bfloat16)
    ref = O.mm_projector(w, feats.float())
    two = _two_gemm_projector(w, feats).float().cpu()
    for rep in range(4):
        one = eng.project(feats.to(DEV)).float().cpu()
        assert torch.isfinite(one).all()
        # same operands, same fp32 accumulation order per output element (tile width may differ): <= 1 bf16 ulp apart
        torch.testing.assert_close(one, two, rtol=2 ** -7, atol=1e-3)
    _check(f"fused projector ({n_img} images)", one, ref)
    eng.close()
