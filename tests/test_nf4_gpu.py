"""GPU: NF4 decoder weights (load_4bit), all through the C ABI.

The quantiser and dequantiser kernels are compared bit for bit with oracle/nf4_oracle.py; gemv_nf4 against the fp64 product
over w_hat; the NF4 engine (built from weights w) against the bf16 engine built from nf4_weights(w): bit-equal wherever both
run the same dense kernels over the same bf16 values (prefill, decode at batch > 8), within a stated tolerance where the
NF4 engine streams 4-bit weights (gemv_nf4, batch <= 8); strict greedy ids on conditioned weights; the loader surface."""
import os
import subprocess
import sys
import textwrap

import pytest
import torch

pytestmark = pytest.mark.gpu

from helpers import make_engine, rel_err  # noqa: E402
from llava import _b2  # noqa: E402
from oracle import llava_oracle as O  # noqa: E402
from oracle import nf4_oracle as Q  # noqa: E402

DEV, BF = "cuda", torch.bfloat16
SHAPES_7B = [(12288, 4096), (4096, 4096), (22016, 4096), (4096, 11008)]


def P(t):
    return _b2.ptr(t)


def S():
    return _b2.stream_ptr()


def lib():
    return _b2.load_library()


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(*shape, generator=g, device=DEV) * scale).to(BF)


def interleaved_gate_up(I, h, seed):
    gate, up = rnd(I, h, scale=h ** -0.5, seed=seed), rnd(I, h, scale=h ** -0.5, seed=seed + 1)
    out = torch.empty(2 * I, h, device=DEV, dtype=BF)
    _b2.check(lib().b2_op_interleave_gate_up(P(gate), P(up), P(out), I, h, S()))
    return out


def op_quantize(w):
    N, K = w.shape
    codes = torch.empty(N, K // 2, device=DEV, dtype=torch.uint8)
    absmax = torch.empty(N, K // 64, device=DEV, dtype=torch.float32)
    _b2.check(lib().b2_op_quantize_nf4(P(w), N, K, P(codes), P(absmax), S()), "b2_op_quantize_nf4")
    return codes, absmax


# ---------------------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("shape", ["12288x4096", "4096x4096", "11008x4096", "4096x11008", "wgu"])
def test_quantize_and_dequantize_kernels_bit_equal_to_oracle(shape):
    w = interleaved_gate_up(11008, 4096, seed=1) if shape == "wgu" else rnd(*map(int, shape.split("x")), scale=0.02, seed=2)
    w[3, 128:192] = 0  # an all-zero block
    w[5, 0] = -w[5, 1:64].abs().max() * 2  # the block's absmax carried by a negative element
    codes, absmax = op_quantize(w)
    torch.cuda.synchronize()
    q_ref, a_ref = Q.quantize_nf4(w.cpu())
    assert torch.equal(absmax.cpu(), a_ref)
    assert torch.equal(codes.cpu(), Q.pack_nf4(q_ref))
    assert int(Q.unpack_nf4(codes.cpu())[3, 128:192].unique().item()) == 7 and float(absmax[3, 2]) == 0.0
    N, K = w.shape
    out = torch.empty(N, K, device=DEV, dtype=BF)
    _b2.check(lib().b2_op_dequantize_nf4(P(codes), P(absmax), N, K, P(out), S()), "b2_op_dequantize_nf4")
    assert torch.equal(out.cpu(), Q.dequantize_nf4(q_ref, a_ref))


def test_kernel_argument_checks():
    w = rnd(64, 96)
    c = torch.empty(64, 48, device=DEV, dtype=torch.uint8)
    a = torch.empty(64, 2, device=DEV)
    assert lib().b2_op_quantize_nf4(P(w), 64, 96, P(c), P(a), S()) == -1  # K % 64
    x, out = rnd(1, 192), torch.empty(1, 64, device=DEV, dtype=BF)
    assert lib().b2_op_gemv_nf4(P(x), 192, P(c), P(a), None, 0.0, None, 0, P(out), 64, 1, 64, 192, 0, S()) == -1  # K % 128
    x = rnd(9, 256)
    assert lib().b2_op_gemv_nf4(P(x), 256, P(c), P(a), None, 0.0, None, 0, P(out), 64, 9, 64, 256, 0, S()) == -1  # B > 8


def gemv_nf4(x, codes_gemv, absmax, N, K, gamma=None, residual=None, act=_b2.ACT_NONE, eps=1e-5):
    B = x.shape[0]
    n_out = N // 2 if act == _b2.ACT_SWIGLU else N
    out = torch.empty(B, n_out, device=DEV, dtype=BF)
    _b2.check(lib().b2_op_gemv_nf4(P(x), x.stride(0), P(codes_gemv), P(absmax), P(gamma), eps, P(residual),
                                   residual.stride(0) if residual is not None else 0, P(out), n_out, B, N, K, act, S()),
              "b2_op_gemv_nf4")
    return out


GEMV_WORST = {}


@pytest.mark.parametrize("B", [1, 2, 4, 8])
@pytest.mark.parametrize("N,K", SHAPES_7B + [(1000, 4096)])
@pytest.mark.parametrize("mode", ["plain", "norm", "residual", "swiglu"])
def test_gemv_nf4_within_bound_of_fp64_product(B, N, K, mode):
    """|y - y_ref| <= 2^-8 * sum_k |x_k w_hat_k| + 1e-6 against the fp64 product over w_hat (norm restated in bf16 as the
    bf16 GEMV tests do); SwiGLU: the bound of each of its two products, carried through silu(g) * u."""
    if mode == "swiglu" and N != 22016:
        pytest.skip("SwiGLU runs on the interleaved gate/up shape")
    w = interleaved_gate_up(N // 2, K, seed=3) if mode == "swiglu" else rnd(N, K, scale=K ** -0.5, seed=3)
    q, a = Q.quantize_nf4(w)
    wh = Q.dequantize_nf4(q, a).double()
    codes = Q.pack_nf4(q, "gemv")
    x = rnd(B, K, seed=4)
    gamma = (1 + 0.1 * torch.randn(K, device=DEV)).to(BF) if mode in ("norm", "swiglu") else None
    res = rnd(B, N, seed=5) if mode == "residual" else None
    xin = x
    if gamma is not None:
        xf = x.float()
        xin = (gamma.float() * (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-5)).to(BF).float()).to(BF)
    xd = xin.double()
    y_lin, bnd = xd @ wh.t(), xd.abs() @ wh.abs().t()
    y = gemv_nf4(x, codes, a, N, K, gamma=gamma, residual=res,
                 act=_b2.ACT_SWIGLU if mode == "swiglu" else _b2.ACT_NONE).double()
    if mode == "swiglu":
        rows = torch.arange(N, device=DEV).view(-1, 128)
        gi, ui = rows[:, :64].reshape(-1), rows[:, 64:].reshape(-1)
        g, u, eg, eu = y_lin[:, gi], y_lin[:, ui], 2 ** -8 * bnd[:, gi] + 1e-6, 2 ** -8 * bnd[:, ui] + 1e-6
        sg = torch.sigmoid(g)
        want = g * sg * u
        dsilu = (sg * (1 + g * (1 - sg))).abs() + eg  # |silu'| over the interval, loosely
        tol = dsilu * eg * (u.abs() + eu) + (g * sg).abs() * eu + 2 ** -8 * want.abs() + 1e-6
    else:
        want = y_lin + (res.double() if res is not None else 0)
        tol = 2 ** -8 * bnd + 1e-6 + (2 ** -8 * res.double().abs() if res is not None else 0)
    err = (y - want).abs()
    ratio = float((err / tol).max())
    GEMV_WORST[(B, N, K, mode)] = ratio
    print(f"gemv_nf4 B={B} N={N} K={K} {mode}: max |err| / bound = {ratio:.4f}")
    assert ratio <= 1.0


# ---------------------------------------------------------------------------------------------- engine
def dev_weights(cfg, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    w = {}
    for key, shape, kind in O.weight_shapes(cfg):
        t = torch.randn(*shape, generator=g, device=DEV) * O.init_std(kind, shape)
        w[key] = (t + 1.0 if kind == "g" else t).to(BF)
    return w


CFG2 = dict(O.CONFIGS["llava-1.5-7b"], layers=2, vit_layers=1)


@pytest.fixture(scope="module")
def pair():
    """NF4 engine from w, bf16 engine from nf4_weights(w): 7B layer shapes, 2 layers."""
    w = dev_weights(CFG2, seed=11)
    e4 = make_engine(CFG2, w, max_batch=32, max_seq=784, max_images=1)
    e4.enable_nf4()
    e16 = make_engine(CFG2, Q.nf4_weights(w, CFG2), max_batch=32, max_seq=784, max_images=1)
    yield e4, e16, w
    e4.close(), e16.close()


def _embeds(B, S_, seed):
    return rnd(B, S_, CFG2["hidden"], seed=seed)


@pytest.mark.parametrize("rope_fused", ["1", "0"])
def test_prefill_logits_bit_equal_to_bf16_engine_on_w_hat(pair, rope_fused, monkeypatch):
    monkeypatch.setenv("B2_ROPE_FUSED", rope_fused)
    e4, e16, _ = pair
    B, S_ = 2, 704
    lens = [704, 650]
    emb = _embeds(B, S_, seed=21)
    for mode in (_b2.LOGITS_LAST, _b2.LOGITS_ALL):
        out = []
        for eng in (e4, e16):
            kv = eng.new_kv(B, 784)
            out.append(eng.prefill(kv, emb, lens, mode).clone())
            if mode == _b2.LOGITS_LAST:  # one offset chunk behind the prompt
                chunk = _embeds(B, 64, seed=22)
                out.append(eng.prefill(kv, chunk, [64, 40], mode, start=[704, 650]).clone())
            kv.close()
        torch.cuda.synchronize()
        half = len(out) // 2
        for a, b in zip(out[:half], out[half:]):
            assert torch.equal(a, b)


def _teacher_forced(e4, e16, B, steps, seed):
    emb = _embeds(B, 128, seed=seed)
    kv4, kv16 = e4.new_kv(B, 784), e16.new_kv(B, 784)
    l4, l16 = e4.prefill(kv4, emb, None, _b2.LOGITS_LAST), e16.prefill(kv16, emb, None, _b2.LOGITS_LAST)
    res = [(l4.clone(), l16.clone())]
    for _ in range(steps):
        tok = l16.argmax(-1).to(torch.int32)
        l4, l16 = e4.decode_step(kv4, tok), e16.decode_step(kv16, tok)
        res.append((l4.clone(), l16.clone()))
    kv4.close(), kv16.close()
    return res


@pytest.mark.parametrize("B", [12, 32])
def test_decode_dequantise_stream_k_bit_equal(pair, B):
    e4, e16, _ = pair
    for a, b in _teacher_forced(e4, e16, B, 8, seed=30 + B):
        assert torch.equal(a, b)


@pytest.mark.parametrize("B", [1, 4, 8])
def test_decode_gemv_nf4_within_tolerance(pair, B, monkeypatch):
    """gemv_nf4 feeds every weight to the MMA as w_hat = bf16(code * absmax), the values the bf16 engine reads; what is left
    is the order of the fp32 accumulation, which bf16 rounding of the activations carries into the logits: max <= 2 %,
    mean <= 0.5 % of the logit std over 8 teacher-forced steps. The bf16 engine decodes with its weight-streaming kernels
    (megakernel at batch 1, GEMV graph at 4 and 8): at batch 8 its default, the stream-K GEMM, has a split-K reduction
    order of its own, which would add its own noise to what this test measures."""
    e4, e16, _ = pair
    if B == 8:
        monkeypatch.setenv("B2_DECODE_SKINNY", "0")  # bf16 engine: GEMV graph at batch 8 (NF4 takes gemv_nf4 regardless)
    res = _teacher_forced(e4, e16, B, 8, seed=40 + B)
    assert torch.equal(res[0][0], res[0][1])  # the prefill is bit-equal
    errs = [rel_err(a, b.float().cpu()) for a, b in res[1:]]
    mx, mn = max(e[0] for e in errs), max(e[1] for e in errs)
    print(f"gemv_nf4 decode B={B}: max {mx:.4f} / mean {mn:.4f} of the logit std")
    assert mx <= 0.02 and mn <= 0.005, (mx, mn)


def test_projector_holds_w_hat(pair):
    e4, e16, _ = pair
    feats = rnd(576, CFG2["vit_hidden"], seed=50)
    assert torch.equal(e4.project(feats), e16.project(feats))


def test_weight_bytes(pair):
    e4, e16, _ = pair
    h, I, L = CFG2["hidden"], CFG2["inter"], CFG2["layers"]
    delta = 0
    for N, K in [(3 * h, h), (h, h), (2 * I, h), (h, I)]:
        delta += -2 * N * K + Q.nf4_linear_bytes(N, K)
    assert e4.weight_bytes() == e16.weight_bytes() + L * delta


def test_error_paths():
    cfg = O.CONFIGS["tiny"]
    w = {k: v.to(DEV, BF) for k, v in O.make_weights(cfg, seed=1).items()}
    from helpers import desc_from_cfg
    eng = _b2.Engine(desc_from_cfg(cfg, max_batch=2, max_seq=64), DEV)
    for k, v in w.items():
        eng.set_weight(k, v)
    with pytest.raises(ValueError, match="not finalized"):
        eng.enable_nf4()
    eng.finalize()
    kv = eng.new_kv(1, 64)
    with pytest.raises(ValueError, match="KV cache"):
        eng.enable_nf4()
    kv.close()
    eng.enable_nf4()
    eng.enable_nf4()  # no-op
    with pytest.raises(ValueError, match="NF4"):
        eng.set_weight("model.layers.0.mlp.down_proj.weight", w["model.layers.0.mlp.down_proj.weight"])
    with pytest.raises(ValueError, match="NF4"):
        eng.set_weight("model.mm_projector.2.weight", w["model.mm_projector.2.weight"])
    with pytest.raises(ValueError, match="NF4"):
        eng.enable_fp8_decode()
    eng.set_weight("model.norm.weight", w["model.norm.weight"])  # not a quantised key
    eng.close()
    eng = make_engine(cfg, w, max_batch=2, max_seq=64)
    eng.enable_fp8_decode()
    with pytest.raises(ValueError, match="fp8"):
        eng.enable_nf4()
    eng.close()


# ---------------------------------------------------------------------------------------------- strict greedy ids
@pytest.fixture(scope="module")
def conditioned_7b():
    """NF4 engine at 7B shapes, 32 layers, on condition_weights(w); oracle ids on nf4_weights of the same weights."""
    torch.set_num_threads(min(32, os.cpu_count() or 1))
    cfg = dict(O.CONFIGS["llava-1.5-7b"], vit_layers=1)
    w = O.condition_weights(dev_weights(cfg, seed=0), cfg, seed=0)
    eng = make_engine(cfg, w, max_batch=12, max_seq=128, max_images=1)
    eng.enable_nf4()
    wq = Q.nf4_weights(w, cfg)
    del w
    w_cpu = {k: v.cpu().float() for k, v in wq.items() if not k.startswith(O.VT)}
    del wq
    g = torch.Generator().manual_seed(5)
    prompt = torch.randint(3, cfg["vocab"], (1, 24), generator=g)
    logits, okv = O.llama_forward(w_cpu, w_cpu["model.embed_tokens.weight"][prompt], cfg, last_only=True)
    want = []
    for _ in range(16):
        nxt = logits[:, -1].argmax(-1)
        want.append(int(nxt))
        logits, okv = O.llama_forward(w_cpu, w_cpu["model.embed_tokens.weight"][nxt][:, None], cfg, kv=okv, last_only=True)
    del w_cpu, okv
    yield eng, prompt, want
    eng.close()


@pytest.mark.parametrize("B,kv_dtype", [(1, "bf16"), (4, "bf16"), (12, "bf16"), (4, "e4m3")])
def test_strict_greedy_ids_7b_32_layers(conditioned_7b, B, kv_dtype):
    eng, prompt, want = conditioned_7b
    kv = eng.new_kv(B, 128, dtype=kv_dtype)
    ids = prompt.repeat(B, 1).to(torch.int32).reshape(-1).to(DEV)
    lg = eng.prefill(kv, eng.splice(ids, None, B, 24), None, _b2.LOGITS_LAST)
    first = eng.argmax(lg)
    rest = eng.decode_greedy(kv, first, 15).cpu()
    got = torch.cat([first.cpu()[None], rest]).t().tolist()
    kv.close()
    for r in got:
        assert r == want, (B, kv_dtype, r, want)


def test_strict_greedy_ids_through_continuous_batching(conditioned_7b):
    """Two slots; slot 0 is freed mid-run and refilled while slot 1 keeps decoding; every request reproduces the oracle ids."""
    eng, prompt, want = conditioned_7b
    kv = eng.new_kv(2, 128)
    eng.batch_begin(kv, 2)
    got, state = {"a": [], "b": [], "c": []}, {"step": 0}
    ids = prompt.to(torch.int32).reshape(-1).to(DEV)

    def admit(slot, name):
        lg = eng.prefill(kv, eng.splice(ids, None, 1, 24), [24], _b2.LOGITS_LAST, slot0=slot)
        first = int(lg.argmax(-1))
        eng.batch_set_row(kv, slot, True, None, first)
        got[name].append(first)

    def step(rows):
        eng.stream_enqueue(kv, 1)
        toks = eng.stream_wait(kv, state["step"], 2)
        state["step"] += 1
        for slot, name in rows.items():
            got[name].append(int(toks[slot]))

    admit(0, "a")
    admit(1, "b")
    for _ in range(5):
        step({0: "a", 1: "b"})
    eng.batch_set_row(kv, 0, False)
    step({1: "b"})
    admit(0, "c")
    for _ in range(6):
        step({0: "c", 1: "b"})
    step({1: "b"})
    kv.close()
    assert got["a"] == want[:6] and got["b"] == want[:14] and got["c"] == want[:7], (got, want)


# ---------------------------------------------------------------------------------------------- loader surface
_LOAD_4BIT = textwrap.dedent("""
    import sys, torch
    sys.path[:0] = [sys.argv[1], sys.argv[2], sys.argv[2] + "/tests"]
    from llava.model.builder import load_pretrained_model
    from llava.constants import IMAGE_TOKEN_INDEX
    from oracle import llava_oracle as O
    from oracle import nf4_oracle as Q
    from helpers import make_model
    ck = sys.argv[3]
    tokenizer, model, image_processor, _ = load_pretrained_model(ck, None, "llava-b2test-7b", load_4bit=True)
    assert model.config.b2_weight_format == "nf4"
    cfg = dict(O.CONFIGS["tiny"], vocab=320)
    w = {k: v.to(torch.float16).to(torch.bfloat16) for k, v in O.condition_weights(O.make_weights(cfg, seed=4), cfg, seed=4).items()}
    direct = make_model(cfg, Q.nf4_weights(w, cfg), max_batch=4, max_seq=256)
    for m in (model, direct):
        m.config.b2_beam_search = 4
        m.config.b2_prefix_cache = True
    a, b = tokenizer("what is in the").input_ids, tokenizer("picture").input_ids[1:]
    ids = torch.tensor([a + [IMAGE_TOKEN_INDEX] + b]).cuda()
    from PIL import Image
    img = Image.new("RGB", (80, 60), (200, 30, 90))
    pixels = image_processor.preprocess(img, return_tensors="pt")["pixel_values"].half().cuda()
    res = {}
    for name, m in (("nf4", model), ("direct", direct)):
        g = m.generate(ids, images=pixels, do_sample=False, max_new_tokens=12, eos_token_id=[])
        turn2 = torch.cat([g, torch.tensor([tokenizer("and then").input_ids[1:]]).cuda()], dim=1)
        g2 = m.generate(turn2, images=pixels, do_sample=False, max_new_tokens=8, eos_token_id=[])  # reuses turn 1's rows
        beam = m.generate(ids, images=pixels, do_sample=False, num_beams=4, max_new_tokens=8, eos_token_id=[])
        res[name] = (g.cpu(), beam.cpu(), g2.cpu())
    assert model._pool.reused_positions > 0
    for x, y in zip(res["nf4"], res["direct"]):
        assert torch.equal(x, y), (x, y)
    print("load-4bit-ok")
""")


def test_load_pretrained_model_load_4bit(tmp_path, repo_root):
    from test_checkpoint_dir import write_fake_hf_cache, write_llava_checkpoint

    cfg = dict(O.CONFIGS["tiny"], vocab=320)
    w = O.condition_weights(O.make_weights(cfg, seed=4), cfg, seed=4)
    hf_home, ck = str(tmp_path / "hf_home"), str(tmp_path / "llava-b2test-7b")
    write_fake_hf_cache(hf_home, cfg, w)
    write_llava_checkpoint(ck, cfg, w)
    env = dict(os.environ, HF_HOME=hf_home, HF_HUB_OFFLINE="1", TRANSFORMERS_OFFLINE="1")
    env.pop("HF_HUB_CACHE", None)
    r = subprocess.run([sys.executable, "-c", _LOAD_4BIT, os.path.join(repo_root, "llava-plus-codebase_b200"), repo_root, ck],
                       env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "load-4bit-ok" in r.stdout, (r.stdout[-1500:], r.stderr[-3000:])
