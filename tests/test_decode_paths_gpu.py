"""GPU: the paths of the multi-kernel decode step, one case per row of decode_plan's table (csrc/model.cu).

Each case prefills a fresh cache and checks that the eager first step at its batch and the graph-replayed steps after it
launch the same kernels, as many as the path implies, and that an eager step and a replayed step from the same prefill give
bit-equal logits. Knobs are set before the cache is created and are read when its step is launched eagerly or captured."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from helpers import make_engine  # noqa: E402
from llava import _b2  # noqa: E402
from oracle import llava_oracle as O  # noqa: E402
from test_nf4_gpu import CFG2, dev_weights, rnd  # noqa: E402

CFGS = {"7b": CFG2, "13b": dict(O.CONFIGS["llava-1.5-13b"], layers=2, vit_layers=1)}
MAX_BATCH, MAX_SEQ, PROMPT = 16, 128, 40

# kernels per layer: GEMV / GEMV_NF4 fuse the norms (qkv, attn, o, gate/up, down); SKINNY / TILE add two RMSNorms; an NF4
# model off GEMV_NF4 dequantises the layer first; SKINNY_FP8 quantises the O and down inputs as well
PER_LAYER = {"GEMV": 5, "GEMV_NF4": 5, "SKINNY": 7, "TILE": 7, "NF4_DENSE": 8, "SKINNY_FP8": 9}

# id: (model, weights, kv dtype, B, env, layer path, head kernels)
CASES = {
    "bf16-skinny-b8": ("7b", "bf16", "bf16", 8, {}, "SKINNY", 2),
    "bf16-skinny-b16": ("7b", "bf16", "bf16", 16, {}, "SKINNY", 2),
    "bf16-tile-b16": ("7b", "bf16", "bf16", 16, {"B2_DECODE_SKINNY": "0"}, "TILE", 2),
    "bf16-gemv-b1-e4m3kv": ("7b", "bf16", "e4m3", 1, {}, "GEMV", 1),
    "bf16-gemv-b4-e4m3kv": ("7b", "bf16", "e4m3", 4, {}, "GEMV", 1),
    "bf16-gemv-b8-e4m3kv": ("7b", "bf16", "e4m3", 8, {"B2_DECODE_SKINNY": "0"}, "GEMV", 1),
    "fp8-skinny8-b16": ("7b", "fp8", "bf16", 16, {}, "SKINNY_FP8", 2),
    "nf4-gemv4-b1": ("7b", "nf4", "bf16", 1, {}, "GEMV_NF4", 1),
    "nf4-gemv4-b4": ("7b", "nf4", "bf16", 4, {}, "GEMV_NF4", 1),
    "nf4-13b-skinny-b8": ("13b", "nf4", "bf16", 8, {}, "NF4_DENSE", 2),
    "nf4-tile-b16": ("7b", "nf4", "bf16", 16, {"B2_DECODE_SKINNY": "0"}, "NF4_DENSE", 2),
}


@pytest.fixture(scope="module")
def engines():
    """Engines by (model, weight format), built on first use: 2 layers, V = 32000."""
    built = {}

    def get(model, fmt):
        if (model, fmt) not in built:
            cfg = CFGS[model]
            eng = make_engine(cfg, dev_weights(cfg, seed=3), max_batch=MAX_BATCH, max_seq=MAX_SEQ, max_images=1)
            if fmt == "fp8":
                eng.enable_fp8_decode()
            elif fmt == "nf4":
                eng.enable_nf4()
            built[(model, fmt)] = eng
        return built[(model, fmt)]

    yield get
    for eng in built.values():
        eng.close()


def _step(eng, kv, tok):
    before = _b2.launch_count()
    logits = eng.decode_step(kv, tok).clone()
    torch.cuda.synchronize()
    return logits, _b2.launch_count() - before


@pytest.mark.parametrize("case", list(CASES))
def test_eager_and_replayed_steps_launch_the_plan_and_agree(engines, case, monkeypatch):
    model, fmt, kv_dtype, B, env, path, head = CASES[case]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    cfg = CFGS[model]
    eng = engines(model, fmt)
    want = 1 + cfg["layers"] * PER_LAYER[path] + head + 1  # embed, layers, head, sample_publish
    emb = rnd(B, PROMPT, cfg["hidden"], seed=60 + B)
    kv = eng.new_kv(B, MAX_SEQ, dtype=kv_dtype)
    tok = eng.argmax(eng.prefill(kv, emb, None, _b2.LOGITS_LAST))
    _step(eng, kv, tok)  # the cache's first step also uploads the sampling state
    monkeypatch.setenv("B2_KV_RESET_GRAPH", "1")  # the reset also forgets the warm batch: the next step is eager again
    kv.reset()
    monkeypatch.delenv("B2_KV_RESET_GRAPH")
    assert torch.equal(eng.argmax(eng.prefill(kv, emb, None, _b2.LOGITS_LAST)), tok)
    eager, n_eager = _step(eng, kv, tok)
    kv.reset()
    eng.prefill(kv, emb, None, _b2.LOGITS_LAST)
    replayed, n_capture = _step(eng, kv, tok)  # captures the graph, then replays it
    _, n_replay = _step(eng, kv, eager.argmax(-1).to(torch.int32))
    kv.close()
    assert (n_eager, n_capture, n_replay) == (want, want, want), (case, n_eager, n_capture, n_replay, want)
    assert torch.equal(eager, replayed), case


def test_bf16_cache_at_batch_1_takes_the_megakernel(engines):
    eng = engines("7b", "bf16")
    kv = eng.new_kv(1, MAX_SEQ)
    first = eng.argmax(eng.prefill(kv, rnd(1, PROMPT, CFG2["hidden"], seed=70), None, _b2.LOGITS_LAST))
    eng.decode_greedy(kv, first, 2)  # the cache's first call also uploads the sampling state
    kv.reset()
    first = eng.argmax(eng.prefill(kv, rnd(1, PROMPT, CFG2["hidden"], seed=70), None, _b2.LOGITS_LAST))
    before = _b2.launch_count()
    eng.decode_greedy(kv, first, 8)
    torch.cuda.synchronize()
    launches = _b2.launch_count() - before
    kv.close()
    assert launches == 8, launches
