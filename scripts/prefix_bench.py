"""Prefill at an offset into a live KV cache (b2_prefill_at) against a prefill from position 0, LLaVA-1.5-7B shapes, random
weights from a seed, batch 1, in ONE process:

  chat      a synthetic 4-turn conversation with one 336 px image: turn t's prompt is the image (576 rows) + 100 text tokens
            per turn so far + the 128-token answers of the earlier turns. Time to first token per turn, with reuse (the cache
            keeps the conversation: prefill of the rows not yet in it at their position, no image encode) and without (encode
            the image, prefill the whole prompt from position 0). The two alternate, three runs each; the median is reported.
            Between turns 128 greedy decode steps write the answer's rows (not timed).
  chunk     the chunk prefill alone: n in {16, 64, 256} new rows at start in {704, 1600}, and the weight-stream bound of one
            pass over the decoder weights at the data-sheet 3.35 TB/s (H100 SXM) beside it.
  attention the offset flash kernel alone (b2_op_flash_attn_kv: n queries over start + n keys, 32 heads) against the plain
            causal kernel over the whole start + n rows (b2_op_flash_attn), one layer.

Times are CUDA-event times around work that ends in a stream synchronise. Needs a GPU (there is no fallback). Prints one JSON
object per measurement and the card's name and power limit.

    python scripts/prefix_bench.py [--runs 3]
"""
import argparse
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (path setup, model table)

import torch  # noqa: E402

M7 = bench.MODELS["7b"]
MAX_SEQ = 2048
IMAGE_ROWS, TEXT_PER_TURN, ANSWER = 576, 100, 128
HBM_BYTES_PER_S = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or f"nvidia-smi failed: {q.stderr.strip()[:200]}"


def build_engine(dev):
    from llava import _b2
    from oracle.llava_oracle import init_std, make_config, weight_shapes  # shapes / init table only

    cfg = make_config(hidden=M7["hidden"], inter=M7["inter"], layers=M7["layers"], heads=M7["heads"])
    desc = dict(image_size=cfg["image_size"], patch_size=cfg["patch_size"], vit_hidden=cfg["vit_hidden"], vit_inter=cfg["vit_inter"],
                vit_layers=cfg["vit_layers"], vit_heads=cfg["vit_heads"], vit_select_layer=cfg["select_layer"], vit_ln_eps=cfg["vit_eps"],
                hidden=cfg["hidden"], inter=cfg["inter"], layers=cfg["layers"], heads=cfg["heads"], vocab=cfg["vocab"],
                rms_eps=cfg["rms_eps"], rope_theta=cfg["rope_theta"], max_batch=1, max_seq=MAX_SEQ, max_images=1)
    eng = _b2.Engine(desc, dev)
    gen = torch.Generator(device=dev).manual_seed(0)
    wbytes = 0
    for key, shape, kind in weight_shapes(cfg):
        t = torch.empty(*shape, device=dev, dtype=torch.bfloat16).normal_(0.0, init_std(kind, shape), generator=gen)
        if kind == "g":
            t.add_(1.0)
        if key.startswith("model.layers.") or key == "lm_head.weight":
            wbytes += t.numel() * 2
        eng.set_weight(key, t)
    eng.finalize()
    return eng, cfg, wbytes


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    out = fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b), out


def chat(eng, cfg, dev, runs, emit):
    from llava import _b2

    g = torch.Generator(device=dev).manual_seed(1)
    pixels = torch.randn(1, 3, cfg["image_size"], cfg["image_size"], device=dev, generator=g).to(torch.bfloat16)
    text = (torch.randn(1, MAX_SEQ, M7["hidden"], device=dev, generator=g) * 0.5).to(torch.bfloat16)
    kv_on, kv_off = eng.new_kv(1, MAX_SEQ), eng.new_kv(1, MAX_SEQ)
    times = {"on": [[] for _ in range(4)], "off": [[] for _ in range(4)]}
    for r in range(runs + 1):                      # run 0 warms every shape up and is not reported
        for mode in ("off", "on"):
            kv = kv_on if mode == "on" else kv_off
            kv.reset()
            cached = 0
            for t in range(4):
                S = IMAGE_ROWS + (t + 1) * TEXT_PER_TURN + t * ANSWER

                def turn():
                    if mode == "on" and t > 0:
                        # the cache holds the earlier turns but the last answer token: prefill from there
                        return eng.argmax(eng.prefill(kv, text[:, cached:S], None, _b2.LOGITS_LAST, start=[cached]))
                    feats = eng.encode_images(pixels)
                    emb = torch.cat([feats, text[:, IMAGE_ROWS:S]], dim=1)
                    kv.reset()
                    return eng.argmax(eng.prefill(kv, emb, None, _b2.LOGITS_LAST))
                ms, first = timed(turn)
                if r:
                    times[mode][t].append(ms)
                eng.decode_greedy(kv, first, ANSWER - 1)
                torch.cuda.synchronize()
                cached = S + ANSWER - 1
    for t in range(4):
        on, off = sorted(times["on"][t]), sorted(times["off"][t])
        S = IMAGE_ROWS + (t + 1) * TEXT_PER_TURN + t * ANSWER
        emit(dict(measure="ttft", turn=t + 1, prompt_rows=S, reuse_ms=on[len(on) // 2], fresh_ms=off[len(off) // 2],
                  ratio=round(on[len(on) // 2] / off[len(off) // 2], 3), runs=runs))
    kv_on.close(), kv_off.close()


def chunks(eng, dev, wbytes, emit):
    from llava import _b2

    g = torch.Generator(device=dev).manual_seed(2)
    x = (torch.randn(1, MAX_SEQ, M7["hidden"], device=dev, generator=g) * 0.5).to(torch.bfloat16)
    kv = eng.new_kv(1, MAX_SEQ)
    for start in (704, 1600):
        kv.reset()
        eng.prefill(kv, x[:, :start], None, _b2.LOGITS_NONE)
        for n in (16, 64, 256):
            run = lambda: eng.prefill(kv, x[:, start:start + n], None, _b2.LOGITS_LAST, start=[start])  # noqa: E731
            for _ in range(3):
                run()
            ms = sorted(timed(run)[0] for _ in range(10))
            emit(dict(measure="chunk_prefill", start=start, n=n, median_ms=round(ms[5], 3), min_ms=round(ms[0], 3),
                      weight_stream_bound_ms=round(wbytes / HBM_BYTES_PER_S * 1e3, 3)))
    kv.close()


def attention(dev, emit):
    from llava import _b2

    lib = _b2.load_library()
    H, D = M7["heads"], 128
    scale = 1 / math.sqrt(D)
    g = torch.Generator(device=dev).manual_seed(3)
    for start in (704, 1600):
        for n in (16, 64, 256):
            L = start + n
            q = torch.randn(1, n, H, D, device=dev, generator=g).to(torch.bfloat16)
            kc, vc = (torch.randn(1, H, L, D, device=dev, generator=g).to(torch.bfloat16) for _ in range(2))
            qf, kf, vf = (torch.randn(1, L, H, D, device=dev, generator=g).to(torch.bfloat16) for _ in range(3))
            o, of = torch.empty_like(q), torch.empty_like(qf)
            pos = torch.tensor([start], device=dev, dtype=torch.int32)
            res = {}
            for name, call in (
                    ("offset", lambda: lib.b2_op_flash_attn_kv(_b2.ptr(q), _b2.ptr(kc), _b2.ptr(vc), _b2.ptr(o), _b2.ptr(pos), None,
                                                               1, n, H, L, scale, _b2.stream_ptr())),
                    ("plain_whole", lambda: lib.b2_op_flash_attn(_b2.ptr(qf), _b2.ptr(kf), _b2.ptr(vf), _b2.ptr(of), None, 1, L, H, D,
                                                                 1, scale, _b2.stream_ptr()))):
                _b2.check(call(), name)
                ms, _ = timed(lambda: [call() for _ in range(50)])
                res[name] = round(ms / 50 * 1e3, 2)
            emit(dict(measure="attention_us", start=start, n=n, keys=L, offset_kernel_us=res["offset"],
                      plain_kernel_whole_sequence_us=res["plain_whole"]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prefix_bench needs a GPU")
    dev = torch.device("cuda", 0)
    emit = lambda d: print(json.dumps(d), flush=True)  # noqa: E731
    emit(dict(card=card()))
    eng, cfg, wbytes = build_engine(dev)
    chat(eng, cfg, dev, a.runs, emit)
    chunks(eng, dev, wbytes, emit)
    attention(dev, emit)
    eng.close()


if __name__ == "__main__":
    main()
