"""A/B of the bf16 and the e4m3 KV cache on the decode step (LLaVA-1.5-7B shapes, random weights from a seed), in ONE process:

  step      per (batch, context): both caches are prefilled with the same inputs, then bf16 and e4m3 runs of `--new` greedy steps
            alternate (decode isolated: prefill -> synchronise -> steps timed with CUDA events); first with bf16 weights, then
            the shapes at batch >= 32 again with e4m3 weights (b2_model_enable_fp8_decode). Bytes per step are computed from
            shapes: the weight stream + B * (context + 1) * bytes per token of the cache in use (scales included).
  kernel    decode attention alone (b2_op_decode_attn vs b2_op_decode_attn_e4m3, one layer, 32 heads) at the same shapes, so a
            shortfall of the step can be attributed to the attention kernel or to the rest of the step.
  capacity  the 7B, batch 64, 2112-token e4m3 cache (its bf16 form, 68 GB, does not fit an 80 GB card beside the weights):
            created once, one slot prefilled, a few decode steps; reports b2_kv_bytes.

Needs a GPU (there is no fallback). Prints one JSON object per measurement and the card's name and power limit.

    python scripts/kv_fp8_bench.py [--shapes 8x704,32x1600] [--new 64] [--out FILE]
"""
import argparse
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (path setup, model table, algorithmic_work)

import torch  # noqa: E402

M7 = bench.MODELS["7b"]
KV_TOKEN_BYTES = {"bf16": 2 * 2 * M7["hidden"] * M7["layers"],                          # 524 288
                  "e4m3": 2 * (M7["hidden"] + 4 * M7["heads"]) * M7["layers"]}          # 270 336: bytes + one fp32 scale per head
WS_ROWS_SEQ = 256   # the engine's workspace holds max_batch * 256 rows: long prompts are prefilled a few slots at a time


def step_bytes(B, context, kv_dtype, fp8_weights):
    return bench.algorithmic_work(M7, B, 1, 2, fp8=fp8_weights)["w_bytes"] + B * (context + 1) * KV_TOKEN_BYTES[kv_dtype]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or f"nvidia-smi failed: {q.stderr.strip()[:200]}"


def build_engine(dev, max_batch):
    """7B engine with seeded random weights, generated tensor by tensor on the device (no second copy of the model)."""
    from llava import _b2
    from oracle.llava_oracle import init_std, make_config, weight_shapes  # shapes / init table only

    cfg = make_config(hidden=M7["hidden"], inter=M7["inter"], layers=M7["layers"], heads=M7["heads"])
    desc = dict(image_size=cfg["image_size"], patch_size=cfg["patch_size"], vit_hidden=cfg["vit_hidden"], vit_inter=cfg["vit_inter"],
                vit_layers=cfg["vit_layers"], vit_heads=cfg["vit_heads"], vit_select_layer=cfg["select_layer"], vit_ln_eps=cfg["vit_eps"],
                hidden=cfg["hidden"], inter=cfg["inter"], layers=cfg["layers"], heads=cfg["heads"], vocab=cfg["vocab"],
                rms_eps=cfg["rms_eps"], rope_theta=cfg["rope_theta"], max_batch=max_batch, max_seq=WS_ROWS_SEQ, max_images=1)
    eng = _b2.Engine(desc, dev)
    gen = torch.Generator(device=dev).manual_seed(0)
    for key, shape, kind in weight_shapes(cfg):
        t = torch.empty(*shape, device=dev, dtype=torch.bfloat16).normal_(0.0, init_std(kind, shape), generator=gen)
        if kind == "g":
            t.add_(1.0)
        eng.set_weight(key, t)
    eng.finalize()
    return eng


def prefill(eng, kv, embeds, B, S):
    """Fill slots 0..B-1 with the same S-token prompts, a workspace-full of slots at a time; returns the first tokens [B]."""
    from llava import _b2

    per = max(1, min(B, eng.desc.max_batch * WS_ROWS_SEQ // S))
    first = []
    for s0 in range(0, B, per):
        n = min(per, B - s0)
        first.append(eng.argmax(eng.prefill(kv, embeds[s0:s0 + n], None, _b2.LOGITS_LAST, slot0=s0)))
    return torch.cat(first)


def measure_steps(eng, dev, shapes, new, reps, fp8_weights, emit):
    g = torch.Generator(device=dev).manual_seed(1)
    for B, ctx in shapes:
        smax = ctx + 16 + reps * new + 8
        need = {d: B * smax * KV_TOKEN_BYTES[d] for d in ("bf16", "e4m3")}
        free = torch.cuda.mem_get_info(dev)[0]
        dtypes = ["bf16", "e4m3"] if need["bf16"] + need["e4m3"] + (3 << 30) < free else ["e4m3"]
        embeds = (torch.randn(B, ctx, M7["hidden"], device=dev, generator=g) * 0.5).to(torch.bfloat16)
        kvs, tok = {}, {}
        for d in dtypes:
            kvs[d] = eng.new_kv(B, smax, dtype=d)
            tok[d] = prefill(eng, kvs[d], embeds, B, ctx)
            tok[d] = eng.decode_greedy(kvs[d], tok[d], 16)[-1]      # warm-up: eager step, graph capture, replays
        del embeds
        torch.cuda.synchronize()
        times = {d: [] for d in dtypes}
        for r in range(reps):                                       # alternate the formats; the context grows by `new` per rep
            for d in dtypes:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                out = eng.decode_greedy(kvs[d], tok[d], new)
                e1.record()
                torch.cuda.synchronize()
                tok[d] = out[-1]
                times[d].append(e0.elapsed_time(e1) / new)
        mid = reps // 2                                             # the headline is the middle rep, at its own mean context
        avg_ctx = ctx + 16 + mid * new + (new - 1) / 2.0
        for d in ("bf16", "e4m3"):
            if d not in dtypes:
                emit(dict(kind="step", B=B, context=ctx, weights="e4m3" if fp8_weights else "bf16", kv=d,
                          skipped=f"a {need[d] / 2**30:.1f} GiB cache does not fit beside the other one"))
                continue
            ms = times[d][mid]
            nbytes = step_bytes(B, avg_ctx, d, fp8_weights)
            emit(dict(kind="step", B=B, context=ctx, avg_context_timed=avg_ctx, weights="e4m3" if fp8_weights else "bf16", kv=d,
                      ms_per_step=round(ms, 4), all_ms=[round(t, 4) for t in times[d]], steps_per_rep=new,
                      bytes_per_step=int(nbytes), gb_per_s=round(nbytes / ms / 1e6, 1), kv_cache_bytes=kvs[d].nbytes))
            kvs[d].close()
        torch.cuda.empty_cache()


def measure_kernel(dev, shapes, launches, emit):
    from llava import _b2

    lib, H, D = _b2.load_library(), M7["heads"], 128
    P, S = _b2.ptr, _b2.stream_ptr
    g = torch.Generator(device=dev).manual_seed(2)
    for B, ctx in shapes:
        smax = (ctx + 8) // 4 * 4
        qkv = torch.randn(B, 3 * H * D, device=dev, generator=g).to(torch.bfloat16)
        cur = torch.full((B,), ctx, device=dev, dtype=torch.int32)
        out = torch.empty(B, H * D, device=dev, dtype=torch.bfloat16)
        kc = torch.randn(B, H, smax, D, device=dev, generator=g).to(torch.bfloat16)
        vc = torch.randn(B, H, smax, D, device=dev, generator=g).to(torch.bfloat16)
        k8 = torch.empty(B, H, smax, D, device=dev, dtype=torch.uint8)
        v8 = torch.empty_like(k8)
        ks, vs = torch.empty(B, H, smax, device=dev), torch.empty(B, H, smax, device=dev)
        _b2.check(lib.b2_op_kv_quantize_e4m3(P(kc), P(vc), P(k8), P(v8), P(ks), P(vs), None, B, smax, H, smax, S()))
        res = {}
        for d, code in (("bf16", _b2.KV_BF16), ("e4m3", _b2.KV_E4M3)):
            ns = lib.b2_op_decode_attn_nsplit(B, H, smax, code)
            scratch = torch.zeros(lib.b2_op_decode_attn_scratch_bytes(B, H, ns), device=dev, dtype=torch.uint8)
            if d == "bf16":
                run = lambda ns=ns, scratch=scratch: lib.b2_op_decode_attn(P(qkv), P(kc), P(vc), P(cur), P(out), P(scratch), B, H, smax,
                                                                           ns, 10000.0, 1 / math.sqrt(D), S())
            else:
                run = lambda ns=ns, scratch=scratch: lib.b2_op_decode_attn_e4m3(P(qkv), P(k8), P(v8), P(ks), P(vs), P(cur), P(out),
                                                                                P(scratch), B, H, smax, ns, 10000.0, 1 / math.sqrt(D), S())
            res[d] = (run, ns, [])
        for _ in range(3):                                      # alternate; the first round is the warm-up
            for d in ("bf16", "e4m3"):
                run, ns, ts = res[d]
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(launches):
                    _b2.check(run())
                e1.record()
                torch.cuda.synchronize()
                ts.append(e0.elapsed_time(e1) / launches * 1e3)
        for d in ("bf16", "e4m3"):
            _, ns, ts = res[d]
            us = min(ts[1:])
            nbytes = B * H * (ctx + 1) * (512 if d == "bf16" else 264)
            emit(dict(kind="decode_attn_kernel", B=B, context=ctx, kv=d, nsplit=ns, us_per_launch=round(us, 2),
                      bytes_per_launch=nbytes, gb_per_s=round(nbytes / us / 1e3, 1), launches=launches))
        del kc, vc, k8, v8, ks, vs
        torch.cuda.empty_cache()


def measure_capacity(eng, dev, emit):
    B, smax, S = 64, 2112, 704
    line = dict(kind="capacity", B=B, max_seq=smax, kv="e4m3", bf16_cache_bytes_computed=B * smax * KV_TOKEN_BYTES["bf16"])
    try:
        kv = eng.new_kv(B, smax, dtype="e4m3")
    except RuntimeError as e:       # reported, not retried
        emit(dict(line, ok=False, error=str(e)[:200]))
        return
    g = torch.Generator(device=dev).manual_seed(3)
    embeds = (torch.randn(1, S, M7["hidden"], device=dev, generator=g) * 0.5).to(torch.bfloat16)
    first = prefill(eng, kv, embeds, 1, S)
    toks = eng.decode_greedy(kv, first, 4)
    torch.cuda.synchronize()
    emit(dict(line, ok=True, kv_cache_bytes=kv.nbytes, prefilled_slots=1, decode_steps=4, lengths=kv.lengths(1), tokens=toks.flatten().tolist()))
    kv.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="8x704,8x1600,32x704,32x1600,64x704,64x1600", help="batch x context, comma separated")
    ap.add_argument("--new", type=int, default=64, help="decode steps per timed run")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--launches", type=int, default=200, help="launches per timing of the attention kernel alone")
    ap.add_argument("--out", default=os.devnull, help="also append every result line to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("kv_fp8_bench needs a CUDA device: there is nothing to measure without one")
    shapes = [tuple(int(x) for x in s.split("x")) for s in a.shapes.split(",")]
    if os.path.dirname(a.out):
        os.makedirs(os.path.dirname(a.out), exist_ok=True)
    fout = open(a.out, "a")

    def emit(d):
        s = json.dumps(d)
        print(s, flush=True)
        fout.write(s + "\n")
        fout.flush()

    dev = torch.device("cuda:0")
    torch.cuda.set_device(0)
    emit(dict(kind="card", name_powerlimit_maxsmclock=card(), kv_bytes_per_token=KV_TOKEN_BYTES))
    stream = torch.cuda.Stream(device=dev)
    with torch.cuda.stream(stream), torch.no_grad():
        measure_kernel(dev, shapes, a.launches, emit)
        eng = build_engine(dev, max(b for b, _ in shapes + [(64, 0)]))
        measure_steps(eng, dev, shapes, a.new, a.reps, False, emit)
        eng.enable_fp8_decode()
        measure_steps(eng, dev, [s for s in shapes if s[0] >= 32], a.new, a.reps, True, emit)
        measure_capacity(eng, dev, emit)
        eng.close()


if __name__ == "__main__":
    main()
