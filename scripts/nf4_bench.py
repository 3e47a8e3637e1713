"""bf16 against NF4 decoder weights (load_4bit), LLaVA-1.5-7B shapes, seeded random weights, both engines in ONE process:

  step      decode step at batch 1, 4, 8, 16, 32 after a 704-row prefill: runs of `--new` greedy steps alternate between the
            engines (prefill -> synchronise -> steps timed with CUDA events), `--reps` per engine, the middle one reported.
            bf16: megakernel at batch 1 and 2, GEMV graph below 7, stream-K GEMM above; NF4: gemv_nf4 at batch <= 8, above it
            each layer is dequantised into a bf16 scratch in front of the same stream-K GEMM.
  prefill   S = 704 prefill at batch 1 (NF4: one dequantisation per layer in front of the wgmma GEMMs), and a 64-row chunk at
            start 704 (b2_prefill_at); median of `--reps` alternating runs.
  gemv      gemv_nf4 against gemv_bf16 on the four 7B decode shapes at batch 1 and 8, 200 launches per timing; GB/s are the
            algorithmic weight bytes (bf16: 2 N K; NF4: N K / 2 codes + 4 N K / 64 absmax) over the time.
  dequant   dequantize_nf4 alone on one 7B layer's four matrices through b2_op_dequantize_nf4 (canonical order, one launch per
            matrix; the engine dequantises the same bytes in GEMV order, four matrices per launch), 200 repeats per timing; GB/s
            are the code + absmax bytes read plus the bf16 bytes written.
  13b       the 13B decode step at batch 1, bf16 (megakernel) against NF4 (gemv_nf4).
  bytes     b2_model_weight_bytes of each engine.

Needs a GPU (there is no fallback). Prints one JSON object per measurement, and the card's name, power limit and maximum SM
clock read in the same run.

    python scripts/nf4_bench.py [--batches 1,4,8,16,32] [--new 32] [--reps 3] [--skip-13b] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "llava-plus-codebase_b200"))

import torch  # noqa: E402

CTX = 704


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or f"nvidia-smi failed: {q.stderr.strip()[:200]}"


def model_cfg(name):
    from oracle.llava_oracle import CONFIGS
    return CONFIGS["llava-1.5-7b" if name == "7b" else "llava-1.5-13b"]


def build_engine(dev, cfg, max_batch, max_seq, nf4):
    """Engine with seeded random weights, generated tensor by tensor on the device (the same weights for both formats)."""
    from llava import _b2
    from oracle.llava_oracle import init_std, weight_shapes

    desc = dict(image_size=cfg["image_size"], patch_size=cfg["patch_size"], vit_hidden=cfg["vit_hidden"], vit_inter=cfg["vit_inter"],
                vit_layers=cfg["vit_layers"], vit_heads=cfg["vit_heads"], vit_select_layer=cfg["select_layer"], vit_ln_eps=cfg["vit_eps"],
                hidden=cfg["hidden"], inter=cfg["inter"], layers=cfg["layers"], heads=cfg["heads"], vocab=cfg["vocab"],
                rms_eps=cfg["rms_eps"], rope_theta=cfg["rope_theta"], max_batch=max_batch, max_seq=max_seq, max_images=1)
    eng = _b2.Engine(desc, dev)
    gen = torch.Generator(device=dev).manual_seed(0)
    for key, shape, kind in weight_shapes(cfg):
        t = torch.empty(*shape, device=dev, dtype=torch.bfloat16).normal_(0.0, init_std(kind, shape), generator=gen)
        if kind == "g":
            t.add_(1.0)
        eng.set_weight(key, t)
        del t
    eng.finalize()
    if nf4:
        eng.enable_nf4()
    torch.cuda.empty_cache()
    return eng


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    r = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), r


def prefill_slots(eng, kv, embeds, B):
    """Prefill slots 0..B-1 with the same prompts, as many slots per call as the workspace holds; returns the first tokens."""
    from llava import _b2

    S = embeds.shape[1]
    per = max(1, min(B, eng.desc.max_batch * eng.desc.max_seq // S))
    first = []
    for s0 in range(0, B, per):
        n = min(per, B - s0)
        first.append(eng.argmax(eng.prefill(kv, embeds[s0:s0 + n], None, _b2.LOGITS_LAST, slot0=s0)))
    return torch.cat(first)


def measure_steps(engines, dev, h, batches, new, reps, emit, tag="7b"):
    g = torch.Generator(device=dev).manual_seed(1)
    for B in batches:
        embeds = (torch.randn(B, CTX, h, device=dev, generator=g) * 0.5).to(torch.bfloat16)
        times = {k: [] for k in engines}
        for r in range(reps + 1):  # rep 0 warms up (eager step, graph capture)
            for name, eng in engines.items():
                kv = eng.new_kv(B, CTX + new + 8)
                tok = prefill_slots(eng, kv, embeds, B)
                torch.cuda.synchronize()
                ms, _ = timed(lambda: eng.decode_greedy(kv, tok, new))
                if r:
                    times[name].append(ms / new)
                kv.close()
        for name in engines:
            t = sorted(times[name])
            emit(dict(kind="step", model=tag, weights=name, B=B, context=CTX, steps_per_run=new, ms_per_step=round(t[len(t) // 2], 4),
                      all_ms=[round(x, 4) for x in times[name]]))
        del embeds
        torch.cuda.empty_cache()


def measure_prefill(engines, dev, h, reps, emit):
    from llava import _b2

    g = torch.Generator(device=dev).manual_seed(2)
    embeds = (torch.randn(1, CTX, h, device=dev, generator=g) * 0.5).to(torch.bfloat16)
    chunk = (torch.randn(1, 64, h, device=dev, generator=g) * 0.5).to(torch.bfloat16)
    res = {k: {"full": [], "chunk": []} for k in engines}
    for r in range(reps + 1):
        for name, eng in engines.items():
            kv = eng.new_kv(1, CTX + 72)
            ms, _ = timed(lambda: eng.prefill(kv, embeds, None, _b2.LOGITS_LAST))
            ms2, _ = timed(lambda: eng.prefill(kv, chunk, None, _b2.LOGITS_LAST, start=[CTX]))
            if r:
                res[name]["full"].append(ms)
                res[name]["chunk"].append(ms2)
            kv.close()
    for name in engines:
        for what, label in (("full", "prefill S=704"), ("chunk", "64-row chunk at start 704")):
            t = sorted(res[name][what])
            emit(dict(kind="prefill", weights=name, what=label, ms=round(t[len(t) // 2], 3), all_ms=[round(x, 3) for x in res[name][what]]))


def measure_gemv(dev, launches, emit):
    from llava import _b2
    from oracle import nf4_oracle as Q

    lib = _b2.load_library()
    S = _b2.stream_ptr
    P = _b2.ptr
    for N, K, act in ((12288, 4096, 0), (4096, 4096, 0), (22016, 4096, _b2.ACT_SWIGLU), (4096, 11008, 0)):
        W = (torch.randn(N, K, device=dev) * K ** -0.5).to(torch.bfloat16)
        q, a = Q.quantize_nf4(W)
        codes = Q.pack_nf4(q, "gemv")
        n_out = N // 2 if act else N
        for B in (1, 8):
            x = torch.randn(B, K, device=dev).to(torch.bfloat16)
            out = torch.empty(B, n_out, device=dev, dtype=torch.bfloat16)
            calls = {
                "bf16": lambda: lib.b2_op_gemv(P(x), K, P(W), K, None, 0.0, None, 0, P(out), n_out, 0, B, N, K, act, S()),
                "nf4": lambda: lib.b2_op_gemv_nf4(P(x), K, P(codes), P(a), None, 0.0, None, 0, P(out), n_out, B, N, K, act, S()),
            }
            nbytes = {"bf16": 2 * N * K, "nf4": Q.nf4_linear_bytes(N, K)}
            best = {}
            for rnd in range(3):  # alternate; the first round warms up
                for name, fn in calls.items():
                    def run():
                        for _ in range(launches):
                            rc = fn()
                            assert rc == 0, _b2.last_error()
                    ms, _ = timed(run)
                    if rnd:
                        best[name] = min(best.get(name, 1e9), ms / launches)
            for name in calls:
                us = best[name] * 1e3
                emit(dict(kind="gemv", weights=name, N=N, K=K, act="swiglu" if act else "none", B=B, us=round(us, 2),
                          gb_per_s=round(nbytes[name] / us / 1e3, 1)))
        del W, q, a, codes
        torch.cuda.empty_cache()


def measure_dequant(dev, launches, emit):
    from llava import _b2
    from oracle import nf4_oracle as Q

    lib = _b2.load_library()
    h, I = 4096, 11008
    shapes = [(3 * h, h), (h, h), (2 * I, h), (h, I)]
    codes = [torch.randint(0, 256, (N, K // 2), device=dev, dtype=torch.uint8) for N, K in shapes]
    absmax = [torch.rand(N, K // 64, device=dev) for N, K in shapes]
    out = [torch.empty(N, K, device=dev, dtype=torch.bfloat16) for N, K in shapes]

    def run():
        for _ in range(launches):
            for c, a, o, (N, K) in zip(codes, absmax, out, shapes):
                rc = lib.b2_op_dequantize_nf4(_b2.ptr(c), _b2.ptr(a), N, K, _b2.ptr(o), _b2.stream_ptr())
                assert rc == 0, _b2.last_error()

    timed(run)
    ms = min(timed(run)[0] for _ in range(2)) / launches
    nbytes = sum(Q.nf4_linear_bytes(N, K) + 2 * N * K for N, K in shapes)
    emit(dict(kind="dequant", what="one 7B layer (4 matrices, canonical order, one launch each)", ms=round(ms, 4),
              gb_per_s=round(nbytes / ms / 1e6, 1)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,4,8,16,32")
    ap.add_argument("--new", type=int, default=32)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--skip-13b", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("nf4_bench needs a CUDA device (sm_90a); there is no CPU path")
    dev = torch.device("cuda", 0)
    rows = []

    def emit(d):
        rows.append(d)
        print(json.dumps(d), flush=True)

    emit(dict(kind="card", name_power_limit_max_sm_clock=card()))
    batches = [int(b) for b in a.batches.split(",")]
    cfg = model_cfg("7b")
    engines = {"bf16": build_engine(dev, cfg, max(batches), CTX + a.new + 96, False),
               "nf4": build_engine(dev, cfg, max(batches), CTX + a.new + 96, True)}
    emit(dict(kind="weight_bytes", model="7b", **{k: e.weight_bytes() for k, e in engines.items()}))
    measure_steps(engines, dev, cfg["hidden"], batches, a.new, a.reps, emit)
    measure_prefill(engines, dev, cfg["hidden"], a.reps, emit)
    for e in engines.values():
        e.close()
    del engines
    torch.cuda.empty_cache()
    measure_gemv(dev, a.launches, emit)
    measure_dequant(dev, a.launches, emit)
    if not a.skip_13b:
        cfg = model_cfg("13b")
        engines = {"bf16": build_engine(dev, cfg, 1, CTX + a.new + 96, False),
                   "nf4": build_engine(dev, cfg, 1, CTX + a.new + 96, True)}
        emit(dict(kind="weight_bytes", model="13b", **{k: e.weight_bytes() for k, e in engines.items()}))
        measure_steps(engines, dev, cfg["hidden"], [1], a.new, a.reps, emit, tag="13b")
        for e in engines.values():
            e.close()
    emit(dict(kind="card", name_power_limit_max_sm_clock=card()))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
