"""History-aware logits processing on the engine (LLaVA-1.5-7B shapes, random weights from a seed), in ONE process.

  step    per (context, batch): ms per decode step of a streamed generation (b2_stream_begin[_ex] + b2_stream_enqueue, CUDA
          events around the enqueued steps) for greedy, greedy + processors, sampled, and sampled + processors
          (no_repeat_ngram_size = 3, repetition_penalty = 1.2, top_k 50 / top_p 0.9 / T 0.8 when sampled). The variants alternate
          `reps` times on one cache whose context grows by `new` tokens per run; every row's history is a random prompt of
          `context` ids, so the n-gram scan covers the whole context.
  kernel  the selection kernel alone: sample_publish_kernel's device time per launch from torch.profiler over one run of
          each variant (a separate, profiled pass).

Needs a GPU (there is no fallback). Prints one JSON object per measurement and the card's name and power limit.

    python scripts/logits_proc_bench.py [--contexts 704,2048] [--batches 1,8,32] [--new 32] [--reps 3] [--out FILE]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(ROOT))
import kv_fp8_bench as kb  # noqa: E402  (7B engine from seeded weights, card())

import torch  # noqa: E402

VARIANTS = ("greedy", "greedy+proc", "sampled", "sampled+proc")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--contexts", default="704,2048")
    ap.add_argument("--batches", default="1,8,32")
    ap.add_argument("--new", type=int, default=32)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from llava import _b2

    dev = torch.device("cuda:0")
    out = open(a.out, "w") if a.out else None

    def emit(d):
        line = json.dumps(d)
        print(line, flush=True)
        if out:
            out.write(line + "\n")

    emit({"card": kb.card()})
    batches = [int(x) for x in a.batches.split(",")]
    eng = kb.build_engine(dev, max(batches))
    V = eng.vocab
    g = torch.Generator(device=dev).manual_seed(1)
    sampled = _b2.make_sampling(True, 0.8, 0.9, 50, seed=7)
    for ctx in [int(x) for x in a.contexts.split(",")]:
        for B in batches:
            smax = ctx + (len(VARIANTS) * (a.reps + 2)) * (a.new + 1) + 8
            kv = eng.new_kv(B, smax)
            embeds = (torch.randn(B, ctx, kb.M7["hidden"], device=dev, generator=g) * 0.5).to(torch.bfloat16)
            kb.prefill(eng, kv, embeds, B, ctx)
            del embeds
            logits = torch.randn(B, V, device=dev, generator=g)  # token 0 of every run is chosen from these
            ids = torch.randint(0, V, (B, ctx), device=dev, dtype=torch.int64, generator=g)
            procs = [_b2.make_logits_proc(ids[b], repetition_penalty=1.2, no_repeat_ngram_size=3) for b in range(B)]
            setup = {"greedy": (None, None), "greedy+proc": (None, procs), "sampled": (sampled, None), "sampled+proc": (sampled, procs)}

            def run(v):
                sp, pr = setup[v]
                eng.stream_begin(kv, logits, sp, pr)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                eng.stream_enqueue(kv, a.new)
                e1.record()
                torch.cuda.synchronize()
                return e0.elapsed_time(e1) / a.new

            for v in VARIANTS:  # warm-up: eager step, graph capture
                run(v)
            times = {v: [] for v in VARIANTS}
            for _ in range(a.reps):
                for v in VARIANTS:
                    times[v].append(run(v))
            for v in VARIANTS:
                emit(dict(kind="step", context=ctx, B=B, variant=v, ms_per_step=round(statistics.median(times[v]), 4),
                          all_ms=[round(t, 4) for t in times[v]], steps_per_run=a.new))
            from torch.profiler import ProfilerActivity, profile
            for v in VARIANTS:
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    run(v)
                ks = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "sample_publish" in e.name]
                us = [e.device_time for e in ks] if ks and hasattr(ks[0], "device_time") else [e.cuda_time for e in ks]
                emit(dict(kind="kernel", context=ctx, B=B, variant=v, launches=len(us),
                          us_per_launch=round(sum(us) / len(us), 2) if us else None))
            kv.close()
            torch.cuda.empty_cache()
    if out:
        out.close()


if __name__ == "__main__":
    main()
