"""Cost of generate(output_scores / output_logits) on the engine (LLaVA-1.5-7B shapes, random weights from a seed), in ONE process.

For each case, ms per decode step with the score and logits rows written (b2_stream_set_outputs / b2_beam_step_out) against the
same steps without them, the two alternating `reps` times on one cache whose context starts at `context` tokens:

  greedy B = 1 (megakernel, plus the rows launch), B = 4 (GEMV graph), B = 32 (stream-K); sampled (T 0.8, top-k 50, top-p 0.9)
  B = 1 and 32: a streamed generation (b2_stream_begin + b2_stream_enqueue, CUDA events around the enqueued steps);
  beam nb = 4 (one sample): b2_beam_step, which synchronises every step, timed with the host clock.

Also printed: the bytes the rows add per step, 2 * rows * V * 4 (computed, not measured), and the card's name, power limit and
SM clock. Needs a GPU (there is no fallback).

    python scripts/scores_bench.py [--context 704] [--new 32] [--reps 5] [--out FILE]
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(ROOT))
import kv_fp8_bench as kb  # noqa: E402  (7B engine from seeded weights, card())

import torch  # noqa: E402

CASES = (("greedy", 1), ("greedy", 4), ("greedy", 32), ("sampled", 1), ("sampled", 32), ("beam", 4))


def sm_clock():
    import subprocess

    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:  # the number is reported beside the card, never needed to run
        return f"unavailable: {e}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--context", type=int, default=704)
    ap.add_argument("--new", type=int, default=32)
    ap.add_argument("--reps", type=int, default=5)
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

    emit({"card": kb.card(), "sm_clock_mhz(now, max)": sm_clock()})
    eng = kb.build_engine(dev, 32)
    V = eng.vocab
    g = torch.Generator(device=dev).manual_seed(1)
    sampled = _b2.make_sampling(True, 0.8, 0.9, 50, seed=7)
    ctx = a.context
    for kind, B in CASES:
        runs = 2 * (a.reps + 1)
        smax = ctx + runs * (a.new + 1) + 8
        kv = eng.new_kv(B, smax)
        embeds = (torch.randn(B, ctx, kb.M7["hidden"], device=dev, generator=g) * 0.5).to(torch.bfloat16)
        kb.prefill(eng, kv, embeds, B, ctx)
        del embeds
        logits = torch.randn(B, V, device=dev, generator=g)
        rows = [torch.empty(a.new + 1, B, V, device=dev) for _ in range(2)]

        def run_stream(on):
            eng.stream_begin(kv, logits, sampled if kind == "sampled" else None, None, *(rows if on else (None, None)))
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            eng.stream_enqueue(kv, a.new)
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / a.new

        step_rows = [torch.empty(B, V, device=dev) for _ in range(2)]

        def run_beam(on):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(a.new):
                eng.beam_step(kv, [], 0, [5] * B, list(range(B)), [0.0] * B, B, 2 * B,
                              **(dict(row_scores=step_rows[0], row_logits=step_rows[1]) if on else {}))
            return (time.perf_counter() - t0) * 1e3 / a.new

        run = run_beam if kind == "beam" else run_stream
        for on in (False, True):  # warm-up: eager step, graph capture
            run(on)
        times = {False: [], True: []}
        for _ in range(a.reps):
            for on in (False, True):
                times[on].append(run(on))
        off_ms, on_ms = statistics.median(times[False]), statistics.median(times[True])
        emit(dict(kind=kind, B=B if kind != "beam" else 1, beams=B if kind == "beam" else 1, context=ctx,
                  ms_per_step_off=round(off_ms, 4), ms_per_step_on=round(on_ms, 4),
                  overhead_pct=round(100.0 * (on_ms - off_ms) / off_ms, 2), all_off=[round(t, 4) for t in times[False]],
                  all_on=[round(t, 4) for t in times[True]], bytes_written_per_step=2 * B * V * 4, steps_per_run=a.new))
        kv.close()
        del rows, step_rows
        torch.cuda.empty_cache()
    if out:
        out.close()


if __name__ == "__main__":
    main()
