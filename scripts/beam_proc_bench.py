"""Cost of logits processors in beam search (LLaVA-1.5-7B shapes, random weights from a seed, batch 1, a 576 + 128 = 704-row
prompt whose 704 ids are the processors' history), in ONE process. eos is off, so every run has its full length.

  step      per num_beams: the beam loop of generate() (b2_beam_step vs b2_beam_step_proc with no_repeat_ngram_size = 3 and
            repetition_penalty = 1.2, begun by b2_op_beam_select_proc + b2_beam_begin_proc), alternated plain / processed
            `--reps` times; ms per beam step on a host clock around work that ends in the step's synchronisation. Reports the
            median of each and the spread (max - min) over the repetitions.
  select    per num_beams: the selection entry points alone on [num_beams, 32000] fp32 logits with CUDA events:
            b2_op_beam_select_out, and b2_op_beam_select_proc with every row processed against a 704-id history. The processed
            call also allocates its scratch state, seeds the histories and synchronises, so it is an upper bound of the
            processed row kernel, not the kernel alone.

Needs a GPU (there is no fallback). Prints one JSON object per measurement and the card's name and power limit.

    python scripts/beam_proc_bench.py [--beams 2,4,8] [--new 64] [--reps 3] [--out FILE]
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

PROMPT = 576 + 128
PROC = dict(repetition_penalty=1.2, no_repeat_ngram_size=3)


def events(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--beams", default="2,4,8")
    ap.add_argument("--new", type=int, default=64)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from llava import _b2
    from llava._b2 import beam as BM

    dev = torch.device("cuda:0")
    out = open(a.out, "w") if a.out else None

    def emit(d):
        line = json.dumps(d)
        print(line, flush=True)
        if out:
            out.write(line + "\n")

    emit({"card": kb.card()})
    beams = [int(x) for x in a.beams.split(",")]
    eng = kb.build_engine(dev, max(beams))
    M7 = kb.M7
    V = eng.vocab
    g = torch.Generator(device=dev).manual_seed(2)
    embeds = (torch.randn(1, PROMPT, M7["hidden"], device=dev, generator=g) * 0.02).to(torch.bfloat16)
    ids = torch.randint(0, V, (1, PROMPT), device=dev, generator=g)
    kv = eng.new_kv(max(beams), PROMPT + a.new + 8)

    def generate(nb, n_new, proc):
        s = BM.BeamSearch(ids.cpu(), nb, n_new, None)
        kv.reset()
        logits = eng.prefill(kv, embeds, None, _b2.LOGITS_LAST)
        step = eng.beam_step
        if proc:
            procs = [_b2.make_logits_proc(ids[0], **PROC)]
            cand = [t.cpu() for t in eng.beam_select_proc(logits, torch.zeros(1), 1, s.K, procs, fan=nb)]
            eng.beam_begin_proc(kv, procs)
            step = eng.beam_step_proc
        else:
            cand = [t.cpu() for t in eng.beam_topk(logits, torch.zeros(1), 1, s.K)]
        plan, rb, steps = BM.SlotPlanner(1, nb), 0, 0
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        while not s.step(*cand):
            cand = step(kv, plan.plan(s.parents), rb, s.next_tokens().tolist(), plan.flat(), s.running_scores.reshape(-1).tolist(),
                        nb, s.K)
            rb, steps = PROMPT, steps + 1
        return (time.perf_counter() - t0) * 1e3 / max(steps, 1)

    for nb in beams:
        generate(nb, 8, False)  # warm-up: graphs / function attributes of batch nb, both selection kernels
        generate(nb, 8, True)
        plain, proc = [], []
        for _ in range(a.reps):
            plain.append(generate(nb, a.new, False))
            proc.append(generate(nb, a.new, True))
        mp, mq = statistics.median(plain), statistics.median(proc)
        emit({"run": "step", "num_beams": nb, "new_tokens": a.new, "plain_ms_per_step": round(mp, 4),
              "proc_ms_per_step": round(mq, 4), "plain_spread_ms": round(max(plain) - min(plain), 4),
              "proc_spread_ms": round(max(proc) - min(proc), 4), "overhead_ms": round(mq - mp, 4),
              "overhead_pct": round(100 * (mq - mp) / mp, 2)})

    lib = _b2.load_library()
    for nb in beams:
        logits = torch.randn(nb, V, device=dev, generator=g)
        sc = torch.zeros(nb, device=dev)
        o = [torch.empty(2 * nb, device=dev, dtype=dt) for dt in (torch.float32, torch.int32, torch.int32)]
        rows = torch.empty(nb, V, device=dev)
        P = _b2.ptr
        base = [P(logits), None, P(sc), 1, nb, V, 2 * nb, None, 0, 1]
        tail = [P(o[0]), P(o[1]), P(o[2]), P(rows), None, _b2.stream_ptr()]
        out_ms = events(lambda: lib.b2_op_beam_select_out(*base, *tail), 100)
        procs = _b2._proc_array([_b2.make_logits_proc(ids[0], **PROC) for _ in range(nb)], nb)
        proc_ms = events(lambda: lib.b2_op_beam_select_proc(P(logits), nb, *base[1:], procs, *tail), 100)
        emit({"run": "select", "num_beams": nb, "vocab": V, "history": PROMPT, "select_out_ms": round(out_ms, 4),
              "select_proc_call_ms": round(proc_ms, 4)})
    emit({"card": kb.card()})


if __name__ == "__main__":
    main()
