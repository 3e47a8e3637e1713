"""Beam search on the engine (LLaVA-1.5-7B shapes, random weights from a seed, batch 1, a 576 + 128 = 704-row prompt), in ONE
process. eos is off, so every run has its full length.

  run       per (num_beams, new tokens): the whole generation (prefill, step-0 selection, then b2_beam_step per token with the
            host bookkeeping of llava/_b2/beam.py) on a host clock; ms per beam step and tokens/s of the best beam against
            greedy decoding of the same prompt (b2_decode_greedy, CUDA events).
  split     per num_beams, with CUDA events: the decode step alone at batch num_beams (b2_decode_step), b2_op_beam_topk alone on
            [num_beams, 32000] logits, and b2_kv_copy_slots of num_beams - 1 slots over the generated rows of a 256-token
            answer (the most a step can copy; bytes moved and GB/s computed from shapes). The host bookkeeping per step
            (llava/_b2/beam.py) is timed on its own inside `run`; the rest of a step beyond the three is the ABI call's own
            host work (argument checks, token upload, the read-back and its synchronisation).

Needs a GPU (there is no fallback). Prints one JSON object per measurement and the card's name and power limit.

    python scripts/beam_bench.py [--beams 1,2,4,5,8] [--new 64,256] [--out FILE]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(ROOT))
import kv_fp8_bench as kb  # noqa: E402  (7B engine from seeded weights, card())

import torch  # noqa: E402

PROMPT = 576 + 128


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
    ap.add_argument("--beams", default="1,2,4,5,8")
    ap.add_argument("--new", default="64,256")
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
    news = [int(x) for x in a.new.split(",")]
    eng = kb.build_engine(dev, max(beams))
    M7 = kb.M7
    g = torch.Generator(device=dev).manual_seed(2)
    embeds = (torch.randn(1, PROMPT, M7["hidden"], device=dev, generator=g) * 0.02).to(torch.bfloat16)
    rows_copied = 256  # generated rows each copy of the split below moves
    cap = PROMPT + max(max(news), rows_copied) + 8
    kv = eng.new_kv(max(beams), cap)
    prompt_ids = torch.full((1, 1), 1, dtype=torch.int64)  # stands for the prompt in the host bookkeeping (ids are not fed back)

    def generate(nb, n_new):
        s = BM.BeamSearch(prompt_ids, nb, n_new, None)
        kv.reset()
        logits = eng.prefill(kv, embeds, None, _b2.LOGITS_LAST)
        cand = [t.cpu() for t in eng.beam_topk(logits, torch.zeros(1), 1, s.K)]
        plan, rb, steps, copies, host = BM.SlotPlanner(1, nb), 0, 0, 0, 0.0
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        while True:
            h0 = time.perf_counter()
            if s.step(*cand):
                break
            c = plan.plan(s.parents)
            args = (c, rb, s.next_tokens().tolist(), plan.flat(), s.running_scores.reshape(-1).tolist(), nb, s.K)
            host += time.perf_counter() - h0
            copies += len(c)
            cand = eng.beam_step(kv, *args)
            rb, steps = PROMPT, steps + 1
        return (time.perf_counter() - t0) * 1e3, steps, copies, host * 1e3

    for n_new in news:
        kv.reset()
        logits = eng.prefill(kv, embeds, None, _b2.LOGITS_LAST)
        first = eng.argmax(logits)
        kv_g = eng.new_kv(1, cap)

        def greedy():
            kv_g.reset()
            eng.prefill(kv_g, embeds, None, _b2.LOGITS_NONE)
            eng.decode_greedy(kv_g, first, n_new - 1)

        prefill_ms = events(lambda: (kv_g.reset(), eng.prefill(kv_g, embeds, None, _b2.LOGITS_NONE)), 3)
        greedy_ms = events(greedy, 3) - prefill_ms
        kv_g.close()
        for nb in beams:
            generate(nb, min(n_new, 8))  # warm-up: graphs / function attributes of batch nb
            ms, steps, copies, host_ms = generate(nb, n_new)
            emit({"run": "generate", "num_beams": nb, "new_tokens": n_new, "beam_steps": steps, "copies": copies,
                  "ms_per_step": round(ms / max(steps, 1), 3), "host_bookkeeping_ms_per_step": round(host_ms / max(steps, 1), 3),
                  "best_beam_tok_s": round(n_new / (ms / 1e3), 1),
                  "greedy_ms_per_step": round(greedy_ms / max(n_new - 1, 1), 3),
                  "greedy_tok_s": round((n_new - 1) / (greedy_ms / 1e3), 1)})

    def fill(cache, nb):
        """slot 0 := the prompt; slots 1 .. nb - 1 := copies of it (the workspace prefills one 704-row prompt at a time)"""
        cache.reset()
        eng.prefill(cache, embeds, None, _b2.LOGITS_NONE)
        if nb > 1:
            eng.kv_copy_slots(cache, [0] * (nb - 1), list(range(1, nb)))

    for nb in beams:
        fill(kv, nb)
        tok = torch.ones(nb, dtype=torch.int32, device=dev)
        eng.decode_step(kv, tok)  # warm-up of the batch size
        decode_ms = events(lambda: eng.decode_step(kv, tok), 20)
        logits = torch.randn(nb, eng.vocab, device=dev, generator=g)
        scores = torch.zeros(nb)
        binding_ms = events(lambda: eng.beam_topk(logits, scores, nb, 2 * nb), 50)
        # the kernels alone: the C entry point on buffers allocated once (no Python-side allocation or host-to-device copy)
        sc_d = torch.zeros(nb, device=dev)
        o = [torch.empty(2 * nb, device=dev, dtype=dt) for dt in (torch.float32, torch.int32, torch.int32)]
        args = [_b2.ptr(logits), None, _b2.ptr(sc_d), 1, nb, eng.vocab, 2 * nb] + [_b2.ptr(t) for t in o] + [_b2.stream_ptr()]
        lib = _b2.load_library()
        topk_ms = events(lambda: lib.b2_op_beam_topk(*args), 200)
        d = {"split": "step", "num_beams": nb, "decode_ms": round(decode_ms, 3), "beam_topk_ms": round(topk_ms, 4),
             "beam_topk_python_call_ms": round(binding_ms, 4)}
        if nb > 1:
            # slot 0 grows by a 256-token answer; each copy then moves rows [PROMPT, PROMPT + 256) of every layer / head, K and V
            fill(kv, 1)
            eng.prefill(kv, torch.zeros(1, rows_copied, M7["hidden"], device=dev, dtype=torch.bfloat16), None, _b2.LOGITS_NONE,
                        start=[PROMPT])
            src, dst = [0] * (nb - 1), list(range(1, nb))
            copy_ms = events(lambda: eng.kv_copy_slots(kv, src, dst, row_begin=PROMPT), 20)
            nbytes = 2 * (nb - 1) * rows_copied * kb.KV_TOKEN_BYTES["bf16"]  # read + write
            d.update({"copies": nb - 1, "copy_rows": rows_copied, "copy_ms": round(copy_ms, 4), "copy_bytes": nbytes,
                      "copy_GBps": round(nbytes / (copy_ms / 1e3) / 1e9, 1)})
        emit(d)
    emit({"card": kb.card()})


if __name__ == "__main__":
    main()
