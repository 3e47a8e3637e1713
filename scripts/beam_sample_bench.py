"""Beam sampling against beam search on the engine (LLaVA-1.5-7B shapes, random weights from a seed, batch 1, a 576 + 128 =
704-row prompt forked into num_beams slots), in ONE process.

  step   per num_beams: ms per b2_beam_step (greedy candidates) and per b2_beam_step_ex (sampled candidates) under each
         warper setting, on a host clock around the synchronising call, the arms alternated in rounds so that drift on the
         host hits all of them alike. Tokens are fed back without slot copies, so a step is decode + selection + read-back.
  op     per num_beams, with CUDA events: b2_op_beam_topk and b2_op_beam_sample alone on [num_beams, 32000] logits, K = 2 nb.

Warper settings: the reference eval scripts' default (temperature 0.2, top_k 50, top_p off) and temperature 0.7 / top_p 0.9.
Needs a GPU (there is no fallback). Prints one JSON object per measurement and the card's name and power limit.

    python scripts/beam_sample_bench.py [--beams 2,4,8] [--steps 40] [--rounds 5] [--out FILE]
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
from beam_bench import PROMPT, events  # noqa: E402

import torch  # noqa: E402

WARPERS = {"T0.2_k50": (0.2, 50, 1.0), "T0.7_k50_p0.9": (0.7, 50, 0.9)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--beams", default="2,4,8")
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--rounds", type=int, default=5)
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
    beams = [int(x) for x in a.beams.split(",")]
    eng = kb.build_engine(dev, max(beams))
    M7 = kb.M7
    g = torch.Generator(device=dev).manual_seed(2)
    embeds = (torch.randn(1, PROMPT, M7["hidden"], device=dev, generator=g) * 0.02).to(torch.bfloat16)
    kv = eng.new_kv(max(beams), PROMPT + a.rounds * (len(WARPERS) + 1) * (a.steps + 1) + 16)
    lib = _b2.load_library()
    arms = {"greedy": None}
    arms.update({k: _b2.make_beam_sampling(T, k_, p, 2, 7) for k, (T, k_, p) in WARPERS.items()})

    for nb in beams:
        kv.reset()
        eng.prefill(kv, embeds, None, _b2.LOGITS_NONE)
        if nb > 1:
            eng.kv_copy_slots(kv, [0] * (nb - 1), list(range(1, nb)))
        K = 2 * nb
        slots, scores = list(range(nb)), [0.0] + [-1.0] * (nb - 1)
        times = {k: [] for k in arms}
        for name, s in arms.items():  # warm-up of every arm
            eng.beam_step(kv, [], 0, [1] * nb, slots, scores, nb, K, sampling=s, step=0)
        for r in range(a.rounds):
            for name, s in arms.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for i in range(a.steps):
                    eng.beam_step(kv, [], 0, [1 + i] * nb, slots, scores, nb, K, sampling=s, step=i + 1)
                times[name].append((time.perf_counter() - t0) * 1e3 / a.steps)
        base = sorted(times["greedy"])[len(times["greedy"]) // 2]
        d = {"run": "step", "num_beams": nb, "K": K, "steps_per_round": a.steps, "rounds": a.rounds}
        for name, ts in times.items():
            med = sorted(ts)[len(ts) // 2]
            d[f"{name}_ms"] = round(med, 3)
            d[f"{name}_spread_ms"] = round(max(ts) - min(ts), 3)
            if name != "greedy":
                d[f"{name}_vs_greedy"] = round(med / base, 4)
        emit(d)

        logits = torch.randn(nb, eng.vocab, device=dev, generator=g) * 3
        sc_d = torch.zeros(nb, device=dev)
        o = [torch.empty(K, device=dev, dtype=dt) for dt in (torch.float32, torch.int32, torch.int32)]
        head = [_b2.ptr(logits), None, _b2.ptr(sc_d), 1, nb, eng.vocab, K]
        tail = [_b2.ptr(t) for t in o] + [_b2.stream_ptr()]
        op = {"run": "op", "num_beams": nb, "K": K, "beam_topk_ms": round(events(lambda: lib.b2_op_beam_topk(*head, *tail), 200), 4)}
        for name, (T, k_, p) in WARPERS.items():
            s = _b2.make_beam_sampling(T, k_, p, 2, 7)
            op[f"beam_sample_{name}_ms"] = round(events(lambda: lib.b2_op_beam_sample(*head, s, 3, *tail), 200), 4)
        emit(op)
    emit({"card": kb.card()})


if __name__ == "__main__":
    main()
