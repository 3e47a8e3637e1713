"""generate(do_sample=True, num_return_sequences=n) at LLaVA-1.5-7B shapes (random weights from a seed), in ONE process.

  step    per (B, n, prompt): the same forked generation (B prompts prefilled once, copied into the n - 1 follower slots of each)
          decoded with the group table armed (b2_stream_begin_groups) and on decode_attn (share_prefix=False), alternated `--reps`
          times; ms per decode step on a host clock around `--new` queued steps that end in a synchronisation. Medians and the
          spread (max - min).
  kernel  per (B, n, prompt): decode_attn_shared alone against decode_attn at the step's shapes (H = 32, the split factor each
          uses in the step, every row at prompt + 64), CUDA events over 200 (decode_attn) and 50 (the shared op entry) calls, and GB/s from the bytes each must read:
          decode_attn every row's prompt + suffix, decode_attn_shared each prompt once plus every row's suffix.
  ttft    per (B, n, prompt): the fork (B prefills + one kv_copy_slots) against one prefill of all B * n rows, CUDA events.

Needs a GPU (there is no fallback). Prints one JSON object per measurement and the card's name and power limit.

    python scripts/num_return_bench.py [--shapes 1x4,1x8,1x16,4x8,2x16] [--prompts 704,1600] [--new 64] [--reps 3] [--out FILE]
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

ROW_BYTES = 2 * 128 * 2  # K + V of one (token, head), bf16


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
    ap.add_argument("--shapes", default="1x4,1x8,1x16,4x8,2x16")
    ap.add_argument("--prompts", default="704,1600")
    ap.add_argument("--new", type=int, default=64)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from llava import _b2
    from llava._b2.fork import ForkPlan

    dev = torch.device("cuda:0")
    out = open(a.out, "w") if a.out else None

    def emit(d):
        line = json.dumps(d)
        print(line, flush=True)
        if out:
            out.write(line + "\n")

    emit({"card": kb.card()})
    shapes = [tuple(int(x) for x in s.split("x")) for s in a.shapes.split(",")]
    prompts = [int(x) for x in a.prompts.split(",")]
    maxb = max(B * n for B, n in shapes)
    eng = kb.build_engine(dev, maxb)
    M7 = kb.M7
    H, V = M7["heads"], eng.vocab
    g = torch.Generator(device=dev).manual_seed(3)
    kv = eng.new_kv(maxb, max(prompts) + a.new + 8)
    lib = _b2.load_library()

    def fork(embeds, B, n, L):
        plan = ForkPlan([L] * B, n)
        kv.reset()
        logits = eng.prefill(kv, embeds, None, _b2.LOGITS_LAST)
        eng.kv_copy_slots(kv, *plan.copies())
        return plan, logits.index_select(0, torch.tensor(plan.prompt_of_slot, device=dev))

    def step_ms(embeds, B, n, L, share):
        plan, logits = fork(embeds, B, n, L)
        eng.stream_begin(kv, logits, _b2.make_sampling(True, 0.8, 0.95, 50, 1), groups=plan.groups(), share_prefix=share)
        eng.stream_enqueue(kv, 2)  # first steps: eager, then the graph capture
        eng.stream_wait(kv, 2, B * n)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        eng.stream_enqueue(kv, a.new)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3 / a.new

    for L in prompts:
        for B, n in shapes:
            embeds = (torch.randn(B, L, M7["hidden"], device=dev, generator=g) * 0.02).to(torch.bfloat16)
            step_ms(embeds, B, n, L, True)
            step_ms(embeds, B, n, L, False)
            on, off = [], []
            for _ in range(a.reps):
                on.append(step_ms(embeds, B, n, L, True))
                off.append(step_ms(embeds, B, n, L, False))
            mo, mf = statistics.median(on), statistics.median(off)
            emit({"run": "step", "B": B, "n": n, "prompt": L, "new_tokens": a.new, "shared_ms_per_step": round(mo, 4),
                  "decode_attn_ms_per_step": round(mf, 4), "shared_spread_ms": round(max(on) - min(on), 4),
                  "decode_attn_spread_ms": round(max(off) - min(off), 4), "speedup": round(mf / mo, 3)})

            # the attention kernels alone at the step's shapes
            N, Smax, pos = B * n, L + 72, L + 64
            plan = ForkPlan([L] * B, n)
            qkv = (torch.randn(N, 3 * H * 128, device=dev, generator=g)).to(torch.bfloat16)
            kc = (torch.randn(N, H, Smax, 128, device=dev, generator=g)).to(torch.bfloat16)
            vc = torch.randn_like(kc)
            cur = torch.full((N,), pos, device=dev, dtype=torch.int32)
            o = torch.empty(N, H * 128, device=dev, dtype=torch.bfloat16)
            ns_d = int(lib.b2_op_decode_attn_nsplit(N, H, Smax, _b2.KV_BF16))
            ns_s = int(lib.b2_op_decode_attn_shared_nsplit(N, H, Smax))
            sd = torch.zeros(int(lib.b2_op_decode_attn_scratch_bytes(N, H, ns_d)), device=dev, dtype=torch.uint8)
            ss = torch.zeros(int(lib.b2_op_decode_attn_shared_scratch_bytes(N, H, ns_s)), device=dev, dtype=torch.uint8)
            grp = _b2._group_array(plan.groups())
            P, st = _b2.ptr, _b2.stream_ptr()
            t_d = events(lambda: lib.b2_op_decode_attn(P(qkv), P(kc), P(vc), P(cur), P(o), P(sd), N, H, Smax, ns_d, 1e4, 128 ** -0.5, st),
                         200)
            # the op entry uploads the group table and synchronises on every call: shared_call_us is an upper bound of the kernel
            lib.b2_op_decode_attn_shared(P(qkv), P(kc), P(vc), P(cur), grp, len(plan.groups()), P(o), P(ss), N, H, Smax, ns_s, 1e4,
                                         128 ** -0.5, st)
            t_s = events(lambda: lib.b2_op_decode_attn_shared(P(qkv), P(kc), P(vc), P(cur), grp, len(plan.groups()), P(o), P(ss), N,
                                                              H, Smax, ns_s, 1e4, 128 ** -0.5, st), 50)
            bytes_d = N * H * (pos + 1) * ROW_BYTES
            bytes_s = (B * L + N * (pos + 1 - L)) * H * ROW_BYTES
            emit({"run": "kernel", "B": B, "n": n, "prompt": L, "rows": N, "nsplit_decode_attn": ns_d, "nsplit_shared": ns_s,
                  "decode_attn_us": round(t_d * 1e3, 2), "decode_attn_GBps": round(bytes_d / t_d / 1e6, 1),
                  "shared_call_us": round(t_s * 1e3, 2), "shared_GBps": round(bytes_s / t_s / 1e6, 1),
                  "bytes_ratio": round(bytes_d / bytes_s, 2)})
            del qkv, kc, vc, sd, ss

            # time to the first token's logits: fork against a prefill of every row
            big = embeds.repeat_interleave(n, 0)
            t_fork = events(lambda: fork(embeds, B, n, L), 3)

            def full():
                kv.reset()
                eng.prefill(kv, big, None, _b2.LOGITS_LAST)
            try:
                t_full = round(events(full, 3), 3)
            except (ValueError, RuntimeError) as e:  # B * n * prompt rows may exceed the engine's prefill workspace
                t_full = f"not measured: {e}"
            emit({"run": "ttft", "B": B, "n": n, "prompt": L, "fork_ms": round(t_fork, 3), "prefill_all_rows_ms": t_full})
    emit({"card": kb.card()})


if __name__ == "__main__":
    main()
