"""Prompt-lookup speculative decoding at LLaVA-1.5-7B shapes, seeded random weights, contexts 704 and 1600 (batch 1):

  verify    the verify forward of R = 1, 2, 4, 8, 12, 16 rows (b2_decode_rows, launched eagerly) against the batch-1 megakernel step
            and the multi-kernel decode step at batch R (b2_decode_step on a cache of R slots in a child process started with
            B2_DECODE_MEGA=0: the GEMV graph up to 6, stream-K above)
  attn      decode_attn_mq alone (R = 8 and 16, the split factor the verify step uses) against decode_attn, H = 32, 200 launches
  e2e       a streamed greedy generation of `--new` tokens, scheduled as generate() schedules it, host clock from the prefill to the
            last token read: plain, lookup on prompt ids that hold the plain stream (the upper bound while the streams agree) and
            lookup on prompt ids that never recur (drafts come from the answer only); K = `--k`
  breakeven the mean accepted draft tokens per step at which a verify step (its no-match time) pays for itself against plain decode

Needs a GPU. Prints one JSON object per measurement and the card's name, power limit and maximum SM clock read in the same run.

    python scripts/spec_bench.py [--k 7] [--new 64] [--reps 3]
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "llava-plus-codebase_b200"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import torch  # noqa: E402

from nf4_bench import build_engine, card, model_cfg  # noqa: E402

DEV = "cuda"


def timed(fn, reps):
    """median ms of fn() over `reps` runs, each bracketed by CUDA events"""
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return sorted(out)[len(out) // 2]


def emit(**kw):
    print(json.dumps(kw), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--k", type=int, default=7)
    ap.add_argument("--new", type=int, default=64)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--batch-steps", action="store_true", help="child mode: only the decode step at batch R")
    args = ap.parse_args()
    from llava import _b2

    if args.batch_steps:
        return batch_steps(args)
    child = subprocess.run([sys.executable, os.path.abspath(__file__), "--batch-steps", "--reps", str(args.reps)],
                           env=dict(os.environ, B2_DECODE_MEGA="0"), capture_output=True, text=True)
    step_at = {}
    for line in child.stdout.splitlines():
        if line.startswith("{"):
            r = json.loads(line)
            step_at[(r["ctx"], r["R"])] = r["ms"]
    if not step_at:
        raise RuntimeError("batch-step child failed: " + child.stderr[-2000:])

    emit(card=card())
    cfg = model_cfg("7b")
    eng = build_engine(DEV, cfg, 16, 2048, False)
    h, V = cfg["hidden"], cfg["vocab"]
    for ctx in (704, 1600):
        emb = (torch.randn(1, ctx, h, device=DEV, generator=torch.Generator(device=DEV).manual_seed(ctx)) * 0.5).to(torch.bfloat16)
        kv = eng.new_kv(1, 2048)

        def plain_stream(n=args.new):
            logits = eng.prefill(kv, emb, None, _b2.LOGITS_LAST)
            eng.stream_begin(kv, logits, _b2.make_sampling())
            eng.stream_enqueue(kv, n - 1)
            return [eng.stream_wait(kv, t, 1)[0] for t in range(n)]

        plain_stream(8)
        # ---- verify forward against the decode steps ----
        eng.prefill(kv, emb, None, _b2.LOGITS_LAST)
        tok = torch.tensor([5], dtype=torch.int32, device=DEV)
        for _ in range(3):
            eng.decode_step(kv, tok)
        mega = timed(lambda: [eng.decode_step(kv, tok, want_logits=False) for _ in range(20)], args.reps) / 20
        emit(ctx=ctx, what="step", path="megakernel B=1", ms=round(mega, 4))
        verify = {}
        for R in (1, 2, 4, 8, 12, 16):
            rows = torch.arange(R, dtype=torch.int32, device=DEV) + 7

            def run_rows():
                eng.prefill(kv, emb, None, _b2.LOGITS_NONE)
                eng.decode_rows(kv, rows)

            run_rows()
            pre = timed(lambda: eng.prefill(kv, emb, None, _b2.LOGITS_NONE), args.reps)
            both = timed(run_rows, args.reps)
            verify[R] = both - pre
            emit(ctx=ctx, what="verify", R=R, verify_ms=round(verify[R], 4), decode_step_batch_R_ms=step_at[(ctx, R)],
                 megakernel_b1_ms=round(mega, 4))
        # ---- attention alone ----
        lib = _b2.load_library()
        H, D = cfg["heads"], 128
        kc = torch.randn(1, H, 2048, D, device=DEV).to(torch.bfloat16)
        vc = torch.randn_like(kc)
        cur = torch.tensor([ctx], dtype=torch.int32, device=DEV)
        ns1 = lib.b2_op_decode_attn_nsplit(1, H, 2048, 0)
        sc1 = torch.zeros(lib.b2_op_decode_attn_scratch_bytes(1, H, ns1), dtype=torch.uint8, device=DEV)
        qkv1 = torch.randn(1, 3 * H * D, device=DEV).to(torch.bfloat16)
        out1 = torch.empty(1, H * D, device=DEV, dtype=torch.bfloat16)
        P, S = _b2.ptr, _b2.stream_ptr

        def da():
            for _ in range(200):
                lib.b2_op_decode_attn(P(qkv1), P(kc), P(vc), P(cur), P(out1), P(sc1), 1, H, 2048, ns1, 10000.0, 1 / math.sqrt(D), S())

        da()
        t_da = timed(da, args.reps) / 200
        for R in (8, 16):
            nsm = lib.b2_op_decode_attn_mq_nsplit(H, 2048)
            scm = torch.zeros(lib.b2_op_decode_attn_mq_scratch_bytes(1, H, nsm), dtype=torch.uint8, device=DEV)
            qkvm = torch.randn(R, 3 * H * D, device=DEV).to(torch.bfloat16)
            outm = torch.empty(R, H * D, device=DEV, dtype=torch.bfloat16)

            def mq():
                for _ in range(200):
                    lib.b2_op_decode_attn_mq(P(qkvm), P(kc), P(vc), P(cur), P(outm), P(scm), 1, R, H, 2048, nsm, 1 / math.sqrt(D), S())

            mq()
            emit(ctx=ctx, what="attn", R=R, decode_attn_mq_us=round(timed(mq, args.reps) / 200 * 1e3, 2),
                 decode_attn_us=round(t_da * 1e3, 2))
        # ---- end to end ----
        def wall(fn):
            out = []
            for _ in range(args.reps):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                out.append((time.perf_counter() - t0) * 1e3)
                torch.cuda.synchronize()
            return sorted(out)[len(out) // 2]

        plain = plain_stream()
        tp = wall(plain_stream)
        z = V - 11
        hit = torch.tensor([z] + plain + [z], dtype=torch.int64)
        miss = torch.arange(1000, 1000 + 2 * args.new, dtype=torch.int64)  # ids the random model does not produce in order

        from llava.model.language_model.llava_llama import _LOOKUP_STEPS_IN_FLIGHT

        def lookup(ids):
            logits = eng.prefill(kv, emb, None, _b2.LOGITS_LAST)
            eng.stream_begin_lookup(kv, logits, _b2.make_sampling(), _b2.make_prompt_lookup(ids.to(DEV), args.k, 2, args.new))
            toks = []
            for t in range(args.new):  # as generate()'s host loop: top the steps in flight up before each token
                eng.stream_enqueue(kv, _LOOKUP_STEPS_IN_FLIGHT)
                toks.append(eng.stream_wait(kv, t, 1)[0])
            return toks

        for name, ids in (("prompt holds the plain stream", hit), ("prompt without matches", miss)):
            toks = lookup(ids)
            torch.cuda.synchronize()
            stats = eng.lookup_stats(kv)
            t = wall(lambda: lookup(ids))
            emit(ctx=ctx, what="e2e", case=name, K=args.k, same_tokens=toks == plain,
                 first_difference=next((i for i, (a, b) in enumerate(zip(toks, plain)) if a != b), None), steps=stats[0],
                 drafted=stats[1], accepted=stats[2], ms=round(t, 2), plain_ms=round(tp, 2),
                 note="host clock from the prefill to the last token read; at most the in-flight steps run after it")
        be = verify[args.k + 1] / mega - 1
        emit(ctx=ctx, what="breakeven", K=args.k, verify_ms=round(verify[args.k + 1], 4), megakernel_ms=round(mega, 4),
             accepted_per_step=round(be, 3))
        kv.close()
    eng.close()


def batch_steps(args):
    """child mode (B2_DECODE_MEGA=0): ms per decode step at batch R on an R-slot cache, one JSON line per (context, R)"""
    from llava import _b2

    cfg = model_cfg("7b")
    eng = build_engine(DEV, cfg, 16, 2048, False)
    for ctx in (704, 1600):
        emb = (torch.randn(1, ctx, cfg["hidden"], device=DEV, generator=torch.Generator(device=DEV).manual_seed(ctx)) * 0.5).to(torch.bfloat16)
        for R in (1, 2, 4, 8, 12, 16):
            kvb = eng.new_kv(R, 2048)
            eng.prefill(kvb, emb.expand(R, ctx, cfg["hidden"]).contiguous(), None, _b2.LOGITS_NONE)
            toks = torch.full((R,), 5, dtype=torch.int32, device=DEV)
            for _ in range(3):
                eng.decode_step(kvb, toks, want_logits=False)
            ms = timed(lambda: [eng.decode_step(kvb, toks, want_logits=False) for _ in range(10)], args.reps) / 10
            kvb.close()
            print(json.dumps(dict(ctx=ctx, R=R, ms=round(ms, 4))), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
