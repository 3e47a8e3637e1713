"""A/B of the batched decode step inside one process (7B): isolated decode timing (prefill -> sync -> N greedy steps) per
batch size under environment variants read at graph-capture time; also the HOST time of the enqueueing call (a replayed
graph returns in ~N x 20 us, launch-by-launch enqueueing takes as long as the GPU work).

    python scripts/decode_ab.py --batches 8,32 --variants "default;B2_DECODE_SKINNY=0"
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import bench  # noqa: E402
import config_sweep  # noqa: E402

import numpy as np  # noqa: E402
import torch  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="7b")
    ap.add_argument("--batches", default="8,32")
    ap.add_argument("--new", type=int, default=64)
    ap.add_argument("--variants", default="default;B2_DECODE_SKINNY=0")
    ap.add_argument("--out", default=os.devnull, help="also append every result line to this file")
    a = ap.parse_args()
    from llava import _b2
    from llava.model.llava_arch import build_source_index

    m = bench.MODELS[a.model]
    dev = torch.device("cuda:0")
    torch.cuda.set_device(0)
    batches = [int(x) for x in a.batches.split(",")]
    S, N = 128 + bench.P_IMG, a.new
    hbm_peak, _, _ = bench.peaks()
    model = config_sweep.build(m, dev, max(batches), S + N + 8, 8)
    engine = model._ensure_engine()
    g = torch.Generator().manual_seed(1)
    fout = open(a.out, "a")
    stream = torch.cuda.Stream(device=dev)
    with torch.cuda.stream(stream), torch.no_grad():
        for B in batches:
            work = bench.algorithmic_work(m, B, S, N + 1)
            ids = torch.randint(3, bench.VOCAB, (B, 129), generator=g)
            ids[:, 0] = 1
            ids[:, 5] = bench.IMAGE_TOKEN
            ids_np = ids.numpy().astype(np.int64)
            src, _, _, _, lens = build_source_index(ids_np, np.ones_like(ids_np, bool), np.full_like(ids_np, -100),
                                                    B * bench.P_IMG, [bench.P_IMG] * B, None, "right")
            feats = (torch.randn(B * bench.P_IMG, m["hidden"], generator=g) * 0.5).to(dev, torch.bfloat16)
            embeds = engine.splice(torch.from_numpy(src.reshape(-1)).to(dev), feats, B, S)
            out = torch.empty(N, B, dtype=torch.int32, device=dev)
            ref = None
            for variant in a.variants.split(";"):
                env = dict(kv.split("=") for kv in variant.split(",") if "=" in kv)
                for k, v in env.items():
                    os.environ[k] = v
                kv = engine.new_kv(B, S + N + 8)  # fresh cache -> freshly captured graph under this environment
                times, host = [], []
                for rep in range(int(env.get("REPS", "4"))):
                    if env.get("FRESHKV") == "1" and rep > 0:   # is a run only fast on a cache object that was just created?
                        kv.close()
                        kv = engine.new_kv(B, S + N + 8)
                    kv.reset()
                    first = engine.argmax(engine.prefill(kv, embeds, lens, _b2.LOGITS_LAST))
                    torch.cuda.synchronize()
                    time.sleep(float(env.get("SLEEP", "0.2")))
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    t0 = time.perf_counter()
                    engine.decode_greedy(kv, first, N, out=out)
                    host.append((time.perf_counter() - t0) * 1e3 / N)
                    e1.record()
                    torch.cuda.synchronize()
                    times.append(e0.elapsed_time(e1) / N)
                # time evolution inside one run: 8-step chunks back to back (is a run slower at its end than at its start?)
                kv.reset()
                first = engine.argmax(engine.prefill(kv, embeds, lens, _b2.LOGITS_LAST))
                torch.cuda.synchronize()
                sampler = bench.ClockSampler(0)
                sampler.start()
                evs = [torch.cuda.Event(enable_timing=True) for _ in range(N // 8 + 1)]
                cur = first
                evs[0].record()
                for c in range(N // 8):
                    chunk = engine.decode_greedy(kv, cur, 8)
                    cur = chunk[7]
                    evs[c + 1].record()
                torch.cuda.synchronize()
                clocks = sampler.stop()
                chunks = [round(evs[c].elapsed_time(evs[c + 1]) / 8, 3) for c in range(N // 8)]
                toks = out.cpu()
                if ref is None:
                    ref = toks.clone()
                best = min(times[1:])
                gbs = work["decode_bytes_per_step"] / best / 1e6
                d = dict(B=B, variant=variant, ms_per_step=best, all_ms=times, host_enqueue_ms_per_step=min(host[1:]),
                         ms_per_step_by_8_step_chunk=chunks, clocks=clocks,
                         frac_hbm_peak=gbs / hbm_peak, tokens_equal_first_variant=bool((toks == ref).all()))
                s = json.dumps(d)
                print(s, flush=True)
                fout.write(s + "\n")
                fout.flush()
                kv.close()
                for k in env:
                    os.environ.pop(k, None)


if __name__ == "__main__":
    main()
