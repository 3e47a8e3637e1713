"""Time b2_op_flash_attn (C-ABI, the wgmma flash-attention kernel) on the path's attention shapes.

    python scripts/attn_bench.py            # prints one line per shape: us, TFLOP/s, max-abs-diff vs torch fp32
"""
import math
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "llava-plus-codebase_b200"))
from llava import _b2  # noqa: E402

SHAPES = [  # B, S, H, D, causal
    (1, 577, 16, 64, 0), (8, 577, 16, 64, 0), (32, 577, 16, 64, 0), (64, 577, 16, 64, 0),
    (1, 704, 32, 128, 1), (8, 704, 32, 128, 1), (32, 704, 32, 128, 1),
    (4, 2048, 32, 128, 1), (4, 2048, 40, 128, 1),
]


def main():
    lib = _b2.load_library()
    _b2.check(lib.b2_init(0))
    dev = torch.device("cuda:0")
    for B, S, H, D, causal in SHAPES:
        g = torch.Generator(device=dev).manual_seed(1)
        q, k, v = (torch.randn(B, S, H, D, device=dev, generator=g).to(torch.bfloat16) for _ in range(3))
        o = torch.empty_like(q)
        st = torch.cuda.current_stream().cuda_stream

        def run():
            _b2.check(lib.b2_op_flash_attn(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), None, B, S, H, D,
                                           causal, 1 / math.sqrt(D), st))
        for _ in range(3):
            run()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n = 20
        e0.record()
        for _ in range(n):
            run()
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 1e3 / n
        flops = 4.0 * B * H * S * S * D * (0.5 if causal else 1.0)
        # fp32 check on the first batch entry / 4 heads
        qf, kf, vf = (t[0, :, :4].float().permute(1, 0, 2) for t in (q, k, v))
        s = qf @ kf.transpose(-1, -2) / math.sqrt(D)
        if causal:
            s = s.masked_fill(torch.triu(torch.ones(S, S, device=dev, dtype=torch.bool), 1), float("-inf"))
        want = (torch.softmax(s, -1) @ vf).permute(1, 0, 2)
        err = (o[0, :, :4].float() - want).abs().max().item()
        print(f"B={B} S={S} H={H} D={D} causal={causal}: {us:9.1f} us  {flops / us / 1e6:8.1f} TFLOP/s  "
              f"max|err|={err:.4f}", flush=True)


if __name__ == "__main__":
    main()
