"""CPU restatement of a prefill chunk appended to an e4m3 KV cache (b2_prefill_at, include/b2llava.h) — TEST INFRASTRUCTURE ONLY.

It extends the rule of oracle/kv_fp8_oracle.py (prefill attends over the unquantised K / V of its own tokens, only what it
stores is quantised) to a chunk that starts at cache position p > 0: the rows [0, p) exist only as stored e4m3 bytes and
scales, so the engine stages them as bf16(float(q) * scale) and the chunk attends over those plus its own unquantised rows.
With a bf16 cache no new rule is needed: oracle/llava_oracle.llama_forward(kv=..., position_ids=...) is the continuation.
"""
import torch

from . import kv_fp8_oracle as KV
from . import llava_oracle as O


def stage_prefix(cache, b, p):
    """The bf16 staging of rows [0, p) of sample b of one layer's cache (b2_op_kv_dequantize_e4m3): (k, v) [1, H, p, 128] bf16."""
    return tuple(KV.dequantize_kv(cache[q8][b:b + 1, :, :p], cache[sc][b:b + 1, :, :p]).to(torch.bfloat16)
                 for q8, sc in (("k8", "ks"), ("v8", "vs")))


def prefill_chunk(w, embeds, cfg, caches, start, seq_lens=None, last_only=False, dtype=torch.float32):
    """Prefill of a chunk appended at cache position start[b] of a quantised cache. embeds [B, n, h]; sample b has
    seq_lens[b] valid rows (None = n). Its rows attend over stage_prefix(..., start[b]) plus their own unquantised K / V
    (llama_forward at positions start[b] + t), and are then stored at rows start[b] .. IN PLACE. Returns fp32 logits
    [B, n, V] (rows past seq_lens[b] are zero), or with last_only [B, V] at each sample's last valid row."""
    B, n = embeds.shape[0], embeds.shape[1]
    out = []
    for b in range(B):
        p, L = int(start[b]), n if seq_lens is None else int(seq_lens[b])
        kv = [tuple(t.to(dtype) for t in stage_prefix(c, b, p)) for c in caches]
        logits, new_kv = O.llama_forward(w, embeds[b:b + 1, :L], cfg, kv=kv, dtype=dtype)
        for c, (k, v) in zip(caches, new_kv):
            for src, q8, sc in ((k, "k8", "ks"), (v, "v8", "vs")):
                q, s = KV.quantize_kv(src[0, :, p:p + L].to(torch.bfloat16))
                c[q8][b, :, p:p + L] = q
                c[sc][b, :, p:p + L] = s
        if last_only:
            out.append(logits[0, L - 1])
        else:
            full = torch.zeros(n, logits.shape[-1])
            full[:L] = logits[0]
            out.append(full)
    return torch.stack(out)
