"""CPU restatement of the e4m3 KV cache (b2_kv_create_ex(B2_KV_E4M3), include/b2llava.h) — TEST INFRASTRUCTURE ONLY.

The reference has no quantised cache, so like oracle/fp8_oracle.py this file DEFINES the arithmetic the CUDA kernels
implement (csrc/attention.cu: kv_quantize_e4m3_kernel, decode_attn_e4m3_kernel) and is what their tolerance is derived from:

  quantize_kv            one row = the 128 elements of one head of one token; fp8_oracle.quantize_rows_e4m3 over it:
                         scale = amax / 448 (1 for a zero row), q = e4m3_rne(x * (448 / amax)). K rows are quantised AFTER
                         RoPE (the roped, bf16-rounded value a bf16 cache would have stored), V rows as projected.
  prefill                attends over the unquantised K / V of its own tokens exactly as with a bf16 cache (so its logits
                         do not depend on the cache format); only what it STORES is quantised           (prefill_cache)
  decode                 attends over what is stored: every key of step t, the one appended in that step included, is the
                         dequantised row float(q) * scale. Scores and softmax in fp32:
                         score = (q . k_q) * k_scale * d^-1/2,  o += p * v_scale * v_q                   (decode_attention)

Layout mirrors the device cache: k8 / v8 [B][H][Smax][128] float8_e4m3fn, ks / vs [B][H][Smax] fp32 per layer.
"""
import torch
import torch.nn.functional as F

from . import fp8_oracle as F8
from . import llava_oracle as O

D = 128
BYTES_PER_HEAD_TOKEN = 2 * (D + 4)        # K and V: 128 e4m3 bytes + one fp32 scale each
BYTES_PER_HEAD_TOKEN_BF16 = 2 * D * 2


def quantize_kv(x):
    """x [..., 128] -> (q float8_e4m3fn [..., 128], scale fp32 [...])."""
    assert x.shape[-1] == D
    return F8.quantize_rows_e4m3(x)


def dequantize_kv(q, scale):
    return q.float() * scale.unsqueeze(-1)


def rope_bf16(x, pos, theta=10000.0):
    """HF apply_rotary_pos_emb with its bf16 rounding points (cos / sin cast to bf16, bf16 products and sum):
    x [B, H, 128] bf16, pos [B] -> bf16."""
    cos, sin = O._rope_cos_sin(pos[:, None], D, theta, torch.bfloat16)     # [B, 1, 128]
    x = x.to(torch.bfloat16)
    return x * cos + O._rotate_half(x) * sin


def empty_cache(B, H, Smax):
    z8 = lambda: torch.zeros(B, H, Smax, D).to(torch.float8_e4m3fn)
    return dict(k8=z8(), v8=z8(), ks=torch.zeros(B, H, Smax), vs=torch.zeros(B, H, Smax))


def store_rows(cache, k, v, seq_lens=None, slot0=0):
    """The prefill cache write: k (roped) / v [B, H, S, 128] -> rows t < seq_lens[b] of slots slot0.. of the cache."""
    B, _, S, _ = k.shape
    for b in range(B):
        n = S if seq_lens is None else int(seq_lens[b])
        for src, q8, sc in ((k, "k8", "ks"), (v, "v8", "vs")):
            q, s = quantize_kv(src[b, :, :n].to(torch.bfloat16))
            cache[q8][slot0 + b, :, :n] = q
            cache[sc][slot0 + b, :, :n] = s


def decode_attention(q, k_new, v_new, cache, lens):
    """One decode-attention call over a quantised cache. q / k_new (both roped) and v_new: [B, H, 128]; lens[b] = rows already
    stored for sample b. Appends the quantised new row at lens[b] IN PLACE and attends over rows 0..lens[b] as stored.
    Returns fp32 [B, H, 128]."""
    B, H, _ = q.shape
    out = torch.empty(B, H, D)
    for b in range(B):
        n = int(lens[b])
        for src, q8, sc in ((k_new, "k8", "ks"), (v_new, "v8", "vs")):
            qq, s = quantize_kv(src[b].to(torch.bfloat16))
            cache[q8][b, :, n] = qq
            cache[sc][b, :, n] = s
        kq, ks = cache["k8"][b, :, :n + 1].float(), cache["ks"][b, :, :n + 1]
        vq, vs = cache["v8"][b, :, :n + 1].float(), cache["vs"][b, :, :n + 1]
        score = torch.einsum("hd,hnd->hn", q[b].float(), kq) * ks * D ** -0.5
        p = torch.softmax(score, dim=-1)
        out[b] = torch.einsum("hn,hnd->hd", p * vs, vq)
    return out


def decode_attn_call(qkv, cache, lens, H, theta=10000.0, k_roped=None):
    """The kernel-level call (b2_op_decode_attn_e4m3): qkv [B, 3*H*128] bf16 rows of the new token, RoPE at position lens[b]
    on q and k, append, attend. `k_roped` [B, H, 128] overrides the roped k (tests pass the row the bf16 kernel stored, whose
    sin / cos may differ from torch's in the last bf16 bit). Returns fp32 [B, H*128]."""
    B = qkv.shape[0]
    v3 = qkv.view(B, 3, H, D)
    pos = torch.as_tensor(lens, dtype=torch.long)
    q = rope_bf16(v3[:, 0], pos, theta)
    k = rope_bf16(v3[:, 1], pos, theta) if k_roped is None else k_roped
    return decode_attention(q, k, v3[:, 2], cache, lens).reshape(B, H * D)


# ---- engine level: prefill that fills a quantised cache, and the decode step over it ---------------------------------
def prefill_cache(w, embeds, cfg, Smax, seq_lens=None, last_only=False):
    """llama_forward over the prompt (unquantised attention: the logits are those of the bf16-cache oracle) plus the
    quantised cache it leaves behind: (logits fp32 [B, S, V] ([B, 1, V] with last_only), [cache per layer])."""
    logits, kv = O.llama_forward(w, embeds, cfg, last_only=last_only)
    B, H = embeds.shape[0], cfg["heads"]
    caches = []
    for k, v in kv:
        c = empty_cache(B, H, Smax)
        store_rows(c, k, v, seq_lens)
        caches.append(c)
    return logits, caches


def decode_step(w, tokens, cfg, caches, lens, dtype=torch.float32):
    """One decode step (O.llama_forward with S = 1, per-sample positions lens[b]) whose attention is decode_attention over
    the quantised caches; q / k / v are rounded to bf16 where the engine's QKV projection stores them. Appends IN PLACE;
    the caller advances lens. Returns fp32 logits [B, V]."""
    h, H = cfg["hidden"], cfg["heads"]
    x = w["model.embed_tokens.weight"].to(dtype)[tokens]                      # [B, h]
    B = x.shape[0]
    pos = torch.as_tensor(lens, dtype=torch.long)
    for i in range(cfg["layers"]):
        p = f"model.layers.{i}."
        W = lambda k: w[p + k].to(dtype)
        y = O._rmsnorm(x, W("input_layernorm.weight"), cfg["rms_eps"])
        q = F.linear(y, W("self_attn.q_proj.weight")).view(B, H, D).to(torch.bfloat16)
        k = F.linear(y, W("self_attn.k_proj.weight")).view(B, H, D).to(torch.bfloat16)
        v = F.linear(y, W("self_attn.v_proj.weight")).view(B, H, D).to(torch.bfloat16)
        a = decode_attention(rope_bf16(q, pos, cfg["rope_theta"]), rope_bf16(k, pos, cfg["rope_theta"]), v, caches[i], lens)
        x = x + F.linear(a.reshape(B, h).to(dtype), W("self_attn.o_proj.weight"))
        y = O._rmsnorm(x, W("post_attention_layernorm.weight"), cfg["rms_eps"])
        x = x + F.linear(F.silu(F.linear(y, W("mlp.gate_proj.weight"))) * F.linear(y, W("mlp.up_proj.weight")),
                         W("mlp.down_proj.weight"))
    x = O._rmsnorm(x, w["model.norm.weight"].to(dtype), cfg["rms_eps"])
    return F.linear(x, w["lm_head.weight"].to(dtype)).float()


def greedy_generate(w, embeds, cfg, max_new_tokens, Smax):
    """Greedy ids [B, N] of equal-length prompts `embeds` [B, S, h] decoded over the quantised cache."""
    logits, caches = prefill_cache(w, embeds, cfg, Smax)
    lens = [embeds.shape[1]] * embeds.shape[0]
    tok = logits[:, -1].argmax(-1)
    toks = [tok]
    for _ in range(max_new_tokens - 1):
        tok = decode_step(w, tok, cfg, caches, lens).argmax(-1)
        lens = [n + 1 for n in lens]
        toks.append(tok)
    return torch.stack(toks, dim=1)


# ---- error model ---------------------------------------------------------------------------------------------------
ROW_REL_ERROR_MAX = 2.0 ** -4      # |deq - x| <= 2^-4 |x| for normal codes (3 mantissa bits, round to nearest) ...
ROW_ABS_ERROR_FLOOR = 2.0 ** -10   # ... and <= 2^-10 * amax * (448/448) in the subnormal range (step 2^-9 of the scaled value)


def expected_attention_error():
    """Error of one decode-attention output relative to its RMS, e4m3 cache vs bf16 cache, on unit-variance q / k / v: each
    stored element carries a relative rounding error of RMS 2^-4 / sqrt(3) ~ 3.6 %. On V it passes through the softmax
    average unchanged in relative terms (signal and noise both shrink as 1 / sqrt(n_eff)): ~3.6 % of the output RMS. On K it
    perturbs every score by ~3.6 % of the score's RMS (1 after the d^-1/2 scaling), i.e. p by ~3.6 % of itself, which adds
    another ~3.6 % in quadrature: ~5.1 % together, independent of the number of keys."""
    return 2.0 ** -4 / 3 ** 0.5 * 2 ** 0.5
