"""Beam sampling as plain PyTorch / numpy over full sequences (test infrastructure; the product never imports it).

`beam_search(..., do_sample=True)` extends oracle/beam_oracle.beam_search with transformers 5.5 `GenerationMixin._beam_search`
under do_sample: per step the running beams' log_softmax rows go through HF's warpers (Temperature -> TopK -> TopP, each
keeping at least min_keep = 1 + n_eos tokens, 2 without eos ids), the running scores are added, and K candidates per sample are
drawn without replacement from softmax over nb * V. Two samplers:
  sampler="torch"   torch.multinomial(softmax(acc), K) exactly as HF calls it (the warpers restated in torch, op for op);
  sampler="philox"  the device rule of b2_op_beam_sample restated in numpy: warpers in fp32 (top-p over 2^-40 fixed-point
                    masses, as csrc/sampling.cu), keys fp32(acc + g) with g = -log(-log u) in fp64 from
                    oracle/sampling_oracle.philox_u64(seed, step, (b * nb + j) * V + token); finite keys first by key, then -inf
                    candidates by flat index, then NaN.
Without do_sample it is oracle/beam_oracle.beam_search."""
import numpy as np
import torch

from oracle import beam_oracle as BO
from oracle import sampling_oracle as SO

M32 = 0xFFFFFFFF


def min_keep_of(eos):
    """HF _get_logits_processor: min_tokens_to_keep = 1 + number of eos ids (an empty list counts 0), 2 without eos ids."""
    return 2 if eos is None else 1 + len(eos)


# ---------------------------------------------------------------------------------------------------- warpers (torch, HF)
def hf_warp(lp, temperature=1.0, top_k=0, top_p=1.0, min_keep=1):
    """HF 5.5 TemperatureLogitsWarper -> TopKLogitsWarper -> TopPLogitsWarper on log-probabilities lp [N, V] (fp32), restated."""
    s = lp
    if temperature != 1.0:
        s = s / temperature
    if top_k:
        k = min(max(int(top_k), min_keep), s.shape[-1])
        s = s.masked_fill(s < torch.topk(s, k)[0][..., -1, None], float("-inf"))
    if top_p is not None and top_p < 1.0:
        srt, idx = torch.sort(s, descending=False)
        cum = srt.softmax(dim=-1).cumsum(dim=-1)
        rm = cum <= (1 - top_p)
        rm[..., -min_keep:] = 0
        s = s.masked_fill(rm.scatter(1, idx, rm), float("-inf"))
    return s


def hf_warp_installed(lp, temperature=1.0, top_k=0, top_p=1.0, min_keep=1):
    """The same through the installed transformers' warper classes."""
    from transformers.generation.logits_process import TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper

    ids = torch.zeros(lp.shape[0], 1, dtype=torch.long)
    s = lp
    if temperature != 1.0:
        s = TemperatureLogitsWarper(float(temperature))(ids, s)
    if top_k:
        s = TopKLogitsWarper(int(top_k), min_tokens_to_keep=min_keep)(ids, s)
    if top_p is not None and top_p < 1.0:
        s = TopPLogitsWarper(float(top_p), min_tokens_to_keep=min_keep)(ids, s)
    return s


# ---------------------------------------------------------------------------------------------- warpers (numpy, device rule)
def log_softmax32(x):
    """fp32 log_softmax in torch's rounding order ((x - max) - lse), NaN skipped in max and sum."""
    x = np.asarray(x, dtype=np.float32)
    fin = ~np.isnan(x)
    mx = np.float32(x[fin].max()) if fin.any() else np.float32(-np.inf)
    lse = np.float32(np.log(np.exp((x[fin] - mx).astype(np.float32)).astype(np.float32).sum(dtype=np.float32)))
    return ((x - mx).astype(np.float32) - lse).astype(np.float32)


def kept_mask(w, top_k=0, top_p=1.0, min_keep=1):
    """Survivors of top-k then top-p over warped scores w (fp32 row) with at least min_keep of each (device rule):
    oracle/sampling_oracle.kept_mask at temperature 1 (its top-p over 2^-40 fixed-point masses) with k = max(top_k, min_keep),
    and the min_keep largest w (ties kept) added back to the top-p survivors. They are also top-k survivors, as k >= min_keep.
    NaN never survives."""
    w = np.asarray(w, dtype=np.float32)
    V = w.shape[0]
    nan = np.isnan(w)
    ws = np.where(nan, -np.inf, w).astype(np.float32)
    k = max(int(top_k), min_keep) if top_k and top_k > 0 else 0
    keep, _ = SO.kept_mask(ws, 1.0, k, top_p)
    if top_p is not None and top_p < 1.0 and min_keep > 1:
        keep |= ws >= np.sort(ws)[V - min_keep]
    return keep & ~nan


def device_warp(x, temperature=1.0, top_k=0, top_p=1.0, min_keep=1):
    """Warped row of the device: fp32 ((x - max) - lse) / T, non-survivors -inf, NaN logits NaN."""
    w = (log_softmax32(x) / np.float32(temperature)).astype(np.float32)
    keep = kept_mask(w, top_k, top_p, min_keep)
    return np.where(keep | np.isnan(w), w, -np.inf).astype(np.float32)


# --------------------------------------------------------------------------------------------------------- Philox keys
def philox_u64_np(seed, index, rows):
    """Vectorised oracle/sampling_oracle.philox_u64 over an array of row counters (uint64 arithmetic on 32-bit words)."""
    rows = np.asarray(rows, dtype=np.uint64)
    m = np.uint64(M32)
    c0 = np.full(rows.shape, index & M32, dtype=np.uint64)
    c1 = rows & m
    c2 = np.zeros_like(c1)
    c3 = np.zeros_like(c1)
    k0, k1 = seed & M32, (seed >> 32) & M32
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * c0
        p1 = np.uint64(0xCD9E8D57) * c2
        c0, c1, c2, c3 = ((p1 >> np.uint64(32)) ^ c1 ^ np.uint64(k0)) & m, p1 & m, ((p0 >> np.uint64(32)) ^ c3 ^ np.uint64(k1)) & m, p0 & m
        k0 = (k0 + 0x9E3779B9) & M32
        k1 = (k1 + 0xBB67AE85) & M32
    return (c0 << np.uint64(32)) | c1


def gumbel(seed, step, flat):
    """g = -log(-log u), u = ((r >> 11) + 0.5) * 2^-53 in fp64, r = Philox(seed; step, flat)."""
    r = philox_u64_np(seed, step, flat)
    u = ((r >> np.uint64(11)).astype(np.float64) + 0.5) * 2.0 ** -53
    return -np.log(-np.log(u))


def philox_select(acc, seed, step, nb, K, sample0=0):
    """acc [B, nb * V] fp32 (warped + running score; -inf dropped, NaN) -> (scores [B, K] fp32, flat [B, K], keys fp64 [B, K]
    of the candidates in key order, and the fp64 keys of every candidate [B, nb * V] with -inf / NaN for the unranked)."""
    acc = np.asarray(acc, dtype=np.float32)
    B, N = acc.shape
    V = N // nb
    out_s, out_i, out_k, allk = [], [], [], []
    for b in range(B):
        a = acc[b]
        fin = np.isfinite(a)
        flat_global = (np.arange(N, dtype=np.uint64) + np.uint64((sample0 + b) * nb * V))
        key64 = np.where(fin, a.astype(np.float64), np.where(np.isnan(a), np.nan, -np.inf))
        key64[fin] += gumbel(seed, step, flat_global[fin])
        key32 = np.where(fin, key64.astype(np.float32).astype(np.float64), -np.inf)
        cls = np.where(fin, 0, np.where(np.isnan(a), 2, 1))
        # finite by fp32 key descending (ties to the lower index), then -inf by index, then NaN by index
        order = np.lexsort((np.arange(N), -np.where(fin, key32, 0.0), cls))[:K]
        out_s.append(a[order])
        out_i.append(order)
        out_k.append(key64[order])
        allk.append(key64)
    return np.stack(out_s), np.stack(out_i), np.stack(out_k), np.stack(allk)


def key_margins(allk, nb, K):
    """Smallest gap between sorted finite keys at the ranks that decide something: K / K+1 (which candidates) and nb / nb+1
    (which may finish a hypothesis), over every sample; inf where fewer finite keys exist."""
    m = float("inf")
    for row in allk:
        s = np.sort(row[np.isfinite(row)])[::-1]
        for r in (nb, K):
            if len(s) > r and s[r - 1] > -1e8:  # keys of beams at -1e9 fill the list by the same fp32 rule in both runs
                m = min(m, float(s[r - 1] - s[r]))
    return m


# --------------------------------------------------------------------------------------------------------- beam search
def beam_search(logits_fn, prompt, num_beams, max_new_tokens, eos_token_id=None, pad_token_id=None, length_penalty=1.0,
                early_stopping=False, num_return_sequences=1, stopping_criteria=None, return_margins=False, do_sample=False,
                temperature=1.0, top_k=50, top_p=1.0, sampler="torch", seed=0):
    """oracle/beam_oracle.beam_search, plus beam sampling with do_sample. With return_margins and sampler="philox" the margins
    are in key space (key_margins per step) followed by the running-selection score gaps, as beam_oracle reports them."""
    if not do_sample:
        return BO.beam_search(logits_fn, prompt, num_beams, max_new_tokens, eos_token_id, pad_token_id, length_penalty,
                              early_stopping, num_return_sequences, stopping_criteria, return_margins)
    prompt = prompt.to("cpu", torch.int64)
    B, Lt = prompt.shape
    nb = num_beams
    eos = None if eos_token_id is None else ([eos_token_id] if isinstance(eos_token_id, int) else list(eos_token_id))
    K = max(2, 1 + len(eos or [])) * nb
    mk = min_keep_of(eos)
    max_length = Lt + max_new_tokens
    fill = -1 if eos is None else (pad_token_id or (eos[0] if eos else -1))
    running = torch.full((B, nb, max_length), fill, dtype=torch.int64)
    running[:, :, :Lt] = prompt[:, None]
    sequences = running.clone()
    run_scores = torch.zeros(B, nb)
    run_scores[:, 1:] = -1e9
    beam_scores = torch.full((B, nb), -1e9)
    gen_len = torch.zeros(B, nb, dtype=torch.int64)
    finished = torch.zeros(B, nb, dtype=torch.bool)
    unsat = torch.ones(B, 1, dtype=torch.bool)
    top_mask = torch.arange(K) < nb
    take = lambda t, i: torch.take_along_dim(t, i.view(*i.shape, *([1] * (t.dim() - 2))), dim=1)
    cur, step = Lt, 0
    margins = []
    while True:
        logits = logits_fn(running[:, :, :cur].reshape(B * nb, cur)).to(torch.float32).cpu()
        V = logits.shape[-1]
        if sampler == "torch":
            w = hf_warp(torch.log_softmax(logits, dim=-1), temperature, top_k, top_p, mk)
            acc = (w.view(B, nb, V) + run_scores[:, :, None]).reshape(B, nb * V)
            top_i = torch.multinomial(torch.softmax(acc, dim=-1), num_samples=K)
            top_s = torch.gather(acc, 1, top_i)
        else:
            w = np.stack([device_warp(r, temperature, top_k, top_p, mk) for r in logits.numpy()])
            acc = (w.reshape(B, nb, V) + run_scores.numpy()[:, :, None].astype(np.float32)).astype(np.float32).reshape(B, nb * V)
            s, i, _, allk = philox_select(acc, seed, step, nb, K)
            top_s, top_i = torch.from_numpy(s.astype(np.float32)), torch.from_numpy(i.astype(np.int64))
            if return_margins:
                margins.append(key_margins(allk, nb, K))
        beams, toks = top_i // V, top_i % V
        cand = take(running, beams)
        cand[:, :, cur] = toks
        ids = cand[:, :, :cur + 1].reshape(B * K, cur + 1)
        hits = torch.full((B * K,), cur + 1 >= max_length)
        if eos:
            hits |= torch.isin(ids[:, -1], torch.tensor(eos))
        for c in stopping_criteria or ():
            r = c(ids, None)
            hits = hits | (r.cpu().bool() if torch.is_tensor(r) else bool(r))
        hits = hits.view(B, K)
        rs = top_s + hits.float() * -1.0e9
        if return_margins and not bool(hits.all()):
            # running selection; candidates at or below -1e8 (hit a criterion, or drawn in the zero-probability fill) tie among
            # themselves, and the host bookkeeping breaks those ties alike for any two runs with the same candidate lists
            srt = torch.sort(rs, dim=1, descending=True)[0]
            gap = srt[:, nb - 1] - srt[:, nb]
            gap = torch.where(srt[:, nb - 1] <= -1e8, torch.full_like(gap, float("inf")), gap)
            margins.append(float(gap.min()))
        nxt = torch.topk(rs, k=nb)[1]
        running, run_scores = take(cand, nxt), take(rs, nxt)
        did = hits & top_mask[None]
        s = top_s / ((cur + 1 - Lt) ** length_penalty)
        s = s + (finished.all(-1, keepdim=True) & (early_stopping is True)).float() * -1.0e9
        s = s + (~unsat).float() * -1.0e9
        s = s + (~did) * -1.0e9
        keep = torch.topk(torch.cat((beam_scores, s), 1), k=nb)[1]
        sequences = take(torch.cat((sequences, cand), 1), keep)
        beam_scores = take(torch.cat((beam_scores, s), 1), keep)
        gen_len = take(torch.cat((gen_len, torch.full((B, K), cur + 1 - Lt)), 1), keep)
        finished = take(torch.cat((finished, did), 1), keep)
        cur += 1
        step += 1
        best_len = (max_length - Lt) if (early_stopping == "never" and length_penalty > 0.0) else (cur - Lt)
        worst = torch.where(finished, beam_scores.min(1, keepdim=True)[0], -1.0e9)
        unsat = unsat & (run_scores[:, :1] / (best_len ** length_penalty) > worst).any(-1, keepdim=True)
        if not (unsat.any() and not (finished.all() and early_stopping is True) and not hits.all()):
            break
    r = num_return_sequences
    n = int(gen_len[:, :r].max())
    out = sequences[:, :r].reshape(B * r, -1)[:, :Lt + n], beam_scores[:, :r].reshape(-1)
    return (out + (margins,)) if return_margins else out
