"""Beam search as plain PyTorch over full sequences (test infrastructure; the product never imports it).

`beam_search(logits_fn, prompt, ...)` restates transformers 5.5 `GenerationMixin._beam_search` (generation/utils.py) with no
KV cache: every step calls `logits_fn(sequences [B*nb, cur]) -> fp32 logits [B*nb, V]` on the running beams' whole sequences,
so it defines what beam search computes independently of how an engine reorders its cache slots.

Candidate selection follows the rule the device kernel documents (b2_op_beam_topk): the K best of
log_softmax(logits) + running score over num_beams * V continuations, ties to the lower beam * V + token. HF uses torch.topk,
whose tie order is unspecified; on untied scores the two agree (tests/test_beam_host.py checks it against the installed
transformers).

`condition_weights_beam` extends llava_oracle.condition_weights for strict-id beam tests (see its docstring)."""
import torch


def select_candidates(log_probs, K):
    """log_probs [B, nb * V] -> (scores, flat indices) [B, K], score descending, ties to the lower flat index."""
    s, i = torch.sort(log_probs, dim=1, descending=True, stable=True)
    return s[:, :K], i[:, :K]


def beam_search(logits_fn, prompt, num_beams, max_new_tokens, eos_token_id=None, pad_token_id=None, length_penalty=1.0,
                early_stopping=False, num_return_sequences=1, stopping_criteria=None, return_margins=False):
    """Returns (sequences [B * num_return_sequences, L], sequences_scores [B * num_return_sequences]) and, with
    return_margins, the score gaps behind every decision of every step: candidate ranks K / K+1 and num_beams / num_beams+1
    of the accumulated log-probabilities, and ranks num_beams / num_beams+1 of the running selection while it is used."""
    prompt = prompt.to("cpu", torch.int64)
    B, Lt = prompt.shape
    nb = num_beams
    eos = None if eos_token_id is None else ([eos_token_id] if isinstance(eos_token_id, int) else list(eos_token_id))
    K = max(2, 1 + len(eos or [])) * nb
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
    cur = Lt
    margins = []
    while True:
        logits = logits_fn(running[:, :, :cur].reshape(B * nb, cur)).to(torch.float32).cpu()
        V = logits.shape[-1]
        lp = torch.log_softmax(logits, dim=-1).view(B, nb, V) + run_scores[:, :, None]
        lp = lp.reshape(B, nb * V)
        if return_margins:  # which K candidates, and which of them are the first num_beams
            srt = torch.sort(lp, dim=1, descending=True)[0]
            margins.append(float(torch.minimum(srt[:, K - 1] - srt[:, K], srt[:, nb - 1] - srt[:, nb]).min()))
        top_s, top_i = select_candidates(lp, K)
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
        if return_margins and not bool(hits.all()):  # which candidates run on (unused once every candidate has stopped)
            srt = torch.sort(rs, dim=1, descending=True)[0]
            margins.append(float((srt[:, nb - 1] - srt[:, nb]).min()))
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
        best_len = (max_length - Lt) if (early_stopping == "never" and length_penalty > 0.0) else (cur - Lt)
        worst = torch.where(finished, beam_scores.min(1, keepdim=True)[0], -1.0e9)
        unsat = unsat & (run_scores[:, :1] / (best_len ** length_penalty) > worst).any(-1, keepdim=True)
        if not (unsat.any() and not (finished.all() and early_stopping is True) and not hits.all()):
            break
    r = num_return_sequences
    n = int(gen_len[:, :r].max())
    out = sequences[:, :r].reshape(B * r, -1)[:, :Lt + n], beam_scores[:, :r].reshape(-1)
    return (out + (margins,)) if return_margins else out


def condition_weights_beam(w, cfg, seed=0, mix=(1.0, 0.71, 0.53, 0.37), layer_gain=None):
    """condition_weights (llava_oracle) for beam search: lm_head is tied to a weighted sum of len(mix) permutations of the
    embedding table, lm_head[perm_i[t]] += mix[i] * embed[t], with incommensurate weights. The hidden state keeps a large cosine
    with the embedding of the token fed, so the logits of the continuations beam search compares are separated by multiples of
    those weights' differences: far above bf16 noise, also after scores are summed over steps. Returns a NEW dict."""
    import math

    g = torch.Generator().manual_seed(2000 + seed)
    V = cfg["vocab"]
    if layer_gain is None:
        layer_gain = min(1.0, 2.0 / math.sqrt(2.0 * cfg["layers"]))
    out = dict(w)
    emb = w["model.embed_tokens.weight"].float()
    head = torch.zeros(V, emb.shape[1], device=emb.device)
    for c in mix:
        head[torch.randperm(V, generator=g).to(emb.device)] += c * emb
    out["lm_head.weight"] = head.to(torch.bfloat16).to(w["lm_head.weight"].dtype)
    for i in range(cfg["layers"]):
        for k in ("self_attn.o_proj.weight", "mlp.down_proj.weight"):
            key = f"model.layers.{i}.{k}"
            out[key] = (w[key].float() * layer_gain).to(torch.bfloat16).to(w[key].dtype)
    return out
