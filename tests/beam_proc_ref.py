"""Beam search and beam sampling with logits processors, as plain PyTorch / numpy over full sequences (test infrastructure; the
product never imports it).

`beam_search(..., repetition_penalty=, no_repeat_ngram_size=, min_new_tokens=, min_length=)` is the loop of
tests/beam_sampling_ref.beam_search (oracle/beam_oracle.beam_search without do_sample) with transformers 5.5's processing step of
`GenerationMixin._beam_search`: each running beam's log_softmax row goes through oracle/logits_proc_oracle.process against that
beam's running sequence (prompt row, then its generated tokens) before the warpers (under do_sample) and before the running score
is added. With every processor off it computes what those two references compute."""
import numpy as np
import torch

import beam_sampling_ref as BSR
from oracle import beam_oracle as BO
from oracle import logits_proc_oracle as P


def processed_rows(lp, seqs, prompt_len, proc):
    """lp [N, V] fp32 log-probabilities, seqs [N, cur] (each row's running sequence) -> the rows processed by `proc` (the
    keyword arguments of logits_proc_oracle.process)."""
    if not proc:
        return lp
    out = [P.process(lp[i].numpy(), seqs[i].tolist(), prompt_len, **proc) for i in range(lp.shape[0])]
    return torch.from_numpy(np.stack(out))


def beam_search(logits_fn, prompt, num_beams, max_new_tokens, eos_token_id=None, pad_token_id=None, length_penalty=1.0,
                early_stopping=False, num_return_sequences=1, stopping_criteria=None, return_margins=False, do_sample=False,
                temperature=1.0, top_k=50, top_p=1.0, sampler="torch", seed=0, repetition_penalty=1.0, no_repeat_ngram_size=0,
                min_new_tokens=0, min_length=0, return_rows=False):
    """Returns (sequences, sequences_scores), then the margins with return_margins (as beam_sampling_ref reports them), then with
    return_rows the per-step score rows [B * nb, V] HF hands to selection (processed, warped under do_sample)."""
    prompt = prompt.to("cpu", torch.int64)
    B, Lt = prompt.shape
    nb = num_beams
    eos = None if eos_token_id is None else ([eos_token_id] if isinstance(eos_token_id, int) else list(eos_token_id))
    proc = {}
    mg = P.min_generated(min_new_tokens, min_length, Lt) if eos else 0
    if repetition_penalty != 1.0 or no_repeat_ngram_size or mg > 0:
        proc = dict(repetition_penalty=repetition_penalty, no_repeat_ngram_size=no_repeat_ngram_size, min_gen=mg,
                    eos_ids=tuple(eos or ()))
    K = max(2, 1 + len(eos or [])) * nb
    mk = BSR.min_keep_of(eos)
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
    margins, rows = [], []
    while True:
        seqs = running[:, :, :cur].reshape(B * nb, cur)
        logits = logits_fn(seqs).to(torch.float32).cpu()
        V = logits.shape[-1]
        if not do_sample:
            w = processed_rows(torch.log_softmax(logits, dim=-1), seqs, Lt, proc)
            lp = (w.view(B, nb, V) + run_scores[:, :, None]).reshape(B, nb * V)
            if return_margins:
                srt = torch.sort(lp, dim=1, descending=True)[0]
                margins.append(float(torch.minimum(srt[:, K - 1] - srt[:, K], srt[:, nb - 1] - srt[:, nb]).min()))
            top_s, top_i = BO.select_candidates(lp, K)
        elif sampler == "torch":
            w = BSR.hf_warp(processed_rows(torch.log_softmax(logits, dim=-1), seqs, Lt, proc), temperature, top_k, top_p, mk)
            acc = (w.view(B, nb, V) + run_scores[:, :, None]).reshape(B, nb * V)
            top_i = torch.multinomial(torch.softmax(acc, dim=-1), num_samples=K)
            top_s = torch.gather(acc, 1, top_i)
        else:
            ls = processed_rows(torch.from_numpy(np.stack([BSR.log_softmax32(r) for r in logits.numpy()])), seqs, Lt, proc).numpy()
            w = (ls / np.float32(temperature)).astype(np.float32)
            keep = np.stack([BSR.kept_mask(r, top_k, top_p, mk) for r in w])
            w = np.where(keep | np.isnan(w), w, -np.inf).astype(np.float32)
            acc = (w.reshape(B, nb, V) + run_scores.numpy()[:, :, None].astype(np.float32)).astype(np.float32).reshape(B, nb * V)
            s, i, _, allk = BSR.philox_select(acc, seed, step, nb, K)
            top_s, top_i = torch.from_numpy(s.astype(np.float32)), torch.from_numpy(i.astype(np.int64))
            w = torch.from_numpy(w)
            if return_margins:
                margins.append(BSR.key_margins(allk, nb, K))
        rows.append(w.clone())
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
    if return_margins:
        out = out + (margins,)
    if return_rows:
        out = out + (tuple(rows),)
    return out
