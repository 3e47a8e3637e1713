"""Host half of beam search (generate(num_beams > 1)).

`BeamSearch` restates the bookkeeping of transformers 5.5 `GenerationMixin._beam_search` (and its helpers
`_get_running_beams_for_next_iteration`, `_update_finished_beams`, `_check_early_stop_heuristic`,
`_beam_search_has_unfinished_sequences`) over the K = max(2, 1 + n_eos) * num_beams candidates per sample that the device
selects each step (b2_op_beam_topk / b2_beam_step): running beams, finished hypotheses with their length penalty, the early-stop
heuristic, termination and the output tensor. The arithmetic on scores is HF's, in fp32 on the CPU, in HF's order. Beside the
running and finished sequences it carries HF's beam-index tensors (the flat running beam b * num_beams + j each generated token
came from), gathered the same way, for generate(return_dict_in_generate=True)'s `beam_indices`.

`SlotPlanner` keeps the map from running beam to KV-cache slot and turns each step's parent vector into a list of slot copies:
a parent's first child stays in the parent's slot (it only appends a row); every further child takes the slot of a parent that
has no child left, as a copy of the parent's rows. No copy then reads a slot another copy of the same step writes, and the
number of copies is num_beams minus the number of distinct surviving parents.

Pure CPU torch: no engine calls.
"""
import torch


def stopping_hits(ids, stopping_criteria, max_length, eos_ids):
    """HF StoppingCriteriaList over candidate sequences ids [N, cur]: the OR of max length, eos on the last token and every
    caller criterion. A criterion returning a plain bool applies to every row."""
    n, cur = ids.shape
    done = torch.full((n,), cur >= max_length, dtype=torch.bool)
    if eos_ids:
        done = done | torch.isin(ids[:, -1], torch.tensor(list(eos_ids), dtype=ids.dtype))
    for crit in stopping_criteria or ():
        r = crit(ids, None)
        done = done | (r.to("cpu", torch.bool) if torch.is_tensor(r) else bool(r))
    return done


class BeamSearch:
    """State of one beam-search generation of B samples. prompt: CPU int64 [B, Lt] (the caller's ids, image placeholders
    included); eos_ids: list of ints or None."""

    def __init__(self, prompt, num_beams, max_new_tokens, eos_ids=None, length_penalty=1.0, early_stopping=False,
                 num_return_sequences=1, pad_token_id=None, stopping_criteria=None):
        if num_return_sequences > num_beams:
            raise ValueError(f"num_return_sequences ({num_return_sequences}) must be <= num_beams ({num_beams})")
        if early_stopping not in (False, True, "never"):
            raise ValueError(f"early_stopping must be False, True or 'never', got {early_stopping!r}")
        prompt = prompt.to("cpu", torch.int64)
        self.B, self.Lt = prompt.shape
        self.nb = nb = int(num_beams)
        self.max_length = self.Lt + int(max_new_tokens)
        self.eos_ids = None if eos_ids is None else [int(e) for e in eos_ids]
        self.K = max(2, 1 + len(self.eos_ids or [])) * nb
        self.length_penalty, self.early_stopping = length_penalty, early_stopping
        self.num_return_sequences = int(num_return_sequences)
        self.criteria = stopping_criteria
        # HF: `pad_token_id or eos_token_id[0] if eos_token_id is not None else -1` (a pad id of 0 falls through to eos)
        if self.eos_ids is None:
            self.fill = -1
        else:
            self.fill = pad_token_id or (self.eos_ids[0] if self.eos_ids else -1)
        B = self.B
        self.running = torch.full((B, nb, self.max_length), self.fill, dtype=torch.int64)
        self.running[:, :, :self.Lt] = prompt[:, None, :]
        self.sequences = self.running.clone()
        self.running_scores = torch.zeros(B, nb, dtype=torch.float32)
        self.running_scores[:, 1:] = -1e9
        self.beam_scores = torch.full((B, nb), -1e9, dtype=torch.float32)
        self.gen_len = torch.zeros(B, nb, dtype=torch.int64)          # generated tokens of each finished hypothesis
        self.is_sent_finished = torch.zeros(B, nb, dtype=torch.bool)
        self.unsatisfied = torch.ones(B, 1, dtype=torch.bool)
        self.top_mask = torch.cat([torch.ones(nb, dtype=torch.bool), torch.zeros(self.K - nb, dtype=torch.bool)])
        self.cur_len = self.Lt
        self.parents = torch.zeros(B, nb, dtype=torch.int64)          # running beam j came from beam parents[b, j]
        # HF's running / finished beam indices: int32, -1 where nothing was generated
        self.running_beam_indices = torch.full((B, nb, self.max_length - self.Lt), -1, dtype=torch.int32)
        self.beam_indices = self.running_beam_indices.clone()
        self.done = False

    @staticmethod
    def _gather(t, idx):
        while idx.dim() < t.dim():
            idx = idx.unsqueeze(-1)
        return torch.take_along_dim(t, idx, dim=1)

    def step(self, topk_scores, topk_tokens, topk_beams):
        """One step from the device's candidates [B, K] (accumulated score, token, beam within the sample; best first).
        Returns True when the search is over."""
        B, K, nb, cur = self.B, self.K, self.nb, self.cur_len
        topk_scores = topk_scores.to("cpu", torch.float32).reshape(B, K)
        topk_tokens = topk_tokens.to("cpu", torch.int64).reshape(B, K)
        topk_beams = topk_beams.to("cpu", torch.int64).reshape(B, K)
        cand = self._gather(self.running, topk_beams)
        cand[:, :, cur] = topk_tokens
        cand_bi = self._gather(self.running_beam_indices, topk_beams)
        cand_bi[:, :, cur - self.Lt] = (topk_beams + torch.arange(B).view(-1, 1) * nb).to(torch.int32)
        hits = stopping_hits(cand[:, :, :cur + 1].reshape(B * K, cur + 1), self.criteria, self.max_length,
                             self.eos_ids).reshape(B, K)

        # running beams of the next step: the best num_beams candidates that did not hit a criterion
        run_scores = topk_scores + hits.to(torch.float32) * -1.0e9
        nxt = torch.topk(run_scores, k=nb)[1]
        self.running = self._gather(cand, nxt)
        self.running_scores = self._gather(run_scores, nxt)
        self.running_beam_indices = self._gather(cand_bi, nxt)
        self.parents = self._gather(topk_beams, nxt)

        # finished hypotheses: candidates among the first num_beams that hit a criterion, length-normalised
        did = hits & self.top_mask[None, :]
        s = topk_scores / ((cur + 1 - self.Lt) ** self.length_penalty)
        full = torch.all(self.is_sent_finished, dim=-1, keepdim=True) & (self.early_stopping is True)
        s = s + full.to(torch.float32) * -1.0e9
        s = s + (~self.unsatisfied).to(torch.float32) * -1.0e9
        s = s + (~did) * -1.0e9
        m_seq = torch.cat((self.sequences, cand), dim=1)
        m_scores = torch.cat((self.beam_scores, s), dim=1)
        m_len = torch.cat((self.gen_len, torch.full((B, K), cur + 1 - self.Lt, dtype=torch.int64)), dim=1)
        m_fin = torch.cat((self.is_sent_finished, did), dim=1)
        m_bi = torch.cat((self.beam_indices, cand_bi), dim=1)
        keep = torch.topk(m_scores, k=nb)[1]
        self.sequences = self._gather(m_seq, keep)
        self.beam_scores = self._gather(m_scores, keep)
        self.gen_len = self._gather(m_len, keep)
        self.is_sent_finished = self._gather(m_fin, keep)
        self.beam_indices = self._gather(m_bi, keep)

        self.cur_len = cur = cur + 1
        if self.early_stopping == "never" and self.length_penalty > 0.0:
            best_len = self.max_length - self.Lt
        else:
            best_len = cur - self.Lt
        best_running = self.running_scores[:, :1] / (best_len ** self.length_penalty)
        worst_finished = torch.where(self.is_sent_finished, torch.min(self.beam_scores, dim=1, keepdim=True)[0], -1.0e9)
        self.unsatisfied = self.unsatisfied & torch.any(best_running > worst_finished, dim=-1, keepdim=True)
        go_on = (bool(torch.any(self.unsatisfied)) and not (bool(torch.all(self.is_sent_finished)) and self.early_stopping is True)
                 and not bool(torch.all(hits)))
        self.done = not go_on
        return self.done

    def next_tokens(self):
        """Token each running beam feeds to the next decode step, [B * nb] in beam order."""
        return self.running[:, :, self.cur_len - 1].reshape(-1)

    def output(self):
        """(sequences [B * num_return_sequences, Lt + longest returned continuation], their scores), best first per sample."""
        r = self.num_return_sequences
        seq = self.sequences[:, :r].reshape(self.B * r, -1)
        n = int(self.gen_len[:, :r].max())
        return seq[:, :self.Lt + n].clone(), self.beam_scores[:, :r].reshape(-1).clone()

    def output_beam_indices(self):
        """HF's `beam_indices` of the returned sequences: int32 [B * num_return_sequences, longest returned continuation], the
        flat running beam each generated token came from, -1 past a sequence's end."""
        r = self.num_return_sequences
        bi = self.beam_indices[:, :r].reshape(self.B * r, -1)
        n = int(((bi + 1) != 0).sum(dim=1).max())
        return bi[:, :n].clone()


class SlotPlanner:
    """Beam -> KV-cache slot map of B samples x nb beams in a cache of >= B * nb slots. Before the first step sample b's prompt
    sits in slot b alone; its other beams are given slots B + b * (nb - 1) + j, which the first plan fills by copying slot b."""

    def __init__(self, B, nb):
        self.B, self.nb = B, nb
        self.slot_of = [[b] + [B + b * (nb - 1) + j for j in range(nb - 1)] for b in range(B)]

    def plan(self, parents):
        """parents [B, nb] (beam j of the next step continues beam parents[b][j]) -> list of (src, dst) slot copies, to be
        applied before the next step's tokens are fed; updates the map."""
        copies = []
        for b in range(self.B):
            old = self.slot_of[b]
            par = [int(p) for p in parents[b]]
            taken = set()
            free = [old[p] for p in range(self.nb) if p not in par]
            new = [None] * self.nb
            later = []
            for j, p in enumerate(par):
                if p not in taken:
                    taken.add(p)
                    new[j] = old[p]
                else:
                    later.append(j)
            for j, slot in zip(later, free):
                new[j] = slot
                copies.append((old[par[j]], slot))
            self.slot_of[b] = new
        return copies

    def flat(self):
        return [s for row in self.slot_of for s in row]
