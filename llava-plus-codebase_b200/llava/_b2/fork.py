"""Host plan of generate(do_sample=True, num_return_sequences=n): B prompts, n samples each, B * n rows of one KV cache.

Prompt b is prefilled once, into slot b (its leader, sample 0). Sample j >= 1 of prompt b is a follower in slot
B + b * (n - 1) + (j - 1), which one b2_kv_copy_slots call fills with the leader's rows [0, len_b): sources [0, B), destinations
[B, B * n), so no slot is both, and none is written twice. The device keeps this slot order for the whole generation; the host
reads every token, score row and stopping-criteria row through `slot_of_row`, which maps HF's row b * n + j (the order
repeat_interleave gives) to its slot.

The decode attention reads a prompt once for all of its samples through the group table (b2_stream_begin_groups): one group
per prompt naming slot b and prefix length len_b, its n rows split into groups of at most 16 that all name slot b.

Pure Python: no engine calls.
"""

GROUP_ROWS = 16


class ForkPlan:
    def __init__(self, lens, n):
        self.B, self.n = len(lens), int(n)
        if self.B < 1 or self.n < 1:
            raise ValueError(f"a fork needs at least one prompt and one sample (got {self.B} prompts, n={n})")
        self.lens = [int(x) for x in lens]
        self.rows = self.B * self.n

    def slot(self, b, j):
        """Cache slot of sample j of prompt b."""
        return b if j == 0 else self.B + b * (self.n - 1) + (j - 1)

    @property
    def slot_of_row(self):
        """slot_of_row[b * n + j] = slot of sample j of prompt b (HF row order -> device slot order)."""
        return [self.slot(b, j) for b in range(self.B) for j in range(self.n)]

    @property
    def prompt_of_slot(self):
        """The prompt whose rows each slot holds, in slot order (the index_select that expands the prefill logits)."""
        out = [0] * self.rows
        for b in range(self.B):
            for j in range(self.n):
                out[self.slot(b, j)] = b
        return out

    def copies(self):
        """(src, dst) slot lists of the one kv_copy_slots call that fills the followers."""
        src = [b for b in range(self.B) for _ in range(1, self.n)]
        dst = [self.slot(b, j) for b in range(self.B) for j in range(1, self.n)]
        return src, dst

    def groups(self):
        """(src_slot, prefix_len, rows) per group: each prompt's n slots, in chunks of at most GROUP_ROWS."""
        out = []
        for b in range(self.B):
            slots = [self.slot(b, j) for j in range(self.n)]
            for i in range(0, self.n, GROUP_ROWS):
                out.append((b, self.lens[b], slots[i:i + GROUP_ROWS]))
        return out
