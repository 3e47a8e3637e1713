"""Conversation prefix reuse for generate() (config.b2_prefix_cache / B2_PREFIX_CACHE=1): host-side bookkeeping only.

A multi-turn caller (llava/serve/cli.py, the model worker behind the Gradio servers) sends the whole conversation on every
turn: the same image and a prompt that extends the previous prompt and answer. A cache released by generate() keeps a record
of what its rows hold; the next call prefills only the part of its prompt that is not already there (b2_prefill_at).

A record is a list of items in spliced order: an int is one token row, a tensor is the pixels of one image placeholder slot
and stands for that slot's feature rows. Two placeholders match only when their pixels are equal (`torch.equal`, same shape,
dtype and device): callers decode the image again for every request, so identity says nothing.
"""
import torch


def item_rows(item, rows_per_image):
    """Spliced rows of one item: 1 for a token, rows_per_image per image in the slot (a [3,H,W] slot holds one image,
    an [n,3,H,W] slot n)."""
    if isinstance(item, int):
        return 1
    return rows_per_image * (item.shape[0] if item.dim() == 4 else 1)


def _same_image(a, b):
    return (a.shape == b.shape and a.dtype == b.dtype and a.device == b.device and bool(torch.equal(a, b)))


def match_rows(cached, new, rows_per_image):
    """Spliced rows at the front of `new` that `cached` already holds: items are compared one by one and the walk stops at
    the first difference (an image counts whole or not at all)."""
    m = 0
    for a, b in zip(cached, new):
        if isinstance(a, int) != isinstance(b, int):
            break
        if isinstance(a, int):
            if a != b:
                break
        elif not _same_image(a, b):
            break
        m += item_rows(a, rows_per_image)
    return m


def reusable_rows(cached, new, rows_per_image):
    """match_rows capped at (spliced length of `new`) - 1: at least one row is always prefilled, because the first token of
    the answer is chosen from the prefill's last-position logits (a regenerated answer re-sends the same prompt)."""
    total = sum(item_rows(it, rows_per_image) for it in new)
    return min(match_rows(cached, new, rows_per_image), total - 1)


def record_after_generation(prompt_items, returned_tokens):
    """What a cache's rows hold once generate() returns: the spliced prompt and every returned token but the last. Token t
    of the answer is written into the cache by the decode step that feeds it; the last returned token may never have been
    fed, and rows of steps queued past the stop are never trusted."""
    return list(prompt_items) + [int(t) for t in list(returned_tokens)[:-1]]


def select(records, new, rows_per_image):
    """Pick the free cache for a prompt: records[i] is the record of free cache i (None = nothing reusable), ordered from
    least to most recently released. Returns (index, rows): the cache with the longest reusable prefix, or (0, 0) — the
    least recently used one — when none has any."""
    best, best_m = 0, 0
    for i, rec in enumerate(records):
        if rec is None:
            continue
        m = reusable_rows(rec, new, rows_per_image)
        if m > best_m:
            best, best_m = i, m
    return best, best_m


def chunk_source_index(src, m, skipped_rows, pad_row):
    """Rows [m, L) of a host splice index (llava_arch.build_source_index, one row), for features of the images that were
    actually encoded: the slots wholly inside the reused prefix (their `skipped_rows` feature rows) are left out of the
    feature tensor, so every feature reference moves down by that many rows."""
    out = src[m:].copy()
    feat = (out < 0) & (out != pad_row)
    out[feat] += skipped_rows
    return out
