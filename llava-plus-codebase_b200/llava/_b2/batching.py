"""Continuous batching of concurrent generate() calls (SURVEY §8f-4).

The reference's worker serves concurrent requests by running up to `limit_model_concurrency` generate() THREADS on one
model (/root/reference/llava/serve/model_worker.py:174-185, :230-243): each is a batch-1 HF loop and the GPU interleaves
them. A decode step at batch 1 and at batch 8 costs almost the same on this hardware (it streams the weights either way), so
here those threads share ONE batched decode step instead: every thread still runs its own host loop (streamer, eos, stopping
criteria — `_stream_decode` in llava_llama.py), but the tokens come from a scheduler that owns a KV cache with `slots` rows:

    admit   a waiting request takes a free slot: its prompt is prefilled INTO that slot (b2_prefill_slots), its first token
            is chosen from the prefill logits with its own sampling parameters, the slot is armed (b2_batch_set_row)
    step    one batched decode step over all slots (b2_stream_enqueue(1)): per-slot greedy / temperature-top-k-top-p
            selection on the device, tokens published to pinned host memory (b2_stream_wait)
    retire  a request that finished (max_new_tokens, or cancelled by its consumer after eos / a stopping criterion)
            frees its slot for the next waiting request

Requests never interact numerically: a row's logits depend on its own cache slot only.
"""
import queue
import threading

import torch

from . import LOGITS_LAST, make_sampling


class Request:
    """One generation in flight. The consumer thread reads tokens with `get()`; `cancel()` retires it early."""

    def __init__(self, embeds, length, sampling, max_new_tokens, proc=None):
        self.embeds, self.length, self.sampling, self.max_new_tokens = embeds, int(length), sampling, int(max_new_tokens)
        self.proc = proc  # LogitsProc over the request's prompt ids (device), or None
        self.tokens = queue.Queue()
        self.produced = 0
        self.cancelled = False
        self.error = None
        self.slot = None

    def get(self, timeout=120.0):
        item = self.tokens.get(timeout=timeout)
        if isinstance(item, BaseException):
            raise item
        return item

    def cancel(self):
        self.cancelled = True


class RequestStream:
    """Engine-shaped view of a Request for `_stream_decode` (stream_begin / stream_enqueue / stream_wait)."""

    def __init__(self, request):
        self.request = request

    def stream_begin(self, kv, logits, sampling):
        pass

    def stream_enqueue(self, kv, n):
        pass  # the scheduler decides when steps run

    def stream_wait(self, kv, index, B, timeout_ms=120000):
        return [self.request.get(timeout=timeout_ms / 1000.0)]


class ContinuousBatcher:
    def __init__(self, engine, slots, max_seq, kv_dtype="bf16", _cuda=None):
        """`kv_dtype`: element format of the shared cache ("bf16" | "e4m3"). `_cuda`: the namespace streams / events come from (torch.cuda; the CPU tests of the scheduling logic pass a stand-in)."""
        self._cuda = _cuda if _cuda is not None else torch.cuda
        if slots < 2:
            raise ValueError("continuous batching needs at least 2 slots")
        self.engine, self.slots, self.max_seq = engine, int(slots), int(max_seq)
        self.kv = engine.new_kv(self.slots, self.max_seq) if kv_dtype == "bf16" else engine.new_kv(self.slots, self.max_seq, dtype=kv_dtype)
        self.pending = queue.Queue()
        self.active = {}                      # slot -> Request
        self.free = list(range(self.slots))[::-1]
        self.step = 0                         # decode steps scheduled so far (= index of the next ring entry)
        self.wake = threading.Event()
        self.closed = False
        self.stats = {"steps": 0, "admitted": 0, "max_active": 0, "rows_stepped": 0}
        self.stream = self._cuda.Stream(device=engine.device)
        with self._cuda.stream(self.stream):
            engine.batch_begin(self.kv, self.slots)
        self.thread = threading.Thread(target=self._loop, name="b2-batcher", daemon=True)
        self.thread.start()

    # ---- consumer side -------------------------------------------------------------------------------------
    def submit(self, embeds, length, sampling=None, max_new_tokens=20, proc=None):
        """embeds: bf16 [1, S, hidden] on the device (already spliced by the caller's thread); proc: the request's LogitsProc
        (its prompt ids produced on the caller's stream, like embeds) or None; returns a Request."""
        if self.closed:
            raise RuntimeError("batcher is closed")
        if length + max_new_tokens > self.max_seq:
            raise ValueError(f"sequence {length} + {max_new_tokens} new tokens exceeds the batcher's cache ({self.max_seq})")
        ready = self._cuda.Event()
        ready.record()                          # the caller's stream produced `embeds`: the scheduler's stream waits for it
        req = Request(embeds, length, sampling or make_sampling(), max_new_tokens, proc)
        req.ready = ready
        self.pending.put(req)
        self.wake.set()
        return req

    def close(self):
        self.closed = True
        self.wake.set()
        self.thread.join(timeout=30)
        self.kv.close()

    # ---- scheduler thread ----------------------------------------------------------------------------------
    def _admit(self, req):
        eng, slot = self.engine, self.free.pop()
        req.slot = slot
        self.stream.wait_event(req.ready)
        logits = eng.prefill(self.kv, req.embeds, [req.length], LOGITS_LAST, slot0=slot)
        if req.proc is None:
            first = int(eng.sample(logits, req.sampling, index=0).cpu()[0])      # admission is a sync point anyway
            eng.check_async_error()
            eng.batch_set_row(self.kv, slot, True, req.sampling, first)
        else:  # the first token is chosen over the prompt history; the slot's history is the prompt and that token
            # the ids were made on the caller's stream and are read on this one, possibly after the caller dropped them
            req.proc.ids.record_stream(self.stream)
            first = int(eng.sample(logits, req.sampling, index=0, procs=[req.proc]).cpu()[0])
            eng.check_async_error()
            eng.batch_set_row(self.kv, slot, True, req.sampling, first, proc=req.proc)
        req.embeds = None
        self.active[slot] = req
        self.stats["admitted"] += 1
        self.stats["max_active"] = max(self.stats["max_active"], len(self.active))
        self._deliver(req, first)

    def _deliver(self, req, token):
        req.produced += 1
        req.tokens.put(token)
        if req.produced >= req.max_new_tokens:
            req.cancelled = True                 # done: retire at the next sweep

    def _retire(self, slot):
        self.engine.batch_set_row(self.kv, slot, False)
        del self.active[slot]
        self.free.append(slot)

    def _loop(self):
        eng = self.engine
        try:
            with self._cuda.stream(self.stream), torch.no_grad():
                while not self.closed:
                    for slot in [s for s, r in self.active.items() if r.cancelled]:
                        self._retire(slot)
                    while self.free and not self.pending.empty():
                        req = self.pending.get_nowait()
                        if req.cancelled:
                            continue
                        try:
                            self._admit(req)
                        except BaseException as e:   # a bad request must not take the batch down
                            if req.slot is not None and req.slot not in self.active:
                                self.free.append(req.slot)
                            req.tokens.put(e)
                    if not self.active:
                        self.wake.wait(timeout=0.05)
                        self.wake.clear()
                        continue
                    eng.stream_enqueue(self.kv, 1)
                    toks = eng.stream_wait(self.kv, self.step, self.slots)
                    self.step += 1
                    self.stats["steps"] += 1
                    self.stats["rows_stepped"] += len(self.active)
                    for slot, req in list(self.active.items()):
                        if not req.cancelled:
                            self._deliver(req, int(toks[slot]))
        except BaseException as e:
            for req in list(self.active.values()):
                req.tokens.put(e)
            while not self.pending.empty():
                self.pending.get_nowait().tokens.put(e)
            self.closed = True
