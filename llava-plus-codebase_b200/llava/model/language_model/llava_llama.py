"""LlavaLlamaForCausalLM on the H100 engine.

Same public surface as the reference's llava/model/language_model/llava_llama.py (LlavaConfig :29-30,
LlavaLlamaModel :33-38, LlavaLlamaForCausalLM.forward :56-99, prepare_inputs_for_generation :101-108) and
the same state-dict key layout (SURVEY.md §5), so `load_pretrained_model`, `llava.serve.model_worker`,
`llava.serve.cli` and the eval scripts can drive it unchanged. The modules here only HOLD checkpoint tensors;
all arithmetic of the path (CLIP ViT, projector, splice, LLaMA prefill + KV-cache decode, lm_head, greedy
argmax) runs in libb2llava.so through the C ABI in include/b2llava.h. There is no PyTorch fallback: without
the CUDA library / an sm_90 device every compute entry point raises.

Compute dtype is bf16 (north-star). Callers that ask for fp16 (`.half()`, torch_dtype=float16 in the
reference's builder.py:43) keep their tensor dtypes at the boundary, the engine computes in bf16.
"""
import json
import os
import threading
import weakref
from typing import List, Optional, Tuple, Union

import numpy as np
import torch
import torch.nn as nn
from transformers import AutoConfig, LlamaConfig
from transformers.modeling_outputs import CausalLMOutputWithPast

from ..llava_arch import LlavaMetaModel, LlavaMetaForCausalLM
from ..multimodal_encoder.clip_encoder import _Holder, _read_checkpoint_dir
from ..._b2 import (Engine, KVCache, LOGITS_ALL, LOGITS_LAST, ERR_SPLICE_SLOTS, INT32_MIN, kv_dtype_code, last_error, make_logits_proc,
                     make_prompt_lookup,
                    make_sampling, make_beam_sampling)
from ..._b2 import prefix as _prefix
from ..._b2.fork import ForkPlan
from ...constants import IMAGE_TOKEN_INDEX
from ..llava_arch import build_source_index


class LlavaConfig(LlamaConfig):
    model_type = "llava"


class _KVPool:
    """KV caches of one engine. Every generate() works on a cache of its own for its whole duration — the reference's
    model_worker runs up to `limit_model_concurrency` generate() threads on one model object
    (llava/serve/model_worker.py:174-185, :230-243), and a shared cache would let request B's prefill overwrite request
    A's context mid-decode. Caches are created on demand (up to `cap`, then acquire() blocks) and reused."""

    def __init__(self, engine, max_batch, max_seq, cap, dtype="bf16"):
        self.engine, self.max_batch, self.max_seq, self.cap, self.dtype = engine, max_batch, max_seq, max(1, int(cap)), dtype
        self._cond = threading.Condition()
        self._free, self._made = [], 0
        self._records = {}   # id(free cache) -> (record of its rows, event recorded at release); prefix reuse only
        # conversation prefix reuse (generate() with config.b2_prefix_cache): spliced rows taken over from a released cache,
        # and images whose encode_images was skipped because they lay inside those rows
        self.reused_positions = 0
        self.skipped_encodes = 0

    def acquire(self):
        with self._cond:
            while not self._free and self._made >= self.cap:
                self._cond.wait()
            if self._free:
                return self._free.pop()
            self._made += 1
        try:
            return _new_kv(self.engine, self.max_batch, self.max_seq, self.dtype)
        except Exception:
            with self._cond:
                self._made -= 1
                self._cond.notify()
            raise

    def acquire_prefix(self, items, rows_per_image):
        """acquire() for a prompt whose spliced items are `items` (llava/_b2/prefix.py): the free cache holding the longest
        reusable prefix of it, else a new cache while fewer than `cap` exist, else the least recently released one.
        Returns (kv, rows to reuse, event recorded when the cache was released)."""
        with self._cond:
            while True:
                if self._free:
                    recs = [self._records.get(id(kv), (None, None))[0] for kv in self._free]
                    i, m = _prefix.select(recs, items, rows_per_image)
                    if m > 0 or self._made >= self.cap:
                        kv = self._free.pop(i)
                        ev = self._records.pop(id(kv), (None, None))[1]
                        return kv, m, (ev if m > 0 else None)
                if self._made < self.cap:
                    self._made += 1
                    break
                self._cond.wait()
        try:
            kv = _new_kv(self.engine, self.max_batch, self.max_seq, self.dtype)
        except Exception:
            with self._cond:
                self._made -= 1
                self._cond.notify()
            raise
        return kv, 0, None

    def count_reuse(self, rows, images):
        with self._cond:
            self.reused_positions += int(rows)
            self.skipped_encodes += int(images)

    def release(self, kv, record=None):
        """`record`: what the cache's rows hold (prefix.record_after_generation), or None. An event on the releasing stream
        orders the next user's prefill after the decode steps this call still has queued (they write rows past the record)."""
        ev = None
        if record is not None:
            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream(self.engine.device))
        with self._cond:
            if record is not None:
                self._records[id(kv)] = (record, ev)
            else:
                self._records.pop(id(kv), None)
            self._free.append(kv)
            self._cond.notify()


def _new_kv(engine, max_batch, max_seq, dtype):
    return engine.new_kv(max_batch, max_seq) if dtype == "bf16" else engine.new_kv(max_batch, max_seq, dtype=dtype)


class PastKeyValues:
    """What forward(use_cache=True) returns as `past_key_values`: a lease on one of the model's forward caches. A later
    forward() may recycle the underlying cache (`config.b2_forward_caches` of them exist, default 2); using a recycled
    lease raises instead of silently decoding against somebody else's context."""

    def __init__(self, kv, serial):
        self.kv, self.serial = kv, serial

    @property
    def valid(self):
        return getattr(self.kv, "_lease_serial", None) == self.serial

    def get_seq_length(self, layer_idx=0):
        return self.kv.get_seq_length()


def _empty_param(*shape, dtype=None, device=None):
    return nn.Parameter(torch.empty(*shape, dtype=dtype, device=device), requires_grad=False)


class _Weight(nn.Module):
    """`<name>.weight` holder (Linear without bias / RMSNorm / Embedding), never initialised on construction."""

    def __init__(self, *shape, dtype=None, device=None):
        super().__init__()
        self.weight = _empty_param(*shape, dtype=dtype, device=device)


class _DecoderWeights(nn.Module):
    """State-dict layout of transformers LlamaModel: embed_tokens, layers.N.{self_attn,mlp,*_layernorm}, norm."""

    def __init__(self, config):
        super().__init__()
        self.config = config
        h, I, V = config.hidden_size, config.intermediate_size, config.vocab_size
        dt = getattr(config, "_b2_param_dtype", torch.bfloat16)
        dev = getattr(config, "_b2_param_device", None)
        self.embed_tokens = _Weight(V, h, dtype=dt, device=dev)
        layers = []
        for _ in range(config.num_hidden_layers):
            L = _Holder()
            L.self_attn = _Holder()
            for n in ("q_proj", "k_proj", "v_proj", "o_proj"):
                setattr(L.self_attn, n, _Weight(h, h, dtype=dt, device=dev))
            L.mlp = _Holder()
            L.mlp.gate_proj = _Weight(I, h, dtype=dt, device=dev)
            L.mlp.up_proj = _Weight(I, h, dtype=dt, device=dev)
            L.mlp.down_proj = _Weight(h, I, dtype=dt, device=dev)
            L.input_layernorm = _Weight(h, dtype=dt, device=dev)
            L.post_attention_layernorm = _Weight(h, dtype=dt, device=dev)
            layers.append(L)
        self.layers = nn.ModuleList(layers)
        self.norm = _Weight(h, dtype=dt, device=dev)


class LlavaLlamaModel(LlavaMetaModel, _DecoderWeights):
    config_class = LlavaConfig

    def __init__(self, config):
        super(LlavaLlamaModel, self).__init__(config)


class LlavaLlamaForCausalLM(nn.Module, LlavaMetaForCausalLM):
    config_class = LlavaConfig

    def __init__(self, config, device=None, dtype=torch.bfloat16, max_batch=None, max_seq=None, max_images=None):
        nn.Module.__init__(self)
        if getattr(config, "num_key_value_heads", config.num_attention_heads) != config.num_attention_heads:
            raise NotImplementedError("grouped-query attention is not part of the LLaVA-1.5 path (kv_heads == heads)")
        if getattr(config, "pretraining_tp", 1) != 1:
            raise NotImplementedError("pretraining_tp != 1")
        self.config = config
        config._b2_param_dtype, config._b2_param_device = dtype, device
        try:
            self.model = LlavaLlamaModel(config)
        finally:
            del config._b2_param_dtype, config._b2_param_device
        self.vocab_size = config.vocab_size
        self.lm_head = _Weight(config.vocab_size, config.hidden_size, dtype=dtype, device=device)
        self._engine = None
        self._batcher = None       # config.b2_continuous_batching = N: concurrent generate() calls share batched decode steps
        self._pool = None          # generate(): one exclusive cache per call
        self._fwd_kvs = []         # forward(use_cache=True): small LRU ring of leased caches
        self._fwd_lock = threading.Lock()
        self._engine_lock = threading.RLock()
        self._limits = {"max_batch": max_batch, "max_seq": max_seq, "max_images": max_images}
        self._attach()

    # ------------------------------------------------------------------ plumbing
    def _attach(self):
        ref = weakref.ref(self)
        self.model._owner = ref
        if getattr(self.model, "mm_projector", None) is not None:
            self.model.mm_projector._owner = ref
        vt = self.model.get_vision_tower()
        if vt is not None:
            vt._owner = ref

    def get_model(self):
        return self.model

    def get_input_embeddings(self):
        return self.model.embed_tokens

    def get_output_embeddings(self):
        return self.lm_head

    @property
    def device(self):
        return self.lm_head.weight.device

    @property
    def dtype(self):
        return self.lm_head.weight.dtype

    def invalidate_engine(self):
        """Weights changed (load_state_dict, resize, tower load): rebuild the device engine lazily."""
        with self._engine_lock:
            if self._batcher is not None:
                self._batcher.close()
                self._batcher = None
            self._pool = None
            self._fwd_kvs = []
            if self._engine is not None:
                self._engine.close()
            self._engine = None

    def load_state_dict(self, state_dict, strict=True, assign=False):
        r = super().load_state_dict(state_dict, strict=strict, assign=assign)
        self.invalidate_engine()
        return r

    def _apply(self, fn, *a, **k):
        r = super()._apply(fn, *a, **k)
        self.invalidate_engine()
        return r

    def resize_token_embeddings(self, new_num_tokens=None):
        old = self.model.embed_tokens.weight
        if new_num_tokens is None or new_num_tokens == old.shape[0]:
            return self.model.embed_tokens
        for mod in (self.model.embed_tokens, self.lm_head):
            w = mod.weight.data
            nw = torch.zeros(new_num_tokens, w.shape[1], dtype=w.dtype, device=w.device)
            n = min(new_num_tokens, w.shape[0])
            nw[:n] = w[:n]
            if new_num_tokens > n:
                nw[n:].normal_(mean=0.0, std=getattr(self.config, "initializer_range", 0.02))
            mod.weight = nn.Parameter(nw, requires_grad=False)
        self.config.vocab_size = self.vocab_size = new_num_tokens
        self.invalidate_engine()
        return self.model.embed_tokens

    def engine_limits(self, max_batch=None, max_seq=None, max_images=None):
        """Workspace sizing of the device engine (KV cache + activations); call before the first forward."""
        for k, v in (("max_batch", max_batch), ("max_seq", max_seq), ("max_images", max_images)):
            if v is not None and v != self._limits[k]:
                self._limits[k] = v
                self.invalidate_engine()

    def _ensure_engine(self) -> Engine:
        eng = self._engine
        if eng is not None:
            return eng
        with self._engine_lock:
            return self._build_engine()

    def _build_engine(self) -> Engine:
        if self._engine is not None:
            return self._engine
        vt = self.get_vision_tower()
        if vt is None or not vt.is_loaded:
            raise RuntimeError("vision tower is not loaded: call model.get_vision_tower().load_model() first")
        if self.device.type != "cuda":
            raise RuntimeError("LlavaLlamaForCausalLM weights must be on a CUDA (sm_90a) device: model.to('cuda'); "
                               "there is no CPU path")
        c, vc = self.config, vt.config
        # KV cache format of every cache this model creates: config.b2_kv_dtype or B2_KV_DTYPE ("bf16" default, "e4m3": half the
        # cache bytes, decode numerics change — include/b2llava.h, b2_kv_create_ex); checked before anything is allocated
        self._kv_dtype = getattr(c, "b2_kv_dtype", None) or os.environ.get("B2_KV_DTYPE") or "bf16"
        kv_dtype_code(self._kv_dtype)
        weight_format = _check_weight_format(c)
        max_seq = self._limits["max_seq"] or min(getattr(c, "max_position_embeddings", 4096), 4096)
        desc = dict(
            image_size=vc.image_size, patch_size=vc.patch_size, vit_hidden=vc.hidden_size,
            vit_inter=vc.intermediate_size, vit_layers=vc.num_hidden_layers, vit_heads=vc.num_attention_heads,
            vit_select_layer=vt.select_layer, vit_ln_eps=vc.layer_norm_eps,
            hidden=c.hidden_size, inter=c.intermediate_size, layers=c.num_hidden_layers,
            heads=c.num_attention_heads, vocab=self.lm_head.weight.shape[0], rms_eps=c.rms_norm_eps,
            rope_theta=float(getattr(c, "rope_theta", None) or (getattr(c, "rope_parameters", None) or {}).get("rope_theta", 10000.0)),
            max_batch=max(self._limits["max_batch"] or 1, int(getattr(c, "b2_continuous_batching", 0) or 0), self._beam_search_cap()),
            max_seq=max_seq, max_images=self._limits["max_images"] or 8,
        )
        if getattr(vc, "hidden_act", "quick_gelu") != "quick_gelu":
            raise NotImplementedError("CLIP tower activation must be quick_gelu (openai/clip-vit-large-patch14-336)")
        eng = Engine(desc, self.device)
        torch.cuda.current_stream(self.device).synchronize()  # set_weight copies on the library's stream: order it after
        for k, v in self.state_dict().items():                # whatever produced the parameters on the caller's stream
            if "position_ids" in k or "inv_freq" in k:
                continue
            eng.set_weight(k, v.to(self.device))
        eng.finalize()
        if weight_format == "nf4":  # load_4bit: before any KV cache exists
            eng.enable_nf4()
        # BASELINE configs[4] opt-in: e4m3 decoder weights for batch >= 7 decode (config.b2_fp8_decode or B2_FP8_DECODE=1)
        if getattr(c, "b2_fp8_decode", False) or os.environ.get("B2_FP8_DECODE") == "1":
            eng.enable_fp8_decode()
        self._pool = _KVPool(eng, desc["max_batch"], desc["max_seq"],
                             getattr(c, "b2_max_concurrent_generations", None) or int(os.environ.get("B2_MAX_GENERATIONS", "8")),
                             dtype=self._kv_dtype)
        self._fwd_kvs = []
        self._engine = eng
        return eng

    def _get_batcher(self, eng):
        slots = int(getattr(self.config, "b2_continuous_batching", 0) or 0)
        if slots < 2:
            return None
        with self._engine_lock:
            if self._batcher is None:
                from ..._b2.batching import ContinuousBatcher
                self._batcher = ContinuousBatcher(eng, slots, eng.desc.max_seq, kv_dtype=self._kv_dtype)
            return self._batcher

    def _check_limits(self, eng, B, need_seq):
        lim_b, lim_s = eng.desc.max_batch, eng.desc.max_seq
        if B > lim_b or need_seq > lim_s:
            raise ValueError(f"batch {B} / sequence {need_seq} exceed the engine limits (max_batch={lim_b}, max_seq={lim_s}); "
                             f"call model.engine_limits(max_batch=..., max_seq=...) before the first forward")

    def _lease_forward_kv(self, eng, B, need_seq):
        """Cache for one forward(use_cache=True): least recently leased of a small ring; earlier leases of it go stale."""
        self._check_limits(eng, B, need_seq)
        with self._fwd_lock:
            cap = max(1, int(getattr(self.config, "b2_forward_caches", 2)))
            if len(self._fwd_kvs) < cap:
                kv = _new_kv(eng, eng.desc.max_batch, eng.desc.max_seq, self._kv_dtype)
                kv._lease_serial = 0
            else:
                kv = self._fwd_kvs.pop(0)
            kv._lease_serial += 1
            self._fwd_kvs.append(kv)
            return PastKeyValues(kv, kv._lease_serial)

    # ------------------------------------------------------------------ forward (ref llava_llama.py:56-99)
    def forward(
        self,
        input_ids: torch.LongTensor = None,
        attention_mask: Optional[torch.Tensor] = None,
        position_ids: Optional[torch.LongTensor] = None,
        past_key_values=None,
        inputs_embeds: Optional[torch.FloatTensor] = None,
        labels: Optional[torch.LongTensor] = None,
        use_cache: Optional[bool] = None,
        output_attentions: Optional[bool] = None,
        output_hidden_states: Optional[bool] = None,
        images: Optional[torch.FloatTensor] = None,
        return_dict: Optional[bool] = None,
    ) -> Union[Tuple, CausalLMOutputWithPast]:
        if output_attentions or output_hidden_states:
            raise NotImplementedError("attention maps / hidden states are never materialised on the fused path")
        engine = self._ensure_engine()

        # ---- decode step: [B,1] ids against an engine cache ----
        if inputs_embeds is None and past_key_values is not None and input_ids is not None and input_ids.shape[1] == 1:
            kv = self._resolve_cache(past_key_values)
            logits = engine.decode_step(kv, input_ids.reshape(-1))
            logits = logits.unsqueeze(1)
            return self._output(logits, past_key_values, labels, return_dict)

        if past_key_values is not None:
            return self._forward_continue(engine, input_ids, inputs_embeds, attention_mask, past_key_values, images, labels,
                                          return_dict)

        if inputs_embeds is None:
            (input_ids, position_ids, attention_mask, past_key_values, inputs_embeds, labels) = \
                self.prepare_inputs_labels_for_multimodal(input_ids, position_ids, attention_mask, past_key_values, labels, images)
            if inputs_embeds is None:  # text-only (no images / no tower): plain embedding lookup on the engine
                ids = input_ids.to(torch.int32).reshape(-1).to(engine.device)
                inputs_embeds = engine.splice(ids, None, input_ids.shape[0], input_ids.shape[1])

        B, S = inputs_embeds.shape[0], inputs_embeds.shape[1]
        lens, left = None, False
        if attention_mask is not None:
            m = attention_mask.to(device=inputs_embeds.device).bool()
            lens = m.sum(dim=1).tolist()
            left = bool((~m[:, 0]).any()) and bool(m[:, -1].all())
            if left:  # engine rows are right-padded: rotate valid tokens to the front (ref pads left only on request)
                inputs_embeds = torch.stack([torch.roll(inputs_embeds[b], shifts=-(S - lens[b]), dims=0) for b in range(B)])
        lease = self._lease_forward_kv(engine, B, S)
        lease.kv.reset()
        logits = engine.prefill(lease.kv, inputs_embeds, lens, LOGITS_ALL)
        if left:
            logits = torch.stack([torch.roll(logits[b], shifts=(S - lens[b]), dims=0) for b in range(B)])
        return self._output(logits, lease if use_cache is not False else None, labels, return_dict)

    def _forward_continue(self, engine, input_ids, inputs_embeds, attention_mask, past_key_values, images, labels, return_dict):
        """HF continuation: the [B, n] chunk is appended to each row's own cache length (b2_prefill_at); image placeholders
        in the chunk are spliced like a prompt's. Returns logits [B, n', V] (n' = spliced chunk length) and the same cache."""
        kv = self._resolve_cache(past_key_values)
        if attention_mask is not None and not bool(attention_mask.bool().all()):
            raise NotImplementedError("a padded attention_mask on a chunk appended to a cache is not supported")
        lens = None
        if inputs_embeds is None:
            embeds, lens = self._prepare_multimodal(input_ids, None, None, None, None, images)
            inputs_embeds = embeds[4]
            if inputs_embeds is None:  # text-only chunk: plain embedding lookup on the engine
                ids = input_ids.to(torch.int32).reshape(-1).to(engine.device)
                inputs_embeds = engine.splice(ids, None, input_ids.shape[0], input_ids.shape[1])
                lens = None
        B, S = inputs_embeds.shape[0], inputs_embeds.shape[1]
        start = kv.lengths(B)
        self._check_limits(engine, B, max(start[b] + (S if lens is None else lens[b]) for b in range(B)))
        logits = engine.prefill(kv, inputs_embeds, lens, LOGITS_ALL, start=start)
        return self._output(logits, past_key_values, labels, return_dict)

    @staticmethod
    def _resolve_cache(past_key_values):
        if isinstance(past_key_values, PastKeyValues):
            if not past_key_values.valid:
                raise RuntimeError("this past_key_values was recycled by a later forward(use_cache=True): the model keeps "
                                   "config.b2_forward_caches (default 2) forward caches alive at a time")
            return past_key_values.kv
        if isinstance(past_key_values, KVCache):
            return past_key_values
        raise ValueError("past_key_values must be the cache object returned by a previous forward of this model")

    def _output(self, logits, kv, labels, return_dict):
        loss = None
        if labels is not None:  # HF LlamaForCausalLM loss: shift by one, ignore_index=-100
            sl = logits[..., :-1, :].contiguous().float()
            tl = labels[..., 1:].contiguous().to(sl.device)
            loss = nn.functional.cross_entropy(sl.view(-1, sl.size(-1)), tl.view(-1), ignore_index=-100)
        if return_dict is False:
            out = (logits, kv)
            return ((loss,) + out) if loss is not None else out
        return CausalLMOutputWithPast(loss=loss, logits=logits, past_key_values=kv)

    def prepare_inputs_for_generation(self, input_ids, past_key_values=None, inputs_embeds=None, **kwargs):
        """ref llava_llama.py:101-108 (kept for API parity; generate() below does not need it)."""
        images = kwargs.pop("images", None)
        if past_key_values is not None:
            input_ids = input_ids[:, -1:]
        model_inputs = {"input_ids": input_ids, "past_key_values": past_key_values,
                        "use_cache": kwargs.get("use_cache"), "attention_mask": kwargs.get("attention_mask")}
        if inputs_embeds is not None and past_key_values is None:
            model_inputs = {"inputs_embeds": inputs_embeds, **{k: v for k, v in model_inputs.items() if k != "input_ids"}}
        if images is not None:
            model_inputs["images"] = images
        return model_inputs

    # ------------------------------------------------------------------ generate
    # generation arguments of HF generate() that change WHAT is generated and that this loop does not implement: raise
    # instead of silently decoding something else (value = the setting that means "off")
    _UNSUPPORTED_GENERATION_ARGS = {
        "repetition_penalty": 1.0, "encoder_repetition_penalty": 1.0, "length_penalty": 1.0, "no_repeat_ngram_size": 0,
        "encoder_no_repeat_ngram_size": 0, "min_new_tokens": None, "min_length": 0, "bad_words_ids": None,
        "force_words_ids": None, "num_beam_groups": 1, "diversity_penalty": 0.0, "penalty_alpha": None, "typical_p": 1.0,
        "epsilon_cutoff": 0.0, "eta_cutoff": 0.0, "num_return_sequences": 1, "logits_processor": None,
        "prefix_allowed_tokens_fn": None, "constraints": None, "suppress_tokens": None, "begin_suppress_tokens": None,
        "forced_bos_token_id": None, "forced_eos_token_id": None, "assistant_model": None, "min_p": None,
    }
    # implemented by the device's logits processing when config.b2_logits_processors / B2_LOGITS_PROCESSORS=1 opts in
    _LOGITS_PROCESSOR_ARGS = ("repetition_penalty", "no_repeat_ngram_size", "min_new_tokens", "min_length")
    # accepted and without effect on this path
    _IGNORED_GENERATION_ARGS = {"synced_gpus", "early_stopping", "output_attentions", "output_hidden_states",
                                "generation_config", "position_ids", "past_key_values", "renormalize_logits", "max_time"}

    @torch.no_grad()
    def generate(self, inputs=None, images=None, do_sample=False, temperature=1.0, top_p=None, top_k=None,
                 num_beams=1, max_new_tokens=None, max_length=None, use_cache=True, streamer=None,
                 stopping_criteria=None, eos_token_id=None, pad_token_id=None, attention_mask=None,
                 input_ids=None, output_scores=False, return_dict_in_generate=False, output_logits=False, **kwargs):
        """Own decoding loop with the side-protocols the reference's callers rely on (SURVEY §8b): prompt ids (with
        IMAGE_TOKEN_INDEX) echoed in the result, `streamer.put/end`, `stopping_criteria` called as
        crit(ids_so_far, scores) -> bool | bool tensor, eos stop, temperature / top-k / top-p sampling.

        Every variant runs the same device-resident loop: token feedback, argmax or the sampling draw are kernels, each
        step publishes its token into pinned host memory, and this thread (usually a worker `Thread`,
        llava/serve/model_worker.py:174-185) reads token t — streamer, eos, stopping criteria — while the device is
        already `config.b2_run_ahead` (default 8) steps further. Steps queued beyond the stop point are discarded.

        With return_dict_in_generate=True the result is transformers' GenerateDecoderOnlyOutput (GenerateBeamDecoderOnlyOutput
        with num_beams > 1): `scores` (output_scores) and `logits` (output_logits) are tuples of one fp32 tensor per generated
        step on the model's device, [B, V] ([B * num_beams, V] for beams, in the running-beam order). A score row is what HF
        hands to selection: the logits after the processors, and when sampling x / T with the tokens top-k / top-p remove at
        -inf; under beam search log_softmax(logits), warped under beam sampling. The decode kernels write the rows while the
        device runs ahead, so they cost no synchronisation per token. A row of a batch that has finished keeps decoding its own
        tokens (the result shows pad there), so its scores and logits after its eos are not the ones HF, which feeds it pad
        ids, would give; every position up to and including its eos is. `past_key_values`, `attentions` and `hidden_states`
        are None. Stopping criteria still receive scores=None: handing them the live device rows would need a synchronisation
        per token. Without return_dict_in_generate the id tensor is returned and output_scores / output_logits are ignored,
        as in HF.

        num_return_sequences=n with do_sample (and num_beams=1) returns B * n rows in HF's order (the n samples of prompt b are
        rows b * n .. b * n + n - 1). Each prompt and its image are encoded and prefilled once; the prompt's cache rows are then
        copied into the slots of its other samples, and the decode attention reads each prompt once for all of its samples. Token
        0 of every sample is drawn from its prompt's prefill logits with the sample's own Philox key, so a seeded run equals HF's
        (which repeats the inputs n times) in distribution, not in ids. Processors, score rows, stopping criteria, eos / pad and
        the streamer see the B * n rows."""
        if inputs is None:
            inputs = input_ids
        if inputs is None:
            raise ValueError("generate() needs input ids")
        want = _output_arguments(return_dict_in_generate, output_scores, output_logits, kwargs)
        proc_args = self._logits_processor_arguments(kwargs)
        beam_args = {}
        if num_beams != 1:
            if proc_args and not _beam_logits_processors_on(self.config):
                raise NotImplementedError("logits processors (repetition_penalty, no_repeat_ngram_size, min_new_tokens, "
                                          "min_length) together with num_beams > 1 are not implemented on the H100 path "
                                          "without config.b2_beam_logits_processors")
            if self._beam_search_cap() < 2:
                raise NotImplementedError("beam search is not used on the LLaVA path (num_beams=1 everywhere)")
            beam_args = self._beam_arguments(num_beams, do_sample, temperature, top_p, top_k, streamer, kwargs)
        prompt = inputs if inputs.dim() == 2 else inputs.unsqueeze(0)
        n_ret = 1 if num_beams != 1 else _num_return_arguments(self.config, kwargs, prompt.shape[0], do_sample, images)
        lookup_args = self._prompt_lookup_arguments(kwargs, prompt.shape[0] * n_ret, num_beams, bool(proc_args))
        if want and (want["scores"] or want["logits"]):
            what = "output_scores / output_logits with return_dict_in_generate"
            if lookup_args:
                raise NotImplementedError(f"{what} together with the prompt-lookup path (b2_prompt_lookup) is not implemented")
            if prompt.shape[0] == 1 and num_beams == 1 and int(getattr(self.config, "b2_continuous_batching", 0) or 0) >= 2:
                raise NotImplementedError(f"{what} together with the continuous batcher (b2_continuous_batching) is not implemented")
        for k, v in kwargs.items():
            if k in self._IGNORED_GENERATION_ARGS:
                continue
            if k in self._UNSUPPORTED_GENERATION_ARGS:
                if v is None or v == self._UNSUPPORTED_GENERATION_ARGS[k]:
                    continue
                raise NotImplementedError(f"generate({k}={v!r}) is not implemented on the H100 path")
            raise NotImplementedError(f"generate() got an unsupported argument {k!r}")
        B, Lt = prompt.shape
        engine = self._ensure_engine()
        if eos_token_id is None:
            eos_token_id = getattr(self.config, "eos_token_id", None)
        eos_ids = set(eos_token_id) if isinstance(eos_token_id, (list, tuple)) else ({eos_token_id} if eos_token_id is not None else set())
        if max_new_tokens is None:
            max_new_tokens = (max_length - Lt) if max_length is not None else 20
        if max_new_tokens <= 0:
            raise ValueError("max_new_tokens must be positive")
        procs = None
        if proc_args:
            # history of row b = the prompt row as passed (placeholders and pad ids included), kept on the device
            prompt_dev = prompt.to(device=engine.device, dtype=torch.int64).contiguous()
            procs = [make_logits_proc(prompt_dev[b], proc_args["repetition_penalty"], proc_args["no_repeat_ngram_size"],
                                      max(proc_args["min_new_tokens"], proc_args["min_length"] - Lt), eos_ids)
                     for b in range(B)]
            if all(p is None for p in procs):
                procs = None
        if beam_args:
            eos_list = (list(eos_token_id) if isinstance(eos_token_id, (list, tuple))
                        else (None if eos_token_id is None else [eos_token_id]))
            return self._beam_generate(engine, prompt, images, attention_mask, num_beams, max_new_tokens, eos_list, pad_token_id,
                                       stopping_criteria, want=want, procs=procs, **beam_args)
        greedy = (not do_sample) or (temperature is not None and temperature <= 1e-5)
        if greedy:
            sampling = make_sampling()
        else:
            if top_p is not None and not (0.0 < top_p <= 1.0):
                raise ValueError(f"top_p must be in (0, 1], got {top_p}")
            # HF GenerationConfig defaults: top_k = 50, top_p = 1.0; the draw is seeded from torch's CPU generator so that
            # torch.manual_seed() makes a run repeatable
            seed = int(torch.randint(0, 2**62, (1,), dtype=torch.int64).item())
            sampling = make_sampling(True, temperature, 1.0 if top_p is None else top_p, 50 if top_k is None else top_k, seed)
        lookup = None  # prompt-lookup speculative decoding (batch 1): lookup(cache rows) -> PromptLookup, or None when K rows no longer fit
        if lookup_args and self._get_batcher(engine) is None:
            def lookup(rows):
                return self._fit_prompt_lookup(engine, prompt, rows, lookup_args, max_new_tokens, eos_ids)
        began_lookup = [False]
        prof = _StageTimer() if os.environ.get("B2_PROFILE_GENERATE") else None

        batcher = self._get_batcher(engine) if B == 1 and n_ret == 1 else None
        if batcher is not None:
            # continuous batching: this thread splices its prompt and runs its own host loop (streamer, eos, criteria); the
            # decode steps are shared with every other generate() in flight (llava/_b2/batching.py)
            from ..._b2.batching import RequestStream
            embeds = lens = None
            if images is not None and self.get_vision_tower() is not None:
                embeds, lens, speculative = self._spliced_embeds(prompt, attention_mask, images)
                if speculative:
                    torch.cuda.current_stream(engine.device).synchronize()
                    if engine.take_async_error() & ERR_SPLICE_SLOTS:
                        embeds, lens, _ = self._spliced_embeds(prompt, attention_mask, images, force_host=True)
            if embeds is None:
                embeds = engine.splice(prompt.to(torch.int32).reshape(-1).to(engine.device), None, 1, Lt)
                lens = [Lt]
            self._check_limits(engine, 1, lens[0] + max_new_tokens)
            req = batcher.submit(embeds, lens[0], sampling, max_new_tokens, proc=procs[0] if procs else None)
            if streamer is not None:
                streamer.put(prompt.cpu())
            pad = pad_token_id if pad_token_id is not None else (next(iter(eos_ids)) if eos_ids else 0)
            try:
                new_tokens = _stream_decode(RequestStream(req), None, None, sampling, 1, max_new_tokens, eos_ids, pad, prompt,
                                            streamer, stopping_criteria, begun=True)
            finally:
                req.cancel()
            if streamer is not None:
                streamer.end()
            out = torch.cat([prompt, new_tokens.to(device=prompt.device, dtype=prompt.dtype)], dim=1)
            return out if not want else _decoder_output(out, None, None)

        # num_return_sequences: the B * n rows in HF's order (repeat_interleave) for the result, the streamer and the criteria;
        # on the device prompt b is prefilled once and forked into the slots of its other samples (llava/_b2/fork.py)
        rows_out = prompt if n_ret == 1 else prompt.repeat_interleave(n_ret, dim=0)
        N = B * n_ret
        fork = None
        if n_ret > 1 and procs is not None:
            procs = [p for p in procs for _ in range(n_ret)]  # HF row order; reordered to slots once the fork is planned
        # score / logits rows of every step the generation may take, written by the device (b2_stream_set_outputs)
        rows = {k: (torch.empty(max_new_tokens, N, engine.vocab, dtype=torch.float32, device=engine.device) if want and want[k] else None)
                for k in ("scores", "logits")}
        # conversation prefix reuse (opt-in, batch 1): the part of the prompt a released cache already holds is not prefilled again
        plan = None
        if B == 1 and n_ret == 1 and self._prefix_cache_on() and (attention_mask is None or bool(attention_mask.bool().all())):
            plan = self._prefix_plan(prompt, images)
        reuse, released_ev = 0, None
        if plan is not None:
            kv, reuse, released_ev = self._pool.acquire_prefix(plan["items"], engine.num_patches)
        else:
            kv = self._pool.acquire()  # exclusive for this call (concurrent generate() threads each get their own)
        record = None
        try:
            # ---- prefill: splice + decoder, last-position logits only; token 0 is chosen on the device ----
            def prefill(force_host):
                nonlocal fork
                embeds, lens, speculative = self._prompt_embeds(engine, prompt, attention_mask, images, force_host)
                if prof: prof.mark("encode_images+splice")
                self._check_limits(engine, N, max(lens) + max_new_tokens)
                kv.reset()
                logits = engine.prefill(kv, embeds, lens, LOGITS_LAST)
                lk = lookup(lens[0]) if lookup is not None else None
                began_lookup[0] = lk is not None
                if lk is not None:
                    engine.stream_begin_lookup(kv, logits, sampling, lk)
                elif n_ret > 1:
                    fork = ForkPlan(lens, n_ret)
                    engine.kv_copy_slots(kv, *fork.copies())
                    # token 0 of every sample from its prompt's prefill row, drawn with the sample's own row key
                    logits = logits.index_select(0, torch.tensor(fork.prompt_of_slot, device=logits.device))
                    slot_procs = None
                    if procs is not None:
                        slot_procs = [None] * N
                        for r, s in enumerate(fork.slot_of_row):
                            slot_procs[s] = procs[r]
                    engine.stream_begin(kv, logits, sampling, slot_procs, rows["scores"], rows["logits"], groups=fork.groups())
                else:
                    engine.stream_begin(kv, logits, sampling, procs, rows["scores"], rows["logits"])
                engine.stream_wait(kv, 0, N)          # first sync of this call: every input check has run by now
                if prof: prof.mark("prefill + first token")
                return speculative

            if plan is not None:
                began_lookup[0] = self._prefill_reusing(engine, kv, plan, reuse, released_ev, sampling, max_new_tokens, procs, lookup,
                                                        rows)
                speculative = False
            else:
                speculative = prefill(False)
            err = engine.take_async_error()
            if speculative and (err & ERR_SPLICE_SLOTS):
                # the rows do not hold n_images / B placeholders each: the shape-only output length was wrong. Redo on the
                # host path, which reproduces the reference's behaviour for that input (extra images ignored / IndexError)
                speculative = prefill(True)
                err = engine.take_async_error()
            if err:
                raise ValueError(last_error())

            if streamer is not None:
                streamer.put(rows_out.cpu())
            pad = pad_token_id if pad_token_id is not None else (next(iter(eos_ids)) if eos_ids else 0)
            new_tokens = _stream_decode(engine, kv, None, sampling, N, max_new_tokens, eos_ids, pad, rows_out,
                                        streamer, stopping_criteria,
                                        run_ahead=int(getattr(self.config, "b2_run_ahead", 8)), begun=True,
                                        lookup_steps=_LOOKUP_STEPS_IN_FLIGHT if began_lookup[0] else 0,
                                        slot_of_row=None if fork is None else fork.slot_of_row)
            engine.check_async_error()
            if prof: prof.mark("decode")
            if plan is not None:
                items = [it if isinstance(it, int) else it.detach().clone() for it in plan["items"]]
                record = _prefix.record_after_generation(items, new_tokens[0].tolist())
        finally:
            self._pool.release(kv, record)
        if streamer is not None:
            streamer.end()
        out = torch.cat([rows_out, new_tokens.to(device=prompt.device, dtype=prompt.dtype)], dim=1)
        if prof: prof.mark("ids to caller"); prof.report()
        if not want:
            return out
        n = new_tokens.shape[1]
        if fork is not None:  # slot order -> HF row order
            order = torch.tensor(fork.slot_of_row, device=engine.device)
            rows = {k: None if v is None else v.index_select(1, order) for k, v in rows.items()}
        return _decoder_output(out, _trim_steps(rows.pop("scores"), n), _trim_steps(rows.pop("logits"), n))

    def compute_transition_scores(self, sequences, scores, beam_indices=None, normalize_logits=False):
        """transformers' GenerationMixin.compute_transition_scores: the score of each generated token from generate()'s
        `scores` (and `beam_indices` after beam search), [batch * num_return_sequences, generated length]."""
        from transformers.generation.utils import GenerationMixin

        return GenerationMixin.compute_transition_scores(self, sequences, scores, beam_indices, normalize_logits)

    def _prompt_embeds(self, engine, prompt, attention_mask, images, force_host):
        """Spliced prompt rows of generate(): (embeds [B, S, hidden], valid rows per sample, whether the device splice was
        used on the shape-only assumption that every row holds n_images / B placeholders)."""
        B, Lt = prompt.shape
        embeds, lens, speculative = None, None, False
        if images is not None and self.get_vision_tower() is not None:
            embeds, lens, speculative = self._spliced_embeds(prompt, attention_mask, images, force_host=force_host)
        if embeds is not None:
            if getattr(self.config, "tokenizer_padding_side", "right") == "left" and len(set(lens)) > 1:
                S = embeds.shape[1]
                embeds = torch.stack([torch.roll(embeds[b], shifts=-(S - lens[b]), dims=0) for b in range(B)])
        else:  # text-only prompt (or a [B,1] prompt, which the multimodal splice passes through)
            if attention_mask is not None and not bool(attention_mask.bool().all()):
                raise NotImplementedError("padded text-only batches: pass equal-length prompts")
            ids = prompt.to(torch.int32).reshape(-1).to(engine.device)
            embeds = engine.splice(ids, None, B, Lt)
            lens = [Lt] * B
        return embeds, lens, speculative

    def _logits_processors_on(self):
        """config.b2_logits_processors or B2_LOGITS_PROCESSORS=1 (off by default, like the other b2_* opt-ins)."""
        v = getattr(self.config, "b2_logits_processors", None)
        return bool(v) if v is not None else os.environ.get("B2_LOGITS_PROCESSORS") == "1"

    def _logits_processor_arguments(self, kwargs):
        """With the opt-in, takes repetition_penalty / no_repeat_ngram_size / min_new_tokens / min_length out of `kwargs` and
        returns them with their off values filled in, or {} when every one is off. Without it they stay in `kwargs`, where
        any value other than the off value raises NotImplementedError."""
        if not self._logits_processors_on():
            return {}
        got = {k: kwargs.pop(k) for k in self._LOGITS_PROCESSOR_ARGS if k in kwargs}
        p = got.get("repetition_penalty")
        p = 1.0 if p is None else float(p)
        if not p > 0.0:
            raise ValueError(f"repetition_penalty has to be a strictly positive float, but is {p}")
        n = got.get("no_repeat_ngram_size")
        n = 0 if n is None else int(n)
        if n < 0:
            raise ValueError(f"no_repeat_ngram_size has to be a non-negative integer, but is {n}")
        mnt = int(got.get("min_new_tokens") or 0)
        ml = int(got.get("min_length") or 0)
        if p == 1.0 and n == 0 and mnt <= 0 and ml <= 0:
            return {}
        return {"repetition_penalty": p, "no_repeat_ngram_size": n, "min_new_tokens": mnt, "min_length": ml}

    # ------------------------------------------------------------------ prompt-lookup speculative decoding
    def _prompt_lookup_cap(self):
        """config.b2_prompt_lookup or B2_PROMPT_LOOKUP: K, the most draft tokens per verify step (0 = off). It caps
        prompt_lookup_num_tokens, and batch-1 calls that do not pass it draft K tokens."""
        v = getattr(self.config, "b2_prompt_lookup", None)
        if v is None:
            v = os.environ.get("B2_PROMPT_LOOKUP")
        try:
            k = int(v or 0)
        except (TypeError, ValueError):
            raise ValueError(f"b2_prompt_lookup must be an integer, got {v!r}")
        if not 0 <= k <= 15:
            raise ValueError(f"b2_prompt_lookup must be in 0..15, got {k}")
        return k

    def _fit_prompt_lookup(self, engine, prompt, rows, lookup_args, max_new_tokens, eos_ids):
        """The PromptLookup of a batch-1 generation whose prompt fills `rows` cache rows. A verify step writes K rows past the
        last token, so K is capped at what the cache leaves free; with no room (or more eos ids than the device keeps) the
        call decodes without speculation, as it would without the opt-in."""
        Lt = prompt.shape[1]
        room = self._pool.max_seq - max(rows, Lt) - max_new_tokens
        k = min(lookup_args["num_tokens"], room)
        if getattr(self.config, "b2_fp8_decode", False) or os.environ.get("B2_FP8_DECODE") == "1":
            k = min(k, engine.desc.max_batch - 1)  # the e4m3 activation buffer holds max_batch rows
        if k < 1 or len(set(eos_ids)) > 8:
            return None
        prompt_dev = prompt.to(device=engine.device, dtype=torch.int64).contiguous()
        return make_prompt_lookup(prompt_dev[0], k, lookup_args["max_ngram"], max_new_tokens, eos_ids)

    def _prompt_lookup_arguments(self, kwargs, B, num_beams, has_procs):
        """With the opt-in, takes prompt_lookup_num_tokens / max_matching_ngram_size out of `kwargs` and returns
        {"num_tokens", "max_ngram"} when this call decodes with prompt lookup, else {}. Without it they stay in `kwargs` and raise
        as any unsupported argument does."""
        K = self._prompt_lookup_cap()
        if K == 0:
            return {}
        k = kwargs.pop("prompt_lookup_num_tokens", None)
        n = kwargs.pop("max_matching_ngram_size", None)
        explicit = k is not None
        if explicit:
            k = int(k)
            if k <= 0:
                raise ValueError("Invalid max_matching_ngram_size or num_output_tokens")
            if B != 1:
                raise ValueError("assisted generate is only supported for batch_size = 1")
            blocker = ("the continuous batcher (b2_continuous_batching)" if int(getattr(self.config, "b2_continuous_batching", 0) or 0)
                       else "num_beams > 1" if num_beams != 1 else "logits processors" if has_procs
                       else "an e4m3 KV cache" if (getattr(self.config, "b2_kv_dtype", None) or os.environ.get("B2_KV_DTYPE") or "bf16") != "bf16"
                       else None)
            if blocker is not None:
                raise NotImplementedError(f"prompt_lookup_num_tokens together with {blocker} is not implemented on the H100 path")
        elif (B != 1 or num_beams != 1 or has_procs
              or (getattr(self.config, "b2_kv_dtype", None) or os.environ.get("B2_KV_DTYPE") or "bf16") != "bf16"):
            return {}
        n = 2 if n is None else int(n)
        if n <= 0:
            raise ValueError("Invalid max_matching_ngram_size or num_output_tokens")
        return {"num_tokens": min(k, K) if explicit else K, "max_ngram": n}

    # ------------------------------------------------------------------ beam search
    def _beam_search_cap(self):
        """config.b2_beam_search or B2_BEAM_SEARCH: the largest num_beams generate() accepts (beam search is off below 2). It
        also sizes the engine's caches, like b2_continuous_batching."""
        v = getattr(self.config, "b2_beam_search", None)
        if v is None:
            v = os.environ.get("B2_BEAM_SEARCH")
        try:
            return int(v or 0)
        except (TypeError, ValueError):
            raise ValueError(f"b2_beam_search must be an integer, got {v!r}")

    def _beam_sample_on(self):
        """config.b2_beam_sample or B2_BEAM_SAMPLE=1: generate(do_sample=True, num_beams > 1) runs beam sampling (off by default:
        its draws come from the engine's Philox stream, so a seeded run equals transformers' in distribution, not in ids)."""
        v = getattr(self.config, "b2_beam_sample", None)
        return bool(v) if v is not None else os.environ.get("B2_BEAM_SAMPLE") == "1"

    def _beam_arguments(self, num_beams, do_sample, temperature, top_p, top_k, streamer, kwargs):
        """Checks what generate(num_beams > 1) does not implement and takes the beam-only arguments out of `kwargs`. With
        do_sample (and a temperature above 1e-5, below which it is beam search) the result carries `sampling`: the warpers of
        beam sampling, HF GenerationConfig's defaults top_k = 50 and top_p = 1.0 filled in."""
        if num_beams < 1 or num_beams > self._beam_search_cap():
            raise ValueError(f"num_beams={num_beams} exceeds config.b2_beam_search={self._beam_search_cap()}")
        sampled = bool(do_sample) and not (temperature is not None and temperature <= 1e-5)
        if sampled and not self._beam_sample_on():
            raise NotImplementedError("beam sampling (do_sample=True with num_beams > 1) is not implemented on the H100 path "
                                      "without config.b2_beam_sample")
        if (kwargs.get("num_beam_groups") or 1) != 1 or (kwargs.get("diversity_penalty") or 0.0) != 0.0:
            raise NotImplementedError("group beam search (num_beam_groups / diversity_penalty) is not implemented on the H100 path")
        if kwargs.get("constraints") is not None:
            raise NotImplementedError("constrained beam search (constraints) is not implemented on the H100 path")
        if streamer is not None:
            raise ValueError("`streamer` cannot be used with beam search (num_beams > 1)")
        sampling = None
        if sampled:
            if top_p is not None and not (0.0 < top_p <= 1.0):
                raise ValueError(f"top_p must be in (0, 1], got {top_p}")
            if top_k is not None and int(top_k) < 0:
                raise ValueError(f"top_k must be a non-negative integer, got {top_k}")
            sampling = dict(temperature=1.0 if temperature is None else float(temperature), top_k=50 if top_k is None else int(top_k),
                            top_p=1.0 if top_p is None else float(top_p))
        lp = kwargs.pop("length_penalty", None)
        es = kwargs.pop("early_stopping", None)
        nrs = kwargs.pop("num_return_sequences", None)
        return dict(length_penalty=1.0 if lp is None else float(lp), early_stopping=False if es is None else es,
                    num_return_sequences=1 if nrs is None else int(nrs), sampling=sampling)

    def _beam_generate(self, engine, prompt, images, attention_mask, num_beams, max_new_tokens, eos_ids, pad_token_id,
                       stopping_criteria, length_penalty, early_stopping, num_return_sequences, sampling=None, want=None, procs=None):
        """Beam search (llava/_b2/beam.py): sample b is prefilled once into slot b of a pool cache; its candidates from the
        prefill logits fork the prompt into nb slots; then every b2_beam_step applies the step's slot copies, decodes the
        B * nb running beams in one batch and returns the K best candidates per sample for the host bookkeeping.

        With `sampling` (beam sampling) the device draws the K candidates of step t with b2_op_beam_sample / b2_beam_step_ex at
        draw index t, seeded from torch's CPU generator. The first draw reads all nb beam rows of a sample, each mapped to its
        prefill row, with running scores [0, -1e9, ...] as HF's first step does: the -1e9 rows matter to which candidates fill
        the list when fewer than K have positive probability.

        `want` (generate()'s _output_arguments): the device also writes each step's score and raw logits rows, [B * nb, V] in
        running-beam order, and the result is a GenerateBeamDecoderOnlyOutput.

        `procs` (config.b2_beam_logits_processors): one LogitsProc (or None) per sample. Each running beam's log-probabilities are
        processed against its own sequence, as HF's _beam_search does: the first candidates come from the prefill row processed
        over the prompt (b2_op_beam_select_proc), then b2_beam_begin_proc gives slot b sample b's processors and prompt history,
        and every b2_beam_step_proc carries the histories along the slot copies and appends each step's tokens. The host
        bookkeeping is unchanged: the candidates' scores are already the processed accumulated scores, and the score rows the
        processed (warped) rows."""
        from ..._b2 import beam as _beam

        B = prompt.shape[0]
        nb = num_beams
        search = _beam.BeamSearch(prompt, nb, max_new_tokens, eos_ids, length_penalty, early_stopping, num_return_sequences,
                                  pad_token_id, stopping_criteria)
        if engine.vocab < search.K:
            raise ValueError(f"beam search keeps {search.K} candidates per step, more than the vocabulary ({engine.vocab})")
        bs = None
        if sampling is not None:
            # HF _get_logits_processor: min_tokens_to_keep = 1 + number of eos ids, 2 when there are none
            min_keep = 2 if eos_ids is None else 1 + len(eos_ids)
            seed = int(torch.randint(0, 2**62, (1,), dtype=torch.int64).item())
            bs = make_beam_sampling(sampling["temperature"], sampling["top_k"], sampling["top_p"], min_keep, seed)
        self._check_limits(engine, B * nb, 1)
        rows = {k: (torch.empty(max_new_tokens, B * nb, engine.vocab, dtype=torch.float32, device=engine.device)
                    if want and want[k] else None) for k in ("scores", "logits")}
        at = lambda k, t: None if rows[k] is None else rows[k][t]  # noqa: E731  (step t's [B * nb, V] rows)
        kv = self._pool.acquire()  # exclusive for this call; never recorded for prefix reuse
        try:
            def first_candidates(force_host):
                embeds, lens, speculative = self._prompt_embeds(engine, prompt, attention_mask, images, force_host)
                self._check_limits(engine, B * nb, max(lens) + max_new_tokens)
                kv.reset()
                logits = engine.prefill(kv, embeds, lens, LOGITS_LAST)
                if procs is not None:  # processed over each sample's prompt; a sample's prefill row feeds all of its beams
                    if bs is None:
                        cand = engine.beam_select_proc(logits, torch.zeros(B), 1, search.K, procs, at("scores", 0), at("logits", 0),
                                                       fan=nb)
                    else:
                        cand = engine.beam_select_proc(logits, search.running_scores.reshape(-1), nb, search.K, procs, at("scores", 0),
                                                       at("logits", 0), sampling=bs, step=0,
                                                       row_of_beam=[b for b in range(B) for _ in range(nb)])
                    cand = [t.cpu() for t in cand]
                    if bs is not None:
                        cand[2].zero_()
                elif want:  # the same selection, also writing step 0's rows (the one prefill row of a sample fills its nb rows)
                    if bs is None:
                        cand = engine.beam_select_out(logits, torch.zeros(B), 1, search.K, at("scores", 0), at("logits", 0), fan=nb)
                    else:
                        cand = engine.beam_select_out(logits, search.running_scores.reshape(-1), nb, search.K, at("scores", 0),
                                                      at("logits", 0), sampling=bs, step=0,
                                                      row_of_beam=[b for b in range(B) for _ in range(nb)])
                    cand = [t.cpu() for t in cand]
                    if bs is not None:
                        cand[2].zero_()
                elif bs is None:
                    cand = [t.cpu() for t in engine.beam_topk(logits, torch.zeros(B), 1, search.K)]  # synchronises
                else:
                    cand = [t.cpu() for t in engine.beam_sample(logits, search.running_scores.reshape(-1), nb, search.K, bs, 0,
                                                                row_of_beam=[b for b in range(B) for _ in range(nb)])]
                    cand[2].zero_()  # every beam still holds the bare prompt, which only slot b has: all descend from beam 0
                return cand, lens, speculative

            cand, lens, speculative = first_candidates(False)
            err = engine.take_async_error()
            if speculative and (err & ERR_SPLICE_SLOTS):
                cand, lens, _ = first_candidates(True)
                err = engine.take_async_error()
            if err:
                raise ValueError(last_error())
            beam_step = engine.beam_step
            if procs is not None:
                engine.beam_begin_proc(kv, procs)
                beam_step = engine.beam_step_proc
            planner = _beam.SlotPlanner(B, nb)
            row_begin = 0  # the first plan copies whole prompts; later ones only rows behind the shortest prompt
            step = 0
            while not search.step(*cand):
                step += 1
                copies = planner.plan(search.parents)
                cand = beam_step(kv, copies, row_begin, search.next_tokens().tolist(), planner.flat(),
                                        search.running_scores.reshape(-1).tolist(), nb, search.K, sampling=bs, step=step,
                                        **({"row_scores": at("scores", step), "row_logits": at("logits", step)} if want else {}))
                row_begin = min(lens)
            engine.check_async_error()
        finally:
            self._pool.release(kv)
        seq, seq_scores = search.output()
        seq = seq.to(device=prompt.device, dtype=prompt.dtype)
        if not want:
            return seq
        from transformers.generation.utils import GenerateBeamDecoderOnlyOutput

        n = search.cur_len - search.Lt  # steps taken: b2_beam_step synchronised on every one
        return GenerateBeamDecoderOnlyOutput(
            sequences=seq, sequences_scores=seq_scores.to(engine.device) if want["scores"] else None,
            scores=_trim_steps(rows.pop("scores"), n), logits=_trim_steps(rows.pop("logits"), n),
            beam_indices=search.output_beam_indices().to(engine.device), attentions=None, hidden_states=None, past_key_values=None)

    def _prefix_cache_on(self):
        """config.b2_prefix_cache or B2_PREFIX_CACHE=1 (off by default: logits of reused answer rows, which the decode kernels
        wrote, differ from a fresh prefill's by bf16 rounding). Not used when config.b2_continuous_batching routes generate()
        to the batcher."""
        v = getattr(self.config, "b2_prefix_cache", None)
        return bool(v) if v is not None else os.environ.get("B2_PREFIX_CACHE") == "1"

    def _prefix_plan(self, prompt, images):
        """The spliced items of a batch-1 prompt (llava/_b2/prefix.py), or None when the prompt is outside what the host splice
        reproduces exactly here (placeholders and image slots do not pair up, truncation, negative ids without images)."""
        ids = [int(t) for t in prompt[0].tolist()]
        tower = self.get_vision_tower()
        if images is None or tower is None:
            return None if any(t < 0 for t in ids) else {"items": ids, "slots": [], "images": None}
        if isinstance(images, (list, tuple)):
            slots = list(images)
            if any(not torch.is_tensor(x) or x.dim() != 4 for x in slots):
                return None
        elif images.dim() in (4, 5):
            slots = [images[j] for j in range(images.shape[0])]
        else:
            return None
        if sum(t == IMAGE_TOKEN_INDEX for t in ids) != len(slots) or len(ids) < 2:
            return None
        it = iter(slots)
        items = [next(it) if t == IMAGE_TOKEN_INDEX else t for t in ids]
        total = sum(_prefix.item_rows(x, tower.num_patches) for x in items)
        max_len = getattr(self.config, "tokenizer_model_max_length", None)
        if max_len is not None and total > max_len:
            return None
        return {"items": items, "slots": slots, "images": images}

    def _prefill_reusing(self, engine, kv, plan, m, released_ev, sampling, max_new_tokens, procs=None, lookup=None, out_rows=None):
        """Prefill of a planned prompt that keeps the first m spliced rows of `kv`: image slots wholly inside them are not
        encoded, rows [m, L) are spliced on the host-index path and prefilled at position m (b2_prefill_at). m == 0 is an
        ordinary prefill from position 0. Chooses and publishes token 0 like generate()'s own prefill. Returns whether the
        generation decodes with prompt lookup (`lookup`: generate()'s lookup(rows) or None). `out_rows`: generate()'s score / logits
        buffers ({"scores", "logits"}, entries may be None)."""
        P = engine.num_patches
        items, slots = plan["items"], plan["slots"]
        rows = [_prefix.item_rows(x, P) for x in slots]
        L = sum(_prefix.item_rows(x, P) for x in items)
        self._check_limits(engine, 1, L + max_new_tokens)
        ends, pos = [], 0
        for x in items:
            pos += _prefix.item_rows(x, P)
            if not isinstance(x, int):
                ends.append(pos)
        skip = sum(e <= m for e in ends)       # leading slots that lie wholly inside the reused rows
        if slots:
            ids_np = np.asarray([[IMAGE_TOKEN_INDEX if not isinstance(x, int) else x for x in items]], dtype=np.int64)
            src = build_source_index(ids_np, np.ones_like(ids_np, dtype=bool), np.zeros_like(ids_np), sum(rows), rows, None,
                                     "right", vocab_size=self.get_model().embed_tokens.weight.shape[0])[0][0]
            chunk = _prefix.chunk_source_index(src, m, sum(rows[:skip]), INT32_MIN)
        else:  # text only: the ids are the embedding rows (out-of-range ids are flagged by the splice kernel)
            chunk = np.asarray(items[m:], dtype=np.int32)
        feats = None
        if skip < len(slots):
            images = plan["images"]
            todo = images[skip:] if torch.is_tensor(images) and images.dim() == 4 else list(slots[skip:])
            feats, _ = self._image_features(todo)
        embeds = engine.splice(torch.from_numpy(chunk).to(engine.device), feats, 1, L - m)
        if m > 0:
            if released_ev is not None:
                torch.cuda.current_stream(engine.device).wait_event(released_ev)
            logits = engine.prefill(kv, embeds, None, LOGITS_LAST, start=[m])
            self._pool.count_reuse(m, sum(x.shape[0] if x.dim() == 4 else 1 for x in slots[:skip]))
        else:
            kv.reset()
            logits = engine.prefill(kv, embeds, None, LOGITS_LAST)
        lk = lookup(L) if lookup is not None else None
        if lk is not None:
            engine.stream_begin_lookup(kv, logits, sampling, lk)
        else:
            out_rows = out_rows or {}
            engine.stream_begin(kv, logits, sampling, procs, out_rows.get("scores"), out_rows.get("logits"))
        engine.stream_wait(kv, 0, 1)
        return lk is not None

    # ------------------------------------------------------------------ checkpoints
    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, *model_args, config=None, torch_dtype=None,
                        low_cpu_mem_usage=True, device_map=None, device=None, **kwargs):
        """Minimal HF-style loader: `config.json` + safetensors / pytorch_model*.bin shards in a local directory
        (ref builder.py:105-106 calls this). 4-bit loading (`load_in_4bit=True`, or a `quantization_config` — a
        transformers BitsAndBytesConfig or a dict — with load_in_4bit and bnb_4bit_quant_type "nf4") sets
        config.b2_weight_format = "nf4": the engine then holds NF4 decoder Linears (include/b2llava.h,
        b2_model_enable_nf4). 8-bit loading and FP4 are not part of the H100 path."""
        nf4 = _nf4_requested(kwargs)
        path = pretrained_model_name_or_path
        if not os.path.isdir(path):
            raise ValueError(f"{path!r} is not a local checkpoint directory (no network access on this path)")
        if config is None:
            with open(os.path.join(path, "config.json")) as f:
                config = LlavaConfig(**json.load(f))
        if nf4:
            config.b2_weight_format = "nf4"
            _check_weight_format(config)
        dev = device
        if dev is None and isinstance(device_map, (str, torch.device)) and str(device_map) not in ("auto",):
            dev = device_map
        if dev is None:
            dev = "cuda"
        model = cls(config, device=dev, dtype=torch.bfloat16)
        sd = _read_checkpoint_dir(path)
        if not sd:
            raise RuntimeError(f"no weight files found under {path!r}")
        own = model.state_dict()
        sd = {k: v for k, v in sd.items() if k in own}
        missing = [k for k in own if k not in sd and "vision_tower" not in k]
        if missing:
            raise RuntimeError(f"checkpoint is missing tensors: {missing[:8]} ...")
        model.load_state_dict(sd, strict=False)
        return model

    def eval(self):
        return super().eval()


def _beam_logits_processors_on(config):
    """config.b2_beam_logits_processors or B2_BEAM_LOGITS_PROCESSORS=1: generate(num_beams > 1) runs the logits processors that
    config.b2_logits_processors enables (off by default, like the other b2_* opt-ins)."""
    v = getattr(config, "b2_beam_logits_processors", None)
    return bool(v) if v is not None else os.environ.get("B2_BEAM_LOGITS_PROCESSORS") == "1"


def _nf4_requested(kwargs):
    """True when from_pretrained's arguments ask for bitsandbytes NF4 (the reference's load_4bit); raises NotImplementedError
    for the quantised loads this package does not serve (8-bit, FP4)."""
    qc = kwargs.get("quantization_config")
    if kwargs.get("load_in_8bit"):
        raise NotImplementedError("8-bit (LLM.int8) loading is not part of the H100 path")
    if qc is None:
        return bool(kwargs.get("load_in_4bit"))
    get = qc.get if isinstance(qc, dict) else (lambda k, d=None: getattr(qc, k, d))
    if get("load_in_8bit", False):
        raise NotImplementedError("8-bit (LLM.int8) loading is not part of the H100 path")
    if not get("load_in_4bit", False):
        raise NotImplementedError("quantization_config without load_in_4bit: only bitsandbytes NF4 is served")
    qt = get("bnb_4bit_quant_type", "fp4")  # BitsAndBytesConfig's own default
    if qt != "nf4":
        raise NotImplementedError(f"bnb_4bit_quant_type={qt!r}: only 'nf4' is served")
    return True


def _check_weight_format(config):
    """config.b2_weight_format: None / "bf16" (default) or "nf4"; NF4 and the e4m3 decode weights do not combine."""
    fmt = getattr(config, "b2_weight_format", None) or "bf16"
    if fmt not in ("bf16", "nf4"):
        raise ValueError(f"unknown b2_weight_format {fmt!r}: expected 'bf16' or 'nf4'")
    if fmt == "nf4" and (getattr(config, "b2_fp8_decode", False) or os.environ.get("B2_FP8_DECODE") == "1"):
        raise ValueError("b2_weight_format='nf4' (load_4bit) cannot be combined with b2_fp8_decode (e4m3 decode weights)")
    return fmt


def _output_arguments(return_dict_in_generate, output_scores, output_logits, kwargs):
    """{"scores", "logits"}: which per-step rows a generate(return_dict_in_generate=True) call returns, or None when generate()
    returns the id tensor (output_scores / output_logits are then ignored, as HF ignores them)."""
    if not return_dict_in_generate:
        return None
    for k in ("output_attentions", "output_hidden_states"):
        if kwargs.get(k):
            raise NotImplementedError(f"{k}=True with return_dict_in_generate: attention maps / hidden states are never "
                                      "materialised on the fused path")
    return {"scores": bool(output_scores), "logits": bool(output_logits)}


def _num_return_arguments(config, kwargs, B, do_sample, images):
    """generate(num_return_sequences=n) without beams: takes n out of `kwargs` and checks what the fork does not serve. Greedy
    raises transformers' GenerationConfig.validate error; do_sample with temperature <= 1e-5 decodes greedily and returns n
    equal rows."""
    n = kwargs.pop("num_return_sequences", None)
    n = 1 if n is None else int(n)
    if n == 1:
        return 1
    if n < 1:
        raise ValueError(f"num_return_sequences must be a positive integer, got {n}")
    if not do_sample:
        from transformers import GenerationConfig

        GenerationConfig(num_return_sequences=n).validate()
    if kwargs.get("prompt_lookup_num_tokens") is not None:
        raise ValueError(f"num_return_sequences has to be 1 when doing assisted generate, but is {n}.")
    if images is not None and not torch.is_tensor(images):
        raise NotImplementedError("num_return_sequences > 1 with a list of images: transformers does not expand a list to the "
                                  "samples of each prompt; pass the images as one tensor")
    if B == 1 and int(getattr(config, "b2_continuous_batching", 0) or 0) >= 2:
        raise NotImplementedError("num_return_sequences > 1 together with the continuous batcher (b2_continuous_batching) is "
                                  "not implemented")
    return n


def _trim_steps(buf, n):
    """generate()'s rows [max_new_tokens, rows, V] -> a tuple of the first n steps' [rows, V] tensors. The decode steps were
    ordered before later work on the caller's current stream when they were queued, so reading there is safe; a buffer with
    an unused tail is copied, so the tail is not kept alive by the returned views."""
    if buf is None:
        return None
    if n < buf.shape[0]:
        buf = buf[:n].clone()
    return tuple(buf.unbind(0))


def _decoder_output(sequences, scores, logits):
    from transformers.generation.utils import GenerateDecoderOnlyOutput

    return GenerateDecoderOnlyOutput(sequences=sequences, scores=scores, logits=logits, attentions=None, hidden_states=None,
                                     past_key_values=None)


# verify steps a prompt-lookup generation keeps queued in front of the host: two keep the device busy while the host handles a
# step's tokens, and bound what runs after the host stops
_LOOKUP_STEPS_IN_FLIGHT = 2


def _stream_decode(engine, kv, logits, sampling, B, max_new_tokens, eos_ids, pad, prompt, streamer, stopping_criteria,
                   run_ahead=8, begun=False, lookup_steps=0, slot_of_row=None):
    """Host half of the decode loop. The device chooses token 0 from the prefill `logits` and then runs up to `run_ahead`
    steps in front of this loop; `engine.stream_wait(kv, t, B)` hands over token t as soon as its kernel has written it
    to pinned memory. Per token, in the order HF's loop uses: finished rows show `pad`; streamer.put; eos bookkeeping;
    stopping criteria on cat(prompt, tokens so far) (the reference's KeywordsStoppingCriteria looks at the tail of that
    tensor, llava/mm_utils.py:92-114). Returns a CPU int64 tensor [B, n], 1 <= n <= max_new_tokens.
    lookup_steps > 0 (a prompt-lookup generation): a step publishes a varying number of tokens, so instead of counting tokens the
    loop asks the engine before each token to keep `lookup_steps` verify steps in flight (b2_stream_enqueue tops them up against
    the steps the device has retired and queues none once max_new_tokens are published).
    slot_of_row (a forked generation, llava/_b2/fork.py): row r of the result, of the streamer and of the criteria is the device's
    slot slot_of_row[r]."""
    Lt = prompt.shape[1]
    crit_buf = None
    if stopping_criteria:
        crit_buf = torch.empty(B, Lt + max_new_tokens, dtype=torch.long)
        crit_buf[:, :Lt] = prompt.to("cpu", torch.long)
    run_ahead = max(1, int(run_ahead))
    if not begun:  # generate() begins the stream itself (it confirms its input checks on token 0 before any output)
        engine.stream_begin(kv, logits, sampling)
    scheduled = 1                                   # tokens whose kernels have been queued (token 0 = begin)
    finished = [False] * B
    cols = []
    for t in range(max_new_tokens):
        if lookup_steps > 0:
            engine.stream_enqueue(kv, lookup_steps)
        # keep the device `run_ahead` tokens in front of the host (queued in blocks: one call per ~run_ahead/2 tokens)
        elif scheduled < max_new_tokens and scheduled - t <= (run_ahead + 1) // 2:
            n = min(run_ahead - (scheduled - t) + 1, max_new_tokens - scheduled)
            if n > 0:
                engine.stream_enqueue(kv, n)
                scheduled += n
        toks = engine.stream_wait(kv, t, B)
        if slot_of_row is not None:
            toks = [toks[s] for s in slot_of_row]
        col = [pad if finished[b] else int(toks[b]) for b in range(B)]
        cols.append(col)
        if streamer is not None:
            streamer.put(torch.tensor(col, dtype=torch.long))
        for b in range(B):
            if col[b] in eos_ids:
                finished[b] = True
        stop = bool(eos_ids) and all(finished)
        if crit_buf is not None:
            crit_buf[:, Lt + t] = torch.tensor(col, dtype=torch.long)
            view = crit_buf[:, :Lt + t + 1]
            for crit in stopping_criteria:
                r = crit(view, None)
                stop = stop or (bool(r.all()) if torch.is_tensor(r) else bool(r))
        if stop:
            break
    return torch.tensor(cols, dtype=torch.long).t().contiguous()


class _StageTimer:
    """B2_PROFILE_GENERATE=1: wall-clock per stage of generate() with a device sync at every mark (debug aid; the
    syncs serialise host and device, so the stages add up to MORE than an unprofiled call)."""

    def __init__(self):
        import time
        self._t, self._clock, self._rows = time.perf_counter(), time.perf_counter, []

    def mark(self, name):
        torch.cuda.synchronize()
        t = self._clock()
        self._rows.append((name, (t - self._t) * 1e3))
        self._t = t

    def report(self):
        import sys
        print("generate stages (ms): " + ", ".join(f"{n} {ms:.2f}" for n, ms in self._rows), file=sys.stderr)


try:  # the installed transformers may already ship a "llava" model type (ref llava_llama.py:110-111)
    AutoConfig.register("llava", LlavaConfig, exist_ok=True)
except Exception:  # pragma: no cover - registry differences across transformers versions
    pass
