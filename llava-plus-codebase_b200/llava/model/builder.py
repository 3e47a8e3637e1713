"""load_pretrained_model — the loader contract of the reference's llava/model/builder.py:26-151
(`(tokenizer, model, image_processor, context_len)`), restricted to what the H100 path serves: full LLaVA-1.5
(LLaMA/Vicuna) checkpoints from a local directory. `load_4bit=True` passes the reference's own BitsAndBytesConfig
(builder.py:32-38) and loads NF4 decoder Linears, quantised at load from the ordinary checkpoint
(include/b2llava.h, b2_model_enable_nf4; DESIGN.md §2 states where the arithmetic differs from bitsandbytes).
LoRA merging, MPT, projector-only checkpoints on a base LLM and 8-bit (LLM.int8) loading are outside the hot path
and raise NotImplementedError.
"""
import os

import torch
from transformers import AutoTokenizer, BitsAndBytesConfig

from .language_model.llava_llama import LlavaLlamaForCausalLM
from ..constants import DEFAULT_IMAGE_PATCH_TOKEN, DEFAULT_IM_START_TOKEN, DEFAULT_IM_END_TOKEN


def load_pretrained_model(model_path, model_base, model_name, load_8bit=False, load_4bit=False, device_map="auto",
                          device="cuda"):
    if load_8bit:
        raise NotImplementedError("bitsandbytes 8-bit (LLM.int8) loading is not part of the H100 path")
    kwargs = {}
    if load_4bit:  # ref builder.py:32-38
        kwargs["quantization_config"] = BitsAndBytesConfig(load_in_4bit=True, bnb_4bit_compute_dtype=torch.float16,
                                                           bnb_4bit_use_double_quant=True, bnb_4bit_quant_type="nf4")
    if "llava" not in model_name.lower():
        raise NotImplementedError("only LLaVA (LLaMA/Vicuna) checkpoints are served by this package")
    if "lora" in model_name.lower() or model_base is not None or "mpt" in model_name.lower():
        raise NotImplementedError("LoRA / delta / MPT checkpoints: merge offline with the reference's scripts first")
    if device != "cuda" and not str(device).startswith("cuda"):
        raise RuntimeError("the H100 path needs a CUDA (sm_90a) device; there is no CPU fallback")

    tokenizer = AutoTokenizer.from_pretrained(model_path, use_fast=False)
    model = LlavaLlamaForCausalLM.from_pretrained(model_path, low_cpu_mem_usage=True, device=device, **kwargs)

    # ref builder.py:131-138
    if getattr(model.config, "mm_use_im_patch_token", True):
        tokenizer.add_tokens([DEFAULT_IMAGE_PATCH_TOKEN], special_tokens=True)
    if getattr(model.config, "mm_use_im_start_end", False):
        tokenizer.add_tokens([DEFAULT_IM_START_TOKEN, DEFAULT_IM_END_TOKEN], special_tokens=True)
    model.resize_token_embeddings(len(tokenizer))

    # ref builder.py:140-144: the tower weights come from the separate CLIP checkpoint
    vision_tower = model.get_vision_tower()
    if not vision_tower.is_loaded:
        vision_tower.load_model()
    vision_tower.to(device=device, dtype=torch.bfloat16)
    image_processor = vision_tower.image_processor

    context_len = getattr(model.config, "max_sequence_length", 2048)  # ref builder.py:146-149
    return tokenizer, model, image_processor, context_len
