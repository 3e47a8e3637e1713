"""ctypes binding of libb2llava.so (C ABI: include/b2llava.h).

PyTorch is used here only for device memory and streams: every call passes raw `tensor.data_ptr()` values
and `torch.cuda.current_stream().cuda_stream` across the ABI. There is no CPU or eager fallback: if the
library is missing or the device is not sm_90, calls raise.
"""
import ctypes
import os
import threading
import weakref

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get(
    "B2LLAVA_LIB", os.path.normpath(os.path.join(_HERE, "..", "..", "lib", "libb2llava.so"))
)

DT_BF16, DT_F16, DT_F32 = 0, 1, 2
ACT_NONE, ACT_QUICK_GELU, ACT_GELU_ERF, ACT_SWIGLU = 0, 1, 2, 3
LOGITS_NONE, LOGITS_LAST, LOGITS_ALL = 0, 1, 2
KV_BF16, KV_E4M3 = 0, 1
KV_DTYPES = {"bf16": KV_BF16, "e4m3": KV_E4M3}
INT32_MIN = -(2**31)
ERR_TOKEN_RANGE, ERR_IMAGE_ROW_RANGE, ERR_SPLICE_SLOTS = 1, 2, 4

_c = ctypes
_vp, _i32, _i64, _f32 = _c.c_void_p, _c.c_int, _c.c_int64, _c.c_float


class ModelDesc(_c.Structure):
    _fields_ = [
        ("image_size", _c.c_int32), ("patch_size", _c.c_int32), ("vit_hidden", _c.c_int32),
        ("vit_inter", _c.c_int32), ("vit_layers", _c.c_int32), ("vit_heads", _c.c_int32),
        ("vit_select_layer", _c.c_int32), ("vit_ln_eps", _c.c_float),
        ("hidden", _c.c_int32), ("inter", _c.c_int32), ("layers", _c.c_int32), ("heads", _c.c_int32),
        ("vocab", _c.c_int32), ("rms_eps", _c.c_float), ("rope_theta", _c.c_float),
        ("max_batch", _c.c_int32), ("max_seq", _c.c_int32), ("max_images", _c.c_int32),
    ]


class Sampling(_c.Structure):
    """b2_sampling (include/b2llava.h): do_sample == 0 -> greedy argmax."""
    _fields_ = [("do_sample", _c.c_int32), ("temperature", _c.c_float), ("top_p", _c.c_float),
                ("top_k", _c.c_int32), ("seed", _c.c_ulonglong)]


class PreprocessPlan(_c.Structure):
    """b2_preprocess_plan (include/b2llava.h)."""
    _fields_ = [("img", _vp), ("H", _c.c_int32), ("W", _c.c_int32), ("pad_top", _c.c_int32), ("pad_left", _c.c_int32),
                ("bg", _c.c_uint8 * 4), ("h_bounds", _vp), ("h_kk", _vp), ("h_ksize", _c.c_int32), ("h_identity", _c.c_int32),
                ("v_bounds", _vp), ("v_kk", _vp), ("v_ksize", _c.c_int32), ("v_identity", _c.c_int32),
                ("y0", _c.c_int32), ("rows", _c.c_int32), ("x_lo", _c.c_int32), ("y_lo", _c.c_int32), ("out", _c.c_int32),
                ("tmp", _vp), ("mean", _c.c_float * 3), ("stdv", _c.c_float * 3), ("rescale", _c.c_float),
                ("pixels", _vp), ("u8_out", _vp)]


class BeamStepArgs(_c.Structure):
    """b2_beam_step_args (include/b2llava.h)."""
    _fields_ = [("copy_src_host", _vp), ("copy_dst_host", _vp), ("n_copies", _c.c_int32), ("row_begin", _c.c_int32),
                ("B", _c.c_int32), ("nb", _c.c_int32), ("K", _c.c_int32), ("tokens_host", _vp), ("slot_of_beam_host", _vp),
                ("beam_scores_host", _vp), ("out_scores_host", _vp), ("out_tokens_host", _vp), ("out_beams_host", _vp)]


class BeamSampling(_c.Structure):
    """b2_beam_sampling (include/b2llava.h): warpers and Philox key of beam sampling."""
    _fields_ = [("temperature", _c.c_float), ("top_k", _c.c_int32), ("top_p", _c.c_float), ("min_keep", _c.c_int32),
                ("seed", _c.c_ulonglong)]


def make_beam_sampling(temperature=1.0, top_k=50, top_p=1.0, min_keep=2, seed=0):
    return BeamSampling(float(temperature), int(top_k or 0), float(1.0 if top_p is None else top_p), int(min_keep),
                        int(seed) & (2**64 - 1))


class LogitsProc(_c.Structure):
    """b2_logits_proc (include/b2llava.h): history-aware logits processors of one row; `prompt_ids` is a device int64 pointer."""
    _fields_ = [("repetition_penalty", _c.c_float), ("no_repeat_ngram_size", _c.c_int32), ("min_generated", _c.c_int32),
                ("n_eos", _c.c_int32), ("eos_ids", _c.c_int32 * 8), ("prompt_ids", _vp), ("prompt_len", _c.c_int32)]


MAX_PROC_EOS = 8


class PrefixGroup(_c.Structure):
    """b2_prefix_group (include/b2llava.h): rows of one batch that read keys [0, prefix_len) from slot src_slot."""
    _fields_ = [("src_slot", _c.c_int32), ("prefix_len", _c.c_int32), ("n_rows", _c.c_int32), ("rows", _c.c_int32 * 16)]


def _group_array(groups):
    """ctypes array of PrefixGroup from (src_slot, prefix_len, rows) triples."""
    arr = (PrefixGroup * len(groups))()
    for i, (src, plen, rows) in enumerate(groups):
        if not 1 <= len(rows) <= 16:
            raise ValueError(f"a prefix group holds 1..16 rows, got {len(rows)}")
        arr[i].src_slot, arr[i].prefix_len, arr[i].n_rows = int(src), int(plen), len(rows)
        for j, r in enumerate(rows):
            arr[i].rows[j] = int(r)
    return arr


class PromptLookup(_c.Structure):
    """b2_prompt_lookup (include/b2llava.h): prompt-lookup speculative decoding of one sample; `prompt_ids` is a device int64
    pointer."""
    _fields_ = [("num_tokens", _c.c_int32), ("max_ngram", _c.c_int32), ("max_new_tokens", _c.c_int32), ("n_eos", _c.c_int32),
                ("eos_ids", _c.c_int32 * 8), ("prompt_ids", _vp), ("prompt_len", _c.c_int32)]


def make_prompt_lookup(prompt_row, num_tokens, max_ngram, max_new_tokens, eos_ids=()):
    """PromptLookup over `prompt_row` (device int64 [L], kept alive as `.ids` of the result)."""
    eos = sorted(set(int(e) for e in eos_ids))
    if len(eos) > MAX_PROC_EOS:
        raise ValueError(f"at most {MAX_PROC_EOS} eos ids are supported with prompt lookup, got {len(eos)}")
    if prompt_row.dtype != torch.int64 or prompt_row.dim() != 1 or not prompt_row.is_cuda or not prompt_row.is_contiguous():
        raise ValueError("prompt_row must be a contiguous 1-D int64 CUDA tensor")
    lk = PromptLookup(int(num_tokens), int(max_ngram), int(max_new_tokens), len(eos))
    for i, e in enumerate(eos):
        lk.eos_ids[i] = e
    lk.prompt_ids = prompt_row.data_ptr() if prompt_row.numel() else None
    lk.prompt_len = int(prompt_row.numel())
    lk.ids = prompt_row
    return lk


def make_logits_proc(prompt_row, repetition_penalty=1.0, no_repeat_ngram_size=0, min_generated=0, eos_ids=()):
    """LogitsProc over `prompt_row` (device int64 [L], kept alive as `.ids` of the result; a caller that hands the struct to
    work on another stream records that stream on it), or None when every processor is at its off value. min_generated: eos ids are banned while fewer tokens were generated."""
    eos = sorted(set(int(e) for e in eos_ids))
    if len(eos) > MAX_PROC_EOS:
        raise ValueError(f"at most {MAX_PROC_EOS} eos ids are supported with logits processors, got {len(eos)}")
    p = float(1.0 if repetition_penalty is None else repetition_penalty)
    n = int(no_repeat_ngram_size or 0)
    mg = int(min_generated or 0) if eos else 0
    if p == 1.0 and n == 0 and mg <= 0:
        return None
    if prompt_row.dtype != torch.int64 or prompt_row.dim() != 1 or not prompt_row.is_cuda or not prompt_row.is_contiguous():
        raise ValueError("prompt_row must be a contiguous 1-D int64 CUDA tensor")
    lp = LogitsProc(p, n, max(mg, 0), len(eos))
    for i, e in enumerate(eos):
        lp.eos_ids[i] = e
    lp.prompt_ids = prompt_row.data_ptr() if prompt_row.numel() else None
    lp.prompt_len = int(prompt_row.numel())
    lp.ids = prompt_row  # the tensor behind prompt_ids: whoever holds the struct keeps the ids alive
    return lp


def _proc_array(procs, B):
    """ctypes array of B LogitsProc (None entries = off), or None when every row is off."""
    if procs is None or all(p is None for p in procs):
        return None
    if len(procs) != B:
        raise ValueError(f"{len(procs)} logits processors for {B} rows")
    arr = (LogitsProc * B)()
    for b, p in enumerate(procs):
        arr[b] = p if p is not None else LogitsProc(1.0, 0, 0, 0)
    return arr


def make_sampling(do_sample=False, temperature=1.0, top_p=1.0, top_k=0, seed=0):
    return Sampling(int(bool(do_sample)), float(temperature), float(1.0 if top_p is None else top_p),
                    int(top_k or 0), int(seed) & (2**64 - 1))


# name -> (restype, argtypes); must list every symbol include/b2llava.h declares (tests check this)
SIGNATURES = {
    "b2_init": (_i32, [_i32]),
    "b2_last_error": (_c.c_char_p, []),
    "b2_version": (_i32, []),
    "b2_launch_count": (_c.c_ulonglong, []),
    "b2_model_create": (_i32, [_c.POINTER(ModelDesc), _c.POINTER(_vp)]),
    "b2_model_set_weight": (_i32, [_vp, _c.c_char_p, _vp, _c.POINTER(_i64), _i32, _i32]),
    "b2_model_finalize": (_i32, [_vp]),
    "b2_model_destroy": (_i32, [_vp]),
    "b2_model_enable_fp8_decode": (_i32, [_vp]),
    "b2_model_enable_nf4": (_i32, [_vp]),
    "b2_model_weight_bytes": (_i64, [_vp]),
    "b2_kv_create": (_i32, [_vp, _i32, _i32, _c.POINTER(_vp)]),
    "b2_kv_create_ex": (_i32, [_vp, _i32, _i32, _i32, _c.POINTER(_vp)]),
    "b2_kv_dtype": (_i32, [_vp]),
    "b2_kv_bytes": (_i64, [_vp]),
    "b2_kv_reset": (_i32, [_vp]),
    "b2_kv_destroy": (_i32, [_vp]),
    "b2_kv_lengths": (_i32, [_vp, _c.POINTER(_c.c_int32), _i32]),
    "b2_vit_encode": (_i32, [_vp, _vp, _i32, _vp, _vp]),
    "b2_project": (_i32, [_vp, _vp, _i32, _vp, _vp]),
    "b2_encode_images": (_i32, [_vp, _vp, _i32, _vp, _vp]),
    "b2_splice": (_i32, [_vp, _vp, _vp, _i32, _i32, _vp, _vp]),
    "b2_splice_ids": (_i32, [_vp, _vp, _i32, _i32, _i32, _c.POINTER(_c.c_int32), _i32, _vp, _i32, _vp, _vp]),
    "b2_async_error": (_i32, [_vp, _c.POINTER(_c.c_int)]),
    "b2_stream_begin": (_i32, [_vp, _vp, _vp, _i32, _c.POINTER(Sampling), _vp]),
    "b2_stream_begin_ex": (_i32, [_vp, _vp, _vp, _i32, _c.POINTER(Sampling), _c.POINTER(LogitsProc), _vp]),
    "b2_stream_begin_groups": (_i32, [_vp, _vp, _vp, _i32, _c.POINTER(Sampling), _c.POINTER(LogitsProc), _c.POINTER(PrefixGroup), _i32,
                                      _vp]),
    "b2_stream_enqueue": (_i32, [_vp, _vp, _i32, _vp]),
    "b2_stream_wait": (_i32, [_vp, _i32, _c.POINTER(_c.c_int32), _i32]),
    "b2_stream_set_outputs": (_i32, [_vp, _vp, _vp, _i32]),
    "b2_stream_begin_lookup": (_i32, [_vp, _vp, _vp, _i32, _c.POINTER(Sampling), _c.POINTER(PromptLookup), _vp]),
    "b2_stream_lookup_stats": (_i32, [_vp, _c.POINTER(_c.c_int32), _c.POINTER(_c.c_int32), _c.POINTER(_c.c_int32)]),
    "b2_decode_rows": (_i32, [_vp, _vp, _i32, _vp, _i32, _vp, _vp]),
    "b2_op_preprocess_clip": (_i32, [_c.POINTER(PreprocessPlan), _vp]),
    "b2_op_sample": (_i32, [_vp, _i32, _i32, _c.POINTER(Sampling), _i32, _vp, _vp]),
    "b2_op_sample_ex": (_i32, [_vp, _i32, _i32, _c.POINTER(Sampling), _c.POINTER(LogitsProc), _i32, _vp, _vp, _vp]),
    "b2_prefill": (_i32, [_vp, _vp, _vp, _c.POINTER(_c.c_int32), _i32, _i32, _vp, _i32, _vp]),
    "b2_prefill_slots": (_i32, [_vp, _vp, _vp, _c.POINTER(_c.c_int32), _i32, _i32, _i32, _vp, _i32, _vp]),
    "b2_prefill_at": (_i32, [_vp, _vp, _vp, _c.POINTER(_c.c_int32), _c.POINTER(_c.c_int32), _i32, _i32, _i32, _vp, _i32, _vp]),
    "b2_batch_begin": (_i32, [_vp, _vp, _i32, _vp]),
    "b2_batch_set_row": (_i32, [_vp, _vp, _i32, _i32, _c.POINTER(Sampling), _i32, _vp]),
    "b2_batch_set_row_ex": (_i32, [_vp, _vp, _i32, _i32, _c.POINTER(Sampling), _c.POINTER(LogitsProc), _i32, _vp]),
    "b2_decode_step": (_i32, [_vp, _vp, _vp, _i32, _vp, _vp, _vp]),
    "b2_decode_greedy": (_i32, [_vp, _vp, _vp, _i32, _i32, _vp, _vp]),
    "b2_argmax": (_i32, [_vp, _i32, _i32, _vp, _vp]),
    "b2_kv_copy_slots": (_i32, [_vp, _vp, _c.POINTER(_c.c_int32), _c.POINTER(_c.c_int32), _i32, _i32, _vp]),
    "b2_op_beam_topk": (_i32, [_vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp]),
    "b2_beam_step": (_i32, [_vp, _vp, _c.POINTER(BeamStepArgs), _vp]),
    "b2_op_beam_sample": (_i32, [_vp, _vp, _vp, _i32, _i32, _i32, _i32, _c.POINTER(BeamSampling), _c.c_uint32, _vp, _vp, _vp, _vp]),
    "b2_beam_step_ex": (_i32, [_vp, _vp, _c.POINTER(BeamStepArgs), _c.POINTER(BeamSampling), _c.c_uint32, _vp]),
    "b2_op_beam_select_out": (_i32, [_vp, _vp, _vp, _i32, _i32, _i32, _i32, _c.POINTER(BeamSampling), _c.c_uint32, _i32, _vp, _vp,
                                     _vp, _vp, _vp, _vp]),
    "b2_beam_step_out": (_i32, [_vp, _vp, _c.POINTER(BeamStepArgs), _c.POINTER(BeamSampling), _c.c_uint32, _vp, _vp, _vp]),
    "b2_op_beam_select_proc": (_i32, [_vp, _i32, _vp, _vp, _i32, _i32, _i32, _i32, _c.POINTER(BeamSampling), _c.c_uint32, _i32,
                                      _c.POINTER(LogitsProc), _vp, _vp, _vp, _vp, _vp, _vp]),
    "b2_beam_begin_proc": (_i32, [_vp, _vp, _i32, _c.POINTER(LogitsProc), _vp]),
    "b2_beam_step_proc": (_i32, [_vp, _vp, _c.POINTER(BeamStepArgs), _c.POINTER(BeamSampling), _c.c_uint32, _vp, _vp, _vp]),
    "b2_op_gemm": (_i32, [_vp, _i32, _vp, _i32, _vp, _vp, _i32, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _vp]),
    "b2_op_gemv": (_i32, [_vp, _i64, _vp, _i32, _vp, _f32, _vp, _i32, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _vp]),
    "b2_op_quantize_nf4": (_i32, [_vp, _i32, _i32, _vp, _vp, _vp]),
    "b2_op_dequantize_nf4": (_i32, [_vp, _vp, _i32, _i32, _vp, _vp]),
    "b2_op_gemv_nf4": (_i32, [_vp, _i64, _vp, _vp, _vp, _f32, _vp, _i32, _vp, _i32, _i32, _i32, _i32, _i32, _vp]),
    "b2_op_gemm_skinny": (_i32, [_vp, _i32, _vp, _i32, _vp, _i32, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _i64, _vp, _vp]),
    "b2_op_gemm_skinny_fp8": (_i32, [_vp, _i32, _vp, _vp, _i32, _vp, _vp, _i32, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _i64, _vp, _vp]),
    "b2_op_quantize_rows_e4m3": (_i32, [_vp, _i64, _i32, _i32, _vp, _i64, _vp, _vp]),
    "b2_op_rmsnorm_quant_e4m3": (_i32, [_vp, _vp, _vp, _vp, _i32, _i32, _f32, _vp]),
    "b2_op_gemm_skinny_workspace_bytes": (_i64, [_i32, _i32, _i32]),
    "b2_op_gemm_skinny_counter_bytes": (_i64, [_i32]),
    "b2_op_layernorm": (_i32, [_vp, _vp, _vp, _vp, _i32, _i32, _f32, _vp]),
    "b2_op_rmsnorm": (_i32, [_vp, _vp, _vp, _i32, _i32, _f32, _vp]),
    "b2_op_flash_attn": (_i32, [_vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _f32, _vp]),
    "b2_op_rope_kv_write": (_i32, [_vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _f32, _vp]),
    "b2_op_flash_attn_kv": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _f32, _vp]),
    "b2_op_rope_kv_write_at": (_i32, [_vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _f32, _vp]),
    "b2_op_decode_attn": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _f32, _f32, _vp]),
    "b2_op_decode_attn_scratch_bytes": (_i64, [_i32, _i32, _i32]),
    "b2_op_decode_attn_e4m3": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _f32, _f32, _vp]),
    "b2_op_decode_attn_nsplit": (_i32, [_i32, _i32, _i32, _i32]),
    "b2_op_decode_attn_mq": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _f32, _vp]),
    "b2_op_decode_attn_mq_scratch_bytes": (_i64, [_i32, _i32, _i32]),
    "b2_op_decode_attn_mq_nsplit": (_i32, [_i32, _i32]),
    "b2_op_decode_attn_shared": (_i32, [_vp, _vp, _vp, _vp, _c.POINTER(PrefixGroup), _i32, _vp, _vp, _i32, _i32, _i32, _i32, _f32, _f32,
                                        _vp]),
    "b2_op_decode_attn_shared_scratch_bytes": (_i64, [_i32, _i32, _i32]),
    "b2_op_decode_attn_shared_nsplit": (_i32, [_i32, _i32, _i32]),
    "b2_op_prompt_lookup": (_i32, [_vp, _i32, _i32, _i32, _i32, _c.POINTER(_c.c_int32), _i32, _i32, _vp, _vp, _vp]),
    "b2_op_kv_quantize_e4m3": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp]),
    "b2_op_kv_quantize_e4m3_at": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _vp]),
    "b2_op_kv_dequantize_e4m3": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp]),
    "b2_op_interleave_gate_up": (_i32, [_vp, _vp, _vp, _i32, _i32, _vp]),
    "b2_op_im2col": (_i32, [_vp, _vp, _i32, _i32, _i32, _i32, _vp]),
}

_lib = None
_lib_lock = threading.Lock()
_inited_devices = set()


def load_library():
    """Load libb2llava.so (no GPU needed to load and resolve symbols)."""
    global _lib
    with _lib_lock:
        if _lib is None:
            if not os.path.exists(LIB_PATH):
                raise RuntimeError(
                    f"libb2llava.so not found at {LIB_PATH}: build it with "
                    f"`python llava-plus-codebase_b200/build.py` (there is no fallback path)"
                )
            lib = ctypes.CDLL(LIB_PATH)
            for name, (res, args) in SIGNATURES.items():
                fn = getattr(lib, name)
                fn.restype = res
                fn.argtypes = args
            _lib = lib
    return _lib


def last_error():
    return load_library().b2_last_error().decode("utf-8", "replace")


def check(rc, what=""):
    """Error convention of the reference's callers (SURVEY §8b): ValueError for bad arguments,
    RuntimeError for CUDA / state failures; never abort."""
    if rc == 0:
        return
    msg = f"{what}: {last_error()}" if what else last_error()
    if rc == -1:
        raise ValueError(msg)
    raise RuntimeError(msg)


def init(device_index):
    lib = load_library()
    if device_index not in _inited_devices:
        if not torch.cuda.is_available():
            raise RuntimeError("b2llava needs a CUDA device (sm_90a); no CPU fallback exists")
        check(lib.b2_init(int(device_index)), "b2_init")
        _inited_devices.add(device_index)
    return lib


def stream_ptr():
    return _vp(torch.cuda.current_stream().cuda_stream)


def ptr(t):
    if t is None:
        return _vp(0)
    return _vp(t.data_ptr())


def kv_dtype_code(dtype):
    """"bf16" | "e4m3" -> B2_KV_*; anything else is a ValueError (before anything is allocated)."""
    if dtype not in KV_DTYPES:
        raise ValueError(f"unknown KV cache dtype {dtype!r}: expected one of {sorted(KV_DTYPES)}")
    return KV_DTYPES[dtype]


def launch_count():
    return int(load_library().b2_launch_count())


_TORCH_DT = {torch.bfloat16: DT_BF16, torch.float16: DT_F16, torch.float32: DT_F32}


class KVCache:
    """Device KV cache handle (b2_kv): [layers][B][heads][max_seq][128] for K and V; bf16, or with dtype="e4m3" one byte per
    element plus an fp32 scale per (layer, sample, head, token) — 0.516 x the bytes, different decode numerics (b2llava.h)."""

    def __init__(self, engine, max_batch, max_seq, dtype="bf16"):
        self.engine = engine
        self.max_batch, self.max_seq, self.dtype = int(max_batch), int(max_seq), dtype
        code = kv_dtype_code(dtype)
        h = _vp()
        check(engine.lib.b2_kv_create_ex(engine.handle, self.max_batch, self.max_seq, code, ctypes.byref(h)), "b2_kv_create_ex")
        self.handle = h

    @property
    def nbytes(self):
        """Device bytes of K, V and their scales."""
        return int(self.engine.lib.b2_kv_bytes(self.handle))

    def reset(self):
        check(self.engine.lib.b2_kv_reset(self.handle), "b2_kv_reset")

    def lengths(self, n=None):
        n = self.max_batch if n is None else n
        arr = (_c.c_int32 * n)()
        check(self.engine.lib.b2_kv_lengths(self.handle, arr, n), "b2_kv_lengths")
        return list(arr)

    def get_seq_length(self, layer_idx=0):
        return self.lengths(1)[0]

    def close(self):
        if getattr(self, "handle", None) is not None and self.handle.value:
            self.engine.lib.b2_kv_destroy(self.handle)
            self.handle = _vp(0)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Engine:
    """Thin owner of a b2_model handle. All tensors are torch CUDA tensors used as raw device memory."""

    def __init__(self, desc: dict, device):
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("b2llava Engine requires a CUDA device; there is no CPU path")
        self.index = self.device.index if self.device.index is not None else torch.cuda.current_device()
        self.lib = init(self.index)
        self.desc = ModelDesc(**desc)
        h = _vp()
        with torch.cuda.device(self.index):
            check(self.lib.b2_model_create(ctypes.byref(self.desc), ctypes.byref(h)), "b2_model_create")
        self.handle = h
        self.hidden, self.vocab = desc["hidden"], desc["vocab"]
        self.vit_hidden = desc["vit_hidden"]
        self.num_patches = (desc["image_size"] // desc["patch_size"]) ** 2
        self.finalized = False
        self._kvs = weakref.WeakSet()

    # -- weights ------------------------------------------------------------------------------------
    def set_weight(self, key, tensor):
        t = tensor.detach()
        if t.dtype not in _TORCH_DT:
            t = t.float()
        t = t.contiguous()
        shape = (_i64 * max(t.dim(), 1))(*([int(s) for s in t.shape] or [1]))
        with torch.cuda.device(self.index):
            check(self.lib.b2_model_set_weight(self.handle, key.encode(), ptr(t), shape, max(t.dim(), 1),
                                               _TORCH_DT[t.dtype]), f"set_weight({key})")

    def finalize(self):
        with torch.cuda.device(self.index):
            check(self.lib.b2_model_finalize(self.handle), "b2_model_finalize")
        self.finalized = True

    def enable_fp8_decode(self):
        """BASELINE configs[4]: e4m3 weights for decode at batch >= 7 (see include/b2llava.h): W8A8 numerics, opt-in."""
        with torch.cuda.device(self.index):
            check(self.lib.b2_model_enable_fp8_decode(self.handle), "b2_model_enable_fp8_decode")

    def enable_nf4(self):
        """load_4bit: NF4 decoder Linears and a w_hat projector (see include/b2llava.h). Call after finalize() and before any
        KV cache exists; it cannot be combined with enable_fp8_decode()."""
        with torch.cuda.device(self.index):
            check(self.lib.b2_model_enable_nf4(self.handle), "b2_model_enable_nf4")

    def weight_bytes(self):
        """Device bytes of the weights the engine holds (workspaces excluded)."""
        return int(self.lib.b2_model_weight_bytes(self.handle))

    def new_kv(self, max_batch, max_seq, dtype="bf16"):
        with torch.cuda.device(self.index):
            kv = KVCache(self, max_batch, max_seq, dtype)
        self._kvs.add(kv)
        return kv

    # -- hot path -----------------------------------------------------------------------------------
    def _bf16(self, t):
        return t.to(device=self.device, dtype=torch.bfloat16).contiguous()

    def vit_encode(self, pixels):
        pixels = self._bf16(pixels)
        B = pixels.shape[0]
        out = torch.empty(B, self.num_patches, self.vit_hidden, dtype=torch.bfloat16, device=self.device)
        with torch.cuda.device(self.index):
            check(self.lib.b2_vit_encode(self.handle, ptr(pixels), B, ptr(out), stream_ptr()), "b2_vit_encode")
        return out

    def project(self, feats):
        feats = self._bf16(feats)
        rows = feats.numel() // self.vit_hidden
        out = torch.empty(*feats.shape[:-1], self.hidden, dtype=torch.bfloat16, device=self.device)
        with torch.cuda.device(self.index):
            check(self.lib.b2_project(self.handle, ptr(feats), rows, ptr(out), stream_ptr()), "b2_project")
        return out

    def encode_images(self, pixels):
        pixels = self._bf16(pixels)
        B = pixels.shape[0]
        out = torch.empty(B, self.num_patches, self.hidden, dtype=torch.bfloat16, device=self.device)
        with torch.cuda.device(self.index):
            check(self.lib.b2_encode_images(self.handle, ptr(pixels), B, ptr(out), stream_ptr()), "b2_encode_images")
        return out

    def splice(self, src_index, image_feats, B, S):
        """src_index: int32 device tensor [B*S]; image_feats: bf16 [n_rows, hidden] or None. Ids / rows out of range
        become zero rows and are reported by check_async_error() (never an out-of-bounds read)."""
        out = torch.empty(B, S, self.hidden, dtype=torch.bfloat16, device=self.device)
        n_rows = 0 if image_feats is None else int(image_feats.shape[0])
        with torch.cuda.device(self.index):
            check(self.lib.b2_splice(self.handle, ptr(src_index), ptr(image_feats), n_rows, B * S, ptr(out), stream_ptr()),
                  "b2_splice")
        return out

    def splice_ids(self, input_ids, k_per_row, feat_rows, image_feats):
        """Device-side splice for equal-length unpadded rows: input_ids int64 [B, Lt] ON THE DEVICE, k_per_row image
        placeholders per row, feat_rows[j] = feature rows of image slot j (row-major slot order). Returns embeds
        [B, S, hidden] with S = Lt - k + sum(feat rows of one row) and no host synchronisation. A wrong placeholder count is
        reported by take_async_error() (ERR_SPLICE_SLOTS) once the stream has run."""
        B, Lt = input_ids.shape
        n_img = len(feat_rows)
        assert n_img == B * k_per_row and input_ids.dtype == torch.int64 and input_ids.is_cuda and input_ids.is_contiguous()
        per_row = [sum(feat_rows[b * k_per_row:(b + 1) * k_per_row]) for b in range(B)]
        assert len(set(per_row)) == 1, "rows must receive the same number of feature rows"
        S = Lt - k_per_row + per_row[0]
        off = (_c.c_int32 * (n_img + 1))(*([0] + [sum(feat_rows[:j + 1]) for j in range(n_img)]))
        out = torch.empty(B, S, self.hidden, dtype=torch.bfloat16, device=self.device)
        with torch.cuda.device(self.index):
            check(self.lib.b2_splice_ids(self.handle, ptr(input_ids), B, Lt, int(k_per_row), off, n_img, ptr(image_feats), S,
                                         ptr(out), stream_ptr()), "b2_splice_ids")
        return out

    def take_async_error(self):
        """Bit mask of the input problems kernels have flagged since the last call (ERR_* below); clears it."""
        code = _c.c_int(0)
        check(self.lib.b2_async_error(self.handle, ctypes.byref(code)), "b2_async_error")
        return code.value

    def check_async_error(self):
        """Raise ValueError if a kernel flagged bad inputs (ids outside the embedding table, image placeholder without
        features). Call after a point where the stream has been synchronised (e.g. once the first token is on the host)."""
        if self.take_async_error():
            raise ValueError(last_error())

    def prefill(self, kv, embeds, seq_lens=None, logits_mode=LOGITS_LAST, slot0=0, start=None):
        """`slot0`: first cache slot to fill (continuous batching); the other slots keep their contents. `start` (list of B
        ints, or None = all 0): cache position where each sample's chunk goes (b2_prefill_at); the cache rows in front of it
        are attended, a start below the slot's current length rewinds it."""
        embeds = self._bf16(embeds)
        B, S = embeds.shape[0], embeds.shape[1]
        lens = pos = None
        if seq_lens is not None:
            lens = (_c.c_int32 * B)(*[int(x) for x in seq_lens])
        if start is not None:
            if len(start) != B:
                raise ValueError(f"start has {len(start)} entries for a batch of {B}")
            pos = (_c.c_int32 * B)(*[int(x) for x in start])
        logits = None
        if logits_mode == LOGITS_LAST:
            logits = torch.empty(B, self.vocab, dtype=torch.float32, device=self.device)
        elif logits_mode == LOGITS_ALL:
            logits = torch.empty(B, S, self.vocab, dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.index):
            check(self.lib.b2_prefill_at(self.handle, kv.handle, ptr(embeds), pos, lens, B, S, int(slot0), ptr(logits), logits_mode,
                                         stream_ptr()), "b2_prefill")
        return logits

    def decode_step(self, kv, tokens, want_logits=True):
        """tokens: int32 tensor [B] (cpu or cuda). Returns fp32 logits [B, vocab] (device)."""
        tokens = tokens.to(torch.int32).contiguous()
        B = tokens.numel()
        logits = torch.empty(B, self.vocab, dtype=torch.float32, device=self.device) if want_logits else None
        with torch.cuda.device(self.index):
            check(self.lib.b2_decode_step(self.handle, kv.handle, ptr(tokens), B, ptr(logits), _vp(0), stream_ptr()),
                  "b2_decode_step")
        return logits

    def decode_greedy(self, kv, first_tokens, n_steps, out=None):
        """Runs n_steps greedy steps on the device (CUDA-graph replay). Returns int32 [n_steps, B];
        `out` may be a pinned CPU tensor to receive the tokens directly."""
        first_tokens = first_tokens.to(torch.int32).contiguous()
        B = first_tokens.numel()
        if out is None:
            out = torch.empty(n_steps, B, dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.index):
            check(self.lib.b2_decode_greedy(self.handle, kv.handle, ptr(first_tokens), B, int(n_steps), ptr(out),
                                            stream_ptr()), "b2_decode_greedy")
        return out

    # -- streaming decode (device runs ahead, host reads tokens from mapped pinned memory) ---------------
    def stream_begin(self, kv, logits, sampling=None, procs=None, out_scores=None, out_logits=None, groups=None, share_prefix=True):
        """Token 0 is chosen from the prefill logits [B, vocab] on the device and published as ring index 0. `procs`: one
        LogitsProc (or None) per row; rows with processors keep their history on the device for the whole generation.
        `out_scores` / `out_logits` (device fp32 [steps, B, vocab], or None): the step that publishes token t writes its score
        row (what selection read: processed, and when sampling divided by T and filtered) and its raw logits row to index t
        (b2_stream_set_outputs). Keep them alive until the generation's steps have run. `groups` ((src_slot, prefix_len, rows)
        triples, see llava/_b2/fork.py): rows that hold copies of one prompt's cache rows, whose decode attention then reads the
        prompt once per group (b2_stream_begin_groups); share_prefix=False runs the same generation with every row reading its
        own copy."""
        logits = logits.contiguous()
        sp = sampling if sampling is not None else make_sampling()
        B = int(logits.shape[0])
        arr = _proc_array(procs, B)
        cap = 0
        for o in (out_scores, out_logits):
            if o is not None:
                if o.dtype != torch.float32 or o.dim() != 3 or tuple(o.shape[1:]) != (B, self.vocab) or not o.is_contiguous():
                    raise ValueError(f"output rows must be contiguous fp32 [steps, {B}, {self.vocab}], got {tuple(o.shape)}")
                cap = int(o.shape[0]) if cap == 0 else min(cap, int(o.shape[0]))
        with torch.cuda.device(self.index):
            # always armed (NULLs included): a begin never inherits buffers a failed call left behind
            check(self.lib.b2_stream_set_outputs(kv.handle, ptr(out_scores), ptr(out_logits), cap), "b2_stream_set_outputs")
            if groups and share_prefix:
                g = _group_array(groups)
                check(self.lib.b2_stream_begin_groups(self.handle, kv.handle, ptr(logits), B, ctypes.byref(sp), arr, g, len(groups),
                                                      stream_ptr()), "b2_stream_begin_groups")
            elif arr is None:
                check(self.lib.b2_stream_begin(self.handle, kv.handle, ptr(logits), B, ctypes.byref(sp), stream_ptr()),
                      "b2_stream_begin")
            else:
                check(self.lib.b2_stream_begin_ex(self.handle, kv.handle, ptr(logits), B, ctypes.byref(sp), arr, stream_ptr()),
                      "b2_stream_begin_ex")

    def stream_begin_lookup(self, kv, logits, sampling, lookup):
        """stream_begin of a batch-1 prompt-lookup generation (`lookup`: make_prompt_lookup); stream_enqueue(n) then queues n
        verify steps, each publishing at least one token."""
        logits = logits.contiguous()
        sp = sampling if sampling is not None else make_sampling()
        with torch.cuda.device(self.index):
            check(self.lib.b2_stream_begin_lookup(self.handle, kv.handle, ptr(logits), int(logits.shape[0]), ctypes.byref(sp),
                                                  ctypes.byref(lookup), stream_ptr()), "b2_stream_begin_lookup")

    def lookup_stats(self, kv):
        """(verify steps, drafted tokens, accepted draft tokens) of the cache's last lookup generation; waits for its steps."""
        out = [_c.c_int32(0) for _ in range(3)]
        with torch.cuda.device(self.index):
            check(self.lib.b2_stream_lookup_stats(kv.handle, *[ctypes.byref(o) for o in out]), "b2_stream_lookup_stats")
        return tuple(int(o.value) for o in out)

    def decode_rows(self, kv, tokens, slot=0):
        """The verify forward: tokens int [R] appended at slot `slot`'s length; returns fp32 logits [R, vocab] (device)."""
        tokens = torch.as_tensor(tokens).to(device=self.device, dtype=torch.int32).contiguous()
        R = tokens.numel()
        logits = torch.empty(R, self.vocab, dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.index):
            check(self.lib.b2_decode_rows(self.handle, kv.handle, int(slot), ptr(tokens), R, ptr(logits), stream_ptr()),
                  "b2_decode_rows")
        return logits

    def batch_begin(self, kv, B):
        with torch.cuda.device(self.index):
            check(self.lib.b2_batch_begin(self.handle, kv.handle, int(B), stream_ptr()), "b2_batch_begin")

    def batch_set_row(self, kv, slot, active, sampling=None, first_token=0, proc=None):
        sp = sampling if sampling is not None else make_sampling()
        with torch.cuda.device(self.index):
            if proc is None:
                check(self.lib.b2_batch_set_row(self.handle, kv.handle, int(slot), int(bool(active)), ctypes.byref(sp),
                                                int(first_token), stream_ptr()), "b2_batch_set_row")
            else:
                check(self.lib.b2_batch_set_row_ex(self.handle, kv.handle, int(slot), int(bool(active)), ctypes.byref(sp),
                                                   ctypes.byref(proc), int(first_token), stream_ptr()), "b2_batch_set_row_ex")

    def stream_enqueue(self, kv, n_steps):
        with torch.cuda.device(self.index):
            check(self.lib.b2_stream_enqueue(self.handle, kv.handle, int(n_steps), stream_ptr()), "b2_stream_enqueue")

    def stream_wait(self, kv, index, B, timeout_ms=60000):
        """Blocks (GIL released by ctypes) until token `index` is visible; returns a list of B ints."""
        out = (_c.c_int32 * B)()
        check(self.lib.b2_stream_wait(kv.handle, int(index), out, int(timeout_ms)), "b2_stream_wait")
        return list(out)

    def sample(self, logits, sampling, index=0, procs=None, want_processed=False):
        """One selection per row of fp32 logits [B, V] with csrc/sampling.cu (greedy or temperature/top-k/top-p). `procs`: one
        LogitsProc (or None) per row, applied over its prompt history first. With want_processed, returns (tokens, the
        processed logits [B, V] before temperature)."""
        logits = logits.to(device=self.device, dtype=torch.float32).contiguous()
        B, V = logits.shape
        out = torch.empty(B, dtype=torch.int32, device=self.device)
        arr = _proc_array(procs, B)
        processed = torch.empty(B, V, dtype=torch.float32, device=self.device) if want_processed else None
        with torch.cuda.device(self.index):
            if arr is None and processed is None:
                check(self.lib.b2_op_sample(ptr(logits), B, V, ctypes.byref(sampling), int(index), ptr(out), stream_ptr()),
                      "b2_op_sample")
            else:
                check(self.lib.b2_op_sample_ex(ptr(logits), B, V, ctypes.byref(sampling), arr, int(index), ptr(out),
                                               None if processed is None else ptr(processed), stream_ptr()), "b2_op_sample_ex")
        return (out, processed) if want_processed else out

    # -- beam search (generate(num_beams > 1); host half in llava/_b2/beam.py) ------------------------------------------------
    def kv_copy_slots(self, kv, src, dst, row_begin=0):
        """Rows [row_begin, len(src[i])) of slot src[i] -> slot dst[i], all layers; afterwards len(dst[i]) == len(src[i])."""
        n = len(src)
        if len(dst) != n:
            raise ValueError(f"{n} sources for {len(dst)} destinations")
        s, d = (_c.c_int32 * max(n, 1))(*src), (_c.c_int32 * max(n, 1))(*dst)
        with torch.cuda.device(self.index):
            check(self.lib.b2_kv_copy_slots(self.handle, kv.handle, s, d, n, int(row_begin), stream_ptr()), "b2_kv_copy_slots")

    def beam_topk(self, logits, beam_scores, nb, K, row_of_beam=None):
        """logits fp32 [rows, V] (device); beam_scores [B*nb]; row_of_beam int [B*nb] or None (identity). Returns device
        tensors (scores fp32, tokens int32, beams int32), each [B, K], best first (b2_op_beam_topk)."""
        V = logits.shape[-1]
        scores = beam_scores.to(device=self.device, dtype=torch.float32).contiguous()
        B = scores.numel() // nb
        rows = None if row_of_beam is None else torch.as_tensor(row_of_beam, dtype=torch.int32).to(self.device).contiguous()
        out_s = torch.empty(B, K, dtype=torch.float32, device=self.device)
        out_t = torch.empty(B, K, dtype=torch.int32, device=self.device)
        out_b = torch.empty(B, K, dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.index):
            check(self.lib.b2_op_beam_topk(ptr(logits), ptr(rows), ptr(scores), B, int(nb), V, int(K), ptr(out_s), ptr(out_t),
                                           ptr(out_b), stream_ptr()), "b2_op_beam_topk")
        return out_s, out_t, out_b

    def beam_sample(self, logits, beam_scores, nb, K, sampling, step, row_of_beam=None):
        """beam_topk with the candidates drawn without replacement (b2_op_beam_sample): `sampling` a BeamSampling, `step` the
        index of the draw. Returns device tensors (scores fp32, tokens int32, beams int32), each [B, K], in draw order."""
        V = logits.shape[-1]
        scores = beam_scores.to(device=self.device, dtype=torch.float32).contiguous()
        B = scores.numel() // nb
        rows = None if row_of_beam is None else torch.as_tensor(row_of_beam, dtype=torch.int32).to(self.device).contiguous()
        out_s = torch.empty(B, K, dtype=torch.float32, device=self.device)
        out_t = torch.empty(B, K, dtype=torch.int32, device=self.device)
        out_b = torch.empty(B, K, dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.index):
            check(self.lib.b2_op_beam_sample(ptr(logits), ptr(rows), ptr(scores), B, int(nb), V, int(K), ctypes.byref(sampling),
                                             int(step), ptr(out_s), ptr(out_t), ptr(out_b), stream_ptr()), "b2_op_beam_sample")
        return out_s, out_t, out_b

    def beam_select_out(self, logits, beam_scores, nb, K, row_scores, row_logits, sampling=None, step=0, row_of_beam=None, fan=1):
        """beam_topk (or beam_sample with `sampling`) that also writes each beam row's score row (log_softmax, warped under
        sampling) and raw logits row to row_scores / row_logits (device fp32 [B*nb*fan, V] or None), `fan` copies per beam
        row (b2_op_beam_select_out)."""
        V = logits.shape[-1]
        scores = beam_scores.to(device=self.device, dtype=torch.float32).contiguous()
        B = scores.numel() // nb
        rows = None if row_of_beam is None else torch.as_tensor(row_of_beam, dtype=torch.int32).to(self.device).contiguous()
        for o in (row_scores, row_logits):
            if o is not None and (o.dtype != torch.float32 or o.numel() != B * nb * fan * V or not o.is_contiguous()):
                raise ValueError(f"output rows must be contiguous fp32 [{B * nb * fan}, {V}]")
        out_s = torch.empty(B, K, dtype=torch.float32, device=self.device)
        out_t = torch.empty(B, K, dtype=torch.int32, device=self.device)
        out_b = torch.empty(B, K, dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.index):
            check(self.lib.b2_op_beam_select_out(ptr(logits), ptr(rows), ptr(scores), B, int(nb), V, int(K),
                                                 None if sampling is None else ctypes.byref(sampling), int(step), int(fan), ptr(out_s),
                                                 ptr(out_t), ptr(out_b), ptr(row_scores), ptr(row_logits), stream_ptr()),
                  "b2_op_beam_select_out")
        return out_s, out_t, out_b

    def beam_select_proc(self, logits, beam_scores, nb, K, procs, row_scores=None, row_logits=None, sampling=None, step=0,
                         row_of_beam=None, fan=1):
        """beam_select_out with logits processors (b2_op_beam_select_proc): `procs` holds one LogitsProc (or None) per logits row,
        processing that row's log-probabilities against its prompt ids. Returns device tensors (scores fp32, tokens int32, beams
        int32), each [B, K]; synchronises."""
        V = logits.shape[-1]
        rows_n = logits.numel() // V
        scores = beam_scores.to(device=self.device, dtype=torch.float32).contiguous()
        B = scores.numel() // nb
        rows = None if row_of_beam is None else torch.as_tensor(row_of_beam, dtype=torch.int32).to(self.device).contiguous()
        for o in (row_scores, row_logits):
            if o is not None and (o.dtype != torch.float32 or o.numel() != B * nb * fan * V or not o.is_contiguous()):
                raise ValueError(f"output rows must be contiguous fp32 [{B * nb * fan}, {V}]")
        arr = _proc_array(procs, rows_n)
        out_s = torch.empty(B, K, dtype=torch.float32, device=self.device)
        out_t = torch.empty(B, K, dtype=torch.int32, device=self.device)
        out_b = torch.empty(B, K, dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.index):
            check(self.lib.b2_op_beam_select_proc(ptr(logits), rows_n, ptr(rows), ptr(scores), B, int(nb), V, int(K),
                                                  None if sampling is None else ctypes.byref(sampling), int(step), int(fan), arr,
                                                  ptr(out_s), ptr(out_t), ptr(out_b), ptr(row_scores), ptr(row_logits), stream_ptr()),
                  "b2_op_beam_select_proc")
        return out_s, out_t, out_b

    def beam_begin_proc(self, kv, procs):
        """Arms the logits processors of a beam search on `kv` (b2_beam_begin_proc): slot b gets procs[b] (LogitsProc or None),
        its history seeded from the prompt ids; b2_beam_step_proc (beam_step_proc) then processes every beam against its slot's
        history."""
        arr = _proc_array(procs, len(procs))
        with torch.cuda.device(self.index):
            check(self.lib.b2_beam_begin_proc(self.handle, kv.handle, len(procs), arr, stream_ptr()), "b2_beam_begin_proc")

    def beam_step_proc(self, kv, copies, row_begin, tokens, slot_of_beam, beam_scores, nb, K, sampling=None, step=0,
                       row_scores=None, row_logits=None):
        """beam_step with the processors armed by beam_begin_proc (b2_beam_step_proc)."""
        return self.beam_step(kv, copies, row_begin, tokens, slot_of_beam, beam_scores, nb, K, sampling, step, row_scores,
                              row_logits, _proc=True)

    def beam_step(self, kv, copies, row_begin, tokens, slot_of_beam, beam_scores, nb, K, sampling=None, step=0, row_scores=None,
                  row_logits=None, _proc=False):
        """One step of the running beams (b2_beam_step, or b2_beam_step_ex with a BeamSampling): `copies` = [(src, dst)] applied
        first, tokens[i] fed to slot slot_of_beam[i], one decode step at batch len(tokens), candidates of every sample selected
        (or, with `sampling`, drawn as draw `step`) on the device. Returns CPU tensors (scores fp32, tokens int64, beams int64),
        each [B, K], best (or first drawn) first. `row_scores` / `row_logits` (device fp32 [len(tokens), V] or None) receive the
        step's score rows and raw logits rows in beam order (b2_beam_step_out)."""
        n = len(tokens)
        B = n // nb
        i32 = lambda xs: (_c.c_int32 * max(len(xs), 1))(*[int(x) for x in xs])
        src, dst = i32([c[0] for c in copies]), i32([c[1] for c in copies])
        toks, slots = i32(tokens), i32(slot_of_beam)
        scores = (_c.c_float * n)(*[float(x) for x in beam_scores])
        out_s = torch.empty(B, K, dtype=torch.float32)
        out_t = torch.empty(B, K, dtype=torch.int32)
        out_b = torch.empty(B, K, dtype=torch.int32)
        a = BeamStepArgs(_c.cast(src, _vp), _c.cast(dst, _vp), len(copies), int(row_begin), B, int(nb), int(K), _c.cast(toks, _vp),
                         _c.cast(slots, _vp), _c.cast(scores, _vp), _vp(out_s.data_ptr()), _vp(out_t.data_ptr()),
                         _vp(out_b.data_ptr()))
        with torch.cuda.device(self.index):
            for o in (row_scores, row_logits):
                if o is not None and (o.dtype != torch.float32 or o.numel() != n * self.vocab or not o.is_contiguous()):
                    raise ValueError(f"output rows must be contiguous fp32 [{n}, {self.vocab}]")
            if _proc:
                check(self.lib.b2_beam_step_proc(self.handle, kv.handle, ctypes.byref(a),
                                                 None if sampling is None else ctypes.byref(sampling), int(step), ptr(row_scores),
                                                 ptr(row_logits), stream_ptr()), "b2_beam_step_proc")
            elif row_scores is not None or row_logits is not None:
                check(self.lib.b2_beam_step_out(self.handle, kv.handle, ctypes.byref(a),
                                                None if sampling is None else ctypes.byref(sampling), int(step), ptr(row_scores),
                                                ptr(row_logits), stream_ptr()), "b2_beam_step_out")
            elif sampling is None:
                check(self.lib.b2_beam_step(self.handle, kv.handle, ctypes.byref(a), stream_ptr()), "b2_beam_step")
            else:
                check(self.lib.b2_beam_step_ex(self.handle, kv.handle, ctypes.byref(a), ctypes.byref(sampling), int(step),
                                               stream_ptr()), "b2_beam_step_ex")
        return out_s, out_t.long(), out_b.long()

    def argmax(self, logits):
        B, V = logits.shape
        out = torch.empty(B, dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.index):
            check(self.lib.b2_argmax(ptr(logits), B, V, ptr(out), stream_ptr()), "b2_argmax")
        return out

    def close(self):
        if getattr(self, "handle", None) is not None and self.handle.value:
            for kv in list(self._kvs):  # caches point into the model: release them first
                kv.close()
            self.lib.b2_model_destroy(self.handle)
            self.handle = _vp(0)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
