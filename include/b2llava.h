/* b2llava.h — C ABI of the H100-native LLaVA multimodal forward path (libb2llava.so).
 *
 * The reference (LLaVA-VL/LLaVA-Plus-Codebase) has NO native boundary on this path: its hot path is a Python
 * class surface (llava/model/language_model/llava_llama.py:56-108, llava/model/llava_arch.py:94-240,
 * llava/model/multimodal_encoder/clip_encoder.py:39-51, llava/model/multimodal_projector/builder.py:33-51)
 * sitting directly on HuggingFace transformers + ATen. This header is the boundary we introduce where
 * HF/ATen sit today (SURVEY.md §8b): each entry point names the reference function whose arithmetic it
 * replaces. The Python package `llava` in this repo binds it with ctypes (see INTEGRATION.md).
 *
 * Conventions
 *   - extern "C", plain pointers and sizes, no C++/torch types. cudaStream_t is passed as void*.
 *   - All tensor pointers are DEVICE pointers unless the parameter name ends in _host or the doc says
 *     "host or device". Activations and weights are bf16 (uint16 storage); logits are fp32.
 *   - Return 0 on success, <0 on error (-1 bad argument, -2 CUDA failure, -3 bad state); the message is
 *     available from b2_last_error() (thread-local). Nothing aborts the process; no exceptions cross the ABI.
 *   - The caller owns every input/output buffer and the stream. The library owns weights (copied and
 *     repacked at set_weight/finalize), workspaces and KV caches.
 *   - A b2_model / b2_kv handle may be used from any host thread, one call at a time (calls lock the handle).
 */
#ifndef B2LLAVA_H_
#define B2LLAVA_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct b2_model b2_model;
typedef struct b2_kv b2_kv;

/* dtype codes for b2_model_set_weight */
enum { B2_DT_BF16 = 0, B2_DT_F16 = 1, B2_DT_F32 = 2 };
/* activation codes for b2_op_gemm */
enum { B2_ACT_NONE = 0, B2_ACT_QUICK_GELU = 1, B2_ACT_GELU_ERF = 2, B2_ACT_SWIGLU = 3 };
/* logits modes for b2_prefill */
enum { B2_LOGITS_NONE = 0, B2_LOGITS_LAST = 1, B2_LOGITS_ALL = 2 };
/* element formats of a KV cache (b2_kv_create_ex) */
enum { B2_KV_BF16 = 0, B2_KV_E4M3 = 1 };

typedef struct b2_model_desc {
    /* CLIP vision tower (transformers CLIPVisionConfig; reference clip_encoder.py:22-27) */
    int32_t image_size;       /* 336 */
    int32_t patch_size;       /* 14 */
    int32_t vit_hidden;       /* 1024 */
    int32_t vit_inter;        /* 4096 */
    int32_t vit_layers;       /* 24 (total in the checkpoint) */
    int32_t vit_heads;        /* 16 (head_dim must be 64) */
    int32_t vit_select_layer; /* -2: hidden_states index, reference clip_encoder.py:30 */
    float vit_ln_eps;         /* 1e-5 */
    /* LLaMA decoder (LlavaConfig(LlamaConfig), reference llava_llama.py:29-30) */
    int32_t hidden;           /* 4096 | 5120 */
    int32_t inter;            /* 11008 | 13824 */
    int32_t layers;           /* 32 | 40 */
    int32_t heads;            /* 32 | 40 (head_dim must be 128; kv_heads == heads) */
    int32_t vocab;            /* 32000 */
    float rms_eps;            /* 1e-5 */
    float rope_theta;         /* 10000 */
    /* workspace sizing */
    int32_t max_batch;        /* largest B for prefill/decode */
    int32_t max_seq;          /* largest spliced prefill length S (B*S rows of workspace) */
    int32_t max_images;       /* images encoded per ViT pass (larger batches are chunked) */
} b2_model_desc;

/* Token selection of the decode loop (HF GenerationMixin as the reference calls it: llava/serve/model_worker.py:155-185
 * passes do_sample / temperature / top_p; top_k comes from the GenerationConfig default). do_sample == 0 -> greedy argmax. */
typedef struct b2_sampling {
    int32_t do_sample;
    float temperature;        /* > 0 */
    float top_p;              /* (0, 1]; 1 = off */
    int32_t top_k;            /* 0 = off */
    unsigned long long seed;  /* Philox key; draw t of row b is a pure function of (logits, seed, t, b) */
} b2_sampling;

/* History-aware logits processing of one row, applied before token selection in HF 5.5's order (GenerationMixin
 * _get_logits_processor): repetition penalty -> no-repeat n-gram -> min_length / min_new_tokens -> temperature -> top-k -> top-p.
 * The row's history is prompt_ids[0, prompt_len) (device int64, the caller's prompt row as passed, IMAGE_TOKEN_INDEX
 * placeholders and pad ids included) followed by the tokens generated so far.
 *   repetition_penalty  p > 0, 1 = off: every distinct history id in [0, vocab) gets x < 0 ? x * p : x / p (IEEE fp32)
 *   no_repeat_ngram_size n >= 0, 0 = off: every history n-gram whose first n-1 ids equal the last n-1 ids bans its last id
 *                        (-inf) unless that id is outside [0, vocab); nothing is banned while history length + 1 < n
 *   min_generated        eos_ids[0, n_eos) get -inf while fewer than min_generated tokens were generated
 *                        (max(min_new_tokens, min_length - prompt_len) for HF's two processors); no effect with n_eos == 0
 * A row with every processor off is selected exactly as without this struct. The pointed-to ids are read by the call's
 * stream work only (they must stay valid until it has run). */
typedef struct b2_logits_proc {
    float repetition_penalty;
    int32_t no_repeat_ngram_size;
    int32_t min_generated;
    int32_t n_eos;               /* 0..8 */
    int32_t eos_ids[8];
    const int64_t* prompt_ids;   /* device */
    int32_t prompt_len;
} b2_logits_proc;

/* ---- lifecycle ------------------------------------------------------------------------------------------ */
int b2_init(int device);                 /* cudaSetDevice + capability check (needs sm_90) */
const char* b2_last_error(void);         /* thread-local message of the last failing call */
int b2_version(void);
unsigned long long b2_launch_count(void);/* number of kernels this library has launched (bench.py gpu_launches) */

int b2_model_create(const b2_model_desc* desc, b2_model** out);
/* Copy one checkpoint tensor into the model. `hf_key` uses the reference's state-dict names (SURVEY.md §5):
 * model.embed_tokens.weight, model.layers.{i}.self_attn.{q,k,v,o}_proj.weight,
 * model.layers.{i}.mlp.{gate,up,down}_proj.weight, model.layers.{i}.{input,post_attention}_layernorm.weight,
 * model.norm.weight, lm_head.weight, model.mm_projector.{0,2}.{weight,bias},
 * [model.vision_tower.vision_tower.]vision_model.* (CLIPVisionModel names). `ptr` may be host or device memory,
 * borrowed for the duration of the call. q/k/v are fused into one [3h,h] matrix, gate/up are block-64
 * interleaved for the fused SwiGLU epilogue. Unknown keys return -1; keys that are dead on this path
 * (vision post_layernorm, CLIP layers above the selected one, rotary inv_freq buffers) are accepted and ignored. */
int b2_model_set_weight(b2_model* m, const char* hf_key, const void* ptr, const int64_t* shape, int ndim, int dtype);
int b2_model_finalize(b2_model* m);      /* checks every tensor arrived, allocates workspaces */
int b2_model_destroy(b2_model* m);
/* BASELINE configs[4] ("fp8-weight path"): after finalize, quantise the decoder's Linear weights to e4m3 with one
 * fp32 scale per output channel; decode steps at batch >= 7 then run e4m3 x e4m3 wgmma GEMMs (activations quantised
 * per token on the fly; the KV cache format is a separate choice, b2_kv_create_ex). Prefill and small-batch decode keep the bf16 weights. The reference has no
 * fp8 path; oracle/fp8_oracle.py defines the arithmetic and the tolerance (tests/test_fp8_gpu.py). Off unless this call is
 * made: it changes the numerics of the decode step (W8A8), so it is never a default. */
int b2_model_enable_fp8_decode(b2_model* m);
/* load_4bit (reference llava/model/builder.py:26-41, bitsandbytes NF4): after finalize, quantise the seven decoder Linears
 * of every layer to NF4 (per row, one fp32 absmax per 64-element block, 4-bit codes into the NF4 table; oracle/nf4_oracle.py
 * defines the arithmetic) and free their bf16 buffers; replace both mm_projector weights in place by their dequantised
 * values w_hat = bf16(code * absmax). Decode at batch <= 8 then streams the 4-bit weights (gemv_nf4, whose activation tile
 * must fit shared memory: 13B shapes at batch 5..8 do not); prefill and the other decode batches dequantise one layer at a
 * time into a bf16 scratch and run the dense kernels over it. The CLIP tower,
 * embed_tokens, lm_head and the norms stay bf16. Returns -1 when the model is not finalized, when
 * b2_model_enable_fp8_decode has run, or when a KV cache of this model exists; a second call is a no-op. Afterwards
 * b2_model_enable_fp8_decode and b2_model_set_weight on a decoder Linear or projector weight return -1. */
int b2_model_enable_nf4(b2_model* m);
/* device bytes of the weights the model holds (bf16, e4m3 and NF4 copies with their scales; workspaces excluded) */
int64_t b2_model_weight_bytes(b2_model* m);

int b2_kv_create(b2_model* m, int max_batch, int max_seq, b2_kv** out); /* KV cache [L][2][B][H][Smax][128] bf16 */
/* b2_kv_create with the element format chosen per cache; b2_kv_create == kv_dtype B2_KV_BF16. B2_KV_E4M3 stores K and V as e4m3
 * bytes, [L][B][H][Smax][128], with one fp32 scale per (layer, sample, head, token) for K and one for V, [L][B][H][Smax]: 264
 * bytes per head-token instead of 512 (Smax is rounded up to a multiple of 4 inside). A row's scale is amax / 448 over its 128
 * elements (1 for a zero row) and q = e4m3_rn_satfinite(x / scale), the rule of b2_op_quantize_rows_e4m3; K is quantised after
 * RoPE. Prefill attends over the unquantised bf16 K / V of its own tokens, so its logits are bit-identical to a bf16 cache's;
 * only what it stores is quantised. Every decode step attends over what is stored, the token it appends included: scores
 * and softmax in fp32, score = (q . k_q) * k_scale / sqrt(128), o += p * v_scale * v_q. oracle/kv_fp8_oracle.py defines the
 * arithmetic and the tolerance (tests/test_kv_fp8_gpu.py). It changes the numerics of decode, so it is never a default. Decode
 * on an e4m3 cache runs the multi-kernel step at every batch size (the batch <= 8 megakernel reads bf16 caches only): at
 * small batch the cache is a few percent of a step's bytes, so there the format buys capacity, not speed. Works with bf16 and
 * e4m3 weights, b2_prefill_slots, the streaming calls and continuous batching. Unknown kv_dtype: -1. */
int b2_kv_create_ex(b2_model* m, int max_batch, int max_seq, int kv_dtype, b2_kv** out);
int b2_kv_dtype(b2_kv* kv);              /* B2_KV_BF16 | B2_KV_E4M3 */
int64_t b2_kv_bytes(b2_kv* kv);          /* device bytes of K, V and their scale arrays */
int b2_kv_reset(b2_kv* kv);
int b2_kv_destroy(b2_kv* kv);
int b2_kv_lengths(b2_kv* kv, int32_t* lens_host, int n);  /* current cache length per sample */

/* ---- hot path ------------------------------------------------------------------------------------------- */
/* CLIPVisionTower.forward + feature_select (reference clip_encoder.py:29-51; HF modeling_clip.py:202-217,
 * 300-384, 667-691): pixels [B,3,img,img] bf16 -> patch features [B, P, vit_hidden] bf16 of
 * hidden_states[vit_select_layer] with the CLS token dropped. Layers above the selected one are not computed. */
int b2_vit_encode(b2_model* m, const void* pixels, int B, void* out_feats, void* stream);
/* mm_projector mlp2x_gelu (reference multimodal_projector/builder.py:39-46): [rows, vit_hidden] -> [rows, hidden] */
int b2_project(b2_model* m, const void* feats, int rows, void* out, void* stream);
/* LlavaMetaForCausalLM.encode_images (reference llava_arch.py:94-97) = b2_vit_encode then b2_project:
 * pixels [B,3,img,img] -> [B, P, hidden] */
int b2_encode_images(b2_model* m, const void* pixels, int B, void* out, void* stream);
/* The device half of prepare_inputs_labels_for_multimodal (reference llava_arch.py:150-225). src_index[r]
 * (device int32, one per output row of the padded [B,S] layout) is: >= 0 -> embed_tokens row (token id);
 * < 0 and != INT32_MIN -> row (-src-1) of image_feats [n_img*P, hidden]; INT32_MIN -> zero row (padding).
 * The index is built on the host from input_ids (llava/model/llava_arch.py in this repo). image_feats holds n_feat_rows
 * rows (0 with a NULL pointer for text-only batches). An index outside the embedding table or the feature rows never reads
 * out of bounds: the row is zero-filled and the problem is reported by b2_async_error(). */
int b2_splice(b2_model* m, const int32_t* src_index, const void* image_feats, int n_feat_rows, int rows, void* embeds_out,
              void* stream);
/* The whole splice on the device, for the layout every generation caller of the reference uses (equal-length rows without
 * padding, k_per_row IMAGE_TOKEN_INDEX placeholders per row; llava/serve/model_worker.py:163, llava/eval/model_vqa_loader.py:98):
 * input_ids int64 [B,Lt] stays on the device (no D2H of the ids, no host loop over rows — reference llava_arch.py:143-187);
 * image slot j holds feature rows [feat_offsets_host[j], feat_offsets_host[j+1]) of image_feats, slots are consumed in
 * row-major order. The caller derives S = Lt - k + rows-per-row from shapes alone. A row whose placeholder count is not
 * k_per_row is flagged (b2_async_error code 4) and the caller redoes the splice on the exact host path (b2_splice). */
int b2_splice_ids(b2_model* m, const int64_t* input_ids, int B, int Lt, int k_per_row, const int32_t* feat_offsets_host, int n_img,
                  const void* image_feats, int S, void* embeds_out, void* stream);
/* Input problems that only a kernel can see (ids live on the device): returns in *code_out the OR of 1 = token id outside
 * [0, vocab) or an image placeholder without features, 2 = image-feature row out of range, 4 = more placeholders than
 * images, accumulated since the last call, and clears it. Meaningful after the stream has been synchronised (the codes
 * are written to mapped host memory by the kernels); b2_last_error() then holds the text. */
int b2_async_error(b2_model* m, int* code_out);
/* LlamaModel.forward prefill over inputs_embeds [B,S,hidden] (HF modeling_llama.py:375-425 and :303-332 per
 * layer), right-padded rows with seq_lens_host[b] valid tokens (NULL => all S). Fills the KV cache from
 * position 0 (b2_prefill_at: from a given position). logits_out: B2_LOGITS_LAST -> fp32 [B,vocab] at each sample's last valid position;
 * B2_LOGITS_ALL -> fp32 [B,S,vocab] (the reference's lm_head over all positions, llava_llama.py:88-99). */
int b2_prefill(b2_model* m, b2_kv* kv, const void* embeds, const int32_t* seq_lens_host, int B, int S,
               void* logits_out, int logits_mode, void* stream);
/* b2_prefill into the cache slots [slot0, slot0 + B) — the other slots of the cache are not touched (continuous batching:
 * a new request is prefilled while the rest of the batch keeps its context). b2_prefill == slot0 0. */
int b2_prefill_slots(b2_model* m, b2_kv* kv, const void* embeds, const int32_t* seq_lens_host, int B, int S, int slot0,
                     void* logits_out, int logits_mode, void* stream);
/* Prefill of a chunk appended at a given cache position (multi-turn chat: the turn's new tokens behind the conversation
 * already in the cache). Sample b's S-row chunk (seq_lens_host[b] valid tokens, NULL => all S) goes to positions
 * start_host[b] .. start_host[b] + len - 1 of slot slot0 + b: RoPE at those positions, attention over the cache rows
 * [0, start_host[b]) plus the chunk itself (causal). Needs start_host[b] <= the slot's current length (a smaller start rewinds
 * the slot) and start_host[b] + len <= max_seq; afterwards the slot's length is start_host[b] + len. logits_out as in
 * b2_prefill, over the chunk's positions. start_host NULL (or all zeros) is b2_prefill_slots. On an e4m3 cache the chunk
 * attends over the stored prefix as bf16(q * scale) and its own unquantised K / V, and stores only its own rows. */
int b2_prefill_at(b2_model* m, b2_kv* kv, const void* embeds, const int32_t* start_host, const int32_t* seq_lens_host, int B,
                  int S, int slot0, void* logits_out, int logits_mode, void* stream);
/* One autoregressive step (reference decode branch llava_arch.py:103-112 + HF one-token forward): tokens [B]
 * int32 (host or device) are embedded, run through the decoder against the cache (appending one K/V row per
 * layer), logits_out fp32 [B,vocab] (nullable), next_tokens_out int32 [B] = argmax (nullable, host or device). */
int b2_decode_step(b2_model* m, b2_kv* kv, const int32_t* tokens, int B, void* logits_out, int32_t* next_tokens_out,
                   void* stream);
/* n_steps greedy steps with device-resident token feedback, replayed from a CUDA graph (no host sync between
 * steps): the decode half of HF generate() greedy search as invoked by the reference (model_worker.py:174-185).
 * first_tokens [B] (host or device) is the token fed to step 0; out_tokens [n_steps,B] (host or device) receives
 * the token produced by every step. */
int b2_decode_greedy(b2_model* m, b2_kv* kv, const int32_t* first_tokens, int B, int n_steps, int32_t* out_tokens,
                     void* stream);
int b2_argmax(const float* logits, int B, int V, int32_t* out, void* stream);

/* Streaming decode — what generate() needs when somebody watches every token (the reference always passes a streamer and a
 * stopping criterion: llava/serve/model_worker.py:166-188, llava/serve/cli.py:91-102). The device loop is the same as
 * b2_decode_greedy (token feedback stays on the device, argmax or the temperature/top-k/top-p draw is a kernel), but every
 * step also publishes its token into a ring in mapped pinned host memory, tagged with the generation's epoch, so the host
 * reads token t while step t+k is already running: no D2H copy and no stream synchronisation per token.
 *   b2_stream_begin   selects token 0 from `logits` (device fp32 [B,vocab], the prefill's last-position logits) and
 *                     publishes it as index 0;
 *   b2_stream_enqueue queues n_steps more decode steps (token indices continue from the last one scheduled);
 *   b2_stream_wait    blocks until token `index` is visible and copies it to tokens_host[B] (host). Takes no lock;
 *                     timeout_ms <= 0 waits forever; -3 on timeout, -2 if the device faulted.
 * Steps that were queued past the point where the host decides to stop simply run to completion (rows never interact). */
int b2_stream_begin(b2_model* m, b2_kv* kv, const float* logits, int B, const b2_sampling* sampling, void* stream);
/* b2_stream_begin with logits processors: proc[b] (nullable = all off) for sample b. Token 0 is chosen from the processed
 * prefill logits over the prompt history; every later step of the generation processes against the history kept on the
 * device (prompt, then each chosen token). The cache's processing state is allocated by the first call that turns a processor
 * on (b2_kv_bytes does not count it). b2_stream_begin, b2_batch_begin, b2_decode_step, b2_decode_greedy and b2_beam_step turn
 * every row's processors off, and disarm the processing of a beam search (b2_beam_begin_proc). -1 for repetition_penalty <= 0, a negative n-gram size, n_eos outside [0, 8] or a prompt longer
 * than the cache's max_seq. */
int b2_stream_begin_ex(b2_model* m, b2_kv* kv, const float* logits, int B, const b2_sampling* sampling, const b2_logits_proc* proc,
                       void* stream);
/* Shared-prefix decode of forked samples (generate(num_return_sequences=n)): rows that hold copies of one prompt's cache rows
 * (b2_kv_copy_slots) form a group, and while the group table is armed the decode attention reads keys [0, prefix_len) of every
 * row of a group once, from the group's source slot, instead of once per row from the row's own copy. The result is the one the
 * rows' own copies give, up to the order of floating-point sums.
 *   src_slot    the slot whose rows [0, prefix_len) the group's rows read;
 *   prefix_len  1 <= prefix_len <= the current length of src_slot and of every member row;
 *   rows        n_rows (1..16) rows of the batch; a row belongs to at most one group, and rows outside every group attend their
 *               own slot only. Split more than 16 rows of a prompt into several groups naming the same source. */
typedef struct {
    int32_t src_slot;
    int32_t prefix_len;
    int32_t n_rows;
    int32_t rows[16];
} b2_prefix_group;
/* b2_stream_begin_ex that also arms `groups[0..G)` (G in 1..B, src_slot < B) for the decode steps of this generation. -1 (nothing
 * queued) for a table that breaks the rules above. The table's device state is allocated by the first call (b2_kv_bytes does not
 * count it). Only the multi-kernel decode step over a bf16 cache reads the table: the megakernel (batch <= 2) and an e4m3
 * cache read every row's own copy. Every other call that begins a generation or decodes on the cache (b2_stream_begin*,
 * b2_stream_begin_lookup, b2_batch_begin, b2_decode_step, b2_decode_greedy, b2_decode_rows, b2_beam_step*) and b2_kv_reset
 * disarm it. Arming or disarming drops the cache's captured decode graph. */
int b2_stream_begin_groups(b2_model* m, b2_kv* kv, const float* logits, int B, const b2_sampling* sampling, const b2_logits_proc* proc,
                           const b2_prefix_group* groups, int G, void* stream);
int b2_stream_enqueue(b2_model* m, b2_kv* kv, int n_steps, void* stream);
int b2_stream_wait(b2_kv* kv, int index, int32_t* tokens_host, int timeout_ms);
/* Score and logits rows of a streaming generation (generate(output_scores / output_logits, return_dict_in_generate)).
 *   b2_stream_set_outputs  arms device fp32 buffers [cap_steps][B][vocab] (either nullable; both NULL disarms) for the next
 *                          b2_stream_begin / b2_stream_begin_ex on this cache, which takes them over whether or not it succeeds.
 *                          The step that publishes token t of that generation writes row t = [B][vocab] of each: `logits` gets
 *                          the raw fp32 logits it selected from, `scores` the row HF hands to selection: the logits after the
 *                          processors, and when sampling x / T (IEEE division) with the tokens the top-k / top-p filters remove
 *                          at -inf. Token 0 is written by the begin, from the prefill logits. Steps queued past cap_steps write
 *                          nothing. The buffers are written by every step of the generation on the stream the steps run on, so
 *                          they must stay allocated until the steps queued for it have run (b2_stream_enqueue orders them before
 *                          later work on the caller's stream) and until the next call that begins a generation or decodes on the
 *                          cache (b2_stream_begin*, b2_batch_begin, b2_decode_step, b2_decode_greedy, b2_beam_step*). A finished
 *                          row keeps decoding its own tokens, so its rows after its eos are not HF's. b2_stream_begin_lookup and
 *                          b2_batch_begin return -1 while buffers are armed. */
int b2_stream_set_outputs(b2_kv* kv, float* scores, float* logits, int cap_steps);

/* Prompt-lookup speculative decoding of one sample (HF generate(prompt_lookup_num_tokens=K, max_matching_ngram_size=n): the draft is
 * copied from the conversation itself). Every step drafts up to K tokens from the history on the device (the prompt ids, then the
 * published tokens), runs the pending token and the draft as K + 1 rows of one forward over the weights, and accepts the draft's
 * leading tokens that equal the tokens selected at the rows before them, plus the token selected after the last match. Row j of
 * a step is selected (greedy, or the temperature / top-k / top-p draw) as token index t0 + j of the generation, keyed as plain
 * streaming keys it, so greedy output equals plain decoding's up to the logits' numerics.
 *   b2_stream_begin_lookup  b2_stream_begin for B == 1 on a bf16 cache. Afterwards b2_stream_enqueue(n) keeps n verify steps in
 *                           flight: it queues as many as the device has not yet retired below n (read from mapped host memory, no
 *                           synchronisation), and none once the generation's max_new_tokens are published. Every step publishes at
 *                           least one token, so token `index` may be waited for (b2_stream_wait) once index < published + steps in
 *                           flight; a host that calls b2_stream_enqueue(n >= 1) before each b2_stream_wait always may. b2_kv_lengths
 *                           then reports an upper bound of the cache length. -1 for B != 1, an e4m3 cache, num_tokens outside
 *                           1..15, max_ngram or max_new_tokens < 1, n_eos outside 0..8, or prompt_len (or the cache length) +
 *                           max_new_tokens + num_tokens > max_seq. Logits processors cannot be combined with it.
 *   b2_stream_lookup_stats  the generation's steps that published tokens, the tokens they drafted and the draft tokens accepted
 *                           (host int32, nullable), as of the last step the device has finished; it does not wait (synchronise the
 *                           stream first for the final counts).
 *   b2_decode_rows          the verify forward alone: tokens [R] (host or device, R in 1..16) are appended at slot `slot`'s length
 *                           (bf16 cache), its length advances by R, logits_out (nullable, host or device) receives fp32 [R, vocab].
 *                           Rewind with b2_prefill_at's start. */
typedef struct b2_prompt_lookup {
    int32_t num_tokens;          /* K: draft tokens per step, 1..15 */
    int32_t max_ngram;           /* max_matching_ngram_size, >= 1 */
    int32_t max_new_tokens;      /* the generation publishes at most this many tokens */
    int32_t n_eos;               /* 0..8: a draft ends before the first eos id */
    int32_t eos_ids[8];
    const int64_t* prompt_ids;   /* device, the prompt row as passed (IMAGE_TOKEN_INDEX placeholders end a draft) */
    int32_t prompt_len;
} b2_prompt_lookup;
int b2_stream_begin_lookup(b2_model* m, b2_kv* kv, const float* logits, int B, const b2_sampling* sampling, const b2_prompt_lookup* lookup,
                           void* stream);
int b2_stream_lookup_stats(b2_kv* kv, int32_t* steps, int32_t* drafted, int32_t* accepted);
int b2_decode_rows(b2_model* m, b2_kv* kv, int slot, const int32_t* tokens, int R, float* logits_out, void* stream);

/* Continuous batching (SURVEY §8f-4: the reference's worker runs up to limit_model_concurrency generate() threads on one
 * model, llava/serve/model_worker.py:230-243, each a batch-1 HF loop; here they share ONE batched decode step). The B slots of
 * a cache are a pool: b2_batch_begin puts the cache in per-slot mode (every slot idle, streaming ring armed);
 * b2_prefill_slots fills one slot; b2_batch_set_row(active=1) arms it with its own sampling parameters and the token chosen
 * from its prefill logits; b2_stream_enqueue(n) then advances ALL slots by n steps in one batched step each (idle slots keep
 * their length and are ignored) and b2_stream_wait hands the step's B tokens to the host; b2_batch_set_row(active=0) frees a
 * slot. Token selection is per slot: greedy or temperature/top-k/top-p with the slot's own Philox stream. */
int b2_batch_begin(b2_model* m, b2_kv* kv, int B, void* stream);
int b2_batch_set_row(b2_model* m, b2_kv* kv, int slot, int active, const b2_sampling* sampling, int first_token, void* stream);
/* b2_batch_set_row with the slot's logits processors (nullable = off): its history is proc's prompt ids followed by first_token
 * (chosen by the caller, e.g. with b2_op_sample_ex over the same prompt). A freed slot's processors are turned off. */
int b2_batch_set_row_ex(b2_model* m, b2_kv* kv, int slot, int active, const b2_sampling* sampling, const b2_logits_proc* proc,
                        int first_token, void* stream);

/* Beam search (generate(num_beams > 1): HF GenerationMixin._beam_search of the installed transformers 5.5, as the reference's eval
 * scripts call it with --num_beams, llava/eval/run_llava.py:121,153). The B*nb running beams of B samples live in cache slots;
 * the host (llava/_b2/beam.py) keeps the beam -> slot map and decides which slot becomes a copy of which after every step.
 *   b2_kv_copy_slots   for each i, rows [row_begin, len(src_host[i])) of every layer's K and V (bytes and fp32 scales on an e4m3
 *                      cache) are copied from slot src_host[i] to slot dst_host[i], and len(dst) := len(src). Rows below
 *                      row_begin of dst are not touched. -1 when a dst is also a src of the call, a dst repeats, a slot is out
 *                      of range or row_begin > len(src).
 *   b2_op_beam_topk    per sample b, the K best continuations (score, token, beam) among nb beams x V tokens, where
 *                      score = log_softmax(logits[row_of_beam[b*nb + j]]) + beam_scores[b*nb + j] in fp32 over the raw logits,
 *                      sorted by score descending; equal scores go to the lower beam * V + token. NaN logits rank below -inf.
 *                      row_of_beam (device int32 [B*nb]) may be NULL (= identity); beam_scores device fp32 [B*nb]; outputs
 *                      device [B, K] (beam = index within the sample). nb <= 32, K <= 128, K <= nb * V.
 *   b2_beam_step       one step of the running beams: the copies, then tokens_host[i] is fed to slot slot_of_beam_host[i]
 *                      (every slot [0, B*nb) of the cache must hold one beam), one decode step at batch B*nb (the same path
 *                      b2_decode_step takes), then b2_op_beam_topk over its logits with row_of_beam = slot_of_beam_host and
 *                      the running scores, candidates written to the host arrays; returns after one stream synchronisation. */
typedef struct b2_beam_step_args {
    const int32_t* copy_src_host;     /* [n_copies] */
    const int32_t* copy_dst_host;     /* [n_copies] */
    int32_t n_copies;
    int32_t row_begin;                /* first cache row the copies move (rows below are shared, e.g. the prompt) */
    int32_t B, nb, K;
    const int32_t* tokens_host;       /* [B*nb] token fed to running beam i (sample i / nb) */
    const int32_t* slot_of_beam_host; /* [B*nb] cache slot of running beam i (after the copies) */
    const float* beam_scores_host;    /* [B*nb] running score of beam i */
    float* out_scores_host;           /* [B*K] */
    int32_t* out_tokens_host;         /* [B*K] */
    int32_t* out_beams_host;          /* [B*K] beam index within the sample */
} b2_beam_step_args;
int b2_kv_copy_slots(b2_model* m, b2_kv* kv, const int32_t* src_host, const int32_t* dst_host, int n, int row_begin, void* stream);
int b2_op_beam_topk(const float* logits, const int32_t* row_of_beam, const float* beam_scores, int B, int nb, int V, int K,
                    float* out_scores, int32_t* out_tokens, int32_t* out_beams, void* stream);
int b2_beam_step(b2_model* m, b2_kv* kv, const b2_beam_step_args* args, void* stream);

/* Beam sampling (generate(do_sample=True, num_beams > 1): HF 5.5 _beam_search with do_sample). The candidates of a sample are
 * drawn without replacement instead of taken best first:
 *   b2_op_beam_sample  per beam row, w = log_softmax(logits[row_of_beam[b*nb + j]]) / temperature (fp32: ((x - max) - lse) / T),
 *                      then top-k (ties kept) and top-p over w, each keeping at least min_keep tokens, the others -inf; the
 *                      accumulated score acc = w + beam_scores[b*nb + j]; every finite acc gets the key fp32(acc + g) with
 *                      g = -log(-log u) in fp64 and u = ((r >> 11) + 0.5) * 2^-53, r = Philox4x32-10(seed; step,
 *                      (b*nb + j) * V + token). Per sample the K largest keys are returned in key order, each with its
 *                      unperturbed acc as the score: torch.multinomial(softmax(acc), K) in distribution and in draw order.
 *                      -inf candidates rank below every finite key by lower beam * V + token, NaN logits below them
 *                      (a NaN logit stays NaN through the warpers, score NaN).
 *                      Arguments as b2_op_beam_topk, plus temperature > 0, top_k >= 0 (0 = off), top_p in (0, 1] (1 = off),
 *                      1 <= min_keep <= K, B * nb * V <= 2^32.
 *   b2_beam_step_ex    b2_beam_step whose candidates come from b2_op_beam_sample at `step` (NULL sampling = b2_beam_step). */
typedef struct b2_beam_sampling {
    float temperature;
    int32_t top_k;
    float top_p;
    int32_t min_keep;         /* HF: 1 + number of eos ids, 2 when there are none */
    unsigned long long seed;
} b2_beam_sampling;
int b2_op_beam_sample(const float* logits, const int32_t* row_of_beam, const float* beam_scores, int B, int nb, int V, int K,
                      const b2_beam_sampling* sampling, uint32_t step, float* out_scores, int32_t* out_tokens, int32_t* out_beams,
                      void* stream);
int b2_beam_step_ex(b2_model* m, b2_kv* kv, const b2_beam_step_args* args, const b2_beam_sampling* sampling, uint32_t step,
                    void* stream);
/* Score and logits rows of beam search (generate(output_scores / output_logits, return_dict_in_generate) with num_beams > 1).
 *   b2_op_beam_select_out  b2_op_beam_topk (sampling NULL) or b2_op_beam_sample that also writes, for every beam row
 *                          i = b*nb + j it reads, its score row to row_scores[(i*fan + r) * vocab ...] and the raw logits row to
 *                          row_logits[...] for r < fan (device fp32, either nullable). The score row is log_softmax of the logits
 *                          (fp32, ((x - max) - lse)), under sampling warped as b2_op_beam_sample warps it, -inf outside the
 *                          survivors. fan > 1 (1..32, greedy only) fills the nb running rows of a sample from its one prefill row
 *                          (nb = 1, fan = num_beams), as HF's first step of beam search has nb equal rows.
 *   b2_beam_step_out       b2_beam_step_ex that writes the step's rows, [B*nb][vocab] in running-beam order (beam i reads the
 *                          logits of slot slot_of_beam_host[i]), to row_scores / row_logits (device, nullable). */
int b2_op_beam_select_out(const float* logits, const int32_t* row_of_beam, const float* beam_scores, int B, int nb, int V, int K,
                          const b2_beam_sampling* sampling, uint32_t step, int fan, float* out_scores, int32_t* out_tokens,
                          int32_t* out_beams, float* row_scores, float* row_logits, void* stream);
int b2_beam_step_out(b2_model* m, b2_kv* kv, const b2_beam_step_args* args, const b2_beam_sampling* sampling, uint32_t step,
                     float* row_scores, float* row_logits, void* stream);

/* Logits processors in beam search (generate(num_beams > 1, repetition_penalty / no_repeat_ngram_size / min_new_tokens /
 * min_length): HF 5.5 _beam_search runs them over each running beam's log_softmax row against that beam's own sequence, before the
 * running score is added and, under beam sampling, before temperature / top-k / top-p). The processors of b2_logits_proc act on
 * the fp32 log-probabilities ((x - max) - lse): a penalised history id's score is multiplied by p when negative; a log-prob of
 * exactly 0 stays 0. The score rows written (row_scores) are the processed rows (warped under sampling).
 *   b2_op_beam_select_proc  b2_op_beam_select_out over `rows` logits rows, where logits row r is processed against the history
 *                           proc[r].prompt_ids (proc: [rows] structs, NULL = every row off; row_of_beam NULL needs rows == B*nb).
 *                           Every beam row that reads logits row r (fan, row_of_beam) sees the same processed row. With every
 *                           processor off, candidates and rows are those of b2_op_beam_select_out. Synchronises the stream.
 *   b2_beam_begin_proc      arms the processing of a beam search on the cache: slot b < B gets proc[b] (NULL entry or NULL
 *                           array = off) with its history seeded from proc[b]'s prompt ids; every other slot is off. Call it after
 *                           the prompts are prefilled into slots 0..B-1, before the first b2_beam_step_proc.
 *   b2_beam_step_proc       b2_beam_step_out with the armed processing: a copy moves the source slot's history (ids, presence
 *                           bitmap and counters) with its K/V rows; then tokens_host[i] joins the history of slot
 *                           slot_of_beam_host[i], and beam i's log_softmax row is processed against that history before selection.
 *                           The decode step inside neither processes nor appends. One more kernel launch than b2_beam_step_out
 *                           (the tokens to the device), plus one per 64 copies when the step copies slots.
 * -1 (nothing queued) for the checks of b2_stream_begin_ex on a processor, and from b2_beam_step_proc on a cache where the
 * processing is not armed. The calls that turn every row's processors off (see b2_stream_begin_ex) disarm it. */
int b2_op_beam_select_proc(const float* logits, int rows, const int32_t* row_of_beam, const float* beam_scores, int B, int nb, int V,
                           int K, const b2_beam_sampling* sampling, uint32_t step, int fan, const b2_logits_proc* proc, float* out_scores,
                           int32_t* out_tokens, int32_t* out_beams, float* row_scores, float* row_logits, void* stream);
int b2_beam_begin_proc(b2_model* m, b2_kv* kv, int B, const b2_logits_proc* proc, void* stream);
int b2_beam_step_proc(b2_model* m, b2_kv* kv, const b2_beam_step_args* args, const b2_beam_sampling* sampling, uint32_t step,
                      float* row_scores, float* row_logits, void* stream);

/* ---- single-kernel entry points (unit-level parity tests; same kernels the hot path launches) ----------- */
int b2_op_gemm(const void* A, int lda, const void* W, int ldw, const void* bias, const void* residual, int ld_res,
               void* out, int ld_out, int out_fp32, int M, int N, int K, int act, int bn_override, void* stream);
int b2_op_gemv(const void* x, int64_t ldx, const void* W, int ldw, const void* norm_gamma, float eps,
               const void* residual, int ld_res, void* out, int ld_out, int out_fp32, int B, int N, int K, int act,
               void* stream);
/* NF4 (b2_model_enable_nf4). Canonical layout: codes [N, K/2] bytes, element 2j in the high nibble of byte j; absmax
 * [N, K/64] fp32. quantize: w bf16 [N, K] contiguous, K % 64 == 0. dequantize: out bf16 [N, K] = w_hat. */
int b2_op_quantize_nf4(const void* w, int N, int K, void* codes, float* absmax, void* stream);
int b2_op_dequantize_nf4(const void* codes, const float* absmax, int N, int K, void* out, void* stream);
/* b2_op_gemv over NF4 weights: codes in the GEMV order (oracle/nf4_oracle.py pack_nf4(order="gemv")), absmax [N, K/64];
 * K % 128 == 0, bf16 output; out = (rmsnorm(x) | x) . w_hat^T (+ residual), or SwiGLU over block-64 interleaved rows. */
int b2_op_gemv_nf4(const void* x, int64_t ldx, const void* codes, const float* absmax, const void* norm_gamma, float eps,
                   const void* residual, int ld_res, void* out, int ld_out, int B, int N, int K, int act, void* stream);
/* decode Linear at batch 9..128 (swap-AB stream-K wgmma GEMM, csrc/gemm_skinny.cu): out[B,N] = x[B,K]·W[N,K]^T
 * (+ residual); act = B2_ACT_NONE | B2_ACT_SWIGLU (out [B,N/2], W rows block-64 interleaved). `workspace` (fp32,
 * >= b2_op_gemm_skinny_workspace_bytes) and `counters` (int32, >= b2_op_gemm_skinny_counter_bytes, zero-filled once
 * by the caller; the kernel leaves them zero) are caller-owned scratch. */
int b2_op_gemm_skinny(const void* x, int ldx, const void* W, int ldw, const void* residual, int ld_res, void* out,
                      int ld_out, int out_fp32, int B, int N, int K, int act, void* workspace, int64_t workspace_bytes,
                      void* counters, void* stream);
/* fp8 variant of b2_op_gemm_skinny: xq [B,K] / Wq [N,K] e4m3 bytes (ld in bytes), x_scale [B], w_scale [N] fp32:
 * out = (xq·Wq^T) * x_scale[b] * w_scale[n] (+ residual). Same scratch contract. */
int b2_op_gemm_skinny_fp8(const void* xq, int ldx, const float* x_scale, const void* Wq, int ldw, const float* w_scale,
                          const void* residual, int ld_res, void* out, int ld_out, int out_fp32, int B, int N, int K, int act,
                          void* workspace, int64_t workspace_bytes, void* counters, void* stream);
/* scale[r] = amax_r / 448 (1 for a zero row); q[r,k] = e4m3_rn_satfinite(x[r,k] * (448 / amax_r)); x bf16, ld in elements */
int b2_op_quantize_rows_e4m3(const void* x, int64_t ldx, int rows, int K, void* q, int64_t ldq, float* scale, void* stream);
/* LlamaRMSNorm (HF rounding points) fused with the per-token quantisation of its output; contiguous rows */
int b2_op_rmsnorm_quant_e4m3(const void* x, const void* gamma, void* q, float* scale, int rows, int cols, float eps,
                             void* stream);
int64_t b2_op_gemm_skinny_workspace_bytes(int B, int N, int K);
int64_t b2_op_gemm_skinny_counter_bytes(int N);
int b2_op_layernorm(const void* x, const void* gamma, const void* beta, void* y, int rows, int cols, float eps,
                    void* stream);
int b2_op_rmsnorm(const void* x, const void* gamma, void* y, int rows, int cols, float eps, void* stream);
/* q,k,v,o: [B,S,H,D] bf16 contiguous; seq_lens device int32 [B] or NULL */
int b2_op_flash_attn(const void* q, const void* k, const void* v, void* o, const int32_t* seq_lens, int B, int S,
                     int H, int D, int causal, float scale, void* stream);
/* causal attention of a chunk against a KV cache: q, o [B,S,H,128] bf16; kcache/vcache [B,H,Smax,128] bf16; pos0 / seq_lens
 * device int32 [B] (seq_lens nullable = S). Query row t of sample b sits at position pos0[b] + t and attends cache rows
 * 0 .. pos0[b] + t; the cache must already hold the chunk's own rows (b2_op_rope_kv_write_at). wgmma kernel only. */
int b2_op_flash_attn_kv(const void* q, const void* kcache, const void* vcache, void* o, const int32_t* pos0, const int32_t* seq_lens,
                        int B, int S, int H, int Smax, float scale, void* stream);
/* qkv [B*S, 3*H*D] (q roped in place); kcache/vcache [B,H,Smax,D] */
int b2_op_rope_kv_write(void* qkv, void* kcache, void* vcache, int B, int S, int H, int D, int Smax, float theta,
                        void* stream);
/* b2_op_rope_kv_write for a chunk at cache position pos0[b] (device int32 [B]): row t of sample b is rotated for position
 * pos0[b] + t and stored at that cache row; rows at or beyond Smax are rotated but not stored */
int b2_op_rope_kv_write_at(void* qkv, void* kcache, void* vcache, const int32_t* pos0, int B, int S, int H, int D, int Smax,
                           float theta, void* stream);
/* qkv [B,3*H*128]; caches [B,H,Smax,128]; cur_len device int32 [B]; out [B,H*128]; scratch from b2_op_decode_attn_scratch */
int b2_op_decode_attn(const void* qkv, void* kcache, void* vcache, const int32_t* cur_len, void* out, void* scratch,
                      int B, int H, int Smax, int nsplit, float theta, float scale, void* stream);
int64_t b2_op_decode_attn_scratch_bytes(int B, int H, int nsplit); /* caller zero-fills the scratch once */
/* b2_op_decode_attn over an e4m3 cache: k8 / v8 [B,H,Smax,128] e4m3 bytes, kscale / vscale [B,H,Smax] fp32, all 16-byte
 * aligned, Smax % 4 == 0. Appends the quantised row of the new token (bytes and scale) and attends over the stored values. */
int b2_op_decode_attn_e4m3(const void* qkv, void* k8, void* v8, float* kscale, float* vscale, const int32_t* cur_len, void* out,
                           void* scratch, int B, int H, int Smax, int nsplit, float theta, float scale, void* stream);
/* multi-query decode attention of the prompt-lookup verify step: qkv [B*R, 3*H*128] with q already roped and rows j < R of sample
 * b already stored at cache rows cur_len[b] + j (b2_op_rope_kv_write_at with pos0 = cur_len); row j attends cache rows
 * 0 .. cur_len[b] + j; out [B*R, H*128] bf16. R in 1..16. scratch: b2_op_decode_attn_mq_scratch_bytes, zero-filled once. */
int b2_op_decode_attn_mq(const void* qkv, const void* kcache, const void* vcache, const int32_t* cur_len, void* out, void* scratch,
                         int B, int R, int H, int Smax, int nsplit, float scale, void* stream);
int64_t b2_op_decode_attn_mq_scratch_bytes(int B, int H, int nsplit);
/* the split factor the verify step uses for b2_op_decode_attn_mq at H heads and a cache of Smax rows (from the kernel's occupancy) */
int b2_op_decode_attn_mq_nsplit(int H, int Smax);
/* b2_op_decode_attn with the group table `groups_host` (host, G groups, the rules of b2_prefix_group; prefix_len is checked against
 * Smax only, the caller keeps it <= cur_len of the source and of every member): row b's keys [0, prefix_len) come from its group's
 * source slot. The table is copied into `scratch` (b2_op_decode_attn_shared_scratch_bytes, zero-filled once); synchronises. */
int b2_op_decode_attn_shared(const void* qkv, void* kcache, void* vcache, const int32_t* cur_len, const b2_prefix_group* groups_host,
                             int G, void* out, void* scratch, int B, int H, int Smax, int nsplit, float theta, float scale,
                             void* stream);
int64_t b2_op_decode_attn_shared_scratch_bytes(int B, int H, int nsplit);
/* the split factor the decode step uses for b2_op_decode_attn_shared at B rows, H heads and a cache of Smax rows */
int b2_op_decode_attn_shared_nsplit(int B, int H, int Smax);
/* the draft of one prompt-lookup step: hist device int32 [len] (the last id is the pending token), max_length = prompt length +
 * max_new_tokens of the generation; out_tokens device int32 [num_tokens + 1] = pending, draft, padding; out_draft_len device int32.
 * Synchronises the stream. */
int b2_op_prompt_lookup(const int32_t* hist, int len, int num_tokens, int max_ngram, int max_length, const int32_t* eos_host, int n_eos,
                        int V, int32_t* out_tokens, int32_t* out_draft_len, void* stream);
/* the split-KV factor a decode step uses for this shape and cache format (from the resident CTAs per SM of the kernel it launches) */
int b2_op_decode_attn_nsplit(int B, int H, int Smax, int kv_dtype);
/* prefill's cache write of an e4m3 cache: kstage / vstage [B,H,S,128] bf16 (roped K, V of one layer) -> rows t < seq_lens[b]
 * (device int32 [B], NULL = S) of k8 / v8 [B,H,Smax,128] and kscale / vscale [B,H,Smax]; rows beyond seq_lens[b] are not written */
int b2_op_kv_quantize_e4m3(const void* kstage, const void* vstage, void* k8, void* v8, float* kscale, float* vscale,
                           const int32_t* seq_lens, int B, int S, int H, int Smax, void* stream);
/* b2_op_kv_quantize_e4m3 of a chunk at cache position pos0[b] (device int32 [B]): kstage / vstage [B,H,S_src,128]; chunk row
 * t < seq_lens[b] (NULL = S) is read from slab row pos0[b] + t and stored at cache row pos0[b] + t; nothing else is written */
int b2_op_kv_quantize_e4m3_at(const void* kstage, const void* vstage, void* k8, void* v8, float* kscale, float* vscale,
                              const int32_t* pos0, const int32_t* seq_lens, int B, int S, int S_src, int H, int Smax, void* stream);
/* the stored prefix of an e4m3 cache as bf16: rows t < pos0[b] (device int32 [B]) of k8 / v8 [B,H,Smax,128] with kscale / vscale
 * [B,H,Smax] -> kdst / vdst [B,H,S_dst,128] row t = bf16(float(q) * scale); rows >= min(pos0[b], S_dst) are not written */
int b2_op_kv_dequantize_e4m3(const void* k8, const void* v8, const float* kscale, const float* vscale, const int32_t* pos0,
                             void* kdst, void* vdst, int B, int H, int Smax, int S_dst, void* stream);
int b2_op_interleave_gate_up(const void* gate, const void* up, void* out, int I, int h, void* stream);
int b2_op_im2col(const void* pixels, void* out, int B, int img, int patch, int kpad, void* stream);
/* Image preprocessing on the device (csrc/preprocess.cu): the reference's llava/mm_utils.py:16-44 (`expand2square` +
 * CLIPImageProcessor.preprocess = PIL bicubic shortest-edge resize, centre crop, rescale, normalise) for ONE uint8 RGB image.
 * The caller (llava/_b2/preprocess.py) supplies the resize plan: PIL's fixed-point coefficient tables for both axes
 * (bounds[2*i] = first tap, bounds[2*i+1] = tap count, kk[i*ksize + t] = 22-bit fixed-point weight; *_identity != 0 when
 * the axis is not resized), the virtual padding, the crop origin and the source-row window of the vertical pass. All
 * pointers are device pointers. pixels: bf16 [3,out,out] (nullable); u8_out: uint8 [out,out,3] before normalisation (nullable). */
typedef struct b2_preprocess_plan {
    const uint8_t* img; int32_t H, W;
    int32_t pad_top, pad_left; uint8_t bg[4];
    const int32_t *h_bounds, *h_kk; int32_t h_ksize, h_identity;
    const int32_t *v_bounds, *v_kk; int32_t v_ksize, v_identity;
    int32_t y0, rows, x_lo, y_lo, out;
    uint8_t* tmp;                /* scratch, >= rows*out*3 bytes */
    float mean[3], stdv[3], rescale;
    void* pixels; uint8_t* u8_out;
} b2_preprocess_plan;
int b2_op_preprocess_clip(const b2_preprocess_plan* plan, void* stream);
/* one selection per row from fp32 logits [B,V] (csrc/sampling.cu): out_tokens device int32 [B]; `index` is the draw index
 * that keys the Philox stream (token position within a generation). Synchronises the stream. */
int b2_op_sample(const float* logits, int B, int V, const b2_sampling* sampling, int index, int32_t* out_tokens, void* stream);
/* b2_op_sample with logits processors: proc (nullable) [B], row b's history is proc[b]'s prompt ids (nothing generated yet).
 * out_processed (nullable, device fp32 [B,V]) receives each row's logits after the processors and before temperature. */
int b2_op_sample_ex(const float* logits, int B, int V, const b2_sampling* sampling, const b2_logits_proc* proc, int index,
                    int32_t* out_tokens, float* out_processed, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B2LLAVA_H_ */
