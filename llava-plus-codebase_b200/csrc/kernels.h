// Internal launcher declarations for the b2llava kernels (C++ side, not part of the C ABI).
// All tensors are device pointers; activations/weights are bf16 unless stated otherwise.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace b2 {

enum { ACT_NONE = 0, ACT_QUICK_GELU = 1, ACT_GELU_ERF = 2, ACT_SWIGLU = 3, ACT_ROPE_QKV = 4 };

// ACT_ROPE_QKV (CTA-pair kernel only): the GEMM is LLaMA's fused QKV projection of a prefill, rows = b*S + t. The epilogue
// rounds the projection to bf16, applies RoPE (HF rounding points, cos/sin from `table`) to the q and k heads, writes q to
// `out` and k / v straight into the KV cache [b][head][Smax][128] — the standalone rope_kv_write pass over qkv disappears.
struct RopeQkv {
    const void* table = nullptr;   // uint32 [Smax][64]: bf16 cos | bf16 sin << 16 of position t, frequency i (rope_table_build)
    void* kcache = nullptr;        // this layer's K slab of the first batch row written
    void* vcache = nullptr;
    int S = 0, H = 0, Smax = 0;
    // device int32 [B] or null: row t of sample b is position pos0[b] + t (table entry and cache row); rows at or beyond Smax
    // store no k / v. Smax must not exceed the table's rows.
    const int32_t* pos0 = nullptr;
};
enum { DT_BF16 = 0, DT_F16 = 1, DT_F32 = 2 };

int num_sms();

// ---- wgmma GEMM (gemm_wgmma.cu) ----------------------------------------------------------------
// out[M, N] = act(A[M,K] · W[N,K]^T + bias) + residual      (ACT_NONE / QUICK_GELU / GELU_ERF)
// out[M, N/2] = silu(gate) * up                               (ACT_SWIGLU; W rows block-64 interleaved)
struct GemmArgs {
    const void* A = nullptr; int lda = 0;        // bf16 [M, K]
    const void* W = nullptr; int ldw = 0;        // bf16 [N, K]
    const void* bias = nullptr;                  // bf16 [N] or null
    const void* residual = nullptr; int ld_res = 0;  // bf16 [M, N] or null (may alias out)
    void* out = nullptr; int ld_out = 0; int out_fp32 = 0;
    int M = 0, N = 0, K = 0;
    int act = ACT_NONE;
    int bn_override = 0;  // 0 = cost-model heuristic, else 64/128/192/256 (2 = CTA-pair kernel)
    RopeQkv rope;         // ACT_ROPE_QKV only
};
int gemm_bf16(const GemmArgs& g, cudaStream_t stream);
// mm_projector mlp2x_gelu as ONE kernel (gemm_wgmma.cu, projector_fused_kernel): out = gelu_erf(X W1^T + b1) W2^T + b2.
// H [M,N1] bf16 and row_done int[ceil(M/128)] are caller scratch.
int projector_fused_bf16(const void* X, int ldx, const void* W1, const void* b1, const void* W2, const void* b2, void* H,
                         void* out, int ld_out, int M, int K1, int N1, int N2, int* row_done, cudaStream_t stream);
// CTA-pair (clusters of two, 256x256 pair tiles, W multicast) variant, gemm_wgmma.cu (chosen by gemm_bf16's cost model, or bn_override == 2)
int gemm_bf16_2cta(const GemmArgs& g, cudaStream_t stream);

// ---- swap-AB stream-K GEMM for decode at batch 9..128 (gemm_skinny.cu) ------------------------------------
// out[B, N] = x[B,K] · W[N,K]^T (+ residual); ACT_SWIGLU: out[B, N/2] (W rows block-64 interleaved).
struct SkinnyArgs {
    const void* x = nullptr; int ldx = 0;        // bf16 [B, K]
    const void* W = nullptr; int ldw = 0;        // bf16 [N, K]
    const void* residual = nullptr; int ld_res = 0;  // bf16 [B, N] or null (may alias out)
    void* out = nullptr; int ld_out = 0; int out_fp32 = 0;
    int B = 0, N = 0, K = 0;
    int act = ACT_NONE;                          // ACT_NONE | ACT_SWIGLU
    float* partial = nullptr; size_t partial_bytes = 0;  // >= gemm_skinny_workspace_bytes(B, N, K)
    int* counters = nullptr;                     // >= gemm_skinny_counter_bytes(N), zero-initialised once
    const float* w_scale = nullptr;              // fp8 variant: [N] per weight row; x / W then hold e4m3 bytes
    const float* x_scale = nullptr;              // fp8 variant: [B] per token
};
int gemm_skinny_bf16(const SkinnyArgs& g, cudaStream_t stream);
int gemm_skinny_fp8(const SkinnyArgs& g, cudaStream_t stream);
size_t gemm_skinny_workspace_bytes(int B, int N, int K);
size_t gemm_skinny_counter_bytes(int N);

// ---- e4m3 row quantisation for the fp8 decode path (quant_fp8.cu) ----------------------
// scale[r] = amax_r / 448 (1 for a zero row); q[r,k] = e4m3_rn_satfinite(x[r,k] * (448 / amax_r)); ld* in elements
int quantize_rows_e4m3(const void* x, int64_t ldx, int rows, int K, void* q, int64_t ldq, float* scale, cudaStream_t stream);
// RMSNorm (HF rounding points) fused with the per-token quantisation of its output
int rmsnorm_quant_e4m3(const void* x, int64_t x_row_stride, const void* gamma, void* q, int64_t ldq, float* scale, int rows,
                       int cols, float eps, cudaStream_t stream);

// ---- weight-streaming GEMV for decode (gemv.cu) ---------------------------------------------------
// out[B, N] = (rmsnorm(x) or x)[B,K] · W[N,K]^T (+ residual); B <= 8. ACT_SWIGLU: out[B, N/2].
struct GemvArgs {
    const void* x = nullptr; int64_t ldx = 0;   // bf16 [B, K], row stride ldx (elements)
    const void* W = nullptr; int ldw = 0;        // bf16 [N, K]
    const void* norm_gamma = nullptr; float eps = 0.f;  // fused RMSNorm on x when non-null
    const void* residual = nullptr; int ld_res = 0;     // bf16 [B, N] or null (may alias out)
    void* out = nullptr; int ld_out = 0; int out_fp32 = 0;
    int B = 0, N = 0, K = 0;
    int act = ACT_NONE;
};
int gemv_bf16(const GemvArgs& g, cudaStream_t stream);
bool gemv_fits(int B, int N, int K, int act);  // activation tile + partial table fit in shared memory

// ---- NF4 weights (nf4.cu; format in DESIGN.md §2-3) ------------------------------------------------------------
// w bf16 [N, K] (row pitch ldw) -> codes [N, K/2] bytes + absmax [N, K/64] fp32; K % 64 == 0. gemv_order = 0: canonical
// layout (element 2j in the high nibble of byte j); 1: the order gemv_nf4 reads (K % 128 == 0)
int quantize_nf4(const void* w, int64_t ldw, int N, int K, void* q, float* absmax, int gemv_order, cudaStream_t stream);
struct Nf4Matrix {
    const void* q = nullptr; const float* absmax = nullptr;
    void* out = nullptr;  // bf16 [N, K], contiguous
    int N = 0, K = 0;
};
// w_hat = bf16(code * absmax) of up to four matrices in one launch
int dequantize_nf4(const Nf4Matrix* mats, int n, int gemv_order, cudaStream_t stream);
// gemv_bf16's contract over NF4 weights in GEMV order (g.W unused; bf16 output only); K % 128 == 0
int gemv_nf4(const GemvArgs& g, const void* q, const float* absmax, cudaStream_t stream);
bool gemv_nf4_fits(int B, int N, int K, int act);

// ---- norms (norms.cu) ------------------------------------------------------------------------------
int layernorm_bf16(const void* x, const void* gamma, const void* beta, void* y, int rows, int cols, float eps,
                   cudaStream_t stream);
// HF LlamaRMSNorm semantics: y = gamma * bf16(x * rsqrt(mean(x^2) + eps)); x rows may be strided.
int rmsnorm_bf16(const void* x, int64_t x_row_stride, const void* gamma, void* y, int rows, int cols, float eps,
                 cudaStream_t stream);
// gather variant: row r of y is the RMSNorm of x[row_index[r]] (row_index on device)
int rmsnorm_gather_bf16(const void* x, const int32_t* row_index, const void* gamma, void* y, int rows, int cols,
                        float eps, cudaStream_t stream);

// ---- ViT helpers (vit_ops.cu) ----------------------------------------------------------------------
// pixels [B,3,img,img] bf16 -> patches [B*P, kpad] (k = c*patch*patch + i*patch + j, zero padded to kpad)
int vit_im2col(const void* pixels, void* out, int B, int img, int patch, int kpad, cudaStream_t stream);
// hidden[b, 0] = LN(cls + pos[0]); hidden[b, 1+p] = LN(patch_out[b*P+p] + pos[1+p])   (pre_layrnorm fused)
int vit_embed_ln(const void* patch_out, const void* cls, const void* pos, const void* gamma, const void* beta,
                 void* hidden, int B, int P, int D, float eps, cudaStream_t stream);
// out[b, p, :] = hidden[b, 1 + p, :]   (feature_select 'patch': drop CLS)
int vit_drop_cls(const void* hidden, void* out, int B, int P, int D, cudaStream_t stream);

// ---- attention (attention_wgmma.cu, attention.cu) ---------------------------------------------------
struct FlashArgs {
    const void* q = nullptr; int64_t q_bs = 0, q_ts = 0, q_hs = 0;  // element strides: batch, token, head
    const void* k = nullptr; int64_t k_bs = 0, k_ts = 0, k_hs = 0;
    const void* v = nullptr; int64_t v_bs = 0, v_ts = 0, v_hs = 0;
    void* o = nullptr;       int64_t o_bs = 0, o_ts = 0, o_hs = 0;
    const int32_t* seq_lens = nullptr;  // device [B] or null (=S)
    // device [B] or null: query row t of sample b sits at absolute position pos0[b] + t and attends keys 0 .. pos0[b] + t of
    // k / v, which then hold Skv rows per (b, head) (a KV cache). Causal, D = 128.
    const int32_t* pos0 = nullptr;
    int Skv = 0;
    int B = 0, H = 0, S = 0, D = 0;     // S = padded/query length; D in {64, 128}
    int causal = 0;
    float scale = 1.f;
};
int flash_attn_bf16(const FlashArgs& a, cudaStream_t stream);  // attention_wgmma.cu: wgmma + TMA

// prefill: RoPE on q (in place) and k inside qkv [B*S, 3*H*D]; roped k and v written to the cache
// kcache/vcache: [Bmax, H, Smax, D] for one layer. Positions are 0..S-1 (right-padded rows).
// (cos, sin) table of rope_kv_write's positions 0..Smax-1 (head_dim D): uint32 [Smax][D/2], bf16 cos | bf16 sin << 16
int rope_table_build(void* table, int Smax, int D, float theta, cudaStream_t stream);
// pos0 (device int32 [B] or null): row t of sample b is the token at absolute position pos0[b] + t (its RoPE angle and its
// cache row); rows at or beyond Smax are rotated but not stored. pos0 == null: positions t, S <= Smax.
int rope_kv_write(void* qkv, void* kcache, void* vcache, int B, int S, int H, int D, int Smax, float theta,
                  cudaStream_t stream, const int32_t* pos0 = nullptr);

// decode: q/k/v of the new token from qkv [B, 3*H*D]; RoPE at position cur_len[b]; append k,v to the cache;
// split-KV attention over cur_len[b]+1 keys; out [B, H*D] bf16.
struct DecodeAttnArgs {
    const void* qkv = nullptr;
    void* kcache = nullptr; void* vcache = nullptr;  // layer base, [Bmax, H, Smax, D] (bf16, or e4m3 bytes)
    float* kscale = nullptr; float* vscale = nullptr;  // e4m3 cache only: layer base, [Bmax, H, Smax] fp32
    const int32_t* cur_len = nullptr;                // device [B]
    void* out = nullptr;
    float* partial = nullptr;                        // workspace [B*H*nsplit*(D+2)] fp32
    int32_t* counters = nullptr;                     // workspace [B*H], zero-initialised, self-resetting
    int B = 0, H = 0, D = 128, Smax = 0, nsplit = 1;
    float theta = 10000.f, scale = 1.f;
    int R = 1;  // decode_attn_mq only: query rows per sample
};
int decode_attn_ctas_per_sm();
int decode_attn_bf16(const DecodeAttnArgs& a, cudaStream_t stream);
// multi-query decode (prompt-lookup verify step) over a bf16 cache: qkv [B*R, 3*H*D] with q already roped and the R rows'
// K / V already stored at cache rows cur_len[b] .. cur_len[b] + R - 1 (rope_kv_write at pos0 = cur_len); row j attends rows
// 0 .. cur_len[b] + j; out [B*R, H*D]. R <= 16. partial: [B*H*nsplit*16*(D+2)] fp32; counters as decode_attn's. The cache
// length is not advanced. No RoPE, no cache write.
int decode_attn_mq_ctas_per_sm();
size_t decode_attn_mq_scratch_bytes(int B, int H, int nsplit);  // partial then counters
int decode_attn_mq_bf16(const DecodeAttnArgs& a, cudaStream_t stream);
// shared-prefix decode (the forked samples of one prompt): decode_attn_bf16's result for every row, with keys [0, prefix_len) of
// a group's rows read once per group from its source slot. Same layout as b2_prefix_group (include/b2llava.h).
constexpr int kPrefixGroupRows = 16;
struct PrefixGroup {
    int32_t src_slot, prefix_len, n_rows;
    int32_t rows[kPrefixGroupRows];
};
// groups: device [G]; row_prefix: device [B], the prefix_len of the row's group (0 outside every group). G <= B, every row in
// at most one group, 1 <= prefix_len <= cur_len of the source and of every member. partial: [B*H*2*nsplit*(D+2)] fp32, then the
// counters [B*H] (decode_attn_shared_scratch_bytes)
int decode_attn_shared_ctas_per_sm();
size_t decode_attn_shared_scratch_bytes(int B, int H, int nsplit);  // partial then counters
int decode_attn_shared_bf16(const DecodeAttnArgs& a, const PrefixGroup* groups, const int32_t* row_prefix, int G,
                            cudaStream_t stream);
// the same step over an e4m3 cache (rows of 128 bytes + one fp32 scale per row); Smax % 4 == 0
int decode_attn_e4m3_ctas_per_sm();
int decode_attn_e4m3(const DecodeAttnArgs& a, cudaStream_t stream);
// prefill cache write of an e4m3 cache: roped bf16 K / V of one layer, [B, H, S, D] contiguous, -> rows t < seq_lens[b]
// (device, null = S) of k8 / v8 [B, H, Smax, D] bytes and kscale / vscale [B, H, Smax]
// With pos0 (device int32 [B]): the slabs are [B, H, S_src, D] (0 = S) and chunk row t < seq_lens[b] is read from and stored
// at row pos0[b] + t; rows outside the slab or the cache are skipped.
int kv_quantize_e4m3(const void* ksrc, const void* vsrc, void* k8, void* v8, float* kscale, float* vscale,
                     const int32_t* seq_lens, int B, int S, int H, int D, int Smax, cudaStream_t stream,
                     const int32_t* pos0 = nullptr, int S_src = 0);
// the stored prefix as bf16: rows t < pos0[b] (device int32 [B]) of k8 / v8 [B, H, Smax, 128] and their scales ->
// bf16(float(q) * scale) at row t of kdst / vdst [B, H, S_dst, 128]
int kv_dequantize_e4m3(const void* k8, const void* v8, const float* kscale, const float* vscale, const int32_t* pos0, void* kdst,
                       void* vdst, int B, int H, int Smax, int S_dst, cudaStream_t stream);

// ---- persistent decode-step megakernel (decode_mega.cu), batch <= 8 ------------------------------------
struct MegaLayer {
    const __nv_bfloat16 *ln1, *wqkv, *wo, *ln2, *wgu, *wd;
    __nv_bfloat16 *kcache, *vcache;  // this layer's [Bmax, H, Smax, 128] slabs
};
struct MegaParams {
    const MegaLayer* layers = nullptr;  // device array [L]
    int L = 0, h = 0, I = 0, H = 0, V = 0, B = 0, Smax = 0, nsplit = 1;
    const __nv_bfloat16 *embed = nullptr, *final_norm = nullptr, *lm_head = nullptr;
    int32_t *tok = nullptr, *cur_len = nullptr, *out_tokens = nullptr, *step_counter = nullptr;
    __nv_bfloat16 *x = nullptr, *qkv = nullptr, *attn = nullptr, *act = nullptr;
    float* logits = nullptr;
    float* attn_partial = nullptr;      // [B*H*nsplit*(128+2)]
    int32_t* attn_counters = nullptr;   // [B*H], zero-initialised, self-resetting
    unsigned int *bar_count = nullptr, *done_count = nullptr;  // zero-initialised
    unsigned int bar_base = 0;  // barrier-counter value before this launch = launches so far * (5L+2) * grid
    float eps = 1e-5f, theta = 10000.f, scale_log2 = 1.f;
    long long* trace = nullptr;  // optional [n_phases+2][4] SM-clock timestamps of CTA 0 (B2_MEGA_TRACE=<file>)
    // token publication to the host ring (sampling.cu): non-null only for greedy streaming; with do_sample the separate
    // sample_publish kernel that follows the launch overrides the fused argmax and publishes instead
    struct SampleState* sstate = nullptr;
    int32_t* ring = nullptr;
    int ring_cap = 0;
    const struct RowState* rows = nullptr;  // continuous batching: only active slots advance their cache length
};
// one launch = embed -> all layers -> lm_head -> argmax -> token store; cur_len/step_counter advance on device
int decode_mega(const MegaParams& p, cudaStream_t stream);
bool decode_mega_fits(int B, int h, int I);

// ---- token selection + host-ring publication (sampling.cu) --------------------------------------------------
// Device-resident state of one generation (lives in the b2_kv): read by the kernels, so a captured CUDA graph of the decode
// step stays valid when the sampling parameters change.
struct SampleState {
    int do_sample;            // 0 = greedy argmax
    float temperature, top_p;
    int top_k;                // 0 = off
    unsigned long long seed;  // Philox key
    int tag;                  // generation epoch 1..2047 published with every token; 0 = do not publish to the host ring
    int pub_counter;          // index of the next token of this generation
    unsigned int done;        // rows finished in the current launch (self-resetting)
    int per_row;              // continuous batching: selection parameters and liveness come from RowState[b] instead
    // generate(output_scores / output_logits): fp32 rows [out_cap][B][V] (nullable). The step that publishes token t writes
    // row t of each: the processed row it selected from (scores) and the raw logits it read (logits); t >= out_cap is skipped
    float* out_scores;
    float* out_logits;
    int out_cap;
};
// One cache slot of a continuously batched decode (llava/_b2/batching.py): requests join and leave between steps, each with
// its own sampling parameters and its own Philox draw index; a slot that is not active keeps its cache length and token.
struct RowState {
    int active;
    int do_sample; float temperature, top_p; int top_k;
    unsigned long long seed;
    int index;                // draws made for this request so far
};
// History-aware logits processing of one row (HF RepetitionPenalty -> NoRepeatNGram -> MinLength / MinNewTokens), applied by
// sample_publish before selection. Device-resident like RowState, so a captured decode graph stays valid when it changes.
constexpr int kProcMaxEos = 8;
struct ProcRow {
    int on;                   // 0: the row is selected from its raw logits and its history is not kept
    float penalty;            // repetition penalty, 1 = off
    int ngram;                // no_repeat_ngram_size, 0 = off
    int min_gen;              // eos ids are banned while fewer than min_gen tokens were generated
    int n_eos;
    int eos[kProcMaxEos];
    int prompt_len;           // history[0, prompt_len) is the caller's prompt row; what follows was generated
    int hist_len;
};
// Per-cache processing state: rows[B], history int32 [B][cap] (cap = max_seq + 1), presence bitmap uint32 [B][words] of the
// history's ids in [0, V). rows == nullptr: no row of this cache has ever had processors on.
struct ProcState {
    ProcRow* rows;
    int32_t* hist;
    uint32_t* bits;
    int cap, words;
};
// Prompt-lookup speculative decoding of one sample (b2_stream_begin_lookup), device-resident so the verify step is a CUDA
// graph: prompt_lookup drafts from the history, the verify forward runs R = K + 1 rows, sample_publish's multi-row mode accepts.
constexpr int kSpecMaxRows = 16;
struct SpecState {
    int K;                    // draft tokens per step (R = K + 1 rows)
    int ngram;                // max_matching_ngram_size
    int max_new;              // the generation never publishes more tokens
    int n_eos;
    int eos[kProcMaxEos];     // a draft ends before the first eos id
    int prompt_len;
    int hist_len;             // history (ProcState row 0) = the prompt, then every published token but the pending one (tok[0])
    int draft_len;            // draft of the step in flight (rows[1 .. draft_len])
    int32_t rows[kSpecMaxRows];  // the step's input tokens: the pending token, the draft, padding
    int steps, drafted, accepted;  // steps that published tokens, tokens they drafted, draft tokens accepted
    int retired;              // verify steps finished, including those queued after the generation was complete
    int32_t sel[kSpecMaxRows];  // token selected from each row's logits
    int* mirror;              // mapped host int[6]: steps, drafted, accepted, cache length, retired, tokens published
};
// one CTA: history hist[0, hist_len) + tok[0] -> draft (HF PromptLookupCandidateGenerator.get_candidates, cut before the first eos
// id or id outside [0, V)) -> spec->rows = tok[0], the draft, tok[0] as padding up to R; spec->draft_len. st->pub_counter = tokens
// published so far.
int prompt_lookup(int32_t* hist, SpecState* spec, const SampleState* st, const int32_t* tok, int V, int R, cudaStream_t stream);

enum { SP_SELECT = 1,     // choose from `logits` (argmax or sample) and write tok[b]; otherwise tok[b] is already chosen
       SP_WRITE_OUT = 2,  // out_tokens[(*step_counter + step_offset) * B + b] = token
       SP_BUMP = 4 };     // last row: *step_counter += 1, cur_len[b] += 1
int sample_state_set(SampleState* st_dev, const SampleState& v, cudaStream_t stream);
// `proc` processes rows whose ProcRow is on (and appends the chosen token to their history); `processed_out` (nullable, fp32
// [B,V]) receives each selected row's logits after processing and before temperature.
// With `spec` (multi-row acceptance of a verify step, sample 0 only): the B rows are the step's R rows; row j is selected as
// draw pub_counter + j (Philox row 0, as plain streaming keys it) unless j > draft_len; the last CTA accepts n = matches + 1
// tokens (HF's n_matches rule, capped by max_new), appends them to the history (proc.hist row 0), publishes them at ring indices
// pub_counter .. + n - 1, sets tok[0] to the last one and advances cur_len[0] and pub_counter by n. flags must be SP_SELECT.
int sample_publish(const float* logits, int V, int B, SampleState* st_dev, RowState* rows_dev, int32_t* tok, int32_t* out_tokens,
                   int32_t* step_counter, int32_t* cur_len, int32_t* ring_dev, int ring_cap, int flags, int step_offset,
                   const ProcState& proc, float* processed_out, cudaStream_t stream, SpecState* spec = nullptr);
// the output rows of the step whose token the decode megakernel's fused argmax has just published (token pub_counter - 1): the
// raw logits [B, V] to st->out_scores and st->out_logits (greedy without processors: the score row is the logits row). Selects
// nothing, publishes nothing and leaves the counters alone.
int publish_rows(const float* logits, int V, int B, const SampleState* st_dev, cudaStream_t stream);
// row := v, its history := ids[0, len) (int64, device) followed by `first_token` when >= 0, and its bitmap rebuilt from those ids
int proc_seed(const ProcState& proc, int row, const ProcRow& v, const int64_t* ids, int len, int first_token, int V,
              cudaStream_t stream);
int row_state_set(RowState* row_dev, const RowState& v, int32_t* tok_dev, int token, cudaStream_t stream);

// ---- beam search (beam.cu) ---------------------------------------------------------------------------------------------------
// per sample b, the K best (score, token, beam) of score = log_softmax(logits[row_of_beam[b*nb + j]]) + beam_scores[b*nb + j]
// over its nb beams x V tokens, sorted by score descending, ties to the lower beam * V + token; row_of_beam null = identity.
// nb <= 32, K <= min(128, nb * V); workspace >= beam_topk_workspace_bytes(B, nb, K)
size_t beam_topk_workspace_bytes(int B, int nb, int K);
// generate(output_scores / output_logits) of beam search: each beam row b*nb + j also writes its score row (log_softmax, warped
// under beam sampling) to scores[(b*nb + j) * fan + r] and the raw logits it read to logits[...], r < fan, fp32 [V] each (both
// nullable). fan > 1 fills the nb running rows of a sample from its one prefill row (the first step of beam search, nb = 1).
struct BeamRowsOut {
    float* scores = nullptr;
    float* logits = nullptr;
    int fan = 1;
};
// Logits processors of beam search (HF's processors over each running beam's log_softmax row, against its own sequence):
// beam row b*nb + j reads logits row r = row_of_beam[b*nb + j] and, when proc.rows[r].on, first appends append[b*nb + j] to
// history r (when `append` is non-null), then processes its log-probabilities against history r (process_row) before the
// running score is added (and, under beam sampling, before the warpers). proc.rows == nullptr: processing off, the kernels of
// the unprocessed selection run.
struct BeamProc {
    ProcState proc = {};
    const int32_t* append = nullptr;
};
int beam_topk(const float* logits, const int32_t* row_of_beam, const float* beam_scores, int B, int nb, int V, int K,
              void* workspace, float* out_scores, int32_t* out_tokens, int32_t* out_beams, cudaStream_t stream,
              const BeamRowsOut& rows_out = BeamRowsOut{}, const BeamProc& proc = BeamProc{});
// beam sampling: the same selection over Gumbel-perturbed keys of the warped scores (beam_row_sample_kernel in beam.cu); each
// candidate's score is its unperturbed accumulated score. T > 0, top_k >= 0 (0 = off), top_p in (0, 1], min_keep >= 1.
struct BeamSampleParams {
    float temperature;
    int top_k;
    float top_p;
    int min_keep;
    unsigned long long seed;
    uint32_t step;
};
size_t beam_sample_workspace_bytes(int B, int nb, int K);
int beam_sample(const float* logits, const int32_t* row_of_beam, const float* beam_scores, int B, int nb, int V, int K,
                const BeamSampleParams& sp, void* workspace, float* out_scores, int32_t* out_tokens, int32_t* out_beams,
                cudaStream_t stream, const BeamRowsOut& rows_out = BeamRowsOut{}, const BeamProc& proc = BeamProc{});
struct KvCopyPairs {
    static constexpr int kMax = 64;
    int32_t src[kMax], dst[kMax], end[kMax];
};
// for each pair i: rows [row_begin, end[i]) of cache slot src[i] -> slot dst[i], every layer / head / K and V (k / v bases of
// [L][max_batch][H][pitch][row_bytes] bytes; kscale / vscale [L][max_batch][H][pitch] fp32 or null), and len_dev[dst[i]] = end[i].
// No dst may be a src of the same call.
int kv_copy_slots(void* k, void* v, float* kscale, float* vscale, const int32_t* src, const int32_t* dst, const int32_t* end, int n,
                  int row_begin, int L, int H, int max_batch, int pitch, int row_bytes, int32_t* len_dev, cudaStream_t stream);
// for each pair i: history row src[i] of `proc` -> row dst[i]: its ProcRow, history ids [0, hist_len) and presence bitmap
// (one CTA per pair). No dst may be a src of the same call.
int proc_copy_slots(const ProcState& proc, const int32_t* src, const int32_t* dst, int n, cudaStream_t stream);

// ---- image preprocessing (preprocess.cu): uint8 HWC -> CLIP pixel_values, PIL-exact bicubic resize ------------------------
struct PreprocessArgs {
    const uint8_t* img = nullptr; int H = 0, W = 0;        // device, RGB HWC
    int pad_top = 0, pad_left = 0; uint8_t bg[3] = {0, 0, 0};  // virtual expand2square: reads outside the image return bg
    const int32_t *h_bounds = nullptr, *h_kk = nullptr; int h_ksize = 0, h_identity = 0;  // tables over the resized WIDTH
    const int32_t *v_bounds = nullptr, *v_kk = nullptr; int v_ksize = 0, v_identity = 0;  // tables over the resized HEIGHT
    int y0 = 0, rows = 0;        // source rows the vertical pass reads: [y0, y0 + rows)
    int x_lo = 0, y_lo = 0;      // centre-crop origin inside the resized image
    int cols = 0, out = 0;       // cols == out: crop width / output size
    uint8_t* tmp = nullptr;      // [rows, cols, 3] scratch
    float mean[3] = {0, 0, 0}, stdv[3] = {1, 1, 1}, rescale = 1.f / 255.f;
    void* pixels = nullptr;      // bf16 [3, out, out] or null
    uint8_t* u8_out = nullptr;   // uint8 [out, out, 3] (the resized + cropped image before normalisation) or null
};
int preprocess_clip_image(const PreprocessArgs& a, cudaStream_t stream);

// ---- misc (misc_ops.cu) ----------------------------------------------------------------------------
// out[r, :] = src_index[r] >= 0 ? table[src_index[r]] : (src_index[r] == INT32_MIN ? 0 : feats[-src_index[r]-1]).
// Rows whose index is outside [0, vocab) / [0, n_feat_rows) are written as zeros and reported through *err_flag
// (mapped host memory, B2_ERR_* codes, may be null): nothing is ever read out of bounds.
int splice_embed(const int32_t* src_index, const void* table, const void* feats, void* out, int rows, int h, int vocab,
                 int n_feat_rows, int* err_flag, cudaStream_t stream);
// device-built source index for equal-length unpadded rows with k_per_row image placeholders each (misc_ops.cu):
// ids int64 [B, Lt] on the device; feat_offsets_host[n_img + 1] = prefix sums of the feature rows of the image slots
int splice_index(const long long* ids, int B, int Lt, int k_per_row, const int32_t* feat_offsets_host, int n_img, int image_token,
                 int S, int32_t* src_index, int* err_flag, cudaStream_t stream);
int embed_tokens(const int32_t* tokens, const void* table, void* out, int rows, int h, int vocab, int* err_flag,
                 cudaStream_t stream);
enum { B2_ERR_TOKEN_RANGE = 1, B2_ERR_IMAGE_ROW_RANGE = 2, B2_ERR_SPLICE_SLOTS = 4 };
int argmax_f32(const float* logits, int B, int V, int32_t* out, cudaStream_t stream);
struct I32Pack { int32_t v[128]; };
// dst_a[i] = a_host[i] (and dst_b[i] = b_host[i] when dst_b != null), i < n: values travel as kernel parameters
int set_i32_pairs(int32_t* dst_a, const int32_t* a_host, int32_t* dst_b, const int32_t* b_host, int n, cudaStream_t stream);
int convert_to_bf16(const void* src, int src_dtype, void* dst, int64_t n, cudaStream_t stream);
// out[2I, h]: within each 128-row group g: rows [0,64) = gate[g*64 .. +64), rows [64,128) = up[g*64 .. +64)
int interleave_gate_up(const void* gate, const void* up, void* out, int I, int h, cudaStream_t stream);

}  // namespace b2
