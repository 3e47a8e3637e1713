// Engine + C ABI of libb2llava.so: weight ingestion/repack, workspaces, and the orchestration of the
// hot path (CLIP ViT -> mm_projector -> splice -> LLaMA prefill -> KV-cache decode) over the kernels in this
// directory. Entry points are declared in include/b2llava.h, which cites the reference function each replaces.
#include <cuda_fp16.h>
#include <limits.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

#include <array>
#include <atomic>
#include <utility>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/b2llava.h"
#include "common.cuh"
#include "kernels.h"

namespace b2 {

static thread_local char g_err[1024] = {0};
unsigned long long g_launch_count = 0;

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

namespace {
typedef __nv_bfloat16 bf16;

struct DevBuf {
    void* p = nullptr;
    size_t bytes = 0;
    int alloc(size_t n) {
        free();
        if (n == 0) return 0;
        cudaError_t e = cudaMalloc(&p, n);
        if (e != cudaSuccess) {
            p = nullptr;
            set_error("cudaMalloc(%zu bytes) failed: %s", n, cudaGetErrorString(e));
            return -2;
        }
        bytes = n;
        return 0;
    }
    void free() {
        if (p) cudaFree(p);
        p = nullptr;
        bytes = 0;
    }
    template <typename T>
    T* as() const { return reinterpret_cast<T*>(p); }
};

struct VitLayer {
    DevBuf ln1_g, ln1_b, wqkv, bqkv, wo, bo, ln2_g, ln2_b, w1, b1, w2, b2;
    unsigned qkv_w = 0, qkv_b = 0;  // bit j set: part j (q/k/v) of the fused buffer has arrived
};
// One decoder Linear [N, K] in each format it can be held in: the bf16 weight w, its e4m3 copy w8 + per-row fp32 scales s8
// (b2_model_enable_fp8_decode), and its NF4 codes q in GEMV order [N, K/2] + absmax a [N, K/64] (b2_model_enable_nf4, which
// frees w)
struct Linear {
    DevBuf w;
    DevBuf w8, s8;
    DevBuf q, a;
    void free() { for (DevBuf* b : {&w, &w8, &s8, &q, &a}) b->free(); }
    size_t bytes() const { return w.bytes + w8.bytes + s8.bytes + q.bytes + a.bytes; }
};
struct LlamaLayer {
    DevBuf ln1, ln2;
    Linear qkv, o, gu, d;  // gu: gate / up rows interleaved in blocks of 64 (interleave_gate_up)
    std::array<Linear*, 4> linears() { return {&qkv, &o, &gu, &d}; }  // the order of layer_shapes
    unsigned qkv_parts = 0;
    DevBuf tmp_gate, tmp_up;  // staging until both halves arrived
    bool has_gate = false, has_up = false;
};
struct LinearShape { int N, K, act; };
// N, K and activation of a decoder layer's Linears: QKV, O, gate/up (SwiGLU), down
std::array<LinearShape, 4> layer_shapes(const b2_model_desc& d) {
    const int h = d.hidden, I = d.inter;
    return {{{3 * h, h, ACT_NONE}, {h, h, ACT_NONE}, {2 * I, h, ACT_SWIGLU}, {h, I, ACT_NONE}}};
}
}  // namespace
}  // namespace b2

using namespace b2;

struct b2_model {
    b2_model_desc d;
    int device = 0;
    std::mutex mu;
    bool finalized = false;
    // derived
    int P = 0, T = 0, kpad = 0, vit_live = 0, vit_hd = 64, hd = 128;
    // weights
    DevBuf patch_w, cls, pos, pre_g, pre_b;
    std::vector<VitLayer> vit;
    DevBuf p0_w, p0_b, p2_w, p2_b;
    DevBuf embed, final_norm;
    Linear head;  // lm_head: w, and w8 / s8 with fp8 decode (never NF4)
    std::vector<LlamaLayer> ll;
    // errors detected by kernels (bad token ids / image rows): int[8] in mapped pinned host memory, slot = log2(B2_ERR_*)
    int* err_host = nullptr;
    int* err_dev = nullptr;
    // the workspaces below are shared by every call on this model: a call on stream B must not start before the previous
    // call's kernels on stream A are done with them (calls on one stream are ordered anyway)
    cudaEvent_t ws_event = nullptr;
    cudaStream_t ws_stream = nullptr;
    bool ws_valid = false;
    // ViT workspace (per chunk of max_images)
    DevBuf v_col, v_patch, v_hidden, v_xn, v_qkv, v_attn, v_mlp, v_feats, p_mid, p_done;
    // LLaMA workspace
    DevBuf x, xn, qkv, attn, act, last_idx, xlast, logits, splice_idx;
    DevBuf chunk_pos;  // b2_prefill_at: int32 [2][max_batch] = start position, then chunk length, of each sample
    // encode_images replays a CUDA graph per chunk size (~190 launches per image, 5-20 us each at B = 1: the host cannot
    // keep the GPU fed launch by launch). Inputs/outputs are staged through fixed buffers so the captured pointers stay valid.
    DevBuf enc_pixels, enc_out;
    std::vector<cudaGraphExec_t> enc_graph;  // index = images in the chunk (0 = unused)
    std::vector<char> enc_warm;              // an eager run has set the function attributes for this chunk size
    cudaStream_t enc_stream = nullptr;       // capture is illegal on the legacy default stream: such callers run here
    cudaEvent_t enc_fork = nullptr, enc_join = nullptr;
    int enc_launches = 0;                    // kernels in one captured chunk (b2_launch_count bookkeeping)
    // fp8 decode (BASELINE configs[4]): quantised activation row buffer + per-token scales
    bool fp8_decode = false;
    DevBuf xq8, xscale;
    // e4m3 KV caches: one layer of roped bf16 K / V, [B][H][S][128], that prefill attends over before it is quantised into
    // the cache (allocated with the first e4m3 cache)
    DevBuf kstage, vstage;
    // NF4 decoder Linears (b2_model_enable_nf4): the dense kernels read one layer's w_hat from this bf16 scratch
    // (wqkv | wo | wgu | wd, dequantised by one launch per layer); a workspace like the ones above
    bool nf4 = false;
    DevBuf nf4_scratch;
    std::atomic<int> kv_live{0};  // KV caches created on this model and not destroyed
};

struct b2_kv {
    b2_model* m = nullptr;
    int max_batch = 0, max_seq = 0;
    int dtype = B2_KV_BF16;
    int pitch = 0;       // tokens per (layer, sample, head) slab: max_seq, rounded up to a multiple of 4 for an e4m3 cache
    DevBuf k, v;         // [L][B][H][pitch][D] bf16, or e4m3 bytes
    DevBuf kscale, vscale;  // e4m3 cache: [L][B][H][pitch] fp32, one scale per stored row
    DevBuf len_dev, tok, step_counter, out_tokens, attn_partial, attn_counters;
    DevBuf sk_partial, sk_counters;  // stream-K workspace of the skinny decode GEMM (batch 9..128)
    std::vector<int32_t> len_host;
    int out_capacity = 0;  // steps
    // cached decode-step graph
    cudaGraphExec_t graph = nullptr;
    int graph_B = 0;
    int graph_launches = 0;  // kernels in the captured step (b2_launch_count bookkeeping)
    // stream capture is illegal on the legacy default stream (torch's default current stream): decode steps
    // run on this library-owned stream, ordered against the caller's stream with events
    unsigned int mega_bar_base = 0;  // value of the grid-barrier counter before the next megakernel launch
    DevBuf mega_layers, mega_sync;  // MegaLayer[L] table and {bar_count, bar_gen, done_count}
    DevBuf rope_tab;                // uint32 [max_seq][hd/2]: bf16 (cos, sin) per position for the QKV GEMM's fused RoPE epilogue
    cudaStream_t own_stream = nullptr;
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    int warm_B = 0;  // an eager step has run for this B (function attributes set, driver entry points resolved)
    // token selection state (sampling.cu) + the host-visible token ring of the streaming decode API
    DevBuf sstate;                 // SampleState on the device
    SampleState samp_host = {};    // what was last written there (pub_counter / done excluded: the device advances them)
    bool samp_valid = false;
    int32_t* ring_host = nullptr;  // cudaHostAlloc(mapped) [ring_cap][max_batch]; entry = tag << 20 | token
    int32_t* ring_dev = nullptr;
    int ring_cap = 0;
    int epoch = 0;                 // generations started on this cache (tag = 1 + epoch % 2047)
    int stream_B = 0, stream_tag = 0, stream_scheduled = 0;  // streaming generation in progress: tokens scheduled so far
    // output rows armed by b2_stream_set_outputs for the next b2_stream_begin(_ex), which takes them over (SampleState::out_*)
    float* next_scores = nullptr;
    float* next_logits = nullptr;
    int next_cap = 0;
    DevBuf rows_dev;               // RowState[max_batch] (continuous batching)
    std::vector<RowState> rows_host;
    // b2_beam_step (allocated by the first call): beam -> slot map and running scores [2][max_batch], the per-row candidate
    // keys of beam_topk, and its [B, K] outputs (scores, tokens, beams)
    DevBuf beam_in, beam_ws, beam_out;
    // history-aware logits processing (b2_stream_begin_ex / b2_batch_set_row_ex; allocated by the first call that turns it on):
    // ProcRow[max_batch], history int32 [max_batch][max_seq + 1], presence bitmap uint32 [max_batch][ceil(V / 32)]
    DevBuf proc_rows, proc_hist, proc_bits;
    std::vector<char> proc_on;  // host copy of ProcRow::on per slot
    bool any_proc() const { for (char c : proc_on) if (c) return true; return false; }
    // beam search with logits processors (b2_beam_begin_proc, allocated by its first call): ProcRow[max_batch] of the beams'
    // cache slots. Their histories and bitmaps share proc_hist / proc_bits (a cache runs one kind of generation at a time), while
    // the rows stay apart from proc_rows, which every decode step clears and whose rows the decode step's selection would append
    // its own choice to. Armed until a call turns every row's processors off.
    DevBuf beam_proc_rows;
    bool beam_proc_on = false;
    // prompt-lookup speculative decoding (b2_stream_begin_lookup / b2_decode_rows; allocated by the first call): SpecState, the
    // verify forward's logits fp32 [16][V], decode_attn_mq's partials and counters, a mapped host mirror of the step counters,
    // and one captured verify step per row count R. The history lives in proc_hist row 0.
    DevBuf spec_state, spec_logits, spec_attn;
    int* spec_mirror = nullptr;  // cudaHostAlloc(mapped) int[6]: SpecState::mirror
    int spec_nsplit = 0;
    int spec_R = 0;              // rows of the lookup generation in progress (0: none)
    int spec_max_new = 0;
    int spec_queued = 0;         // verify steps queued in the generation
    int spec_len0 = 0;           // cache length when it began
    std::array<cudaGraphExec_t, kSpecMaxRows + 1> spec_graph{};
    std::array<int, kSpecMaxRows + 1> spec_launches{};
    std::array<char, kSpecMaxRows + 1> spec_warm{};
    // shared-prefix decode (b2_stream_begin_groups; allocated by its first call, not counted by b2_kv_bytes): the group table
    // PrefixGroup[max_batch] then row_prefix int32 [max_batch], and decode_attn_shared's partials and counters. share_G > 0 while
    // a generation runs with the table armed; the multi-kernel step over a bf16 cache then reads it.
    DevBuf share_tab, share_attn;
    int share_G = 0;
    bool counted = false;  // included in m->kv_live
    bool e4m3() const { return dtype == B2_KV_E4M3; }
    size_t elem_bytes() const { return e4m3() ? 1 : 2; }
    size_t layer_rows() const { return (size_t)max_batch * m->d.heads * pitch; }  // = the layer stride of the scale arrays
    size_t layer_stride() const { return layer_rows() * m->hd; }                  // elements of k / v
    char* k_layer(int l) const { return k.as<char>() + (size_t)l * layer_stride() * elem_bytes(); }
    char* v_layer(int l) const { return v.as<char>() + (size_t)l * layer_stride() * elem_bytes(); }
};

namespace {

ProcState proc_state(const b2_kv* kv) {
    ProcState p = {};
    if (kv->proc_rows.p == nullptr) return p;
    p.rows = kv->proc_rows.as<ProcRow>(); p.hist = kv->proc_hist.as<int32_t>(); p.bits = kv->proc_bits.as<uint32_t>();
    p.cap = kv->max_seq + 1; p.words = (kv->m->d.vocab + 31) / 32;
    return p;
}
ProcState beam_proc_state(const b2_kv* kv) {
    ProcState p = proc_state(kv);
    p.rows = kv->beam_proc_rows.as<ProcRow>();
    return p;
}

bool starts_with(const std::string& s, const char* p) { return s.rfind(p, 0) == 0; }

// copy `n` elements of `dtype` from host-or-device `src` into bf16 device memory `dst` (contiguous)
int ingest(const void* src, int dtype, void* dst, int64_t n, cudaStream_t st) {
    if (dtype == DT_BF16) {
        B2_CUDA_CHECK(cudaMemcpyAsync(dst, src, (size_t)n * 2, cudaMemcpyDefault, st));
        B2_CUDA_CHECK(cudaStreamSynchronize(st));
        return 0;
    }
    const size_t esz = dtype == DT_F32 ? 4 : 2;
    cudaPointerAttributes attr;
    bool on_device = false;
    if (cudaPointerGetAttributes(&attr, src) == cudaSuccess)
        on_device = attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged;
    else
        cudaGetLastError();
    DevBuf tmp;
    const void* dsrc = src;
    if (!on_device) {
        B2_TRY(tmp.alloc((size_t)n * esz));
        B2_CUDA_CHECK(cudaMemcpy(tmp.p, src, (size_t)n * esz, cudaMemcpyDefault));
        dsrc = tmp.p;
    }
    int r = convert_to_bf16(dsrc, dtype, dst, n, st);
    cudaError_t e = cudaStreamSynchronize(st);
    tmp.free();
    if (r != 0) return r;
    B2_CUDA_CHECK(e);
    return 0;
}

int64_t numel(const int64_t* shape, int ndim) {
    int64_t n = 1;
    for (int i = 0; i < ndim; ++i) n *= shape[i];
    return n;
}

int expect_shape(const char* key, const int64_t* shape, int ndim, int64_t a, int64_t b = -1) {
    const int64_t n = numel(shape, ndim);
    const int64_t want = b < 0 ? a : a * b;
    bool ok = n == want;
    if (ok && b >= 0 && ndim >= 2) ok = shape[0] == a;
    if (!ok) {
        set_error("set_weight(%s): unexpected shape (numel %lld, expected %lld x %lld)", key, (long long)n,
                  (long long)a, (long long)(b < 0 ? 1 : b));
        return -1;
    }
    return 0;
}

// alloc-if-needed + ingest into dst buffer at element offset `off`
int put(DevBuf& buf, size_t total_elems, size_t off, const void* src, int dtype, int64_t n) {
    if (buf.p == nullptr) B2_TRY(buf.alloc(total_elems * 2));
    return ingest(src, dtype, buf.as<bf16>() + off, n, 0);
}

int gemm(const void* A, int lda, const void* W, int ldw, const void* bias, const void* res, int ld_res, void* out,
         int ld_out, int out_fp32, int M, int N, int K, int act, cudaStream_t st) {
    GemmArgs g;
    g.A = A; g.lda = lda; g.W = W; g.ldw = ldw; g.bias = bias; g.residual = res; g.ld_res = ld_res;
    g.out = out; g.ld_out = ld_out; g.out_fp32 = out_fp32; g.M = M; g.N = N; g.K = K; g.act = act;
    return gemm_bf16(g, st);
}

int gemv(const void* x, int64_t ldx, const void* W, int ldw, const void* gamma, float eps, const void* res,
         int ld_res, void* out, int ld_out, int out_fp32, int B, int N, int K, int act, cudaStream_t st) {
    GemvArgs g;
    g.x = x; g.ldx = ldx; g.W = W; g.ldw = ldw; g.norm_gamma = gamma; g.eps = eps; g.residual = res;
    g.ld_res = ld_res; g.out = out; g.ld_out = ld_out; g.out_fp32 = out_fp32; g.B = B; g.N = N; g.K = K;
    g.act = act;
    return gemv_bf16(g, st);
}

// Batch 7..128: below that the GEMV path (5 kernels/layer, RMSNorm fused) has fewer launches per layer than the stream-K GEMM
// path (7 kernels/layer) and wins. B2_DECODE_SKINNY=0 selects the other paths for A/B runs (GEMV kernels for B <= 8, tile GEMM
// with the batch padded to M=128 above).
bool use_skinny(const b2_kv* kv, int B) {
    if (B < 7 || B > 128 || kv->sk_partial.p == nullptr) return false;
    const char* e = getenv("B2_DECODE_SKINNY");
    return !(e != nullptr && e[0] == '0');
}

// bf16 weights of decoder layer l for the dense kernels (wgmma tile GEMMs, stream-K GEMM): the ingested buffers, or on an NF4
// model the layer's w_hat, dequantised into the model's one-layer scratch by one launch
struct LayerW { const void *wqkv, *wo, *wgu, *wd; };
int layer_weights(b2_model* m, int l, LayerW* w, cudaStream_t st) {
    LlamaLayer& L = m->ll[l];
    if (!m->nf4) { *w = {L.qkv.w.p, L.o.w.p, L.gu.w.p, L.d.w.p}; return 0; }
    const auto lin = L.linears();
    const auto sh = layer_shapes(m->d);
    Nf4Matrix mt[4];
    bf16* out = m->nf4_scratch.as<bf16>();
    for (int i = 0; i < 4; ++i) {
        mt[i].q = lin[i]->q.p; mt[i].absmax = lin[i]->a.as<float>(); mt[i].out = out; mt[i].N = sh[i].N; mt[i].K = sh[i].K;
        out += (size_t)sh[i].N * sh[i].K;
    }
    B2_TRY(dequantize_nf4(mt, 4, 1, st));
    *w = {mt[0].out, mt[1].out, mt[2].out, mt[3].out};
    return 0;
}
// NF4 decode at batch <= 8: gemv_nf4 for the seven decoder Linears when every shape fits its shared-memory budget
bool use_gemv_nf4(const b2_model* m, int B) {
    if (!m->nf4 || B > 8) return false;
    for (const LinearShape& s : layer_shapes(m->d))
        if (!gemv_nf4_fits(B, s.N, s.K, s.act)) return false;
    return true;
}

enum DecodePath { GEMV_NF4, SKINNY_FP8, GEMV, SKINNY, TILE };
struct DecodePlan { DecodePath layer, head; };
// Paths of the Linears of one multi-kernel decode step at batch B; the first row whose condition holds applies:
//   condition                                     layer Linears   head
//   use_gemv_nf4(m, B)                            GEMV_NF4        GEMV if gemv_fits(B, V, h), else TILE
//   use_skinny(kv, B) && fp8 decode               SKINNY_FP8      SKINNY_FP8
//   use_skinny(kv, B)                             SKINNY          SKINNY
//   not NF4, B <= 8, gemv_fits every shape        GEMV            GEMV
//   otherwise                                     TILE            TILE
// GEMV: tensor-core GEMV kernels. SKINNY: swap-AB stream-K GEMM over the kv-owned workspace (weights streamed once, all SMs
// busy); SKINNY_FP8 is the same GEMM on e4m3 weights x e4m3 activations. TILE: the wgmma tile GEMM. On an NF4 model SKINNY
// and TILE read the layer layer_weights dequantised.
DecodePlan decode_plan(const b2_model* m, const b2_kv* kv, int B) {
    if (use_gemv_nf4(m, B)) return {GEMV_NF4, gemv_fits(B, m->d.vocab, m->d.hidden, ACT_NONE) ? GEMV : TILE};
    if (use_skinny(kv, B)) return m->fp8_decode ? DecodePlan{SKINNY_FP8, SKINNY_FP8} : DecodePlan{SKINNY, SKINNY};
    bool small = !m->nf4 && B <= 8 && gemv_fits(B, m->d.vocab, m->d.hidden, ACT_NONE);
    for (const LinearShape& s : layer_shapes(m->d)) small = small && gemv_fits(B, s.N, s.K, s.act);
    return small ? DecodePlan{GEMV, GEMV} : DecodePlan{TILE, TILE};
}

// One Linear of the multi-kernel decode step on `path`: out[B, N] = (rmsnorm(x; gamma) or x)[B, K] · W^T, plus out itself
// when `residual` (x += ...). w_bf16 is the bf16 weight the GEMV / SKINNY / TILE paths read. GEMV and GEMV_NF4 fuse the norm;
// SKINNY and TILE normalise into xn first; SKINNY_FP8 normalises (or only quantises) into xq8 / xscale.
int decode_linear(b2_model* m, b2_kv* kv, DecodePath path, const Linear& lin, const void* w_bf16, const void* x, int ldx,
                  const void* gamma, bool residual, void* out, int ld_out, int out_fp32, int B, int N, int K, int act,
                  cudaStream_t st) {
    const float eps = gamma ? m->d.rms_eps : 0.f;
    const void* res = residual ? out : nullptr;
    const int ld_res = residual ? ld_out : 0;
    if (path == GEMV) return gemv(x, ldx, w_bf16, K, gamma, eps, res, ld_res, out, ld_out, out_fp32, B, N, K, act, st);
    if (path == GEMV_NF4) {
        GemvArgs g;
        g.x = x; g.ldx = ldx; g.norm_gamma = gamma; g.eps = eps; g.residual = res; g.ld_res = ld_res;
        g.out = out; g.ld_out = ld_out; g.out_fp32 = out_fp32; g.B = B; g.N = N; g.K = K; g.act = act;
        return gemv_nf4(g, lin.q.p, lin.a.as<float>(), st);
    }
    if (path == SKINNY_FP8) {
        if (gamma) B2_TRY(rmsnorm_quant_e4m3(x, ldx, gamma, m->xq8.p, K, m->xscale.as<float>(), B, K, eps, st));
        else B2_TRY(quantize_rows_e4m3(x, ldx, B, K, m->xq8.p, K, m->xscale.as<float>(), st));
        x = m->xq8.p;
        ldx = K;
    } else if (gamma) {
        B2_TRY(rmsnorm_bf16(x, ldx, gamma, m->xn.p, B, K, eps, st));
        x = m->xn.p;
        ldx = K;
    }
    if (path == TILE) return gemm(x, ldx, w_bf16, K, nullptr, res, ld_res, out, ld_out, out_fp32, B, N, K, act, st);
    SkinnyArgs g;
    g.x = x; g.ldx = ldx; g.W = path == SKINNY_FP8 ? lin.w8.p : w_bf16; g.ldw = K; g.residual = res; g.ld_res = ld_res;
    g.out = out; g.ld_out = ld_out; g.out_fp32 = out_fp32; g.B = B; g.N = N; g.K = K; g.act = act;
    g.partial = kv->sk_partial.as<float>(); g.partial_bytes = kv->sk_partial.bytes;
    g.counters = kv->sk_counters.as<int>();
    if (path == SKINNY) return gemm_skinny_bf16(g, st);
    g.w_scale = lin.s8.as<float>(); g.x_scale = m->xscale.as<float>();
    return gemm_skinny_fp8(g, st);
}

int decode_nsplit(int B, int H, int max_seq, int ctas_per_sm) {
    // Split-KV factor of the multi-kernel decode step. The kernel is register-limited to `occ` resident CTAs per SM, so one wave
    // is occ*SMs CTAs. Few (batch, head) pairs: fill one wave; otherwise 3 splits (short enough ranges for the tail wave to
    // overlap, few enough partials for the merge to stay cheap).
    const int cap = ctas_per_sm * num_sms();
    int n = cap / (B * H);
    if (n < 3) n = 3;
    if (n > 16) n = 16;
    const int n_hi = max_seq / 64;  // keep >= 64 keys per split at the cache's capacity
    if (n > n_hi) n = n_hi < 1 ? 1 : n_hi;
    return n;
}

// ------------------------------------------------------------------------------------------------------
// weight routing
// ------------------------------------------------------------------------------------------------------
int set_vision_weight(b2_model* m, const std::string& k, const void* ptr, const int64_t* shape, int ndim, int dt) {
    const int D = m->d.vit_hidden, I = m->d.vit_inter;
    const char* key = k.c_str();
    if (k == "embeddings.class_embedding") {
        B2_TRY(expect_shape(key, shape, ndim, D));
        return put(m->cls, D, 0, ptr, dt, D);
    }
    if (k == "embeddings.patch_embedding.weight") {
        const int kk = 3 * m->d.patch_size * m->d.patch_size;
        B2_TRY(expect_shape(key, shape, ndim, D, kk));
        // [D, 3, ps, ps] -> rows of kpad (zero padded) so the TMA row pitch is a multiple of 16 B
        DevBuf tmp;
        B2_TRY(tmp.alloc((size_t)D * kk * 2));
        B2_TRY(ingest(ptr, dt, tmp.p, (int64_t)D * kk, 0));
        if (m->patch_w.p == nullptr) B2_TRY(m->patch_w.alloc((size_t)D * m->kpad * 2));
        B2_CUDA_CHECK(cudaMemset(m->patch_w.p, 0, (size_t)D * m->kpad * 2));
        B2_CUDA_CHECK(cudaMemcpy2D(m->patch_w.p, (size_t)m->kpad * 2, tmp.p, (size_t)kk * 2, (size_t)kk * 2, D,
                                   cudaMemcpyDeviceToDevice));
        return 0;
    }
    if (k == "embeddings.position_embedding.weight") {
        B2_TRY(expect_shape(key, shape, ndim, m->T, D));
        return put(m->pos, (size_t)m->T * D, 0, ptr, dt, (int64_t)m->T * D);
    }
    if (k == "embeddings.position_ids") return 0;  // buffer in old checkpoints
    if (k == "pre_layrnorm.weight") { B2_TRY(expect_shape(key, shape, ndim, D)); return put(m->pre_g, D, 0, ptr, dt, D); }
    if (k == "pre_layrnorm.bias") { B2_TRY(expect_shape(key, shape, ndim, D)); return put(m->pre_b, D, 0, ptr, dt, D); }
    if (starts_with(k, "post_layernorm.")) return 0;  // dead for select_layer=-2 (SURVEY App. B.4)
    if (starts_with(k, "encoder.layers.")) {
        int li = -1, consumed = 0;
        if (sscanf(key, "encoder.layers.%d.%n", &li, &consumed) != 1 || li < 0 || li >= m->d.vit_layers) {
            set_error("set_weight: bad vision layer index in '%s'", key);
            return -1;
        }
        if (li >= m->vit_live) return 0;  // layers above the selected hidden state are never computed
        VitLayer& L = m->vit[li];
        const std::string s = k.substr(consumed);
        if (s == "layer_norm1.weight") { B2_TRY(expect_shape(key, shape, ndim, D)); return put(L.ln1_g, D, 0, ptr, dt, D); }
        if (s == "layer_norm1.bias") { B2_TRY(expect_shape(key, shape, ndim, D)); return put(L.ln1_b, D, 0, ptr, dt, D); }
        if (s == "layer_norm2.weight") { B2_TRY(expect_shape(key, shape, ndim, D)); return put(L.ln2_g, D, 0, ptr, dt, D); }
        if (s == "layer_norm2.bias") { B2_TRY(expect_shape(key, shape, ndim, D)); return put(L.ln2_b, D, 0, ptr, dt, D); }
        const char* names[3] = {"self_attn.q_proj.", "self_attn.k_proj.", "self_attn.v_proj."};
        for (int j = 0; j < 3; ++j) {
            if (starts_with(s, names[j])) {
                if (s == std::string(names[j]) + "weight") {
                    B2_TRY(expect_shape(key, shape, ndim, D, D));
                    B2_TRY(put(L.wqkv, (size_t)3 * D * D, (size_t)j * D * D, ptr, dt, (int64_t)D * D));
                    L.qkv_w |= 1u << j;
                    return 0;
                }
                if (s != std::string(names[j]) + "bias") break;
                B2_TRY(expect_shape(key, shape, ndim, D));
                B2_TRY(put(L.bqkv, (size_t)3 * D, (size_t)j * D, ptr, dt, D));
                L.qkv_b |= 1u << j;
                return 0;
            }
        }
        if (s == "self_attn.out_proj.weight") { B2_TRY(expect_shape(key, shape, ndim, D, D)); return put(L.wo, (size_t)D * D, 0, ptr, dt, (int64_t)D * D); }
        if (s == "self_attn.out_proj.bias") { B2_TRY(expect_shape(key, shape, ndim, D)); return put(L.bo, D, 0, ptr, dt, D); }
        if (s == "mlp.fc1.weight") { B2_TRY(expect_shape(key, shape, ndim, I, D)); return put(L.w1, (size_t)I * D, 0, ptr, dt, (int64_t)I * D); }
        if (s == "mlp.fc1.bias") { B2_TRY(expect_shape(key, shape, ndim, I)); return put(L.b1, I, 0, ptr, dt, I); }
        if (s == "mlp.fc2.weight") { B2_TRY(expect_shape(key, shape, ndim, D, I)); return put(L.w2, (size_t)D * I, 0, ptr, dt, (int64_t)D * I); }
        if (s == "mlp.fc2.bias") { B2_TRY(expect_shape(key, shape, ndim, D)); return put(L.b2, D, 0, ptr, dt, D); }
    }
    set_error("set_weight: unknown vision key '%s'", key);
    return -1;
}

int set_llama_layer_weight(b2_model* m, int li, const std::string& s, const char* key, const void* ptr,
                           const int64_t* shape, int ndim, int dt) {
    const int h = m->d.hidden, I = m->d.inter;
    LlamaLayer& L = m->ll[li];
    if (m->nf4 && (starts_with(s, "self_attn.") || starts_with(s, "mlp.")) && s != "self_attn.rotary_emb.inv_freq") {
        set_error("set_weight(%s): the decoder Linears of this model are NF4 (b2_model_enable_nf4); they cannot be reloaded", key);
        return -1;
    }
    if (s == "input_layernorm.weight") { B2_TRY(expect_shape(key, shape, ndim, h)); return put(L.ln1, h, 0, ptr, dt, h); }
    if (s == "post_attention_layernorm.weight") { B2_TRY(expect_shape(key, shape, ndim, h)); return put(L.ln2, h, 0, ptr, dt, h); }
    const char* names[3] = {"self_attn.q_proj.weight", "self_attn.k_proj.weight", "self_attn.v_proj.weight"};
    for (int j = 0; j < 3; ++j) {
        if (s == names[j]) {
            B2_TRY(expect_shape(key, shape, ndim, h, h));
            B2_TRY(put(L.qkv.w, (size_t)3 * h * h, (size_t)j * h * h, ptr, dt, (int64_t)h * h));
            L.qkv_parts |= 1u << j;
            return 0;
        }
    }
    if (s == "self_attn.o_proj.weight") { B2_TRY(expect_shape(key, shape, ndim, h, h)); return put(L.o.w, (size_t)h * h, 0, ptr, dt, (int64_t)h * h); }
    if (s == "mlp.down_proj.weight") { B2_TRY(expect_shape(key, shape, ndim, h, I)); return put(L.d.w, (size_t)h * I, 0, ptr, dt, (int64_t)h * I); }
    if (s == "mlp.gate_proj.weight" || s == "mlp.up_proj.weight") {
        B2_TRY(expect_shape(key, shape, ndim, I, h));
        const bool is_gate = s == "mlp.gate_proj.weight";
        DevBuf& tmp = is_gate ? L.tmp_gate : L.tmp_up;
        B2_TRY(put(tmp, (size_t)I * h, 0, ptr, dt, (int64_t)I * h));
        (is_gate ? L.has_gate : L.has_up) = true;
        if (L.has_gate && L.has_up) {
            if (L.gu.w.p == nullptr) B2_TRY(L.gu.w.alloc((size_t)2 * I * h * 2));
            B2_TRY(interleave_gate_up(L.tmp_gate.p, L.tmp_up.p, L.gu.w.p, I, h, 0));
            B2_CUDA_CHECK(cudaStreamSynchronize(0));
            L.tmp_gate.free();
            L.tmp_up.free();
            L.has_gate = L.has_up = false;  // allow a later reload
        }
        return 0;
    }
    if (s == "self_attn.rotary_emb.inv_freq") return 0;  // buffer in 4.31-era checkpoints
    set_error("set_weight: unknown decoder key '%s'", key);
    return -1;
}

// ------------------------------------------------------------------------------------------------------
// forward passes (caller holds the model lock)
// ------------------------------------------------------------------------------------------------------
int vit_forward_chunk(b2_model* m, const void* pixels, int B, void* out_feats, cudaStream_t st) {
    const b2_model_desc& d = m->d;
    const int D = d.vit_hidden, I = d.vit_inter, H = d.vit_heads, P = m->P, T = m->T;
    const int rows = B * T;
    B2_TRY(vit_im2col(pixels, m->v_col.p, B, d.image_size, d.patch_size, m->kpad, st));
    B2_TRY(gemm(m->v_col.p, m->kpad, m->patch_w.p, m->kpad, nullptr, nullptr, 0, m->v_patch.p, D, 0, B * P, D,
                m->kpad, ACT_NONE, st));
    B2_TRY(vit_embed_ln(m->v_patch.p, m->cls.p, m->pos.p, m->pre_g.p, m->pre_b.p, m->v_hidden.p, B, P, D,
                        d.vit_ln_eps, st));
    for (int l = 0; l < m->vit_live; ++l) {
        VitLayer& L = m->vit[l];
        B2_TRY(layernorm_bf16(m->v_hidden.p, L.ln1_g.p, L.ln1_b.p, m->v_xn.p, rows, D, d.vit_ln_eps, st));
        B2_TRY(gemm(m->v_xn.p, D, L.wqkv.p, D, L.bqkv.p, nullptr, 0, m->v_qkv.p, 3 * D, 0, rows, 3 * D, D,
                    ACT_NONE, st));
        FlashArgs fa;
        bf16* qkv = m->v_qkv.as<bf16>();
        fa.q = qkv;         fa.q_bs = (int64_t)T * 3 * D; fa.q_ts = 3 * D; fa.q_hs = m->vit_hd;
        fa.k = qkv + D;     fa.k_bs = fa.q_bs; fa.k_ts = 3 * D; fa.k_hs = m->vit_hd;
        fa.v = qkv + 2 * D; fa.v_bs = fa.q_bs; fa.v_ts = 3 * D; fa.v_hs = m->vit_hd;
        fa.o = m->v_attn.p; fa.o_bs = (int64_t)T * D; fa.o_ts = D; fa.o_hs = m->vit_hd;
        fa.B = B; fa.H = H; fa.S = T; fa.D = m->vit_hd; fa.causal = 0;
        fa.scale = 1.0f / sqrtf((float)m->vit_hd);
        B2_TRY(flash_attn_bf16(fa, st));
        B2_TRY(gemm(m->v_attn.p, D, L.wo.p, D, L.bo.p, m->v_hidden.p, D, m->v_hidden.p, D, 0, rows, D, D, ACT_NONE,
                    st));
        B2_TRY(layernorm_bf16(m->v_hidden.p, L.ln2_g.p, L.ln2_b.p, m->v_xn.p, rows, D, d.vit_ln_eps, st));
        B2_TRY(gemm(m->v_xn.p, D, L.w1.p, D, L.b1.p, nullptr, 0, m->v_mlp.p, I, 0, rows, I, D, ACT_QUICK_GELU, st));
        B2_TRY(gemm(m->v_mlp.p, I, L.w2.p, I, L.b2.p, m->v_hidden.p, D, m->v_hidden.p, D, 0, rows, D, I, ACT_NONE,
                    st));
    }
    B2_TRY(vit_drop_cls(m->v_hidden.p, out_feats, B, P, D, st));
    return 0;
}

int project_rows(b2_model* m, const void* feats, int rows, void* out, cudaStream_t st) {
    const int D = m->d.vit_hidden, h = m->d.hidden;
    const int max_rows = m->d.max_images * m->P;
    for (int r0 = 0; r0 < rows; r0 += max_rows) {
        const int n = rows - r0 < max_rows ? rows - r0 : max_rows;
        const bf16* a = reinterpret_cast<const bf16*>(feats) + (size_t)r0 * D;
        bf16* o = reinterpret_cast<bf16*>(out) + (size_t)r0 * h;
        // north_star: "mm_projector as one fused GEMM->GELU->GEMM kernel" (phase-2 tiles gated on per-row-block counters)
        B2_TRY(projector_fused_bf16(a, D, m->p0_w.p, m->p0_b.p, m->p2_w.p, m->p2_b.p, m->p_mid.p, o, h, n, D, h, h,
                                    m->p_done.as<int>(), st));
    }
    return 0;
}

// Captures the kernels fn() enqueues on st and instantiates them as *exec. A capture records launches without running them:
// g_launch_count is left as it was, and *launches receives the kernel count, which the caller adds on each replay.
template <typename F>
int capture_graph(cudaStream_t st, cudaGraphExec_t* exec, int* launches, F fn) {
    cudaGraph_t graph = nullptr;
    B2_CUDA_CHECK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
    const unsigned long long launches_before = g_launch_count;
    const int r = fn();
    *launches = (int)(g_launch_count - launches_before);
    g_launch_count = launches_before;
    cudaError_t e = cudaStreamEndCapture(st, &graph);
    if (r != 0) { if (graph) cudaGraphDestroy(graph); return r; }
    B2_CUDA_CHECK(e);
    e = cudaGraphInstantiate(exec, graph, 0);
    cudaGraphDestroy(graph);
    B2_CUDA_CHECK(e);
    return 0;
}

// vision tower + projector for one chunk of n <= max_images images: pixels -> out [n*P, hidden]. First call per chunk size runs
// eagerly (function attributes, driver entry points), the second captures, later ones replay.
int encode_chunk(b2_model* m, const void* pixels, int n, void* out, cudaStream_t st) {
    const b2_model_desc& d = m->d;
    const size_t in_bytes = (size_t)n * 3 * d.image_size * d.image_size * 2, out_bytes = (size_t)n * m->P * d.hidden * 2;
    cudaStream_t run = st;
    if (st == nullptr || st == cudaStreamLegacy) {
        if (m->enc_stream == nullptr) {
            B2_CUDA_CHECK(cudaStreamCreateWithFlags(&m->enc_stream, cudaStreamNonBlocking));
            B2_CUDA_CHECK(cudaEventCreateWithFlags(&m->enc_fork, cudaEventDisableTiming));
            B2_CUDA_CHECK(cudaEventCreateWithFlags(&m->enc_join, cudaEventDisableTiming));
        }
        B2_CUDA_CHECK(cudaEventRecord(m->enc_fork, st));
        B2_CUDA_CHECK(cudaStreamWaitEvent(m->enc_stream, m->enc_fork, 0));
        run = m->enc_stream;
    }
    B2_CUDA_CHECK(cudaMemcpyAsync(m->enc_pixels.p, pixels, in_bytes, cudaMemcpyDeviceToDevice, run));
    if (!m->enc_warm[n]) {
        B2_TRY(vit_forward_chunk(m, m->enc_pixels.p, n, m->v_feats.p, run));
        B2_TRY(project_rows(m, m->v_feats.p, n * m->P, m->enc_out.p, run));
        m->enc_warm[n] = 1;
    } else {
        if (m->enc_graph[n] == nullptr)
            B2_TRY(capture_graph(run, &m->enc_graph[n], &m->enc_launches, [&] {
                B2_TRY(vit_forward_chunk(m, m->enc_pixels.p, n, m->v_feats.p, run));
                return project_rows(m, m->v_feats.p, n * m->P, m->enc_out.p, run);
            }));
        B2_CUDA_CHECK(cudaGraphLaunch(m->enc_graph[n], run));
        g_launch_count += (unsigned long long)m->enc_launches;
    }
    B2_CUDA_CHECK(cudaMemcpyAsync(out, m->enc_out.p, out_bytes, cudaMemcpyDeviceToDevice, run));
    if (run != st) {
        B2_CUDA_CHECK(cudaEventRecord(m->enc_join, run));
        B2_CUDA_CHECK(cudaStreamWaitEvent(st, m->enc_join, 0));
    }
    return 0;
}

// the counters at the front of kv->share_attn (every row of the cache, 256-byte aligned partials behind them)
size_t share_counter_bytes(const b2_kv* kv) { return ((size_t)kv->max_batch * kv->m->d.heads * sizeof(int32_t) + 255) / 256 * 256; }

// one decode step on kv-owned buffers: tok -> logits (m->logits) -> argmax -> tok, out_tokens[step], len += 1
int decode_step_launch(b2_model* m, b2_kv* kv, int B, cudaStream_t st) {
    const b2_model_desc& d = m->d;
    const int h = d.hidden, I = d.inter, H = d.heads, V = d.vocab;
    const bool shared = kv->share_G > 0 && !kv->e4m3();
    const int nsplit = decode_nsplit(B, H, kv->max_seq, kv->e4m3() ? decode_attn_e4m3_ctas_per_sm()
                                                        : shared ? decode_attn_shared_ctas_per_sm() : decode_attn_ctas_per_sm());
    const DecodePlan plan = decode_plan(m, kv, B);
    const DecodePath p = plan.layer;
    B2_TRY(embed_tokens(kv->tok.as<int32_t>(), m->embed.p, m->x.p, B, h, V, m->err_dev, st));
    for (int l = 0; l < d.layers; ++l) {
        LlamaLayer& L = m->ll[l];
        LayerW lw = {};
        if (p != GEMV_NF4) B2_TRY(layer_weights(m, l, &lw, st));
        B2_TRY(decode_linear(m, kv, p, L.qkv, lw.wqkv, m->x.p, h, L.ln1.p, false, m->qkv.p, 3 * h, 0, B, 3 * h, h, ACT_NONE, st));
        DecodeAttnArgs da;
        da.qkv = m->qkv.p;
        da.kcache = kv->k_layer(l);
        da.vcache = kv->v_layer(l);
        da.cur_len = kv->len_dev.as<int32_t>();
        da.out = m->attn.p;
        da.partial = kv->attn_partial.as<float>();
        da.counters = kv->attn_counters.as<int32_t>();
        da.B = B; da.H = H; da.D = m->hd; da.Smax = kv->pitch; da.nsplit = nsplit;
        da.theta = d.rope_theta;
        da.scale = 1.0f / sqrtf((float)m->hd);
        if (kv->e4m3()) {
            da.kscale = kv->kscale.as<float>() + (size_t)l * kv->layer_rows();
            da.vscale = kv->vscale.as<float>() + (size_t)l * kv->layer_rows();
            B2_TRY(decode_attn_e4m3(da, st));
        } else if (shared) {
            const PrefixGroup* groups = kv->share_tab.as<PrefixGroup>();
            // counters first, at a place that does not move with B and nsplit: they stay zero between launches
            da.counters = kv->share_attn.as<int32_t>();
            da.partial = reinterpret_cast<float*>(kv->share_attn.as<char>() + share_counter_bytes(kv));
            B2_TRY(decode_attn_shared_bf16(da, groups, reinterpret_cast<const int32_t*>(groups + kv->max_batch), kv->share_G, st));
        } else {
            B2_TRY(decode_attn_bf16(da, st));
        }
        B2_TRY(decode_linear(m, kv, p, L.o, lw.wo, m->attn.p, h, nullptr, true, m->x.p, h, 0, B, h, h, ACT_NONE, st));
        B2_TRY(decode_linear(m, kv, p, L.gu, lw.wgu, m->x.p, h, L.ln2.p, false, m->act.p, I, 0, B, 2 * I, h, ACT_SWIGLU, st));
        B2_TRY(decode_linear(m, kv, p, L.d, lw.wd, m->act.p, I, nullptr, true, m->x.p, h, 0, B, h, I, ACT_NONE, st));
    }
    B2_TRY(decode_linear(m, kv, plan.head, m->head, m->head.w.p, m->x.p, h, m->final_norm.p, false, m->logits.p, V, 1, B, V, h,
                         ACT_NONE, st));
    // argmax or temperature/top-k/top-p draw (device-resident SampleState), token feedback, host-ring publication and the
    // step / cache-length counters in one launch
    B2_TRY(sample_publish(m->logits.as<float>(), V, B, kv->sstate.as<SampleState>(), kv->rows_dev.as<RowState>(), kv->tok.as<int32_t>(),
                          kv->out_tokens.as<int32_t>(), kv->step_counter.as<int32_t>(), kv->len_dev.as<int32_t>(),
                          kv->ring_dev, kv->ring_cap, SP_SELECT | SP_WRITE_OUT | SP_BUMP, 0, proc_state(kv), nullptr, st));
    return 0;
}

// caller stream -> stream the decode steps run on (fork), and back (join)
int fork_stream(b2_kv* kv, cudaStream_t st, cudaStream_t* run) {
    if (st != nullptr && st != cudaStreamLegacy) { *run = st; return 0; }
    if (kv->own_stream == nullptr) {
        B2_CUDA_CHECK(cudaStreamCreateWithFlags(&kv->own_stream, cudaStreamNonBlocking));
        B2_CUDA_CHECK(cudaEventCreateWithFlags(&kv->ev_fork, cudaEventDisableTiming));
        B2_CUDA_CHECK(cudaEventCreateWithFlags(&kv->ev_join, cudaEventDisableTiming));
    }
    B2_CUDA_CHECK(cudaEventRecord(kv->ev_fork, st));
    B2_CUDA_CHECK(cudaStreamWaitEvent(kv->own_stream, kv->ev_fork, 0));
    *run = kv->own_stream;
    return 0;
}
int join_stream(b2_kv* kv, cudaStream_t st, cudaStream_t run) {
    if (run == st) return 0;
    B2_CUDA_CHECK(cudaEventRecord(kv->ev_join, run));
    B2_CUDA_CHECK(cudaStreamWaitEvent(st, kv->ev_join, 0));
    return 0;
}

// run one step, through the cached CUDA graph when possible
bool use_mega(const b2_model* m, const b2_kv* kv, int B) {
    if (kv->e4m3()) return false;  // the megakernel reads bf16 caches only: an e4m3 cache takes the multi-kernel step at every batch
    if (m->nf4) return false;      // ... and bf16 weights only
    if (!decode_mega_fits(B, m->d.hidden, m->d.inter) || m->d.layers > 48) return false;
    static int flag = -1;
    if (flag < 0) {
        const char* e = getenv("B2_DECODE_MEGA");
        flag = (e != nullptr && e[0] == '0') ? 0 : 1;
    }
    return flag == 1;
}

int decode_step_mega(b2_model* m, b2_kv* kv, int B, cudaStream_t st) {
    const b2_model_desc& d = m->d;
    MegaParams p;
    p.layers = kv->mega_layers.as<MegaLayer>();
    p.L = d.layers; p.h = d.hidden; p.I = d.inter; p.H = d.heads; p.V = d.vocab; p.B = B; p.Smax = kv->pitch;
    int ns = (num_sms() * 16) / (B * d.heads);
    p.nsplit = ns < 1 ? 1 : (ns > 64 ? 64 : ns);
    p.embed = m->embed.as<bf16>(); p.final_norm = m->final_norm.as<bf16>(); p.lm_head = m->head.w.as<bf16>();
    p.tok = kv->tok.as<int32_t>(); p.cur_len = kv->len_dev.as<int32_t>();
    p.out_tokens = kv->out_tokens.as<int32_t>(); p.step_counter = kv->step_counter.as<int32_t>();
    p.x = m->x.as<bf16>(); p.qkv = m->qkv.as<bf16>(); p.attn = m->attn.as<bf16>(); p.act = m->act.as<bf16>();
    p.logits = m->logits.as<float>();
    p.attn_partial = kv->attn_partial.as<float>(); p.attn_counters = kv->attn_counters.as<int32_t>();
    unsigned int* sync = kv->mega_sync.as<unsigned int>();
    p.bar_count = sync; p.done_count = sync + 2;
    p.bar_base = kv->mega_bar_base;
    kv->mega_bar_base += (unsigned int)(5 * d.layers + 2) * (unsigned int)num_sms();
    p.eps = d.rms_eps; p.theta = d.rope_theta;
    p.scale_log2 = (1.0f / sqrtf((float)m->hd)) * 1.4426950408889634f;
    // greedy streaming: the kernel's fused argmax publishes to the host ring itself; with do_sample (or logits processors) the
    // sample_publish launch below overrides the fused argmax (token feedback, out_tokens slot) and publishes instead
    const bool sampling = kv->samp_host.do_sample != 0 || kv->samp_host.per_row != 0 || kv->any_proc();
    if (!sampling && kv->samp_host.tag != 0) { p.sstate = kv->sstate.as<SampleState>(); p.ring = kv->ring_dev; p.ring_cap = kv->ring_cap; }
    if (kv->samp_host.per_row) p.rows = kv->rows_dev.as<RowState>();
    static int trace_mode = -1;
    if (trace_mode < 0) { const char* e = getenv("B2_MEGA_TRACE"); trace_mode = (e && e[0] != 0) ? 1 : 0; }
    if (trace_mode == 1) {
        // debug (B2_MEGA_TRACE=<file>): per-phase SM-clock timestamps of CTA 0 for one step, written to <file>
        static int steps_seen = 0;
        if (++steps_seen == 40) {
            const int n = (5 * d.layers + 2) * 4;
            DevBuf tb;
            B2_TRY(tb.alloc((size_t)n * 8));
            cudaMemset(tb.p, 0, (size_t)n * 8);
            p.trace = tb.as<long long>();
            int r = decode_mega(p, st);
            cudaStreamSynchronize(st);
            std::vector<long long> host(n);
            cudaMemcpy(host.data(), tb.p, (size_t)n * 8, cudaMemcpyDeviceToHost);
            FILE* f = fopen(getenv("B2_MEGA_TRACE"), "w");
            if (f) {
                for (int ph = 0; ph <= 5 * d.layers; ++ph)
                    fprintf(f, "%d %lld %lld %lld %lld %lld\n", ph, host[ph * 4], host[ph * 4 + 1], host[ph * 4 + 2],
                            host[ph * 4 + 3], host[(ph + 1) * 4]);
                fclose(f);
            }
            tb.free();
            return r;
        }
    }
    B2_TRY(decode_mega(p, st));
    // output rows of the token the fused argmax published (the sampling launch below writes its own)
    if (!sampling && p.ring != nullptr && kv->samp_host.out_cap > 0)
        B2_TRY(publish_rows(m->logits.as<float>(), d.vocab, B, kv->sstate.as<SampleState>(), st));
    if (sampling)
        B2_TRY(sample_publish(m->logits.as<float>(), d.vocab, B, kv->sstate.as<SampleState>(), kv->rows_dev.as<RowState>(), kv->tok.as<int32_t>(),
                              kv->out_tokens.as<int32_t>(), kv->step_counter.as<int32_t>(), kv->len_dev.as<int32_t>(),
                              kv->ring_dev, kv->ring_cap, SP_SELECT | SP_WRITE_OUT, -1, proc_state(kv), nullptr, st));
    return 0;
}

// the shared-prefix group table (b2_stream_begin_groups) := G groups armed, 0 disarmed. A change drops the captured decode graph
// and makes the next step eager, as a first step at a batch size is (it sets the shared kernel's function attributes).
static void share_arm(b2_kv* kv, int G) {
    if (kv->share_G == G) return;
    if (kv->graph) { cudaGraphExecDestroy(kv->graph); kv->graph = nullptr; kv->graph_B = 0; }
    kv->warm_B = 0;
    kv->share_G = G;
}
int decode_step_run(b2_model* m, b2_kv* kv, int B, cudaStream_t st) {
    // B <= 8: one persistent cooperative launch per token (no graph needed: launches queue asynchronously)
    if (use_mega(m, kv, B)) return decode_step_mega(m, kv, B, st);
    if (kv->warm_B != B) {
        // first step for this batch size runs eagerly: sets function attributes, resolves driver entry points
        if (kv->graph) { cudaGraphExecDestroy(kv->graph); kv->graph = nullptr; kv->graph_B = 0; }
        B2_TRY(decode_step_launch(m, kv, B, st));
        kv->warm_B = B;
        return 0;
    }
    if (kv->graph == nullptr || kv->graph_B != B) {
        if (kv->graph) { cudaGraphExecDestroy(kv->graph); kv->graph = nullptr; }
        B2_TRY(capture_graph(st, &kv->graph, &kv->graph_launches, [&] { return decode_step_launch(m, kv, B, st); }));
        kv->graph_B = B;
    }
    B2_CUDA_CHECK(cudaGraphLaunch(kv->graph, st));
    g_launch_count += (unsigned long long)kv->graph_launches;
    return 0;
}

// ---- prompt-lookup speculative decoding ----------------------------------------------------------------------------------
int32_t* spec_rows(b2_kv* kv) { return reinterpret_cast<int32_t*>(kv->spec_state.as<char>() + offsetof(SpecState, rows)); }

// The verify forward of R rows of slot `slot` (bf16 cache): tokens spec->rows -> K / V at cache rows len .. len + R - 1 of every
// layer -> logits fp32 [R, V] in kv->spec_logits. Every Linear runs at R rows on decode_plan(m, kv, R)'s path; the cache length is
// not advanced.
int rows_forward(b2_model* m, b2_kv* kv, int slot, int R, cudaStream_t st) {
    const b2_model_desc& d = m->d;
    const int h = d.hidden, I = d.inter, H = d.heads, V = d.vocab;
    const DecodePlan plan = decode_plan(m, kv, R);
    const DecodePath p = plan.layer;
    const int32_t* len = kv->len_dev.as<int32_t>() + slot;
    const size_t slot_off = (size_t)slot * H * kv->pitch * m->hd * kv->elem_bytes();
    const size_t attn_partial = decode_attn_mq_scratch_bytes(1, H, kv->spec_nsplit) - (size_t)H * sizeof(int32_t);
    B2_TRY(embed_tokens(spec_rows(kv), m->embed.p, m->x.p, R, h, V, m->err_dev, st));
    for (int l = 0; l < d.layers; ++l) {
        LlamaLayer& L = m->ll[l];
        LayerW lw = {};
        if (p != GEMV_NF4) B2_TRY(layer_weights(m, l, &lw, st));
        B2_TRY(decode_linear(m, kv, p, L.qkv, lw.wqkv, m->x.p, h, L.ln1.p, false, m->qkv.p, 3 * h, 0, R, 3 * h, h, ACT_NONE, st));
        B2_TRY(rope_kv_write(m->qkv.p, kv->k_layer(l) + slot_off, kv->v_layer(l) + slot_off, 1, R, H, m->hd, kv->pitch,
                             d.rope_theta, st, len));
        DecodeAttnArgs da;
        da.qkv = m->qkv.p;
        da.kcache = kv->k_layer(l) + slot_off;
        da.vcache = kv->v_layer(l) + slot_off;
        da.cur_len = len;
        da.out = m->attn.p;
        da.partial = kv->spec_attn.as<float>();
        da.counters = reinterpret_cast<int32_t*>(kv->spec_attn.as<char>() + attn_partial);
        da.B = 1; da.R = R; da.H = H; da.D = m->hd; da.Smax = kv->pitch; da.nsplit = kv->spec_nsplit;
        da.scale = 1.0f / sqrtf((float)m->hd);
        B2_TRY(decode_attn_mq_bf16(da, st));
        B2_TRY(decode_linear(m, kv, p, L.o, lw.wo, m->attn.p, h, nullptr, true, m->x.p, h, 0, R, h, h, ACT_NONE, st));
        B2_TRY(decode_linear(m, kv, p, L.gu, lw.wgu, m->x.p, h, L.ln2.p, false, m->act.p, I, 0, R, 2 * I, h, ACT_SWIGLU, st));
        B2_TRY(decode_linear(m, kv, p, L.d, lw.wd, m->act.p, I, nullptr, true, m->x.p, h, 0, R, h, I, ACT_NONE, st));
    }
    return decode_linear(m, kv, plan.head, m->head, m->head.w.p, m->x.p, h, m->final_norm.p, false, kv->spec_logits.p, V, 1, R, V,
                         h, ACT_NONE, st);
}

// one verify step of the lookup generation on slot 0: draft -> forward of the R rows -> acceptance (publication, history, length)
int verify_step_launch(b2_model* m, b2_kv* kv, int R, cudaStream_t st) {
    SpecState* spec = kv->spec_state.as<SpecState>();
    SampleState* sst = kv->sstate.as<SampleState>();
    B2_TRY(prompt_lookup(kv->proc_hist.as<int32_t>(), spec, sst, kv->tok.as<int32_t>(), m->d.vocab, R, st));
    B2_TRY(rows_forward(m, kv, 0, R, st));
    return sample_publish(kv->spec_logits.as<float>(), m->d.vocab, R, sst, nullptr, kv->tok.as<int32_t>(), nullptr,
                          kv->step_counter.as<int32_t>(), kv->len_dev.as<int32_t>(), kv->ring_dev, kv->ring_cap, SP_SELECT, 0,
                          proc_state(kv), nullptr, st, spec);
}

// the verify step through its CUDA graph (one per R): the first step at an R runs eagerly, the second captures, later ones replay
int verify_step_run(b2_model* m, b2_kv* kv, int R, cudaStream_t st) {
    if (!kv->spec_warm[R]) {
        B2_TRY(verify_step_launch(m, kv, R, st));
        kv->spec_warm[R] = 1;
        return 0;
    }
    if (kv->spec_graph[R] == nullptr)
        B2_TRY(capture_graph(st, &kv->spec_graph[R], &kv->spec_launches[R], [&] { return verify_step_launch(m, kv, R, st); }));
    B2_CUDA_CHECK(cudaGraphLaunch(kv->spec_graph[R], st));
    g_launch_count += (unsigned long long)kv->spec_launches[R];
    return 0;
}

// makes `dev` current for the duration of an ABI call and restores the caller's device afterwards
struct DeviceGuard {
    int prev = -1;
    explicit DeviceGuard(int dev) {
        if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
        if (prev != dev) cudaSetDevice(dev); else prev = -1;
    }
    ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
    DeviceGuard(const DeviceGuard&) = delete;
    DeviceGuard& operator=(const DeviceGuard&) = delete;
};

// Cross-stream ordering of the shared model workspaces (see b2_model::ws_event). Caller holds the model lock.
int ws_enter(b2_model* m, cudaStream_t st) {
    if (m->ws_valid && m->ws_stream != st) B2_CUDA_CHECK(cudaStreamWaitEvent(st, m->ws_event, 0));
    return 0;
}
int ws_leave(b2_model* m, cudaStream_t st) {
    B2_CUDA_CHECK(cudaEventRecord(m->ws_event, st));
    m->ws_stream = st;
    m->ws_valid = true;
    return 0;
}

}  // namespace

// ==========================================================================================================
// C ABI
// ==========================================================================================================
extern "C" {

int b2_init(int device) {
    B2_CUDA_CHECK(cudaSetDevice(device));
    cudaDeviceProp prop;
    B2_CUDA_CHECK(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9) {
        set_error("b2_init: device %d is sm_%d%d; this library only contains sm_90a code (no fallback path)", device,
                  prop.major, prop.minor);
        return -3;
    }
    return 0;
}

const char* b2_last_error(void) { return g_err; }
int b2_version(void) { return 11; }
unsigned long long b2_launch_count(void) { return g_launch_count; }

int b2_model_create(const b2_model_desc* desc, b2_model** out) {
    B2_CHECK_ARG(desc != nullptr && out != nullptr, "b2_model_create: null argument");
    const b2_model_desc& d = *desc;
    B2_CHECK_ARG(d.vit_hidden > 0 && d.vit_heads > 0 && d.vit_hidden / d.vit_heads == 64 &&
                     d.vit_hidden % 256 == 0 && d.vit_hidden <= 2048,
                 "b2_model_create: vision head_dim must be 64 and hidden a multiple of 256 (hidden=%d heads=%d)",
                 d.vit_hidden, d.vit_heads);
    B2_CHECK_ARG(d.hidden > 0 && d.heads > 0 && d.hidden / d.heads == 128 && d.hidden % 256 == 0,
                 "b2_model_create: decoder head_dim must be 128 and hidden a multiple of 256 (hidden=%d heads=%d)",
                 d.hidden, d.heads);
    B2_CHECK_ARG(d.inter % 256 == 0 && d.vit_inter % 8 == 0 && d.vocab % 8 == 0,
                 "b2_model_create: inter %% 256, vit_inter %% 8, vocab %% 8 must be 0");
    B2_CHECK_ARG(d.image_size % d.patch_size == 0, "b2_model_create: image_size not a multiple of patch_size");
    B2_CHECK_ARG(d.max_batch >= 1 && d.max_seq >= 1 && d.max_images >= 1, "b2_model_create: bad workspace sizing");
    const int live = d.vit_select_layer < 0 ? d.vit_layers + 1 + d.vit_select_layer : d.vit_select_layer;
    B2_CHECK_ARG(live >= 0 && live <= d.vit_layers, "b2_model_create: vit_select_layer %d out of range",
                 d.vit_select_layer);
    b2_model* m = new b2_model();
    m->d = d;
    cudaGetDevice(&m->device);
    const int g = d.image_size / d.patch_size;
    m->P = g * g;
    m->T = m->P + 1;
    const int kk = 3 * d.patch_size * d.patch_size;
    m->kpad = (kk + 7) / 8 * 8;
    m->vit_live = live;  // hidden_states[live] = output of encoder layer `live` (0 = embeddings)
    m->vit.resize(live);
    m->ll.resize(d.layers);
    *out = m;
    return 0;
}

int b2_model_set_weight(b2_model* m, const char* hf_key, const void* ptr, const int64_t* shape, int ndim, int dtype) {
    B2_CHECK_ARG(m && hf_key && ptr && shape, "b2_model_set_weight: null argument");
    B2_CHECK_ARG(dtype == DT_BF16 || dtype == DT_F16 || dtype == DT_F32, "b2_model_set_weight: bad dtype %d", dtype);
    std::lock_guard<std::mutex> lk(m->mu);
    DeviceGuard dg(m->device);
    std::string k(hf_key);
    const int h = m->d.hidden, V = m->d.vocab, D = m->d.vit_hidden;
    int r = -1;
    size_t pos;
    if ((pos = k.find("vision_model.")) != std::string::npos) {
        r = set_vision_weight(m, k.substr(pos + strlen("vision_model.")), ptr, shape, ndim, dtype);
    } else if (k == "model.embed_tokens.weight") {
        B2_TRY(expect_shape(hf_key, shape, ndim, V, h));
        r = put(m->embed, (size_t)V * h, 0, ptr, dtype, (int64_t)V * h);
    } else if (k == "model.norm.weight") {
        B2_TRY(expect_shape(hf_key, shape, ndim, h));
        r = put(m->final_norm, h, 0, ptr, dtype, h);
    } else if (k == "lm_head.weight") {
        B2_TRY(expect_shape(hf_key, shape, ndim, V, h));
        r = put(m->head.w, (size_t)V * h, 0, ptr, dtype, (int64_t)V * h);
    } else if (m->nf4 && (k == "model.mm_projector.0.weight" || k == "model.mm_projector.2.weight")) {
        set_error("set_weight(%s): the projector of this model holds its NF4 w_hat (b2_model_enable_nf4); it cannot be reloaded", hf_key);
        return -1;
    } else if (k == "model.mm_projector.0.weight") {
        B2_TRY(expect_shape(hf_key, shape, ndim, h, D));
        r = put(m->p0_w, (size_t)h * D, 0, ptr, dtype, (int64_t)h * D);
    } else if (k == "model.mm_projector.0.bias") {
        B2_TRY(expect_shape(hf_key, shape, ndim, h));
        r = put(m->p0_b, h, 0, ptr, dtype, h);
    } else if (k == "model.mm_projector.2.weight") {
        B2_TRY(expect_shape(hf_key, shape, ndim, h, h));
        r = put(m->p2_w, (size_t)h * h, 0, ptr, dtype, (int64_t)h * h);
    } else if (k == "model.mm_projector.2.bias") {
        B2_TRY(expect_shape(hf_key, shape, ndim, h));
        r = put(m->p2_b, h, 0, ptr, dtype, h);
    } else if (starts_with(k, "model.layers.")) {
        int li = -1, consumed = 0;
        if (sscanf(hf_key, "model.layers.%d.%n", &li, &consumed) != 1 || li < 0 || li >= m->d.layers) {
            set_error("set_weight: bad decoder layer index in '%s'", hf_key);
            return -1;
        }
        r = set_llama_layer_weight(m, li, k.substr(consumed), hf_key, ptr, shape, ndim, dtype);
    } else {
        set_error("set_weight: unknown key '%s'", hf_key);
        return -1;
    }
    return r;
}

int b2_model_finalize(b2_model* m) {
    B2_CHECK_ARG(m != nullptr, "b2_model_finalize: null model");
    std::lock_guard<std::mutex> lk(m->mu);
    DeviceGuard dg(m->device);
    const b2_model_desc& d = m->d;
    // completeness
    std::string missing;
    auto need = [&](const DevBuf& b, const char* name) {
        if (b.p == nullptr) { if (missing.size() < 600) { missing += name; missing += ' '; } }
    };
    need(m->patch_w, "patch_embedding"); need(m->cls, "class_embedding"); need(m->pos, "position_embedding");
    need(m->pre_g, "pre_layrnorm.weight"); need(m->pre_b, "pre_layrnorm.bias");
    for (size_t i = 0; i < m->vit.size(); ++i) {
        VitLayer& L = m->vit[i];
        const DevBuf* bs[12] = {&L.ln1_g, &L.ln1_b, &L.wqkv, &L.bqkv, &L.wo, &L.bo, &L.ln2_g, &L.ln2_b, &L.w1, &L.b1, &L.w2, &L.b2};
        for (int j = 0; j < 12; ++j)
            if (bs[j]->p == nullptr) { char t[64]; snprintf(t, sizeof t, "vision.layer%zu.#%d", i, j); need(*bs[j], t); }
    }
    need(m->p0_w, "mm_projector.0.weight"); need(m->p0_b, "mm_projector.0.bias");
    need(m->p2_w, "mm_projector.2.weight"); need(m->p2_b, "mm_projector.2.bias");
    need(m->embed, "embed_tokens"); need(m->final_norm, "model.norm"); need(m->head.w, "lm_head");
    for (size_t i = 0; i < m->ll.size(); ++i) {
        LlamaLayer& L = m->ll[i];
        const DevBuf* bs[6] = {&L.ln1, &L.qkv.w, &L.o.w, &L.ln2, &L.gu.w, &L.d.w};
        for (int j = 0; j < 6; ++j)
            if (bs[j]->p == nullptr) { char t[64]; snprintf(t, sizeof t, "layers.%zu.#%d", i, j); need(*bs[j], t); }
    }
    if (!missing.empty()) {
        set_error("b2_model_finalize: missing weights: %s", missing.c_str());
        return -3;
    }
    // fused buffers are filled piecewise (q/k/v): every part must have arrived, or the buffer holds uninitialised memory
    // (gate/up is only materialised once both halves are there, so its pointer check above is already exact)
    for (size_t i = 0; i < m->vit.size(); ++i)
        if (m->vit[i].qkv_w != 7u || m->vit[i].qkv_b != 7u) {
            set_error("b2_model_finalize: vision layer %zu is missing q/k/v parts (weights mask %u, bias mask %u of 7)", i,
                      m->vit[i].qkv_w, m->vit[i].qkv_b);
            return -3;
        }
    for (size_t i = 0; i < m->ll.size(); ++i)
        if (m->ll[i].qkv_parts != 7u) {
            set_error("b2_model_finalize: decoder layer %zu is missing q/k/v projections (mask %u of 7)", i, m->ll[i].qkv_parts);
            return -3;
        }
    if (m->err_host == nullptr) {
        B2_CUDA_CHECK(cudaHostAlloc(reinterpret_cast<void**>(&m->err_host), 8 * sizeof(int), cudaHostAllocMapped));
        memset(m->err_host, 0, 8 * sizeof(int));
        B2_CUDA_CHECK(cudaHostGetDevicePointer(reinterpret_cast<void**>(&m->err_dev), m->err_host, 0));
        B2_CUDA_CHECK(cudaEventCreateWithFlags(&m->ws_event, cudaEventDisableTiming));
    }
    // workspaces
    const int D = d.vit_hidden, I = d.vit_inter, h = d.hidden;
    const size_t vrows = (size_t)d.max_images * m->T, prow = (size_t)d.max_images * m->P;
    B2_TRY(m->v_col.alloc(prow * m->kpad * 2));
    B2_TRY(m->v_patch.alloc(prow * D * 2));
    B2_TRY(m->v_hidden.alloc(vrows * D * 2));
    B2_TRY(m->v_xn.alloc(vrows * D * 2));
    B2_TRY(m->v_qkv.alloc(vrows * 3 * D * 2));
    B2_TRY(m->v_attn.alloc(vrows * D * 2));
    B2_TRY(m->v_mlp.alloc(vrows * I * 2));
    B2_TRY(m->v_feats.alloc(prow * D * 2));
    B2_TRY(m->p_mid.alloc(prow * h * 2));
    B2_TRY(m->p_done.alloc(((prow + 127) / 128 + 1) * sizeof(int)));
    B2_TRY(m->enc_pixels.alloc((size_t)d.max_images * 3 * d.image_size * d.image_size * 2));
    B2_TRY(m->enc_out.alloc(prow * h * 2));
    m->enc_graph.assign(d.max_images + 1, nullptr);
    m->enc_warm.assign(d.max_images + 1, 0);
    const size_t rows = (size_t)d.max_batch * d.max_seq;
    B2_TRY(m->x.alloc(rows * h * 2));
    B2_TRY(m->xn.alloc(rows * h * 2));
    B2_TRY(m->qkv.alloc(rows * 3 * h * 2));
    B2_TRY(m->attn.alloc(rows * h * 2));
    B2_TRY(m->act.alloc(rows * d.inter * 2));
    B2_TRY(m->last_idx.alloc((size_t)d.max_batch * 4));
    B2_TRY(m->chunk_pos.alloc((size_t)d.max_batch * 2 * 4));
    B2_TRY(m->splice_idx.alloc(rows * 4));
    B2_TRY(m->xlast.alloc((size_t)d.max_batch * h * 2));
    B2_TRY(m->logits.alloc((size_t)d.max_batch * d.vocab * 4));
    m->finalized = true;
    return 0;
}

int b2_model_destroy(b2_model* m) {
    if (m == nullptr) return 0;
    DeviceGuard dg(m->device);
    cudaDeviceSynchronize();
    if (m->err_host) cudaFreeHost(m->err_host);
    if (m->ws_event) cudaEventDestroy(m->ws_event);
    for (cudaGraphExec_t g : m->enc_graph) if (g) cudaGraphExecDestroy(g);
    if (m->enc_stream) cudaStreamDestroy(m->enc_stream);
    if (m->enc_fork) cudaEventDestroy(m->enc_fork);
    if (m->enc_join) cudaEventDestroy(m->enc_join);
    DevBuf* top[] = {&m->patch_w, &m->cls, &m->pos, &m->pre_g, &m->pre_b, &m->p0_w, &m->p0_b, &m->p2_w, &m->p2_b,
                     &m->embed, &m->final_norm, &m->v_col, &m->v_patch, &m->v_hidden, &m->v_xn,
                     &m->v_qkv, &m->v_attn, &m->v_mlp, &m->v_feats, &m->p_mid, &m->p_done, &m->enc_pixels, &m->enc_out, &m->x, &m->xn, &m->qkv, &m->attn,
                     &m->act, &m->last_idx, &m->chunk_pos, &m->xlast, &m->logits, &m->splice_idx, &m->xq8, &m->xscale,
                     &m->kstage, &m->vstage, &m->nf4_scratch};
    for (DevBuf* b : top) b->free();
    m->head.free();
    for (VitLayer& L : m->vit) {
        DevBuf* bs[12] = {&L.ln1_g, &L.ln1_b, &L.wqkv, &L.bqkv, &L.wo, &L.bo, &L.ln2_g, &L.ln2_b, &L.w1, &L.b1, &L.w2, &L.b2};
        for (DevBuf* b : bs) b->free();
    }
    for (LlamaLayer& L : m->ll) {
        for (DevBuf* b : {&L.ln1, &L.ln2, &L.tmp_gate, &L.tmp_up}) b->free();
        for (Linear* lin : L.linears()) lin->free();
    }
    delete m;
    return 0;
}

// BASELINE configs[4]: quantise every decode Linear to e4m3 with per-output-channel scales (the bf16 copies stay: prefill
// and the B <= 6 decode paths keep using them). Decode steps at batch >= 7 then stream 1-byte weights.
int b2_model_enable_fp8_decode(b2_model* m) {
    B2_CHECK_ARG(m != nullptr, "b2_model_enable_fp8_decode: null model");
    B2_CHECK_ARG(m->finalized, "b2_model_enable_fp8_decode: model not finalized");
    std::lock_guard<std::mutex> lk(m->mu);
    DeviceGuard dg(m->device);
    if (m->fp8_decode) return 0;
    B2_CHECK_ARG(!m->nf4, "b2_model_enable_fp8_decode: the decoder Linears are NF4 (b2_model_enable_nf4); the two formats do not combine");
    const b2_model_desc& d = m->d;
    const int h = d.hidden, I = d.inter, V = d.vocab;
    B2_CHECK_ARG(h % 16 == 0 && I % 16 == 0, "b2_model_enable_fp8_decode: hidden/inter must be multiples of 16");
    // gate/up rows stay block-64 interleaved; its scales follow the physical rows
    auto quant = [&](Linear& lin, int N, int K) -> int {
        B2_TRY(lin.w8.alloc((size_t)N * K));
        B2_TRY(lin.s8.alloc((size_t)N * sizeof(float)));
        return quantize_rows_e4m3(lin.w.p, K, N, K, lin.w8.p, K, lin.s8.as<float>(), nullptr);
    };
    const auto sh = layer_shapes(d);
    for (LlamaLayer& L : m->ll) {
        const auto lin = L.linears();
        for (int i = 0; i < 4; ++i) B2_TRY(quant(*lin[i], sh[i].N, sh[i].K));
    }
    B2_TRY(quant(m->head, V, h));
    const int mb = d.max_batch > 128 ? 128 : d.max_batch;
    B2_TRY(m->xq8.alloc((size_t)mb * (h > I ? h : I)));
    B2_TRY(m->xscale.alloc((size_t)mb * sizeof(float)));
    B2_CUDA_CHECK(cudaDeviceSynchronize());
    m->fp8_decode = true;
    return 0;
}

// load_4bit (reference llava/model/builder.py:26-41): the seven decoder Linears of every layer become NF4 (codes in GEMV order
// + fp32 absmax per 64-element block) and their bf16 buffers are freed; both projector weights are replaced by their w_hat in
// place (the projector kernels stay bf16); the one-layer dequantisation scratch of prefill and batch > 8 decode is allocated.
int b2_model_enable_nf4(b2_model* m) {
    B2_CHECK_ARG(m != nullptr, "b2_model_enable_nf4: null model");
    std::lock_guard<std::mutex> lk(m->mu);
    DeviceGuard dg(m->device);
    B2_CHECK_ARG(m->finalized, "b2_model_enable_nf4: model not finalized");
    if (m->nf4) return 0;
    B2_CHECK_ARG(!m->fp8_decode, "b2_model_enable_nf4: e4m3 decode weights are enabled (b2_model_enable_fp8_decode); the two formats do not combine");
    B2_CHECK_ARG(m->kv_live.load() == 0, "b2_model_enable_nf4: %d KV cache(s) exist; enable NF4 before creating any (the megakernel "
                 "tables of existing caches point at the bf16 weights)", m->kv_live.load());
    const b2_model_desc& d = m->d;
    const int h = d.hidden, D = d.vit_hidden;
    auto quant = [&](Linear& lin, int N, int K) -> int {
        B2_TRY(lin.q.alloc((size_t)N * K / 2));
        B2_TRY(lin.a.alloc((size_t)N * (K / 64) * sizeof(float)));
        return quantize_nf4(lin.w.p, K, N, K, lin.q.p, lin.a.as<float>(), 1, nullptr);
    };
    const auto sh = layer_shapes(d);
    size_t scratch = 0;  // elements of one dequantised layer
    for (const LinearShape& s : sh) scratch += (size_t)s.N * s.K;
    int r = 0;
    for (LlamaLayer& L : m->ll) {
        const auto lin = L.linears();
        for (int i = 0; i < 4 && r == 0; ++i) r = quant(*lin[i], sh[i].N, sh[i].K);
        if (r != 0) break;
    }
    // projector: w -> codes (canonical) -> w_hat, in place
    DevBuf pq, pa;
    // w -> codes (canonical) -> w_hat into a new buffer; the projector's own buffers are swapped in only when both succeeded
    auto roundtrip = [&](const DevBuf& w, int N, int K, DevBuf& out) -> int {
        B2_TRY(pq.alloc((size_t)N * K / 2));
        B2_TRY(pa.alloc((size_t)N * (K / 64) * sizeof(float)));
        B2_TRY(out.alloc((size_t)N * K * 2));
        B2_TRY(quantize_nf4(w.p, K, N, K, pq.p, pa.as<float>(), 0, nullptr));
        Nf4Matrix mt;
        mt.q = pq.p; mt.absmax = pa.as<float>(); mt.out = out.p; mt.N = N; mt.K = K;
        B2_TRY(dequantize_nf4(&mt, 1, 0, nullptr));
        B2_CUDA_CHECK(cudaStreamSynchronize(nullptr));
        return 0;
    };
    DevBuf p0_hat, p2_hat;
    if (r == 0) r = m->nf4_scratch.alloc(scratch * 2);
    if (r == 0 && cudaDeviceSynchronize() != cudaSuccess) { set_error("b2_model_enable_nf4: quantisation failed: %s", cudaGetErrorString(cudaGetLastError())); r = -2; }
    if (r == 0) r = roundtrip(m->p0_w, h, D, p0_hat);
    if (r == 0) r = roundtrip(m->p2_w, h, h, p2_hat);
    pq.free();
    pa.free();
    if (r != 0) {  // nothing of the model has changed yet
        for (LlamaLayer& L : m->ll)
            for (Linear* lin : L.linears()) { lin->q.free(); lin->a.free(); }
        m->nf4_scratch.free();
        p0_hat.free();
        p2_hat.free();
        return r;
    }
    std::swap(m->p0_w, p0_hat);
    std::swap(m->p2_w, p2_hat);
    p0_hat.free();  // now the bf16 originals
    p2_hat.free();
    for (LlamaLayer& L : m->ll)
        for (Linear* lin : L.linears()) lin->w.free();
    m->nf4 = true;
    return 0;
}

int64_t b2_model_weight_bytes(b2_model* m) {
    B2_CHECK_ARG(m != nullptr, "b2_model_weight_bytes: null model");
    std::lock_guard<std::mutex> lk(m->mu);
    size_t n = 0;
    for (const DevBuf* b : {&m->patch_w, &m->cls, &m->pos, &m->pre_g, &m->pre_b, &m->p0_w, &m->p0_b, &m->p2_w, &m->p2_b, &m->embed,
                            &m->final_norm})
        n += b->bytes;
    n += m->head.bytes();
    for (const VitLayer& L : m->vit)
        for (const DevBuf* b : {&L.ln1_g, &L.ln1_b, &L.wqkv, &L.bqkv, &L.wo, &L.bo, &L.ln2_g, &L.ln2_b, &L.w1, &L.b1, &L.w2, &L.b2})
            n += b->bytes;
    for (LlamaLayer& L : m->ll) {
        n += L.ln1.bytes + L.ln2.bytes;
        for (const Linear* lin : L.linears()) n += lin->bytes();
    }
    return (int64_t)n;
}

int b2_kv_create(b2_model* m, int max_batch, int max_seq, b2_kv** out) {
    return b2_kv_create_ex(m, max_batch, max_seq, B2_KV_BF16, out);
}

int b2_kv_create_ex(b2_model* m, int max_batch, int max_seq, int kv_dtype, b2_kv** out) {
    B2_CHECK_ARG(m && out, "b2_kv_create: null argument");
    B2_CHECK_ARG(kv_dtype == B2_KV_BF16 || kv_dtype == B2_KV_E4M3, "b2_kv_create: unknown kv_dtype %d (B2_KV_BF16 = 0, B2_KV_E4M3 = 1)",
                 kv_dtype);
    B2_CHECK_ARG(max_batch >= 1 && max_batch <= m->d.max_batch, "b2_kv_create: max_batch %d exceeds model max_batch %d",
                 max_batch, m->d.max_batch);
    B2_CHECK_ARG(max_seq >= 1, "b2_kv_create: max_seq must be positive");
    std::lock_guard<std::mutex> lk(m->mu);
    DeviceGuard dg(m->device);
    b2_kv* kv = new b2_kv();
    kv->m = m;
    kv->max_batch = max_batch;
    kv->max_seq = max_seq;
    kv->dtype = kv_dtype;
    kv->pitch = kv->e4m3() ? (max_seq + 3) / 4 * 4 : max_seq;  // decode_attn_e4m3 loads 4 scales as one 16-byte vector
    const size_t per = (size_t)m->d.layers * kv->layer_stride() * kv->elem_bytes();
    const size_t per_scale = kv->e4m3() ? (size_t)m->d.layers * kv->layer_rows() * sizeof(float) : 0;
    int r = 0;
    if (kv->e4m3() && m->kstage.p == nullptr) {
        const size_t stage = (size_t)m->d.max_batch * m->d.max_seq * m->d.hidden * 2;
        if ((r = m->kstage.alloc(stage)) != 0 || (r = m->vstage.alloc(stage)) != 0) {
            m->kstage.free();
            delete kv;
            return r;
        }
    }
    if ((r = kv->k.alloc(per)) != 0 || (r = kv->v.alloc(per)) != 0 ||
        (r = kv->kscale.alloc(per_scale)) != 0 || (r = kv->vscale.alloc(per_scale)) != 0 ||
        (r = kv->len_dev.alloc((size_t)max_batch * 4)) != 0 || (r = kv->tok.alloc((size_t)max_batch * 4)) != 0 ||
        (r = kv->step_counter.alloc(4)) != 0) {
        b2_kv_destroy(kv);
        return r;
    }
    kv->out_capacity = max_seq;
    const int max_split = 64;
    if (!m->nf4) {  // the megakernel reads bf16 weights; an NF4 model never takes it (use_mega)
        std::vector<MegaLayer> tbl(m->d.layers);
        for (int l = 0; l < m->d.layers; ++l) {
            LlamaLayer& L = m->ll[l];
            tbl[l].ln1 = L.ln1.as<bf16>(); tbl[l].wqkv = L.qkv.w.as<bf16>(); tbl[l].wo = L.o.w.as<bf16>();
            tbl[l].ln2 = L.ln2.as<bf16>(); tbl[l].wgu = L.gu.w.as<bf16>(); tbl[l].wd = L.d.w.as<bf16>();
            tbl[l].kcache = reinterpret_cast<bf16*>(kv->k_layer(l));  // read by the megakernel, which a bf16 cache alone reaches
            tbl[l].vcache = reinterpret_cast<bf16*>(kv->v_layer(l));
        }
        if ((r = kv->mega_layers.alloc(tbl.size() * sizeof(MegaLayer))) != 0 || (r = kv->mega_sync.alloc(64)) != 0) {
            b2_kv_destroy(kv);
            return r;
        }
        cudaMemcpy(kv->mega_layers.p, tbl.data(), tbl.size() * sizeof(MegaLayer), cudaMemcpyHostToDevice);
        cudaMemset(kv->mega_sync.p, 0, 64);
    }
    if ((r = kv->out_tokens.alloc((size_t)kv->out_capacity * max_batch * 4)) != 0 ||
        (r = kv->attn_partial.alloc(((size_t)max_batch * m->d.heads * max_split + 1024) * (128 + 2) * 4)) != 0 ||
        (r = kv->attn_counters.alloc((size_t)max_batch * m->d.heads * 4)) != 0) {
        b2_kv_destroy(kv);
        return r;
    }
    if (max_batch >= 7 && max_batch <= 128) {  // the batches use_skinny takes
        size_t ws = 0;
        int nmax = 0;
        auto fit = [&](int N, int K) {
            const size_t b = gemm_skinny_workspace_bytes(max_batch, N, K);
            ws = b > ws ? b : ws;
            nmax = N > nmax ? N : nmax;
        };
        for (const LinearShape& sh : layer_shapes(m->d)) fit(sh.N, sh.K);
        fit(m->d.vocab, m->d.hidden);
        if ((r = kv->sk_partial.alloc(ws)) != 0 || (r = kv->sk_counters.alloc(gemm_skinny_counter_bytes(nmax))) != 0) {
            b2_kv_destroy(kv);
            return r;
        }
        cudaMemset(kv->sk_counters.p, 0, gemm_skinny_counter_bytes(nmax));
    }
    kv->ring_cap = max_seq;
    if ((r = kv->sstate.alloc(sizeof(SampleState))) != 0 || (r = kv->rows_dev.alloc((size_t)max_batch * sizeof(RowState))) != 0) {
        b2_kv_destroy(kv);
        return r;
    }
    cudaMemset(kv->sstate.p, 0, sizeof(SampleState));
    cudaMemset(kv->rows_dev.p, 0, (size_t)max_batch * sizeof(RowState));
    kv->rows_host.assign(max_batch, RowState{});
    if (cudaHostAlloc(reinterpret_cast<void**>(&kv->ring_host), (size_t)kv->ring_cap * max_batch * 4, cudaHostAllocMapped) != cudaSuccess ||
        cudaHostGetDevicePointer(reinterpret_cast<void**>(&kv->ring_dev), kv->ring_host, 0) != cudaSuccess) {
        set_error("b2_kv_create: cannot allocate the pinned token ring (%d x %d)", kv->ring_cap, max_batch);
        cudaGetLastError();
        b2_kv_destroy(kv);
        return -2;
    }
    memset(kv->ring_host, 0, (size_t)kv->ring_cap * max_batch * 4);
    cudaMemset(kv->k.p, 0, per);
    cudaMemset(kv->v.p, 0, per);
    if (per_scale) { cudaMemset(kv->kscale.p, 0, per_scale); cudaMemset(kv->vscale.p, 0, per_scale); }
    cudaMemset(kv->len_dev.p, 0, (size_t)max_batch * 4);
    cudaMemset(kv->tok.p, 0, (size_t)max_batch * 4);
    cudaMemset(kv->step_counter.p, 0, 4);
    cudaMemset(kv->attn_counters.p, 0, (size_t)max_batch * m->d.heads * 4);
    if ((r = kv->rope_tab.alloc((size_t)max_seq * (m->hd / 2) * sizeof(uint32_t))) != 0 ||
        (r = rope_table_build(kv->rope_tab.p, max_seq, m->hd, m->d.rope_theta, nullptr)) != 0) {
        b2_kv_destroy(kv);
        return r;
    }
    // The memsets above run on the legacy stream; the caller's stream may be a non-blocking one (torch side streams are) and
    // is NOT ordered against it: a prefill issued right after this call would race with the zero-fill of the cache it writes
    // (seen in scripts/decode_ab.py FRESHKV=1: different tokens on a cache that was created a moment earlier).
    B2_CUDA_CHECK(cudaDeviceSynchronize());
    kv->len_host.assign(max_batch, 0);
    kv->counted = true;
    m->kv_live++;
    *out = kv;
    return 0;
}

int b2_kv_reset(b2_kv* kv) {
    B2_CHECK_ARG(kv != nullptr, "b2_kv_reset: null");
    std::lock_guard<std::mutex> lk(kv->m->mu);
    DeviceGuard dg(kv->m->device);
    // Host bookkeeping only. The device-side lengths are rewritten by the next b2_prefill and the step counter by the next
    // decode call, both on the CALLER's stream; a cudaMemset here would run on the legacy stream, unordered against work
    // still in flight on a non-blocking caller stream (e.g. two forward() calls issued back to back).
    kv->len_host.assign(kv->max_batch, 0);
    share_arm(kv, 0);  // the table names prefix lengths of the contents just dropped
    {   // measurement knob: drop the captured decode graph so that the next run starts with an eager step + a new capture
        const char* e = getenv("B2_KV_RESET_GRAPH");
        if (e != nullptr && e[0] == '1') {
            if (kv->graph) { cudaGraphExecDestroy(kv->graph); kv->graph = nullptr; kv->graph_B = 0; }
            kv->warm_B = 0;
        }
    }
    return 0;
}

int b2_kv_destroy(b2_kv* kv) {
    if (kv == nullptr) return 0;
    DeviceGuard dg(kv->m->device);
    cudaDeviceSynchronize();
    if (kv->counted) kv->m->kv_live--;
    if (kv->ring_host) cudaFreeHost(kv->ring_host);
    if (kv->graph) cudaGraphExecDestroy(kv->graph);
    for (cudaGraphExec_t g : kv->spec_graph) if (g) cudaGraphExecDestroy(g);
    if (kv->spec_mirror) cudaFreeHost(kv->spec_mirror);
    if (kv->own_stream) cudaStreamDestroy(kv->own_stream);
    if (kv->ev_fork) cudaEventDestroy(kv->ev_fork);
    if (kv->ev_join) cudaEventDestroy(kv->ev_join);
    DevBuf* bs[] = {&kv->k, &kv->v, &kv->kscale, &kv->vscale, &kv->len_dev, &kv->tok, &kv->step_counter, &kv->out_tokens, &kv->attn_partial,
                    &kv->attn_counters, &kv->mega_layers, &kv->mega_sync, &kv->sk_partial, &kv->sk_counters, &kv->sstate, &kv->rows_dev, &kv->rope_tab,
                    &kv->beam_in, &kv->beam_ws, &kv->beam_out, &kv->proc_rows, &kv->proc_hist, &kv->proc_bits,
                    &kv->beam_proc_rows, &kv->spec_state, &kv->spec_logits, &kv->spec_attn};
    for (DevBuf* b : bs) b->free();
    delete kv;
    return 0;
}

int b2_kv_dtype(b2_kv* kv) {
    B2_CHECK_ARG(kv != nullptr, "b2_kv_dtype: null");
    return kv->dtype;
}

int64_t b2_kv_bytes(b2_kv* kv) {
    B2_CHECK_ARG(kv != nullptr, "b2_kv_bytes: null");
    return (int64_t)(kv->k.bytes + kv->v.bytes + kv->kscale.bytes + kv->vscale.bytes);
}

int b2_kv_lengths(b2_kv* kv, int32_t* lens_host, int n) {
    B2_CHECK_ARG(kv && lens_host && n >= 0 && n <= kv->max_batch, "b2_kv_lengths: bad argument");
    for (int i = 0; i < n; ++i) lens_host[i] = kv->len_host[i];
    return 0;
}

// ---------------------------------------------------------------------------------------------------------
int b2_vit_encode(b2_model* m, const void* pixels, int B, void* out_feats, void* stream) {
    B2_CHECK_ARG(m && pixels && out_feats && B >= 1, "b2_vit_encode: bad argument");
    B2_CHECK_ARG(m->finalized, "b2_vit_encode: model not finalized");
    std::lock_guard<std::mutex> lk(m->mu);
    DeviceGuard dg(m->device);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    B2_TRY(ws_enter(m, st));
    const size_t img_elems = (size_t)3 * m->d.image_size * m->d.image_size;
    for (int b0 = 0; b0 < B; b0 += m->d.max_images) {
        const int n = B - b0 < m->d.max_images ? B - b0 : m->d.max_images;
        B2_TRY(vit_forward_chunk(m, reinterpret_cast<const bf16*>(pixels) + b0 * img_elems, n,
                                 reinterpret_cast<bf16*>(out_feats) + (size_t)b0 * m->P * m->d.vit_hidden, st));
    }
    return ws_leave(m, st);
}

int b2_project(b2_model* m, const void* feats, int rows, void* out, void* stream) {
    B2_CHECK_ARG(m && feats && out && rows >= 1, "b2_project: bad argument");
    B2_CHECK_ARG(m->finalized, "b2_project: model not finalized");
    std::lock_guard<std::mutex> lk(m->mu);
    DeviceGuard dg(m->device);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    B2_TRY(ws_enter(m, st));
    B2_TRY(project_rows(m, feats, rows, out, st));
    return ws_leave(m, st);
}

int b2_encode_images(b2_model* m, const void* pixels, int B, void* out, void* stream) {
    B2_CHECK_ARG(m && pixels && out && B >= 1, "b2_encode_images: bad argument");
    B2_CHECK_ARG(m->finalized, "b2_encode_images: model not finalized");
    std::lock_guard<std::mutex> lk(m->mu);
    DeviceGuard dg(m->device);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    B2_TRY(ws_enter(m, st));
    const size_t img_elems = (size_t)3 * m->d.image_size * m->d.image_size;
    for (int b0 = 0; b0 < B; b0 += m->d.max_images) {
        const int n = B - b0 < m->d.max_images ? B - b0 : m->d.max_images;
        B2_TRY(encode_chunk(m, reinterpret_cast<const bf16*>(pixels) + b0 * img_elems, n,
                            reinterpret_cast<bf16*>(out) + (size_t)b0 * m->P * m->d.hidden, st));
    }
    return ws_leave(m, st);
}

int b2_splice(b2_model* m, const int32_t* src_index, const void* image_feats, int n_feat_rows, int rows, void* embeds_out,
              void* stream) {
    B2_CHECK_ARG(m && src_index && embeds_out && rows >= 1 && n_feat_rows >= 0, "b2_splice: bad argument");
    B2_CHECK_ARG(image_feats != nullptr || n_feat_rows == 0, "b2_splice: n_feat_rows=%d without image_feats", n_feat_rows);
    B2_CHECK_ARG(m->finalized, "b2_splice: model not finalized");
    std::lock_guard<std::mutex> lk(m->mu);
    DeviceGuard dg(m->device);
    return splice_embed(src_index, m->embed.p, image_feats, embeds_out, rows, m->d.hidden, m->d.vocab, n_feat_rows,
                        m->err_dev, reinterpret_cast<cudaStream_t>(stream));
}

int b2_splice_ids(b2_model* m, const int64_t* input_ids, int B, int Lt, int k_per_row, const int32_t* feat_offsets_host, int n_img,
                  const void* image_feats, int S, void* embeds_out, void* stream) {
    B2_CHECK_ARG(m && input_ids && feat_offsets_host && embeds_out, "b2_splice_ids: null argument");
    B2_CHECK_ARG(m->finalized, "b2_splice_ids: model not finalized");
    B2_CHECK_ARG(B >= 1 && S >= 1 && (size_t)B * S <= (size_t)m->d.max_batch * m->d.max_seq,
                 "b2_splice_ids: B*S=%d exceeds the workspace (%d rows)", B * S, m->d.max_batch * m->d.max_seq);
    B2_CHECK_ARG(image_feats != nullptr || n_img == 0, "b2_splice_ids: image slots without image_feats");
    std::lock_guard<std::mutex> lk(m->mu);
    DeviceGuard dg(m->device);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    B2_TRY(ws_enter(m, st));
    B2_TRY(splice_index(reinterpret_cast<const long long*>(input_ids), B, Lt, k_per_row, feat_offsets_host, n_img, -200, S,
                        m->splice_idx.as<int32_t>(), m->err_dev, st));
    B2_TRY(splice_embed(m->splice_idx.as<int32_t>(), m->embed.p, image_feats, embeds_out, B * S, m->d.hidden, m->d.vocab,
                        n_img > 0 ? feat_offsets_host[n_img] : 0, m->err_dev, st));
    return ws_leave(m, st);
}

int b2_async_error(b2_model* m, int* code_out) {
    B2_CHECK_ARG(m && code_out, "b2_async_error: null argument");
    int code = 0;
    if (m->err_host != nullptr)
        for (int i = 0; i < 8; ++i)
            if (reinterpret_cast<volatile int*>(m->err_host)[i] != 0) {
                code |= 1 << i;
                reinterpret_cast<volatile int*>(m->err_host)[i] = 0;
            }
    *code_out = code;
    if (code != 0)
        set_error("device-side input check failed:%s%s%s", (code & B2_ERR_TOKEN_RANGE) ? " token id outside [0, vocab) (or an image placeholder without image features)" : "",
                  (code & B2_ERR_IMAGE_ROW_RANGE) ? " image-feature row outside the encoded images" : "",
                  (code & B2_ERR_SPLICE_SLOTS) ? " more image placeholders than images" : "");
    return 0;
}

int b2_prefill(b2_model* m, b2_kv* kv, const void* embeds, const int32_t* seq_lens_host, int B, int S,
               void* logits_out, int logits_mode, void* stream) {
    return b2_prefill_at(m, kv, embeds, nullptr, seq_lens_host, B, S, 0, logits_out, logits_mode, stream);
}

int b2_prefill_slots(b2_model* m, b2_kv* kv, const void* embeds, const int32_t* seq_lens_host, int B, int S, int slot0,
                     void* logits_out, int logits_mode, void* stream) {
    return b2_prefill_at(m, kv, embeds, nullptr, seq_lens_host, B, S, slot0, logits_out, logits_mode, stream);
}

int b2_prefill_at(b2_model* m, b2_kv* kv, const void* embeds, const int32_t* start_host, const int32_t* seq_lens_host, int B,
                  int S, int slot0, void* logits_out, int logits_mode, void* stream) {
    B2_CHECK_ARG(m && kv && embeds && kv->m == m, "b2_prefill: bad handle");
    B2_CHECK_ARG(m->finalized, "b2_prefill: model not finalized");
    B2_CHECK_ARG(B >= 1 && slot0 >= 0 && slot0 + B <= kv->max_batch && S >= 1 && S <= kv->max_seq,
                 "b2_prefill: B=%d S=%d slot0=%d exceed the KV cache (max_batch=%d max_seq=%d)", B, S, slot0, kv->max_batch, kv->max_seq);
    B2_CHECK_ARG((size_t)B * S <= (size_t)m->d.max_batch * m->d.max_seq,
                 "b2_prefill: B*S=%d exceeds the workspace (%d rows)", B * S, m->d.max_batch * m->d.max_seq);
    B2_CHECK_ARG(logits_mode == B2_LOGITS_NONE || logits_out != nullptr, "b2_prefill: logits_out is null");
    std::lock_guard<std::mutex> lk(m->mu);
    DeviceGuard dg(m->device);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const b2_model_desc& d = m->d;
    const int h = d.hidden, I = d.inter, H = d.heads, V = d.vocab, T = B * S;

    std::vector<int32_t> lens(B), last(B), start(B, 0), total(B);
    int max_start = 0;
    for (int b = 0; b < B; ++b) {
        lens[b] = seq_lens_host ? seq_lens_host[b] : S;
        B2_CHECK_ARG(lens[b] >= 1 && lens[b] <= S, "b2_prefill: seq_lens[%d]=%d out of range (S=%d)", b, lens[b], S);
        if (start_host != nullptr) {
            start[b] = start_host[b];
            B2_CHECK_ARG(start[b] >= 0 && start[b] <= kv->len_host[slot0 + b],
                         "b2_prefill_at: start[%d]=%d outside [0, current length %d]", b, start[b], kv->len_host[slot0 + b]);
            B2_CHECK_ARG(start[b] + lens[b] <= kv->max_seq, "b2_prefill_at: start[%d]=%d + %d tokens exceed the cache (max_seq=%d)",
                         b, start[b], lens[b], kv->max_seq);
        }
        max_start = start[b] > max_start ? start[b] : max_start;
        total[b] = start[b] + lens[b];
        last[b] = b * S + lens[b] - 1;
    }
    // a chunk at position 0 everywhere is an ordinary prefill (the same kernels, bit for bit)
    const bool offset = max_start > 0;
    const bool q8 = kv->e4m3();
    // e4m3 cache: the producers below write one layer of roped bf16 K / V into the staging slab [B][H][kv_pitch][128] (a cache
    // with Smax = kv_pitch), attention reads it there, and kv_quantize_e4m3 then stores the layer's chunk rows and scales. At an
    // offset the slab also holds the stored prefix, dequantised (rows [0, start)), in front of the chunk's rows.
    const int kv_pitch = !q8 ? kv->pitch : (offset ? (max_start + S < kv->max_seq ? max_start + S : kv->max_seq) : S);
    B2_CHECK_ARG(!q8 || (size_t)B * kv_pitch <= (size_t)d.max_batch * d.max_seq,
                 "b2_prefill_at: %d samples x %d rows exceed the staging slab (%d rows)", B, kv_pitch, d.max_batch * d.max_seq);
    B2_TRY(ws_enter(m, st));
    // lengths / last-row indices travel as kernel parameters: no pinned staging, no stream sync in this call
    B2_TRY(set_i32_pairs(kv->len_dev.as<int32_t>() + slot0, total.data(), m->last_idx.as<int32_t>(), last.data(), B, st));
    int32_t* pos_dev = m->chunk_pos.as<int32_t>();  // [0, B): start, [max_batch, +B): chunk length
    int32_t* clen_dev = pos_dev + d.max_batch;
    if (offset) B2_TRY(set_i32_pairs(pos_dev, start.data(), clen_dev, lens.data(), B, st));
    for (int b = 0; b < B; ++b) kv->len_host[slot0 + b] = total[b];
    const size_t slot_rows = (size_t)slot0 * H * kv->pitch;  // cache rows in front of the first slot this call fills

    B2_CUDA_CHECK(cudaMemcpyAsync(m->x.p, embeds, (size_t)T * h * 2, cudaMemcpyDeviceToDevice, st));
    // RoPE + KV write fused into the QKV GEMM where the CTA-pair kernel is the one that runs anyway (M >= 512; 256-column pair
    // tiles must hold whole 128-wide heads of ONE of q / k / v: hidden % 256 == 0). B2_ROPE_FUSED=0: standalone pass (A/B, tests).
    bool rope_fused = T >= 512 && m->hd == 128 && h % 256 == 0;
    { const char* e = getenv("B2_ROPE_FUSED"); if (e != nullptr && e[0] == '0') rope_fused = false; }
    for (int l = 0; l < d.layers; ++l) {
        LlamaLayer& L = m->ll[l];
        LayerW lw;
        B2_TRY(layer_weights(m, l, &lw, st));
        bf16* kc = q8 ? m->kstage.as<bf16>() : reinterpret_cast<bf16*>(kv->k_layer(l)) + slot_rows * m->hd;
        bf16* vc = q8 ? m->vstage.as<bf16>() : reinterpret_cast<bf16*>(kv->v_layer(l)) + slot_rows * m->hd;
        const size_t row0 = (size_t)l * kv->layer_rows() + slot_rows;  // e4m3: first scale / row of this layer's slots
        if (q8 && offset)
            B2_TRY(kv_dequantize_e4m3(kv->k.as<uint8_t>() + row0 * m->hd, kv->v.as<uint8_t>() + row0 * m->hd,
                                      kv->kscale.as<float>() + row0, kv->vscale.as<float>() + row0, pos_dev, kc, vc, B, H,
                                      kv->pitch, kv_pitch, st));
        B2_TRY(rmsnorm_bf16(m->x.p, h, L.ln1.p, m->xn.p, T, h, d.rms_eps, st));
        if (rope_fused) {
            // QKV projection with RoPE and the cache write in its epilogue (CTA-pair kernel): q -> qkv buffer, k / v -> cache
            GemmArgs g;
            g.A = m->xn.p; g.lda = h; g.W = lw.wqkv; g.ldw = h; g.out = m->qkv.p; g.ld_out = 3 * h;
            g.M = T; g.N = 3 * h; g.K = h; g.act = ACT_ROPE_QKV;
            g.rope.table = kv->rope_tab.p; g.rope.kcache = kc; g.rope.vcache = vc; g.rope.S = S; g.rope.H = H; g.rope.Smax = kv_pitch;
            g.rope.pos0 = offset ? pos_dev : nullptr;
            B2_TRY(gemm_bf16_2cta(g, st));
        } else {
            B2_TRY(gemm(m->xn.p, h, lw.wqkv, h, nullptr, nullptr, 0, m->qkv.p, 3 * h, 0, T, 3 * h, h, ACT_NONE, st));
            B2_TRY(rope_kv_write(m->qkv.p, kc, vc, B, S, H, m->hd, kv_pitch, d.rope_theta, st, offset ? pos_dev : nullptr));
        }
        FlashArgs fa;
        fa.q = m->qkv.p; fa.q_bs = (int64_t)S * 3 * h; fa.q_ts = 3 * h; fa.q_hs = m->hd;
        fa.k = kc; fa.k_bs = (int64_t)H * kv_pitch * m->hd; fa.k_ts = m->hd; fa.k_hs = (int64_t)kv_pitch * m->hd;
        fa.v = vc; fa.v_bs = fa.k_bs; fa.v_ts = m->hd; fa.v_hs = fa.k_hs;
        fa.o = m->attn.p; fa.o_bs = (int64_t)S * h; fa.o_ts = h; fa.o_hs = m->hd;
        fa.seq_lens = offset ? clen_dev : kv->len_dev.as<int32_t>() + slot0;
        if (offset) { fa.pos0 = pos_dev; fa.Skv = kv_pitch; }
        fa.B = B; fa.H = H; fa.S = S; fa.D = m->hd; fa.causal = 1;
        fa.scale = 1.0f / sqrtf((float)m->hd);
        B2_TRY(flash_attn_bf16(fa, st));
        if (q8) {
            B2_TRY(kv_quantize_e4m3(kc, vc, kv->k.as<uint8_t>() + row0 * m->hd, kv->v.as<uint8_t>() + row0 * m->hd,
                                    kv->kscale.as<float>() + row0, kv->vscale.as<float>() + row0,
                                    offset ? clen_dev : kv->len_dev.as<int32_t>() + slot0, B, S, H, m->hd, kv->pitch, st,
                                    offset ? pos_dev : nullptr, kv_pitch));
        }
        B2_TRY(gemm(m->attn.p, h, lw.wo, h, nullptr, m->x.p, h, m->x.p, h, 0, T, h, h, ACT_NONE, st));
        B2_TRY(rmsnorm_bf16(m->x.p, h, L.ln2.p, m->xn.p, T, h, d.rms_eps, st));
        B2_TRY(gemm(m->xn.p, h, lw.wgu, h, nullptr, nullptr, 0, m->act.p, I, 0, T, 2 * I, h, ACT_SWIGLU, st));
        B2_TRY(gemm(m->act.p, I, lw.wd, I, nullptr, m->x.p, h, m->x.p, h, 0, T, h, I, ACT_NONE, st));
    }
    if (logits_mode == B2_LOGITS_LAST) {
        // only the last valid position per sample feeds generation (the reference computes lm_head on all S)
        B2_TRY(rmsnorm_gather_bf16(m->x.p, m->last_idx.as<int32_t>(), m->final_norm.p, m->xlast.p, B, h, d.rms_eps, st));
        if (B <= 8 && gemv_fits(B, V, h, ACT_NONE))
            B2_TRY(gemv(m->xlast.p, h, m->head.w.p, h, nullptr, 0.f, nullptr, 0, logits_out, V, 1, B, V, h, ACT_NONE, st));
        else
            B2_TRY(gemm(m->xlast.p, h, m->head.w.p, h, nullptr, nullptr, 0, logits_out, V, 1, B, V, h, ACT_NONE, st));
    } else if (logits_mode == B2_LOGITS_ALL) {
        B2_TRY(rmsnorm_bf16(m->x.p, h, m->final_norm.p, m->xn.p, T, h, d.rms_eps, st));
        B2_TRY(gemm(m->xn.p, h, m->head.w.p, h, nullptr, nullptr, 0, logits_out, V, 1, T, V, h, ACT_NONE, st));
    }
    return ws_leave(m, st);
}

static int copy_tokens_in(b2_kv* kv, const int32_t* tokens, int B, cudaStream_t st) {
    B2_CUDA_CHECK(cudaMemcpyAsync(kv->tok.p, tokens, (size_t)B * 4, cudaMemcpyDefault, st));
    return 0;
}

// device-resident selection state := v (pub_counter restarts at 0); launched only when something changed
static int set_sampling(b2_kv* kv, const SampleState& v, bool force, cudaStream_t st) {
    const SampleState& c = kv->samp_host;
    if (!force && kv->samp_valid && c.do_sample == v.do_sample && c.temperature == v.temperature && c.top_p == v.top_p &&
        c.top_k == v.top_k && c.seed == v.seed && c.tag == v.tag && c.per_row == v.per_row && c.out_scores == v.out_scores &&
        c.out_logits == v.out_logits && c.out_cap == v.out_cap)
        return 0;
    B2_TRY(sample_state_set(kv->sstate.as<SampleState>(), v, st));
    kv->samp_host = v;
    kv->samp_valid = true;
    return 0;
}
// every slot selects from its raw logits again (a no-op on a cache whose processors are off); beam processing is disarmed
// unless keep_beam (the step of a processed beam search itself), and so is the shared-prefix group table
static int proc_all_off(b2_kv* kv, cudaStream_t st, bool keep_beam = false) {
    share_arm(kv, 0);
    if (!keep_beam) kv->beam_proc_on = false;
    if (!kv->any_proc()) return 0;
    B2_CUDA_CHECK(cudaMemsetAsync(kv->proc_rows.p, 0, kv->proc_rows.bytes, st));
    kv->proc_on.assign(kv->max_batch, 0);
    return 0;
}
static int set_greedy_unpublished(b2_kv* kv, cudaStream_t st, bool keep_beam = false) {
    SampleState v = {};
    v.temperature = 1.f; v.top_p = 1.f;
    kv->stream_B = 0;  // any streaming generation on this cache is over
    kv->spec_R = 0;
    B2_TRY(proc_all_off(kv, st, keep_beam));
    return set_sampling(kv, v, false, st);
}
// b2_logits_proc -> ProcRow (on = 0 when every processor is at its off value); prompt ids are checked against `cap`
static int proc_row_of(const b2_logits_proc* lp, int cap, ProcRow* out, const char* who) {
    *out = ProcRow{};
    out->penalty = 1.f;
    if (lp == nullptr) return 0;
    B2_CHECK_ARG(lp->repetition_penalty > 0.f && lp->repetition_penalty < INFINITY, "%s: repetition_penalty must be positive and finite (got %g)",
                 who, (double)lp->repetition_penalty);
    B2_CHECK_ARG(lp->no_repeat_ngram_size >= 0, "%s: no_repeat_ngram_size must be >= 0 (got %d)", who, lp->no_repeat_ngram_size);
    B2_CHECK_ARG(lp->n_eos >= 0 && lp->n_eos <= kProcMaxEos, "%s: n_eos must be in [0, %d] (got %d)", who, kProcMaxEos, lp->n_eos);
    B2_CHECK_ARG(lp->prompt_len >= 0 && (lp->prompt_len == 0 || lp->prompt_ids != nullptr), "%s: bad prompt ids", who);
    out->penalty = lp->repetition_penalty;
    out->ngram = lp->no_repeat_ngram_size;
    out->n_eos = lp->n_eos;
    for (int i = 0; i < lp->n_eos; ++i) out->eos[i] = lp->eos_ids[i];
    out->min_gen = lp->n_eos > 0 && lp->min_generated > 0 ? lp->min_generated : 0;
    out->on = (out->penalty != 1.f || out->ngram > 0 || out->min_gen > 0) ? 1 : 0;
    out->prompt_len = lp->prompt_len;
    out->hist_len = lp->prompt_len;
    B2_CHECK_ARG(!out->on || lp->prompt_len + 1 <= cap, "%s: prompt of %d ids exceeds the history capacity %d", who, lp->prompt_len, cap);
    return 0;
}
// the cache's processing state, allocated on first use; a decode graph captured before then does not read it and is dropped.
// Every row starts off, zeroed on the caller's stream `st`: the seeding and the decode steps that read the state are ordered
// after it there, which a memset on the legacy stream would not be when `st` is a non-blocking stream.
static int proc_alloc(b2_kv* kv, cudaStream_t st) {
    if (kv->proc_rows.p != nullptr) return 0;
    const size_t words = (size_t)(kv->m->d.vocab + 31) / 32;
    int r = kv->proc_rows.alloc((size_t)kv->max_batch * sizeof(ProcRow));
    if (r == 0) r = kv->proc_hist.alloc((size_t)kv->max_batch * (kv->max_seq + 1) * sizeof(int32_t));
    if (r == 0) r = kv->proc_bits.alloc((size_t)kv->max_batch * words * sizeof(uint32_t));
    if (r == 0 && cudaMemsetAsync(kv->proc_rows.p, 0, kv->proc_rows.bytes, st) != cudaSuccess) {
        set_error("proc_alloc: %s", cudaGetErrorString(cudaGetLastError()));
        r = -2;
    }
    if (r != 0) {  // all or nothing: proc_rows != nullptr means the whole state exists
        kv->proc_rows.free(); kv->proc_hist.free(); kv->proc_bits.free();
        return r;
    }
    kv->proc_on.assign(kv->max_batch, 0);
    if (kv->graph) { cudaGraphExecDestroy(kv->graph); kv->graph = nullptr; kv->graph_B = 0; }
    return 0;
}
// slot `row` := v; its history seeded from the prompt ids (and first_token when >= 0) when v is on
static int proc_set_row(b2_kv* kv, int row, const ProcRow& v, const int64_t* ids, int first_token, cudaStream_t st) {
    if (!v.on) {
        if (kv->proc_rows.p != nullptr && kv->proc_on[row]) {
            B2_CUDA_CHECK(cudaMemsetAsync(kv->proc_rows.as<ProcRow>() + row, 0, sizeof(ProcRow), st));
            kv->proc_on[row] = 0;
        }
        return 0;
    }
    B2_TRY(proc_alloc(kv, st));
    ProcRow r = v;
    if (first_token >= 0) r.hist_len += 1;
    B2_TRY(proc_seed(proc_state(kv), row, r, ids, v.prompt_len, first_token, kv->m->d.vocab, st));
    kv->proc_on[row] = 1;
    return 0;
}
// The lookup state of a bf16 cache, allocated on first use (b2_kv_bytes does not count it), and a stream-K workspace for R rows
// when decode_plan takes SKINNY there. A workspace that grows is reallocated, so graphs captured over the old one are dropped.
static int spec_alloc(b2_model* m, b2_kv* kv, int R, cudaStream_t st) {
    B2_CHECK_ARG(!kv->e4m3(), "prompt lookup: the verify step reads a bf16 KV cache (this one is e4m3)");
    B2_CHECK_ARG(R >= 1 && R <= kSpecMaxRows, "prompt lookup: %d rows per step (1..%d)", R, kSpecMaxRows);
    B2_CHECK_ARG(!m->fp8_decode || R <= m->d.max_batch, "prompt lookup: %d rows exceed the e4m3 activation buffer (model max_batch %d)",
                 R, m->d.max_batch);
    B2_TRY(proc_alloc(kv, st));
    if (kv->spec_state.p == nullptr) {
        const int H = m->d.heads;
        const int nsplit = decode_nsplit(1, H, kv->max_seq, decode_attn_mq_ctas_per_sm());
        const size_t attn = decode_attn_mq_scratch_bytes(1, H, nsplit);
        int r = kv->spec_state.alloc(sizeof(SpecState));
        if (r == 0) r = kv->spec_logits.alloc((size_t)kSpecMaxRows * m->d.vocab * sizeof(float));
        if (r == 0) r = kv->spec_attn.alloc(attn);
        if (r == 0 && (cudaHostAlloc(reinterpret_cast<void**>(&kv->spec_mirror), 6 * sizeof(int), cudaHostAllocMapped) != cudaSuccess ||
                       cudaMemsetAsync(kv->spec_attn.p, 0, attn, st) != cudaSuccess)) {
            set_error("prompt lookup: %s", cudaGetErrorString(cudaGetLastError()));
            r = -2;
        }
        if (r != 0) {
            kv->spec_state.free(); kv->spec_logits.free(); kv->spec_attn.free();
            if (kv->spec_mirror) { cudaFreeHost(kv->spec_mirror); kv->spec_mirror = nullptr; }
            return r;
        }
        memset(kv->spec_mirror, 0, 6 * sizeof(int));
        kv->spec_nsplit = nsplit;
    }
    if (R >= 7) {  // use_skinny's batches: the stream-K GEMM needs its workspace at R rows
        size_t ws = 0;
        int nmax = 0;
        for (const LinearShape& sh : layer_shapes(m->d)) { ws = std::max(ws, gemm_skinny_workspace_bytes(R, sh.N, sh.K)); nmax = std::max(nmax, sh.N); }
        ws = std::max(ws, gemm_skinny_workspace_bytes(R, m->d.vocab, m->d.hidden));
        nmax = std::max(nmax, m->d.vocab);
        if (kv->sk_partial.bytes < ws || kv->sk_counters.bytes < gemm_skinny_counter_bytes(nmax)) {
            B2_CUDA_CHECK(cudaStreamSynchronize(st));
            if (kv->graph) { cudaGraphExecDestroy(kv->graph); kv->graph = nullptr; kv->graph_B = 0; }
            for (cudaGraphExec_t& g : kv->spec_graph) if (g) { cudaGraphExecDestroy(g); g = nullptr; }
            const size_t cb = gemm_skinny_counter_bytes(nmax);
            kv->sk_partial.free(); kv->sk_counters.free();
            int r = kv->sk_partial.alloc(ws);
            if (r == 0) r = kv->sk_counters.alloc(cb);
            if (r != 0) { kv->sk_partial.free(); kv->sk_counters.free(); return r; }
            B2_CUDA_CHECK(cudaMemsetAsync(kv->sk_counters.p, 0, cb, st));
        }
    }
    return 0;
}

static bool is_device_pointer(const void* p) {
    cudaPointerAttributes attr;
    if (cudaPointerGetAttributes(&attr, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged;
}

int b2_decode_step(b2_model* m, b2_kv* kv, const int32_t* tokens, int B, void* logits_out, int32_t* next_tokens_out,
                   void* stream) {
    B2_CHECK_ARG(m && kv && tokens && kv->m == m, "b2_decode_step: bad handle");
    B2_CHECK_ARG(m->finalized, "b2_decode_step: model not finalized");
    B2_CHECK_ARG(B >= 1 && B <= kv->max_batch, "b2_decode_step: B=%d exceeds cache batch %d", B, kv->max_batch);
    std::lock_guard<std::mutex> lk(m->mu);
    DeviceGuard dg(m->device);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    for (int b = 0; b < B; ++b)
        B2_CHECK_ARG(kv->len_host[b] >= 1 && kv->len_host[b] < kv->max_seq,
                     "b2_decode_step: sample %d has cache length %d (capacity %d; prefill first)", b, kv->len_host[b],
                     kv->max_seq);
    B2_TRY(ws_enter(m, st));
    B2_TRY(copy_tokens_in(kv, tokens, B, st));
    B2_CUDA_CHECK(cudaMemsetAsync(kv->step_counter.p, 0, 4, st));
    B2_TRY(set_greedy_unpublished(kv, st));
    cudaStream_t run = nullptr;
    B2_TRY(fork_stream(kv, st, &run));
    B2_TRY(decode_step_run(m, kv, B, run));
    B2_TRY(join_stream(kv, st, run));
    for (int b = 0; b < B; ++b) kv->len_host[b]++;
    if (logits_out)
        B2_CUDA_CHECK(cudaMemcpyAsync(logits_out, m->logits.p, (size_t)B * m->d.vocab * 4, cudaMemcpyDefault, st));
    if (next_tokens_out)
        B2_CUDA_CHECK(cudaMemcpyAsync(next_tokens_out, kv->tok.p, (size_t)B * 4, cudaMemcpyDefault, st));
    B2_TRY(ws_leave(m, st));
    if (next_tokens_out && !is_device_pointer(next_tokens_out)) B2_CUDA_CHECK(cudaStreamSynchronize(st));
    return 0;
}

int b2_decode_greedy(b2_model* m, b2_kv* kv, const int32_t* first_tokens, int B, int n_steps, int32_t* out_tokens,
                     void* stream) {
    B2_CHECK_ARG(m && kv && first_tokens && out_tokens && kv->m == m, "b2_decode_greedy: bad handle");
    B2_CHECK_ARG(m->finalized, "b2_decode_greedy: model not finalized");
    B2_CHECK_ARG(B >= 1 && B <= kv->max_batch && n_steps >= 1, "b2_decode_greedy: bad B=%d n_steps=%d", B, n_steps);
    B2_CHECK_ARG(n_steps <= kv->out_capacity, "b2_decode_greedy: n_steps=%d exceeds capacity %d", n_steps,
                 kv->out_capacity);
    std::lock_guard<std::mutex> lk(m->mu);
    DeviceGuard dg(m->device);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    for (int b = 0; b < B; ++b)
        B2_CHECK_ARG(kv->len_host[b] >= 1 && kv->len_host[b] + n_steps <= kv->max_seq,
                     "b2_decode_greedy: sample %d cache length %d + %d steps exceeds capacity %d", b, kv->len_host[b],
                     n_steps, kv->max_seq);
    B2_TRY(ws_enter(m, st));
    B2_TRY(copy_tokens_in(kv, first_tokens, B, st));
    B2_CUDA_CHECK(cudaMemsetAsync(kv->step_counter.p, 0, 4, st));
    B2_TRY(set_greedy_unpublished(kv, st));
    cudaStream_t run = nullptr;
    B2_TRY(fork_stream(kv, st, &run));
    for (int s = 0; s < n_steps; ++s) B2_TRY(decode_step_run(m, kv, B, run));
    B2_TRY(join_stream(kv, st, run));
    for (int b = 0; b < B; ++b) kv->len_host[b] += n_steps;
    B2_CUDA_CHECK(cudaMemcpyAsync(out_tokens, kv->out_tokens.p, (size_t)n_steps * B * 4, cudaMemcpyDefault, st));
    B2_TRY(ws_leave(m, st));
    // a device destination stays asynchronous on the caller's stream; a host destination must be complete on return
    if (!is_device_pointer(out_tokens)) B2_CUDA_CHECK(cudaStreamSynchronize(st));
    return 0;
}

// ---- beam search: slot copies, candidate selection, one step of the running beams --------------------------------------
// Checks a copy list against the cache (no side effects); end[i] = current length of src[i].
static int check_copies(b2_kv* kv, const int32_t* src, const int32_t* dst, int n, int row_begin, std::vector<int32_t>& end) {
    B2_CHECK_ARG(n >= 0 && n <= kv->max_batch && (n == 0 || (src != nullptr && dst != nullptr)) && row_begin >= 0,
                 "b2_kv_copy_slots: bad argument (n=%d row_begin=%d)", n, row_begin);
    std::vector<char> is_src(kv->max_batch, 0), is_dst(kv->max_batch, 0);
    end.assign(n, 0);
    for (int i = 0; i < n; ++i) {
        B2_CHECK_ARG(src[i] >= 0 && src[i] < kv->max_batch && dst[i] >= 0 && dst[i] < kv->max_batch,
                     "b2_kv_copy_slots: pair %d (%d -> %d) outside the cache's %d slots", i, src[i], dst[i], kv->max_batch);
        B2_CHECK_ARG(row_begin <= kv->len_host[src[i]], "b2_kv_copy_slots: row_begin %d beyond the length %d of slot %d", row_begin,
                     kv->len_host[src[i]], src[i]);
        is_src[src[i]] = 1;
        end[i] = kv->len_host[src[i]];
    }
    for (int i = 0; i < n; ++i) {
        B2_CHECK_ARG(!is_dst[dst[i]], "b2_kv_copy_slots: slot %d is the destination of two copies", dst[i]);
        B2_CHECK_ARG(!is_src[dst[i]], "b2_kv_copy_slots: slot %d is both a source and a destination", dst[i]);
        is_dst[dst[i]] = 1;
    }
    return 0;
}

static int launch_copies(b2_model* m, b2_kv* kv, const int32_t* src, const int32_t* dst, const std::vector<int32_t>& end, int n,
                         int row_begin, cudaStream_t st) {
    if (n == 0) return 0;
    B2_TRY(kv_copy_slots(kv->k.p, kv->v.p, kv->e4m3() ? kv->kscale.as<float>() : nullptr, kv->e4m3() ? kv->vscale.as<float>() : nullptr,
                         src, dst, end.data(), n, row_begin, m->d.layers, m->d.heads, kv->max_batch, kv->pitch,
                         (int)(m->hd * kv->elem_bytes()), kv->len_dev.as<int32_t>(), st));
    for (int i = 0; i < n; ++i) kv->len_host[dst[i]] = end[i];
    return 0;
}

int b2_kv_copy_slots(b2_model* m, b2_kv* kv, const int32_t* src_host, const int32_t* dst_host, int n, int row_begin, void* stream) {
    B2_CHECK_ARG(m && kv && kv->m == m, "b2_kv_copy_slots: bad handle");
    std::lock_guard<std::mutex> lk(m->mu);
    DeviceGuard dg(m->device);
    std::vector<int32_t> end;
    B2_TRY(check_copies(kv, src_host, dst_host, n, row_begin, end));
    return launch_copies(m, kv, src_host, dst_host, end, n, row_begin, reinterpret_cast<cudaStream_t>(stream));
}

int b2_op_beam_topk(const float* logits, const int32_t* row_of_beam, const float* beam_scores, int B, int nb, int V, int K,
                    float* out_scores, int32_t* out_tokens, int32_t* out_beams, void* stream) {
    B2_CHECK_ARG(B >= 1 && nb >= 1 && nb <= 32 && K >= 1 && K <= 128, "b2_op_beam_topk: B=%d nb=%d K=%d", B, nb, K);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    void* ws = nullptr;
    B2_CUDA_CHECK(cudaMallocAsync(&ws, beam_topk_workspace_bytes(B, nb, K), st));
    const int r = beam_topk(logits, row_of_beam, beam_scores, B, nb, V, K, ws, out_scores, out_tokens, out_beams, st);
    B2_CUDA_CHECK(cudaFreeAsync(ws, st));
    return r;
}

static BeamSampleParams beam_sample_params(const b2_beam_sampling* s, uint32_t step) {
    BeamSampleParams p;
    p.temperature = s->temperature;
    p.top_k = s->top_k;
    p.top_p = s->top_p;
    p.min_keep = s->min_keep;
    p.seed = s->seed;
    p.step = step;
    return p;
}

int b2_op_beam_sample(const float* logits, const int32_t* row_of_beam, const float* beam_scores, int B, int nb, int V, int K,
                      const b2_beam_sampling* sampling, uint32_t step, float* out_scores, int32_t* out_tokens, int32_t* out_beams,
                      void* stream) {
    B2_CHECK_ARG(sampling != nullptr, "b2_op_beam_sample: null sampling");
    B2_CHECK_ARG(B >= 1 && nb >= 1 && nb <= 32 && K >= 1 && K <= 128, "b2_op_beam_sample: B=%d nb=%d K=%d", B, nb, K);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    void* ws = nullptr;
    B2_CUDA_CHECK(cudaMallocAsync(&ws, beam_sample_workspace_bytes(B, nb, K), st));
    const int r = beam_sample(logits, row_of_beam, beam_scores, B, nb, V, K, beam_sample_params(sampling, step), ws, out_scores,
                              out_tokens, out_beams, st);
    B2_CUDA_CHECK(cudaFreeAsync(ws, st));
    return r;
}

int b2_op_beam_select_out(const float* logits, const int32_t* row_of_beam, const float* beam_scores, int B, int nb, int V, int K,
                          const b2_beam_sampling* sampling, uint32_t step, int fan, float* out_scores, int32_t* out_tokens,
                          int32_t* out_beams, float* row_scores, float* row_logits, void* stream) {
    B2_CHECK_ARG(B >= 1 && nb >= 1 && nb <= 32 && K >= 1 && K <= 128, "b2_op_beam_select_out: B=%d nb=%d K=%d", B, nb, K);
    B2_CHECK_ARG(fan >= 1 && fan <= 32 && (sampling == nullptr || fan == 1),
                 "b2_op_beam_select_out: fan %d (1..32, and 1 with sampling)", fan);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    BeamRowsOut ro;
    ro.scores = row_scores; ro.logits = row_logits; ro.fan = fan;
    void* ws = nullptr;
    B2_CUDA_CHECK(cudaMallocAsync(&ws, beam_sample_workspace_bytes(B, nb, K), st));  // >= beam_topk's
    const int r = sampling != nullptr
                      ? beam_sample(logits, row_of_beam, beam_scores, B, nb, V, K, beam_sample_params(sampling, step), ws, out_scores,
                                    out_tokens, out_beams, st, ro)
                      : beam_topk(logits, row_of_beam, beam_scores, B, nb, V, K, ws, out_scores, out_tokens, out_beams, st, ro);
    B2_CUDA_CHECK(cudaFreeAsync(ws, st));
    return r;
}

int b2_op_beam_select_proc(const float* logits, int rows, const int32_t* row_of_beam, const float* beam_scores, int B, int nb, int V,
                           int K, const b2_beam_sampling* sampling, uint32_t step, int fan, const b2_logits_proc* proc, float* out_scores,
                           int32_t* out_tokens, int32_t* out_beams, float* row_scores, float* row_logits, void* stream) {
    B2_CHECK_ARG(B >= 1 && nb >= 1 && nb <= 32 && K >= 1 && K <= 128, "b2_op_beam_select_proc: B=%d nb=%d K=%d", B, nb, K);
    B2_CHECK_ARG(fan >= 1 && fan <= 32 && (sampling == nullptr || fan == 1),
                 "b2_op_beam_select_proc: fan %d (1..32, and 1 with sampling)", fan);
    B2_CHECK_ARG(rows >= 1 && (row_of_beam != nullptr || rows == B * nb), "b2_op_beam_select_proc: %d logits rows for B=%d nb=%d", rows,
                 B, nb);
    B2_CHECK_ARG(V >= 1, "b2_op_beam_select_proc: vocab %d", V);
    // processors: a scratch state whose row r holds proc[r]'s prompt ids as its history
    std::vector<ProcRow> pr(proc ? rows : 0);
    int cap = 1;
    bool any = false;
    for (int r = 0; r < (int)pr.size(); ++r) {
        B2_TRY(proc_row_of(proc + r, INT_MAX, &pr[r], "b2_op_beam_select_proc"));
        cap = std::max(cap, proc[r].prompt_len + 1);
        any = any || pr[r].on;
    }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const int words = (V + 31) / 32;
    const size_t ws_bytes = beam_sample_workspace_bytes(B, nb, K);  // >= beam_topk's
    const size_t off_rows = (ws_bytes + 255) / 256 * 256, off_hist = off_rows + (size_t)rows * sizeof(ProcRow);
    const size_t off_bits = off_hist + (size_t)rows * cap * sizeof(int32_t);
    DevBuf tmp;  // one scratch buffer: the selection's workspace, then (with processors) ProcRow[rows], history [rows][cap], bitmap
    B2_TRY(tmp.alloc(any ? off_bits + (size_t)rows * words * sizeof(uint32_t) : ws_bytes));
    BeamProc bp;
    int r = 0;
    if (any) {
        ProcState& ps = bp.proc;
        ps.rows = reinterpret_cast<ProcRow*>(tmp.as<char>() + off_rows);
        ps.hist = reinterpret_cast<int32_t*>(tmp.as<char>() + off_hist);
        ps.bits = reinterpret_cast<uint32_t*>(tmp.as<char>() + off_bits);
        ps.cap = cap; ps.words = words;
        if (cudaMemsetAsync(ps.rows, 0, (size_t)rows * sizeof(ProcRow), st) != cudaSuccess) {
            set_error("b2_op_beam_select_proc: %s", cudaGetErrorString(cudaGetLastError()));
            r = -2;
        }
        for (int i = 0; i < rows && r == 0; ++i)
            if (pr[i].on) r = proc_seed(ps, i, pr[i], proc[i].prompt_ids, pr[i].prompt_len, -1, V, st);
    }
    BeamRowsOut ro;
    ro.scores = row_scores; ro.logits = row_logits; ro.fan = fan;
    if (r == 0)
        r = sampling != nullptr ? beam_sample(logits, row_of_beam, beam_scores, B, nb, V, K, beam_sample_params(sampling, step), tmp.p,
                                              out_scores, out_tokens, out_beams, st, ro, bp)
                                : beam_topk(logits, row_of_beam, beam_scores, B, nb, V, K, tmp.p, out_scores, out_tokens, out_beams, st, ro, bp);
    cudaError_t e = cudaStreamSynchronize(st);
    tmp.free();
    if (r != 0) return r;
    B2_CUDA_CHECK(e);
    return 0;
}

int b2_beam_begin_proc(b2_model* m, b2_kv* kv, int B, const b2_logits_proc* proc, void* stream) {
    B2_CHECK_ARG(m && kv && kv->m == m, "b2_beam_begin_proc: bad handle");
    B2_CHECK_ARG(B >= 1 && B <= kv->max_batch, "b2_beam_begin_proc: B=%d exceeds the cache's %d slots", B, kv->max_batch);
    std::vector<ProcRow> pr(B);
    for (int b = 0; b < B; ++b) B2_TRY(proc_row_of(proc ? proc + b : nullptr, kv->max_seq + 1, &pr[b], "b2_beam_begin_proc"));
    std::lock_guard<std::mutex> lk(m->mu);
    DeviceGuard dg(m->device);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    B2_TRY(proc_all_off(kv, st));
    B2_TRY(proc_alloc(kv, st));
    if (kv->beam_proc_rows.p == nullptr) B2_TRY(kv->beam_proc_rows.alloc((size_t)kv->max_batch * sizeof(ProcRow)));
    B2_CUDA_CHECK(cudaMemsetAsync(kv->beam_proc_rows.p, 0, kv->beam_proc_rows.bytes, st));
    for (int b = 0; b < B; ++b)
        if (pr[b].on) B2_TRY(proc_seed(beam_proc_state(kv), b, pr[b], proc[b].prompt_ids, pr[b].prompt_len, -1, m->d.vocab, st));
    kv->beam_proc_on = true;
    return 0;
}

static int beam_step(b2_model* m, b2_kv* kv, const b2_beam_step_args* a, const b2_beam_sampling* sampling, uint32_t step,
                     float* row_scores, float* row_logits, bool proc, void* stream);

int b2_beam_step(b2_model* m, b2_kv* kv, const b2_beam_step_args* a, void* stream) {
    return b2_beam_step_ex(m, kv, a, nullptr, 0u, stream);
}

int b2_beam_step_ex(b2_model* m, b2_kv* kv, const b2_beam_step_args* a, const b2_beam_sampling* sampling, uint32_t step, void* stream) {
    return b2_beam_step_out(m, kv, a, sampling, step, nullptr, nullptr, stream);
}

int b2_beam_step_out(b2_model* m, b2_kv* kv, const b2_beam_step_args* a, const b2_beam_sampling* sampling, uint32_t step,
                     float* row_scores, float* row_logits, void* stream) {
    return beam_step(m, kv, a, sampling, step, row_scores, row_logits, false, stream);
}

int b2_beam_step_proc(b2_model* m, b2_kv* kv, const b2_beam_step_args* a, const b2_beam_sampling* sampling, uint32_t step,
                      float* row_scores, float* row_logits, void* stream) {
    return beam_step(m, kv, a, sampling, step, row_scores, row_logits, true, stream);
}

static int beam_step(b2_model* m, b2_kv* kv, const b2_beam_step_args* a, const b2_beam_sampling* sampling, uint32_t step,
                     float* row_scores, float* row_logits, bool proc, void* stream) {
    B2_CHECK_ARG(m && kv && a && kv->m == m, "b2_beam_step: bad handle");
    B2_CHECK_ARG(m->finalized, "b2_beam_step: model not finalized");
    const int B = a->B, nb = a->nb, K = a->K, n = a->B * a->nb;
    B2_CHECK_ARG(B >= 1 && nb >= 1 && nb <= 32 && n <= kv->max_batch, "b2_beam_step: B=%d x nb=%d beams exceed the cache's %d slots",
                 B, nb, kv->max_batch);
    B2_CHECK_ARG(K >= 1 && K <= 128 && (long long)K <= (long long)nb * m->d.vocab, "b2_beam_step: K=%d outside [1, min(128, nb*V)]", K);
    // the sampling arguments are checked before the step changes the cache, as every other argument is
    B2_CHECK_ARG(sampling == nullptr || (sampling->temperature > 0.f && sampling->top_p > 0.f && sampling->top_p <= 1.f &&
                                         sampling->top_k >= 0 && sampling->min_keep >= 1 && sampling->min_keep <= K),
                 "b2_beam_step_ex: bad sampling (temperature > 0, top_p in (0, 1], top_k >= 0, 1 <= min_keep <= K)");
    B2_CHECK_ARG(sampling == nullptr || (long long)n * m->d.vocab <= 0xFFFFFFFFll,
                 "b2_beam_step_ex: B*nb*V exceeds the 32-bit Philox row");
    B2_CHECK_ARG(a->tokens_host && a->slot_of_beam_host && a->beam_scores_host && a->out_scores_host && a->out_tokens_host &&
                 a->out_beams_host, "b2_beam_step: null array");
    std::lock_guard<std::mutex> lk(m->mu);
    DeviceGuard dg(m->device);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    B2_CHECK_ARG(!proc || kv->beam_proc_on, "b2_beam_step_proc: beam processing is not armed on this cache (b2_beam_begin_proc)");
    std::vector<int32_t> end;
    B2_TRY(check_copies(kv, a->copy_src_host, a->copy_dst_host, a->n_copies, a->row_begin, end));
    std::vector<int32_t> len(kv->len_host.begin(), kv->len_host.begin() + n), tok(n, -1);
    for (int i = 0; i < a->n_copies; ++i)
        if (a->copy_dst_host[i] < n) len[a->copy_dst_host[i]] = end[i];
    for (int i = 0; i < n; ++i) {
        const int s = a->slot_of_beam_host[i];
        B2_CHECK_ARG(s >= 0 && s < n && tok[s] < 0, "b2_beam_step: slot_of_beam is not a permutation of [0, %d)", n);
        B2_CHECK_ARG(a->tokens_host[i] >= 0, "b2_beam_step: negative token %d for beam %d", a->tokens_host[i], i);
        tok[s] = a->tokens_host[i];
    }
    for (int s = 0; s < n; ++s)
        B2_CHECK_ARG(len[s] >= 1 && len[s] < kv->max_seq, "b2_beam_step: slot %d has cache length %d (capacity %d)", s, len[s],
                     kv->max_seq);
    if (kv->beam_in.p == nullptr) {
        B2_TRY(kv->beam_in.alloc((size_t)3 * kv->max_batch * 4));
        B2_TRY(kv->beam_ws.alloc(beam_sample_workspace_bytes(kv->max_batch, 1, 128)));  // >= beam_topk's
        B2_TRY(kv->beam_out.alloc((size_t)kv->max_batch * 128 * 12));
    }
    B2_TRY(ws_enter(m, st));
    B2_TRY(launch_copies(m, kv, a->copy_src_host, a->copy_dst_host, end, a->n_copies, a->row_begin, st));
    // a copied slot takes its source's history with its K/V rows (the whole history: it is in token space, not cache rows)
    if (proc && a->n_copies > 0) B2_TRY(proc_copy_slots(beam_proc_state(kv), a->copy_src_host, a->copy_dst_host, a->n_copies, st));
    B2_TRY(copy_tokens_in(kv, tok.data(), n, st));
    B2_CUDA_CHECK(cudaMemsetAsync(kv->step_counter.p, 0, 4, st));
    B2_TRY(set_greedy_unpublished(kv, st, proc));
    cudaStream_t run = nullptr;
    B2_TRY(fork_stream(kv, st, &run));
    B2_TRY(decode_step_run(m, kv, n, run));
    B2_TRY(join_stream(kv, st, run));
    for (int s = 0; s < n; ++s) kv->len_host[s]++;
    int32_t* rows = kv->beam_in.as<int32_t>();
    B2_TRY(set_i32_pairs(rows, a->slot_of_beam_host, rows + kv->max_batch, reinterpret_cast<const int32_t*>(a->beam_scores_host), n, st));
    float* o_s = kv->beam_out.as<float>();
    int32_t* o_t = reinterpret_cast<int32_t*>(o_s + B * K);
    int32_t* o_b = o_t + B * K;
    const float* run_scores = reinterpret_cast<const float*>(rows + kv->max_batch);
    BeamRowsOut ro;
    ro.scores = row_scores; ro.logits = row_logits;
    BeamProc bp;
    if (proc) {  // each beam's token joins its slot's history inside the row kernel, before the row is processed
        int32_t* append = rows + 2 * kv->max_batch;
        B2_TRY(set_i32_pairs(append, a->tokens_host, nullptr, nullptr, n, st));
        bp.proc = beam_proc_state(kv);
        bp.append = append;
    }
    if (sampling != nullptr)
        B2_TRY(beam_sample(m->logits.as<float>(), rows, run_scores, B, nb, m->d.vocab, K, beam_sample_params(sampling, step), kv->beam_ws.p,
                           o_s, o_t, o_b, st, ro, bp));
    else
        B2_TRY(beam_topk(m->logits.as<float>(), rows, run_scores, B, nb, m->d.vocab, K, kv->beam_ws.p, o_s, o_t, o_b, st, ro, bp));
    B2_CUDA_CHECK(cudaMemcpyAsync(a->out_scores_host, o_s, (size_t)B * K * 4, cudaMemcpyDeviceToHost, st));
    B2_CUDA_CHECK(cudaMemcpyAsync(a->out_tokens_host, o_t, (size_t)B * K * 4, cudaMemcpyDeviceToHost, st));
    B2_CUDA_CHECK(cudaMemcpyAsync(a->out_beams_host, o_b, (size_t)B * K * 4, cudaMemcpyDeviceToHost, st));
    B2_TRY(ws_leave(m, st));
    B2_CUDA_CHECK(cudaStreamSynchronize(st));
    return 0;
}

// ---- streaming decode: the device runs ahead, the host reads tokens from mapped pinned memory ---------------------------
int b2_stream_set_outputs(b2_kv* kv, float* scores, float* logits, int cap_steps) {
    B2_CHECK_ARG(kv != nullptr, "b2_stream_set_outputs: null cache");
    const bool any = scores != nullptr || logits != nullptr;
    B2_CHECK_ARG(!any || cap_steps >= 1, "b2_stream_set_outputs: cap_steps %d must be >= 1", cap_steps);
    std::lock_guard<std::mutex> lk(kv->m->mu);
    kv->next_scores = scores; kv->next_logits = logits; kv->next_cap = any ? cap_steps : 0;
    return 0;
}

// the shared-prefix state of a cache, allocated by the first armed generation: the table, and the counters of max_batch rows
// (zeroed on `st`; they self-reset after every launch) followed by partials for the largest split decode_nsplit gives (16)
static int share_alloc(b2_model* m, b2_kv* kv, cudaStream_t st) {
    if (kv->share_tab.p != nullptr) return 0;
    const size_t attn = share_counter_bytes(kv) + decode_attn_shared_scratch_bytes(kv->max_batch, m->d.heads, 16);
    int r = kv->share_tab.alloc((size_t)kv->max_batch * (sizeof(PrefixGroup) + sizeof(int32_t)));
    if (r == 0) r = kv->share_attn.alloc(attn);
    if (r == 0 && cudaMemsetAsync(kv->share_attn.p, 0, attn, st) != cudaSuccess) {
        set_error("b2_stream_begin_groups: %s", cudaGetErrorString(cudaGetLastError()));
        r = -2;
    }
    if (r != 0) { kv->share_tab.free(); kv->share_attn.free(); }
    return r;
}
static int stream_begin(b2_model* m, b2_kv* kv, const float* logits, int B, const b2_sampling* sp, const b2_logits_proc* proc,
                        const b2_prefix_group* groups, int G, void* stream);

int b2_stream_begin(b2_model* m, b2_kv* kv, const float* logits, int B, const b2_sampling* sp, void* stream) {
    return b2_stream_begin_ex(m, kv, logits, B, sp, nullptr, stream);
}

int b2_stream_begin_ex(b2_model* m, b2_kv* kv, const float* logits, int B, const b2_sampling* sp, const b2_logits_proc* proc,
                       void* stream) {
    return stream_begin(m, kv, logits, B, sp, proc, nullptr, 0, stream);
}

int b2_stream_begin_groups(b2_model* m, b2_kv* kv, const float* logits, int B, const b2_sampling* sp, const b2_logits_proc* proc,
                           const b2_prefix_group* groups, int G, void* stream) {
    B2_CHECK_ARG(G >= 1 && groups != nullptr, "b2_stream_begin_groups: G=%d groups (at least one)", G);
    return stream_begin(m, kv, logits, B, sp, proc, groups, G, stream);
}

static int stream_begin(b2_model* m, b2_kv* kv, const float* logits, int B, const b2_sampling* sp, const b2_logits_proc* proc,
                        const b2_prefix_group* groups, int G, void* stream) {
    B2_CHECK_ARG(m && kv && logits && kv->m == m, "b2_stream_begin: bad handle");
    // the rows armed by b2_stream_set_outputs belong to this call, whether or not it begins a generation
    float *out_scores, *out_logits;
    int out_cap;
    {
        std::lock_guard<std::mutex> lk(m->mu);
        out_scores = kv->next_scores; out_logits = kv->next_logits; out_cap = kv->next_cap;
        kv->next_scores = kv->next_logits = nullptr; kv->next_cap = 0;
    }
    B2_CHECK_ARG(m->finalized, "b2_stream_begin: model not finalized");
    B2_CHECK_ARG(B >= 1 && B <= kv->max_batch, "b2_stream_begin: B=%d exceeds cache batch %d", B, kv->max_batch);
    SampleState v = {};
    v.temperature = 1.f; v.top_p = 1.f;
    if (sp != nullptr && sp->do_sample) {
        B2_CHECK_ARG(sp->temperature > 0.f, "b2_stream_begin: temperature must be positive when sampling (got %g)", (double)sp->temperature);
        B2_CHECK_ARG(sp->top_p > 0.f && sp->top_p <= 1.f, "b2_stream_begin: top_p must be in (0, 1] (got %g)", (double)sp->top_p);
        B2_CHECK_ARG(sp->top_k >= 0, "b2_stream_begin: top_k must be >= 0");
        v.do_sample = 1; v.temperature = sp->temperature; v.top_p = sp->top_p; v.top_k = sp->top_k; v.seed = sp->seed;
    }
    std::lock_guard<std::mutex> lk(m->mu);
    DeviceGuard dg(m->device);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    v.out_scores = out_scores; v.out_logits = out_logits; v.out_cap = out_cap;
    for (int b = 0; b < B; ++b)
        B2_CHECK_ARG(kv->len_host[b] >= 1, "b2_stream_begin: sample %d has an empty cache (prefill first)", b);
    std::vector<ProcRow> pr(B);
    for (int b = 0; b < B; ++b) B2_TRY(proc_row_of(proc ? proc + b : nullptr, kv->max_seq + 1, &pr[b], "b2_stream_begin_ex"));
    // the group table: checked against the cache before anything is queued
    std::vector<PrefixGroup> tab(G);
    std::vector<int32_t> row_prefix(kv->max_batch, 0);
    if (G > 0) {
        B2_CHECK_ARG(G <= B, "b2_stream_begin_groups: G=%d groups for %d rows", G, B);
        std::vector<char> seen(B, 0);
        for (int g = 0; g < G; ++g) {
            const b2_prefix_group& x = groups[g];
            B2_CHECK_ARG(x.n_rows >= 1 && x.n_rows <= kPrefixGroupRows, "b2_stream_begin_groups: group %d has %d rows (1..%d)", g,
                         x.n_rows, kPrefixGroupRows);
            B2_CHECK_ARG(x.src_slot >= 0 && x.src_slot < B, "b2_stream_begin_groups: group %d source slot %d outside [0, %d)", g,
                         x.src_slot, B);
            B2_CHECK_ARG(x.prefix_len >= 1 && x.prefix_len <= kv->len_host[x.src_slot],
                         "b2_stream_begin_groups: group %d prefix_len %d outside [1, %d] (the length of slot %d)", g, x.prefix_len,
                         kv->len_host[x.src_slot], x.src_slot);
            tab[g].src_slot = x.src_slot; tab[g].prefix_len = x.prefix_len; tab[g].n_rows = x.n_rows;
            for (int r = 0; r < kPrefixGroupRows; ++r) tab[g].rows[r] = r < x.n_rows ? x.rows[r] : 0;
            for (int r = 0; r < x.n_rows; ++r) {
                const int row = x.rows[r];
                B2_CHECK_ARG(row >= 0 && row < B, "b2_stream_begin_groups: group %d row %d outside [0, %d)", g, row, B);
                B2_CHECK_ARG(!seen[row], "b2_stream_begin_groups: row %d belongs to two groups", row);
                B2_CHECK_ARG(x.prefix_len <= kv->len_host[row], "b2_stream_begin_groups: group %d prefix_len %d exceeds the length %d "
                             "of its row %d", g, x.prefix_len, kv->len_host[row], row);
                seen[row] = 1;
                row_prefix[row] = x.prefix_len;
            }
        }
    }
    kv->epoch += 1;
    v.tag = 1 + kv->epoch % 2047;
    kv->spec_R = 0;
    B2_TRY(ws_enter(m, st));
    B2_TRY(set_sampling(kv, v, true, st));
    B2_CUDA_CHECK(cudaMemsetAsync(kv->step_counter.p, 0, 4, st));
    B2_TRY(proc_all_off(kv, st));
    for (int b = 0; b < B; ++b) B2_TRY(proc_set_row(kv, b, pr[b], proc ? proc[b].prompt_ids : nullptr, -1, st));
    // token 0: chosen from the prefill's last-position logits (processed over the prompt history), published as ring entry 0,
    // fed to the first decode step
    B2_TRY(sample_publish(logits, m->d.vocab, B, kv->sstate.as<SampleState>(), kv->rows_dev.as<RowState>(), kv->tok.as<int32_t>(), nullptr,
                          kv->step_counter.as<int32_t>(), kv->len_dev.as<int32_t>(), kv->ring_dev, kv->ring_cap, SP_SELECT, 0,
                          proc_state(kv), nullptr, st));
    kv->stream_B = B; kv->stream_tag = v.tag; kv->stream_scheduled = 1;
    if (G > 0) {
        B2_TRY(share_alloc(m, kv, st));
        B2_CUDA_CHECK(cudaMemcpyAsync(kv->share_tab.p, tab.data(), (size_t)G * sizeof(PrefixGroup), cudaMemcpyHostToDevice, st));
        B2_CUDA_CHECK(cudaMemcpyAsync(kv->share_tab.as<PrefixGroup>() + kv->max_batch, row_prefix.data(),
                                      (size_t)kv->max_batch * sizeof(int32_t), cudaMemcpyHostToDevice, st));
        B2_CUDA_CHECK(cudaStreamSynchronize(st));  // pageable host sources
        share_arm(kv, G);
    }
    return ws_leave(m, st);
}

int b2_stream_begin_lookup(b2_model* m, b2_kv* kv, const float* logits, int B, const b2_sampling* sp, const b2_prompt_lookup* lk,
                           void* stream) {
    B2_CHECK_ARG(m && kv && logits && lk && kv->m == m, "b2_stream_begin_lookup: bad handle");
    B2_CHECK_ARG(m->finalized, "b2_stream_begin_lookup: model not finalized");
    B2_CHECK_ARG(B == 1, "b2_stream_begin_lookup: prompt lookup decodes one sample (B=%d)", B);
    B2_CHECK_ARG(!kv->e4m3(), "b2_stream_begin_lookup: the verify step reads a bf16 KV cache");
    B2_CHECK_ARG(lk->num_tokens >= 1 && lk->num_tokens < kSpecMaxRows, "b2_stream_begin_lookup: num_tokens %d outside 1..%d",
                 lk->num_tokens, kSpecMaxRows - 1);
    B2_CHECK_ARG(lk->max_ngram >= 1 && lk->max_new_tokens >= 1, "b2_stream_begin_lookup: max_ngram and max_new_tokens must be >= 1");
    B2_CHECK_ARG(lk->n_eos >= 0 && lk->n_eos <= kProcMaxEos, "b2_stream_begin_lookup: n_eos must be in [0, %d]", kProcMaxEos);
    B2_CHECK_ARG(lk->prompt_len >= 0 && (lk->prompt_len == 0 || lk->prompt_ids != nullptr), "b2_stream_begin_lookup: bad prompt ids");
    B2_CHECK_ARG((int64_t)lk->prompt_len + lk->max_new_tokens + lk->num_tokens <= kv->max_seq,
                 "b2_stream_begin_lookup: prompt %d + max_new_tokens %d + num_tokens %d exceed the cache's max_seq %d", lk->prompt_len,
                 lk->max_new_tokens, lk->num_tokens, kv->max_seq);
    SampleState v = {};
    v.temperature = 1.f; v.top_p = 1.f;
    if (sp != nullptr && sp->do_sample) {
        B2_CHECK_ARG(sp->temperature > 0.f && sp->top_p > 0.f && sp->top_p <= 1.f && sp->top_k >= 0, "b2_stream_begin_lookup: bad sampling parameters");
        v.do_sample = 1; v.temperature = sp->temperature; v.top_p = sp->top_p; v.top_k = sp->top_k; v.seed = sp->seed;
    }
    const int R = lk->num_tokens + 1;
    std::lock_guard<std::mutex> lk_(m->mu);
    DeviceGuard dg(m->device);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    B2_CHECK_ARG(kv->next_scores == nullptr && kv->next_logits == nullptr,
                 "b2_stream_begin_lookup: a prompt-lookup generation writes no score or logits rows (b2_stream_set_outputs)");
    // the last step writes rows up to len + (max_new_tokens - 1) + R - 1
    B2_CHECK_ARG(kv->len_host[0] >= 1 && (int64_t)kv->len_host[0] + lk->max_new_tokens + lk->num_tokens <= kv->max_seq,
                 "b2_stream_begin_lookup: cache length %d + max_new_tokens %d + num_tokens %d exceed max_seq %d", kv->len_host[0],
                 lk->max_new_tokens, lk->num_tokens, kv->max_seq);
    B2_TRY(ws_enter(m, st));
    B2_TRY(spec_alloc(m, kv, R, st));
    kv->epoch += 1;
    v.tag = 1 + kv->epoch % 2047;
    B2_TRY(set_sampling(kv, v, true, st));
    B2_CUDA_CHECK(cudaMemsetAsync(kv->step_counter.p, 0, 4, st));
    B2_TRY(proc_all_off(kv, st));
    ProcRow off = {};
    off.penalty = 1.f;
    B2_TRY(proc_seed(proc_state(kv), 0, off, lk->prompt_ids, lk->prompt_len, -1, m->d.vocab, st));  // the history: prompt ids
    SpecState ss = {};
    ss.K = lk->num_tokens; ss.ngram = lk->max_ngram; ss.max_new = lk->max_new_tokens; ss.n_eos = lk->n_eos;
    for (int i = 0; i < lk->n_eos; ++i) ss.eos[i] = lk->eos_ids[i];
    ss.prompt_len = lk->prompt_len; ss.hist_len = lk->prompt_len;
    B2_CUDA_CHECK(cudaHostGetDevicePointer(reinterpret_cast<void**>(&ss.mirror), kv->spec_mirror, 0));
    B2_CUDA_CHECK(cudaMemcpyAsync(kv->spec_state.p, &ss, sizeof ss, cudaMemcpyHostToDevice, st));
    B2_CUDA_CHECK(cudaStreamSynchronize(st));  // `ss` is a pageable host source; earlier steps on this cache are done
    memset(kv->spec_mirror, 0, 6 * sizeof(int));
    kv->spec_mirror[5] = 1;  // token 0, published below
    // token 0 from the prefill logits, published as ring entry 0 and pending for the first verify step
    B2_TRY(sample_publish(logits, m->d.vocab, 1, kv->sstate.as<SampleState>(), kv->rows_dev.as<RowState>(), kv->tok.as<int32_t>(), nullptr,
                          kv->step_counter.as<int32_t>(), kv->len_dev.as<int32_t>(), kv->ring_dev, kv->ring_cap, SP_SELECT, 0,
                          proc_state(kv), nullptr, st));
    kv->stream_B = 1; kv->stream_tag = v.tag; kv->stream_scheduled = 1;
    kv->spec_R = R; kv->spec_max_new = lk->max_new_tokens; kv->spec_queued = 0; kv->spec_len0 = kv->len_host[0];
    return ws_leave(m, st);
}

// b2_stream_enqueue of a lookup generation: tops the verify steps in flight (queued, not yet retired on the device) up to n, and
// queues none once the generation's tokens are published. A step publishes a varying number of tokens, so steps are scheduled
// against what the device has retired, read from the mapped mirror without a synchronisation. Every step in flight publishes at
// least one token until max_new_tokens are out, so the host may wait for token published + in flight - 1.
static int lookup_enqueue(b2_model* m, b2_kv* kv, int n_steps, cudaStream_t st) {
    const volatile int* mr = kv->spec_mirror;
    const int published = mr[5];  // before `retired`: the device writes retired first
    __sync_synchronize();
    const int retired = mr[4];
    int in_flight = kv->spec_queued - retired;
    if (published < kv->spec_max_new && in_flight < n_steps) {
        const int q = n_steps - in_flight;
        B2_TRY(ws_enter(m, st));
        cudaStream_t run = nullptr;
        B2_TRY(fork_stream(kv, st, &run));
        for (int s = 0; s < q; ++s) B2_TRY(verify_step_run(m, kv, kv->spec_R, run));
        B2_TRY(join_stream(kv, st, run));
        B2_TRY(ws_leave(m, st));
        kv->spec_queued += q;
        in_flight += q;
        // an upper bound of the cache length (the exact one is in the mirror once the steps have run)
        kv->len_host[0] = kv->spec_len0 + std::min(kv->spec_max_new - 1, kv->spec_queued * kv->spec_R);
    }
    const int guaranteed = published >= kv->spec_max_new ? kv->spec_max_new : std::min(kv->spec_max_new, published + in_flight);
    kv->stream_scheduled = std::max(kv->stream_scheduled, guaranteed);
    return 0;
}

int b2_stream_lookup_stats(b2_kv* kv, int32_t* steps, int32_t* drafted, int32_t* accepted) {
    B2_CHECK_ARG(kv != nullptr, "b2_stream_lookup_stats: null cache");
    B2_CHECK_ARG(kv->spec_mirror != nullptr, "b2_stream_lookup_stats: no lookup generation has run on this cache");
    const volatile int* mr = kv->spec_mirror;
    if (steps) *steps = mr[0];
    if (drafted) *drafted = mr[1];
    if (accepted) *accepted = mr[2];
    return 0;
}

int b2_decode_rows(b2_model* m, b2_kv* kv, int slot, const int32_t* tokens, int R, float* logits_out, void* stream) {
    B2_CHECK_ARG(m && kv && tokens && kv->m == m, "b2_decode_rows: bad handle");
    B2_CHECK_ARG(m->finalized, "b2_decode_rows: model not finalized");
    B2_CHECK_ARG(slot >= 0 && slot < kv->max_batch, "b2_decode_rows: slot %d outside the cache's %d", slot, kv->max_batch);
    std::lock_guard<std::mutex> lk(m->mu);
    DeviceGuard dg(m->device);
    B2_CHECK_ARG(kv->len_host[slot] >= 1 && kv->len_host[slot] + R <= kv->max_seq,
                 "b2_decode_rows: slot %d cache length %d + %d rows exceeds capacity %d (prefill first)", slot, kv->len_host[slot], R,
                 kv->max_seq);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    B2_TRY(ws_enter(m, st));
    B2_TRY(spec_alloc(m, kv, R, st));
    B2_TRY(set_greedy_unpublished(kv, st));
    B2_CUDA_CHECK(cudaMemcpyAsync(spec_rows(kv), tokens, (size_t)R * 4, cudaMemcpyDefault, st));
    cudaStream_t run = nullptr;
    B2_TRY(fork_stream(kv, st, &run));
    B2_TRY(rows_forward(m, kv, slot, R, run));
    B2_TRY(join_stream(kv, st, run));
    const int32_t len = kv->len_host[slot] + R;
    B2_TRY(set_i32_pairs(kv->len_dev.as<int32_t>() + slot, &len, nullptr, nullptr, 1, st));
    kv->len_host[slot] = len;
    if (logits_out)
        B2_CUDA_CHECK(cudaMemcpyAsync(logits_out, kv->spec_logits.p, (size_t)R * m->d.vocab * 4, cudaMemcpyDefault, st));
    B2_TRY(ws_leave(m, st));
    // host sources are copied before return; a host destination must be complete on return
    if (!is_device_pointer(tokens) || (logits_out && !is_device_pointer(logits_out))) B2_CUDA_CHECK(cudaStreamSynchronize(st));
    return 0;
}

int b2_stream_enqueue(b2_model* m, b2_kv* kv, int n_steps, void* stream) {
    B2_CHECK_ARG(m && kv && kv->m == m && n_steps >= 1, "b2_stream_enqueue: bad argument");
    std::lock_guard<std::mutex> lk(m->mu);
    DeviceGuard dg(m->device);
    B2_CHECK_ARG(kv->stream_B >= 1, "b2_stream_enqueue: no streaming generation on this cache (b2_stream_begin first)");
    if (kv->spec_R > 0) return lookup_enqueue(m, kv, n_steps, reinterpret_cast<cudaStream_t>(stream));
    const int B = kv->stream_B;
    const bool per_row = kv->samp_host.per_row != 0;
    // one generation never outgrows the ring (ring_cap = max_seq); a continuously batched cache runs indefinitely and wraps
    B2_CHECK_ARG(per_row || kv->stream_scheduled + n_steps <= kv->ring_cap, "b2_stream_enqueue: %d tokens exceed the ring capacity %d",
                 kv->stream_scheduled + n_steps, kv->ring_cap);
    for (int b = 0; b < B; ++b)
        B2_CHECK_ARG((per_row && !kv->rows_host[b].active) || kv->len_host[b] + n_steps <= kv->max_seq,
                     "b2_stream_enqueue: sample %d cache length %d + %d steps exceeds capacity %d", b, kv->len_host[b], n_steps, kv->max_seq);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    B2_TRY(ws_enter(m, st));
    cudaStream_t run = nullptr;
    B2_TRY(fork_stream(kv, st, &run));
    for (int s = 0; s < n_steps; ++s) B2_TRY(decode_step_run(m, kv, B, run));
    B2_TRY(join_stream(kv, st, run));
    for (int b = 0; b < B; ++b)
        if (!per_row || kv->rows_host[b].active) kv->len_host[b] += n_steps;
    kv->stream_scheduled += n_steps;
    return ws_leave(m, st);
}

// ---- continuous batching: requests join and leave the slots of one cache between decode steps ----------------------------
int b2_batch_begin(b2_model* m, b2_kv* kv, int B, void* stream) {
    B2_CHECK_ARG(m && kv && kv->m == m && B >= 1 && B <= kv->max_batch, "b2_batch_begin: bad argument");
    std::lock_guard<std::mutex> lk(m->mu);
    DeviceGuard dg(m->device);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    B2_CHECK_ARG(kv->next_scores == nullptr && kv->next_logits == nullptr,
                 "b2_batch_begin: a continuously batched cache writes no score or logits rows (b2_stream_set_outputs)");
    SampleState v = {};
    v.temperature = 1.f; v.top_p = 1.f; v.per_row = 1;
    kv->spec_R = 0;
    kv->epoch += 1;
    v.tag = 1 + kv->epoch % 2047;
    B2_TRY(ws_enter(m, st));
    B2_TRY(set_sampling(kv, v, true, st));
    B2_CUDA_CHECK(cudaMemsetAsync(kv->step_counter.p, 0, 4, st));
    B2_TRY(proc_all_off(kv, st));
    B2_CUDA_CHECK(cudaMemsetAsync(kv->rows_dev.p, 0, (size_t)kv->max_batch * sizeof(RowState), st));
    B2_CUDA_CHECK(cudaMemsetAsync(kv->len_dev.p, 0, (size_t)kv->max_batch * 4, st));
    B2_CUDA_CHECK(cudaMemsetAsync(kv->tok.p, 0, (size_t)kv->max_batch * 4, st));
    kv->rows_host.assign(kv->max_batch, RowState{});
    kv->len_host.assign(kv->max_batch, 0);
    kv->stream_B = B; kv->stream_tag = v.tag; kv->stream_scheduled = 0;
    return ws_leave(m, st);
}

int b2_batch_set_row(b2_model* m, b2_kv* kv, int slot, int active, const b2_sampling* sp, int first_token, void* stream) {
    return b2_batch_set_row_ex(m, kv, slot, active, sp, nullptr, first_token, stream);
}

int b2_batch_set_row_ex(b2_model* m, b2_kv* kv, int slot, int active, const b2_sampling* sp, const b2_logits_proc* proc,
                        int first_token, void* stream) {
    B2_CHECK_ARG(m && kv && kv->m == m && slot >= 0 && slot < kv->stream_B, "b2_batch_set_row: bad slot %d", slot);
    B2_CHECK_ARG(kv->samp_host.per_row != 0, "b2_batch_set_row: b2_batch_begin first");
    RowState v = {};
    v.active = active ? 1 : 0; v.temperature = 1.f; v.top_p = 1.f; v.index = 1;  // draw 0 chose first_token
    if (active && sp != nullptr && sp->do_sample) {
        B2_CHECK_ARG(sp->temperature > 0.f && sp->top_p > 0.f && sp->top_p <= 1.f && sp->top_k >= 0, "b2_batch_set_row: bad sampling parameters");
        v.do_sample = 1; v.temperature = sp->temperature; v.top_p = sp->top_p; v.top_k = sp->top_k; v.seed = sp->seed;
    }
    ProcRow pr;
    B2_TRY(proc_row_of(active ? proc : nullptr, kv->max_seq + 1, &pr, "b2_batch_set_row_ex"));
    B2_CHECK_ARG(!pr.on || (first_token >= 0 && first_token < m->d.vocab), "b2_batch_set_row_ex: first_token %d out of range", first_token);
    std::lock_guard<std::mutex> lk(m->mu);
    DeviceGuard dg(m->device);
    B2_CHECK_ARG(!active || kv->len_host[slot] >= 1, "b2_batch_set_row: slot %d has an empty cache (prefill it first)", slot);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    B2_TRY(ws_enter(m, st));
    B2_TRY(proc_set_row(kv, slot, pr, proc ? proc->prompt_ids : nullptr, first_token, st));  // history: prompt, then first_token
    B2_TRY(row_state_set(kv->rows_dev.as<RowState>() + slot, v, active ? kv->tok.as<int32_t>() + slot : nullptr, first_token, st));
    if (!active) {  // a freed slot restarts from an empty cache
        B2_CUDA_CHECK(cudaMemsetAsync(kv->len_dev.as<int32_t>() + slot, 0, 4, st));
        kv->len_host[slot] = 0;
    }
    kv->rows_host[slot] = v;
    return ws_leave(m, st);
}

// Blocks (the Python binding releases the GIL around it) until token `index` of the current generation is in the ring.
// Takes no lock: other threads keep issuing work on the model while this one waits.
int b2_stream_wait(b2_kv* kv, int index, int32_t* tokens_host, int timeout_ms) {
    B2_CHECK_ARG(kv && tokens_host && index >= 0, "b2_stream_wait: bad argument");
    const int B = kv->stream_B;
    B2_CHECK_ARG(B >= 1, "b2_stream_wait: no streaming generation on this cache");
    B2_CHECK_ARG(index < kv->stream_scheduled, "b2_stream_wait: token %d has not been scheduled (%d scheduled)", index,
                 kv->stream_scheduled);
    volatile int32_t* slot = kv->ring_host + (size_t)(index % kv->ring_cap) * B;
    const int tag = 1 + (kv->stream_tag - 1 + index / kv->ring_cap) % 2047;  // the tag advances when the ring wraps (sampling.cu)
    struct timespec t0, t1;
    clock_gettime(CLOCK_MONOTONIC, &t0);
    for (unsigned long long spins = 0;; ++spins) {
        bool ready = true;
        for (int b = 0; b < B; ++b)
            if ((slot[b] >> 20) != tag) { ready = false; break; }
        if (ready) {
            for (int b = 0; b < B; ++b) tokens_host[b] = slot[b] & 0xFFFFF;
            return 0;
        }
        if (spins < 4096) continue;                 // ~ tens of microseconds of pure polling, then back off
        struct timespec nap = {0, 20000};
        nanosleep(&nap, nullptr);
        if ((spins & 255) == 0) {
            clock_gettime(CLOCK_MONOTONIC, &t1);
            const double ms = (t1.tv_sec - t0.tv_sec) * 1e3 + (t1.tv_nsec - t0.tv_nsec) * 1e-6;
            cudaError_t e = cudaPeekAtLastError();  // a sticky fault (illegal address, trap) would never publish the token
            if (e != cudaSuccess) { set_error("b2_stream_wait: CUDA error while waiting for token %d: %s", index, cudaGetErrorString(e)); return -2; }
            if (timeout_ms > 0 && ms > timeout_ms) { set_error("b2_stream_wait: token %d not published after %d ms", index, timeout_ms); return -3; }
        }
    }
}

int b2_op_preprocess_clip(const b2_preprocess_plan* pl, void* stream) {
    B2_CHECK_ARG(pl != nullptr, "b2_op_preprocess_clip: null plan");
    PreprocessArgs a;
    a.img = pl->img; a.H = pl->H; a.W = pl->W; a.pad_top = pl->pad_top; a.pad_left = pl->pad_left;
    for (int i = 0; i < 3; ++i) { a.bg[i] = pl->bg[i]; a.mean[i] = pl->mean[i]; a.stdv[i] = pl->stdv[i]; }
    a.h_bounds = pl->h_bounds; a.h_kk = pl->h_kk; a.h_ksize = pl->h_ksize; a.h_identity = pl->h_identity;
    a.v_bounds = pl->v_bounds; a.v_kk = pl->v_kk; a.v_ksize = pl->v_ksize; a.v_identity = pl->v_identity;
    a.y0 = pl->y0; a.rows = pl->rows; a.x_lo = pl->x_lo; a.y_lo = pl->y_lo; a.cols = pl->out; a.out = pl->out;
    a.tmp = pl->tmp; a.rescale = pl->rescale; a.pixels = pl->pixels; a.u8_out = pl->u8_out;
    return preprocess_clip_image(a, reinterpret_cast<cudaStream_t>(stream));
}

// standalone selection (unit tests, first-token choice outside a streaming generation): out_tokens[b] (device int32)
int b2_op_sample(const float* logits, int B, int V, const b2_sampling* sp, int index, int32_t* out_tokens, void* stream) {
    return b2_op_sample_ex(logits, B, V, sp, nullptr, index, out_tokens, nullptr, stream);
}

int b2_op_sample_ex(const float* logits, int B, int V, const b2_sampling* sp, const b2_logits_proc* proc, int index, int32_t* out_tokens,
                    float* out_processed, void* stream) {
    B2_CHECK_ARG(logits && out_tokens && B >= 1 && V >= 1 && index >= 0, "b2_op_sample: bad argument");
    SampleState v = {};
    v.temperature = 1.f; v.top_p = 1.f;
    if (sp != nullptr && sp->do_sample) {
        B2_CHECK_ARG(sp->temperature > 0.f && sp->top_p > 0.f && sp->top_p <= 1.f && sp->top_k >= 0, "b2_op_sample: bad sampling parameters");
        v.do_sample = 1; v.temperature = sp->temperature; v.top_p = sp->top_p; v.top_k = sp->top_k; v.seed = sp->seed;
    }
    v.pub_counter = index;
    // processors: a scratch state whose row b holds proc[b]'s prompt ids as its history
    std::vector<ProcRow> pr(proc ? B : 0);
    int cap = 1;
    bool any = false;
    for (int b = 0; b < (int)pr.size(); ++b) {
        B2_TRY(proc_row_of(proc + b, INT_MAX, &pr[b], "b2_op_sample_ex"));
        cap = std::max(cap, proc[b].prompt_len + 1);
        any = any || pr[b].on;
    }
    // one scratch buffer: SampleState, then (with processors) ProcRow[B], history int32 [B][cap] and the bitmap [B][words]
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const int words = (V + 31) / 32;
    static_assert(sizeof(SampleState) <= 256, "b2_op_sample_ex scratch layout");
    const size_t off_rows = 256, off_hist = off_rows + (size_t)B * sizeof(ProcRow), off_bits = off_hist + (size_t)B * cap * sizeof(int32_t);
    DevBuf tmp;
    B2_TRY(tmp.alloc(any ? off_bits + (size_t)B * words * sizeof(uint32_t) : sizeof(SampleState) + 64));
    ProcState ps = {};
    int r = 0;
    if (any) {
        ps.rows = reinterpret_cast<ProcRow*>(tmp.as<char>() + off_rows);
        ps.hist = reinterpret_cast<int32_t*>(tmp.as<char>() + off_hist);
        ps.bits = reinterpret_cast<uint32_t*>(tmp.as<char>() + off_bits);
        ps.cap = cap; ps.words = words;
        if (cudaMemsetAsync(ps.rows, 0, (size_t)B * sizeof(ProcRow), st) != cudaSuccess) {
            set_error("b2_op_sample_ex: %s", cudaGetErrorString(cudaGetLastError()));
            r = -2;
        }
        for (int b = 0; b < B && r == 0; ++b)
            if (pr[b].on) r = proc_seed(ps, b, pr[b], proc[b].prompt_ids, pr[b].prompt_len, -1, V, st);
    }
    if (r == 0) r = sample_state_set(tmp.as<SampleState>(), v, st);
    if (r == 0)
        r = sample_publish(logits, V, B, tmp.as<SampleState>(), nullptr, out_tokens, nullptr, nullptr, nullptr, nullptr, 0, SP_SELECT, 0,
                           ps, out_processed, st);
    cudaError_t e = cudaStreamSynchronize(st);
    tmp.free();
    if (r != 0) return r;
    B2_CUDA_CHECK(e);
    return 0;
}

int b2_argmax(const float* logits, int B, int V, int32_t* out, void* stream) {
    B2_CHECK_ARG(logits && out, "b2_argmax: null argument");
    return argmax_f32(logits, B, V, out, reinterpret_cast<cudaStream_t>(stream));
}

// ---------------------------------------------------------------------------------------------------------
// single-kernel entry points
// ---------------------------------------------------------------------------------------------------------
int b2_op_gemm(const void* A, int lda, const void* W, int ldw, const void* bias, const void* residual, int ld_res,
               void* out, int ld_out, int out_fp32, int M, int N, int K, int act, int bn_override, void* stream) {
    B2_CHECK_ARG(A && W && out, "b2_op_gemm: null argument");
    GemmArgs g;
    g.A = A; g.lda = lda; g.W = W; g.ldw = ldw; g.bias = bias; g.residual = residual; g.ld_res = ld_res;
    g.out = out; g.ld_out = ld_out; g.out_fp32 = out_fp32; g.M = M; g.N = N; g.K = K; g.act = act;
    g.bn_override = bn_override;
    return gemm_bf16(g, reinterpret_cast<cudaStream_t>(stream));
}

int b2_op_gemv(const void* x, int64_t ldx, const void* W, int ldw, const void* norm_gamma, float eps,
               const void* residual, int ld_res, void* out, int ld_out, int out_fp32, int B, int N, int K, int act,
               void* stream) {
    B2_CHECK_ARG(x && W && out, "b2_op_gemv: null argument");
    return gemv(x, ldx, W, ldw, norm_gamma, eps, residual, ld_res, out, ld_out, out_fp32, B, N, K, act,
                reinterpret_cast<cudaStream_t>(stream));
}

int b2_op_quantize_nf4(const void* w, int N, int K, void* codes, float* absmax, void* stream) {
    return quantize_nf4(w, K, N, K, codes, absmax, 0, reinterpret_cast<cudaStream_t>(stream));
}

int b2_op_dequantize_nf4(const void* codes, const float* absmax, int N, int K, void* out, void* stream) {
    Nf4Matrix mt;
    mt.q = codes; mt.absmax = absmax; mt.out = out; mt.N = N; mt.K = K;
    return dequantize_nf4(&mt, 1, 0, reinterpret_cast<cudaStream_t>(stream));
}

int b2_op_gemv_nf4(const void* x, int64_t ldx, const void* codes, const float* absmax, const void* norm_gamma, float eps,
                   const void* residual, int ld_res, void* out, int ld_out, int B, int N, int K, int act, void* stream) {
    B2_CHECK_ARG(x && codes && absmax && out, "b2_op_gemv_nf4: null argument");
    GemvArgs g;
    g.x = x; g.ldx = ldx; g.norm_gamma = norm_gamma; g.eps = eps; g.residual = residual; g.ld_res = ld_res;
    g.out = out; g.ld_out = ld_out; g.B = B; g.N = N; g.K = K; g.act = act;
    return gemv_nf4(g, codes, absmax, reinterpret_cast<cudaStream_t>(stream));
}

int b2_op_gemm_skinny(const void* x, int ldx, const void* W, int ldw, const void* residual, int ld_res, void* out,
                      int ld_out, int out_fp32, int B, int N, int K, int act, void* workspace, int64_t workspace_bytes,
                      void* counters, void* stream) {
    B2_CHECK_ARG(x && W && out && workspace && counters, "b2_op_gemm_skinny: null argument");
    SkinnyArgs g;
    g.x = x; g.ldx = ldx; g.W = W; g.ldw = ldw; g.residual = residual; g.ld_res = ld_res;
    g.out = out; g.ld_out = ld_out; g.out_fp32 = out_fp32; g.B = B; g.N = N; g.K = K; g.act = act;
    g.partial = reinterpret_cast<float*>(workspace); g.partial_bytes = (size_t)workspace_bytes;
    g.counters = reinterpret_cast<int*>(counters);
    return gemm_skinny_bf16(g, reinterpret_cast<cudaStream_t>(stream));
}
int b2_op_gemm_skinny_fp8(const void* xq, int ldx, const float* x_scale, const void* Wq, int ldw, const float* w_scale,
                          const void* residual, int ld_res, void* out, int ld_out, int out_fp32, int B, int N, int K, int act,
                          void* workspace, int64_t workspace_bytes, void* counters, void* stream) {
    B2_CHECK_ARG(xq && Wq && x_scale && w_scale && out && workspace && counters, "b2_op_gemm_skinny_fp8: null argument");
    SkinnyArgs g;
    g.x = xq; g.ldx = ldx; g.W = Wq; g.ldw = ldw; g.residual = residual; g.ld_res = ld_res;
    g.out = out; g.ld_out = ld_out; g.out_fp32 = out_fp32; g.B = B; g.N = N; g.K = K; g.act = act;
    g.partial = reinterpret_cast<float*>(workspace); g.partial_bytes = (size_t)workspace_bytes;
    g.counters = reinterpret_cast<int*>(counters);
    g.w_scale = w_scale; g.x_scale = x_scale;
    return gemm_skinny_fp8(g, reinterpret_cast<cudaStream_t>(stream));
}
int b2_op_quantize_rows_e4m3(const void* x, int64_t ldx, int rows, int K, void* q, int64_t ldq, float* scale, void* stream) {
    B2_CHECK_ARG(x && q && scale, "b2_op_quantize_rows_e4m3: null argument");
    return quantize_rows_e4m3(x, ldx, rows, K, q, ldq, scale, reinterpret_cast<cudaStream_t>(stream));
}
int b2_op_rmsnorm_quant_e4m3(const void* x, const void* gamma, void* q, float* scale, int rows, int cols, float eps,
                             void* stream) {
    B2_CHECK_ARG(x && gamma && q && scale, "b2_op_rmsnorm_quant_e4m3: null argument");
    return rmsnorm_quant_e4m3(x, cols, gamma, q, cols, scale, rows, cols, eps, reinterpret_cast<cudaStream_t>(stream));
}
int64_t b2_op_gemm_skinny_workspace_bytes(int B, int N, int K) {
    if (B < 1 || B > 128 || N < 1 || K < 1) return -1;
    return (int64_t)gemm_skinny_workspace_bytes(B, N, K);
}
int64_t b2_op_gemm_skinny_counter_bytes(int N) { return N < 1 ? -1 : (int64_t)gemm_skinny_counter_bytes(N); }

int b2_op_layernorm(const void* x, const void* gamma, const void* beta, void* y, int rows, int cols, float eps,
                    void* stream) {
    B2_CHECK_ARG(x && gamma && beta && y, "b2_op_layernorm: null argument");
    return layernorm_bf16(x, gamma, beta, y, rows, cols, eps, reinterpret_cast<cudaStream_t>(stream));
}

int b2_op_rmsnorm(const void* x, const void* gamma, void* y, int rows, int cols, float eps, void* stream) {
    B2_CHECK_ARG(x && gamma && y, "b2_op_rmsnorm: null argument");
    return rmsnorm_bf16(x, cols, gamma, y, rows, cols, eps, reinterpret_cast<cudaStream_t>(stream));
}

int b2_op_flash_attn(const void* q, const void* k, const void* v, void* o, const int32_t* seq_lens, int B, int S,
                     int H, int D, int causal, float scale, void* stream) {
    B2_CHECK_ARG(q && k && v && o, "b2_op_flash_attn: null argument");
    FlashArgs fa;
    const int64_t ts = (int64_t)H * D, bs = (int64_t)S * H * D;
    fa.q = q; fa.q_bs = bs; fa.q_ts = ts; fa.q_hs = D;
    fa.k = k; fa.k_bs = bs; fa.k_ts = ts; fa.k_hs = D;
    fa.v = v; fa.v_bs = bs; fa.v_ts = ts; fa.v_hs = D;
    fa.o = o; fa.o_bs = bs; fa.o_ts = ts; fa.o_hs = D;
    fa.seq_lens = seq_lens; fa.B = B; fa.H = H; fa.S = S; fa.D = D; fa.causal = causal; fa.scale = scale;
    return flash_attn_bf16(fa, reinterpret_cast<cudaStream_t>(stream));
}

int b2_op_rope_kv_write(void* qkv, void* kcache, void* vcache, int B, int S, int H, int D, int Smax, float theta,
                        void* stream) {
    B2_CHECK_ARG(qkv && kcache && vcache, "b2_op_rope_kv_write: null argument");
    return rope_kv_write(qkv, kcache, vcache, B, S, H, D, Smax, theta, reinterpret_cast<cudaStream_t>(stream));
}

int64_t b2_op_decode_attn_mq_scratch_bytes(int B, int H, int nsplit) {
    if (B < 1 || H < 1 || nsplit < 1) return -1;
    return (int64_t)decode_attn_mq_scratch_bytes(B, H, nsplit);
}

int b2_op_decode_attn_mq_nsplit(int H, int Smax) {
    B2_CHECK_ARG(H >= 1 && Smax >= 1, "b2_op_decode_attn_mq_nsplit: bad shape");
    return decode_nsplit(1, H, Smax, decode_attn_mq_ctas_per_sm());
}

int b2_op_decode_attn_mq(const void* qkv, const void* kcache, const void* vcache, const int32_t* cur_len, void* out, void* scratch,
                         int B, int R, int H, int Smax, int nsplit, float scale, void* stream) {
    B2_CHECK_ARG(qkv && kcache && vcache && cur_len && out && scratch, "b2_op_decode_attn_mq: null argument");
    B2_CHECK_ARG(B >= 1 && H >= 1 && nsplit >= 1 && Smax >= 1, "b2_op_decode_attn_mq: bad shape");
    DecodeAttnArgs da;
    da.qkv = qkv; da.kcache = const_cast<void*>(kcache); da.vcache = const_cast<void*>(vcache); da.cur_len = cur_len; da.out = out;
    da.partial = reinterpret_cast<float*>(scratch);
    da.counters = reinterpret_cast<int32_t*>(reinterpret_cast<char*>(scratch) + decode_attn_mq_scratch_bytes(B, H, nsplit) -
                                             (size_t)B * H * sizeof(int32_t));
    da.B = B; da.R = R; da.H = H; da.D = 128; da.Smax = Smax; da.nsplit = nsplit; da.scale = scale;
    return decode_attn_mq_bf16(da, reinterpret_cast<cudaStream_t>(stream));
}

int b2_op_prompt_lookup(const int32_t* hist, int len, int num_tokens, int max_ngram, int max_length, const int32_t* eos_host, int n_eos,
                        int V, int32_t* out_tokens, int32_t* out_draft_len, void* stream) {
    B2_CHECK_ARG(hist && out_tokens && out_draft_len && len >= 1, "b2_op_prompt_lookup: bad argument");
    B2_CHECK_ARG(num_tokens >= 1 && num_tokens < kSpecMaxRows && max_ngram >= 1 && max_length >= 1,
                 "b2_op_prompt_lookup: num_tokens must be in 1..%d, max_ngram and max_length >= 1", kSpecMaxRows - 1);
    B2_CHECK_ARG(n_eos >= 0 && n_eos <= kProcMaxEos && (n_eos == 0 || eos_host), "b2_op_prompt_lookup: bad eos ids");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    // scratch: SpecState, SampleState, tok[1], history [len]
    const size_t off_st = (sizeof(SpecState) + 255) / 256 * 256, off_tok = off_st + 256, off_hist = off_tok + 256;
    DevBuf tmp;
    B2_TRY(tmp.alloc(off_hist + (size_t)len * 4));
    SpecState ss = {};
    ss.K = num_tokens; ss.ngram = max_ngram; ss.max_new = max_length; ss.n_eos = n_eos;
    for (int i = 0; i < n_eos; ++i) ss.eos[i] = eos_host[i];
    ss.hist_len = len - 1;  // hist[len - 1] is the pending token
    SampleState sst = {};
    int32_t* tok = reinterpret_cast<int32_t*>(tmp.as<char>() + off_tok);
    int32_t* h = reinterpret_cast<int32_t*>(tmp.as<char>() + off_hist);
    int r = 0;
    if (cudaMemcpyAsync(tmp.p, &ss, sizeof ss, cudaMemcpyHostToDevice, st) != cudaSuccess ||
        cudaMemcpyAsync(tmp.as<char>() + off_st, &sst, sizeof sst, cudaMemcpyHostToDevice, st) != cudaSuccess ||
        cudaMemcpyAsync(h, hist, (size_t)len * 4, cudaMemcpyDefault, st) != cudaSuccess ||
        cudaMemcpyAsync(tok, hist + len - 1, 4, cudaMemcpyDefault, st) != cudaSuccess) {
        set_error("b2_op_prompt_lookup: %s", cudaGetErrorString(cudaGetLastError()));
        r = -2;
    }
    SpecState* dss = tmp.as<SpecState>();
    if (r == 0) r = prompt_lookup(h, dss, reinterpret_cast<SampleState*>(tmp.as<char>() + off_st), tok, V, num_tokens + 1, st);
    if (r == 0 && (cudaMemcpyAsync(out_tokens, tmp.as<char>() + offsetof(SpecState, rows), (size_t)(num_tokens + 1) * 4, cudaMemcpyDefault, st) != cudaSuccess ||
                   cudaMemcpyAsync(out_draft_len, tmp.as<char>() + offsetof(SpecState, draft_len), 4, cudaMemcpyDefault, st) != cudaSuccess)) {
        set_error("b2_op_prompt_lookup: %s", cudaGetErrorString(cudaGetLastError()));
        r = -2;
    }
    cudaError_t e = cudaStreamSynchronize(st);
    tmp.free();
    if (r != 0) return r;
    B2_CUDA_CHECK(e);
    return 0;
}

int64_t b2_op_decode_attn_shared_scratch_bytes(int B, int H, int nsplit) {
    if (B < 1 || H < 1 || nsplit < 1) return -1;
    return (int64_t)(decode_attn_shared_scratch_bytes(B, H, nsplit) + (size_t)B * (sizeof(PrefixGroup) + sizeof(int32_t)));
}

int b2_op_decode_attn_shared_nsplit(int B, int H, int Smax) {
    B2_CHECK_ARG(B >= 1 && H >= 1 && Smax >= 1, "b2_op_decode_attn_shared_nsplit: bad shape");
    return decode_nsplit(B, H, Smax, decode_attn_shared_ctas_per_sm());
}

int b2_op_decode_attn_shared(const void* qkv, void* kcache, void* vcache, const int32_t* cur_len, const b2_prefix_group* groups_host,
                             int G, void* out, void* scratch, int B, int H, int Smax, int nsplit, float theta, float scale,
                             void* stream) {
    B2_CHECK_ARG(qkv && kcache && vcache && cur_len && out && scratch && (G == 0 || groups_host), "b2_op_decode_attn_shared: null argument");
    B2_CHECK_ARG(B >= 1 && H >= 1 && nsplit >= 1 && Smax >= 1 && G >= 0 && G <= B, "b2_op_decode_attn_shared: bad shape");
    std::vector<PrefixGroup> tab(G);
    std::vector<int32_t> row_prefix(B, 0);
    for (int g = 0; g < G; ++g) {
        const b2_prefix_group& x = groups_host[g];
        B2_CHECK_ARG(x.n_rows >= 1 && x.n_rows <= kPrefixGroupRows && x.src_slot >= 0 && x.src_slot < B && x.prefix_len >= 1 &&
                     x.prefix_len <= Smax, "b2_op_decode_attn_shared: bad group %d", g);
        tab[g].src_slot = x.src_slot; tab[g].prefix_len = x.prefix_len; tab[g].n_rows = x.n_rows;
        for (int r = 0; r < kPrefixGroupRows; ++r) tab[g].rows[r] = r < x.n_rows ? x.rows[r] : 0;
        for (int r = 0; r < x.n_rows; ++r) {
            B2_CHECK_ARG(x.rows[r] >= 0 && x.rows[r] < B && row_prefix[x.rows[r]] == 0, "b2_op_decode_attn_shared: group %d row %d", g,
                         x.rows[r]);
            row_prefix[x.rows[r]] = x.prefix_len;
        }
    }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const size_t attn = decode_attn_shared_scratch_bytes(B, H, nsplit);
    PrefixGroup* dtab = reinterpret_cast<PrefixGroup*>(reinterpret_cast<char*>(scratch) + attn);
    int32_t* dprefix = reinterpret_cast<int32_t*>(dtab + B);
    if (G > 0) B2_CUDA_CHECK(cudaMemcpyAsync(dtab, tab.data(), (size_t)G * sizeof(PrefixGroup), cudaMemcpyHostToDevice, st));
    B2_CUDA_CHECK(cudaMemcpyAsync(dprefix, row_prefix.data(), (size_t)B * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    DecodeAttnArgs da;
    da.qkv = qkv; da.kcache = kcache; da.vcache = vcache; da.cur_len = cur_len; da.out = out;
    da.partial = reinterpret_cast<float*>(scratch);
    da.counters = reinterpret_cast<int32_t*>(reinterpret_cast<char*>(scratch) + attn - (size_t)B * H * sizeof(int32_t));
    da.B = B; da.H = H; da.D = 128; da.Smax = Smax; da.nsplit = nsplit; da.theta = theta; da.scale = scale;
    B2_TRY(decode_attn_shared_bf16(da, dtab, dprefix, G, st));
    B2_CUDA_CHECK(cudaStreamSynchronize(st));  // pageable host sources
    return 0;
}

int64_t b2_op_decode_attn_scratch_bytes(int B, int H, int nsplit) {
    return (int64_t)B * H * 4 /*counters*/ + 256 + (int64_t)B * H * nsplit * (128 + 2) * 4;
}

int b2_op_decode_attn(const void* qkv, void* kcache, void* vcache, const int32_t* cur_len, void* out, void* scratch,
                      int B, int H, int Smax, int nsplit, float theta, float scale, void* stream) {
    B2_CHECK_ARG(qkv && kcache && vcache && cur_len && out && scratch, "b2_op_decode_attn: null argument");
    DecodeAttnArgs da;
    da.qkv = qkv; da.kcache = kcache; da.vcache = vcache; da.cur_len = cur_len; da.out = out;
    da.counters = reinterpret_cast<int32_t*>(scratch);
    const size_t off = ((size_t)B * H * 4 + 255) / 256 * 256;
    da.partial = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(scratch) + off);
    da.B = B; da.H = H; da.D = 128; da.Smax = Smax; da.nsplit = nsplit; da.theta = theta; da.scale = scale;
    return decode_attn_bf16(da, reinterpret_cast<cudaStream_t>(stream));
}

int b2_op_decode_attn_e4m3(const void* qkv, void* k8, void* v8, float* kscale, float* vscale, const int32_t* cur_len, void* out,
                           void* scratch, int B, int H, int Smax, int nsplit, float theta, float scale, void* stream) {
    B2_CHECK_ARG(qkv && k8 && v8 && kscale && vscale && cur_len && out && scratch, "b2_op_decode_attn_e4m3: null argument");
    DecodeAttnArgs da;
    da.qkv = qkv; da.kcache = k8; da.vcache = v8; da.kscale = kscale; da.vscale = vscale; da.cur_len = cur_len; da.out = out;
    da.counters = reinterpret_cast<int32_t*>(scratch);
    da.partial = reinterpret_cast<float*>(reinterpret_cast<char*>(scratch) + (((size_t)B * H * 4 + 255) / 256) * 256);
    da.B = B; da.H = H; da.D = 128; da.Smax = Smax; da.nsplit = nsplit; da.theta = theta; da.scale = scale;
    return decode_attn_e4m3(da, reinterpret_cast<cudaStream_t>(stream));
}

int b2_op_decode_attn_nsplit(int B, int H, int Smax, int kv_dtype) {
    B2_CHECK_ARG(B >= 1 && H >= 1 && Smax >= 1, "b2_op_decode_attn_nsplit: bad shape");
    B2_CHECK_ARG(kv_dtype == B2_KV_BF16 || kv_dtype == B2_KV_E4M3, "b2_op_decode_attn_nsplit: unknown kv_dtype %d", kv_dtype);
    return decode_nsplit(B, H, Smax, kv_dtype == B2_KV_E4M3 ? decode_attn_e4m3_ctas_per_sm() : decode_attn_ctas_per_sm());
}

int b2_op_kv_quantize_e4m3(const void* kstage, const void* vstage, void* k8, void* v8, float* kscale, float* vscale,
                           const int32_t* seq_lens, int B, int S, int H, int Smax, void* stream) {
    B2_CHECK_ARG(kstage && vstage && k8 && v8 && kscale && vscale, "b2_op_kv_quantize_e4m3: null argument");
    return kv_quantize_e4m3(kstage, vstage, k8, v8, kscale, vscale, seq_lens, B, S, H, 128, Smax, reinterpret_cast<cudaStream_t>(stream));
}

int b2_op_flash_attn_kv(const void* q, const void* kcache, const void* vcache, void* o, const int32_t* pos0, const int32_t* seq_lens,
                        int B, int S, int H, int Smax, float scale, void* stream) {
    B2_CHECK_ARG(q && kcache && vcache && o && pos0, "b2_op_flash_attn_kv: null argument");
    B2_CHECK_ARG(B >= 1 && S >= 1 && H >= 1 && Smax >= 1, "b2_op_flash_attn_kv: bad shape B=%d S=%d H=%d Smax=%d", B, S, H, Smax);
    const int D = 128;
    FlashArgs fa;
    fa.q = q; fa.q_bs = (int64_t)S * H * D; fa.q_ts = (int64_t)H * D; fa.q_hs = D;
    fa.k = kcache; fa.k_bs = (int64_t)H * Smax * D; fa.k_ts = D; fa.k_hs = (int64_t)Smax * D;
    fa.v = vcache; fa.v_bs = fa.k_bs; fa.v_ts = D; fa.v_hs = fa.k_hs;
    fa.o = o; fa.o_bs = fa.q_bs; fa.o_ts = fa.q_ts; fa.o_hs = D;
    fa.seq_lens = seq_lens; fa.pos0 = pos0; fa.Skv = Smax;
    fa.B = B; fa.H = H; fa.S = S; fa.D = D; fa.causal = 1; fa.scale = scale;
    return flash_attn_bf16(fa, reinterpret_cast<cudaStream_t>(stream));
}

int b2_op_rope_kv_write_at(void* qkv, void* kcache, void* vcache, const int32_t* pos0, int B, int S, int H, int D, int Smax,
                           float theta, void* stream) {
    B2_CHECK_ARG(qkv && kcache && vcache && pos0, "b2_op_rope_kv_write_at: null argument");
    return rope_kv_write(qkv, kcache, vcache, B, S, H, D, Smax, theta, reinterpret_cast<cudaStream_t>(stream), pos0);
}

int b2_op_kv_dequantize_e4m3(const void* k8, const void* v8, const float* kscale, const float* vscale, const int32_t* pos0,
                             void* kdst, void* vdst, int B, int H, int Smax, int S_dst, void* stream) {
    return kv_dequantize_e4m3(k8, v8, kscale, vscale, pos0, kdst, vdst, B, H, Smax, S_dst, reinterpret_cast<cudaStream_t>(stream));
}

int b2_op_kv_quantize_e4m3_at(const void* kstage, const void* vstage, void* k8, void* v8, float* kscale, float* vscale,
                              const int32_t* pos0, const int32_t* seq_lens, int B, int S, int S_src, int H, int Smax, void* stream) {
    B2_CHECK_ARG(kstage && vstage && k8 && v8 && kscale && vscale && pos0, "b2_op_kv_quantize_e4m3_at: null argument");
    B2_CHECK_ARG(S_src >= 1, "b2_op_kv_quantize_e4m3_at: S_src=%d", S_src);
    return kv_quantize_e4m3(kstage, vstage, k8, v8, kscale, vscale, seq_lens, B, S, H, 128, Smax, reinterpret_cast<cudaStream_t>(stream),
                            pos0, S_src);
}

int b2_op_interleave_gate_up(const void* gate, const void* up, void* out, int I, int h, void* stream) {
    B2_CHECK_ARG(gate && up && out, "b2_op_interleave_gate_up: null argument");
    return interleave_gate_up(gate, up, out, I, h, reinterpret_cast<cudaStream_t>(stream));
}

int b2_op_im2col(const void* pixels, void* out, int B, int img, int patch, int kpad, void* stream) {
    B2_CHECK_ARG(pixels && out, "b2_op_im2col: null argument");
    return vit_im2col(pixels, out, B, img, patch, kpad, reinterpret_cast<cudaStream_t>(stream));
}

}  // extern "C"
