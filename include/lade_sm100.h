/*
 * lade_sm100.h -- C ABI of the H100-native lookahead/verification decoding step.
 *
 * Drop-in boundary for ONE hot path of hao-ai-lab/LookaheadDecoding ("lade"): the Jacobi lookahead +
 * n-gram verification step.  Every entry point names the reference interface it replaces
 * (paths relative to the reference checkout, file:line).  Plain C: device tensors are passed as raw
 * device pointers (torch `tensor.data_ptr()`), `stream` is a `cudaStream_t` passed as void*.
 *
 * Conventions
 *   - every function returns 0 (LADE_OK) or a negative LADE_E* code; no C++ exception crosses the
 *     boundary, nothing calls exit().  `lade_strerror` maps codes to text; `lade_last_cuda_error`
 *     returns the text of the last CUDA error seen by the calling thread's library calls.
 *   - all work is stream-ordered on the caller's stream; no hidden synchronisation; every launch is
 *     CUDA-graph capturable (per-step scalars such as the KV length live in device memory).
 *   - ownership: the caller owns every tensor (weights, activations, KV cache, scratch); the library
 *     owns only `LadeCtx` (device-resident int32 window / n-gram pool / token buffers).
 *   - one `LadeCtx` per generate() call per rank, driven by a single host thread.
 *
 * Data layouts (all row-major, innermost last)
 *   KV cache of one layer : K and V each [n_kv_heads][kv_capacity][head_dim] bf16
 *   Q (post-RoPE)         : [n_heads][q_pad][head_dim] bf16
 *   attention output      : [q_rows][n_heads*head_dim] bf16
 *   step rows             : ids/pos/rowdesc int32 [q_pad] ; rowmask uint32 [q_pad][mask_words]
 *   step meta             : int32 [LADE_META_INTS] (indices LADE_M_*)
 *   lm rows / argmax slots: int32 [lm_cap], lm_cap = 1 + (W+N-3) + G*(N-1):
 *                             slot 0 = row predicting the next token, slots [1, 1+W+N-3) = rows of the
 *                             newest window level, slots [1+W+N-3, lm_cap) = verification rows.
 */
#ifndef LADE_SM100_H_
#define LADE_SM100_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LADE_OK 0
#define LADE_EINVAL (-1)      /* bad argument / unsupported shape */
#define LADE_ECUDA (-2)       /* a CUDA runtime call failed (see lade_last_cuda_error) */
#define LADE_ENOMEM (-3)
#define LADE_EUNSUPPORTED (-4)
#define LADE_ESTATE (-5)      /* call sequence violated */

/* row classes carried by the row descriptors (rowdesc = class<<30 | block<<15 | index) */
#define LADE_ROW_PREFIX 0
#define LADE_ROW_WINDOW 1
#define LADE_ROW_GUESS 2
#define LADE_ROW_PAD 3

/* indices into the device-resident step meta record */
enum {
  LADE_M_Q_LEN = 0,       /* live rows of this step                                   */
  LADE_M_KV_LEN = 1,      /* committed KV rows before this step                       */
  LADE_M_N_INPUT = 2,     /* re-fed input rows (prompt length on the first step)      */
  LADE_M_LEVEL_OFFSET = 3,/* modeling_llama.py:136                                    */
  LADE_M_ALL_OFFSET = 4,  /* level_offset + dist_offset, modeling_llama.py:188        */
  LADE_M_TINY = 5,        /* level_sizes[-1], modeling_llama.py:132                   */
  LADE_M_N_LEVELS = 6,
  LADE_M_N_GUESS_TOK = 7, /* len(guess_tokens)                                        */
  LADE_M_IS_PREFILL = 8,
  LADE_M_PHASE = 9,       /* 0 prefill step, 1 window-fill step, 2 steady step        */
  LADE_M_Q_PAD = 10,      /* rows materialised (>= q_len; extra rows are PAD rows)    */
  LADE_M_DONE = 11,       /* generation finished: the step is a no-op                 */
  LADE_M_STEP = 12,
  LADE_META_INTS = 16
};

/* per-step result record written by lade_accept_update (device int32[LADE_RES_INTS]) */
enum {
  LADE_R_N_EMIT = 0,      /* tokens appended to the output this step (<= N-1)         */
  LADE_R_MAX_HIT = 1,
  LADE_R_MAX_HIT_IDX = 2,
  LADE_R_KV_SRC = 3,      /* first cache row of the accepted n-gram (decoding.py:1156)*/
  LADE_R_KV_DST = 4,      /* kvcache_len                                              */
  LADE_R_KV_LEN = 5,      /* committed rows after the step                            */
  LADE_R_DONE = 6,
  LADE_R_N_OUT = 7,       /* len(input_ids) after the step                            */
  LADE_R_STEPS = 8,
  LADE_R_N_GUESS = 9,     /* n-grams verified this step                               */
  LADE_R_HITS = 16,       /* hits[0..N-2]                                             */
  LADE_RES_INTS = 48
};

typedef struct LadeCtx LadeCtx;

/* lade.config_lade(...) knobs (lade/utils.py:13-37) + model shape */
typedef struct LadeConfig {
  int32_t window_size;      /* WINDOW_SIZE (W)                                        */
  int32_t level;            /* LEVEL (N) >= 3 (lade/decoding.py:902)                   */
  int32_t guess_set_size;   /* GUESS_SET_SIZE (G) > 0; -1 (unbounded set) unsupported */
  int32_t pool_from_prompt; /* POOL_FROM_PROMPT                                       */
  int32_t vocab_size;
  int32_t max_total_len;    /* capacity of the token buffers (prompt + new + N)       */
  int32_t n_eos;            /* number of eos ids (0..4)                               */
  int32_t eos_token_id[4];  /* eos_token_id[0] is the one decoding.py:1169 tests      */
  int32_t dist_workers;     /* DIST_WORKERS (lookahead parallelism), 1 = off          */
  int32_t rank;             /* LOCAL_RANK                                             */
} LadeConfig;

/* Greedy logits processors applied on device by lade_argmax_processed (HF transformers 5.5,
 * generation/logits_process.py).  The reference forbids any processor on its greedy path (lade/decoding.py:968);
 * greedy lookahead stays lossless under a processor that depends only on the prefix a row stands for, which is what
 * these three do.  One record per generate() call, written to device memory by lade_processors_upload. */
enum {
  LADE_PROC_REPETITION_PENALTY = 1, /* RepetitionPenaltyLogitsProcessor(penalty, prompt_ignore_length)           */
  LADE_PROC_NO_REPEAT_NGRAM = 2,    /* NoRepeatNGramLogitsProcessor(ngram_size)                                  */
  LADE_PROC_MIN_LENGTH = 4,         /* MinLengthLogitsProcessor / MinNewTokensLengthLogitsProcessor              */
  LADE_PROC_MAX_NGRAM = 64,
  LADE_PROC_MAX_EOS = 8
};
typedef struct LadeProcessors {
  int32_t flags;                  /* LADE_PROC_* bits of the active processors                                */
  uint32_t penalty_bits;          /* fp32 bits of the repetition penalty (> 0, finite)                        */
  int32_t prompt_ignore_length;   /* the penalty acts on prefix[prompt_ignore_length:]                       */
  int32_t ngram_size;             /* 1 .. LADE_PROC_MAX_NGRAM                                                 */
  int32_t eos_bound;              /* eos ids score -inf while the prefix is shorter: max(min_length,
                                     prompt_length_to_skip + min_new_tokens)                                  */
  int32_t n_eos;                  /* 0 .. LADE_PROC_MAX_EOS                                                   */
  int32_t eos_token_id[8];
} LadeProcessors;

/* Sampling warpers of lade_sample_verify_warped, in HF's list order (transformers 5.5,
 * GenerationMixin._get_logits_processor): TemperatureLogitsWarper -> TopKLogitsWarper -> TopPLogitsWarper ->
 * MinPLogitsWarper -> EpsilonLogitsWarper -> EtaLogitsWarper, every one with min_tokens_to_keep = 1 and filter value
 * -inf.  top_k = 0, top_p = 1 and 0 for the last three switch a warper off. */
typedef struct LadeWarpers {
  float temperature;   /* > 0                                                                         */
  int32_t top_k;       /* >= 0                                                                        */
  float top_p;         /* (0, 1]                                                                      */
  float min_p;         /* [0, 1]: drop probs < min_p * max(probs)                    (MinPLogitsWarper) */
  float epsilon;       /* 0 or (0, 1): drop probs < epsilon, never the maximum    (EpsilonLogitsWarper) */
  float eta;           /* 0 or (0, 1): drop probs < min(eta, sqrt(eta) * exp(-entropy)), never the maximum
                          (EtaLogitsWarper)                                                           */
} LadeWarpers;

/* ---- context --------------------------------------------------------------------------------- */

/* Allocates the device-resident decode state (window, n-gram pool, token buffers).
 * Replaces the python locals of jacobi_greedy_search_multilevel, lade/decoding.py:854-916. */
int lade_ctx_create(const LadeConfig* cfg, LadeCtx** out);
/* Frees the device state (the reference relies on python GC of the loop's locals, decoding.py:1221-1259). */
int lade_ctx_destroy(LadeCtx* ctx);

/* Start a generate() call: upload prompt ids and the initial lookahead window level 0
 * (W+N-3 tokens, drawn by the caller exactly as lade/decoding.py:887-902 does, so the python
 * `random` stream is consumed identically), clear the pool and, if POOL_FROM_PROMPT, fill it from
 * the prompt (lade/decoding.py:104-127, :915-916).  Host pointers; copied before return is NOT
 * guaranteed -- the buffers must stay valid until the stream reaches this point. */
int lade_ctx_reset(LadeCtx* ctx, void* stream, const int32_t* prompt_host, int32_t n_prompt,
                   const int32_t* window0_host, int32_t n_window0, int32_t max_length);

/* ---- step layout ------------------------------------------------------------------------------ */

/* Build the rows of the next step on device: token ids, position ids, row descriptors (mask classes),
 * the lm_head row list and the step meta record.  `q_pad` rows are written (rows past the live count
 * are PAD rows).  Replaces LlamaForCausalLM.jforward_multilevel's input assembly
 * (lade/models/modeling_llama.py:1458-1511), the pool lookup of lade/decoding.py:948-954 and the
 * mask of j_make_causal_mask_multilevel (modeling_llama.py:115-207) in its compact forms: one class
 * descriptor per row (`rowdesc`) and, for non-prefill steps, the visibility bitmask of the step block
 * (`rowmask`, bit c of row r = row r attends step column c; mask_words >= ceil(q_pad/32)). */
int lade_step_layout(LadeCtx* ctx, void* stream, int32_t q_pad, int32_t* ids_out, int32_t* pos_out,
                     int32_t* rowdesc_out, int32_t* lm_rows_out, int32_t* meta_out,
                     uint32_t* rowmask_out /* [q_pad][mask_words], nullable */, int32_t mask_words);

/* Expected live row count of the upcoming step as a pure function of the step index (host side, no
 * sync): prefill = P + W+N-3 ; fill step k ; steady = (N-1)*(W+G).  Returns the count or <0.
 * Mirrors the lengths of the tensors jforward_multilevel concatenates (modeling_llama.py:1458-1511) for the
 * fill_level schedule of decoding.py:1038-1066. */
int lade_step_rows_bound(const LadeConfig* cfg, int32_t n_prompt, int32_t step_index);

/* ---- floating-point kernels of the decoder layer ---------------------------------------------- */

/* out = weight * bf16(x_f32 * rsqrt(mean(x^2)+eps)) with optional fused residual add
 * (h = bf16(x + delta) is written to `h_out` first).  LlamaRMSNorm, modeling_llama.py:222-227 and the
 * residual adds of LlamaDecoderLayer.forward :883-889. */
int lade_rmsnorm(void* stream, const void* x, const void* delta /*nullable*/, const void* weight,
                 void* h_out /*nullable unless delta*/, void* out, int32_t rows, int32_t hidden, float eps);

/* Final-norm variant that gathers rows: out[i] = rmsnorm(x[rows_idx[i]] (+ delta[rows_idx[i]])).
 * LlamaModel.norm (modeling_llama.py:1240) restricted to the rows whose logits the loop reads (:1570-1606). */
int lade_rmsnorm_gather(void* stream, const void* x, const void* delta, const void* weight,
                        const int32_t* rows_idx, void* out, int32_t n_rows, int32_t hidden, float eps);

/* Rotary embedding + KV append: reads the fused QKV projection [rows][(Hq+2Hkv)*D], writes
 * Q'[Hq][q_pad][D] and appends K', V to the layer's cache at rows kv_len + r (kv_len from `meta`).
 * apply_rotary_pos_emb (modeling_llama.py:342-346, bf16 rounding of each product and of the sum) and
 * the torch.cat KV append (:513-516). cos/sin: [max_pos][D] in the model dtype (:255-256,:264-265). */
int lade_rope_append(void* stream, const void* qkv, const void* cos_tab, const void* sin_tab,
                     const int32_t* pos, const int32_t* meta, void* q_out, void* k_cache, void* v_cache,
                     int32_t rows, int32_t q_pad, int32_t n_heads, int32_t n_kv_heads, int32_t head_dim,
                     int32_t kv_capacity, int32_t max_pos);

/* Qwen3 variant (Qwen3ForCausalLM): the per-head RMSNorm of q and of k in front of the rotary embedding, fused into the
 * same pass.  Qwen3Attention.forward (transformers modeling_qwen3.py):
 *     query_states = self.q_norm(self.q_proj(hidden_states).view(hidden_shape))      (the same for k with k_norm)
 *     query_states, key_states = apply_rotary_pos_emb(query_states, key_states, cos, sin)
 * with Qwen3RMSNorm.forward, the rounding points of LlamaRMSNorm, over each head of D elements:
 *     rstd = rsqrt(sum(x^2) / D + eps)  (fp32),  n = T(x * rstd),  y = T(w * n)
 * then the rotary embedding of lade_rope_append on y, with its roundings.  V is appended unchanged.
 * q_norm_w, k_norm_w: device T[head_dim] (the two modules' weights), 16-byte aligned; eps: the modules'
 * variance_epsilon.  Arguments, layouts and errors otherwise as lade_rope_append; LADE_EINVAL also for a null or
 * misaligned weight, eps negative or not finite, and head_dim / 16 not a power of two.  Nothing is launched on an
 * error.  _f16: fp16 models. */
int lade_rope_append_qknorm(void* stream, const void* qkv, const void* cos_tab, const void* sin_tab,
                            const int32_t* pos, const int32_t* meta, void* q_out, void* k_cache, void* v_cache,
                            int32_t rows, int32_t q_pad, int32_t n_heads, int32_t n_kv_heads, int32_t head_dim,
                            int32_t kv_capacity, int32_t max_pos, const void* q_norm_w, const void* k_norm_w, float eps);
int lade_rope_append_qknorm_f16(void* stream, const void* qkv, const void* cos_tab, const void* sin_tab,
                                const int32_t* pos, const int32_t* meta, void* q_out, void* k_cache, void* v_cache,
                                int32_t rows, int32_t q_pad, int32_t n_heads, int32_t n_kv_heads, int32_t head_dim,
                                int32_t kv_capacity, int32_t max_pos, const void* q_norm_w, const void* k_norm_w,
                                float eps);

/* Qwen2 / Qwen2.5 variant (Qwen2ForCausalLM): q_proj, k_proj and v_proj carry a bias, added before the rotary
 * embedding.  Qwen2Attention.forward (transformers modeling_qwen2.py):
 *     query_states = self.q_proj(hidden_states).view(hidden_shape).transpose(1, 2)      (the same for k and v)
 *     query_states, key_states = apply_rotary_pos_emb(query_states, key_states, cos, sin)
 * nn.Linear with a bias is addmm: the bias is added to the fp32 accumulator and the sum is rounded once.  So `qkv` is
 * here the fused projection's fp32 accumulator [rows][(Hq+2Hkv)*D] (float, 16-byte aligned), and every element is first
 * x = T(acc + float(bias)); RoPE of lade_rope_append then runs on q and k, v is appended as x.  bias: device
 * T[(Hq+2Hkv)*D], the three biases concatenated in qkv's column order, 16-byte aligned.  Arguments, layouts and
 * errors otherwise as lade_rope_append; LADE_EINVAL also for a null or misaligned bias or qkv.  Nothing is launched on
 * an error.  _f16: fp16 models. */
int lade_rope_append_bias(void* stream, const void* qkv, const void* cos_tab, const void* sin_tab,
                          const int32_t* pos, const int32_t* meta, void* q_out, void* k_cache, void* v_cache,
                          int32_t rows, int32_t q_pad, int32_t n_heads, int32_t n_kv_heads, int32_t head_dim,
                          int32_t kv_capacity, int32_t max_pos, const void* bias);
int lade_rope_append_bias_f16(void* stream, const void* qkv, const void* cos_tab, const void* sin_tab,
                              const int32_t* pos, const int32_t* meta, void* q_out, void* k_cache, void* v_cache,
                              int32_t rows, int32_t q_pad, int32_t n_heads, int32_t n_kv_heads, int32_t head_dim,
                              int32_t kv_capacity, int32_t max_pos, const void* bias);

/* Lookahead attention over the persistent KV cache (the roofline kernel).  softmax(QK^T/sqrt(D) +
 * lookahead mask) V with the mask bits of `rowmask` tested in registers (prefill steps: plain causal,
 * rowmask unused); all step rows see the committed cache.  Replaces LlamaAttention.forward's attention core (modeling_llama.py:520-541), the
 * dense mask of j_make_causal_mask_multilevel (:115-207) and flash_attn_lade.flash_attn_func(...,
 * lookahead=[...]) (:705-713).  `scratch` holds split-KV partials: lade_attn_scratch_bytes().
 * head_dim 128: wgmma/TMA kernel (impl 0 or 2) or the mma.sync kernel (impl 1); head_dim 64 (TinyLlama-style): the
 * mma.sync kernel (impl 0 or 1).  Other head dimensions: LADE_EUNSUPPORTED.
 * impl 3 (head_dim 128): the wgmma kernel's REFERENCE-ORDER variant -- the probabilities are normalised by the sum
 * of the whole row in fp32 and rounded to the model dtype afterwards, exactly the order of :530-541 (impl 2 is an online
 * softmax: it rounds exp(x - max) before the sum is known, which changes the last bit of about half of the outputs).
 * Every K/V tile of a KV split stays in shared memory, so kv_bound must be a true bound of kv_len + q_len and at most
 * 384 * n_splits (n_splits <= 8): LADE_EUNSUPPORTED otherwise.  Slower; a parity mode. */
int lade_attn_fwd(void* stream, const void* q, const void* k_cache, const void* v_cache, void* out,
                  const uint32_t* rowmask, int32_t mask_words, const int32_t* meta, void* scratch, int32_t q_pad,
                  int32_t n_heads, int32_t n_kv_heads, int32_t head_dim, int32_t kv_capacity,
                  int32_t kv_bound /* host upper bound of kv_len + q_len */, int32_t n_splits,
                  int32_t impl /* 0 = default (= 2), 1 = mma.sync path, 2 = wgmma/TMA path, 3 = its reference-order variant */);
/* Bytes of zero-initialised scratch `lade_attn_fwd` needs for a shape.  Every impl merges its KV splits through it:
 * [16384 int32 ticket counters, one per (head, q tile), zero at rest][(m, l) fp32 per split row][fp32 O per split row],
 * split-major, rows padded to 128.  Each split writes its partial rows and takes a ticket; the CTA that draws the last
 * one combines the splits and puts the counter back to 0, so the buffer needs no clearing between launches.  impl 3
 * also exchanges its row maxima and row sums through the (m, l) table.  Launches that share a scratch buffer must be
 * stream-ordered.  No reference counterpart. */
int64_t lade_attn_scratch_bytes(int32_t q_pad, int32_t n_heads, int32_t head_dim, int32_t n_splits);
/* Profiling aid: when set (device buffer of 16 int64 per CTA, or NULL to disable) the wgmma kernel records
 * %globaltimer (ns) at its phase boundaries in slots 0-7 (start, first K tile landed, first S ready, O final, partials
 * written, ticket drawn, -, end) and the SM it ran on in slot 15. */
int lade_debug_attn_timing(void* dev_buffer);

/* Measurement aid: force the programmatic-dependent-launch attribute of lade_attn_fwd on (1) / off (0), or back to the
 * environment default (-1, LADE_PDL).  With it on, a launch that follows a kernel which triggers its dependents early
 * (lade_rope_append in the decode step; another lade_attn_fwd in a back-to-back loop) overlaps its set-up with the
 * predecessor's tail; bench.py reports the kernel both ways. */
int lade_debug_attn_pdl(int32_t enable);

/* Projection GEMM of the lookahead step: c[m][n] (row stride ldc) = a[m][k] . w[n][k]^T, bf16 in/out, fp32
 * accumulation on the tensor cores (wgmma); w is an nn.Linear weight ([out_features][in_features], row-major).
 * Replaces q/k/v_proj (modeling_llama.py:447-449), o_proj (:541), gate/up/down_proj (:378) and lm_head (:1608)
 * for step row counts m <= 128; `a_rows` >= m is the number of addressable rows of the `a` buffer (rows >= m
 * are read but never stored).  tile_n / split_k = 0 lets the library pick (one wave of CTAs over the SMs);
 * tuning knobs ride in tile_n: bits [16,20) = pipeline depth cap, bit 20 = do not prefill the ring during CTA set-up.
 * Returns LADE_EUNSUPPORTED for m > 128, k % 64 != 0 or n % 8 != 0 (callers then use a library GEMM), and for
 * m < 1, a_rows < m, n < 1, k < 1, ldc < n or ldc % 8 != 0; LADE_EINVAL for a, w or c not 16-byte aligned.
 * Forced configurations (the low 16 bits of tile_n, or split_k, non-zero; a zero split_k is then 1, a zero tile the
 * library's choice) launch nothing and return LADE_EINVAL unless all of these hold:
 *   tile is a multiple of 32 in [32, 256]; split_k is 1, 2, 4 or 8 and divides the k / 64 k-blocks;
 *   with split_k > 1 the fp32 staging tile of the split reduction fits the pipeline ring it reuses:
 *     128 * (tile + 4) * 4 <= stages * (16384 + 128 * tile)  bytes, where
 *     stages = min(floor(231232 / (16384 + 128 * tile)), 11, k / 64 / split_k, depth cap if given).
 * Rows [m, a_rows) of `a` may hold anything, NaN included: output rows are independent and only rows < m and columns
 * < n of `c` are written, whatever ldc is. */
int lade_gemm_bf16(void* stream, const void* a, const void* w, void* c, int32_t m, int32_t a_rows, int32_t n, int32_t k,
                   int32_t ldc, int32_t tile_n, int32_t split_k);

/* FP8 projection, T = bf16 (lade_gemm_fp8) or fp16 (lade_gemm_fp8_f16); not on the engine's step (DESIGN.md §7.2):
 *   c[r][n] = T( __fmul_rn(__fmul_rn(sum_k a[r][k] * w[n][k], a_scale[r]), w_scale[n]) )
 * a: [a_rows][k] and w: [n][k] float8_e4m3fn bytes, row-major (the nn.Linear layout, K-major for wgmma); a_scale: [m]
 * and w_scale: [n] fp32, the scales of the row quantisation of lade_quant_rows_fp8 (see there).  The sum runs over
 * 128-deep k-blocks: each block on the tensor cores (m64nNk32 e4m3 wgmma into a zeroed accumulator), then added in fp32
 * on the CUDA cores; K splits are added in split order before the scales.  Requires k % 128 == 0, n % 8 == 0,
 * ldc % 8 == 0, ldc >= n, 16-byte aligned a / w / c.  Up to 256 rows stream each weight once; larger m loops over
 * 256-row chunks.  tile_n (32..128, multiple of 32; bits 16-19 a ring-depth cap, bit 20 = no ring prefill before the
 * CTA barrier) and split_k as for lade_gemm_bf16; the automatic choice depends on (n, k) only, so an output row is
 * the same bits whatever m is.  A rejected configuration returns LADE_EINVAL before anything is written. */
int lade_gemm_fp8(void* stream, const void* a, const float* a_scale, const void* w, const float* w_scale, void* c,
                  int32_t m, int32_t a_rows, int32_t n, int32_t k, int32_t ldc, int32_t tile_n, int32_t split_k);
int lade_gemm_fp8_f16(void* stream, const void* a, const float* a_scale, const void* w, const float* w_scale, void* c,
                      int32_t m, int32_t a_rows, int32_t n, int32_t k, int32_t ldc, int32_t tile_n, int32_t split_k);

/* e4m3 row quantisation, the same for activations (per token) and weights (per output channel).  For a row x of T:
 *   amax = max |x| (fp32); s = amax / 448 (fp32), or 1 when amax is 0 or not finite; q = e4m3(x / s) with the division
 *   in fp32, round to nearest even, saturated to +-448 (float8_e4m3fn).  A row holding inf or NaN quantises to
 *   undefined bytes.
 * lade_rmsnorm_quant_fp8: lade_rmsnorm's output row T(w * n), quantised to q_out [rows][hidden] / s_out [rows] instead
 *   of stored (h_out as in lade_rmsnorm).
 * lade_swiglu_quant_fp8: lade_swiglu's row T(T(silu(g)) * u), quantised to q_out [rows][inter] / s_out [rows].
 * lade_quant_rows_fp8: plain rows x [rows][cols] to q_out [rows][cols] / s_out [rows].
 * Every output row depends only on its own input row.  _f16: the fp16 twins. */
int lade_rmsnorm_quant_fp8(void* stream, const void* x, const void* delta, const void* weight, void* h_out, void* q_out,
                           float* s_out, int32_t rows, int32_t hidden, float eps);
int lade_rmsnorm_quant_fp8_f16(void* stream, const void* x, const void* delta, const void* weight, void* h_out, void* q_out,
                               float* s_out, int32_t rows, int32_t hidden, float eps);
int lade_swiglu_quant_fp8(void* stream, const void* gate_up, void* q_out, float* s_out, int32_t rows, int32_t inter);
int lade_swiglu_quant_fp8_f16(void* stream, const void* gate_up, void* q_out, float* s_out, int32_t rows, int32_t inter);
int lade_quant_rows_fp8(void* stream, const void* x, void* q_out, float* s_out, int32_t rows, int32_t cols);
int lade_quant_rows_fp8_f16(void* stream, const void* x, void* q_out, float* s_out, int32_t rows, int32_t cols);

/* Profiling aid: when set (device buffer of 4 * 1024 * 8 int64, or NULL to disable) the GEMM kernel records
 * %globaltimer (ns) at its phase boundaries per CTA, the last 4 launches round-robin. */
int lade_debug_gemm_timing(void* dev_buffer);

/* act = bf16(silu(gate)) * up on the fused [rows][2*inter] projection.  LlamaMLP, modeling_llama.py:378. */
int lade_swiglu(void* stream, const void* gate_up, void* out, int32_t rows, int32_t inter);

/* fp16 models (the dtype of the reference's README.md:159 / minimal.py:19; the BASELINE configs are bf16): the same
 * kernels instantiated on the element type -- every rounding point of the bf16 entry point of the same name without the
 * suffix happens in fp16 instead.  Arguments, layouts and error codes are those of the unsuffixed function.
 * lade_attn_fwd_f16 picks its kernel like lade_attn_fwd (wgmma/TMA for head_dim 128, mma.sync for 64 or impl 1). */
int lade_rmsnorm_f16(void* stream, const void* x, const void* delta, const void* weight, void* h_out, void* out,
                     int32_t rows, int32_t hidden, float eps);
int lade_rmsnorm_gather_f16(void* stream, const void* x, const void* delta, const void* weight,
                            const int32_t* rows_idx, void* out, int32_t n_rows, int32_t hidden, float eps);
int lade_rope_append_f16(void* stream, const void* qkv, const void* cos_tab, const void* sin_tab,
                         const int32_t* pos, const int32_t* meta, void* q_out, void* k_cache, void* v_cache,
                         int32_t rows, int32_t q_pad, int32_t n_heads, int32_t n_kv_heads, int32_t head_dim,
                         int32_t kv_capacity, int32_t max_pos);
int lade_swiglu_f16(void* stream, const void* gate_up, void* out, int32_t rows, int32_t inter);
int lade_argmax_rows_f16(void* stream, const void* logits, int32_t n_rows, int32_t vocab, int32_t ld,
                         int32_t* out_idx);
int lade_attn_fwd_f16(void* stream, const void* q, const void* k_cache, const void* v_cache, void* out,
                      const uint32_t* rowmask, int32_t mask_words, const int32_t* meta, void* scratch, int32_t q_pad,
                      int32_t n_heads, int32_t n_kv_heads, int32_t head_dim, int32_t kv_capacity,
                      int32_t kv_bound, int32_t n_splits, int32_t impl);
int lade_sample_verify_f16(LadeCtx* ctx, void* stream, const void* logits, int32_t ld, int32_t vocab,
                           const int32_t* argmax_slots, const int32_t* meta, float temperature, int32_t top_k, float top_p,
                           uint64_t* rng_state, int32_t* decision_out, float* debug_uniforms);

/* ---- token selection / accept / pool update ---------------------------------------------------- */

/* Row-wise argmax with lowest-index tie-break over bf16 logits [n_rows][vocab], rows `ld` >= vocab elements apart
 * (torch.argmax at lade/decoding.py:1021,1041,1052,1072,1102).  -inf and +inf compete like any value; a row of
 * nothing but -inf gives 0.  NaN is outside the contract (torch.argmax would return its index; this does not). */
int lade_argmax_rows(void* stream, const void* logits, int32_t n_rows, int32_t vocab, int32_t ld,
                     int32_t* out_idx);

/* lade_argmax_rows under the greedy logits processors of `proc_dev` (device LadeProcessors): every lm slot is scored
 * as HF's greedy _sample scores the position it stands for, argmax(processors(prefix, fp32(logits[slot]))), lowest
 * index on ties.  Prefix of slot 0: the committed ids out_ids[0, n_out); of verification slot 1+(W+N-3)+i (i below the
 * step's guess-token count; n-gram e = i / (N-1), position u = i % (N-1)): the committed ids followed by the n-gram's
 * tokens 0..u.  Window slots are plain argmax.  Lifts the reference's "no logits processors" restriction
 * (lade/decoding.py:968) for RepetitionPenaltyLogitsProcessor, NoRepeatNGramLogitsProcessor, MinLengthLogitsProcessor
 * and MinNewTokensLengthLogitsProcessor.  Reads n_out, the guess count and the guess tokens from the ctx state, so it
 * runs after lade_step_layout of the same step.  LADE_EUNSUPPORTED for vocab > 163840 (shared-memory bitmaps) or a
 * lookahead-parallel ctx.  With no flag set the output equals lade_argmax_rows. */
int lade_argmax_processed(LadeCtx* ctx, void* stream, const void* logits, int32_t n_rows, int32_t vocab, int32_t ld,
                          const LadeProcessors* proc_dev, int32_t* out_idx);
int lade_argmax_processed_f16(LadeCtx* ctx, void* stream, const void* logits, int32_t n_rows, int32_t vocab, int32_t ld,
                              const LadeProcessors* proc_dev, int32_t* out_idx);
/* Validate a host LadeProcessors record and copy it to `dev` on `stream` (stream-ordered; the host record may be
 * reused on return).  LADE_EINVAL for unknown flags, a penalty that is not finite and > 0, a negative
 * prompt_ignore_length, ngram_size outside 1..LADE_PROC_MAX_NGRAM, or more than LADE_PROC_MAX_EOS eos ids. */
int lade_processors_upload(void* stream, const LadeProcessors* host, LadeProcessors* dev);

/* Verification + state update of one step, fully on device: longest-prefix accept
 * (lade/decoding.py:1071-1084), window fill / shift (:1038-1066,:1119-1124), n-gram pool LRU update
 * (:37-63,:1116), emission with the EOS scan and POOL_FROM_PROMPT appends (:1165-1177), stopping
 * (:1205-1219).  `argmax_slots` uses the lm-row slot layout above.  Writes `result` (LADE_R_*). */
int lade_accept_update(LadeCtx* ctx, void* stream, const int32_t* argmax_slots, const int32_t* meta,
                       int32_t* result);

/* Sampling verification ON DEVICE for the reference's warper set {temperature, top-k, top-p} (decoding.py:375-377;
 * top_k = 0 and top_p = 1 switch the filters off) -- replaces the host loop of
 * jacobi_sample_multilevel, lade/decoding.py:445-546 (softmax of out_logits / T :445,:485; per n-gram position the
 * accept test over the n-grams still alive :495-516 (u <= min(1, p[token]) for the uniform u in (0, 1], which accepts
 * with probability p like the reference's random.random() < p), zero-and-renormalise on reject :518-520 (each test
 * normalised by the kept mass not yet rejected, summed afresh in float64: a sole survivor has p = 1),
 * residual multinomial draw :533-535; single multinomial draw on steps without candidates :458-480,:543-546) and
 * filter_window (:131-135,:578-580).  One kernel, one CTA; random numbers from a Philox4x32-10 stream whose
 * (seed, offset) live in `rng_state[2]` (device, uint64; the kernel advances the offset), so a sampling step replays
 * from a CUDA graph with no host round trip.  `logits`: bf16 [lm slots][ld], slot order of lade_step_layout's
 * lm_rows; `argmax_slots`: lade_argmax_rows of the same slots (the window advances by argmax, :466,:478,:549).
 * Writes the decision record lade_commit_decision consumes.  `debug_uniforms` (nullable, device float[>= 2 + G*(N-1) + W]):
 * [count, u0, u1, ...] the uniforms consumed, for tests.  Top-k keeps every score >= the k-th largest (ties included,
 * TopKLogitsWarper); top-p drops scores in ascending order while their cumulative probability stays <= 1 - top_p
 * (TopPLogitsWarper, min_tokens_to_keep = 1) -- the logits are bf16, so both cut-offs are exact thresholds found with
 * two 256-bin histogram passes, and scores of equal value are kept or dropped together. */
int lade_sample_verify(LadeCtx* ctx, void* stream, const void* logits, int32_t ld, int32_t vocab,
                       const int32_t* argmax_slots, const int32_t* meta, float temperature, int32_t top_k, float top_p,
                       uint64_t* rng_state, int32_t* decision_out, float* debug_uniforms);

/* lade_sample_verify under the full warper record `warpers` (host memory, read at launch: a captured graph keeps the
 * values of its capture).  After top-p, every row the verification visits -- slot 0 and the row after each accepted
 * token -- is cut further, each warper acting on the softmax of what the previous ones kept (logits_process.py):
 *   MinPLogitsWarper     probs = softmax(scores); remove probs < min_p * probs.amax()
 *                        (with e_t = exp(score_t - max): e_t < min_p);
 *   EpsilonLogitsWarper  remove softmax(scores) < epsilon & scores < topk(scores, 1);
 *   EtaLogitsWarper      entropy = Categorical(logits=scores).entropy(); eta = min(epsilon, sqrt(epsilon) * exp(-entropy));
 *                        remove softmax(scores) < eta & scores < topk(scores, 1).
 * Each kept set is every score at or above a threshold, so each cut is one more threshold on the key (one pass over
 * the vocabulary; eta one more for the entropy), evaluated in fp32; the accept tests, the residual and the plain draw
 * use e_t / S' with S' summed over the final kept set.  The cuts consume no random numbers: the Philox stream and its
 * advance are those of lade_sample_verify, and with the three cuts off the decision is bit for bit the same.
 * `debug_cuts` (nullable, device float[>= 1 + 2 (N-1)]): [rows visited, then per row its final threshold key (the
 * 16-bit order key of the smallest kept logit) and S'], for tests.  LADE_EINVAL for min_p outside [0, 1], epsilon or
 * eta outside {0} or (0, 1), any NaN, or the temperature / top_k / top_p ranges of lade_sample_verify. */
int lade_sample_verify_warped(LadeCtx* ctx, void* stream, const void* logits, int32_t ld, int32_t vocab,
                              const int32_t* argmax_slots, const int32_t* meta, const LadeWarpers* warpers,
                              uint64_t* rng_state, int32_t* decision_out, float* debug_uniforms, float* debug_cuts);
int lade_sample_verify_warped_f16(LadeCtx* ctx, void* stream, const void* logits, int32_t ld, int32_t vocab,
                                  const int32_t* argmax_slots, const int32_t* meta, const LadeWarpers* warpers,
                                  uint64_t* rng_state, int32_t* decision_out, float* debug_uniforms, float* debug_cuts);

/* Apply an externally made decision (sampling path: the caller runs the reference's rejection-sampling
 * verification, lade/decoding.py:484-540, against the device logits with its own RNG streams).
 * `decision` (device) = lade_lp_record_ints() ints [first_token, max_hit, n_new, hits[N-1], new_window_tokens[W+N-3]]
 * followed by [max_hit_idx, flags, finished, 0] and, when flags bit1 is set, W ints: the newest window level
 * after filter_window (decoding.py:131-135,578-580; the pool still receives the unfiltered tokens).
 * flags bit0: sampling emission semantics (decoding.py:594-603). */
int lade_commit_decision(LadeCtx* ctx, void* stream, const int32_t* decision, const int32_t* meta,
                         int32_t* result);

/* Per-token logits capture (return_dict_in_generate with output_logits / output_scores, which the reference refuses,
 * lade/decoding.py:411, :967).  Launched after the step's commit (lade_accept_update or lade_commit_decision) on the
 * same stream, inside the same CUDA graph: for each token j the step emitted, the lm slot row it was decided from,
 * logits[slot][0:vocab] (bf16; _f16: fp16), is copied to out[r][0:vocab], r = n_out_before - n_prompt + j, where
 * n_out_before = result[LADE_R_N_OUT] - result[LADE_R_N_EMIT] and n_prompt is the prompt length of lade_ctx_reset: row r
 * of `out` is generated token r.  Slot of token j: 0 for j = 0; for j >= 1 the verification slot (e, j-1) of n-gram
 * e = result[LADE_R_MAX_HIT_IDX] when `sampling` is 0 (greedy: lade_accept_update emits the argmax of those slots), and
 * e = the lowest-index n-gram whose tokens 0..j-1 equal hits[0..j-1] when `sampling` is 1 (the row the sampling chain
 * drew token j from: the first candidate carrying each accepted token is the one that accepted it).  The n-grams'
 * tokens are read from the step's rows, ids[lm_rows[slot]] (lade_step_layout of the same step).  Writes nothing when
 * the step ran on a finished state (meta[LADE_M_DONE]) or emitted nothing, and never a row >= out_rows.  Rows are
 * `ld` / `ld_out` elements apart (>= vocab); 16-byte copies where both rows allow them.  LADE_EINVAL for a null
 * pointer, vocab < 1, ld or ld_out < vocab, out_rows < 1, `sampling` not 0 or 1, a pointer not aligned to its element
 * (nothing is launched); LADE_EUNSUPPORTED for a lookahead-parallel ctx. */
int lade_capture_rows(LadeCtx* ctx, void* stream, const void* logits, int32_t ld, int32_t vocab, const int32_t* ids,
                      const int32_t* lm_rows, const int32_t* meta, const int32_t* result, int32_t sampling, void* out,
                      int32_t ld_out, int32_t out_rows);
int lade_capture_rows_f16(LadeCtx* ctx, void* stream, const void* logits, int32_t ld, int32_t vocab, const int32_t* ids,
                          const int32_t* lm_rows, const int32_t* meta, const int32_t* result, int32_t sampling,
                          void* out, int32_t ld_out, int32_t out_rows);

/* Move the accepted n-gram's K/V rows to the cache tail for every layer (lade/decoding.py:1156-1163): rows
 * [R_KV_SRC, R_KV_SRC + h) of every head go to [R_KV_DST, R_KV_DST + h), h = min(R_MAX_HIT, max_rows); nothing moves when
 * R_MAX_HIT is 0 or R_KV_SRC < 0.  k_base/v_base point at layer 0; layers are `layer_stride_elems` apart (at least
 * n_kv_heads * kv_capacity * head_dim); 16-bit payloads of either model dtype.
 * Precondition: the two row ranges do not overlap, R_KV_SRC - R_KV_DST >= R_MAX_HIT (every row is copied by its own
 * CTA, in no order).  The results of lade_accept_update / lade_commit_decision satisfy it: the source rows are the
 * step's guess rows, which lie behind all of its window rows, the destination the first rows after the input token. */
int lade_kv_compact(void* stream, const int32_t* result, void* k_base, void* v_base,
                    int64_t layer_stride_elems, int32_t n_layers, int32_t n_kv_heads,
                    int32_t kv_capacity, int32_t head_dim, int32_t max_rows);

/* Copy the generated ids (device) out: out_ids_dev int32[max_total_len]; count via result.
 * The reference returns them as `input_ids` grown by torch.cat each step (decoding.py:1165-1177,1221-1225). */
int lade_ctx_output_ids(LadeCtx* ctx, void* stream, int32_t* out_host, int32_t n);
/* Debug/test access to the device state: the n-gram pool (`token_map`, decoding.py:911) as cnt[V], tup[V][G][N-1]
 * and the lookahead window (`past_tokens`, :902) as rows of W+N-3 ints with their live lengths. */
int lade_ctx_pool_snapshot(LadeCtx* ctx, void* stream, int32_t* cnt_host, int32_t* tup_host);
int lade_ctx_window_snapshot(LadeCtx* ctx, void* stream, int32_t* win_host, int32_t* len_host);

/* ---- lookahead parallelism (lade_distributed; lade/decoding.py:905-906,956-984,1023-1107,1148-1153) ---
 * Every rank holds a model replica and the same window + pool; rank r evaluates window columns
 * [ws, we) and its share of the candidate n-grams (lade_step_layout does the slicing from
 * LadeConfig.dist_workers / .rank).  Per step each rank writes ONE fixed-size int32 record
 *   [first_guess, max_hit, n_new, hits[N-1], new_tokens[W+N-3]]
 * with lade_lp_verify; the caller all-gathers the records (a single ncclAllGather over NVLink, rank order);
 * lade_lp_commit reduces them identically on every rank (max hit, lowest rank wins ties; window tokens
 * concatenated in rank order) and applies the state update -- this replaces the pickled object
 * collectives of decoding.py:1024,1045,1057,1090,1096,1106.  With a hit, no KV is copied: the accepted
 * tokens are re-fed next step (decoding.py:1148-1153). */
int lade_lp_record_ints(const LadeConfig* cfg);
int lade_lp_verify(LadeCtx* ctx, void* stream, const int32_t* argmax_slots, const int32_t* meta,
                   int32_t* record_out);
int lade_lp_commit(LadeCtx* ctx, void* stream, const int32_t* records_all /* [D][record_ints] */,
                   const int32_t* meta, int32_t* result);

/* Lookahead-parallel exchange INSIDE the library (SURVEY 8(b)): one ncclAllGather of the per-rank int32 record
 * (lade_lp_record_ints ints) on `stream` -- capturable, so verify -> exchange -> commit replay as part of the step's
 * CUDA graph.  Replaces dist.broadcast_object_list / dist.all_gather_object of python lists, lade/decoding.py:1023-1024,
 * :1043-1058, :1088-1107.  `nccl_comm` is an ncclComm_t: the caller's own, or one made by lade_nccl_comm_create (NCCL is
 * resolved at run time from the libnccl.so.2 already mapped into the process; LADE_EUNSUPPORTED when there is none).
 * lade_nccl_unique_id: rank 0 fills 128 bytes, the host broadcasts them (any transport), every rank then calls
 * lade_nccl_comm_create (collective) with its CUDA device current. */
int lade_nccl_available(void);
int lade_nccl_unique_id(void* id128);
int lade_nccl_comm_create(const void* id128, int32_t world, int32_t rank, void** comm_out);
int lade_nccl_comm_destroy(void* nccl_comm);
int lade_lp_exchange(LadeCtx* ctx, void* stream, void* nccl_comm, const int32_t* record_in, int32_t* records_all_out);

/* Error text for a LADE_E* code / the last CUDA runtime error string seen by this library (the reference raises
 * python exceptions or asserts, e.g. lade/utils.py:33, decoding.py:375-377,412); ABI version of this header. */
const char* lade_strerror(int code);
const char* lade_last_cuda_error(void);
int lade_version(void);

#ifdef __cplusplus
}
#endif
#endif /* LADE_SM100_H_ */
