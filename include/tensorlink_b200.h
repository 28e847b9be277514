/* tensorlink_b200 — C ABI of the H100-native shard executor.
 *
 * The reference (tensorlink-lab/tensorlink) has no FFI: its shard operator is Python
 * (`LayerGroupModule.forward(**kwargs)`, tensorlink/ml/injector.py:154-281) and the arithmetic is
 * whatever Hugging Face `transformers` does inside `decoder_layer(...)`.  This header is the plain-C
 * boundary that sits UNDER that operator: every entry point replaces one group of ATen library calls
 * the reference's worker makes per layer (`module(**kwargs)`, tensorlink/ml/worker.py:333) or its
 * autograd (`assoc_output.backward(loss)`, tensorlink/ml/worker.py:271).  INTEGRATION.md shows the
 * ctypes binding a maintainer would add on the reference side.
 *
 * Conventions
 *  - all pointers are DEVICE pointers on the current device unless the name ends in `_host`;
 *    bf16 tensors are `void*`; row-major, innermost dimension contiguous, 16-byte aligned.
 *  - `stream` is a `cudaStream_t` passed as `void*`; every call is asynchronous on that stream.
 *  - no entry point allocates or frees device memory; workspaces are passed in.  One exception:
 *    tl_gemv_bf16 / tl_gemv_bf16_pf allocate their pool of ticket counters (a few KB) once per device.
 *  - return value: 0 on success, a negative `tl_status` otherwise; `tl_last_error()` gives the
 *    (thread-local) message.  There is no CPU fallback: on a machine without an sm_90 device
 *    compute calls return TL_ERR_NO_DEVICE.
 *  - rounding points replicate the reference's bf16 pipeline (each HF op output is rounded to bf16
 *    before the next op consumes it); accumulation is fp32.
 */
#ifndef TENSORLINK_B200_H
#define TENSORLINK_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TL_ABI_VERSION 1

typedef enum {
    TL_OK = 0,
    TL_ERR_INVALID = -1,   /* bad shape / alignment / flag combination */
    TL_ERR_CUDA = -2,      /* a CUDA runtime / driver call failed       */
    TL_ERR_NO_DEVICE = -3, /* no sm_90 device visible                  */
    TL_ERR_WORKSPACE = -4  /* workspace too small                       */
} tl_status;

/* epilogue / operand flags for tl_gemm_bf16 and tl_gemv_bf16 */
#define TL_EPI_BIAS 1      /* + bias[N] (bf16), added in fp32 before the output rounding (oneDNN post-op)  */
#define TL_EPI_RESIDUAL 2  /* out = bf16(bf16(acc) + residual[M,N])  — HF `residual + hidden_states`        */
#define TL_EPI_SWIGLU 4    /* rows of B interleave gate/up (2j, 2j+1); out[M,N/2] = silu(gate)*up, HF rounding */
#define TL_EPI_OUT_F32 8   /* C is fp32 instead of bf16                                                     */
#define TL_EPI_ACCUM 16    /* C += result (bf16 read-modify-write; gradient accumulation)                   */
#define TL_A_MN_MAJOR 32   /* A is given as [K, M] row-major (contraction dim outermost)                     */
#define TL_B_MN_MAJOR 64   /* B is given as [K, N] row-major                                                 */

int tl_abi_version(void);
const char* tl_last_error(void);
/* sm_count / compute capability of the current device; TL_ERR_NO_DEVICE if none */
int tl_device_info(int* sm_count, int* cc_major, int* cc_minor);

/* ---- K1  Qwen2RMSNorm.forward (site-packages/transformers/models/qwen2/modeling_qwen2.py:258-263)
 * y[r,:] = w * bf16(x[r,:] * rsqrt(mean(x[r,:]^2) + eps)); rstd_out (fp32[rows]) optional, for backward */
int tl_rmsnorm_fwd(const void* x, const void* w, void* y, float* rstd_out, int rows, int H, float eps, void* stream);

/* ---- K7  embed_tokens gather (modeling_qwen2.py:367): out[n,:] = table[ids[n],:] */
int tl_embed_fwd(const int64_t* ids, const void* table, void* out, int n_tokens, int H, int vocab, void* stream);

/* ---- K2/K5/K6/K7  nn.Linear as one wgmma GEMM: C[M,N] = A[M,K] * B[N,K]^T (+ epilogue flags above).
 * lda/ldb/ldc in elements.  Replaces q/k/v_proj (modeling_qwen2.py:217-219, fused into one B), o_proj (:244),
 * gate/up/down_proj (:46-48), lm_head (:474-476) and, with the MN-major flags, their dgrad/wgrad. */
int tl_gemm_bf16(const void* A, const void* B, void* C, int M, int N, int K, int lda, int ldb, int ldc,
                 const void* bias, const void* residual, int flags, void* stream);

/* same contract with a caller-provided workspace (>= tl_gemm_splitk_ws(M, N) bytes): batched-decode shapes (M <= 128) whose
 * few output tiles cannot occupy every SM are split along K (fp32 partials + one reduce/epilogue pass) */
size_t tl_gemm_splitk_ws(int M, int N);
int tl_gemm_bf16_ws(const void* A, const void* B, void* C, int M, int N, int K, int lda, int ldb, int ldc,
                    const void* bias, const void* residual, int flags, void* workspace, size_t ws_bytes, void* stream);
/* ... and the RMSNorm that follows this Linear in the decoder layer (modeling_qwen2.py:296 / :280 of the next layer):
 * with norm_w != NULL also writes H_out[M,N] = norm_w * bf16(C * rstd(C)), C being the bf16 result above (ldc == N <= 8192,
 * bias / residual epilogue only).  Fused into the split-K reduce pass when that path runs, otherwise one extra
 * tl_rmsnorm_fwd launch (C identical either way; H may differ in a last bf16 bit: the row's sum of squares is reduced
 * in another order). */
int tl_gemm_bf16_ws_norm(const void* A, const void* B, void* C, int M, int N, int K, int lda, int ldb, int ldc,
                         const void* bias, const void* residual, int flags, void* workspace, size_t ws_bytes,
                         const void* norm_w, float eps, void* H_out, void* stream);

/* ---- decode-shaped Linear (M <= 8 tokens), HBM-bound weight streaming:
 * y[M,N] = f(norm(x)[M,K] * W[N,K]^T).  norm_w != NULL fuses the preceding RMSNorm (K1) as a prologue.
 * The kernel hands out its rows by ticket from a block of device counter words (see tl_gemv_bf16_ctr); these two
 * entry points take one from a per-device pool the library allocates at its first call on a device (which therefore
 * must not be inside a graph capture). */
int tl_gemv_bf16(const void* x, const void* W, void* y, int M, int N, int K, const void* bias,
                 const void* residual, const void* norm_w, float eps, int flags, void* stream);
/* same, plus a hint: once its own weight loads are issued the kernel queues L2 prefetches of the first next_bytes of
 * next_W (the weights the NEXT launch on this stream will read; 16-byte aligned, may be NULL), so HBM keeps streaming
 * across the launch boundary and the next kernel starts from L2.  Purely a performance hint: results are identical. */
int tl_gemv_bf16_pf(const void* x, const void* W, void* y, int M, int N, int K, const void* bias,
                    const void* residual, const void* norm_w, float eps, int flags, const void* next_W,
                    size_t next_bytes, void* stream);
/* same, with the caller's counter block: TL_GEMV_COUNTER_WORDS device words (4-byte aligned), zero before the first
 * call; every call leaves them zero.  A call site that owns a block (a launch inside a captured graph) never shares it
 * with a launch that can run at the same time: the next launch on the stream may start before this one has ended
 * (programmatic dependent launch).  NULL = a block from the pool. */
#define TL_GEMV_COUNTER_WORDS 4
int tl_gemv_bf16_ctr(const void* x, const void* W, void* y, int M, int N, int K, const void* bias,
                     const void* residual, const void* norm_w, float eps, int flags, unsigned* counter,
                     const void* next_W, size_t next_bytes, void* stream);

/* ---- FP8 weights (HF's fine-grained FP8 checkpoints, weight-only): W[N,K] float8_e4m3fn with fp32 scales[N][K/128],
 * one per row and 128-column group (HF's weight_scale_inv of the row's 128x128 block).  The weight used is
 * bf16(float(W[n,k]) * scales[n][k/128]), the bf16 weight of HF's dequantized checkpoint.
 * tl_gemv_fp8 / tl_gemv_fp8_ctr: tl_gemv_bf16 / tl_gemv_bf16_ctr over that weight (same flags, counter block and
 * prefetch hint; next_bytes counts bytes of whatever the next launch streams).  The result equals tl_gemv_bf16's over
 * the dequantized matrix bit for bit.  Needs K % 128 == 0 and a 16-byte aligned W.
 * tl_dequant_fp8: out[N,K] bf16 = that weight, for the GEMM paths (prefill, batched decode); HBM-bound. */
#define TL_FP8_BLOCK 128
int tl_gemv_fp8(const void* x, const void* W, const float* scales, void* y, int M, int N, int K, const void* bias,
                const void* residual, const void* norm_w, float eps, int flags, void* stream);
int tl_gemv_fp8_ctr(const void* x, const void* W, const float* scales, void* y, int M, int N, int K, const void* bias,
                    const void* residual, const void* norm_w, float eps, int flags, unsigned* counter,
                    const void* next_W, size_t next_bytes, void* stream);
int tl_dequant_fp8(const void* W, const float* scales, void* out, int N, int K, void* stream);

/* ---- K3  rotary tables (modeling_qwen2.py:102-113): cos/sin[pos, d/2] = bf16(cos/sin(pos * inv_freq)) */
int tl_rope_table(const float* inv_freq, void* cos_tab, void* sin_tab, int max_pos, int half_dim, void* stream);

/* ---- K3 + KV-cache append (+ Qwen3 q/k RMSNorm, modeling_qwen3.py:248-264):
 * qkv[n, (n_h+2n_kv)*d] (post-bias) -> q_out[n, n_h*d] rotated; K/V written to
 * cache[b, kv_head, pos, d] with b = n / S, pos = *pos0 + n % S (pos0 read from device memory so a
 * captured CUDA graph can be replayed while the position advances). q_norm_w/k_norm_w may be NULL. */
int tl_rope_kv_fwd(const void* qkv, void* q_out, void* k_cache, void* v_cache, const int32_t* pos0_dev,
                   const void* cos_tab, const void* sin_tab, const void* q_norm_w, const void* k_norm_w,
                   float eps, int n_tokens, int S, int n_h, int n_kv, int d, int T_max, void* stream);

/* ---- K4  causal GQA attention, prefill / training forward (modeling_qwen2.py:161-184 SDPA contract).
 * q[B,S,n_h,d]; caches [B,n_kv,T_max,d] hold keys 0..past_len+S-1; out[B,S,n_h*d];
 * lse (fp32 [B,n_h,S], natural log) optional, kept for backward. */
int tl_attn_prefill_fwd(const void* q, const void* k_cache, const void* v_cache, void* out, float* lse, int B,
                        int S, int past_len, int n_h, int n_kv, int d, int T_max, float scale, void* stream);

/* ---- K4  decode attention, one query token per batch row, split over the KV length.
 * kv_len_dev: device int32, number of valid keys (same for all rows).  workspace >= tl_attn_decode_ws(...) */
size_t tl_attn_decode_ws(int B, int n_h, int d, int T_max);
int tl_attn_decode_fwd(const void* q, const void* k_cache, const void* v_cache, void* out,
                       const int32_t* kv_len_dev, void* workspace, size_t ws_bytes, int B, int n_h, int n_kv,
                       int d, int T_max, float scale, void* stream);

/* ---- K4  verify attention (prompt-lookup decoding): q[q_len, n_h, d] are q_len <= 16 consecutive query tokens of cache
 * row 0 whose keys and values tl_rope_kv_fwd (S = q_len) already appended at slots *pos_dev .. *pos_dev + q_len - 1.
 * Query i attends to keys 0..*pos_dev + i; slots above that are never read into an output (they may hold anything,
 * NaN included).  out[q_len, n_h*d].  Split over the KV length; workspace >= tl_attn_verify_ws(...) bytes. */
size_t tl_attn_verify_ws(int q_len, int n_h, int d, int T_max);
int tl_attn_verify_fwd(const void* q, const void* k_cache, const void* v_cache, void* out, const int32_t* pos_dev,
                       void* workspace, size_t ws_bytes, int q_len, int n_h, int n_kv, int d, int T_max, float scale,
                       void* stream);

/* ---- K3 + K4 fused for decode, T_max <= 2048: RoPE (+q/k-norm) of the new token, KV-cache append at *pos_dev and
 * single-pass attention over keys 0..*pos_dev, one launch per layer.  qkv[B, (n_h+2n_kv)*d] post-bias; out[B, n_h*d] */
int tl_attn_decode_fused(const void* qkv, void* k_cache, void* v_cache, void* out, const int32_t* pos_dev,
                         const void* cos_tab, const void* sin_tab, const void* q_norm_w, const void* k_norm_w,
                         float eps, int B, int n_h, int n_kv, int d, int T_max, float scale, void* stream);

/* ---- left-padded batches (HF's layout for batched generation): the four entry points above, each with one more
 * argument, kv_start_dev (device int32[B]).  kv_start[b] is the number of leading pad slots of row b (at most its
 * cache length - 1, so every row keeps at least one real key):
 *   - cache slot t of row b holds the token at rotary position t - kv_start[b]; pad slots (t < kv_start[b]) are
 *     still written, rotated at position 0, and are never attended;
 *   - attention reads keys kv_start[b]..(last valid key) of row b only: the cache below kv_start may hold anything
 *     (NaN included) and is not read by the tensor-core kernels, and split-KV partials lying wholly below it are skipped;
 *   - a query row below kv_start[b] (a pad token of the prompt) gets out = 0 and lse = -inf.
 * The write position and the KV length stay scalar and shared by all rows, as in the entry points above.  With every
 * kv_start[b] = 0 each result equals the plain entry point's bit for bit. */
int tl_rope_kv_fwd_rows(const void* qkv, void* q_out, void* k_cache, void* v_cache, const int32_t* pos0_dev,
                        const void* cos_tab, const void* sin_tab, const void* q_norm_w, const void* k_norm_w,
                        float eps, int n_tokens, int S, int n_h, int n_kv, int d, int T_max,
                        const int32_t* kv_start_dev, void* stream);
int tl_attn_prefill_fwd_rows(const void* q, const void* k_cache, const void* v_cache, void* out, float* lse, int B,
                             int S, int past_len, int n_h, int n_kv, int d, int T_max, float scale,
                             const int32_t* kv_start_dev, void* stream);
int tl_attn_decode_fwd_rows(const void* q, const void* k_cache, const void* v_cache, void* out,
                            const int32_t* kv_len_dev, void* workspace, size_t ws_bytes, int B, int n_h, int n_kv,
                            int d, int T_max, float scale, const int32_t* kv_start_dev, void* stream);
int tl_attn_decode_fused_rows(const void* qkv, void* k_cache, void* v_cache, void* out, const int32_t* pos_dev,
                              const void* cos_tab, const void* sin_tab, const void* q_norm_w, const void* k_norm_w,
                              float eps, int B, int n_h, int n_kv, int d, int T_max, float scale,
                              const int32_t* kv_start_dev, void* stream);
/* The attention backward of a left-padded training batch: tl_attn_bwd (below) with kv_start_dev as above, for the
 * output of tl_attn_prefill_fwd_rows at past_len = 0 (k/v caches hold keys 0..S-1):
 *   - the q, dout, out and lse rows of pad queries (s < kv_start[b]) and the K/V slots below kv_start[b] may hold
 *     anything, NaN included; they are never read, or meet the backward through a select only;
 *   - on exit dq is 0 on pad query rows and dk/dv are 0 on slots below kv_start[b]; every output is finite;
 *   - with every kv_start[b] = 0 each result equals tl_attn_bwd's bit for bit.
 * Dispatch is tl_attn_bwd's (wgmma kernels from S >= 64, mma.sync below; TL_ATTN_BWD=mma|wgmma forces a path). */
int tl_attn_bwd_rows(const void* q, const void* k_cache, const void* v_cache, const void* out, const void* dout,
                     const float* lse, void* dq, void* dk, void* dv, void* workspace, size_t ws_bytes, int B, int S,
                     int n_h, int n_kv, int d, int T_max, float scale, const int32_t* kv_start_dev, void* stream);

/* ---- K7  final norm + lm_head + greedy argmax for M <= 8 rows: ids[m] = argmax_v bf16(norm(x)[m,:]·W[v,:])
 * (lowest index wins ties, as torch.argmax).  logits_out (bf16 [M,V]) optional.
 * workspace >= tl_lmhead_ws(M, V) bytes; gemv_counter: the lm_head GEMV's counter block (tl_gemv_bf16_ctr), may be NULL. */
size_t tl_lmhead_ws(int M, int V);
int tl_lmhead_argmax(const void* x, const void* W, const void* norm_w, float eps, int64_t* ids_out,
                     void* logits_out, void* workspace, size_t ws_bytes, int M, int V, int H, unsigned* gemv_counter,
                     void* stream);

/* argmax over bf16 logits[M,V] (any M); workspace >= M*64*8 bytes */
int tl_argmax_bf16(const void* logits, int64_t* ids_out, void* workspace, size_t ws_bytes, int M, int V, void* stream);

/* ---- the score log of generate(output_scores / output_logits): the _log twins of tl_argmax_bf16, tl_argmax_proc,
 * tl_sample and tl_sample_proc pick the same ids (same draws, counters and histories) and also store each row into column
 * c = log_col[0] of fp32 logs [n_cols, B_total, V] (column stride B_total*V, 64-bit offsets), launch row m at log row
 * row0 + m: raw_log = float(bf16 logit); score_log = HF's score: the processed value (the logit itself without logits
 * processors) for the argmax, and x / temperature (IEEE division) on the sampler's kept set, -inf elsewhere, for the
 * samplers (x: the processed value for tl_sample_proc_log).  Either log may be NULL, not both.  log_col: int32[2] in
 * device memory, {column, exit word}; the exit word must be 0 and is left 0.  The call advances the column by one, so a
 * captured graph logs each replay into the next column; a column >= n_cols is not written.  A NULL log_col, row0 + M >
 * B_total, or n_cols*B_total*V beyond int64 is rejected (TL_ERR_INVALID).  No launch is added. */
int tl_argmax_bf16_log(const void* logits, int64_t* ids_out, void* workspace, size_t ws_bytes, int M, int V, float* raw_log,
                       float* score_log, int32_t* log_col, int n_cols, int B_total, int row0, void* stream);

/* ---- token sampling on the device (csrc/sample.cu): what HF `generate(do_sample=True)` does on the host's copy of the
 * logits (the reference delegates to it, tensorlink/ml/module.py:763-769, ml/worker.py:403-404): temperature -> top-k
 * (every logit >= the k-th largest is kept; 0 = off) -> top-p (a token is kept while the probability mass above it is
 * < top_p; ties at the threshold are kept) -> min_p -> typical_p -> epsilon -> eta -> one multinomial draw per row from
 * Philox4x32-10(seed; row, counter).  The last four arguments are HF's MinP / Typical / Epsilon / Eta warpers
 * (min_tokens_to_keep 1), each over the set the stages before it kept, p = softmax(x / T) over that set, H its entropy:
 * min_p keeps p >= min_p * p_max; typical_p = m keeps a group of equal distance |E[x/T] - x/T| while the mass of the
 * strictly closer tokens is < m (it may drop the top tokens); epsilon keeps p >= epsilon; eta keeps p >=
 * min(eta, sqrt(eta) * exp(-H)); the last two always keep the set's top value.  Off at min_p 0, typical_p 1, epsilon 0,
 * eta 0, which run the sampler as without them; 0 <= min_p <= 1, 0 < typical_p <= 1, 0 <= epsilon < 1 and
 * 0 <= eta < 1, else TL_ERR_INVALID.  The kept set is always one interval of values.  The same four arguments act alike
 * in tl_sample_proc and tl_spec_accept.  They need no more workspace, except tl_spec_accept's 8 bytes per row for the
 * interval's top.
 * counters_dev: int32[M] in device memory, advanced by the kernel (a captured graph draws a fresh number per replay).
 * workspace >= tl_sample_ws(M) bytes.  logits bf16 [M,V] row-major; ids_out int64[M]. */
size_t tl_sample_ws(int M);
int tl_sample(const void* logits, int64_t* ids_out, int M, int V, float temperature, int top_k, float top_p,
              unsigned long long seed, int32_t* counters_dev, void* workspace, size_t ws_bytes, void* stream, float min_p,
              float typical_p, float epsilon, float eta);
int tl_sample_log(const void* logits, int64_t* ids_out, int M, int V, float temperature, int top_k, float top_p,
                  unsigned long long seed, int32_t* counters_dev, void* workspace, size_t ws_bytes, float* raw_log,
                  float* score_log, int32_t* log_col, int n_cols, int B_total, int row0, void* stream, float min_p,
                  float typical_p, float epsilon, float eta);
/* speculative sampling after a verify pass (Leviathan et al. Algorithm 1, HF _speculative_sampling), one row: the
 * target's rows p_logits bf16 [K+1, V_p] and the assistant's q_logits bf16 [K, V_q], each warped by tl_sample's rules
 * with the same temperature / top_k / top_p; the drafts d_i = in_ids[i+1] for i < n = min(*n_cand, K).  Draft i is kept
 * while u_i * q_i(d_i) < p_i(d_i) (u_i: Philox row i); at the first rejection n the next token is drawn from
 * norm((p_n - q_n)+) with d_n excluded (from p_n without d_n when that mass rounds to 0), else from p_n (Philox row 16).
 * An id >= V_q has q = 0, a draft >= V_p has p = 0 (always rejected): exact over the union of the vocabularies.
 * Output in tl_prompt_lookup_accept's form: ids_out[i] = in_ids[i+1] for i < n, ids_out[n] = the drawn token (never
 * in_ids[n+1]); ids_out[n+1..K] are not written.  counter_dev: one int32 in device memory, advanced by one per call.
 * workspace >= tl_spec_accept_ws(K) bytes.  Two launches: 2K+1 CTAs (one per row), then one CTA. */
size_t tl_spec_accept_ws(int K);
int tl_spec_accept(const void* p_logits, int V_p, const void* q_logits, int V_q, int K, const int64_t* in_ids,
                   const int32_t* n_cand, float temperature, int top_k, float top_p, unsigned long long seed,
                   int32_t* counter_dev, int64_t* ids_out, void* workspace, size_t ws_bytes, void* stream, float min_p,
                   float typical_p, float epsilon, float eta);

/* ---- logits processors (csrc/logits_process.cu): HF's RepetitionPenaltyLogitsProcessor -> NoRepeatNGramLogitsProcessor
 * -> MinNewTokensLengthLogitsProcessor on the fp32 copy of the bf16 logits, before the argmax or the warpers above.
 * Each row keeps its token history in device memory: log int32[M, L] (row pitch L), len int32[M] and a presence
 * bitmap bits uint32[M, ceil(V/32)].  params_dev int32[TL_LP_PARAMS]: the penalty (float bits), n, min_new_tokens,
 * the prompt length (history entries that are not generated), the number of EOS ids and the ids.  The picking kernel
 * appends its id to the row's history, so a captured graph stays right on every replay.
 * flags & TL_LP_BAN: compute the ban set (n-gram completions, EOS ids below min_new_tokens); otherwise only the
 * penalty applies.  workspace >= tl_logits_proc_ws(M, V) bytes. */
#define TL_LP_PENALTY 0
#define TL_LP_NGRAM 1
#define TL_LP_MIN_NEW 2
#define TL_LP_PROMPT 3
#define TL_LP_N_EOS 4
#define TL_LP_EOS 5
#define TL_LP_MAX_EOS 8
#define TL_LP_PARAMS (TL_LP_EOS + TL_LP_MAX_EOS)
#define TL_LP_BAN 1
size_t tl_logits_proc_ws(int M, int V);
/* history of row m = prompt[m, 0:S] (int64 [M,S]); len = S; the bitmap holds exactly those ids */
int tl_history_fill(const int64_t* prompt, int32_t* log, int32_t* len, uint32_t* bits, int M, int S, int L, int V,
                    void* stream);
/* ids[m] = the lowest index of the largest processed value (torch.argmax); 0 when every value is -inf */
int tl_argmax_proc(const void* logits, int64_t* ids_out, int32_t* log, int32_t* len, uint32_t* bits,
                   const int32_t* params_dev, int flags, void* workspace, size_t ws_bytes, int M, int V, int L, void* stream);
/* tl_sample's rules over the processed values (32-bit keys: the top-k and top-p boundaries are resolved exactly, and the
 * probability mass is summed as 64-bit fixed-point integers, so a seed reproduces its tokens) */
int tl_sample_proc(const void* logits, int64_t* ids_out, int32_t* log, int32_t* len, uint32_t* bits,
                   const int32_t* params_dev, int flags, int M, int V, int L, float temperature, int top_k, float top_p,
                   unsigned long long seed, int32_t* counters_dev, void* workspace, size_t ws_bytes, void* stream, float min_p,
                   float typical_p, float epsilon, float eta);
/* the score-log twins (see tl_argmax_bf16_log) */
int tl_argmax_proc_log(const void* logits, int64_t* ids_out, int32_t* log, int32_t* len, uint32_t* bits,
                       const int32_t* params_dev, int flags, void* workspace, size_t ws_bytes, int M, int V, int L,
                       float* raw_log, float* score_log, int32_t* log_col, int n_cols, int B_total, int row0, void* stream);
int tl_sample_proc_log(const void* logits, int64_t* ids_out, int32_t* log, int32_t* len, uint32_t* bits,
                       const int32_t* params_dev, int flags, int M, int V, int L, float temperature, int top_k, float top_p,
                       unsigned long long seed, int32_t* counters_dev, void* workspace, size_t ws_bytes, float* raw_log,
                       float* score_log, int32_t* log_col, int n_cols, int B_total, int row0, void* stream, float min_p,
                       float typical_p, float epsilon, float eta);

/* ---- prompt-lookup decoding (csrc/prompt_lookup.cu), one row: a verify step runs in_ids[0..K] (the last history token
 * and K drafts) as K+1 rows and keeps the drafts the model agrees with.  The history is the logits processors' (log, len,
 * bits above, row 0).  params_dev int32[TL_PL_PARAMS]: the largest n-gram size, max_length (prompt + max_new_tokens:
 * the history never grows past it), the number of EOS ids and the ids. */
#define TL_PL_NGRAM 0
#define TL_PL_MAX_LEN 1
#define TL_PL_N_EOS 2
#define TL_PL_EOS 3
#define TL_PL_MAX_EOS 8
#define TL_PL_PARAMS (TL_PL_EOS + TL_PL_MAX_EOS)
#define TL_PL_MAX_DRAFT 15
/* HF PromptLookupCandidateGenerator.get_candidates on the history: in_ids[0] = its last token, in_ids[1..n] = the
 * candidates, in_ids[n+1..K] = filler (the last token), *n_cand = n (0..K) */
int tl_prompt_lookup_draft(const int32_t* log, const int32_t* len, int L, const int32_t* params_dev, int K, int64_t* in_ids,
                           int32_t* n_cand, void* stream);
/* ids[0..K]: the model's next token after each of in_ids[0..K].  a = the largest value <= *n_cand with ids[i] ==
 * in_ids[i+1] for every i < a; e = min(a+1, max_length - len) tokens ids[0..e) join the history and out_log[*count..],
 * and *count, *pos_dev and *kv_len_dev (= the new *pos_dev) advance by e.  bits may be NULL. */
int tl_prompt_lookup_accept(const int64_t* ids, const int64_t* in_ids, const int32_t* n_cand, int32_t* log, int32_t* len,
                            uint32_t* bits, int L, int V, const int32_t* params_dev, int64_t* out_log, int32_t* count,
                            int out_cap, int32_t* pos_dev, int32_t* kv_len_dev, int K, void* stream);
/* assisted decoding (an assistant model drafts in_ids[1..K]), one row: with P = *len - 1, the history's log[P-1], log[P]
 * -> asst_in[0..1] (the assistant's 2-row catch-up at cache slots P-1, P), log[P] -> in_ids[0], and the assistant's
 * *asst_pos = *asst_kv_len = P - 1.  Nothing else is written. */
int tl_assist_prep(const int32_t* log, const int32_t* len, int L, int64_t* asst_in, int64_t* in_ids, int32_t* asst_pos,
                   int32_t* asst_kv_len, void* stream);

/* ---- small device-side helpers used by the captured decode graph */
int tl_advance_pos(int32_t* pos_dev, int32_t* kv_len_dev, int delta, void* stream); /* pos += delta; kv_len = pos */
/* out_tokens[b, *step_dev] = ids[b] for b < B (row pitch ld), then ++*step_dev: the generated-token log
 * (replaces the per-token TOKEN packet, tensorlink/p2p/torch_node.py:543-551) */
int tl_append_token(const int64_t* ids, int64_t* out_tokens, int32_t* step_dev, int B, int ld, void* stream);

/* ---- a chain of dependent decode-step jobs as ONE persistent kernel (csrc/decode_chain.cu) ----------------
 * The job list replaces the per-layer launch sequence of `DistributedWorker._handle_forward` ->
 * `module(**kwargs)` (tensorlink/ml/worker.py:297-357) for single-token rows (M <= 4): one CTA per SM walks the
 * list; the producer warp streams the weights of EVERY GEMV job through one shared-memory ring without ever waiting
 * for a dependency, a dependency between jobs is one release/acquire counter, the attention job is split-KV over
 * all CTAs (one group per row and kv head).  Typical chain = one decoder layer:
 *   ATTN(j) -> GEMV o(j) -> GEMV gate/up(j) -> GEMV down(j) -> GEMV qkv(j+1). */
#define TL_JOB_GEMV 0     /* y[M,N or N/2] = f(norm(x)[M,K] W[N,K]^T): same semantics and flags as tl_gemv_bf16 */
#define TL_JOB_ATTN 1     /* RoPE (+ q/k norm) + KV append + attention for one new token per row: x = qkv[M,(n_h+2n_kv)d]
                           * (post-bias), y = out[M,n_h*d]; reads the position from *pos_dev (cached keys 0..pos-1) */
#define TL_ATTN_POS_PER_ROW 1   /* flags of an ATTN job: pos_dev is int32[M], one position per row (ragged batches) */
#define TL_DECODE_CHAIN_MAX_JOBS 16
#define TL_DECODE_CHAIN_SYNC_BYTES 1024   /* per launch site, zero-initialised once; the kernel leaves it zeroed */
typedef struct tl_decode_job {
    int32_t type, N, K, flags;
    int32_t n_h, n_kv, d, T_max;
    float eps, scale;
    const void* W;
    const void* x;
    void* y;
    const void* bias;
    const void* residual;
    const void* norm_w;
    const void* pos_dev;
    const void* cos_tab;
    const void* sin_tab;
    const void* q_norm_w;
    const void* k_norm_w;
    void* k_cache;
    void* v_cache;
} tl_decode_job;
/* bytes of the attention-partials workspace shared by every chain launch of a stage */
size_t tl_decode_chain_ws(int M, int n_h, int n_kv, int d);
/* host only: the shared-memory ring tl_decode_chain builds for M rows whose widest GEMV job has K = k_max.  stage_kb < 0
 * takes the process's TL_CHAIN_STAGE_KB (what tl_decode_chain uses), 0 the default geometry, > 0 forces a slot size.
 * out[4] = {slot bytes, slots, consumer warps NW, K chunk}; TL_ERR_INVALID when the launcher cannot place the shape. */
int tl_decode_chain_geometry(int M, int k_max, int stage_kb, int* out);
/* jobs: HOST array (copied into kernel parameter space).  sync_slot: TL_DECODE_CHAIN_SYNC_BYTES of device memory
 * private to this launch site (consecutive launches under programmatic dependent launch must not share one); word 2
 * is an error flag the kernel raises instead of hanging when a dependency wait exceeds 2 s.  pf_ptr/pf_bytes:
 * optional L2 prefetch hint = the weights the NEXT launch streams first. */
int tl_decode_chain(const tl_decode_job* jobs, int n_jobs, int M, void* sync_slot, void* attn_ws, size_t attn_ws_bytes,
                    const void* pf_ptr, size_t pf_bytes, void* stream);
/* debugging aid: device buffer of n_slots * 2*(TL_DECODE_CHAIN_MAX_JOBS+1)*4 uint64; every later chain launch takes the
 * next slot and stamps it with globaltimer values (CTA 0 and the last CTA; per job: start / input staged / work done /
 * dependency passed; last row: kernel entry / previous grid done / exit); NULL = off */
int tl_decode_chain_trace(void* buf, int n_slots);

/* ---- peer-memory mailboxes: the inter-shard hop of a decode step (csrc/peer.cu) ---------------------------
 * Replace the per-hop send of `DistributedModel.forward` (tensorlink/ml/module.py:438-462: tensor -> bytes ->
 * shared memory -> node process -> socket) and the worker's pickup (tensorlink/ml/worker.py:297-305) on one
 * NVSwitch node: the receiver's input buffer is mapped into the sender (CUDA IPC), the sender's last kernel stores
 * its rows there over NVLink, and a sequence number published with release/acquire at system scope hands it over.
 * All counters are device-resident and advance inside the kernels, so a captured CUDA graph replays unchanged. */
/* cudaMalloc + zero `bytes` and export the allocation: handle64 = the 64-byte cudaIpcMemHandle_t */
int tl_peer_alloc(size_t bytes, void** ptr, unsigned char* handle64);
/* map another process's allocation (peer access enabled lazily); *ptr is valid on this process's device */
int tl_peer_open(const unsigned char* handle64, void** ptr);
int tl_peer_close(void* ptr);   /* unmap a tl_peer_open mapping */
int tl_peer_free(void* ptr);    /* free a tl_peer_alloc allocation */
/* ++*want_dev, then wait until *flag_local >= *want_dev (mod 2^32).  After timeout_ns (0 = 10 s) sets *err_dev = 1
 * and returns instead of hanging; once *err_dev is set every later wait returns at once.  wait_ns_dev (optional) accumulates the nanoseconds spent waiting. */
int tl_peer_wait(const uint32_t* flag_local, uint32_t* want_dev, uint32_t* err_dev, uint64_t* wait_ns_dev,
                 uint64_t timeout_ns, int32_t* bump_dev, void* stream);   /* bump_dev (optional): ++*bump_dev as well */
/* ++*sent_dev, then publish it in the peer's flag after every earlier write of this stream (release, system scope) */
int tl_peer_signal(uint32_t* flag_peer, uint32_t* sent_dev, int32_t* bump_dev, void* stream);   /* bump_dev as above */
/* copy `bytes` (multiple of 16, both 16-byte aligned) into the peer buffer, then signal as above */
int tl_peer_put(void* dst_peer, const void* src, size_t bytes, uint32_t* flag_peer, uint32_t* sent_dev, void* stream);

/* ---- training-only pieces (K8/K9/K10): replace the autograd graph of `assoc_output.backward(loss)`
 * (tensorlink/ml/worker.py:271) and `optimizer.step()` (tensorlink/ml/worker.py:1317) ------------------------- */
/* SwiGLU on interleaved gate/up pre-activations gu[M,2I] (col 2j = gate_j, 2j+1 = up_j): h[M,I], HF rounding */
int tl_swiglu_fwd(const void* gu, void* h, int M, int I, void* stream);
/* dgu[M,2I] from dh[M,I] */
int tl_swiglu_bwd(const void* gu, const void* dh, void* dgu, int M, int I, void* stream);
/* RMSNorm backward: dx = rstd*(dy*w - n*mean(dy*w*n)) (+ dx_add if non-NULL); dw_accum (fp32 [H]) += sum dy*n */
int tl_rmsnorm_bwd(const void* x, const void* w, const void* dy, const float* rstd, const void* dx_add, void* dx,
                   float* dw_accum, int rows, int H, void* stream);
/* RoPE backward + KV gather: dqkv[n, (n_h+2n_kv)*d] from dq[n, n_h*d] and dk/dv[B, n_h, T_max, d] (one partial per
 * query head as written by tl_attn_bwd; the n_h/n_kv partials of a kv head are summed in fp32) */
int tl_rope_kv_bwd(const void* dq, const void* dk, const void* dv, void* dqkv, const void* cos_tab,
                   const void* sin_tab, int n_tokens, int S, int n_h, int n_kv, int d, int T_max, void* stream);
/* Qwen3 q/k-norm backward, in place on the q and k slices of dqkv[n, (n_h+2n_kv)*d] (gradient w.r.t. the
 * normalised vectors on entry, w.r.t. the pre-norm vectors on exit); gain gradients accumulate in fp32 [d] */
int tl_qk_norm_bwd(const void* qkv_pre, void* dqkv, const void* q_norm_w, const void* k_norm_w, float* dqn_accum,
                   float* dkn_accum, float eps, int n_tokens, int n_h, int n_kv, int d, void* stream);
/* attention backward (recompute P from lse): dq[B,S,n_h,d]; dk/dv[B,n_h,T_max,d] rows < S, one partial per query head */
size_t tl_attn_bwd_ws(int B, int S, int n_h);
int tl_attn_bwd(const void* q, const void* k_cache, const void* v_cache, const void* out, const void* dout,
                const float* lse, void* dq, void* dk, void* dv, void* workspace, size_t ws_bytes, int B, int S,
                int n_h, int n_kv, int d, int T_max, float scale, void* stream);
/* cross-entropy on bf16 logits[M,V] (fp32 math): *loss_sum += sum_rows (lse - logit[label]); *n_valid += rows
 * with a valid label; dlogits = (softmax - onehot) * grad_scale (may alias logits); label outside [0,V) ignored */
int tl_ce_fwd_bwd(const void* logits, const int64_t* labels, float* loss_sum, int32_t* n_valid, void* dlogits,
                  float grad_scale, int M, int V, void* stream);
/* embedding backward: dtable[ids[n],:] += dout[n,:]  (bf16x2 atomics into the bf16 gradient) */
int tl_embed_bwd(const int64_t* ids, const void* dout, void* dtable, int n_tokens, int H, int vocab, void* stream);
/* bias gradient: db_accum[N] (fp32) += sum_m dy[m,:N] (row pitch ld) */
int tl_colsum(const void* dy, float* db_accum, int M, int N, int ld, void* stream);
/* dst[n] (+)= src[n]: fp32 accumulator into a bf16 gradient */
int tl_f32_to_bf16_accum(const float* src, void* dst, size_t n, int accumulate, void* stream);
/* a[n] += b[n] over bf16 (n %% 8 == 0) */
int tl_add_inplace(void* a, const void* b, size_t n, void* stream);
/* a[n] = (accumulate ? a[n] : 0) + scale * b[n]: commits a pending gradient with the upstream gradient's scale
 * (the reference gets this from autograd: ml/worker.py:271 `assoc_output.backward(loss)`); bf16 (n %% 8 == 0) / fp32 */
int tl_scale_add_bf16(void* a, const void* b, float scale, int accumulate, size_t n, void* stream);
int tl_scale_add_f32(float* a, const float* b, float scale, int accumulate, size_t n, void* stream);
/* fused Adam / AdamW (torch.optim update rule, fp32 math and moments) over a flat bf16 parameter arena
 * (all four arrays 16-byte aligned; n arbitrary) */
int tl_adamw_step(void* param, const void* grad, float* exp_avg, float* exp_avg_sq, size_t n, float lr,
                  float beta1, float beta2, float eps, float weight_decay, int step, int decoupled,
                  void* stream);


/* ---- Qwen3-MoE sparse MLP (HF Qwen3MoeSparseMoeBlock with eager experts; tensorlink_b200/csrc/moe.cu)
 * tl_moe_route: per token (N rows of bf16 logits [N,E], E <= 256, 1 <= k <= min(16,E)): the top-k of the fp32 softmax,
 *   ties toward the lower expert, ids[N,k] sorted ascending and wts[N,k] fp32 (renormalised over the picks if
 *   norm_topk).  counts/offsets/row_of/tiles (all or none): the grouped-GEMM plan — counts[E], offsets[E+1] (segments
 *   padded to 128 rows), row_of[N*k] (token, slot) -> segment row in ascending token order, tiles[max_tiles][2] =
 *   (expert or -1, valid rows) per 128-row M-tile; max_tiles >= tl_moe_max_tiles(N, E, k).
 * tl_moe_gather: hg[row_of[t*k+s], :] = h[t, :].
 * tl_moe_gemm: C[r, :] = A[r, :] · W[e]^T (W [E*N, K], expert e = rows e*N..) for the valid rows of every tile; flags
 *   0 (bf16 out) or TL_EPI_SWIGLU (interleaved gate/up rows, C [rows, N/2]); N % 128 == 0.
 * tl_moe_combine: out[t] = bf16(x[t] + acc), acc = +0 then acc = bf16(acc + bf16(y[row_of[t*k+s]] * wts[t,s])) for
 *   s = 0..k-1 (ascending expert).  out may alias x.
 * tl_moe_gemv: M <= 16 decode rows, weights of the picked experts only.  TL_EPI_SWIGLU: y[M*k, N/2] per (row, pick)
 *   from x[M,K] and W [E, N, K] with interleaved gate/up rows.  TL_EPI_RESIDUAL: x = act [M*k, K], W [E, N, K];
 *   y[M, N] = the combine above with residual [M, N] (y may alias residual). */
int tl_moe_max_tiles(int N, int E, int k);
int tl_moe_route(const void* logits, int N, int E, int k, int norm_topk, int32_t* ids, float* wts, int32_t* counts,
                 int32_t* offsets, int32_t* row_of, int32_t* tiles, int max_tiles, void* stream);
int tl_moe_gather(const void* h, const int32_t* row_of, void* hg, int N, int k, int H, void* stream);
int tl_moe_gemm(const void* A, const void* W, void* C, const int32_t* tiles, int max_tiles, int E, int N, int K, int ldc,
                int flags, void* stream);
int tl_moe_combine(const void* y, const int32_t* row_of, const float* wts, const void* x, void* out, int N, int k, int H,
                   void* stream);
int tl_moe_gemv(const void* x, const void* W, void* y, const int32_t* ids, const float* wts, const void* residual, int M,
                int k, int N, int K, int flags, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TENSORLINK_B200_H */
