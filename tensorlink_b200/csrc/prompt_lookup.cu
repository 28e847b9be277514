// Prompt-lookup decoding on the device: the draft of a verify step and the accept step after it, for one row.
//
// HF ``generate(prompt_lookup_num_tokens=K)`` (PromptLookupCandidateGenerator.get_candidates) proposes the up to K tokens
// that followed the first occurrence, from the left, of the sequence's last n-gram, runs them with the current token as
// K+1 rows in one pass over the weights and keeps the longest prefix the model agrees with plus the model's own next
// token.  Both halves run inside the captured verify graph, so the host only replays it and reads the token count
// now and then.  The row's token history is the logits processors' (csrc/logits_process.cu, tl_history_fill): an int32
// log of row pitch L, a length and a presence bitmap.
//   * draft kernel    one CTA: for n = min(ngram, len-1) .. 1, the lowest start whose n tokens equal the last n and
//                     whose continuation is not empty; in_ids = [last token, up to K candidates cut at the first EOS,
//                     filler], n_cand = the number of candidates
//   * accept kernel   one warp: a = the agreeing prefix of the candidates; ids[0..a] join the history and the output
//                     log, the count, the cache position and the KV length advance by a+1.
//   * assist prep     one thread: with an assistant model as the draft source (assisted decoding), its catch-up input
//                     and cache position for the round, and the target's current token.
#include <limits.h>

#include "common.cuh"

namespace tl {

constexpr int PL_THREADS = 256;

__global__ void __launch_bounds__(PL_THREADS) pl_draft_kernel(const int32_t* __restrict__ log, const int32_t* __restrict__ len_dev,
                                                              int L_cap, const int32_t* __restrict__ params, int K,
                                                              int64_t* __restrict__ in_ids, int32_t* __restrict__ n_cand_out) {
    __shared__ int s_best;
    const int tid = threadIdx.x;
    const int L = min(*len_dev, L_cap);
    const int max_len = params[TL_PL_MAX_LEN];
    const int last = L > 0 ? log[L - 1] : 0;
    int start = 0, n = 0;                                  // the continuation: log[start .. start + n)
    if (max_len != L + 1) {                                // (HF: the model's own token would already reach max_length)
        const int end = min(L, max_len);                   // a continuation ends before min(L, max_length)
        for (int ng = min(params[TL_PL_NGRAM], L - 1); ng >= 1; --ng) {
            if (tid == 0) s_best = INT_MAX;
            __syncthreads();
            const int tail = L - ng;
            for (int idx = tid; idx + ng < end; idx += PL_THREADS) {
                bool same = true;
                for (int j = 0; j < ng && same; ++j) same = log[idx + j] == log[tail + j];
                if (same) {
                    atomicMin(&s_best, idx);
                    break;                                 // this thread's later starts are larger
                }
            }
            __syncthreads();
            const int best = s_best;
            __syncthreads();                               // every thread has read s_best before it is reset
            if (best != INT_MAX) {
                start = best + ng;
                n = min(K, end - start);
                break;
            }
        }
    }
    // the candidates stop before the first EOS id
    const int n_eos = min(params[TL_PL_N_EOS], TL_PL_MAX_EOS);
    for (int j = 0; j < n && n_eos > 0; ++j) {
        const int id = log[start + j];
        bool eos = false;
        for (int e = 0; e < n_eos; ++e) eos |= id == params[TL_PL_EOS + e];
        if (eos) {
            n = j;
            break;
        }
    }
    if (tid <= K) in_ids[tid] = (tid >= 1 && tid <= n) ? log[start + tid - 1] : last;    // filler: the last token
    if (tid == 0) *n_cand_out = n;
}

__global__ void pl_accept_kernel(const int64_t* __restrict__ ids, const int64_t* __restrict__ in_ids,
                                 const int32_t* __restrict__ n_cand_dev, int32_t* __restrict__ log, int32_t* __restrict__ len_dev,
                                 uint32_t* __restrict__ bits, int L_cap, int W, const int32_t* __restrict__ params,
                                 int64_t* __restrict__ out_log, int32_t* __restrict__ count_dev, int out_cap,
                                 int32_t* __restrict__ pos_dev, int32_t* __restrict__ kv_len_dev, int K) {
    const int lane = threadIdx.x;
    const int len = *len_dev, count = *count_dev, pos = *pos_dev;
    const int nc = max(0, min(*n_cand_dev, K));
    int a = 0;
    while (a < nc && ids[a] == in_ids[a + 1]) ++a;
    // at most max_length - len tokens remain to be generated (none: nothing moves)
    const int e = max(0, min(a + 1, params[TL_PL_MAX_LEN] - len));
    __syncwarp();                                          // every lane has read the counters before lane 0 moves them
    if (lane < e) {
        const int64_t id = ids[lane];
        if (len + lane < L_cap) log[len + lane] = (int32_t)id;
        if (bits && id >= 0 && id < (int64_t)W * 32) atomicOr(&bits[id >> 5], 1u << (id & 31));
        if (count + lane < out_cap) out_log[count + lane] = id;
    }
    if (lane == 0) {
        *len_dev = len + e;
        *count_dev = count + e;
        *pos_dev = pos + e;
        *kv_len_dev = pos + e;
    }
}

// Assisted decoding: a second (smaller) model drafts the K tokens.  Every round starts with a 2-row catch-up of the
// assistant at cache slots P-1 and P (P = len - 1, the slot of the last history token): slot P-1 is the one it never fed
// when all K drafts of the previous round were accepted, slot P may hold a rejected draft.  Its drafts then overwrite
// any slot above P that still holds one, so this and the positions are the whole rollback.
__global__ void assist_prep_kernel(const int32_t* __restrict__ log, const int32_t* __restrict__ len_dev, int L_cap,
                                   int64_t* __restrict__ asst_in, int64_t* __restrict__ in_ids,
                                   int32_t* __restrict__ asst_pos, int32_t* __restrict__ asst_kv_len) {
    const int P = max(min(*len_dev, L_cap) - 1, 1);       // the history holds the prompt and one token at least
    asst_in[0] = log[P - 1];
    asst_in[1] = log[P];
    in_ids[0] = log[P];
    *asst_pos = P - 1;
    *asst_kv_len = P - 1;
}

}  // namespace tl

extern "C" {

int tl_assist_prep(const int32_t* log, const int32_t* len, int L, int64_t* asst_in, int64_t* in_ids, int32_t* asst_pos,
                   int32_t* asst_kv_len, void* stream) {
    using namespace tl;
    TL_REQUIRE(log && len && asst_in && in_ids && asst_pos && asst_kv_len, TL_ERR_INVALID, "tl_assist_prep: null argument");
    TL_REQUIRE(L >= 2, TL_ERR_INVALID, "tl_assist_prep: bad shape L=%d", L);
    assist_prep_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(log, len, L, asst_in, in_ids, asst_pos, asst_kv_len);
    return check_launch("tl_assist_prep");
}

int tl_prompt_lookup_draft(const int32_t* log, const int32_t* len, int L, const int32_t* params_dev, int K, int64_t* in_ids,
                           int32_t* n_cand, void* stream) {
    using namespace tl;
    TL_REQUIRE(log && len && params_dev && in_ids && n_cand, TL_ERR_INVALID, "tl_prompt_lookup_draft: null argument");
    TL_REQUIRE(K >= 1 && K <= TL_PL_MAX_DRAFT && L >= 1, TL_ERR_INVALID, "tl_prompt_lookup_draft: bad shape K=%d L=%d", K, L);
    pl_draft_kernel<<<1, PL_THREADS, 0, (cudaStream_t)stream>>>(log, len, L, params_dev, K, in_ids, n_cand);
    return check_launch("tl_prompt_lookup_draft");
}

int tl_prompt_lookup_accept(const int64_t* ids, const int64_t* in_ids, const int32_t* n_cand, int32_t* log, int32_t* len,
                            uint32_t* bits, int L, int V, const int32_t* params_dev, int64_t* out_log, int32_t* count,
                            int out_cap, int32_t* pos_dev, int32_t* kv_len_dev, int K, void* stream) {
    using namespace tl;
    TL_REQUIRE(ids && in_ids && n_cand && log && len && params_dev && out_log && count && pos_dev && kv_len_dev,
               TL_ERR_INVALID, "tl_prompt_lookup_accept: null argument");
    TL_REQUIRE(K >= 1 && K <= TL_PL_MAX_DRAFT && L >= 1 && V >= 1 && out_cap >= 1, TL_ERR_INVALID,
               "tl_prompt_lookup_accept: bad shape K=%d L=%d V=%d out_cap=%d", K, L, V, out_cap);
    pl_accept_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(ids, in_ids, n_cand, log, len, bits, L, lp_words(V), params_dev,
                                                          out_log, count, out_cap, pos_dev, kv_len_dev, K);
    return check_launch("tl_prompt_lookup_accept");
}

}  // extern "C"
