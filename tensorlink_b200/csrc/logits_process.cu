// Logits processors on the device: the per-row token history and the ban set of one decode step.
//
// HF ``generate`` runs RepetitionPenaltyLogitsProcessor -> NoRepeatNGramLogitsProcessor -> MinNewTokensLengthLogitsProcessor
// on the fp32 copy of the logits, with the row's whole ``input_ids`` (prompt, pads included, plus every generated token) as
// the history.  Here the logits never leave the last stage, so each row keeps that history in device memory: a token log
// (for the n-gram scan) and a presence bitmap of V bits (for the penalty, read per logit by the argmax / sampler).
//   * tl_history_fill   one CTA per row: the prompt into the log and the bitmap
//   * ban kernel        one CTA per row: the ids that would complete an n-gram already in the log (a scan of the log in
//                       index order, O(L n)), plus the EOS ids while fewer than min_new_tokens tokens were generated, as a
//                       bitmap of V bits in the workspace
//   * the pick          tl_argmax_proc (lmhead.cu) / tl_sample_proc (sample.cu) apply the penalty and the ban set as they
//                       read each logit, and append the picked id to the history.
#include "common.cuh"

namespace tl {

constexpr int LP_THREADS = 1024;

__global__ void __launch_bounds__(LP_THREADS) history_fill_kernel(const int64_t* __restrict__ prompt, int32_t* __restrict__ log,
                                                                  int32_t* __restrict__ len, uint32_t* __restrict__ bits, int S,
                                                                  int L, int W) {
    const int m = blockIdx.x;
    uint32_t* b = bits + (size_t)m * W;
    for (int i = threadIdx.x; i < W; i += LP_THREADS) b[i] = 0u;
    __syncthreads();
    for (int i = threadIdx.x; i < S; i += LP_THREADS) {
        const int id = (int)prompt[(size_t)m * S + i];
        log[(size_t)m * L + i] = id;
        if (id >= 0 && id < W * 32) atomicOr(&b[id >> 5], 1u << (id & 31));
    }
    if (threadIdx.x == 0) len[m] = S;
}

__global__ void __launch_bounds__(LP_THREADS) ban_kernel(LpRows h, uint32_t* __restrict__ ban_all, int V) {
    const int m = blockIdx.x;
    uint32_t* ban = ban_all + (size_t)m * h.W;
    for (int i = threadIdx.x; i < h.W; i += LP_THREADS) ban[i] = 0u;
    __syncthreads();
    const int32_t* lg = h.log + (size_t)m * h.L;
    const int len = min(h.len[m], h.L);
    const int n = h.params[TL_LP_NGRAM];
    // NoRepeatNGram: while cur_len + 1 >= n, ban lg[i + n - 1] for every i whose n-1 tokens equal the last n-1 tokens
    if (n > 0 && len + 1 >= n) {
        const int tail = len - (n - 1);
        for (int i = threadIdx.x; i + n <= len; i += LP_THREADS) {
            bool same = true;
            for (int j = 0; j < n - 1 && same; ++j) same = lg[i + j] == lg[tail + j];
            if (same) {
                const int id = lg[i + n - 1];
                if (id >= 0 && id < V) atomicOr(&ban[id >> 5], 1u << (id & 31));
            }
        }
    }
    // MinNewTokensLength: every EOS id while fewer than min_new_tokens tokens were generated
    if (threadIdx.x < h.params[TL_LP_N_EOS] && h.len[m] - h.params[TL_LP_PROMPT] < h.params[TL_LP_MIN_NEW]) {
        const int id = h.params[TL_LP_EOS + threadIdx.x];
        if (id >= 0 && id < V) atomicOr(&ban[id >> 5], 1u << (id & 31));
    }
}

int lp_ban_launch(const LpRows& h, uint32_t* ban, int M, int V, cudaStream_t stream) {
    ban_kernel<<<M, LP_THREADS, 0, stream>>>(h, ban, V);
    return check_launch("logits processors: ban set");
}

}  // namespace tl

extern "C" {

size_t tl_logits_proc_ws(int M, int V) {
    // the ban bitmaps, then the argmax partials or the sampler's 65536-bin 64-bit histograms (the larger)
    return tl::lp_ban_bytes(M, V) + (size_t)(M > 0 ? M : 0) * 65536 * sizeof(unsigned long long);
}

int tl_history_fill(const int64_t* prompt, int32_t* log, int32_t* len, uint32_t* bits, int M, int S, int L, int V,
                    void* stream) {
    using namespace tl;
    TL_REQUIRE(prompt && log && len && bits, TL_ERR_INVALID, "tl_history_fill: null argument");
    TL_REQUIRE(M >= 1 && S >= 1 && V >= 1 && S <= L, TL_ERR_INVALID, "tl_history_fill: bad shape M=%d S=%d L=%d V=%d", M, S, L, V);
    history_fill_kernel<<<M, LP_THREADS, 0, (cudaStream_t)stream>>>(prompt, log, len, bits, S, L, lp_words(V));
    return check_launch("tl_history_fill");
}

}  // extern "C"
