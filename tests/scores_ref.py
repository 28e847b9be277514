"""CPU reference of the scores ``generate(return_dict_in_generate=True, output_scores=True)`` returns: HF's own logits
processors and warpers applied in torch fp32 to the fp32 copy of a bf16 logits row, in HF's order
(RepetitionPenalty -> NoRepeatNGram -> MinNewTokensLength, then Temperature -> TopK -> TopP when sampling)."""
import torch


def hf_processed(logits_bf16, hist, penalty=1.0, ngram=0, min_new=0, prompt_len=0, eos=()):
    """HF's processed scores (fp32) of each row of ``logits_bf16`` [M, V] with the token history ``hist[r]`` (int64)."""
    from transformers.generation.logits_process import (MinNewTokensLengthLogitsProcessor, NoRepeatNGramLogitsProcessor,
                                                        RepetitionPenaltyLogitsProcessor)
    out = []
    for r, h in enumerate(hist):
        s = logits_bf16[r:r + 1].float().clone()
        ids = h.view(1, -1)
        if penalty != 1.0:
            s = RepetitionPenaltyLogitsProcessor(penalty)(ids, s)
        if ngram:
            s = NoRepeatNGramLogitsProcessor(ngram)(ids, s)
        if min_new and eos:
            s = MinNewTokensLengthLogitsProcessor(prompt_len, min_new, list(eos))(ids, s)
        out.append(s)
    return torch.cat(out)


def hf_warped_scores(scores, temperature=1.0, top_k=0, top_p=1.0):
    """HF's TemperatureLogitsWarper -> TopKLogitsWarper -> TopPLogitsWarper on fp32 scores [M, V]: the removed entries
    become -inf.  (HF adds each warper only when it is not neutral; so does this.)"""
    from transformers.generation.logits_process import TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper
    s = scores.clone()
    if temperature != 1.0:
        s = TemperatureLogitsWarper(temperature)(None, s)
    if top_k:
        s = TopKLogitsWarper(top_k)(None, s)
    if top_p < 1.0:
        s = TopPLogitsWarper(top_p)(None, s)
    return s


def kept_scores(scores, kept, temperature):
    """What the sampler logs: scores / temperature (IEEE fp32 division) where ``kept`` (bool [M, V]), -inf elsewhere."""
    return torch.where(kept, scores / torch.tensor(temperature, dtype=torch.float32), torch.tensor(float("-inf")))
