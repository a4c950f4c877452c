"""The distribution HF ``GenerationMixin.sample`` draws from with ``top_p`` set: ``oracle.navillm_oracle.sampling_probs``
(TemperatureLogitsWarper -> TopKLogitsWarper -> softmax) with transformers' TopPLogitsWarper between top-k and the softmax.
The warper sorts ascending, takes the bf16 softmax and its cumsum, removes every position whose running sum is <= 1 - top_p
(the Python scalar takes the bf16 dtype) and keeps the largest.  Torch leaves the order of equal scores unspecified; this
restatement sorts stably, so a tie group at the cut loses its lowest token indices first, as ``nv_sample`` does.  On CPU
tensors the cumsum is torch's CPU rule that ``nv_sample`` follows (an fp32 running sum, each partial rounded to bf16)."""
import torch
import torch.nn.functional as F

from oracle import navillm_oracle as O


def top_p_filter(s: torch.Tensor, top_p: float) -> torch.Tensor:
    srt, idx = torch.sort(s, dim=-1, descending=False, stable=True)
    cum = srt.softmax(dim=-1).cumsum(dim=-1)
    remove = cum <= (1 - top_p)
    remove[..., -1:] = False
    return s.masked_fill(remove.scatter(-1, idx, remove), float("-inf"))


def sampling_probs(scores: torch.Tensor, temperature: float = 1.0, top_k: int = 50, top_p: float = 1.0) -> torch.Tensor:
    """``oracle.navillm_oracle.sampling_probs`` with the top-p warper between its top-k and its softmax.  The oracle's own
    distribution gives the top-k survivors (its nonzero entries); a finite score whose bf16 probability underflows to 0 sits
    at the front of the ascending order with a running sum of 0, which top-p removes anyway, so masking it first changes
    nothing."""
    probs = O.sampling_probs(scores, temperature, top_k)
    if top_p >= 1.0:                          # generation adds the top-p warper only below 1
        return probs
    s = scores / temperature if temperature != 1.0 else scores
    return F.softmax(top_p_filter(s.masked_fill(probs == 0, float("-inf")), top_p), dim=-1)
