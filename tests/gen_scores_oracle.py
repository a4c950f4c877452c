"""CPU restatements for generate()'s per-step scores (return_dict_in_generate=True, output_scores=True): a literal transcription
of transformers 4.28's ``GenerationMixin.compute_transition_scores`` and torch statements of the values each decoding mode stores
(the warped sampling scores, the beams' processed log-probs)."""
import torch


def compute_transition_scores_428(sequences, scores, beam_indices=None, normalize_logits=False, vocab_size=None):
    """transformers 4.28 ``compute_transition_scores``, step by step (``self.config.vocab_size`` is ``vocab_size``)."""
    # 1. In absence of `beam_indices`, we can assume that we come from e.g. greedy search, which is equivalent
    # to a beam search approach were the first (and only) beam is always selected
    if beam_indices is None:
        beam_indices = torch.arange(scores[0].shape[0]).view(-1, 1).to(sequences.device)
        beam_indices = beam_indices.expand(-1, len(scores))

    # 2. reshape scores as [batch_size*vocab_size, # generation steps] with # generation steps being
    # seq_len - input_length
    scores = torch.stack(scores).reshape(len(scores), -1).transpose(0, 1)

    # 3. Optionally normalize the logits (across the vocab dimension)
    if normalize_logits:
        scores = scores.reshape(-1, vocab_size, scores.shape[-1])
        scores = torch.nn.functional.log_softmax(scores, dim=1)
        scores = scores.reshape(-1, scores.shape[-1])

    # 4. cut beam_indices to longest beam length
    beam_indices_mask = beam_indices < 0
    max_beam_length = (1 - beam_indices_mask.long()).sum(-1).max()
    beam_indices = beam_indices.clone()[:, :max_beam_length]
    beam_indices_mask = beam_indices_mask[:, :max_beam_length]

    # 5. Set indices of beams that finished early to 0
    # such indices will be masked correctly afterwards
    beam_indices[beam_indices_mask] = 0

    # 6. multiply beam_indices with vocab size to gather correctly from scores
    beam_sequence_indices = beam_indices * vocab_size

    # 7. Define which indices contributed to scores
    cut_idx = sequences.shape[-1] - max_beam_length
    indices = sequences[:, cut_idx:] + beam_sequence_indices

    # 8. Compute scores
    transition_scores = scores.gather(0, indices)

    # 9. Mask out transition_scores of beams that stopped early
    transition_scores[beam_indices_mask] = 0

    return transition_scores


def warped_scores(logits, special, temperature, top_k):
    """4.28's sample(): bf16 next-token scores (special ids -inf), TemperatureLogitsWarper in bf16, TopKLogitsWarper (ties at the
    k-th value stay).  Returns the bf16 scores after top-k."""
    v = (logits.float() / temperature).to(torch.bfloat16).float()
    v[:, special] = float("-inf")
    v = torch.nan_to_num(v, nan=float("-inf"))
    if top_k > 0:
        kth = torch.topk(v, min(top_k, v.shape[1]), dim=1).values[:, -1:]
        v = torch.where(v < kth, torch.full_like(v, float("-inf")), v)
    return v.to(torch.bfloat16)


def beam_logprobs(logits, special):
    """nv_beam_topk's per-token log-probs before the beam-score add: special ids -inf, fp32 max m, fp64 sum of exp(x - m),
    ls = fp32(log(sum)), bf16((x - m) - ls) in fp32."""
    x = logits.float().clone()
    x[:, special] = float("-inf")
    m = x.max(dim=1, keepdim=True).values
    ls = torch.log(torch.exp(x.double() - m.double()).sum(dim=1, keepdim=True)).float()
    return ((x - m) - ls).to(torch.bfloat16)


def teacher_forced_logits(sd, cfg, input_ids, attention_mask, path, cand_vis=None):
    """The oracle's bf16 next-token logits [B, V] before each generated column of ``path`` [B, S + n] (the device's own tokens
    fed back, a KV cache as in 4.28's loop): entry t is what step t of a greedy / sampled / contrastive / lookup call reads
    before its processors.  ``modified_lm_forward`` of oracle/navillm_oracle.py."""
    import sys
    from pathlib import Path
    sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
    from oracle import navillm_oracle as O
    B, S = input_ids.shape
    mask = attention_mask.clone()
    past: list = [None] * cfg.n_layers
    pos = (mask.long().cumsum(-1) - 1).masked_fill(mask == 0, 1)
    out = O.modified_lm_forward(sd, cfg, input_ids, mask, cand_vis=cand_vis, position_ids=pos, past_kv=past)
    steps = []
    for t in range(path.shape[1] - S):
        steps.append(out["logits"][:, -1].to(torch.bfloat16))
        if t + 1 == path.shape[1] - S:
            break
        mask = torch.cat([mask, mask.new_ones(B, 1)], dim=1)
        pos = (mask.long().cumsum(-1) - 1)[:, -1:]
        out = O.modified_lm_forward(sd, cfg, path[:, S + t:S + t + 1], mask, position_ids=pos, past_kv=past)
    return steps


def processed_scores(logits, special, history, S, proc=None, trie=None, eos=2):
    """4.28's next-token scores of a greedy / contrastive step: the logits with the special ids -inf, the processors of
    tests/processors_oracle.py on the histories ``history`` [R, S + t] (padded prompt, then the generated tokens), then the trie
    mask (tests/trie_beam_oracle.py) on the generated tokens."""
    from tests import processors_oracle as PO
    from tests import trie_beam_oracle as TB
    s = logits.clone()
    s[:, special] = float("-inf")
    if proc:
        s = PO.process(s, history, S, eos_token_id=eos, **proc)
    if trie is not None:
        s = TB.trie_mask(s, [h[S:].tolist() for h in history], trie)
    return s


def processed_beam_logprobs(logits, special, history, S, proc=None, trie=None, eos=2):
    """``beam_logprobs`` followed by the processors and the trie mask, as 4.28's beam_search applies them to log_softmax's
    output (``next_token_scores_processed``)."""
    from tests import processors_oracle as PO
    from tests import trie_beam_oracle as TB
    lp = beam_logprobs(logits, special)
    if proc:
        lp = PO.process(lp, history, S, eos_token_id=eos, **proc)
    if trie is not None:
        lp = TB.trie_mask(lp, [h[S:].tolist() for h in history], trie)
    return lp


def ulp_bf16(x: torch.Tensor) -> torch.Tensor:
    """One bf16 ulp at |x| (elementwise)."""
    return torch.exp2(torch.floor(torch.log2(x.abs().clamp_min(1e-30))) - 7)


def compare(got, want, ulps: float):
    """The same -inf pattern, then per finite element |got - want| <= ulps bf16 ulp of the row's largest |want| (the noise floor
    of a differently ordered forward).  Returns (finite values, exactly equal, outside the bound, max diff in row ulps)."""
    g, w = got.float(), want.float()
    assert torch.equal(torch.isfinite(g), torch.isfinite(w)), "-inf pattern differs"
    fin = torch.isfinite(w)
    scale = ulp_bf16(torch.where(fin, w, torch.zeros_like(w)).abs().amax(dim=-1, keepdim=True)).expand_as(w)
    d = (g - w).abs()[fin] / scale[fin]
    return int(fin.sum()), int((d == 0).sum()), int((d > ulps).sum()), float(d.max()) if d.numel() else 0.0
