"""``ModifiedLlamaForCausalLM.generate``'s decoding (HF GenerationMixin greedy / sampling / beam / contrastive search): the call's
record, the decode states, the prefill, the graph-replayed step loop and the drivers ``decode``, ``lookup_decode``,
``beam_search`` and ``contrastive_search``."""
from __future__ import annotations

import collections
import dataclasses
from types import SimpleNamespace
from typing import Optional

import numpy as np
import torch

from . import llama as llama_mod
from . import ops

bf16 = torch.bfloat16
BEAM_MAX = 8                   # beams per prompt the beam kernels are built for


@dataclasses.dataclass(frozen=True)
class Decoding:
    """One ``generate()`` call's decoding rule, after validation.  Fields a mode does not use are None."""
    eos: int
    pad: int
    stop_on_eos: Optional[bool]          # None for beams: a prompt stops when its hypotheses are done
    mode: str                            # "greedy", "sample", "trie", "trie+sample", "beam", "contrastive", "lookup" or
                                         # "trie_score" (``score_answers``)
    kv: str                              # the KV cache format, "bf16" or "fp8"
    temperature: Optional[float] = None  # sampled modes
    top_k: Optional[int] = None          # sampled modes, and contrastive search's candidates per prompt (= n)
    top_p: Optional[float] = None
    trie_eos: Optional[int] = None       # trie modes: the flattened trie's end-of-answer id
    n: int = 1                           # rows per prompt: samples, or beams
    early_stopping: Optional[bool] = None
    proc: Optional[tuple] = None         # the device logits processors (``processors``)
    n_return: int = 1                    # beams: sequences returned per prompt (host finalisation)
    length_penalty: Optional[float] = None   # beams: its normalisers are copied into the state every call
    penalty_alpha: Optional[float] = None    # contrastive search: the degeneration penalty's weight
    lookup_k: Optional[int] = None           # prompt-lookup decoding: drafts per step (the window is lookup_k + 1 rows)
    lookup_ngram: Optional[int] = None       # prompt-lookup decoding: max_matching_ngram_size
    scores: bool = False                     # return_dict_in_generate + output_scores: the step stores HF's per-step scores
    groups: int = 1                          # beams: num_beam_groups (diverse beam search when > 1)
    diversity_penalty: Optional[float] = None    # diverse beam search: the Hamming diversity penalty
    batch_invariant: bool = False            # ModifiedLlamaForCausalLM.set_batch_invariant: the step runs other kernels

    @property
    def sampled(self) -> bool:
        return self.mode in ("sample", "trie+sample")

    def key(self) -> tuple:
        """The graph key: every field a captured step bakes in (not ``n_return`` or ``length_penalty``), the format last."""
        return (self.eos, self.pad, self.stop_on_eos, self.mode, self.temperature, self.top_k, self.top_p, self.trie_eos, self.n,
                self.early_stopping, self.proc, self.penalty_alpha, self.lookup_k, self.lookup_ngram, self.scores, self.groups,
                self.diversity_penalty, self.batch_invariant, self.kv)


def processors(repetition_penalty, no_repeat_ngram_size, min_length, min_new_tokens, eos: int) -> Optional[tuple]:
    """Validate HF's processor kwargs as transformers does; returns (penalty, n, min_length, min_new_tokens, eos) for the
    kernels, or None when every one is at its default (off), which keeps the call on the processor-free path."""
    p = 1.0 if repetition_penalty is None else repetition_penalty
    if p != 1.0 and (isinstance(p, bool) or not isinstance(p, float) or not p > 0):
        raise ValueError(f"generate(repetition_penalty={repetition_penalty!r}): has to be a strictly positive float")
    named = (("no_repeat_ngram_size", no_repeat_ngram_size), ("min_length", min_length), ("min_new_tokens", min_new_tokens))
    ints = []
    for name, v in named:
        v = 0 if v is None else v
        if isinstance(v, bool) or not isinstance(v, int) or v < 0:
            raise ValueError(f"generate({name}={v!r}): has to be a non-negative integer")
        ints.append(v)
    if p == 1.0 and not any(ints):
        return None
    return (float(p), *ints, int(eos))


def logits_buffer(rows: int, V: int, device) -> torch.Tensor:
    """Uninitialised bf16 [rows, V] logits whose rows start 16-byte aligned (a row stride of V rounded up to 64)."""
    return torch.empty((rows, (V + 63) // 64 * 64), dtype=bf16, device=device)[:, :V]


class DecodeStates(collections.OrderedDict):
    """A model's persistent decode states by key (shapes and ``Decoding.key()``), least recently used first.  A state holds
    the KV caches, the step's I/O buffers and -- once captured -- the CUDA graph of ONE decode step.  Capturing and
    instantiating the ~260-node graph costs more than the 127 replays of a C3 generation save, so a state is kept for later
    calls with the same key (evaluation loops call generate with the same shapes over and over), at most ``max_states`` of
    them.  Whatever changes the weight buffers or the kernels a captured graph launches must ``clear()`` them."""

    max_states = 2

    def lookup(self, key, build, want_graph: bool):
        """The state under ``key``, now the most recently used, or a new one from ``build()``.  A call that will not replay a
        graph neither looks up nor keeps a state."""
        if not want_graph:
            return build()
        if key in self:
            self.move_to_end(key)
            return self[key]
        st = self[key] = build()
        while len(self) > self.max_states:
            self.popitem(last=False)
        return st


def _grow(st, cap_name: str, need: tuple, alloc) -> tuple:
    """Capacities ``getattr(st, cap_name)`` of persistent buffers of ``st`` (a captured graph keeps their pointers): when
    ``need`` exceeds them, each grows to the next power of two (a need of 0 stays 0), ``alloc(*caps)`` re-allocates the
    buffers and the state's graph is dropped.  Returns the capacities."""
    cap = getattr(st, cap_name, (0,) * len(need))
    if any(n > c for n, c in zip(need, cap)):
        cap = tuple(max(c, 1 << (n - 1).bit_length() if n else 0) for n, c in zip(need, cap))
        alloc(*cap)
        setattr(st, cap_name, cap)
        st.graph = None
    return cap


def load_trie(st, table) -> tuple:
    """Copy a flattened trie into the state's ``trie_buf`` in one host-to-device copy (a trie that outgrows it drops the
    state's graph).  Returns the kernels' (node_ptr, child_tok, child_node, n_nodes) views."""
    def alloc(ncap, ecap):
        st.trie_buf = torch.empty(ncap + 2 + 2 * ecap, dtype=torch.int32, device=st.next_ids.device)
    ncap, ecap = _grow(st, "trie_cap", (table.n_nodes, max(table.n_edges, 1)), alloc)
    st.trie_buf.copy_(torch.from_numpy(table.pack(ncap, ecap)))
    o = ncap + 2
    return st.trie_buf[:o], st.trie_buf[o:o + ecap], st.trie_buf[o + ecap:], ncap


def load_scores(st, planes: int, rows: int, V: int) -> None:
    """The per-step scores of a ``dec.scores`` call in persistent buffers of ``st``: ``st.scores`` bf16 [>= planes, rows, V]
    (``ops.scores_buffer``; a captured step writes plane ``st.score_t[0]`` and advances it, so the counter is zeroed here) and
    ``st.score_prev`` int32 [rows] (prompt lookup: the columns emitted before a step)."""
    dev = st.next_ids.device

    def alloc(cap):
        st.scores = ops.scores_buffer(cap, rows, V, dev)
        st.score_t = torch.zeros((1,), dtype=torch.int32, device=dev)
        st.score_prev = torch.zeros((rows,), dtype=torch.int32, device=dev)
    _grow(st, "score_cap", (max(planes, 1),), alloc)
    st.score_t.zero_()


def take_scores(st, n: int) -> tuple:
    """HF's ``scores`` tuple: the first ``n`` planes copied once into a fresh tensor (the next call reuses the state's
    buffer), one [rows, V] entry per plane."""
    return tuple(st.scores[:n].clone().unbind(0))


def load_proc(st, input_ids, rows: int, G: int) -> None:
    """The logits processors' device state in persistent buffers of ``st``: the padded prompt ids ``proc_ids`` [P, >= S] and
    their width S ``proc_width`` [1], copied once per call, and -- for ``rows`` > 0 -- the generated history ``proc_hist``
    [rows, >= G] with its per-row length ``proc_len`` (zeroed; the step appends to it)."""
    P, S = input_ids.shape
    dev = st.next_ids.device

    def alloc(scap, gcap):
        st.proc_ids = torch.zeros((P, scap), dtype=torch.int32, device=dev)
        st.proc_width = torch.zeros((1,), dtype=torch.int32, device=dev)
        if rows:
            st.proc_hist = torch.zeros((rows, gcap), dtype=torch.int32, device=dev)
            st.proc_len = torch.zeros((rows,), dtype=torch.int32, device=dev)
    _grow(st, "proc_cap", (S, G if rows else 0), alloc)
    st.proc_ids[:, :S].copy_(input_ids.to(torch.int32))
    st.proc_width.fill_(S)
    if rows:
        st.proc_len.zero_()


def prefill(lm, dec: Decoding, input_ids, attention_mask, vis, max_new_tokens: int, want_graph: bool, host: bool = False):
    """Pack the prompts (positions = cumsum(mask) - 1, as HF generate), find or build the call's decode state and run the
    prompt forward into its cache; the visual rows (cand, hist, obj) are injected here only, as in
    models/modified_lm.py:195-197.  Returns the packed prompt, the state and the last hidden row of every prompt.

    One sequence per prompt: kc / vc [B, G, D] per layer hold each row's prompt and generated keys.  Several samples, or
    beams, per prompt (``dec.n`` > 1): the prompt keys go to a prompt cache ``pk`` / ``pv`` [B, Sp, D] that the n rows of a
    prompt share (``plens`` keys each), and kc / vc [B * n, G, D] hold only the generated keys, read through the source table
    ``src`` (``st.beam``), so no K/V is copied.  Sampling adds its uniform numbers ``u`` (the host processors draw their
    own), tries their masked logits and walk state (beams walk statelessly inside ``ops.beam_topk_trie``), beams the scorer's
    buffers (``ops.beam_select``).

    Contrastive search (``dec.n`` = k candidates per prompt): the prompt cache holds the prompt and then the selected tokens
    (Sp = bucket(longest prompt + max_new_tokens)), kc / vc [B * k, 1, D] the candidates' own keys, one slot each; the logits,
    ids and flags are per prompt ([B]), and the prefill returns every prompt row of the last layer (the context).  See
    ``contrastive_search``.

    Prompt-lookup decoding (``dec.lookup_k`` = k): one sequence per prompt in a cache of bucket(longest prompt + max_new_tokens
    + k) rows, so that every verify window's k + 1 writes fit, and [B * (k + 1)] logits rows.  See ``lookup_decode``.

    Answer scoring (``dec.mode`` "trie_score", ``max_new_tokens`` = the trie's N' tree rows): one sequence per prompt in a
    zeroed cache of bucket(longest prompt + N') rows (the tree attention reads rows past kv_len as masked zeros), never
    graphed.  See ``score_answers``."""
    from .modified_lm import PackedPrompt           # modified_lm imports this module
    dev, d = lm._device(), lm.dims
    pp = PackedPrompt(input_ids, attention_mask, lm, dev, generate_positions=True)
    vis = lm.cat_vis(*vis, pp)
    bucket = lambda n: (n + 127) // 128 * 128       # cache lengths in multiples of 128: more calls share a state
    B, n, V = pp.B, dec.n, lm.lm_head.weight.shape[0]
    R, shared, cs = B * n, n > 1, dec.mode == "contrastive"
    Sp, G = (bucket(max(pp.seqlens)), bucket(max_new_tokens)) if shared else (0, bucket(max(pp.seqlens) + max_new_tokens))
    if cs:
        Sp, G = bucket(max(pp.seqlens) + max_new_tokens), 1
    W = 1 if dec.lookup_k is None else dec.lookup_k + 1   # decode rows per sequence in a step
    if W > 1:
        G = bucket(max(pp.seqlens) + max_new_tokens + dec.lookup_k)
    P = B if cs else R                              # rows with their own logits, ids and finished flag

    def build():
        cache = lambda rows, length: llama_mod.kv_cache(d, rows, length, dec.kv, dev, zero=dec.mode == "trie_score")
        zeros = lambda dtype, *shape: torch.zeros(shape, dtype=dtype, device=dev)
        i32 = lambda *shape: zeros(torch.int32, *shape)
        st = SimpleNamespace(kc=cache(R, G), vc=cache(R, G), logits=logits_buffer(P * W, V, dev), next_ids=i32(P), lens=i32(R),
                             Sp=Sp, G=G, graph=None)
        if dec.mode == "beam":
            c = 2 * n // dec.groups                                         # candidates per prompt (and group) and step
            st.beam_score, st.cand_score, st.cand_tok = zeros(torch.float32, R), zeros(torch.float32, B, c), i32(B, c)
            st.cand_par, st.hist, st.src, st.hyp_score = i32(B, c), i32(R, G), i32(R, G), zeros(torch.float64, B, n + 1)
            st.hyp_meta, st.hyp_tok, st.pstate, st.norm = i32(B, n, 2), i32(B, n, G), i32(B, 5), zeros(torch.float64, G)
            if dec.scores:                                                  # 4.28's beam_indices (ops.beam_select trace=)
                st.par_hist, st.hyp_par, st.done_step = i32(R, G), i32(B, n, G), i32(B)
        else:
            st.finished = i32(P)
            if shared:                                                      # the identity source table
                st.src = torch.arange(R, dtype=torch.int32, device=dev)[:, None].expand(R, G).contiguous()
        if shared:
            st.pk, st.pv, st.plens = cache(B, Sp), cache(B, Sp), i32(B)
            st.beam = SimpleNamespace(pk=st.pk, pv=st.pv, plens=st.plens, src=st.src, K=n)
        if cs:
            st.cand_p, st.cand_ids, st.sel, st.pen_key = zeros(bf16, B, n), i32(B, n), i32(B), i32(R)
            st.ctx, st.ctx_len, st.hsel = zeros(bf16, B, Sp, d.hidden), i32(B), zeros(bf16, B, d.hidden)
            st.commit_table = ops.contrastive_commit_table(st.kc, st.vc, st.pk, st.pv)
        if dec.sampled and not host:
            st.u = torch.empty((R,), dtype=torch.float32, device=dev)
        if dec.trie_eos is not None and dec.mode != "beam":
            st.masked, st.node, st.miss = logits_buffer(R, V, dev), i32(R), i32(1)
        return st
    # a verify step bakes max_new_tokens into its accept launch
    st = lm._decode_states.lookup((R, G, (B, Sp) if shared else None, max_new_tokens if W > 1 else None) + dec.key(), build,
                                  want_graph)
    if shared:
        st.plens.copy_(torch.tensor(pp.seqlens, dtype=torch.int32), non_blocking=True)
    x = ops.embed_fwd(pp.ids, lm.model.embed_tokens.weight.data, pp.vis_src if vis is not None else None, vis)
    h, _ = lm.core.forward(x, pp.pos, pp.cu, pp.seqlens, save=False, kv_store=(st.pk, st.pv) if shared else (st.kc, st.vc),
                           out_rows=None if cs else pp.last_rows)
    return pp, st, h


def decode_head(lm, h_rows: torch.Tensor, out: torch.Tensor) -> None:
    """Final RMSNorm + lm_head of decode rows into ``out`` [rows, V] bf16 (the fp8 weight copy when there is one)."""
    hn, _ = ops.rmsnorm_fwd(h_rows, lm.model.norm.weight.data, lm.dims.rms_eps)
    lm_head_rows(lm, hn, out)


def lm_head_rows(lm, hn: torch.Tensor, out: torch.Tensor) -> None:
    """lm_head of final-norm rows ``hn`` into ``out`` [rows, V] bf16 (the fp8 weight copy when there is one)."""
    B = hn.shape[0]
    fp8_head = lm._fp8.view([lm.lm_head.weight], tuple(lm.lm_head.weight.shape)) if lm.core.fp8 is not None else None
    if lm.core.batch_invariant:
        ops.gemm_bi(hn, lm.lm_head.weight.data, out=out)
    elif B <= 16 and fp8_head is not None:
        ops.gemm_skinny_fp8(hn, *fp8_head, out=out)
    elif B <= llama_mod.FP8_MAX_ROWS and fp8_head is not None:
        ops.gemm_fp8w(hn, *fp8_head, out=out)
    elif B <= 16:
        ops.gemm_skinny(hn, lm.lm_head.weight.data, out=out)
    else:
        ops.gemm(hn, lm.lm_head.weight.data, out=out)


def step_loop(st, step, n_tokens: int, done, every: int, graphed: bool, before=None, after=None) -> tuple:
    """Steps for tokens 1 .. n_tokens - 1: ``step()``, or -- ``graphed`` -- replays of ``st.graph``, captured after the eager
    step of the first iteration that finds none (which yields that iteration's token).  ``done()`` (if not None) is asked
    every ``every`` tokens and ends the loop; ``before()`` / ``after()`` run around each step.  Returns (steps, replays)."""
    it, replays = 1, 0
    while it < n_tokens:
        if done is not None and it % every == 0 and done():
            break
        if before is not None:
            before()
        if graphed and st.graph is not None:
            st.graph.replay()
            replays += 1
        else:
            step()
        if after is not None:
            after()
        if graphed and st.graph is None:
            g = torch.cuda.CUDAGraph()
            torch.cuda.synchronize()
            with torch.cuda.graph(g):
                step()
            st.graph = g
        it += 1
    return it - 1, replays


class PhaseTimer:
    """Device-side phase times of one call for ``stats=`` (bench.py reads prefill_ms, decode_ms and decode_steps): events at
    the start, after the prefill's token (``mark()``) and after the decode steps; one synchronise at the end."""

    def __init__(self, stats: Optional[dict]):
        self.stats, self.ev = stats, []
        self.mark()

    def mark(self) -> None:
        if self.stats is not None:
            self.ev.append(torch.cuda.Event(enable_timing=True))
            self.ev[-1].record()

    def finish(self, pp, steps: int, replays: int, kv_rows: int, **extra) -> None:
        if self.stats is not None:
            self.mark()
            torch.cuda.synchronize()
            ev = self.ev
            self.stats.update({"prefill_ms": ev[0].elapsed_time(ev[1]), "decode_ms": ev[1].elapsed_time(ev[2]) if steps else None,
                              "decode_steps": steps, "graph_replays": replays, "kv_rows": kv_rows,
                              "prompt_lens": list(pp.seqlens), **extra})


def decode(lm, input_ids, attention_mask, vis, max_new_tokens, use_cuda_graph, stats, dec: Decoding, procs=(), table=None,
           out_fields: Optional[dict] = None):
    """``generate`` without beams, with the host processors ``procs`` (the host path when not empty) or the flattened trie
    ``table`` walked on the device; returns None when the device walk reported a miss.  ``dec.n`` > 1 (sampling without
    processors): the n samples of a prompt start from its last hidden row, over its prompt cache; the visual tokens of
    prompt b reach all n samples of prompt b.  ``dec.scores``: every pick also stores what it read -- the processed (trie-masked)
    logits with the special ids -inf (``ops.scores_store``), or the warped scores of ``ops.sample`` -- in plane ``st.score_t``
    of ``st.scores``, inside the captured step; ``out_fields["scores"]`` gets one [R, V] entry per generated column."""
    timer = PhaseTimer(stats)
    host = bool(procs)                                        # processors walk the generated ids on the host
    graphed = use_cuda_graph and not host
    pp, st, hid_last = prefill(lm, dec, input_ids, attention_mask, vis, max_new_tokens, graphed, host)
    dev, n = lm._device(), dec.n
    R, shared = pp.B * n, n > 1                               # decode rows; shared: a prompt cache per prompt
    logits, next_ids, finished, lens = st.logits, st.next_ids, st.finished, st.lens
    if table is not None:
        trie_csr = load_trie(st, table)
        st.node.zero_()                                       # every row starts at the root
        st.miss.zero_()
    if dec.proc is not None:
        load_proc(st, input_ids, R, max_new_tokens)
    if dec.scores:
        load_scores(st, max_new_tokens, R, logits.shape[1])
    finished.zero_()
    lens.copy_(torch.tensor(pp.seqlens, dtype=torch.int32).repeat_interleave(n), non_blocking=True)
    if shared:                                                # the n samples of a prompt start from its last row
        hid_last = hid_last.repeat_interleave(n, dim=0)
    special, eos, pad, stop = lm.special_ids_dev, dec.eos, dec.pad, dec.stop_on_eos

    def head(h_rows, append=None):
        """lm_head into `logits`, then the logits processors, whose history first takes the token in `append`."""
        decode_head(lm, h_rows, logits)
        if dec.proc is not None:
            ops.logits_process_(logits, st.proc_ids, st.proc_width, st.proc_hist, st.proc_len, append, dec.proc,
                                rows_per_prompt=n)

    def pick_host(all_ids_host):
        """next token from `logits` -> next_ids (device), through the host processors."""
        lg = logits.float()
        lg[:, lm.special_token_ids] = float("-inf")
        for p in procs:
            lg = p(torch.tensor(all_ids_host, device=dev), lg)
        if dec.sampled:
            ops.sample(lg.to(torch.bfloat16), special, finished, eos, pad, stop, dec.temperature, dec.top_k, dec.top_p,
                       torch.rand(R, device=dev, dtype=torch.float32), next_ids, **scored)
            if dec.scores:
                ops.add_int_(st.score_t, 1)
            return
        if dec.scores:
            ops.scores_store(lg.to(torch.bfloat16), special, st.scores, st.score_t)
            ops.add_int_(st.score_t, 1)
        nxt = lg.argmax(dim=-1)
        fin = finished.bool()
        nxt = torch.where(fin, torch.full_like(nxt, pad), nxt)
        if stop:
            finished.copy_((fin | (nxt == eos)).to(torch.int32))
        next_ids.copy_(nxt.to(torch.int32))

    def pick(advance):
        """next token from `logits` -> next_ids (device) without host work; with a trie, the row's node first advances by
        the token in next_ids (``advance``) and the pick reads the trie-masked copy of the logits."""
        src = logits
        if table is not None:
            ops.trie_mask(logits, st.masked, *trie_csr, table.eos, special, st.node, next_ids if advance else None, st.miss)
            src = st.masked
        if dec.sampled:
            st.u.uniform_()                                   # = torch.rand(R): the same numbers, into a static buffer
            ops.sample(src, special, finished, eos, pad, stop, dec.temperature, dec.top_k, dec.top_p, st.u, next_ids, **scored)
        else:
            if dec.scores:
                ops.scores_store(src, special, st.scores, st.score_t)
            ops.argmax_masked(src, special, finished, eos, pad, stop, next_ids)
        if dec.scores:
            ops.add_int_(st.score_t, 1)

    scored = dict(scores=st.scores, step=st.score_t) if dec.scores else {}
    head(hid_last)
    host_ids = [row.tolist() for row in input_ids.cpu()] if host else None
    if host:
        pick_host(host_ids)
    else:
        pick(advance=False)
    out_tokens = [next_ids.clone()]
    timer.mark()

    def step():
        with ops.pdl():                         # programmatic dependent launch along the whole decode chain
            xt = ops.embed_fwd(next_ids, lm.model.embed_tokens.weight.data)
            h = lm.core.decode_step(xt, lens, st.kc, st.vc, beam=st.beam if shared else None)
            head(h, append=next_ids)
            ops.add_int_(lens, 1)
            if not host:
                pick(advance=True)
        if host:
            pick_host(host_ids)

    def append_host_ids():
        for bn, t in enumerate(out_tokens[-1].tolist()):
            host_ids[bn].append(t)

    # HF stops when every sequence has finished.  Asking the device after EVERY token would serialise host and device
    # (one blocking read per token); finished rows only emit pad tokens, so the greedy and sampled loops look every
    # `check_every` tokens and the surplus pad columns are trimmed below -- same ids as a per-token check.  Trie-constrained
    # answers are a handful of tokens: there the check stays per token, as on the host path.
    check_every = 1 if host or table is not None else 8
    steps, replays = step_loop(st, step, max_new_tokens, (lambda: bool(finished.all())) if stop else None, check_every, graphed,
                               before=append_host_ids if host else None, after=lambda: out_tokens.append(next_ids.clone()))
    miss = False
    if table is not None:
        # one more advance, outside the graph: a token picked at the last step that is not a child is a miss as well
        ops.trie_mask(logits, st.masked, *trie_csr, table.eos, special, st.node, next_ids, st.miss)
        miss = bool(st.miss.item())
    timer.finish(pp, steps, replays, st.Sp + st.G)
    if miss:
        return None
    new = torch.stack(out_tokens, dim=1).to(torch.int64)
    if stop and check_every > 1:
        new = trim_after_eos(new, eos)                        # see check_every above
    if out_fields is not None:
        out_fields["scores"] = take_scores(st, new.shape[1]) if dec.scores else None
    return torch.cat([input_ids.to(dev).repeat_interleave(n, dim=0), new], dim=1)


# ---- answer scoring: every answer of a trie teacher-forced in one tree-masked forward over the prompt cache ----
TREE_MAX_ROWS = 16384          # tree rows (prompts x N') per suffix forward: bounds its activations and the [rows, V] logits


def score_answers(lm, input_ids, attention_mask, vis, rows, length_penalty: float, stats, dec: Decoding) -> dict:
    """The log-probability of every answer of a trie under each prompt (``ModifiedLlamaForCausalLM.score_answers``).  ``rows``:
    the trie's ``trie.TreeRows`` (N' nodes, A answers).  The prompts are prefilled once into a zeroed cache of
    bucket(longest prompt + N') rows (``prefill``, mode "trie_score"); then, for chunks of prompts with at most
    ``TREE_MAX_ROWS`` tree rows in all, the N' tree tokens of each prompt run as one suffix forward with the tree mask
    (``forward_suffix(tree_end=...)``: node (t_1 .. t_i) holds t_i at position p_b + i - 1 and attends to the prompt and to
    t_1 .. t_i, the keys decode steps along that path would have), the final RMSNorm and the lm_head run on the prompt's last
    row and the tree rows, and ``ops.trie_score`` folds each answer's bf16 log-probs in fp32.  One device-to-host copy at the
    end.  Returns dict(answers, logprob fp32 [B, A], score fp64 [B, A], best int64 [B]) on the host; score is
    logprob / (S + d) ** length_penalty in Python floats, as ``nv_beam_select`` scores that hypothesis."""
    N, A = rows.n, len(rows.paths)
    if N > TREE_MAX_ROWS:
        raise NotImplementedError(f"score_answers: a trie of {N} nodes; at most {TREE_MAX_ROWS} (TREE_MAX_ROWS) are built")
    timer = [torch.cuda.Event(enable_timing=True) for _ in range(2)] if stats is not None else None
    if timer:
        timer[0].record()
    pp, st, hid_last = prefill(lm, dec, input_ids, attention_mask, vis, N, False)
    if timer:
        timer[1].record()
    dev, d, B, G, S = lm._device(), lm.dims, pp.B, st.G, int(input_ids.shape[1])
    R = N + 1                                                  # logits rows per prompt: the prompt's last row, then the tree
    # one host-to-device copy: tok | end | depth - 1 | path_off | path_rows (never empty, so no view has a null pointer)
    path_off = np.concatenate([[0], np.cumsum([len(p) for p in rows.paths])])
    path_rows = np.array([r for p in rows.paths for r in p], dtype=np.int64)
    host = np.concatenate([rows.tok, rows.end, rows.depth - 1, path_off, path_rows, [0]]).astype(np.int32)
    buf = torch.from_numpy(host).to(dev)
    o = np.cumsum([0, N, N, N, A + 1, len(path_rows)])
    tok, tree_end, dpos, poff, prow = (buf[o[i]:o[i + 1]] for i in range(5))
    plens = torch.tensor(pp.seqlens, dtype=torch.int32, device=dev)
    per = max(1, TREE_MAX_ROWS // max(N, 1))                   # prompts per chunk
    norm_w, eps, E = lm.model.norm.weight.data, d.rms_eps, lm.model.embed_tokens.weight.data
    V = lm.lm_head.weight.shape[0]
    logprob = torch.empty((B, A), dtype=torch.float32, device=dev)
    events, chunks = [], 0
    for c0 in range(0, B, per):
        c1 = min(B, c0 + per)
        nb = c1 - c0
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)] if stats is not None else None
        if ev:
            ev[0].record()
        h = torch.empty((nb, R, d.hidden), dtype=bf16, device=dev)
        h[:, 0] = hid_last[c0:c1]
        if N:
            pl = plens[c0:c1]
            x = ops.embed_fwd(tok.repeat(nb), E)
            pos = (pl[:, None] + dpos[None, :]).view(-1)
            cu = torch.arange(0, (nb + 1) * N, N, dtype=torch.int32, device=dev)
            kv_start = torch.arange(0, nb * G, G, dtype=torch.int32, device=dev)
            part = lambda caches: [(c[0][c0:c1], c[1][c0:c1]) if isinstance(c, tuple) else c[c0:c1] for c in caches]
            h[:, 1:] = lm.core.forward_suffix(x, pos, cu, [N] * nb, part(st.kc), part(st.vc), pl, kv_start, pl + N,
                                              tree_end=tree_end).view(nb, N, d.hidden)
        if ev:
            ev[1].record()
        hn, _ = ops.rmsnorm_fwd(h.view(nb * R, d.hidden), norm_w, eps)
        logits = logits_buffer(nb * R, V, dev)
        lm_head_rows(lm, hn, logits)
        ops.trie_score(logits, lm.special_ids_dev, tok, poff, prow, rows.eos, nb, logprob=logprob[c0:c1])
        if ev:
            ev[2].record()
            events.append(ev)
        chunks += 1
    lp = logprob.cpu()
    norm = torch.tensor([(S + len(p)) ** length_penalty for p in rows.paths], dtype=torch.float64)
    score = lp.to(torch.float64) / norm
    best = score.argmax(dim=1)                                 # the first of equal maxima: the lowest answer index
    if stats is not None:
        stats.update({"prefill_ms": timer[0].elapsed_time(timer[1]),
                      "tree_ms": sum(e[0].elapsed_time(e[1]) for e in events),
                      "score_ms": sum(e[1].elapsed_time(e[2]) for e in events),
                      "tree_rows": B * N, "chunks": chunks, "prompt_lens": list(pp.seqlens)})
    return {"answers": [list(a) for a in rows.answers], "logprob": lp, "score": score, "best": best}


# ---- prompt-lookup speculative decoding (HF generate(prompt_lookup_num_tokens=k), greedy) ----
# A step that accepts drafts finishes a row in fewer steps than greedy's 8-step check interval would notice; a check is one
# blocking read between two graph replays.
LOOKUP_CHECK_EVERY = 4


def lookup_history(input_ids, attention_mask, cap: int) -> tuple:
    """Each prompt's non-pad ids, left-aligned in an int32 [B, cap] host array, and their counts: where the drafts of
    ``ops.lookup_draft`` are looked up (the generated tokens are appended on the device)."""
    ids = input_ids.detach().cpu().numpy()
    msk = np.ones(ids.shape, dtype=bool) if attention_mask is None else attention_mask.detach().cpu().numpy().astype(bool)
    hist = np.zeros((ids.shape[0], cap), dtype=np.int32)
    lens = msk.sum(1).astype(np.int32)
    for b in range(ids.shape[0]):
        hist[b, :lens[b]] = ids[b][msk[b]]
    return hist, lens


def lookup_decode(lm, input_ids, attention_mask, vis, max_new_tokens, use_cuda_graph, stats, dec: Decoding,
                  out_fields: Optional[dict] = None):
    """Greedy decoding that verifies k = ``dec.lookup_k`` drafted tokens per step.  After the prefill and its first token (as
    in ``decode``), a step is: ``ops.lookup_draft`` proposes k tokens per prompt from n-grams of its history (prompt and
    generated tokens, HF's PromptLookupCandidateGenerator); the last token and the k drafts run as one causal window of k + 1
    decode rows per prompt (``decode_step(window=k + 1)``, all rows through the lm_head); ``ops.lookup_accept`` keeps the drafts
    that equal the argmax of the row before them and emits those plus one token, 1 .. k + 1 per prompt and step.  A row's tokens
    are the argmax of its own prefix, so the ids are greedy decoding's whatever the drafts are; they differ from ``decode`` only
    where a different row count in a GEMM moves a near tie.  Static shapes: the step is captured once and replayed; the
    generated ids stay on the device until one copy at the end.  Returns [B, S0 + n_new] with ``decode``'s width and pads.
    ``dec.scores``: column c of prompt b gets the logits row that picked its token (``ops.lookup_scores`` after the accept, inside
    the captured step); the planes start at -inf, so a column after a row's EOS, which that row never runs, stays -inf."""
    k, eos, pad, stop, special = dec.lookup_k, dec.eos, dec.pad, dec.stop_on_eos, lm.special_ids_dev
    W, n_out = k + 1, max(max_new_tokens, 1)
    timer = PhaseTimer(stats)
    pp, st, hid_last = prefill(lm, dec, input_ids, attention_mask, vis, max_new_tokens, use_cuda_graph)
    B, dev = pp.B, lm._device()
    hist0, plens = lookup_history(input_ids, attention_mask, int(input_ids.shape[1]) + n_out)

    def alloc(hcap, ocap):
        i32 = lambda *shape: torch.zeros(shape, dtype=torch.int32, device=dev)
        st.hist, st.out, st.drafts, st.win = i32(B, hcap), i32(B, ocap), i32(B, k), i32(B, W)
        st.hist_len, st.n_out, st.n_acc = i32(B), i32(B), i32(B)
    _grow(st, "lookup_cap", (hist0.shape[1], n_out), alloc)
    st.hist[:, :hist0.shape[1]].copy_(torch.from_numpy(hist0), non_blocking=True)
    st.finished.zero_()
    st.lens.copy_(torch.from_numpy(plens), non_blocking=True)
    decode_head(lm, hid_last, st.logits[:B])
    ops.argmax_masked(st.logits[:B], special, st.finished, eos, pad, stop, st.next_ids)
    st.hist.scatter_(1, st.lens[:, None].long(), st.next_ids[:, None])        # the first token ends the history
    st.hist_len.copy_(st.lens).add_(1)
    st.out.fill_(pad)
    st.out[:, 0].copy_(st.next_ids)
    st.n_out.fill_(1)
    st.n_acc.zero_()
    if dec.scores:
        load_scores(st, n_out, B, st.logits.shape[1])
        st.scores[:n_out].fill_(float("-inf"))
        ops.scores_store(st.logits[:B], special, st.scores, st.score_t)       # plane 0: the first token's row
    if n_out == 1:
        st.finished.fill_(1)
    timer.mark()

    def step():
        with ops.pdl():
            ops.lookup_draft(st.hist, st.hist_len, st.finished, special, eos, dec.lookup_ngram, st.drafts, st.win)
            xt = ops.embed_fwd(st.win.view(-1), lm.model.embed_tokens.weight.data)
            h = lm.core.decode_step(xt, st.lens, st.kc, st.vc, window=W)
            decode_head(lm, h, st.logits)
            if dec.scores:
                st.score_prev.copy_(st.n_out)
            ops.lookup_accept(st.logits, special, st.drafts, st.finished, eos, stop, n_out, st.out, st.hist, st.hist_len,
                              st.n_out, st.lens, st.n_acc)
            if dec.scores:
                ops.lookup_scores(st.logits, special, st.score_prev, st.n_out, W, st.scores)

    # every row is done once it emitted EOS or n_out tokens; the device is asked every LOOKUP_CHECK_EVERY steps, and a done
    # row's extra steps emit nothing.  At most n_out - 1 steps: each emits at least one token per unfinished row.
    steps, replays = step_loop(st, step, n_out, lambda: bool(st.finished.all()), LOOKUP_CHECK_EVERY, use_cuda_graph)
    counts = torch.cat([st.n_out, st.n_acc, st.out.flatten()]).cpu()
    n_emit, n_acc, out = counts[:B], counts[B:2 * B], counts[2 * B:].view(B, -1)[:, :n_out]
    timer.finish(pp, steps, replays, st.G, lookup_steps=steps, lookup_tokens=int(n_emit.sum()) - B,
                 lookup_accepted=int(n_acc.sum()))
    new = out.to(torch.int64)
    if stop:
        new = trim_after_eos(new, eos)
    if out_fields is not None:
        out_fields["scores"] = take_scores(st, new.shape[1]) if dec.scores else None
    return torch.cat([input_ids.to(dev), new.to(dev)], dim=1)


def trim_after_eos(new: torch.Tensor, eos: int) -> torch.Tensor:
    """The generated columns [rows, n] without those after the step at which the last row emitted EOS: a loop that asks the
    device only every few tokens whether every row has finished runs a few steps too many, and they only emit pad."""
    if new.shape[1] > 1:
        is_eos = (new == eos)
        if bool(is_eos.any(dim=1).all()):
            last = int(is_eos.float().argmax(dim=1).max())        # first EOS per row; the slowest row decides
            new = new[:, :last + 1]
    return new


# ---- contrastive search (HF GenerationMixin.contrastive_search / _ranking_fast, transformers 4.28) ----
def contrastive_search(lm, input_ids, attention_mask, vis, max_new_tokens, use_cuda_graph, stats, dec: Decoding,
                       out_fields: Optional[dict] = None):
    """Contrastive search (Su et al. 2022) over B prompts with k = ``dec.n`` candidates and alpha = ``dec.penalty_alpha``.  The
    prefill keeps the normalised final-norm row of every prompt position as the prompt's context (``ops.contrastive_context``)
    and the last row's logits.  A step: the processors (``dec.proc``) on the B logits rows, the k most probable tokens
    (``ops.contrastive_topk``), the B * k candidates as one decode step over the prompt caches (each candidate's own key in its
    one-slot cache), their final-norm rows ranked against the context (``ops.contrastive_rank``: the token, the context grows by
    the selected row), the selected candidate's K/V committed to the prompt cache (``ops.contrastive_commit``) and the lm_head
    on its row only.  All on the device and replayed as a CUDA graph; ids, trimming and ``stats`` as in greedy decoding.
    ``dec.scores``: each step first stores the processed logits whose top-k formed its candidates (4.28's
    processed_logit_for_next_step, special ids -inf; ``ops.scores_store``)."""
    k, eos, pad, stop, proc, special = dec.n, dec.eos, dec.pad, dec.stop_on_eos, dec.proc, lm.special_ids_dev
    timer = PhaseTimer(stats)
    pp, st, h_all = prefill(lm, dec, input_ids, attention_mask, vis, max_new_tokens, use_cuda_graph)
    B, H, norm_w, eps = pp.B, lm.dims.n_heads, lm.model.norm.weight.data, lm.dims.rms_eps
    fp8_kv = llama_mod.is_fp8_kv(st.kc)
    if proc is not None:
        load_proc(st, input_ids, B, max_new_tokens)
    st.finished.zero_()
    st.pen_key.zero_()
    st.ctx_len.zero_()
    if dec.scores:
        load_scores(st, max_new_tokens, B, st.logits.shape[1])
    st.lens.copy_(torch.tensor(pp.seqlens, dtype=torch.int32).repeat_interleave(k), non_blocking=True)
    hn_all, _ = ops.rmsnorm_fwd(h_all, norm_w, eps)
    ops.contrastive_context(hn_all, pp.cu, st.ctx, st.ctx_len)

    def head_topk(hn_rows, append=None):
        lm_head_rows(lm, hn_rows, st.logits)
        if proc is not None:
            ops.logits_process_(st.logits, st.proc_ids, st.proc_width, st.proc_hist, st.proc_len, append, proc)
        ops.contrastive_topk(st.logits, special, k, st.cand_p, st.cand_ids)

    head_topk(ops.gather_rows(hn_all, pp.last_rows))

    def step():
        with ops.pdl():
            if dec.scores:
                ops.scores_store(st.logits, special, st.scores, st.score_t)
                ops.add_int_(st.score_t, 1)
            xt = ops.embed_fwd(st.cand_ids.view(-1), lm.model.embed_tokens.weight.data)
            h = lm.core.decode_step(xt, st.lens, st.kc, st.vc, beam=st.beam)
            hn, _ = ops.rmsnorm_fwd(h, norm_w, eps)
            ops.contrastive_rank(hn, st.ctx, st.ctx_len, st.pen_key, st.cand_p, st.cand_ids, dec.penalty_alpha, st.finished, eos,
                                 pad, stop, st.next_ids, st.sel, st.hsel, st.plens, st.lens)
            ops.contrastive_commit(st.commit_table, st.sel, st.plens, k, st.Sp, H, fp8_kv)
            head_topk(st.hsel, append=st.next_ids)

    timer.mark()                                                  # prefill_ms: the prefill and the first candidates
    out_tokens = []
    # every token, the first included, is a candidate step: max_new_tokens steps, timed as decode_ms
    steps, replays = step_loop(st, step, max_new_tokens + 1, (lambda: bool(st.finished.all())) if stop else None, 8,
                               use_cuda_graph, after=lambda: out_tokens.append(st.next_ids.clone()))
    timer.finish(pp, steps, replays, st.Sp, contrastive_steps=steps)
    new = (torch.stack(out_tokens, dim=1).to(torch.int64) if out_tokens else
           torch.zeros((B, 0), dtype=torch.int64, device=lm._device()))
    if stop:
        new = trim_after_eos(new, eos)
    if out_fields is not None:
        out_fields["scores"] = take_scores(st, new.shape[1]) if dec.scores else None
    return torch.cat([input_ids.to(lm._device()), new], dim=1)


# ---- beam search (HF GenerationMixin.beam_search / BeamSearchScorer, transformers 4.28 as the reference pins it) ----
def beam_search(lm, input_ids, attention_mask, vis, max_new_tokens, use_cuda_graph, stats, dec: Decoding, table=None,
                out_fields: Optional[dict] = None):
    """Beam search over B prompts with K = ``dec.n`` beams each.  The prefill runs once per prompt into the prompt cache, whose
    keys the K beams of the prompt share; generated keys live in a [B * K, G] cache that is written once per slot and read
    through the source table ``src`` (reordering the beams gathers ``src``, never K/V).  Each step is ``nv_beam_topk`` (2K
    best candidates per prompt) and ``nv_beam_select`` (the scorer), all on the device, and is replayed as a CUDA graph; the
    hypotheses are finalized on the host after one device-to-host copy.  The visual tokens of prompt b reach all K beams of
    prompt b (the reference's HF expansion of ``cand_vis`` would hand them to other rows' slots).  With logits processors
    (``dec.proc``) the scoring is ``nv_beam_topk_processed`` over the beams' histories (prompt ids, ``hist``).  With the
    flattened trie ``table`` it is ``nv_beam_topk_trie`` (processors or not): each beam walks its own generated tokens from the
    root, and the log-probs its node does not allow become -inf after the processors, as 4.28's PrefixConstrainedLogitsProcessor
    masks log_softmax's output; the trie is loaded as in ``decode``, and one that outgrows the buffers is recaptured.

    Diverse beam search (``dec.groups`` = G > 1, transformers 4.28's group_beam_search): the K beams of a prompt form G groups
    of Kg = K / G, and only the first beam of each group starts with score 0.  The decode step runs over all B * K rows as
    above; then, for g = 0 .. G - 1 in order, ``nv_beam_topk_group`` takes group g's 2Kg best candidates (each log-prob first
    lowered by ``dec.diversity_penalty`` times the count of its token among the tokens groups 0 .. g - 1 chose in this step,
    which their selects have just written to ``next_ids``) and ``nv_beam_select_group`` runs process for the group against the
    prompt's one set of K hypotheses and reorders the group's rows.  All 2G launches are in the captured step.

    ``out_fields`` (return_dict_in_generate) gets ``sequences_scores`` fp32 [B * n], the returned hypotheses' scores from the host
    finalisation.  ``dec.scores`` (and output_scores) adds ``scores``: the top-k kernel of step t writes each beam's processed
    log-probs to plane t (``prompt_state[:, 0]``), one entry per step 4.28 runs (until every prompt is done, not the extra steps
    of the every-8-steps check); and ``beam_indices`` int64 [B * n, L]: ``nv_beam_select_scores`` keeps each beam's rows
    (``par_hist``) and each hypothesis' rows (``hyp_par``), padded with -1."""
    K, eos, pad, proc, special, n_groups = dec.n, dec.eos, dec.pad, dec.proc, lm.special_ids_dev, dec.groups
    if K > BEAM_MAX:
        raise NotImplementedError(f"generate(num_beams={K}): at most {BEAM_MAX} beams are built")
    if max_new_tokens < 1:
        raise ValueError("generate(num_beams > 1) needs max_new_tokens >= 1")
    timer = PhaseTimer(stats)
    pp, st, hid_last = prefill(lm, dec, input_ids, attention_mask, vis, max_new_tokens, use_cuda_graph)
    B, S, G = pp.B, int(input_ids.shape[1]), st.G
    if proc is not None or table is not None:
        load_proc(st, input_ids, 0, G)
    if table is not None:
        trie_csr = load_trie(st, table)
    st.beam_score.view(B, K).fill_(-1e9)[:, ::K // n_groups] = 0.0   # only beam 0 of a prompt (of each group) expands first
    st.hyp_score.zero_()
    st.hyp_score[:, K] = 1e9                                      # BeamHypotheses.worst_score starts at 1e9
    st.hyp_meta.zero_()
    st.pstate.zero_()
    st.pstate[:, 1].copy_(st.plens)
    if dec.scores:
        load_scores(st, max_new_tokens, B * K, st.logits.shape[1])      # step t writes plane t < max_new_tokens
        st.done_step.zero_()
    sc = dict(scores=st.scores, prompt_state=st.pstate) if dec.scores else {}
    trace = (st.par_hist, st.hyp_par, st.done_step) if dec.scores else None
    st.norm.copy_(ops.beam_norm(S, G, dec.length_penalty))
    decode_head(lm, hid_last, st.logits[:B])
    sel = lambda: ops.beam_select(st.cand_score, st.cand_tok, st.cand_par, st.beam_score, st.hist, st.src, st.hyp_score,
                                  st.hyp_meta, st.hyp_tok, st.pstate, st.next_ids, st.lens, st.norm, eos, pad,
                                  dec.early_stopping, trace=trace)

    def group_step(first_step=False):
        for g in range(n_groups):
            ops.beam_topk_group(st.logits, special, st.beam_score, K, n_groups, g, st.cand_score, st.cand_tok, st.cand_par,
                                st.next_ids, dec.diversity_penalty, first_step=first_step, proc=proc, prompt_ids=st.proc_ids
                                if proc is not None else None, prompt_width=st.proc_width if proc is not None else None,
                                hist=st.hist, prompt_state=st.pstate, scores=sc.get("scores"))
            ops.beam_select_group(st.cand_score, st.cand_tok, st.cand_par, st.beam_score, st.hist, st.src, st.hyp_score, st.hyp_meta,
                                  st.hyp_tok, st.pstate, st.next_ids, st.lens, st.norm, eos, pad, dec.early_stopping, n_groups, g,
                                  trace=trace)

    def topk(first_step=False):
        if table is not None:
            ops.beam_topk_trie(st.logits, special, st.beam_score, K, st.cand_score, st.cand_tok, st.cand_par, st.proc_ids,
                               st.proc_width, st.hist, st.pstate, proc, *trie_csr, table.eos, first_step=first_step,
                               scores=sc.get("scores"))
        elif proc is None:
            ops.beam_topk(st.logits, special, st.beam_score, K, st.cand_score, st.cand_tok, st.cand_par, first_step=first_step, **sc)
        else:
            ops.beam_topk_processed(st.logits, special, st.beam_score, K, st.cand_score, st.cand_tok, st.cand_par, st.proc_ids,
                                    st.proc_width, st.hist, st.pstate, proc, first_step=first_step, scores=sc.get("scores"))

    if n_groups > 1:
        group_step(first_step=True)
    else:
        topk(first_step=True)
        sel()
    timer.mark()

    def step():
        with ops.pdl():
            xt = ops.embed_fwd(st.next_ids, lm.model.embed_tokens.weight.data)
            h = lm.core.decode_step(xt, st.lens, st.kc, st.vc, beam=st.beam)
            decode_head(lm, h, st.logits)
            if n_groups > 1:
                group_step()
            else:
                topk()
                sel()

    # like the greedy loop, ask the device whether every prompt is done only every few steps: a done prompt's steps leave
    # its hypotheses unchanged, so the extra steps change no output
    steps, replays = step_loop(st, step, max_new_tokens, lambda: bool(st.pstate[:, 4].all()), 8, use_cuda_graph)
    timer.finish(pp, steps, replays, st.Sp + G, beam_steps=steps + 1)          # beam steps: tokens generated
    # one copy; the fp64 scores go first, so their view starts at an even int32 offset whatever B and K are
    parts = [st.hyp_score.flatten().view(torch.int32), st.hist.flatten(), st.hyp_meta.flatten(), st.hyp_tok.flatten(),
             st.pstate.flatten(), st.beam_score.view(torch.int32)]
    if dec.scores:
        parts += [st.par_hist.flatten(), st.hyp_par.flatten(), st.done_step]
    hyp_score, hist, hyp_meta, hyp_tok, pstate, beam_score, *tr = torch.cat(parts).cpu().split([t.numel() for t in parts])
    hyp_score, beam_score = hyp_score.view(torch.float64).view(B, K + 1), beam_score.view(torch.float32)
    hist, hyp_meta, hyp_tok, pstate = hist.view(B * K, G), hyp_meta.view(B, K, 2), hyp_tok.view(B, K, G), pstate.view(B, 5)
    T_done = int(pstate[0, 0])
    if dec.scores:
        par_hist, hyp_par, done_step = tr[0].view(B * K, G), tr[1].view(B, K, G), tr[2]
    # the beam rows of each hypothesis (beam_indices) ride along as a third element when they are kept
    idx = (lambda rows, n: (rows[:n].tolist(),)) if dec.scores else (lambda rows, n: ())
    hyps, running = [], []
    for b in range(B):
        n = int(pstate[b, 2])
        kept = sorted(range(n), key=lambda i: int(hyp_meta[b, i, 1]))          # insertion order
        hyps.append([(float(hyp_score[b, i]), hyp_tok[b, i, :int(hyp_meta[b, i, 0])].tolist(),
                      *idx(hyp_par[b, i] if dec.scores else None, int(hyp_meta[b, i, 0]) + 1)) for i in kept])
        running.append(None if int(pstate[b, 4]) else
                       [(float(beam_score[b * K + k]), hist[b * K + k, :T_done].tolist(),
                         *idx(par_hist[b * K + k] if dec.scores else None, T_done)) for k in range(K)])
    best = beam_finalize(hyps, [float(hyp_score[b, K]) for b in range(B)], running, S, T_done, K, dec.n_return,
                         dec.length_penalty, entries=True)
    seqs = [[e[1] for e in per] for per in best]
    out = beam_output(input_ids.cpu(), seqs, S, S + max_new_tokens, eos, pad)
    if out_fields is not None:
        out_fields["sequences_scores"] = torch.tensor([e[0] for per in best for e in per], dtype=torch.float32).to(lm._device())
        out_fields["scores"] = out_fields["beam_indices"] = None
        if dec.scores:
            # 4.28 stops once every prompt is done; the device checks every 8 steps, and its extra steps are not 4.28's
            n_steps = int(done_step.max()) if bool(pstate[:, 4].all()) else T_done
            out_fields["scores"] = take_scores(st, n_steps)
            bi = torch.full(out.shape, -1, dtype=torch.int64)
            for i, e in enumerate(e for per in best for e in per):
                bi[i, :len(e[2])] = torch.tensor(e[2], dtype=torch.int64)
            out_fields["beam_indices"] = bi.to(lm._device())
    return out.to(lm._device())


def beam_finalize(hyps, worst, running, S: int, T: int, K: int, n_return: int, length_penalty: float, entries: bool = False):
    """BeamSearchScorer.finalize of transformers 4.28: prompts that are not done add their K running beams (score
    sum_logprobs / (S + T) ** length_penalty, the Python float arithmetic of BeamHypotheses.add), then each prompt returns its
    ``n_return`` best hypotheses, best first; of equal scores the one added last wins (a stable sort, popped from the end).
    hyps[b]: the kept (score, generated tokens) in insertion order; worst[b]: their worst_score; running[b]: the K (running
    score, tokens) of a prompt that is not done, else None.  Returns [[generated tokens] * n_return] per prompt; with ``entries``
    the whole (score, tokens, ...) entries instead (an entry may carry more elements, e.g. its beam rows; they ride along)."""
    out = []
    for b, beams in enumerate(hyps):
        beams, w = list(beams), worst[b]
        for sc, toks, *rest in (running[b] or []):
            score = sc / ((S + T) ** length_penalty)
            if len(beams) < K or score > w:
                beams.append((score, toks, *rest))
                if len(beams) > K:
                    order = sorted([(e[0], i) for i, e in enumerate(beams)])
                    del beams[order[0][1]]
                    w = order[1][0]
                else:
                    w = min(score, w)
        ranked = sorted(beams, key=lambda x: x[0])
        out.append([ranked.pop() if entries else ranked.pop()[1] for _ in range(n_return)])
    return out


def beam_output(prompt_ids: torch.Tensor, seqs, S: int, max_length: int, eos: int, pad: int) -> torch.Tensor:
    """HF ``sequences`` of a beam search: [B * n, L] int64 rows of prompt ids and generated tokens, L = min(longest + 1,
    max_length); a row shorter than L gets EOS after its tokens, then pad."""
    rows = [(b, toks) for b, per in enumerate(seqs) for toks in per]
    L = min(max(S + len(t) for _, t in rows) + 1, max_length)
    out = torch.full((len(rows), L), pad, dtype=torch.int64)
    for i, (b, toks) in enumerate(rows):
        n = S + len(toks)
        out[i, :S] = prompt_ids[b]
        out[i, S:n] = torch.tensor(toks, dtype=torch.int64)
        if n < L:
            out[i, n] = eos
    return out
