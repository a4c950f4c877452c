"""Batch-invariant mode without a GPU: the setter and its environment default, the refusals of the quantized paths, the graph
key, and the split-count rules of the panorama encoder GEMMs as functions of (N, K) alone."""
import dataclasses
from pathlib import Path
from types import SimpleNamespace

import pytest

from navillm_b200 import generation
from navillm_b200.modified_lm import ModifiedLlamaForCausalLM

ROOT = Path(__file__).resolve().parents[1]


def _lm():
    cfg = SimpleNamespace(hidden_size=256, intermediate_size=256, num_hidden_layers=1, num_attention_heads=2, vocab_size=64,
                          rms_norm_eps=1e-6)
    return ModifiedLlamaForCausalLM(cfg, SimpleNamespace(precision="amp_bf16"))


def test_setter_returns_previous_and_defaults_off(monkeypatch):
    monkeypatch.delenv("NAVILLM_BATCH_INVARIANT", raising=False)
    lm = _lm()
    assert lm.batch_invariant is False
    assert lm.set_batch_invariant(True) is False
    assert lm.set_batch_invariant(True) is True
    assert lm.set_batch_invariant(False) is True
    assert lm.batch_invariant is False


def test_environment_sets_the_default(monkeypatch):
    monkeypatch.setenv("NAVILLM_BATCH_INVARIANT", "1")
    assert _lm().batch_invariant is True
    monkeypatch.setenv("NAVILLM_BATCH_INVARIANT", "0")
    assert _lm().batch_invariant is False


def test_refuses_quantized_paths():
    lm = _lm()
    lm.set_batch_invariant(True)
    with pytest.raises(ValueError, match="batch-invariant"):
        lm.quantize_weights_fp8()
    with pytest.raises(ValueError, match="batch-invariant"):
        lm.quantize_weights_int4()
    with pytest.raises(ValueError, match="batch-invariant"):
        lm.set_activation_dtype("fp8")
    assert lm.activation_dtype == "bf16"
    lm.set_batch_invariant(False)
    lm.set_activation_dtype("fp8")
    with pytest.raises(ValueError, match="batch-invariant mode does not combine with fp8 activations"):
        lm.set_batch_invariant(True)
    assert lm.batch_invariant is False
    lm.__dict__["_fp8"] = object()                  # a weight copy present (built on the GPU in practice)
    lm.set_activation_dtype("bf16")
    with pytest.raises(ValueError, match="fp8 weight copy"):
        lm.set_batch_invariant(True)
    lm.__dict__["_fp8"], lm.__dict__["_int4"] = None, object()
    with pytest.raises(ValueError, match="int4 weight copy"):
        lm.set_batch_invariant(True)


def test_graph_key_separates_the_modes():
    dec = generation.Decoding(2, 0, True, "greedy", "bf16")
    inv = dataclasses.replace(dec, batch_invariant=True)
    assert dec.key() != inv.key()
    assert dec.key()[-1] == inv.key()[-1] == "bf16"             # the format stays last


@pytest.mark.parametrize("N,K", [(768, 768), (3072, 768), (768, 3072), (768, 640), (2048, 4096), (768, 7)])
def test_fixed_split_counts_depend_on_k_alone(N, K):
    """With nv_set_fixed_splits on, the loops of nv_sgemm and nv_gemm_tf32 give one split count for every tile count (the
    number of views) and every SM count."""
    pano = (ROOT / "navillm_b200/csrc/pano_ops.cu").read_text()
    tf32 = (ROOT / "navillm_b200/csrc/gemm_tf32.cu").read_text()
    assert "(g_fixed_splits || tiles * splits < 3 * sm_count())" in pano
    assert "(g_fixed_splits || tiles * splits * 2 <= 2u * (uint32_t)sm_count())" in tf32

    def sgemm_splits(tiles, sms, fixed):
        s = 1
        while s < 8 and (fixed or tiles * s < 3 * sms) and K // (s * 2) >= 256:
            s *= 2
        return s

    def tf32_splits(tiles, sms, fixed):
        kb = (K + 31) // 32
        s = 1
        while s < 8 and (fixed or tiles * s * 2 <= 2 * sms) and kb // (s * 2) >= 8:
            s *= 2
        return s

    for rule in (sgemm_splits, tf32_splits):
        got = {rule(tiles, sms, True) for tiles in (1, 3, 17, 80, 400, 5000) for sms in (66, 114, 132)}
        assert len(got) == 1, (rule.__name__, got)
        # off: the count follows the batch (the reason for the switch)
        if K >= 1024:
            assert rule(1, 132, False) != rule(5000, 132, False)


def test_invariant_predicate_follows_training():
    """One predicate decides positions, heads, prefix offsets and encoder splits: the mode is on and the call does not
    train (grad enabled with training enabled)."""
    import torch
    lm = _lm()
    assert lm.invariant_inference() is False
    lm.set_batch_invariant(True)
    with torch.no_grad():
        assert lm.invariant_inference() is True
    with torch.enable_grad():
        assert lm.invariant_inference() is False
        lm.training_enabled = False
        assert lm.invariant_inference() is True


@pytest.mark.parametrize("invariant", [False, True])
def test_prefix_plan_offsets(invariant):
    """A prefix-cached row's rotary offset: the reference's left padding S - L, or 0 in batch-invariant mode (then a row's
    positions do not follow the longest prompt of its batch)."""
    import numpy as np
    from navillm_b200.modified_lm import plan_prefix_reuse
    from tests.test_host_logic_cpu import _left_pad
    CAND, HIST, CLS = 900, 901, 902
    cache = SimpleNamespace(B=2, max_len=64, ids=[np.zeros(0, dtype=np.int64) for _ in range(2)], off=[None, None])
    rows = [[1, 5, 6, 7, 20, 21, 40, CAND, 22, CLS], [1, 9, 20, 21, 40, CAND, 41, CAND, 22, CLS, 3, 4]]
    ids, msk = _left_pad(rows)
    tok, pos, vis, ql, cached, kvl, cls = plan_prefix_reuse(ids, msk, cache, [0, 0], 3, CAND, HIST, CLS, invariant=invariant)
    S = ids.shape[1]
    want = [0, 0] if invariant else [S - len(rows[0]), S - len(rows[1])]
    assert cache.off == want
    assert pos[0].tolist() == list(range(want[0], want[0] + len(rows[0])))
