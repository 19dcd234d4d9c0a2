"""CPU tests: the oracle (oracle/magma_oracle.py) reproduces the outputs of the REFERENCE ITSELF.

The fixtures in tests/golden/ were produced by oracle/make_golden.py, which runs the reference's own Python
(imported from a reference checkout under shims) with HF GPT-J / HF CLIP-ViT as the third-party arithmetic. fp32 on both
sides, so tolerances are tight; integer results (labels, greedy token ids, filters' -inf pattern) must be identical.
"""
import os

import numpy as np
import pytest
import torch

from oracle import magma_oracle as O
from conftest import oracle_cfg_from_record

VARIANTS = ["v1_mlp_normal", "v2_mlp_attn_normal", "parallel", "no_adapters"]


def _load(golden_dir, name):
    return torch.load(os.path.join(golden_dir, name), map_location="cpu", weights_only=False)


def test_adapter_matches_reference(golden_dir):
    rec = _load(golden_dir, "adapter.pt")
    w = {"a." + k: v for k, v in rec["weights"].items()}
    y = O.adapter_forward(rec["x"], w, "a")
    torch.testing.assert_close(y, rec["y"], rtol=1e-5, atol=1e-6)


def test_build_labels_bit_exact(golden_dir):
    rec = _load(golden_dir, "build_labels.pt")
    for case in rec["cases"]:
        got = O.build_labels(case["L"], case["captions"].numpy(), rec["eos"])
        assert got.dtype == np.int64
        assert np.array_equal(got, case["labels"].numpy()), f"L={case['L']}"


def test_build_labels_edge_cases():
    eos = 9
    # no eos at all, eos first, prefix == seq (every label masked), empty prefix
    caps = np.array([[1, 2, 3, 4], [9, 1, 2, 3], [1, 9, 9, 2]], dtype=np.int64)
    assert O.build_labels(0, caps, eos).shape == (3, 0)  # reference quirk: captions[:, :-0] is empty
    assert np.array_equal(O.build_labels(1, caps, eos), [[-100, 1, 2, 3], [-100, 9, -100, -100], [-100, 1, 9, -100]])
    assert np.array_equal(O.build_labels(4, caps, eos), np.full((3, 4), -100))
    assert np.array_equal(O.build_labels(2, caps, eos), [[-100, -100, 1, 2], [-100, -100, 9, -100], [-100, -100, 1, 9]])
    with pytest.raises(AssertionError):
        O.build_labels(5, caps, eos)  # prefix longer than the sequence: reference asserts (utils.py:349)


def test_sampling_filters_match_reference(golden_dir):
    rec = _load(golden_dir, "sampling_filters.pt")
    assert torch.equal(O.top_k_filter(rec["logits"].clone(), 5), rec["top_k_5"])
    assert torch.equal(O.top_p_filter(rec["logits"].clone(), 0.9), rec["top_p_0.9"])
    assert torch.equal(O.top_p_filter(rec["logits"].clone(), 0.5), rec["top_p_0.5"])
    # the inverted-nucleus behaviour of sampling.py:7-19 is part of the contract
    q5 = O.top_p_filter(rec["quirk_probs"].clone(), 0.5)
    assert torch.equal(q5, rec["quirk_0.5"]) and torch.isinf(q5[0, 1]) and not torch.isinf(q5[0, 0])
    assert torch.equal(O.top_p_filter(rec["quirk_probs"].clone(), 0.9), rec["quirk_0.9"])


@pytest.mark.parametrize("tag", VARIANTS)
def test_magma_forward_backward_matches_reference(golden_dir, tag):
    rec = _load(golden_dir, f"magma_{tag}.pt")
    cfg = oracle_cfg_from_record(rec)
    trainable = set(rec["grads"].keys())
    w = {k: v.clone().requires_grad_(k in trainable) for k, v in rec["weights"].items()}
    loss, logits, labels = O.magma_forward(rec["images"], rec["captions"], w, cfg)
    torch.testing.assert_close(loss.detach(), rec["loss"], rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(logits.detach(), rec["logits"], rtol=1e-3, atol=1e-4)
    loss.backward()
    for k, gref in rec["grads"].items():
        torch.testing.assert_close(w[k].grad, gref, rtol=2e-3, atol=1e-6, msg=lambda m, k=k: f"{k}: {m}")


def test_vit_embed_and_greedy_generate_match_reference(golden_dir):
    rec = _load(golden_dir, "magma_v1_mlp_normal.pt")
    cfg = oracle_cfg_from_record(rec)
    w = rec["weights"]
    with torch.no_grad():
        feats = O.vit_forward(rec["images"], w, cfg)
        torch.testing.assert_close(feats, rec["enc_feats"], rtol=1e-3, atol=1e-5)
        emb = O.magma_embed([rec["images"], rec["text"]], w, cfg)
        torch.testing.assert_close(emb, rec["embeddings"], rtol=1e-3, atol=1e-5)
        toks = O.generate_greedy(rec["embeddings"], w, cfg, max_steps=10)
    assert torch.equal(toks, rec["greedy_tokens"])  # token ids are integers: exact


def test_remove_tokens_after_eos():
    t = torch.tensor([255, 255, 5, 6, 254, 7, 8])
    assert O.remove_tokens_after_eos(t, 254, 255) == [5, 6]
    assert O.remove_tokens_after_eos(torch.tensor([1, 2, 3]), 254, 255) == [1, 2, 3]
