"""The launch records of the production passes (tools/plan_trace.py, written by the CPU emulation in trace mode) and the
checker tests/test_production_launches_gpu.py holds each distinct configuration to.

- Every record is complete: its op's full argument set, every pointer resolved to a region of the traced pass.
- The number of distinct launch configurations per pass is pinned: a schedule change that adds or removes one updates
  the pin on purpose, and the GPU file, which derives its cases from the same records, follows it. Every non-GEMM
  configuration has a replay there, and the ones too large for their float64 checker are pinned by name.
- The element-wise checker fails on a doctored result: one element one bf16 rounding past its bound, one row block
  shifted by a row.
- The cheap GEMM configurations (M <= 32) and the decode attention configurations are replayed on the CPU emulation of
  the operators by the GPU file's bodies.
"""
import math
import os
import sys

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tools"))
import plan_trace  # noqa: E402

# distinct launch configurations (op, scalars, alignment class, aliasing) of each production pass
PINNED = {
    "config2_train": 37,
    "gptj_recompute_train_S2048": 29,
    "magma_v2_train": 25,
    "vit_train": 38,
    "prefill_S2048": 12,
    "decode_pos136": 10,
    "decode_last": 10,
}

# mb200_gemm_args as recorded: every scalar of the call, every pointer as [region, byte offset]
GEMM_FIELDS = {"op", "M", "N", "K", "nb0", "nb1", "A", "a_ld", "a_bs0", "a_bs1", "a_mn", "B", "b_ld", "b_bs0", "b_bs1",
               "b_mn", "b_static", "c_dtype", "C", "ldc", "c_bs0", "c_bs1", "alpha", "act", "dact", "accumulate", "bias",
               "aux_out", "aux_in", "res1", "res2", "ld_res", "force_bn", "generic_epilogue", "rope_mode", "rope_tab",
               "rope_S", "rope_hd", "rope_rot", "rope_ncols", "splitk_ws", "splitk_ws_bytes"}
# pointers a launch of the op cannot do without
REQUIRED = {"gemm": ("A", "B", "C"), "layernorm_fwd": ("x", "gamma", "beta", "y"), "softmax_bwd": ("dp", "p", "ds"),
            "cross_entropy": ("logits", "labels", "loss"), "attn_fwd_flash": ("q", "k", "v", "O"),
            "attn_decode": ("qkv", "kc", "vc", "out"), "kv_append": ("qkv", "kc", "vc"), "colsum": ("x", "out")}


@pytest.fixture(scope="module")
def records():
    return {name: plan_trace.pass_records(name) for name in plan_trace.PASSES}


def test_records_are_complete(records):
    for name, (rows, recs) in records.items():
        assert len(recs) == len(rows), f"{name}: {len(recs)} records for {len(rows)} traced launches"
        fields = {}
        for r in recs:
            assert fields.setdefault(r["op"], set(r)) == set(r), f"{name}: {r['op']} records differ in their fields"
            for k in plan_trace.POINTERS[r["op"]]:
                p = r[k]
                assert p is None or (isinstance(p[0], str) and p[1] >= 0), f"{name}: {r['op']}.{k} = {p}"
            for k in REQUIRED.get(r["op"], ()):
                assert r[k] is not None, f"{name}: {r['op']} without {k}"
            assert all(isinstance(v, (int, float)) for k, v in r.items() if k != "op" and k not in plan_trace.POINTERS[r["op"]])
        assert fields["gemm"] == GEMM_FIELDS


def test_distinct_configurations_are_pinned(records):
    counts = {name: len(plan_trace.distinct_configs(recs)) for name, (rows, recs) in records.items()}
    for name, n in counts.items():
        print(f"[configs] {name}: {n} distinct launch configurations of {len(records[name][1])} launches")
    assert counts == PINNED


def test_records_show_the_production_risks(records):
    """The launches the element-wise GEMM tests had no shape for: K % 8 != 0, 2^31-byte batched outputs, in place."""
    recs = [r for _, rs in records.values() for r in rs]
    gemm = [r for r in recs if r["op"] == "gemm"]
    assert any(r["K"] == 50258 and r["M"] == 16384 and r["b_mn"] for r in gemm)  # LM-head dgrad, S = 2048
    assert any(r["K"] == 588 and r["a_ld"] == 592 for r in gemm)  # ViT-L/14 patch embedding
    assert any(r["nb0"] * r["nb1"] == 128 and r["M"] == r["N"] == 2048 and r["c_dtype"] == 1 for r in gemm)
    assert any(r["M"] <= 32 and r["splitk_ws_bytes"] > 0 for r in gemm)  # decode: the split-K plans
    assert any(r["res1"] == r["C"] for r in gemm)  # the residual added in place
    ce = [r for r in recs if r["op"] == "cross_entropy"]
    assert {(r["B"] * r["S"], r["V"], r["ldv"]) for r in ce} >= {(16384, 50258, 50304), (1024, 50258, 50304)}


def test_aliasing_and_alignment_separate_configurations():
    base = {"op": "colsum", "x": ["workspace", 4096], "ldx": 64, "rows": 8, "cols": 64, "out": ["g", 0], "accumulate": 0}
    moved = dict(base, x=["workspace", 4096 + 16])
    aliased = dict(base, out=["workspace", 4096])
    other_region = dict(base, x=["x", 4096])
    keys = {plan_trace.config_key(r) for r in (base, moved, aliased)}
    assert len(keys) == 3
    assert plan_trace.config_key(other_region) == plan_trace.config_key(base)


# non-GEMM configurations whose float64 checker holds whole >= 2 GiB tensors several times over: not replayed on the GPU
TOO_LARGE = {
    "cross_entropy B=8 S=2048 V=50258 ldv=50304",
    "attn_fwd_flash B=8 Sq=2048 Sk=2048 H=16 hd=256 causal=1",
    "softmax_bwd nz=128 Sq=2048 Sk=2048",
}


def test_every_other_configuration_has_a_replay():
    import test_production_launches_gpu as P

    large = set()
    for cid, r, passes in P.OTHERS:
        assert callable(P.other_replay(r)), cid
        if P.too_large(r):
            large.add(_short(r))
    assert large == TOO_LARGE


def _short(r):
    keys = dict(cross_entropy=("B", "S", "V", "ldv"), attn_fwd_flash=("B", "Sq", "Sk", "H", "hd", "causal"),
                softmax_bwd=("nz", "Sq", "Sk"))[r["op"]]
    return r["op"] + " " + " ".join(f"{k}={r[k]}" for k in keys)


def _doctor_case():
    import torch

    from test_gemm_reference_gpu import _reference

    from _refcheck import bf16_rne, ulp_bf16

    gen = torch.Generator().manual_seed(3)
    M, N, K = 256, 96, 520
    A = torch.randn(M, K, generator=gen, dtype=torch.float64).to(torch.bfloat16)
    B = (torch.randn(N, K, generator=gen, dtype=torch.float64) / math.sqrt(K)).to(torch.bfloat16)
    ref, pre, bound, amb = _reference(A, B, alpha=1.0, bias=None, act=0, dact=0, aux_in=None, res1=None, res2=None,
                                      rope=None, c_old=None)
    return ref, bound, bf16_rne(ref), ulp_bf16


def test_checker_fails_one_rounding_past_the_bound():
    from test_gemm_reference_gpu import _check

    ref, bound, good, ulp_bf16 = _doctor_case()
    _check("exact rounding", good, ref, bound, False)
    bad = good.clone()
    i, j = 100, 37
    limit = ref[i, j] + ulp_bf16(ref[i, j]) + bound[i, j]  # the largest error the bound allows
    v = good[i, j]
    while v <= limit:  # walk up the bf16 grid to the first value past the bound
        v = v + ulp_bf16(v)
    bad[i, j] = v
    with pytest.raises(pytest.fail.Exception, match=r"1 of .* outside the bound; worst at \(100, 37\)"):
        _check("one element past its bound", bad, ref, bound, False)
    bad[i, j] = v - ulp_bf16(v)  # one rounding back: inside
    _check("one element at its bound", bad, ref, bound, False)


def test_checker_fails_a_shifted_row_block():
    from test_gemm_reference_gpu import _check

    ref, bound, good, _ = _doctor_case()
    bad = good.clone()
    bad[128:192] = good[129:193]  # one 64-row block of a 128-row tile written one row off
    with pytest.raises(pytest.fail.Exception, match="outside the bound"):
        _check("row block shifted", bad, ref, bound, False)


def _cheap_gemms():
    import test_production_launches_gpu as P

    return [c for c in P.CONFIGS if c[1]["M"] <= 32]


def _decode_attention():
    import test_production_launches_gpu as P

    return [c for c in P.OTHERS if c[1]["op"] == "attn_decode"]


@pytest.mark.parametrize("cid,rec,passes", _decode_attention(), ids=[c[0] for c in _decode_attention()])
def test_decode_attention_on_emulation(emul_ops, monkeypatch, cid, rec, passes):
    import test_production_launches_gpu as P

    monkeypatch.setenv("MB200_TEST_DEVICE", "cpu")
    P.other_replay(rec)()


@pytest.mark.parametrize("cid,rec,passes", _cheap_gemms(), ids=[c[0] for c in _cheap_gemms()])
def test_cheap_configurations_on_emulation(emul_ops, monkeypatch, cid, rec, passes):
    import test_production_launches_gpu as P

    monkeypatch.setenv("MB200_TEST_DEVICE", "cpu")
    P.replay_gemm(cid, rec, passes)
