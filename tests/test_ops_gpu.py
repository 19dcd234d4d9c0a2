"""GPU parity tests of the HBM-bound operators (layernorm, rotary, softmax, cross-entropy, build_labels, embedding
assembly, reductions, argmax, fused AdamW) through the C ABI against torch-fp32 / the oracle. Integer results are
compared bit-exactly."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def test_ops_group():
    import torch

    from tools import model_check

    assert model_check.group_ops(torch.device("cuda:0"))


def test_build_labels_golden_and_edges(golden_dir):
    """CUDA build_labels vs the fixtures produced by the reference's own build_labels (magma/utils.py:334-364)."""
    import os

    import torch

    from magma_b200.utils import build_labels
    from oracle import magma_oracle as O

    dev = torch.device("cuda:0")
    rec = torch.load(os.path.join(golden_dir, "build_labels.pt"), weights_only=False)
    for case in rec["cases"]:
        emb = torch.zeros(case["captions"].shape[0], case["L"], 8, device=dev)
        got = build_labels(emb, case["captions"].to(dev), rec["eos"], dev)
        assert got.dtype == torch.int64 and torch.equal(got.cpu(), case["labels"]), f"L={case['L']}"
    # full-size shapes (B=8, S=2048 — the reference's literal seq_len), random eos placement, property checks
    g = torch.Generator().manual_seed(0)
    caps = torch.randint(0, 50257, (8, 2048), generator=g)
    caps[3, 100:] = 50256
    for L in (2, 144):
        got = build_labels(torch.zeros(8, L, 4, device=dev), caps.to(dev), 50256, dev).cpu().numpy()
        want = O.build_labels(L, caps.numpy(), 50256)
        assert np.array_equal(got, want)
        assert (got[:, :L] == -100).all()
    with pytest.raises(AssertionError):
        build_labels(torch.zeros(8, 3000, 4, device=dev), caps.to(dev), 50256, dev)


def test_adapter_standalone_matches_golden(golden_dir):
    """magma_b200.adapters.Adapter (fused GEMM epilogues) vs the reference Adapter's own output."""
    import os

    import torch

    from magma_b200.adapters import Adapter

    dev = torch.device("cuda:0")
    rec = torch.load(os.path.join(golden_dir, "adapter.pt"), weights_only=False)
    ad = Adapter(64, 4).to(dev)
    ad.load_state_dict(rec["weights"])
    x = rec["x"].to(dev).requires_grad_(True)
    y = ad(x)
    rel = ((y.float().cpu() - rec["y"]).norm() / rec["y"].norm()).item()
    assert rel < 2e-2, rel
    # backward against autograd of the fp32 restatement
    from oracle import magma_oracle as O

    w = {"a." + k: v.clone().requires_grad_(True) for k, v in rec["weights"].items()}
    xo = rec["x"].clone().requires_grad_(True)
    go = torch.randn(3, 5, 64, generator=torch.Generator().manual_seed(1))
    O.adapter_forward(xo, w, "a").backward(go)
    y.backward(go.to(dev))
    assert ((x.grad.cpu() - xo.grad).norm() / xo.grad.norm()).item() < 1e-1  # relu mask decided near 0
    gup = ad.adapter[2].weight.grad.cpu()
    assert ((gup - w["a.adapter.2.weight"].grad).norm() / w["a.adapter.2.weight"].grad.norm()).item() < 3e-2


def test_sumsq_is_bit_identical_for_any_grid():
    """mb200_sumsq (the clipping norm): B200Engine caps the optimizer kernels' grids when the optimizer runs beside the
    next step's GEMMs; the result must not depend on the grid (data-parallel replicas / pipelined vs in-stream optimizer
    stay bit-identical) and must equal the fp64 sum to fp32 accuracy."""
    import torch

    from magma_b200 import ops
    from magma_b200._lib import lib

    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(0)
    x = torch.randn(241_332_224 // 8 + 4 * 3 + 1, generator=g).to(dev)
    outs = []
    try:
        for cap in (0, 296, 148, 7):
            lib().mb200_set_optimizer_grid(cap)
            for view in (x[:-1], x[1:]):       # 16-byte aligned / not
                o = torch.zeros(1, device=dev)
                ops.sumsq(view, o)
                outs.append((cap, float(o), float((view.double() ** 2).sum())))
    finally:
        lib().mb200_set_optimizer_grid(0)
    for cap, got, want in outs:
        assert abs(got - want) < 2e-5 * want, (cap, got, want)
    assert len({o[1] for o in outs[0::2]}) == 1 and len({o[1] for o in outs[1::2]}) == 1, outs
