"""CPU replay of the tile, epilogue and batch test bodies of tests/test_gemm_reference_gpu.py on the emulated operator
(oracle/cabi_emul.cpp::mb200_gemm) at small sizes: keeps the float64 reference, the element-wise bound and the sentinel
and input checks honest without a GPU; the kernel itself is verified by the `-m gpu` run only. The emulation counts no
launches and has no split-K plans, so the split-K and SM-limit bodies are GPU-only. Also holds ops.gemm's layout
validation of the epilogue tensors, which no C ABI can check on raw pointers."""
import pytest

import test_gemm_reference_gpu as G


@pytest.mark.parametrize("shape", [(65, 203, 40), (127, 45, 8), (129, 67, 72), (33, 45, 12), (20, 37, 588)],
                         ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, False), (True, True)],
                         ids=["KK", "KMN", "MNK", "MNMN"])
def test_tiles_and_majors_body_on_emulation(emul_ops, monkeypatch, a_mn, b_mn, shape):
    monkeypatch.setenv("MB200_TEST_DEVICE", "cpu")
    G.test_tiles_and_majors(64, a_mn, b_mn, shape)


@pytest.mark.parametrize("form", list(G.EPILOGUES))
def test_epilogue_forms_body_on_emulation(emul_ops, monkeypatch, form):
    monkeypatch.setenv("MB200_TEST_DEVICE", "cpu")
    G.test_epilogue_forms(64, form, shape=(70, 203, 40))


@pytest.mark.parametrize("form", list(G.BATCH_FORMS))
def test_batched_body_on_emulation(emul_ops, monkeypatch, form):
    monkeypatch.setenv("MB200_TEST_DEVICE", "cpu")
    G.test_batched(True, True, form, shape=(33, 45, 24))


def test_batched_attention_style_output_body_on_emulation(emul_ops, monkeypatch):
    monkeypatch.setenv("MB200_TEST_DEVICE", "cpu")
    G.test_batched_attention_style_output(64, S=20, H=2, hd=16, Sk=24)


def test_ops_gemm_rejects_misshaped_epilogue_tensors(emul_ops):
    import torch

    from magma_b200 import ops

    bf = torch.bfloat16
    M, N, K = 16, 24, 32
    A, B = torch.zeros(M, K, dtype=bf), torch.zeros(N, K, dtype=bf)
    mn = torch.zeros(M, N, dtype=bf)
    ops.gemm(A, B, bias=torch.zeros(N, dtype=bf), res1=mn, res2=mn, aux_out=mn.clone())  # the valid layout runs
    for bad in (torch.zeros(N + 8, dtype=bf), torch.zeros(2 * N, dtype=bf)[::2], torch.zeros(1, N, dtype=bf)):
        with pytest.raises(ValueError, match="bias"):
            ops.gemm(A, B, bias=bad)
    small = torch.zeros(M - 1, N, dtype=bf)
    for name in ("aux_out", "aux_in", "res1", "res2"):
        kw = {name: small}
        if name == "aux_in":
            kw["dact"] = ops.DACT_RELU
        with pytest.raises(ValueError, match=name):
            ops.gemm(A, B, **kw)
    # batched: out [2, 3, M, N]; residuals may change the row stride but not the batch dims or batch strides
    Ab, Bb = torch.zeros(2, 3, M, K, dtype=bf), torch.zeros(2, 3, N, K, dtype=bf)
    out = torch.zeros(2, 3, M, N, dtype=bf)
    wide = torch.zeros(2, 3, M, N + 8, dtype=bf)  # row stride N + 8: batch strides differ from out's
    with pytest.raises(ValueError, match="res1"):
        ops.gemm(Ab, Bb, out=out, res1=wide[..., :N])
    same_batch = torch.zeros(6 * M * N + 128, dtype=bf).as_strided((2, 3, M, N), (3 * M * N, M * N, N + 8, 1))
    ops.gemm(Ab, Bb, out=out, res1=same_batch)  # only the row stride differs
    ops.gemm(Ab, Bb, out=out, res1=torch.zeros(2, 3, M, N, dtype=bf), res2=torch.zeros(2, 3, M, N, dtype=bf))
    with pytest.raises(ValueError, match="res2"):
        ops.gemm(Ab, Bb, out=out, res2=torch.zeros(3, 2, M, N, dtype=bf).transpose(0, 1))
    with pytest.raises(ValueError, match="res1"):
        ops.gemm(Ab, Bb, out=out, res1=torch.zeros(3, M, N, dtype=bf))
    with pytest.raises(ValueError, match="aux_out"):
        ops.gemm(Ab, Bb, out=out, aux_out=torch.zeros(2, 3, M, N + 8, dtype=bf)[..., :N])
