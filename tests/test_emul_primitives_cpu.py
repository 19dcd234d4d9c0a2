"""The CPU emulation of the primitive operators (oracle/cabi_emul.cpp) is itself held to independent torch formulas:
every dry run in this suite is only as good as the emulation of mb200_gemm, so its operand majors, batch strides and the
whole epilogue (bias, activations, saved pre-activation, derivative multipliers, residuals, fp32 accumulate, rotary
embedding) are checked here on small shapes; the elementwise / reduction operators replay the same `group_ops` harness
the real kernels are held to on the GPU (tests/test_ops_gpu.py)."""
import pytest
import torch
import torch.nn.functional as F


def rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-12)).item()


def mk(g, *shape, scale=1.0):
    return (torch.randn(*shape, generator=g) * scale).to(torch.bfloat16)


@pytest.mark.parametrize("a_mn", [False, True])
@pytest.mark.parametrize("b_mn", [False, True])
def test_gemm_operand_majors_and_ragged_shapes(emul_ops, a_mn, b_mn):
    from magma_b200 import ops

    g = torch.Generator().manual_seed(0)
    M, N, K = 37, 24, 56                                  # ragged M; N, K multiples of 8 (leading dimensions)
    A = mk(g, K, 40) if a_mn else mk(g, M, K)             # [K, M(ld 40)] or [M, K]
    B = mk(g, K, N) if b_mn else mk(g, N, K)
    Av = A[:, :M] if a_mn else A
    want = (Av.float().t() if a_mn else Av.float()) @ (B.float() if b_mn else B.float().t())
    got = ops.gemm(Av, B, a_mn=a_mn, b_mn=b_mn)
    assert got.shape == (M, N) and rel(got, want) < 5e-3
    got32 = ops.gemm(Av, B, a_mn=a_mn, b_mn=b_mn, out_dtype=torch.float32, alpha=0.5)
    assert got32.dtype == torch.float32 and rel(got32, 0.5 * want) < 1e-5


def test_gemm_epilogue_options(emul_ops):
    from magma_b200 import ops

    g = torch.Generator().manual_seed(1)
    M, N, K = 16, 32, 24
    A, B = mk(g, M, K), mk(g, N, K)
    bias, r1, r2 = mk(g, N), mk(g, M, N), mk(g, M, N)
    acc = A.float() @ B.float().t() + bias.float()
    gelu_new = lambda x: 0.5 * x * (1 + torch.tanh(0.7978845608028654 * (x + 0.044715 * x ** 3)))  # noqa: E731
    # bias + activation, pre-activation saved
    aux = torch.empty(M, N, dtype=torch.bfloat16)
    y = ops.gemm(A, B, bias=bias, act=ops.ACT_GELU_NEW, aux_out=aux)
    assert rel(aux, acc) < 5e-3 and rel(y, gelu_new(acc)) < 5e-3
    assert rel(ops.gemm(A, B, bias=bias, act=ops.ACT_QUICK_GELU), acc * torch.sigmoid(1.702 * acc)) < 5e-3
    assert rel(ops.gemm(A, B, bias=bias, act=ops.ACT_RELU), F.relu(acc)) < 5e-3
    # residuals, and ReLU applied AFTER them
    assert rel(ops.gemm(A, B, bias=bias, res1=r1, res2=r2), acc + r1.float() + r2.float()) < 5e-3
    assert rel(ops.gemm(A, B, bias=bias, res1=r1, act=ops.ACT_RELU_POST), F.relu(acc + r1.float())) < 5e-3
    # derivative multipliers (backward epilogues)
    pre = mk(g, M, N)
    x = pre.float().requires_grad_(True)
    gelu_new(x).sum().backward()
    assert rel(ops.gemm(A, B, aux_in=pre, dact=ops.DACT_GELU_NEW), (A.float() @ B.float().t()) * x.grad) < 5e-3
    assert rel(ops.gemm(A, B, aux_in=pre, dact=ops.DACT_RELU), (A.float() @ B.float().t()) * (pre.float() > 0)) < 5e-3
    # fp32 accumulate
    out = torch.full((M, N), 2.0)
    ops.gemm(A, B, out=out, accumulate=True)
    assert rel(out, 2.0 + A.float() @ B.float().t()) < 1e-5


def test_gemm_batched_strides_address_heads_inside_a_fused_qkv_buffer(emul_ops):
    """The attention GEMMs read Q / K / V of head h straight from the fused [B*S, 3*H*hd] buffer through batch strides
    (hd, S*3d) and write O as [B, S, H, hd]: scores = Q K^T per (b, h), O = P V with V as an MN-major operand."""
    from magma_b200 import ops

    g = torch.Generator().manual_seed(2)
    Bb, S, H, hd = 2, 9, 3, 16
    d = H * hd
    qkv = mk(g, Bb * S, 3 * d)
    q4 = qkv.view(Bb, S, 3, H, hd)
    Q = q4[:, :, 0].permute(0, 2, 1, 3)       # [B, H, S, hd] strided views of the same memory
    K = q4[:, :, 1].permute(0, 2, 1, 3)
    V = q4[:, :, 2].permute(0, 2, 1, 3)
    ldS = 16
    scores = torch.zeros(Bb, H, S, ldS)
    ops.gemm(Q, K, out=scores[..., :S])
    want = Q.float() @ K.float().transpose(-1, -2)
    assert rel(scores[..., :S], want) < 1e-5
    P = torch.softmax(want, -1).to(torch.bfloat16)
    Pp = torch.zeros(Bb, H, S, ldS, dtype=torch.bfloat16)
    Pp[..., :S] = P
    O = torch.empty(Bb, S, H, hd, dtype=torch.bfloat16)
    ops.gemm(Pp[..., :S], V, b_mn=True, out=O.permute(0, 2, 1, 3))
    assert rel(O.permute(0, 2, 1, 3), P.float() @ V.float()) < 5e-3


def test_gemm_rotary_epilogue_equals_the_rope_kernel_and_inverts(emul_ops):
    from magma_b200 import ops

    g = torch.Generator().manual_seed(3)
    Bb, S, H, hd, rot = 2, 5, 2, 16, 8
    d = H * hd
    x, W = mk(g, Bb * S, 24), mk(g, 3 * d, 24)
    tab = ops.rope_table(S, rot, 0, device=torch.device("cpu"))
    fused = ops.gemm(x, W, rope_tab=tab, rope_mode=1, rope_S=S, rope_hd=hd, rope_rot=rot, rope_ncols=2 * d)
    plain = ops.gemm(x, W, out_dtype=torch.float32).to(torch.bfloat16)
    ops.rope_(plain, S, H, hd, rot)           # the standalone kernel's semantics: q and k rotated, v untouched
    assert rel(fused, plain) < 8e-3
    # rotate_every_two against the HF formula (modeling_gptj.py:57-67) on q of head 0
    from oracle import magma_oracle as O

    sin, cos = O.rope_tables(torch.arange(S), rot)
    q0 = ops.gemm(x, W, out_dtype=torch.float32).view(Bb, S, 3, H, hd)[:, :, 0, 0]
    want = O.apply_rope(q0[:, :, None, :], sin, cos, rot)[:, :, 0]
    assert rel(fused.view(Bb, S, 3, H, hd)[:, :, 0, 0], want) < 8e-3


def test_elementwise_harness_of_the_gpu_suite_replays_on_the_emulation(emul_ops, monkeypatch, capsys):
    from tools import model_check

    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    assert model_check.group_ops(torch.device("cpu"))
    assert "[FAIL]" not in capsys.readouterr().out
