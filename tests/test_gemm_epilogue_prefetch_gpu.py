"""The GEMM epilogue reads its [M, N] inputs (aux_in, res1, res2) one of two ways: staged into shared memory by TMA
through the operand ring, when every such input has a 16-byte-aligned base and row and batch strides that are multiples
of 8 elements, or loaded from global memory by the epilogue threads otherwise. Both must give the same bits.

Each case runs once on inputs at 16-byte-aligned addresses (TMA path) and once on the same values stored one element
past a 16-byte boundary (register path); out and aux_out must be bit-identical, and each call one launch. Unused storage
around the inputs holds NaN, so a read outside [M, N] would show in the output.
"""
import pytest

from _refcheck import bits as _bits, dev as _dev, launches as _launches, rand as _rand

pytestmark = pytest.mark.gpu

ACT_GELU_NEW, ACT_RELU_POST = 1, 4
DACT_GELU_NEW, DACT_RELU = 1, 3


def _place(vals, ld, bstrides, shift):
    """vals copied into a NaN-filled storage as a view with row stride ld, batch strides bstrides, at element `shift`."""
    import torch

    lead, (M, N) = vals.shape[:-2], vals.shape[-2:]
    size = shift + sum((n - 1) * s for n, s in zip(lead, bstrides)) + (M - 1) * ld + N + 8
    st = torch.full((size,), float("nan"), dtype=vals.dtype, device=vals.device)
    v = st.as_strided(vals.shape, (*bstrides, ld, 1), shift)
    v.copy_(vals)
    return v


def _run(M, N, K, *, lead=(), b_mn=False, bias=False, act=0, aux_out=False, dact=0, res=(), ld_res=None, force_bn=0,
         seed=0):
    import torch

    from magma_b200 import ops

    dev = _dev()
    gen = torch.Generator().manual_seed(seed * 7919 + M * 31 + N * 17 + K)
    A = _rand((*lead, M, K), gen, 1.0, dev)
    B = _rand((*lead, K, N) if b_mn else (*lead, N, K), gen, K**-0.5, dev)
    ldc = (N + 7) // 8 * 8 + 8
    ld_r = ldc if ld_res is None else ldc + ld_res
    plane = (M + 3) * max(ldc, ld_r)
    # non-contiguous batch strides: the outer dim has the smaller stride, with a gap after the inner batches
    bstrides = (plane, (lead[0] + 1) * plane) if len(lead) == 2 else ()
    ins = {}
    if dact:
        ins["aux_in"] = (_rand((*lead, M, N), gen, 1.5, dev), ldc)
    for name in res:
        ins[name] = (_rand((*lead, M, N), gen, 1.0, dev), ld_r)
    kw = dict(b_mn=b_mn, act=act, dact=dact, force_bn=force_bn)
    if bias:
        kw["bias"] = _rand((N,), gen, 0.5, dev)

    results = []
    for shift in (0, 1):  # 0: TMA-staged inputs; 1: base one element past a 16-byte boundary -> register loads
        call = dict(kw)
        for name, (vals, ld) in ins.items():
            call[name] = _place(vals, ld, bstrides, shift)
        out = _place(torch.zeros((*lead, M, N), dtype=torch.bfloat16, device=dev), ldc, bstrides, 0)
        if aux_out:
            call["aux_out"] = _place(torch.zeros((*lead, M, N), dtype=torch.bfloat16, device=dev), ldc, bstrides, 0)
        n0 = _launches()
        ops.gemm(A, B, out=out, **call)
        assert _launches() - n0 == 1
        torch.cuda.synchronize()
        results.append((out, call.get("aux_out")))
    (o_tma, x_tma), (o_reg, x_reg) = results
    assert not torch.isnan(o_tma.float()).any()
    assert torch.equal(_bits(o_tma), _bits(o_reg)), "out differs between the TMA and register input paths"
    if aux_out:
        assert torch.equal(_bits(x_tma), _bits(x_reg)), "aux_out differs between the TMA and register input paths"


FORMS = {
    "dact_gelu": dict(dact=DACT_GELU_NEW),
    "dact_relu": dict(dact=DACT_RELU),
    "res1": dict(res=("res1",)),
    "res2": dict(res=("res2",)),
    "res1+res2": dict(res=("res1", "res2")),
    "dact_gelu+res1+res2": dict(dact=DACT_GELU_NEW, res=("res1", "res2")),
    "bias+relu_post+res1": dict(bias=True, act=ACT_RELU_POST, res=("res1",)),
    "bias+gelu+aux+res1+res2": dict(bias=True, act=ACT_GELU_NEW, aux_out=True, res=("res1", "res2")),
}


@pytest.mark.parametrize("shape", [(65, 203, 72), (129, 1001, 136), (256, 512, 64)], ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("form", list(FORMS))
@pytest.mark.parametrize("bn", [64, 128, 256])
def test_input_forms(bn, form, shape):
    M, N, K = shape
    _run(M, N, K, force_bn=bn, **FORMS[form])


@pytest.mark.parametrize("ld_res", [+24, -8], ids=["ld_res>ldc", "ld_res<ldc"])
@pytest.mark.parametrize("bn", [64, 128, 256])
def test_residual_row_stride(bn, ld_res):
    _run(200, 1001, 136, dact=DACT_RELU, res=("res1", "res2"), ld_res=ld_res, force_bn=bn)


BATCH_FORMS = {
    "dact_relu+res1+res2": dict(dact=DACT_RELU, res=("res1", "res2")),
    "bias+gelu+aux+res1": dict(bias=True, act=ACT_GELU_NEW, aux_out=True, res=("res1",)),
}


@pytest.mark.parametrize("form", list(BATCH_FORMS))
@pytest.mark.parametrize("bn", [64, 128, 256])
def test_two_batch_dims(bn, form):
    _run(130, 200, 72, lead=(2, 3), b_mn=True, force_bn=bn, **BATCH_FORMS[form])


# GPT-J-6B (d = 4096) and its MLP adapters (r = 1024) at M = 1024 tokens, automatic tile width
GPTJ = {
    "out fwd +res1": dict(N=4096, K=4096, res=("res1",)),
    "fc_out dgrad dgelu": dict(N=16384, K=4096, b_mn=True, dact=DACT_GELU_NEW),
    "qkv dgrad +res1": dict(N=4096, K=12288, b_mn=True, res=("res1",)),
    "adapter up bias+res1+res2": dict(N=4096, K=1024, bias=True, res=("res1", "res2")),
    "adapter dgrad-up drelu": dict(N=1024, K=4096, b_mn=True, dact=DACT_RELU),
    "adapter dgrad-down +res1": dict(N=4096, K=1024, b_mn=True, res=("res1",)),
}


@pytest.mark.parametrize("case", list(GPTJ))
def test_gptj_shapes(case):
    c = dict(GPTJ[case])
    _run(1024, c.pop("N"), c.pop("K"), **c)


@pytest.mark.parametrize("form", ["res1+res2", "dact_gelu"])
@pytest.mark.parametrize("M", [1, 7, 32])
def test_small_m(M, form):
    kw = dict(res=("res1", "res2")) if form == "res1+res2" else dict(dact=DACT_GELU_NEW)
    _run(M, 1003, 4096, **kw)
