"""The ViT-L/14 forward's GEMMs have compiled epilogue forms (bias + res1 for out and proj, bias + QuickGELU for fc) and
the tile planner weighs the epilogue form, so at M = 2056 (8 images x 257 tokens) they run at the 256-wide tile with a
compiled form instead of 64-wide tiles with the runtime form. Compiled and runtime form must give the same bits, the
planner must pick the same width whether or not the runtime form is forced, and the GPT-J GEMMs of a training step
must keep the plans they had before the epilogue entered the cost model.
"""
import pytest

from test_gemm_epilogue_forms_gpu import _call, _inputs, _same

pytestmark = pytest.mark.gpu

ACT_QUICK_GELU = 2

# the four GEMMs of a ViT-L/14 block (width 1024, MLP 4096) at M = 2056
VIT = {
    "qkv: bias": dict(N=3072, K=1024, bias=True),
    "out: bias+res1": dict(N=1024, K=1024, bias=True, res=("res1",)),
    "fc: bias+quick_gelu": dict(N=4096, K=1024, bias=True, act=ACT_QUICK_GELU),
    "proj: bias+res1": dict(N=1024, K=4096, bias=True, res=("res1",)),
}


def _vit(name, M=2056, **shape):
    c = dict(VIT[name])
    c.update(shape)
    return _inputs(M, c.pop("N"), c.pop("K"), **c)


@pytest.mark.parametrize("gemm", list(VIT))
def test_vit_shape_compiled_equals_runtime_form(gemm):
    from magma_b200 import ops

    case = _vit(gemm, force_bn=0)
    got = _call(*case)
    assert ops.gemm_last_plan() == (256, 1)
    want = _call(*case, generic_epilogue=True)
    assert ops.gemm_last_plan() == (256, 1), "the plan must not depend on generic_epilogue"
    _same(got, want, "between the compiled and the runtime form")


@pytest.mark.parametrize("gemm", [g for g in VIT if g != "qkv: bias"])
def test_vit_form_ragged_shape(gemm):
    """M = 1000: the last row block is partial; N = 4090: the last 4-column group has two columns"""
    case = _vit(gemm, M=1000, N=4090, K=264)
    _same(_call(*case), _call(*case, generic_epilogue=True), "between the compiled and the runtime form")


def test_quick_gelu_matches_fp64():
    """bias + QuickGELU on the compiled form against x * sigmoid(1.702 x) in fp64"""
    import torch

    A, B, kw, outputs = _vit("fc: bias+quick_gelu", M=1000, N=4090, K=264)
    got = _call(A, B, kw, outputs)[0]
    x = A.double() @ B.double().t() + kw["bias"].double()
    want = x * torch.sigmoid(1.702 * x)
    out = got.view(torch.bfloat16).double()
    err = (out - want).abs() / (want.abs() + 1e-2)
    assert err.max().item() < 2e-2


# (M, N, K, majors and features, width) of the GEMMs of a config-2 training step (GPT-J-6B, its adapters, the ViT
# patch embedding) that run unsplit without a scratch, and the width they ran at before
GPTJ = [
    (1024, 16384, 4096, dict(bias=True, act=1, aux_out=True), 256),
    (1024, 4096, 16384, dict(bias=True), 256),
    (1024, 12288, 4096, dict(), 256),
    (1024, 4096, 4096, dict(res=("res1",)), 256),
    (1024, 50258, 4096, dict(bias=True), 256),
    (1024, 4096, 1024, dict(bias=True, res=("res1", "res2")), 256),
    (1024, 16384, 4096, dict(b_mn=True, dact=1), 256),
    (1024, 4096, 16384, dict(b_mn=True), 256),
    (1024, 4096, 12288, dict(b_mn=True, res=("res1",)), 256),
    (1024, 1024, 4096, dict(bias=True, act=3), 64),
    (1024, 1024, 4096, dict(b_mn=True, dact=3), 64),
    (1024, 4096, 50258, dict(b_mn=True), 256),
    (2048, 1024, 588, dict(), 128),
    (4096, 1024, 1024, dict(a_mn=True, b_mn=True, f32=True), 256),
    (1024, 4096, 1024, dict(a_mn=True, b_mn=True, f32=True), 256),
]


@pytest.mark.parametrize("M,N,K,feat,bn", GPTJ)
def test_gptj_plans_unchanged(M, N, K, feat, bn):
    import torch

    from magma_b200 import ops

    A, B, kw, outputs = _inputs(M, N, K, force_bn=0, **feat)
    out, aux = outputs()
    if aux is not None:
        kw = dict(kw, aux_out=aux.view)
    ops.gemm(A, B, out=out.view, **kw)
    torch.cuda.synchronize()
    assert ops.gemm_last_plan() == (bn, 1)
