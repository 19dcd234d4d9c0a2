"""The GEMM core compiles its epilogue once per epilogue form: a runtime form that reads every feature from the launch
parameters, and compiled forms for the feature sets a GPT-J training step launches at the 256-wide tile, in which the
absent features are not generated and the row loop is unrolled. Both must give the same bits.

Each case calls ops.gemm twice on the same seeded inputs, once as the host selects (a compiled form) and once with
generic_epilogue (the runtime form), at the GPT-J shape the form serves and at a ragged shape whose last row block and
last 4-column group are partial. out and aux_out lie in sentinel-filled buffers: they must be bit-identical and the
padding untouched, and each call is one launch. Inputs lie in NaN-filled buffers, so a read outside [M, N] would show.
"""
import pytest

from _refcheck import SENTINEL, Buf, bits as _bits, dev as _dev, launches as _launches, rand as _rand

pytestmark = pytest.mark.gpu

ACT_GELU_NEW, DACT_GELU_NEW = 1, 1


def _placed(vals):
    """vals as a padded-row view (row stride a multiple of 8 elements) into NaN-filled storage"""
    b = Buf((), vals.shape[0], vals.shape[1], vals.dtype, vals.device, float("nan"))
    b.view.copy_(vals)
    return b.view


def _inputs(M, N, K, *, a_mn=False, b_mn=False, bias=False, act=0, aux_out=False, dact=0, res=(), rope=False, f32=False,
            accumulate=False, bias_shift=0, force_bn=256):
    """(A, B, keyword arguments of ops.gemm, makers of the output buffers) of one case"""
    import torch

    from magma_b200 import ops

    dev = _dev()
    gen = torch.Generator().manual_seed(M * 31 + N * 17 + K)
    A = _placed(_rand((K, M) if a_mn else (M, K), gen, 1.0, dev))
    B = _placed(_rand((K, N) if b_mn else (N, K), gen, K**-0.5, dev))
    kw = dict(a_mn=a_mn, b_mn=b_mn, act=act, dact=dact, accumulate=accumulate, force_bn=force_bn)
    if bias:  # bias_shift = 1: one element past an 8-byte boundary
        st = torch.full((N + 8,), float("nan"), dtype=torch.bfloat16, device=dev)
        kw["bias"] = st[bias_shift:bias_shift + N]
        kw["bias"].copy_(_rand((N,), gen, 0.5, dev))
    if dact:
        kw["aux_in"] = _placed(_rand((M, N), gen, 1.5, dev))
    for name in res:
        kw[name] = _placed(_rand((M, N), gen, 1.0, dev))
    if rope:  # GPT-J: 256-wide heads, 64 rotary dims, on the q and k thirds of a fused qkv output
        ncols = 2 * N // 3 // 256 * 256
        kw.update(rope_tab=ops.rope_table(128, 64, device=dev), rope_mode=1, rope_S=128, rope_hd=256, rope_rot=64,
                  rope_ncols=ncols)
    old = _rand((M, N), gen, 1.0, dev, torch.float32) if accumulate else None

    def outputs():
        out = Buf((), M, N, torch.float32 if f32 else torch.bfloat16, dev, SENTINEL)
        if accumulate:
            out.view.copy_(old)
        aux = Buf((), M, N, torch.bfloat16, dev, SENTINEL) if aux_out else None
        return out, aux

    return A, B, kw, outputs


def _call(A, B, kw, outputs, **extra):
    import torch

    from magma_b200 import ops

    out, aux = outputs()
    call = dict(kw, **extra)
    if aux is not None:
        call["aux_out"] = aux.view
    n0 = _launches()
    ops.gemm(A, B, out=out.view, **call)
    assert _launches() - n0 == 1
    torch.cuda.synchronize()
    assert out.overwritten() == 0 and (aux is None or aux.overwritten() == 0), "wrote outside [M, N]"
    assert not torch.isnan(out.view.float()).any()
    return _bits(out.view), (_bits(aux.view) if aux is not None else None)


def _same(got, want, what):
    import torch

    assert torch.equal(got[0], want[0]), f"out differs {what}"
    if want[1] is not None:
        assert torch.equal(got[1], want[1]), f"aux_out differs {what}"


# the compiled forms, each at the GPT-J-6B shape (M = 1024 tokens, d = 4096, adapters r = 1024) it serves
FORMS = {
    "qkv fwd: rotary": dict(N=12288, K=4096, rope=True),
    "out fwd: res1": dict(N=4096, K=4096, res=("res1",)),
    "fc_in fwd: bias+gelu+aux_out": dict(N=16384, K=4096, bias=True, act=ACT_GELU_NEW, aux_out=True),
    "fc_out fwd: bias": dict(N=4096, K=16384, bias=True),
    "adapter up: bias+res1+res2": dict(N=4096, K=1024, bias=True, res=("res1", "res2")),
    "fc_out dgrad: dgelu": dict(N=16384, K=4096, b_mn=True, dact=DACT_GELU_NEW),
    "fc_in dgrad: no features": dict(N=4096, K=16384, b_mn=True),
    "qkv dgrad: res1": dict(N=4096, K=12288, b_mn=True, res=("res1",)),
    "adapter wgrad: fp32 store": dict(M=4096, N=1024, K=1024, a_mn=True, b_mn=True, f32=True),
    "adapter wgrad: fp32 accumulate": dict(M=4096, N=1024, K=1024, a_mn=True, b_mn=True, f32=True, accumulate=True),
}


def _form(name, **shape):
    c = dict(M=1024)
    c.update(FORMS[name])
    c.update(shape)
    return _inputs(c.pop("M"), c.pop("N"), c.pop("K"), **c)


@pytest.mark.parametrize("form", list(FORMS))
def test_gptj_shape(form):
    case = _form(form, force_bn=0)  # the tile width the step gets: 256
    _same(_call(*case), _call(*case, generic_epilogue=True), "between the compiled and the runtime form")


@pytest.mark.parametrize("form", list(FORMS))
def test_ragged_shape(form):
    """M = 1000: the last row block is partial; N = 4090: the last 4-column group has two columns"""
    case = _form(form, M=1000, N=4090, K=264)
    _same(_call(*case), _call(*case, generic_epilogue=True), "between the compiled and the runtime form")


def test_lm_head_shape():
    """bias form at the GPT-J vocabulary, N = 50258 = 4 x 12564 + 2"""
    case = _inputs(1024, 50258, 4096, bias=True, force_bn=0)
    _same(_call(*case), _call(*case, generic_epilogue=True), "between the compiled and the runtime form")


def test_misaligned_bias_is_still_correct():
    """A bias one element past an 8-byte boundary cannot be read as vectors: the launch must not take the compiled form"""
    want = _call(*_inputs(1000, 4090, 264, bias=True))
    _same(_call(*_inputs(1000, 4090, 264, bias=True, bias_shift=1)), want, "with a misaligned bias")


def _kernel(A, B, kw, outputs, **extra):
    """name of the kernel the call launches"""
    import torch
    from torch.profiler import ProfilerActivity, profile

    from magma_b200 import ops

    out, aux = outputs()
    call = dict(kw, **extra)
    if aux is not None:
        call["aux_out"] = aux.view
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ops.gemm(A, B, out=out.view, **call)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if "gemm_wgmma_kernel" in e.name]
    assert len(names) == 1, names
    return names[0]


@pytest.mark.parametrize("form", list(FORMS))
def test_table_launches_select_a_compiled_form(form):
    """Without this a host that always fell back to the runtime form would pass every comparison above."""
    case = _form(form, M=256, N=512, K=64)
    assert _kernel(*case) != _kernel(*case, generic_epilogue=True)


def test_misaligned_bias_selects_the_runtime_form():
    generic = _kernel(*_inputs(256, 512, 64, bias=True), generic_epilogue=True)
    assert _kernel(*_inputs(256, 512, 64, bias=True, bias_shift=1)) == generic
