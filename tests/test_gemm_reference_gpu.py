"""Element-wise float64 reference tests of the wgmma GEMM core (ops.gemm -> mb200_gemm), across its tile widths, operand
majors, epilogue forms, batch layouts, split-K plans and the persistent schedule under an SM limit.

Every output element (and every saved pre-activation) must satisfy

    |got - ref| <= ulp_out(ref) + 2 * gamma_K * |alpha| * (|A| @ |B|^T),    gamma_K = ceil(K / 16) * 2^-23

ref restates the epilogue order of include/magma_b200.h in float64 from the same bf16 inputs. ulp_out is one bf16 ulp at
|ref| (2^-22 |ref| for fp32 outputs), gamma_K bounds the fp32 accumulation over the wgmma k-steps, and the factor 2 covers
the slope of the epilogue (GELU <= 1.13; a rotated pair uses the larger |A| @ |B|^T of its two columns). ReLU decisions
whose float64 argument lies within that bound of zero are not compared; they must stay under 1 % of the elements.

Outputs live inside larger buffers filled with a sentinel (>= 3 extra rows and >= 8 extra columns, gaps between batches)
that must stay untouched; the padding of every input holds NaN, so a read outside [M, N] or [M|N, K] poisons the result.
Every input is compared byte for byte before and after each call.

The device comes from MB200_TEST_DEVICE (default cuda:0): tests/test_gemm_reference_twin_cpu.py replays the bodies of the
tile, epilogue and batch tests on the CPU emulation of the operator, where no launches are counted.
"""
import math
import os

import pytest

pytestmark = pytest.mark.gpu

SENTINEL = -1.5e38
ACT = dict(none=0, gelu_new=1, quick_gelu=2, relu=3, relu_post=4)
DACT = dict(none=0, gelu_new=1, relu=3)


def _dev():
    """cuda:0 — or the CPU when tests/test_gemm_reference_twin_cpu.py replays a test body on the emulated operator."""
    import torch

    return torch.device(os.environ.get("MB200_TEST_DEVICE", "cuda:0"))


def _launches():
    from magma_b200._lib import lib

    return lib().mb200_launch_count()


class _Buf:
    """A [*lead, rows, cols] view into a flat storage filled with `fill`: row stride `ld` (default: cols rounded up to 8,
    plus 8), 3 spare rows per batch and, unless given, batch strides that are not those of a contiguous tensor (the
    outer batch dim has the smaller stride, and a gap of one batch follows)."""

    def __init__(self, lead, rows, cols, dtype, dev, fill, ld=None, bstrides=None):
        import torch

        ld = ld or (cols + 7) // 8 * 8 + 8
        plane = (rows + 3) * ld
        if bstrides is None:
            bstrides = (plane, (lead[0] + 1) * plane)[: len(lead)] if len(lead) == 2 else (2 * plane,) * len(lead)
        size = sum((n - 1) * s for n, s in zip(lead, bstrides)) + plane + 8
        self.shape, self.strides = (*lead, rows, cols), (*bstrides, ld, 1)
        self.storage = torch.full((size,), fill, dtype=dtype, device=dev)
        self.view = self.storage.as_strided(self.shape, self.strides)
        inside = torch.zeros(size, dtype=torch.bool, device=dev)
        inside.as_strided(self.shape, self.strides).fill_(True)
        self.outside = ~inside
        self.fill = torch.full((1,), fill, dtype=dtype, device=dev)

    def overwritten(self):
        return int((self.storage[self.outside] != self.fill).sum().item())


def _rand(shape, gen, scale, dev, dtype=None):
    import torch

    t = torch.randn(*shape, generator=gen, dtype=torch.float64) * scale
    return t.to(dtype or torch.bfloat16).to(dev)


def _bits(t):
    import torch

    t = t.contiguous()
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32).clone()


def _rope_params(M, N):
    hd = 96 if N > 400 else 48
    return dict(S=37 if M > 37 else max(1, M // 2), hd=hd, rot=hd // 3 // 4 * 4, ncols=N * 3 // 5 // 4 * 4, pos0=5)


def _reference(Al, Bl, *, alpha, bias, act, dact, aux_in, res1, res2, rope, c_old):
    """float64 restatement of the documented epilogue. Returns (out, pre-activation, accumulation bound, ambiguous mask)."""
    import torch

    A64, B64 = Al.double(), Bl.double()
    K = A64.shape[-1]
    acc = A64 @ B64.transpose(-1, -2)
    mag = A64.abs() @ B64.abs().transpose(-1, -2)
    v = alpha * acc
    if bias is not None:
        v = v + bias.double()
    if rope is not None:
        tab, mode, S, hd, rot, ncols = rope
        M, N = v.shape[-2:]
        c = torch.arange(0, N - 1, 2, device=v.device)
        c = c[(c < ncols) & (c % hd < rot)]
        cs = tab.double()[torch.arange(M, device=v.device) % S][:, (c % hd) // 2]  # [M, pairs, 2]
        cos, sin = cs[..., 0], cs[..., 1] * (1.0 if mode > 0 else -1.0)
        x0, x1 = v[..., c].clone(), v[..., c + 1].clone()
        v = v.clone()
        v[..., c], v[..., c + 1] = x0 * cos - x1 * sin, x1 * cos + x0 * sin
        mag = mag.clone()
        pair = torch.maximum(mag[..., c], mag[..., c + 1])
        mag[..., c], mag[..., c + 1] = pair, pair
    bound_acc = 2.0 * math.ceil(K / 16) * 2.0**-23 * abs(alpha) * mag
    amb = torch.zeros_like(v, dtype=torch.bool)
    pre = v
    if act == ACT["gelu_new"]:
        v = 0.5 * v * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (v + 0.044715 * v**3)))
    elif act == ACT["quick_gelu"]:
        v = v * torch.sigmoid(1.702 * v)
    elif act == ACT["relu"]:
        amb |= v.abs() <= bound_acc + 2.0**-22 * v.abs()
        v = v.clamp(min=0.0)
    if dact == DACT["gelu_new"]:
        x = aux_in.double()
        k0, k1 = math.sqrt(2.0 / math.pi), 0.044715
        t = torch.tanh(k0 * (x + k1 * x**3))
        v = v * (0.5 * (1.0 + t) + 0.5 * x * (1.0 - t * t) * k0 * (1.0 + 3.0 * k1 * x * x))
    elif dact == DACT["relu"]:
        v = v * (aux_in.double() > 0)  # the mask comes from an exact input: never ambiguous
    size = v.abs()
    for r in (res1, res2):
        if r is not None:
            v = v + r.double()
            size = size + r.double().abs()
    if act == ACT["relu_post"]:
        amb |= v.abs() <= bound_acc + 2.0**-22 * size
        v = v.clamp(min=0.0)
    if c_old is not None:
        v = v + c_old.double()
    return v, pre, bound_acc, amb


def _check(name, got, ref, bound_acc, f32, amb=None):
    """The element-wise criterion; prints the largest err / bound ratio, or fails with the worst element."""
    import torch

    ref_abs = ref.abs()
    if f32:
        ulp = ref_abs * 2.0**-22
    else:
        _, e = torch.frexp(ref_abs.clamp(min=2.0**-126))  # |ref| in [2^(e-1), 2^e): bf16 ulp 2^(e-8)
        ulp = torch.ldexp(torch.ones_like(ref), e - 8)
    bound = ulp + bound_acc
    err = (got.double() - ref).abs()
    ratio = torch.nan_to_num(err / bound, nan=math.inf)
    if amb is not None:
        n_amb = int(amb.sum().item())
        assert n_amb < 0.01 * ref.numel(), f"{name}: {n_amb} of {ref.numel()} ReLU decisions within the bound of zero"
        ratio = ratio.masked_fill(amb, 0.0)
    bad = int((ratio > 1.0).sum().item())
    worst = int(ratio.argmax().item())
    r_max = float(ratio.reshape(-1)[worst].item())
    if bad:
        idx = [int(i) for i in torch.unravel_index(torch.tensor(worst), ref.shape)]
        pytest.fail(f"{name}: {bad} of {ref.numel()} elements outside the bound; worst at {tuple(idx)} (batch..., row, "
                    f"col): got {got.double().reshape(-1)[worst].item():.6g}, ref {ref.reshape(-1)[worst].item():.6g}, "
                    f"err/bound {r_max:.3g}")
    print(f"[ratio] {name}: max err/bound {r_max:.3f}")


def _run(name, M, N, K, *, lead=(), a_mn=False, b_mn=False, out_f32=False, accumulate=False, alpha=1.0, bias=False,
         act="none", aux_out=False, dact="none", res=0, ld_res=None, rope=0, force_bn=0, splitk_ws=None, b_static=False,
         launches=1, out_layout=None, seed=0):
    """One ops.gemm call on freshly drawn inputs, held to the float64 reference. Returns (out, aux_out) copies."""
    import torch

    from magma_b200 import ops

    dev = _dev()
    gen = torch.Generator().manual_seed(seed * 7919 + M * 31 + N * 17 + K)
    nan = float("nan")
    bf = torch.bfloat16

    def operand(rows, scale, mn):
        buf = _Buf(lead, K, rows, bf, dev, nan) if mn else _Buf(lead, rows, K, bf, dev, nan)
        buf.view.copy_(_rand(buf.shape, gen, scale, dev))
        return buf.view, (buf.view.transpose(-1, -2) if mn else buf.view)

    A, Al = operand(M, 1.0, a_mn)
    B, Bl = operand(N, 1.0 / math.sqrt(K), b_mn)
    layout = out_layout or {}
    out = _Buf(lead, M, N, torch.float32 if out_f32 else bf, dev, SENTINEL, **layout)
    c_old = None
    if accumulate:
        out.view.copy_(_rand(out.shape, gen, 1.0, dev, torch.float32))
        c_old = out.view.clone()
    kw = dict(a_mn=a_mn, b_mn=b_mn, alpha=alpha, act=ACT[act], dact=DACT[dact], accumulate=accumulate,
              force_bn=force_bn, splitk_ws=splitk_ws, b_static=b_static)
    inputs = {"A": A, "B": B}
    if bias:
        bstore = torch.full((N + 8,), nan, dtype=bf, device=dev)
        bstore[:N] = _rand((N,), gen, 0.5, dev)
        kw["bias"] = inputs["bias"] = bstore[:N]
    aux = None
    if aux_out:
        aux = _Buf(lead, M, N, bf, dev, SENTINEL, **layout)
        kw["aux_out"] = aux.view
    if dact != "none":
        ai = _Buf(lead, M, N, bf, dev, nan, **layout)
        ai.view.copy_(_rand(ai.shape, gen, 1.5, dev))
        kw["aux_in"] = inputs["aux_in"] = ai.view
    for i in range(res):
        rl = dict(layout) if ld_res is None else dict(ld=ld_res)
        rb = _Buf(lead, M, N, bf, dev, nan, **rl)
        rb.view.copy_(_rand(rb.shape, gen, 1.0, dev))
        kw[f"res{i + 1}"] = inputs[f"res{i + 1}"] = rb.view
    rope_ref = None
    if rope:
        rp = _rope_params(M, N)
        tab = ops.rope_table(rp["S"], rp["rot"], pos0=rp["pos0"], device=dev)
        kw.update(rope_tab=tab, rope_mode=rope, rope_S=rp["S"], rope_hd=rp["hd"], rope_rot=rp["rot"],
                  rope_ncols=rp["ncols"])
        rope_ref = (tab, rope, rp["S"], rp["hd"], rp["rot"], rp["ncols"])
        inputs["rope_tab"] = tab
    before = {k: _bits(t) for k, t in inputs.items()}

    n0 = _launches()
    ops.gemm(A, B, out=out.view, **kw)
    n1 = _launches()
    if dev.type == "cuda":
        torch.cuda.synchronize()
        assert n1 - n0 == launches, f"{name}: {n1 - n0} kernel launches, expected {launches}"

    for k, t in inputs.items():
        assert torch.equal(_bits(t), before[k]), f"{name}: the call modified its input {k}"
    ref, pre, bound_acc, amb = _reference(Al, Bl, alpha=alpha, bias=kw.get("bias"), act=ACT[act], dact=DACT[dact],
                                          aux_in=kw.get("aux_in"), res1=kw.get("res1"), res2=kw.get("res2"),
                                          rope=rope_ref, c_old=c_old)
    _check(f"{name} out", out.view, ref, bound_acc, out_f32, amb)
    assert out.overwritten() == 0, f"{name}: {out.overwritten()} sentinel elements of the output buffer overwritten"
    if aux is not None:
        _check(f"{name} aux_out", aux.view, pre, bound_acc, False)
        assert aux.overwritten() == 0, f"{name}: {aux.overwritten()} sentinel elements of the aux_out buffer overwritten"
    return out.view.clone(), (aux.view.clone() if aux is not None else None)


def _same(a, b):
    import torch

    return torch.equal(_bits(a), _bits(b))


# ---------------------------------------------------------------------------------------------
# A. tile widths x operand majors on ragged shapes (M at warpgroup / tile boundaries, N % 4 in {1, 3}, K < 64)
# ---------------------------------------------------------------------------------------------
TILE_SHAPES = [(65, 203, 40), (129, 257, 72), (200, 1001, 328), (127, 1003, 8)]


@pytest.mark.parametrize("shape", TILE_SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, False), (True, True)],
                         ids=["KK", "KMN", "MNK", "MNMN"])
@pytest.mark.parametrize("bn", [64, 128, 256])
def test_tiles_and_majors(bn, a_mn, b_mn, shape):
    M, N, K = shape
    _run(f"bn={bn} a_mn={a_mn:d} b_mn={b_mn:d} {M}x{N}x{K}", M, N, K, a_mn=a_mn, b_mn=b_mn, force_bn=bn)


def test_large_automatic_tile():
    _run("1024x4096x4096 auto", 1024, 4096, 4096)


# ---------------------------------------------------------------------------------------------
# B. every epilogue form at every tile width
# ---------------------------------------------------------------------------------------------
EPI_SHAPE = (200, 1001, 328)
EPILOGUES = {
    "bias": dict(bias=True),
    "gelu_new": dict(bias=True, act="gelu_new"),
    "gelu_new+aux": dict(bias=True, act="gelu_new", aux_out=True),
    "quick_gelu": dict(bias=True, act="quick_gelu"),
    "quick_gelu+aux": dict(bias=True, act="quick_gelu", aux_out=True),
    "relu": dict(bias=True, act="relu"),
    "relu+aux": dict(bias=True, act="relu", aux_out=True),
    "relu_post+res1": dict(bias=True, act="relu_post", res=1),
    "dact_gelu": dict(dact="gelu_new"),
    "dact_relu": dict(dact="relu"),
    "alpha=0.5": dict(bias=True, alpha=0.5),
    "alpha=-1.25": dict(bias=True, alpha=-1.25),
    "res1+res2 ld_res>ldc": dict(res=2, ld_res=+24),
    "res1+res2 ld_res<ldc": dict(res=2, ld_res=-8),
    "f32": dict(out_f32=True),
    "f32 accumulate": dict(out_f32=True, accumulate=True, alpha=0.5),
    "rope fwd": dict(bias=True, rope=1),
    "rope inv": dict(rope=-1, aux_out=True),
}


@pytest.mark.parametrize("form", list(EPILOGUES))
@pytest.mark.parametrize("bn", [64, 128, 256])
def test_epilogue_forms(bn, form, shape=EPI_SHAPE):
    M, N, K = shape
    kw = dict(EPILOGUES[form])
    if "ld_res" in kw:  # residual row stride relative to ldc = round_up(N, 8) + 8
        kw["ld_res"] += (N + 7) // 8 * 8 + 8
    _run(f"{form} bn={bn} {M}x{N}x{K}", M, N, K, force_bn=bn, **kw)


# ---------------------------------------------------------------------------------------------
# C. two batch dims with non-contiguous batch strides on A, B, C, aux and residuals
# ---------------------------------------------------------------------------------------------
BATCH_FORMS = {
    "plain f32": dict(out_f32=True),
    "bias+gelu+aux+res1": dict(bias=True, act="gelu_new", aux_out=True, res=1),
    "dact_relu+res1+res2": dict(dact="relu", res=2, alpha=-0.75),
}


@pytest.mark.parametrize("form", list(BATCH_FORMS))
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, False), (True, True)],
                         ids=["KK", "KMN", "MNK", "MNMN"])
def test_batched(a_mn, b_mn, form, shape=(130, 203, 72)):
    M, N, K = shape
    _run(f"batched {form} a_mn={a_mn:d} b_mn={b_mn:d}", M, N, K, lead=(2, 3), a_mn=a_mn, b_mn=b_mn,
         **BATCH_FORMS[form])


@pytest.mark.parametrize("bn", [64, 256])
def test_batched_attention_style_output(bn, S=100, H=3, hd=64, Sk=136):
    """P V into o.permute(0, 2, 1, 3) of o [B, S, H, hd]: batch dims (B, H), heads interleaved within each row."""
    hdp = hd + 8
    ld = H * hdp
    layout = dict(ld=ld, bstrides=((S + 3) * ld, hdp))
    _run(f"attention-style output bn={bn}", S, hd, Sk, lead=(2, H), b_mn=True, res=1, force_bn=bn,
         out_layout=layout)


# ---------------------------------------------------------------------------------------------
# D. split-K plans: the host rules of gemm.cu select a split (2 launches: partial tiles + finalize)
# ---------------------------------------------------------------------------------------------
SMALL_M_EPI = {
    "bias+gelu+aux": dict(bias=True, act="gelu_new", aux_out=True),
    "alpha": dict(alpha=-1.25),
    "res1+res2": dict(res=2),
    "dact_gelu": dict(dact="gelu_new"),
}
# N = 4096, K = 4096 is served best unsplit by the small-M plan (64 tiles of BN = 64); N = 3072 splits.
SPLIT_CASES = {
    **{f"smallm M={M} N={N} K={K} {e}": dict(M=M, N=N, K=K, **kw)
       for M in (1, 7, 32) for (N, K) in ((1003, 4096), (1003, 16384), (3072, 4096), (4096, 16384))
       for e, kw in SMALL_M_EPI.items()},
    "smallm decode qkv rope M=4": dict(M=4, N=3072, K=8192, rope=1),
    "mid M=33 N=4096 K=8192 bias+gelu+aux": dict(M=33, N=4096, K=8192, bias=True, act="gelu_new", aux_out=True),
    "mid M=100 N=1003 K=16384 alpha+res1+res2": dict(M=100, N=1003, K=16384, alpha=0.5, res=2),
    "mid M=128 N=8192 K=8192 f32 accumulate MN-major A": dict(M=128, N=8192, K=8192, a_mn=True, out_f32=True,
                                                             accumulate=True),
    "mid M=100 N=2048 K=16384 MN-major A dact_gelu": dict(M=100, N=2048, K=16384, a_mn=True, dact="gelu_new"),
    "mid M=32 N=1003 K=8192 MN-major A relu": dict(M=32, N=1003, K=8192, a_mn=True, bias=True, act="relu"),
    "few vit out-proj wgrad": dict(M=1024, N=1024, K=2056, a_mn=True, b_mn=True, out_f32=True, accumulate=True),
    "few conv-trunk bias+relu": dict(M=1152, N=768, K=6912, bias=True, act="relu"),
    "few conv-trunk bias+relu_post+res1": dict(M=1152, N=768, K=6912, bias=True, act="relu_post", res=1),
}


def _scratch(n_floats):
    import torch

    return torch.full((n_floats,), float("nan"), dtype=torch.float32, device=_dev())


@pytest.mark.parametrize("case", list(SPLIT_CASES))
def test_split_k_plan(case):
    c = dict(SPLIT_CASES[case])
    M, N, K = c.pop("M"), c.pop("N"), c.pop("K")
    ws = _scratch(16 << 20)
    split = _run(f"{case} split", M, N, K, splitk_ws=ws, launches=2, **c)
    again = _run(f"{case} split rerun", M, N, K, splitk_ws=_scratch(16 << 20), launches=2, **c)
    assert all(a is None or _same(a, b) for a, b in zip(split, again)), f"{case}: split-K rerun not bit-identical"
    _run(f"{case} single pass", M, N, K, launches=1, **c)


@pytest.mark.parametrize("case", ["smallm M=7 N=1003 K=16384 res1+res2", "few vit out-proj wgrad",
                                  "mid M=33 N=4096 K=8192 bias+gelu+aux"])
def test_split_k_scratch_size(case):
    """Scratch of exactly splits * M * round_up(N, 4) fp32 runs the same plan; scratch too small for two splits
    runs a single pass."""
    c = dict(SPLIT_CASES[case])
    M, N, K = c.pop("M"), c.pop("N"), c.pop("K")
    slice_ = M * ((N + 3) // 4 * 4)
    ws = _scratch(16 << 20)
    big = _run(f"{case} ample scratch", M, N, K, splitk_ws=ws, launches=2, **c)
    used = int((~ws.isnan()).sum().item())
    assert used % slice_ == 0 and used >= 2 * slice_, f"{case}: {used} scratch floats written"
    splits = used // slice_
    exact = _scratch(splits * slice_)
    got = _run(f"{case} exact scratch ({splits} splits)", M, N, K, splitk_ws=exact, launches=2, **c)
    assert not bool(exact.isnan().any()), f"{case}: exact scratch not fully used by {splits} splits"
    assert all(a is None or _same(a, b) for a, b in zip(big, got))
    _run(f"{case} scratch below two splits", M, N, K, splitk_ws=_scratch(2 * slice_ - 1), launches=1, **c)


# ---------------------------------------------------------------------------------------------
# E. the persistent schedule under a CTA limit (each CTA loops over many tiles, the mbarrier ring wraps its phase)
# ---------------------------------------------------------------------------------------------
PERSISTENT_CASES = {
    "1024x4096x4096 bn=256": dict(M=1024, N=4096, K=4096, force_bn=256),
    "ragged batched": dict(M=200, N=1001, K=328, lead=(2, 3), b_mn=True, bias=True, act="gelu_new", aux_out=True,
                           res=1),
    "split_few conv-trunk": dict(M=1152, N=768, K=6912, bias=True, act="relu_post", res=1, split=True),
}


@pytest.fixture
def gemm_sm_limit():
    from magma_b200._lib import lib

    L = lib()
    L.mb200_set_gemm_sm_limit(0)
    yield L.mb200_set_gemm_sm_limit
    L.mb200_set_gemm_sm_limit(int(os.environ.get("MB200_GEMM_SMS", "0") or 0))


@pytest.mark.parametrize("limit", [1, 3, 17])
@pytest.mark.parametrize("case", list(PERSISTENT_CASES))
def test_persistent_schedule_under_sm_limit(gemm_sm_limit, case, limit):
    c = dict(PERSISTENT_CASES[case])
    M, N, K = c.pop("M"), c.pop("N"), c.pop("K")
    split = c.pop("split", False)
    ws = (lambda: _scratch(16 << 20)) if split else (lambda: None)
    n = 2 if split else 1
    full = _run(f"{case} all SMs", M, N, K, splitk_ws=ws(), launches=n, **c)
    assert gemm_sm_limit(limit) == limit
    got = _run(f"{case} {limit} SMs", M, N, K, splitk_ws=ws(), launches=n, **c)
    assert all(a is None or _same(a, b) for a, b in zip(full, got)), f"{case}: limit {limit} changed the result"


# ---------------------------------------------------------------------------------------------
# F. b_static (frozen weights) gives the same bits
# ---------------------------------------------------------------------------------------------
STATIC_CASES = {
    "dense bias+gelu+aux": dict(M=200, N=1001, K=328, bias=True, act="gelu_new", aux_out=True),
    "batched MN-major B": dict(M=130, N=203, K=72, lead=(2, 3), b_mn=True, res=1),
    "split small-M": dict(M=7, N=1003, K=16384, bias=True, split=True),
}


@pytest.mark.parametrize("case", list(STATIC_CASES))
def test_b_static_is_bit_identical(case):
    c = dict(STATIC_CASES[case])
    M, N, K = c.pop("M"), c.pop("N"), c.pop("K")
    split = c.pop("split", False)
    n = 2 if split else 1
    plain = _run(f"{case} b_static=False", M, N, K, splitk_ws=_scratch(16 << 20) if split else None, launches=n, **c)
    static = _run(f"{case} b_static=True", M, N, K, splitk_ws=_scratch(16 << 20) if split else None, launches=n,
                  b_static=True, **c)
    assert all(a is None or _same(a, b) for a, b in zip(plain, static))
