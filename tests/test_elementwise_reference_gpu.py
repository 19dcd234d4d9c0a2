"""Element-wise float64 reference tests of the HBM-bound kernels of csrc/elementwise.cu (bodies in elt_kernels.cuh and
train_kernels.cuh): LayerNorm, cross-entropy, the column reductions, the optimizer, the layout / gather kernels, the
casts, dropout, argmax, the rotary table and the decode-loop kernels.

Every reference is computed in float64 on the device from the same bf16 / fp32 inputs. u = 2^-24 is the fp32 unit
roundoff. The library is built without --use_fast_math, so division and sqrtf round correctly and sincosf, powf and
logf are the accurate library versions. Their bounds are the ones in the tables "Single-Precision Mathematical Standard
Library Functions with Maximum ULP Error" and "Single-Precision Floating-Point Intrinsic Functions" of the CUDA C++
Programming Guide: rsqrtf 2 ulp, logf 1 ulp, sinf / cosf / sincosf 2 ulp, powf 4 ulp, __expf(x) 2 + floor(1.173 |x|)
ulp. One ulp of a result r is at most 2u |r| (2^-149 below 2^-126).

Sums. A sum computed in fp32 in a known order differs from the exact sum by at most u times the sum of the magnitudes
of its partial sums (the running-error bound; the partial sums are taken in float64 from the exact terms, and the
factor 1.001 covers the second-order terms). The kernels' orders:
  - block_sum over 256 (512) threads: each thread first adds its own terms serially, then 5 xor-shuffle levels
    (16, 8, 4, 2, 1; a level's partial sums are the sums over the lanes of one residue class), then the 8 (16) warp
    totals go through the same 5 levels in warp 0. LayerNorm: thread t holds the 8-element vectors t, t + 256, ...
    (at most 4, so at most 32 terms), in that order. Cross-entropy: thread t holds vectors t, t + 512, ..., then one
    element of the scalar tail.
  - colsum and layernorm_param_grad_rows: per 64-row chunk, row group g (0..7) adds rows g, g + 8, ... serially, the 8
    group sums are added in order, then one atomicAdd per chunk into the column. col_moments: the same with 128-row
    chunks. The atomics land in any order, so that step is bounded by (chunks) u (sum of |chunk totals| + |start|).
  - dot: thread t of block b adds vectors b 256 + t + k 256 grid serially, then block_sum, then one atomicAdd per block.
  - layernorm_param_grad (few rows): one thread per column adds the rows serially.

LayerNorm. mean and rstd (fp32 outputs) are held to the float64 mean and 1 / sqrt(var + eps): the mean to the sum's
bound / d plus the division's rounding; the variance sums (x - mean_k)^2 with the kernel's mean, so it carries
d e_mean^2 and 2 |x - mean| e_mean + u |x - mean_k|^2 per term besides its own sum bound; rstd = rsqrtf(var + eps) is
within 0.5 dv / v + 4u relative. y is then held by the rounding rule to (x - mean_k) rstd_k gamma + beta with the
kernel's own statistics (exact fp32 inputs): three roundings of the product and one of the sum. A constant row has an
exact mean, zero variance and y == beta bitwise. The backward takes mean and rstd as exact inputs: xhat carries 2u,
the two row sums their running-error bounds, and the result five roundings (six with res).

Cross-entropy. The row sum of __expf(x_j - m) (x_j - m rounds once) carries each term's __expf bound and the running
error; lse = m + logf(sum) adds 1 ulp of logf and two roundings; the row loss one more. The mean over rows is a
block_sum<1024> of the row losses (bounded as one sum of n terms, depth n) and one division. dlogits_j =
(__expf(x_j - m) / sum - [j = target]) * grad_scale / n_valid rounds by the rule with
delta = g (p_j (eps_exp + u |x_j - m| + eps_sum + 2u) + u |p_j - onehot|) + 2u |ref| + 2^-149. A label is valid when
it lies in [0, V); any other label (-100, -1, V, ldv - 1) gives the same loss and the same dlogits bits as -100.

The rounding rule for bf16 outputs (tests/_refcheck.py::check_rounded): the output must equal the float64 reference
rounded to nearest even unless [ref - delta, ref + delta] holds a rounding midpoint. delta is a few fp32 ulps here,
so the ambiguous share is capped at 0.1 % (AMBIGUOUS_MAX) and printed. Exceptions: the LayerNorm backward, whose delta
adds up eight roundings and the two row sums' bounds (AMBIGUOUS_MAX_LN_BWD, 0.3 %), and two kernels whose delta is
dominated by __expf's argument-dependent bound, quick_gelu_bwd over [-20, 20] (|1.702 x| up to 34 is 42 ulp) and
cross-entropy's dlogits (the row sum's bound enters every element): AMBIGUOUS_MAX_EXP, 1 %. A sum of bf16 values that
fp32 holds exactly (|sum| < 2^24 times the smallest spacing of its terms) adds no delta: add, scale_add without s,
vit_assemble, avgpool and col2im3x3 are bit-exact wherever their sums are.

Other derived bounds: rope_table against sin / cos of fl(pos * inv_freq) with GPT-J's fp32 inv_freq (torch); the
kernel's inv_freq = 1 / powf(10000, 2p / rot) is within 4 ulp + 2 roundings of 10000^(-2p/rot) and torch's within
2 roundings more, so the argument is off by pos * 12u * inv_freq + 2u |theta| at most, plus the 2 ulp of sincosf.
bn_finalize_fwd: var = s2 / n - mean^2 carries 2u E[z^2] + 5u mean^2 + u var, a relative error of about
u (2 + 5 mean^2 / var), the cancellation term; rstd then follows as above. AdamW: each of 3 steps is held to float64
from the fp32 state before the step, with every constant's rounding (powf 1 ulp on the host, rsqrtf 2 ulp) and one
rounding per operation.

Bit-exact: the gathers (ids outside [0, vocab) read row 0), decode_advance (token, EOS flag, pos += 1; no token write
when pos + 1 == ld_tok), patchify, im2col3x3, nchw_to_nhwc8 (channels C..7 are +0), both casts, dropout against a
numpy restatement of hash32 with y = RNE(fl(x fl(1 / (1 - p)))), argmax against torch.argmax(x.float()) (ties go to
the lowest index), rope_table_dev against rope_table and the AdamW bf16 shadow against RNE(master). argmax ignores NaN:
a row with NaN entries returns the index of its largest other entry, an all-NaN row returns 2^31 - 1.

Layouts. Outputs sit in sentinel-filled buffers with row strides larger than the row (and spare rows), which must stay
untouched; input padding holds NaN; every input is compared byte for byte before and after each call; each call's
launch count is checked (CUDA only); kernels without atomics give bit-identical reruns.

The device comes from MB200_TEST_DEVICE (default cuda:0): tests/test_elementwise_reference_twin_cpu.py replays the
bodies at small sizes on the kernel source executed on the CPU (oracle/kernel_host_exec.cpp).
"""
import math
import zlib

import numpy as np
import pytest

from _refcheck import SENTINEL, Buf, bf16_rne, bits, check_rounded, dev as _dev, launches

pytestmark = pytest.mark.gpu

U = 2.0**-24
TINY = 2.0**-149
AMBIGUOUS_MAX = 0.001
AMBIGUOUS_MAX_LN_BWD = 0.003
AMBIGUOUS_MAX_EXP = 0.01
F32 = np.float32


def _gen(*key):
    import torch

    return torch.Generator().manual_seed(zlib.crc32(repr(key).encode()))


def _count():
    return launches() if _dev().type == "cuda" else 0


def _launched(name, n0, want=1):
    import torch

    if _dev().type == "cuda":
        torch.cuda.synchronize()
        n = launches() - n0
        assert n == want, f"{name}: {n} kernel launches, expected {want}"


def _same(a, b):
    import torch

    return torch.equal(bits(a), bits(b))


def _untouched(name, *bufs):
    for tag, b in bufs:
        n = b.overwritten()
        assert n == 0, f"{name}: {n} sentinel elements of {tag} overwritten"


class _Inputs:
    """Byte snapshots of the inputs of a call."""

    def __init__(self, *ts):
        self.ts = [t for t in ts if t is not None]
        self.before = [bits(t.reshape(-1).view(-1)) for t in self.ts]

    def unchanged(self, name):
        import torch

        for t, b in zip(self.ts, self.before):
            assert torch.equal(bits(t.reshape(-1)), b), f"{name}: an input was modified"


def _nanbuf(rows, cols, values, dtype=None):
    """A [rows, cols] view with row stride cols + 8 (rounded to 8) in a NaN-filled storage, holding `values`."""
    import torch

    b = Buf((), rows, cols, dtype or torch.bfloat16, _dev(), float("nan"))
    b.view.copy_(values)
    return b


def _check_bound(name, got, ref, bound):
    """|got - ref| <= bound element by element (fp32 outputs); prints the largest err / bound."""
    import torch

    err = (got.double() - ref).abs()
    ratio = torch.where(err == 0, 0.0, torch.nan_to_num(err / bound, nan=math.inf))
    worst = int(ratio.reshape(-1).argmax().item())
    r = float(ratio.reshape(-1)[worst].item())
    if r > 1.0:
        pytest.fail(f"{name}: {int((ratio > 1).sum().item())} of {ref.numel()} elements outside the bound; worst at "
                    f"{worst}: got {got.double().reshape(-1)[worst].item():.9g}, ref {ref.reshape(-1)[worst].item():.9g}, "
                    f"err/bound {r:.3g}")
    print(f"[ratio] {name}: max err/bound {r:.3f}")
    return r


def _quantum(x):
    """The spacing every value of the float64 tensor x (exact bf16 values) is a multiple of; inf for zeros."""
    import torch

    from _refcheck import ulp_bf16

    return torch.where(x == 0, math.inf, ulp_bf16(x))


def _add_err(total, q):
    """Error of one fp32 addition whose exact result `total` is a multiple of q: none when |total| < 2^24 q (the
    result is representable), else u |total|. Sums of a few bf16 values are mostly exact in fp32."""
    import torch

    return torch.where(total.abs() < 2.0**24 * q, 0.0, U * total.abs())


def _ulp32(x):
    """One fp32 ulp at |x| (float64)."""
    import torch

    _, e = torch.frexp(x.abs().clamp(min=2.0**-126))
    return torch.ldexp(torch.ones_like(x, dtype=torch.float64), e - 24)


# ---------------------------------------------------------------------------------------------
# running-error bounds of the kernels' summation orders
# ---------------------------------------------------------------------------------------------
def _block_tree(T):
    """Sum of |partial sums| of block_sum over thread totals T [..., n_threads] (n_threads = 256 or 512)."""
    import torch

    nw = T.shape[-1] // 32
    lanes = T.reshape(*T.shape[:-1], nw, 32)
    tot = torch.zeros(T.shape[:-1], dtype=T.dtype, device=T.device)
    for m in (16, 8, 4, 2, 1):
        tot = tot + lanes.reshape(*T.shape[:-1], nw, 32 // m, m).sum(-2).abs().sum((-1, -2))
    w = torch.zeros(*T.shape[:-1], 32, dtype=T.dtype, device=T.device)
    w[..., :nw] = lanes.sum(-1)
    for m in (16, 8, 4, 2, 1):
        tot = tot + w.reshape(*T.shape[:-1], 32 // m, m).sum(-2).abs().sum(-1)
    return tot


def _ln_sum_err(v):
    """Running-error sum (without the factor u) of the LayerNorm kernels' row sums of v [rows, d]."""
    import torch

    rows, d = v.shape
    full = torch.zeros(rows, 4 * 256 * 8, dtype=v.dtype, device=v.device)
    full[:, :d] = v
    per = full.view(rows, 4, 256, 8).permute(0, 2, 1, 3).reshape(rows, 256, 32)
    cum = per.cumsum(-1)
    return cum[..., 1:].abs().sum((-1, -2)) + _block_tree(cum[..., -1])


def _chunked_err(T, chunk, base=None):
    """(exact column sums, running-error bound) of the colsum / param_grad_rows / col_moments order over T [rows, cols]."""
    import torch

    rows, cols = T.shape
    nch = (rows + chunk - 1) // chunk
    full = torch.zeros(nch * chunk, cols, dtype=T.dtype, device=T.device)
    full[:rows] = T
    per = full.view(nch, chunk // 8, 8, cols)  # row r = k * 8 + g within the chunk
    cum = per.cumsum(1)
    serial = cum[:, 1:].abs().sum((0, 1, 2))
    groups = cum[:, -1].cumsum(1)  # the 8 group sums added in order
    smem = groups[:, 1:].abs().sum((0, 1))
    ctot = groups[:, -1]
    start = base.abs() if base is not None else torch.zeros(cols, dtype=T.dtype, device=T.device)
    atom = (nch + 1) * (ctot.abs().sum(0) + start)
    s = ctot.sum(0) + (base if base is not None else 0)
    return s, U * 1.001 * (serial + smem + atom) + TINY


# ---------------------------------------------------------------------------------------------
# A. LayerNorm
# ---------------------------------------------------------------------------------------------
LN_DISTS = ("normal", "offset64", "outliers", "constant")


def _ln_x(gen, rows, d, dist):
    import torch

    x = torch.randn(rows, d, generator=gen, dtype=torch.float64)
    if dist == "offset64":
        x = x + 64.0
    elif dist == "outliers":
        x[:, 1], x[:, d - 2] = 300.0, -300.0
    elif dist == "constant":
        x = (4.0 * torch.randn(rows, 1, generator=gen, dtype=torch.float64)).expand(rows, d)
    return x.to(torch.bfloat16)


def _layernorm(rows, d, dist):
    import torch

    from magma_b200 import ops

    name = f"layernorm rows={rows} d={d} {dist}"
    dev, bf = _dev(), torch.bfloat16
    gen = _gen("ln", rows, d, dist)
    xb = _nanbuf(rows, d, _ln_x(gen, rows, d, dist).to(dev))
    gamma = (1 + 0.1 * torch.randn(d, generator=gen, dtype=torch.float64)).to(bf).to(dev)
    beta = (0.1 * torch.randn(d, generator=gen, dtype=torch.float64)).to(bf).to(dev)
    eps = float(F32(1e-5))
    inp = _Inputs(xb.storage, gamma, beta)

    def fwd(stats=True):
        yb = Buf((), rows, d, bf, dev, SENTINEL)
        n0 = _count()
        _, mean, rstd = ops.layernorm_fwd(xb.view, gamma, beta, 1e-5, save_stats=stats, out=yb.view)
        _launched(name, n0)
        return yb, mean, rstd

    yb, mk, rk = fwd()
    inp.unchanged(name)
    _untouched(name, ("y", yb))
    x = xb.view.double()
    g, b = gamma.double(), beta.double()
    # statistics
    mean = x.mean(1)
    e_mean = 1.001 * U * (_ln_sum_err(x) / d + mean.abs()) + TINY
    _check_bound(f"{name} mean", mk, mean, e_mean)
    t = (x - mean[:, None]).abs()
    a = t + e_mean[:, None]
    dt = e_mean[:, None] + U * a
    dq = (2 * a * dt + dt * dt + U * a * a).sum(1) + U * _ln_sum_err(a * a)
    var = (t * t).sum(1) / d
    dvar = 1.001 * (dq / d + U * (var + dq / d))
    v = var + eps
    dv = dvar + U * v
    rstd = 1.0 / v.sqrt()
    _check_bound(f"{name} rstd", rk, rstd, rstd * 1.001 * (0.5 * dv / v + 4 * U) + TINY)
    # y from the kernel's own statistics
    m32, r32 = mk.double()[:, None], rk.double()[:, None]
    p = (x - m32) * r32
    ref = p * g + b
    delta = 1.001 * (3 * U * (p * g).abs() + U * ref.abs()) + TINY
    keep = torch.ones(1, dtype=torch.bool, device=dev)
    check_rounded(f"{name} y", yb.view, ref, delta, keep, limit=AMBIGUOUS_MAX)
    if dist == "constant":
        assert torch.equal(mk.double(), x[:, 0]), f"{name}: the mean of a constant row is not exact"
        assert _same(yb.view, beta.expand(rows, d)), f"{name}: y of a constant row is not beta"
    yb2, _, _ = fwd(stats=False)
    assert _same(yb.view, yb2.view), f"{name}: y without saved statistics differs"
    return xb, gamma, mk, rk


def _layernorm_bwd(rows, d, dist, with_res):
    import torch

    from magma_b200 import ops

    name = f"layernorm_bwd rows={rows} d={d} {dist} res={int(with_res)}"
    dev, bf = _dev(), torch.bfloat16
    xb, gamma, mk, rk = _layernorm(rows, d, dist)
    gen = _gen("lnb", rows, d, dist, with_res)
    dyb = _nanbuf(rows, d, torch.randn(rows, d, generator=gen, dtype=torch.float64).to(bf).to(dev))
    rb = _nanbuf(rows, d, torch.randn(rows, d, generator=gen, dtype=torch.float64).to(bf).to(dev)) if with_res else None
    inp = _Inputs(xb.storage, dyb.storage, gamma, mk, rk, rb.storage if rb else None)

    def bwd():
        ob = Buf((), rows, d, bf, dev, SENTINEL)
        n0 = _count()
        ops.layernorm_bwd(dyb.view, xb.view, gamma, mk, rk, res=rb.view if rb else None, out=ob.view)
        _launched(name, n0)
        return ob

    ob = bwd()
    inp.unchanged(name)
    _untouched(name, ("dx", ob))
    x, dy = xb.view.double(), dyb.view.double()
    mu, rs = mk.double()[:, None], rk.double()[:, None]
    g = dy * gamma.double()
    xh = (x - mu) * rs
    e_xh = 2.001 * U * xh.abs()
    m1 = g.sum(1, keepdim=True) / d
    m2 = (g * xh).sum(1, keepdim=True) / d
    e_m1 = 1.001 * U * (_ln_sum_err(g)[:, None] / d + m1.abs())
    e_m2 = 1.001 * ((g.abs() * e_xh).sum(1, keepdim=True) / d + U * ((g * xh).abs().sum(1, keepdim=True)
                    + _ln_sum_err(g * xh)[:, None]) / d + U * m2.abs())
    h = g - m1 - xh * m2
    e_h = e_m1 + xh.abs() * e_m2 + m2.abs() * e_xh + U * ((g - m1).abs() + (xh * m2).abs() + h.abs())
    ref = rs * h
    delta = rs * e_h + U * ref.abs()
    if rb is not None:
        ref = ref + rb.view.double()
        delta = delta + U * ref.abs()
    check_rounded(f"{name} dx", ob.view, ref, 1.001 * delta + TINY, torch.ones(1, dtype=torch.bool, device=dev),
                  limit=AMBIGUOUS_MAX_LN_BWD)
    assert _same(ob.view, bwd().view), f"{name}: rerun not bit-identical"


LN_SHAPES = [(1, 4096), (2056, 1024), (16384, 4096), (3, 8), (5, 8192), (7, 1032)]


@pytest.mark.parametrize("rows,d", LN_SHAPES)
def test_layernorm(rows, d):
    _layernorm_bwd(rows, d, "normal", True)


@pytest.mark.parametrize("dist", LN_DISTS)
@pytest.mark.parametrize("d", [1032, 4096, 8192])
def test_layernorm_distributions(d, dist):
    _layernorm_bwd(64, d, dist, dist != "constant")


def _ln_param_grad(rows, d, many, accumulate):
    import torch

    from magma_b200 import ops

    name = f"layernorm_param_grad{'_rows' if many else ''} rows={rows} d={d} acc={int(accumulate)}"
    dev = _dev()
    gen = _gen("lnpg", rows, d, many, accumulate)
    xb = _nanbuf(rows, d, _ln_x(gen, rows, d, "normal").to(dev))
    dyb = _nanbuf(rows, d, torch.randn(rows, d, generator=gen, dtype=torch.float64).to(torch.bfloat16).to(dev))
    x = xb.view.double()
    mk = x.mean(1).float().contiguous()
    rk = (1.0 / (x.var(1, unbiased=False) + 1e-5).sqrt()).float().contiguous()
    base = torch.randn(2, d, generator=gen, dtype=torch.float64).float().to(dev)
    dg, db = base[0].clone(), base[1].clone()
    inp = _Inputs(xb.storage, dyb.storage, mk, rk)
    n0 = _count()
    fn = ops.layernorm_param_grad_rows if many else ops.layernorm_param_grad
    fn(dyb.view, xb.view, mk, rk, dg, db, accumulate=accumulate)
    _launched(name, n0)
    inp.unchanged(name)
    dy = dyb.view.double()
    xh = (x - mk.double()[:, None]) * rk.double()[:, None]
    tg = dy * xh
    b0 = base.double() if accumulate else None
    if many:
        sg, eg = _chunked_err(tg, 64, None if b0 is None else b0[0])
        sb, eb = _chunked_err(dy, 64, None if b0 is None else b0[1])
    else:
        def serial(T, start):  # one thread per column adds the rows, then (accumulate) adds the sum to the output
            c = T.cumsum(0)
            tot = c[-1] + (start if start is not None else 0)
            extra = tot.abs() if start is not None else 0
            return tot, U * 1.001 * (c[1:].abs().sum(0) + extra) + TINY
        sg, eg = serial(tg, None if b0 is None else b0[0])
        sb, eb = serial(dy, None if b0 is None else b0[1])
    eg = eg + 3.001 * U * tg.abs().sum(0)
    _check_bound(f"{name} dgamma", dg, sg, eg)
    _check_bound(f"{name} dbeta", db, sb, eb)


@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("rows,d", [(2056, 1024), (150, 4104), (16384, 64), (1, 1024)])
def test_layernorm_param_grad_rows(rows, d, accumulate):
    _ln_param_grad(rows, d, True, accumulate)


@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("rows,d", [(16, 1024), (3, 4100)])
def test_layernorm_param_grad(rows, d, accumulate):
    _ln_param_grad(rows, d, False, accumulate)


# ---------------------------------------------------------------------------------------------
# B. cross-entropy
# ---------------------------------------------------------------------------------------------
def _ce_sum_terms(e, V):
    """Running-error sum (without u) of ce_row_kernel's row sum of the positive terms e [rows, V]."""
    import torch

    rows = e.shape[0]
    nvec = V // 8
    K = (nvec + 511) // 512
    full = torch.zeros(rows, K * 512 * 8, dtype=e.dtype, device=e.device)
    full[:, :nvec * 8] = e[:, :nvec * 8]
    per = full.view(rows, K, 512, 8).permute(0, 2, 1, 3).reshape(rows, 512, K * 8)
    tail = torch.zeros(rows, 512, 1, dtype=e.dtype, device=e.device)
    tail[:, :V - nvec * 8, 0] = e[:, nvec * 8:]
    cum = torch.cat([per, tail], -1).cumsum(-1)
    return cum[..., 1:].abs().sum((-1, -2)) + _block_tree(cum[..., -1])


def _cross_entropy(B, S, V, ldv, in_place=False, ignore_frac=0.2, labels=None, scale=2.0, grad_scale=1.0):
    import torch

    from magma_b200 import ops

    name = f"cross_entropy B={B} S={S} V={V} ldv={ldv}"
    dev, bf = _dev(), torch.bfloat16
    gen = _gen("ce", B, S, V, ldv)
    M = B * S
    lg = torch.full((M + 2, ldv), float("nan"), dtype=bf, device=dev)  # NaN in the columns [V, ldv)
    lg[:M, :V] = (scale * torch.randn(M, V, generator=gen, dtype=torch.float64)).to(bf).to(dev)
    logits = lg[:M].view(B, S, ldv)
    if labels is None:
        labels = torch.randint(0, V, (B, S), generator=gen)
        labels[torch.rand(B, S, generator=gen) < ignore_frac] = -100
    labels = labels.to(dev)
    x = logits[..., :V].double().reshape(M, V)
    lab = labels.reshape(-1).cpu()
    tgt = torch.full((M,), -1, dtype=torch.long)
    for r in range(M):
        if r % S + 1 < S and 0 <= int(lab[r + 1]) < V:
            tgt[r] = int(lab[r + 1])
    valid = (tgt >= 0).to(dev)
    tgt = tgt.clamp(min=0).to(dev)
    n_valid = int(valid.sum().item())

    def run(inplace):
        snap = lg.clone()
        rl = torch.full((M + 8,), SENTINEL, dtype=torch.float32, device=dev)
        dst = snap if inplace else torch.full_like(lg, SENTINEL)
        lv = snap[:M].view(B, S, ldv)
        inp = _Inputs(labels, *(() if inplace else (snap,)))
        n0 = _count()
        loss, _ = ops.cross_entropy(lv, labels, V, grad_scale=grad_scale, dlogits=dst[:M].view(B, S, ldv),
                                    row_loss=rl[:M])
        _launched(name, n0, 3)
        inp.unchanged(name)
        assert bool((rl[M:] == SENTINEL).all()), f"{name}: row_loss written past B * S"
        if not inplace:
            assert _same(dst[M:], torch.full_like(dst[M:], SENTINEL)), f"{name}: dlogits written past B * S rows"
            assert _same(dst[:M, V:], torch.full_like(dst[:M, V:], SENTINEL)), f"{name}: dlogits written in [V, ldv)"
        else:
            assert _same(dst[:M, V:], lg[:M, V:]), f"{name}: the padding [V, ldv) of the logits was written"
        return loss, rl[:M], dst[:M, :V]

    loss, rl, dl = run(in_place)
    m = x.amax(1, keepdim=True)
    xm = x - m
    e = torch.exp(xm)
    ssum = e.sum(1, keepdim=True)
    p = e / ssum
    eps_exp = (2.0 + 1.173 * xm.abs()) * 2.0**-23 + U * xm.abs()
    eps_sum = 1.001 * ((e * eps_exp).sum(1, keepdim=True) + U * _ce_sum_terms(e, V)[:, None]) / ssum
    lse = m + torch.log(ssum)
    tl = x.gather(1, tgt[:, None])
    loss_ref = (lse - tl).squeeze(1)
    log_s = torch.log(ssum)
    d_lse = eps_sum * 1.001 + 2 * U * log_s.abs() + U * lse.abs()
    d_row = (d_lse + U * (lse - tl).abs()).squeeze(1) + TINY
    zero = torch.zeros_like(loss_ref)
    _check_bound(f"{name} row_loss", rl, torch.where(valid, loss_ref, zero), torch.where(valid, d_row, zero))
    assert _same(rl[~valid], torch.zeros_like(rl[~valid])), f"{name}: an ignored row's loss is not +0"
    nv = max(n_valid, 1)
    mean_ref = torch.where(valid, loss_ref, zero).sum() / nv
    d_mean = (torch.where(valid, d_row, zero).sum() + M * U * torch.where(valid, loss_ref, zero).abs().sum()) / nv
    _check_bound(f"{name} loss", loss, mean_ref.reshape(1), (1.001 * d_mean + U * mean_ref.abs() + TINY).reshape(1))
    gs = float(F32(grad_scale)) / nv
    onehot = torch.zeros_like(p).scatter_(1, tgt[:, None], 1.0)
    ref = (p - onehot) * gs
    delta = gs * (p * (eps_exp + eps_sum + 2 * U) + U * (p - onehot).abs()) + 2 * U * ref.abs()
    vrows = valid[:, None]
    check_rounded(f"{name} dlogits", dl, torch.where(vrows, ref, 0.0), 1.001 * delta + TINY, vrows, limit=AMBIGUOUS_MAX_EXP)
    assert _same(dl[~valid], torch.zeros_like(dl[~valid])), f"{name}: an ignored row's dlogits are not +0"
    _, rl2, dl2 = run(not in_place)
    assert _same(dl, dl2) and _same(rl, rl2), f"{name}: in-place and separate dlogits differ"
    return loss, dl


@pytest.mark.parametrize("in_place", [True, False], ids=["in_place", "separate"])
def test_cross_entropy_gptj_vocab(in_place):
    _cross_entropy(2, 150, 50400, 50432, in_place)


@pytest.mark.parametrize("B,S,V,ldv", [(8, 2048, 96, 96), (2, 9, 1003, 1008), (1, 5, 8, 8), (3, 4, 4100, 4104)])
def test_cross_entropy_shapes(B, S, V, ldv):
    _cross_entropy(B, S, V, ldv)


def test_cross_entropy_all_rows_ignored():
    import torch

    loss, dl = _cross_entropy(2, 6, 1003, 1008, labels=torch.full((2, 6), -100, dtype=torch.long))
    assert float(loss.item()) == 0.0


def test_cross_entropy_ignores_every_label_outside_the_vocabulary():
    """Labels V, ldv - 1, -1 and -100 are all ignored alike: the same loss and dlogits bits as four -100."""
    import torch

    V, ldv = 1003, 1008
    gen = _gen("ce_ignore")
    labels = torch.randint(0, V, (2, 8), generator=gen)
    odd = labels.clone()
    for (b, s), v in zip(((0, 2), (0, 5), (1, 1), (1, 6)), (V, ldv - 1, -1, -100)):
        odd[b, s] = v
        labels[b, s] = -100
    l1, d1 = _cross_entropy(2, 8, V, ldv, labels=odd, grad_scale=0.75)
    l2, d2 = _cross_entropy(2, 8, V, ldv, labels=labels, grad_scale=0.75)
    assert _same(l1, l2) and _same(d1, d2), f"loss {float(l1)} vs {float(l2)}"


# ---------------------------------------------------------------------------------------------
# C. column reductions and dot
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("rows,cols", [(16384, 4096), (2056, 1030), (63, 130), (1, 2)])
def test_colsum(rows, cols, accumulate):
    import torch

    from magma_b200 import ops

    name = f"colsum rows={rows} cols={cols} acc={int(accumulate)}"
    dev = _dev()
    gen = _gen("colsum", rows, cols, accumulate)
    xb = _nanbuf(rows, cols, torch.randn(rows, cols, generator=gen, dtype=torch.float64).to(torch.bfloat16).to(dev))
    base = torch.randn(cols, generator=gen, dtype=torch.float64).float().to(dev)
    outb = torch.full((cols + 8,), SENTINEL, dtype=torch.float32, device=dev)
    outb[:cols] = base
    inp = _Inputs(xb.storage)
    n0 = _count()
    ops.colsum(xb.view, out=outb[:cols], accumulate=accumulate)
    _launched(name, n0)
    inp.unchanged(name)
    assert bool((outb[cols:] == SENTINEL).all()), f"{name}: written past cols"
    s, e = _chunked_err(xb.view.double(), 64, base.double() if accumulate else None)
    _check_bound(name, outb[:cols], s, e)


@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("rows,cols", [(2056 * 49, 64), (300, 130), (1, 2)])
def test_col_moments(rows, cols, masked):
    import torch

    from magma_b200 import ops

    name = f"col_moments rows={rows} cols={cols} mask={int(masked)}"
    dev, bf = _dev(), torch.bfloat16
    gen = _gen("colmom", rows, cols, masked)

    def r(scale=1.0, off=0.0):
        return (off + scale * torch.randn(rows, cols, generator=gen, dtype=torch.float64)).to(bf).to(dev)

    ub, vb = _nanbuf(rows, cols, r(2.0, 0.5)), _nanbuf(rows, cols, r())
    mb = _nanbuf(rows, cols, r()) if masked else None
    inp = _Inputs(ub.storage, vb.storage, mb.storage if mb else None)
    n0 = _count()
    o1, o2 = ops.col_moments(ub.view, vb.view, mb.view if mb else None)
    _launched(name, n0)
    inp.unchanged(name)
    u = ub.view.double()
    if mb is not None:
        u = u * (mb.view.double() > 0)
    s1, e1 = _chunked_err(u, 128)
    t = u * vb.view.double()
    s2, e2 = _chunked_err(t, 128)
    _check_bound(f"{name} sum u", o1, s1, e1)
    _check_bound(f"{name} sum u v", o2, s2, e2 + 1.001 * U * t.abs().sum(0))


@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("n", [2056 * 1024, 4096 * 8 + 8, 8])
def test_dot(n, accumulate):
    import torch

    from magma_b200 import ops

    name = f"dot n={n} acc={int(accumulate)}"
    dev = _dev()
    gen = _gen("dot", n, accumulate)
    a = torch.randn(n, generator=gen, dtype=torch.float64).to(torch.bfloat16).to(dev)
    b = torch.randn(n, generator=gen, dtype=torch.float64).to(torch.bfloat16).to(dev)
    out = torch.full((2,), 3.25, dtype=torch.float32, device=dev)
    inp = _Inputs(a, b)
    n0 = _count()
    ops.dot(a, b, out[:1], accumulate=accumulate)
    _launched(name, n0)
    inp.unchanged(name)
    assert float(out[1]) == 3.25
    nvec = n // 8
    if dev.type == "cuda":
        sms = torch.cuda.get_device_properties(dev).multi_processor_count
        grid = min(max(1, min((nvec + 255) // 256, 16 * sms)), 1024)
    else:
        grid = max(1, min((nvec + 255) // 256, 4))
    K = (nvec + 256 * grid - 1) // (256 * grid)
    terms = torch.zeros(K * grid * 256 * 8, dtype=torch.float64, device=dev)
    terms[:n] = a.double() * b.double()
    per = terms.view(K, grid, 256, 8).permute(1, 2, 0, 3).reshape(grid, 256, K * 8)
    cum = per.cumsum(-1)
    blocks = cum[..., -1].sum(-1)
    start = 3.25 if accumulate else 0.0
    err = cum[..., 1:].abs().sum() + _block_tree(cum[..., -1]).sum() + (grid + 1) * (blocks.abs().sum() + abs(start))
    ref = terms.sum() + start
    _check_bound(name, out[:1], ref.reshape(1), (1.001 * U * (err + terms.abs().sum()) + TINY).reshape(1))


# ---------------------------------------------------------------------------------------------
# D. rounded element-wise kernels
# ---------------------------------------------------------------------------------------------
def _rounded(name, got, ref, delta, limit=AMBIGUOUS_MAX):
    import torch

    check_rounded(name, got, ref, 1.001 * delta + TINY, torch.ones(1, dtype=torch.bool, device=ref.device), limit=limit)


def test_quick_gelu_bwd(n=None):
    """n: the element count (tests/test_production_launches_gpu.py replays the production one)."""
    import torch

    from magma_b200 import ops

    name = "quick_gelu_bwd"
    dev, bf = _dev(), torch.bfloat16
    n = n or (1 << 18 if dev.type == "cuda" else 4096)
    gen = _gen("qgelu", n)
    pre = torch.linspace(-20, 20, n, dtype=torch.float64).to(bf).to(dev)
    dy = torch.randn(n, generator=gen, dtype=torch.float64).to(bf).to(dev)
    out = torch.full((n + 64,), SENTINEL, dtype=bf, device=dev)
    inp = _Inputs(pre, dy)
    n0 = _count()
    ops.quick_gelu_bwd(dy, pre, out=out[:n])
    _launched(name, n0)
    inp.unchanged(name)
    assert _same(out[n:], torch.full((64,), SENTINEL, dtype=bf, device=dev)), f"{name}: written past n"
    k = float(F32(1.702))
    x, g = pre.double(), dy.double()
    t = -k * x
    E = torch.exp(t)
    s = 1.0 / (1.0 + E)
    eps_s = (E / (1 + E)) * ((2.0 + 1.173 * t.abs()) * 2.0**-23 + U * t.abs()) + 2 * U
    ds = eps_s * s
    oms = 1 - s
    d_oms = ds + U * oms.abs()
    kx = k * x
    Bt = kx * s * oms
    dBt = kx.abs() * (s * oms * 3 * U + ds * oms + s * d_oms)
    inner = s + Bt
    ref = g * inner
    _rounded(name, out[:n], ref, g.abs() * (ds + dBt + U * inner.abs()) + U * ref.abs(), AMBIGUOUS_MAX_EXP)
    buf = dy.clone()
    ops.quick_gelu_bwd(buf, pre, out=buf)
    assert _same(buf, out[:n]), f"{name}: in place differs"


@pytest.mark.parametrize("with_s,with_r1,with_r2", [(1, 1, 1), (1, 0, 0), (0, 1, 0), (0, 0, 0)])
def test_scale_add(with_s, with_r1, with_r2):
    import torch

    from magma_b200 import ops

    name = f"scale_add s={with_s} r1={with_r1} r2={with_r2}"
    dev, bf = _dev(), torch.bfloat16
    n = 1024 * 4096 if dev.type == "cuda" else 4096
    gen = _gen("scale_add", with_s, with_r1, with_r2)
    u, r1, r2 = (torch.randn(n, generator=gen, dtype=torch.float64).to(bf).to(dev) for _ in range(3))
    s = torch.tensor([0.3712], dtype=torch.float32, device=dev) if with_s else None
    r1, r2 = (r1 if with_r1 else None), (r2 if with_r2 else None)
    out = torch.full((n + 64,), SENTINEL, dtype=bf, device=dev)
    inp = _Inputs(u, s, r1, r2)
    n0 = _count()
    ops.scale_add(u, s, r1, r2, out=out[:n])
    _launched(name, n0)
    inp.unchanged(name)
    assert _same(out[n:], torch.full((64,), SENTINEL, dtype=bf, device=dev))
    a = u.double() * (s.double() if with_s else 1.0)
    d = U * a.abs() if with_s else torch.zeros_like(a)
    q = _quantum(u.double()) if not with_s else torch.zeros_like(a)  # u * s rounds to an fp32 value: no quantum
    for r in (r1, r2):
        if r is not None:
            q = torch.minimum(q, _quantum(r.double()))
            a = a + r.double()
            d = d + _add_err(a, q)
    _rounded(name, out[:n], a, d)
    out2 = ops.scale_add(u, s, r1, r2)
    assert _same(out2, out[:n]), f"{name}: rerun differs"


@pytest.mark.parametrize("with_c", [False, True])
def test_add(with_c):
    import torch

    from magma_b200 import ops

    name = f"add c={int(with_c)}"
    dev, bf = _dev(), torch.bfloat16
    n = 1024 * 4096 if dev.type == "cuda" else 4096
    gen = _gen("add", with_c)
    a, b, c = (torch.randn(n, generator=gen, dtype=torch.float64).to(bf).to(dev) for _ in range(3))
    c = c if with_c else None
    out = torch.full((n + 64,), SENTINEL, dtype=bf, device=dev)
    inp = _Inputs(a, b, c)
    n0 = _count()
    ops.add(a, b, c, out=out[:n])
    _launched(name, n0)
    inp.unchanged(name)
    assert _same(out[n:], torch.full((64,), SENTINEL, dtype=bf, device=dev))
    a64, b64 = a.double(), b.double()
    q = torch.minimum(_quantum(a64), _quantum(b64))
    bc, d = b64, 0.0
    if with_c:
        c64 = c.double()
        q = torch.minimum(q, _quantum(c64))
        bc = b64 + c64
        d = _add_err(bc, torch.minimum(_quantum(b64), _quantum(c64)))
    ref = a64 + bc
    _rounded(name, out[:n], ref, d + _add_err(ref, q))


def test_vit_assemble(shape=None):
    """shape: (B, T, w) (tests/test_production_launches_gpu.py replays the production one)."""
    import torch

    from magma_b200 import ops

    dev, bf = _dev(), torch.bfloat16
    B, T, w = shape or ((2, 257, 1024) if dev.type == "cuda" else (2, 5, 16))
    name = f"vit_assemble B={B} T={T} w={w}"
    gen = _gen("vit_assemble", B, T, w)
    pe, cls, pos = (torch.randn(*s, generator=gen, dtype=torch.float64).to(bf).to(dev)
                    for s in ((B, T - 1, w), (w,), (T, w)))
    x = torch.full((B + 1, T, w), SENTINEL, dtype=bf, device=dev)
    inp = _Inputs(pe, cls, pos)
    n0 = _count()
    ops.vit_assemble(x[:B], pe, cls, pos)
    _launched(name, n0)
    inp.unchanged(name)
    assert _same(x[B:], torch.full_like(x[B:], SENTINEL))
    base = torch.cat([cls.double().expand(B, 1, w), pe.double()], 1)
    ref = base + pos.double()
    _rounded(name, x[:B], ref, _add_err(ref, torch.minimum(_quantum(base), _quantum(pos.double()))))


@pytest.mark.parametrize("B,H,W,C,k", [(2, 48, 48, 256, 2), (1, 7, 9, 8, 3), (3, 4, 4, 16, 4), (1, 1, 1, 8, 1)])
def test_avgpool_fwd_bwd(B, H, W, C, k):
    import torch

    from magma_b200 import ops

    name = f"avgpool B={B} H={H} W={W} C={C} k={k}"
    dev, bf = _dev(), torch.bfloat16
    gen = _gen("avgpool", B, H, W, C, k)
    x = torch.randn(B, H, W, C, generator=gen, dtype=torch.float64).to(bf).to(dev)
    Ho, Wo = H // k, W // k
    out = torch.full((B + 1, Ho, Wo, C), SENTINEL, dtype=bf, device=dev)
    inp = _Inputs(x)
    n0 = _count()
    ops.avgpool_nhwc(x, k, out=out[:B])
    _launched(name, n0)
    inp.unchanged(name)
    assert _same(out[B:], torch.full_like(out[B:], SENTINEL))
    win = x.double()[:, :Ho * k, :Wo * k].reshape(B, Ho, k, Wo, k, C).permute(0, 1, 3, 2, 4, 5).reshape(B, Ho, Wo, k * k, C)
    cum = win.cumsum(3)
    qm = _quantum(win).cummin(3).values
    ref = cum[:, :, :, -1] / (k * k)
    scale_err = 0.0 if (k * k) & (k * k - 1) == 0 else 2 * U  # fl(1 / k^2) and the product are exact for k^2 = 2^j
    _rounded(name, out[:B], ref, _add_err(cum[:, :, :, 1:], qm[:, :, :, 1:]).sum(3) / (k * k) + scale_err * ref.abs())
    # backward
    dy = torch.randn(B, Ho, Wo, C, generator=gen, dtype=torch.float64).to(bf).to(dev)
    dx = torch.full((B + 1, H, W, C), SENTINEL, dtype=bf, device=dev)
    inp = _Inputs(dy)
    n0 = _count()
    ops.avgpool_nhwc_bwd(dy, H, W, k, out=dx[:B])
    _launched(name + " bwd", n0)
    inp.unchanged(name)
    assert _same(dx[B:], torch.full_like(dx[B:], SENTINEL))
    ref = torch.zeros(B, H, W, C, dtype=torch.float64, device=dev)
    ref[:, :Ho * k, :Wo * k] = dy.double().repeat_interleave(k, 1).repeat_interleave(k, 2) / (k * k)
    _rounded(name + " bwd", dx[:B], ref, scale_err * ref.abs())
    assert _same(dx[:B, Ho * k:], torch.zeros_like(dx[:B, Ho * k:])) and \
        _same(dx[:B, :, Wo * k:], torch.zeros_like(dx[:B, :, Wo * k:])), f"{name}: uncovered pixels are not +0"


def _im2col_ref(x, stride):
    import torch

    B, H, W, C = x.shape
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    xp = torch.zeros(B, H + 2, W + 2, C, dtype=x.dtype, device=x.device)
    xp[:, 1:H + 1, 1:W + 1] = x
    taps = [xp[:, kh:kh + stride * (Ho - 1) + 1:stride, kw:kw + stride * (Wo - 1) + 1:stride]
            for kh in range(3) for kw in range(3)]
    return torch.stack(taps, 3).reshape(B * Ho * Wo, 9 * C), Ho, Wo


CONV_SHAPES = [(2, 24, 24, 64, 1), (2, 24, 24, 64, 2), (1, 7, 5, 8, 2), (2, 5, 9, 16, 1), (1, 1, 6, 8, 1), (3, 1, 1, 8, 2)]


@pytest.mark.parametrize("B,H,W,C,s", CONV_SHAPES)
def test_im2col_col2im(B, H, W, C, s):
    import torch

    from magma_b200 import ops

    name = f"im2col3x3 B={B} H={H} W={W} C={C} stride={s}"
    dev, bf = _dev(), torch.bfloat16
    gen = _gen("im2col", B, H, W, C, s)
    x = torch.randn(B, H, W, C, generator=gen, dtype=torch.float64).to(bf).to(dev)
    ref, Ho, Wo = _im2col_ref(x, s)
    out = torch.full((B * Ho * Wo + 3, 9 * C), SENTINEL, dtype=bf, device=dev)
    inp = _Inputs(x)
    n0 = _count()
    ops.im2col3x3(x, s, out=out[:B * Ho * Wo])
    _launched(name, n0)
    inp.unchanged(name)
    assert _same(out[B * Ho * Wo:], torch.full_like(out[B * Ho * Wo:], SENTINEL))
    assert _same(out[:B * Ho * Wo], ref), f"{name}: not bit-identical to the float64 gather"
    # col2im3x3: the adjoint, summing the taps in (kh, kw) order
    dcols = torch.randn(B * Ho * Wo, 9 * C, generator=gen, dtype=torch.float64).to(bf).to(dev)
    dx = torch.full((B + 1, H, W, C), SENTINEL, dtype=bf, device=dev)
    inp = _Inputs(dcols)
    n0 = _count()
    ops.col2im3x3(dcols, B, H, W, C, s, out=dx[:B])
    _launched(name + " col2im", n0)
    inp.unchanged(name)
    assert _same(dx[B:], torch.full_like(dx[B:], SENTINEL))
    dc = dcols.double().view(B, Ho, Wo, 3, 3, C)
    acc = torch.zeros(B, H + 2, W + 2, C, dtype=torch.float64, device=dev)
    err = torch.zeros_like(acc)
    qm = torch.full_like(acc, math.inf)
    for kh in range(3):
        for kw in range(3):
            sl = (slice(None), slice(kh, kh + s * (Ho - 1) + 1, s), slice(kw, kw + s * (Wo - 1) + 1, s))
            t = dc[:, :, :, kh, kw]
            acc[sl] += t
            qm[sl] = torch.minimum(qm[sl], _quantum(t))
            err[sl] += _add_err(acc[sl], qm[sl])
    ref = acc[:, 1:H + 1, 1:W + 1]
    _rounded(name + " col2im", dx[:B], ref, err[:, 1:H + 1, 1:W + 1])


@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("full", [False, True])
def test_channel_affine(full, relu):
    import torch

    from magma_b200 import ops

    name = f"channel_affine full={int(full)} relu={int(relu)}"
    dev, bf = _dev(), torch.bfloat16
    rows, C = (4096, 256) if dev.type == "cuda" else (40, 24)
    gen = _gen("chaff", full, relu)

    def r():
        return torch.randn(rows, C, generator=gen, dtype=torch.float64).to(bf).to(dev)

    def c():
        return torch.randn(C, generator=gen, dtype=torch.float64).float().to(dev)

    x1, a1 = r(), c()
    x2, a2, c0, mask, res = (r(), c(), c(), r(), r()) if full else (None,) * 5
    out = torch.full((rows + 3, C), SENTINEL, dtype=bf, device=dev)
    inp = _Inputs(x1, a1, x2, a2, c0, mask, res)
    n0 = _count()
    ops.channel_affine(x1, a1, x2, a2, c0, mask, res, relu, out=out[:rows])
    _launched(name, n0)
    inp.unchanged(name)
    assert _same(out[rows:], torch.full_like(out[rows:], SENTINEL))
    f = x1.double()
    if full:
        f = f * (mask.double() > 0)
    t = f * a1.double()
    d = U * t.abs()
    if full:
        t = t + c0.double()
        d = d + U * t.abs()
        p2 = x2.double() * a2.double()
        t = t + p2
        d = d + U * (p2.abs() + t.abs())
        t = t + res.double()
        d = d + U * t.abs()
    if relu:  # relu(fl(t)) lies between relu(t - d) and relu(t + d)
        lo, hi = (t - d).clamp(min=0), (t + d).clamp(min=0)
        t, d = (lo + hi) / 2, (hi - lo) / 2
    _rounded(name, out[:rows], t, d)


# ---------------------------------------------------------------------------------------------
# E. bit-exact layout, gathers, casts, dropout, argmax
# ---------------------------------------------------------------------------------------------
def test_patchify_vit_front_end(shape=None):
    """shape: (B, R, P) (tests/test_production_launches_gpu.py replays the production one)."""
    import torch

    from magma_b200 import ops

    dev, bf = _dev(), torch.bfloat16
    B, R, P = shape or ((2, 224, 14) if dev.type == "cuda" else (2, 28, 14))
    g = R // P
    K = 3 * P * P
    name = f"patchify B={B} R={R} P={P}"
    img = torch.randn(B, 3, R, R, generator=_gen("patchify"), dtype=torch.float64).to(bf).to(dev)
    pb = Buf((), B * g * g, K, bf, dev, SENTINEL)
    inp = _Inputs(img)
    n0 = _count()
    ops.patchify(img, P, pb.view)
    _launched(name, n0)
    inp.unchanged(name)
    _untouched(name, ("patches", pb))
    ref = img.view(B, 3, g, P, g, P).permute(0, 2, 4, 1, 3, 5).reshape(B * g * g, K)
    assert _same(pb.view, ref), f"{name}: not bit-identical"


@pytest.mark.parametrize("C", [3, 8, 1])
def test_nchw_to_nhwc8(C):
    import torch

    from magma_b200 import ops

    dev, bf = _dev(), torch.bfloat16
    B, H, W = 2, 17, 9
    x = torch.randn(B, C, H, W, generator=_gen("nhwc8", C), dtype=torch.float64).to(bf).to(dev)
    x[0, 0, 0, 0] = -0.0
    out = torch.full((B + 1, H, W, 8), SENTINEL, dtype=bf, device=dev)
    inp = _Inputs(x)
    n0 = _count()
    ops.nchw_to_nhwc8(x, out=out[:B])
    _launched("nchw_to_nhwc8", n0)
    inp.unchanged("nchw_to_nhwc8")
    assert _same(out[B:], torch.full_like(out[B:], SENTINEL))
    assert _same(out[:B, ..., :C], x.permute(0, 2, 3, 1))
    assert int((bits(out[:B, ..., C:]) != 0).sum()) == 0, "channels C..7 are not +0"


def _gather_ids(gen, n, V):
    import torch

    ids = torch.randint(0, V, (n,), generator=gen)
    ids[:4] = torch.tensor([-1, V, V + 5, -100])
    ids[4], ids[5] = 0, V - 1
    return ids


def test_embed_assemble_and_gather():
    import torch

    from magma_b200 import ops

    dev, bf = _dev(), torch.bfloat16
    V, d = 1000, 256
    gen = _gen("embed")
    wte = torch.randn(V, d, generator=gen, dtype=torch.float64).to(bf).to(dev)
    for B, S, L in ((3, 12, 4), (2, 7, 0), (2, 5, 5)):
        name = f"embed_assemble B={B} S={S} L={L}"
        caps = _gather_ids(gen, B * (S - L + 3), V).view(B, S - L + 3).to(dev)
        prefix = torch.randn(B, L, d, generator=gen, dtype=torch.float64).to(bf).to(dev) if L else None
        out = torch.full((B + 1, S, d), SENTINEL, dtype=bf, device=dev)
        inp = _Inputs(wte, caps, prefix)
        n0 = _count()
        ops.embed_assemble(caps, wte, prefix, S=S, out=out[:B])
        _launched(name, n0)
        inp.unchanged(name)
        assert _same(out[B:], torch.full_like(out[B:], SENTINEL))
        ids = caps[:, :S - L]
        ids = torch.where((ids < 0) | (ids >= V), 0, ids)
        ref = wte[ids]
        if L:
            ref = torch.cat([prefix, ref], 1)
        assert _same(out[:B], ref), f"{name}: not bit-identical"
    ids = _gather_ids(gen, 37, V).to(dev)
    out = torch.full((38, d), SENTINEL, dtype=bf, device=dev)
    n0 = _count()
    ops.embed_gather(ids, wte, out=out[:37])
    _launched("embed_gather", n0)
    assert _same(out[37:], torch.full_like(out[37:], SENTINEL))
    assert _same(out[:37], wte[torch.where((ids < 0) | (ids >= V), 0, ids)])


def test_casts():
    import torch

    from magma_b200 import ops

    dev = _dev()
    specials = [0.0, -0.0, math.inf, -math.inf, math.nan, 1e-40, -3e-42, 2.0**-149, 2.0**-126, 1.17e-38,
                3.4e38, -3.39e38, 3.3961e38, float.fromhex("0x1.fefffep+127"), 65504.0]
    ties = [float(np.array([b], dtype=np.uint32).view(np.float32)[0])
            for b in (0x3F808000, 0x3F818000, 0xBF808000, 0x00008000, 0x00018000, 0x7F7F8000)]
    rnd = torch.randn(100000, generator=_gen("cast"), dtype=torch.float64) * 10.0 ** torch.randint(-40, 38, (100000,),
                                                                                                     generator=_gen("e"))
    src = torch.cat([torch.tensor(specials + ties, dtype=torch.float64), rnd]).float().to(dev)
    n = src.numel()
    out = torch.full((n + 8,), SENTINEL, dtype=torch.bfloat16, device=dev)
    inp = _Inputs(src)
    n0 = _count()
    ops.cast_f32_to_bf16(src, out[:n])
    _launched("cast_f32_to_bf16", n0)
    inp.unchanged("cast_f32_to_bf16")
    assert _same(out[n:], torch.full((8,), SENTINEL, dtype=torch.bfloat16, device=dev))
    s64 = src.double()
    ref = bf16_rne(s64)
    ref = torch.where(ref.abs() >= 2.0**128, torch.copysign(torch.full_like(ref, math.inf), s64), ref)
    ref = torch.where(s64.isinf(), s64, ref)
    got = out[:n].double()
    fin = ~s64.isnan()
    assert bool(got[~fin].isnan().all()), "cast_f32_to_bf16: NaN did not stay NaN"
    bad = (got[fin] != ref[fin]) | (torch.signbit(got[fin]) != torch.signbit(ref[fin]))
    assert int(bad.sum()) == 0, f"cast_f32_to_bf16: {int(bad.sum())} values not RNE, first {s64[fin][bad][:4].tolist()}"
    # bf16 -> fp32 is exact (every bf16 bit pattern, NaN payloads included)
    allb = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(torch.bfloat16).to(dev)
    f = torch.full((65536 + 8,), SENTINEL, dtype=torch.float32, device=dev)
    n0 = _count()
    ops.cast_bf16_to_f32(allb, f[:65536])
    _launched("cast_bf16_to_f32", n0)
    assert bool((f[65536:] == SENTINEL).all())
    want = allb.view(torch.int16).to(torch.int64).bitwise_and(0xFFFF).bitwise_left_shift(16)
    got = f[:65536].view(torch.int32).to(torch.int64).bitwise_and(0xFFFFFFFF)
    assert torch.equal(got, want), "cast_bf16_to_f32 is not a bit shift"


def _hash32(k):
    k = k ^ (k >> np.uint64(33))
    k = k * np.uint64(0xFF51AFD7ED558CCD)
    k = k ^ (k >> np.uint64(33))
    k = k * np.uint64(0xC4CEB9FE1A85EC53)
    k = k ^ (k >> np.uint64(33))
    return (k & np.uint64(0xFFFFFFFF)).astype(np.uint32)


@pytest.mark.parametrize("p", [0.0, 0.1, 0.5, 0.9])
def test_dropout(p):
    import torch

    from magma_b200 import ops

    dev, bf = _dev(), torch.bfloat16
    n = (1 << 20) + 3 if dev.type == "cuda" else 5000
    seed = 0x1234_5678_9ABC + int(p * 10)
    name = f"dropout p={p}"
    x = torch.randn(n, generator=_gen("dropout", p), dtype=torch.float64).to(bf).to(dev)
    y = torch.full((n + 8,), SENTINEL, dtype=bf, device=dev)
    inp = _Inputs(x)
    n0 = _count()
    _, mask = ops.dropout_fwd(x, p, seed, out=y[:n])
    _launched(name, n0)
    inp.unchanged(name)
    assert _same(y[n:], torch.full((8,), SENTINEL, dtype=bf, device=dev))
    with np.errstate(over="ignore"):
        k = np.uint64(seed) * np.uint64(0x9E3779B97F4A7C15) + np.arange(n, dtype=np.uint64)
    u = (_hash32(k) >> np.uint32(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)
    keep = torch.from_numpy((u >= np.float32(p)).astype(np.uint8))
    assert torch.equal(mask.cpu(), keep), f"{name}: mask differs from the hash restatement"
    scale = torch.tensor(np.float32(1.0) / (np.float32(1.0) - np.float32(p)))
    ref = torch.where(keep.bool(), x.cpu().float() * scale, torch.zeros(n)).to(bf)
    assert _same(y[:n].cpu(), ref), f"{name}: y != RNE(fl(x * fl(1 / (1 - p))))"
    if p == 0.0:
        assert _same(y[:n], x), "dropout p = 0 is not the identity"
    y2 = torch.full((n + 8,), SENTINEL, dtype=bf, device=dev)
    n0 = _count()
    ops.dropout_apply(x, mask, p, out=y2[:n])
    _launched(name + " apply", n0)
    assert _same(y2, y), f"{name}: dropout_apply with the forward's mask differs from the forward"


def _argmax_case(name, x, V):
    import torch

    from magma_b200 import ops

    rows = x.shape[0]
    out = torch.full((rows + 2,), -7, dtype=torch.int64, device=x.device)
    inp = _Inputs(x)
    n0 = _count()
    ops.argmax(x, V, out=out[:rows])
    _launched(name, n0)
    inp.unchanged(name)
    assert bool((out[rows:] == -7).all())
    return out[:rows]


def test_argmax():
    import torch

    dev, bf = _dev(), torch.bfloat16
    gen = _gen("argmax")
    for V, ld in ((50400, 50432), (100, 104), (511, 512), (513, 520), (1, 8)):
        rows = 9
        store = torch.randn(rows, ld, generator=gen, dtype=torch.float64).to(bf)
        store[:, V:] = 1e30  # larger values in the padding, which must be ignored
        store[0, 0] = 1e20
        store[1, V - 1] = 1e20
        mx = store[2, :V].max()
        store[2, V // 3], store[2, V - 1] = mx + 1, mx + 1  # a tie: the lower index wins
        store[3, :V] = -math.inf
        store[4, :V] = 2.5  # all equal
        x = store.to(dev)
        got = _argmax_case(f"argmax V={V} ld={ld}", x, V)
        want = torch.argmax(store[:, :V].float(), -1)
        assert torch.equal(got.cpu(), want), f"argmax V={V}: {got.cpu().tolist()} vs {want.tolist()}"
    # NaN entries never win; an all-NaN row returns 2^31 - 1
    store = torch.randn(2, 64, generator=gen, dtype=torch.float64).to(bf)
    store[0, 5] = math.nan
    store[1, :] = math.nan
    got = _argmax_case("argmax NaN", store.to(dev), 64)
    assert int(got[0]) == int(torch.argmax(torch.nan_to_num(store[0].float(), nan=-math.inf)))
    assert int(got[1]) == 2**31 - 1


# ---------------------------------------------------------------------------------------------
# F. rotary table, BatchNorm bookkeeping, AdamW
# ---------------------------------------------------------------------------------------------
def _torch_inv_freq(rot):
    import torch

    return 1.0 / (10000 ** (torch.arange(0, rot, 2, dtype=torch.int64).float() / rot))


@pytest.mark.parametrize("S,rot,pos0", [(2048, 64, 0), (7, 64, 2040), (300, 128, 5), (1, 2, 0)])
def test_rope_table(S, rot, pos0):
    import torch

    from magma_b200 import ops

    name = f"rope_table S={S} rot={rot} pos0={pos0}"
    dev = _dev()
    n0 = _count()
    tab = ops.rope_table(S, rot, pos0, device=dev)
    _launched(name, n0)
    inv = _torch_inv_freq(rot).to(dev)
    pos = torch.arange(pos0, pos0 + S, dtype=torch.float32, device=dev)
    theta = (pos[:, None] * inv[None, :]).double()  # fl(pos * inv_freq), as GPT-J forms it
    dth = pos.double()[:, None] * 12.0 * U * inv.double()[None, :] + 2 * U * theta.abs()
    c, s = torch.cos(theta), torch.sin(theta)
    _check_bound(f"{name} cos", tab[..., 0], c, 1.001 * (dth + 2 * _ulp32(c.abs() + dth)) + TINY)
    _check_bound(f"{name} sin", tab[..., 1], s, 1.001 * (dth + 2 * _ulp32(s.abs() + dth)) + TINY)
    if dev.type == "cuda":
        out = torch.full((S + 1, rot // 2, 2), SENTINEL, dtype=torch.float32, device=dev)
        p0 = torch.tensor([pos0], dtype=torch.int32, device=dev)
        n0 = _count()
        ops.rope_table_dev(S, rot, p0, out=out[:S])
        _launched(name + " dev", n0)
        assert _same(out[:S], tab), f"{name}: rope_table_dev differs from rope_table"
        assert bool((out[S:] == SENTINEL).all())


@pytest.mark.parametrize("ratio", [0.0, 1.0, 4.0])
def test_bn_finalize_and_bwd_coeffs(ratio):
    import torch

    from magma_b200 import ops

    name = f"bn |mean|/std={ratio}"
    dev = _dev()
    gen = _gen("bn", ratio)
    C, R = 256, 2056 * 49
    std = 0.5 + torch.rand(C, generator=gen, dtype=torch.float64)
    mu = ratio * std * torch.where(torch.rand(C, generator=gen) < 0.5, -1.0, 1.0)
    z = mu + std * torch.randn(512, C, generator=gen, dtype=torch.float64)  # the moments of R rows, drawn at 512
    s1 = (z.mean(0) * R).float().to(dev)
    s2 = ((z * z).mean(0) * R).float().to(dev)
    gamma = (1 + 0.1 * torch.randn(C, generator=gen, dtype=torch.float64)).float().to(dev)
    beta = (0.1 * torch.randn(C, generator=gen, dtype=torch.float64)).float().to(dev)
    rm0 = (0.1 * torch.randn(C, generator=gen, dtype=torch.float64)).float().to(dev)
    rv0 = (1 + 0.2 * torch.rand(C, generator=gen, dtype=torch.float64)).float().to(dev)
    rm, rv = rm0.clone(), rv0.clone()
    eps, mom = float(F32(1e-5)), float(F32(0.1))
    inp = _Inputs(s1, s2, gamma, beta)
    n0 = _count()
    mean, rstd, scale, shift = ops.bn_finalize_fwd(s1, s2, gamma, beta, R, 1e-5, 0.1, rm, rv)
    _launched(name, n0)
    inp.unchanged(name)
    S1, S2, g, b = s1.double(), s2.double(), gamma.double(), beta.double()
    m = S1 / R
    e2 = S2 / R
    var = (e2 - m * m).clamp(min=0)
    dm = 2.001 * U * m.abs()
    dvar = 2.001 * U * e2 + 5.001 * U * m * m + U * var
    v = var + eps
    dv = dvar + U * v
    r = 1.0 / v.sqrt()
    er = 1.001 * (0.5 * dv / v + 4 * U)
    _check_bound(f"{name} mean", mean, m, dm + TINY)
    rr = _check_bound(f"{name} rstd", rstd, r, r * er + TINY)
    err_rstd = float(((rstd.double() - r).abs() / r).max())
    print(f"[bn] |mean|/std={ratio}: measured rstd relative error {err_rstd:.3g} (bound ratio {rr:.3f})")
    sc = g * r
    dsc = sc.abs() * (er + U) * 1.001
    _check_bound(f"{name} scale", scale, sc, dsc + TINY)
    sh = b - m * sc
    _check_bound(f"{name} shift", shift, sh, 1.001 * (m.abs() * dsc + sc.abs() * dm + U * (m * sc).abs() + U * sh.abs()) + TINY)
    unb = R / (R - 1)
    rm_ref = (1 - mom) * rm0.double() + mom * m
    d_rm = 1.001 * (U * (1 - mom) * rm0.double().abs() + mom * (dm + 2 * U * m.abs()) + U * rm_ref.abs()) + TINY
    _check_bound(f"{name} running_mean", rm, rm_ref, d_rm + U * (1 - mom) * rm0.double().abs())
    rv_ref = (1 - mom) * rv0.double() + mom * var * unb
    d_rv = 1.001 * (2 * U * (1 - mom) * rv0.double().abs() + mom * unb * (dvar + 4 * U * var) + U * rv_ref.abs()) + TINY
    _check_bound(f"{name} running_var", rv, rv_ref, d_rv)
    # backward coefficients from the kernel's own mean / rstd
    t = (S1 * 0.3 + 0.7 * std.to(dev) * R).float()
    d1 = (0.01 * R * torch.randn(C, generator=gen, dtype=torch.float64)).float().to(dev)
    dg0 = torch.randn(C, generator=gen, dtype=torch.float64).float().to(dev)
    db0 = torch.randn(C, generator=gen, dtype=torch.float64).float().to(dev)
    for acc in (False, True):
        dg, db = dg0.clone(), db0.clone()
        n0 = _count()
        A, Bc, Cc = ops.bn_bwd_coeffs(d1, t, mean, rstd, gamma, R, dg, db, accumulate=acc)
        _launched(name + " bwd", n0)
        mk, rk, D1, T = mean.double(), rstd.double(), d1.double(), t.double()
        inr = 1.0 / R
        inner = T - mk * D1
        s2r = rk * inner
        ds2 = 1.001 * (rk * U * ((mk * D1).abs() + inner.abs()) + U * s2r.abs())
        gref = (dg0.double() if acc else 0) + s2r
        _check_bound(f"{name} dgamma acc={int(acc)}", dg, gref, ds2 + U * gref.abs() + TINY)
        bref = (db0.double() if acc else 0) + D1
        _check_bound(f"{name} dbeta acc={int(acc)}", db, bref, U * bref.abs() + TINY)
        a = g * rk
        _check_bound(f"{name} A", A, a, U * a.abs() + TINY)
        k2 = a * rk * s2r * inr
        dk2 = 1.001 * (4 * U * k2.abs() + (a * rk * inr).abs() * ds2) + TINY
        _check_bound(f"{name} Bc", Bc, -k2, dk2)
        c3 = a * D1 * inr
        cc = k2 * mk - c3
        dcc = 1.001 * (dk2 * mk.abs() + U * (k2 * mk).abs() + 3 * U * c3.abs() + U * cc.abs()) + TINY
        _check_bound(f"{name} Cc", Cc, cc, dcc)


def _adamw_step_ref(w, g, m, v, lr, b1, b2, eps, wd, gs, gn, max_norm, step):
    """float64 AdamW step from the fp32 state and its bound (w, m, v, and their bounds)."""
    import torch

    p1, p2 = b1**step, b2**step
    bc1, bc2 = 1 - p1, 1 - p2
    e_bc1 = (2 * U * p1 + U * bc1) / bc1
    e_bc2 = (2 * U * p2 + U * bc2) / bc2
    stp, e_stp = lr / bc1, e_bc1 + U
    isb, e_isb = 1 / math.sqrt(bc2), 0.5 * e_bc2 + 4 * U
    decay = 1 - lr * wd
    d_decay = U * lr * wd + U * decay
    coef, e_coef = gs, 0.0
    if gn is not None and max_norm > 0:
        ratio = max_norm / (math.sqrt(gn) * gs + float(F32(1e-6)))
        coef, e_coef = gs * min(1.0, ratio), 5.001 * U
    gi = g * coef
    dgi = gi.abs() * (e_coef + U)
    wi = w * decay
    dwi = w.abs() * (d_decay + U * decay)
    a = b1 * m + (1 - b1) * gi
    da = U * (b1 * m).abs() + (1 - b1) * (dgi + U * gi.abs()) + U * a.abs()
    vv = b2 * v + (1 - b2) * gi * gi
    dvv = U * (b2 * v).abs() + (1 - b2) * (2 * gi.abs() * dgi + 2 * U * gi * gi) + U * vv
    sq = vv.sqrt()
    dsq = torch.minimum(dvv / (2 * sq).clamp(min=1e-300), dvv.sqrt()) + U * sq
    den = sq * isb + eps
    dden = isb * dsq + sq * isb * (e_isb + U) + U * den
    q = a / den
    dq = (da + q.abs() * dden) / den + U * q.abs()
    upd = stp * q
    dupd = stp * dq + upd.abs() * (e_stp + U)
    w2 = wi - upd
    dw = dwi + dupd + U * w2.abs()
    return w2, a, vv, 1.01 * dw + TINY, 1.01 * da + TINY, 1.01 * dvv + TINY


@pytest.mark.parametrize("case", ["plain", "clip_scale", "late_step", "no_decay_no_zero"])
def test_adamw(case):
    import torch

    from magma_b200 import ops

    name = f"adamw {case}"
    dev = _dev()
    n = (1 << 20) + 64 if dev.type == "cuda" else 4096
    gen = _gen("adamw", case)
    lr, b1, b2, eps = (float(F32(v)) for v in (1e-3, 0.9, 0.95, 1e-8))
    wd = 0.0 if case == "no_decay_no_zero" else float(F32(0.1))
    gs = float(F32(0.5)) if case == "clip_scale" else 1.0
    max_norm = float(F32(1.0)) if case == "clip_scale" else 0.0
    step0 = 1000 if case == "late_step" else 1
    zero_grad = case != "no_decay_no_zero"
    w0 = torch.randn(n, generator=gen, dtype=torch.float64).float().to(dev)
    m0 = torch.zeros(n, device=dev) if step0 == 1 else (0.01 * torch.randn(n, generator=gen, dtype=torch.float64)).float().to(dev)
    v0 = torch.zeros(n, device=dev) if step0 == 1 else (1e-4 * torch.rand(n, generator=gen, dtype=torch.float64)).float().to(dev)
    grads = [(0.1 * torch.randn(n, generator=gen, dtype=torch.float64)).float().to(dev) for _ in range(3)]

    def run(cap):
        if cap is not None:
            ops.set_optimizer_grid(cap)
        try:
            w, m, v = w0.clone(), m0.clone(), v0.clone()
            sh = torch.full((n + 8,), SENTINEL, dtype=torch.bfloat16, device=dev)
            states = []
            for k, g0 in enumerate(grads):
                g = g0.clone()
                gn = torch.tensor([float((g0.double() ** 2).sum())], dtype=torch.float32, device=dev) \
                    if max_norm > 0 else None
                prev = (w.clone(), m.clone(), v.clone())
                n0 = _count()
                ops.adamw_step(w, g, m, v, sh[:n], lr, b1, b2, eps, wd, gs, gn, max_norm, step0 + k, zero_grad)
                _launched(name, n0)
                if zero_grad:
                    assert _same(g, torch.zeros_like(g)), f"{name}: gradients not zeroed"
                else:
                    assert _same(g, g0), f"{name}: gradients modified with zero_grad = 0"
                assert _same(sh[n:], torch.full((8,), SENTINEL, dtype=torch.bfloat16, device=dev))
                states.append((prev, g0, None if gn is None else float(gn), w.clone(), m.clone(), v.clone(),
                               sh[:n].clone()))
            return states
        finally:
            if cap is not None:
                ops.set_optimizer_grid(0)

    states = run(None)
    for k, ((w, m, v), g, gn, w2, m2, v2, sh) in enumerate(states):
        rw, rm, rv, dw, dm, dv = _adamw_step_ref(w.double(), g.double(), m.double(), v.double(), lr, b1, b2, eps, wd,
                                                 gs, gn, max_norm, step0 + k)
        _check_bound(f"{name} step {step0 + k} master", w2, rw, dw)
        _check_bound(f"{name} step {step0 + k} exp_avg", m2, rm, dm)
        _check_bound(f"{name} step {step0 + k} exp_avg_sq", v2, rv, dv)
        assert _same(sh, w2.to(torch.bfloat16)), f"{name}: the bf16 shadow is not RNE(master)"
    if dev.type == "cuda":
        for cap in (1, 7, 264):
            other = run(cap)
            for a, b in zip(states, other):
                assert all(_same(x, y) for x, y in zip(a[3:], b[3:])), f"{name}: optimizer grid cap {cap} changes bits"


# ---------------------------------------------------------------------------------------------
# G. decode-loop kernels
# ---------------------------------------------------------------------------------------------
def test_decode_embed_and_advance():
    import torch

    from magma_b200 import ops

    dev, bf = _dev(), torch.bfloat16
    V, d, B, ld = 1000, 4096, 5, 12
    gen = _gen("decode")
    wte = torch.randn(V, d, generator=gen, dtype=torch.float64).to(bf).to(dev)
    tokens = torch.randint(0, V, (B, ld), generator=gen).to(dev)
    tokens[:4, 3] = torch.tensor([-1, V, V + 7, 0], device=dev)
    for pos in (3, 0, ld - 1):
        pos_dev = torch.tensor([pos], dtype=torch.int32, device=dev)
        out = torch.full((B + 1, d), SENTINEL, dtype=bf, device=dev)
        inp = _Inputs(wte, tokens, pos_dev)
        n0 = _count()
        ops.decode_embed(tokens, pos_dev, wte, out[:B])
        _launched("decode_embed", n0)
        inp.unchanged("decode_embed")
        ids = tokens[:, pos]
        assert _same(out[:B], wte[torch.where((ids < 0) | (ids >= V), 0, ids)]), f"decode_embed pos={pos}"
        assert _same(out[B:], torch.full_like(out[B:], SENTINEL))
    eos = 7
    for pos, nxt_all_eos in ((3, False), (4, True), (ld - 1, True)):
        toks = tokens.clone()
        pos_dev = torch.tensor([pos], dtype=torch.int32, device=dev)
        nxt = torch.full((B,), eos, dtype=torch.int64, device=dev)
        if not nxt_all_eos:
            nxt[2] = 11
        flags = torch.full((ld + 2,), 9, dtype=torch.uint8, device=dev)
        s0 = 2
        n0 = _count()
        ops.decode_advance(nxt, toks, pos_dev, eos, flags[:ld - s0], s0)
        _launched("decode_advance", n0)
        want = tokens.clone()
        if pos + 1 < ld:
            want[:, pos + 1] = nxt
        assert torch.equal(toks, want), f"decode_advance pos={pos}: tokens"
        assert int(pos_dev.item()) == pos + 1
        wf = torch.full_like(flags, 9)
        if 0 <= pos + 1 - s0 < ld - s0:
            wf[pos + 1 - s0] = int(nxt_all_eos)
        assert torch.equal(flags, wf), f"decode_advance pos={pos}: flags {flags.tolist()}"


# ---------------------------------------------------------------------------------------------
# H. rejected arguments: nothing is launched
# ---------------------------------------------------------------------------------------------
def test_misaligned_views_are_rejected():
    import torch

    from magma_b200 import ops
    from magma_b200._lib import MB200Error

    dev, bf = _dev(), torch.bfloat16
    rows, d = 4, 64
    store = torch.zeros(4096, dtype=bf, device=dev)
    fstore = torch.zeros(4096, dtype=torch.float32, device=dev)

    def mis(n, shape=None, dt=bf):
        t = (store if dt == bf else fstore)[1:1 + n]
        return t.view(*shape) if shape else t

    def ok(n, shape=None, dt=bf):
        t = torch.zeros(n, dtype=dt, device=dev)
        return t.view(*shape) if shape else t

    g, b = ok(d), ok(d)
    st = ok(rows, dt=torch.float32)
    x2 = ok(rows * d, (rows, d))
    nhwc = (1, 2, 4, 8)
    cases = {
        "layernorm_fwd x": lambda: ops.layernorm_fwd(mis(rows * d, (rows, d)), g, b),
        "layernorm_fwd gamma": lambda: ops.layernorm_fwd(x2, mis(d), b),
        "layernorm_fwd out": lambda: ops.layernorm_fwd(x2, g, b, out=mis(rows * d, (rows, d))),
        "layernorm_bwd dy": lambda: ops.layernorm_bwd(mis(rows * d, (rows, d)), x2, g, st, st),
        "layernorm_bwd res": lambda: ops.layernorm_bwd(x2, x2, g, st, st, res=mis(rows * d, (rows, d))),
        "layernorm_bwd dx": lambda: ops.layernorm_bwd(x2, x2, g, st, st, out=mis(rows * d, (rows, d))),
        "cross_entropy logits": lambda: ops.cross_entropy(mis(2 * d, (1, 2, d)), ok(2, dt=torch.int64).view(1, 2), d),
        "cross_entropy dlogits": lambda: ops.cross_entropy(ok(2 * d, (1, 2, d)), ok(2, dt=torch.int64).view(1, 2), d,
                                                           dlogits=mis(2 * d, (1, 2, d))),
        "embed_assemble wte": lambda: ops.embed_assemble(ok(4, dt=torch.int64).view(1, 4), mis(2 * d, (2, d)), None),
        "embed_assemble prefix": lambda: ops.embed_assemble(ok(4, dt=torch.int64).view(1, 4), ok(2 * d, (2, d)),
                                                            mis(d, (1, 1, d))),
        "embed_assemble out": lambda: ops.embed_assemble(ok(4, dt=torch.int64).view(1, 4), ok(2 * d, (2, d)), None,
                                                         out=mis(4 * d, (1, 4, d))),
        "embed_gather wte": lambda: ops.embed_gather(ok(3, dt=torch.int64), mis(2 * d, (2, d))),
        "embed_gather out": lambda: ops.embed_gather(ok(3, dt=torch.int64), ok(2 * d, (2, d)), out=mis(3 * d, (3, d))),
        "decode_embed wte": lambda: ops.decode_embed(ok(4, dt=torch.int64).view(2, 2), ok(1, dt=torch.int32),
                                                     mis(2 * d, (2, d)), ok(2 * d, (2, d))),
        "decode_embed out": lambda: ops.decode_embed(ok(4, dt=torch.int64).view(2, 2), ok(1, dt=torch.int32),
                                                     ok(2 * d, (2, d)), mis(2 * d, (2, d))),
        "add": lambda: ops.add(mis(d), ok(d)),
        "add c": lambda: ops.add(ok(d), ok(d), mis(d)),
        "add out": lambda: ops.add(ok(d), ok(d), out=mis(d)),
        "im2col3x3": lambda: ops.im2col3x3(mis(64, nhwc)),
        "im2col3x3 out": lambda: ops.im2col3x3(ok(64).view(nhwc), out=mis(8 * 72, (8, 72))),
        "col2im3x3": lambda: ops.col2im3x3(ok(8 * 72, (8, 72)), 1, 2, 4, 8, out=mis(64, nhwc)),
        "avgpool_nhwc": lambda: ops.avgpool_nhwc(mis(64, nhwc), 2),
        "avgpool_nhwc_bwd": lambda: ops.avgpool_nhwc_bwd(ok(16, (1, 1, 2, 8)), 2, 4, 2, out=mis(64, nhwc)),
        "nchw_to_nhwc8": lambda: ops.nchw_to_nhwc8(ok(24, (1, 3, 2, 4)), out=mis(64, nhwc)),
        "adamw master": lambda: ops.adamw_step(mis(64, dt=torch.float32), ok(64, dt=torch.float32),
                                               ok(64, dt=torch.float32), ok(64, dt=torch.float32), None, 1e-3, 0.9,
                                               0.95, 1e-8, 0.0, 1.0, None, 0.0, 1),
        "adamw exp_avg_sq": lambda: ops.adamw_step(ok(64, dt=torch.float32), ok(64, dt=torch.float32),
                                                   ok(64, dt=torch.float32), mis(64, dt=torch.float32), None, 1e-3,
                                                   0.9, 0.95, 1e-8, 0.0, 1.0, None, 0.0, 1),
        "adamw shadow": lambda: ops.adamw_step(ok(64, dt=torch.float32), ok(64, dt=torch.float32),
                                               ok(64, dt=torch.float32), ok(64, dt=torch.float32), mis(64), 1e-3,
                                               0.9, 0.95, 1e-8, 0.0, 1.0, None, 0.0, 1),
        "colsum": lambda: ops.colsum(mis(rows * d, (rows, d))),
        "layernorm_param_grad_rows": lambda: ops.layernorm_param_grad_rows(
            mis(rows * d, (rows, d)), x2, st, st, ok(d, dt=torch.float32), ok(d, dt=torch.float32)),
        "col_moments": lambda: ops.col_moments(mis(rows * d, (rows, d)), x2),
        "col_moments mask": lambda: ops.col_moments(x2, x2, mis(rows * d, (rows, d))),
    }
    n0 = _count()
    for tag, call in cases.items():
        with pytest.raises(MB200Error, match="aligned"):
            call()
    with pytest.raises(MB200Error, match="ldx"):
        ops.argmax(ok(2 * d, (2, d)), d + 8)
    assert _count() == n0, "a rejected call launched a kernel"
