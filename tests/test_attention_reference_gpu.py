"""Element-wise float64 reference tests of the attention kernels: the single-tile forward and backward
(ops.attn_fwd_tile / attn_bwd_tile), the multi-tile forward (ops.attn_fwd_flash, with and without a KV cache), the KV
cache append and the fused decode step (ops.kv_append / attn_decode / attn_decode_dev), and the materialised softmax
(ops.softmax_fwd / softmax_bwd).

Every reference is computed in float64 on the device from the same bf16 (or fp32) inputs. u = 2^-24 is the fp32 unit
roundoff and gamma_n = ceil(n / 16) * 2^-23 bounds a wgmma fp32 accumulation over n products; k-steps whose products
are all zero (masked keys past the last visible one) leave the accumulator unchanged, so n counts keys up to the last
visible one.

Scores. s_j = q . k_j / sqrt(hd) with
    ds_j = (gamma_hd |q| . |k_j| + c_scale |q . k_j|) / sqrt(hd)
c_scale = 3u for the tile and flash kernels (sqrtf, the division 1 / sqrtf and the product with it each round once),
5u for the decode step (rsqrtf is within 2 ulp, plus the product). The decode step sums the head dim per lane (two
roundings per bf16 pair: the products of bf16 values are exact in fp32) and then over the warp, so its gamma_hd is
(8 ceil(hd / 256) + 5) u. For softmax_fwd the scores are exact fp32 inputs: ds_j = u |scale * s_j|.

Probabilities. With x_j = s_j - max_i s_i, the kernel's fp32 exp(x_j) carries the score error ds_j and
    eta_j = u |x_j| + eps_exp(x_j),    eps_exp(x) = (2 + 1.173 |x|) 2^-23
(the rounding of the argument and the documented bound of __expf); the error of the row maximum cancels between
numerator and sum. A term of the fp32 row sum goes through at most `depth` additions: 32 + 2 in the tile kernel (a
thread's columns, then two quad shuffles), 35 + n_tiles in the multi-tile forward, ceil(Sk / 32) + 5 in softmax_fwd
(lane-strided, then the warp), ceil(nk / 256) + 13 in the decode step (then 8 warps in sequence). So the sum has
relative error eps_l = sum_j p_j (ds_j + eta_j) + depth u. The multi-tile forward rescales its running sum once per
key tile at most: each rescale adds 2 * 2^-23 + 2u, and 1.173 * 2^-23 times the total rise of the running maximum (at
most the row's score range plus 2 max ds). The probability then has relative error
    E_j = 1.001 * (ds_j + eta_j + eps_l + 2u)
(the reciprocal and the product round once each; 1.001 covers the second-order terms), plus 2^-149 absolute where the
product is an fp32 subnormal.

The rule for rounded intermediates. P (and dS in the backward) is rounded to bf16. The reference rounds the float64
value to nearest even. Where the interval [ref - delta, ref + delta] holds a rounding midpoint the element is
ambiguous and may take any bf16 value between the roundings of the interval ends; elsewhere it must equal the
reference rounding exactly. The ambiguous share is printed and capped by AMBIGUOUS_MAX: the worst-case wgmma bound
is wide enough that a 1 % cap cannot hold at head_dim 256. __expf flushes results below 2^-126 to zero, so a
probability whose exp(x_j) (1 - E_j) lies below 2^-126 may also be +0 (the flush band, reported apart). Masked and
padding columns of P must be exactly +0. A one-hot row of P gives D = dP_j exactly, so dS = 0 exactly there.

Outputs. O against sum_j P_j v_j:
    |O - sum_j P_j v_j| <= ulp_bf16(ref) + gamma_nk sum_j P_j |v_j|
with the kernel's own P where it is returned. The decode step accumulates P V sequentially in fp32 (nk u instead of
gamma_nk) and returns no P: it is held to the reference-rounded P, with (upper - lower rounding) |v_j| added for every
ambiguous j. Flash statistics: the row maximum within max_j ds_j of the float64 maximum, and
inv * sum_j exp(s_j - m) within max_j E_j of 1.

Tile backward (the kernel's forward P is an exact input). dP = dO V^T with ddP = gamma_hd |dO| |V|^T;
D_i = sum_j P_ij dP_ij with dD_i = sum_j P_ij ddP_ij + (4 ceil(S / 8) + 2) u sum_j P_ij |dP_ij| (a thread sums its
nonzero columns with at most two roundings per pair, then two quad shuffles); dS = P (dP - D) / sqrt(hd) with
ddS = P (ddP + dD) / sqrt(hd) + 5u |dS| + 2^-149, rounded by the rule above. dQ = dS K and dK = dS^T Q are held to
ulp_bf16 + gamma_S |dS| |K| (resp. |dS|^T |Q|), plus (upper - lower rounding) of each ambiguous dS times |K| (|Q|).
The inverse rotary rotation is applied in float64 with the kernel's fp32 table; a rotated pair takes the larger
bound of its two columns times (|cos| + |sin|), plus 2u (|x0| + |x1|) for the rotation's own rounding.
dV = P^T dO: ulp_bf16 + gamma_S P^T |dO|. softmax_bwd: D sums lane-strided, then over the warp, so
dD = (ceil(Sk / 32) + 5) u sum_j P_j |dP_j| and ddS = P dD scale + 3u |dS| + 2^-149.

Layouts. qkv is a view with row stride 3 H hd + 8 and NaN in the padding and in spare rows after the last batch;
KV caches hold NaN beyond their valid rows. O, P, dqkv, stats and the softmax outputs sit in sentinel-filled buffers
with larger row strides and spare rows, which must stay untouched except where each kernel's contract writes:
the tile forward writes P columns [0, min(ldP, 128)), flash writes [0, ldP), softmax_fwd writes [0, Sk). Every input
is compared byte for byte before and after each call, each call is exactly one launch, and reruns are bit-identical.

Inputs come in four score distributions: scores with std about 2, peaked scores with std about 20 (most exponentials
underflow), all-equal scores (q = 0), and scores that rise along the key index (the running maximum of the multi-tile
forward changes in every key tile).

The device comes from MB200_TEST_DEVICE (default cuda:0): tests/test_attention_reference_twin_cpu.py replays the
bodies on the CPU emulation of the operators (softmax on the kernel source executed on the CPU), where no launches are
counted.
"""
import ctypes
import math
import zlib

import pytest

from _refcheck import SENTINEL, Buf, bf16_rne, bits, check_rounded, dev as _dev, launches, ulp_bf16
from _refcheck import roundings as _roundings

pytestmark = pytest.mark.gpu

U = 2.0**-24
TINY = 2.0**-149  # one fp32 subnormal step
DISTS = ("std2", "peaked", "equal", "rising")
# Largest share of ambiguous rounded elements (plus 8, for the tiny S = 1, 2 cases). The worst-case wgmma bound
# gamma_hd |q| . |k| grows with head_dim and with the score scale, so it makes up to about 8 % of the std-2
# probabilities ambiguous at head_dim 256, and a third of the peaked ones.
AMBIGUOUS_MAX = {"std2": 0.08, "peaked": 0.4}


def _fp32_inv_sqrt(hd):
    """The kernels' scale 1.0f / sqrtf((float)hd), as a Python float."""
    import numpy as np

    return float(np.float32(1.0) / np.sqrt(np.float32(hd)))


# ---------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------
def _draw(gen, B, n, H, hd, dist, pos0=0, span=None):
    """float64 q, k, v [B, n, H, hd] at sequence positions pos0.. (span: the key count the rising scores run over)."""
    import torch

    def g(scale):
        return torch.randn(B, n, H, hd, generator=gen, dtype=torch.float64) * scale

    v = g(1.0)
    if dist == "std2":
        return g(2.0**0.5), g(2.0**0.5), v
    if dist == "peaked":
        return g(20.0**0.5), g(20.0**0.5), v
    if dist == "equal":
        return torch.zeros(B, n, H, hd, dtype=torch.float64), g(1.0), v
    assert dist == "rising"  # s_j ~ 24 * position / span
    pos = torch.arange(pos0, pos0 + n, dtype=torch.float64)[None, :, None, None]
    return 2.0 + g(0.1), g(0.1) + 12.0 / math.sqrt(hd) * pos / (span or n), v


class _Qkv:
    """The fused qkv rows [B*S, 3*H*hd] as a view with row stride 3 H hd + 8, NaN in the padding columns and in 5 spare
    rows after the last batch; q / k / v hold the bf16 values as float64 [B, H, S, hd]."""

    def __init__(self, gen, B, S, H, hd, dist, pos0=0, span=None):
        import torch

        d = H * hd
        ld = 3 * d + 8
        self.storage = torch.full(((B * S + 5) * ld,), float("nan"), dtype=torch.bfloat16, device=_dev())
        self.view = self.storage.as_strided((B * S, 3 * d), (ld, 1))
        q, k, v = _draw(gen, B, S, H, hd, dist, pos0, span)
        self.view.copy_(torch.stack([q, k, v], 2).reshape(B * S, 3 * d).to(torch.bfloat16))
        self.q, self.k, self.v = self.view.double().view(B, S, 3, H, hd).permute(2, 0, 3, 1, 4)
        self.before = bits(self.storage)

    def unchanged(self):
        import torch

        return torch.equal(bits(self.storage), self.before)


def _gen(*key):
    import torch

    return torch.Generator().manual_seed(zlib.crc32(repr(key).encode()))


def _one_launch(name, n0):
    import torch

    if _dev().type == "cuda":
        torch.cuda.synchronize()
        n = launches() - n0
        assert n == 1, f"{name}: {n} kernel launches, expected 1"


def _count():
    return launches() if _dev().type == "cuda" else 0


def _same(a, b):
    import torch

    return torch.equal(bits(a), bits(b))


# ---------------------------------------------------------------------------------------------
# references and checks
# ---------------------------------------------------------------------------------------------
def _gamma(n):
    return math.ceil(n / 16) * 2.0**-23


def _acc(a, b):
    """Bound of the wgmma fp32 accumulation of a @ b (float64 operands, exact in bf16)."""
    return _gamma(a.shape[-1]) * (a.abs() @ b.abs())


def _scores(q, k, hd, c_scale, lane_gamma=None):
    """float64 scores q k^T / sqrt(hd) and their bound ds (wgmma accumulation unless lane_gamma is given)."""
    r = 1.0 / math.sqrt(hd)
    qk = q @ k.transpose(-1, -2)
    if lane_gamma is None:
        acc = _acc(q, k.transpose(-1, -2))
    else:
        acc = lane_gamma * (q.abs() @ k.abs().transpose(-1, -2))
    return qk * r, (acc + c_scale * qk.abs()) * r


def _probs(s, ds, vis, depth, rescales=0):
    """float64 softmax over the visible scores, the relative bound E of the kernel's probability and the flush band.
    depth: the most additions any term of the kernel's row sum goes through."""
    import torch

    zero = torch.zeros((), dtype=s.dtype, device=s.device)
    m = torch.where(vis, s, -math.inf).amax(-1, keepdim=True)
    x = torch.where(vis, s - m, zero)
    e = torch.where(vis, torch.exp(x), zero)
    p = e / e.sum(-1, keepdim=True)
    ds = torch.where(vis, ds, zero)
    dmax = ds.amax(-1, keepdim=True)
    ax = x.abs()
    eta = U * ax + (2.0 + 1.173 * ax) * 2.0**-23
    eps_l = (p * (ds + eta)).sum(-1, keepdim=True) + depth * U
    if rescales:
        eps_l = eps_l + rescales * (2 * 2.0**-23 + 2 * U) + 1.173 * 2.0**-23 * (ax.amax(-1, keepdim=True) + 2 * dmax)
    E = 1.001 * (ds + eta + eps_l + 2 * U)
    flush = vis & (e * (1 - E) < 2.0**-126)
    return p, E, flush


def _check_rounded(name, got, ref, delta, keep, band=None, dist="std2"):
    """The rounding rule (tests/_refcheck.py) with this file's ambiguous-share cap for the score distribution."""
    return check_rounded(name, got, ref, delta, keep, band, AMBIGUOUS_MAX.get(dist, AMBIGUOUS_MAX["std2"]))


def _check_bound(name, got, ref, extra):
    """|got - ref| <= ulp_bf16(ref) + extra, element by element; prints the largest err / bound ratio."""
    import torch

    bound = ulp_bf16(ref) + extra
    err = (got.double() - ref).abs()
    ratio = torch.nan_to_num(err / bound, nan=math.inf)
    worst = int(ratio.argmax().item())
    r = float(ratio.reshape(-1)[worst].item())
    if r > 1.0:
        idx = tuple(int(t) for t in torch.unravel_index(torch.tensor(worst), ref.shape))
        pytest.fail(f"{name}: {int((ratio > 1).sum().item())} of {ref.numel()} elements outside the bound; worst at "
                    f"{idx}: got {got.double().reshape(-1)[worst].item():.6g}, ref {ref.reshape(-1)[worst].item():.6g}, "
                    f"err/bound {r:.3g}")
    print(f"[ratio] {name}: max err/bound {r:.3f}")


def _check_zero(name, t, mask=None):
    """Masked / padding probabilities must be exactly +0."""
    b = bits(t)
    if mask is not None:
        b = b[mask.expand(t.shape)]
    assert int((b != 0).sum().item()) == 0, f"{name}: {int((b != 0).sum().item())} masked elements are not +0"


def _untouched(name, *bufs):
    for tag, b in bufs:
        n = b.overwritten()
        assert n == 0, f"{name}: {n} sentinel elements of {tag} overwritten"


def _inv_rope(x, bound, tab, rot):
    """The kernel's inverse rotation of the first `rot` columns ([B, H, S, hd], row i uses table row i) in float64."""
    import torch

    if tab is None:
        return x, bound
    cs = tab.double()
    c, s = cs[..., 0], cs[..., 1]
    x0, x1 = x[..., 0:rot:2], x[..., 1:rot:2]
    y = x.clone()
    y[..., 0:rot:2], y[..., 1:rot:2] = x0 * c + x1 * s, x1 * c - x0 * s
    bm = torch.maximum(bound[..., 0:rot:2], bound[..., 1:rot:2]) * (c.abs() + s.abs()) + 2 * U * (x0.abs() + x1.abs())
    nb = bound.clone()
    nb[..., 0:rot:2], nb[..., 1:rot:2] = bm, bm
    return y, nb


# ---------------------------------------------------------------------------------------------
# A. single-tile forward and backward
# ---------------------------------------------------------------------------------------------
def _tile(B, S, H, hd, rot, dist="std2"):
    import torch

    from magma_b200 import ops

    name = f"tile B={B} S={S} H={H} hd={hd} rot={rot} {dist}"
    dev, bf = _dev(), torch.bfloat16
    gen = _gen("tile", B, S, H, hd, rot, dist)
    x = _Qkv(gen, B, S, H, hd, dist)
    ldP = (S + 7) // 8 * 8 + 8
    ncols = min(ldP, 128)  # the columns the tile forward writes
    nan = float("nan")

    def fwd():
        Pb = Buf((B, H), S, ncols, bf, dev, SENTINEL, ld=ldP, bstrides=(H * S * ldP, S * ldP))
        Ob = Buf((), B * S, H * hd, bf, dev, SENTINEL)
        n0 = _count()
        ops.attn_fwd_tile(x.view, B, S, H, hd, O=Ob.view, P=Pb.view)
        _one_launch(name, n0)
        return Ob, Pb

    Ob, Pb = fwd()
    assert x.unchanged(), f"{name}: the forward modified qkv"
    _untouched(name, ("O", Ob), ("P", Pb))
    s, ds = _scores(x.q, x.k, hd, 3 * U)
    vis = torch.ones(S, S, dtype=torch.bool, device=dev).tril()
    p, E, flush = _probs(s, ds, vis, 32 + 2)
    P = Pb.view[..., :S]
    _check_rounded(f"{name} P", P, p, p * E + TINY, vis, flush, dist)
    _check_zero(f"{name} P above the diagonal", P, ~vis)
    _check_zero(f"{name} P columns [S, min(ldP, 128))", Pb.view[..., S:])
    Ph = P.double()
    O = Ob.view.unflatten(1, (H, hd)).unflatten(0, (B, S)).permute(0, 2, 1, 3)
    _check_bound(f"{name} O", O, Ph @ x.v, _acc(Ph, x.v))
    Ob2, Pb2 = fwd()
    assert _same(Ob.view, Ob2.view) and _same(Pb.view, Pb2.view), f"{name}: forward rerun not bit-identical"

    # ---- backward, from the kernel's own P ----
    dOb = Buf((), B * S, H * hd, bf, dev, nan)
    dOb.view.copy_((torch.randn(B * S, H * hd, generator=gen, dtype=torch.float64)).to(bf))
    dO = dOb.view.double().unflatten(1, (H, hd)).unflatten(0, (B, S)).permute(0, 2, 1, 3)
    tab = ops.rope_table(S, rot, 0, device=dev) if rot else None
    inputs = [dOb.storage, Pb.storage] + ([tab] if rot else [])
    before = [bits(t) for t in inputs]

    def bwd():
        Db = Buf((), B * S, 3 * H * hd, bf, dev, SENTINEL)
        n0 = _count()
        ops.attn_bwd_tile(x.view, dOb.view, Pb.view, B, S, H, hd, rope_tab=tab, rot=rot, dqkv=Db.view)
        _one_launch(name + " bwd", n0)
        return Db

    Db = bwd()
    assert x.unchanged(), f"{name}: the backward modified qkv"
    for t, b0 in zip(inputs, before):
        assert torch.equal(bits(t), b0), f"{name}: the backward modified dO, P or the rope table"
    _untouched(name, ("dqkv", Db))
    dP = dO @ x.v.transpose(-1, -2)
    ddP = _acc(dO, x.v.transpose(-1, -2))
    D = (Ph * dP).sum(-1, keepdim=True)
    dD = (Ph * ddP).sum(-1, keepdim=True) + (4 * math.ceil(S / 8) + 2) * U * (Ph * dP.abs()).sum(-1, keepdim=True)
    r = 1.0 / math.sqrt(hd)
    dS = Ph * (dP - D) * r
    # a one-hot row of P (a single visible key, or a peaked row) has D = dP_j exactly in fp32 too, so dS = 0 exactly
    one_hot = ((Ph == 1).sum(-1, keepdim=True) == 1) & ((Ph != 0).sum(-1, keepdim=True) == 1)
    ddS = torch.where(one_hot, torch.zeros_like(dS), Ph * (ddP + dD) * r + 5 * U * dS.abs() + TINY)
    dSb = bf16_rne(dS)  # dS is internal to the kernel: the rule bounds its choices, the reference takes this one
    w = _check_rounded(f"{name} dS", dSb, dS, ddS, vis, dist=dist)
    g = Db.view.unflatten(1, (3, H, hd)).unflatten(0, (B, S)).permute(2, 0, 3, 1, 4)
    kt, qt = x.k, x.q
    dq, bq = dSb @ kt, _acc(dSb, kt) + w @ kt.abs()
    dk = dSb.transpose(-1, -2) @ qt
    bk = _acc(dSb.transpose(-1, -2), qt) + w.transpose(-1, -2) @ qt.abs()
    dq, bq = _inv_rope(dq, bq, tab, rot)
    dk, bk = _inv_rope(dk, bk, tab, rot)
    _check_bound(f"{name} dQ", g[0], dq, bq)
    _check_bound(f"{name} dK", g[1], dk, bk)
    _check_bound(f"{name} dV", g[2], Ph.transpose(-1, -2) @ dO, _acc(Ph.transpose(-1, -2), dO))
    assert _same(Db.view, bwd().view), f"{name}: backward rerun not bit-identical"


TILE_HD, TILE_S = (64, 128, 192, 256), (1, 2, 63, 64, 65, 127, 128)


@pytest.mark.parametrize("rot", ["none", "64", "hd"])
@pytest.mark.parametrize("H", [1, 3])
@pytest.mark.parametrize("S", TILE_S)
@pytest.mark.parametrize("hd", TILE_HD)
def test_tile_forward_backward(hd, S, H, rot):
    _tile(2, S, H, hd, dict(none=0, hd=hd).get(rot, 64))


def test_tile_production_shape():
    _tile(8, 128, 16, 256, 64)


def test_tile_backward_fused_inverse_rope():
    """The inverse rotary rotation fused into the backward's dQ / dK stores, at a length between the grid's S values:
    held element-wise to the float64 inverse rotation with the kernel's table."""
    _tile(2, 96, 2, 128, 64)


@pytest.mark.parametrize("dist", DISTS)
@pytest.mark.parametrize("hd,S", [(128, 128), (256, 65)])
def test_tile_distributions(hd, S, dist):
    _tile(2, S, 3, hd, 64, dist)


# ---------------------------------------------------------------------------------------------
# B. multi-tile forward (fused qkv, or keys / values from a KV cache)
# ---------------------------------------------------------------------------------------------
def _flash_check(name, x, kv, B, Sq, Sk, H, hd, causal, cache=None, dist="std2"):
    """One flash call with O, P and stats in sentinel buffers, held to the reference; then the same call without the
    optional outputs, and a rerun, both bit-identical. kv: float64 keys / values [B, H, Sk, hd]."""
    import torch

    from magma_b200 import ops

    dev, bf = _dev(), torch.bfloat16
    cache = cache or {}
    ldP = (Sk + 7) // 8 * 8 + 8
    guarded = [t for t in (cache.get("kcache"), cache.get("vcache")) if t is not None]
    before = [bits(t) for t in guarded]

    def run(with_outputs):
        Ob = Buf((), B * Sq, H * hd, bf, dev, SENTINEL)
        Pb = Buf((B, H), Sq, ldP, bf, dev, SENTINEL, ld=ldP, bstrides=(H * Sq * ldP, Sq * ldP))
        st = torch.full((B * H * Sq * 2 + 64,), SENTINEL, dtype=torch.float32, device=dev)
        kw = dict(P=Pb.view, stats=st[: B * H * Sq * 2].view(B, H, Sq, 2)) if with_outputs else {}
        n0 = _count()
        ops.attn_fwd_flash(x.view, B, Sq, H, hd, causal=causal, O=Ob.view, **kw, **cache)
        _one_launch(name, n0)
        return Ob, Pb, st

    Ob, Pb, st = run(True)
    assert x.unchanged(), f"{name}: the call modified qkv"
    assert all(torch.equal(bits(t), b0) for t, b0 in zip(guarded, before)), f"{name}: the call modified the cache"
    _untouched(name, ("O", Ob), ("P", Pb))
    n_st = B * H * Sq * 2
    assert bool((st[n_st:] == SENTINEL).all()), f"{name}: stats written past [B, H, Sq, 2]"
    k, v = kv
    s, ds = _scores(x.q, k, hd, 3 * U)
    i = torch.arange(Sq, device=dev)[:, None]
    j = torch.arange(Sk, device=dev)[None, :]
    vis = (j <= i + (Sk - Sq)) if causal else torch.ones(Sq, Sk, dtype=torch.bool, device=dev)
    n_kv = (Sk + 127) // 128
    p, E, flush = _probs(s, ds, vis, 35 + n_kv, rescales=n_kv)
    P = Pb.view[..., :Sk]
    _check_rounded(f"{name} P", P, p, p * E + TINY, vis, flush, dist)
    _check_zero(f"{name} P masked", P, ~vis)
    _check_zero(f"{name} P columns [Sk, ldP)", Pb.view[..., Sk:])
    Ph = P.double()
    O = Ob.view.unflatten(1, (H, hd)).unflatten(0, (B, Sq)).permute(0, 2, 1, 3)
    _check_bound(f"{name} O", O, Ph @ v, _acc(Ph, v))
    # statistics: the row maximum, and 1 / sum
    stats = st[:n_st].view(B, H, Sq, 2).double()
    m_k, inv_k = stats[..., 0], stats[..., 1]
    zero = torch.zeros((), dtype=s.dtype, device=dev)
    m_ref = torch.where(vis, s, -math.inf).amax(-1)
    dmax = torch.where(vis, ds, zero).amax(-1)
    err_m = (m_k - m_ref).abs()
    assert bool((err_m <= dmax).all()), f"{name}: row maximum off by {float((err_m - dmax).max()):.3g} past its bound"
    tot = torch.where(vis, torch.exp(s - m_k[..., None]), zero).sum(-1) * inv_k
    e_max = torch.where(vis, E, zero).amax(-1)
    err_l = (tot - 1).abs()
    assert bool((err_l <= e_max).all()), f"{name}: inv * sum exp(s - m) off from 1 by {float(err_l.max()):.3g}"
    print(f"[ratio] {name} stats: max err/bound m {float((err_m / dmax.clamp(min=1e-300)).max()):.3f}, "
          f"1/sum {float((err_l / e_max).max()):.3f}")
    Ob2, _, _ = run(False)
    assert _same(Ob.view, Ob2.view), f"{name}: O without P / stats differs from O with them"
    Ob3, Pb3, st3 = run(True)
    assert _same(Ob.view, Ob3.view) and _same(Pb.view, Pb3.view) and _same(st, st3), f"{name}: rerun not bit-identical"
    return Pb


def _flash(B, S, H, hd, causal, dist="std2"):
    name = f"flash B={B} S={S} H={H} hd={hd} causal={int(causal)} {dist}"
    x = _Qkv(_gen("flash", B, S, H, hd, causal, dist), B, S, H, hd, dist)
    return x, _flash_check(name, x, (x.k, x.v), B, S, S, H, hd, causal, dist=dist)


FLASH_S = (1, 127, 128, 129, 255, 256, 257, 300, 640, 2048)


@pytest.mark.parametrize("S", FLASH_S)
@pytest.mark.parametrize("causal", [True, False], ids=["causal", "full"])
@pytest.mark.parametrize("hd", TILE_HD)
def test_flash(hd, causal, S):
    _flash(2 if S <= 300 else 1, S, 2, hd, causal)


@pytest.mark.parametrize("dist", DISTS)
@pytest.mark.parametrize("hd,S,causal", [(128, 640, True), (192, 300, False), (256, 2048, True)])
def test_flash_distributions(hd, S, causal, dist):
    _flash(1, S, 2, hd, causal, dist)


def test_flash_vit_shape():
    _flash(2, 257, 16, 64, False)


def test_flash_gptj_shape():
    _flash(1, 2048, 4, 256, True)


def _prefill(B, S, H, hd, pos0, dist="std2"):
    """kv_append of S new positions at pos0 into NaN-filled caches holding pos0 valid rows, then flash over the cache."""
    import torch

    from magma_b200 import ops

    name = f"prefill B={B} S={S} H={H} hd={hd} pos0={pos0} {dist}"
    dev, bf = _dev(), torch.bfloat16
    Sk, Smax = pos0 + S, pos0 + S + 9
    gen = _gen("prefill", B, S, H, hd, pos0, dist)
    _, k0, v0 = _draw(gen, B, pos0, H, hd, dist, 0, Sk)
    x = _Qkv(gen, B, S, H, hd, dist, pos0, Sk)
    caches = []
    for t in (k0, v0):
        c = torch.full((B, H, Smax, hd), float("nan"), dtype=bf, device=dev)
        c[:, :, :pos0] = t.permute(0, 2, 1, 3).to(bf).to(dev)
        caches.append(c)
    kc, vc = caches
    old = [c.clone() for c in caches]
    n0 = _count()
    ops.kv_append(x.view, kc, vc, B, S, H, hd, pos0)
    _one_launch(name + " kv_append", n0)
    assert x.unchanged(), f"{name}: kv_append modified qkv"
    d = H * hd
    new = x.view.unflatten(0, (B, S))
    for which, c, o in ((1, kc, old[0]), (2, vc, old[1])):
        src = new[:, :, which * d:(which + 1) * d].unflatten(2, (H, hd)).permute(0, 2, 1, 3)
        assert _same(c[:, :, pos0:Sk], src), f"{name}: cache rows [pos0, pos0 + S) are not qkv's bytes"
        keep = torch.ones(Smax, dtype=torch.bool, device=dev)
        keep[pos0:Sk] = False
        assert _same(c[:, :, keep], o[:, :, keep]), f"{name}: kv_append changed cache rows outside [pos0, pos0 + S)"
    _flash_check(name, x, (kc[:, :, :Sk].double(), vc[:, :, :Sk].double()), B, S, Sk, H, hd, True,
                 dict(kcache=kc, vcache=vc, pos0=pos0), dist)


@pytest.mark.parametrize("S", [100, 200])
@pytest.mark.parametrize("pos0", [1, 127, 128, 129, 300])
@pytest.mark.parametrize("hd", [64, 256])
def test_prefill_continuation(hd, pos0, S):
    _prefill(2, S, 2, hd, pos0)


@pytest.mark.parametrize("dist", DISTS)
def test_prefill_distributions(dist):
    _prefill(1, 200, 2, 128, 300, dist)


# ---------------------------------------------------------------------------------------------
# C. fused decode step
# ---------------------------------------------------------------------------------------------
def _decode(B, H, hd, pos, dist="std2", Smax=None):
    import torch

    from magma_b200 import ops

    name = f"decode B={B} H={H} hd={hd} pos={pos} {dist}"
    dev, bf = _dev(), torch.bfloat16
    Smax = Smax or pos + 9
    nk = pos + 1
    gen = _gen("decode", B, H, hd, pos, dist)
    _, k0, v0 = _draw(gen, B, pos, H, hd, dist, 0, nk)
    x = _Qkv(gen, B, 1, H, hd, dist, pos, nk)
    caches = []
    for t in (k0, v0):
        c = torch.full((B, H, Smax, hd), float("nan"), dtype=bf, device=dev)
        c[:, :, :pos] = t.permute(0, 2, 1, 3).to(bf).to(dev)
        caches.append(c)
    old = [c.clone() for c in caches]

    def run(dev_pos):
        kc, vc = (c.clone() for c in old)
        ob = Buf((), B, H * hd, bf, dev, SENTINEL)
        n0 = _count()
        if dev_pos:
            ops.attn_decode_dev(x.view, kc, vc, B, H, hd, torch.tensor([pos], dtype=torch.int32, device=dev),
                                out=ob.view)
        else:
            ops.attn_decode(x.view, kc, vc, B, H, hd, pos, out=ob.view)
        _one_launch(name, n0)
        return ob, kc, vc

    ob, kc, vc = run(False)
    assert x.unchanged(), f"{name}: the step modified qkv"
    _untouched(name, ("out", ob))
    d = H * hd
    keep = torch.ones(Smax, dtype=torch.bool, device=dev)
    keep[pos] = False
    for which, c, o in ((1, kc, old[0]), (2, vc, old[1])):
        src = x.view[:, which * d:(which + 1) * d].unflatten(1, (H, hd))
        assert _same(c[:, :, pos], src), f"{name}: cache row pos is not qkv's k / v bytes"
        assert _same(c[:, :, keep], o[:, :, keep]), f"{name}: the step changed cache rows other than pos"
    k, v = kc[:, :, :nk].double(), vc[:, :, :nk].double()
    q = x.q  # [B, H, 1, hd]
    s, ds = _scores(q, k, hd, 5 * U, lane_gamma=(8 * math.ceil(hd / 256) + 5) * U)
    vis = torch.ones(1, nk, dtype=torch.bool, device=dev)
    p, E, flush = _probs(s, ds, vis, math.ceil(nk / 256) + 5 + 8)
    rlo, rhi = _roundings(p, p * E + TINY, flush)
    either = rlo != rhi
    n_amb = int((either & ~flush).sum().item())
    limit = AMBIGUOUS_MAX.get(dist, AMBIGUOUS_MAX["std2"])
    assert n_amb <= limit * p.numel() + 8, f"{name}: {n_amb} of {p.numel()} probabilities ambiguous"
    print(f"[ambiguous] {name} P: {n_amb} of {p.numel()} ({int((either & flush).sum().item())} more in the flush band)")
    Pb = bf16_rne(p)
    extra = nk * U * (Pb @ v.abs()) + torch.where(either, rhi - rlo, torch.zeros_like(p)) @ v.abs()
    _check_bound(f"{name} out", ob.view.unflatten(1, (H, hd))[:, :, None], Pb @ v, extra)
    for dev_pos in (False, True):
        ob2, kc2, vc2 = run(dev_pos)
        tag = "decode_dev" if dev_pos else "rerun"
        assert _same(ob.view, ob2.view) and _same(kc, kc2) and _same(vc, vc2), f"{name}: {tag} not bit-identical"


@pytest.mark.parametrize("pos", [0, 1, 31, 32, 127, 2047])
@pytest.mark.parametrize("hd", [8, 40, 64, 256])
def test_decode(hd, pos):
    B, H = (8, 16) if pos <= 127 else (2, 3)
    _decode(B, H, hd, pos)


@pytest.mark.parametrize("dist", DISTS)
@pytest.mark.parametrize("hd,pos", [(64, 2047), (256, 127)])
def test_decode_distributions(hd, pos, dist):
    _decode(2, 3, hd, pos, dist)


def test_decode_long_cache():
    """Positions past 12,250 need more than the 48 KB of shared memory a launch gets without opting in."""
    _decode(1, 2, 64, 16000, Smax=16384)


# ---------------------------------------------------------------------------------------------
# D. materialised softmax
# ---------------------------------------------------------------------------------------------
def _softmax(nz, Sq, Sk, causal, koff, dist="std2", hd=128):
    import torch

    from magma_b200 import ops

    name = f"softmax nz={nz} Sq={Sq} Sk={Sk} causal={int(causal)} koff={koff} {dist}"
    dev = _dev()
    gen = _gen("softmax", nz, Sq, Sk, causal, koff, dist)
    scale = _fp32_inv_sqrt(hd)
    nan = float("nan")
    sb = Buf((nz,), Sq, Sk, torch.float32, dev, nan)  # padded row and batch strides, NaN padding
    z = torch.randn(nz, Sq, Sk, generator=gen, dtype=torch.float64)
    jj = torch.arange(Sk, dtype=torch.float64)
    x0 = dict(std2=2.0 * z, peaked=20.0 * z, equal=0.0 * z, rising=24.0 * jj / Sk + 0.2 * z)[dist]
    sb.view.copy_((x0 / scale).to(torch.float32))
    pb = Buf((nz,), Sq, Sk, torch.bfloat16, dev, SENTINEL)
    s_before = bits(sb.storage)
    n0 = _count()
    ops.softmax_fwd(sb.view, scale, causal, koff, out=pb.view)
    _one_launch(name, n0)
    assert torch.equal(bits(sb.storage), s_before), f"{name}: softmax_fwd modified its scores"
    _untouched(name, ("P", pb))
    xs = sb.view.double() * scale
    i = torch.arange(Sq, device=dev)[:, None]
    j = torch.arange(Sk, device=dev)[None, :]
    vis = (j <= i + koff) if causal else torch.ones(Sq, Sk, dtype=torch.bool, device=dev)
    p, E, flush = _probs(xs, U * xs.abs(), vis, math.ceil(Sk / 32) + 5)
    _check_rounded(f"{name} P", pb.view, p, p * E + TINY, vis, flush, dist)
    _check_zero(f"{name} P masked", pb.view, ~vis)
    pb2 = Buf((nz,), Sq, Sk, torch.bfloat16, dev, SENTINEL)
    ops.softmax_fwd(sb.view, scale, causal, koff, out=pb2.view)
    assert _same(pb.view, pb2.view), f"{name}: rerun not bit-identical"

    # ---- backward: fp32 dP and the kernel's bf16 P are exact inputs ----
    dpb = Buf((nz,), Sq, Sk, torch.float32, dev, nan)
    dpb.view.copy_(torch.randn(nz, Sq, Sk, generator=gen, dtype=torch.float64).to(torch.float32))
    inputs = (dpb.storage, pb.storage)
    before = [bits(t) for t in inputs]
    dsb = Buf((nz,), Sq, Sk, torch.bfloat16, dev, SENTINEL)
    n0 = _count()
    ops.softmax_bwd(dpb.view, pb.view, scale, out=dsb.view)
    _one_launch(name + " bwd", n0)
    assert all(torch.equal(bits(t), b0) for t, b0 in zip(inputs, before)), f"{name}: softmax_bwd modified dP or P"
    _untouched(name + " bwd", ("dS", dsb))
    P, dp = pb.view.double(), dpb.view.double()
    D = (P * dp).sum(-1, keepdim=True)
    dD = (math.ceil(Sk / 32) + 5) * U * (P * dp).abs().sum(-1, keepdim=True)
    dS = P * (dp - D) * scale
    one_hot = ((P == 1).sum(-1, keepdim=True) == 1) & ((P != 0).sum(-1, keepdim=True) == 1)  # dS = 0 exactly
    _check_rounded(f"{name} dS", dsb.view, dS, torch.where(one_hot, 0.0, P * dD * scale + 3 * U * dS.abs() + TINY),
                   torch.ones(1, dtype=torch.bool, device=dev), dist=dist)


SOFTMAX_SK = (1, 31, 32, 33, 257, 2048)


@pytest.mark.parametrize("Sk", SOFTMAX_SK)
@pytest.mark.parametrize("causal", [True, False], ids=["causal", "full"])
def test_softmax(causal, Sk):
    _softmax(3, Sk // 2 + 2, Sk, causal, 3 if causal else 0)


@pytest.mark.parametrize("dist", DISTS)
def test_softmax_distributions(dist):
    _softmax(2, 300, 2048, True, 1748, dist)


# ---------------------------------------------------------------------------------------------
# E. flash's saved P against the materialised path (fp32 GEMM scores, then softmax_fwd)
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,S,H,hd,causal", [(2, 257, 16, 64, False), (1, 2048, 4, 256, True)], ids=["vit", "gptj"])
def test_flash_p_against_materialised_softmax(B, S, H, hd, causal):
    import torch

    from magma_b200 import ops

    name = f"materialised B={B} S={S} H={H} hd={hd} causal={int(causal)}"
    x, Pb = _flash(B, S, H, hd, causal)
    qkv5 = x.view.unflatten(1, (3, H, hd)).unflatten(0, (B, S))  # [B, S, 3, H, hd]
    q4, k4 = (qkv5[:, :, w].permute(0, 2, 1, 3) for w in (0, 1))  # [B, H, S, hd], row stride 3 H hd + 8
    ld = (S + 7) // 8 * 8 + 8
    sc = torch.empty(B, H, S, ld, dtype=torch.float32, device=_dev())[..., :S]
    ops.gemm(q4, k4, out=sc)  # unscaled fp32 scores, as the GEMM path of the schedules computes them
    assert x.unchanged()
    pm = ops.softmax_fwd(sc.flatten(0, 1), _fp32_inv_sqrt(hd), causal)
    s, ds = _scores(x.q, x.k, hd, 3 * U)
    vis = torch.ones(S, S, dtype=torch.bool, device=_dev())
    if causal:
        vis = vis.tril()
    p, E, flush = _probs(s, ds, vis, math.ceil(S / 32) + 5)
    pm4 = pm.unflatten(0, (B, H))
    _check_rounded(f"{name} materialised P", pm4, p, p * E + TINY, vis, flush)
    pf = Pb.view[..., :S]
    n_diff = int((bits(pf) != bits(pm4)).sum().item())
    # Both follow the rounding rule; they sum exp(s - m) in different orders (lane-strided warp sums against per-tile
    # quad sums with a running rescale), so 1 / sum may differ in its last bits and a rounding may flip.
    print(f"[materialised] {name}: flash P and materialised P differ in {n_diff} of {pf.numel()} elements")


# ---------------------------------------------------------------------------------------------
# F. rejected shapes
# ---------------------------------------------------------------------------------------------
def _raw_flash(qkv, B, Sq, Sk, H, hd, P, ldP, causal):
    """mb200_attn_fwd_flash on the fused qkv buffer with arguments ops.attn_fwd_flash would refuse."""
    from magma_b200 import ops
    from magma_b200._lib import lib

    c64, vp = ctypes.c_int64, ctypes.c_void_p
    d, ld, p = H * hd, qkv.stride(0), qkv.data_ptr()
    out = qkv.new_empty(B * Sq, d)
    return lib().mb200_attn_fwd_flash(vp(p), c64(ld), c64(hd), c64(Sq * ld), vp(p + 2 * d), c64(ld), c64(hd),
                                      c64(Sk * ld), vp(p + 4 * d), c64(ld), c64(hd), c64(Sk * ld), vp(out.data_ptr()),
                                      c64(d), vp(P.data_ptr()), c64(ldP), None, B, Sq, Sk, H, hd, int(causal),
                                      ops._stream())


def test_rejections():
    import torch

    from magma_b200 import ops
    from magma_b200._lib import MB200Error, lib

    dev, bf = _dev(), torch.bfloat16
    n0 = _count()
    with pytest.raises(MB200Error, match="unsupported"):
        ops.attn_fwd_tile(torch.zeros(2 * 129, 3 * 64, device=dev, dtype=bf), 2, 129, 1, 64)
    with pytest.raises(MB200Error, match="unsupported"):
        ops.attn_fwd_tile(torch.zeros(2 * 16, 3 * 48, device=dev, dtype=bf), 2, 16, 1, 48)
    qkv = torch.zeros(256, 3 * 64, device=dev, dtype=bf)
    P = torch.zeros(1, 1, 256, 256, device=dev, dtype=bf)
    with pytest.raises(ValueError, match="P must be"):  # ldP < Sk
        ops.attn_fwd_flash(qkv[:200], 1, 200, 1, 64, P=P[:, :, :200, :192].contiguous())
    assert _raw_flash(qkv, 1, 200, 200, 1, 64, P, 192, False) != 0
    assert b"ldP" in lib().mb200_last_error()
    assert _raw_flash(qkv, 1, 256, 128, 1, 64, P, 256, True) != 0  # causal with Sk < Sq
    assert b"causal needs Sk >= Sq" in lib().mb200_last_error()
    kc = torch.zeros(1, 1, 16, 64, device=dev, dtype=bf)
    with pytest.raises(MB200Error, match="attn_decode"):
        ops.attn_decode(qkv[:1], kc, kc.clone(), 1, 1, 64, 16)  # pos >= S_kv_max
    with pytest.raises(MB200Error, match="kv_append"):
        ops.kv_append(qkv[:8], kc, kc.clone(), 1, 8, 1, 64, 9)  # pos0 + S > S_kv_max
    long_kc = torch.zeros(1, 1, 60000, 8, device=dev, dtype=bf)
    q8 = torch.zeros(1, 3 * 8, device=dev, dtype=bf)
    with pytest.raises(MB200Error, match="shared memory"):
        ops.attn_decode(q8, long_kc, long_kc.clone(), 1, 1, 8, 52000)
    with pytest.raises(MB200Error, match="shared memory"):
        ops.attn_decode_dev(q8, long_kc, long_kc.clone(), 1, 1, 8, torch.zeros(1, dtype=torch.int32, device=dev))
    assert _count() == n0, "a rejected call launched a kernel"
