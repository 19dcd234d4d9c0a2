"""Float64 reference tests of mb200_sample (csrc/elt_abi.cuh, body in csrc/samp_kernels.cuh): the top-k filter, the
reference's inverted nucleus filter, softmax(x / T) and the Philox multinomial draw, which `generate` runs for every
token at temperature > 0.

The reference rule, in float64 on the device from the same bf16 / fp32 logits x:
  - order: stable descending, -0 == +0, ties by index; NaN reads as -inf (both signs);
  - K = the first top_k of that order (the whole row when top_k == 0 or top_k >= V); M = max over K, top1 = rank 0;
  - masses w_r = exp(x_r - M) over K in rank order, Z = sum w, C_r the inclusive cumulative mass;
  - p32 = float32(top_p), what the kernel receives; when p32 > 0, m = #{r : C_r < (1 - p32) Z} capped at |K| - 1, and
    ranks 1..m are removed (sampling.py:13-17 shifts the removal mask right by one); keep = K minus those ranks;
  - draw weights g_j = exp((x_j - M) / T32) over keep, in index order, G their inclusive cumulative sum, W = G[-1];
  - u = curand_uniform of Philox4x32-10 with key = seed, counter = (offset // 4 in the low 64 bits, row in the high 64),
    output word offset % 4, f32(word) * 2^-32 + 2^-33 in fp32 (_philox_uniform restates it bit for bit); the token is
    the first kept index with G >= u W.
  - A row whose entries are all -inf (or NaN) has no distribution: the kernel returns top1 = index 0, and keep = K when
    top_p == 0, {top1} otherwise. The header states this next to mb200_sample.

Bounds. The library is built without --use_fast_math: expf is the Math API's expf (2 ulp, so a relative 2^-22), and
u = 2^-24. A mass expf(x - M) is off by 2^-22 + u |x - M| relative (the subtraction rounds once), a draw weight
expf((x - M) * fl(1 / T)) by 2^-22 + 3u |(x - M) / T| (three roundings of the argument); both carry an absolute 2^-147
besides, for results in or below the subnormal range, and a factor 1.001 for second-order terms. Entries equal to the
maximum carry no error: x - M = 0 exactly and expf(0) = 1, so ties at the top (an all-equal row) have exact masses and
m is exact there. The kernel adds in
double, in its own order: at most n 2^-52 of the total. With d_r the sum of those term errors over ranks <= r:
  - Mask. The kernel's comparison C'_r < thr' differs from the reference's by at most D_r = d_r + d_Z + n 2^-52 Z, so
    the kernel's m' lies in [#{C_r + D_r < thr}, #{C_r - D_r < thr}]. The removed set must be exactly ranks 1..m' of the
    stable order for that m'; a row whose window holds more than one m is "ambiguous". Every other mask byte is exact.
  - Token. The kernel picks i when C'_excl(i) < u W' <= C'_incl(i). Index i is acceptable when it is kept and
    G_excl(i) - E_i < u W <= G(i) + E_i with E_i = e_i + e_W + n 2^-52 W (e: the draw weights' term errors). The
    predicted token is always acceptable; a draw with more than one acceptable index is "ambiguous" and may take any
    of them. All other draws must equal the predicted token.
  Both ambiguous shares are printed and capped (AMBIGUOUS_MAX of the rows, plus 2); flat rows of 50k nearly equal
  masses are where the windows are widest (each mass is ~2e-5 Z, the window ~5e-7 Z).

Layouts and contract: logits are a view with row stride V + 24 in a NaN-filled storage with a spare NaN row (reading
the padding would poison every sum), tokens and the keep mask land in sentinel buffers of which exactly rows and
rows x V entries may change, the logits stay unchanged byte for byte, each call is one launch, and a rerun gives the
same bits (the mass histogram adds doubles with atomicAdd; a rerun that differs is a finding). Bad arguments return
their error code without a launch. `generate` at temperature > 0 is checked call by call against the same rule.

The device comes from MB200_TEST_DEVICE (default cuda:0): tests/test_sampling_reference_twin_cpu.py replays these
bodies at small sizes on the kernel source executed on the CPU (oracle/kernel_host_exec.cpp).
"""
import ctypes
import math
import os
import zlib

import numpy as np
import pytest

from _refcheck import bits, dev as _dev, launches

pytestmark = pytest.mark.gpu

U = 2.0**-24
EXP_ULP2 = 2.0**-22
ABS_TINY = 2.0**-147
AMBIGUOUS_MAX = 0.05
NAN_PAD = 24
BIG_SEEDS = (0x9E3779B97F4A7C15, 2**62 + 12345, 0xFFFFFFFF00000001, 7)
OFFSETS = (0, 1, 3, 4, 5, 2**32 + 3, 2**34 + 5)
E_SHAPE, E_DTYPE, E_ARG = -1, -2, -7


def _gen(*key):
    import torch

    return torch.Generator().manual_seed(zlib.crc32(repr(key).encode()))


def _count():
    return launches() if _dev().type == "cuda" else 0


# ---------------------------------------------------------------------------------------------
# Philox4x32-10 as curand_init(seed, subsequence = row, offset) + curand_uniform computes it
# ---------------------------------------------------------------------------------------------
def _philox_word(seed, row, offset):
    m32 = 0xFFFFFFFF
    n = offset // 4
    c = [n & m32, (n >> 32) & m32, row & m32, (row >> 32) & m32]
    k = [seed & m32, (seed >> 32) & m32]
    for r in range(10):
        p0, p1 = 0xD2511F53 * c[0], 0xCD9E8D57 * c[2]
        c = [(p1 >> 32) ^ c[1] ^ k[0], p1 & m32, (p0 >> 32) ^ c[3] ^ k[1], p0 & m32]
        k = [(k[0] + 0x9E3779B9) & m32, (k[1] + 0xBB67AE85) & m32]
    return c[offset % 4]


def _philox_uniform(seed, row, offset):
    f32 = np.float32
    return float(f32(_philox_word(seed, row, offset)) * f32(2.0**-32) + f32(2.0**-33))


# ---------------------------------------------------------------------------------------------
# the reference rule
# ---------------------------------------------------------------------------------------------
def _canonical(x):
    """float64 copy with NaN -> -inf and -0 -> +0 (x + 0.0 is +0 for either zero)."""
    import torch

    x = x.double()
    return torch.where(torch.isnan(x), torch.full_like(x, -math.inf), x) + 0.0


def _check(name, x, top_k, top_p, T, seed, offset, tokens, keep):
    """Holds the kernel's tokens [R] and keep mask [R, V] to the reference rule. Returns (ambiguous mask rows,
    ambiguous draws, exactly predicted draws, rows)."""
    import torch

    R, V = x.shape
    dev = x.device
    x = _canonical(x)
    keep = keep.bool()
    tokens = tokens.to(dev)
    ar = torch.arange(R, device=dev)
    vals, order = torch.sort(x, dim=1, descending=True, stable=True)
    rank = torch.empty_like(order)
    rank.scatter_(1, order, torch.arange(V, device=dev).expand(R, V).contiguous())
    kk = V if top_k == 0 or top_k >= V else top_k
    in_k = rank < kk
    M = vals[:, :1]
    dead = torch.isneginf(M[:, 0])
    top1 = order[:, 0]
    p32 = float(np.float32(top_p))

    # --- mask ---
    if p32 > 0:
        w = torch.exp(vals[:, :kk] - M)
        dw = torch.where((w > 0) & (w < 1), w * (EXP_ULP2 + U * (vals[:, :kk] - M).abs()) * 1.001, torch.zeros_like(w))
        dw = dw + torch.where(w < 1, ABS_TINY, 0.0)
        C = torch.cumsum(w, 1)
        Z = C[:, -1:]
        d = torch.cumsum(dw, 1)
        D = d + d[:, -1:] + kk * 2.0**-52 * Z
        thr = (1.0 - p32) * Z
        m_lo = (C + D < thr).sum(1).clamp(max=kk - 1)
        m_hi = (C - D < thr).sum(1).clamp(max=kk - 1)
        m_lo = torch.where(dead, torch.full_like(m_lo, kk - 1), m_lo)
        m_hi = torch.where(dead, torch.full_like(m_hi, kk - 1), m_hi)
    else:
        m_lo = m_hi = torch.zeros(R, dtype=torch.int64, device=dev)
    assert not bool((keep & ~in_k).any()), f"{name}: a token outside the top-k set is kept"
    removed = in_k & ~keep
    m = removed.sum(1)
    bad_m = (m < m_lo) | (m > m_hi)
    if bool(bad_m.any()):
        r = int(bad_m.nonzero()[0])
        pytest.fail(f"{name}: row {r} removes {int(m[r])} ranks, the reference window is [{int(m_lo[r])}, {int(m_hi[r])}]")
    want_removed = in_k & (rank >= 1) & (rank <= m[:, None])
    bad = removed != want_removed
    if bool(bad.any()):
        r, i = (int(t) for t in bad.nonzero()[0])
        pytest.fail(f"{name}: row {r}: index {i} (rank {int(rank[r, i])}, value {float(x[r, i])!r}) is "
                    f"{'removed' if bool(removed[r, i]) else 'kept'}; the stable order removes ranks 1..{int(m[r])}")
    n_amb_mask = int((m_lo != m_hi).sum())

    # --- draw ---
    assert bool(((tokens >= 0) & (tokens < V)).all()), f"{name}: token out of range {tokens.tolist()}"
    assert bool(keep[ar, tokens].all()), f"{name}: a drawn token is not kept"
    live = ~dead
    assert torch.equal(tokens[dead], top1[dead]), f"{name}: an all -inf row does not return top1"
    T32 = float(np.float32(T))
    a = torch.where(keep, (x - M) / T32, torch.full_like(x, -math.inf))
    g = torch.exp(a)
    g = torch.where(keep & live[:, None], g, torch.zeros_like(g))
    dg = torch.where((g > 0) & (g < 1), g * (EXP_ULP2 + 3 * U * a.abs()) * 1.001, torch.zeros_like(g))
    dg = dg + (keep & (g < 1)) * ABS_TINY
    G = torch.cumsum(g, 1)
    W = G[:, -1:]
    e = torch.cumsum(dg, 1)
    E = e + e[:, -1:] + V * 2.0**-52 * W
    f = torch.tensor([_philox_uniform(seed, r, offset) for r in range(R)], dtype=torch.float64, device=dev)
    target = f[:, None] * W
    pred = torch.searchsorted(G, target).clamp(max=V - 1)[:, 0]
    ok = keep & (G - g - E < target) & (target <= G + E)
    n_ok = ok.sum(1)
    bad = live & ~ok[ar, tokens]
    if bool(bad.any()):
        r = int(bad.nonzero()[0])
        pytest.fail(f"{name}: row {r} drew {int(tokens[r])}, predicted {int(pred[r])} (u = {float(f[r])!r}, acceptable "
                    f"{ok[r].nonzero()[:, 0].tolist()[:8]})")
    n_amb_draw = int((live & (n_ok > 1)).sum())
    n_exact = int((live & (tokens == pred)).sum()) + int(dead.sum())
    assert bool((tokens[live & (n_ok == 1)] == pred[live & (n_ok == 1)]).all())
    return n_amb_mask, n_amb_draw, n_exact, R


# ---------------------------------------------------------------------------------------------
# one call of the C ABI, with its layout, launch and rerun checks
# ---------------------------------------------------------------------------------------------
def _raw(logits_ptr, dtype_code, ld, R, V, T, top_k, top_p, seed, offset, tok_ptr, mask_ptr):
    from magma_b200 import ops
    from magma_b200._lib import lib

    return lib().mb200_sample(ctypes.c_void_p(logits_ptr), int(dtype_code), ctypes.c_int64(ld), int(R), int(V),
                              ctypes.c_float(T), int(top_k), ctypes.c_float(top_p), ctypes.c_uint64(seed),
                              ctypes.c_uint64(offset), ctypes.c_void_p(tok_ptr), ctypes.c_void_p(mask_ptr), ops._stream())


def _sample(name, x, top_k, top_p, T, seed, offset):
    """x [R, V] bf16 / fp32 on the device, copied into a NaN-padded view; returns (tokens, keep) of the kernel."""
    import torch

    R, V = x.shape
    ld = V + NAN_PAD
    store = torch.full(((R + 1) * ld,), math.nan, dtype=x.dtype, device=x.device)
    view = store[: R * ld].view(R, ld)[:, :V]
    view.copy_(x)
    before = bits(store)
    code = 0 if x.dtype == torch.bfloat16 else 1
    outs = []
    for _ in range(2):
        tok = torch.full((R + 4,), -7, dtype=torch.int64, device=x.device)
        mask = torch.full((R * V + 64,), 0xAB, dtype=torch.uint8, device=x.device)
        n0 = _count()
        rc = _raw(view.data_ptr(), code, ld, R, V, T, top_k, top_p, seed, offset, tok.data_ptr(), mask.data_ptr())
        assert rc == 0, f"{name}: rc {rc}"
        if x.device.type == "cuda":
            torch.cuda.synchronize()
            assert launches() - n0 == 1, f"{name}: {launches() - n0} launches"
        assert torch.equal(bits(store), before), f"{name}: the logits were modified"
        assert bool((tok[R:] == -7).all()), f"{name}: tokens written past row {R}"
        assert bool((mask[R * V:] == 0xAB).all()), f"{name}: keep mask written past {R} x {V}"
        k = mask[: R * V].view(R, V)
        assert bool(((k == 0) | (k == 1)).all()), f"{name}: keep mask bytes other than 0 / 1"
        outs.append((tok[:R].clone(), k.clone()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1]), f"{name}: rerun differs"
    return outs[0]


def _case(name, x, top_k, top_p, T, seed, offset):
    tokens, keep = _sample(name, x, top_k, top_p, T, seed, offset)
    return _check(name, x, top_k, top_p, T, seed, offset, tokens, keep)


def _logits(dist, R, V, dtype, gen):
    """float64 CPU logits of a distribution, rounded to dtype."""
    import torch

    r = torch.randn(R, V, generator=gen, dtype=torch.float64)
    if dist == "peaked":
        x = r * 4
    elif dist == "flat":
        x = r * 0.05
    elif dist == "mid":
        x = r * 1.5
    elif dist == "huge":
        x = r * 1e4
    elif dist == "steps":  # a few values, many ties
        x = -0.5 * torch.randint(0, 6, (R, V), generator=gen).double()
    elif dist == "const":
        x = torch.full((R, V), 2.5, dtype=torch.float64)
    elif dist == "zeros":  # -0 and +0 are ties; -1 below them
        s = torch.randint(0, 3, (R, V), generator=gen)
        x = torch.where(s == 0, torch.full_like(r, -0.0), torch.where(s == 1, torch.zeros_like(r), -torch.ones_like(r)))
    elif dist == "neginf":  # about 7 in 8 entries -inf
        x = torch.where(torch.rand(R, V, generator=gen) < 0.875, torch.full_like(r, -math.inf), r * 1.5)
        x[:, 0] = r[:, 0]
    elif dist == "single":  # one finite entry per row
        x = torch.full((R, V), -math.inf, dtype=torch.float64)
        x[torch.arange(R), torch.randint(0, V, (R,), generator=gen)] = r[:, 0] * 3
    else:
        raise ValueError(dist)
    return x.to(dtype)


def _tie_k(x):
    """A k whose boundary falls inside a tie group of row 0 (the k-th and (k+1)-th of the stable order are equal)."""
    import torch

    v = torch.sort(_canonical(x[0]), descending=True, stable=True).values
    V = v.numel()
    for r in list(range(V // 3, V)) + list(range(1, V // 3)):
        if v[r - 1] == v[r] and not math.isinf(float(v[r])):
            return r
    return 1


def _k(spec, V, x):
    if spec == "tie":
        return _tie_k(x)
    return {"V-1": V - 1, "V": V, "V+5": V + 5, "half": max(1, V // 2)}.get(spec, spec)


# (distribution, top_k, top_p) — every call runs with one of the temperatures, seeds and offsets in turn
FILTERS = [("mid", 0, 0.9), ("flat", 0, 0.5), ("peaked", 40, 0.0), ("mid", 1, 0.9), ("flat", "V-1", 1e-6),
           ("steps", "V", 0.5), ("peaked", "V+5", 1.0), ("steps", "tie", 0.9), ("neginf", "half", 0.9),
           ("neginf", 40, 0.0), ("single", 40, 0.5), ("huge", 0, 0.9), ("const", 0, 0.3), ("zeros", 0, 0.5),
           ("steps", 0, "tie"), ("mid", 0, 0.0)]
TEMPS = (0.05, 0.7, 1.0, 5.0)
ROWS = (1, 3, 64)


def _tie_p(x):
    """A top_p whose boundary (1 - p) Z falls strictly inside the tie group that holds rank V // 2 of row 0, halfway
    between two of its cumulative masses (so the boundary is not ambiguous)."""
    v = _canonical(x[0]).sort(descending=True, stable=True).values
    w = (v - v[0]).exp()
    C = w.cumsum(0)
    r = v.numel() // 2
    tgt = float((C[r - 1] + C[r]) / 2 / C[-1]) if r >= 1 else 0.5
    return 1.0 - tgt


def _run_filters(dtype, V, rows=ROWS, filters=FILTERS, tag=""):
    import torch

    dev = _dev()
    amb_m = amb_d = exact = n = 0
    for ci, (dist, kspec, p) in enumerate(filters):
        R = rows[ci % len(rows)]
        x = _logits(dist, R, V, dtype, _gen("sample", tag, str(dtype), V, ci))
        k = _k(kspec, V, x)
        if p == "tie":
            p = _tie_p(x)
        T, seed, off = TEMPS[ci % len(TEMPS)], BIG_SEEDS[ci % len(BIG_SEEDS)], OFFSETS[ci % len(OFFSETS)]
        name = f"sample {dtype} V={V} R={R} {dist} k={k} p={p:.6g} T={T} seed={seed:#x} offset={off}"
        am, ad, ex, nn = _case(name, x.to(dev), k, p, T, seed, off)
        amb_m, amb_d, exact, n = amb_m + am, amb_d + ad, exact + ex, n + nn
    print(f"[ambiguous] sample {dtype} V={V}: mask rows {amb_m} of {n}, draws {amb_d} of {n}; "
          f"{exact} draws predicted exactly")
    assert amb_m <= AMBIGUOUS_MAX * n + 2, f"{amb_m} of {n} mask rows ambiguous"
    assert amb_d <= AMBIGUOUS_MAX * n + 2, f"{amb_d} of {n} draws ambiguous"
    return exact, n


def test_philox_restatement_known_value():
    """curand_uniform after curand_init(123, 5, 7): 0x3f07db65 (the host-compiled curand header gives the same)."""
    assert np.float32(_philox_uniform(123, 5, 7)).view(np.uint32) == 0x3F07DB65


@pytest.mark.parametrize("V", [1, 2, 31, 1023, 1024, 1025, 4097, 50257, 50258, 50400])
@pytest.mark.parametrize("dtype", ["bf16", "fp32"])
def test_sample_against_reference(dtype, V):
    import torch

    _run_filters(torch.bfloat16 if dtype == "bf16" else torch.float32, V)


def test_sample_1024_rows_one_subsequence_each():
    """1024 rows, each drawing from its own Philox subsequence (row = blockIdx.x), with an offset whose counter needs
    the high word."""
    import torch

    dev = _dev()
    R, V = 1024, 1025
    x = _logits("mid", R, V, torch.bfloat16, _gen("sample rows"))
    am, ad, ex, n = _case("sample R=1024", x.to(dev), 0, 0.9, 0.7, BIG_SEEDS[0], 2**34 + 5)
    print(f"[ambiguous] sample R=1024: mask rows {am} of {n}, draws {ad} of {n}; {ex} draws predicted exactly")
    assert am <= AMBIGUOUS_MAX * n + 2 and ad <= AMBIGUOUS_MAX * n + 2
    assert ex >= n - ad


def test_signed_zeros_are_ties():
    """-0 and +0 are one value to the order (torch.sort / torch.topk): ties go by index."""
    import torch

    dev = _dev()
    for dtype in (torch.float32, torch.bfloat16):
        x = torch.tensor([[-0.0, 0.0, -0.0, 0.0]], dtype=dtype, device=dev)
        tok, keep = _sample("+-0 top_p 0.5", x, 0, 0.5, 1.0, 1, 0)
        # cum = .25, .5, .75, 1: ranks with cum < 0.5, shifted by one, remove rank 1 only, which is index 1
        assert keep[0].tolist() == [1, 0, 1, 1], keep[0].tolist()
        _check("+-0 top_p 0.5", x, 0, 0.5, 1.0, 1, 0, tok, keep)
        x = torch.tensor([[-0.0, 0.0]], dtype=dtype, device=dev)
        tok, keep = _sample("+-0 top_k 1", x, 1, 0.0, 1.0, 1, 0)
        assert keep[0].tolist() == [1, 0] and int(tok[0]) == 0, (keep[0].tolist(), tok.tolist())
    _run_filters(torch.bfloat16, 1031, rows=(5,), filters=[("zeros", 0, 0.5), ("zeros", 40, 0.9), ("zeros", "tie", 0.0)],
                 tag="zeros")


def _nan(dtype, negative):
    import torch

    if dtype == torch.bfloat16:
        return torch.tensor([-64 if negative else 0x7FC0], dtype=torch.int16).view(torch.bfloat16)
    return torch.tensor([-4194304 if negative else 0x7FC00000], dtype=torch.int32).view(torch.float32)


@pytest.mark.parametrize("dtype", ["bf16", "fp32"])
def test_nan_reads_as_minus_infinity(dtype):
    """NaN of either sign is read as -inf (rows with NaN are outside the reference's domain: torch.multinomial raises);
    an all -inf or all-NaN row returns index 0."""
    import torch

    dt = torch.bfloat16 if dtype == "bf16" else torch.float32
    dev = _dev()
    V = 300
    x = _logits("mid", 4, V, dt, _gen("nan", dtype))
    g = _gen("nan pos", dtype)
    pos = torch.randperm(V, generator=g)[:80].view(2, 40)
    x[0, pos[0]] = _nan(dt, False)
    x[0, pos[1]] = _nan(dt, True)
    x[1, :] = _nan(dt, True)
    x[1, 7] = 1.0
    x[2, :] = -math.inf
    x[3, :] = _nan(dt, False)
    x[3, 1::2] = _nan(dt, True)
    assert bool(torch.signbit(x[0, pos[1]].float()).all()) and not bool(torch.signbit(x[0, pos[0]].float()).any())
    for k, p in ((0, 0.9), (0, 0.0), (40, 0.5), (V + 5, 1.0)):
        name = f"NaN {dtype} k={k} p={p}"
        tok, keep = _sample(name, x.to(dev), k, p, 0.7, 99, 3)
        _check(name, x.to(dev), k, p, 0.7, 99, 3, tok, keep)
        assert int(tok[1]) == 7 and int(tok[2]) == 0 and int(tok[3]) == 0, tok.tolist()
        kk = V if k == 0 or k >= V else k
        for r in (2, 3):  # all -inf: keep = K (the first kk indices), or {0} when top_p > 0
            want = torch.zeros(V, dtype=torch.uint8)
            want[: (1 if p > 0 else kk)] = 1
            assert torch.equal(keep[r].cpu(), want), (r, keep[r].nonzero()[:, 0].tolist()[:8])


def test_reference_filters_golden():
    """The keep mask is the reference's own top_k_filter / top_p_filter output (tests/golden/sampling_filters.pt, made by
    magma/sampling.py): kept exactly where the golden logits are finite."""
    import torch

    dev = _dev()
    rec = torch.load(os.path.join(os.path.dirname(__file__), "golden", "sampling_filters.pt"))
    for key, src, k, p in (("top_k_5", "logits", 5, 0.0), ("top_p_0.9", "logits", 0, 0.9), ("top_p_0.5", "logits", 0, 0.5),
                           ("quirk_0.5", "quirk_probs", 0, 0.5), ("quirk_0.9", "quirk_probs", 0, 0.9)):
        x = rec[src].float().to(dev)
        tok, keep = _sample(f"golden {key}", x, k, p, 1.0, 5, 0)
        want = (rec[key] > -math.inf).to(torch.uint8)
        assert torch.equal(keep.cpu(), want), f"golden {key}: {keep.cpu().tolist()} vs {want.tolist()}"
        _check(f"golden {key}", x, k, p, 1.0, 5, 0, tok, keep)


def test_argument_checks_do_not_launch():
    import torch

    dev = _dev()
    x = torch.zeros(2, 64, dtype=torch.bfloat16, device=dev)
    tok = torch.full((4,), -7, dtype=torch.int64, device=dev)
    good = dict(code=0, ld=64, R=2, V=64, T=1.0, k=0, p=0.9)
    bad = [("rows=0", dict(R=0), E_SHAPE), ("rows<0", dict(R=-1), E_SHAPE), ("V=0", dict(V=0), E_SHAPE),
           ("V<0", dict(V=-3), E_SHAPE), ("ld<V", dict(ld=63), E_SHAPE), ("T=0", dict(T=0.0), E_ARG),
           ("T<0", dict(T=-1.0), E_ARG), ("T=NaN", dict(T=math.nan), E_ARG), ("top_k<0", dict(k=-1), E_ARG),
           ("top_p<0", dict(p=-0.1), E_ARG), ("top_p>1", dict(p=1.5), E_ARG), ("top_p=NaN", dict(p=math.nan), E_ARG),
           ("dtype", dict(code=7), E_DTYPE)]
    for name, change, want in bad:
        a = dict(good, **change)
        n0 = launches()
        rc = _raw(x.data_ptr(), a["code"], a["ld"], a["R"], a["V"], a["T"], a["k"], a["p"], 1, 0, tok.data_ptr(), 0)
        if dev.type == "cuda":
            torch.cuda.synchronize()
        assert rc == want, f"{name}: rc {rc}, expected {want}"
        assert launches() == n0, f"{name}: launched"
        assert bool((tok == -7).all()), f"{name}: tokens written"


@pytest.mark.parametrize("top_k,top_p", [(0, 0.9), (20, 0.0)])
def test_generate_samples_by_the_reference_rule(monkeypatch, top_k, top_p):
    """generate(temperature=0.7) on a small model: every ops.sample call is held to the reference rule, the seed is one
    per call of generate, the offset is the step index, the logits view is V wide with the LM head's row stride, and
    the emitted ids are the recorded draws in order."""
    import torch

    from _gpu_util import build_magma_from_weights
    from magma_b200 import ops
    from oracle import magma_oracle as O
    from tools.model_check import small_cfg

    dev = _dev()
    cfg = small_cfg(n_layer=2, vocab=1031)
    w = O.init_weights(cfg, seed=21)
    w["lm.lm_head.weight"] = w["lm.lm_head.weight"] * 4
    w16 = {k: v.to(torch.bfloat16).float() for k, v in w.items()}
    model = build_magma_from_weights(w16, cfg, {"mlp": {"adapter_type": "normal", "downsample_factor": 4}}, 40, dev,
                                     vit_name="clip_vit_sample_case")
    model.eval()
    emb = (torch.randn(3, 6, cfg.d, generator=_gen("generate")) * 0.5).to(torch.bfloat16).to(dev)
    calls = []
    orig = ops.sample

    def recording(logits, temperature, top_k=0, top_p=0.0, seed=0, offset=0, return_mask=False):
        tok = orig(logits, temperature, top_k=top_k, top_p=top_p, seed=seed, offset=offset, return_mask=return_mask)
        calls.append({"x": logits.clone(), "shape": tuple(logits.shape), "stride": logits.stride(), "T": temperature,
                      "k": top_k, "p": top_p, "seed": seed, "offset": offset, "tok": tok.clone()})
        return tok

    monkeypatch.setattr(ops, "sample", recording)
    out = model.generate(emb, max_steps=24, temperature=0.7, top_k=top_k, top_p=top_p, decode=False)
    assert calls, "generate did not sample"
    V, ldv = cfg.vocab, model.lm.ldv
    n_steps = out.shape[1] - emb.shape[1]
    assert len(calls) >= n_steps
    amb_m = amb_d = exact = n = 0
    for i, c in enumerate(calls):
        assert c["shape"] == (emb.shape[0], V) and c["stride"] == (ldv, 1), (c["shape"], c["stride"], ldv)
        assert c["seed"] == calls[0]["seed"] and c["offset"] == i and c["T"] == 0.7
        assert c["k"] == top_k and c["p"] == top_p
        tok, keep = orig(c["x"], c["T"], top_k=c["k"], top_p=c["p"], seed=c["seed"], offset=c["offset"], return_mask=True)
        assert torch.equal(tok, c["tok"]), f"step {i}: the draw depends on the keep mask being written"
        am, ad, ex, nn = _check(f"generate step {i}", c["x"], c["k"], c["p"], c["T"], c["seed"], c["offset"], tok, keep)
        amb_m, amb_d, exact, n = amb_m + am, amb_d + ad, exact + ex, n + nn
    drawn = torch.stack([c["tok"] for c in calls[:n_steps]], 1).cpu()
    assert torch.equal(out[:, emb.shape[1]:].cpu(), drawn)
    print(f"[ambiguous] generate k={top_k} p={top_p}: mask rows {amb_m} of {n}, draws {amb_d} of {n}; {exact} exact")
