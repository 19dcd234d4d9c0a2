"""Shared pieces of the element-wise float64 reference tests (tests/test_gemm_reference_gpu.py,
tests/test_attention_reference_gpu.py, tests/test_elementwise_reference_gpu.py): sentinel-filled output buffers, bit
snapshots of inputs, bf16 ulps and round-to-nearest-even from float64, the rounding rule for bf16 outputs, the device
under test and the launch counter."""
import os

import pytest

SENTINEL = -1.5e38


def dev():
    """cuda:0 — or the CPU when a *_twin_cpu.py file replays a test body on the emulated operators."""
    import torch

    return torch.device(os.environ.get("MB200_TEST_DEVICE", "cuda:0"))


def launches():
    from magma_b200._lib import lib

    return lib().mb200_launch_count()


class Buf:
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


def rand(shape, gen, scale, dev, dtype=None):
    import torch

    t = torch.randn(*shape, generator=gen, dtype=torch.float64) * scale
    return t.to(dtype or torch.bfloat16).to(dev)


def bits(t):
    import torch

    t = t.contiguous()
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32).clone()


def ulp_bf16(x):
    """One bf16 ulp at |x| (float64): 2^(e-8) for |x| in [2^(e-1), 2^e), the subnormal spacing 2^-133 below 2^-126."""
    import torch

    _, e = torch.frexp(x.abs().clamp(min=2.0**-126))
    return torch.ldexp(torch.ones_like(x, dtype=torch.float64), e - 8)


def bf16_rne(x):
    """float64 -> the nearest bf16 value (ties to even), as float64: one rounding, not float64 -> fp32 -> bf16."""
    import torch

    u = ulp_bf16(x)
    return torch.round(x / u) * u  # torch.round rounds half to even; x / u is exact (u is a power of two)


def roundings(ref, delta, band=None):
    """bf16 roundings of the interval ends (the lower end is 0 in the flush band)."""
    import torch

    lo = ref - delta
    if band is not None:
        lo = torch.where(band, torch.zeros_like(lo), lo)
    return bf16_rne(lo), bf16_rne(ref + delta)


def check_rounded(name, got, ref, delta, keep, band=None, limit=0.001):
    """The rounding rule: a bf16 output whose float computation is within `delta` of the float64 `ref` must equal the
    reference rounding unless [ref - delta, ref + delta] holds a rounding midpoint; then it may take either rounding of
    the interval ends. At most `limit` of the kept elements (plus 8) may be ambiguous. Returns the width
    (upper - lower rounding) of every element that may take either value."""
    import torch

    keep = keep.expand(ref.shape)
    rlo, rhi = roundings(ref, delta, band)
    g = got.double()
    bad = ~((g >= rlo) & (g <= rhi)) & keep
    either = (rlo != rhi) & keep
    n_flush = int((either & band).sum().item()) if band is not None else 0
    n_amb = int(either.sum().item()) - n_flush
    n = int(keep.sum().item())
    if int(bad.sum().item()):
        i = int(bad.reshape(-1).nonzero()[0].item())
        idx = tuple(int(t) for t in torch.unravel_index(torch.tensor(i), ref.shape))
        pytest.fail(f"{name}: {int(bad.sum().item())} of {n} elements break the rounding rule; first at {idx}: got "
                    f"{g.reshape(-1)[i].item():.9g}, reference {ref.reshape(-1)[i].item():.9g} rounds to "
                    f"[{rlo.reshape(-1)[i].item():.9g}, {rhi.reshape(-1)[i].item():.9g}]")
    assert n_amb <= limit * n + 8, f"{name}: {n_amb} of {n} elements ambiguous (limit {limit:.1%})"
    print(f"[ambiguous] {name}: {n_amb} of {n} ({n_flush} more in the flush band)")
    return torch.where(either, rhi - rlo, torch.zeros_like(ref))
