"""mb200_peer_reduce_bcast (csrc/elt_kernels.cuh::peer_reduce_bcast_kernel), the data-parallel gradient exchange, on one
device: the kernel only loads from and stores to the `world` pointers it is given, so buffers that all live on one GPU
stand in for the peer-mapped buffers of `world` ranks.

Contract: elements [offset, offset + n) of every buffer end equal, bit for bit, to the fp32 sum in rank order
(acc = b_0; acc += b_r for r = 1..world-1, one rounding per add, as torch computes it element-wise). Values of 1e8, 1
and -1e8 side by side make that order visible in the bits. Every other element of every buffer stays untouched, the
grid cap (max_blocks) does not change a bit, n = 0 launches nothing, and bad arguments (world outside [1, 16], offset or
n not a multiple of 4, a null or misaligned buffer) return their error code without a launch.

The device comes from MB200_TEST_DEVICE (default cuda:0): tests/test_sampling_reference_twin_cpu.py replays the bodies
at small sizes on the kernel source executed on the CPU (oracle/kernel_host_exec.cpp).
"""
import ctypes
import zlib

import pytest

from _refcheck import bits, dev as _dev, launches

pytestmark = pytest.mark.gpu

E_ALIGN, E_ARG = -3, -7


def _count():
    return launches() if _dev().type == "cuda" else 0


def _sync():
    import torch

    if _dev().type == "cuda":
        torch.cuda.synchronize()


def _buffers(world, total, seed):
    import torch

    g = torch.Generator().manual_seed(seed)
    pick = torch.randint(0, 4, (world, total), generator=g)
    big = torch.tensor([1e8, 1.0, -1e8, 0.0], dtype=torch.float64)[pick]
    x = torch.where(pick == 3, torch.randn(world, total, generator=g, dtype=torch.float64) * 3, big)
    x = x * (1 + torch.rand(world, total, generator=g, dtype=torch.float64))
    return [x[r].float().to(_dev()) for r in range(world)]


def _run(bufs, offset, n, max_blocks):
    from magma_b200 import ops

    n0 = _count()
    ops.peer_reduce_bcast([b.data_ptr() for b in bufs], offset, n, max_blocks)
    _sync()
    if _dev().type == "cuda":
        assert launches() - n0 == (1 if n else 0)


def _case(world, total, offset, n):
    import torch

    ref = _buffers(world, total, zlib.crc32(repr((world, total, offset, n)).encode()))
    acc = ref[0][offset: offset + n].clone()
    for r in range(1, world):
        acc += ref[r][offset: offset + n]
    results = []
    for mb in (0, 1, 7):
        bufs = [b.clone() for b in ref]
        _run(bufs, offset, n, mb)
        for r, (b, b0) in enumerate(zip(bufs, ref)):
            assert torch.equal(bits(b[:offset]), bits(b0[:offset])), f"rank {r}: elements before the shard changed"
            assert torch.equal(bits(b[offset + n:]), bits(b0[offset + n:])), f"rank {r}: elements after the shard changed"
            assert torch.equal(bits(b[offset: offset + n]), bits(acc)), \
                f"world {world} offset {offset} n {n} max_blocks {mb}: rank {r} differs from the rank-order fp32 sum"
        results.append(bits(bufs[0]))
    assert all(torch.equal(results[0], r) for r in results[1:])
    if n >= 1020 and world > 2:  # the values make the order visible: another order gives other bits somewhere
        other = ref[world - 1][offset: offset + n].clone()
        for r in range(world - 2, -1, -1):
            other += ref[r][offset: offset + n]
        assert not torch.equal(bits(other), bits(acc))


@pytest.mark.parametrize("world", [1, 2, 3, 8, 16])
def test_peer_reduce_is_the_rank_order_sum(world):
    total = 3 * 65536 + 40
    for offset, n in ((0, 4), (4, 1020), (1028, 4096), (0, total), (36, 3 * 65536)):
        _case(world, total, offset, n)


def test_peer_reduce_n0_launches_nothing():
    import torch

    ref = _buffers(3, 64, 1)
    bufs = [b.clone() for b in ref]
    _run(bufs, 8, 0, 0)
    assert all(torch.equal(bits(a), bits(b)) for a, b in zip(bufs, ref))


def test_peer_reduce_argument_checks_do_not_launch():
    import torch

    from magma_b200._lib import lib

    bufs = [torch.zeros(64, device=_dev()) for _ in range(17)]
    ptrs = [b.data_ptr() for b in bufs]

    def call(p, world, offset, n):
        arr = (ctypes.c_void_p * len(p))(*[ctypes.c_void_p(q) for q in p])
        n0 = launches()
        rc = lib().mb200_peer_reduce_bcast(arr, world, ctypes.c_int64(offset), ctypes.c_int64(n), 0, None)
        _sync()
        assert launches() == n0
        return rc

    assert call(ptrs, 0, 0, 16) == E_ARG
    assert call(ptrs, 17, 0, 16) == E_ARG
    assert call(ptrs[:2], 2, 2, 16) == E_ALIGN
    assert call(ptrs[:2], 2, 0, 6) == E_ALIGN
    assert call([ptrs[0], 0], 2, 0, 16) == E_ALIGN
    assert call([ptrs[0], ptrs[1] + 4], 2, 0, 16) == E_ALIGN
    assert all(bool((b == 0).all()) for b in bufs)
