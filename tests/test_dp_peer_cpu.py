"""Host logic of the peer-memory gradient exchange (magma_b200/dp.py::PeerExchange): the shard partition, and the
reduce + broadcast primitive's contract on the emulated C ABI — "ranks" are plain host buffers here; the kernel itself
runs on 2 GPUs in tests/test_dp_gpu.py."""
import torch

from magma_b200 import dp


def test_shard_bounds_cover_the_slice_in_aligned_contiguous_pieces():
    for lo, hi, w in [(0, 1024, 2), (64, 64 + 64 * 25, 8), (0, 64, 8), (128, 128, 2), (0, 241_332_224, 8)]:
        b = dp.shard_bounds(lo, hi, w)
        assert len(b) == w and b[0][0] == lo and b[-1][1] == hi
        assert all(b[i][1] == b[i + 1][0] for i in range(w - 1))
        assert all((s0 - lo) % dp.ALIGN == 0 and (s1 - s0) % 4 == 0 for s0, s1 in b)
        sizes = [s1 - s0 for s0, s1 in b]
        assert sizes == sorted(sizes, reverse=True) and sum(sizes) == hi - lo   # equal shards, ragged / empty tail only


def test_every_rank_ends_with_the_same_sum(emul_ops):
    from magma_b200 import ops

    world, n = 4, 64 * 9
    g = torch.Generator().manual_seed(0)
    grads = [torch.randn(n, generator=g) for _ in range(world)]
    want = torch.stack(grads).sum(0)
    E = [x.clone() for x in grads]                       # each rank's exchange buffer after "E <- grad"
    ptrs = [e.data_ptr() for e in E]
    for rank in range(world):                            # every rank reduces + broadcasts its own shard
        s0, s1 = dp.shard_bounds(0, n, world)[rank]
        if s1 > s0:
            ops.peer_reduce_bcast(ptrs, s0, s1 - s0)
    for e in E:
        assert torch.equal(e, E[0]) and torch.allclose(e, want, atol=1e-6)


def test_exchange_selection_and_plain_gradient_buffer_without_a_process_group(monkeypatch):
    """NCCL is the default exchange; the symmetric gradient buffer is only asked for in a multi-rank
    GPU job that selected the peer kernel — everywhere else (CPU, single process) the arena gets a plain zeroed buffer."""
    monkeypatch.delenv("MB200_DP_EXCHANGE", raising=False)
    assert dp.exchange_mode() == "nccl"
    monkeypatch.setenv("MB200_DP_EXCHANGE", "PEER")
    assert dp.exchange_mode() == "peer"
    monkeypatch.setenv("MB200_DP_EXCHANGE", "something-else")
    assert dp.exchange_mode() == "nccl"
    monkeypatch.setenv("MB200_DP_EXCHANGE", "peer")
    buf, symmetric = dp.alloc_gradient_buffer(192, "cpu")
    assert not symmetric and buf.dtype == torch.float32 and buf.shape == (192,) and float(buf.abs().sum()) == 0.0


def test_partitions_hold_for_arbitrary_sizes():
    """Property checks (hypothesis) of the two partitions the data-parallel path relies on: shard_bounds cuts any aligned
    slice into `world` contiguous, aligned, non-increasing shards; layer_chunks covers [0, n_layer) exactly once from
    the top down for any bucket count."""
    from hypothesis import given, settings
    from hypothesis import strategies as st

    @settings(max_examples=200, deadline=None)
    @given(st.integers(0, 1 << 16), st.integers(0, 1 << 14), st.integers(1, 16))
    def shards(lo64, n64, world):
        lo, hi = lo64 * dp.ALIGN, (lo64 + n64) * dp.ALIGN
        b = dp.shard_bounds(lo, hi, world)
        assert len(b) == world and b[0][0] == lo and b[-1][1] == hi
        assert all(b[i][1] == b[i + 1][0] for i in range(world - 1))
        assert all((s0 - lo) % dp.ALIGN == 0 and (s1 - s0) % 4 == 0 and s1 >= s0 for s0, s1 in b)
        sizes = [s1 - s0 for s0, s1 in b]
        assert sizes == sorted(sizes, reverse=True)

    @settings(max_examples=200, deadline=None)
    @given(st.integers(1, 96), st.integers(1, 128))
    def chunks(n_layer, n_buckets):
        c = dp.layer_chunks(n_layer, n_buckets)
        assert c[0][0] == n_layer and c[-1][1] == 0 and all(hi > lo for hi, lo in c)
        assert all(c[i][1] == c[i + 1][0] for i in range(len(c) - 1))
        assert len(c) == min(n_buckets, n_layer)

    shards()
    chunks()
