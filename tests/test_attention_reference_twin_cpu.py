"""CPU replay of the test bodies of tests/test_attention_reference_gpu.py at small sizes: the tile, flash, cache, append
and decode bodies on the emulated operators (oracle/cabi_emul.cpp), the softmax bodies on the kernel source of
csrc/elt_kernels.cuh executed on the CPU (oracle/kernel_host_exec.cpp). Keeps the float64 references, the bounds, the
rounding rule and the sentinel and input checks honest without a GPU; the kernels themselves are verified by the
`-m gpu` run only. Launches are counted on the GPU only."""
import pytest

import test_attention_reference_gpu as A


@pytest.fixture
def on_cpu(monkeypatch):
    monkeypatch.setenv("MB200_TEST_DEVICE", "cpu")


@pytest.mark.parametrize("dist", A.DISTS)
@pytest.mark.parametrize("S,hd,rot", [(1, 64, 0), (9, 64, 64), (13, 128, 64)])
def test_tile_body_on_emulation(emul_ops, on_cpu, S, hd, rot, dist):
    A._tile(2, S, 2, hd, rot, dist)


@pytest.mark.parametrize("dist", A.DISTS)
@pytest.mark.parametrize("S,causal", [(1, True), (130, True), (70, False)])
def test_flash_body_on_emulation(emul_ops, on_cpu, S, causal, dist):
    A._flash(1, S, 1, 64, causal, dist)


def test_prefill_body_on_emulation(emul_ops, on_cpu):
    for pos0, S in ((1, 20), (129, 3)):  # the causal limit of the first query tile before / past a key-tile boundary
        A._prefill(2, S, 1, 64, pos0)


@pytest.mark.parametrize("dist", A.DISTS)
@pytest.mark.parametrize("hd,pos", [(8, 0), (40, 33), (64, 300)])
def test_decode_body_on_emulation(emul_ops, on_cpu, hd, pos, dist):
    A._decode(2, 3, hd, pos, dist)


@pytest.mark.parametrize("dist", A.DISTS)
@pytest.mark.parametrize("Sk,causal", [(1, False), (33, True), (257, True)])
def test_softmax_body_on_kernel_source(kernel_ops, on_cpu, Sk, causal, dist):
    A._softmax(2, Sk // 2 + 2, Sk, causal, 3 if causal else 0, dist)
