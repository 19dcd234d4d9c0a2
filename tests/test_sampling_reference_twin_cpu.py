"""CPU replay of the test bodies of tests/test_sampling_reference_gpu.py and tests/test_peer_reduce_reference_gpu.py at
small sizes, on the kernel source of csrc/samp_kernels.cuh and csrc/elt_kernels.cuh and their C-ABI wrappers in
csrc/elt_abi.cuh executed on the CPU (oracle/kernel_host_exec.cpp, 1024 threads per block as on the GPU). Keeps the
float64 reference rule, its bounds, the Philox restatement, the layout checks and the argument checks honest without a
GPU. The executor's expf is the host library's and its double atomics land in thread-scheduling order, so it says
nothing about GPU bits."""
import ctypes

import numpy as np
import pytest

import test_peer_reduce_reference_gpu as P
import test_sampling_reference_gpu as S


@pytest.fixture
def on_cpu(monkeypatch):
    monkeypatch.setenv("MB200_TEST_DEVICE", "cpu")


def test_philox_restatement_matches_host_compiled_curand(kernel_ops):
    f = kernel_ops.hx_curand_uniform
    f.restype = ctypes.c_float
    f.argtypes = [ctypes.c_ulonglong] * 3
    for seed in S.BIG_SEEDS + (123,):
        for row in (0, 1, 5, 1023, 2**32 + 1):
            for off in S.OFFSETS + (7, 2**64 - 1):
                assert np.float32(f(seed, row, off)) == np.float32(S._philox_uniform(seed, row, off)), (seed, row, off)


@pytest.mark.parametrize("V", [1, 2, 31, 1025])
def test_sample_body_on_kernel_source(kernel_ops, on_cpu, V):
    import torch

    S._run_filters(torch.bfloat16, V, rows=(1, 2))
    S._run_filters(torch.float32, V, rows=(1,), filters=S.FILTERS[1::3], tag="fp32")


def test_signed_zeros_on_kernel_source(kernel_ops, on_cpu):
    import torch

    dev = torch.device("cpu")
    for dtype in (torch.float32, torch.bfloat16):
        x = torch.tensor([[-0.0, 0.0, -0.0, 0.0]], dtype=dtype, device=dev)
        tok, keep = S._sample("+-0 top_p 0.5", x, 0, 0.5, 1.0, 1, 0)
        assert keep[0].tolist() == [1, 0, 1, 1], keep[0].tolist()
        x = torch.tensor([[-0.0, 0.0]], dtype=dtype, device=dev)
        tok, keep = S._sample("+-0 top_k 1", x, 1, 0.0, 1.0, 1, 0)
        assert keep[0].tolist() == [1, 0] and int(tok[0]) == 0, (keep[0].tolist(), tok.tolist())
    S._run_filters(torch.bfloat16, 67, rows=(2,), filters=[("zeros", 0, 0.5), ("zeros", 5, 0.9), ("zeros", "tie", 0.0)],
                   tag="zeros")


def test_nan_rule_on_kernel_source(kernel_ops, on_cpu):
    S.test_nan_reads_as_minus_infinity("bf16")


def test_reference_filters_golden_on_kernel_source(kernel_ops, on_cpu):
    S.test_reference_filters_golden()


def test_peer_reduce_on_kernel_source(kernel_ops, on_cpu):
    for world in (1, 3, 16):
        for offset, n in ((0, 4), (4, 1020), (8, 1040)):
            P._case(world, 1100, offset, n)
    P.test_peer_reduce_n0_launches_nothing()


def test_argument_checks_on_kernel_source(kernel_ops, on_cpu):
    S.test_argument_checks_do_not_launch()
    P.test_peer_reduce_argument_checks_do_not_launch()
