"""CPU replay of the kernel-level bodies of tests/test_sampled_decode_graph_gpu.py at small sizes, on the kernel source
of csrc/samp_kernels.cuh and its C-ABI wrappers in csrc/elt_abi.cuh executed on the CPU (oracle/kernel_host_exec.cpp):
mb200_sample_dev, with its offset read from the position in memory, draws the tokens of mb200_sample at offset
pos - s0 + 1, and rejects bad arguments (a NULL position among them) without a launch."""
import pytest

import test_sampled_decode_graph_gpu as G


@pytest.fixture
def on_cpu(monkeypatch):
    monkeypatch.setenv("MB200_TEST_DEVICE", "cpu")


def test_sample_dev_matches_sample_on_kernel_source(kernel_ops, on_cpu):
    import torch

    G._sample_dev_matches_sample(torch.bfloat16, 1031, 2, G.FILTERS[:3], temps=(0.7,))
    G._sample_dev_matches_sample(torch.float32, 1031, 1, G.FILTERS[3:], temps=(1.3,))


def test_sample_dev_argument_checks_on_kernel_source(kernel_ops, on_cpu):
    G._argument_checks()
