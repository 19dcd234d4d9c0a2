"""CPU replay of tests/test_logits_grad_gpu.py's kernel body at small sizes, on the kernel source of
mb200_logits_grad_combine (csrc/elt_kernels.cuh, csrc/elt_abi.cuh) executed on the CPU (oracle/kernel_host_exec.cpp): the
float64 reference, the rounding rule, the sentinel and input checks and the row alignments the kernel branches on."""
import pytest

import test_logits_grad_gpu as G


@pytest.fixture
def on_cpu(monkeypatch):
    monkeypatch.setenv("MB200_TEST_DEVICE", "cpu")


@pytest.mark.parametrize("alpha", [0.0, 1.0, 0.125])
@pytest.mark.parametrize("M,V,ld_g", [(3, 1031, 1031), (2, 1031, 1088), (3, 8202, 8202), (2, 13, 13), (1, 5, 7)])
def test_logits_grad_combine_on_kernel_source(kernel_ops, on_cpu, M, V, ld_g, alpha):
    G.combine_body(M, V, ld_g, alpha)
