"""GPU parity tests of the wgmma GEMM core through the C ABI (mb200_gemm) against an fp32 matmul of the same bf16
inputs. Tolerance: relative Frobenius error < 2e-2 (bf16 output rounding is ~2^-9 relative; fp32 outputs < 5e-3)."""
import pytest

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("group", ["basic", "majors", "tails", "epilogue", "batched", "pair", "streamk", "splitk", "smallm"])
def test_gemm_group(group):
    import torch

    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but no CUDA device is visible (magma_b200 has no CPU fallback)")
    from tools import gemm_check

    assert gemm_check.run_group(group) == 0


def test_gemm_argument_validation():
    import torch

    from magma_b200 import ops
    from magma_b200._lib import MB200Error

    dev = torch.device("cuda:0")
    a = torch.zeros(64, 64, device=dev, dtype=torch.bfloat16)
    with pytest.raises(MB200Error, match="ld"):
        ops.gemm(a[:, :60][:, ::1].as_strided((64, 60), (62, 1)), a[:, :60].as_strided((64, 60), (62, 1)))
    with pytest.raises(TypeError):
        ops.gemm(a.float(), a)
    with pytest.raises(MB200Error, match="accumulate"):
        ops.gemm(a, a, accumulate=True)  # accumulate needs an f32 output
