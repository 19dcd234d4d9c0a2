"""CPU replay of the test bodies of tests/test_elementwise_reference_gpu.py at small sizes, on the kernel source of
csrc/elt_kernels.cuh and csrc/train_kernels.cuh and the C-ABI wrappers of csrc/elt_abi.cuh executed on the CPU
(oracle/kernel_host_exec.cpp). Keeps the float64 references, the bounds, the rounding rule, the sentinel and input checks
and the wrappers' argument checks honest without a GPU. The executor runs the grid of a one-SM device and the accurate
expf for __expf, so it says nothing about GPU bits or launch counts."""
import pytest

import test_elementwise_reference_gpu as E


@pytest.fixture
def on_cpu(monkeypatch):
    monkeypatch.setenv("MB200_TEST_DEVICE", "cpu")


@pytest.mark.parametrize("rows,d,dist", [(2, 8192, "normal"), (3, 1032, "outliers"), (2, 2048, "offset64"),
                                         (2, 64, "constant"), (1, 8, "normal")])
def test_layernorm_body_on_kernel_source(kernel_ops, on_cpu, rows, d, dist):
    E._layernorm_bwd(rows, d, dist, dist != "constant")


@pytest.mark.parametrize("many", [False, True])
@pytest.mark.parametrize("accumulate", [False, True])
def test_layernorm_param_grad_body_on_kernel_source(kernel_ops, on_cpu, many, accumulate):
    E._ln_param_grad(150 if many else 5, 136, many, accumulate)


@pytest.mark.parametrize("B,S,V,ldv,in_place", [(1, 3, 1003, 1008, True), (2, 2, 4100, 4104, False), (1, 2, 8, 8, False)])
def test_cross_entropy_body_on_kernel_source(kernel_ops, on_cpu, B, S, V, ldv, in_place):
    E._cross_entropy(B, S, V, ldv, in_place)


def test_cross_entropy_ignore_rule_on_kernel_source(kernel_ops, on_cpu):
    E.test_cross_entropy_ignores_every_label_outside_the_vocabulary()
    E.test_cross_entropy_all_rows_ignored()


@pytest.mark.parametrize("rows,cols", [(150, 130), (1, 2)])
def test_column_reductions_on_kernel_source(kernel_ops, on_cpu, rows, cols):
    for acc in (False, True):
        E.test_colsum(rows, cols, acc)
    for masked in (False, True):
        E.test_col_moments(rows, cols, masked)


@pytest.mark.parametrize("n", [8, 4096 * 8 + 8])
def test_dot_on_kernel_source(kernel_ops, on_cpu, n):
    E.test_dot(n, False)
    E.test_dot(n, True)


def test_rounded_elementwise_on_kernel_source(kernel_ops, on_cpu):
    E.test_quick_gelu_bwd()
    for args in ((1, 1, 1), (0, 0, 0), (1, 0, 0)):
        E.test_scale_add(*args)
    E.test_add(False)
    E.test_add(True)
    E.test_vit_assemble()
    for full in (False, True):
        E.test_channel_affine(full, full)


@pytest.mark.parametrize("B,H,W,C,s", [(1, 7, 5, 8, 2), (2, 5, 9, 16, 1), (3, 1, 1, 8, 2)])
def test_conv_layout_on_kernel_source(kernel_ops, on_cpu, B, H, W, C, s):
    E.test_im2col_col2im(B, H, W, C, s)
    E.test_avgpool_fwd_bwd(B, max(H, 3), max(W, 3), C, 3 if s == 2 else 1)


def test_layout_gather_cast_on_kernel_source(kernel_ops, on_cpu):
    E.test_patchify_vit_front_end()
    for C in (3, 8):
        E.test_nchw_to_nhwc8(C)
    E.test_embed_assemble_and_gather()
    E.test_casts()


@pytest.mark.parametrize("p", [0.0, 0.5])
def test_dropout_on_kernel_source(kernel_ops, on_cpu, p):
    E.test_dropout(p)


def test_argmax_on_kernel_source(kernel_ops, on_cpu):
    E.test_argmax()


def test_rope_table_on_kernel_source(kernel_ops, on_cpu):
    E.test_rope_table(7, 64, 2040)
    E.test_rope_table(3, 2, 0)


@pytest.mark.parametrize("ratio", [0.0, 4.0])
def test_batchnorm_bookkeeping_on_kernel_source(kernel_ops, on_cpu, ratio):
    E.test_bn_finalize_and_bwd_coeffs(ratio)


@pytest.mark.parametrize("case", ["plain", "clip_scale", "late_step", "no_decay_no_zero"])
def test_adamw_on_kernel_source(kernel_ops, on_cpu, case):
    E.test_adamw(case)


def test_decode_loop_on_kernel_source(kernel_ops, on_cpu):
    E.test_decode_embed_and_advance()


def test_argument_checks_on_kernel_source(kernel_ops, on_cpu):
    E.test_misaligned_views_are_rejected()
