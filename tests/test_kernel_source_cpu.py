"""The SOURCE of the training kernels (magma_b200/csrc/train_kernels.cuh), executed on the CPU.

oracle/kernel_host_exec.cpp compiles those kernels and their C-ABI wrappers (csrc/elt_abi.cuh) unchanged as host C++ and
runs them with the CUDA execution model emulated (threads of a block = OS threads, __syncthreads = barrier, warp shuffles
and atomicAdd emulated, blocks in sequence); the hx_* names are the wrappers without their stream argument. Here each
kernel is held to the torch formula its GPU test uses (tests/test_training_paths_gpu.py): this checks what a kernel
COMPUTES — indexing, 8-wide vector handling, masks, smem reductions, row-chunk accumulation through atomics — not what
the hardware does with it."""
import ctypes

import pytest
import torch
import torch.nn.functional as F


@pytest.fixture(scope="module")
def kx():
    from oracle import build_emul

    return ctypes.CDLL(build_emul.build_kernel_exec())


def rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-12)).item()


def P(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def bf(g, *shape, scale=1.0):
    return (torch.randn(*shape, generator=g) * scale).to(torch.bfloat16)


LL = ctypes.c_longlong


def test_quick_gelu_bwd_kernel_source(kx):
    g = torch.Generator().manual_seed(0)
    pre, dy = bf(g, 37, 64, scale=2.0), bf(g, 37, 64)
    x = pre.float().requires_grad_(True)
    (x * torch.sigmoid(1.702 * x)).backward(dy.float())
    out = torch.empty_like(dy)
    kx.hx_quick_gelu_bwd(P(dy), P(pre), P(out), LL(dy.numel()))
    assert rel(out, x.grad) < 5e-3
    buf = dy.clone()
    kx.hx_quick_gelu_bwd(P(buf), P(pre), P(buf), LL(buf.numel()))   # in place
    assert torch.equal(buf, out)


def test_scale_add_and_dot_kernel_source(kx):
    g = torch.Generator().manual_seed(1)
    u, r1, r2 = bf(g, 20, 48), bf(g, 20, 48), bf(g, 20, 48)
    s = torch.tensor([0.625])
    out = torch.empty_like(u)
    kx.hx_scale_add(P(u), P(s), P(r1), P(r2), P(out), LL(u.numel()))
    assert rel(out, 0.625 * u.float() + r1.float() + r2.float()) < 5e-3
    kx.hx_scale_add(P(u), None, None, None, P(out), LL(u.numel()))
    assert torch.equal(out, u)
    a, b = bf(g, 4096 + 64), bf(g, 4096 + 64)
    acc = torch.tensor([3.0])
    kx.hx_dot(P(a), P(b), LL(a.numel()), P(acc), 0)
    want = float((a.float() * b.float()).sum())
    assert abs(float(acc) - want) < 1e-3 * (a.float().norm() * b.float().norm()).item()
    kx.hx_dot(P(a), P(b), LL(a.numel()), P(acc), 1)
    assert abs(float(acc) - 2 * want) < 2e-3 * (a.float().norm() * b.float().norm()).item()


def test_layernorm_param_grad_rows_kernel_source(kx):
    g = torch.Generator().manual_seed(2)
    rows, d, ld = 150, 96, 104                      # ragged rows (3 chunks of 64), d not a multiple of 64, padded rows
    xs, dys = bf(g, rows, ld), bf(g, rows, ld)
    x, dy = xs[:, :d], dys[:, :d]
    mean = x.float().mean(1).contiguous()
    rstd = torch.rsqrt(x.float().var(1, unbiased=False) + 1e-5).contiguous()
    xh = (x.float() - mean[:, None]) * rstd[:, None]
    dg, db = torch.full((d,), 9.0), torch.full((d,), 9.0)
    kx.hx_layernorm_param_grad_rows(P(dys), LL(ld), P(xs), LL(ld), P(mean), P(rstd), P(dg), P(db), rows, d, 0)
    assert rel(dg, (dy.float() * xh).sum(0)) < 1e-5 and rel(db, dy.float().sum(0)) < 1e-5
    kx.hx_layernorm_param_grad_rows(P(dys), LL(ld), P(xs), LL(ld), P(mean), P(rstd), P(dg), P(db), rows, d, 1)
    assert rel(dg, 2 * (dy.float() * xh).sum(0)) < 1e-5 and rel(db, 2 * dy.float().sum(0)) < 1e-5


def test_col_moments_and_channel_affine_kernel_source(kx):
    g = torch.Generator().manual_seed(3)
    R, C = 300, 96                                   # 3 row chunks of 128, 2 column strips
    u, v, m = bf(g, R, C), bf(g, R, C), bf(g, R, C)
    o1, o2 = torch.empty(C), torch.empty(C)
    kx.hx_col_moments(P(u), LL(C), P(v), LL(C), P(m), LL(C), R, C, P(o1), P(o2))
    um = u.float() * (m.float() > 0)
    assert rel(o1, um.sum(0)) < 1e-5 and rel(o2, (um * v.float()).sum(0)) < 1e-5
    kx.hx_col_moments(P(u), LL(C), P(u), LL(C), None, LL(0), R, C, P(o1), P(o2))
    assert rel(o1, u.float().sum(0)) < 1e-5 and rel(o2, (u.float() ** 2).sum(0)) < 1e-5
    a1, a2, c0 = torch.randn(C, generator=g), torch.randn(C, generator=g), torch.randn(C, generator=g)
    y = torch.empty_like(u)
    kx.hx_channel_affine(P(u), P(a1), P(v), P(a2), P(c0), P(m), P(v), 1, P(y), LL(R), C)
    assert rel(y, F.relu(um * a1 + v.float() * a2 + c0 + v.float())) < 5e-3
    kx.hx_channel_affine(P(u), P(a1), None, None, None, None, None, 0, P(y), LL(R), C)
    assert rel(y, u.float() * a1) < 5e-3


@pytest.mark.parametrize("B,H,W,C,s", [(2, 6, 6, 8, 1), (2, 6, 6, 16, 2), (1, 7, 5, 8, 2), (1, 5, 9, 8, 1)])
def test_col2im3x3_kernel_source_is_the_adjoint_of_im2col(kx, B, H, W, C, s):
    g = torch.Generator().manual_seed(4)
    Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
    dcols = bf(g, B * Ho * Wo, 9 * C)
    x = torch.zeros(B, H, W, C, requires_grad=True)
    xu = F.unfold(x.permute(0, 3, 1, 2), 3, padding=1, stride=s)
    xu = xu.view(B, C, 9, Ho * Wo).permute(0, 3, 2, 1).reshape(B * Ho * Wo, 9 * C)
    xu.backward(dcols.float())
    dx = torch.empty(B, H, W, C, dtype=torch.bfloat16)
    kx.hx_col2im3x3(P(dcols), P(dx), B, H, W, C, s)
    assert rel(dx, x.grad) < 5e-3


def test_avgpool_nhwc_bwd_kernel_source(kx):
    g = torch.Generator().manual_seed(5)
    for (B, H, W, C, k) in ((2, 6, 8, 16, 2), (1, 7, 9, 8, 3)):          # 7x9 with k = 3: the last row / columns get no gradient
        dy = bf(g, B, H // k, W // k, C)
        x = torch.zeros(B, H, W, C, requires_grad=True)
        F.avg_pool2d(x.permute(0, 3, 1, 2), k).backward(dy.float().permute(0, 3, 1, 2))
        dx = torch.empty(B, H, W, C, dtype=torch.bfloat16)
        kx.hx_avgpool_nhwc_bwd(P(dy), P(dx), B, H, W, C, k)
        assert rel(dx, x.grad) < 5e-3


def test_gpu_verified_kernel_source_passes_the_gpu_ops_harness(kernel_ops, monkeypatch, capsys):
    """Calibration of the executor itself: the kernels of csrc/elt_kernels.cuh ARE verified on the GPU
    (tests/test_ops_gpu.py); executed on the CPU under the emulated thread model, their source passes the very same
    harness (LayerNorm fwd / bwd / parameter gradients, rotary, softmax fwd / bwd, build_labels bit-exact, cross-entropy,
    gathers, colsum, argmax tie rule, fused AdamW against torch.optim.AdamW, dropout) — so a pass of the NEW kernels under
    this executor means what it would mean for these."""
    from tools import model_check

    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    assert model_check.group_ops(torch.device("cpu"))
    assert "[FAIL]" not in capsys.readouterr().out


def _both(monkeypatch, fn):
    """Run fn() once on the kernel-source executor and once on the operator emulation; returns the two results."""
    import ctypes as C

    from magma_b200 import _lib, ops
    from oracle import build_emul

    out = []
    for path in (build_emul.build_kernel_exec(), build_emul.build()):
        L = C.CDLL(path)
        L.mb200_last_error.restype = C.c_char_p
        monkeypatch.setattr(_lib, "_lib", L)
        monkeypatch.setattr(ops, "_stream", lambda: None)
        out.append(fn())
    return out


def test_operator_emulation_agrees_with_the_kernel_source(monkeypatch):
    """Every dry run in this suite goes through oracle/cabi_emul.cpp, a RESTATEMENT of the operators. Here that
    restatement is compared, operator by operator on the same inputs, with the kernel source itself executed on the CPU:
    identical integers / bf16 values for the layout and gather kernels, fp32-reassociation-level agreement for reductions."""
    from magma_b200 import ops

    g = torch.Generator().manual_seed(7)

    def close(a, b, tol=2e-3):
        assert a.shape == b.shape and rel(a, b) < tol, rel(a, b)

    # LayerNorm forward / backward / parameter gradients
    x, dy, res = bf(g, 9, 64), bf(g, 9, 64), bf(g, 9, 64)
    gam, bet = (1 + 0.1 * torch.randn(64, generator=g)).to(torch.bfloat16), bf(g, 64, scale=0.1)
    (yk, mk, rk), (ye, me, re_) = _both(monkeypatch, lambda: ops.layernorm_fwd(x, gam, bet, 1e-5))
    close(yk, ye), close(mk, me, 1e-5), close(rk, re_, 1e-5)
    dk, de = _both(monkeypatch, lambda: ops.layernorm_bwd(dy, x, gam, mk, rk, res=res))
    close(dk, de)
    def pg():
        a, b = torch.zeros(64), torch.zeros(64)
        ops.layernorm_param_grad(dy, x, mk, rk, a, b)
        return torch.stack([a, b])
    close(*_both(monkeypatch, pg), tol=1e-5)
    # softmax forward (causal with offset) / backward
    s = torch.randn(3, 5, 16, generator=g)
    pk, pe = _both(monkeypatch, lambda: ops.softmax_fwd(s, 0.25, True, koff=3))
    close(pk, pe)
    dp = torch.randn(3, 5, 16, generator=g)
    close(*_both(monkeypatch, lambda: ops.softmax_bwd(dp, pk.contiguous(), 0.25)))
    # shifted cross-entropy: loss and gradient (V = 70 columns of a 72-wide row)
    logits = bf(g, 2, 3, 72)
    labels = torch.randint(0, 70, (2, 3), generator=g)
    labels[0, 2] = -100
    (lk, gk), (le, ge) = _both(monkeypatch, lambda: ops.cross_entropy(logits, labels, 70, write_grad=True))
    assert abs(float(lk) - float(le)) < 1e-5
    close(gk[..., :70], ge[..., :70])
    # integer / layout kernels: identical
    caps = torch.randint(0, 50, (3, 12), generator=g)
    caps[1, 4:] = 49
    a, b = _both(monkeypatch, lambda: ops.build_labels(caps, 3, 49))
    assert torch.equal(a, b)
    img = bf(g, 2, 3, 16, 16)
    a, b = _both(monkeypatch, lambda: ops.nchw_to_nhwc8(img))
    assert torch.equal(a, b)
    t = bf(g, 2, 6, 6, 8)
    for st in (1, 2):
        (ca, _, _), (cb, _, _) = _both(monkeypatch, lambda: ops.im2col3x3(t, st))
        assert torch.equal(ca, cb)
    a, b = _both(monkeypatch, lambda: ops.avgpool_nhwc(t, 2))
    close(a, b)
    rows = bf(g, 5, 96)
    a, b = _both(monkeypatch, lambda: ops.argmax(rows, 90))
    assert torch.equal(a, b)
    a, b = _both(monkeypatch, lambda: ops.colsum(rows))
    close(a, b, 1e-6)
    (ya, ma), (yb, mb) = _both(monkeypatch, lambda: ops.dropout_fwd(rows, 0.3, 11))
    assert torch.equal(ma, mb) and torch.equal(ya, yb)       # same counter-based hash, same mask
    # the training kernels: emulation vs source
    u, v, m = bf(g, 40, 16), bf(g, 40, 16), bf(g, 40, 16)
    (a1, a2), (b1, b2) = _both(monkeypatch, lambda: ops.col_moments(u, v, m))
    close(a1, b1, 1e-5), close(a2, b2, 1e-5)
    co = torch.randn(16, generator=g)
    close(*_both(monkeypatch, lambda: ops.channel_affine(u, co, x2=v, a2=co, c0=co, mask=m, res=v, relu=True)))
    dcols = bf(g, 2 * 3 * 3, 9 * 8)
    close(*_both(monkeypatch, lambda: ops.col2im3x3(dcols, 2, 6, 6, 8, 2)))
    close(*_both(monkeypatch, lambda: ops.quick_gelu_bwd(u, v)))


def test_batchnorm_bookkeeping_kernel_source(kx):
    """bn_finalize_fwd / bn_bwd_coeffs (one thread per channel) against nn.BatchNorm2d semantics and autograd."""
    g = torch.Generator().manual_seed(9)
    R, C = 200, 40
    z = torch.randn(R, C, generator=g) * 2 + 0.5
    gamma, beta = 1 + 0.1 * torch.randn(C, generator=g), 0.1 * torch.randn(C, generator=g)
    rm, rv = torch.randn(C, generator=g) * 0.1, 1 + 0.2 * torch.rand(C, generator=g)
    s1, s2 = z.sum(0).contiguous(), (z * z).sum(0).contiguous()
    bn = torch.nn.BatchNorm2d(C, momentum=0.1)
    with torch.no_grad():
        bn.weight.copy_(gamma), bn.bias.copy_(beta), bn.running_mean.copy_(rm), bn.running_var.copy_(rv)
    zz = z.clone().requires_grad_(True)
    y = bn(zz.t().reshape(1, C, R, 1))                       # training mode: batch statistics over the R positions
    rm_k, rv_k = rm.clone(), rv.clone()
    out = [torch.empty(C) for _ in range(4)]
    F32 = ctypes.c_float
    rc = kx.mb200_bn_finalize_fwd(P(s1), P(s2), P(gamma), P(beta), LL(R), F32(1e-5), F32(0.1), P(rm_k), P(rv_k),
                                  P(out[0]), P(out[1]), P(out[2]), P(out[3]), C, None)
    assert rc == 0
    mean, rstd, scale, shift = out
    assert torch.allclose(z * scale + shift, y.reshape(C, R).t(), rtol=1e-4, atol=1e-4)
    assert torch.allclose(rm_k, bn.running_mean, rtol=1e-5, atol=1e-6) and torch.allclose(rv_k, bn.running_var, rtol=1e-4, atol=1e-5)
    dy = torch.randn(R, C, generator=g)
    y.backward(dy.t().reshape(1, C, R, 1))
    t = (dy * z).sum(0).contiguous()
    d1 = dy.sum(0).contiguous()
    dg, db = torch.full((C,), 2.0), torch.full((C,), 2.0)
    co = [torch.empty(C) for _ in range(3)]
    rc = kx.mb200_bn_bwd_coeffs(P(d1), P(t), P(mean), P(rstd), P(gamma), LL(R), P(dg), P(db), 1, P(co[0]), P(co[1]), P(co[2]),
                                C, None)
    assert rc == 0
    assert torch.allclose(dg, 2.0 + bn.weight.grad, rtol=1e-3, atol=1e-3) and torch.allclose(db, 2.0 + bn.bias.grad, rtol=1e-4, atol=1e-4)
    dz = dy * co[0] + z * co[1] + co[2]
    assert torch.allclose(dz, zz.grad, rtol=1e-3, atol=1e-4)


def test_sumsq_kernel_source_parts_cover_every_element(kx):
    """The grid-independent squared norm (elt_kernels.cuh::sumsq_kernel): 2048 logical parts over float4 chunks, a scalar
    tail, and the scalar path for a view that is not 16-byte aligned. (The CPU executor runs it on a 16-block grid, the
    grid of one SM; the GPU test checks that any grid gives the same bits.)"""
    g = torch.Generator().manual_seed(3)
    for n in (150 * 256 * 4 + 4 * 77 + 3, 1000, 5):   # (inputs long enough for several chunks per part: GPU test)
        x = torch.randn(n + 1, generator=g)
        for view in ((x[:n], x[1:]) if n <= 1000 else (x[:n],)):   # aligned / 4-byte-offset view
            out = torch.full((1,), 2.0)
            assert kx.mb200_sumsq(P(view), LL(n), P(out), None) == 0
            want = 2.0 + float((view.double() ** 2).sum())
            assert abs(float(out) - want) < 2e-5 * want, (n, float(out), want)
