"""Thin Python wrappers over the C ABI (include/magma_b200.h). Tensors are torch CUDA tensors used purely as
device-memory handles; every op is enqueued on torch's current CUDA stream."""
import ctypes

import torch

from . import _lib
from ._lib import GemmArgs, check, lib

ACT_NONE, ACT_GELU_NEW, ACT_QUICK_GELU, ACT_RELU, ACT_RELU_POST = 0, 1, 2, 3, 4
DACT_NONE, DACT_GELU_NEW, DACT_RELU = 0, 1, 3


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _ptr(t):
    return t.data_ptr() if t is not None else None


def _mat_meta(t, name):
    """(rows, cols, ld, nb0, nb1, bs0, bs1) of a [..., rows, cols] tensor with unit inner stride."""
    if t.dim() < 2 or t.dim() > 4:
        raise ValueError(f"{name}: expected 2-4 dims, got {t.dim()}")
    if t.stride(-1) != 1 and t.shape[-1] != 1:
        raise ValueError(f"{name}: innermost stride must be 1, got {t.stride()}")
    rows, cols = t.shape[-2], t.shape[-1]
    ld = t.stride(-2) if rows > 1 else max(cols, t.stride(-2))
    nb0 = t.shape[-3] if t.dim() >= 3 else 1
    bs0 = t.stride(-3) if t.dim() >= 3 else 0
    nb1 = t.shape[-4] if t.dim() >= 4 else 1
    bs1 = t.stride(-4) if t.dim() >= 4 else 0
    return rows, cols, ld, nb0, nb1, bs0, bs1


def gemm(
    A,
    B,
    out=None,
    *,
    a_mn=False,
    b_mn=False,
    out_dtype=torch.bfloat16,
    alpha=1.0,
    bias=None,
    act=ACT_NONE,
    aux_out=None,
    aux_in=None,
    dact=DACT_NONE,
    res1=None,
    res2=None,
    accumulate=False,
    force_bn=0,
    generic_epilogue=False,
    rope_tab=None,
    rope_mode=0,
    rope_S=0,
    rope_hd=0,
    rope_rot=0,
    rope_ncols=0,
    splitk_ws=None,
    b_static=False,
):
    """C[..., M, N] = epilogue(alpha * A @ B^T) on the wgmma GEMM core.

    A is [..., M, K] (a_mn=False) or [..., K, M] (a_mn=True); B is [..., N, K] (b_mn=False) or
    [..., K, N] (b_mn=True). Up to two leading batch dims with arbitrary (8-element aligned) strides.
    """
    if A.dtype != torch.bfloat16 or B.dtype != torch.bfloat16:
        raise TypeError("gemm operands must be bf16")
    ra, ca, lda, anb0, anb1, abs0, abs1 = _mat_meta(A, "A")
    rb, cb, ldb, bnb0, bnb1, bbs0, bbs1 = _mat_meta(B, "B")
    M, K = (ca, ra) if a_mn else (ra, ca)
    N, Kb = (cb, rb) if b_mn else (rb, cb)
    if K != Kb:
        raise ValueError(f"gemm K mismatch: {K} vs {Kb}")
    nb0, nb1 = max(anb0, bnb0), max(anb1, bnb1)
    # broadcast of a non-batched operand over the batch: stride 0 is not TMA-legal, so only allow equal batch
    if (anb0, anb1) != (nb0, nb1) or (bnb0, bnb1) != (nb0, nb1):
        raise ValueError("gemm: A and B must have identical batch dims")
    if out is None:
        shape = ([nb1] if A.dim() >= 4 else []) + ([nb0] if A.dim() >= 3 else []) + [M, N]
        out = torch.empty(shape, dtype=out_dtype, device=A.device)
    rc_, cc, ldc, cnb0, cnb1, cbs0, cbs1 = _mat_meta(out, "out")
    if (rc_, cc) != (M, N) or (cnb0, cnb1) != (nb0, nb1):
        raise ValueError(f"gemm: out shape {tuple(out.shape)} does not match M={M} N={N} batch=({nb1},{nb0})")
    g = GemmArgs()
    g.M, g.N, g.K, g.nb0, g.nb1 = M, N, K, nb0, nb1
    g.c_dtype = 1 if out.dtype == torch.float32 else 0
    if out.dtype not in (torch.float32, torch.bfloat16):
        raise TypeError("gemm out must be bf16 or f32")
    g.A.ptr, g.A.ld, g.A.bs0, g.A.bs1, g.A.mn_major = A.data_ptr(), lda, abs0, abs1, int(a_mn)
    g.B.ptr, g.B.ld, g.B.bs0, g.B.bs1, g.B.mn_major = B.data_ptr(), ldb, bbs0, bbs1, int(b_mn)
    g.B.static_data = int(bool(b_static))  # frozen weights: first tiles may load ahead of the PDL dependency
    g.C, g.ldc, g.c_bs0, g.c_bs1 = out.data_ptr(), ldc, cbs0, cbs1
    g.alpha, g.act, g.dact, g.accumulate = float(alpha), int(act), int(dact), int(bool(accumulate))
    for name, t in (("bias", bias), ("aux_out", aux_out), ("aux_in", aux_in), ("res1", res1), ("res2", res2)):
        if t is not None:
            if t.dtype != torch.bfloat16:
                raise TypeError(f"gemm {name} must be bf16")
            setattr(g, name, t.data_ptr())
    # The kernel gets raw pointers: bias is read as [N] with unit stride, aux and residual tensors at C's batch offsets
    # (aux also at C's row stride), so any other layout would be read or written out of place.
    if bias is not None and (tuple(bias.shape) != (N,) or (N > 1 and bias.stride(0) != 1)):
        raise ValueError(f"gemm bias must be a contiguous [N={N}] vector, got shape {tuple(bias.shape)}")
    for name, t in (("aux_out", aux_out), ("aux_in", aux_in), ("res1", res1), ("res2", res2)):
        if t is not None and tuple(t.shape) != tuple(out.shape):
            raise ValueError(f"gemm {name} shape {tuple(t.shape)} must equal out's {tuple(out.shape)}")
    for name, t in (("aux_out", aux_out), ("aux_in", aux_in)):
        if t is not None and _mat_meta(t, name)[2:] != (ldc, cnb0, cnb1, cbs0, cbs1):
            raise ValueError(f"gemm {name} must share out's strides")
    ld_res = 0
    for name, t in (("res1", res1), ("res2", res2)):
        if t is not None:
            m = _mat_meta(t, name)
            if (cnb0 > 1 and m[5] != cbs0) or (cnb1 > 1 and m[6] != cbs1):
                raise ValueError(f"gemm {name} must share out's batch strides (its row stride may differ)")
            if ld_res and m[2] != ld_res:
                raise ValueError("res1/res2 must share a row stride")
            ld_res = m[2]
    g.ld_res = ld_res
    g.force_bn = force_bn
    g.generic_epilogue = int(bool(generic_epilogue))
    if rope_tab is not None and rope_mode:
        g.rope_tab, g.rope_mode = rope_tab.data_ptr(), int(rope_mode)
        g.rope_S, g.rope_hd, g.rope_rot, g.rope_ncols = int(rope_S), int(rope_hd), int(rope_rot), int(rope_ncols)
    if splitk_ws is not None:
        g.splitk_ws, g.splitk_ws_bytes = splitk_ws.data_ptr(), splitk_ws.numel() * splitk_ws.element_size()
    check(lib().mb200_gemm(ctypes.byref(g), _stream()))
    return out


def gemm_last_plan():
    """(tile width, K splits) of this thread's last gemm call"""
    v = [ctypes.c_int32() for _ in range(2)]
    lib().mb200_gemm_last_plan(*[ctypes.byref(x) for x in v])
    return tuple(x.value for x in v)


# --------------------------------------------------------------------------------------------
# HBM-bound operators
# --------------------------------------------------------------------------------------------
def _rows(t):
    """(rows, d, ld) of a [..., d] tensor whose leading dims collapse to a constant row stride."""
    d = t.shape[-1]
    if t.dim() == 1:
        return 1, d, d
    t2 = t.reshape(-1, d) if t.is_contiguous() else None
    if t2 is not None:
        return t2.shape[0], d, d
    if t.dim() == 2:
        return t.shape[0], d, t.stride(0)
    raise ValueError("non-contiguous >2-D tensor: pass a 2-D view with an explicit row stride")


def layernorm_fwd(x, gamma, beta, eps=1e-5, save_stats=True, out=None):
    rows, d, ldx = _rows(x)
    y = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device) if out is None else out
    mean = torch.empty(rows, dtype=torch.float32, device=x.device) if save_stats else None
    rstd = torch.empty(rows, dtype=torch.float32, device=x.device) if save_stats else None
    check(lib().mb200_layernorm_fwd(_ptr(x), ldx, _ptr(gamma), _ptr(beta), _ptr(y), _rows(y)[2], _ptr(mean), _ptr(rstd),
                                    rows, d, eps, _stream()))
    return y, mean, rstd


def layernorm_bwd(dy, x, gamma, mean, rstd, res=None, out=None):
    """dx of LayerNorm (+ res); into `out` (any row stride) when given."""
    rows, d, ldx = _rows(x)
    dx = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device) if out is None else out
    check(lib().mb200_layernorm_bwd(_ptr(dy), _rows(dy)[2], _ptr(x), ldx, _ptr(gamma), _ptr(mean), _ptr(rstd),
                                    _ptr(res), _rows(res)[2] if res is not None else 0, _ptr(dx), _rows(dx)[2], rows, d,
                                    _stream()))
    return dx


def layernorm_param_grad(dy, x, mean, rstd, dgamma, dbeta, accumulate=False):
    rows, d, ldx = _rows(x)
    check(lib().mb200_layernorm_param_grad(_ptr(dy), _rows(dy)[2], _ptr(x), ldx, _ptr(mean), _ptr(rstd), _ptr(dgamma),
                                           _ptr(dbeta), rows, d, accumulate, _stream()))


def layernorm_param_grad_rows(dy, x, mean, rstd, dgamma, dbeta, accumulate=False):
    """Same result as layernorm_param_grad with a (column strip) x (row chunk) grid — for thousands of rows."""
    rows, d, ldx = _rows(x)
    check(lib().mb200_layernorm_param_grad_rows(_ptr(dy), _rows(dy)[2], _ptr(x), ldx, _ptr(mean), _ptr(rstd),
                                                _ptr(dgamma), _ptr(dbeta), rows, d, accumulate, _stream()))


def quick_gelu_bwd(dy, pre, out=None):
    """dx = dy * d/dx[x sigmoid(1.702 x)] at x = pre (CLIP QuickGELU backward); `out` may be dy itself."""
    out = torch.empty_like(dy) if out is None else out
    check(lib().mb200_quick_gelu_bwd(_ptr(dy), _ptr(pre), _ptr(out), dy.numel(), _stream()))
    return out


def rope_(qkv, S, H, hd, rot, pos0=0, inverse=False):
    """In place on a [rows, 3*H*hd] fused qkv buffer."""
    rows = qkv.shape[0]
    check(lib().mb200_rope(_ptr(qkv), qkv.stride(0), rows, S, H, hd, rot, pos0, inverse, _stream()))
    return qkv


def rope_table(S, rot, pos0=0, device=None):
    tab = torch.empty(S, rot // 2, 2, dtype=torch.float32, device=device or torch.device("cuda"))
    check(lib().mb200_rope_table(_ptr(tab), S, rot, pos0, _stream()))
    return tab


def softmax_fwd(s, scale, causal, koff=0, out=None):
    """s: fp32 [nz, Sq, Sk(ld)] -> bf16 probabilities with the same padded layout, or into `out` (bf16 [nz, Sq, Sk] with
    unit column stride, any row and batch strides). Columns [0, Sk) of each row are written."""
    nz, Sq, Sk = s.shape
    lds = s.stride(1)
    p = torch.zeros(nz, Sq, lds, dtype=torch.bfloat16, device=s.device)[..., :Sk] if out is None else out
    _batched_out(p, "out", (nz, Sq, Sk))
    check(lib().mb200_softmax_fwd(_ptr(s), lds, s.stride(0), _ptr(p), p.stride(1), p.stride(0), nz, Sq, Sk, scale,
                                  causal, koff, _stream()))
    return p


def _batched_out(t, name, shape):
    if t.dtype != torch.bfloat16 or tuple(t.shape) != shape or (shape[-1] > 1 and t.stride(-1) != 1):
        raise ValueError(f"{name} must be a bf16 {list(shape)} view with unit column stride, got {t.dtype} "
                         f"{tuple(t.shape)} strides {t.stride()}")


def softmax_bwd(dp, p, scale, out=None):
    """dS = P * (dP - rowsum(dP * P)) * scale: fp32 dp and bf16 p [nz, Sq, Sk] -> bf16, in the padded layout of p or
    into `out` (bf16 [nz, Sq, Sk] with unit column stride)."""
    nz, Sq, Sk = dp.shape
    ds = torch.zeros(nz, Sq, p.stride(1), dtype=torch.bfloat16, device=dp.device)[..., :Sk] if out is None else out
    _batched_out(ds, "out", (nz, Sq, Sk))
    check(lib().mb200_softmax_bwd(_ptr(dp), dp.stride(1), dp.stride(0), _ptr(p), p.stride(1), p.stride(0), _ptr(ds),
                                  ds.stride(1), ds.stride(0), nz, Sq, Sk, scale, _stream()))
    return ds


def build_labels(captions, prefix_len, eos_token):
    """magma/utils.py:334-364 on device; captions int64 [B,S] -> labels int64 [B,S]."""
    B, S = captions.shape
    if captions.dtype != torch.int64:
        raise TypeError("captions must be int64")
    labels = torch.empty(B, S, dtype=torch.int64, device=captions.device)
    check(lib().mb200_build_labels(_ptr(captions), captions.stride(0), _ptr(labels), B, S, int(prefix_len),
                                   int(eos_token), _stream()))
    return labels


def embed_assemble(captions, wte, prefix, S=None, out=None):
    B, Sc = captions.shape
    S = Sc if S is None else S
    L = 0 if prefix is None else prefix.shape[1]
    V, d = wte.shape
    x = torch.empty(B, S, d, dtype=torch.bfloat16, device=wte.device) if out is None else out
    check(lib().mb200_embed_assemble(_ptr(captions), captions.stride(0), _ptr(wte), _ptr(prefix), L,
                                     _ptr(x), B, S, d, V, _stream()))
    return x


def embed_gather(ids, wte, out=None):
    V, d = wte.shape
    flat = ids.reshape(-1).contiguous()
    out = torch.empty(*ids.shape, d, dtype=torch.bfloat16, device=wte.device) if out is None else out
    check(lib().mb200_embed_gather(_ptr(flat), _ptr(wte), _ptr(out), flat.numel(), d, V, _stream()))
    return out


def cross_entropy(logits, labels, V, write_grad=False, grad_scale=1.0, dlogits=None, row_loss=None):
    """logits bf16 [B,S,ldv]; returns (loss fp32 [1], dlogits or None). `dlogits` (same strides as logits; may be
    logits itself) receives the gradient instead of a new buffer; `row_loss` (fp32 [B*S]) the per-row losses."""
    B, S = labels.shape
    ldv = logits.stride(-2)
    if row_loss is None:
        row_loss = torch.empty(B * S, dtype=torch.float32, device=logits.device)
    n_valid = torch.zeros(4, dtype=torch.int32, device=logits.device)
    loss = torch.empty(1, dtype=torch.float32, device=logits.device)
    if dlogits is not None and dlogits.stride() != logits.stride():
        raise ValueError("cross_entropy: dlogits must share the strides of logits")
    dl = dlogits if dlogits is not None else (torch.zeros_like(logits) if write_grad else None)
    check(lib().mb200_cross_entropy(_ptr(logits), ldv, _ptr(labels), B, S, V, _ptr(row_loss),
                                    _ptr(n_valid), _ptr(loss), _ptr(dl), grad_scale, _stream()))
    return loss, dl


def colsum(x, out=None, accumulate=False):
    rows, cols = x.shape
    if out is None:
        out = torch.empty(cols, dtype=torch.float32, device=x.device)
    check(lib().mb200_colsum(_ptr(x), x.stride(0), rows, cols, _ptr(out), accumulate, _stream()))
    return out


def dropout_fwd(x, p, seed, out=None):
    y = torch.empty_like(x) if out is None else out
    mask = torch.empty(x.numel(), dtype=torch.uint8, device=x.device)
    check(lib().mb200_dropout_fwd(_ptr(x), _ptr(y), _ptr(mask), x.numel(), p, seed, _stream()))
    return y, mask


def dropout_apply(x, mask, p, out=None):
    y = torch.empty_like(x) if out is None else out
    check(lib().mb200_dropout_apply(_ptr(x), _ptr(mask), _ptr(y), x.numel(), p, _stream()))
    return y


def argmax(x, V=None, out=None):
    rows = x.shape[0]
    V = x.shape[1] if V is None else V
    if out is None:
        out = torch.empty(rows, dtype=torch.int64, device=x.device)
    check(lib().mb200_argmax(_ptr(x), x.stride(0), rows, V, _ptr(out), _stream()))
    return out


def decode_embed(tokens, pos_dev, wte, out):
    """out[b] = wte[tokens[b, pos]] with the column `pos` read from DEVICE memory (int32 [1]) — the input embedding of
    a graph-replayed decode step (mb200_decode_embed)."""
    V, d = wte.shape
    check(lib().mb200_decode_embed(_ptr(tokens), tokens.stride(0), _ptr(pos_dev), _ptr(wte), _ptr(out),
                                   tokens.shape[0], d, V, _stream()))
    return out


def decode_advance(next_tokens, tokens, pos_dev, eos, flags, s0):
    """tokens[:, pos + 1] = next_tokens; flags[pos + 1 - s0] = all rows emitted `eos`; pos += 1 (all on the device)."""
    check(lib().mb200_decode_advance(_ptr(next_tokens), _ptr(tokens), tokens.stride(0), _ptr(pos_dev),
                                     -1 if eos is None else int(eos), _ptr(flags), int(s0),
                                     flags.numel() if flags is not None else 0, tokens.shape[0], _stream()))


def nchw_to_nhwc8(x, out=None):
    """[B, C<=8, H, W] bf16 -> [B, H, W, 8] bf16 with zero-padded channels (conv-trunk stem input)."""
    assert x.dtype == torch.bfloat16 and x.is_contiguous() and x.ndim == 4
    B, C, H, W = x.shape
    y = torch.empty(B, H, W, 8, dtype=torch.bfloat16, device=x.device) if out is None else out
    check(lib().mb200_nchw_to_nhwc8(_ptr(x), _ptr(y), B, C, H, W, _stream()))
    return y


def im2col3x3(x, stride=1, out=None):
    """NHWC [B,H,W,C] bf16 -> [B*Ho*Wo, 9*C] bf16 (3x3, padding 1), columns ordered (kh, kw, c)."""
    assert x.dtype == torch.bfloat16 and x.is_contiguous() and x.ndim == 4
    B, H, W, C = x.shape
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    y = torch.empty(B * Ho * Wo, 9 * C, dtype=torch.bfloat16, device=x.device) if out is None else out
    check(lib().mb200_im2col3x3(_ptr(x), _ptr(y), B, H, W, C, stride, _stream()))
    return y, Ho, Wo


def avgpool_nhwc(x, k, out=None):
    """nn.AvgPool2d(k) on NHWC bf16: [B,H,W,C] -> [B,H//k,W//k,C]."""
    assert x.dtype == torch.bfloat16 and x.is_contiguous() and x.ndim == 4
    B, H, W, C = x.shape
    y = torch.empty(B, H // k, W // k, C, dtype=torch.bfloat16, device=x.device) if out is None else out
    check(lib().mb200_avgpool_nhwc(_ptr(x), _ptr(y), B, H, W, C, k, _stream()))
    return y


def col_moments(u, v, mask=None):
    """Per-channel (sum u', sum u' * v) over the rows of [rows, C] bf16 tensors, u' = u * 1[mask > 0]; fp32 [C] each."""
    rows, C = u.shape
    assert u.dtype == v.dtype == torch.bfloat16 and v.shape == u.shape and u.stride(1) == 1 and v.stride(1) == 1
    o1 = torch.empty(C, dtype=torch.float32, device=u.device)
    o2 = torch.empty(C, dtype=torch.float32, device=u.device)
    check(lib().mb200_col_moments(_ptr(u), u.stride(0), _ptr(v), v.stride(0), _ptr(mask),
                                  mask.stride(0) if mask is not None else 0, rows, C, _ptr(o1), _ptr(o2),
                                  _stream()))
    return o1, o2


def channel_affine(x1, a1, x2=None, a2=None, c0=None, mask=None, res=None, relu=False, out=None):
    """y = relu?(a1[c] * x1 * 1[mask > 0] + a2[c] * x2 + c0[c] + res) over contiguous [rows, C] bf16 tensors with fp32
    per-channel coefficients (BatchNorm forward / backward, ReLU backward)."""
    rows, C = x1.shape
    for t in (x1, x2, mask, res):
        assert t is None or (t.dtype == torch.bfloat16 and t.is_contiguous() and t.shape == x1.shape)
    for t in (a1, a2, c0):
        assert t is None or (t.dtype == torch.float32 and t.is_contiguous() and t.numel() == C)
    y = torch.empty_like(x1) if out is None else out
    check(lib().mb200_channel_affine(_ptr(x1), _ptr(a1), _ptr(x2), _ptr(a2), _ptr(c0), _ptr(mask), _ptr(res), relu,
                                     _ptr(y), rows, C, _stream()))
    return y


def bn_finalize_fwd(s1, s2, gamma, beta, rows, eps, momentum, running_mean=None, running_var=None):
    """(sum z, sum z^2) -> (mean, rstd, scale, shift) fp32 [C]; updates the running statistics in place when given."""
    C = s1.numel()
    for t in (s1, s2, gamma, beta, running_mean, running_var):
        assert t is None or (t.dtype == torch.float32 and t.is_contiguous() and t.numel() == C)
    out = torch.empty(4, C, dtype=torch.float32, device=s1.device)
    check(lib().mb200_bn_finalize_fwd(_ptr(s1), _ptr(s2), _ptr(gamma), _ptr(beta), rows, eps,
                                      momentum, _ptr(running_mean), _ptr(running_var), _ptr(out[0]),
                                      _ptr(out[1]), _ptr(out[2]), _ptr(out[3]), C, _stream()))
    return out[0], out[1], out[2], out[3]


def bn_bwd_coeffs(s1, t, mean, rstd, gamma, rows, dgamma, dbeta, accumulate=False):
    """(sum dy', sum dy' * z) -> dgamma / dbeta (written or accumulated in place) and the coefficients (A, Bc, Cc) of
    dz = A * dy' + Bc * z + Cc."""
    C = s1.numel()
    for x in (s1, t, mean, rstd, gamma, dgamma, dbeta):
        assert x.dtype == torch.float32 and x.is_contiguous() and x.numel() == C
    out = torch.empty(3, C, dtype=torch.float32, device=s1.device)
    check(lib().mb200_bn_bwd_coeffs(_ptr(s1), _ptr(t), _ptr(mean), _ptr(rstd), _ptr(gamma), rows,
                                    _ptr(dgamma), _ptr(dbeta), accumulate, _ptr(out[0]), _ptr(out[1]), _ptr(out[2]), C,
                                    _stream()))
    return out[0], out[1], out[2]


def col2im3x3(dcols, B, H, W, C, stride=1, out=None):
    """Adjoint of im2col3x3: [B*Ho*Wo, 9*C] bf16 -> [B, H, W, C] bf16."""
    assert dcols.dtype == torch.bfloat16 and dcols.is_contiguous() and dcols.shape[1] == 9 * C
    dx = torch.empty(B, H, W, C, dtype=torch.bfloat16, device=dcols.device) if out is None else out
    check(lib().mb200_col2im3x3(_ptr(dcols), _ptr(dx), B, H, W, C, stride, _stream()))
    return dx


def avgpool_nhwc_bwd(dy, H, W, k, out=None):
    """Adjoint of avgpool_nhwc: [B, H//k, W//k, C] -> [B, H, W, C]."""
    assert dy.dtype == torch.bfloat16 and dy.is_contiguous() and dy.ndim == 4
    B, _, _, C = dy.shape
    dx = torch.empty(B, H, W, C, dtype=torch.bfloat16, device=dy.device) if out is None else out
    check(lib().mb200_avgpool_nhwc_bwd(_ptr(dy), _ptr(dx), B, H, W, C, k, _stream()))
    return dx


def sample(logits, temperature, top_k=0, top_p=0.0, seed=0, offset=0, return_mask=False):
    """One token per row of `logits` [rows, V] (bf16 or fp32, unit column stride) sampled like magma/sampling.py:97-105
    (top-k filter, the reference's nucleus filter, softmax(logits / T), multinomial)."""
    assert logits.ndim == 2 and logits.stride(1) == 1 and logits.dtype in (torch.bfloat16, torch.float32)
    rows, V = logits.shape
    out = torch.empty(rows, dtype=torch.int64, device=logits.device)
    mask = torch.empty(rows, V, dtype=torch.uint8, device=logits.device) if return_mask else None
    check(lib().mb200_sample(_ptr(logits), 0 if logits.dtype == torch.bfloat16 else 1, logits.stride(0), rows, V,
                             temperature, int(top_k), top_p, seed & (2**64 - 1), offset, _ptr(out), _ptr(mask),
                             _stream()))
    return (out, mask) if return_mask else out


def sample_dev(logits, pos_dev, s0, temperature, top_k, top_p, seed, out):
    """`sample` with the Philox offset read on the device, pos_dev[0] - s0 + 1 (pos_dev: int32 [1], the decode loop's
    cache position; s0: the prompt length), into the preallocated int64 `out` [rows] — capturable in a CUDA graph of
    the decode step (mb200_sample_dev)."""
    assert logits.ndim == 2 and logits.stride(1) == 1 and logits.dtype in (torch.bfloat16, torch.float32)
    assert out.dtype == torch.int64 and out.numel() == logits.shape[0] and pos_dev.dtype == torch.int32
    rows, V = logits.shape
    check(lib().mb200_sample_dev(_ptr(logits), 0 if logits.dtype == torch.bfloat16 else 1, logits.stride(0), rows, V,
                                 temperature, int(top_k), top_p, seed & (2**64 - 1), _ptr(pos_dev), int(s0), _ptr(out),
                                 None, _stream()))
    return out


def add(a, b, c=None, out=None):
    y = torch.empty_like(a) if out is None else out
    check(lib().mb200_add(_ptr(a), _ptr(b), _ptr(c), _ptr(y), a.numel(), _stream()))
    return y


def logits_grad_combine(dce, g, out, alpha):
    """mb200_logits_grad_combine: out[:, :V] = alpha * dce[:, :V] + g for bf16 rows; dce and out share the row stride,
    g [M, V] may have any."""
    M, V = g.shape
    assert dce.stride(0) == out.stride(0) and g.stride(1) == 1
    check(lib().mb200_logits_grad_combine(_ptr(dce), out.stride(0), _ptr(g), g.stride(0), _ptr(out), M, V, alpha,
                                          _stream()))
    return out


def peer_reduce_bcast(buffer_ptrs, offset, n, max_blocks=0):
    """mb200_peer_reduce_bcast: `buffer_ptrs` = device addresses of every rank's exchange buffer as mapped here."""
    arr = (ctypes.c_void_p * len(buffer_ptrs))(*[int(p) for p in buffer_ptrs])
    check(lib().mb200_peer_reduce_bcast(arr, len(buffer_ptrs), offset, n, int(max_blocks),
                                        _stream()))


def cast_f32_to_bf16(src, dst):
    check(lib().mb200_cast_f32_to_bf16(_ptr(src), _ptr(dst), src.numel(), _stream()))


def cast_bf16_to_f32(src, dst):
    check(lib().mb200_cast_bf16_to_f32(_ptr(src), _ptr(dst), src.numel(), _stream()))


def patchify(img, P, out):
    """images bf16 [B, 3, R, R] -> out [B * (R/P)^2, >= 3 P P] (row stride out.stride(0)), columns ordered (c, py, px)."""
    B, _, R, _ = img.shape
    check(lib().mb200_patchify(_ptr(img), _ptr(out), out.stride(0), B, R, P, _stream()))
    return out


def vit_assemble(x, pe, cls, pos):
    """x [B, T, w] = [cls; pe] + pos with pe [B, T-1, w], cls [w], pos [T, w] (all contiguous bf16)."""
    B, T, w = x.shape
    check(lib().mb200_vit_assemble(_ptr(x), _ptr(pe), _ptr(cls), _ptr(pos), B, T, w, _stream()))
    return x


def scale_add(u, s=None, r1=None, r2=None, out=None):
    """out = s[0] * u + r1 + r2 (s: device fp32 scalar or None for 1; r1 / r2 optional), bf16."""
    out = torch.empty_like(u) if out is None else out
    check(lib().mb200_scale_add(_ptr(u), _ptr(s), _ptr(r1), _ptr(r2), _ptr(out), u.numel(), _stream()))
    return out


def dot(a, b, out, accumulate=False):
    """out[0] (+)= sum a * b over bf16 vectors, fp32."""
    check(lib().mb200_dot(_ptr(a), _ptr(b), a.numel(), _ptr(out), accumulate, _stream()))
    return out


def rope_table_dev(S, rot, pos0_dev, out=None):
    """rope_table with the first position read from device memory (int32 [1])."""
    tab = torch.empty(S, rot // 2, 2, dtype=torch.float32, device=pos0_dev.device) if out is None else out
    check(lib().mb200_rope_table_dev(_ptr(tab), S, rot, _ptr(pos0_dev), _stream()))
    return tab


def set_optimizer_grid(n_blocks):
    """Cap the grid of the optimizer kernels (sumsq, adamw) at n_blocks (0: no cap). Returns the cap in force."""
    return lib().mb200_set_optimizer_grid(int(n_blocks))


def sumsq(x, out):
    check(lib().mb200_sumsq(_ptr(x), x.numel(), _ptr(out), _stream()))


def adamw_step(master, grad, m1, m2, shadow, lr, beta1, beta2, eps, wd, grad_scale, gnorm_sq, max_norm, step,
               zero_grad=True):
    check(lib().mb200_adamw_step(_ptr(master), _ptr(grad), _ptr(m1), _ptr(m2), _ptr(shadow), master.numel(), lr, beta1,
                                 beta2, eps, wd, grad_scale, _ptr(gnorm_sq), max_norm, int(step), zero_grad, _stream()))


def _rows_out(t, name, rows, cols, dtype=torch.bfloat16):
    """Row stride of a caller-supplied [rows, cols] output with unit column stride."""
    if t.dtype != dtype or tuple(t.shape) != (rows, cols) or (cols > 1 and t.stride(1) != 1):
        raise ValueError(f"{name} must be a {dtype} [{rows}, {cols}] view with unit column stride, got "
                         f"{t.dtype} {tuple(t.shape)} strides {t.stride()}")
    return t.stride(0) if rows > 1 else max(cols, t.stride(0))


def _p_out(P, B, H, S, min_cols):
    """Row stride ldP of a caller-supplied P [B, H, S, ldP]: the kernels address row (b, h, i) at ((b H + h) S + i) ldP,
    so the view must be contiguous apart from its last dim, which may be cut short of the row stride."""
    ldP = P.stride(2)
    want = (H * S * ldP, S * ldP, ldP)
    if (P.dtype != torch.bfloat16 or P.dim() != 4 or tuple(P.shape[:3]) != (B, H, S) or P.stride(3) != 1
            or any(n > 1 and s != w for n, s, w in zip(P.shape[:3], P.stride()[:3], want)) or ldP % 8
            or ldP < min_cols):
        raise ValueError(f"P must be a bf16 [B={B}, H={H}, S={S}, >= {min_cols}] view of a [B, H, S, ldP] buffer "
                         f"(ldP % 8 == 0), got shape {tuple(P.shape)} strides {P.stride()}")
    return ldP


def attn_fwd_tile(qkv, B, S, H, hd, O=None, P=None):
    """Fused single-tile causal attention (S <= 128). qkv: bf16 [B*S, 3*H*hd] already rotated.
    Returns (O [B*S, H*hd], P [B, H, S, ldP]). O and P may be given with padded row strides; the kernel writes columns
    [0, min(ldP, 128)) of every row of P."""
    if P is None:
        P = torch.zeros(B, H, S, (S + 7) // 8 * 8, dtype=torch.bfloat16, device=qkv.device)
    ldP = _p_out(P, B, H, S, S)
    if O is None:
        O = torch.empty(B * S, H * hd, dtype=torch.bfloat16, device=qkv.device)
    ldo = _rows_out(O, "O", B * S, H * hd)
    check(lib().mb200_attn_fwd_tile(_ptr(qkv), qkv.stride(0), _ptr(P), ldP, _ptr(O), ldo, B, S, H, hd, _stream()))
    return O, P


def attn_fwd_flash(qkv, B, S, H, hd, causal=True, want_p=False, want_stats=False, kcache=None, vcache=None, pos0=0,
                   O=None, P=None, stats=None):
    """Multi-tile attention forward for any sequence length (mb200_attn_fwd_flash). qkv: bf16 [B*S, 3*H*hd] (already
    rotated) supplies the queries and — without a cache — the keys / values. With kcache / vcache ([B, H, Smax, hd],
    positions [0, pos0 + S) valid) the keys / values come from the cache (prefill continuation: queries are the last S
    of the pos0 + S positions). Returns O [B*S, H*hd] (+ P [B, H, S, ldP]) (+ stats [B, H, S, 2]). O and P may be
    given with padded row strides (P then need not be asked for with want_p; every column [0, ldP) is written), stats
    as a contiguous fp32 [B, H, S, 2]."""
    d = H * hd
    Sk = pos0 + S if kcache is not None else S
    if O is None:
        O = torch.empty(B * S, d, dtype=torch.bfloat16, device=qkv.device)
    ldo = _rows_out(O, "O", B * S, d)
    if P is None and want_p:
        P = torch.empty(B, H, S, (Sk + 7) // 8 * 8, dtype=torch.bfloat16, device=qkv.device)
    ldP = _p_out(P, B, H, S, Sk) if P is not None else 0
    if stats is None and want_stats:
        stats = torch.empty(B, H, S, 2, dtype=torch.float32, device=qkv.device)
    if stats is not None and (stats.dtype != torch.float32 or tuple(stats.shape) != (B, H, S, 2)
                              or not stats.is_contiguous()):
        raise ValueError(f"stats must be a contiguous fp32 [{B}, {H}, {S}, 2] tensor")
    ld = qkv.stride(0)
    if kcache is not None:
        Smax = kcache.shape[2]
        kk, vv, ldk, bsh, bsb = kcache.data_ptr(), vcache.data_ptr(), hd, Smax * hd, H * Smax * hd
    else:
        kk, vv, ldk, bsh, bsb = qkv.data_ptr() + 2 * d, qkv.data_ptr() + 4 * d, ld, hd, S * ld
    check(lib().mb200_attn_fwd_flash(_ptr(qkv), ld, hd, S * ld, kk, ldk, bsh, bsb, vv, ldk, bsh, bsb, _ptr(O), ldo,
                                     _ptr(P), ldP, _ptr(stats), B, S, Sk, H, hd, bool(causal), _stream()))
    out = (O,)
    if want_p:
        out += (P,)
    if want_stats:
        out += (stats,)
    return out if len(out) > 1 else O


def attn_bwd_tile(qkv, dO, P, B, S, H, hd, rope_tab=None, rot=0, dqkv=None):
    """Backward of attn_fwd_tile -> dqkv [B*S, 3*H*hd] (inverse rotary applied to dq, dk when rope_tab is given).
    dqkv may be given with a padded row stride."""
    if dqkv is None:
        dqkv = torch.empty(B * S, 3 * H * hd, dtype=torch.bfloat16, device=qkv.device)
    ld = _rows_out(dqkv, "dqkv", B * S, 3 * H * hd)
    check(lib().mb200_attn_bwd_tile(_ptr(qkv), qkv.stride(0), _ptr(dO), dO.stride(0), _ptr(P), _p_out(P, B, H, S, S),
                                    _ptr(dqkv), ld, _ptr(rope_tab), int(rot), B, S, H, hd, _stream()))
    return dqkv


def kv_append(qkv, kcache, vcache, B, S, H, hd, pos0):
    """K / V of the fused qkv rows [B*S, 3*H*hd] (row stride qkv.stride(0)) into the caches [B, H, Smax, hd] at
    positions [pos0, pos0 + S) (mb200_kv_append)."""
    check(lib().mb200_kv_append(_ptr(qkv), qkv.stride(0), _ptr(kcache), _ptr(vcache), B, S, H, hd,
                                kcache.shape[2], pos0, _stream()))


def attn_decode(qkv, kcache, vcache, B, H, hd, pos, out=None):
    """One decode step (mb200_attn_decode): qkv [B, 3*H*hd] (one already-rotated row per batch, row stride
    qkv.stride(0)) appends its k, v at cache position `pos` of kcache / vcache [B, H, Smax, hd], then attends over
    [0, pos]. Returns out [B, H*hd] (may be given with a padded row stride)."""
    if out is None:
        out = torch.empty(B, H * hd, dtype=torch.bfloat16, device=qkv.device)
    ldo = _rows_out(out, "out", B, H * hd)
    check(lib().mb200_attn_decode(_ptr(qkv), qkv.stride(0), _ptr(kcache), _ptr(vcache), _ptr(out), ldo, B, H, hd,
                                  kcache.shape[2], int(pos), _stream()))
    return out


def attn_decode_dev(qkv, kcache, vcache, B, H, hd, pos_dev, out=None):
    """attn_decode with the cache position read from device memory (int32 [1]; mb200_attn_decode_dev)."""
    if out is None:
        out = torch.empty(B, H * hd, dtype=torch.bfloat16, device=qkv.device)
    ldo = _rows_out(out, "out", B, H * hd)
    check(lib().mb200_attn_decode_dev(_ptr(qkv), qkv.stride(0), _ptr(kcache), _ptr(vcache), _ptr(out), ldo, B, H, hd,
                                      kcache.shape[2], _ptr(pos_dev), _stream()))
    return out
