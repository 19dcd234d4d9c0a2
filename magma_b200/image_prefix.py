"""ImagePrefix — drop-in for magma/image_prefix.py: enc(x) -> Linear(enc_dim, out_dim*seq) -> reshape -> Dropout ->
LayerNorm, with the projection on the wgmma GEMM core (bias fused), dropout and LayerNorm as bf16 kernels, and a
hand-written backward (wgrad GEMM with MN-major operands, bias/LN-parameter reductions) that writes fp32 gradients
straight into the trainable-parameter arena."""
import torch
import torch.nn as nn

from . import ops
from .config import MultimodalConfig
from .image_encoders import get_image_encoder

# fixed-sequence-length encoders (no pooling) — magma/image_prefix.py:11-14
ENCODER_SEQ_LENS = {"clip_resnet": 49, "clip_resnet_large": 144}
# encoder output dims — magma/image_prefix.py:16-21, extended with the ViT-L/14 entry
ENCODER_OUT_DIMS = {"nfresnet50": 2048, "clip": 512, "clip_resnet": 2560, "clip_resnet_large": 3072,
                    "clip_vit_large": 768}


class _PrefixFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, mod, feats, w, b, lnw, lnb):
        B = feats.shape[0]
        arena = mod._arena
        w16 = arena.shadow_of(w) if arena is not None else w.to(torch.bfloat16)
        b16 = arena.shadow_of(b) if arena is not None else b.to(torch.bfloat16)
        y = ops.gemm(feats, w16, bias=b16)                                  # [B, out_dim * s]
        rows = y.view(-1, mod.out_dim) if mod.reshape_seq else y.view(-1, mod.out_dim)
        mask = None
        p = mod.dropout.p if mod.training else 0.0
        if p > 0:
            mod._seed += 1
            rows, mask = ops.dropout_fwd(rows.contiguous(), p, mod._seed)
        mean = rstd = None
        out = rows
        if mod.use_layernorm:
            g16 = arena.shadow_of(lnw) if arena is not None else lnw.to(torch.bfloat16)
            be16 = arena.shadow_of(lnb) if arena is not None else lnb.to(torch.bfloat16)
            out, mean, rstd = ops.layernorm_fwd(rows, g16, be16, mod.ln.eps)
            ctx.g16 = g16
        ctx.mod, ctx.p, ctx.mask, ctx.w16 = mod, p, mask, w16
        ctx.save_for_backward(feats, rows, mean, rstd)
        seq = mod.out_seq_len if mod.reshape_seq else rows.shape[0] // B
        return out.view(B, seq, mod.out_dim)

    @staticmethod
    def backward(ctx, gout):
        mod = ctx.mod
        feats, rows, mean, rstd = ctx.saved_tensors
        arena = mod._arena
        acc = bool(getattr(arena, "_accumulate_current", False)) if arena is not None else False
        g = gout.to(torch.bfloat16).reshape(-1, mod.out_dim).contiguous()

        def gbuf(p):
            return arena.grad_of(p) if arena is not None else torch.zeros(p.shape, dtype=torch.float32, device=g.device)

        gl_w = gl_b = None
        if mod.use_layernorm:
            gl_w, gl_b = gbuf(mod.ln.weight), gbuf(mod.ln.bias)
            ops.layernorm_param_grad(g, rows, mean, rstd, gl_w, gl_b, accumulate=acc)
            g = ops.layernorm_bwd(g, rows, ctx.g16, mean, rstd)
        if ctx.p > 0:
            g = ops.dropout_apply(g, ctx.mask, ctx.p)
        B = feats.shape[0]
        g2 = g.view(B, -1) if mod.reshape_seq else g
        gw, gb = gbuf(mod.proj.weight), gbuf(mod.proj.bias)
        ops.gemm(g2, feats, out=gw, a_mn=True, b_mn=True, accumulate=acc)   # dW[out, in] = g^T feats
        ops.colsum(g2, out=gb, accumulate=acc)
        dfeats = None
        if ctx.needs_input_grad[1]:  # trainable encoder (freeze_img_encoder: false): dfeats = g W
            dfeats = ops.gemm(g2.contiguous(), ctx.w16, b_mn=True)
        if arena is not None:
            arena.publish_grads()
            return None, dfeats, None, None, None, None
        return None, dfeats, gw.to(mod.proj.weight.dtype), gb, gl_w, gl_b


class ImagePrefix(nn.Module):
    """magma/image_prefix.py:24-109 (same constructor, attributes `.enc .proj .dropout .ln .out_seq_len`)."""

    def __init__(self, config: MultimodalConfig, out_dim: int = 2048, device=None):
        super().__init__()
        self.device = device or torch.device("cuda" if torch.cuda.is_available() else "cpu")
        self.config = config
        self.encoder_type = config.encoder_name
        self.enc = get_image_encoder(config.encoder_name, device=self.device, pretrained=config.pretrained_img_encoder)
        self.encoder_out_dim = ENCODER_OUT_DIMS[self.encoder_type]
        self.out_dim = out_dim
        self.out_seq_len = (config.image_seq_len if config.encoder_name not in ENCODER_SEQ_LENS
                            else ENCODER_SEQ_LENS[config.encoder_name])
        self.reshape_seq = self.encoder_type not in ENCODER_SEQ_LENS
        proj_out_dim = (self.out_dim * self.out_seq_len) if self.reshape_seq else self.out_dim
        self.proj = nn.Linear(self.encoder_out_dim, proj_out_dim).to(self.device)
        self.dropout = nn.Dropout(config.image_embed_dropout_prob)
        self.use_layernorm = config.use_image_embed_layernorm
        if self.use_layernorm:
            self.ln = nn.LayerNorm(self.out_dim).to(self.device)
        self._arena = None
        self._seed = 0x5EED

    def attach_arena(self, arena):
        self._arena = arena
        if hasattr(self.enc, "attach_arena"):
            self.enc.attach_arena(arena)

    def forward(self, x):
        feats = self.enc(x)  # image_prefix.py:83
        if feats.ndim == 4:
            feats = feats[:, :, 0, 0]  # "b d 1 1 -> b d" (:86-87)
        seq_shape = None
        if feats.ndim == 3:  # conv trunks: one token per spatial position, projected individually (:89-93)
            assert self.encoder_type in ENCODER_SEQ_LENS and feats.shape[1] == self.out_seq_len, tuple(feats.shape)
            seq_shape = (feats.shape[0], feats.shape[1], self.out_dim)
            feats = feats.reshape(-1, feats.shape[-1])
        else:
            assert feats.ndim == 2
        feats = feats.to(torch.bfloat16).contiguous()
        if self._arena is not None:
            self._arena.sync_shadow()
        lnw = self.ln.weight if self.use_layernorm else None
        lnb = self.ln.bias if self.use_layernorm else None
        if torch.is_grad_enabled() and self.proj.weight.requires_grad:
            out = _PrefixFn.apply(self, feats, self.proj.weight, self.proj.bias, lnw, lnb)
        else:
            with torch.no_grad():
                out = _PrefixFn.forward(_NoCtx(), self, feats, self.proj.weight, self.proj.bias, lnw, lnb)
        return out.view(seq_shape) if seq_shape is not None else out


class _NoCtx:
    def save_for_backward(self, *a):
        pass
