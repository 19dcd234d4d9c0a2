"""Image encoders — drop-in for magma/image_encoders.py (`get_image_encoder`) re-backed by the CUDA runtime.

The reference obtains its encoders from openai/CLIP (`clip.load(name)[0].visual`, image_encoders.py:65) and timm;
neither package is vendored. This module implements CLIP's VisionTransformer family natively (patchify-conv as
im2col + GEMM, 24x [LN -> QKV GEMM+bias -> attention -> out GEMM+bias+residual -> LN -> fc GEMM+bias+
QuickGELU -> proj GEMM+bias+residual], ln_post(CLS) @ proj) with openai/CLIP's parameter names, and extends the
reference's name table with `clip_vit_large` (ViT-L/14, BASELINE.json config 2) following the reference's own ViT
convention (pooled [b, D] features; `"clip"` = ViT-B/32 -> 512, image_prefix.py:18).

CLIP's conv trunks (`clip_resnet` = RN50x4, `clip_resnet_large` = RN50x16, the encoder MAGMA_v1.yml ships with) are
implemented as `B200ModifiedResNet`: NHWC bf16 activations, 1x1 convolutions as plain GEMMs, 3x3 convolutions
as im2col + GEMM, eval-mode BatchNorm folded into the packed weights / GEMM bias, ReLU and the bottleneck residual in
the GEMM epilogue, the anti-aliasing average pools as one HBM-bound kernel; attention pool replaced by the
"b d h w -> b (h w) d" reshape exactly as the reference does (image_encoders.py:69-74). timm's `nfresnet50` raises.
"""
from collections import OrderedDict
import ctypes
import os

import torch
import torch.nn as nn

from . import ops
from ._lib import MB200Error, VitGradsC, VitLayerC, VitLayerGradsC, VitModelC, check, lib

# name -> (width, layers, heads, patch, input_resolution, mlp, out_dim)
VIT_CONFIGS = {
    "clip": (768, 12, 12, 32, 224, 3072, 512),             # ViT-B/32 (image_encoders.py:56-57)
    "ViT-B/32": (768, 12, 12, 32, 224, 3072, 512),
    "clip_vit_large": (1024, 24, 16, 14, 224, 4096, 768),  # ViT-L/14 (extension)
    "ViT-L/14": (1024, 24, 16, 14, 224, 4096, 768),
}


def register_vit(name, width, layers, heads, patch, input_resolution, mlp, out_dim):
    """Add a CLIP-ViT geometry under `name` (must contain "clip", like the reference's dispatch at
    image_encoders.py:87) — used by the tests for small configurations."""
    from . import image_prefix

    VIT_CONFIGS[name] = (width, layers, heads, patch, input_resolution, mlp, out_dim)
    image_prefix.ENCODER_OUT_DIMS[name] = out_dim


def _p(*shape, device):
    return nn.Parameter(torch.empty(*shape, dtype=torch.bfloat16, device=device), requires_grad=False)


class _Lin(nn.Module):
    def __init__(self, i, o, device):
        super().__init__()
        self.weight, self.bias = _p(o, i, device=device), _p(o, device=device)


class _LN(nn.Module):
    def __init__(self, d, device):
        super().__init__()
        self.weight, self.bias = _p(d, device=device), _p(d, device=device)


class _Attn(nn.Module):
    def __init__(self, w, device):
        super().__init__()
        self.in_proj_weight, self.in_proj_bias = _p(3 * w, w, device=device), _p(3 * w, device=device)
        self.out_proj = _Lin(w, w, device)


class _MLP(nn.Module):
    def __init__(self, w, m, device):
        super().__init__()
        self.c_fc, self.c_proj = _Lin(w, m, device), _Lin(m, w, device)


class _ResBlock(nn.Module):
    def __init__(self, w, m, device):
        super().__init__()
        self.ln_1, self.attn, self.ln_2, self.mlp = _LN(w, device), _Attn(w, device), _LN(w, device), _MLP(w, m, device)


class _Transformer(nn.Module):
    def __init__(self, w, n, m, device):
        super().__init__()
        self.resblocks = nn.ModuleList([_ResBlock(w, m, device) for _ in range(n)])


class _Conv(nn.Module):
    def __init__(self, w, patch, device):
        super().__init__()
        self.weight = _p(w, 3, patch, patch, device=device)


_VIT_LAYER_FIELDS = (("ln1_g", "ln_1.weight"), ("ln1_b", "ln_1.bias"), ("w_qkv", "attn.in_proj_weight"),
                     ("b_qkv", "attn.in_proj_bias"), ("w_out", "attn.out_proj.weight"), ("b_out", "attn.out_proj.bias"),
                     ("ln2_g", "ln_2.weight"), ("ln2_b", "ln_2.bias"), ("w_fc", "mlp.c_fc.weight"),
                     ("b_fc", "mlp.c_fc.bias"), ("w_proj", "mlp.c_proj.weight"), ("b_proj", "mlp.c_proj.bias"))
_VIT_TOP_FIELDS = (("cls", "class_embedding"), ("pos", "positional_embedding"), ("ln_pre_g", "ln_pre.weight"),
                   ("ln_pre_b", "ln_pre.bias"), ("ln_post_g", "ln_post.weight"), ("ln_post_b", "ln_post.bias"))


class _VitTrainFn(torch.autograd.Function):
    """feats = ViT(images) with the hand-written backward of csrc/vit_sched.cu (`freeze_img_encoder: false`): every
    parameter gradient is written as fp32 straight into the trainable-parameter arena. `anchor` is one trainable
    parameter: it makes autograd call backward although the pixels carry no gradient."""

    @staticmethod
    def forward(ctx, enc, x, anchor):
        feats = enc._run_forward_train(x)
        ctx.enc, ctx.B, ctx.generation = enc, x.shape[0], enc._generation
        return feats

    @staticmethod
    def backward(ctx, dfeats):
        enc = ctx.enc
        if ctx.generation != enc._generation:
            raise MB200Error("backward called after another training forward overwrote the saved ViT activations")
        enc._run_backward(dfeats.to(torch.bfloat16).contiguous(), ctx.B)
        return None, None, None


class B200VisionTransformer(nn.Module):
    """CLIP VisionTransformer with openai/CLIP state-dict names (conv1, class_embedding, positional_embedding,
    ln_pre, transformer.resblocks.{i}.{ln_1,attn.{in_proj_weight,in_proj_bias,out_proj},ln_2,mlp.{c_fc,c_proj}},
    ln_post, proj). Attribute `input_resolution` is read by Magma.__init__ (magma/magma.py:69)."""

    supports_training = True  # Magma(freeze_img_encoder=False) sets requires_grad on this encoder's parameters

    def __init__(self, width, layers, heads, patch, input_resolution, mlp, out_dim, device=None):
        super().__init__()
        dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self._device = dev
        self.input_resolution = input_resolution
        self.width, self.layers, self.heads, self.patch, self.mlp_dim, self.output_dim = width, layers, heads, patch, mlp, out_dim
        T = (input_resolution // patch) ** 2 + 1
        self.conv1 = _Conv(width, patch, dev)
        self.class_embedding = _p(width, device=dev)
        self.positional_embedding = _p(T, width, device=dev)
        self.ln_pre = _LN(width, dev)
        self.transformer = _Transformer(width, layers, mlp, dev)
        self.ln_post = _LN(width, dev)
        self.proj = _p(width, out_dim, device=dev)
        self._cache = None
        self._gcache = None
        self._ws = {}
        self._ws_train = {}
        self._arena = None
        self._generation = 0

    @torch.no_grad()
    def init_weights(self, seed=0, std=0.02):
        g = torch.Generator(device=self._device).manual_seed(seed)
        for name, p in self.named_parameters():
            r = std * torch.randn(p.shape, generator=g, device=self._device)
            if name.endswith(("ln_1.weight", "ln_2.weight", "ln_pre.weight", "ln_post.weight")):
                r = 1.0 + r
            p.data.copy_(r)
        self.invalidate()
        return self

    def invalidate(self):
        self._cache = None
        self._gcache = None

    def load_state_dict(self, *a, **kw):  # the packed conv1 / proj^T copies the kernels read are derived from the weights
        self.invalidate()
        return super().load_state_dict(*a, **kw)

    def _load_from_state_dict(self, *a, **kw):  # reached when a parent module loads a checkpoint
        self.invalidate()
        return super()._load_from_state_dict(*a, **kw)

    def attach_arena(self, arena):
        """Trainable encoder (freeze_img_encoder: false): parameters are fp32 master views of the arena and the
        kernels read the arena's bf16 compute copy."""
        self._arena = arena
        self.invalidate()

    def _trainable(self):
        flags = [p.requires_grad for p in self.parameters()]
        if any(flags) and not all(flags):
            raise MB200Error("the ViT encoder trains all of its parameters or none (mixed requires_grad is not supported)")
        return all(flags)

    def _w(self, name, p):
        """The bf16 tensor the kernels read for parameter p."""
        if p.requires_grad:
            if self._arena is None:
                raise MB200Error("trainable ViT parameters need the parameter arena (Magma.finalize())")
            return self._arena.shadow_of(p)
        if p.dtype != torch.bfloat16 or p.device.type != self._device.type:
            raise MB200Error(f"frozen ViT parameter {name} must be bf16 on {self._device}")
        return p.data

    def _refresh_packed(self):
        """conv1 is staged as [w, 3P^2 padded to 8] and proj transposed; with a trainable encoder both follow the
        optimizer, so they are rewritten from the compute copy before every pass (0.7 M elements)."""
        _, _, conv, proj_t = self._cache
        K = 3 * self.patch * self.patch
        conv[:, :K].copy_(self._w("conv1.weight", self.conv1.weight).reshape(self.width, K))
        proj_t.copy_(self._w("proj", self.proj).t())

    def _cmodel(self):
        if self._cache is not None:
            return self._cache
        named = dict(self.named_parameters())
        K = 3 * self.patch * self.patch
        ldk = (K + 7) // 8 * 8
        conv = torch.zeros(self.width, ldk, dtype=torch.bfloat16, device=self._device)
        proj_t = torch.empty(self.output_dim, self.width, dtype=torch.bfloat16, device=self._device)
        layers = (VitLayerC * self.layers)()
        for i in range(self.layers):
            for f, k in _VIT_LAYER_FIELDS:
                n = f"transformer.resblocks.{i}.{k}"
                setattr(layers[i], f, self._w(n, named[n]).data_ptr())
        m = VitModelC()
        m.n_layer, m.width, m.n_head, m.patch = self.layers, self.width, self.heads, self.patch
        m.image, m.mlp, m.out_dim = self.input_resolution, self.mlp_dim, self.output_dim
        m.w_conv, m.ld_conv = conv.data_ptr(), ldk
        for f, k in _VIT_TOP_FIELDS:
            setattr(m, f, self._w(k, named[k]).data_ptr())
        m.proj_t = proj_t.data_ptr()
        m.layers = ctypes.cast(layers, ctypes.POINTER(VitLayerC))
        self._cache = (m, layers, conv, proj_t)
        self._refresh_packed()
        return self._cache

    def _cgrads(self):
        """mb200_vit_grads over the arena's fp32 gradient views (parameter shapes; conv1 as [w, 3P^2])."""
        if self._gcache is None:
            named, ar = dict(self.named_parameters()), self._arena
            lg = (VitLayerGradsC * self.layers)()
            for i in range(self.layers):
                for f, k in _VIT_LAYER_FIELDS:
                    setattr(lg[i], f, ar.grad_of(named[f"transformer.resblocks.{i}.{k}"]).data_ptr())
            G = VitGradsC()
            G.w_conv = ar.grad_of(self.conv1.weight).data_ptr()
            for f, k in _VIT_TOP_FIELDS:
                setattr(G, f, ar.grad_of(named[k]).data_ptr())
            G.proj = ar.grad_of(self.proj).data_ptr()
            G.layers = ctypes.cast(lg, ctypes.POINTER(VitLayerGradsC))
            self._gcache = (G, lg)
        return self._gcache[0]

    def _train_ws(self, B):
        if B not in self._ws_train:
            n = lib().mb200_vit_train_workspace_bytes(ctypes.byref(self._cmodel()[0]), B)
            if n == 0:
                raise MB200Error(f"vit_train_workspace_bytes: {lib().mb200_last_error().decode()}")
            self._ws_train[B] = torch.empty(n, dtype=torch.uint8, device=self._device)
        return self._ws_train[B]

    def _run_forward_train(self, x):
        B = x.shape[0]
        self._arena.sync_shadow()
        m = self._cmodel()[0]
        self._refresh_packed()
        ws = self._train_ws(B)
        self._generation += 1
        feats = torch.empty(B, self.output_dim, dtype=torch.bfloat16, device=self._device)
        check(lib().mb200_vit_forward_train(ctypes.byref(m), ops._ptr(x), ops._ptr(feats), B, ops._ptr(ws), ws.numel(),
                                            ops._stream()))
        return feats

    def _run_backward(self, dfeats, B):
        ar = self._arena
        ws = self._train_ws(B)
        acc = bool(getattr(ar, "_accumulate_current", False))
        check(lib().mb200_vit_backward(ctypes.byref(self._cmodel()[0]), ctypes.byref(self._cgrads()), ops._ptr(dfeats),
                                       acc, B, ops._ptr(ws), ws.numel(), ops._stream()))
        ar.publish_grads()

    def forward(self, x):
        """[b, 3, R, R] -> [b, out_dim] (pooled CLS features, like clip's `.visual`)."""
        B, C, R, R2 = x.shape
        if C != 3 or R != self.input_resolution or R2 != R:
            raise ValueError(f"expected [b,3,{self.input_resolution},{self.input_resolution}], got {tuple(x.shape)}")
        x = x.to(device=self._device, dtype=torch.bfloat16).contiguous()
        if self._trainable():
            if torch.is_grad_enabled():
                return _VitTrainFn.apply(self, x, self.class_embedding)
            self._arena.sync_shadow()
            self._cmodel()
            self._refresh_packed()
        m = self._cmodel()[0]
        if B not in self._ws:
            n = lib().mb200_vit_workspace_bytes(ctypes.byref(m), B)
            self._ws[B] = torch.empty(n, dtype=torch.uint8, device=self._device)
        ws = self._ws[B]
        feats = torch.empty(B, self.output_dim, dtype=torch.bfloat16, device=self._device)
        check(lib().mb200_vit_forward(ctypes.byref(m), ops._ptr(x), ops._ptr(feats), B, ops._ptr(ws), ws.numel(),
                                      ops._stream()))
        return feats


# name -> (layers, width, input_resolution) of CLIP's ModifiedResNet family (output dim = width * 32)
RESNET_CONFIGS = {
    "clip_resnet": ((4, 6, 10, 6), 80, 288),          # RN50x4 (image_encoders.py:58-59) -> 2560
    "RN50x4": ((4, 6, 10, 6), 80, 288),
    "clip_resnet_large": ((6, 8, 18, 8), 96, 384),    # RN50x16 (image_encoders.py:60-61) -> 3072, 12x12 = 144 tokens
    "RN50x16": ((6, 8, 18, 8), 96, 384),
}


def register_resnet(name, layers, width, input_resolution):
    """Add a ModifiedResNet geometry under `name` (must contain "clip") — used by the tests for small trunks."""
    from . import image_prefix

    RESNET_CONFIGS[name] = (tuple(layers), width, input_resolution)
    image_prefix.ENCODER_OUT_DIMS[name] = width * 32
    image_prefix.ENCODER_SEQ_LENS[name] = (input_resolution // 32) ** 2


class _Conv2d(nn.Module):
    def __init__(self, ci, co, k, device):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(co, ci, k, k, dtype=torch.float32, device=device), requires_grad=False)


class _BatchNorm(nn.Module):
    """Eval-mode BatchNorm2d parameters/buffers under torch's names (so CLIP / MAGMA checkpoints load)."""

    def __init__(self, c, device):
        super().__init__()
        self.eps = 1e-5
        self.weight = nn.Parameter(torch.ones(c, dtype=torch.float32, device=device), requires_grad=False)
        self.bias = nn.Parameter(torch.zeros(c, dtype=torch.float32, device=device), requires_grad=False)
        self.register_buffer("running_mean", torch.zeros(c, dtype=torch.float32, device=device))
        self.register_buffer("running_var", torch.ones(c, dtype=torch.float32, device=device))
        self.register_buffer("num_batches_tracked", torch.zeros((), dtype=torch.long, device=device))


def fold_conv_bn(conv_w: torch.Tensor, bn: "_BatchNorm", pad_cin_to: int = 0):
    """Conv (no bias) followed by eval BatchNorm == conv with weight W * s and bias (beta - mean * s),
    s = gamma / sqrt(var + eps). Returns (packed bf16 [Cout, kh*kw*Cin] in (kh, kw, c) column order — the order
    mb200_im2col3x3 writes —, bf16 bias [Cout])."""
    s = bn.weight.float() / torch.sqrt(bn.running_var.float() + bn.eps)
    w = conv_w.float() * s[:, None, None, None]
    b = bn.bias.float() - bn.running_mean.float() * s
    if pad_cin_to and w.shape[1] < pad_cin_to:
        w = torch.cat([w, w.new_zeros(w.shape[0], pad_cin_to - w.shape[1], *w.shape[2:])], 1)
    packed = w.permute(0, 2, 3, 1).reshape(w.shape[0], -1)
    return packed.to(torch.bfloat16).contiguous(), b.to(torch.bfloat16).contiguous()


class _Bottleneck(nn.Module):
    def __init__(self, inplanes, planes, stride, device):
        super().__init__()
        self.stride = stride
        self.conv1, self.bn1 = _Conv2d(inplanes, planes, 1, device), _BatchNorm(planes, device)
        self.conv2, self.bn2 = _Conv2d(planes, planes, 3, device), _BatchNorm(planes, device)
        self.conv3, self.bn3 = _Conv2d(planes, planes * 4, 1, device), _BatchNorm(planes * 4, device)
        self.downsample = None
        if stride > 1 or inplanes != planes * 4:  # CLIP names: downsample.{-1: AvgPool2d, 0: conv, 1: bn}
            self.downsample = nn.Sequential(OrderedDict([("-1", nn.AvgPool2d(stride)),
                                                         ("0", _Conv2d(inplanes, planes * 4, 1, device)),
                                                         ("1", _BatchNorm(planes * 4, device))]))


class _ResNetTrainFn(torch.autograd.Function):
    """feats = trunk(images) with BatchNorm in TRAINING mode and the hand-scheduled backward of
    B200ModifiedResNet._train_backward (`freeze_img_encoder: false` with a conv trunk — MAGMA_v1.yml / MAGMA_v2.yml).
    Parameter gradients go straight into the arena; `anchor` is one trainable parameter (the pixels carry no gradient)."""

    @staticmethod
    def forward(ctx, enc, x, anchor):
        feats, tape = enc._train_forward(x)
        enc._generation += 1
        ctx.enc, ctx.tape, ctx.generation = enc, tape, enc._generation
        return feats

    @staticmethod
    def backward(ctx, dfeats):
        enc = ctx.enc
        enc._train_backward(ctx.tape, dfeats.to(torch.bfloat16).contiguous())
        ctx.tape = None
        return None, None, None


class B200ModifiedResNet(nn.Module):
    """CLIP ModifiedResNet trunk with openai/CLIP state-dict names (conv1..3 / bn1..3, layer{1..4}.{i}.{conv1,bn1,
    conv2,bn2,conv3,bn3,downsample.{0,1}}); `attnpool` is the reshape "b d h w -> b (h w) d" of
    magma/image_encoders.py:69-74, so forward returns [b, (R/32)^2, width*32].

    Frozen (the measured configuration): eval-mode BatchNorm folded into the packed weights, one CUDA graph per batch
    size. Trainable (`freeze_img_encoder: false`, what MAGMA_v1.yml / v2.yml ship): BatchNorm in training mode (batch
    statistics by `col_moments`, normalisation + residual + ReLU by `channel_affine`, running statistics updated with
    momentum 0.1) and a hand-scheduled backward — BatchNorm / ReLU backward from the same two kernels, convolution
    wgrad and dgrad as GEMMs over the saved im2col matrix (MN-major operands), `col2im3x3` and `avgpool_nhwc_bwd` as
    the adjoints of the layout kernels. Checked on the GPU in tests/test_training_paths_gpu.py and dry-run on the CPU
    against the oracle's autograd in tests/test_host_dryrun_cpu.py."""

    supports_training = True
    bn_momentum = 0.1
    # The reference never puts a frozen encoder in eval(): under model.train() its BatchNorm layers use batch statistics
    # and keep updating their running statistics even when freeze_img_encoder is true (magma/magma.py:98-100 only clears
    # requires_grad). Setting this to True reproduces that (forward through the training-mode schedule, no backward);
    # the default keeps the frozen trunk on the folded (eval-mode BatchNorm) path.
    bn_batch_stats_when_frozen = False

    def __init__(self, layers, width, input_resolution, device=None):
        super().__init__()
        dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        assert width % 16 == 0 and input_resolution % 32 == 0, "channel counts must be multiples of 8 (16-byte rows)"
        self._device = dev
        self.input_resolution, self.width, self.layers_cfg = input_resolution, width, tuple(layers)
        self.output_dim = width * 32
        self.conv1, self.bn1 = _Conv2d(3, width // 2, 3, dev), _BatchNorm(width // 2, dev)
        self.conv2, self.bn2 = _Conv2d(width // 2, width // 2, 3, dev), _BatchNorm(width // 2, dev)
        self.conv3, self.bn3 = _Conv2d(width // 2, width, 3, dev), _BatchNorm(width, dev)
        inpl = width
        for li, n in enumerate(self.layers_cfg):
            planes, blocks = width * (2 ** li), []
            for b in range(n):
                blocks.append(_Bottleneck(inpl, planes, 2 if (b == 0 and li > 0) else 1, dev))
                inpl = planes * 4
            setattr(self, f"layer{li + 1}", nn.Sequential(*blocks))
        self._packed = None
        self._graphs = {}
        self._splitk_ws = None
        self._arena = None
        self._generation = 0

    def attach_arena(self, arena):
        self._arena = arena
        self._packed = None
        self._graphs = {}

    def _trainable(self):
        flags = [p.requires_grad for p in self.parameters()]
        if any(flags) and not all(flags):
            raise MB200Error("the conv trunk trains all of its parameters or none (mixed requires_grad is not supported)")
        return all(flags)

    # ---- training path -------------------------------------------------------------------------------------------
    def _w16(self, p):
        """bf16 values of a (trainable, fp32) parameter: the arena's compute copy when there is one."""
        if self._arena is not None and p.requires_grad:
            return self._arena.shadow_of(p)
        return p.data.to(torch.bfloat16)

    def _pack_conv(self, conv, pad_cin_to=0):
        """[Cout, Cin, k, k] -> bf16 [Cout, k*k*Cin] in the (kh, kw, c) column order im2col3x3 writes."""
        w = self._w16(conv.weight)
        if pad_cin_to and w.shape[1] < pad_cin_to:
            w = torch.cat([w, w.new_zeros(w.shape[0], pad_cin_to - w.shape[1], *w.shape[2:])], 1)
        return w.permute(0, 2, 3, 1).reshape(w.shape[0], -1).contiguous()

    def _put_grad(self, p, value, acc):
        """Write / accumulate an fp32 gradient (parameter shape) for p: into the arena's view, or p.grad without one."""
        value = value.to(torch.float32)
        if self._arena is not None:
            g = self._arena.grad_of(p)
            g.add_(value) if acc else g.copy_(value)
        else:
            p.grad = value.clone() if (p.grad is None or not acc) else p.grad + value

    def _conv_bn_fwd(self, tape, t, conv, bn, k, stride, relu, res=None, pad_cin_to=0, need_dx=True):
        """conv (no bias) -> BatchNorm(batch statistics) [-> + res] [-> ReLU] on NHWC t; records what backward needs."""
        B, H, W, Cin = t.shape
        wp = self._pack_conv(conv, pad_cin_to)
        if k == 3:
            cols, Ho, Wo = ops.im2col3x3(t, stride)
        else:
            cols, Ho, Wo = t.reshape(-1, Cin), H, W
        z = ops.gemm(cols, wp)                                    # conv output, [R, Cout] bf16
        R = z.shape[0]
        s1, s2 = ops.col_moments(z, z)                            # sum z, sum z^2 per channel (fp32)
        gamma = bn.weight.data if bn.weight.dtype == torch.float32 else bn.weight.data.float()
        beta = bn.bias.data if bn.bias.dtype == torch.float32 else bn.bias.data.float()
        # one launch: batch statistics, scale = gamma * rstd, shift = beta - mean * scale, and nn.BatchNorm2d's
        # running statistics (momentum 0.1, unbiased variance)
        mean, rstd, scale, shift = ops.bn_finalize_fwd(s1, s2, gamma.contiguous(), beta.contiguous(), R, bn.eps,
                                                       self.bn_momentum, bn.running_mean, bn.running_var)
        res2 = res.reshape(R, -1) if res is not None else None
        y = ops.channel_affine(z, scale, c0=shift, res=res2, relu=relu)
        bn.num_batches_tracked += 1
        tape.append({"conv": conv, "bn": bn, "k": k, "stride": stride, "in_shape": (B, H, W, Cin), "cols": cols, "wp": wp,
                     "z": z, "mean": mean, "rstd": rstd, "gamma": gamma, "y": y if relu else None,
                     "has_res": res is not None, "pad": pad_cin_to, "need_dx": need_dx})
        return y.view(B, Ho, Wo, -1)

    def _conv_bn_bwd(self, rec, dy, acc):
        """dy: gradient w.r.t. the unit's output [R, Cout]. Returns (gradient w.r.t. the NHWC input or None, gradient
        w.r.t. the residual input or None)."""
        z, mean, rstd, gamma, mask = rec["z"], rec["mean"], rec["rstd"], rec["gamma"], rec["y"]
        R, Cout = z.shape
        s1, t = ops.col_moments(dy, z, mask)                      # sum dy', sum dy' * z   (dy' = dy * 1[y > 0])
        bn = rec["bn"]
        if self._arena is not None:                               # dgamma / dbeta straight into the arena's gradient views
            dg, db, bn_acc = self._arena.grad_of(bn.weight), self._arena.grad_of(bn.bias), acc
        else:
            dg, db, bn_acc = torch.empty_like(s1), torch.empty_like(s1), False
        # one launch: dgamma = sum dy' * xhat, dbeta = sum dy', and the coefficients of dz = A dy' + Bc z + Cc
        A, Bc, Cc = ops.bn_bwd_coeffs(s1, t, mean, rstd, gamma.contiguous(), R, dg, db, accumulate=bn_acc)
        if self._arena is None:
            self._put_grad(bn.weight, dg, acc)
            self._put_grad(bn.bias, db, acc)
        dz = ops.channel_affine(dy, A, x2=z, a2=Bc, c0=Cc, mask=mask)   # gamma * rstd * (dy' - s1/R - xhat * s2/R)
        dres = None
        if rec["has_res"]:
            dres = dy if mask is None else ops.channel_affine(dy, torch.ones_like(A), mask=mask)
        conv, k, pad = rec["conv"], rec["k"], rec["pad"]
        B, H, W, Cin = rec["in_shape"]
        dwp = ops.gemm(dz, rec["cols"], a_mn=True, b_mn=True, out_dtype=torch.float32)   # [Cout, k*k*Cin] = dz^T cols
        dw = dwp.view(Cout, k, k, Cin).permute(0, 3, 1, 2)
        self._put_grad(conv.weight, dw[:, : conv.weight.shape[1]] if pad else dw, acc)
        if not rec["need_dx"]:
            return None, dres
        dcols = ops.gemm(dz, rec["wp"], b_mn=True)                # [R, k*k*Cin] = dz Wp
        dx = ops.col2im3x3(dcols, B, H, W, Cin, rec["stride"]) if k == 3 else dcols.view(B, H, W, Cin)
        return dx, dres

    def _train_forward(self, x):
        if self._arena is not None:
            self._arena.sync_shadow()
        self._packed = None  # the folded (eval) weights go stale with every optimizer step
        B = x.shape[0]
        tape = {"stem": [], "blocks": []}
        t = ops.nchw_to_nhwc8(x)
        t = self._conv_bn_fwd(tape["stem"], t, self.conv1, self.bn1, 3, 2, True, pad_cin_to=8, need_dx=False)
        t = self._conv_bn_fwd(tape["stem"], t, self.conv2, self.bn2, 3, 1, True)
        t = self._conv_bn_fwd(tape["stem"], t, self.conv3, self.bn3, 3, 1, True)
        tape["stem_pool_in"] = t.shape
        t = ops.avgpool_nhwc(t, 2)
        for blk in self.blocks():
            rec = {"units": [], "stride": blk.stride, "in_shape": t.shape, "ds": blk.downsample is not None}
            out = self._conv_bn_fwd(rec["units"], t, blk.conv1, blk.bn1, 1, 1, True)
            out = self._conv_bn_fwd(rec["units"], out, blk.conv2, blk.bn2, 3, 1, True)
            rec["pool_in"] = out.shape
            if blk.stride > 1:
                out = ops.avgpool_nhwc(out, blk.stride)
            idn = t
            if blk.downsample is not None:
                if blk.stride > 1:
                    idn = ops.avgpool_nhwc(t, blk.stride)
                idn = self._conv_bn_fwd(rec["units"], idn, blk.downsample[1], blk.downsample[2], 1, 1, False)
            t = self._conv_bn_fwd(rec["units"], out, blk.conv3, blk.bn3, 1, 1, True, res=idn)  # relu(bn3(conv3) + idn)
            tape["blocks"].append(rec)
        return t.reshape(B, -1, t.shape[-1]), tape

    def _train_backward(self, tape, dfeats):
        ar = self._arena
        acc = bool(getattr(ar, "_accumulate_current", False)) if ar is not None else False
        g = dfeats.reshape(-1, dfeats.shape[-1])                  # [B*h*w, C]: NHWC rows, like the forward reshape
        for rec in reversed(tape["blocks"]):
            units = rec["units"]
            u1, u2, u3 = units[0], units[1], units[-1]
            d_out, d_idn = self._conv_bn_bwd(u3, g, acc)
            if rec["stride"] > 1:
                _, H, W, _ = rec["pool_in"]
                d_out = ops.avgpool_nhwc_bwd(d_out, H, W, rec["stride"])
            d2, _ = self._conv_bn_bwd(u2, d_out.reshape(-1, d_out.shape[-1]), acc)
            d1, _ = self._conv_bn_bwd(u1, d2.reshape(-1, d2.shape[-1]), acc)
            Bx, Hx, Wx, Cx = rec["in_shape"]
            if rec["ds"]:
                dd, _ = self._conv_bn_bwd(units[2], d_idn, acc)
                if rec["stride"] > 1:
                    dd = ops.avgpool_nhwc_bwd(dd, Hx, Wx, rec["stride"])
            else:
                dd = d_idn
            g = ops.add(d1.reshape(-1, Cx), dd.reshape(-1, Cx))
        _, H, W, C = tape["stem_pool_in"]
        g = ops.avgpool_nhwc_bwd(g.view(-1, H // 2, W // 2, C), H, W, 2)
        for rec in reversed(tape["stem"]):
            g, _ = self._conv_bn_bwd(rec, g.reshape(-1, g.shape[-1]), acc)
        if ar is not None:
            ar.publish_grads()

    @torch.no_grad()
    def init_weights(self, seed=0):
        g = torch.Generator(device=self._device).manual_seed(seed)
        for name, p in self.named_parameters():
            if p.ndim == 4:
                fan = p.shape[1] * p.shape[2] * p.shape[3]
                p.data.copy_(torch.randn(p.shape, generator=g, device=self._device) * (2.0 / fan) ** 0.5)
            elif name.endswith("bn3.weight") or name.endswith("downsample.1.weight"):
                p.data.fill_(0.5)
        self._packed = None
        return self

    def invalidate(self):
        self._packed = None

    def load_state_dict(self, *a, **kw):
        self._packed = None
        return super().load_state_dict(*a, **kw)

    def _load_from_state_dict(self, *a, **kw):  # reached when a parent module loads a checkpoint
        self._packed = None
        return super()._load_from_state_dict(*a, **kw)

    def blocks(self):
        for li in range(4):
            yield from getattr(self, f"layer{li + 1}")

    def _pack(self):
        if self._packed is None:
            pk = {"stem": [fold_conv_bn(self.conv1.weight, self.bn1, pad_cin_to=8), fold_conv_bn(self.conv2.weight, self.bn2),
                           fold_conv_bn(self.conv3.weight, self.bn3)], "blocks": []}
            for blk in self.blocks():
                ds = fold_conv_bn(blk.downsample[1].weight, blk.downsample[2]) if blk.downsample is not None else None
                pk["blocks"].append((fold_conv_bn(blk.conv1.weight, blk.bn1), fold_conv_bn(blk.conv2.weight, blk.bn2),
                                     fold_conv_bn(blk.conv3.weight, blk.bn3), ds))
            self._packed = pk
        return self._packed

    def forward(self, x):
        """[b, 3, R, R] -> [b, (R/32)^2, width*32]."""
        B, C, R, R2 = x.shape
        if C != 3 or R != self.input_resolution or R2 != R:
            raise ValueError(f"expected [b,3,{self.input_resolution},{self.input_resolution}], got {tuple(x.shape)}")
        x = x.to(device=self._device, dtype=torch.bfloat16).contiguous()
        if self._trainable() and self.training and torch.is_grad_enabled():
            return _ResNetTrainFn.apply(self, x, self.conv1.weight)       # BatchNorm in training mode + backward
        if self.training and self.bn_batch_stats_when_frozen and not self._trainable():
            with torch.no_grad():
                return self._train_forward(x)[0]                          # reference-literal frozen trunk under train()
        # frozen, or a trainable trunk in eval mode: running statistics folded into the weights (re-packed from the
        # current fp32 parameters after every training forward, which resets self._packed)
        if x.is_cuda and os.environ.get("MB200_RESNET_GRAPH", "1") != "0" and \
                not torch.cuda.is_current_stream_capturing():
            return self._forward_graphed(x)
        return self._forward_eager(x)

    def _forward_graphed(self, x):
        """The trunk is ~300 short launches with static shapes: replay them as one CUDA graph per batch size (the
        host-side launch cost, not the GPU, bounds the eager version). The result is copied out of the graph's static
        buffer, so it stays valid across later calls."""
        B = x.shape[0]
        entry = self._graphs.get(B)
        if entry is None or entry[3] is not self._pack():
            pk = self._pack()
            static_in = torch.empty_like(x)
            static_in.copy_(x)
            s = torch.cuda.Stream(device=self._device)
            s.wait_stream(torch.cuda.current_stream(self._device))
            with torch.cuda.stream(s):
                self._forward_eager(static_in)  # warm-up outside capture (function attributes, allocator)
            torch.cuda.current_stream(self._device).wait_stream(s)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                static_out = self._forward_eager(static_in)
            entry = (g, static_in, static_out, pk)
            self._graphs[B] = entry
        g, static_in, static_out, _ = entry
        static_in.copy_(x)
        g.replay()
        return static_out.clone()

    def _forward_eager(self, x):
        B = x.shape[0]
        pk = self._pack()
        x = ops.nchw_to_nhwc8(x)

        if self._splitk_ws is None:  # fp32 split-K scratch for the few-tile / long-K convolutions of the late stages
            self._splitk_ws = torch.empty(16 << 20, dtype=torch.float32, device=self._device)
        ws = self._splitk_ws

        def conv3x3(t, wb, stride):
            cols, Ho, Wo = ops.im2col3x3(t, stride)
            return ops.gemm(cols, wb[0], bias=wb[1], act=ops.ACT_RELU, splitk_ws=ws).view(t.shape[0], Ho, Wo, -1)

        def conv1x1(t, wb, **kw):
            return ops.gemm(t.reshape(-1, t.shape[-1]), wb[0], bias=wb[1], splitk_ws=ws, **kw).view(*t.shape[:3], -1)

        x = conv3x3(x, pk["stem"][0], 2)
        x = conv3x3(x, pk["stem"][1], 1)
        x = conv3x3(x, pk["stem"][2], 1)
        x = ops.avgpool_nhwc(x, 2)
        for blk, (w1, w2, w3, wd) in zip(self.blocks(), pk["blocks"]):
            out = conv1x1(x, w1, act=ops.ACT_RELU)
            out = conv3x3(out, w2, 1)
            if blk.stride > 1:
                out = ops.avgpool_nhwc(out, blk.stride)
            idn = x
            if wd is not None:
                idn = conv1x1(ops.avgpool_nhwc(x, blk.stride) if blk.stride > 1 else x, wd)
            x = conv1x1(out, w3, act=ops.ACT_RELU_POST, res1=idn.reshape(-1, idn.shape[-1]))  # relu(bn3(conv3) + identity)
        return x.reshape(B, -1, x.shape[-1])


def clip_encoder(device=None, name: str = "clip") -> nn.Module:
    """magma/image_encoders.py:48-76."""
    if name in RESNET_CONFIGS:
        return B200ModifiedResNet(*RESNET_CONFIGS[name], device=device)
    if name not in VIT_CONFIGS:
        raise ValueError(f"encoder {name} not recognized")
    return B200VisionTransformer(*VIT_CONFIGS[name], device=device)


def get_image_encoder(name: str, device=None, pretrained: bool = False) -> nn.Module:
    """magma/image_encoders.py:79-91. Weights are uninitialised/random: no checkpoint source exists offline."""
    if name == "nfresnet50":
        raise NotImplementedError("nfresnet50 (timm NF-ResNet conv trunk) is not re-backed")
    if "clip" in name or name in VIT_CONFIGS or name in RESNET_CONFIGS:
        return clip_encoder(device=device, name=name)
    raise ValueError(f"image encoder {name} not recognized")
