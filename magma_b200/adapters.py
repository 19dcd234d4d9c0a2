"""Adapter modules — drop-in for magma/adapters.py (same class names, constructor signatures and state-dict
keys `adapter.{0,2}.{weight,bias}`), re-backed by the wgmma GEMM core.

Inside the LM the adapters are executed by the C++ GPT-J runtime (csrc/gptj_sched.cu), which discovers them through the
same `block.mlp` / `block.attn` rewiring the reference performs (magma/magma.py:128-169). `forward` below is the
standalone path (an adapter called on its own): down-proj GEMM with fused bias+ReLU epilogue, up-proj GEMM with
fused bias+residual epilogue; backward = two dgrad GEMMs (MN-major weight operand, ReLU mask fused) and two wgrad
GEMMs (MN-major activations, fp32 output)."""
import torch
import torch.nn as nn

from . import ops


def _bf16(t):
    return t if t.dtype == torch.bfloat16 else t.to(torch.bfloat16)


def activation_kind(activation) -> int:
    """The bottleneck activation as the kernels know it: 0 = ReLU (the reference default, adapters.py:11), 1 = GeLU in
    the tanh form the GPT-J MLP itself uses (nn.GELU(approximate="tanh") / transformers' NewGELUActivation) — both are
    fused into the down-projection's GEMM epilogue (the GeLU one also saves its pre-activation for the backward pass).
    `activation` is what the reference passes: a module CLASS (or any zero-argument factory) instantiated once."""
    if activation is nn.ReLU:
        return 0
    probe = activation() if callable(activation) and not isinstance(activation, nn.Module) else activation
    if isinstance(probe, nn.ReLU):
        return 0
    if isinstance(probe, nn.GELU) and getattr(probe, "approximate", "none") == "tanh":
        return 1
    if type(probe).__name__ in ("NewGELUActivation", "GELUTanh"):
        return 1
    raise NotImplementedError(
        f"adapter activation {activation!r}: magma_b200 fuses ReLU (the reference default, adapters.py:11) or the tanh "
        "GeLU (nn.GELU(approximate='tanh')) into the bottleneck GEMMs; exact-erf GELU and others are not re-backed")


class _AdapterFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, wd, bd, wu, bu, residual, act=0):
        shp = x.shape
        x2 = _bf16(x).reshape(-1, shp[-1]).contiguous()
        wd16, bd16, wu16, bu16 = _bf16(wd), _bf16(bd), _bf16(wu), _bf16(bu)
        if act == 0:
            t = ops.gemm(x2, wd16, bias=bd16, act=ops.ACT_RELU)
            pre = t  # the ReLU mask is read off the output
        else:
            pre = torch.empty(x2.shape[0], wd16.shape[0], dtype=torch.bfloat16, device=x2.device)
            t = ops.gemm(x2, wd16, bias=bd16, act=ops.ACT_GELU_NEW, aux_out=pre)
        y = ops.gemm(t, wu16, bias=bu16, res1=x2 if residual else None)
        ctx.save_for_backward(x2, t, wd16, wu16, pre)
        ctx.act = act
        ctx.residual = residual
        ctx.shape = shp
        ctx.dtypes = (x.dtype, wd.dtype)
        return y.reshape(shp).to(x.dtype)

    @staticmethod
    def backward(ctx, gy):
        x2, t, wd16, wu16, pre = ctx.saved_tensors
        g = _bf16(gy).reshape(-1, ctx.shape[-1]).contiguous()
        dt = ops.gemm(g, wu16, b_mn=True, aux_in=pre,                            # (g Wu) * act'(pre)   (ReLU: 1[t>0])
                      dact=ops.DACT_RELU if ctx.act == 0 else ops.DACT_GELU_NEW)
        dwu = ops.gemm(g, t, a_mn=True, b_mn=True, out_dtype=torch.float32)       # g^T t
        dbu = ops.colsum(g)
        dwd = ops.gemm(dt, x2, a_mn=True, b_mn=True, out_dtype=torch.float32)     # dt^T x
        dbd = ops.colsum(dt)
        dx = ops.gemm(dt, wd16, b_mn=True, res1=g if ctx.residual else None)      # dt Wd (+ g)
        xd, wdt = ctx.dtypes
        return dx.reshape(ctx.shape).to(xd), dwd.to(wdt), dbd.to(wdt), dwu.to(wdt), dbu.to(wdt), None, None


class Adapter(nn.Module):
    """magma/adapters.py:6-39."""

    def __init__(self, dim: int, downsample_factor: int = 4, activation: nn.Module = nn.ReLU,
                 add_layernorm: bool = False):
        super().__init__()
        self.act_kind = activation_kind(activation)  # raises for activations the kernels do not fuse
        layers = []
        if add_layernorm:
            layers.append(nn.LayerNorm(dim))
        layers.extend([nn.Linear(dim, dim // downsample_factor), activation(), nn.Linear(dim // downsample_factor, dim)])
        self.adapter = nn.Sequential(*layers)
        self.add_layernorm = add_layernorm
        self.dim = dim
        self.bottleneck = dim // downsample_factor
        self.adapter.apply(self.init_weights)

    def init_weights(self, m: nn.Module, std=1e-3):
        """N(0, std) clamped to +-2 std for Linear weight and bias; LN -> (1, 0)  (adapters.py:28-36)."""
        if isinstance(m, nn.Linear):
            torch.nn.init.normal_(m.weight, std=std)
            torch.nn.init.normal_(m.bias, std=std)
            m.weight.data = torch.clamp(m.weight.data, min=-2 * std, max=2 * std)
            m.bias.data = torch.clamp(m.bias.data, min=-2 * std, max=2 * std)
        elif isinstance(m, nn.LayerNorm):
            m.bias.data.zero_()
            m.weight.data.fill_(1.0)

    @property
    def down(self):
        return self.adapter[1 if self.add_layernorm else 0]

    @property
    def up(self):
        return self.adapter[3 if self.add_layernorm else 2]

    def bottleneck_fn(self, x, residual):
        if self.add_layernorm:
            raise NotImplementedError("add_layernorm adapters are not re-backed yet")
        return _AdapterFn.apply(x, self.down.weight, self.down.bias, self.up.weight, self.up.bias, residual, self.act_kind)

    def forward(self, x):
        return self.bottleneck_fn(x, True)  # self.adapter(x) + x


class ParallelAdapter(Adapter):
    """magma/adapters.py:42-66."""

    def __init__(self, module: nn.Module, dim: int, downsample_factor: int = 4, scaled: bool = False,
                 add_layernorm: bool = False, activation: nn.Module = nn.ReLU):
        super().__init__(dim, downsample_factor, add_layernorm=add_layernorm, activation=activation)
        self.module = module
        if scaled:
            self.adapter_scale = nn.Parameter(torch.ones(1))
        else:
            self.adapter_scale = 1

    def forward(self, x, **module_kwargs):
        y = self.module(x, **module_kwargs)
        z = self.bottleneck_fn(x, False)
        return y + (z * self.adapter_scale)


class ParallelAdapterWrapper(ParallelAdapter):
    """magma/adapters.py:69-92 (attention variant: passes through (present, attentions))."""

    def forward(self, x, *attn_args, **attn_kwargs):
        attn_outputs = self.module(x, *attn_args, **attn_kwargs)
        attn_output, outputs = attn_outputs[0], attn_outputs[1:]
        hidden_states = attn_output + (self.bottleneck_fn(x, False) * self.adapter_scale)
        return (hidden_states,) + outputs


class AdapterWrapper(Adapter):
    """magma/adapters.py:95-116."""

    def __init__(self, attn_block: nn.Module, dim: int, downsample_factor: int = 4, activation: nn.Module = nn.ReLU,
                 add_layernorm: bool = False):
        super().__init__(dim, downsample_factor, activation, add_layernorm)
        self.attn_block = attn_block

    def forward(self, x, *attn_args, **attn_kwargs):
        attn_outputs = self.attn_block(x, *attn_args, **attn_kwargs)
        attn_output, outputs = attn_outputs[0], attn_outputs[1:]
        hidden_states = self.bottleneck_fn(attn_output, True)
        return (hidden_states,) + outputs
