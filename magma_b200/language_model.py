"""GPT-J language model — drop-in for magma/language_model.py (`get_gptj`) re-backed by the C++/CUDA runtime.

`get_gptj()` returns an object that honours every use the reference makes of its LM:
`.config.{max_position_embeddings,hidden_size,pad_token_id}`, `.resize_token_embeddings(n)`, `.transformer.wte`
(callable on int64 ids), `.transformer.h[l].{mlp,attn}` (get/settable — the seam `Magma.add_adapters` rewires,
magma/magma.py:128-169), `named_parameters()` with "adapter" in adapter names, and
`__call__(inputs_embeds=|input_ids=, labels=, use_cache=, past_key_values=, output_hidden_states=, output_attentions=)`
returning an object with `.loss`, `.logits`, `.past_key_values`, `.hidden_states` (and `.attentions` when asked for).

All frozen weights are bf16 tensors on the GPU; parameter names follow HF GPT-J (`attn.q_proj.weight`, `mlp.fc_in.*`,
`ln_1`, `ln_f`, `lm_head`) — the executable stand-in for the reference's fork. The whole
28-block forward and backward run inside libmagma_b200.so (csrc/gptj_sched.cu); this file only owns tensors and plumbing.
"""
import ctypes
import math
import os
from dataclasses import dataclass

import torch
import torch.nn as nn

from . import ops
from ._lib import (AdapterExC, GptjLayerExC, GptjModelExC, MB200Error, check,
                   lib)
from .adapters import Adapter, AdapterWrapper, ParallelAdapter, ParallelAdapterWrapper
from .arena import ParamArena

ADAPTER_NONE, ADAPTER_NORMAL, ADAPTER_PARALLEL = 0, 1, 2


@dataclass
class GPTJConfig:
    """Architecture of magma/language_model.py:12-24 (gpt-neo-2.7B config mutated into GPT-J-6B)."""

    vocab_size: int = 50400
    max_position_embeddings: int = 2048
    hidden_size: int = 4096
    num_layers: int = 28
    num_heads: int = 16
    rotary_dim: int = 64
    layer_norm_epsilon: float = 1e-5
    intermediate_size: int = None
    pad_token_id: int = None
    gradient_checkpointing: bool = False  # accepted for API parity; the runtime decides (_use_recompute)
    use_cache: bool = True

    def __post_init__(self):
        if self.intermediate_size is None:
            self.intermediate_size = 4 * self.hidden_size


class LMOutput(dict):
    """Attribute + key access like transformers' ModelOutput."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e

    __setattr__ = dict.__setitem__


class KVCache:
    """Static KV cache [n_layer, B, H, S_max, hd] x {k, v}; `pos` = number of valid positions."""

    def __init__(self, n_layer, B, H, S_max, hd, device):
        self.k = torch.empty(n_layer, B, H, S_max, hd, dtype=torch.bfloat16, device=device)
        self.v = torch.empty_like(self.k)
        self.pos = 0
        self.S_max = S_max
        self.B = B


def _frozen(*shape, device):
    return nn.Parameter(torch.empty(*shape, dtype=torch.bfloat16, device=device), requires_grad=False)


class Linear(nn.Module):
    """Weight holder (frozen, bf16) with a standalone GEMM forward."""

    def __init__(self, in_f, out_f, bias, device, weight_view=None):
        super().__init__()
        self.in_features, self.out_features = in_f, out_f
        self.weight = _frozen(out_f, in_f, device=device) if weight_view is None else nn.Parameter(
            weight_view, requires_grad=False)
        self.bias = _frozen(out_f, device=device) if bias else None

    def forward(self, x):
        x2 = x.reshape(-1, x.shape[-1]).to(torch.bfloat16).contiguous()
        return ops.gemm(x2, self.weight, bias=self.bias).reshape(*x.shape[:-1], self.out_features)


class LayerNorm(nn.Module):
    def __init__(self, d, eps, device):
        super().__init__()
        self.weight = _frozen(d, device=device)
        self.bias = _frozen(d, device=device)
        self.eps = eps

    def forward(self, x):
        return ops.layernorm_fwd(x.to(torch.bfloat16).contiguous(), self.weight, self.bias, self.eps, False)[0]


class WordEmbedding(nn.Module):
    def __init__(self, V, d, device):
        super().__init__()
        self.weight = _frozen(V, d, device=device)

    def forward(self, ids):
        return ops.embed_gather(ids.to(self.weight.device), self.weight)


class GPTJAttention(nn.Module):
    def __init__(self, cfg, device):
        super().__init__()
        d = cfg.hidden_size
        self._fused = torch.empty(3 * d, d, dtype=torch.bfloat16, device=device)
        self.q_proj = Linear(d, d, False, device, self._fused[0:d])
        self.k_proj = Linear(d, d, False, device, self._fused[d : 2 * d])
        self.v_proj = Linear(d, d, False, device, self._fused[2 * d :])
        self.out_proj = Linear(d, d, False, device)

    def fused_qkv(self):
        """[3d, d] = cat(q, k, v) weights in one buffer (re-fused if a .to()/load split the views)."""
        d = self.q_proj.weight.shape[0]
        base, esz = self._fused.data_ptr(), 2
        ptrs = [p.weight.data_ptr() for p in (self.q_proj, self.k_proj, self.v_proj)]
        if ptrs != [base, base + d * d * esz, base + 2 * d * d * esz] or self._fused.device != self.q_proj.weight.device:
            dev = self.q_proj.weight.device
            fused = torch.cat([p.weight.data.to(torch.bfloat16) for p in (self.q_proj, self.k_proj, self.v_proj)], 0).to(dev)
            self._fused = fused
            for i, p in enumerate((self.q_proj, self.k_proj, self.v_proj)):
                p.weight.data = fused[i * d : (i + 1) * d]
        return self._fused

    def forward(self, *a, **k):
        raise MB200Error("GPTJAttention runs inside the fused GPT-J runtime (call the LM, not the block)")


class GPTJMLP(nn.Module):
    def __init__(self, cfg, device):
        super().__init__()
        self.fc_in = Linear(cfg.hidden_size, cfg.intermediate_size, True, device)
        self.fc_out = Linear(cfg.intermediate_size, cfg.hidden_size, True, device)

    def forward(self, *a, **k):
        raise MB200Error("GPTJMLP runs inside the fused GPT-J runtime (call the LM, not the block)")


class GPTJBlock(nn.Module):
    def __init__(self, cfg, device):
        super().__init__()
        self.ln_1 = LayerNorm(cfg.hidden_size, cfg.layer_norm_epsilon, device)
        self.attn = GPTJAttention(cfg, device)
        self.mlp = GPTJMLP(cfg, device)


class GPTJTransformer(nn.Module):
    def __init__(self, cfg, device):
        super().__init__()
        self.wte = WordEmbedding(cfg.vocab_size, cfg.hidden_size, device)
        self.h = nn.ModuleList([GPTJBlock(cfg, device) for _ in range(cfg.num_layers)])
        self.ln_f = LayerNorm(cfg.hidden_size, cfg.layer_norm_epsilon, device)


def _split_mlp(mlp):
    if isinstance(mlp, GPTJMLP):
        return ADAPTER_NONE, mlp, None
    if isinstance(mlp, nn.Sequential) and len(mlp) == 2 and isinstance(mlp[1], Adapter):
        return ADAPTER_NORMAL, mlp[0], mlp[1]  # magma/magma.py:143-148
    if isinstance(mlp, ParallelAdapter):
        return ADAPTER_PARALLEL, mlp.module, mlp
    raise MB200Error(f"unsupported mlp wrapper {type(mlp).__name__}")


def _split_attn(attn):
    if isinstance(attn, GPTJAttention):
        return ADAPTER_NONE, attn, None
    if isinstance(attn, AdapterWrapper):
        return ADAPTER_NORMAL, attn.attn_block, attn
    if isinstance(attn, ParallelAdapterWrapper):
        return ADAPTER_PARALLEL, attn.module, attn
    raise MB200Error(f"unsupported attention wrapper {type(attn).__name__}")


def _ptr_array(tensors):
    """A C array of the tensors' data pointers (NULL for None) for the per-hidden-state arguments of the C ABI."""
    return (ctypes.c_void_p * len(tensors))(*[None if t is None else t.data_ptr() for t in tensors])


def _use_recompute(stored_bytes, other_bytes, free_bytes):
    """Whether a training pass recomputes block activations in its backward: yes when the stored-activation workspace
    plus the pass's other allocations does not fit in the memory the process can still allocate. Both paths run the
    same kernels on the same block inputs (the results agree bit for bit apart from the run-to-run last-bit variation
    of the atomically reduced 1-D gradients), so this only trades time (one more forward of the blocks) for memory."""
    return stored_bytes + other_bytes > free_bytes


def _free_bytes(device):
    """Memory a new allocation on `device` can use: free on the device plus what the caching allocator holds unused."""
    if device.type != "cuda":
        return math.inf  # the CPU emulation the host-side tests run on has no device memory to run out of
    free, _ = torch.cuda.mem_get_info(device)
    return free + torch.cuda.memory_reserved(device) - torch.cuda.memory_allocated(device)


def _backward_scale(model, dloss):
    """The loss gradient the LM head's backward scales the cross-entropy gradient by: 0 when the loss does not read
    `.loss` (also under B200Engine.backward: its hint must not add a CE term the loss does not have), else
    B200Engine.backward's hint, else dloss (a host sync). Gradients a loss sends through the logits, hidden states or
    attentions are not scaled by it."""
    if dloss is None:
        return 0.0
    if model._loss_scale_hint is not None:
        return model._loss_scale_hint
    return float(dloss)


class _LMTrainFn(torch.autograd.Function):
    """(loss, logits) = LM(inputs_embeds, labels) with the backward pass of the C++ runtime (LM frozen: dgrad through
    every GEMM, wgrad only for adapters, written straight into the parameter arena's fp32 gradient buffer). loss is None
    without labels. With want_hidden the n_layer + 1 hidden states follow (loss, logits) as outputs, then with want_attn
    the n_layer attention probabilities ([B, H, S, S rounded up to 8]); the gradients of the logits, the hidden states
    and the attentions flow back through the same backward pass."""

    @staticmethod
    def forward(ctx, model, x, labels, anchor, want_hidden=False, want_attn=False):
        loss, logits, hidden, attn = model._run_forward(x, labels, training=True, want_hidden=want_hidden,
                                                        want_attn=want_attn)
        ctx.model = model
        ctx.generation = model._generation
        ctx.shape = x.shape
        ctx.x_dtype = x.dtype
        ctx.n_hidden = len(hidden or ())
        ctx.has_labels = labels is not None
        ctx.set_materialize_grads(False)  # an output the loss does not read has no gradient to add
        return (loss, logits, *(hidden or ()), *(attn or ()))

    @staticmethod
    def backward(ctx, dloss, dlogits, *douts):
        model = ctx.model
        if ctx.generation != model._generation:
            raise MB200Error("backward called after another training forward overwrote the saved activations")
        scale = _backward_scale(model, dloss) if ctx.has_labels else None
        dx = model._run_backward(ctx.shape, scale, douts[: ctx.n_hidden], douts[ctx.n_hidden :], dlogits)
        return None, dx.to(ctx.x_dtype), None, None, None, None


class B200GPTJForCausalLM(nn.Module):
    def __init__(self, config: GPTJConfig = None, device=None):
        super().__init__()
        self.config = config or GPTJConfig()
        dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self._device = dev
        self.transformer = GPTJTransformer(self.config, dev)
        self.lm_head = Linear(self.config.hidden_size, self.config.vocab_size, True, dev)
        self._arena = None
        self._own_arena = False
        self._cmodel_ex_cache = None
        self._ws = {}
        self._generation = 0
        self._generation_recompute = False  # whether the training forward of _generation recomputes in its backward
        self._loss_scale_hint = None
        self._bwd_chunks = None       # list of (layer_hi, layer_lo); None = single chunk
        self._after_chunk = None      # callback(layer_hi, layer_lo) for gradient all-reduce overlap

    # ---- construction helpers -------------------------------------------------------------
    @torch.no_grad()
    def init_weights(self, seed=0, std=0.02):
        """Synthetic weights of the benchmark protocol: N(0, 0.02) linears, LN ~ (1, 0)."""
        g = torch.Generator(device=self._device).manual_seed(seed)
        for name, p in self.named_parameters():
            if "adapter" in name:
                continue
            if name.endswith("ln_1.weight") or name.endswith("ln_f.weight"):
                p.data.copy_(1.0 + std * torch.randn(p.shape, generator=g, device=self._device))
            else:
                p.data.copy_(std * torch.randn(p.shape, generator=g, device=self._device))
        self._cmodel_ex_cache = None
        return self

    def resize_token_embeddings(self, n):
        """magma/magma.py:50 — wte and lm_head both shrink/grow to n rows."""
        dev = self._device
        for mod, names in ((self.transformer.wte, ("weight",)), (self.lm_head, ("weight", "bias"))):
            for nm in names:
                old = getattr(mod, nm)
                new = torch.zeros(n, *old.shape[1:], dtype=old.dtype, device=dev)
                k = min(n, old.shape[0])
                new[:k] = old.data[:k]
                setattr(mod, nm, nn.Parameter(new, requires_grad=False))
        self.lm_head.out_features = n
        self.config.vocab_size = n
        self._cmodel_ex_cache = None
        return self.transformer.wte

    def adapter_parameters(self):
        return [(n, p) for n, p in self.named_parameters() if "adapter" in n]

    def attach_arena(self, arena: ParamArena):
        self._arena = arena
        self._own_arena = False
        self._cmodel_ex_cache = None

    def _ensure_arena(self):
        if self._arena is None:
            params = self.adapter_parameters()
            # backward visits layers last-to-first: order the arena the same way for all-reduce overlap
            params.sort(key=lambda np_: -int(np_[0].split(".h.")[1].split(".")[0]) if ".h." in np_[0] else 0)
            self._arena = ParamArena(params, self._device) if params else None
            self._own_arena = True
        return self._arena

    # ---- C model struct ---------------------------------------------------------------------
    def _adapter_struct_ex(self, ad):
        c = AdapterExC()
        if ad is None:
            return c
        ar = self._arena
        fields = [("wd", ad.down.weight), ("bd", ad.down.bias), ("wu", ad.up.weight), ("bu", ad.up.bias)]
        if ad.add_layernorm:
            fields += [("ln_g", ad.adapter[0].weight), ("ln_b", ad.adapter[0].bias)]
        for cname, p in fields:
            setattr(c, cname, ar.shadow_of(p).data_ptr())
            if p.requires_grad:
                setattr(c, "g_" + cname, ar.grad_of(p).data_ptr())
        sc = getattr(ad, "adapter_scale", 1)
        if isinstance(sc, nn.Parameter):  # read as fp32 straight from the arena's master copy
            c.scale = sc.data.data_ptr()
            if sc.requires_grad:
                c.g_scale = ar.grad_of(sc).data_ptr()
        return c

    def _cmodel_ex(self):
        """mb200_gptj_model_ex: frozen-weight pointers and the adapter tables (every adapter form of the reference)."""
        self._ensure_arena()
        if self._cmodel_ex_cache is not None:
            return self._cmodel_ex_cache
        cfg = self.config
        n = len(self.transformer.h)
        layers = (GptjLayerExC * n)()
        kinds, rm, ra = set(), 0, 0
        for l, blk in enumerate(self.transformer.h):
            mk, mlp, mad = _split_mlp(blk.mlp)
            ak, attn, aad = _split_attn(blk.attn)
            kinds.add((mk, ak))
            L = layers[l]
            L.ln1_g, L.ln1_b = blk.ln_1.weight.data_ptr(), blk.ln_1.bias.data_ptr()
            L.w_qkv, L.w_out = attn.fused_qkv().data_ptr(), attn.out_proj.weight.data_ptr()
            L.w_fc_in, L.b_fc_in = mlp.fc_in.weight.data_ptr(), mlp.fc_in.bias.data_ptr()
            L.w_fc_out, L.b_fc_out = mlp.fc_out.weight.data_ptr(), mlp.fc_out.bias.data_ptr()
            L.mlp_ad, L.attn_ad = self._adapter_struct_ex(mad), self._adapter_struct_ex(aad)
            rm = mad.bottleneck if mad is not None else rm
            ra = aad.bottleneck if aad is not None else ra
        if len(kinds) != 1:
            raise MB200Error("all blocks must carry the same adapter configuration")
        mk, ak = kinds.pop()
        acts = {getattr(ad, "act_kind", 0) for blk in self.transformer.h
                for ad in (_split_mlp(blk.mlp)[2], _split_attn(blk.attn)[2]) if ad is not None}
        if len(acts) > 1:
            raise MB200Error("all adapters must use the same activation")
        for name, p in self.named_parameters():
            if "adapter" not in name and (p.dtype != torch.bfloat16 or p.device.type != self._device.type):
                raise MB200Error(f"frozen LM parameter {name} must be bf16 on {self._device} (got {p.dtype}, {p.device})")
        m = GptjModelExC()
        m.n_layer, m.d, m.n_head, m.rotary_dim = n, cfg.hidden_size, cfg.num_heads, cfg.rotary_dim
        m.vocab, m.d_ff = self.lm_head.weight.shape[0], cfg.intermediate_size
        m.mlp_adapter, m.mlp_adapter_r, m.attn_adapter, m.attn_adapter_r = mk, rm, ak, ra
        m.ln_eps = cfg.layer_norm_epsilon
        m.adapter_act = acts.pop() if acts else 0
        m.layers = ctypes.cast(layers, ctypes.POINTER(GptjLayerExC))
        m.lnf_g, m.lnf_b = self.transformer.ln_f.weight.data_ptr(), self.transformer.ln_f.bias.data_ptr()
        m.w_lm, m.b_lm = self.lm_head.weight.data_ptr(), self.lm_head.bias.data_ptr()
        self._cmodel_ex_cache = (m, layers)
        return self._cmodel_ex_cache

    def _workspace_ex(self, B, S):
        """(training workspace for [B, S], whether its pass recomputes block activations). The path is chosen once,
        when the workspace is allocated, and kept with it, so a run does not switch paths between steps."""
        key = ("ex", B, S)
        if key not in self._ws:
            m = ctypes.byref(self._cmodel_ex()[0])
            stored = lib().mb200_gptj_sched_workspace_bytes(m, B, S)
            if stored == 0:
                raise MB200Error(lib().mb200_last_error().decode())
            for k in [k for k in self._ws if isinstance(k, tuple) and k[0] == "ex"]:
                del self._ws[k]
            other = B * S * (self.ldv + self.config.hidden_size) * 2  # the pass's bf16 logits and dx
            recompute = _use_recompute(stored, other, _free_bytes(self._device))
            nbytes = lib().mb200_gptj_sched_recompute_workspace_bytes(m, B, S) if recompute else stored
            self._ws[key] = (torch.empty(nbytes, dtype=torch.uint8, device=self._device), recompute)
        return self._ws[key]

    def invalidate(self):
        """Call after replacing parameters/modules (e.g. add_adapters) so the C model struct is rebuilt."""
        self._cmodel_ex_cache = None
        if self._own_arena:
            self._arena = None

    @property
    def ldv(self):
        return (self.lm_head.weight.shape[0] + 63) // 64 * 64

    # ---- passes --------------------------------------------------------------------------------
    def _run_forward(self, x, labels, training, cache=None, last_only=False, want_hidden=False, want_logits=True,
                     want_attn=False):
        """(loss, logits, hidden states, attentions): the hidden states are output_hidden_states' tuple of n_layer + 1
        [B, S, d] tensors when want_hidden, else None; the attentions n_layer [B, H, S, ld] bf16 probability buffers
        when want_attn, else None (ld = S_kv rounded up to 8; columns from S_kv on are not part of the result)."""
        B, S, d = x.shape
        x = x.to(torch.bfloat16).contiguous()
        if self._arena is not None or self.adapter_parameters():
            self._ensure_arena().sync_shadow()
        return self._run_pass(x, labels, training, cache, last_only, want_hidden, want_logits, want_attn)

    def _run_pass(self, x, labels, training, cache, last_only, want_hidden, want_logits, want_attn=False):
        """csrc/gptj_sched.cu: the training pass (activations saved for backward) when a loss is asked for, else the
        inference pass — full sequence, KV-cache prefill / decode step, last-position logits, every hidden state,
        every block's attention probabilities."""
        B, S, d = x.shape
        m = self._cmodel_ex()[0]
        V, ldv = self.lm_head.weight.shape[0], self.ldv
        n, H = len(self.transformer.h), self.config.num_heads
        if labels is not None or training:
            if cache is not None or last_only:
                raise MB200Error("a loss together with a KV cache / last-position logits is not supported")
            ws, recompute = self._workspace_ex(B, S)
            logits = torch.empty(B * S, ldv, dtype=torch.bfloat16, device=x.device) if want_logits else None
            loss = torch.zeros(1, dtype=torch.float32, device=x.device) if labels is not None else None
            if labels is not None:
                labels = labels.to(device=x.device, dtype=torch.int64).contiguous()
            self._generation += 1  # this pass records its activations in the workspace
            self._generation_recompute = recompute
            attn = None
            if want_attn:  # written by the forward as each block runs, in the layout of the saved probabilities
                ld_attn = (S + 7) // 8 * 8
                attn = tuple(torch.empty(B, H, S, ld_attn, dtype=torch.bfloat16, device=x.device) for _ in range(n))
                fwd = (lib().mb200_gptj_sched_forward_attn_recompute if recompute
                       else lib().mb200_gptj_sched_forward_attn)
                check(fwd(ctypes.byref(m), ops._ptr(x), ops._ptr(labels), ops._ptr(logits), ldv, ops._ptr(loss),
                          _ptr_array(attn), ld_attn, B, S, ops._ptr(ws), ws.numel(), ops._stream()))
            else:
                fwd = lib().mb200_gptj_sched_forward_recompute if recompute else lib().mb200_gptj_sched_forward
                check(fwd(ctypes.byref(m), ops._ptr(x), ops._ptr(labels), ops._ptr(logits), ldv, ops._ptr(loss), B, S,
                          ops._ptr(ws), ws.numel(), ops._stream()))
            hidden = None
            if want_hidden:  # copied out of the workspace, which the next forward overwrites
                hidden = tuple(torch.empty(B, S, d, dtype=torch.bfloat16, device=x.device)
                               for _ in range(len(self.transformer.h) + 1))
                copy = (lib().mb200_gptj_sched_hidden_states_recompute if recompute
                        else lib().mb200_gptj_sched_hidden_states)
                check(copy(ctypes.byref(m), _ptr_array(hidden), B, S, ops._ptr(ws), ws.numel(), ops._stream()))
            lg = logits.view(B, S, ldv)[..., :V] if logits is not None else None
            return (loss.squeeze(0) if loss is not None else None), lg, hidden, attn
        S_kv = cache.S_max if cache is not None else S
        # ONE grow-only inference workspace: a serving process sees many (B, prompt length, cache length) combinations,
        # and the C side only needs `nbytes` of scratch for the pass at hand (nothing survives between calls)
        nbytes = lib().mb200_gptj_sched_infer_workspace_bytes(ctypes.byref(m), B, S, S_kv)
        if nbytes == 0:
            raise MB200Error(lib().mb200_last_error().decode())
        ws = self._ws.get("infer")
        if ws is None or ws.numel() < nbytes:
            self._ws.pop("infer", None)
            ws = self._ws["infer"] = torch.empty(nbytes, dtype=torch.uint8, device=self._device)
        rows = B if last_only else B * S
        logits = torch.empty(rows, ldv, dtype=torch.bfloat16, device=x.device) if want_logits else None
        kv = (ops._ptr(cache.k), ops._ptr(cache.v), S_kv, cache.pos) if cache is not None else (None, None, 0, 0)
        hidden = attn = None
        if want_hidden:  # one buffer, entry l at l * B*S*d: each block writes its output into its entry
            hidden = torch.empty(len(self.transformer.h) + 1, B, S, d, dtype=torch.bfloat16, device=x.device)
        if want_attn:  # one buffer, entry l the [B, H, S, ld_attn] probabilities block l multiplies V with
            S_kv = S + (cache.pos if cache is not None else 0)
            ld_attn = (S_kv + 7) // 8 * 8
            attn = torch.empty(n, B, H, S, ld_attn, dtype=torch.bfloat16, device=x.device)
            check(lib().mb200_gptj_sched_infer_attn(
                ctypes.byref(m), ops._ptr(x), ops._ptr(logits), ldv, last_only, ops._ptr(hidden),
                hidden.stride(0) if hidden is not None else 0, _ptr_array(attn.unbind(0)), ld_attn, *kv, B, S,
                ops._ptr(ws), ws.numel(), ops._stream()))
            attn = attn.unbind(0)
        elif want_hidden:
            check(lib().mb200_gptj_sched_infer_hidden(
                ctypes.byref(m), ops._ptr(x), ops._ptr(logits), ldv, last_only, ops._ptr(hidden), hidden.stride(0), *kv,
                B, S, ops._ptr(ws), ws.numel(), ops._stream()))
        else:
            check(lib().mb200_gptj_sched_infer(
                ctypes.byref(m), ops._ptr(x), ops._ptr(logits), ldv, last_only, None, *kv, B, S, ops._ptr(ws),
                ws.numel(), ops._stream()))
        if cache is not None:
            cache.pos += S
        if hidden is not None:
            hidden = hidden.unbind(0)
        lg = logits.view(B, 1 if last_only else S, ldv)[..., :V] if logits is not None else None
        return None, lg, hidden, attn

    def _run_backward(self, shape, loss_scale, dhidden=(), dattn=(), dlogits=None):
        """loss_scale: the factor of the cross-entropy gradient, None when the forward had no labels; dhidden: the
        gradients of the hidden states the forward returned (each None or [B, S, d]); dattn: those of its attention
        buffers (each None or [B, H, S, S rounded up to 8]); dlogits: that of its logits (None or [B, S, V]), used as
        autograd delivers it. All None or empty runs the backward of the loss alone."""
        B, S, d = shape
        arena = self._arena
        dx = torch.empty(B, S, d, dtype=torch.bfloat16, device=self._device)
        ws, recompute = self._workspace_ex(B, S)
        if recompute != self._generation_recompute:
            raise MB200Error("backward called on a workspace of the other activation path (stored / recomputed) than "
                             "its forward's")

        def prep(gs):
            return [None if g is None else g.to(device=self._device, dtype=torch.bfloat16).contiguous() for g in gs]

        if dlogits is not None or loss_scale is None:  # the logits' gradient joins the CE term at the LM head
            dh, da = prep(dhidden), prep(dattn)
            g, comb, ld_g = None, None, 0
            if dlogits is not None:
                V = dlogits.shape[-1]
                # rows [B*S, V] of stride ld_g >= V: what autograd hands over, unless the loss's backward built a
                # broadcast or a layout no [B*S, V] view has; those are copied into fresh rows. The stride is read off
                # the 2-D view, because torch does not define the stride of a size-1 dim (S == 1).
                g = dlogits.to(device=self._device, dtype=torch.bfloat16).reshape(B * S, V)
                if g.stride(1) != 1 or (B * S > 1 and g.stride(0) < V):
                    g = torch.empty(B * S, V, dtype=torch.bfloat16, device=self._device).copy_(g)
                ld_g = g.stride(0) if B * S > 1 else V
                comb = torch.empty(B * S, self.ldv, dtype=torch.bfloat16, device=self._device)
            extra = (_ptr_array(dh) if any(t is not None for t in dh) else None,
                     _ptr_array(da) if any(t is not None for t in da) else None, (S + 7) // 8 * 8,
                     ops._ptr(g), ld_g, ops._ptr(comb))
            loss_scale = loss_scale or 0.0
            bwd = (lib().mb200_gptj_sched_backward_range_logits_recompute if recompute
                   else lib().mb200_gptj_sched_backward_range_logits)
        elif any(g is not None for g in dattn):  # hidden-state and attention gradients in one pass
            dh, da = prep(dhidden), prep(dattn)
            extra = (_ptr_array(dh) if any(g is not None for g in dh) else None, _ptr_array(da), (S + 7) // 8 * 8)
            bwd = (lib().mb200_gptj_sched_backward_range_attn_recompute if recompute
                   else lib().mb200_gptj_sched_backward_range_attn)
        elif any(g is not None for g in dhidden):
            dh = prep(dhidden)
            extra = (_ptr_array(dh),)
            bwd = (lib().mb200_gptj_sched_backward_range_hidden_recompute if recompute
                   else lib().mb200_gptj_sched_backward_range_hidden)
        else:
            extra = ()
            bwd = lib().mb200_gptj_sched_backward_range_recompute if recompute else lib().mb200_gptj_sched_backward_range
        accumulate = arena is not None and arena.grads_live()
        for hi, lo in (self._bwd_chunks or [(len(self.transformer.h), 0)]):
            check(bwd(ctypes.byref(self._cmodel_ex()[0]), ops._ptr(dx) if lo == 0 else None, *extra, loss_scale, hi, lo,
                      accumulate, B, S, ops._ptr(ws), ws.numel(), ops._stream()))
            if self._after_chunk is not None:
                self._after_chunk(hi, lo)
        if arena is not None and self._own_arena:
            arena.publish_grads()
        return dx

    def forward(self, input_ids=None, inputs_embeds=None, labels=None, use_cache=False, past_key_values=None,
                output_hidden_states=False, output_attentions=False, max_cache_len=None, **_unused):
        """GPTJForCausalLM.forward. Under grad, with trainable adapters or an input that requires grad and without
        use_cache, it runs the training pass, with or without labels: `.logits` then has a grad_fn, and the gradient of
        any loss on it joins the cross-entropy gradient at the LM head in the one backward pass (it reaches the
        adapters and inputs_embeds). That gradient is used as autograd delivers it: B200Engine's 1/grad_accum scaling
        applies to the cross-entropy term only, as it does for the hidden-state and attention gradients, and a loss
        that does not read `.loss` gets no cross-entropy term, under B200Engine as well. The backward
        of a loss on the logits takes one more bf16 [B*S, vocab rounded up to 64] buffer, the size of the logits.

        output_attentions=True adds `.attentions`: one bf16 [B, H, S, S_kv] tensor per
        block (S_kv = S, or pos0 + S over a KV cache), the probabilities the block multiplied V with, as
        `attn_weights.to(value.dtype)` of hf:gptj/modeling_gptj.py:145-146 returns them; entries above the causal
        diagonal are 0. They are views of buffers whose rows are S_kv rounded up to 8 long. In training they are outputs
        of the autograd function, and the gradient of a loss that reads them joins the one backward pass. Not covered:
        the gradient of the loss with respect to the attentions themselves (HF's retain_grad on an intermediate), and an
        output_attentions argument of Magma.forward, which the reference does not have. generate() never asks for
        them."""
        if (input_ids is None) == (inputs_embeds is None):
            raise ValueError("pass exactly one of input_ids / inputs_embeds")
        if inputs_embeds is None:
            inputs_embeds = self.transformer.wte(input_ids)
        B, S, _ = inputs_embeds.shape
        out = LMOutput(loss=None, logits=None, past_key_values=None, hidden_states=None)
        has_trainable = any(p.requires_grad for _, p in self.adapter_parameters()) or inputs_embeds.requires_grad
        if torch.is_grad_enabled() and has_trainable and not use_cache:
            anchor = next((p for _, p in self.adapter_parameters() if p.requires_grad), None)
            res = _LMTrainFn.apply(self, inputs_embeds, labels, anchor, output_hidden_states, output_attentions)
            out.loss, out.logits = res[0], res[1]
            nh = len(self.transformer.h) + 1 if output_hidden_states else 0
            if output_hidden_states:
                out.hidden_states = tuple(res[2 : 2 + nh])
            if output_attentions:
                out.attentions = tuple(a[..., :S] for a in res[2 + nh :])
            return out
        cache = past_key_values
        if use_cache and cache is None:
            S_max = max_cache_len or self.config.max_position_embeddings
            cfg = self.config
            cache = KVCache(cfg.num_layers, B, cfg.num_heads, S_max, cfg.hidden_size // cfg.num_heads, self._device)
        S_kv = S + (cache.pos if use_cache else 0)
        with torch.no_grad():
            loss, logits, hidden, attn = self._run_forward(inputs_embeds, labels, training=False,
                                                           cache=cache if use_cache else None, last_only=False,
                                                           want_hidden=output_hidden_states,
                                                           want_attn=output_attentions)
        out.loss, out.logits, out.hidden_states = loss, logits, hidden
        if output_attentions:
            out.attentions = tuple(a[..., :S_kv] for a in attn)
        out.past_key_values = cache if use_cache else None
        return out

    @torch.no_grad()
    def decode_step_dev(self, x, cache, pos_dev, logits):
        """One decode step (S = 1, last-position logits into the preallocated `logits` [B, ldv]) whose cache position is
        read from DEVICE memory (`pos_dev`, int32 [1]): no host-side argument changes from token to token, so
        sampling.generate captures the step once in a CUDA graph and replays it (mb200_gptj_sched_decode_step). The
        caller advances `pos_dev` (ops.decode_advance) and keeps `cache.pos` in step."""
        B, S, d = x.shape
        assert S == 1 and x.dtype == torch.bfloat16 and x.is_contiguous()
        m = self._cmodel_ex()[0]
        nbytes = lib().mb200_gptj_sched_infer_workspace_bytes(ctypes.byref(m), B, 1, cache.S_max)
        if nbytes == 0:
            raise MB200Error(lib().mb200_last_error().decode())
        ws = self._ws.get("infer")
        if ws is None or ws.numel() < nbytes:
            self._ws.pop("infer", None)
            ws = self._ws["infer"] = torch.empty(nbytes, dtype=torch.uint8, device=self._device)
        check(lib().mb200_gptj_sched_decode_step(ctypes.byref(m), ops._ptr(x), ops._ptr(logits), logits.stride(0),
                                                 ops._ptr(cache.k), ops._ptr(cache.v), cache.S_max, ops._ptr(pos_dev),
                                                 B, ops._ptr(ws), ws.numel(), ops._stream()))
        return logits

    @torch.no_grad()
    def decode_logits(self, inputs_embeds, cache):
        """Last-position logits only (what magma/sampling.py:92 consumes): the LM head runs on B rows, not B*S."""
        _, lg, _, _ = self._run_forward(inputs_embeds, None, training=False, cache=cache, last_only=True)
        return lg[:, 0, :]


LANGUAGE_MODELS = ["gptj"]


def gptj_config():
    """magma/language_model.py:12-24."""
    return GPTJConfig(vocab_size=50400, max_position_embeddings=2048, hidden_size=4096, num_layers=28, num_heads=16,
                      rotary_dim=64)


def get_gptj(gradient_checkpointing: bool = True, from_pretrained=False, config: GPTJConfig = None, device=None):
    """magma/language_model.py:27-45 — returns the (uninitialised-weights) LM. `gradient_checkpointing` is accepted
    for signature parity and ignored: the runtime stores every block's activations when they fit in free device memory
    (3.2 GiB at B=8, S=128) and otherwise keeps only each block's input and recomputes the block in the backward
    (13.6 GiB instead of 78.6 GiB at B=8, S=2048). Both compute the same results."""
    if from_pretrained:
        raise NotImplementedError("GPTJ pretrained not implemented")  # same behaviour as the reference (:41-42)
    cfg = config or gptj_config()
    cfg.gradient_checkpointing = gradient_checkpointing
    return B200GPTJForCausalLM(cfg, device=device)
