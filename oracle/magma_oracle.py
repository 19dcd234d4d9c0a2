"""TEST INFRASTRUCTURE — CPU oracle: a plain torch-fp32 / numpy restatement of the MAGMA hot path.

Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s cpu_baseline / `--impl reference` leg may import this
module, and only as the checker / reported CPU baseline. Nothing in `magma_b200/` imports it.

Parity status: the reference repository ships no tests or golden vectors, so this oracle is
pinned against *outputs of the reference itself*: `oracle/make_golden.py` imports
the reference's own `magma.{adapters,image_prefix,magma,utils,sampling}` from a reference checkout under shims
(oracle/ref_shims.py), with mainline HF `GPTJForCausalLM` / `CLIPVisionModelWithProjection` standing in for the
un-vendored transformers fork / openai-CLIP, and writes the fixtures in tests/golden/. tests/test_oracle_golden.py
checks every function below against those fixtures.

Each function cites the reference lines it restates (paths relative to the reference repository's root, or
`hf:` = site-packages/transformers).

Weight naming follows the reference state dict (magma/magma.py:52-53,143-149; HF GPT-J names for the LM,
openai/CLIP `.visual` names for the ViT):
  lm.transformer.wte.weight                      lm.transformer.h.{l}.ln_1.{weight,bias}
  lm.transformer.h.{l}.attn.{q,k,v,out}_proj.weight
  lm.transformer.h.{l}.mlp.0.fc_in.{weight,bias}  lm.transformer.h.{l}.mlp.0.fc_out.{weight,bias}
  lm.transformer.h.{l}.mlp.1.adapter.{0,2}.{weight,bias}          (adapter_type "normal", mlp)
  lm.transformer.h.{l}.attn.adapter.{0,2}.{weight,bias}           (attention adapters; attn weights move to
                                                                   attn.attn_block.* in the reference)
  lm.transformer.ln_f.{weight,bias}              lm.lm_head.{weight,bias}
  image_prefix.enc.*  image_prefix.proj.{weight,bias}  image_prefix.ln.{weight,bias}
"""
import math
from dataclasses import dataclass, field
from typing import Dict, Optional

import numpy as np
import torch
import torch.nn.functional as F


@dataclass
class OracleConfig:
    # language model (magma/language_model.py:12-24)
    d: int = 4096
    n_layer: int = 28
    n_head: int = 16
    rotary_dim: int = 64
    vocab: int = 50258  # len(tokenizer) after resize (magma/magma.py:50)
    ln_eps: float = 1e-5
    # adapter activation (magma/adapters.py:11: `activation: nn.Module = nn.ReLU`): "relu" (every shipped config) or
    # "gelu" = the tanh GeLU of the GPT-J MLP (NewGELUActivation / nn.GELU(approximate="tanh")) — north_star's variant
    adapter_act: str = "relu"
    # adapters (magma/magma.py:73-90): None | dict(adapter_type=..., downsample_factor=...)
    mlp_adapter: Optional[dict] = field(default_factory=lambda: {"adapter_type": "normal", "downsample_factor": 4})
    attn_adapter: Optional[dict] = None
    # image prefix (magma/image_prefix.py)
    image_seq_len: int = 2
    enc_out_dim: int = 768
    use_image_embed_layernorm: bool = True
    # ViT (openai/CLIP VisionTransformer; HF CLIPVisionModelWithProjection)
    vit_width: int = 1024
    vit_layers: int = 24
    vit_heads: int = 16
    vit_patch: int = 14
    vit_image: int = 224
    vit_mlp: int = 4096
    # conv trunk (openai/CLIP ModifiedResNet: RN50x16 = width 96, layers (6,8,18,8), 384 px; RN50x4 = 80, (4,6,10,6), 288)
    rn_width: int = 96
    rn_layers: tuple = (6, 8, 18, 8)
    rn_image: int = 384
    eos_token: int = 50256
    image_token: int = 50257


# ------------------------------------------------------------------------------------------------
# elementary functions
# ------------------------------------------------------------------------------------------------
def gelu_new(x):
    """hf:activations.py:59-66 (NewGELUActivation)."""
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * torch.pow(x, 3.0))))


def quick_gelu(x):
    """hf:activations.py QuickGELUActivation / openai-CLIP QuickGELU: x * sigmoid(1.702 x)."""
    return x * torch.sigmoid(1.702 * x)


def layer_norm(x, w, b, eps=1e-5):
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).mean(-1, keepdim=True)
    return (x - mu) / torch.sqrt(var + eps) * w + b


def rope_tables(positions, rotary_dim):
    """hf:gptj/modeling_gptj.py:47-50 — sin/cos of pos * 10000^(-2i/rotary_dim), i < rotary_dim/2."""
    inv_freq = 1.0 / (10000 ** (torch.arange(0, rotary_dim, 2, dtype=torch.int64) / rotary_dim))
    ang = positions.float()[:, None] * inv_freq[None, :]
    return torch.sin(ang), torch.cos(ang)


def apply_rope(x, sin, cos, rotary_dim):
    """hf:gptj/modeling_gptj.py:57-67,190-207 — rotate_every_two on the first rotary_dim features.
    x: [B, S, H, hd]; sin/cos: [S, rotary_dim/2]."""
    xr, xp = x[..., :rotary_dim], x[..., rotary_dim:]
    x1, x2 = xr[..., 0::2], xr[..., 1::2]
    s, c = sin[None, :, None, :], cos[None, :, None, :]
    o1 = x1 * c - x2 * s
    o2 = x2 * c + x1 * s
    out = torch.stack((o1, o2), dim=-1).flatten(-2)
    return torch.cat((out, xp), dim=-1)


# ------------------------------------------------------------------------------------------------
# adapters — magma/adapters.py
# ------------------------------------------------------------------------------------------------
def adapter_mlp(x, w, prefix, act="relu"):
    """The bottleneck only: Linear(d, d/f) -> act -> Linear(d/f, d)  (magma/adapters.py:16-25)."""
    keys = sorted(k for k in w if k.startswith(prefix + ".adapter."))
    has_ln = any(k.endswith("adapter.3.weight") for k in keys)  # add_layernorm shifts indices by one
    i0 = 1 if has_ln else 0
    h = x
    if has_ln:
        h = layer_norm(h, w[f"{prefix}.adapter.0.weight"], w[f"{prefix}.adapter.0.bias"])
    h = F.linear(h, w[f"{prefix}.adapter.{i0}.weight"], w[f"{prefix}.adapter.{i0}.bias"])
    h = torch.relu(h) if act == "relu" else gelu_new(h)
    return F.linear(h, w[f"{prefix}.adapter.{i0 + 2}.weight"], w[f"{prefix}.adapter.{i0 + 2}.bias"])


def adapter_forward(x, w, prefix, act="relu"):
    """Adapter.forward: self.adapter(x) + x  (magma/adapters.py:38-39)."""
    return adapter_mlp(x, w, prefix, act) + x


# ------------------------------------------------------------------------------------------------
# build_labels — magma/utils.py:334-364 (integer path, numpy, bit-exact)
# ------------------------------------------------------------------------------------------------
def build_labels(prefix_len: int, captions: np.ndarray, eos_token: int) -> np.ndarray:
    captions = np.asarray(captions, dtype=np.int64)
    b, s = captions.shape
    assert s >= prefix_len  # utils.py:349
    # utils.py:352-355, literally: cat(-100 * [b, L], captions[:, :-L]). NB for L == 0 the slice `[:, :-0]` is EMPTY,
    # so the reference returns a [b, 0] tensor; reproduced here because integer paths are bit-exact by contract.
    labels = np.concatenate([np.full((b, prefix_len), -100, dtype=np.int64), captions[:, : s - prefix_len if prefix_len else 0]],
                            axis=1)
    for i in range(b):  # utils.py:358-362: everything AFTER the first eos becomes -100 (the eos itself stays)
        hits = np.nonzero(labels[i] == eos_token)[0]
        if hits.size:
            labels[i, hits[0] + 1 :] = -100
    return labels


# ------------------------------------------------------------------------------------------------
# GPT-J — hf:gptj/modeling_gptj.py (stand-in for the fork's GPTNeo(jax=True, rotary=True))
# ------------------------------------------------------------------------------------------------
def gptj_attention(h, w, pre, cfg: OracleConfig, positions, past_kv=None):
    """hf:gptj/modeling_gptj.py:166-225 + _attn :129-151. h: LN1 output [B,S,d]. Returns (out, (k, v))."""
    B, S, d = h.shape
    H = cfg.n_head
    hd = d // H
    q = F.linear(h, w[f"{pre}.q_proj.weight"]).view(B, S, H, hd)
    k = F.linear(h, w[f"{pre}.k_proj.weight"]).view(B, S, H, hd)
    v = F.linear(h, w[f"{pre}.v_proj.weight"]).view(B, S, H, hd)
    sin, cos = rope_tables(positions, cfg.rotary_dim)
    q = apply_rope(q, sin, cos, cfg.rotary_dim).permute(0, 2, 1, 3)
    k = apply_rope(k, sin, cos, cfg.rotary_dim).permute(0, 2, 1, 3)
    v = v.permute(0, 2, 1, 3)
    if past_kv is not None:
        k = torch.cat((past_kv[0], k), dim=2)
        v = torch.cat((past_kv[1], v), dim=2)
    Sk = k.shape[2]
    att = torch.matmul(q.float(), k.float().transpose(-1, -2)) / math.sqrt(hd)  # :136-140 (fp32 scores)
    qpos = positions[:, None]
    kpos = torch.arange(Sk)[None, :]
    att = att.masked_fill(kpos > qpos, torch.finfo(att.dtype).min)  # causal mask (:502-505)
    att = torch.softmax(att, dim=-1).to(v.dtype)  # :145-146
    o = torch.matmul(att, v).permute(0, 2, 1, 3).reshape(B, S, d)  # :149, _merge_heads
    return F.linear(o, w[f"{pre}.out_proj.weight"]), (k, v)


def gptj_mlp(h, w, pre):
    """hf:gptj/modeling_gptj.py:374-379 (fc_in -> gelu_new -> fc_out; dropout 0)."""
    a = gelu_new(F.linear(h, w[f"{pre}.fc_in.weight"], w[f"{pre}.fc_in.bias"]))
    return F.linear(a, w[f"{pre}.fc_out.weight"], w[f"{pre}.fc_out.bias"])


def gptj_block(x, w, l, cfg: OracleConfig, positions, past_kv=None):
    """hf:gptj/modeling_gptj.py:400-413 (parallel residual) with the MAGMA adapter rewiring of
    magma/magma.py:128-169: mlp := Sequential(mlp, Adapter) / ParallelAdapter; attn := AdapterWrapper / Parallel."""
    p = f"lm.transformer.h.{l}"
    h = layer_norm(x, w[f"{p}.ln_1.weight"], w[f"{p}.ln_1.bias"], cfg.ln_eps)
    # attention branch
    if cfg.attn_adapter:
        kind = cfg.attn_adapter.get("adapter_type", "normal")
        inner = f"{p}.attn.attn_block" if kind == "normal" else f"{p}.attn.module"
        a, kv = gptj_attention(h, w, inner, cfg, positions, past_kv)
        if kind == "normal":  # AdapterWrapper.forward, adapters.py:109-116
            a = adapter_mlp(a, w, f"{p}.attn", cfg.adapter_act) + a
        else:  # ParallelAdapterWrapper.forward, adapters.py:85-92
            scale = w.get(f"{p}.attn.adapter_scale", torch.ones(1))
            a = a + adapter_mlp(h, w, f"{p}.attn", cfg.adapter_act) * scale
    else:
        a, kv = gptj_attention(h, w, f"{p}.attn", cfg, positions, past_kv)
    # mlp branch
    if cfg.mlp_adapter:
        kind = cfg.mlp_adapter.get("adapter_type", "normal")
        if kind == "normal":  # nn.Sequential(mlp, Adapter), magma.py:143-148
            m = gptj_mlp(h, w, f"{p}.mlp.0")
            m = adapter_forward(m, w, f"{p}.mlp.1", cfg.adapter_act)
        else:  # ParallelAdapter.forward, adapters.py:63-66
            scale = w.get(f"{p}.mlp.adapter_scale", torch.ones(1))
            m = gptj_mlp(h, w, f"{p}.mlp.module") + adapter_mlp(h, w, f"{p}.mlp", cfg.adapter_act) * scale
    else:
        m = gptj_mlp(h, w, f"{p}.mlp")
    return a + m + x, kv  # :411


def cross_entropy_shifted(logits, labels):
    """hf:loss/loss_utils.py:28-67 ForCausalLMLoss — fp32 logits, shift by one, ignore_index=-100, mean."""
    logits = logits.float()
    lab = F.pad(labels, (0, 1), value=-100)[:, 1:].contiguous()
    return F.cross_entropy(logits.view(-1, logits.shape[-1]), lab.view(-1), ignore_index=-100, reduction="mean")


def gptj_lm(inputs_embeds, w, cfg: OracleConfig, labels=None, past=None, return_hidden=False):
    """GPTJForCausalLM.forward with inputs_embeds (hf:gptj/modeling_gptj.py:487-530,567-639)."""
    B, S, _ = inputs_embeds.shape
    past_len = 0 if past is None else past[0][0].shape[2]
    positions = torch.arange(past_len, past_len + S)
    x = inputs_embeds
    new_past = []
    for l in range(cfg.n_layer):
        x, kv = gptj_block(x, w, l, cfg, positions, None if past is None else past[l])
        new_past.append(kv)
    x = layer_norm(x, w["lm.transformer.ln_f.weight"], w["lm.transformer.ln_f.bias"], cfg.ln_eps)
    logits = F.linear(x, w["lm.lm_head.weight"], w["lm.lm_head.bias"])
    loss = cross_entropy_shifted(logits, labels) if labels is not None else None
    if return_hidden:
        return loss, logits, new_past, x
    return loss, logits, new_past


# ------------------------------------------------------------------------------------------------
# CLIP ViT — openai/CLIP model.py VisionTransformer == hf:clip/modeling_clip.py vision tower
# ------------------------------------------------------------------------------------------------
def vit_forward(images, w, cfg: OracleConfig, pre="image_prefix.enc"):
    """conv1(stride=patch, no bias) -> [cls; patches] + pos -> ln_pre -> L x (x+attn(ln_1 x); x+mlp(ln_2 x))
    -> ln_post(x[:,0]) @ proj   (hf:clip/modeling_clip.py:138-219,282-386,647-694,1015-1069)."""
    B = images.shape[0]
    wd, H = cfg.vit_width, cfg.vit_heads
    hd = wd // H
    x = F.conv2d(images, w[f"{pre}.conv1.weight"], stride=cfg.vit_patch)  # [B, w, g, g]
    x = x.reshape(B, wd, -1).permute(0, 2, 1)
    cls = w[f"{pre}.class_embedding"].expand(B, 1, wd)
    x = torch.cat((cls, x), dim=1) + w[f"{pre}.positional_embedding"]
    x = layer_norm(x, w[f"{pre}.ln_pre.weight"], w[f"{pre}.ln_pre.bias"])
    T = x.shape[1]
    for i in range(cfg.vit_layers):
        p = f"{pre}.transformer.resblocks.{i}"
        h = layer_norm(x, w[f"{p}.ln_1.weight"], w[f"{p}.ln_1.bias"])
        qkv = F.linear(h, w[f"{p}.attn.in_proj_weight"], w[f"{p}.attn.in_proj_bias"])
        q, k, v = qkv.view(B, T, 3, H, hd).permute(2, 0, 3, 1, 4)
        att = torch.softmax(torch.matmul(q, k.transpose(-1, -2)) * hd**-0.5, dim=-1)
        o = torch.matmul(att, v).permute(0, 2, 1, 3).reshape(B, T, wd)
        x = x + F.linear(o, w[f"{p}.attn.out_proj.weight"], w[f"{p}.attn.out_proj.bias"])
        h = layer_norm(x, w[f"{p}.ln_2.weight"], w[f"{p}.ln_2.bias"])
        h = quick_gelu(F.linear(h, w[f"{p}.mlp.c_fc.weight"], w[f"{p}.mlp.c_fc.bias"]))
        x = x + F.linear(h, w[f"{p}.mlp.c_proj.weight"], w[f"{p}.mlp.c_proj.bias"])
    pooled = layer_norm(x[:, 0], w[f"{pre}.ln_post.weight"], w[f"{pre}.ln_post.bias"])
    return pooled @ w[f"{pre}.proj"]


# ------------------------------------------------------------------------------------------------
# CLIP ModifiedResNet (RN50x4 / RN50x16) with the attention pool replaced by "b d h w -> b (h w) d"
# (magma/image_encoders.py:65-74). PARITY UNPINNED: openai/CLIP is not vendored and nothing in this image carries its
# ModifiedResNet, so this follows the published architecture (CLIP model.py: Bottleneck / ModifiedResNet — 3-conv stem
# with stride-2 first conv and a 2x2 average pool, anti-aliased bottlenecks where the stride is an average pool after
# conv2 and in front of the 1x1 downsample conv, BatchNorm in eval mode) with its state-dict names.
# ------------------------------------------------------------------------------------------------
def _bn_eval(x, w, p, eps=1e-5, train=False, momentum=0.1):
    """nn.BatchNorm2d: eval mode (running statistics) or, with train=True, training mode — batch statistics, and the
    running_mean / running_var tensors in `w` are updated IN PLACE with `momentum` like the module does."""
    return F.batch_norm(x, w[f"{p}.running_mean"], w[f"{p}.running_var"], w[f"{p}.weight"], w[f"{p}.bias"], train,
                        momentum if train else 0.0, eps)


def resnet_block_specs(cfg: OracleConfig):
    """[(name, inplanes, planes, stride)] for layer1..layer4 (CLIP model.py ModifiedResNet._make_layer)."""
    specs, inpl = [], cfg.rn_width
    for li, n in enumerate(cfg.rn_layers):
        planes = cfg.rn_width * (2 ** li)
        for b in range(n):
            specs.append((f"layer{li + 1}.{b}", inpl, planes, 2 if (b == 0 and li > 0) else 1))
            inpl = planes * 4
    return specs


def resnet_forward(images, w, cfg: OracleConfig, pre="image_prefix.enc", train_bn=False, relu=F.relu, store=None):
    """train_bn=True: BatchNorm in training mode (the reference leaves the encoder in train() when
    freeze_img_encoder is false, magma/magma.py:98-100) — batch statistics, running statistics in `w` updated in place.
    `relu` lets a test substitute x * given_mask for the ReLUs (called in network order). `store` (default identity) is
    applied wherever the CUDA training path writes a tensor to HBM — convolution output, unit output, pooled tensors —
    so a test can pass a straight-through bf16 rounding and compare like with like: through ~18 BatchNorm units with
    batch statistics, bf16 storage alone moves the features by ~5 % relative to this function run in pure fp32."""
    t = train_bn
    st = store if store is not None else (lambda v: v)
    x = images

    def unit(v, conv_w, bn, stride=1, padding=0, act=True, res=None):
        z = st(F.conv2d(v, w[conv_w], stride=stride, padding=padding))
        y = _bn_eval(z, w, bn, train=t)
        if res is not None:
            y = y + res
        return st(relu(y) if act else y)

    for i, stride in ((1, 2), (2, 1), (3, 1)):  # stem
        x = unit(x, f"{pre}.conv{i}.weight", f"{pre}.bn{i}", stride=stride, padding=1)
    x = st(F.avg_pool2d(x, 2))
    for name, inpl, planes, stride in resnet_block_specs(cfg):
        p = f"{pre}.{name}"
        out = unit(x, f"{p}.conv1.weight", f"{p}.bn1")
        out = unit(out, f"{p}.conv2.weight", f"{p}.bn2", padding=1)
        if stride > 1:
            out = st(F.avg_pool2d(out, stride))
        idn = x
        if stride > 1 or inpl != planes * 4:
            idn = st(F.avg_pool2d(x, stride)) if stride > 1 else x
            idn = unit(idn, f"{p}.downsample.0.weight", f"{p}.downsample.1", act=False)
        x = unit(out, f"{p}.conv3.weight", f"{p}.bn3", res=idn)  # relu(bn3(conv3(out)) + identity)
    B, D = x.shape[:2]
    return x.reshape(B, D, -1).permute(0, 2, 1)  # image_encoders.py:71-73


def init_resnet_weights(cfg: OracleConfig, seed=0, pre="image_prefix.enc", dtype=torch.float32):
    """He-normal convs, BatchNorm statistics away from (0, 1) so that folding errors show."""
    g = torch.Generator().manual_seed(seed)
    w = {}

    def conv(name, co, ci, k):
        w[f"{name}.weight"] = (torch.randn(co, ci, k, k, generator=g) * math.sqrt(2.0 / (ci * k * k))).to(dtype)

    def bn(name, c, gain=1.0):
        w[f"{name}.weight"] = (gain * (1.0 + 0.1 * torch.randn(c, generator=g))).to(dtype)
        w[f"{name}.bias"] = (0.1 * torch.randn(c, generator=g)).to(dtype)
        w[f"{name}.running_mean"] = (0.1 * torch.randn(c, generator=g)).to(dtype)
        w[f"{name}.running_var"] = (1.0 + 0.2 * torch.rand(c, generator=g)).to(dtype)

    wd = cfg.rn_width
    conv(f"{pre}.conv1", wd // 2, 3, 3), bn(f"{pre}.bn1", wd // 2)
    conv(f"{pre}.conv2", wd // 2, wd // 2, 3), bn(f"{pre}.bn2", wd // 2)
    conv(f"{pre}.conv3", wd, wd // 2, 3), bn(f"{pre}.bn3", wd)
    for name, inpl, planes, stride in resnet_block_specs(cfg):
        p = f"{pre}.{name}"
        conv(f"{p}.conv1", planes, inpl, 1), bn(f"{p}.bn1", planes)
        conv(f"{p}.conv2", planes, planes, 3), bn(f"{p}.bn2", planes)
        conv(f"{p}.conv3", planes * 4, planes, 1), bn(f"{p}.bn3", planes * 4, gain=0.5)
        if stride > 1 or inpl != planes * 4:
            conv(f"{p}.downsample.0", planes * 4, inpl, 1), bn(f"{p}.downsample.1", planes * 4, gain=0.5)
    return w


# ------------------------------------------------------------------------------------------------
# ImagePrefix — magma/image_prefix.py:78-109
# ------------------------------------------------------------------------------------------------
def image_prefix_from_features(feats, w, cfg: OracleConfig, fixed_seq=False, dropout_mask=None, dropout_p=0.0):
    """feats = enc(x): [b,D] | [b,D,1,1] | [b,s,D]. proj -> (b (s d) -> b s d) -> dropout -> LN."""
    if feats.ndim == 4:
        feats = feats[:, :, 0, 0]  # image_prefix.py:86-87
    logits = F.linear(feats, w["image_prefix.proj.weight"], w["image_prefix.proj.bias"])  # :93
    if not fixed_seq:
        logits = logits.view(logits.shape[0], cfg.image_seq_len, cfg.d)  # :96-101
    if dropout_mask is not None:  # :104 (train mode; mask supplied so the oracle is deterministic)
        logits = logits * dropout_mask / (1.0 - dropout_p)
    if cfg.use_image_embed_layernorm:  # :106-107
        logits = layer_norm(logits, w["image_prefix.ln.weight"], w["image_prefix.ln.bias"])
    return logits


def image_prefix(images, w, cfg: OracleConfig, dropout_mask=None, dropout_p=0.0):
    return image_prefix_from_features(vit_forward(images, w, cfg), w, cfg, False, dropout_mask, dropout_p)


# ------------------------------------------------------------------------------------------------
# Magma.forward / embed — magma/magma.py:195-212,238-276
# ------------------------------------------------------------------------------------------------
def magma_forward(images, captions, w, cfg: OracleConfig, input_embeddings=None, dropout_mask=None, dropout_p=0.0):
    """Returns (loss, logits, labels). captions: int64 [B, S] padded to seq_len (magma.py:249-251)."""
    if input_embeddings is None:
        input_embeddings = image_prefix(images, w, cfg, dropout_mask, dropout_p)  # :253-254
    L = input_embeddings.shape[1]
    labels = torch.from_numpy(build_labels(L, captions.numpy(), cfg.eos_token))  # :255-257
    word = F.embedding(captions, w["lm.transformer.wte.weight"])  # :258
    x = torch.cat((input_embeddings, word[:, : captions.shape[1] - L, :]), dim=1)  # :261-267
    loss, logits, _ = gptj_lm(x, w, cfg, labels=labels)  # :270-274
    return loss, logits, labels


def magma_embed(inputs, w, cfg: OracleConfig):
    """Magma.embed (magma.py:195-212): 2-D -> word embedding, 4-D -> image prefix; cat on dim 1."""
    out = []
    for x in inputs:
        if x.ndim == 2:
            out.append(F.embedding(x, w["lm.transformer.wte.weight"]))
        elif x.ndim == 4:
            out.append(image_prefix(x.float(), w, cfg))
        else:
            raise ValueError(f"Expected 2d or 4d tensor, got {x.ndim}d")
    return torch.cat(out, dim=1)


# ------------------------------------------------------------------------------------------------
# sampling — magma/sampling.py
# ------------------------------------------------------------------------------------------------
def top_k_filter(logits, k):
    """sampling.py:22-30."""
    assert k > 0
    val, ind = torch.topk(logits, k)
    probs = torch.full_like(logits, float("-inf"))
    probs.scatter_(1, ind, val)
    return probs


def top_p_filter(logits, threshold=0.9):
    """sampling.py:7-19 — including its inverted-nucleus behaviour (cum_probs < 1 - threshold, shifted by one)."""
    sorted_logits, sorted_indices = torch.sort(logits, descending=True)
    cum_probs = torch.cumsum(F.softmax(sorted_logits, dim=-1), dim=-1)
    remove = cum_probs < (1 - threshold)
    remove[..., 1:] = remove[..., :-1].clone()
    remove[..., 0] = 0
    sorted_logits[remove] = float("-inf")
    return sorted_logits.scatter(1, sorted_indices, sorted_logits)


def generate_greedy(embeddings, w, cfg: OracleConfig, max_steps):
    """sampling.py:43-121 at temperature 0: prefill with inputs_embeds, then one token at a time with the
    KV cache; argmax over fp32 last-token logits (:92,97); stop when every row emits eos (:109)."""
    b, s, _ = embeddings.shape
    out = torch.full((b, s), cfg.image_token, dtype=torch.long)  # :75
    past = None
    for i in range(max_steps):
        if i == 0:
            _, logits, past = gptj_lm(embeddings, w, cfg, past=None)
        else:
            x = F.embedding(out[:, -1:], w["lm.transformer.wte.weight"])
            _, logits, past = gptj_lm(x, w, cfg, past=past)
        nxt = torch.argmax(logits[:, -1, :].float(), dim=-1, keepdim=True)
        out = torch.cat((out, nxt), dim=-1)
        if (nxt == cfg.eos_token).all():
            break
    return out


def remove_tokens_after_eos(tensor, eos_token, image_token):
    """sampling.py:33-40."""
    t = tensor.clone()
    idx = (t == eos_token).nonzero()
    if idx.any():
        t[idx[0] :] = eos_token
    return [i for i in t.tolist() if i != image_token and i != eos_token]


# ------------------------------------------------------------------------------------------------
# synthetic weights: normal(0, 0.02) linears, LN 1/0, adapters per adapters.py:28-36
# ------------------------------------------------------------------------------------------------
def init_weights(cfg: OracleConfig, seed=0, with_vit=True, dtype=torch.float32) -> Dict[str, torch.Tensor]:
    g = torch.Generator().manual_seed(seed)
    w = {}

    def normal(*shape, std=0.02):
        return (torch.randn(*shape, generator=g) * std).to(dtype)

    def adapter(prefix, f, std=1e-3):
        r = cfg.d // f
        for idx, shape in ((0, (r, cfg.d)), (2, (cfg.d, r))):
            w[f"{prefix}.adapter.{idx}.weight"] = torch.clamp(normal(*shape, std=std), -2 * std, 2 * std)
            w[f"{prefix}.adapter.{idx}.bias"] = torch.clamp(normal(shape[0], std=std), -2 * std, 2 * std)

    d = cfg.d
    w["lm.transformer.wte.weight"] = normal(cfg.vocab, d)
    for l in range(cfg.n_layer):
        p = f"lm.transformer.h.{l}"
        w[f"{p}.ln_1.weight"] = (1.0 + normal(d, std=0.02)).to(dtype)
        w[f"{p}.ln_1.bias"] = normal(d)
        attn = f"{p}.attn"
        if cfg.attn_adapter:
            kind = cfg.attn_adapter.get("adapter_type", "normal")
            adapter(f"{p}.attn", cfg.attn_adapter.get("downsample_factor", 4))
            attn = f"{p}.attn.attn_block" if kind == "normal" else f"{p}.attn.module"
        for n in ("q_proj", "k_proj", "v_proj", "out_proj"):
            w[f"{attn}.{n}.weight"] = normal(d, d)
        mlp = f"{p}.mlp"
        if cfg.mlp_adapter:
            kind = cfg.mlp_adapter.get("adapter_type", "normal")
            if kind == "normal":
                mlp = f"{p}.mlp.0"
                adapter(f"{p}.mlp.1", cfg.mlp_adapter.get("downsample_factor", 4))
            else:
                mlp = f"{p}.mlp.module"
                adapter(f"{p}.mlp", cfg.mlp_adapter.get("downsample_factor", 4))
        w[f"{mlp}.fc_in.weight"] = normal(4 * d, d)
        w[f"{mlp}.fc_in.bias"] = normal(4 * d)
        w[f"{mlp}.fc_out.weight"] = normal(d, 4 * d)
        w[f"{mlp}.fc_out.bias"] = normal(d)
    w["lm.transformer.ln_f.weight"] = (1.0 + normal(d)).to(dtype)
    w["lm.transformer.ln_f.bias"] = normal(d)
    w["lm.lm_head.weight"] = normal(cfg.vocab, d)
    w["lm.lm_head.bias"] = normal(cfg.vocab)
    w["image_prefix.proj.weight"] = normal(cfg.d * cfg.image_seq_len, cfg.enc_out_dim)
    w["image_prefix.proj.bias"] = normal(cfg.d * cfg.image_seq_len)
    w["image_prefix.ln.weight"] = (1.0 + normal(d)).to(dtype)
    w["image_prefix.ln.bias"] = normal(d)
    if with_vit:
        e, wd = "image_prefix.enc", cfg.vit_width
        T = (cfg.vit_image // cfg.vit_patch) ** 2 + 1
        w[f"{e}.conv1.weight"] = normal(wd, 3, cfg.vit_patch, cfg.vit_patch)
        w[f"{e}.class_embedding"] = normal(wd)
        w[f"{e}.positional_embedding"] = normal(T, wd)
        for n in ("ln_pre", "ln_post"):
            w[f"{e}.{n}.weight"] = (1.0 + normal(wd)).to(dtype)
            w[f"{e}.{n}.bias"] = normal(wd)
        for i in range(cfg.vit_layers):
            p = f"{e}.transformer.resblocks.{i}"
            for n in ("ln_1", "ln_2"):
                w[f"{p}.{n}.weight"] = (1.0 + normal(wd)).to(dtype)
                w[f"{p}.{n}.bias"] = normal(wd)
            w[f"{p}.attn.in_proj_weight"] = normal(3 * wd, wd)
            w[f"{p}.attn.in_proj_bias"] = normal(3 * wd)
            w[f"{p}.attn.out_proj.weight"] = normal(wd, wd)
            w[f"{p}.attn.out_proj.bias"] = normal(wd)
            w[f"{p}.mlp.c_fc.weight"] = normal(cfg.vit_mlp, wd)
            w[f"{p}.mlp.c_fc.bias"] = normal(cfg.vit_mlp)
            w[f"{p}.mlp.c_proj.weight"] = normal(wd, cfg.vit_mlp)
            w[f"{p}.mlp.c_proj.bias"] = normal(wd)
        w[f"{e}.proj"] = normal(wd, cfg.enc_out_dim)
    return w


def synthetic_batch(cfg: OracleConfig, B, S, seed=1234, prefix_len=None):
    """Synthetic batch: images ~ N(0,1); captions randint(0, 50256) with per-row length U[S/4, S-L], EOS padded
    (mimics tokenizer(..., padding='max_length') with pad=eos; datasets/dataset.py:136-142)."""
    g = torch.Generator().manual_seed(seed)
    L = cfg.image_seq_len if prefix_len is None else prefix_len
    images = torch.randn(B, 3, cfg.vit_image, cfg.vit_image, generator=g)
    hi = min(cfg.eos_token, cfg.vocab - 1)
    captions = torch.randint(0, hi, (B, S), generator=g)
    lo_len, hi_len = max(1, S // 4), max(2, S - L)
    lens = torch.randint(lo_len, hi_len + 1, (B,), generator=g)
    pos = torch.arange(S)[None, :]
    captions = torch.where(pos >= lens[:, None], torch.full_like(captions, cfg.eos_token), captions)
    return images, captions
