"""Dry run of the product's host-only schedule files on the CPU.

magma_b200/csrc/vit_sched.cu (ViT inference forward, training forward + backward) contains no kernels: it carves a workspace and issues
primitive C-ABI operators. Here the SAME source file is compiled as plain C++ against oracle/cabi_emul.cpp (a scalar
CPU emulation of those primitives with bf16 storage, test infrastructure only) and run on CPU tensors, so every
pointer offset, leading dimension, operand major, batch stride and accumulate flag of the schedule is held to torch
autograd of the oracle (oracle/magma_oracle.py::vit_forward). What this cannot check is the CUDA kernels themselves —
that is the job of the `-m gpu` tests."""
import ctypes

import pytest
import torch

from magma_b200._lib import VitGradsC, VitLayerC, VitLayerGradsC, VitModelC
from oracle import magma_oracle as O

LAYER_KEYS = [("ln1_g", "ln_1.weight"), ("ln1_b", "ln_1.bias"), ("w_qkv", "attn.in_proj_weight"),
              ("b_qkv", "attn.in_proj_bias"), ("w_out", "attn.out_proj.weight"), ("b_out", "attn.out_proj.bias"),
              ("ln2_g", "ln_2.weight"), ("ln2_b", "ln_2.bias"), ("w_fc", "mlp.c_fc.weight"), ("b_fc", "mlp.c_fc.bias"),
              ("w_proj", "mlp.c_proj.weight"), ("b_proj", "mlp.c_proj.bias")]
TOP_KEYS = [("cls", "class_embedding"), ("pos", "positional_embedding"), ("ln_pre_g", "ln_pre.weight"),
            ("ln_pre_b", "ln_pre.bias"), ("ln_post_g", "ln_post.weight"), ("ln_post_b", "ln_post.bias")]


@pytest.fixture(scope="module")
def emul():
    from oracle import build_emul

    L = ctypes.CDLL(build_emul.build())
    L.mb200_last_error.restype = ctypes.c_char_p
    L.mb200_vit_train_workspace_bytes.restype = ctypes.c_size_t
    return L


def rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-12)).item()


def ptr(t):
    return ctypes.c_void_p(t.data_ptr())


def make_case(seed=0, B=3):
    cfg = O.OracleConfig(d=64, n_layer=1, n_head=2, rotary_dim=8, vocab=64, enc_out_dim=48, vit_width=64, vit_layers=2,
                         vit_heads=4, vit_patch=8, vit_image=32, vit_mlp=128)
    pre = "image_prefix.enc"
    w = {k: v for k, v in O.init_weights(cfg, seed=seed).items() if k.startswith(pre)}
    g = torch.Generator().manual_seed(seed + 1)
    for k in w:  # larger weights than the 0.02 init so every gradient is well above bf16 noise
        if k.endswith(("in_proj_weight", "out_proj.weight", "c_fc.weight", "c_proj.weight", "conv1.weight", ".proj")):
            w[k] = w[k] * 4
    w16 = {k: v.to(torch.bfloat16) for k, v in w.items()}
    images = torch.randn(B, 3, cfg.vit_image, cfg.vit_image, generator=g).to(torch.bfloat16)
    dfeats = torch.randn(B, cfg.enc_out_dim, generator=g).to(torch.bfloat16)
    return cfg, pre, w16, images, dfeats


def c_model(cfg, pre, w16, keep):
    K = 3 * cfg.vit_patch ** 2
    ldk = (K + 7) // 8 * 8
    conv = torch.zeros(cfg.vit_width, ldk, dtype=torch.bfloat16)
    conv[:, :K] = w16[f"{pre}.conv1.weight"].reshape(cfg.vit_width, K)
    proj_t = w16[f"{pre}.proj"].t().contiguous()
    layers = (VitLayerC * cfg.vit_layers)()
    for i in range(cfg.vit_layers):
        for f, k in LAYER_KEYS:
            setattr(layers[i], f, w16[f"{pre}.transformer.resblocks.{i}.{k}"].data_ptr())
    m = VitModelC()
    m.n_layer, m.width, m.n_head, m.patch = cfg.vit_layers, cfg.vit_width, cfg.vit_heads, cfg.vit_patch
    m.image, m.mlp, m.out_dim = cfg.vit_image, cfg.vit_mlp, cfg.enc_out_dim
    m.w_conv, m.ld_conv = conv.data_ptr(), ldk
    for f, k in TOP_KEYS:
        setattr(m, f, w16[f"{pre}.{k}"].data_ptr())
    m.proj_t = proj_t.data_ptr()
    m.layers = ctypes.cast(layers, ctypes.POINTER(VitLayerC))
    keep += [conv, proj_t, layers]
    return m


def c_grads(cfg, pre, w16, keep, fill=0.0):
    """fp32 gradient buffers with each parameter's own shape; returns (struct, {param name: tensor})."""
    out = {}

    def buf(name):
        out[name] = torch.full(w16[name].shape, fill, dtype=torch.float32)
        return out[name].data_ptr()

    lg = (VitLayerGradsC * cfg.vit_layers)()
    for i in range(cfg.vit_layers):
        for f, k in LAYER_KEYS:
            setattr(lg[i], f, buf(f"{pre}.transformer.resblocks.{i}.{k}"))
    G = VitGradsC()
    G.w_conv = buf(f"{pre}.conv1.weight")
    for f, k in TOP_KEYS:
        setattr(G, f, buf(f"{pre}.{k}"))
    G.proj = buf(f"{pre}.proj")
    G.layers = ctypes.cast(lg, ctypes.POINTER(VitLayerGradsC))
    keep.append(lg)
    return G, out


def oracle_grads(cfg, pre, w16, images, dfeats):
    wf = {k: v.float().requires_grad_(True) for k, v in w16.items()}
    feats = O.vit_forward(images.float(), wf, cfg, pre=pre)
    feats.backward(dfeats.float())
    return feats.detach(), {k: v.grad for k, v in wf.items()}


def run_emul(L, cfg, pre, w16, images, dfeats, accumulate=0, fill=0.0):
    keep = []
    m = c_model(cfg, pre, w16, keep)
    B = images.shape[0]
    n = L.mb200_vit_train_workspace_bytes(ctypes.byref(m), B)
    assert n > 0
    ws = torch.empty(n + 256, dtype=torch.uint8)
    off = (-ws.data_ptr()) % 256  # the product hands the schedule a 256-byte aligned torch allocation
    wsp = ctypes.c_void_p(ws.data_ptr() + off)
    feats = torch.empty(B, cfg.enc_out_dim, dtype=torch.bfloat16)
    rc = L.mb200_vit_forward_train(ctypes.byref(m), ptr(images), ptr(feats), B, wsp, ctypes.c_size_t(n), None)
    assert rc == 0, L.mb200_last_error().decode()
    G, grads = c_grads(cfg, pre, w16, keep, fill=fill)
    rc = L.mb200_vit_backward(ctypes.byref(m), ctypes.byref(G), ptr(dfeats), accumulate, B, wsp, ctypes.c_size_t(n), None)
    assert rc == 0, L.mb200_last_error().decode()
    return feats, grads


def test_vit_train_schedule_matches_oracle_autograd(emul):
    cfg, pre, w16, images, dfeats = make_case()
    feats_o, grads_o = oracle_grads(cfg, pre, w16, images, dfeats)
    feats, grads = run_emul(emul, cfg, pre, w16, images, dfeats)
    assert rel(feats, feats_o) < 2e-2
    assert set(grads) == set(grads_o)
    bad = {k: round(rel(g, grads_o[k]), 4) for k, g in grads.items() if rel(g, grads_o[k]) > 2.5e-2}
    assert not bad, bad  # bf16 activations vs the fp32 oracle


def test_vit_train_schedule_accumulates(emul):
    """accumulate != 0 adds into every gradient buffer (gradient accumulation, train_loop.py:10-19)."""
    cfg, pre, w16, images, dfeats = make_case(seed=3, B=2)
    _, g0 = run_emul(emul, cfg, pre, w16, images, dfeats, accumulate=0, fill=7.0)   # overwrite: the 7s must vanish
    _, g1 = run_emul(emul, cfg, pre, w16, images, dfeats, accumulate=1, fill=0.5)
    for k in g0:
        assert torch.allclose(g1[k], g0[k] + 0.5, rtol=1e-4, atol=1e-4), k


def test_vit_train_schedule_rejects_a_small_workspace(emul):
    cfg, pre, w16, images, dfeats = make_case(B=1)
    keep = []
    m = c_model(cfg, pre, w16, keep)
    ws = torch.empty(1024, dtype=torch.uint8)
    feats = torch.empty(1, cfg.enc_out_dim, dtype=torch.bfloat16)
    rc = emul.mb200_vit_forward_train(ctypes.byref(m), ptr(images), ptr(feats), 1, ptr(ws), ctypes.c_size_t(1024), None)
    assert rc != 0 and b"workspace too small" in emul.mb200_last_error()


# ------------------------------------------------------------------------------------------------------------------
# csrc/gptj_sched.cu — GPT-J + adapters, every adapter form of the reference (magma/adapters.py, magma/magma.py:102-174)
# ------------------------------------------------------------------------------------------------------------------
from magma_b200._lib import AdapterExC, GptjLayerExC, GptjModelExC  # noqa: E402

ADAPTER_KIND = {None: 0, "normal": 1, "parallel": 2, "scaled_parallel": 2}


def lm_case(mlp, attn, mlp_ln=False, attn_ln=False, seed=0, B=2, S=12):
    """Oracle weights for a tiny GPT-J with the requested adapter forms; adapter weights O(0.05) with the bottleneck
    biases at +-3 so every ReLU is decided (bf16 and fp32 agree on the mask), LN / scale parameters non-trivial."""
    cfg = O.OracleConfig(d=64, n_layer=2, n_head=4, rotary_dim=8, vocab=96,
                         mlp_adapter=None if mlp is None else {"adapter_type": mlp, "downsample_factor": 4},
                         attn_adapter=None if attn is None else {"adapter_type": attn, "downsample_factor": 8})
    w = {k: v for k, v in O.init_weights(cfg, seed=seed, with_vit=False).items() if k.startswith("lm.")}
    g = torch.Generator().manual_seed(seed + 7)
    for k in list(w):
        if ".adapter." in k:
            w[k] = torch.randn(w[k].shape, generator=g) * (0.05 if k.endswith("weight") else 0.02)
            if k.endswith("adapter.0.bias"):
                w[k] = torch.where(torch.rand(w[k].shape, generator=g) < 0.5, -3.0, 3.0) + 0.02 * torch.randn(w[k].shape, generator=g)
    for l in range(cfg.n_layer):
        for loc, kind, ln in (("mlp", mlp, mlp_ln), ("attn", attn, attn_ln)):
            if kind is None:
                continue
            pre = f"lm.transformer.h.{l}.{loc}" + (".1" if (loc == "mlp" and kind == "normal") else "")
            if ln:  # add_layernorm shifts the Sequential indices by one (adapters.py:16-25)
                for i, j in ((2, 3), (0, 1)):
                    for s in ("weight", "bias"):
                        w[f"{pre}.adapter.{j}.{s}"] = w.pop(f"{pre}.adapter.{i}.{s}")
                w[f"{pre}.adapter.0.weight"] = 1.0 + 0.1 * torch.randn(cfg.d, generator=g)
                w[f"{pre}.adapter.0.bias"] = 0.1 * torch.randn(cfg.d, generator=g)
            if kind == "scaled_parallel":
                w[f"lm.transformer.h.{l}.{loc}.adapter_scale"] = torch.tensor([0.7 + 0.2 * l])
    w16 = {k: v.to(torch.bfloat16) for k, v in w.items()}
    x = (torch.randn(B, S, cfg.d, generator=g) * 0.5).to(torch.bfloat16)
    labels = torch.randint(0, cfg.vocab, (B, S), generator=g)
    labels[:, :2] = -100
    labels[0, 7:] = -100
    return cfg, w16, x, labels


def c_lm_model(cfg, w16, keep, with_grads=True):
    """mb200_gptj_model_ex over the oracle-named bf16 tensors; returns (struct, {param name: fp32 grad tensor})."""
    grads = {}
    w32 = {}

    def adapter(prefix, kind):
        a = AdapterExC()
        if kind is None:
            return a
        ln = f"{prefix}.adapter.3.weight" in w16
        i0 = 1 if ln else 0
        names = {"wd": f"{prefix}.adapter.{i0}.weight", "bd": f"{prefix}.adapter.{i0}.bias",
                 "wu": f"{prefix}.adapter.{i0 + 2}.weight", "bu": f"{prefix}.adapter.{i0 + 2}.bias"}
        if ln:
            names.update({"ln_g": f"{prefix}.adapter.0.weight", "ln_b": f"{prefix}.adapter.0.bias"})
        for f, n in names.items():
            setattr(a, f, w16[n].data_ptr())
            if with_grads:
                grads[n] = torch.full(w16[n].shape, 5.0, dtype=torch.float32)
                setattr(a, "g_" + f, grads[n].data_ptr())
        sk = prefix.rsplit(".1", 1)[0] + ".adapter_scale" if prefix.endswith(".1") else prefix + ".adapter_scale"
        if sk in w16:  # the scale is read as fp32 from the arena's master copy
            w32[sk] = w16[sk].float().contiguous()
            a.scale = w32[sk].data_ptr()
            if with_grads:
                grads[sk] = torch.full((1,), 5.0, dtype=torch.float32)
                a.g_scale = grads[sk].data_ptr()
        return a

    mk = cfg.mlp_adapter["adapter_type"] if cfg.mlp_adapter else None
    ak = cfg.attn_adapter["adapter_type"] if cfg.attn_adapter else None
    layers = (GptjLayerExC * cfg.n_layer)()
    for l in range(cfg.n_layer):
        p = f"lm.transformer.h.{l}"
        attn = f"{p}.attn" + ("" if ak is None else (".attn_block" if ak == "normal" else ".module"))
        mlp = f"{p}.mlp" + ("" if mk is None else (".0" if mk == "normal" else ".module"))
        qkv = torch.cat([w16[f"{attn}.{n}.weight"] for n in ("q_proj", "k_proj", "v_proj")], 0).contiguous()
        keep.append(qkv)
        L = layers[l]
        L.ln1_g, L.ln1_b = w16[f"{p}.ln_1.weight"].data_ptr(), w16[f"{p}.ln_1.bias"].data_ptr()
        L.w_qkv, L.w_out = qkv.data_ptr(), w16[f"{attn}.out_proj.weight"].data_ptr()
        L.w_fc_in, L.b_fc_in = w16[f"{mlp}.fc_in.weight"].data_ptr(), w16[f"{mlp}.fc_in.bias"].data_ptr()
        L.w_fc_out, L.b_fc_out = w16[f"{mlp}.fc_out.weight"].data_ptr(), w16[f"{mlp}.fc_out.bias"].data_ptr()
        L.mlp_ad = adapter(f"{p}.mlp.1" if mk == "normal" else f"{p}.mlp", mk)
        L.attn_ad = adapter(f"{p}.attn", ak)
    m = GptjModelExC()
    m.n_layer, m.d, m.n_head, m.rotary_dim, m.vocab, m.d_ff = cfg.n_layer, cfg.d, cfg.n_head, cfg.rotary_dim, cfg.vocab, 4 * cfg.d
    m.mlp_adapter, m.attn_adapter = ADAPTER_KIND[mk], ADAPTER_KIND[ak]
    m.mlp_adapter_r = cfg.d // cfg.mlp_adapter["downsample_factor"] if mk else 0
    m.attn_adapter_r = cfg.d // cfg.attn_adapter["downsample_factor"] if ak else 0
    m.ln_eps = cfg.ln_eps
    m.layers = ctypes.cast(layers, ctypes.POINTER(GptjLayerExC))
    m.lnf_g, m.lnf_b = w16["lm.transformer.ln_f.weight"].data_ptr(), w16["lm.transformer.ln_f.bias"].data_ptr()
    m.w_lm, m.b_lm = w16["lm.lm_head.weight"].data_ptr(), w16["lm.lm_head.bias"].data_ptr()
    keep += [layers, w32]
    return m, grads


def run_lm_emul(L, cfg, w16, x, labels, accumulate=0):
    keep = []
    m, grads = c_lm_model(cfg, w16, keep)
    B, S = labels.shape
    L.mb200_gptj_sched_workspace_bytes.restype = ctypes.c_size_t
    n = L.mb200_gptj_sched_workspace_bytes(ctypes.byref(m), B, S)
    assert n > 0, L.mb200_last_error().decode()
    ws = torch.empty(n + 256, dtype=torch.uint8)
    wsp = ctypes.c_void_p(ws.data_ptr() + (-ws.data_ptr()) % 256)
    ldv = (cfg.vocab + 63) // 64 * 64
    logits = torch.zeros(B * S, ldv, dtype=torch.bfloat16)
    loss = torch.zeros(1, dtype=torch.float32)
    rc = L.mb200_gptj_sched_forward(ctypes.byref(m), ptr(x), ptr(labels), ptr(logits), ctypes.c_int64(ldv), ptr(loss), B, S,
                                    wsp, ctypes.c_size_t(n), None)
    assert rc == 0, L.mb200_last_error().decode()
    dx = torch.empty_like(x)
    rc = L.mb200_gptj_sched_backward(ctypes.byref(m), ptr(dx), ctypes.c_float(1.0), accumulate, B, S, wsp,
                                     ctypes.c_size_t(n), None)
    assert rc == 0, L.mb200_last_error().decode()
    return float(loss), logits[:, : cfg.vocab].reshape(B, S, cfg.vocab), dx, grads


FORMS = [
    (None, None, False, False),                                  # plain GPT-J
    ("normal", None, False, False),                              # MAGMA_v1.yml
    ("normal", "normal", False, False),                          # MAGMA_v2.yml
    ("parallel", "parallel", False, False),
    ("normal", "normal", True, True),                            # add_layernorm (adapters.py:16-17)
    ("scaled_parallel", "scaled_parallel", False, False),        # adapter_scale (adapters.py:57-61)
    ("scaled_parallel", "normal", True, True),
    ("parallel", "scaled_parallel", True, False),
]


@pytest.mark.parametrize("mlp,attn,mlp_ln,attn_ln", FORMS)
def test_gptj_schedule_matches_oracle_autograd_for_every_adapter_form(emul, mlp, attn, mlp_ln, attn_ln):
    cfg, w16, x, labels = lm_case(mlp, attn, mlp_ln, attn_ln)
    params = {k: v.float().requires_grad_(".adapter" in k) for k, v in w16.items()}
    xf = x.float().requires_grad_(True)
    loss_o, logits_o, _ = O.gptj_lm(xf, params, cfg, labels=labels)
    loss_o.backward()
    loss, logits, dx, grads = run_lm_emul(emul, cfg, w16, x, labels)
    assert abs(loss - float(loss_o.detach())) < 2e-2
    assert rel(logits, logits_o.detach()) < 3e-2
    assert rel(dx, xf.grad) < 2.5e-2
    want = {k for k, v in params.items() if v.requires_grad}
    assert set(grads) == want
    bad = {k: round(rel(g, params[k].grad), 4) for k, g in grads.items() if rel(g, params[k].grad) > 2.5e-2}
    assert not bad, bad


def test_gptj_schedule_accumulates_and_validates(emul):
    cfg, w16, x, labels = lm_case("scaled_parallel", "normal", True, True, seed=2)
    _, _, _, g0 = run_lm_emul(emul, cfg, w16, x, labels, accumulate=0)   # overwrite: the 5.0 fill must vanish
    _, _, _, g1 = run_lm_emul(emul, cfg, w16, x, labels, accumulate=1)   # add onto the 5.0 fill
    for k in g0:
        assert torch.allclose(g1[k], g0[k] + 5.0, rtol=1e-4, atol=1e-4), k
    # adapter_scale on a "normal" adapter is rejected (the reference has no such form)
    keep = []
    m, _ = c_lm_model(cfg, w16, keep)
    one = torch.ones(1)
    layers = ctypes.cast(m.layers, ctypes.POINTER(GptjLayerExC))
    layers[0].attn_ad.scale = one.data_ptr()
    emul.mb200_gptj_sched_workspace_bytes.restype = ctypes.c_size_t
    assert emul.mb200_gptj_sched_workspace_bytes(ctypes.byref(m), 2, 12) == 0
    assert b"parallel adapter forms only" in emul.mb200_last_error()


def test_gptj_schedule_fused_attention_tile_and_chunked_backward(emul):
    """head_dim 64 takes the fused single-tile attention entry points (mb200_attn_fwd_tile / bwd_tile, emulated per their
    documented semantics); the backward issued in two layer ranges (what B200Engine does to overlap the gradient exchange)
    gives the same gradients as one call."""
    cfg = O.OracleConfig(d=128, n_layer=2, n_head=2, rotary_dim=16, vocab=96,
                         mlp_adapter={"adapter_type": "normal", "downsample_factor": 4}, attn_adapter=None)
    w = {k: v for k, v in O.init_weights(cfg, seed=1, with_vit=False).items() if k.startswith("lm.")}
    g = torch.Generator().manual_seed(5)
    for k in list(w):
        if ".adapter." in k:
            w[k] = torch.randn(w[k].shape, generator=g) * (0.05 if k.endswith("weight") else 0.02)
            if k.endswith("adapter.0.bias"):
                w[k] = torch.where(torch.rand(w[k].shape, generator=g) < 0.5, -3.0, 3.0)
    w16 = {k: v.to(torch.bfloat16) for k, v in w.items()}
    B, S = 2, 10
    x = (torch.randn(B, S, cfg.d, generator=g) * 0.5).to(torch.bfloat16)
    labels = torch.randint(0, cfg.vocab, (B, S), generator=g)
    params = {k: v.float().requires_grad_(".adapter" in k) for k, v in w16.items()}
    xf = x.float().requires_grad_(True)
    loss_o, logits_o, _ = O.gptj_lm(xf, params, cfg, labels=labels)
    loss_o.backward()
    loss, logits, dx, grads = run_lm_emul(emul, cfg, w16, x, labels)
    assert abs(loss - float(loss_o.detach())) < 2e-2 and rel(logits, logits_o.detach()) < 3e-2
    assert rel(dx, xf.grad) < 2.5e-2
    assert max(rel(gr, params[k].grad) for k, gr in grads.items()) < 2.5e-2
    # the same backward in two ranges: [2,1) then [1,0)
    keep = []
    m, grads2 = c_lm_model(cfg, w16, keep)
    n = emul.mb200_gptj_sched_workspace_bytes(ctypes.byref(m), B, S)
    ws = torch.empty(n + 256, dtype=torch.uint8)
    wsp = ctypes.c_void_p(ws.data_ptr() + (-ws.data_ptr()) % 256)
    lossb = torch.zeros(1)
    assert emul.mb200_gptj_sched_forward(ctypes.byref(m), ptr(x), ptr(labels), None, ctypes.c_int64(0), ptr(lossb), B, S,
                                         wsp, ctypes.c_size_t(n), None) == 0, emul.mb200_last_error()
    dx2 = torch.empty_like(x)
    for hi, lo in ((2, 1), (1, 0)):
        rc = emul.mb200_gptj_sched_backward_range(ctypes.byref(m), ptr(dx2) if lo == 0 else None, ctypes.c_float(1.0), hi,
                                                  lo, 0, B, S, wsp, ctypes.c_size_t(n), None)
        assert rc == 0, emul.mb200_last_error()
    assert torch.equal(dx2, dx) and all(torch.equal(grads2[k], grads[k]) for k in grads)


def test_launch_plan_trace_of_a_full_size_step():
    """tools/plan_trace.py: the product's own schedules issue a full-size training step (GPT-J-6B + ViT-L/14, B = 8,
    S = 128) on the emulation in trace mode — placeholder pointers, nothing touches memory — and the launch list carries the
    algorithmic FLOPs of bench.py (LM forward + backward, frozen: 2 x 1.5635 + 0.0601 TFLOP/sample + ViT 0.162)."""
    import os
    import sys

    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tools"))
    import plan_trace

    rows = plan_trace.train_step_plan(8, 128)
    gemms = [r for r in rows if r["op"] == "gemm"]
    assert 650 < len(rows) < 900 and len(gemms) > 450
    tflop = sum(r["flops"] for r in rows) / 1e12
    want = 8 * (2 * 1.5635 + 0.0601 + 0.1620)          # per sample -> per step of 8
    assert abs(tflop - want) / want < 0.03, (tflop, want)
    # the frozen-weight GEMMs of one block, forward: qkv, out, fc_in, fc_out at M = B*S = 1024
    shapes = {(int(r["args"]["M"]), int(r["args"]["N"]), int(r["args"]["K"])) for r in gemms}
    assert {(1024, 12288, 4096), (1024, 4096, 4096), (1024, 16384, 4096), (1024, 4096, 16384), (1024, 50258, 4096)} <= shapes
