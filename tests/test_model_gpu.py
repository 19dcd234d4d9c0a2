"""GPU parity tests of the model-level runtime (C ABI mb200_gptj_forward/backward, mb200_vit_forward, decode) and of
the drop-in Python API (Magma.forward / embed / generate, B200Engine) against the CPU oracle on identical seeded
inputs, and against the golden fixtures produced by the REFERENCE ITSELF (tests/golden/, oracle/make_golden.py).

Tolerances (bf16 kernels vs fp32 oracle): |dloss| < 2e-2; logits rel-Frobenius < 3e-2; gradients
rel-Frobenius < 3e-2 — the reference-made fixtures and the full-size case use adapters whose ReLU masks are decided away
from zero (down-projection biases of +-3), so that bf16 and fp32 agree on the mask; only tools/model_check.py's
"free relu mask" case (a flipped mask entry is an O(1) relative error in that entry) uses a wider bound. Integer results
(labels, greedy token ids up to the reference's first top-1/top-2 near-tie) are exact."""
import os

import pytest

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("group", ["lm", "lm_variants", "vit", "resnet", "magma", "generate", "sampling"])
def test_model_group(group):
    import torch

    from tools import model_check

    assert getattr(model_check, "group_" + group)(torch.device("cuda:0"))


@pytest.mark.parametrize("tag", ["v1_mlp_normal", "v2_mlp_attn_normal", "parallel", "no_adapters"])
def test_magma_matches_reference_golden(golden_dir, tag):
    import torch

    from _gpu_util import build_magma_from_weights, gpu_device, rel
    from conftest import oracle_cfg_from_record

    dev = gpu_device()
    rec = torch.load(os.path.join(golden_dir, f"magma_{tag}.pt"), weights_only=False)
    cfg = oracle_cfg_from_record(rec)
    # the reference ran in fp32; the CUDA path stores weights/activations in bf16
    model = build_magma_from_weights(rec["weights"], cfg, rec["adapter_config"], rec["S"], dev, vit_name="clip_vit_golden")
    model.eval()
    out = model(rec["images"].to(dev), rec["captions"].to(dev))
    assert abs(float(out.loss) - float(rec["loss"])) < 2e-2
    assert rel(out.logits, rec["logits"]) < 3e-2
    if rec["grads"]:
        out.loss.backward()
        sd = dict(model.named_parameters())
        # The fixtures are generated with DECIDED ReLU masks (adapter down-projection biases of +-3,
        # oracle/make_golden.py): bf16 and the reference's fp32 take the same mask, so every trainable gradient —
        # including the down-projection ones that pass through the mask — is held to the tight bar.
        bad = {}
        for k, gref in rec["grads"].items():
            assert sd[k].grad is not None, k
            err = rel(sd[k].grad, gref)
            if err >= 3e-2:
                bad[k] = round(err, 4)
        assert not bad, bad


def test_vit_embed_generate_match_reference_golden(golden_dir):
    import torch

    from _gpu_util import build_magma_from_weights, gpu_device, rel
    from conftest import oracle_cfg_from_record

    dev = gpu_device()
    rec = torch.load(os.path.join(golden_dir, "magma_v1_mlp_normal.pt"), weights_only=False)
    cfg = oracle_cfg_from_record(rec)
    model = build_magma_from_weights(rec["weights"], cfg, rec["adapter_config"], rec["S"], dev, vit_name="clip_vit_golden")
    model.eval()
    feats = model.image_prefix.enc(rec["images"].to(dev))
    assert rel(feats, rec["enc_feats"]) < 3e-2
    emb = model.embed([rec["images"].to(dev), rec["text"].to(dev)])
    assert emb.shape == rec["embeddings"].shape and rel(emb, rec["embeddings"]) < 3e-2
    toks = model.generate(rec["embeddings"].to(dev).to(torch.bfloat16), max_steps=10, temperature=0.0, decode=False).cpu()
    ref = rec["greedy_tokens"]
    # Token ids are exact up to (not including) the first greedy step at which the reference's own top-1 / top-2 logit
    # margin is a bf16 near-tie; logits here are O(1), one bf16 ulp of them is ~8e-3, and the
    # accumulated bf16 error of the tiny model's logits is held to 3e-2 relative above.
    s0, tau = rec["embeddings"].shape[1], 0.05
    assert torch.equal(toks[:, :s0], ref[:, :s0])
    margin = rec["greedy_margin"]
    n_exact = 0
    for b in range(ref.shape[0]):
        tied = (margin[b] < tau).nonzero()
        first_tie = int(tied[0]) if len(tied) else margin.shape[1]
        n = min(first_tie, toks.shape[1] - s0)
        assert torch.equal(toks[b, s0:s0 + n], ref[b, s0:s0 + n]), (b, toks[b, s0:], ref[b, s0:], margin[b])
        n_exact += n
    assert n_exact >= ref.shape[0] * 3, (n_exact, margin)  # the fixture must actually pin several steps per row


def test_magma_forward_asserts_like_the_reference():
    import torch

    from _gpu_util import build_magma_from_weights, gpu_device
    from oracle import magma_oracle as O
    from tools.model_check import small_cfg

    dev = gpu_device()
    cfg = small_cfg()
    w = {k: v.to(torch.bfloat16).float() for k, v in O.init_weights(cfg, seed=3).items()}
    model = build_magma_from_weights(w, cfg, {"mlp": {"adapter_type": "normal", "downsample_factor": 4}}, 32, dev)
    images, captions = O.synthetic_batch(cfg, 2, 32, seed=1)
    with pytest.raises(AssertionError, match="captions"):
        model(images.to(dev), None)
    with pytest.raises(AssertionError, match="padded to sequence length"):
        model(images.to(dev), captions[:, :20].to(dev))
    with pytest.raises(AssertionError, match="not both"):
        model(images.to(dev), captions.to(dev), input_embeddings=torch.zeros(2, 2, cfg.d, device=dev))
    with pytest.raises(ValueError, match="already added"):
        model.add_adapters(location="mlp")
    with pytest.raises(ValueError, match="Expected 2d or 4d"):
        model.embed([torch.zeros(3, device=dev)])


def test_full_size_step_properties():
    """BASELINE config-2 sizes (GPT-J-6B + ViT-L/14, B=8, S=128): size-independent properties instead of an oracle
    run — loss ~ ln(V) at random init, finite gradients on every trainable tensor, gradient accumulation is linear,
    the fused optimizer step lowers the loss on the same batch, and a frozen LM weight never changes."""
    import math

    import torch

    from magma_b200.config import MultimodalConfig
    from magma_b200.magma import Magma
    from magma_b200.train_loop import B200Engine

    dev = torch.device("cuda:0")
    mc = MultimodalConfig(batch_size=8, train_steps=1, encoder_name="clip_vit_large",
                          adapter_config={"mlp": {"adapter_type": "normal", "downsample_factor": 4}}, image_seq_len=2,
                          image_embed_dropout_prob=0.0, use_image_embed_layernorm=True, image_size=224, seq_len=128,
                          lr=1e-3, warmup_num_steps=2)
    model = Magma(mc, device=dev, init_seed=0)
    model.train()
    B, S = 8, 128
    g = torch.Generator().manual_seed(0)
    images = torch.randn(B, 3, 224, 224, generator=g).to(dev).to(torch.bfloat16)
    captions = torch.randint(0, 50256, (B, S), generator=g)
    captions[:, 90:] = 50256
    captions = captions.to(dev)
    out = model(images, captions)
    assert out.logits.shape == (B, S, 50258)
    assert abs(float(out.loss) - math.log(50258)) < 1.0
    out.loss.backward()
    n_train = 0
    for n, p in model.named_parameters():
        if p.requires_grad:
            n_train += p.numel()
            assert p.grad is not None and torch.isfinite(p.grad).all(), n
    assert n_train == 28 * 8_393_728 + 768 * 8192 + 8192 + 2 * 4096  # 241.3 M trainable
    g1 = model.arena.grad.clone()
    model(images, captions).loss.backward()  # grads live -> accumulate
    assert ((model.arena.grad - 2 * g1).norm() / (2 * g1).norm()).item() < 1e-2
    frozen_before = model.lm.transformer.h[5].attn.out_proj.weight.clone()
    for p in model.parameters():
        p.grad = None
    model.arena.grad.zero_()
    eng = B200Engine(model, mc)
    losses = []
    for _ in range(3):
        o = eng(images, captions)
        eng.backward(o.loss)
        eng.step()
        losses.append(float(o.loss))
    assert losses[-1] < losses[0], losses
    assert torch.equal(frozen_before, model.lm.transformer.h[5].attn.out_proj.weight)


def _shared_layer_weights(cfg, seed=0):
    """Oracle-named weights of a model whose frozen per-layer tensors are shared by all layers and whose adapters are
    per-layer, O(0.05), with decided ReLU masks (see _shared_layer_case)."""
    import dataclasses

    import torch

    from oracle import magma_oracle as O
    from tools.model_check import boost_adapters

    one = dataclasses.replace(cfg, n_layer=1, vit_layers=1)
    w1 = O.init_weights(one, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    w = {}
    for k, v in w1.items():
        v = v.to(torch.bfloat16).float()  # the oracle sees the bf16-representable values the device stores
        if ".transformer.h.0." in k:
            for l in range(cfg.n_layer):
                kk = k.replace(".transformer.h.0.", f".transformer.h.{l}.")
                w[kk] = torch.randn(v.shape, generator=g) if ".adapter." in k else v
        elif ".resblocks.0." in k:
            for l in range(cfg.vit_layers):
                w[k.replace(".resblocks.0.", f".resblocks.{l}.")] = v
        else:
            w[k] = v
    torch.manual_seed(seed + 2)
    w = boost_adapters(w, True)
    # boost_adapters draws O(0.05) weights, tuned for d = 512: keep the bottleneck pre-activation's spread (~ std * sqrt(d))
    # well inside the +-3 bias at any width, so the ReLU masks stay decided
    for k in w:
        if k.endswith("adapter.0.weight"):
            w[k] = w[k] * min(1.0, (512.0 / cfg.d) ** 0.5) * 0.5
    return {k: (v.to(torch.bfloat16).float() if ".adapter." in k else v) for k, v in w.items()}


def _shared_layer_case(dev, cfg, B, S, seed=0, vit_name="clip_vit_shared_case"):
    """Magma.forward + backward against the oracle on a model whose FROZEN per-layer weights are one set of random
    tensors shared by every GPT-J / ViT layer (the host-memory trick of bench.py's CPU arm: identical shapes, FLOPs
    and kernels per layer, 1/28 of the fp32 host weights), while every layer keeps its OWN adapter parameters, so the
    per-layer trainable gradients are compared one by one. Adapter weights are O(0.05) with down-projection biases of
    +-3 (tools/model_check.py::boost_adapters): every bottleneck ReLU is decided away from zero and bf16 / fp32 agree
    on the mask. Returns the measured errors."""
    import torch

    from _gpu_util import build_magma_from_weights, rel
    from oracle import magma_oracle as O

    w = _shared_layer_weights(cfg, seed)
    model = build_magma_from_weights(w, cfg, {"mlp": cfg.mlp_adapter}, S, dev, vit_name=vit_name)
    model.eval()
    images, captions = O.synthetic_batch(cfg, B, S, seed=seed + 3)
    images = images.to(torch.bfloat16).float()
    trainable = [k for k in w if ".adapter." in k or k.startswith(("image_prefix.proj", "image_prefix.ln"))]
    params = {k: (v.clone().requires_grad_(True) if k in trainable else v) for k, v in w.items()}
    loss_o, logits_o, labels_o = O.magma_forward(images, captions, params, cfg)
    loss_o.backward()
    out = model(images.to(dev), captions.to(dev))
    out.loss.backward()
    sd = dict(model.named_parameters())
    errs = {k: rel(sd[k].grad, params[k].grad) for k in trainable}
    # how decided the masks really are: fraction of bottleneck pre-activations within 0.25 of zero (oracle side)
    return {"dloss": abs(float(out.loss.detach()) - float(loss_o.detach())), "logits": rel(out.logits, logits_o.detach()),
            "grads": errs, "n_trainable": sum(sd[k].numel() for k in trainable), "loss": float(loss_o.detach())}


def test_config2_full_size_matches_oracle():
    """BASELINE.json config 2 at FULL SIZE against the oracle: GPT-J-6B (28 layers, d = 4096, 16 heads of 256, V = 50258
    with the ragged LM head) + CLIP ViT-L/14 (24 layers, T = 257) + MLP adapters f = 4, 224 x 224 images, seq_len 128,
    batch 2 (the oracle's fp32 forward + backward of 2 samples takes seconds on the host; the kernels, tile shapes and
    launch paths are those of the B = 8 benchmark step except for M = 256 instead of 1024 — the CTA-pair GEMM with
    K = 4096 / 16384, head_dim-256 fused attention, the 50258-wide LM head and cross-entropy).
    Bars: |dloss| < 2e-2, logits rel-Frobenius < 3e-2, every trainable gradient < 3e-2."""
    import torch

    from oracle import magma_oracle as O

    r = _shared_layer_case(torch.device(os.environ.get("MB200_TEST_DEVICE", "cuda:0")), O.OracleConfig(), B=2, S=128,
                           vit_name="clip_vit_large_fullsize_case")
    worst = max(r["grads"], key=r["grads"].get)
    by_kind = {}
    for k, e in r["grads"].items():
        kind = k.split(".")[-2] + "." + k.split(".")[-1] if ".adapter." in k else k
        by_kind.setdefault(kind, []).append(e)
    print({k: (round(min(v), 4), round(max(v), 4)) for k, v in by_kind.items()})
    print(f"full-size config 2 vs oracle: loss {r['loss']:.4f} |dloss| {r['dloss']:.2e}, logits rel {r['logits']:.2e}, "
          f"worst gradient rel {r['grads'][worst]:.2e} ({worst}) over {len(r['grads'])} tensors / {r['n_trainable']} parameters")
    assert r["n_trainable"] == 28 * 8_393_728 + 768 * 8192 + 8192 + 2 * 4096
    assert r["dloss"] < 2e-2
    assert r["logits"] < 3e-2
    bad = {k: round(e, 4) for k, e in r["grads"].items() if e >= 3e-2}
    assert not bad, bad


def _kv_decode_case(dev, cfg, B, n_prompt, n_steps, seed=0, vit_name="clip_vit_shared_decode_case"):
    """KV-cache decoding against the oracle, teacher-forced: image prefix + n_prompt prompt ids are prefilled into a static
    cache (`decode_logits`: multi-position attention over the cache, small-M weight-streaming GEMMs, last-position LM
    head), then n_steps single-token steps (fused cache-append + decode attention) each fed the DEVICE's own greedy token.
    The oracle has no cache: one full causal forward over the final sequence gives the logits of every position. Returns
    per-position logits errors and, per emitted token, whether it is the oracle's argmax or inside an oracle near-tie."""
    import torch

    from _gpu_util import build_magma_from_weights, rel
    from magma_b200 import ops
    from magma_b200.language_model import KVCache
    from oracle import magma_oracle as O

    w = _shared_layer_weights(cfg, seed)
    L = cfg.image_seq_len
    S = L + n_prompt + n_steps
    model = build_magma_from_weights(w, cfg, {"mlp": cfg.mlp_adapter}, S, dev, vit_name=vit_name)
    model.eval()
    images, captions = O.synthetic_batch(cfg, B, S, seed=seed + 3)
    images = images.to(torch.bfloat16).float()
    prompt = captions[:, :n_prompt].clamp(max=cfg.eos_token - 1)
    lm, lc = model.lm, model.lm.config
    with torch.no_grad():
        emb = model.embed([images.to(dev), prompt.to(dev)])
        assert emb.shape[1] == L + n_prompt
        cache = KVCache(lc.num_layers, B, lc.num_heads, S, lc.hidden_size // lc.num_heads, dev)
        got, toks = [], []
        logits = lm.decode_logits(emb, cache)
        for i in range(n_steps):
            got.append(logits.float().cpu()[:, : cfg.vocab])
            nxt = ops.argmax(logits.contiguous(), logits.shape[-1])
            toks.append(nxt.cpu())
            if i + 1 < n_steps:
                logits = lm.decode_logits(lm.transformer.wte(nxt[:, None]), cache)
    toks = torch.stack(toks, 1)                                      # [B, n_steps] device-chosen greedy tokens
    full = torch.cat([prompt, toks, torch.full((B, S - n_prompt - n_steps), cfg.eos_token)], 1)[:, : S]
    _, logits_o, _ = O.magma_forward(images, full, w, cfg)            # [B, S, V]; position p sees tokens <= p
    errs, picks = [], []
    for i in range(n_steps):
        ref = logits_o[:, L + n_prompt - 1 + i].detach().float()
        errs.append(rel(got[i], ref))
        top2 = ref.topk(2, dim=-1)
        is_argmax = toks[:, i] == top2.indices[:, 0]
        near_tie = (top2.values[:, 0] - ref.gather(1, toks[:, i:i + 1])[:, 0]) < 0.05 * ref.abs().max(dim=-1).values
        picks.append(bool((is_argmax | near_tie).all()))
    return {"logits": errs, "picks": picks, "toks": toks}


def test_config5_full_size_kv_decode_matches_oracle():
    """BASELINE.json config 5's path at FULL SIZE against the oracle: GPT-J-6B (28 layers, d = 4096, 16 heads of 256,
    V = 50258) + ViT-L/14 prefix + MLP adapters, an 8-position prompt (2 prefix + 6 ids) prefilled into the static KV
    cache, then greedy single-token steps — the small-M weight-streaming GEMMs with their split-K plans at K = 4096 /
    16384, cache attention at head_dim 256 and the ragged LM head that `bench.py --workload decode` times. Batch 4 keeps
    the oracle's fp32 forward to seconds; the kernels and split plans are those of every M <= 32.
    Bars: logits rel-Frobenius < 3e-2 at every position; every emitted token is the oracle's argmax or inside a near-tie."""
    import torch

    from oracle import magma_oracle as O

    r = _kv_decode_case(torch.device(os.environ.get("MB200_TEST_DEVICE", "cuda:0")), O.OracleConfig(), B=4, n_prompt=6,
                        n_steps=4, vit_name="clip_vit_large_fullsize_decode_case")
    print(f"full-size KV decode vs oracle: logits rel per position {[round(e, 4) for e in r['logits']]}, tokens "
          f"{r['toks'][0].tolist()} ...")
    assert max(r["logits"]) < 3e-2, r["logits"]
    assert all(r["picks"]), r["picks"]


def test_graph_replayed_decode_emits_the_same_tokens_as_the_host_driven_loop(monkeypatch):
    """magma/sampling.py:78-109 at temperature 0: the device-resident decode loop (one CUDA graph of the decode step
    replayed per token, cache position in device memory) against the host-driven loop over the same kernels — every
    emitted id identical, including the early exit when all rows hit EOS."""
    import torch

    from _gpu_util import build_magma_from_weights, gpu_device
    from oracle import magma_oracle as O
    from tools.model_check import small_cfg

    dev = gpu_device()
    cfg = small_cfg(n_layer=3)
    w = O.init_weights(cfg, seed=9)
    w["lm.lm_head.weight"] = w["lm.lm_head.weight"] * 8  # sharpen the head: greedy ids not decided by bf16 near-ties
    w16 = {k: v.to(torch.bfloat16).float() for k, v in w.items()}
    model = build_magma_from_weights(w16, cfg, {"mlp": {"adapter_type": "normal", "downsample_factor": 4}}, 32, dev)
    model.eval()
    g = torch.Generator().manual_seed(3)
    emb = (torch.randn(4, 7, cfg.d, generator=g) * 0.5).to(torch.bfloat16).to(dev)
    monkeypatch.setenv("MB200_DECODE_GRAPH", "0")
    host = model.generate(emb, max_steps=40, temperature=0.0, decode=False).cpu()
    monkeypatch.setenv("MB200_DECODE_GRAPH", "1")
    graph = model.generate(emb, max_steps=40, temperature=0.0, decode=False).cpu()
    assert host.shape == graph.shape and torch.equal(host, graph)
    # early exit: make EOS the argmax of every row from some step on (bias the EOS logit hard), both loops stop alike
    model.lm.lm_head.bias.data[cfg.eos_token] = 1e4
    model.lm.invalidate()
    model.lm.attach_arena(model.arena)
    monkeypatch.setenv("MB200_DECODE_GRAPH", "0")
    host = model.generate(emb, max_steps=40, temperature=0.0, decode=False).cpu()
    monkeypatch.setenv("MB200_DECODE_GRAPH", "1")
    graph = model.generate(emb, max_steps=40, temperature=0.0, decode=False).cpu()
    assert host.shape == graph.shape and torch.equal(host, graph) and host.shape[1] < 7 + 40
