"""TEST INFRASTRUCTURE — generates tests/golden/*.pt by running the REFERENCE ITSELF.

    python oracle/make_golden.py          # needs MAGMA_REFERENCE_ROOT (a reference checkout) and HF transformers

What runs: the reference's own Python (`magma.adapters.Adapter*`, `magma.image_prefix.ImagePrefix`,
`magma.utils.build_labels`, `magma.sampling.{top_k_filter,top_p_filter,generate}`, `magma.magma.Magma.__init__ /
forward / embed / generate`) imported from the reference checkout under the shims of oracle/ref_shims.py, with mainline HF
`GPTJForCausalLM` (eager attention) standing in for the reference's un-vendored transformers fork and HF
`CLIPVisionModelWithProjection` standing in for openai/CLIP's VisionTransformer. Everything is fp32
on CPU with seeded random weights at tiny sizes, so the fixtures stay small. Inputs, weights (re-keyed to the
oracle's naming = the reference state-dict naming) and outputs are stored; tests/test_oracle_golden.py replays the
inputs through oracle/magma_oracle.py and compares.
"""
import os
import sys

import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
OUT = os.path.join(HERE, "..", "tests", "golden")

from oracle.ref_shims import StubTokenizer, load_reference  # noqa: E402

TINY_LM = dict(vocab_size=300, n_positions=64, n_embd=64, n_layer=2, n_head=4, rotary_dim=8)
TINY_VIT = dict(hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=4, image_size=32,
                patch_size=8, projection_dim=48, hidden_act="quick_gelu", layer_norm_eps=1e-5)
EOS, CLS, NTOK = 254, 255, 256


class TinyTokenizer(StubTokenizer):
    cls_token_id = CLS
    eos_token_id = EOS
    pad_token_id = EOS

    def __len__(self):
        return NTOK


def hf_clip_to_openai_names(sd, prefix="image_prefix.enc"):
    """HF CLIPVisionModelWithProjection state dict -> openai/CLIP `.visual` names (the names the reference's
    checkpoints use for `image_prefix.enc.*`)."""
    out = {}
    v = "vision_model."
    out[f"{prefix}.conv1.weight"] = sd[v + "embeddings.patch_embedding.weight"]
    out[f"{prefix}.class_embedding"] = sd[v + "embeddings.class_embedding"]
    out[f"{prefix}.positional_embedding"] = sd[v + "embeddings.position_embedding.weight"]
    for a, b in (("ln_pre", "pre_layrnorm"), ("ln_post", "post_layernorm")):
        out[f"{prefix}.{a}.weight"] = sd[v + b + ".weight"]
        out[f"{prefix}.{a}.bias"] = sd[v + b + ".bias"]
    i = 0
    while v + f"encoder.layers.{i}.layer_norm1.weight" in sd:
        s, d = v + f"encoder.layers.{i}.", f"{prefix}.transformer.resblocks.{i}."
        for a, b in (("ln_1", "layer_norm1"), ("ln_2", "layer_norm2")):
            out[d + a + ".weight"] = sd[s + b + ".weight"]
            out[d + a + ".bias"] = sd[s + b + ".bias"]
        out[d + "attn.in_proj_weight"] = torch.cat([sd[s + f"self_attn.{n}_proj.weight"] for n in "qkv"], 0)
        out[d + "attn.in_proj_bias"] = torch.cat([sd[s + f"self_attn.{n}_proj.bias"] for n in "qkv"], 0)
        out[d + "attn.out_proj.weight"] = sd[s + "self_attn.out_proj.weight"]
        out[d + "attn.out_proj.bias"] = sd[s + "self_attn.out_proj.bias"]
        out[d + "mlp.c_fc.weight"] = sd[s + "mlp.fc1.weight"]
        out[d + "mlp.c_fc.bias"] = sd[s + "mlp.fc1.bias"]
        out[d + "mlp.c_proj.weight"] = sd[s + "mlp.fc2.weight"]
        out[d + "mlp.c_proj.bias"] = sd[s + "mlp.fc2.bias"]
        i += 1
    out[f"{prefix}.proj"] = sd["visual_projection.weight"].t().contiguous()
    return out


class ClipVisualStandIn(nn.Module):
    """What `clip.load(name)[0].visual` is to the reference: images -> pooled projected features [b, D]."""

    def __init__(self):
        super().__init__()
        from transformers import CLIPVisionConfig, CLIPVisionModelWithProjection

        cfg = CLIPVisionConfig(**TINY_VIT)
        cfg._attn_implementation = "eager"
        self.m = CLIPVisionModelWithProjection(cfg)
        self.input_resolution = TINY_VIT["image_size"]

    def forward(self, x):
        return self.m(pixel_values=x).image_embeds


def randomize(module, seed, std=0.05):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n, p in module.named_parameters():
            r = torch.randn(p.shape, generator=g) * std
            if "ln" in n.split(".")[-2] or "norm" in n.split(".")[-2] or "layernorm" in n.split(".")[-2]:
                if n.endswith("weight"):
                    r = 1.0 + r
            p.copy_(r)


def magma_state_to_oracle(model):
    """Reference Magma state dict (HF GPT-J inside) -> oracle naming. Only the encoder needs re-keying."""
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    enc = {k[len("image_prefix.enc.m."):]: v for k, v in sd.items() if k.startswith("image_prefix.enc.m.")}
    out = {k: v for k, v in sd.items() if not k.startswith("image_prefix.enc.") and "embed_positions" not in k
           and not k.endswith("attn.bias") and not k.endswith("masked_bias")}
    out.update(hf_clip_to_openai_names(enc))
    return out


def main():
    os.makedirs(OUT, exist_ok=True)
    torch.manual_seed(0)
    ref = load_reference(gptj_kwargs=TINY_LM, encoder_factory=lambda name, device=None, pretrained=False: ClipVisualStandIn())
    ref.magma.get_tokenizer = lambda *a, **k: TinyTokenizer()
    ref.image_prefix.ENCODER_OUT_DIMS["clip"] = TINY_VIT["projection_dim"]
    import magma.config as mcfg

    # ---------------- 1. Adapter (magma/adapters.py:6-39) ----------------
    ad = ref.adapters.Adapter(64, 4)
    randomize(ad, 1, 0.2)
    x = torch.randn(3, 5, 64)
    torch.save({"weights": {k: v.clone() for k, v in ad.state_dict().items()}, "x": x, "y": ad(x).detach()},
               os.path.join(OUT, "adapter.pt"))

    # ---------------- 2. build_labels (magma/utils.py:334-364) ----------------
    cases = []
    g = torch.Generator().manual_seed(2)
    for L, S, B in ((2, 16, 4), (0, 9, 3), (5, 5, 2), (7, 33, 5), (1, 2, 2)):
        caps = torch.randint(0, 250, (B, S), generator=g)
        if B > 1:
            caps[0, S // 2:] = EOS
            caps[1, 0] = EOS
        if S > 3:
            caps[-1, S - 1] = EOS
        emb = torch.zeros(B, L, 4)
        labels = ref.utils.build_labels(emb, caps.clone(), EOS, "cpu")
        cases.append({"L": L, "captions": caps, "labels": labels})
    torch.save({"eos": EOS, "cases": cases}, os.path.join(OUT, "build_labels.pt"))

    # ---------------- 3. sampling filters (magma/sampling.py:7-30) ----------------
    lg = torch.randn(4, 50, generator=g) * 2
    filt = {"logits": lg,
            "top_k_5": ref.sampling.top_k_filter(lg.clone(), 5),
            "top_p_0.9": ref.sampling.top_p_filter(lg.clone(), 0.9),
            "top_p_0.5": ref.sampling.top_p_filter(lg.clone(), 0.5),
            "quirk_probs": torch.tensor([[.3, .25, .2, .15, .1]]).log()}
    filt["quirk_0.5"] = ref.sampling.top_p_filter(filt["quirk_probs"].clone(), 0.5)
    filt["quirk_0.9"] = ref.sampling.top_p_filter(filt["quirk_probs"].clone(), 0.9)
    torch.save(filt, os.path.join(OUT, "sampling_filters.pt"))

    # ---------------- 4. full reference Magma, three adapter wirings ----------------
    variants = {
        "v1_mlp_normal": {"mlp": {"adapter_type": "normal", "downsample_factor": 4}},
        "v2_mlp_attn_normal": {"mlp": {"adapter_type": "normal", "downsample_factor": 8},
                               "attention": {"adapter_type": "normal", "downsample_factor": 8}},
        "parallel": {"mlp": {"adapter_type": "parallel", "downsample_factor": 4},
                     "attention": {"adapter_type": "parallel", "downsample_factor": 4}},
        "no_adapters": None,
    }
    S, B = 24, 3
    for i, (tag, ac) in enumerate(variants.items()):
        cfg = mcfg.MultimodalConfig(batch_size=B, train_steps=1, encoder_name="clip", adapter_config=ac,
                                    image_seq_len=2, use_image_embed_layernorm=True, image_embed_dropout_prob=0.0,
                                    image_size=32)
        model = ref.magma.Magma(cfg, device="cpu")
        randomize(model, 10 + i, 0.08)
        # Decided ReLU masks: every adapter down-projection bias is +-3 (random sign) so that no bottleneck pre-activation
        # sits within bf16 rounding of zero — a bf16 run then takes the same mask as this fp32 run and the gradients can be
        # held to the tight bar (a flipped mask entry is an O(1) relative error in that entry, not a kernel defect).
        gm = torch.Generator().manual_seed(500 + i)
        with torch.no_grad():
            for n, p in model.named_parameters():
                if n.endswith("adapter.0.bias"):
                    p.copy_(torch.where(torch.rand(p.shape, generator=gm) < 0.5, -3.0, 3.0)
                            + 0.02 * torch.randn(p.shape, generator=gm))
        model.eval()
        model.seq_len = S  # plain attribute
        gi = torch.Generator().manual_seed(100 + i)
        images = torch.randn(B, 3, 32, 32, generator=gi)
        caps = torch.randint(0, 250, (B, S), generator=gi)
        caps[0, 15:] = EOS
        caps[1, 9:] = EOS
        for p in model.parameters():
            p.requires_grad_(False)
        trainable = [n for n, _ in model.named_parameters()
                     if "adapter" in n or n.startswith("image_prefix.proj") or n.startswith("image_prefix.ln")]
        for n, p in model.named_parameters():
            if n in trainable:
                p.requires_grad_(True)
        out = model(images, caps)
        out.loss.backward()
        grads = {n: p.grad.detach().clone() for n, p in model.named_parameters() if n in trainable}
        rec = {"adapter_config": ac, "S": S, "images": images, "captions": caps, "loss": out.loss.detach(),
               "logits": out.logits.detach(), "grads": grads, "weights": magma_state_to_oracle(model),
               "eos": EOS, "cls": CLS, "lm": TINY_LM, "vit": TINY_VIT}
        if tag == "v1_mlp_normal":
            # embed + greedy generate (magma.py:195-236, sampling.py:43-121 at temperature 0).
            # NB reference embed() forces images to .half() (magma.py:207); the fp32-CPU model cannot consume that,
            # so the prefix is taken from image_prefix() directly, exactly what embed() does after the cast.
            with torch.no_grad():
                text = torch.randint(0, 250, (B, 4), generator=gi)
                emb = torch.cat([model.image_prefix(images), model.word_embedding(text)], dim=1)
                toks = ref.sampling.generate(model, emb, max_steps=10, temperature=0.0, decode=False)
                feats = model.image_prefix.enc(images)
                # top-1 minus top-2 logit at every greedy step (teacher-forced full forward over the generated ids): a
                # bf16 run is required to emit the same ids up to the first step whose margin is a near-tie
                s0 = emb.shape[1]
                full = torch.cat([emb, model.word_embedding(toks[:, s0:])], dim=1)
                lg = model.lm(inputs_embeds=full).logits[:, s0 - 1:-1].float()
                top2 = lg.topk(2, dim=-1).values
                margin = top2[..., 0] - top2[..., 1]
                assert torch.equal(lg.argmax(-1), toks[:, s0:])
            rec.update({"text": text, "embeddings": emb, "greedy_tokens": toks, "enc_feats": feats,
                        "greedy_margin": margin})
        torch.save(rec, os.path.join(OUT, f"magma_{tag}.pt"))
        print(tag, "loss", float(out.loss), "n_trainable", len(trainable))
    print("golden fixtures written to", os.path.abspath(OUT))
    for f in sorted(os.listdir(OUT)):
        print(f"  {f}: {os.path.getsize(os.path.join(OUT, f)) / 1024:.0f} KiB")


if __name__ == "__main__":
    main()
