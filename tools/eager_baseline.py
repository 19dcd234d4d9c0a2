"""GPU-eager baseline: the reference assembly in plain PyTorch on the same GPU —
HF GPTJForCausalLM (eager attention; the executable stand-in for the reference's transformers fork) with the
reference's adapter wiring (mlp := Sequential(mlp, Adapter), magma/magma.py:143-148), HF CLIP ViT-L/14 as the image
encoder, Linear+Dropout+LayerNorm prefix, bf16, LM and encoder frozen, batch 8, 224x224, seq_len 128, fwd+bwd+AdamW.
No code from magma_b200 or oracle/ is used: every FLOP goes through ATen/cuBLAS. Reported next to bench.py's number
as the denominator of north_star's ">= 6x over the PyTorch-eager path" target; it is not part of the product."""
import argparse
import json
import time

import torch
import torch.nn as nn


class Adapter(nn.Module):
    def __init__(self, dim, f=4):
        super().__init__()
        self.adapter = nn.Sequential(nn.Linear(dim, dim // f), nn.ReLU(), nn.Linear(dim // f, dim))
        for m in self.adapter:
            if isinstance(m, nn.Linear):
                nn.init.normal_(m.weight, std=1e-3)
                nn.init.normal_(m.bias, std=1e-3)

    def forward(self, x):
        return self.adapter(x) + x


def run(steps=10, warmup=3, checkpointing=False, device="cuda:0"):
    """One process-local run of the eager step; returns the result dict (bench.py calls this for its `gpu_eager` key)."""
    import types

    a = types.SimpleNamespace(steps=steps, warmup=warmup, checkpointing=checkpointing)
    from transformers import CLIPVisionConfig, CLIPVisionModelWithProjection, GPTJConfig, GPTJForCausalLM

    dev = torch.device(device)
    B, S, L, V = 8, 128, 2, 50258
    prev_dtype = torch.get_default_dtype()
    torch.set_default_dtype(torch.bfloat16)
    try:
        return _run(a, dev, B, S, L, V, CLIPVisionConfig, CLIPVisionModelWithProjection, GPTJConfig, GPTJForCausalLM)
    finally:
        torch.set_default_dtype(prev_dtype)


def _run(a, dev, B, S, L, V, CLIPVisionConfig, CLIPVisionModelWithProjection, GPTJConfig, GPTJForCausalLM):
    t0 = time.time()
    with torch.device(dev):
        cfg = GPTJConfig(vocab_size=V, n_positions=2048, n_embd=4096, n_layer=28, n_head=16, rotary_dim=64,
                         resid_pdrop=0.0, embd_pdrop=0.0, attn_pdrop=0.0, tie_word_embeddings=False)
        cfg._attn_implementation = "eager"
        lm = GPTJForCausalLM(cfg)
        vcfg = CLIPVisionConfig(hidden_size=1024, intermediate_size=4096, num_hidden_layers=24, num_attention_heads=16,
                                image_size=224, patch_size=14, projection_dim=768)
        vcfg._attn_implementation = "eager"
        vit = CLIPVisionModelWithProjection(vcfg)
        proj = nn.Linear(768, 4096 * L)
        drop = nn.Dropout(0.1)
        ln = nn.LayerNorm(4096)
        for blk in lm.transformer.h:
            blk.mlp = nn.Sequential(blk.mlp, Adapter(4096, 4))
    for p in lm.parameters():
        p.requires_grad_(False)
    for p in vit.parameters():
        p.requires_grad_(False)
    train = [p for n, p in lm.named_parameters() if "adapter" in n] + list(proj.parameters()) + list(ln.parameters())
    for p in train:
        p.requires_grad_(True)
    if a.checkpointing:
        lm.gradient_checkpointing_enable()
        lm.config.use_cache = False
    lm.train()
    opt = torch.optim.AdamW(train, lr=8e-4, betas=(0.9, 0.95))
    torch.cuda.synchronize()
    build_s = time.time() - t0
    images = torch.randn(B, 3, 224, 224, device=dev)
    captions = torch.randint(0, 50256, (B, S), device=dev)
    captions[:, 100:] = 50256

    def step():
        with torch.no_grad():
            feats = vit(pixel_values=images).image_embeds
        prefix = ln(drop(proj(feats).view(B, L, 4096)))
        labels = torch.cat([torch.full((B, L), -100, device=dev), captions[:, : S - L]], 1)
        for row in labels:  # the reference's build_labels loop (utils.py:358-362), host-synchronous
            for k, tok in enumerate(row):
                if tok == 50256:
                    row[k + 1:] = -100
                    break
        x = torch.cat([prefix, lm.transformer.wte(captions)[:, : S - L]], 1)
        out = lm(inputs_embeds=x, labels=labels)
        out.loss.backward()
        opt.step()
        opt.zero_grad(set_to_none=True)
        return out.loss

    for _ in range(a.warmup):
        loss = step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.steps):
        loss = step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / a.steps
    return {"impl": "gpu-eager (HF GPT-J eager + reference adapter wiring, bf16, LM frozen)",
            "value": B / ms * 1e3, "unit": "samples/s", "ms_per_step": ms, "steps": a.steps,
            "checkpointing": a.checkpointing, "loss": float(loss.detach()), "build_s": build_s,
            "max_mem_gib": torch.cuda.max_memory_allocated() / 2**30}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--checkpointing", action="store_true", help="gradient checkpointing like language_model.py:23")
    a = ap.parse_args()
    print(json.dumps(run(a.steps, a.warmup, a.checkpointing)))


if __name__ == "__main__":
    main()
