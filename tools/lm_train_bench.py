"""Step time of config 2 with GPT-J's own weights training, on one GPU.

Magma with a frozen ViT-L/14, GPT-J-6B with config 2's MLP adapters (normal, downsample_factor 4), B = 8, S = 128, one
B200Engine step (forward, backward, fused AdamW) per timed call, with CUDA events around synchronised steps. The
variants are alternated round by round; each round rebuilds the parameter arena for its variant (untimed) and times
`--steps` steps after one untimed warm-up step:
  * frozen: the adapters and the image prefix train (config 2);
  * top2_head: also blocks 26 and 27, ln_f and lm_head;
  * ln_bias: also every LayerNorm and every bias of the LM (BitFit).
Then mb200_embed_grad alone at Magma's shape on padding-heavy captions. The card's name, power limit and clock are read
in the same run. One JSON line per variant.

    python tools/lm_train_bench.py [--rounds 3] [--steps 5] [--out FILE]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from tools.hidden_states_bench import card, timed  # noqa: E402

VARIANTS = {
    "frozen": lambda n: False,
    "top2_head": lambda n: n.startswith(("lm.transformer.h.26.", "lm.transformer.h.27.", "lm.transformer.ln_f.",
                                         "lm.lm_head.")),
    "ln_bias": lambda n: n.startswith("lm.") and (".ln_" in n or n.endswith(".bias")),
}


def embed_grad_row(rounds, info):
    """mb200_embed_grad alone at Magma's shape (B = 8, 126 caption tokens, d = 4096, vocabulary 50258) on captions whose
    last 60% is padding (one id repeated 600 times), accumulating into the table; median over 20 calls per round."""
    from magma_b200 import ops

    g = torch.Generator().manual_seed(1)
    ids = torch.randint(0, 50256, (8, 126), generator=g)
    ids[:, 50:] = 50256
    ids = ids.cuda()
    dx = torch.randn(8, 128, 4096, device="cuda").to(torch.bfloat16)
    dwte = torch.zeros(50258, 4096, device="cuda")
    ts = [timed(lambda: [ops.embed_grad(ids, dx[:, 2:], dwte, accumulate=True) for _ in range(20)]) / 20
          for _ in range(rounds + 1)][1:]
    return {"variant": "embed_grad_kernel", "n": 8 * 126, "d": 4096, "padding_repeats": 8 * 76,
            "median_ms": round(statistics.median(ts), 4), "min_ms": round(min(ts), 4), "max_ms": round(max(ts), 4),
            **info}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    from magma_b200.config import MultimodalConfig
    from magma_b200.magma import Magma
    from magma_b200.train_loop import B200Engine

    dev = torch.device("cuda:0")
    mc = MultimodalConfig(batch_size=8, train_steps=1, encoder_name="clip_vit_large",
                          adapter_config={"mlp": {"adapter_type": "normal", "downsample_factor": 4}}, image_seq_len=2,
                          image_embed_dropout_prob=0.0, use_image_embed_layernorm=True, image_size=224, seq_len=128,
                          lr=1e-4, freeze_img_encoder=True)
    model = Magma(mc, device=dev, init_seed=0)
    model.train()
    g = torch.Generator().manual_seed(0)
    images = torch.randn(8, 3, 224, 224, generator=g).to(dev).to(torch.bfloat16)
    captions = torch.randint(0, 50256, (8, 128), generator=g).to(dev)

    def select(kind):
        for n, p in model.named_parameters():
            if n.startswith("lm.") and "adapter" not in n:
                p.requires_grad_(VARIANTS[kind](n))
        model.finalize()
        torch.cuda.empty_cache()
        return B200Engine(model, mc), sum(p.numel() for p in model.arena.params)

    def step(eng):
        o = eng(images, captions)
        eng.backward(o.loss)
        eng.step()

    times = {k: [] for k in VARIANTS}
    trainable = {}
    for _ in range(a.rounds):
        for kind in VARIANTS:
            eng, trainable[kind] = select(kind)
            timed(lambda: step(eng))
            # the optimizer of the last step runs on the engine's side stream: it is inside the timed interval
            times[kind].extend(t / a.steps for t in [timed(lambda: ([step(eng) for _ in range(a.steps)],
                                                                   eng.synchronize()))])
            del eng
    info = card()
    rows = []
    base = statistics.median(times["frozen"])
    for kind, ts in times.items():
        med = statistics.median(ts)
        rows.append({"variant": kind, "B": 8, "S": 128, "trainable_params": trainable[kind],
                     "step_median_ms": round(med, 2), "min_ms": round(min(ts), 2), "max_ms": round(max(ts), 2),
                     "rounds": len(ts), "steps_per_round": a.steps, "added_ms": round(med - base, 2), **info})
    rows.append(embed_grad_row(a.rounds, info))
    text = "\n".join(json.dumps(r) for r in rows)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
