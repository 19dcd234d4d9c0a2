"""Cost of output_attentions at full size on one GPU.

Times, with CUDA events around synchronised calls and the variants alternated round by round:
  * the GPT-J-6B training step of a BASELINE.json config-2 run (MLP adapters with downsample factor 4, B = 8, S = 128,
    gradients to the input embeddings as the image prefix takes them): forward + loss.backward() without
    output_attentions, with it (the 28 maps returned, the loss unchanged) and with an auxiliary loss on all 28 (their
    gradients join the backward pass);
  * a 2048-token prefill of GPT-J-6B into a KV cache (B = 1), with and without output_attentions;
  * one host-driven decode step of GPT-J-6B at B = 32 over a 264-position cache, with and without output_attentions.
Each variant prints one JSON line with the median and spread of its times and the bytes the attentions take; the
card's name, power limit and maximum SM clock are read in the same run.

    python tools/attentions_bench.py [--rounds 7] [--warmup 2] [--out FILE]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from hidden_states_bench import alternate, card  # noqa: E402


def summary(case, times, attn_bytes):
    import statistics

    out = []
    base = statistics.median(next(iter(times.values())))
    for k, ts in times.items():
        med = statistics.median(ts)
        out.append({"case": case, "variant": k, "median_ms": round(med, 3), "min_ms": round(min(ts), 3),
                    "max_ms": round(max(ts), 3), "overhead_ms": round(med - base, 3), "rounds": len(ts),
                    "attention_bytes": attn_bytes if k != "off" else 0})
    return out


def lm_with_adapters():
    from magma_b200.adapters import Adapter
    from magma_b200.language_model import get_gptj

    lm = get_gptj(device="cuda:0").init_weights(seed=0)
    d = lm.config.hidden_size
    for blk in lm.transformer.h:  # magma/magma.py:143-148: Sequential(mlp, Adapter(d, 4))
        blk.mlp = torch.nn.Sequential(blk.mlp, Adapter(d, 4).to("cuda:0"))
    lm.invalidate()
    return lm


def train_step_case(lm, rounds, warmup):
    B, S = 8, 128
    cfg = lm.config
    g = torch.Generator(device="cuda").manual_seed(0)
    x = (0.5 * torch.randn(B, S, cfg.hidden_size, generator=g, device="cuda")).to(torch.bfloat16)
    labels = torch.randint(0, cfg.vocab_size, (B, S), generator=g, device="cuda")
    labels[:, :2] = -100
    c = [torch.randn(B, cfg.num_heads, S, S, generator=g, device="cuda") for _ in range(cfg.num_layers)]

    def step(attn, aux=False):
        xr = x.clone().requires_grad_(True)
        out = lm(inputs_embeds=xr, labels=labels, output_attentions=attn)
        loss = out.loss + sum((ci * a.float()).sum() for ci, a in zip(c, out.attentions)) if aux else out.loss
        loss.backward()

    times = alternate({"off": lambda: step(False), "on": lambda: step(True), "on_aux_loss": lambda: step(True, True)},
                      rounds, warmup)
    return summary("train_step_config2_B8_S128", times, cfg.num_layers * B * cfg.num_heads * S * S * 2)


def prefill_case(lm, rounds, warmup):
    B, S = 1, 2048
    cfg = lm.config
    x = (0.5 * torch.randn(B, S, cfg.hidden_size, device="cuda")).to(torch.bfloat16)

    @torch.no_grad()
    def prefill(attn):
        lm(inputs_embeds=x, use_cache=True, max_cache_len=S, output_attentions=attn)

    times = alternate({"off": lambda: prefill(False), "on": lambda: prefill(True)}, rounds, warmup)
    return summary("prefill_B1_S2048", times, cfg.num_layers * B * cfg.num_heads * S * S * 2)


def decode_case(lm, rounds, warmup):
    B, P = 32, 263  # the step writes position 263: 264 keys
    cfg = lm.config
    x = (0.5 * torch.randn(B, P + 1, cfg.hidden_size, device="cuda")).to(torch.bfloat16)
    with torch.no_grad():
        cache = lm(inputs_embeds=x[:, :P], use_cache=True, max_cache_len=P + 1).past_key_values
    step_x = x[:, P:].contiguous()

    @torch.no_grad()
    def step(attn):
        lm(inputs_embeds=step_x, use_cache=True, past_key_values=cache, output_attentions=attn)
        cache.pos -= 1  # every round decodes the same position

    times = alternate({"off": lambda: step(False), "on": lambda: step(True)}, rounds, warmup)
    return summary("decode_B32_pos263", times, cfg.num_layers * B * cfg.num_heads * ((P + 1 + 7) // 8 * 8) * 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("attentions_bench needs a CUDA device")
    info = card()
    lm = lm_with_adapters()
    rows = train_step_case(lm, a.rounds, a.warmup) + prefill_case(lm, a.rounds, a.warmup) + \
        decode_case(lm, a.rounds, a.warmup)
    lines = [json.dumps({**r, **info}) for r in rows]
    print("\n".join(lines))
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
