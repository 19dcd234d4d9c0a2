"""Cost of output_hidden_states at full size on one GPU.

Times, with CUDA events around synchronised calls and the variants alternated round by round:
  * a BASELINE.json config-2 training step (GPT-J-6B + ViT-L/14 + MLP adapters, B = 8, S = 128): Magma.forward +
    loss.backward() without output_hidden_states, with it (the 29 states returned, the loss unchanged) and with an
    auxiliary loss on every state (their gradients join the backward pass);
  * a 2048-token prefill of GPT-J-6B into a KV cache (B = 1), with and without output_hidden_states.
Each variant prints one JSON line with the median and spread of its times and the bytes the states take; the card's
name and power limit are read in the same run.

    python tools/hidden_states_bench.py [--rounds 10] [--warmup 2] [--out FILE]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (s.strip() for s in q.split(","))
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def timed(fn):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def alternate(variants, rounds, warmup):
    """{name: [ms per round]}: every variant once per round, in turn, after `warmup` untimed rounds."""
    times = {k: [] for k in variants}
    for r in range(warmup + rounds):
        for k, fn in variants.items():
            t = timed(fn)
            if r >= warmup:
                times[k].append(t)
    return times


def summary(case, times, state_bytes):
    out = []
    base = statistics.median(next(iter(times.values())))
    for k, ts in times.items():
        med = statistics.median(ts)
        out.append({"case": case, "variant": k, "median_ms": round(med, 3), "min_ms": round(min(ts), 3),
                    "max_ms": round(max(ts), 3), "overhead_ms": round(med - base, 3), "rounds": len(ts),
                    "hidden_state_bytes": state_bytes if k != "off" else 0})
    return out


def train_step_case(rounds, warmup):
    from magma_b200.config import MultimodalConfig
    from magma_b200.magma import Magma

    B, S = 8, 128
    mc = MultimodalConfig(batch_size=B, train_steps=1, encoder_name="clip_vit_large",
                          adapter_config={"mlp": {"adapter_type": "normal", "downsample_factor": 4}}, image_seq_len=2,
                          image_embed_dropout_prob=0.0, use_image_embed_layernorm=True, image_size=224, seq_len=S)
    model = Magma(mc, device=torch.device("cuda:0"), init_seed=0)
    model.train()
    g = torch.Generator().manual_seed(0)
    images = torch.randn(B, 3, 224, 224, generator=g).cuda().to(torch.bfloat16)
    captions = torch.randint(0, 50256, (B, S), generator=g)
    captions[:, 90:] = 50256
    captions = captions.cuda()
    n = model.lm.config.num_layers + 1
    c = [1e-3 * torch.randn(B, S, model.lm.config.hidden_size, device="cuda") for _ in range(n)]

    def step(hidden, aux=False):
        out = model(images, captions, output_hidden_states=hidden)
        loss = out.loss + sum((ci * h.float()).sum() for ci, h in zip(c, out.hidden_states)) if aux else out.loss
        loss.backward()

    times = alternate({"off": lambda: step(False), "on": lambda: step(True), "on_aux_loss": lambda: step(True, True)},
                      rounds, warmup)
    res = summary("train_step_config2_B8_S128", times, n * B * S * model.lm.config.hidden_size * 2)
    del model
    torch.cuda.empty_cache()
    return res


def prefill_case(rounds, warmup):
    from magma_b200.language_model import get_gptj

    lm = get_gptj(device="cuda:0").init_weights(seed=0)
    B, S = 1, 2048
    x = (0.5 * torch.randn(B, S, lm.config.hidden_size, device="cuda")).to(torch.bfloat16)

    @torch.no_grad()
    def prefill(hidden):
        lm(inputs_embeds=x, use_cache=True, max_cache_len=S, output_hidden_states=hidden)

    times = alternate({"off": lambda: prefill(False), "on": lambda: prefill(True)}, rounds, warmup)
    return summary("prefill_B1_S2048", times, (lm.config.num_layers + 1) * B * S * lm.config.hidden_size * 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("hidden_states_bench needs a CUDA device")
    info = card()
    rows = train_step_case(a.rounds, a.warmup) + prefill_case(a.rounds, a.warmup)
    lines = [json.dumps({**r, **info}) for r in rows]
    print("\n".join(lines))
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
