"""Sampled decoding (temperature 0.7, top_p 0.9: the reference's defaults) with the decode step replayed as one CUDA
graph per token against the host-driven loop (MB200_DECODE_GRAPH=1 / 0), greedy decoding in the same run for
reference. GPT-J-6B + ViT-L/14 + MLP adapters, random weights, EOS suppressed so that every call runs all its steps.

Cases:
  * config5: B = 32, prompt of 8 positions (2 image + 6 text), 256 steps (BASELINE.json config 5);
  * example: B = 1, the reference example's 149-position prompt (144 image + 5 text), 100 steps (generate's default);
  * example_short: the same prompt and the example's max_steps = 6.
Each variant is one whole `Magma.generate` call (prefill, graph capture and the lazy EOS checks included), timed with
CUDA events around synchronised calls; the variants are alternated round by round. Each sampled or greedy pair is run
under the same torch.manual_seed, and whether the graph and the host loop emitted the same ids is reported. The card's
name, power limit and SM clock (sampled during the timed rounds) are read in the same run.

    python tools/sampled_decode_bench.py [--rounds 5] [--warmup 1] [--out FILE]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from bench import ClockSampler  # noqa: E402
from tools.hidden_states_bench import card, timed  # noqa: E402

SAMPLED = dict(temperature=0.7, top_k=0, top_p=0.9)
GREEDY = dict(temperature=0.0)
VARIANTS = {"sampled_graph": (SAMPLED, "1"), "sampled_host": (SAMPLED, "0"), "greedy_graph": (GREEDY, "1"),
            "greedy_host": (GREEDY, "0")}


def build_model():
    from magma_b200.config import MultimodalConfig
    from magma_b200.magma import Magma

    mc = MultimodalConfig(batch_size=32, train_steps=1, encoder_name="clip_vit_large",
                          adapter_config={"mlp": {"adapter_type": "normal", "downsample_factor": 4}}, image_seq_len=2,
                          use_image_embed_layernorm=True, image_size=224)
    model = Magma(mc, device=torch.device("cuda:0"), init_seed=0)
    model.eval()
    model.lm.lm_head.bias.data[model.eos_token] = -1e4  # never emit EOS: every call runs all its steps
    model.lm.invalidate()
    return model


def prompts(model):
    g = torch.Generator().manual_seed(0)
    images = torch.randn(32, 3, 224, 224, generator=g).cuda().to(torch.bfloat16)
    text = torch.randint(0, 50000, (32, 6), generator=g).cuda()
    config5 = model.embed([images, text])
    # 149 positions as the example's embeddings have them; the values are text-token embeddings (random ids)
    example = model.word_embedding(torch.randint(0, 50000, (1, 149), generator=g).cuda()).to(torch.bfloat16)
    return {"config5": (config5, 256), "example": (example, 100), "example_short": (example, 6)}


def run_case(model, name, emb, steps, rounds, warmup):
    outs = {}

    def call(kw, graph_env, key):
        def fn():
            os.environ["MB200_DECODE_GRAPH"] = graph_env
            torch.manual_seed(1234)
            outs[key] = model.generate(emb, max_steps=steps, decode=False, **kw)
        return fn

    fns = {k: call(kw, env, k) for k, (kw, env) in VARIANTS.items()}
    times = {k: [] for k in fns}
    sampler = ClockSampler()
    for r in range(warmup + rounds):
        if r == warmup:
            sampler.mark()
        for k, fn in fns.items():
            t = timed(fn)
            if r >= warmup:
                times[k].append(t)
    clocks = sampler.stop()
    B, s0 = emb.shape[0], emb.shape[1]
    same = {"sampled": bool(torch.equal(outs["sampled_graph"], outs["sampled_host"])),
            "greedy": bool(torch.equal(outs["greedy_graph"], outs["greedy_host"]))}
    rows = []
    for k, ts in times.items():
        n_new = outs[k].shape[1] - s0
        med = statistics.median(ts)
        rows.append({"case": name, "variant": k, "batch": B, "prompt_len": s0, "new_tokens": n_new,
                     "median_ms": round(med, 2), "min_ms": round(min(ts), 2), "max_ms": round(max(ts), 2),
                     "ms_per_step": round(med / n_new, 3), "tokens_per_s": round(B * n_new / (med / 1e3), 1),
                     "rounds": len(ts), "ids_equal_graph_vs_host": same[k.split("_")[0]], "clocks": clocks})
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--cases", default="config5,example,example_short")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sampled_decode_bench needs a CUDA device")
    info = card()
    model = build_model()
    cases = prompts(model)
    lines = []
    for name in a.cases.split(","):
        emb, steps = cases[name]
        for row in run_case(model, name, emb, steps, a.rounds, a.warmup):
            lines.append(json.dumps({**row, **info}))
            print(lines[-1], flush=True)
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
