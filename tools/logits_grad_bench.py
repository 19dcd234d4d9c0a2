"""Cost of a loss on the training logits at full size on one GPU.

GPT-J-6B with config 2's MLP adapters (normal, downsample_factor 4) and Magma's vocabulary of 50258 (the logits'
gradient rows 4-byte aligned) through B200GPTJForCausalLM, at config 2's B = 8,
S = 128 (stored activations) and at B = 8, S = 2048 (recomputed activations). With CUDA events around synchronised
steps (forward + loss.backward()), the variants alternated round by round:
  * ce: the runtime's own out.loss;
  * ce_aux: out.loss + 1e-4 * z-loss on out.logits (the logits' gradient joins the CE gradient at the LM head);
  * logits_only: no labels, F.cross_entropy on out.logits in PyTorch.
Reported separately, each as median and spread:
  * the PyTorch loss's own time (forward + backward of the auxiliary loss on a detached logits tensor);
  * the runtime's added time: ce_aux's step minus ce's step minus the PyTorch loss's time;
  * mb200_logits_grad_combine alone, and its achieved bytes/s (6 bytes per logit: read dCE and G, write the sum)
    against the H100 SXM data sheet's 3.35 TB/s, at V = 50258 and at get_gptj's V = 50400 (16-byte aligned rows).
The card's name and power limit are read in the same run. One JSON line per result.

    python tools/logits_grad_bench.py [--rounds 5] [--warmup 2] [--out FILE]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from tools.hidden_states_bench import alternate, card, timed  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def spread(ts):
    return {"median_ms": round(statistics.median(ts), 4), "min_ms": round(min(ts), 4), "max_ms": round(max(ts), 4),
            "n": len(ts)}


def model():
    from magma_b200.adapters import Adapter
    from magma_b200.language_model import get_gptj

    lm = get_gptj(device="cuda:0").init_weights(seed=0)
    lm.resize_token_embeddings(50258)  # Magma's vocabulary (magma/magma.py:50)
    torch.manual_seed(0)
    for blk in lm.transformer.h:
        blk.mlp = torch.nn.Sequential(blk.mlp, Adapter(dim=lm.config.hidden_size, downsample_factor=4).to("cuda:0"))
    lm.invalidate()
    return lm


def case(lm, B, S, rounds, warmup):
    from magma_b200 import ops

    V = lm.config.vocab_size
    g = torch.Generator(device="cuda").manual_seed(0)
    x = (0.5 * torch.randn(B, S, lm.config.hidden_size, generator=g, device="cuda")).to(torch.bfloat16)
    labels = torch.randint(0, V, (B, S), generator=g, device="cuda")
    params = [p for _, p in lm.adapter_parameters()]

    def zloss(logits):
        return 1e-4 * (torch.logsumexp(logits.float(), -1) ** 2).mean()

    def ce(logits):
        return F.cross_entropy(logits[:, :-1].float().reshape(-1, V), labels[:, 1:].reshape(-1))

    def step(kind):
        for p in params:
            p.grad = None
        xr = x.clone().requires_grad_(True)
        out = lm(inputs_embeds=xr, labels=None if kind == "logits_only" else labels)
        loss = {"ce": lambda: out.loss, "ce_aux": lambda: out.loss + zloss(out.logits),
                "logits_only": lambda: ce(out.logits)}[kind]()
        loss.backward()

    lm._ws.clear()
    steps = alternate({k: (lambda k=k: step(k)) for k in ("ce", "ce_aux", "logits_only")}, rounds, warmup)
    recompute = lm._workspace_ex(B, S)[1]
    lm._ws.clear()

    # the PyTorch loss alone, on logits of the runtime's layout
    lg = torch.randn(B * S, lm.ldv, device="cuda").to(torch.bfloat16).view(B, S, lm.ldv)[..., :V]

    def torch_loss(f):
        z = lg.detach().requires_grad_(True)
        torch.autograd.grad(f(z), z)

    loss_t = alternate({"zloss": lambda: torch_loss(zloss), "ce": lambda: torch_loss(ce)}, rounds, warmup)

    med = {k: statistics.median(v) for k, v in steps.items()}
    added = [t - med["ce"] - statistics.median(loss_t["zloss"]) for t in steps["ce_aux"]]
    tag = {"B": B, "S": S, "V": V, "recompute": recompute}
    rows = [{**tag, "result": f"step_{k}", **spread(v)} for k, v in steps.items()]
    rows += [{**tag, "result": f"torch_loss_{k}", **spread(v)} for k, v in loss_t.items()]
    rows.append({**tag, "result": "runtime_added_ce_aux", **spread(added)})
    del lg
    # mb200_logits_grad_combine alone, G as autograd hands it over ([B*S, V] contiguous): at Magma's V = 50258 its
    # rows are 4-byte aligned only (3 rows in 4 take the four-u32 loads), at get_gptj's V = 50400 all 16-byte aligned
    M = B * S
    reps = 20
    for Vk in (V, 50400):
        ldv = (Vk + 63) // 64 * 64
        dce = torch.randn(M, ldv, device="cuda").to(torch.bfloat16)
        G = torch.randn(M, Vk, device="cuda").to(torch.bfloat16)
        out = torch.empty(M, ldv, dtype=torch.bfloat16, device="cuda")

        def combine():
            for _ in range(reps):
                ops.logits_grad_combine(dce, G, out, 1.0)

        comb = [t / reps for t in alternate({"c": combine}, rounds, warmup)["c"]]
        moved = 6 * M * Vk
        rows.append({**tag, "V": Vk, "result": "combine_kernel", **spread(comb), "bytes": moved,
                     "bytes_per_s": round(moved / (statistics.median(comb) * 1e-3), 1),
                     "share_of_3.35TB/s": round(moved / (statistics.median(comb) * 1e-3) / HBM_BYTES_PER_S, 3),
                     "lower_bound_ms": round(moved / HBM_BYTES_PER_S * 1e3, 4)})
        del dce, G, out
    torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("logits_grad_bench needs a CUDA device")
    info = card()
    lm = model()
    rows = case(lm, 8, 128, a.rounds, a.warmup) + case(lm, 8, 2048, a.rounds, a.warmup)
    lines = [json.dumps({**r, **info}) for r in rows]
    print("\n".join(lines))
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
