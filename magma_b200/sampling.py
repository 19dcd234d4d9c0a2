"""Sampling / decode loop — drop-in for magma/sampling.py (same function names and arguments).

`generate` keeps the reference's structure (prefill with inputs_embeds, then one token per step through the KV
cache) but: the cache is a static [layer,B,H,S_max,hd] buffer appended in place by the fused decode-attention
kernel (no torch.cat growth), the LM head runs on the B last-position rows only, temperature-0 argmax is a device
kernel with torch.argmax tie-breaking (lowest index), and the all-EOS early-exit check (sampling.py:109) is polled
every `eos_check_every` steps instead of forcing a host sync per token — emitted tokens are identical because
rows are truncated at the first all-EOS step afterwards. On the GPU the decode step, greedy or sampled, runs as ONE
replayed CUDA graph whose state (cache position included) lives in device memory.

`top_p_filter`, `top_k_filter` and `remove_tokens_after_eos` below are the reference's public host-side helpers kept
VERBATIM in behaviour and near-verbatim in text (magma/sampling.py:7-40, ~20 lines, each cited): callers of the
reference import them by name and the nucleus filter's inverted comparison is a quirk that must be reproduced, not
fixed. `generate` itself does not use them — it samples with the one-launch kernel `mb200_sample` (`mb200_sample_dev` in
the replayed graph)."""
import os
from typing import List, Union

import torch
import torch.nn.functional as F

from . import ops

# The library's sampler. A caller may replace ops.sample (a custom draw, a recorder); generate then keeps calling it
# once per step (see use_graph below), as it did before sampled decoding was captured in the graph.
_LIB_SAMPLE = ops.sample


def top_p_filter(logits, threshold: float = 0.9):
    """magma/sampling.py:7-19 — reproduced including its inverted-nucleus comparison (`cum_probs < 1 - threshold`,
    shifted right by one). This torch statement is the public filter function of the reference API; `generate` itself
    samples with the fused device kernel (`ops.sample` -> mb200_sample), which applies the same rule without a sort."""
    sorted_logits, sorted_indices = torch.sort(logits, descending=True)
    cum_probs = torch.cumsum(F.softmax(sorted_logits, dim=-1), dim=-1)
    sorted_indices_to_remove = cum_probs < (1 - threshold)
    sorted_indices_to_remove[..., 1:] = sorted_indices_to_remove[..., :-1].clone()
    sorted_indices_to_remove[..., 0] = 0
    sorted_logits[sorted_indices_to_remove] = float("-inf")
    return sorted_logits.scatter(1, sorted_indices, sorted_logits)


def top_k_filter(logits, k):
    """magma/sampling.py:22-30."""
    assert k > 0
    val, ind = torch.topk(logits, k)
    probs = torch.full_like(logits, float("-inf"))
    probs.scatter_(1, ind, val)
    return probs


def remove_tokens_after_eos(tensor, eos_token, image_token):
    """magma/sampling.py:33-40."""
    eos_index = (tensor == eos_token).nonzero()
    if eos_index.any():
        tensor[eos_index[0]:] = eos_token
    tensor = tensor.tolist()
    return [i for i in tensor if (not i == image_token) and (not i == eos_token)]


@torch.no_grad()
def generate(model, embeddings, max_steps: int = 100, temperature: float = 0.7, top_k: int = 0, top_p: float = 0.9,
             eos_token: int = None, decode: bool = True, eos_check_every: int = 16) -> Union[List[str], torch.Tensor]:
    """magma/sampling.py:43-121."""
    eos_token = eos_token or model.eos_token
    was_training = model.training
    model.eval()
    lm = model.lm
    b, s, _ = embeddings.shape
    dev = embeddings.device
    out = torch.full((b, s + max_steps), model.image_token, dtype=torch.long, device=dev)  # :75, preallocated
    cache = None
    n_done = max_steps
    all_eos = torch.zeros(max_steps, dtype=torch.bool, device=dev)
    # Philox seed of this call, drawn from torch's CPU generator: reproducible under torch.manual_seed, new per call
    sample_seed = int(torch.randint(0, 2**62, (1,)).item()) if temperature != 0.0 else 0
    # On the GPU, after the prefill, ONE decode step — embedding of the token emitted last, the LM step, the next token
    # (argmax at T = 0, else mb200_sample_dev), store + EOS flag + position increment — is captured in a CUDA graph whose
    # only state is device memory (the cache position included) and replayed per token: no per-step host work besides the
    # replay, same kernels in the same order as the host-driven loop. The sampler reads its Philox offset from the cache
    # position (position - s + 1 = the step index i the host loop passes), so with the same seed every draw, and every
    # token id, is identical. MB200_DECODE_GRAPH=0 keeps the host-driven loop, and so does a replaced ops.sample at T > 0:
    # the graph would bypass it.
    use_graph = (dev.type == "cuda" and max_steps > 2 and os.environ.get("MB200_DECODE_GRAPH", "1") != "0"
                 and (temperature == 0.0 or ops.sample is _LIB_SAMPLE))
    graph = None
    for i in range(max_steps):
        if i == 0:
            from .language_model import KVCache

            cfg = lm.config
            cache = KVCache(cfg.num_layers, b, cfg.num_heads, s + max_steps, cfg.hidden_size // cfg.num_heads, dev)
            logits = lm.decode_logits(embeddings, cache)                       # :81-85 (prefill)
        elif use_graph:
            if graph is None:
                pos_dev = torch.tensor([s], dtype=torch.int32, device=dev)      # column of the token fed next
                flags = torch.zeros(max_steps, dtype=torch.uint8, device=dev)
                x_buf = torch.empty(b, 1, cfg.hidden_size, dtype=torch.bfloat16, device=dev)
                lg_buf = torch.empty(b, lm.ldv, dtype=torch.bfloat16, device=dev)
                nxt_buf = torch.empty(b, dtype=torch.int64, device=dev)
                V = lm.lm_head.weight.shape[0]
                eos_i = -1 if eos_token is None else int(eos_token)
                wte = lm.transformer.wte.compute_weight()  # the bf16 table, also while the embedding trains

                def dev_step():
                    ops.decode_embed(out, pos_dev, wte, x_buf)
                    lm.decode_step_dev(x_buf, cache, pos_dev, lg_buf)
                    if temperature == 0.0:
                        ops.argmax(lg_buf, V, out=nxt_buf)
                    else:
                        ops.sample_dev(lg_buf[:, :V], pos_dev, s, temperature, top_k, top_p, sample_seed, nxt_buf)
                    ops.decode_advance(nxt_buf, out, pos_dev, eos_i, flags, s)

                dev_step()                                                      # step 1 eagerly (also warms every launch)
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph):
                    dev_step()
            else:
                graph.replay()
            cache.pos += 1
            if eos_token is not None and ((i + 1) % eos_check_every == 0 or i == max_steps - 1):
                hit = (all_eos[: i + 1] | flags[: i + 1].bool()).nonzero()      # :109, evaluated lazily
                if hit.numel():
                    n_done = int(hit[0]) + 1
                    break
            continue
        else:
            x = lm.transformer.wte(out[:, s + i - 1: s + i])                    # :88-90 (input_ids path)
            logits = lm.decode_logits(x, cache)
        if temperature == 0.0:
            next_token = ops.argmax(logits.contiguous() if logits.stride(-1) != 1 else logits, logits.shape[-1])  # :97
        else:
            # :92-105 in one launch: top-k filter, the reference's nucleus filter, softmax(logits / T), multinomial
            lg = logits if logits.stride(-1) == 1 else logits.contiguous()
            next_token = ops.sample(lg, temperature, top_k=top_k, top_p=top_p, seed=sample_seed, offset=i)
        out[:, s + i] = next_token                                              # :107
        if eos_token is not None:
            all_eos[i] = (next_token == eos_token).all()                        # :109, evaluated lazily
            if (i + 1) % eos_check_every == 0 or i == max_steps - 1:
                hit = all_eos[: i + 1].nonzero()
                if hit.numel():
                    n_done = int(hit[0]) + 1
                    break
    out = out[:, : s + n_done]
    if decode:
        captions = []
        for row in out:
            row = remove_tokens_after_eos(row, eos_token, model.image_token)
            captions.append(model.tokenizer.decode(row))
        out = captions
    model.train(was_training)
    return out
