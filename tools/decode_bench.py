"""Decode benchmark (BASELINE.json config 5): Magma.generate, batch 32, 224x224 image prefix (+6 text tokens),
256 autoregressive steps, temperature 0 (greedy), KV cache. Reports tokens/s and the HBM roofline fraction
(algorithmic bytes/step = bf16 weights 12.16 GB + KV read)."""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=256)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--temperature", type=float, default=0.0, help="0 = greedy (argmax kernel), > 0 = mb200_sample")
    a = ap.parse_args()
    import torch

    from magma_b200.config import MultimodalConfig
    from magma_b200.magma import Magma

    dev = torch.device("cuda:0")
    mc = MultimodalConfig(batch_size=a.batch, train_steps=1, encoder_name="clip_vit_large",
                          adapter_config={"mlp": {"adapter_type": "normal", "downsample_factor": 4}}, image_seq_len=2,
                          use_image_embed_layernorm=True, image_size=224)
    model = Magma(mc, device=dev, init_seed=0)
    model.eval()
    B = a.batch
    images = torch.randn(B, 3, 224, 224, device=dev).to(torch.bfloat16)
    text = torch.randint(0, 50000, (B, 6), device=dev)
    # never emit EOS so that every run executes all steps (random weights)
    model.lm.lm_head.bias.data[50256] = -1e4
    model.lm.invalidate()
    emb = model.embed([images, text])
    out = model.generate(emb, max_steps=8, temperature=a.temperature, decode=False)  # warm-up
    torch.cuda.synchronize()
    best = None
    for _ in range(a.reps):
        t0 = time.time()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = model.generate(emb, max_steps=a.steps, temperature=a.temperature, decode=False)
        e1.record()
        host_ms = (time.time() - t0) * 1e3  # time to ENQUEUE the whole generation (host-bound if ~ the device time)
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
        best = ms if best is None else min(best, ms)
    n_new = out.shape[1] - emb.shape[1]
    s0 = emb.shape[1]
    ms_step = best / n_new
    w_bytes = 28 * 201_355_264 * 2 + 235_024_384 * 2 + (50258 * 4096 + 50258) * 2
    kv_bytes = B * (s0 + n_new / 2) * 28 * 2 * 4096 * 2
    peaks = json.load(open(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json"))) if os.path.exists(
        os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")) else {"hbm_gbs": 6650.0}
    gbs = (w_bytes + kv_bytes) / (ms_step / 1e3) / 1e9
    print(json.dumps({"metric": "decode tokens/s (%s, KV cache)" % ("greedy" if a.temperature == 0 else f"sampled T={a.temperature} top_p=0.9"), "value": B * n_new / (best / 1e3), "unit": "tokens/s",
                      "batch": B, "prompt_len": s0, "new_tokens": n_new, "ms_per_step": ms_step,
                      "host_enqueue_ms_per_step": host_ms / n_new,
                      "roofline": {"bound": "hbm", "achieved": gbs, "peak": peaks["hbm_gbs"], "unit": "GB/s",
                                   "frac": gbs / peaks["hbm_gbs"], "bytes_per_step": w_bytes + kv_bytes},
                      "tokens_head": out[0, s0:s0 + 8].tolist()}))


if __name__ == "__main__":
    main()
