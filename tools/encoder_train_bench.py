"""Step time with a TRAINABLE image encoder (freeze_img_encoder: false, MAGMA_v1.yml's encoder setting) next to the
frozen-encoder step of bench.py: BASELINE config 2 sizes (ViT-L/14 + GPT-J-6B + MLP adapters, B = 8, S = 128).

  python tools/encoder_train_bench.py [--steps 10]

Prints one JSON line per variant: ms/step, samples/s, trainable parameters, and the ViT's share of algorithmic FLOPs
(forward 0.162 TFLOP/image, backward 2x)."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))


def run(freeze, steps, image_enc_lr):
    import torch

    from magma_b200.config import MultimodalConfig
    from magma_b200.magma import Magma
    from magma_b200.train_loop import B200Engine

    dev = torch.device("cuda:0")
    B, S = 8, 128
    mc = MultimodalConfig(batch_size=B, train_steps=steps, encoder_name="clip_vit_large",
                          adapter_config={"mlp": {"adapter_type": "normal", "downsample_factor": 4}}, image_seq_len=2,
                          image_embed_dropout_prob=0.1, use_image_embed_layernorm=True, image_size=224, seq_len=S,
                          freeze_img_encoder=freeze, image_enc_lr=image_enc_lr, lr=8e-4, lr_decay_iters=300000)
    model = Magma(mc, device=dev, init_seed=0)
    model.train()
    eng = B200Engine(model, mc)
    g = torch.Generator().manual_seed(0)
    images = torch.randn(B, 3, 224, 224, generator=g).to(dev).to(torch.bfloat16)
    caps = torch.randint(0, 50256, (B, S), generator=g)
    caps[:, 100:] = 50256
    caps = caps.to(dev)

    def step():
        out = eng(images, caps)
        eng.backward(out.loss)
        eng.step()
        return out.loss

    for _ in range(3):
        loss = step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        loss = step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    line = {"freeze_img_encoder": freeze, "image_enc_lr": image_enc_lr, "ms_per_step": ms,
            "samples_per_s": B / (ms / 1e3), "trainable_params": int(model.arena.numel), "loss": float(loss),
            "max_mem_gib": torch.cuda.max_memory_allocated() / 2**30}
    print(json.dumps(line), flush=True)
    del eng, model
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    a = ap.parse_args()
    run(True, a.steps, None)
    run(False, a.steps, 2.0e-6)


if __name__ == "__main__":
    main()
