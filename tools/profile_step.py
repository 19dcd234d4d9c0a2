"""Profiling driver for ncu :

  ncu --profile-from-start off --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum \
      --clock-control none --csv --log-file launches_step.csv python tools/profile_step.py
  ncu --profile-from-start off --set full --clock-control none --import-source on -k regex:gemm_wgmma \
      -o prof_gemm python tools/profile_step.py --gemm-only

Default mode: build the BASELINE config-2 model, warm up, then run exactly ONE train step inside a
cudaProfilerStart/Stop range. --gemm-only: the main GEMM shapes of one GPT-J block, standalone, inside the range."""
import argparse
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gemm-only", action="store_true")
    ap.add_argument("--decode", action="store_true")
    a = ap.parse_args()
    import torch

    dev = torch.device("cuda:0")
    if a.gemm_only:
        from magma_b200 import ops

        M, d = 1024, 4096
        shapes = [  # (name, M, N, K, a_mn, b_mn, f32)
            ("qkv_fwd", M, 3 * d, d, False, False, False),
            ("out_fwd", M, d, d, False, False, False),
            ("fc_in_fwd", M, 4 * d, d, False, False, False),
            ("fc_out_fwd", M, d, 4 * d, False, False, False),
            ("fc_out_dgrad", M, 4 * d, d, False, True, False),
            ("fc_in_dgrad", M, d, 4 * d, False, True, False),
            ("adapter_wgrad", d, 1024, M, True, True, True),
            ("lm_head", M, 50258, d, False, False, False),
        ]
        bufs = []
        for name, m, n, k, amn, bmn, f32 in shapes:
            A = torch.randn((k, m) if amn else (m, k), device=dev).to(torch.bfloat16)
            B = torch.randn((k, n) if bmn else (n, k), device=dev).to(torch.bfloat16)
            ldc = (n + 63) // 64 * 64
            C = torch.empty(m, ldc, device=dev, dtype=torch.float32 if f32 else torch.bfloat16)[:, :n]
            bufs.append((A, B, C, amn, bmn))
        for A, B, C, amn, bmn in bufs:  # warm-up
            ops.gemm(A, B, out=C, a_mn=amn, b_mn=bmn)
        torch.cuda.synchronize()
        torch.cuda.profiler.start()
        for A, B, C, amn, bmn in bufs:
            ops.gemm(A, B, out=C, a_mn=amn, b_mn=bmn)
        torch.cuda.synchronize()
        torch.cuda.profiler.stop()
        print("profiled shapes:", [s[0] for s in shapes])
        return
    from magma_b200.config import MultimodalConfig
    from magma_b200.magma import Magma
    from magma_b200.train_loop import B200Engine

    mc = MultimodalConfig(batch_size=8, train_steps=1, encoder_name="clip_vit_large",
                          adapter_config={"mlp": {"adapter_type": "normal", "downsample_factor": 4}}, image_seq_len=2,
                          image_embed_dropout_prob=0.1, use_image_embed_layernorm=True, image_size=224, seq_len=128)
    model = Magma(mc, device=dev, init_seed=0)
    if a.decode:
        model.eval()
        B = 32
        images = torch.randn(B, 3, 224, 224, device=dev).to(torch.bfloat16)
        emb = model.embed([images, torch.randint(0, 50000, (B, 6), device=dev)])
        model.generate(emb, max_steps=8, temperature=0.0, decode=False)
        torch.cuda.synchronize()
        torch.cuda.profiler.start()
        model.generate(emb, max_steps=8, temperature=0.0, decode=False)
        torch.cuda.synchronize()
        torch.cuda.profiler.stop()
        return
    model.train()
    eng = B200Engine(model, mc)
    images = torch.randn(8, 3, 224, 224, device=dev).to(torch.bfloat16)
    captions = torch.randint(0, 50256, (8, 128), device=dev)
    captions[:, 100:] = 50256

    def step():
        out = eng(images, captions)
        eng.backward(out.loss)
        eng.step()

    for _ in range(2):
        step()
    torch.cuda.synchronize()
    torch.cuda.profiler.start()
    step()
    torch.cuda.synchronize()
    torch.cuda.profiler.stop()
    print("profiled one train step")


if __name__ == "__main__":
    main()
