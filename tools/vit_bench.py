"""Time the frozen ViT-L/14 image encoder (mb200_vit_forward) at B images of 224 px: CUDA events over many forwards
after warm-up, then one forward with the per-launch GEMM timing on (mb200_prof_enable / mb200_prof_read) and, in a run
of its own, one under torch.profiler for the kernel time of attention and of everything else. The weights are seeded
random values at the scale of a trained model (power draw and clocks depend on the data). Prints the card name, power
limit and max SM clock read in the same run.

  python tools/vit_bench.py [--B 8] [--reps 50]"""
import argparse
import ctypes
import os
import subprocess
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=8)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    import torch

    from magma_b200._lib import lib
    from magma_b200.image_encoders import B200VisionTransformer

    if not torch.cuda.is_available():
        raise SystemExit("vit_bench: no CUDA device")
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    enc = B200VisionTransformer(1024, 24, 16, 14, 224, 4096, 768, device=dev).eval()
    with torch.no_grad():
        for name, p in enc.named_parameters():
            if p.dim() >= 2:  # matrices, the conv kernel, embeddings: unit-variance outputs
                p.normal_(0.0, (p.numel() // p.shape[0]) ** -0.5)
            elif name.endswith("weight"):  # LayerNorm gains
                p.fill_(1.0)
            else:  # biases
                p.normal_(0.0, 0.02)
    x = torch.randn(a.B, 3, 224, 224, device=dev)
    print(f"[VIT] card: {card()}", flush=True)
    with torch.no_grad():
        for _ in range(a.warmup):
            enc(x)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.reps):
            enc(x)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / a.reps
        L = lib()
        L.mb200_prof_enable(1)
        enc(x)
        torch.cuda.synchronize()
        g_ms, g_fl, g_by, n = ctypes.c_double(), ctypes.c_double(), ctypes.c_double(), ctypes.c_longlong()
        L.mb200_prof_read(ctypes.byref(g_ms), ctypes.byref(g_fl), ctypes.byref(g_by), ctypes.byref(n))
        L.mb200_prof_enable(0)
        from torch.profiler import ProfilerActivity, profile

        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            enc(x)
            torch.cuda.synchronize()
    kern = {"gemm": 0.0, "attention": 0.0, "other": 0.0}
    for e in prof.key_averages():
        us = e.self_device_time_total
        if us <= 0:
            continue
        kind = "gemm" if "gemm_wgmma" in e.key or "splitk" in e.key else "attention" if "attn_" in e.key else "other"
        kern[kind] += us / 1e3
    print(f"[VIT] forward B={a.B}: {ms:.3f} ms per forward over {a.reps} reps", flush=True)
    print(f"[VIT] GEMMs of one forward (per-launch events): {n.value} launches, {g_ms.value:.3f} ms "
          f"({g_fl.value / max(g_ms.value, 1e-9) / 1e9:.1f} TFLOP/s)", flush=True)
    print(f"[VIT] kernel time of one forward (torch.profiler): GEMM {kern['gemm']:.3f} ms, attention "
          f"{kern['attention']:.3f} ms ({kern['attention'] / ms * 100:.1f} % of the forward), other kernels "
          f"(LayerNorm, embedding) {kern['other']:.3f} ms", flush=True)


if __name__ == "__main__":
    main()
