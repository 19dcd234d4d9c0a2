"""Device-side timing (CUDA graph replay, no host launch cost in the number) of the GEMM core on the shapes where the
fixed per-launch cost and the epilogue dominate: single-wave GEMMs of the GPT-J block at M = 1024, the adapter pair, the
short-K ViT-L/14 GEMMs at M = 2056, and a K sweep that separates fixed cost (ramp + exposed last epilogue) from the
mainloop slope. Weights rotate through > L2 for the long-K shapes; activations stay L2-resident as in the step.

  python tools/epi_bench.py [--only sweep,vit,adapter,block]"""
import argparse
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))


def timed(fn, reps, s):
    import torch

    with torch.cuda.stream(s):
        for i in range(3):
            fn(i)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            for i in range(reps):
                fn(i)
        g.replay()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(s)
        for _ in range(3):
            g.replay()
        e1.record(s)
        torch.cuda.synchronize()
    return e0.elapsed_time(e1) / (3 * reps) * 1e3  # us


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default="sweep,vit,adapter,block")
    a = ap.parse_args()
    only = set(a.only.split(","))
    import torch

    from magma_b200 import ops

    dev = torch.device("cuda:0")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())

    def rnd(*shape, scale=0.05):
        return (torch.randn(*shape, device=dev) * scale).to(torch.bfloat16)

    def case(tag, M, N, K, *, bias=False, act=0, res=0, aux=False, a_mn=False, b_mn=False, f32=False, force_bn=0,
             dact=0, check=True, use_ws=True, rope=0, cublas=False):
        nbuf = max(1, min(8, int(200e6 // (N * K * 2)) + 1)) if N * K * 2 > 30e6 else 1
        Bs = [rnd(K, N) if b_mn else rnd(N, K) for _ in range(nbuf)]
        A = rnd(K, M, scale=1.0) if a_mn else rnd(M, K, scale=1.0)
        C = torch.empty(M, N, device=dev, dtype=torch.float32 if f32 else torch.bfloat16)
        kw = dict(a_mn=a_mn, b_mn=b_mn, force_bn=force_bn, b_static=not a_mn)  # K-major-A cases are weight GEMMs
        if bias:
            kw["bias"] = rnd(N)
        if act:
            kw["act"] = act
        if aux:
            kw["aux_out"] = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
        if dact:
            kw["dact"] = dact
            kw["aux_in"] = rnd(M, N, scale=1.0)
        if res >= 1:
            kw["res1"] = rnd(M, N, scale=1.0)
        if res >= 2:
            kw["res2"] = rnd(M, N, scale=1.0)
        if rope:  # GPT-J's rotary epilogue on the q,k thirds of a fused qkv output (S = 128, head_dim 256, 64 rotary dims)
            kw.update(rope_tab=ops.rope_table(128, 64, device=dev), rope_mode=rope, rope_S=128, rope_hd=256, rope_rot=64,
                      rope_ncols=(2 * N // 3) if rope > 0 else N)
            check = False
        if use_ws:  # scratch lent to the GEMM core (split-K of few-tile long-K shapes), as the schedules do
            kw["splitk_ws"] = torch.empty(32 << 20, device=dev, dtype=torch.float32)
        us = timed(lambda i: ops.gemm(A, Bs[i % nbuf], out=C, **kw), max(8, 2 * nbuf), s)
        tf = 2.0 * M * N * K / us / 1e6
        # the same launch on the runtime epilogue form (the same kernel when no compiled form matches the case)
        us_rt = timed(lambda i: ops.gemm(A, Bs[i % nbuf], out=C, generic_epilogue=True, **kw), max(8, 2 * nbuf), s)
        ref = f"  runtime form {us_rt:8.1f} us"
        if cublas:  # torch.matmul on the same operands (no epilogue): the rate this card reaches at this shape
            Ct = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
            Af = A.t() if a_mn else A
            us_ref = timed(lambda i: torch.matmul(Af, Bs[i % nbuf] if b_mn else Bs[i % nbuf].t(), out=Ct),
                           max(8, 2 * nbuf), s)
            ref += f"  cuBLAS {us_ref:8.1f} us {2.0 * M * N * K / us_ref / 1e6:7.1f} TFLOP/s"
        err = float("nan")
        if check:
            ops.gemm(A, Bs[0], out=C, **kw)
            torch.cuda.synchronize()
            Af = A.float().t() if a_mn else A.float()
            Bf = Bs[0].float() if b_mn else Bs[0].float().t()
            want = Af @ Bf
            if bias:
                want = want + kw["bias"].float()
            if act == ops.ACT_RELU:
                want = torch.relu(want)
            elif act == ops.ACT_GELU_NEW:
                want = torch.nn.functional.gelu(want, approximate="tanh")
            elif act == ops.ACT_QUICK_GELU:
                want = want * torch.sigmoid(1.702 * want)
            if dact:
                want = None
            if want is not None:
                if res >= 1:
                    want = want + kw["res1"].float()
                if res >= 2:
                    want = want + kw["res2"].float()
                err = ((C.float() - want).norm() / want.norm()).item()
        print(f"[EPI] {tag:34s} M={M:5d} N={N:5d} K={K:5d}  {us:8.1f} us  {tf:7.1f} TFLOP/s  rel_err={err:.1e}{ref}",
              flush=True)
        return us

    if "sweep" in only:
        # fixed cost vs mainloop slope: 128 tiles of 128 x 256 (one per CTA, one wave), plain / residual epilogues
        for K in (64, 256, 1024, 4096, 16384):
            case("sweep plain", 1024, 4096, K)
        for K in (64, 1024, 4096):
            case("sweep bias+res2", 1024, 4096, K, bias=True, res=2)
        # epilogue pace: 2048 tiles of 128 x 256, 15.5 per CTA, one or four k-blocks each (time / tiles-per-CTA =
        # epilogue time per tile)
        for K in (64, 256):
            case("pace plain   (15.5 tiles/CTA)", 8192, 8192, K)
            case("pace gelu+aux(15.5 tiles/CTA)", 8192, 8192, K, bias=True, act=ops.ACT_GELU_NEW, aux=True)
            case("pace res1    (15.5 tiles/CTA)", 8192, 8192, K, res=1)
            case("pace dact    (15.5 tiles/CTA)", 8192, 8192, K, dact=ops.DACT_GELU_NEW)
    if "block" in only:
        M, d = 1024, 4096
        case("qkv fwd", M, 3 * d, d, cublas=True)
        case("qkv fwd (+rope epilogue)", M, 3 * d, d, rope=1, cublas=True)
        case("out fwd (+res1)", M, d, d, res=1, cublas=True)
        case("fc_in fwd (bias+gelu+aux)", M, 4 * d, d, bias=True, act=ops.ACT_GELU_NEW, aux=True, cublas=True)
        case("fc_out fwd (+bias)", M, d, 4 * d, bias=True, cublas=True)
        case("fc_out dgrad (dgelu)", M, 4 * d, d, b_mn=True, dact=ops.DACT_GELU_NEW, cublas=True)
        case("fc_out dgrad shape, plain", M, 4 * d, d, b_mn=True)  # the floor for the dgelu epilogue above
        case("fc_in dgrad", M, d, 4 * d, b_mn=True, cublas=True)
        case("qkv dgrad (+res1)", M, d, 3 * d, b_mn=True, res=1, cublas=True)
        case("lm_head", M, 50258 // 8 * 8, d, bias=True, cublas=True)
    if "adapter" in only:
        M, d, r = 1024, 4096, 1024
        case("adapter down (bias+relu)", M, r, d, bias=True, act=ops.ACT_RELU)
        case("adapter down (no scratch: bn=64)", M, r, d, bias=True, act=ops.ACT_RELU, use_ws=False)
        case("adapter dgrad-up (no scratch)", M, r, d, b_mn=True, dact=ops.DACT_RELU, use_ws=False)
        case("adapter up (bias+res2)", M, d, r, bias=True, res=2)
        case("adapter dgrad-up (drelu)", M, r, d, b_mn=True, dact=ops.DACT_RELU)
        case("adapter dgrad-down (+res1)", M, d, r, b_mn=True, res=1)
        case("adapter wgrad Wu (f32)", d, r, M, a_mn=True, b_mn=True, f32=True)
        case("adapter wgrad Wd (f32)", r, d, M, a_mn=True, b_mn=True, f32=True)
    if "vit" in only:
        M, w = 2056, 1024
        case("vit qkv (+bias)", M, 3 * w, w, bias=True)
        case("vit out (+bias+res1)", M, w, w, bias=True, res=1)
        case("vit fc (+bias+quickgelu)", M, 4 * w, w, bias=True, act=ops.ACT_QUICK_GELU)
        case("vit proj (+bias+res1)", M, w, 4 * w, bias=True, res=1)


if __name__ == "__main__":
    main()
