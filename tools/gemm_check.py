"""GPU diagnostic sweep for the wgmma GEMM core (development tool; the judged parity tests live in tests/).

Usage on an H100:  python tools/gemm_check.py            # runs every group in its own subprocess
                      python tools/gemm_check.py --group majors
Each case prints max-abs / relative-Frobenius error against an fp32 torch matmul of the same bf16 inputs.
"""
import argparse
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

GROUPS = ["basic", "majors", "tails", "epilogue", "batched", "pair", "splitk", "smallm", "perf"]


def ref_gemm(A, B, a_mn, b_mn):
    import torch

    Af = A.float().transpose(-1, -2) if a_mn else A.float()
    Bf = B.float() if b_mn else B.float().transpose(-1, -2)
    return Af @ Bf


def report(name, got, want, tol=2e-2):
    import torch

    got = got.float()
    err = (got - want).abs().max().item()
    rel = ((got - want).norm() / (want.norm() + 1e-12)).item()
    ok = rel < tol and err == err
    print(f"[{'OK' if ok else 'FAIL'}] {name}: max_abs={err:.4e} rel_fro={rel:.4e}", flush=True)
    return ok


def untouched(name, t, value):
    """Sentinel check: a region the GEMM must not write still holds `value` everywhere."""
    bad = int((t != value).sum().item())
    print(f"[{'OK' if bad == 0 else 'FAIL'}] {name}: {bad} of {t.numel()} sentinel elements overwritten", flush=True)
    return bad == 0


def mk(shape, a_mn, dev, scale=1.0):
    import torch

    *b, r, c = shape
    t = torch.randn(*b, c, r, device=dev) if a_mn else torch.randn(*b, r, c, device=dev)
    return (t * scale).to(torch.bfloat16)


def run_group(g):
    import torch

    from magma_b200 import ops

    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    ok = True
    if g == "basic":
        for bn in (128, 64, 256):
            A, B = mk((256, 256), False, dev), mk((256, 256), False, dev)
            C = ops.gemm(A, B, force_bn=bn)
            torch.cuda.synchronize()
            ok &= report(f"basic KK M=N=K=256 bn={bn}", C, ref_gemm(A, B, False, False))
        A, B = mk((1024, 4096), False, dev), mk((4096, 4096), False, dev)
        C = ops.gemm(A, B)
        torch.cuda.synchronize()
        ok &= report("basic KK 1024x4096x4096 auto", C, ref_gemm(A, B, False, False))
    elif g == "majors":
        for a_mn in (False, True):
            for b_mn in (False, True):
                for bn in (64, 128, 256):
                    M, N, K = 384, 512, 320
                    A, B = mk((M, K), a_mn, dev), mk((N, K), b_mn, dev)
                    C = ops.gemm(A, B, a_mn=a_mn, b_mn=b_mn, force_bn=bn)
                    torch.cuda.synchronize()
                    ok &= report(f"majors a_mn={int(a_mn)} b_mn={int(b_mn)} bn={bn}", C, ref_gemm(A, B, a_mn, b_mn))
    elif g == "tails":
        for a_mn in (False, True):
            for b_mn in (False, True):
                M, N, K = 200, 328, 328  # M tail, N tail (bn=128 -> 72 cols in last tile), K tail (328 = 5*64+8)
                A, B = mk((M, K), a_mn, dev), mk((N, K), b_mn, dev)
                C = ops.gemm(A, B, a_mn=a_mn, b_mn=b_mn, force_bn=128)
                torch.cuda.synchronize()
                ok &= report(f"tails a_mn={int(a_mn)} b_mn={int(b_mn)} M=200 N=328 K=328", C, ref_gemm(A, B, a_mn, b_mn))
        # ragged N with padded ldc (lm_head style: N not a multiple of 8)
        M, N, K, ldc = 130, 1002, 256, 1008
        A, B = mk((M, K), False, dev), mk((N, K), False, dev)
        buf = torch.full((M, ldc), 7.0, device=dev, dtype=torch.bfloat16)
        ops.gemm(A, B, out=buf[:, :N])
        torch.cuda.synchronize()
        ok &= report("tails ragged N=1002 ldc=1008", buf[:, :N], ref_gemm(A, B, False, False))
        ok &= bool((buf[:, N:] == 7.0).all().item())
        print("   padding untouched:", bool((buf[:, N:] == 7.0).all().item()))
        # tiny M (image-prefix style) and K-as-MN-major with ragged K
        A, B = mk((8, 768), False, dev), mk((8192, 768), False, dev)
        C = ops.gemm(A, B)
        torch.cuda.synchronize()
        ok &= report("tails tiny M=8 N=8192 K=768", C, ref_gemm(A, B, False, False))
        # f32 output + accumulate
        A, B = mk((256, 192), True, dev), mk((320, 192), True, dev)
        C = torch.ones(256, 320, device=dev, dtype=torch.float32)
        ops.gemm(A, B, out=C, a_mn=True, b_mn=True, accumulate=True)
        torch.cuda.synchronize()
        ok &= report("f32 accumulate (wgrad style, MN/MN)", C, ref_gemm(A, B, True, True) + 1.0, tol=5e-3)
    elif g == "epilogue":
        import torch.nn.functional as F

        M, N, K = 256, 512, 256
        A, B = mk((M, K), False, dev, 0.5), mk((N, K), False, dev, 0.125)
        bias = (torch.randn(N, device=dev)).to(torch.bfloat16)
        base = ref_gemm(A, B, False, False)
        pre = base + bias.float()
        aux = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
        C = ops.gemm(A, B, bias=bias, act=ops.ACT_GELU_NEW, aux_out=aux)
        torch.cuda.synchronize()
        ok &= report("bias+gelu_new", C, F.gelu(pre, approximate="tanh"))
        ok &= report("aux_out (pre-activation)", aux, pre)
        C = ops.gemm(A, B, bias=bias, act=ops.ACT_RELU)
        ok &= report("bias+relu", C, F.relu(pre))
        C = ops.gemm(A, B, bias=bias, act=ops.ACT_QUICK_GELU)
        ok &= report("bias+quick_gelu", C, pre * torch.sigmoid(1.702 * pre))
        r1, r2 = mk((M, N), False, dev), mk((M, N), False, dev)
        C = ops.gemm(A, B, bias=bias, res1=r1, res2=r2, alpha=0.5)
        ok &= report("alpha+bias+res1+res2", C, 0.5 * base + bias.float() + r1.float() + r2.float())
        # dact gelu: out = acc * gelu'(aux_in)
        x = mk((M, N), False, dev)
        xf = x.float().requires_grad_(True)
        F.gelu(xf, approximate="tanh").sum().backward()
        C = ops.gemm(A, B, aux_in=x, dact=ops.DACT_GELU_NEW)
        ok &= report("dact gelu_new", C, base * xf.grad)
        C = ops.gemm(A, B, aux_in=x, dact=ops.DACT_RELU)
        ok &= report("dact relu", C, base * (x.float() > 0).float())
        torch.cuda.synchronize()
        # fused rotary epilogue == standalone rope kernel on the plain GEMM output (fwd and inverse)
        Sx, H, hd, rot = 32, 2, 128, 64
        Mx = 4 * Sx
        A2, B2 = mk((Mx, 256), False, dev, 0.5), mk((3 * H * hd, 256), False, dev, 0.125)
        tab = ops.rope_table(Sx, rot, pos0=7, device=dev)
        for mode in (1, -1):
            fused = ops.gemm(A2, B2, rope_tab=tab, rope_mode=mode, rope_S=Sx, rope_hd=hd, rope_rot=rot,
                             rope_ncols=2 * H * hd)
            plain = ops.gemm(A2, B2, out_dtype=torch.float32)
            q = plain.view(Mx // Sx, Sx, 3, H, hd).clone()
            cs = tab[None, :, None, None, :, 0]
            sn = tab[None, :, None, None, :, 1] * mode
            x1, x2 = q[:, :, :2, :, 0:rot:2].clone(), q[:, :, :2, :, 1:rot:2].clone()
            q[:, :, :2, :, 0:rot:2] = x1 * cs - x2 * sn
            q[:, :, :2, :, 1:rot:2] = x2 * cs + x1 * sn
            ok &= report(f"fused rope epilogue mode={mode}", fused, q.view(Mx, -1))
        torch.cuda.synchronize()
    elif g == "batched":
        # attention-style strided batches: qkv [B,S,3,H,hd] -> Q/K/V views [B,H,S,hd]
        Bsz, S, H, hd = 2, 128, 4, 256
        qkv = (torch.randn(Bsz, S, 3, H, hd, device=dev) * 0.3).to(torch.bfloat16)
        q = qkv[:, :, 0].permute(0, 2, 1, 3)  # [B,H,S,hd] strided
        k = qkv[:, :, 1].permute(0, 2, 1, 3)
        v = qkv[:, :, 2].permute(0, 2, 1, 3)
        s = ops.gemm(q, k, out_dtype=torch.float32)
        torch.cuda.synchronize()
        ok &= report("batched QK^T (KK, strided, f32 out)", s, q.float() @ k.float().transpose(-1, -2), tol=5e-3)
        p = torch.softmax(s / 16.0, -1).to(torch.bfloat16)
        o = torch.empty(Bsz, S, H, hd, device=dev, dtype=torch.bfloat16)
        ops.gemm(p, v, out=o.permute(0, 2, 1, 3), b_mn=True)
        torch.cuda.synchronize()
        ok &= report("batched PV (K / MN, strided out)", o.permute(0, 2, 1, 3), p.float() @ v.float())
        # dK-style: A = dS^T (MN-major), B = Q (MN-major)
        dk = ops.gemm(p, q, a_mn=True, b_mn=True)
        torch.cuda.synchronize()
        ok &= report("batched dS^T Q (MN/MN)", dk, p.float().transpose(-1, -2) @ q.float())
        # ViT style ragged T=257, hd=64
        T, hd2, H2 = 257, 64, 3
        qkv2 = (torch.randn(Bsz, T, 3, H2, hd2, device=dev) * 0.5).to(torch.bfloat16)
        q2 = qkv2[:, :, 0].permute(0, 2, 1, 3)
        k2 = qkv2[:, :, 1].permute(0, 2, 1, 3)
        v2 = qkv2[:, :, 2].permute(0, 2, 1, 3)
        sbuf = torch.zeros(Bsz, H2, T, 264, device=dev, dtype=torch.float32)
        ops.gemm(q2, k2, out=sbuf[..., :T])
        torch.cuda.synchronize()
        ok &= report("batched ViT QK^T T=257", sbuf[..., :T], q2.float() @ k2.float().transpose(-1, -2), tol=5e-3)
        pbuf = torch.zeros(Bsz, H2, T, 264, device=dev, dtype=torch.bfloat16)
        pbuf[..., :T] = torch.softmax(sbuf[..., :T] / 8.0, -1).to(torch.bfloat16)
        o2 = torch.empty(Bsz, T, H2, hd2, device=dev, dtype=torch.bfloat16)
        ops.gemm(pbuf[..., :T], v2, out=o2.permute(0, 2, 1, 3), b_mn=True)
        torch.cuda.synchronize()
        ok &= report("batched ViT PV T=257 (ragged K)", o2.permute(0, 2, 1, 3), pbuf[..., :T].float() @ v2.float())
    elif g == "pair":
        # the 256-wide tile (force_bn=256) across every epilogue form
        import torch.nn.functional as F

        for a_mn in (False, True):
            for b_mn in (False, True):
                M, N, K = 512, 768, 320
                A, B = mk((M, K), a_mn, dev), mk((N, K), b_mn, dev)
                C = ops.gemm(A, B, a_mn=a_mn, b_mn=b_mn, force_bn=256)
                torch.cuda.synchronize()
                ok &= report(f"pair majors a_mn={int(a_mn)} b_mn={int(b_mn)}", C, ref_gemm(A, B, a_mn, b_mn))
                M, N, K = (304 if a_mn else 300), (1000 if b_mn else 1002), 328  # MN-major operands need ld % 8 == 0
                A, B = mk((M, K), a_mn, dev), mk((N, K), b_mn, dev)
                buf = torch.full((M, 1008), 7.0, device=dev, dtype=torch.bfloat16)
                ops.gemm(A, B, out=buf[:, :N], a_mn=a_mn, b_mn=b_mn, force_bn=256)
                torch.cuda.synchronize()
                ok &= report(f"pair tails a_mn={int(a_mn)} b_mn={int(b_mn)} M={M} N={N} K=328", buf[:, :N], ref_gemm(A, B, a_mn, b_mn))
                ok &= untouched(f"pair tails a_mn={int(a_mn)} b_mn={int(b_mn)} columns >= N", buf[:, N:], 7.0)
        M, N, K = 1024, 4096, 4096
        A, B = mk((M, K), False, dev), mk((N, K), False, dev)
        C = ops.gemm(A, B, force_bn=256)
        torch.cuda.synchronize()
        ok &= report("pair 1024x4096x4096", C, ref_gemm(A, B, False, False))
        M, N, K = 512, 1024, 256
        A, B = mk((M, K), False, dev, 0.5), mk((N, K), False, dev, 0.125)
        bias = torch.randn(N, device=dev).to(torch.bfloat16)
        base = ref_gemm(A, B, False, False)
        pre = base + bias.float()
        aux = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
        C = ops.gemm(A, B, bias=bias, act=ops.ACT_GELU_NEW, aux_out=aux, force_bn=256)
        ok &= report("pair bias+gelu_new+aux", C, F.gelu(pre, approximate="tanh"))
        ok &= report("pair aux_out", aux, pre)
        r1, r2 = mk((M, N), False, dev), mk((M, N), False, dev)
        C = ops.gemm(A, B, bias=bias, res1=r1, res2=r2, force_bn=256)
        ok &= report("pair bias+res1+res2", C, pre + r1.float() + r2.float())
        x = mk((M, N), False, dev)
        C = ops.gemm(A, B, aux_in=x, dact=ops.DACT_RELU, force_bn=256)
        ok &= report("pair dact relu", C, base * (x.float() > 0).float())
        Cf = torch.ones(M, N, device=dev, dtype=torch.float32)
        ops.gemm(A, B, out=Cf, accumulate=True, force_bn=256)
        ok &= report("pair f32 accumulate", Cf, base + 1.0, tol=5e-3)
        # batched (2 x 3 batches of 256 x 512 x 192)
        Ab = mk((2, 3, 256, 192), False, dev)
        Bb = mk((2, 3, 512, 192), False, dev)
        Cb = ops.gemm(Ab, Bb, force_bn=256)
        torch.cuda.synchronize()
        ok &= report("pair batched", Cb, Ab.float() @ Bb.float().transpose(-1, -2))
        # every specialised epilogue of the row-per-thread / TMA-store path (epilogue v3)
        C = ops.gemm(A, B, bias=bias, act=ops.ACT_RELU, force_bn=256)
        ok &= report("pair bias+relu", C, F.relu(pre))
        C = ops.gemm(A, B, bias=bias, act=ops.ACT_QUICK_GELU, force_bn=256)
        ok &= report("pair bias+quick_gelu", C, pre * torch.sigmoid(1.702 * pre))
        C = ops.gemm(A, B, bias=bias, act=ops.ACT_GELU_NEW, force_bn=256)
        ok &= report("pair bias+gelu_new (no aux)", C, F.gelu(pre, approximate="tanh"))
        xf = x.float().requires_grad_(True)
        F.gelu(xf, approximate="tanh").sum().backward()
        C = ops.gemm(A, B, aux_in=x, dact=ops.DACT_GELU_NEW, force_bn=256)
        ok &= report("pair dact gelu_new", C, base * xf.grad)
        C = ops.gemm(A, B, bias=bias, res1=r1, alpha=0.5, force_bn=256)
        ok &= report("pair alpha+bias+res1", C, 0.5 * base + bias.float() + r1.float())
        C = ops.gemm(A, B, bias=bias, res1=r1, act=ops.ACT_RELU_POST, force_bn=256)
        ok &= report("pair bias+res1+relu_post", C, F.relu(pre + r1.float()))
        Cf = torch.full((M, N), 3.0, device=dev, dtype=torch.float32)
        ops.gemm(A, B, out=Cf, force_bn=256)
        ok &= report("pair f32 plain (overwrites)", Cf, base, tol=5e-3)
        # ragged N (not a multiple of 8, like the 50258-wide LM head) and ragged M, with bias / residual / aux / f32
        Mr, Nr, Kr = 520, 1002, 320
        Ar, Br = mk((Mr, Kr), False, dev, 0.5), mk((Nr, Kr), False, dev, 0.125)
        br = torch.randn(Nr, device=dev).to(torch.bfloat16)
        rr_ = torch.full((Mr, 1008), 0.0, device=dev, dtype=torch.bfloat16)
        rr_[:, :Nr] = mk((Mr, Nr), False, dev)
        baser = ref_gemm(Ar, Br, False, False) + br.float()
        buf = torch.full((Mr, 1008), 7.0, device=dev, dtype=torch.bfloat16)
        ops.gemm(Ar, Br, out=buf[:, :Nr], bias=br, res1=rr_[:, :Nr], force_bn=256)
        ok &= report("pair ragged M=520 N=1002 bias+res1", buf[:, :Nr], baser + rr_[:, :Nr].float())
        ok &= untouched("pair ragged bias+res1 columns >= N", buf[:, Nr:], 7.0)
        auxr = torch.full((Mr, 1008), 5.0, device=dev, dtype=torch.bfloat16)
        buf.fill_(7.0)
        ops.gemm(Ar, Br, out=buf[:, :Nr], bias=br, act=ops.ACT_GELU_NEW, aux_out=auxr[:, :Nr], force_bn=256)
        ok &= report("pair ragged gelu+aux: C", buf[:, :Nr], F.gelu(baser, approximate="tanh"))
        ok &= report("pair ragged gelu+aux: aux", auxr[:, :Nr], baser)
        ok &= untouched("pair ragged gelu+aux C columns >= N", buf[:, Nr:], 7.0)
        ok &= untouched("pair ragged gelu+aux aux columns >= N", auxr[:, Nr:], 5.0)
        buff = torch.full((Mr, 1004), 2.0, device=dev, dtype=torch.float32)
        ops.gemm(Ar, Br, out=buff[:, :Nr], accumulate=True, force_bn=256)
        ok &= report("pair ragged f32 accumulate", buff[:, :Nr], baser - br.float() + 2.0, tol=5e-3)
        ok &= untouched("pair ragged f32 accumulate columns >= N", buff[:, Nr:], 2.0)
        # fused rotary epilogue (forward and inverse) on the pair kernel == rotation of the plain fp32 product
        Sx, H, hd, rot = 64, 2, 128, 64
        Mx = 4 * Sx
        A2, B2 = mk((Mx, 512), False, dev, 0.5), mk((3 * H * hd, 512), False, dev, 0.125)
        tab = ops.rope_table(Sx, rot, pos0=7, device=dev)
        for mode in (1, -1):
            fused = ops.gemm(A2, B2, rope_tab=tab, rope_mode=mode, rope_S=Sx, rope_hd=hd, rope_rot=rot,
                             rope_ncols=2 * H * hd, force_bn=256)
            plain = ops.gemm(A2, B2, out_dtype=torch.float32)
            qq = plain.view(Mx // Sx, Sx, 3, H, hd).clone()
            cs = tab[None, :, None, None, :, 0]
            sn = tab[None, :, None, None, :, 1] * mode
            x1, x2 = qq[:, :, :2, :, 0:rot:2].clone(), qq[:, :, :2, :, 1:rot:2].clone()
            qq[:, :, :2, :, 0:rot:2] = x1 * cs - x2 * sn
            qq[:, :, :2, :, 1:rot:2] = x2 * cs + x1 * sn
            ok &= report(f"pair fused rope epilogue mode={mode}", fused, qq.view(Mx, -1))
        # strided-batch output (attention-style: heads interleaved in the row), forced pair
        Bsz, S_, H_, hd_ = 2, 256, 2, 256
        pb = torch.softmax(torch.randn(Bsz, H_, S_, S_, device=dev), -1).to(torch.bfloat16)
        vb = (torch.randn(Bsz, S_, H_, hd_, device=dev) * 0.3).to(torch.bfloat16)
        ob = torch.empty(Bsz, S_, H_, hd_, device=dev, dtype=torch.bfloat16)
        ops.gemm(pb, vb.permute(0, 2, 1, 3), out=ob.permute(0, 2, 1, 3), b_mn=True, force_bn=256)
        ok &= report("pair batched PV into [B,S,H,hd]", ob.permute(0, 2, 1, 3), pb.float() @ vb.permute(0, 2, 1, 3).float())
    elif g == "splitk":
        import torch.nn.functional as F

        ws = torch.full((16 * 128 * 8192,), float('nan'), device=dev, dtype=torch.float32)  # scratch needs no init
        for (M, N, K, bmn) in ((32, 4096, 16384, False), (32, 4096, 8192, True), (7, 1002, 8200, False),
                               (100, 1000, 16384, False), (32, 4096, 4096, False),
                               (1152, 768, 6912, False), (300, 248, 2120, True)):  # few tiles, long K, M > 128
            A, B = mk((M, K), False, dev, 0.5), mk((N, K), bmn, dev, 0.125)
            ldc = (N + 63) // 64 * 64
            bias = torch.randn(N, device=dev).to(torch.bfloat16)
            res = mk((M, ldc), False, dev)[:, :N]
            C = torch.empty(M, ldc, device=dev, dtype=torch.bfloat16)[:, :N]
            ops.gemm(A, B, out=C, b_mn=bmn, bias=bias, act=ops.ACT_GELU_NEW, res1=res, splitk_ws=ws)
            torch.cuda.synchronize()
            want = F.gelu(ref_gemm(A, B, False, bmn) + bias.float(), approximate="tanh") + res.float()
            ok &= report(f"splitk M={M} N={N} K={K} bmn={int(bmn)} bias+gelu+res", C, want)
            C2 = torch.empty(M, ldc, device=dev, dtype=torch.bfloat16)[:, :N]
            ops.gemm(A, B, out=C2, b_mn=bmn, bias=bias, act=ops.ACT_GELU_NEW, res1=res, splitk_ws=ws)
            ok &= bool(torch.equal(C, C2))  # deterministic
        # rope epilogue through the finalize kernel (decode qkv): M=4 rows at position 9
        Sx, H, hd, rot = 1, 4, 256, 64
        A2, B2 = mk((4, 8192), False, dev, 0.5), mk((3 * H * hd, 8192), False, dev, 0.05)
        tab = ops.rope_table(1, rot, pos0=9, device=dev)
        kw = dict(rope_tab=tab, rope_mode=1, rope_S=1, rope_hd=hd, rope_rot=rot, rope_ncols=2 * H * hd)
        a = ops.gemm(A2, B2, splitk_ws=ws, **kw)
        b = ops.gemm(A2, B2, **kw)
        torch.cuda.synchronize()
        ok &= report("splitk rope epilogue == single-pass rope epilogue", a, b.float())
    elif g == "smallm":
        # M <= 32: 32-row A ring (deeper pipeline). All tile widths, both B majors, fused epilogues, ragged N/K.
        import torch.nn.functional as F

        for M in (1, 7, 32):
            for (N, K, bmn) in ((4096, 4096, False), (1000, 328, True), (12288, 4096, False), (264, 16384, False)):
                A, B = mk((M, K), False, dev, 0.5), mk((N, K), bmn, dev, 0.125)
                ldc = (N + 63) // 64 * 64
                bias = torch.randn(N, device=dev).to(torch.bfloat16)
                res = mk((M, ldc), False, dev)[:, :N]
                C = torch.full((M, ldc), 7.0, device=dev, dtype=torch.bfloat16)
                ops.gemm(A, B, out=C[:, :N], b_mn=bmn, bias=bias, act=ops.ACT_RELU, res1=res)
                torch.cuda.synchronize()
                want = F.relu(ref_gemm(A, B, False, bmn) + bias.float()) + res.float()
                ok &= report(f"smallm M={M} N={N} K={K} bmn={int(bmn)}", C[:, :N], want)
                ok &= bool((C[:, N:] == 7.0).all().item())
        for bn in (64, 128, 256):
            A, B = mk((32, 512), False, dev), mk((512, 512), False, dev)
            ok &= report(f"smallm forced bn={bn}", ops.gemm(A, B, force_bn=bn), ref_gemm(A, B, False, False))
    elif g == "perf":
        shapes = [
            (1024, 4096, 4096, False, False, "out/qkv-like fwd"),
            (1024, 12288, 4096, False, False, "qkv fwd"),
            (1024, 16384, 4096, False, False, "fc_in fwd"),
            (1024, 4096, 16384, False, False, "fc_out fwd"),
            (1024, 4096, 16384, False, True, "fc_in dgrad (B MN-major)"),
            (1024, 16384, 4096, False, True, "fc_out dgrad (B MN-major)"),
            (1024, 50304, 4096, False, False, "lm_head"),
            (1024, 4096, 1024, True, True, "adapter wgrad (MN/MN)"),
            (8192, 8192, 8192, False, False, "square 8192"),
        ]
        if os.environ.get("MB200_PERF_SHORT"):
            shapes = [shapes[0], shapes[7]]
        for M, N, K, a_mn, b_mn, name in shapes:
            A, B = mk((M, K), a_mn, dev), mk((N, K), b_mn, dev)
            C = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
            for bn in (128, 256):
                for _ in range(3):
                    ops.gemm(A, B, out=C, a_mn=a_mn, b_mn=b_mn, force_bn=bn)
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                iters = 20
                e0.record()
                for _ in range(iters):
                    ops.gemm(A, B, out=C, a_mn=a_mn, b_mn=b_mn, force_bn=bn)
                e1.record()
                torch.cuda.synchronize()
                ms = e0.elapsed_time(e1) / iters
                tf = 2.0 * M * N * K / ms / 1e9
                print(f"[PERF] {name} M={M} N={N} K={K} bn={bn}: {ms*1000:.1f} us  {tf:.1f} TFLOP/s", flush=True)
            # cuBLAS reference for the same shape (context only)
            Af = A.t() if a_mn else A
            Bf = B if b_mn else B.t()
            for _ in range(3):
                torch.matmul(Af, Bf, out=C)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(20):
                torch.matmul(Af, Bf, out=C)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / 20
            print(f"[PERF]   cuBLAS same shape: {ms*1000:.1f} us  {2.0*M*N*K/ms/1e9:.1f} TFLOP/s", flush=True)
            ok &= report(f"perf-shape correctness {name}", C, ref_gemm(A, B, a_mn, b_mn))
        # split-K vs single pass and the small-M plan (weight-streaming GEMMs)
        ws = torch.full((16 * 128 * 8192,), float("nan"), device=dev, dtype=torch.float32)
        for (M, N, K) in ((32, 12288, 4096), (32, 16384, 4096), (32, 4096, 16384), (32, 4096, 4096), (32, 1024, 4096), (32, 50258, 4096)):
            A, B = mk((M, K), False, dev), mk((N, K), False, dev)
            ldc = (N + 63) // 64 * 64
            C = torch.empty(M, ldc, device=dev, dtype=torch.bfloat16)[:, :N]
            for use in (False, True):
                kw = dict(splitk_ws=ws) if use else {}
                for _ in range(3):
                    ops.gemm(A, B, out=C, **kw)
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(20):
                    ops.gemm(A, B, out=C, **kw)
                e1.record()
                torch.cuda.synchronize()
                ms = e0.elapsed_time(e1) / 20
                print(f"[PERF] M={M} N={N} K={K} {'splitk' if use else 'single'}: {ms*1000:.1f} us  {N*K*2/ms/1e6:.0f} GB/s weights", flush=True)
        for (M, N, K) in ((32, 12288, 4096), (32, 16384, 4096), (32, 4096, 4096), (32, 1024, 4096), (32, 4096, 1024)):
            A, B = mk((M, K), False, dev), mk((N, K), False, dev)
            C = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
            for _ in range(3):
                ops.gemm(A, B, out=C)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(20):
                ops.gemm(A, B, out=C)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / 20
            print(f"[PERF] smallm M={M} N={N} K={K}: {ms*1000:.1f} us  {N*K*2/ms/1e6:.0f} GB/s weights", flush=True)
    print(f"GROUP {g}: {'PASS' if ok else 'FAIL'}", flush=True)
    return 0 if ok else 1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--group", default=None)
    ap.add_argument("--timeout", type=int, default=240)
    args = ap.parse_args()
    if args.group:
        sys.exit(run_group(args.group))
    rc = 0
    for g in GROUPS:
        t0 = time.time()
        try:
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--group", g], timeout=args.timeout)
            code = r.returncode
        except subprocess.TimeoutExpired:
            code = -999
            print(f"GROUP {g}: TIMEOUT", flush=True)
        print(f"== group {g} exit={code} ({time.time()-t0:.1f}s)", flush=True)
        rc |= code != 0
    sys.exit(rc)


if __name__ == "__main__":
    main()
