"""Launch plan of a full-size pass, produced WITHOUT a GPU by the product's own schedule code.

The host schedules (csrc/gptj_sched.cu, vit_sched.cu) are compiled as plain C++ into the CPU emulation library
(oracle/build_emul.py). With the emulation's trace mode on, every primitive logs (operator, shape, algorithmic FLOPs and
bytes) and returns without touching memory, so the schedule can be "issued" at BASELINE.json's sizes — GPT-J-6B, B = 8,
S = 128 — with placeholder pointers in milliseconds. The result is the exact list of launches a step makes, which this
tool summarises against the measured peaks (MEASURED_PEAKS.json): per-launch FLOPs / bytes, the roofline time of each
launch, tile counts of the GEMMs and how full their last wave is on the 132 SMs of an H100 SXM.

  python tools/plan_trace.py [--B 8] [--S 128] [--out step_launch_plan.txt]

This is an ANALYTIC plan (a lower bound per launch), not a measurement: compare it with a measured launch list of the
same step."""
import argparse
import collections
import ctypes
import json
import math
import os
import sys
import tempfile

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)

FAKE = 0x10000000  # placeholder "device pointer": never dereferenced while the trace is on


def gptj_model(L, d, H, rot, V, r, n_layer=28):
    from magma_b200._lib import GptjLayerExC as GptjLayerC, GptjModelExC as GptjModelC

    layers = (GptjLayerC * n_layer)()
    for l in range(n_layer):
        lay = layers[l]
        for f, _ in GptjLayerC._fields_:
            if f in ("mlp_ad", "attn_ad"):
                continue
            setattr(lay, f, FAKE)
        for f in ("wd", "bd", "wu", "bu", "g_wd", "g_bd", "g_wu", "g_bu"):
            setattr(lay.mlp_ad, f, FAKE)
    m = GptjModelC()
    m.n_layer, m.d, m.n_head, m.rotary_dim, m.vocab, m.d_ff = n_layer, d, H, rot, V, 4 * d
    m.mlp_adapter, m.mlp_adapter_r, m.attn_adapter, m.attn_adapter_r = 1, r, 0, 0
    m.ln_eps = 1e-5
    m.layers = ctypes.cast(layers, ctypes.POINTER(GptjLayerC))
    m.lnf_g = m.lnf_b = m.w_lm = m.b_lm = FAKE
    return m, layers


def vit_model(L):
    from magma_b200._lib import VitLayerC, VitModelC

    layers = (VitLayerC * 24)()
    for l in range(24):
        for f, _ in VitLayerC._fields_:
            setattr(layers[l], f, FAKE)
    m = VitModelC()
    m.n_layer, m.width, m.n_head, m.patch, m.image, m.mlp, m.out_dim = 24, 1024, 16, 14, 224, 4096, 768
    m.w_conv, m.ld_conv = FAKE, 592
    for f in ("cls", "pos", "ln_pre_g", "ln_pre_b", "ln_post_g", "ln_post_b", "proj_t"):
        setattr(m, f, FAKE)
    m.layers = ctypes.cast(layers, ctypes.POINTER(VitLayerC))
    return m, layers


def trace(fn):
    from magma_b200._lib import configure
    from oracle import build_emul

    L = configure(ctypes.CDLL(build_emul.build()))
    with tempfile.NamedTemporaryFile("r", suffix=".trace", delete=False) as t:
        path = t.name
    L.mb200_emul_trace(path.encode())
    try:
        fn(L)
    finally:
        L.mb200_emul_trace(None)
    rows = []
    for line in open(path):
        parts = line.rstrip("\n").split("\t")
        kv = dict(p.split("=") for p in parts[1].split()) if len(parts) > 1 and parts[1] else {}
        rows.append({"op": parts[0], "args": kv, "flops": float(parts[-2].split("=")[1]), "bytes": float(parts[-1].split("=")[1])})
    os.unlink(path)
    return rows


def check(L, rc):
    if rc:
        raise RuntimeError(L.mb200_last_error().decode())


def train_step_plan(B, S):
    gm, keep1 = gptj_model(None, 4096, 16, 64, 50258, 1024)
    vm, keep2 = vit_model(None)

    def issue(L):
        ws = ctypes.c_void_p(FAKE)
        n = L.mb200_vit_workspace_bytes(ctypes.byref(vm), B)
        check(L, L.mb200_vit_forward(ctypes.byref(vm), FAKE, FAKE, B, ws, ctypes.c_size_t(n), None))
        n = L.mb200_gptj_sched_workspace_bytes(ctypes.byref(gm), B, S)
        check(L, L.mb200_gptj_sched_forward(ctypes.byref(gm), FAKE, FAKE, None, ctypes.c_int64(0), FAKE, B, S, ws,
                                            ctypes.c_size_t(n), None))
        check(L, L.mb200_gptj_sched_backward(ctypes.byref(gm), FAKE, ctypes.c_float(1.0), 0, B, S, ws, ctypes.c_size_t(n),
                                             None))

    return trace(issue)


def decode_step_plan(B, pos, S_max=264):
    """One KV-cache decode step (BASELINE config 5: B = 32) at cache position `pos`: S = 1, last-position logits."""
    gm, keep = gptj_model(None, 4096, 16, 64, 50258, 1024)

    def issue(L):
        ws = ctypes.c_void_p(FAKE)
        n = L.mb200_gptj_sched_infer_workspace_bytes(ctypes.byref(gm), B, 1, S_max)
        check(L, L.mb200_gptj_sched_infer(ctypes.byref(gm), FAKE, FAKE, ctypes.c_int64(50304), 1, None, FAKE, FAKE, S_max,
                                          pos, B, 1, ws, ctypes.c_size_t(n), None))

    return trace(issue)


def gemm_tiles(a):
    """Tile counts of one GEMM launch of csrc/gemm.cu, approximated as 128 x BN tiles with BN = 256 unless N is small
    (the kernel's own choice also weighs wave quantisation), on a persistent grid of one CTA per SM."""
    M, N, nb = int(a["M"]), int(a["N"]), int(a["nb"])
    bn = 256 if N >= 256 else (128 if N > 64 else 64)
    t = math.ceil(M / 128) * math.ceil(N / bn) * nb
    return f"128x{bn}", t, 132


def summarise(rows, B, S, peaks, out):
    tf, gbs = peaks["bf16_tflops"] * 1e12, peaks["hbm_gbs"] * 1e9
    total_t = 0.0
    groups = collections.OrderedDict()
    for r in rows:
        t = max(r["flops"] / tf, r["bytes"] / gbs)
        total_t += t
        if r["op"] == "gemm":
            a = r["args"]
            key = f"gemm M={a['M']} N={a['N']} K={a['K']} nb={a['nb']} {'T' if a['a_mn'] == '1' else 'N'}{'T' if a['b_mn'] == '1' else 'N'} {a['c']}"
        else:
            key = r["op"] + " " + " ".join(f"{k}={v}" for k, v in r["args"].items())
        g = groups.setdefault(key, {"n": 0, "flops": 0.0, "bytes": 0.0, "t": 0.0, "row": r})
        g["n"] += 1
        g["flops"] += r["flops"]
        g["bytes"] += r["bytes"]
        g["t"] += t
    title = (f"launch plan of one training step (ViT-L/14 forward + GPT-J-6B forward + backward, B={B}, S={S}, MLP adapters f=4),"
             if S else f"launch plan of one KV-cache decode step (GPT-J-6B + MLP adapters, B={B}, S=1, last-position logits),")
    lines = [title,
             "issued by the product's own host schedules on the CPU emulation in trace mode - analytic, not measured.",
             f"peaks: {peaks['bf16_tflops']:.1f} TFLOP/s (burst bf16), {peaks['hbm_gbs']:.1f} GB/s (MEASURED_PEAKS.json)", "",
             f"{len(rows)} launches, {sum(r['flops'] for r in rows) / 1e12:.2f} TFLOP, {sum(r['bytes'] for r in rows) / 1e9:.2f} GB "
             f"algorithmic; sum of per-launch roofline times {total_t * 1e3:.2f} ms "
             f"(= {B / total_t:.0f} {'samples' if S else 'tokens'}/s if every launch ran at its roofline with no gaps)", "",
             f"{'n':>4} {'roofline us':>11} {'each us':>8} {'bound':>6} {'tiles':>6} {'last wave':>9}  launch"]
    for key, g in sorted(groups.items(), key=lambda kv: -kv[1]["t"]):
        r = g["row"]
        bound = "tensor" if r["flops"] / tf >= r["bytes"] / gbs else "hbm"
        tiles = wave = ""
        if r["op"] == "gemm" and int(r["args"]["M"]) > 128:  # small-M GEMMs are tiled by plan_small_m (tile width x split-K)
            kind, t, slots = gemm_tiles(r["args"])
            waves = t / slots
            wave = f"{(t % slots or slots) / slots:.2f}"
            tiles = f"{t}"
            key += f"  [{kind}, {waves:.2f} waves]"
        lines.append(f"{g['n']:>4} {g['t'] * 1e6:>11.1f} {g['t'] / g['n'] * 1e6:>8.2f} {bound:>6} {tiles:>6} {wave:>9}  {key}")
    text = "\n".join(lines) + "\n"
    if out:
        open(out, "w").write(text)
    print(text)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=8)
    ap.add_argument("--S", type=int, default=128)
    ap.add_argument("--out", default=None)
    ap.add_argument("--decode", action="store_true", help="plan of one decode step (B defaults to 32, --pos the cache position)")
    ap.add_argument("--pos", type=int, default=136)
    a = ap.parse_args()
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    peaks = json.load(open(p)) if os.path.exists(p) else {"bf16_tflops": 989.0, "hbm_gbs": 3350.0}  # H100 SXM data sheet
    if a.decode:
        B = a.B if a.B != 8 else 32
        summarise(decode_step_plan(B, a.pos), B, 0, peaks, a.out)
        return
    rows = train_step_plan(a.B, a.S)
    summarise(rows, a.B, a.S, peaks, a.out)


if __name__ == "__main__":
    main()
