"""Launch plan of a full-size pass, produced WITHOUT a GPU by the product's own schedule code.

The host schedules (csrc/gptj_sched.cu, vit_sched.cu) are compiled as plain C++ into the CPU emulation library
(oracle/build_emul.py). With the emulation's trace mode on, every primitive logs (operator, shape, algorithmic FLOPs and
bytes) and returns without touching memory, so the schedule can be "issued" at BASELINE.json's sizes — GPT-J-6B, B = 8,
S = 128 — with placeholder pointers in milliseconds. The result is the exact list of launches a step makes, which this
tool summarises against the measured peaks (MEASURED_PEAKS.json): per-launch FLOPs / bytes, the roofline time of each
launch, tile counts of the GEMMs and how full their last wave is on the 132 SMs of an H100 SXM.

  python tools/plan_trace.py [--B 8] [--S 128] [--out step_launch_plan.txt]

This is an ANALYTIC plan (a lower bound per launch), not a measurement: compare it with a measured launch list of the
same step.

The *_records functions (PASSES) return, per production pass, one launch record per primitive: every scalar argument and
each pointer as [region, byte offset], with the workspace and every tensor the pass is given in a region of its own.
tests/test_production_launches_*.py deduplicate them into launch configurations (config_key) and replay each one."""
import argparse
import collections
import ctypes
import functools
import json
import math
import os
import sys
import tempfile

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)

STEP = 1 << 40  # placeholder "device memory": every tensor a pass is given starts at its own multiple of 2^40


class Regions:
    """Placeholder tensors of one traced pass. Each gets its own base (never dereferenced while the trace is on), so a
    recorded address resolves to (region, byte offset): the workspace and every weight, gradient and I/O tensor are
    regions of their own, and the bases are aligned far beyond 256 bytes like a caching allocator's blocks."""

    def __init__(self):
        self.names, self.sizes = [], []

    def new(self, name, size=STEP):
        """size: the bytes the region holds when the pass states it (the workspace), else the whole stride."""
        self.names.append(name)
        self.sizes.append(size)
        return len(self.names) * STEP

    def resolve(self, addr):
        if not addr:
            return None
        i = addr // STEP - 1
        if not 0 <= i < len(self.names) or addr % STEP >= self.sizes[i]:
            raise ValueError(f"address {addr:#x} lies in no region")
        return [self.names[i], addr % STEP]


def gptj_model(R, d, H, rot, V, r_mlp, r_attn=0, n_layer=28):
    """GPT-J with normal adapters (no leading LayerNorm, scale 1) of bottleneck r_mlp on the MLP and r_attn on attention
    (0 = none); every adapter trains, the LM is frozen."""
    from magma_b200._lib import GptjLayerExC as GptjLayerC, GptjModelExC as GptjModelC

    layers = (GptjLayerC * n_layer)()
    for l in range(n_layer):
        lay = layers[l]
        for f, _ in GptjLayerC._fields_:
            if f not in ("mlp_ad", "attn_ad"):
                setattr(lay, f, R.new(f"lm.h{l}.{f}"))
        for ad, r in (("mlp_ad", r_mlp), ("attn_ad", r_attn)):
            if r:
                for f in ("wd", "bd", "wu", "bu", "g_wd", "g_bd", "g_wu", "g_bu"):
                    setattr(getattr(lay, ad), f, R.new(f"lm.h{l}.{ad}.{f}"))
    m = GptjModelC()
    m.n_layer, m.d, m.n_head, m.rotary_dim, m.vocab, m.d_ff = n_layer, d, H, rot, V, 4 * d
    m.mlp_adapter, m.mlp_adapter_r = (1, r_mlp) if r_mlp else (0, 0)
    m.attn_adapter, m.attn_adapter_r = (1, r_attn) if r_attn else (0, 0)
    m.ln_eps = 1e-5
    m.layers = ctypes.cast(layers, ctypes.POINTER(GptjLayerC))
    for f in ("lnf_g", "lnf_b", "w_lm", "b_lm"):
        setattr(m, f, R.new(f"lm.{f}"))
    return m, layers


def gptj6b(R, r_mlp=1024, r_attn=0):
    return gptj_model(R, 4096, 16, 64, 50258, r_mlp, r_attn)


LDV = 50304  # the logits row stride the runtime allocates: the vocabulary rounded up to 64


def vit_model(R):
    from magma_b200._lib import VitLayerC, VitModelC

    layers = (VitLayerC * 24)()
    for l in range(24):
        for f, _ in VitLayerC._fields_:
            setattr(layers[l], f, R.new(f"vit.l{l}.{f}"))
    m = VitModelC()
    m.n_layer, m.width, m.n_head, m.patch, m.image, m.mlp, m.out_dim = 24, 1024, 16, 14, 224, 4096, 768
    m.w_conv, m.ld_conv = R.new("vit.w_conv"), 592
    for f in ("cls", "pos", "ln_pre_g", "ln_pre_b", "ln_post_g", "ln_post_b", "proj_t"):
        setattr(m, f, R.new(f"vit.{f}"))
    m.layers = ctypes.cast(layers, ctypes.POINTER(VitLayerC))
    return m, layers


def vit_grads(R):
    from magma_b200._lib import VitGradsC, VitLayerGradsC

    layers = (VitLayerGradsC * 24)()
    for l in range(24):
        for f, _ in VitLayerGradsC._fields_:
            setattr(layers[l], f, R.new(f"vit.l{l}.g_{f}"))
    g = VitGradsC()
    for f, _ in VitGradsC._fields_:
        if f != "layers":
            setattr(g, f, R.new(f"vit.g_{f}"))
    g.layers = ctypes.cast(layers, ctypes.POINTER(VitLayerGradsC))
    return g, layers


def trace(fn, R=None):
    """Issues fn(L) on the emulation in trace mode. Returns the summary rows, or (rows, launch records) when a Regions
    table is given: one dict per primitive with every scalar argument and each pointer as [region, byte offset]."""
    from magma_b200._lib import configure
    from oracle import build_emul

    L = configure(ctypes.CDLL(build_emul.build()))
    L.mb200_emul_record.argtypes = [ctypes.c_char_p]
    with tempfile.TemporaryDirectory() as d:
        path, rec = os.path.join(d, "trace"), os.path.join(d, "records")
        L.mb200_emul_trace(path.encode())
        L.mb200_emul_record(rec.encode() if R is not None else None)
        try:
            fn(L)
        finally:
            L.mb200_emul_trace(None)
            L.mb200_emul_record(None)
        rows = []
        for line in open(path):
            parts = line.rstrip("\n").split("\t")
            kv = dict(p.split("=") for p in parts[1].split()) if len(parts) > 1 and parts[1] else {}
            rows.append({"op": parts[0], "args": kv, "flops": float(parts[-2].split("=")[1]),
                         "bytes": float(parts[-1].split("=")[1])})
        if R is None:
            return rows
        records = [json.loads(line) for line in open(rec)]
    for r in records:
        for k in POINTERS[r["op"]]:
            r[k] = R.resolve(r[k])
    return rows, records


# the pointer arguments of each recorded primitive (every other field is a scalar)
POINTERS = {
    "gemm": ("A", "B", "C", "bias", "aux_out", "aux_in", "res1", "res2", "rope_tab", "splitk_ws"),
    "layernorm_fwd": ("x", "gamma", "beta", "y", "mean", "rstd"),
    "layernorm_bwd": ("dy", "x", "gamma", "mean", "rstd", "res", "dx"),
    "layernorm_param_grad": ("dy", "x", "mean", "rstd", "dgamma", "dbeta"),
    "layernorm_param_grad_rows": ("dy", "x", "mean", "rstd", "dgamma", "dbeta"),
    "softmax_fwd": ("s", "p"),
    "softmax_bwd": ("dp", "p", "ds"),
    "colsum": ("x", "out"),
    "quick_gelu_bwd": ("dy", "pre", "dx"),
    "scale_add": ("u", "s", "r1", "r2", "out"),
    "dot": ("a", "b", "out"),
    "rope_table": ("tab",),
    "cross_entropy": ("logits", "labels", "row_loss", "n_valid", "loss", "dlogits"),
    "attn_fwd_tile": ("qkv", "P", "O"),
    "attn_fwd_flash": ("q", "k", "v", "O", "P", "stats"),
    "attn_bwd_tile": ("qkv", "dO", "P", "dqkv", "rope_tab"),
    "kv_append": ("qkv", "kc", "vc"),
    "attn_decode": ("qkv", "kc", "vc", "out"),
    "patchify": ("img", "patches"),
    "vit_assemble": ("x", "pe", "cls", "pos"),
    "logits_grad_combine": ("dce", "g", "out"),
}


def check(L, rc):
    if rc:
        raise RuntimeError(L.mb200_last_error().decode())


def _ws(R, n):
    return ctypes.c_void_p(R.new("workspace", n)), ctypes.c_size_t(n)


def _gptj_train(L, R, gm, B, S, recompute):
    """A training pass as language_model.py issues it: logits [B*S][LDV], labels and loss, dx for the image prefix."""
    P = "_recompute" if recompute else ""
    n = (L.mb200_gptj_sched_recompute_workspace_bytes if recompute else L.mb200_gptj_sched_workspace_bytes)(
        ctypes.byref(gm), B, S)
    ws, nb = _ws(R, n)
    check(L, getattr(L, f"mb200_gptj_sched_forward{P}")(ctypes.byref(gm), R.new("x"), R.new("labels"), R.new("logits"),
                                                         ctypes.c_int64(LDV), R.new("loss"), B, S, ws, nb, None))
    check(L, getattr(L, f"mb200_gptj_sched_backward_range{P}")(ctypes.byref(gm), R.new("dx"), ctypes.c_float(1.0),
                                                                gm.n_layer, 0, 0, B, S, ws, nb, None))


def _vit_infer(L, R, vm, B):
    ws, nb = _ws(R, L.mb200_vit_workspace_bytes(ctypes.byref(vm), B))
    check(L, L.mb200_vit_forward(ctypes.byref(vm), R.new("images"), R.new("feats"), B, ws, nb, None))


def config2_train_records(B=8, S=128):
    """Config 2: ViT-L/14 forward (frozen) + GPT-J-6B with MLP adapters (f = 4) forward and backward, stored path."""
    R = Regions()
    gm, k1 = gptj6b(R)
    vm, k2 = vit_model(R)
    return trace(lambda L: (_vit_infer(L, R, vm, B), _gptj_train(L, R, gm, B, S, False)), R)


def gptj_recompute_train_records(B=8, S=2048):
    """GPT-J-6B with MLP adapters at the reference's sequence length, on the recompute path."""
    R = Regions()
    gm, k = gptj6b(R)
    return trace(lambda L: _gptj_train(L, R, gm, B, S, True), R)


def magma_v2_train_records(B=8, S=128):
    """MAGMA_v2 adapter wiring: normal adapters of downsample factor 8 on the MLP and on attention."""
    R = Regions()
    gm, k = gptj6b(R, r_mlp=512, r_attn=512)
    return trace(lambda L: _gptj_train(L, R, gm, B, S, False), R)


def vit_train_records(B=8):
    """The trainable ViT-L/14 forward and backward (configs/MAGMA_v1_vit_trainable_encoder.yml)."""
    R = Regions()
    vm, k1 = vit_model(R)
    g, k2 = vit_grads(R)

    def issue(L):
        ws, nb = _ws(R, L.mb200_vit_train_workspace_bytes(ctypes.byref(vm), B))
        check(L, L.mb200_vit_forward_train(ctypes.byref(vm), R.new("images"), R.new("feats"), B, ws, nb, None))
        check(L, L.mb200_vit_backward(ctypes.byref(vm), ctypes.byref(g), R.new("dfeats"), 0, B, ws, nb, None))

    return trace(issue, R)


def _infer(L, R, gm, B, S, S_max, pos0):
    n = L.mb200_gptj_sched_infer_workspace_bytes(ctypes.byref(gm), B, S, S_max)
    ws, nb = _ws(R, n)
    check(L, L.mb200_gptj_sched_infer(ctypes.byref(gm), R.new("x"), R.new("logits"), ctypes.c_int64(LDV), 1, None,
                                      R.new("kcache"), R.new("vcache"), S_max, pos0, B, S, ws, nb, None))


def prefill_records(B=1, S=2048):
    """KV-cache prefill of a prompt of S tokens, last-position logits."""
    R = Regions()
    gm, k = gptj6b(R)
    return trace(lambda L: _infer(L, R, gm, B, S, S, 0), R)


def decode_records(B=32, pos=136, S_max=264):
    """One KV-cache decode step (BASELINE config 5: B = 32) at cache position `pos`: S = 1, last-position logits."""
    R = Regions()
    gm, k = gptj6b(R)
    return trace(lambda L: _infer(L, R, gm, B, 1, S_max, pos), R)


# every production pass whose launches tests/test_production_launches_*.py replay
PASSES = {
    "config2_train": config2_train_records,
    "gptj_recompute_train_S2048": gptj_recompute_train_records,
    "magma_v2_train": magma_v2_train_records,
    "vit_train": vit_train_records,
    "prefill_S2048": prefill_records,
    "decode_pos136": lambda: decode_records(32, 136),
    "decode_last": lambda: decode_records(32, 263),
}


def config_key(rec):
    """The launch configuration of a record: the op, every scalar, each pointer's alignment class (byte offset mod 16 and
    mod 256, or absent) and its aliasing (the first earlier pointer argument with the same address, if any). Launches
    with equal keys run the same kernel, plan and compiled form on equally laid-out memory."""
    ptrs = POINTERS[rec["op"]]
    scalars = tuple((k, v) for k, v in rec.items() if k not in ptrs)
    seen, cls = {}, []
    for k in ptrs:
        p = rec[k]
        if p is None:
            cls.append((k, None))
            continue
        alias = seen.setdefault(tuple(p), k)
        cls.append((k, p[1] % 16, p[1] % 256, alias if alias != k else None))
    return scalars + tuple(cls)


def distinct_configs(records):
    """{key: (first record of that configuration, number of launches)} in issue order."""
    out = collections.OrderedDict()
    for r in records:
        k = config_key(r)
        out[k] = (out[k][0], out[k][1] + 1) if k in out else (r, 1)
    return out


@functools.lru_cache(maxsize=None)
def pass_records(name):
    """(summary rows, launch records) of PASSES[name], traced once per process. Callers must not modify them."""
    return PASSES[name]()


def train_step_plan(B, S):
    R = Regions()
    gm, k1 = gptj6b(R)
    vm, k2 = vit_model(R)
    return trace(lambda L: (_vit_infer(L, R, vm, B), _gptj_train(L, R, gm, B, S, False)))


def decode_step_plan(B, pos, S_max=264):
    """One KV-cache decode step (BASELINE config 5: B = 32) at cache position `pos`: S = 1, last-position logits."""
    R = Regions()
    gm, k = gptj6b(R)
    return trace(lambda L: _infer(L, R, gm, B, 1, S_max, pos))


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
