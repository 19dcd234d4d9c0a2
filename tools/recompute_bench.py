"""Cost of activation recomputation in the GPT-J training schedule, at full size on one GPU.

Runs GPT-J-6B with MLP adapters (MAGMA_v1.yml) at S = 2048 through the C ABI with the path forced: the stored-activation
entry points (mb200_gptj_sched_forward / _backward_range) and the recompute ones (..._forward_recompute /
_backward_range_recompute). For B = 4 stored, B = 4 recompute and B = 8 recompute it prints one JSON line with the LM
step time (forward + backward, host clock around synchronised steps), the training workspace and
torch.cuda.max_memory_allocated, which includes the model's weights. B = 8 on the stored path needs a 78.6 GiB workspace
and is reported from workspace arithmetic only. Then `bench.py --gpus 1 --no-gpu-eager --no-cpu-baseline` runs once
in a child process (BASELINE.json config 2, which stays on the stored path). The card's name and power limit are read in the same run.

    python tools/recompute_bench.py [--steps 3] [--warmup 1] [--bench-steps 20] [--out FILE]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (s.strip() for s in q.split(","))
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def lm_step_case(model, B, S, recompute, steps, warmup):
    from magma_b200 import ops
    from magma_b200._lib import check, lib

    L = lib()
    lm = model.lm
    m = lm._cmodel_ex()[0]
    n_layer, d, ldv = len(lm.transformer.h), lm.config.hidden_size, lm.ldv
    sfx = "_recompute" if recompute else ""
    nbytes = getattr(L, f"mb200_gptj_sched{sfx}_workspace_bytes")(ctypes.byref(m), B, S)
    fwd = getattr(L, f"mb200_gptj_sched_forward{sfx}")
    bwd = getattr(L, f"mb200_gptj_sched_backward_range{sfx}")
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    g = torch.Generator(device="cuda").manual_seed(0)
    x = (0.5 * torch.randn(B, S, d, generator=g, device="cuda")).to(torch.bfloat16)
    labels = torch.randint(0, lm.lm_head.weight.shape[0], (B, S), generator=g, device="cuda")
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    logits = torch.empty(B * S, ldv, dtype=torch.bfloat16, device="cuda")
    loss = torch.zeros(1, dtype=torch.float32, device="cuda")
    dx = torch.empty_like(x)

    def step():
        check(fwd(ctypes.byref(m), ops._ptr(x), ops._ptr(labels), ops._ptr(logits), ctypes.c_int64(ldv), ops._ptr(loss),
                  B, S, ops._ptr(ws), ctypes.c_size_t(nbytes), ops._stream()))
        check(bwd(ctypes.byref(m), ops._ptr(dx), ctypes.c_float(1.0), n_layer, 0, 0, B, S, ops._ptr(ws),
                  ctypes.c_size_t(nbytes), ops._stream()))

    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        step()
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3 / steps
    out = {"B": B, "S": S, "path": "recompute" if recompute else "stored", "lm_step_ms": round(ms, 1),
           "lm_samples_per_s": round(B * 1e3 / ms, 3), "workspace_gib": round(nbytes / 2**30, 2),
           "max_memory_allocated_gib": round(torch.cuda.max_memory_allocated() / 2**30, 2),
           "loss": round(float(loss), 4), "dx_finite": bool(torch.isfinite(dx.float()).all())}
    del ws, logits, dx
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--bench-steps", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("recompute_bench: needs a CUDA device")
    rows = [dict(card(), what="device")]

    def emit(row):
        rows.append(row)
        print(json.dumps(row), flush=True)

    print(json.dumps(rows[0]), flush=True)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", str(args.bench_steps),
                        "--warmup", "3", "--no-gpu-eager", "--no-cpu-baseline"],
                       capture_output=True, text=True, cwd=ROOT)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    emit({"what": "bench.py --gpus 1", "rc": r.returncode, "result": json.loads(lines[-1]) if lines else r.stderr[-2000:]})

    from magma_b200.config import MultimodalConfig
    from magma_b200.magma import Magma

    S = 2048
    mc = MultimodalConfig(batch_size=8, train_steps=1, encoder_name="clip_vit_large",
                          adapter_config={"mlp": {"adapter_type": "normal", "downsample_factor": 4}}, image_seq_len=2,
                          image_embed_dropout_prob=0.0, use_image_embed_layernorm=True, image_size=224, seq_len=S)
    model = Magma(mc, device="cuda", init_seed=0)
    m = model.lm._cmodel_ex()[0]
    from magma_b200._lib import lib

    for B, recompute in ((4, False), (4, True), (8, True)):
        emit(dict(lm_step_case(model, B, S, recompute, args.steps, args.warmup), what="lm step"))
    stored8 = lib().mb200_gptj_sched_workspace_bytes(ctypes.byref(m), 8, S)
    free, total = torch.cuda.mem_get_info()
    emit({"what": "lm step", "B": 8, "S": S, "path": "stored", "lm_step_ms": "not measured",
          "workspace_gib": round(stored8 / 2**30, 2), "free_gib_with_model_loaded": round(free / 2**30, 2)})
    st, rc4 = (next(r for r in rows if r.get("B") == 4 and r.get("path") == p) for p in ("stored", "recompute"))
    emit({"what": "recompute overhead at B = 4", "lm_time_ratio": round(rc4["lm_step_ms"] / st["lm_step_ms"], 3)})
    if args.out:
        with open(args.out, "w") as f:
            f.writelines(json.dumps(r) + "\n" for r in rows)


if __name__ == "__main__":
    main()
