#!/usr/bin/env python
"""bench.py — MAGMA hot-path benchmark (BASELINE.json metric: image-caption samples/sec, fwd+bwd).

  python bench.py --gpus N --steps K --warmup W            # this repo's kernels (H100, sm_90a)
  python bench.py --impl reference --gpus N --steps K ...  # the reference's CPU path (oracle port) on host cores

A "step" is one `train_step`: Magma.forward (CLIP ViT-L/14 -> ImagePrefix -> GPT-J-6B + MLP adapters -> LM head ->
shifted CE) + backward (LM and encoder frozen: dgrad everywhere, wgrad for adapters/prefix) + gradient all-reduce
(N > 1) + fused AdamW on the trainable set, at BASELINE.json config 2: batch 8 per GPU, 224x224, seq_len 128, bf16,
random-init weights of the real architecture, synthetic data.

Prints ONE JSON line (rank 0). `value` = samples/s with inputs resident in HBM; `e2e` = the same through the public
`train_step(config, loader, engine)` call with pinned HOST batches (H2D copy + loss D2H read inside the timed
region). `roofline` is for the dominant kernel (the wgmma GEMM core): algorithmic FLOPs of its launches / the sum
of their CUDA-event durations, measured in a second pass of the same steps with per-launch events enabled.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

B_PER_GPU, S, RES = 8, 128, 224
# algorithmic FLOPs / sample, fwd+bwd, LM + encoder frozen
D, R_AD, V, NL = 4096, 1024, 50258, 28
LM_FWD = NL * (24 * D * D + 4 * D * R_AD) * S + 2 * D * V * S + NL * 4 * S * S * D
VIT_FWD = 24 * (24 * 1024 * 1024 * 257 + 4 * 257 * 257 * 1024) + 2 * 588 * 1024 * 256
FLOPS_PER_SAMPLE = 2 * LM_FWD + NL * 4 * D * R_AD * S + VIT_FWD


def peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return d.get("bf16_tflops_sustained", d.get("bf16_tflops")), d.get("hbm_gbs"), "measured (MEASURED_PEAKS.json, sustained)"
    return 989.0, 3350.0, "H100 SXM data sheet (dense BF16, HBM3; 700 W card)"


class ClockSampler:
    """SM clock / throttle-reason samples DURING the timed region. Primary: NVML polled from a thread every 10 ms
    (first sample immediately, so even a 0.3 s region is covered); fallback: an `nvidia-smi -lms 100` child process
    (slow to start: it must already be running when the region begins, so construct the sampler before the warm-up
    and call mark() when the timed region starts)."""
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")
    REASONS = ((0x8, "hw_slowdown"), (0x40, "hw_thermal_slowdown"), (0x20, "sw_thermal_slowdown"), (0x4, "sw_power_cap"))

    def __init__(self, gpu_index=0, nvml=None):
        self.samples, self.t_mark, self.p, self.f, self.thread = [], None, None, None, None
        self._stop = threading.Event()
        self.h = self.nvml = None
        try:
            if nvml is None:
                import pynvml as nvml
            nvml.nvmlInit()
            vis = os.environ.get("CUDA_VISIBLE_DEVICES", "")
            ids = [v for v in vis.split(",") if v.strip().isdigit()]
            self.h = nvml.nvmlDeviceGetHandleByIndex(int(ids[gpu_index]) if gpu_index < len(ids) else gpu_index)
            self.nvml = nvml
            self.max_mhz = float(nvml.nvmlDeviceGetMaxClockInfo(self.h, nvml.NVML_CLOCK_SM))
            self._poll()  # fails here, not in the thread, if a query is unsupported
            self.thread = threading.Thread(target=self._run, daemon=True)
            self.thread.start()
        except Exception:
            self.nvml = self.h = None
            self._start_smi(gpu_index)

    def _reasons(self):
        for fn in ("nvmlDeviceGetCurrentClocksEventReasons", "nvmlDeviceGetCurrentClocksThrottleReasons"):
            if hasattr(self.nvml, fn):
                return int(getattr(self.nvml, fn)(self.h))
        return 0

    def _poll(self):
        self.samples.append((time.time(), float(self.nvml.nvmlDeviceGetClockInfo(self.h, self.nvml.NVML_CLOCK_SM)),
                             self._reasons()))

    def _run(self):
        while not self._stop.is_set():
            try:
                self._poll()
            except Exception:
                pass
            self._stop.wait(0.01)

    def _start_smi(self, gpu_index):
        self.f = tempfile.NamedTemporaryFile("w+", suffix=".csv", delete=False)
        try:
            self.p = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                                       "-lms", "100", "-i", str(gpu_index)], stdout=self.f, stderr=subprocess.DEVNULL)
        except Exception:
            self.p = None

    def mark(self):
        """The timed region starts now: only later samples count (NVML path)."""
        self.t_mark = time.time()

    def stop(self):
        out = {"sm_mhz": None, "sm_max_mhz": None, "reasons": []}
        if self.nvml is not None:
            self._stop.set()
            self.thread.join(timeout=2)
            try:
                self._poll()
            except Exception:
                pass
            rows = [r for r in self.samples if self.t_mark is None or r[0] >= self.t_mark] or self.samples[-1:]
            sm = sorted(r[1] for r in rows)
            bits = 0
            for r in rows:
                bits |= r[2]
            return {"sm_mhz": statistics.median(sm[len(sm) // 2:]), "sm_max_mhz": self.max_mhz,
                    "reasons": sorted(n for m, n in self.REASONS if bits & m), "samples": len(sm), "source": "nvml"}
        if self.p is None:
            return out
        self.p.terminate()
        try:
            self.p.wait(timeout=5)
        except Exception:
            self.p.kill()
        self.f.flush()
        rows = [l.strip().split(",") for l in open(self.f.name) if l.strip()]
        os.unlink(self.f.name)
        sm, mx, reasons = [], [], set()
        for r in rows:
            try:
                sm.append(float(r[1]))
                mx.append(float(r[2]))
                for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), r[4:8]):
                    if v.strip().lower().startswith("active"):
                        reasons.add(name)
            except Exception:
                pass
        if sm:
            busy = sorted(sm)[len(sm) // 2:]  # upper half = samples under load
            out = {"sm_mhz": statistics.median(busy), "sm_max_mhz": max(mx), "reasons": sorted(reasons),
                   "samples": len(sm), "source": "nvidia-smi"}
        return out


def synthetic_host_batches(n, seed, batch=B_PER_GPU, seq=S, res=RES, max_caption=None):
    import torch

    g = torch.Generator().manual_seed(seed)
    out = []
    hi = (max_caption if max_caption is not None else seq - 2) + 1
    for _ in range(n):
        images = torch.randn(batch, 3, res, res, generator=g)
        caps = torch.randint(0, 50256, (batch, seq), generator=g)
        lens = torch.randint(min(seq // 4, hi - 1), hi, (batch,), generator=g)
        caps = torch.where(torch.arange(seq)[None, :] >= lens[:, None], torch.full_like(caps, 50256), caps)
        out.append((images.pin_memory(), caps.pin_memory()))
    return out


def cpu_reference_run(steps, warmup, budget_s, n_threads=None, batch=B_PER_GPU):
    """The reference's CPU path for this workload: oracle/magma_oracle.py (a pinned restatement of the reference's
    Python + HF GPT-J/CLIP arithmetic) in fp32 on the host cores. One step = fwd+bwd of one batch of `batch` samples of
    the workload (224x224 images, seq_len 128, full 28-layer GPT-J-6B + ViT-L/14 + adapters, LM/encoder frozen) — the
    GPU arm's per-GPU batch by default, so both arms time the same configuration."""
    import torch

    from oracle import magma_oracle as O

    if not n_threads:
        # torchrun exports OMP_NUM_THREADS=1 to its workers; the reference arm is meant to use every host core it can
        # (physical cores: 128 hyper-threads on the 64-core box ran this 30x slower than 64 threads)
        try:
            n_threads = len(os.sched_getaffinity(0))
        except AttributeError:
            n_threads = os.cpu_count() or 1
        try:
            import psutil

            n_threads = max(1, min(n_threads, psutil.cpu_count(logical=False) or n_threads))
        except Exception:
            pass
    torch.set_num_threads(n_threads)
    cores = torch.get_num_threads()
    cfg = O.OracleConfig()
    t0 = time.time()
    # One set of random layer weights shared by all 28 GPT-J layers / 24 ViT layers: identical FLOPs and bytes per
    # layer, without materialising 24 GB of fp32 host weights (timing-equivalent; values are random either way).
    one = O.OracleConfig(n_layer=1, vit_layers=1)
    w1 = O.init_weights(one, seed=0)
    w = {}
    for k, v in w1.items():
        if ".transformer.h.0." in k:
            for l in range(cfg.n_layer):
                w[k.replace(".transformer.h.0.", f".transformer.h.{l}.")] = v
        elif ".resblocks.0." in k:
            for l in range(cfg.vit_layers):
                w[k.replace(".resblocks.0.", f".resblocks.{l}.")] = v
        else:
            w[k] = v
    trainable = [k for k in w1 if ".adapter." in k or k.startswith("image_prefix.proj") or k.startswith("image_prefix.ln")]
    for k in trainable:
        w1[k].requires_grad_(True)
    images, captions = O.synthetic_batch(cfg, batch, S, seed=1234)
    init_s = time.time() - t0

    def step():
        for k in trainable:
            w1[k].grad = None
        loss, _, _ = O.magma_forward(images, captions, w, cfg)
        loss.backward()
        return float(loss.detach())

    times = []
    t_start = time.time()
    n_warm = min(warmup, 1)
    for _ in range(n_warm):
        step()
    n_timed = 0
    while n_timed < max(1, steps):
        t1 = time.time()
        step()
        times.append(time.time() - t1)
        n_timed += 1
        if time.time() - t_start + statistics.mean(times) > budget_s:
            break
    sec = statistics.median(times)
    return {"samples_per_s": batch / sec, "sec_per_step": sec, "steps_timed": n_timed, "warmup": n_warm, "cores": cores,
            "init_s": init_s, "batch": batch,
            "sample": f"{n_timed} timed step(s) (after {n_warm} warm-up) of one batch of {batch} samples (224x224, seq_len "
                      f"{S}) fwd+bwd through the full GPT-J-6B+ViT-L/14+adapter graph in fp32 on {cores} threads (oracle "
                      f"port of the reference; layer weights shared across layers to bound host memory); median step time"}


def run_reference(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return 0
    r = cpu_reference_run(args.steps, args.warmup, budget_s=170.0)
    line = {
        "impl": "reference", "metric": "image-caption samples/sec (fwd+bwd)", "value": r["samples_per_s"],
        "unit": "samples/s", "n_gpus": args.gpus, "steps": r["steps_timed"], "warmup": r["warmup"],
        "ms_per_step": r["sec_per_step"] * 1e3, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "f32", "data": "synthetic",
        "config": workload_config(args.gpus, "reference CPU path (oracle port), host cores"),
        "cpu_baseline": {"value": r["samples_per_s"], "unit": "samples/s", "cores": r["cores"], "kind": "port",
                         "sample": r["sample"]},
        "e2e": {"value": r["samples_per_s"], "unit": "samples/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
    }
    print(json.dumps(line), flush=True)
    return 0


# BASELINE.json config 4 asks for an NFNet-F6 encoder, which the reference does not have (its conv
# encoders are timm nf_resnet50 and the CLIP ResNets) and this repo has not built; the conv-trunk hot path that IS built is
# the encoder MAGMA_v1.yml actually ships, CLIP RN50x16 (`clip_resnet_large`) at its native 384 px. Its prefix is 144 tokens
# (one per 12 x 12 position), which must fit inside seq_len (fact 3): 144 + 128 caption positions = 272.
CONV = {"batch": 16, "res": 384, "seq": 272, "encoder": "clip_resnet_large"}


def workload_config(n, note="", conv=False):
    if conv:
        return {"workload": "BASELINE.json config 4, conv-trunk variant that exists: CLIP RN50x16 (clip_resnet_large, the "
                            "encoder of MAGMA_v1.yml; NFNet-F6 is in neither the reference nor this repo) at 384x384 -> "
                            "144-token prefix + GPT-J-6B + MLP adapters (normal, f=4), batch 16 per GPU, seq_len 272 "
                            "(= 144 prefix + 128 caption positions), fwd+bwd+AdamW, LM and image encoder frozen (eval-mode "
                            "BatchNorm folded), random-init weights",
                "global_batch": CONV["batch"] * n, "seq_len": CONV["seq"], "image": CONV["res"], "parallelism": f"dp{n}",
                "l2": "working set per step (12.2 GB of bf16 weights streamed) exceeds the 50 MB L2; no explicit flush",
                "note": note}
    return {"workload": "BASELINE.json config 2: CLIP ViT-L/14 (clip_vit_large, pooled -> image_seq_len 2) + GPT-J-6B "
                        "+ MLP adapters (normal, f=4), batch 8 per GPU, 224x224 images, seq_len 128, fwd+bwd+AdamW, "
                        "LM and image encoder frozen, random-init weights",
            "global_batch": B_PER_GPU * n, "seq_len": S, "image": RES, "parallelism": f"dp{n}",
            "l2": "working set per step (12.2 GB of bf16 weights streamed) exceeds the 50 MB L2; no explicit flush",
            "note": note}


def dump_outputs(out_dir, out):
    """What the caller of the timed step receives from its last step: the loss and a fixed, seeded sample of the logits
    (the full [B, S, vocab] tensor is ~200 MB in fp32), as float32 .npy files."""
    import numpy as np
    import torch

    os.makedirs(out_dir, exist_ok=True)
    np.save(os.path.join(out_dir, "loss.npy"), out.loss.detach().float().reshape(1).cpu().numpy())
    if out.logits is not None:
        flat = out.logits.detach().reshape(-1)
        n = min(flat.numel(), 1 << 22)  # 16 MB of fp32
        idx = torch.randint(0, flat.numel(), (n,), generator=torch.Generator().manual_seed(0))
        np.save(os.path.join(out_dir, "logits_sample.npy"), flat[idx.to(flat.device)].float().cpu().numpy())
        last = out.logits.detach()[0, -1].float().cpu().numpy()  # every vocabulary entry of one position
        np.save(os.path.join(out_dir, "logits_b0_last_position.npy"), last)


def run_b200(args):
    import torch
    import torch.distributed as dist

    from magma_b200 import _lib
    from magma_b200.config import MultimodalConfig
    from magma_b200.magma import Magma
    from magma_b200.train_loop import B200Engine, train_step
    from magma_b200.utils import init_distributed

    rank, world, local_rank = init_distributed("nccl")
    assert world == args.gpus, f"--gpus {args.gpus} but WORLD_SIZE={world} (launch with torchrun for N>1)"
    dev = torch.device("cuda", local_rank)
    torch.cuda.set_device(dev)
    L = _lib.lib()
    conv = args.workload == "conv"
    Bw, Sw, Rw = (CONV["batch"], CONV["seq"], CONV["res"]) if conv else (B_PER_GPU, S, RES)
    mc = MultimodalConfig(batch_size=Bw * world, train_steps=args.steps,
                          encoder_name=CONV["encoder"] if conv else "clip_vit_large",
                          adapter_config={"mlp": {"adapter_type": "normal", "downsample_factor": 4}}, image_seq_len=2,
                          image_embed_dropout_prob=0.1, use_image_embed_layernorm=True, image_size=Rw, seq_len=Sw,
                          gradient_accumulation_steps=1, freeze_img_encoder=True, lr=8e-4, lr_decay_iters=300000)
    torch.manual_seed(0)  # adapters / image prefix draw their initial weights from torch's generator: same every run
    model = Magma(mc, device=dev, init_seed=0)
    model.train()
    engine = B200Engine(model, mc)
    host = synthetic_host_batches(4, 1234 + rank, Bw, Sw, Rw, max_caption=(Sw - 144 - 2) if conv else None)
    dev_batches = [(i.to(dev, non_blocking=True).to(torch.bfloat16), c.to(dev, non_blocking=True)) for i, c in host]
    torch.cuda.synchronize()

    def device_step(i):
        images, captions = dev_batches[i % len(dev_batches)]
        out = engine(images, captions)
        engine.backward(out.loss)
        engine.step()
        return out

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def max_over_ranks(ms):
        if world > 1:
            t = torch.tensor([ms], device=dev)
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            return float(t)
        return ms

    # ---- device-resident timing (value) ----
    sampler = ClockSampler(local_rank) if rank == 0 else None  # running before the warm-up (see its docstring)
    for i in range(max(args.warmup, 3)):
        device_step(i)
    barrier()
    if sampler:
        sampler.mark()
    launches0 = L.mb200_launch_count()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(args.steps):
        out = device_step(i)
    e1.record()
    barrier()
    loss = out.loss
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, out)
    ms_mine = e0.elapsed_time(e1)
    ms_total = max_over_ranks(ms_mine)
    rank_ms = None
    if world > 1:  # evidence for the scaling number: every rank's own device time for the same K steps
        t = torch.zeros(world, device=dev)
        t[rank] = ms_mine / args.steps
        dist.all_reduce(t)
        rank_ms = [round(float(x), 3) for x in t]
    launches = L.mb200_launch_count() - launches0
    clocks = sampler.stop() if sampler else None
    last_loss = float(loss.detach())
    ms_step = ms_total / args.steps
    value = Bw * world / (ms_step / 1e3)

    if os.environ.get("MB200_DP_TRACE", "0") == "1":  # diagnostic: event timeline of two consecutive steps, every rank
        engine.trace_report()
        for i in range(2):
            device_step(i)
        rep = engine.trace_report()
        print(f"[trace rank {rank}]\n" + "\n".join(f"  {ms:9.3f} ms  {lab}" for lab, ms in rep), flush=True)

    # ---- end-to-end through train_step with pinned host batches (e2e) ----
    def loader():
        i = 0
        while True:
            yield host[i % len(host)]
            i += 1

    it = loader()
    for _ in range(2):
        train_step(mc, it, engine)
    barrier()
    e0.record()
    for _ in range(args.steps):
        train_step(mc, it, engine)  # .item() on the reduced loss = D2H read every step
    e1.record()
    barrier()
    e2e_ms = max_over_ranks(e0.elapsed_time(e1)) / args.steps
    e2e = {"value": Bw * world / (e2e_ms / 1e3), "unit": "samples/s", "ms_per_step": e2e_ms,
           "h2d_bytes_per_step": host[0][0].numel() * 4 + host[0][1].numel() * 8, "d2h_bytes_per_step": 4,
           "api": "magma_b200.train_loop.train_step(config, loader, engine) with pinned fp32 images + int64 captions"}

    # ---- roofline of the dominant kernel (GEMM core), per-launch CUDA events, same steps ----
    roof = None
    # every rank runs the profiled steps (they contain the gradient all-reduce); only rank 0 records GEMM events
    if rank == 0:
        L.mb200_prof_enable(1)
    n_prof = min(args.steps, 3)
    t_ev0, t_ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t_ev0.record()
    for i in range(n_prof):
        device_step(i)
    t_ev1.record()
    torch.cuda.synchronize()
    if rank == 0:
        import ctypes

        peak_tf, _, peak_src = peaks()
        ms, fl, by, n = ctypes.c_double(), ctypes.c_double(), ctypes.c_double(), ctypes.c_longlong()
        L.mb200_prof_read(ctypes.byref(ms), ctypes.byref(fl), ctypes.byref(by), ctypes.byref(n))
        L.mb200_prof_enable(0)
        prof_step_ms = t_ev0.elapsed_time(t_ev1) / n_prof
        ach = fl.value / (ms.value / 1e3) / 1e12 if ms.value > 0 else 0.0
        roof = {"kernel": "gemm_wgmma_kernel (all GEMM launches of the step)", "bound": "tensor",
                "achieved": ach, "peak": peak_tf, "unit": "TFLOP/s", "frac": ach / peak_tf, "traffic": None,
                "peak_source": peak_src, "launches_per_step": n.value / n_prof,
                "avg_launch_us": ms.value * 1e3 / max(n.value, 1),
                "algorithmic_tflop_per_launch_avg": fl.value / max(n.value, 1) / 1e12,
                # GEMM time comes from a pass with per-launch events (which defeat PDL overlap and run ~10 % slower):
                # its share is given against that profiled pass and, as an upper bound, against the timed step
                "gemm_ms_per_step_profiled": ms.value / n_prof, "profiled_step_ms": prof_step_ms,
                "gemm_share_of_profiled_step": (ms.value / n_prof) / prof_step_ms,
                "gemm_share_of_step": min(1.0, (ms.value / n_prof) / ms_step),
                # whole-step figure: closed-form FLOPs of config 2; for the conv workload the GEMM launches' own counted
                # FLOPs (every conv is a GEMM here) over the timed step
                "step_algorithmic_tflops": (fl.value / n_prof if conv else FLOPS_PER_SAMPLE * Bw) / (ms_step / 1e3) / 1e12,
                "step_frac_of_peak": (fl.value / n_prof if conv else FLOPS_PER_SAMPLE * Bw) / (ms_step / 1e3) / 1e12 / peak_tf}
    if world > 1:
        dist.barrier()

    # ---- gradient exchange in isolation (N > 1): bytes, time and bus bandwidth of the arena all-reduce;
    # measured AFTER the timed regions, never part of `value`. Any failure here leaves the field null.
    allreduce = None
    if world > 1:
        try:
            g = model.arena.grad
            for _ in range(2):
                dist.all_reduce(g)
            torch.cuda.synchronize()
            a0, a1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a0.record()
            for _ in range(5):
                dist.all_reduce(g)
            a1.record()
            torch.cuda.synchronize()
            ar_ms = max_over_ranks(a0.elapsed_time(a1) / 5)
            nbytes = g.numel() * g.element_size()
            allreduce = {"bytes": nbytes, "ms_isolated": ar_ms,
                         "busbw_gbs": 2 * (world - 1) / world * nbytes / (ar_ms / 1e3) / 1e9,
                         "note": "fp32 gradient arena, one NCCL all-reduce, nothing else running; in the step it is issued in "
                                 "slices overlapped with backward"}
            if engine.peer is not None:  # the peer-memory exchange of the whole arena, isolated, same way
                for _ in range(2):
                    engine.peer.allreduce_slice(g, 0, g.numel())
                torch.cuda.synchronize()
                a0.record()
                for _ in range(5):
                    engine.peer.allreduce_slice(g, 0, g.numel())
                a1.record()
                torch.cuda.synchronize()
                pm = max_over_ranks(a0.elapsed_time(a1) / 5)
                allreduce["peer_kernel_ms_isolated"] = pm
                allreduce["peer_kernel_busbw_gbs"] = 2 * (world - 1) / world * nbytes / (pm / 1e3) / 1e9
            g.zero_()
        except Exception as exc:  # diagnostics only
            allreduce = {"error": repr(exc)[:200]}

    cpu = None
    if rank == 0 and world == 1 and not args.no_cpu_baseline and not conv:
        r = cpu_reference_run(steps=1, warmup=1, budget_s=60.0)
        cpu = {"value": r["samples_per_s"], "unit": "samples/s", "cores": r["cores"], "kind": "port", "sample": r["sample"]}

    # ---- the reference's PyTorch-eager path on the SAME GPU in the same run (north_star's ">= 6x over eager" target):
    # HF GPT-J eager + the reference's adapter wiring, bf16, LM frozen (tools/eager_baseline.py: no magma_b200 code)
    gpu_eager = None
    if rank == 0 and world == 1 and not args.no_gpu_eager and not conv:
        try:
            torch.cuda.empty_cache()
            from tools import eager_baseline

            r = eager_baseline.run(steps=min(args.steps, 10), warmup=3, device=f"cuda:{local_rank}")
            gpu_eager = {"value": r["value"], "unit": "samples/s", "ms_per_step": r["ms_per_step"], "impl": r["impl"],
                         "steps": r["steps"], "speedup_e2e": e2e["value"] / r["value"], "speedup_device": value / r["value"]}
        except Exception as exc:  # reported, never fatal for the headline number
            gpu_eager = {"error": repr(exc)[:300]}
        torch.cuda.empty_cache()

    if rank == 0:
        line = {"metric": "image-caption samples/sec (fwd+bwd)", "value": value, "unit": "samples/s",
                "n_gpus": world, "steps": args.steps, "warmup": max(args.warmup, 3), "ms_per_step": ms_step,
                "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "bf16",
                "data": "synthetic", "config": workload_config(world, conv=conv), "e2e": e2e, "gpu_launches": int(launches),
                "clocks": clocks, "roofline": roof, "cpu_baseline": cpu, "gpu_eager": gpu_eager, "allreduce": allreduce,
                "loss": last_loss, "rank_ms_per_step": rank_ms, "gradient_exchange": engine.exchange_kind,
                "trainable_params": int(model.arena.numel)}
        if os.environ.get("MB200_DP_DIAG_NO_EXCHANGE", "0") == "1":
            line["INVALID"] = "diagnostic run: gradient exchange skipped (MB200_DP_DIAG_NO_EXCHANGE=1)"
        print(json.dumps(line), flush=True)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()
    return 0


def run_decode(args):
    """BASELINE.json config 5: Magma.generate, batch 32 per GPU, 224x224 image prefix (2 pooled-ViT tokens) + 6 prompt
    tokens, 256 greedy autoregressive steps over a static KV cache. A "step" of this workload is ONE full generation
    (prefill + 256 decode steps); `value` = generated tokens/s with the prompt embeddings resident in HBM, `e2e` = the
    same through the public API from HOST inputs (pinned fp32 images + int64 prompt ids -> preprocess/embed -> generate ->
    token ids back on the host). Replicas only for N > 1 (inference has no collective). Roofline:
    HBM — algorithmic bytes of a decode step (bf16 weights 12.16 GB + the KV rows read) / its device time."""
    import torch
    import torch.distributed as dist

    from magma_b200 import _lib
    from magma_b200.config import MultimodalConfig
    from magma_b200.magma import Magma
    from magma_b200.utils import init_distributed

    rank, world, local_rank = init_distributed("nccl")
    dev = torch.device("cuda", local_rank)
    torch.cuda.set_device(dev)
    L = _lib.lib()
    B, NEW, NTXT = 32, 256, 6
    mc = MultimodalConfig(batch_size=B, train_steps=1, encoder_name="clip_vit_large",
                          adapter_config={"mlp": {"adapter_type": "normal", "downsample_factor": 4}}, image_seq_len=2,
                          use_image_embed_layernorm=True, image_size=RES)
    model = Magma(mc, device=dev, init_seed=0)
    model.eval()
    model.lm.lm_head.bias.data[50256] = -1e4  # random weights: never emit EOS, so every run executes all 256 steps
    model.lm.invalidate()
    g = torch.Generator().manual_seed(1234 + rank)
    himg = torch.randn(B, 3, RES, RES, generator=g).pin_memory()
    htxt = torch.randint(0, 50000, (B, NTXT), generator=g).pin_memory()

    def embed_from_host():
        return model.embed([himg.to(dev, non_blocking=True).to(torch.bfloat16), htxt.to(dev, non_blocking=True)])

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def max_over_ranks(ms):
        if world > 1:
            t = torch.tensor([ms], device=dev)
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            return float(t)
        return ms

    emb = embed_from_host()
    s0 = emb.shape[1]
    sampler = ClockSampler(local_rank) if rank == 0 else None
    for _ in range(max(1, min(args.warmup, 3))):
        out = model.generate(emb, max_steps=NEW, temperature=0.0, decode=False)
    barrier()
    if sampler:
        sampler.mark()
    launches0 = L.mb200_launch_count()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        out = model.generate(emb, max_steps=NEW, temperature=0.0, decode=False)
    e1.record()
    barrier()
    ms_gen = max_over_ranks(e0.elapsed_time(e1)) / args.steps
    launches = L.mb200_launch_count() - launches0
    clocks = sampler.stop() if sampler else None
    n_new = out.shape[1] - s0
    value = B * world * n_new / (ms_gen / 1e3)
    # e2e: host inputs -> embed (H2D + ViT + prefix) -> generate -> ids on the host
    barrier()
    e0.record()
    for _ in range(args.steps):
        toks = model.generate(embed_from_host(), max_steps=NEW, temperature=0.0, decode=False).cpu()
    e1.record()
    barrier()
    e2e_ms = max_over_ranks(e0.elapsed_time(e1)) / args.steps
    e2e = {"value": B * world * n_new / (e2e_ms / 1e3), "unit": "tokens/s", "ms_per_step": e2e_ms,
           "h2d_bytes_per_step": himg.numel() * 4 + htxt.numel() * 8, "d2h_bytes_per_step": toks.numel() * 8,
           "api": "Magma.embed([images, prompt ids]) -> Magma.generate(embeddings, max_steps=256, temperature=0) -> ids.cpu()"}
    # roofline of the decode step: prefill time is measured separately and excluded from the per-step figure
    barrier()
    e0.record()
    for _ in range(3):
        model.generate(emb, max_steps=1, temperature=0.0, decode=False)
    e1.record()
    barrier()
    ms_prefill = e0.elapsed_time(e1) / 3
    ms_step = (ms_gen - ms_prefill) / max(n_new - 1, 1)
    _, hbm_gbs, peak_src = peaks()
    w_bytes = NL * 201_355_264 * 2 + 235_024_384 * 2 + (V * D + V) * 2
    kv_bytes = B * (s0 + n_new / 2) * NL * 2 * D * 2
    ach = (w_bytes + kv_bytes) / (ms_step / 1e3) / 1e9
    roof = {"kernel": "one decode step (all launches: small-M weight-streaming GEMMs + fused KV-cache attention)",
            "bound": "hbm", "achieved": ach, "peak": hbm_gbs, "unit": "GB/s", "frac": ach / hbm_gbs, "traffic": None,
            "peak_source": peak_src, "algorithmic_bytes_per_step": w_bytes + kv_bytes, "ms_per_decode_step": ms_step,
            "ms_prefill": ms_prefill, "launches_per_generation": int(launches / args.steps)}
    if rank == 0:
        line = {"metric": "decode tokens/sec (greedy, KV cache)", "value": value, "unit": "tokens/s", "n_gpus": world,
                "steps": args.steps, "warmup": max(1, min(args.warmup, 3)), "ms_per_step": ms_gen, "higher_is_better": True,
                "scaling": "weak", "vs_baseline": None, "dtype": "bf16", "data": "synthetic",
                "config": {"workload": "BASELINE.json config 5: Magma.generate, batch 32 per GPU, 224x224 image prefix "
                                       "(ViT-L/14 pooled -> 2 tokens) + 6 prompt tokens, 256 greedy steps, static KV cache, "
                                       "GPT-J-6B + MLP adapters f=4, random-init weights; one step = one full generation",
                           "global_batch": B * world, "prompt_len": s0, "new_tokens": n_new, "parallelism": f"replicas{world}",
                           "l2": "12.2 GB of weights streamed per decode step exceed the 50 MB L2; no explicit flush"},
                "e2e": e2e, "gpu_launches": int(launches), "clocks": clocks, "roofline": roof, "cpu_baseline": None,
                "tokens_head": out[0, s0:s0 + 8].tolist()}
        print(json.dumps(line), flush=True)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()
    return 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write the last timed step's outputs (loss, seeded logits sample) as "
                         "float32 .npy files into DIR")
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-gpu-eager", action="store_true")
    ap.add_argument("--workload", default="train", choices=["train", "decode", "conv"],
                    help="train = BASELINE.json config 2 (the metric's configuration, default); decode = config 5 "
                         "(Magma.generate: batch 32, 224x224 image prefix, 256 greedy steps, KV cache); conv = config 4's "
                         "conv-trunk hot path with the encoder that exists (CLIP RN50x16 @ 384, batch 16, seq_len 272)")
    args = ap.parse_args()
    if args.impl == "reference":
        return run_reference(args)
    if args.workload == "decode":
        if args.dump_outputs:
            ap.error("--dump-outputs writes the outputs of the train / conv step; the decode workload has none")
        return run_decode(args)
    return run_b200(args)


if __name__ == "__main__":
    sys.exit(main())
