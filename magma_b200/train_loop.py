"""Training step — drop-in for magma/train_loop.py (`train_step`, `eval_step`) plus `B200Engine`, the object that
stands where the DeepSpeed engine stood (train.py:103-111): `engine(images, captions)`, `engine.backward(loss)`,
`engine.step()`.

Data parallelism is the reference's only strategy. With the LM frozen the only exchange is the
gradient of the ~0.24 B trainable parameters, which live in one flat fp32 arena: the engine sums contiguous arena
slices across ranks (NCCL all-reduce, or this package's peer-memory kernel: dp.PeerExchange) on a side stream as soon as
the backward pass has finished the layers they belong to (backward is issued in layer chunks), so the exchange overlaps
the remaining backward; the fused AdamW kernel, on a stream of its own, then applies 1/world averaging, global-norm
clipping and the bf16 weight refresh in one pass."""
import os

import torch
import torch.distributed as dist

from . import dp
from .utils import reduce_losses


class B200Engine:
    def __init__(self, model, config, n_buckets: int = None, betas=(0.9, 0.95), eps=1e-8):
        if n_buckets is None:  # gradient buckets of the overlapped all-reduce (tuning knob)
            n_buckets = int(os.environ.get("MB200_DP_BUCKETS", "4"))
        self.module = model
        self.config = config
        self.world = dist.get_world_size() if dist.is_initialized() else 1
        self.grad_accum = max(1, int(getattr(config, "gradient_accumulation_steps", 1) or 1))
        self.micro_step = 0
        self.global_step = 0
        self.betas, self.eps = betas, eps
        on_gpu = getattr(getattr(model, "device", None), "type", "cuda") == "cuda"
        # high priority: the exchange's blocks are placed first when SM resources free up, so a slice — and above all the
        # last one, which the optimizer waits for while the next step's encoder forward already runs — finishes sooner
        self.comm_stream = torch.cuda.Stream(priority=-1) if (self.world > 1 and on_gpu) else None
        # The optimizer (global-norm reduction + fused AdamW: 7.2 GB of HBM traffic, ~1.4 ms at 6 B scale) is issued on
        # its own stream, ordered after backward and the gradient exchange. Nothing in the next step reads a trainable
        # parameter before the image prefix projection, so with a frozen encoder it runs beside the next step's encoder
        # forward, and at N > 1 the tail of the gradient exchange hides there too. Consumers are ordered by ParamArena.wait_ready() (called from sync_shadow(), i.e. by every forward);
        # MB200_PIPELINE_OPT=0 puts the optimizer back on the caller's stream.
        self.opt_stream = torch.cuda.Stream() if (on_gpu and os.environ.get("MB200_PIPELINE_OPT", "1") != "0") else None
        if self.opt_stream is not None:
            # a few optimizer blocks per SM run beside the persistent GEMM grids; the default 16 per SM would own every
            # SM until the optimizer is done
            from ._lib import lib

            n_sm = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
            lib().mb200_set_optimizer_grid(int(os.environ.get("MB200_OPT_BLOCKS_PER_SM", "2")) * n_sm)
        # data-parallel knobs, both off by default: exchange gradients as bf16, and keep a few SMs out of the persistent
        # GEMM grids so NCCL's CTAs run beside the backward GEMMs
        self.comm_dtype = torch.bfloat16 if os.environ.get("MB200_DP_BF16", "0") == "1" else None
        # SM carve-out for the gradient exchange: while an all-reduce is in flight (from the first bucket issued in
        # backward until the optimizer step has waited for the last one) the persistent GEMM grids leave all but n SMs
        # alone, so NCCL's CTAs run BESIDE the backward GEMMs instead of queueing behind full-width grids (each NCCL CTA
        # otherwise takes an SM at a kernel boundary and the next GEMM's last CTAs start only when it leaves).
        # Outside that window every kernel gets all SMs. MB200_DP_GEMM_SMS=0 disables it.
        self.dp_gemm_sms = int(os.environ.get("MB200_DP_GEMM_SMS", "0")) if self.world > 1 else 0
        self._carved = False
        # Gradient exchange: NCCL all-reduce per slice, or (MB200_DP_EXCHANGE=peer) this package's peer-memory kernel
        # (dp.PeerExchange); which one ran is in self.exchange_kind (bench.py prints it). dp.exchange_mode() has the
        # default.
        self.peer = None
        self.exchange_kind = "none" if self.world == 1 else "nccl"
        if self.world > 1 and on_gpu and self.comm_dtype is None and dp.exchange_mode() == "peer":
            try:
                n_sm = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
                self.peer = dp.PeerExchange(model.arena.grad, getattr(model.arena, "grad_is_symmetric", False),
                                            max_blocks=int(os.environ.get("MB200_DP_PEER_BLOCKS", str(n_sm))))
                self.exchange_kind = "peer-memory kernel" + (" (in place)" if self.peer.in_place else " (staged)")
            except Exception as exc:  # no peer access / IPC refused in this container: NCCL carries the exchange
                import sys

                print(f"[magma_b200] peer-memory gradient exchange unavailable ({exc!r}); using NCCL", file=sys.stderr)
        # measurement only: MB200_DP_DIAG_NO_EXCHANGE=1 skips the gradient all-reduce (the ranks then train on their own
        # shards — NOT data parallelism), to separate what the exchange costs from what N GPUs of one box cost each
        # other in clocks (bench.py prints the per-rank step times)
        self._diag_no_exchange = os.environ.get("MB200_DP_DIAG_NO_EXCHANGE", "0") == "1"
        self._pending = []
        # MB200_DP_TRACE=1: CUDA-event timeline of one step (main / comm / optimizer streams), printed by trace_report()
        self._trace = [] if os.environ.get("MB200_DP_TRACE", "0") == "1" and on_gpu else None
        self.chunks = dp.layer_chunks(len(model.lm.transformer.h), n_buckets)  # (hi, lo), last layers first
        self._segments = None  # optimizer parameter groups, built at the first step (utils.configure_param_groups)

    # DeepSpeed-engine surface used by the reference -------------------------------------------------
    def __call__(self, images, captions):
        self._mark("forward: enqueue start (main)")
        out = self.module(images, captions)
        self._mark("forward: end (main)")
        return out

    def train(self, mode=True):
        self.module.train(mode)
        return self

    def eval(self):
        self.module.eval()
        return self

    def _mark(self, label, stream=None):
        if self._trace is None:
            return
        ev = torch.cuda.Event(enable_timing=True)
        ev.record(stream if stream is not None else torch.cuda.current_stream())
        self._trace.append((label, ev))

    def trace_report(self):
        """[(label, ms since the first mark)] of everything marked since the last report (synchronizes)."""
        if not self._trace:
            return []
        torch.cuda.synchronize()
        t0 = self._trace[0][1]
        out = [(lab, t0.elapsed_time(ev)) for lab, ev in self._trace]
        self._trace = []
        return out

    def _is_boundary(self):
        return (self.micro_step + 1) % self.grad_accum == 0

    def _allreduce_slice(self, lo, hi):
        arena = self.module.arena
        if self.world == 1 or lo is None or self._diag_no_exchange:
            return
        if self.comm_stream is None:  # host-side dry run (tests): no streams, same collective
            dp.allreduce_slice(arena.grad, lo, hi, comm_dtype=self.comm_dtype)
            return
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream())
        self._mark(f"backward: slice [{lo}, {hi}) ready (main)")
        self.comm_stream.wait_event(ev)
        with torch.cuda.stream(self.comm_stream):
            self._mark(f"exchange [{lo}, {hi}) start (comm)", self.comm_stream)
            if self.peer is not None:
                self.peer.allreduce_slice(arena.grad, lo, hi)
            else:
                dp.allreduce_slice(arena.grad, lo, hi, comm_dtype=self.comm_dtype)
            self._mark(f"exchange [{lo}, {hi}) end (comm)", self.comm_stream)
        if self.dp_gemm_sms > 0 and not self._carved:  # GEMMs launched from here on leave room for NCCL
            from ._lib import lib

            lib().mb200_set_gemm_sm_limit(self.dp_gemm_sms)
            self._carved = True

    def backward(self, loss):
        """engine.backward (train_loop.py:18): loss/grad_accum scaling, chunked backward with overlapped all-reduce
        at the accumulation boundary."""
        lm = self.module.lm
        arena = self.module.arena
        lm._loss_scale_hint = 1.0 / self.grad_accum
        lm._bwd_chunks = self.chunks
        boundary = self._is_boundary()
        if boundary and self.world > 1:
            n_layer = len(lm.transformer.h)

            def after(hi, lo):  # the first chunk also finished the LM head and ln_f, the last one the word embedding
                prefixes = [f"lm.transformer.h.{l}." for l in range(lo, hi)]
                prefixes += ["lm.lm_head.", "lm.transformer.ln_f."] if hi == n_layer else []
                prefixes += ["lm.transformer.wte."] if lo == 0 else []
                s = arena.slice_for(prefixes)
                self._allreduce_slice(*s)
            lm._after_chunk = after
        else:
            lm._after_chunk = None
        self._mark("backward: enqueue start (main)")
        try:
            loss.backward()
        finally:
            lm._loss_scale_hint = None
            lm._after_chunk = None
        self._mark("backward: end (main)")
        if boundary and self.world > 1:
            self._allreduce_slice(*arena.slice_for(["image_prefix."]))

    def step(self):
        """engine.step (train_loop.py:19): optimizer step at the accumulation boundary only."""
        boundary = self._is_boundary()
        self.micro_step += 1
        if not boundary:
            return
        arena = self.module.arena
        if self.opt_stream is not None:
            arena.wait_ready()  # two optimizer steps in a row without a forward in between stay ordered
            self.opt_stream.wait_stream(torch.cuda.current_stream())
        if self.comm_stream is not None:  # the optimizer reads the exchanged gradients
            (self.opt_stream or torch.cuda.current_stream()).wait_stream(self.comm_stream)
        if self._carved:  # GEMMs launched from here on get all SMs again
            from ._lib import lib

            lib().mb200_set_gemm_sm_limit(0)
            self._carved = False
        cfg = self.config
        lr = cfg.lr_at(self.global_step) if hasattr(cfg, "lr_at") else cfg.lr
        if self._segments is None:
            from .utils import configure_param_groups

            self._segments = configure_param_groups(self.module, cfg)
        segs = [(lo, hi, lr * scale, wd) for lo, hi, scale, wd in self._segments]
        kw = dict(lr=lr, betas=self.betas, eps=self.eps, weight_decay=float(getattr(cfg, "weight_decay", 0.0) or 0.0),
                  grad_scale=1.0 / self.world, max_norm=float(getattr(cfg, "gradient_clipping", 0.0) or 0.0),
                  segments=segs)
        if self.opt_stream is not None:
            with torch.cuda.stream(self.opt_stream):
                self._mark("optimizer start (opt)", self.opt_stream)
                arena.adamw_step(**kw)
                self._mark("optimizer end (opt)", self.opt_stream)
                ev = torch.cuda.Event()
                ev.record(self.opt_stream)
            arena._ready_event = ev
        else:
            arena.adamw_step(**kw)
        self.global_step += 1

    def synchronize(self):
        """Order the caller's stream after the last optimizer step (needed only by code that reads parameters directly
        right after step(); forwards and checkpoints do it themselves)."""
        self.module.arena.wait_ready()


    # DeepSpeed-engine checkpoint surface (magma/utils.py:89-117 call these through save_model / load_model) ----------
    def save_checkpoint(self, save_dir, tag=None, client_state=None, trainable_only=True):
        """Writes <save_dir>/<tag>/{mp_rank_00_model_states.pt, b200_optim_states.pt} and <save_dir>/latest (rank 0).
        trainable_only keeps the 12 GB of frozen LM / encoder weights out of the file (they never change); pass False
        for a self-contained checkpoint `Magma.from_checkpoint` can load on its own."""
        from . import checkpoint as ck

        tag = tag if tag is not None else f"global_step{self.global_step}"
        self.synchronize()
        if dist.is_initialized() and dist.get_rank() != 0:
            dist.barrier()
            return True
        model = self.module
        trainable = {n for n, p in model.named_parameters() if p.requires_grad}
        # buffers of every module that owns a trainable parameter travel with it: a training conv trunk updates its
        # BatchNorm running_mean / running_var / num_batches_tracked each forward (image_encoders.py), and the folded
        # eval path reads them
        stateful = set()
        for mname, mod in model.named_modules():
            if any(p is not None and p.requires_grad for p in mod._parameters.values()):
                stateful.update(f"{mname}.{b}" if mname else b for b, t in mod._buffers.items()
                                if t is not None and b not in mod._non_persistent_buffers_set)
        sd = {k: v for k, v in model.state_dict().items()
              if not k.startswith(("word_embedding.", "transformer.")) and
              (not trainable_only or k in trainable or k in stateful)}
        state = dict(client_state or {})
        state.update({"global_step_engine": self.global_step, "micro_step": self.micro_step,
                      "trainable_only": bool(trainable_only)})
        ck.save_training_checkpoint(save_dir, tag, sd, ck.arena_optimizer_state(model.arena), state)
        if dist.is_initialized():
            dist.barrier()
        return True

    def load_checkpoint(self, load_dir, tag=None, load_optimizer_states=True, load_lr_scheduler_states=True):
        """-> (load_path, client_state) like DeepSpeed; (None, None) when nothing is found. The learning-rate schedule is
        a pure function of the step counter here (config.lr_at), so restoring the counter restores the scheduler."""
        from . import checkpoint as ck

        path, payload, optim = ck.read_training_checkpoint(load_dir, tag)
        if path is None:
            return None, None
        model = self.module
        self.synchronize()
        sd = payload.pop("module")
        missing, unexpected = model.load_state_dict(sd, strict=False)
        if unexpected:
            raise RuntimeError(f"checkpoint has {len(unexpected)} keys the model does not (e.g. {list(unexpected)[:4]})")
        missing = [k for k in missing if not k.startswith(("word_embedding.", "transformer."))]
        if payload.get("trainable_only", False):  # frozen weights are not in the file; everything that trains must be
            need = {n for n, p in model.named_parameters() if p.requires_grad}
            for mname, mod in model.named_modules():
                if any(p is not None and p.requires_grad for p in mod._parameters.values()):
                    need.update(f"{mname}.{b}" if mname else b for b, t in mod._buffers.items()
                                if t is not None and b not in mod._non_persistent_buffers_set)
            missing = [k for k in missing if k in need]
        if missing:
            raise RuntimeError(f"checkpoint lacks {len(missing)} model keys (e.g. {missing[:4]})")
        if optim is not None:
            ck.load_arena_optimizer_state(model.arena, optim, load_optimizer_states)
        else:
            model.arena.sync_shadow(force=True)
        if load_lr_scheduler_states:
            self.global_step = int(payload.get("global_step_engine", payload.get("global_step", 0)))
            self.micro_step = int(payload.get("micro_step", 0))
        model.lm.invalidate()
        model.lm.attach_arena(model.arena)
        if hasattr(model.image_prefix.enc, "invalidate"):
            model.image_prefix.enc.invalidate()
        return path, payload


def _to_device(images, captions):
    return images.cuda(non_blocking=True).to(torch.bfloat16), captions.cuda(non_blocking=True)


def train_step(config, train_loader, model_engine):
    """magma/train_loop.py:7-21 (images.half() there; bf16 here)."""
    losses = []
    for _ in range(config.gradient_accumulation_steps):
        images, captions = next(train_loader)
        images, captions = _to_device(images, captions)
        if config.run_blind:
            images = torch.zeros_like(images)
        outputs = model_engine(images, captions)
        loss = outputs.loss
        losses.append(loss.detach())
        model_engine.backward(loss)
        model_engine.step()
    return reduce_losses(torch.mean(torch.stack(losses))).item()


def eval_step(config, eval_loader, model_engine):
    """magma/train_loop.py:48-60."""
    losses = []
    with torch.no_grad():
        for _ in range(config.eval_steps):
            images, captions = next(eval_loader)
            images, captions = _to_device(images, captions)
            if config.run_blind:
                images = torch.zeros_like(images)
            outputs = model_engine(images, captions)
            losses.append(outputs.loss)
    return reduce_losses(torch.mean(torch.stack(losses))).item()
