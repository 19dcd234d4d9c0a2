"""Flat parameter arena for the trainable set (adapters + ImagePrefix proj/LN, ~0.24 B params, plus whichever GPT-J
weights train).

All trainable parameters are views into ONE fp32 master buffer, with a parallel bf16 compute copy (what the kernels
read) and a parallel fp32 gradient buffer (what wgrad kernels write). One flat buffer means: the data-parallel
gradient exchange is a handful of large NCCL all-reduces over contiguous slices (replacing DeepSpeed ZeRO-2's
reduce-scatter/all-gather, train.py:103-111), and the optimizer step is one fused kernel over the arena."""
import torch

from . import dp, ops
from ._lib import MB200Error

# what one trainable parameter costs: fp32 master, gradient and two Adam moments, and the bf16 copy the kernels read
BYTES_PER_PARAM = 18


def check_fits(numels, released, free):
    """Raise MB200Error when an arena of parameters with these sizes, Adam moments included, does not fit: `free` is
    what the device can still allocate, `released` the bytes of the parameters' current copies, which the arena
    replaces."""
    need = dp.arena_layout(numels)[1] * BYTES_PER_PARAM
    if need > free + released:
        raise MB200Error(f"the {sum(numels)} trainable parameters need {need} bytes ({need / 2**30:.1f} GiB: "
                         f"{BYTES_PER_PARAM} bytes each for the fp32 master, gradient and two Adam moments and the bf16 "
                         f"copy), but only {int(free + released)} bytes ({(free + released) / 2**30:.1f} GiB) can be "
                         "allocated: train fewer parameters")


class ParamArena:
    def __init__(self, named_params, device, previous=None):
        """named_params: list of (name, nn.Parameter) in the order gradients become ready in backward
        (last layer first), so early slices can be all-reduced while the rest of backward runs. previous: the arena this
        one replaces (its memory is released once the caller drops it), or None."""
        from .language_model import _free_bytes

        self.names = [n for n, _ in named_params]
        self.params = [p for _, p in named_params]
        released = previous.nbytes() if previous is not None else 0
        released += sum(p.numel() * p.element_size() for p in self.params
                        if p.device.type == "cuda" and not (previous is not None and previous.holds(p)))
        check_fits([p.numel() for p in self.params], released, _free_bytes(torch.device(device)))
        self.offsets, off = dp.arena_layout([p.numel() for p in self.params])
        self.numel = off
        self.master = torch.zeros(off, dtype=torch.float32, device=device)
        self.shadow = torch.zeros(off, dtype=torch.bfloat16, device=device)
        # In a data-parallel job on GPUs the gradient buffer is symmetric (peer-mappable) memory, so that the gradient
        # exchange kernel reads and writes the ranks' gradients in place over NVLink (dp.PeerExchange); elsewhere plain.
        self.grad, self.grad_is_symmetric = dp.alloc_gradient_buffer(off, device)
        self._grad_views = []
        self._shadow_views = []
        for p, o in zip(self.params, self.offsets):
            n = p.numel()
            view = self.master[o : o + n].view(p.shape)
            view.copy_(p.data.to(device=device, dtype=torch.float32))
            p.data = view
            self._grad_views.append(self.grad[o : o + n].view(p.shape))
            self._shadow_views.append(self.shadow[o : o + n].view(p.shape))
        self._synced_version = None
        self._ready_event = None  # set by B200Engine.step when the optimizer runs on its own stream (wait_ready)
        self.sync_shadow(force=True)
        self.exp_avg = None
        self.exp_avg_sq = None
        self.gnorm_sq = torch.zeros(1, dtype=torch.float32, device=device)
        self.step_count = 0

    def nbytes(self):
        """Device bytes the arena holds: master, bf16 copy, gradient and the Adam moments once allocated."""
        ts = (self.master, self.shadow, self.grad, self.exp_avg, self.exp_avg_sq)
        return sum(t.numel() * t.element_size() for t in ts if t is not None and t.device.type == "cuda")

    def holds(self, p):
        return any(q is p for q in self.params)

    def _version(self):
        return sum(p._version for p in self.params)

    def wait_ready(self):
        """Order the current stream after the last optimizer step. B200Engine.step launches the fused AdamW on a side
        stream so that it runs under the next step's frozen-encoder forward (HBM-bound beside tensor-bound work); every
        consumer of the arena goes through sync_shadow() first, which calls this. Code that reads parameters directly
        right after engine.step() calls engine.synchronize()."""
        if self._ready_event is not None:
            torch.cuda.current_stream().wait_event(self._ready_event)

    def sync_shadow(self, force=False):
        """Refresh the bf16 compute copy when any master parameter changed (load_state_dict, optimizer.step...)."""
        self.wait_ready()
        v = self._version()
        if force or v != self._synced_version:
            for p, o in zip(self.params, self.offsets):  # guard against .data having been re-pointed by .to()/.half()
                if p.data.data_ptr() != self.master.data_ptr() + o * 4:
                    self.master[o : o + p.numel()].view(p.shape).copy_(p.data.float())
                    p.data = self.master[o : o + p.numel()].view(p.shape)
            ops.cast_f32_to_bf16(self.master, self.shadow)
            self._synced_version = self._version()

    def shadow_of(self, p):
        return self._shadow_views[self._index(p)]

    def grad_of(self, p):
        return self._grad_views[self._index(p)]

    def _index(self, p):
        for i, q in enumerate(self.params):
            if q is p:
                return i
        raise KeyError("parameter not in arena")

    def publish_grads(self):
        """Expose the arena gradient slices as .grad of the master parameters (no copies)."""
        for p, g in zip(self.params, self._grad_views):
            p.grad = g

    def grads_live(self):
        """True when the parameters still hold gradients from an earlier backward (=> accumulate)."""
        return any(p.grad is not None for p in self.params)

    def slice_for(self, prefixes):
        """(lo, hi) element range covering every parameter whose name starts with one of the prefixes."""
        return dp.slice_for(self.names, [p.numel() for p in self.params], self.offsets, prefixes)

    def adamw_step(self, lr, betas=(0.9, 0.95), eps=1e-8, weight_decay=0.0, grad_scale=1.0, max_norm=0.0,
                   segments=None):
        """One fused AdamW pass over the arena. `segments` = [(lo, hi, lr, weight_decay), ...] (dp.optimizer_segments)
        runs the same kernel per parameter group instead — the reference's separate image-encoder learning rate and
        its weight-decay exemptions (magma/utils.py:120-215); the clipping norm stays global over all groups."""
        if self.exp_avg is None:
            self.exp_avg = torch.zeros_like(self.master)
            self.exp_avg_sq = torch.zeros_like(self.master)
        self.step_count += 1
        gn = None
        if max_norm and max_norm > 0:
            self.gnorm_sq.zero_()
            ops.sumsq(self.grad, self.gnorm_sq)
            gn = self.gnorm_sq
        if segments is None or (len(segments) == 1 and segments[0][:2] == (0, self.numel)):
            if segments:
                lr, weight_decay = segments[0][2], segments[0][3]
            ops.adamw_step(self.master, self.grad, self.exp_avg, self.exp_avg_sq, self.shadow, lr, betas[0], betas[1],
                           eps, weight_decay, grad_scale, gn, max_norm or 0.0, self.step_count, zero_grad=True)
        else:
            for lo, hi, slr, swd in segments:
                ops.adamw_step(self.master[lo:hi], self.grad[lo:hi], self.exp_avg[lo:hi], self.exp_avg_sq[lo:hi],
                               self.shadow[lo:hi], slr, betas[0], betas[1], eps, swd, grad_scale, gn, max_norm or 0.0,
                               self.step_count, zero_grad=True)
        for p in self.params:
            p.grad = None
        # the fused kernel wrote master and shadow together: they are in sync without bumping tensor versions
        self._synced_version = self._version()
