"""Data-parallel host logic (pure Python, device-agnostic so it is testable with gloo on CPU).

The reference's only parallelism is DP under DeepSpeed ZeRO-2 (train.py:103-111). Here every rank
holds the full (frozen) model and a flat fp32 gradient arena for the ~0.24 B trainable parameters; the arena is
laid out in the order gradients become ready in backward (last GPT-J layer first, image prefix last) and is
all-reduced slice by slice as backward proceeds."""
import re
from typing import List, Sequence, Tuple

import torch
import torch.distributed as dist

ALIGN = 64  # elements; keeps every parameter view 256-byte aligned


def arena_layout(numels: Sequence[int]) -> Tuple[List[int], int]:
    """Offsets (in elements) of each parameter in the flat arena and the total padded length."""
    offs, off = [], 0
    for n in numels:
        offs.append(off)
        off += (n + ALIGN - 1) // ALIGN * ALIGN
    return offs, off


_BLOCK = re.compile(r"(?:^|\.)transformer\.h\.(\d+)\.")
_HEAD = re.compile(r"(?:^|\.)(?:lm_head|transformer\.ln_f)\.")


def backward_order_key(name: str):
    """Sort key in the order the backward produces gradients: the LM head and ln_f, GPT-J layers descending, then
    everything else (the word embedding and the image prefix, from the input gradient). Names may carry a prefix
    (`lm.` in Magma)."""
    if _HEAD.search(name):
        return (0, 0)
    m = _BLOCK.search(name)
    if m:
        return (1, -int(m.group(1)))
    return (2, 0)


def layer_chunks(n_layer: int, n_buckets: int) -> List[Tuple[int, int]]:
    """[(layer_hi, layer_lo), ...] covering [0, n_layer) from the top down in n_buckets nearly equal chunks."""
    nb = max(1, min(n_buckets, n_layer))
    bounds = [round(i * n_layer / nb) for i in range(nb + 1)]
    return [(bounds[i + 1], bounds[i]) for i in reversed(range(nb))]


def slice_for(names: Sequence[str], numels: Sequence[int], offsets: Sequence[int], prefixes: Sequence[str]):
    """(lo, hi) element range of the arena covering all parameters whose name starts with one of `prefixes`
    (None, None when there is none)."""
    lo = hi = None
    for n, k, o in zip(names, numels, offsets):
        if any(n.startswith(p) for p in prefixes):
            e = o + (k + ALIGN - 1) // ALIGN * ALIGN
            lo = o if lo is None else min(lo, o)
            hi = e if hi is None else max(hi, e)
    return lo, hi


def allreduce_slice(flat_grad: torch.Tensor, lo, hi, group=None, comm_dtype=None):
    """SUM all-reduce of one contiguous arena slice (averaging by 1/world is folded into the optimizer kernel).
    comm_dtype=torch.bfloat16 exchanges a bf16 copy of the slice (half the NVLink bytes; the reference exchanged fp16
    gradients under DeepSpeed fp16, train.py:103-111) and writes the summed values back into the fp32 arena."""
    if lo is None or not dist.is_initialized() or dist.get_world_size(group) == 1:
        return None
    view = flat_grad[lo:hi]
    if comm_dtype is None or comm_dtype == view.dtype:
        return dist.all_reduce(view, op=dist.ReduceOp.SUM, group=group)
    buf = view.to(comm_dtype)
    dist.all_reduce(buf, op=dist.ReduceOp.SUM, group=group)
    view.copy_(buf)
    return None


def exchange_mode() -> str:
    """'nccl' (default) or 'peer' (MB200_DP_EXCHANGE): which mechanism carries the gradient exchange. Both are built
    and parity-tested on 2 GPUs."""
    import os

    m = os.environ.get("MB200_DP_EXCHANGE", "nccl").lower()
    return "peer" if m == "peer" else "nccl"


def alloc_gradient_buffer(numel: int, device):
    """(zeroed fp32 buffer, is_symmetric). Symmetric memory (torch.distributed._symmetric_memory) when a multi-rank
    process group exists, the device is a GPU and the peer-memory exchange is selected (the default); a failure to
    allocate it is not an error — the exchange then stages through its own buffer or uses NCCL."""
    import os

    device = torch.device(device)
    if (device.type == "cuda" and dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1
            and exchange_mode() == "peer" and os.environ.get("MB200_DP_BF16", "0") != "1"):
        try:
            import torch.distributed._symmetric_memory as symm

            t = symm.empty(numel, dtype=torch.float32, device=device)
            t.zero_()
            return t, True
        except Exception:
            pass
    return torch.zeros(numel, dtype=torch.float32, device=device), False


def shard_bounds(lo: int, hi: int, world: int, align: int = ALIGN) -> List[Tuple[int, int]]:
    """Cut the arena slice [lo, hi) into `world` contiguous shards (the last ones may be empty), each a multiple of
    `align` elements except possibly the tail: shard r is what rank r reduces in the peer-memory exchange."""
    n = hi - lo
    per = ((n + world - 1) // world + align - 1) // align * align
    out = []
    for r in range(world):
        s0 = min(hi, lo + r * per)
        out.append((s0, min(hi, s0 + per)))
    return out


class PeerExchange:
    """SUM all-reduce of arena slices over NVLink peer memory with this package's own kernel
    (csrc/elt_kernels.cuh::peer_reduce_bcast_kernel) instead of NCCL.

    Why: NCCL's all-reduce kernels need shared memory, so each of their CTAs needs an SM of its own; the persistent GEMM
    grids of backward own every SM, the collective only gets SMs at kernel boundaries, and the GEMM whose CTAs it
    displaces runs a second wave. The kernel here uses no shared memory and ~40 registers, so its blocks can sit BESIDE
    the GEMM CTAs.

    Layout: the arena's fp32 gradient buffer is symmetric memory (torch.distributed._symmetric_memory: allocation, handle
    exchange and the device-side barrier are torch's; the data path is ours), so the exchange works IN PLACE. Per slice,
    on the comm stream: barrier (every rank's slice is final); rank r sums shard r of the slice over all ranks' gradient
    buffers in rank order and stores the sum into all of them (loads / stores over NVLink); barrier. All ranks end with
    identical bits. If a rank's arena predates the process group, a symmetric staging copy E is used instead
    (E <- grad before, grad <- E after).
    """

    def __init__(self, flat_grad: torch.Tensor, grad_is_symmetric: bool, group=None, max_blocks: int = 0):
        import torch.distributed._symmetric_memory as symm

        self.group = group if group is not None else dist.group.WORLD
        self.world, self.rank = dist.get_world_size(self.group), dist.get_rank(self.group)
        # in place when the arena's gradient buffer is itself symmetric on EVERY rank (the usual case: ParamArena
        # allocates it that way once the process group exists); else through a symmetric staging copy E of it
        flags = [None] * self.world
        dist.all_gather_object(flags, bool(grad_is_symmetric), group=self.group)
        self.in_place = all(flags)
        self.E = flat_grad if self.in_place else symm.empty(flat_grad.numel(), dtype=torch.float32,
                                                            device=flat_grad.device)
        self.hdl = symm.rendezvous(self.E, self.group)
        self.ptrs = [int(p) for p in self.hdl.buffer_ptrs]
        assert len(self.ptrs) == self.world and self.ptrs[self.rank] == self.E.data_ptr()
        self.max_blocks = max_blocks

    def allreduce_slice(self, flat_grad: torch.Tensor, lo: int, hi: int):
        from . import ops

        if lo is None or hi <= lo:
            return
        if not self.in_place:
            self.E[lo:hi].copy_(flat_grad[lo:hi])
        self.hdl.barrier(channel=0)                      # every rank's slice is final / published
        s0, s1 = shard_bounds(lo, hi, self.world)[self.rank]
        if s1 > s0:
            ops.peer_reduce_bcast(self.ptrs, s0, s1 - s0, self.max_blocks)
        self.hdl.barrier(channel=0)                      # every shard's sum has landed on every rank
        if not self.in_place:
            flat_grad[lo:hi].copy_(self.E[lo:hi])


def shard_batch(global_batch: int, rank: int, world: int) -> Tuple[int, int]:
    """Rank `rank` takes samples [lo, hi) of the global batch (rank i takes [8i, 8i+8))."""
    per = global_batch // world
    assert per * world == global_batch, "global batch must divide evenly across ranks"
    return rank * per, (rank + 1) * per


def optimizer_segments(names: Sequence[str], numels: Sequence[int], offsets: Sequence[int], no_decay: Sequence[bool],
                       lr: float, image_enc_lr, weight_decay: float, enc_prefix: str = "image_prefix.enc."):
    """Parameter groups of the reference optimizer (magma/utils.py:120-215) mapped onto the flat arena: contiguous runs
    [(lo, hi, lr, weight_decay), ...] of parameters sharing a learning rate and decay. The image encoder gets
    `image_enc_lr` when it is set (utils.py:173-177); LayerNorm / embedding parameters and biases are exempt from
    weight decay (utils.py:128-146). With weight_decay == 0 and no separate encoder rate this is ONE run — the whole
    arena in one fused kernel launch."""
    segs = []
    for n, k, o, nd in zip(names, numels, offsets, no_decay):
        plr = image_enc_lr if (image_enc_lr is not None and n.startswith(enc_prefix)) else lr
        pwd = 0.0 if (nd or weight_decay == 0.0) else weight_decay
        hi = o + (k + ALIGN - 1) // ALIGN * ALIGN
        if segs and segs[-1][1] == o and segs[-1][2] == plr and segs[-1][3] == pwd:
            segs[-1] = (segs[-1][0], hi, plr, pwd)
        else:
            segs.append((o, hi, plr, pwd))
    return segs
