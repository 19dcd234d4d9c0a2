"""CPU tests of the data-parallel host logic with torch.distributed(gloo), world_size 2:
sharding by batch + SUM all-reduce of contiguous arena slices in backward order reproduces the single-process
gradient of the concatenated batch."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from magma_b200 import dp


def test_layout_and_chunks():
    offs, total = dp.arena_layout([10, 64, 65, 1])
    assert offs == [0, 64, 128, 256] and total == 320
    assert dp.layer_chunks(28, 4) == [(28, 21), (21, 14), (14, 7), (7, 0)]
    assert dp.layer_chunks(2, 8) == [(2, 1), (1, 0)]
    ch = dp.layer_chunks(28, 3)
    assert ch[0][0] == 28 and ch[-1][1] == 0 and all(a[1] == b[0] for a, b in zip(ch, ch[1:]))
    names = ["lm.transformer.h.0.mlp.1.adapter.0.weight", "image_prefix.proj.weight",
             "lm.transformer.h.3.mlp.1.adapter.0.weight", "lm.transformer.h.12.attn.adapter.2.bias"]
    order = sorted(names, key=dp.backward_order_key)
    assert [n.split(".h.")[1].split(".")[0] for n in order[:3]] == ["12", "3", "0"] and order[3].startswith("image_prefix")
    assert dp.shard_batch(64, 3, 8) == (24, 32)
    with pytest.raises(AssertionError):
        dp.shard_batch(10, 0, 4)


def test_slice_for_is_contiguous_per_layer_chunk():
    names, numels = [], []
    for l in reversed(range(6)):
        for p, n in (("adapter.0.weight", 100), ("adapter.0.bias", 7), ("adapter.2.weight", 100), ("adapter.2.bias", 3)):
            names.append(f"lm.transformer.h.{l}.mlp.1.{p}")
            numels.append(n)
    names += ["image_prefix.proj.weight", "image_prefix.ln.bias"]
    numels += [50, 5]
    offs, total = dp.arena_layout(numels)
    covered = []
    for hi, lo in dp.layer_chunks(6, 3):
        s = dp.slice_for(names, numels, offs, [f"lm.transformer.h.{l}." for l in range(lo, hi)])
        covered.append(s)
    covered.append(dp.slice_for(names, numels, offs, ["image_prefix."]))
    assert covered[0][0] == 0 and covered[-1][1] == total
    assert all(a[1] == b[0] for a, b in zip(covered, covered[1:]))  # slices tile the arena in backward order
    assert dp.slice_for(names, numels, offs, ["nothing."]) == (None, None)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        torch.manual_seed(0)
        n_layer, dim = 4, 16
        # a toy "trainable set" with the arena layout of the product: per-layer weight+bias, then a prefix tensor
        names, shapes = [], []
        for l in reversed(range(n_layer)):
            names += [f"lm.transformer.h.{l}.mlp.1.adapter.0.weight", f"lm.transformer.h.{l}.mlp.1.adapter.0.bias"]
            shapes += [(dim, dim), (dim,)]
        names.append("image_prefix.proj.weight")
        shapes.append((dim, 3))
        numels = [int(torch.tensor(s).prod()) for s in shapes]
        offs, total = dp.arena_layout(numels)
        params = [torch.randn(*s) for s in shapes]  # identical on both ranks (same seed)
        X = torch.randn(8, dim)                      # global batch of 8, identical on both ranks
        lo, hi = dp.shard_batch(8, rank, world)

        def loss_and_grads(x):
            ps = [p.clone().requires_grad_(True) for p in params]
            h = x
            for l in range(n_layer):
                i = 2 * (n_layer - 1 - l)
                h = torch.tanh(h @ ps[i].t() + ps[i + 1])
            out = (h @ ps[-1]).pow(2).sum() / x.shape[0]
            out.backward()
            return out.detach(), [p.grad for p in ps]

        _, g_local = loss_and_grads(X[lo:hi])
        flat = torch.zeros(total)
        for g, o, n in zip(g_local, offs, numels):
            flat[o:o + n] = g.reshape(-1)
        # exchange slice by slice in backward order, exactly like B200Engine.backward
        for c_hi, c_lo in dp.layer_chunks(n_layer, 2):
            s = dp.slice_for(names, numels, offs, [f"lm.transformer.h.{l}." for l in range(c_lo, c_hi)])
            dp.allreduce_slice(flat, *s)
        dp.allreduce_slice(flat, *dp.slice_for(names, numels, offs, ["image_prefix."]))
        flat /= world  # the product folds this into the fused AdamW kernel (grad_scale = 1/world)
        _, g_full = loss_and_grads(X)
        ok = all(torch.allclose(flat[o:o + n].view(s), g, atol=1e-5) for g, o, n, s in zip(g_full, offs, numels, shapes))
        # bf16 exchange option: same sums up to bf16 rounding of each rank's contribution, result back in fp32
        flat2 = torch.zeros(total)
        for g, o, n in zip(g_local, offs, numels):
            flat2[o:o + n] = g.reshape(-1)
        dp.allreduce_slice(flat2, 0, total, comm_dtype=torch.bfloat16)
        flat2 /= world
        ok = ok and flat2.dtype == torch.float32 and \
            ((flat2 - flat).norm() / flat.norm()).item() < 1e-2 and not torch.equal(flat2, flat)
        # reduce_losses (magma/utils.py:26-34)
        from magma_b200.utils import reduce_losses

        r = reduce_losses(torch.tensor(float(rank + 1)))
        ok = ok and abs(float(r) - 1.5) < 1e-6
        q.put((rank, ok))
    finally:
        dist.destroy_process_group()


def test_two_rank_gradient_exchange_matches_single_process():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert sorted(res) == [(0, True), (1, True)]
