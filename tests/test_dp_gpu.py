"""Hardware data-parallel parity ("Distributed"): on 2 GPUs, with the gradient exchange carried by
this package's peer-memory kernel (default), by NCCL, and by NCCL with a bf16 wire format, the gradients the engine
holds after its overlapped exchange — divided by the world size, as the fused optimizer kernel does — equal the
single-GPU gradients of the CONCATENATED batch, and one optimizer step leaves every rank with identical parameters
that equal the single-GPU step. Reference semantics: DeepSpeed data parallelism averages the per-rank mean losses'
gradients (train.py:103-111, magma/utils.py:26-34), which equals the gradient of the mean over the concatenated batch
when every rank holds the same number of valid label tokens — the captions below are built that way.

Needs 2 visible GPUs; skipped otherwise."""
import os

import pytest

pytestmark = pytest.mark.gpu


def _worker(rank, world, port, out_dir, mode):
    import torch
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    comm_bf16 = mode == "nccl-bf16"
    if comm_bf16:
        os.environ["MB200_DP_BF16"] = "1"
    os.environ["MB200_DP_EXCHANGE"] = "peer" if mode == "peer" else "nccl"
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world)
    from _gpu_util import build_magma_from_weights
    from magma_b200.train_loop import B200Engine
    from oracle import magma_oracle as O
    from tools.model_check import boost_adapters, small_cfg

    dev = torch.device("cuda", rank)
    cfg = small_cfg(n_layer=4)
    torch.manual_seed(5)
    w = boost_adapters(O.init_weights(cfg, seed=5), True)
    w16 = {k: v.to(torch.bfloat16).float() for k, v in w.items()}
    S, B = 32, 4  # global batch 4: rank r takes samples [2r, 2r + 2)
    images, captions = O.synthetic_batch(cfg, B, S, seed=11)
    captions = captions.clone()
    captions[:, 20:] = cfg.eos_token   # every row: the same number of valid label tokens
    captions[:, :20] = captions[:, :20].clamp(max=cfg.eos_token - 1)
    model = build_magma_from_weights(w16, cfg, {"mlp": {"adapter_type": "normal", "downsample_factor": 4}}, S, dev)
    model.train()
    model.config.image_embed_dropout_prob = 0.0
    eng = B200Engine(model, model.config, n_buckets=2)
    if mode == "peer":  # no silent NCCL fallback in the test of the peer-memory kernel
        assert eng.exchange_kind == "peer-memory kernel (in place)", eng.exchange_kind
    lo, hi = rank * (B // world), (rank + 1) * (B // world)
    out = eng(images[lo:hi].to(dev).to(torch.bfloat16), captions[lo:hi].to(dev))
    eng.backward(out.loss)
    torch.cuda.current_stream().wait_stream(eng.comm_stream)
    torch.cuda.synchronize()
    grads = (model.arena.grad / world).float().cpu()
    eng.global_step = 5  # WarmupLR gives lr = 0 at step 0; take the step at a non-zero learning rate
    eng.step()
    torch.cuda.synchronize()
    torch.save({"grads": grads, "loss": float(out.loss.detach()), "master": model.arena.master.float().cpu()},
               os.path.join(out_dir, f"rank{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


def _single(out_dir):
    import torch

    from _gpu_util import build_magma_from_weights
    from oracle import magma_oracle as O
    from tools.model_check import boost_adapters, small_cfg

    dev = torch.device("cuda", 0)
    cfg = small_cfg(n_layer=4)
    torch.manual_seed(5)
    w = boost_adapters(O.init_weights(cfg, seed=5), True)
    w16 = {k: v.to(torch.bfloat16).float() for k, v in w.items()}
    S, B = 32, 4
    images, captions = O.synthetic_batch(cfg, B, S, seed=11)
    captions = captions.clone()
    captions[:, 20:] = cfg.eos_token
    captions[:, :20] = captions[:, :20].clamp(max=cfg.eos_token - 1)
    model = build_magma_from_weights(w16, cfg, {"mlp": {"adapter_type": "normal", "downsample_factor": 4}}, S, dev)
    model.train()
    model.config.image_embed_dropout_prob = 0.0
    out = model(images.to(dev).to(torch.bfloat16), captions.to(dev))
    out.loss.backward()
    torch.cuda.synchronize()
    return model.arena.grad.float().cpu(), float(out.loss.detach()), model.arena.names


@pytest.mark.parametrize("mode", ["peer", "nccl", "nccl-bf16"])
def test_allreduced_gradients_equal_the_concatenated_batch(tmp_path, mode):
    import torch
    import torch.multiprocessing as mp

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    world = 2
    comm_bf16 = mode == "nccl-bf16"
    port = 29500 + (os.getpid() % 1000) + {"peer": 0, "nccl": 7, "nccl-bf16": 14}[mode]
    mp.spawn(_worker, args=(world, port, str(tmp_path), mode), nprocs=world, join=True)
    r0 = torch.load(tmp_path / "rank0.pt")
    r1 = torch.load(tmp_path / "rank1.pt")
    g_ref, loss_ref, _ = _single(str(tmp_path))
    rel = lambda a, b: ((a - b).norm() / (b.norm() + 1e-12)).item()
    # every rank ends with the same summed gradients (bit-identical: one NCCL all-reduce result) and parameters
    assert torch.equal(r0["grads"], r1["grads"])
    assert torch.equal(r0["master"], r1["master"])
    # mean of the rank losses = loss of the concatenated batch (equal valid-token counts)
    assert abs(0.5 * (r0["loss"] + r1["loss"]) - loss_ref) < 5e-3
    # all-reduced / world == single-GPU gradients of the concatenated batch. fp32 exchange: only the bf16 storage of
    # activations differs between a batch-2 and a batch-4 run (none — rows are independent), so the match is tight;
    # bf16 exchange rounds each rank's gradient once (2^-9 relative).
    tol = 1.5e-2 if comm_bf16 else 2e-3
    e = rel(r0["grads"], g_ref)
    print(f"DP parity (N = 2, {mode} exchange): rel-Frobenius {e:.2e} over {g_ref.numel()} "
          f"gradient elements; loss {loss_ref:.4f}")
    assert e < tol, e
