"""Activation recomputation in the GPT-J training schedule on the H100: the recompute pass (each block's input kept,
the block rerun right before its backward) gives the stored-activation pass's loss, logits, dx and weight gradients bit
for bit (the 1-D gradients, reduced with atomics, to fp32 reordering; see assert_same), through the C ABI at small and
full width and through Magma.forward + loss.backward(); and it lets GPT-J-6B train at B = 8, S = 2048 on one 80 GB
card, where the stored activations alone would take 78.6 GiB."""
import math

import pytest
import torch

from oracle import magma_oracle as O
from test_gptj_recompute_cpu import assert_identical, case, run
from test_sched_emul_cpu import FORMS

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    from magma_b200 import _lib, build

    build.build()
    return _lib.lib()


def assert_same(got, want):
    """Bit for bit, except the 1-D parameter gradients (biases, LayerNorm parameters, adapter_scale): their kernels
    (colsum_kernel in csrc/elt_kernels.cuh, the LayerNorm parameter gradient and dot_kernel in csrc/train_kernels.cuh)
    add per-chunk fp32 partial sums with atomicAdd, in an order that varies from run to run on the stored path as well.
    Those must agree to within 1e-4 of the vector's largest magnitude, far below what a wrong activation would cause."""
    assert set(got) == set(want)
    reordered = {k for k, v in want.items() if k != "loss" and v.dim() == 1}
    assert_identical({k: got[k] for k in want if k not in reordered}, {k: want[k] for k in want if k not in reordered})
    bad = [k for k in reordered
           if not (got[k] - want[k]).abs().max() <= 1e-4 * want[k].abs().max() + 1e-30]
    assert not bad, bad


def on_gpu(L, cfg, w16, x, labels, recompute, **kw):
    with torch.device("cuda:0"):  # the gradient buffers and workspace the helper allocates
        return run(L, cfg, w16, x, labels, recompute, **kw)


@pytest.mark.parametrize("path", ["tile", "flash"])
@pytest.mark.parametrize("act", [0, 1], ids=["relu", "gelu"])
@pytest.mark.parametrize("mlp,attn,mlp_ln,attn_ln", FORMS)
def test_recompute_matches_stored_at_small_width(lib, path, act, mlp, attn, mlp_ln, attn_ln):
    cfg, w16, x, labels = case(path, mlp, attn, mlp_ln, attn_ln)
    w16 = {k: v.cuda() for k, v in w16.items()}
    x, labels = x.cuda(), labels.cuda()
    stored = on_gpu(lib, cfg, w16, x, labels, False, act=act, accumulate=(0, 1))
    recomputed = on_gpu(lib, cfg, w16, x, labels, True, act=act, accumulate=(0, 1))
    assert torch.isfinite(stored["loss"]).all() and torch.isfinite(stored["dx/0"].float()).all()
    assert_same(recomputed, stored)


def full_width_case(B, S, seed=0):
    """Two GPT-J-6B blocks (d = 4096, 16 heads, rotary 64) with MLP adapters (MAGMA_v1.yml), random weights on the GPU."""
    cfg = O.OracleConfig(d=4096, n_layer=2, n_head=16, rotary_dim=64, vocab=8192,
                         mlp_adapter={"adapter_type": "normal", "downsample_factor": 4}, attn_adapter=None)
    d, dff, r, V = cfg.d, 4 * cfg.d, cfg.d // 4, cfg.vocab
    g = torch.Generator(device="cuda").manual_seed(seed)

    def rnd(*shape, std=0.02, mean=0.0):
        return (mean + std * torch.randn(*shape, generator=g, device="cuda")).to(torch.bfloat16)

    w = {"lm.transformer.ln_f.weight": rnd(d, mean=1.0), "lm.transformer.ln_f.bias": rnd(d),
         "lm.lm_head.weight": rnd(V, d), "lm.lm_head.bias": rnd(V)}
    for l in range(cfg.n_layer):
        p = f"lm.transformer.h.{l}"
        w.update({f"{p}.ln_1.weight": rnd(d, mean=1.0), f"{p}.ln_1.bias": rnd(d),
                  f"{p}.mlp.0.fc_in.weight": rnd(dff, d), f"{p}.mlp.0.fc_in.bias": rnd(dff),
                  f"{p}.mlp.0.fc_out.weight": rnd(d, dff), f"{p}.mlp.0.fc_out.bias": rnd(d),
                  f"{p}.mlp.1.adapter.0.weight": rnd(r, d), f"{p}.mlp.1.adapter.0.bias": rnd(r),
                  f"{p}.mlp.1.adapter.2.weight": rnd(d, r), f"{p}.mlp.1.adapter.2.bias": rnd(d)})
        for n in ("q_proj", "k_proj", "v_proj", "out_proj"):
            w[f"{p}.attn.{n}.weight"] = rnd(d, d)
    x = rnd(B, S, d, std=0.5)
    labels = torch.randint(0, V, (B, S), generator=g, device="cuda")
    labels[:, :2] = -100
    return cfg, w, x, labels


@pytest.mark.parametrize("B,S", [(8, 128), (2, 300), (1, 2048)])
def test_recompute_matches_stored_at_full_width(lib, B, S):
    """S = 128: fused single-tile attention; S = 300 and 2048: multi-tile forward + materialised backward, with the
    split-K GEMM scratch in use. The chunked recompute backward equals the stored single-range one."""
    cfg, w16, x, labels = full_width_case(B, S)
    stored = on_gpu(lib, cfg, w16, x, labels, False, accumulate=(0, 1))
    recomputed = on_gpu(lib, cfg, w16, x, labels, True, accumulate=(0, 1))
    assert torch.isfinite(stored["loss"]).all() and torch.isfinite(stored["dx/0"].float()).all()
    assert_same(recomputed, stored)
    del recomputed
    chunked = on_gpu(lib, cfg, w16, x, labels, True, chunks=[(2, 1), (1, 0)])
    assert_same(chunked, {k: v for k, v in stored.items() if not k.endswith("/1")})


def test_magma_forward_backward_matches_with_recompute_forced(monkeypatch):
    """Magma.forward + loss.backward() (the _EmbedLMFn path, image prefix gradients included) with the path forced
    through the selection function: loss, logits and every trainable gradient agree (assert_same)."""
    from magma_b200 import language_model
    from _gpu_util import build_magma_from_weights

    dev = torch.device("cuda:0")
    cfg = O.OracleConfig(d=512, n_layer=2, n_head=4, rotary_dim=64, vocab=1024, image_seq_len=2, enc_out_dim=96,
                         vit_width=128, vit_layers=2, vit_heads=4, vit_patch=16, vit_image=64, vit_mlp=256,
                         eos_token=1000, image_token=1001)
    w16 = {k: v.to(torch.bfloat16).float() for k, v in O.init_weights(cfg, seed=5).items()}
    S, B = 160, 2
    model = build_magma_from_weights(w16, cfg, {"mlp": {"adapter_type": "normal", "downsample_factor": 4}}, S, dev,
                                     vit_name="clip_vit_recompute")
    model.eval()
    images, captions = O.synthetic_batch(cfg, B, S, seed=11)
    images, captions = images.to(dev).to(torch.bfloat16), captions.to(dev)
    names = [n for n, p in model.named_parameters() if p.requires_grad]
    sd = dict(model.named_parameters())
    results = {}
    for recompute in (False, True):
        monkeypatch.setattr(language_model, "_use_recompute", lambda *a, r=recompute: r)
        model.lm._ws.clear()
        for p in model.parameters():
            p.grad = None
        model.arena.grad.zero_()
        out = model(images, captions)
        out.loss.backward()
        assert model.lm._workspace_ex(B, S)[1] is recompute
        results[recompute] = {"loss": out.loss.detach().clone(), "logits": out.logits.clone(),
                              **{n: sd[n].grad.clone() for n in names}}
    assert any(n.startswith("image_prefix.") for n in names) and any(".adapter." in n for n in names)
    assert_same(results[True], results[False])


def test_gptj6b_trains_at_2048_tokens_with_batch_8():
    """MAGMA_v1.yml's sequence length at B = 8 per GPU: the stored activations (78.6 GiB) do not fit next to the
    weights, so the first train_step selects recompute; it completes with a finite loss and moves the adapters."""
    from magma_b200.config import MultimodalConfig
    from magma_b200.magma import Magma
    from magma_b200.train_loop import B200Engine, train_step

    dev = torch.device("cuda:0")
    B, S = 8, 2048
    mc = MultimodalConfig(batch_size=B, train_steps=1, encoder_name="clip_vit_large",
                          adapter_config={"mlp": {"adapter_type": "normal", "downsample_factor": 4}}, image_seq_len=2,
                          image_embed_dropout_prob=0.0, use_image_embed_layernorm=True, image_size=224, seq_len=S,
                          lr=1e-3, min_lr=1e-4, warmup_num_steps=2)
    model = Magma(mc, device=dev, init_seed=0)
    model.train()
    g = torch.Generator().manual_seed(0)
    images = torch.randn(B, 3, 224, 224, generator=g)
    captions = torch.randint(0, 50256, (B, S), generator=g)
    captions[:, 1500:] = 50256
    eng = B200Engine(model, mc)
    before = model.arena.master.clone()  # fp32 master copy of every trainable parameter (adapters, image prefix)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(dev)
    loss = train_step(mc, iter([(images, captions)]), eng)
    eng.synchronize()
    peak = torch.cuda.max_memory_allocated(dev)
    ws, recompute = model.lm._workspace_ex(B, S)
    print(f"B={B} S={S}: recompute={recompute} workspace {ws.numel() / 2**30:.2f} GiB, loss {loss:.4f}, "
          f"peak allocated {peak / 2**30:.2f} GiB on {torch.cuda.get_device_name(dev)}")
    assert recompute
    assert math.isfinite(loss) and abs(loss - math.log(50258)) < 2.0
    lo, hi = model.arena.slice_for(["lm.transformer.h."])
    assert not torch.equal(model.arena.master[lo:hi], before[lo:hi])  # the adapters moved
    assert peak < torch.cuda.get_device_properties(dev).total_memory
