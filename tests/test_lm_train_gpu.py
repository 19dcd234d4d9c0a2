"""Training GPT-J's own weights on the GPU.

  * the CPU tests' C-ABI cases (every LM gradient against the oracle's autograd) at small width on the device;
  * every launch configuration the pass adds at GPT-J-6B shapes, replayed against float64;
  * mb200_embed_grad at GPT-J's size against float64, and bit for bit over two runs;
  * GPT-J-6B in Magma with config 2's MLP adapters and the top 2 blocks + ln_f + lm_head trainable, B = 8, S = 128:
    engine steps on a fixed batch lower the loss, the trained weights change and the frozen ones stay bit-identical,
    the peak allocation stays within the estimate from shapes, and a checkpoint restores the trained LM weights."""
import pytest
import torch

from test_gptj_recompute_cpu import case
from test_hidden_states_gpu import on_gpu
from test_lm_train_cpu import LM_TRACE_PASSES, check, new_lm_train_configs, run_train, subset
from test_sched_emul_cpu import FORMS

pytestmark = pytest.mark.gpu


def _lm_trace_cases():
    out, seen = [], set()
    for name in LM_TRACE_PASSES:
        for r, n in new_lm_train_configs(name):
            key = tuple(sorted((k, str(v)) for k, v in r.items() if not isinstance(v, list)))
            if key not in seen:
                seen.add(key)
                out.append((f"{name}-{len(out):02d}-{r['op']}", r))
    return out


LM_TRACE_CASES = _lm_trace_cases()


@pytest.mark.parametrize("cid,rec", LM_TRACE_CASES, ids=[c[0] for c in LM_TRACE_CASES])
def test_lm_train_launch_against_float64(cid, rec):
    """Each launch configuration the LM-training pass adds at GPT-J-6B shapes (tests/test_lm_train_cpu.py pins them),
    replayed with its recorded arguments and held to float64 by the checkers of the production-launch and element-wise
    tests. The fp32 wgrads are replayed again accumulating onto drawn values, as gradient accumulation runs them."""
    import test_elementwise_reference_gpu as ELT
    from test_production_launches_gpu import replay_gemm

    op = rec["op"]
    if op == "gemm":
        replay_gemm(cid, rec, [cid])
        if rec["c_dtype"] == 1:
            _accumulating_wgrad(cid, rec)
    elif op == "colsum":
        for acc in (False, True):
            ELT.test_colsum(rec["rows"], rec["cols"], acc)
    elif op == "layernorm_param_grad_rows":
        for acc in (False, True):
            ELT._ln_param_grad(rec["rows"], rec["d"], True, acc)
    elif op == "logits_grad_combine":
        _combine_in_place_of_itself(rec)
    else:
        raise AssertionError(f"no replay for {op}")


def _accumulating_wgrad(cid, r):
    """The recorded wgrad (MN-major operands at their recorded leading dimensions, the recorded split-K scratch) adding
    onto drawn fp32 values, held to float64 with the old values in the reference."""
    from magma_b200 import ops
    from test_gemm_reference_gpu import _check, _reference

    assert r["a_mn"] and r["b_mn"]
    M, N, K = r["M"], r["N"], r["K"]
    g = torch.Generator(device="cuda").manual_seed(M + 3 * N + 7 * K)
    A = torch.randn(K, r["a_ld"], generator=g, device="cuda").to(torch.bfloat16)[:, :M]
    B = (torch.randn(K, r["b_ld"], generator=g, device="cuda") / K**0.5).to(torch.bfloat16)[:, :N]
    C = torch.randn(M, N, generator=g, device="cuda")
    c_old = C.clone()
    ws = torch.full((r["splitk_ws_bytes"] // 4,), float("nan"), device="cuda")
    ops.gemm(A, B, out=C, a_mn=True, b_mn=True, accumulate=True, splitk_ws=ws)
    torch.cuda.synchronize()
    ref, _, bound, amb = _reference(A.t(), B.t(), alpha=1.0, bias=None, act=0, dact=0, aux_in=None, res1=None, res2=None,
                                 rope=None, c_old=c_old)
    _check(f"{cid} accumulate", C, ref, bound, True, amb)


def _combine_in_place_of_itself(r):
    """The combine the LM head's gradient is formed with when no loss reads the logits: g is the CE gradient itself,
    out = (loss_scale - 1) * dce + dce in fp32, one rounding to bf16. Both products are exact for a bf16 dce and a
    scale of a few bits, so the result is known bit for bit."""
    from magma_b200 import ops

    M, V, ldv, alpha = r["M"], r["V"], r["ldv"], r["alpha"]
    g = torch.Generator(device="cuda").manual_seed(M + V)
    dce = (1e-3 * torch.randn(M, ldv, generator=g, device="cuda")).to(torch.bfloat16)
    before = dce.clone()
    out = torch.full((M, ldv), float("nan"), dtype=torch.bfloat16, device="cuda")
    ops.logits_grad_combine(dce, dce[:, :V], out, alpha)
    torch.cuda.synchronize()
    assert torch.equal(dce.view(torch.int16), before.view(torch.int16))
    want = (dce[:, :V].double() * (1.0 + alpha)).float().to(torch.bfloat16)
    assert torch.equal(out[:, :V].view(torch.int16), want.view(torch.int16))
    assert bool(out[:, V:].isnan().all())


@pytest.mark.parametrize("recompute", [False, True], ids=["stored", "recompute"])
@pytest.mark.parametrize("mlp,attn,mlp_ln,attn_ln", FORMS)
def test_every_lm_gradient_on_device(recompute, mlp, attn, mlp_ln, attn_ln):
    from magma_b200._lib import lib

    cfg, w16, x, labels = case("gemm", mlp, attn, mlp_ln, attn_ln)
    train = subset(cfg, "all")
    check(on_gpu(run_train, lib(), cfg, w16, x, labels, recompute, train), cfg, w16, x, labels, train)


@pytest.mark.parametrize("which", ["last_block", "ln_bias", "head"])
def test_subsets_on_device(which):
    from magma_b200._lib import lib

    cfg, w16, x, labels = case("flash", "normal", "parallel", True, False, seed=2)
    train = subset(cfg, which)
    check(on_gpu(run_train, lib(), cfg, w16, x, labels, False, train), cfg, w16, x, labels, train, tol=5e-2)


def test_embed_grad_against_float64_and_bit_for_bit():
    """Magma's layout: ids = captions[:, :S - L], rows dx[:, L:] of GPT-J width, vocabulary 50258, many repeats, ids
    outside the vocabulary counted as 0."""
    from magma_b200 import ops

    B, S, L, d, V = 8, 128, 2, 4096, 50258
    g = torch.Generator().manual_seed(0)
    captions = torch.randint(0, 64, (B, S), generator=g)
    captions[:, 100:] = 50256  # padding: every row ends in the same token
    captions[0, 5] = -100
    dx = torch.randn(B, S, d, generator=g).to(torch.bfloat16)
    ids = captions[:, : S - L]
    want = torch.zeros(V, d, dtype=torch.float64)
    want.index_add_(0, ids.where((ids >= 0) & (ids < V), 0).reshape(-1), dx[:, L:].double().reshape(-1, d))
    dxd, idd = dx.cuda(), captions.cuda()[:, : S - L]
    outs = [ops.embed_grad(idd, dxd[:, L:], torch.full((V, d), float("nan"), device="cuda")) for _ in range(2)]
    assert torch.equal(outs[0], outs[1])
    n_max = int(torch.bincount(ids.where(ids >= 0, 0).reshape(-1)).max())
    err = (outs[0].cpu().double() - want).abs()
    bound = n_max * 2.0**-24 * want.abs().clamp_min(dx.double().abs().max()) * 2
    assert bool((err <= bound).all()), float(err.max())
    acc = ops.embed_grad(idd, dxd[:, L:], outs[0].clone(), accumulate=True)
    assert torch.allclose(acc, 2 * outs[0], rtol=1e-6, atol=1e-6)


def test_gptj6b_top2_blocks_and_head_train_and_checkpoint(tmp_path):
    from magma_b200.arena import BYTES_PER_PARAM
    from magma_b200.config import MultimodalConfig
    from magma_b200.magma import Magma
    from magma_b200.train_loop import B200Engine

    dev = torch.device("cuda:0")
    torch.cuda.set_device(0)
    mc = MultimodalConfig(batch_size=8, train_steps=1, encoder_name="clip_vit_large",
                          adapter_config={"mlp": {"adapter_type": "normal", "downsample_factor": 4}}, image_seq_len=2,
                          image_embed_dropout_prob=0.0, use_image_embed_layernorm=True, image_size=224, seq_len=128,
                          lr=1e-4, freeze_img_encoder=True)
    model = Magma(mc, device=dev, init_seed=0)
    model.train()
    chosen = ("lm.transformer.h.26.", "lm.transformer.h.27.", "lm.transformer.ln_f.", "lm.lm_head.")
    lm_train = [n for n, _ in model.named_parameters() if n.startswith(chosen) and "adapter" not in n]
    for n, p in model.named_parameters():
        if n in lm_train:
            p.requires_grad_(True)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    model.finalize()
    n_lm = sum(p.numel() for n, p in model.named_parameters() if n in lm_train)
    assert abs(n_lm - (2 * 201.4e6 + 205.9e6)) < 1e6
    frozen = {n: p.detach().clone() for n, p in model.named_parameters()
              if n.startswith(("lm.transformer.h.25.", "lm.transformer.wte.", "lm.transformer.h.0.")) and
              not p.requires_grad}
    before = {n: p.detach().clone() for n, p in model.named_parameters() if n in lm_train}
    g = torch.Generator().manual_seed(0)
    images = torch.randn(8, 3, 224, 224, generator=g).to(dev).to(torch.bfloat16)
    captions = torch.randint(0, 50256, (8, 128), generator=g).to(dev)
    torch.cuda.reset_peak_memory_stats()
    eng = B200Engine(model, mc)
    losses = []
    for _ in range(4):
        o = eng(images, captions)
        eng.backward(o.loss)
        eng.step()
        losses.append(float(o.loss))
    eng.synchronize()
    assert losses[-1] < losses[0], losses
    sd = dict(model.named_parameters())
    assert all(not torch.equal(sd[n], before[n]) for n in lm_train)
    assert all(torch.equal(sd[n], frozen[n]) for n in frozen)
    # estimate from shapes: the model before finalize, the arena with its Adam moments (minus the bf16 copies it
    # replaced), the stored-activation workspace, the logits, the combined logits gradient and its autograd twin, dx
    ws = model.lm._workspace_ex(8, 128)[0].numel()
    lm_bytes = (8 * 128) * (model.lm.ldv * 2 * 3 + 4096 * 2 * 2)
    estimate = base + BYTES_PER_PARAM * model.arena.numel - 2 * n_lm + ws + lm_bytes + (2 << 30)
    peak = torch.cuda.max_memory_allocated()
    assert peak <= estimate, (peak / 2**30, estimate / 2**30)
    # a trainable-only checkpoint carries the trained LM weights; loading it restores them after another step
    eng.save_checkpoint(str(tmp_path), tag="t")
    saved = {n: sd[n].detach().clone() for n in lm_train}
    o = eng(images, captions)
    eng.backward(o.loss)
    eng.step()
    eng.synchronize()
    assert not torch.equal(sd[lm_train[0]], saved[lm_train[0]])
    path, _ = eng.load_checkpoint(str(tmp_path), tag="t")
    assert path is not None
    sd = dict(model.named_parameters())
    assert all(torch.equal(sd[n], saved[n]) for n in lm_train)
