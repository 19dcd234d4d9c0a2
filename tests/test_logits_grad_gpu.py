"""Gradients through the training logits on the GPU.

  * mb200_logits_grad_combine element by element against float64, bit for bit: the gradient rows at the strides autograd hands
    over (V = 50258 gives 4-byte aligned rows, an odd V 2-byte aligned ones), alpha 0 over a NaN-filled CE gradient,
    ragged M, sentinel-guarded output, inputs unchanged byte for byte;
  * the CPU tests' C-ABI cases at small width on the GPU;
  * GPT-J-6B with config 2's MLP adapters and Magma's vocabulary of 50258 through B200GPTJForCausalLM, stored (B = 8, S = 128) and recompute
    (B = 1, S = 2048): F.cross_entropy on the logits of a pass without labels gives the gradients of the runtime's own
    loss, and the gradients are linear in the loss."""
import pytest
import torch
import torch.nn.functional as F

import test_elementwise_reference_gpu as E
from _refcheck import SENTINEL, dev as _dev
from test_gptj_recompute_cpu import case
from test_hidden_states_gpu import on_gpu, rel_dev
from test_logits_grad_cpu import check, loss_fn, run_train

pytestmark = pytest.mark.gpu


def combine_body(M, V, ld_g, alpha):
    """One mb200_logits_grad_combine call against float64: out = bf16(fp32 fma(alpha, dce, g))."""
    from magma_b200 import ops

    dev, bf = _dev(), torch.bfloat16
    name = f"logits_grad_combine M={M} V={V} ld_g={ld_g} alpha={alpha}"
    ldv = (V + 63) // 64 * 64
    gen = E._gen("logits_grad_combine", M, V, ld_g, alpha)
    dce = torch.full((M, ldv), float("nan"), dtype=bf, device=dev)
    if alpha != 0:  # alpha == 0 must never read it: left NaN
        dce[:, :V] = (torch.randn(M, V, generator=gen, dtype=torch.float64) * 1e-4).to(bf).to(dev)
    gs = torch.full((M * ld_g + 8,), float("nan"), dtype=bf, device=dev)
    g = gs[: M * ld_g].view(M, ld_g)[:, :V]
    g.copy_((torch.randn(M, V, generator=gen, dtype=torch.float64) * 1e-3).to(bf).to(dev))
    out = torch.full((M + 2, ldv), SENTINEL, dtype=bf, device=dev)
    inp = E._Inputs(dce, gs)
    n0 = E._count()
    ops.logits_grad_combine(dce, g, out[:M], alpha)
    E._launched(name, n0)
    inp.unchanged(name)
    keep = torch.ones_like(out, dtype=torch.bool)
    keep[:M, :V] = False
    assert E._same(out[keep], torch.full_like(out[keep], SENTINEL)), f"{name}: sentinel overwritten"
    # alpha is a power of two (or 0) and both operands are bf16, so alpha * dce + g is exact in float64: the one fp32
    # rounding of the kernel's fma is the float64 -> float32 rounding, and its bf16 result is known bit for bit
    ref = g.double() + (alpha * dce[:, :V].double() if alpha != 0 else 0.0)
    want = ref.to(torch.float32).to(bf)
    bad = int((E.bits(out[:M, :V]) != E.bits(want)).sum().item())
    assert bad == 0, f"{name}: {bad} of {M * V} elements differ from the float64 reference rounded fp32 -> bf16"


@pytest.mark.parametrize("alpha", [0.0, 1.0, 0.125])
@pytest.mark.parametrize("V,ld", [(50258, "V"), (50258, "ldv"), (1031, "V"), (1031, "ldv")])
@pytest.mark.parametrize("M", [1024, 37])
def test_logits_grad_combine_against_float64(M, V, ld, alpha):
    combine_body(M, V, V if ld == "V" else (V + 63) // 64 * 64, alpha)


def test_logits_grad_combine_rejects_bad_arguments():
    from magma_b200._lib import lib

    t = torch.zeros(4, 64, dtype=torch.bfloat16, device="cuda")
    p = t.data_ptr()
    assert lib().mb200_logits_grad_combine(p, 64, p, 31, p, 4, 32, 1.0, None) != 0  # ld_g < V
    assert lib().mb200_logits_grad_combine(p + 2, 64, p, 64, p, 4, 32, 1.0, None) != 0  # dce not 16-byte aligned
    assert lib().mb200_logits_grad_combine(None, 64, p, 64, p, 4, 32, 1.0, None) != 0  # NULL dce with alpha != 0
    assert lib().mb200_logits_grad_combine(None, 64, p, 64, p, 4, 32, 0.0, None) == 0


# ---- small width through the C ABI --------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    from magma_b200 import _lib, build

    build.build()
    return _lib.lib()


@pytest.mark.parametrize("kind", ["ce_lin", "kl", "zlin_no_labels"])
@pytest.mark.parametrize("recompute", [False, True], ids=["stored", "recompute"])
@pytest.mark.parametrize("path", ["tile", "flash"])
def test_logits_loss_gradients_at_small_width(lib, kind, recompute, path):
    cfg, w16, x, labels = case(path, "normal", "normal", False, False)
    B, S = labels.shape
    f, reads_ce = loss_fn(kind, cfg.vocab, B, S)
    lab = labels if kind != "zlin_no_labels" else None
    got = on_gpu(run_train, lib, cfg, w16, x, lab, recompute, f=f, ld_g=cfg.vocab + 1, reads_ce=reads_ce)
    check(got, cfg, w16, x, labels, f, reads_ce)


# ---- full size: GPT-J-6B + config 2's MLP adapters ----------------------------------------------------------------
@pytest.fixture(scope="module")
def gptj6b_adapters():
    from magma_b200.adapters import Adapter
    from magma_b200.language_model import get_gptj

    torch.cuda.set_device(0)
    lm = get_gptj(device="cuda:0").init_weights(seed=0)
    lm.resize_token_embeddings(50258)  # as Magma does (magma/magma.py:50): G's rows are 4-byte aligned only
    torch.manual_seed(0)
    for blk in lm.transformer.h:  # magma/magma.py:143-148 with config 2's {"adapter_type": "normal", "downsample_factor": 4}
        ad = Adapter(dim=lm.config.hidden_size, downsample_factor=4)
        ad.adapter[-1].weight.data.normal_(std=2e-2)  # an up projection that moves the residual stream
        blk.mlp = torch.nn.Sequential(blk.mlp, ad.to("cuda:0"))
    lm.invalidate()
    return lm


# Bound: the runtime's own CE gradient and F.cross_entropy's are each the bf16 rounding of (softmax - onehot) / n, so
# they differ element by element by at most one bf16 ulp (2^-8 relative). The backward is linear in the LM head's input
# gradient apart from its own bf16 roundings, so the gradients agree to 2^-8 of their norm plus those roundings, which
# differ between two runs with different inputs; 2^-6 covers both.
BOUND = 2.0**-6


@pytest.mark.parametrize("B,S,recompute", [(8, 128, False), (1, 2048, True)], ids=["stored-8x128", "recompute-1x2048"])
def test_gptj6b_logits_gradients(gptj6b_adapters, monkeypatch, B, S, recompute):
    from magma_b200 import language_model

    lm = gptj6b_adapters
    monkeypatch.setattr(language_model, "_use_recompute", lambda *a: recompute)
    lm._ws.clear()
    V = lm.config.vocab_size
    g = torch.Generator(device="cuda").manual_seed(1)
    x = (0.5 * torch.randn(B, S, lm.config.hidden_size, generator=g, device="cuda")).to(torch.bfloat16)
    labels = torch.randint(0, V, (B, S), generator=g, device="cuda")
    labels[:, :2] = -100
    C = 1e-3 * torch.randn(B, S, V, generator=g, device="cuda")
    params = [p for _, p in lm.adapter_parameters() if p.requires_grad]

    def grads(loss_of, with_labels=True):
        for p in params:
            p.grad = None
        xr = x.clone().requires_grad_(True)
        out = lm(inputs_embeds=xr, labels=labels if with_labels else None)
        assert out.logits.grad_fn is not None and (out.loss is None) != with_labels
        loss_of(out).backward()
        assert lm._workspace_ex(B, S)[1] is recompute
        return [xr.grad.clone()] + [p.grad.clone() for p in params]

    def ce(o):
        return F.cross_entropy(o.logits[:, :-1].float().reshape(-1, V), labels[:, 1:].reshape(-1), ignore_index=-100)

    def lin(o):
        return (C * o.logits.float()).sum()

    own = grads(lambda o: o.loss)
    torch_ce = grads(ce, with_labels=False)
    bad = [i for i, (a, b) in enumerate(zip(torch_ce, own)) if rel_dev(a, b) > BOUND]
    assert not bad, [(i, rel_dev(torch_ce[i], own[i])) for i in bad]
    lam = 0.5
    both = grads(lambda o: o.loss + lam * lin(o))
    aux = grads(lin, with_labels=False)
    assert rel_dev(both[0], own[0]) > 0.05  # the auxiliary term matters
    bad = [i for i, (a, b, c) in enumerate(zip(both, own, aux)) if rel_dev(a, b + lam * c) > BOUND]
    assert not bad, [(i, rel_dev(both[i], own[i] + lam * aux[i])) for i in bad]
    # a loss on out.loss alone: the plain backward, bit for bit on a rerun of the same forward
    assert all(torch.equal(a, b) for a, b in zip(grads(lambda o: o.loss)[:1], own[:1]))
    lm._ws.clear()
