"""Activation recomputation in the GPT-J training schedule (csrc/gptj_sched.cu), on its CPU build.

The recompute pass keeps each block's input only and reruns the block's forward right before the block's backward. It
issues the same operators in the same order on the same inputs as the stored-activation pass, so loss, logits, dx and
every gradient must equal the stored pass's bit for bit: every comparison here is torch.equal. The cases reuse the
tiny GPT-J builders of test_sched_emul_cpu.py; head_dim 16 takes the batched-GEMM attention, head_dim 64 the fused
single-tile kernels (S <= 128) or the multi-tile forward with the materialised backward (S > 128)."""
import ctypes

import pytest
import torch

from magma_b200._lib import GptjLayerExC, GptjModelExC
from oracle import magma_oracle as O
from test_sched_emul_cpu import FORMS, c_lm_model, lm_case, ptr

ENTRY = {False: ("mb200_gptj_sched_workspace_bytes", "mb200_gptj_sched_forward", "mb200_gptj_sched_backward_range"),
         True: ("mb200_gptj_sched_recompute_workspace_bytes", "mb200_gptj_sched_forward_recompute",
                "mb200_gptj_sched_backward_range_recompute")}
# attention path -> (n_head of the d = 64 model, S)
PATHS = {"gemm": (4, 12), "tile": (1, 40), "flash": (1, 136)}


@pytest.fixture(scope="module")
def emul():
    from oracle import build_emul

    L = ctypes.CDLL(build_emul.build())
    L.mb200_last_error.restype = ctypes.c_char_p
    L.mb200_gptj_sched_workspace_bytes.restype = ctypes.c_size_t
    L.mb200_gptj_sched_recompute_workspace_bytes.restype = ctypes.c_size_t
    return L


def case(path, mlp, attn, mlp_ln, attn_ln, seed=0, B=2):
    n_head, S = PATHS[path]
    orig = O.OracleConfig

    def cfg_with_heads(**kw):
        return orig(**{**kw, "n_head": n_head})

    O.OracleConfig = cfg_with_heads
    try:
        return lm_case(mlp, attn, mlp_ln, attn_ln, seed=seed, B=B, S=S)
    finally:
        O.OracleConfig = orig


def aligned_ws(n):
    ws = torch.empty(n + 256, dtype=torch.uint8)
    return ws, ctypes.c_void_p(ws.data_ptr() + (-ws.data_ptr()) % 256)


def run(L, cfg, w16, x, labels, recompute, act=0, chunks=None, accumulate=(0,)):
    """Forward, then one backward per entry of `accumulate` (each in the layer ranges `chunks`); returns every output
    and every gradient after each backward."""
    keep = []
    m, grads = c_lm_model(cfg, w16, keep)
    m.adapter_act = act
    B, S = labels.shape
    nbytes, fwd, bwd = (getattr(L, f) for f in ENTRY[recompute])
    n = nbytes(ctypes.byref(m), B, S)
    assert n > 0, L.mb200_last_error().decode()
    ws, wsp = aligned_ws(n)
    ldv = (cfg.vocab + 63) // 64 * 64
    logits = torch.zeros(B * S, ldv, dtype=torch.bfloat16)
    loss = torch.zeros(1, dtype=torch.float32)
    rc = fwd(ctypes.byref(m), ptr(x), ptr(labels), ptr(logits), ctypes.c_int64(ldv), ptr(loss), B, S, wsp,
             ctypes.c_size_t(n), None)
    assert rc == 0, L.mb200_last_error().decode()
    out = {"loss": loss, "logits": logits}
    for i, acc in enumerate(accumulate):
        dx = torch.full_like(x, float("nan"))
        for hi, lo in chunks or [(cfg.n_layer, 0)]:
            rc = bwd(ctypes.byref(m), ptr(dx) if lo == 0 else None, ctypes.c_float(0.75), hi, lo, acc, B, S, wsp,
                     ctypes.c_size_t(n), None)
            assert rc == 0, L.mb200_last_error().decode()
        out[f"dx/{i}"] = dx
        out.update({f"{k}/{i}": g.clone() for k, g in grads.items()})
    return out


def assert_identical(got, want):
    assert set(got) == set(want)
    diff = [k for k in want if not torch.equal(got[k], want[k])]
    assert not diff, diff


@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("act", [0, 1], ids=["relu", "gelu"])
@pytest.mark.parametrize("mlp,attn,mlp_ln,attn_ln", FORMS)
def test_recompute_is_bit_identical_to_stored(emul, path, act, mlp, attn, mlp_ln, attn_ln):
    """Every adapter form, both adapter activations, every attention path; the second backward accumulates onto the
    first's gradients."""
    cfg, w16, x, labels = case(path, mlp, attn, mlp_ln, attn_ln)
    stored = run(emul, cfg, w16, x, labels, False, act, accumulate=(0, 1))
    recomputed = run(emul, cfg, w16, x, labels, True, act, accumulate=(0, 1))
    assert torch.isfinite(stored["loss"]).all() and not torch.isnan(stored["dx/0"].float()).any()
    if mlp is not None:
        assert len(stored) > 4  # adapter gradients are part of the comparison
    assert_identical(recomputed, stored)


@pytest.mark.parametrize("path", ["tile", "flash"])
def test_chunked_and_repeated_recompute_backward(emul, path):
    """The backward in layer ranges [2,1) then [1,0) (how B200Engine overlaps the gradient exchange) equals one range,
    and running the backward twice leaves the same result: the recomputed layers never overwrite a saved block input."""
    cfg, w16, x, labels = case(path, "scaled_parallel", "normal", True, True, seed=3)
    one = run(emul, cfg, w16, x, labels, True, accumulate=(0, 0))
    chunked = run(emul, cfg, w16, x, labels, True, chunks=[(2, 1), (1, 0)], accumulate=(0, 0))
    assert_identical(chunked, one)
    again = {k[:-2]: v for k, v in one.items() if k.endswith("/1")}
    assert_identical(again, {k[:-2]: v for k, v in one.items() if k.endswith("/0")})
    assert_identical(one, run(emul, cfg, w16, x, labels, False, accumulate=(0, 0)))


def full_size_model(keep):
    """GPT-J-6B with MLP adapters (MAGMA_v1.yml) for workspace arithmetic: no tensor is touched, so the pointers are
    placeholders."""
    layers = (GptjLayerExC * 28)()
    m = GptjModelExC()
    m.n_layer, m.d, m.n_head, m.rotary_dim, m.vocab, m.d_ff = 28, 4096, 16, 64, 50258, 16384
    m.mlp_adapter, m.mlp_adapter_r, m.ln_eps = 1, 1024, 1e-5
    m.layers = ctypes.cast(layers, ctypes.POINTER(GptjLayerExC))
    keep.append(layers)
    return m


@pytest.mark.parametrize("B,S", [(1, 1), (8, 128), (1, 2048), (4, 2048), (8, 2048)])
def test_full_size_recompute_workspace_is_smaller(emul, B, S):
    keep = []
    m = full_size_model(keep)
    stored = emul.mb200_gptj_sched_workspace_bytes(ctypes.byref(m), B, S)
    recompute = emul.mb200_gptj_sched_recompute_workspace_bytes(ctypes.byref(m), B, S)
    assert 0 < recompute < stored
    if (B, S) == (8, 2048):
        assert stored > 78 * 2**30 and recompute < 16 * 2**30


def test_recompute_rejects_a_small_workspace(emul):
    cfg, w16, x, labels = case("gemm", "normal", None, False, False)
    keep = []
    m, _ = c_lm_model(cfg, w16, keep)
    B, S = labels.shape
    n = emul.mb200_gptj_sched_recompute_workspace_bytes(ctypes.byref(m), B, S)
    assert 0 < n < emul.mb200_gptj_sched_workspace_bytes(ctypes.byref(m), B, S)
    ws, wsp = aligned_ws(n)
    loss = torch.zeros(1)
    rc = emul.mb200_gptj_sched_forward_recompute(ctypes.byref(m), ptr(x), ptr(labels), None, ctypes.c_int64(0),
                                                 ptr(loss), B, S, wsp, ctypes.c_size_t(n - 1), None)
    assert rc != 0 and b"workspace too small" in emul.mb200_last_error()
    rc = emul.mb200_gptj_sched_backward_range_recompute(ctypes.byref(m), None, ctypes.c_float(1.0), 2, 0, 0, B, S, wsp,
                                                        ctypes.c_size_t(n - 1), None)
    assert rc != 0 and b"workspace too small" in emul.mb200_last_error()


def test_selection_picks_stored_when_it_fits():
    from magma_b200.language_model import _use_recompute

    GiB = 2**30
    assert not _use_recompute(10 * GiB, 1 * GiB, 11 * GiB)
    assert _use_recompute(10 * GiB, 1 * GiB, 11 * GiB - 1)
    # GPT-J-6B on an 80 GB card with about 66 GiB left after the weights: bench config 2 (B = 8, S = 128) stays on the
    # stored path, B = 8 at S = 2048 recomputes
    logits_dx = lambda B, S: B * S * (50304 + 4096) * 2  # noqa: E731
    assert not _use_recompute(3.21 * GiB, logits_dx(8, 128), 66 * GiB)
    assert _use_recompute(78.57 * GiB, logits_dx(8, 2048), 66 * GiB)


def _tiny_lm():
    from magma_b200.language_model import GPTJConfig, get_gptj

    cfg = GPTJConfig(vocab_size=96, hidden_size=64, num_layers=2, num_heads=4, rotary_dim=8)
    lm = get_gptj(config=cfg, device="cpu").init_weights(seed=1, std=0.2)
    g = torch.Generator().manual_seed(2)
    x = (torch.randn(2, 12, 64, generator=g) * 0.5).to(torch.bfloat16)
    labels = torch.randint(0, 96, (2, 12), generator=g)
    return lm, x, labels


def _loss_and_dx(lm, x, labels):
    xr = x.clone().requires_grad_(True)
    out = lm(inputs_embeds=xr, labels=labels)
    out.loss.backward()
    return out.loss.detach(), out.logits, xr.grad


def test_language_model_follows_the_selection_and_checks_the_mode(emul_ops, monkeypatch):
    """B200GPTJForCausalLM runs the path _use_recompute picks (same results bit for bit), keeps it with the workspace,
    and refuses a backward whose workspace belongs to the other path than its forward's."""
    from magma_b200 import _lib, language_model

    emul_ops.mb200_gptj_sched_recompute_workspace_bytes.restype = ctypes.c_size_t
    lm, x, labels = _tiny_lm()
    assert lm._workspace_ex(2, 12)[1] is False  # the emulation has no device memory to run out of
    stored = _loss_and_dx(lm, x, labels)
    lm._ws.clear()
    monkeypatch.setattr(language_model, "_use_recompute", lambda *a: True)
    recomputed = _loss_and_dx(lm, x, labels)
    assert lm._workspace_ex(2, 12)[1] is True
    assert all(torch.equal(a, b) for a, b in zip(recomputed, stored))
    monkeypatch.setattr(language_model, "_use_recompute", lambda *a: False)
    assert lm._workspace_ex(2, 12)[1] is True  # decided once per workspace
    # a forward on the recompute workspace, then a backward on a stored one
    xr = x.clone().requires_grad_(True)
    out = lm(inputs_embeds=xr, labels=labels)
    lm._ws.clear()
    with pytest.raises(_lib.MB200Error, match="other activation path"):
        out.loss.backward()
