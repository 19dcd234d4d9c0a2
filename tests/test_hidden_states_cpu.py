"""output_hidden_states of the GPT-J runtime (csrc/gptj_sched.cu) on its CPU build, held to the oracle's autograd.

The LM returns n_layer + 1 hidden states as GPTNeoModel.forward does: the input embeddings, the outputs of blocks
1 .. n_layer-1 and ln_f of the last block's output. In training they come out of the workspace the backward already
holds, and a loss that reads them sends its gradients back through the same backward pass (stored and recompute). The
inference pass writes them straight from the blocks, over a full sequence or a KV-cache prefill and its decode steps."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from oracle import magma_oracle as O
from test_gptj_recompute_cpu import ENTRY, aligned_ws, case
from test_sched_emul_cpu import FORMS, c_lm_model, ptr, rel

BWD_HIDDEN = {False: "mb200_gptj_sched_backward_range_hidden", True: "mb200_gptj_sched_backward_range_hidden_recompute"}
COPY_HIDDEN = {False: "mb200_gptj_sched_hidden_states", True: "mb200_gptj_sched_hidden_states_recompute"}


@pytest.fixture(scope="module")
def emul():
    from magma_b200 import _lib
    from oracle import build_emul

    return _lib.configure(ctypes.CDLL(build_emul.build()))


def ptrs(ts):
    return (ctypes.c_void_p * len(ts))(*[None if t is None else t.data_ptr() for t in ts])


def run_train(L, cfg, w16, x, labels, recompute, dh, act=0, chunks=None):
    """Training forward, the hidden-state copy-out, then the backward with the hidden-state gradients dh (a list of
    n_layer + 1 tensors or None; dh=None runs the plain backward_range). Returns outputs and gradients."""
    keep = []
    m, grads = c_lm_model(cfg, w16, keep)
    m.adapter_act = act
    B, S = labels.shape
    nbytes, fwd, bwd = (getattr(L, f) for f in ENTRY[recompute])
    n = nbytes(ctypes.byref(m), B, S)
    ws, wsp = aligned_ws(n)
    ldv = (cfg.vocab + 63) // 64 * 64
    logits = torch.zeros(B * S, ldv, dtype=torch.bfloat16)
    loss = torch.zeros(1, dtype=torch.float32)
    assert fwd(ctypes.byref(m), ptr(x), ptr(labels), ptr(logits), ldv, ptr(loss), B, S, wsp, n, None) == 0, \
        L.mb200_last_error()
    hidden = [torch.full_like(x, float("nan")) for _ in range(cfg.n_layer + 1)]
    assert getattr(L, COPY_HIDDEN[recompute])(ctypes.byref(m), ptrs(hidden), B, S, wsp, n, None) == 0, L.mb200_last_error()
    dx = torch.full_like(x, float("nan"))
    for hi, lo in chunks or [(cfg.n_layer, 0)]:
        dxp = ptr(dx) if lo == 0 else None
        if dh is None:
            rc = bwd(ctypes.byref(m), dxp, 1.0, hi, lo, 0, B, S, wsp, n, None)
        else:
            rc = getattr(L, BWD_HIDDEN[recompute])(ctypes.byref(m), dxp, ptrs(dh), 1.0, hi, lo, 0, B, S, wsp, n, None)
        assert rc == 0, L.mb200_last_error()
    return {"loss": loss, "logits": logits, "dx": dx, **{f"h{l}": h for l, h in enumerate(hidden)},
            **{k: g.clone() for k, g in grads.items()}}


def aux_weights(cfg, x, which, seed=4):
    """Fixed random c_l of loss = CE + sum_l <c_l, h_l> for the states in `which` (None elsewhere). At this size the
    auxiliary term's gradients are several times the CE term's, so an auxiliary gradient added in the wrong place or
    twice is far outside the tolerance, while the CE term still shows."""
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(x.shape, generator=g) * 1e-2).to(torch.bfloat16) if l in which else None
            for l in range(cfg.n_layer + 1)]


def oracle_lm(x, w, cfg, labels=None):
    """GPTJForCausalLM.forward with output_hidden_states=True, composed from the oracle's block, LayerNorm and loss
    (oracle/magma_oracle.py::gptj_lm without a cache): (loss, logits, states). The states are those of GPTNeoModel: the
    input embeddings, the outputs of blocks 1 .. n_layer-1 and ln_f of the last block's output."""
    positions = torch.arange(x.shape[1])
    states = [x]
    for l in range(cfg.n_layer):
        states.append(O.gptj_block(states[-1], w, l, cfg, positions)[0])
    states[-1] = O.layer_norm(states[-1], w["lm.transformer.ln_f.weight"], w["lm.transformer.ln_f.bias"], cfg.ln_eps)
    logits = F.linear(states[-1], w["lm.lm_head.weight"], w["lm.lm_head.bias"])
    loss = O.cross_entropy_shifted(logits, labels) if labels is not None else None
    return loss, logits, tuple(states)


def oracle(cfg, w16, x, labels, c, act=0):
    cfg.adapter_act = ("relu", "gelu")[act]
    params = {k: v.float().requires_grad_(".adapter" in k) for k, v in w16.items()}
    xf = x.float().requires_grad_(True)
    loss, logits, states = oracle_lm(xf, params, cfg, labels=labels)
    total = loss + sum((ci.float() * h).sum() for ci, h in zip(c, states) if ci is not None)
    total.backward()
    return loss.detach(), logits.detach(), [h.detach() for h in states], xf.grad, params


def check_against_oracle(got, cfg, w16, x, labels, c, act=0):
    loss_o, logits_o, states_o, dx_o, params = oracle(cfg, w16, x, labels, c, act)
    assert abs(float(got["loss"]) - float(loss_o)) < 2e-2
    assert rel(got["logits"][:, : cfg.vocab].reshape(logits_o.shape), logits_o) < 3e-2
    assert len(states_o) == cfg.n_layer + 1
    bad = {l: round(rel(got[f"h{l}"], h), 4) for l, h in enumerate(states_o) if rel(got[f"h{l}"], h) > 2e-2}
    assert not bad, bad
    assert rel(got["dx"], dx_o) < 2.5e-2
    grads = {k: v for k, v in got.items() if k in params}
    assert set(grads) == {k for k, v in params.items() if v.requires_grad}
    bad = {k: round(rel(g, params[k].grad), 4) for k, g in grads.items() if rel(g, params[k].grad) > 2.5e-2}
    assert not bad, bad


@pytest.mark.parametrize("recompute", [False, True], ids=["stored", "recompute"])
@pytest.mark.parametrize("act", [0, 1], ids=["relu", "gelu"])
@pytest.mark.parametrize("mlp,attn,mlp_ln,attn_ln", FORMS)
def test_training_states_and_aux_loss_gradients_match_oracle(emul, recompute, act, mlp, attn, mlp_ln, attn_ln):
    """Every adapter form and activation, both activation paths: the n_layer + 1 states, and every trainable gradient
    and dx of CE + sum_l <c_l, h_l> over all states."""
    cfg, w16, x, labels = case("gemm", mlp, attn, mlp_ln, attn_ln)
    c = aux_weights(cfg, x, range(cfg.n_layer + 1))
    got = run_train(emul, cfg, w16, x, labels, recompute, c, act=act)
    check_against_oracle(got, cfg, w16, x, labels, c, act)


@pytest.mark.parametrize("recompute", [False, True], ids=["stored", "recompute"])
@pytest.mark.parametrize("which", [[0], [1], [2]], ids=["entry0", "block1", "ln_f"])
def test_one_state_gradient_matches_oracle(emul, recompute, which):
    """A gradient on one state only: entry 0 (it reaches dx alone), a block output, the ln_f entry."""
    cfg, w16, x, labels = case("gemm", "scaled_parallel", "normal", True, True)
    c = aux_weights(cfg, x, which, seed=6)
    got = run_train(emul, cfg, w16, x, labels, recompute, c)
    check_against_oracle(got, cfg, w16, x, labels, c)


@pytest.mark.parametrize("path", ["gemm", "tile", "flash"])
def test_hidden_gradients_in_layer_ranges_and_none(emul, path):
    """The backward in layer ranges [2,1) then [1,0) adds each state's gradient once (equal to one range, stored and
    recompute alike); every pointer NULL equals the plain backward; the states are the same on both paths."""
    cfg, w16, x, labels = case(path, "normal", "parallel", True, False, seed=2)
    c = aux_weights(cfg, x, range(cfg.n_layer + 1))
    one = run_train(emul, cfg, w16, x, labels, False, c)
    for recompute in (False, True):
        chunked = run_train(emul, cfg, w16, x, labels, recompute, c, chunks=[(2, 1), (1, 0)])
        diff = [k for k in one if not torch.equal(chunked[k], one[k])]
        assert not diff, (recompute, diff)
        plain = run_train(emul, cfg, w16, x, labels, recompute, None)
        none = run_train(emul, cfg, w16, x, labels, recompute, [None] * (cfg.n_layer + 1))
        diff = [k for k in plain if not torch.equal(none[k], plain[k])]
        assert not diff, (recompute, diff)


# ---- inference: full sequence, KV-cache prefill + decode -------------------------------------------------------
def run_infer(L, cfg, w16, x, hidden=True, last_only=0, cache=None, pos0=0, S_max=0):
    keep = []
    m, _ = c_lm_model(cfg, w16, keep, with_grads=False)
    B, S, d = x.shape
    n = L.mb200_gptj_sched_infer_workspace_bytes(ctypes.byref(m), B, S, S_max if cache else S)
    ws, wsp = aligned_ws(n)
    ldv = (cfg.vocab + 63) // 64 * 64
    logits = torch.zeros(B if last_only else B * S, ldv, dtype=torch.bfloat16)
    kc, vc = (ptr(cache[0]), ptr(cache[1])) if cache else (None, None)
    if hidden:
        states = torch.full((cfg.n_layer + 1, B, S, d), float("nan"), dtype=torch.bfloat16)
        rc = L.mb200_gptj_sched_infer_hidden(ctypes.byref(m), ptr(x), ptr(logits), ldv, last_only, ptr(states),
                                             states.stride(0), kc, vc, S_max, pos0, B, S, wsp, n, None)
    else:
        states = torch.full((B if last_only else B * S, d), float("nan"), dtype=torch.bfloat16)  # the ln_f output
        rc = L.mb200_gptj_sched_infer(ctypes.byref(m), ptr(x), ptr(logits), ldv, last_only, ptr(states), kc, vc, S_max,
                                      pos0, B, S, wsp, n, None)
    assert rc == 0, L.mb200_last_error()
    return logits, states


@pytest.mark.parametrize("path", ["gemm", "tile"])
def test_inference_states_match_oracle_and_the_ln_f_output(emul, path):
    cfg, w16, x, _ = case(path, "normal", "scaled_parallel", False, True, seed=3)
    logits, states = run_infer(emul, cfg, w16, x)
    params = {k: v.float() for k, v in w16.items()}
    _, logits_o, states_o = oracle_lm(x.float(), params, cfg)
    assert torch.equal(logits_o, O.gptj_lm(x.float(), params, cfg)[1])  # the composition is the oracle's LM
    bad = {l: round(rel(states[l], h), 4) for l, h in enumerate(states_o) if rel(states[l], h) > 2e-2}
    assert not bad, bad
    assert torch.equal(states[0], x)
    # logits and the ln_f entry bit for bit as the pass without hidden states computes them
    logits_ref, lnf = run_infer(emul, cfg, w16, x, hidden=False)
    assert torch.equal(logits, logits_ref) and torch.equal(states[-1].reshape(lnf.shape), lnf)
    # last-position logits: the ln_f entry still covers every row
    last, states_last = run_infer(emul, cfg, w16, x, last_only=1)
    last_ref, _ = run_infer(emul, cfg, w16, x, hidden=False, last_only=1)
    assert torch.equal(last, last_ref) and torch.equal(states_last, states)


def test_prefill_then_decode_states_match_the_full_sequence(emul):
    """With a KV cache the states are those of the S new positions: a 7-token prefill and three decode steps give the
    matching slices of one 10-token call."""
    cfg, w16, x, _ = case("gemm", "normal", None, False, False, seed=5, B=2)
    x = x[:, :10].contiguous()
    B, S, d = x.shape
    H, hd, S_max = cfg.n_head, cfg.d // cfg.n_head, 16
    _, full = run_infer(emul, cfg, w16, x)
    cache = [torch.zeros(cfg.n_layer, B, H, S_max, hd, dtype=torch.bfloat16) for _ in range(2)]
    parts = [run_infer(emul, cfg, w16, x[:, :7].contiguous(), cache=cache, pos0=0, S_max=S_max)[1]]
    for p in range(7, 10):
        parts.append(run_infer(emul, cfg, w16, x[:, p:p + 1].contiguous(), cache=cache, pos0=p, S_max=S_max)[1])
    stepped = torch.cat(parts, dim=2)
    bad = {l: round(rel(stepped[l], full[l]), 4) for l in range(cfg.n_layer + 1) if rel(stepped[l], full[l]) > 1e-2}
    assert not bad, bad


def test_infer_hidden_rejects_a_short_stride(emul):
    cfg, w16, x, _ = case("gemm", None, None, False, False)
    keep = []
    m, _ = c_lm_model(cfg, w16, keep, with_grads=False)
    B, S, d = x.shape
    n = emul.mb200_gptj_sched_infer_workspace_bytes(ctypes.byref(m), B, S, S)
    ws, wsp = aligned_ws(n)
    states = torch.empty(cfg.n_layer + 1, B, S, d, dtype=torch.bfloat16)
    rc = emul.mb200_gptj_sched_infer_hidden(ctypes.byref(m), ptr(x), None, 0, 0, ptr(states), B * S * d - 8, None, None,
                                            0, 0, B, S, wsp, n, None)
    assert rc != 0 and b"ld_hidden" in emul.mb200_last_error()


# ---- the Python surface: B200GPTJForCausalLM.forward and Magma.forward -------------------------------------------
def test_language_model_returns_every_state(emul_ops):
    from test_gptj_recompute_cpu import _tiny_lm

    lm, x, labels = _tiny_lm()
    n = len(lm.transformer.h)
    inf = lm(inputs_embeds=x, output_hidden_states=True)
    assert len(inf.hidden_states) == n + 1 and all(h.shape == x.shape for h in inf.hidden_states)
    assert torch.equal(inf.hidden_states[0], x)
    assert torch.equal(inf.logits, lm(inputs_embeds=x).logits)
    with torch.no_grad():  # a loss without backward: the training pass, states copied out of its workspace
        tr = lm(inputs_embeds=x, labels=labels, output_hidden_states=True)
    assert len(tr.hidden_states) == n + 1
    assert all(torch.equal(a, b) for a, b in zip(tr.hidden_states, inf.hidden_states))


def test_magma_forward_trains_through_hidden_states(emul_ops, monkeypatch):
    """Magma.forward(output_hidden_states=True) on the training path: CE + sum_l <c_l, h_l> gives the oracle's adapter
    gradients and prefix gradient; leaving the states out of the loss gives the gradients of a run without
    output_hidden_states, bit for bit."""
    from test_e2e_dryrun_cpu import build, oracle_weights, tiny_cfg

    cfg = tiny_cfg(mlp_adapter={"adapter_type": "normal", "downsample_factor": 4})
    S, B = 16, 2
    w = oracle_weights(cfg)
    model, _ = build(monkeypatch, cfg, w, S, freeze_enc=True)
    model.eval()
    images, captions = O.synthetic_batch(cfg, B, S, seed=11)
    images = images.to(torch.bfloat16).float()
    with torch.no_grad():
        prefix = O.image_prefix(images, w, cfg).to(torch.bfloat16)
    names = [n for n, p in model.named_parameters() if p.requires_grad and n.startswith("lm.")]
    sd = dict(model.named_parameters())

    def run(loss_of, hidden):
        model.arena.grad.zero_()
        for p in model.parameters():
            p.grad = None
        pr = prefix.float().requires_grad_(True)  # dprefix: what _EmbedLMFn routes back to the image prefix
        out = model(None, captions, input_embeddings=pr, output_hidden_states=hidden)
        assert (out.hidden_states is not None) == hidden
        loss_of(out).backward()
        return {"dprefix": pr.grad.clone(), **{n: sd[n].grad.clone() for n in names}}

    plain = run(lambda out: out.loss, False)
    unused = run(lambda out: out.loss, True)
    assert all(torch.equal(unused[k], plain[k]) for k in plain)

    g = torch.Generator().manual_seed(3)
    c = [torch.randn(B, S, cfg.d, generator=g) * 0.02 for _ in range(cfg.n_layer + 1)]
    got = run(lambda out: out.loss + sum((ci * h.float()).sum() for ci, h in zip(c, out.hidden_states)), True)
    params = {k: v.clone().requires_grad_(k in names) for k, v in w.items()}
    pf = prefix.float().requires_grad_(True)
    _, _, labels = O.magma_forward(None, captions, params, cfg, input_embeddings=pf.detach())
    x = torch.cat([pf, params["lm.transformer.wte.weight"][captions[:, : S - cfg.image_seq_len]]], dim=1)
    loss_o, _, states = oracle_lm(x, params, cfg, labels=labels)
    (loss_o + sum((ci * h).sum() for ci, h in zip(c, states))).backward()
    want = {"dprefix": pf.grad, **{k: params[k].grad for k in names}}
    bad = {k: round(rel(got[k], v), 4) for k, v in want.items() if rel(got[k], v) > 5e-2}
    assert not bad, bad
