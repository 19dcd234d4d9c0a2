"""Gradients through the training logits of the GPT-J runtime (csrc/gptj_sched.cu) on its CPU build, held to the
oracle's autograd.

A loss on the logits sends its gradient G into the same backward pass as the cross-entropy term: the LM head's dgrad
reads loss_scale * dCE + G (mb200_logits_grad_combine into a caller buffer), so the workspace's cross-entropy gradient
stays as the forward wrote it. A forward without labels never writes it, and its backward never reads it. The schedule's
CPU build links tests/logits_grad_emul.cpp and tests/attention_emul.cpp next to oracle/cabi_emul.cpp."""
import ctypes
import os
import subprocess

import pytest
import torch
import torch.nn.functional as F

from oracle import magma_oracle as O
from test_attentions_cpu import attn_weights, oracle_attn_lm
from test_gptj_recompute_cpu import ENTRY, aligned_ws, case
from test_hidden_states_cpu import aux_weights, oracle_lm, ptrs
from test_sched_emul_cpu import FORMS, c_lm_model, ptr, rel

BWD_LOGITS = {False: "mb200_gptj_sched_backward_range_logits", True: "mb200_gptj_sched_backward_range_logits_recompute"}
HERE = os.path.dirname(os.path.abspath(__file__))
EXT_SRC = [os.path.join(HERE, "attention_emul.cpp"), os.path.join(HERE, "logits_grad_emul.cpp")]


def build_logits_emul():
    """oracle/_build/libsched_emul_logits.so: the objects of oracle/build_emul.py's schedule emulation plus the two
    emulations above."""
    from oracle import build_emul

    build_emul.build()
    out = os.path.join(build_emul.OUT_DIR, "libsched_emul_logits.so")
    objs = [os.path.join(build_emul.OUT_DIR, os.path.basename(f).rsplit(".", 1)[0] + ".o")
            for f in build_emul.SCHEDULES + [build_emul.EMUL]]
    deps = objs + EXT_SRC + [os.path.join(build_emul.ROOT, "include", "magma_b200.h")]
    if os.path.exists(out) and os.path.getmtime(out) >= max(os.path.getmtime(d) for d in deps):
        return out
    ext = [os.path.join(build_emul.OUT_DIR, os.path.basename(s).rsplit(".", 1)[0] + "_lg.o") for s in EXT_SRC]
    for src, o in zip(EXT_SRC, ext):
        r = subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-Wall", "-c", src, "-o", o], capture_output=True,
                           text=True)
        assert r.returncode == 0, r.stdout + r.stderr
    r = subprocess.run(["g++", "-shared", "-o", out, *objs, *ext], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return out


@pytest.fixture(scope="module")
def emul():
    from magma_b200 import _lib

    return _lib.configure(ctypes.CDLL(build_logits_emul()))


@pytest.fixture
def emul_logits_ops(monkeypatch):
    """The conftest's emul_ops with the library that also emulates mb200_logits_grad_combine."""
    from magma_b200 import _lib, ops

    L = _lib.configure(ctypes.CDLL(build_logits_emul()))
    monkeypatch.setattr(_lib, "_lib", L)
    monkeypatch.setattr(ops, "_stream", lambda: None)
    return L


# ---- the losses on the logits ----------------------------------------------------------------------------------------
def loss_fn(kind, V, B, S, seed=11):
    """(f(logits [B, S, V] float) -> scalar, reads_ce): the auxiliary loss and whether the total adds the CE loss.
    ce_lin: CE + <C, logits>; kl: KL(teacher || softmax(logits)) per row, summed; zlin: 0.2 <C, logits> + 0.1 z-loss
    (no labels)."""
    g = torch.Generator().manual_seed(seed)
    C = torch.randn(B, S, V, generator=g) * 0.05
    teacher = torch.softmax(torch.randn(B, S, V, generator=g) * 2.0, -1)
    if kind == "ce_lin":
        return (lambda z: (C * z).sum()), True
    if kind == "kl":
        return (lambda z: (teacher * (teacher.log() - torch.log_softmax(z, -1))).sum()), False
    return (lambda z: 0.2 * (C * z).sum() + 0.1 * (torch.logsumexp(z, -1) ** 2).sum()), False


def optr(t):
    return None if t is None else t.data_ptr()


def grad_of(f, logits):
    z = logits.detach().float().cpu().requires_grad_(True)
    f(z).backward()
    return z.grad.to(logits.device)


# ---- the schedule's C ABI ------------------------------------------------------------------------------------------
def run_train(L, cfg, w16, x, labels, recompute, f=None, dh=None, da=None, act=0, chunks=None, ld_g=None, plain=False,
              reads_ce=True):
    """Training forward (labels may be None), then the backward: plain runs the old backward_range entry; otherwise
    backward_range_logits with G = d f / d logits (taken on the runtime's own logits, as autograd would, in a
    NaN-padded buffer of row stride ld_g), hidden-state gradients dh and attention gradients da. reads_ce: whether the
    loss adds the CE loss (loss_scale 1, else 0, as _backward_scale gives for a loss that does not read it)."""
    keep = []
    m, grads = c_lm_model(cfg, w16, keep)
    m.adapter_act = act
    B, S, V = x.shape[0], x.shape[1], cfg.vocab
    nbytes, fwd, bwd = (getattr(L, fn) for fn in ENTRY[recompute])
    n = nbytes(ctypes.byref(m), B, S)
    ws, wsp = aligned_ws(n)
    ws.fill_(255)  # NaN bf16 everywhere the forward does not write: P.dlogits of a forward without labels among them
    ldv = (V + 63) // 64 * 64
    logits = torch.zeros(B * S, ldv, dtype=torch.bfloat16)
    loss = torch.zeros(1, dtype=torch.float32)
    assert fwd(ctypes.byref(m), ptr(x), optr(labels), ptr(logits), ldv, ptr(loss), B, S, wsp, n, None) == 0, \
        L.mb200_last_error()
    G = None
    if f is not None:
        ld_g = ld_g or V
        G = torch.full((B * S, ld_g), float("nan"), dtype=torch.bfloat16)
        G[:, :V] = grad_of(f, logits[:, :V].reshape(B, S, V)).reshape(B * S, V).to(torch.bfloat16)
    comb = torch.full((B * S, ldv), float("nan"), dtype=torch.bfloat16)
    dx = torch.full_like(x, float("nan"))
    scale = 1.0 if labels is not None and reads_ce else 0.0
    for hi, lo in chunks or [(cfg.n_layer, 0)]:
        dxp = ptr(dx) if lo == 0 else None
        if plain:
            rc = bwd(ctypes.byref(m), dxp, scale, hi, lo, 0, B, S, wsp, n, None)
        else:
            rc = getattr(L, BWD_LOGITS[recompute])(ctypes.byref(m), dxp, None if dh is None else ptrs(dh),
                                                   None if da is None else ptrs(da), (S + 7) // 8 * 8, optr(G),
                                                   ld_g or 0, ptr(comb), scale, hi, lo, 0, B, S, wsp, n, None)
        assert rc == 0, L.mb200_last_error()
    return {"loss": loss, "logits": logits, "dx": dx, **{k: g.clone() for k, g in grads.items()}}


def oracle(cfg, w16, x, labels, f, reads_ce, act=0, ch=None, ca=None):
    """dx and trainable gradients of [CE +] f(logits) [+ sum <ch_l, h_l>] [+ sum <ca_l, A_l>] on the oracle."""
    cfg.adapter_act = ("relu", "gelu")[act]
    params = {k: v.float().requires_grad_(".adapter" in k) for k, v in w16.items()}
    xf = x.float().requires_grad_(True)
    S = x.shape[1]
    loss, logits, states = oracle_lm(xf, params, cfg, labels=labels if reads_ce else None)
    total = f(logits) if f is not None else 0.0
    if reads_ce:
        total = total + loss
    if ch is not None:
        total = total + sum((c.float() * h).sum() for c, h in zip(ch, states) if c is not None)
    if ca is not None:
        attn = oracle_attn_lm(xf, params, cfg)[2]
        total = total + sum((c[..., :S].float() * a).sum() for c, a in zip(ca, attn) if c is not None)
    total.backward()
    return logits.detach(), xf.grad, params


def check(got, cfg, w16, x, labels, f, reads_ce, act=0, ch=None, ca=None, tol=3e-2):
    logits_o, dx_o, params = oracle(cfg, w16, x, labels, f, reads_ce, act, ch, ca)
    assert rel(got["logits"][:, : cfg.vocab].reshape(logits_o.shape), logits_o) < 3e-2
    assert rel(got["dx"], dx_o) < tol, rel(got["dx"], dx_o)
    grads = {k: v for k, v in got.items() if k in params}
    assert set(grads) == {k for k, v in params.items() if v.requires_grad}
    # adapter_scale's gradient is one bf16 dot product over every row: twice the bar
    bad = {k: round(rel(g, params[k].grad), 4) for k, g in grads.items()
           if rel(g, params[k].grad) > (2 * tol if g.numel() == 1 else tol)}
    assert not bad, bad


LOSSES = ["ce_lin", "kl", "zlin_no_labels"]


@pytest.mark.parametrize("kind", LOSSES)
@pytest.mark.parametrize("recompute", [False, True], ids=["stored", "recompute"])
@pytest.mark.parametrize("act", [0, 1], ids=["relu", "gelu"])
@pytest.mark.parametrize("mlp,attn,mlp_ln,attn_ln", FORMS)
def test_logits_loss_gradients_match_oracle(emul, kind, recompute, act, mlp, attn, mlp_ln, attn_ln):
    """Every adapter form and activation, both activation paths, each loss: every trainable gradient and dx. G sits in
    rows of odd stride V + 1 (2-byte aligned rows, NaN in the padding)."""
    cfg, w16, x, labels = case("gemm", mlp, attn, mlp_ln, attn_ln)
    B, S = labels.shape
    f, reads_ce = loss_fn(kind, cfg.vocab, B, S)
    lab = labels if kind != "zlin_no_labels" else None
    got = run_train(emul, cfg, w16, x, lab, recompute, f=f, act=act, ld_g=cfg.vocab + 1, reads_ce=reads_ce)
    check(got, cfg, w16, x, labels, f, reads_ce, act)


@pytest.mark.parametrize("kind", LOSSES)
@pytest.mark.parametrize("path", ["gemm", "tile"])
def test_with_hidden_and_attention_gradients_in_layer_ranges(emul, kind, path):
    """Logits, hidden-state and attention gradients in one pass; layer ranges [2,1) then [1,0) give the one-range
    result bit for bit on both paths, and stored and recompute agree."""
    cfg, w16, x, labels = case(path, "normal", "parallel", True, False, seed=2)
    B, S = labels.shape
    f, reads_ce = loss_fn(kind, cfg.vocab, B, S, seed=5)
    lab = labels if kind != "zlin_no_labels" else None
    ch = aux_weights(cfg, x, range(cfg.n_layer + 1))
    ca = attn_weights(cfg, B, S, range(cfg.n_layer), scale=4.0)
    one = run_train(emul, cfg, w16, x, lab, False, f=f, dh=ch, da=ca, reads_ce=reads_ce)
    check(one, cfg, w16, x, labels, f, reads_ce, ch=ch, ca=ca, tol=5e-2)
    for recompute in (False, True):
        chunked = run_train(emul, cfg, w16, x, lab, recompute, f=f, dh=ch, da=ca, chunks=[(2, 1), (1, 0)],
                            reads_ce=reads_ce)
        diff = [k for k in one if not torch.equal(chunked[k], one[k])]
        assert not diff, (recompute, diff)


@pytest.mark.parametrize("recompute", [False, True], ids=["stored", "recompute"])
def test_all_none_gradients_and_the_plain_backward(emul, recompute):
    """With labels and no logits gradient the new entry equals the plain backward bit for bit; without labels, hidden-
    state gradients alone match the oracle (the NaN left in the workspace's CE gradient is never read) and all-None
    gradients give dx = 0; G = 0 with labels gives the plain backward's gradients."""
    cfg, w16, x, labels = case("gemm", "normal", "normal", False, False, seed=3)
    plain = run_train(emul, cfg, w16, x, labels, recompute, plain=True)
    nones = run_train(emul, cfg, w16, x, labels, recompute, dh=[None] * (cfg.n_layer + 1), da=[None] * cfg.n_layer)
    assert not [k for k in plain if not torch.equal(nones[k], plain[k])]
    zero = run_train(emul, cfg, w16, x, labels, recompute, f=lambda z: 0.0 * z.sum())
    assert not [k for k in plain if k != "logits" and rel(zero[k], plain[k]) > 1e-2]
    ch = aux_weights(cfg, x, range(cfg.n_layer + 1))
    got = run_train(emul, cfg, w16, x, None, recompute, dh=ch)
    check(got, cfg, w16, x, labels, None, False, ch=ch)
    empty = run_train(emul, cfg, w16, x, None, recompute)
    assert torch.equal(empty["dx"], torch.zeros_like(x))


def test_second_backward_gives_the_same_result(emul):
    """The combined gradient goes to the caller's buffer: a second backward over the same forward, with or without G,
    reads the CE gradient the forward wrote."""
    cfg, w16, x, labels = case("gemm", "normal", None, False, False, seed=4)
    B, S = labels.shape
    f, _ = loss_fn("ce_lin", cfg.vocab, B, S)
    keep = []
    m, grads = c_lm_model(cfg, w16, keep)
    n = emul.mb200_gptj_sched_workspace_bytes(ctypes.byref(m), B, S)
    ws, wsp = aligned_ws(n)
    ldv = (cfg.vocab + 63) // 64 * 64
    logits = torch.zeros(B * S, ldv, dtype=torch.bfloat16)
    loss = torch.zeros(1)
    assert emul.mb200_gptj_sched_forward(ctypes.byref(m), ptr(x), ptr(labels), ptr(logits), ldv, ptr(loss), B, S, wsp, n,
                                         None) == 0
    G = grad_of(f, logits[:, : cfg.vocab].reshape(B, S, -1)).reshape(B * S, -1).to(torch.bfloat16)
    comb = torch.empty(B * S, ldv, dtype=torch.bfloat16)
    outs = []
    for g in (G, None, G):
        dx = torch.empty_like(x)
        assert emul.mb200_gptj_sched_backward_range_logits(ctypes.byref(m), ptr(dx), None, None, 0, optr(g), cfg.vocab,
                                                           ptr(comb), 1.0, cfg.n_layer, 0, 0, B, S, wsp, n, None) == 0
        outs.append(dx)
    assert torch.equal(outs[0], outs[2]) and not torch.equal(outs[0], outs[1])


def test_rejects_a_short_ld_dlogits_and_a_missing_buffer(emul):
    cfg, w16, x, labels = case("gemm", None, None, False, False)
    keep = []
    m, _ = c_lm_model(cfg, w16, keep)
    B, S = labels.shape
    n = emul.mb200_gptj_sched_workspace_bytes(ctypes.byref(m), B, S)
    ws, wsp = aligned_ws(n)
    G = torch.zeros(B * S, cfg.vocab, dtype=torch.bfloat16)
    comb = torch.empty(B * S, (cfg.vocab + 63) // 64 * 64, dtype=torch.bfloat16)
    for ld, c in ((cfg.vocab - 1, comb), (cfg.vocab, None)):
        rc = emul.mb200_gptj_sched_backward_range_logits(ctypes.byref(m), None, None, None, 0, optr(G), ld, optr(c), 1.0,
                                                         cfg.n_layer, 0, 0, B, S, wsp, n, None)
        assert rc != 0 and b"ld_dlogits" in emul.mb200_last_error()


# ---- the Python surface ----------------------------------------------------------------------------------------------
def test_language_model_logits_are_differentiable(emul_logits_ops):
    """B200GPTJForCausalLM.forward: under grad the logits have a grad_fn, with or without labels; CE + <C, logits>
    through out.loss and out.logits gives the oracle's dx; a loss on out.loss alone gives the gradients of the plain
    backward bit for bit; F.cross_entropy on the logits of a pass without labels gives out.loss's dx."""
    from test_gptj_recompute_cpu import _tiny_lm

    lm, x, labels = _tiny_lm()
    B, S, _ = x.shape
    V = lm.config.vocab_size
    C = torch.randn(B, S, V, generator=torch.Generator().manual_seed(3)) * 0.05

    def run(loss_of, with_labels=True):
        xr = x.float().requires_grad_(True)
        out = lm(inputs_embeds=xr, labels=labels if with_labels else None)
        assert out.logits.grad_fn is not None
        loss_of(out).backward()
        return out, xr.grad

    _, dx_plain = run(lambda o: o.loss)
    _, dx = run(lambda o: o.loss + (C * o.logits.float()).sum())
    w = {"lm." + n: p.detach().float() for n, p in lm.named_parameters()}
    cfg = O.OracleConfig(d=64, n_layer=2, n_head=4, rotary_dim=8, vocab=V, mlp_adapter=None)
    xf = x.float().requires_grad_(True)
    loss, logits, _ = oracle_lm(xf, w, cfg, labels=labels)
    (loss + (C * logits).sum()).backward()
    assert rel(dx, xf.grad) < 3e-2 and rel(dx, dx_plain) > 0.1
    out, dx_ce = run(lambda o: F.cross_entropy(o.logits[:, :-1].float().reshape(-1, V), labels[:, 1:].reshape(-1)),
                     with_labels=False)
    assert out.loss is None and rel(dx_ce, dx_plain) < 1e-2


def test_logits_gradient_layouts_and_the_engine_hint(emul_logits_ops):
    """G in layouts other than contiguous [B, S, V] rows: S == 1 (torch does not define the stride of a size-1 dim) and
    the stride-0 broadcast logits.sum() sends back; both give the oracle's dx. B200Engine's loss-scale hint does not
    add a CE term to a loss that does not read out.loss."""
    from test_gptj_recompute_cpu import _tiny_lm

    lm, x, labels = _tiny_lm()
    V = lm.config.vocab_size
    w = {"lm." + n: p.detach().float() for n, p in lm.named_parameters()}
    cfg = O.OracleConfig(d=64, n_layer=2, n_head=4, rotary_dim=8, vocab=V, mlp_adapter=None)
    C = torch.randn(2, 12, V, generator=torch.Generator().manual_seed(4)) * 0.05
    cases = [(x[:, :1], lambda z: (C[:, :1] * z).sum()), (x, lambda z: z.sum()), (x[:1, :1], lambda z: z.sum()),
             (x[:, :5], lambda z: (C[:, :5] * z).transpose(0, 1).sum())]
    for xs, f in cases:
        xr = xs.float().requires_grad_(True)
        f(lm(inputs_embeds=xr).logits.float()).backward()
        xf = xs.float().requires_grad_(True)
        f(oracle_lm(xf, w, cfg)[1]).backward()
        assert rel(xr.grad, xf.grad) < 3e-2, (xs.shape, rel(xr.grad, xf.grad))

    def dx_of_logits_loss(hint):
        lm._loss_scale_hint = hint
        try:
            xr = x.float().requires_grad_(True)
            (C * lm(inputs_embeds=xr, labels=labels).logits.float()).sum().backward()
            return xr.grad
        finally:
            lm._loss_scale_hint = None

    assert torch.equal(dx_of_logits_loss(0.5), dx_of_logits_loss(None))


@pytest.mark.parametrize("kind", ["ce_lin", "kl", "zlin"])
def test_magma_forward_trains_through_logits(emul_logits_ops, monkeypatch, kind):
    """Magma.forward, each loss on the logits (kl and zlin do not read out.loss): the oracle's adapter gradients and
    image-prefix gradient; a loss on out.loss alone gives the gradients of a run that never touches the logits."""
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

    def run(loss_of):
        model.arena.grad.zero_()
        for p in model.parameters():
            p.grad = None
        pr = prefix.float().requires_grad_(True)
        out = model(None, captions, input_embeddings=pr)
        assert out.logits.grad_fn is not None
        loss_of(out).backward()
        return {"dprefix": pr.grad.clone(), **{n: sd[n].grad.clone() for n in names}}

    plain = run(lambda out: out.loss)
    touched = run(lambda out: out.loss + 0 * out.logits.float().sum())
    assert all(rel(touched[k], plain[k]) < 1e-2 for k in plain)
    f, reads_ce = loss_fn(kind, cfg.vocab, B, S, seed=3)
    got = run(lambda out: (out.loss if reads_ce else 0.0) + f(out.logits.float()))
    params = {k: v.clone().requires_grad_(k in names) for k, v in w.items()}
    pf = prefix.float().requires_grad_(True)
    _, _, labels = O.magma_forward(None, captions, params, cfg, input_embeddings=pf.detach())
    x = torch.cat([pf, params["lm.transformer.wte.weight"][captions[:, : S - cfg.image_seq_len]]], dim=1)
    loss_o, logits_o, _ = oracle_lm(x, params, cfg, labels=labels)
    ((loss_o if reads_ce else 0.0) + f(logits_o)).backward()
    want = {"dprefix": pf.grad, **{k: params[k].grad for k in names}}
    bad = {k: round(rel(got[k], v), 4) for k, v in want.items() if rel(got[k], v) > 5e-2}
    assert not bad, bad
    assert rel(got["dprefix"], plain["dprefix"]) > 0.1
