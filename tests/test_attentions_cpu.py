"""output_attentions of the GPT-J runtime (csrc/gptj_sched.cu) on its CPU build, held to the oracle and its autograd.

Each block's probabilities, the bf16 values P V used, come out of the training forward (stored and recompute) and the
inference pass (full sequence, KV-cache prefill, decode steps). A loss that reads them sends its gradient into the same
backward pass: it joins dP = dO V^T before rowsum(dP * P), in the tile backward, or as the dP GEMM's residual on the
materialised path.

The reference attentions are composed here from the oracle's pieces (oracle_attn_lm: the probabilities of its
gptj_attention next to its blocks) and pinned to the reference's own (tests/golden/attentions.pt, written by
tools/make_attentions_golden.py). The schedule's CPU build links tests/attention_emul.cpp, the emulation of the two
kernels output_attentions adds, next to oracle/cabi_emul.cpp."""
import ctypes
import math
import os
import subprocess

import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN
from oracle import magma_oracle as O
from test_gptj_recompute_cpu import ENTRY, aligned_ws, case
from test_hidden_states_cpu import aux_weights, oracle_lm, ptrs
from test_sched_emul_cpu import FORMS, c_lm_model, ptr, rel

FWD_ATTN = {False: "mb200_gptj_sched_forward_attn", True: "mb200_gptj_sched_forward_attn_recompute"}
BWD_ATTN = {False: "mb200_gptj_sched_backward_range_attn", True: "mb200_gptj_sched_backward_range_attn_recompute"}


EXT_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "attention_emul.cpp")


def build_attn_emul():
    """oracle/_build/libsched_emul_attn.so: the objects of oracle/build_emul.py's schedule emulation plus
    tests/attention_emul.cpp."""
    from oracle import build_emul

    build_emul.build()
    out = os.path.join(build_emul.OUT_DIR, "libsched_emul_attn.so")
    objs = [os.path.join(build_emul.OUT_DIR, os.path.basename(f).rsplit(".", 1)[0] + ".o")
            for f in build_emul.SCHEDULES + [build_emul.EMUL]]
    deps = objs + [EXT_SRC, os.path.join(build_emul.ROOT, "include", "magma_b200.h")]
    if os.path.exists(out) and os.path.getmtime(out) >= max(os.path.getmtime(d) for d in deps):
        return out
    ext = os.path.join(build_emul.OUT_DIR, "attention_emul.o")
    for cmd in (["g++", "-O2", "-std=c++17", "-fPIC", "-Wall", "-c", EXT_SRC, "-o", ext],
                ["g++", "-shared", "-o", out, *objs, ext]):
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
    return out


@pytest.fixture(scope="module")
def emul():
    from magma_b200 import _lib

    return _lib.configure(ctypes.CDLL(build_attn_emul()))


@pytest.fixture
def emul_attn_ops(monkeypatch):
    """The conftest's emul_ops with the library that also emulates the output_attentions kernels."""
    from magma_b200 import _lib, ops

    L = _lib.configure(ctypes.CDLL(build_attn_emul()))
    monkeypatch.setattr(_lib, "_lib", L)
    monkeypatch.setattr(ops, "_stream", lambda: None)
    return L


def ld8(n):
    return (n + 7) // 8 * 8


# ---- the reference attentions -------------------------------------------------------------------------------------
def oracle_probs(h, w, pre, cfg, positions):
    """The probabilities oracle.magma_oracle.gptj_attention multiplies V with (hf:gptj/modeling_gptj.py:136-146):
    [B, H, S, S] from the ln_1 output h."""
    B, S, d = h.shape
    H = cfg.n_head
    hd = d // H
    sin, cos = O.rope_tables(positions, cfg.rotary_dim)
    q = O.apply_rope(F.linear(h, w[f"{pre}.q_proj.weight"]).view(B, S, H, hd), sin, cos, cfg.rotary_dim)
    k = O.apply_rope(F.linear(h, w[f"{pre}.k_proj.weight"]).view(B, S, H, hd), sin, cos, cfg.rotary_dim)
    q, k = q.permute(0, 2, 1, 3), k.permute(0, 2, 1, 3)
    att = torch.matmul(q.float(), k.float().transpose(-1, -2)) / math.sqrt(hd)
    att = att.masked_fill(torch.arange(k.shape[2])[None, :] > positions[:, None], torch.finfo(att.dtype).min)
    return torch.softmax(att, dim=-1).to(h.dtype)


def oracle_attn_lm(x, w, cfg, labels=None):
    """GPTJForCausalLM.forward(output_attentions=True) composed from the oracle's blocks, LayerNorm and loss, the
    probabilities of each block taken from its ln_1 output: (loss, logits, attentions)."""
    positions = torch.arange(x.shape[1])
    attentions = []
    kind = (cfg.attn_adapter or {}).get("adapter_type")
    for l in range(cfg.n_layer):
        p = f"lm.transformer.h.{l}"
        pre = {None: f"{p}.attn", "normal": f"{p}.attn.attn_block"}.get(kind, f"{p}.attn.module")
        h = O.layer_norm(x, w[f"{p}.ln_1.weight"], w[f"{p}.ln_1.bias"], cfg.ln_eps)
        attentions.append(oracle_probs(h, w, pre, cfg, positions))
        x = O.gptj_block(x, w, l, cfg, positions)[0]
    x = O.layer_norm(x, w["lm.transformer.ln_f.weight"], w["lm.transformer.ln_f.bias"], cfg.ln_eps)
    logits = F.linear(x, w["lm.lm_head.weight"], w["lm.lm_head.bias"])
    loss = O.cross_entropy_shifted(logits, labels) if labels is not None else None
    return loss, logits, tuple(attentions)


@pytest.mark.parametrize("tag", ["mlp_attn_normal", "attn_parallel"])
def test_oracle_attentions_match_the_reference(tag):
    """HF GPT-J (eager) inside the reference's Magma, its blocks wrapped by AdapterWrapper / ParallelAdapterWrapper;
    the weights are rebuilt from the fixture's seed as tools/make_attentions_golden.py built them."""
    rec = torch.load(f"{GOLDEN}/attentions.pt")[tag]
    lm, ac = rec["lm"], rec["adapter_config"]
    cfg = O.OracleConfig(d=lm["n_embd"], n_layer=lm["n_layer"], n_head=lm["n_head"], rotary_dim=lm["rotary_dim"],
                         vocab=rec["vocab"], mlp_adapter=ac.get("mlp"), attn_adapter=ac.get("attention"))
    w = {k: v for k, v in O.init_weights(cfg, seed=rec["seed"], with_vit=False).items() if k.startswith("lm.")}
    for k in w:
        for pat, g in rec["gains"].items():
            if pat in k:
                w[k] = w[k] * g
    _, logits, attn = oracle_attn_lm(rec["x"], w, cfg)
    assert torch.equal(logits, O.gptj_lm(rec["x"], w, cfg)[1])  # the composition is the oracle's LM
    assert torch.allclose(logits, rec["logits"], atol=1e-4, rtol=1e-4)
    assert len(attn) == len(rec["attentions"]) == cfg.n_layer
    for a, r in zip(attn, rec["attentions"]):
        assert a.shape == r.shape and torch.allclose(a, r, atol=1e-5, rtol=1e-4)
    # the fixture is not blind to the adapters: without them block 1's attentions move
    no_adapters = {k: v * 0 if ".adapter" in k else v for k, v in w.items()}
    assert (oracle_attn_lm(rec["x"], no_adapters, cfg)[2][1] - rec["attentions"][1]).abs().max() > 1e-2

# ---- training ------------------------------------------------------------------------------------------------------
def run_train(L, cfg, w16, x, labels, recompute, dh=None, da=None, act=0, chunks=None, attn=True):
    """Training forward (with the attentions when attn), then the backward with hidden-state gradients dh and
    attention gradients da (lists or None; both None runs the plain backward_range)."""
    keep = []
    m, grads = c_lm_model(cfg, w16, keep)
    m.adapter_act = act
    B, S = labels.shape
    H = cfg.n_head
    nbytes, fwd, bwd = (getattr(L, f) for f in ENTRY[recompute])
    n = nbytes(ctypes.byref(m), B, S)
    ws, wsp = aligned_ws(n)
    ldv = (cfg.vocab + 63) // 64 * 64
    logits = torch.zeros(B * S, ldv, dtype=torch.bfloat16)
    loss = torch.zeros(1, dtype=torch.float32)
    out = {}
    if attn:
        A = [torch.full((B, H, S, ld8(S)), float("nan"), dtype=torch.bfloat16) for _ in range(cfg.n_layer)]
        rc = getattr(L, FWD_ATTN[recompute])(ctypes.byref(m), ptr(x), ptr(labels), ptr(logits), ldv, ptr(loss), ptrs(A),
                                             ld8(S), B, S, wsp, n, None)
        out.update({f"a{l}": a[..., :S] for l, a in enumerate(A)})  # the row padding is not part of the result
    else:
        rc = fwd(ctypes.byref(m), ptr(x), ptr(labels), ptr(logits), ldv, ptr(loss), B, S, wsp, n, None)
    assert rc == 0, L.mb200_last_error()
    dx = torch.full_like(x, float("nan"))
    for hi, lo in chunks or [(cfg.n_layer, 0)]:
        dxp = ptr(dx) if lo == 0 else None
        if dh is None and da is None:
            rc = bwd(ctypes.byref(m), dxp, 1.0, hi, lo, 0, B, S, wsp, n, None)
        else:
            rc = getattr(L, BWD_ATTN[recompute])(ctypes.byref(m), dxp, None if dh is None else ptrs(dh),
                                                 None if da is None else ptrs(da), ld8(S), 1.0, hi, lo, 0, B, S, wsp, n,
                                                 None)
        assert rc == 0, L.mb200_last_error()
    return {"loss": loss, "logits": logits, "dx": dx, **out, **{k: g.clone() for k, g in grads.items()}}


def attn_weights(cfg, B, S, which, seed=8, scale=1.0):
    """Fixed random c_l of loss = CE + sum_l <c_l, A_l>, as bf16 [B, H, S, ld8(S)] buffers with NaN in the row
    padding (the runtime must not read it); None for layers not in `which`."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for l in range(cfg.n_layer):
        if l not in which:
            out.append(None)
            continue
        c = torch.full((B, cfg.n_head, S, ld8(S)), float("nan"), dtype=torch.bfloat16)
        c[..., :S] = (torch.randn(B, cfg.n_head, S, S, generator=g) * scale).to(torch.bfloat16)
        out.append(c)
    return out


def oracle(cfg, w16, x, labels, ca, ch=None, act=0):
    """loss, attentions, dx and trainable gradients of CE + sum <c_l, A_l> (+ sum <h_l, ch_l>) on the oracle."""
    cfg.adapter_act = ("relu", "gelu")[act]
    params = {k: v.float().requires_grad_(".adapter" in k) for k, v in w16.items()}
    xf = x.float().requires_grad_(True)
    S = x.shape[1]
    loss, _, attn = oracle_attn_lm(xf, params, cfg, labels=labels)
    total = loss + sum((c[..., :S].float() * a).sum() for c, a in zip(ca, attn) if c is not None)
    if ch is not None:
        _, _, states = oracle_lm(xf, params, cfg)
        total = total + sum((c.float() * h).sum() for c, h in zip(ch, states) if c is not None)
    total.backward()
    return loss.detach(), [a.detach() for a in attn], xf.grad, params


def check(got, cfg, w16, x, labels, ca, ch=None, act=0, tol=3e-2):
    S = x.shape[1]
    loss_o, attn_o, dx_o, params = oracle(cfg, w16, x, labels, ca, ch, act)
    assert abs(float(got["loss"]) - float(loss_o)) < 2e-2
    bad = {l: round(rel(got[f"a{l}"][..., :S], a), 4) for l, a in enumerate(attn_o) if rel(got[f"a{l}"][..., :S], a) > 2e-2}
    assert not bad, bad
    assert rel(got["dx"], dx_o) < tol, rel(got["dx"], dx_o)
    grads = {k: v for k, v in got.items() if k in params}
    assert set(grads) == {k for k, v in params.items() if v.requires_grad}
    # adapter_scale's gradient is one bf16 dot product over every row, which the auxiliary term dominates: twice the bar
    bad = {k: round(rel(g, params[k].grad), 4) for k, g in grads.items()
           if rel(g, params[k].grad) > (2 * tol if g.numel() == 1 else tol)}
    assert not bad, bad


@pytest.mark.parametrize("recompute", [False, True], ids=["stored", "recompute"])
@pytest.mark.parametrize("act", [0, 1], ids=["relu", "gelu"])
@pytest.mark.parametrize("mlp,attn,mlp_ln,attn_ln", FORMS)
def test_training_attentions_and_aux_loss_gradients_match_oracle(emul, recompute, act, mlp, attn, mlp_ln, attn_ln):
    """Every adapter form and activation, both activation paths, materialised attention (head_dim 16): the
    attentions, and every trainable gradient and dx of CE + sum_l <c_l, A_l> over all layers."""
    cfg, w16, x, labels = case("gemm", mlp, attn, mlp_ln, attn_ln)
    B, S = labels.shape
    ca = attn_weights(cfg, B, S, range(cfg.n_layer))
    got = run_train(emul, cfg, w16, x, labels, recompute, da=ca, act=act)
    check(got, cfg, w16, x, labels, ca, act=act)


@pytest.mark.parametrize("path", ["gemm", "tile", "flash"])
@pytest.mark.parametrize("recompute", [False, True], ids=["stored", "recompute"])
def test_attention_gradients_on_every_attention_path(emul, path, recompute):
    """The tile backward with dP_ext (S = 40) and the materialised backward after the fused forward (S = 136): the
    gradient of the auxiliary term is several times the CE term's, so a gradient added in the wrong place or not at
    all is far outside the tolerance."""
    cfg, w16, x, labels = case(path, "normal", "parallel", True, False, seed=1)
    B, S = labels.shape
    ca = attn_weights(cfg, B, S, range(cfg.n_layer), scale=4.0)
    got = run_train(emul, cfg, w16, x, labels, recompute, da=ca)
    check(got, cfg, w16, x, labels, ca)
    plain = run_train(emul, cfg, w16, x, labels, recompute, attn=False)
    assert rel(plain["dx"], got["dx"]) > 0.2  # the auxiliary term matters at this scale


@pytest.mark.parametrize("which", [[0], [1]], ids=["layer0", "layer1"])
def test_one_layer_and_hidden_states_together(emul, which):
    """A gradient on one layer's attentions only, together with hidden-state gradients, in one backward pass."""
    cfg, w16, x, labels = case("tile", "scaled_parallel", "normal", True, True, seed=6)
    B, S = labels.shape
    ca = attn_weights(cfg, B, S, which, seed=7, scale=4.0)
    ch = aux_weights(cfg, x, range(cfg.n_layer + 1))
    for recompute in (False, True):
        got = run_train(emul, cfg, w16, x, labels, recompute, dh=ch, da=ca)
        check(got, cfg, w16, x, labels, ca, ch)


@pytest.mark.parametrize("path", ["gemm", "tile", "flash"])
def test_layer_ranges_zero_gradients_and_paths_agree(emul, path):
    """Layer ranges [2,1) then [1,0) add each gradient once; stored and recompute give the same attentions and
    gradients bit for bit; an all-zero dattn gives the plain backward's results (dx, loss and every weight gradient)
    except the atomically reduced 1-D gradients, which may differ in the last bit; all-NULL pointers equal it exactly."""
    cfg, w16, x, labels = case(path, "normal", "parallel", True, False, seed=2)
    B, S = labels.shape
    ca = attn_weights(cfg, B, S, range(cfg.n_layer), scale=4.0)
    one = run_train(emul, cfg, w16, x, labels, False, da=ca)
    for recompute in (False, True):
        chunked = run_train(emul, cfg, w16, x, labels, recompute, da=ca, chunks=[(2, 1), (1, 0)])
        diff = [k for k in one if not torch.equal(chunked[k], one[k])]
        assert not diff, (recompute, diff)
        plain = run_train(emul, cfg, w16, x, labels, recompute, attn=False)
        nulls = run_train(emul, cfg, w16, x, labels, recompute, da=[None] * cfg.n_layer)
        diff = [k for k in plain if not torch.equal(nulls[k], plain[k])]
        assert not diff, (recompute, diff)
        zeros = [torch.zeros_like(c) for c in ca]
        zero = run_train(emul, cfg, w16, x, labels, recompute, da=zeros)
        diff = [k for k in plain if not torch.equal(zero[k], plain[k])]
        assert not diff, (recompute, diff)


def test_training_rejects_a_short_ld_attn(emul):
    cfg, w16, x, labels = case("gemm", None, None, False, False)
    keep = []
    m, _ = c_lm_model(cfg, w16, keep)
    B, S = labels.shape
    n = emul.mb200_gptj_sched_workspace_bytes(ctypes.byref(m), B, S)
    ws, wsp = aligned_ws(n)
    A = [torch.empty(B, cfg.n_head, S, S, dtype=torch.bfloat16) for _ in range(cfg.n_layer)]
    rc = emul.mb200_gptj_sched_forward_attn(ctypes.byref(m), ptr(x), None, None, 0, None, ptrs(A), S - 4, B, S, wsp, n,
                                            None)
    assert rc != 0 and b"ld_attn" in emul.mb200_last_error()


# ---- inference -----------------------------------------------------------------------------------------------------
def run_infer(L, cfg, w16, x, cache=None, pos0=0, S_max=0, ld=None, hidden=False):
    keep = []
    m, _ = c_lm_model(cfg, w16, keep, with_grads=False)
    B, S, d = x.shape
    n = L.mb200_gptj_sched_infer_workspace_bytes(ctypes.byref(m), B, S, S_max if cache else S)
    ws, wsp = aligned_ws(n)
    ldv = (cfg.vocab + 63) // 64 * 64
    logits = torch.zeros(B * S, ldv, dtype=torch.bfloat16)
    kc, vc = (ptr(cache[0]), ptr(cache[1])) if cache else (None, None)
    S_kv = pos0 + S
    ld = ld or ld8(S_kv)
    A = torch.full((cfg.n_layer, B, cfg.n_head, S, ld), float("nan"), dtype=torch.bfloat16)
    states = torch.full((cfg.n_layer + 1, B, S, d), float("nan"), dtype=torch.bfloat16) if hidden else None
    rc = L.mb200_gptj_sched_infer_attn(ctypes.byref(m), ptr(x), ptr(logits), ldv, 0, ptr(states) if hidden else None,
                                       states.stride(0) if hidden else 0, ptrs(list(A.unbind(0))), ld, kc, vc, S_max,
                                       pos0, B, S, wsp, n, None)
    assert rc == 0, L.mb200_last_error()
    return logits, A[..., :S_kv], states


def check_rows(A, S_kv):
    """Rows sum to 1 within bf16 rounding; entries above the causal diagonal (queries are the last S of S_kv) are 0."""
    S = A.shape[-2]
    sums = A.float().sum(-1)
    assert (sums - 1).abs().max() < S_kv * 2**-8
    above = torch.arange(S_kv)[None, :] > (torch.arange(S) + S_kv - S)[:, None]
    assert torch.equal(A[..., above], torch.zeros_like(A[..., above]))


@pytest.mark.parametrize("path", ["gemm", "tile", "flash"])
def test_inference_attentions_match_oracle(emul, path):
    cfg, w16, x, _ = case(path, "normal", "scaled_parallel", False, True, seed=3)
    S = x.shape[1]
    logits, A, _ = run_infer(emul, cfg, w16, x)
    params = {k: v.float() for k, v in w16.items()}
    _, _, attn_o = oracle_attn_lm(x.float(), params, cfg)
    bad = {l: round(rel(A[l], a), 4) for l, a in enumerate(attn_o) if rel(A[l], a) > 2e-2}
    assert not bad, bad
    check_rows(A, S)
    # the logits are those of the pass without attentions, bit for bit; with hidden states as well, both agree
    m_logits = run_infer_plain(emul, cfg, w16, x)
    assert torch.equal(logits, m_logits)
    logits2, A2, states = run_infer(emul, cfg, w16, x, hidden=True, ld=ld8(S) + 8)
    assert torch.equal(logits2, logits) and torch.equal(A2, A) and not states.isnan().any()


def run_infer_plain(L, cfg, w16, x):
    keep = []
    m, _ = c_lm_model(cfg, w16, keep, with_grads=False)
    B, S, d = x.shape
    n = L.mb200_gptj_sched_infer_workspace_bytes(ctypes.byref(m), B, S, S)
    ws, wsp = aligned_ws(n)
    ldv = (cfg.vocab + 63) // 64 * 64
    logits = torch.zeros(B * S, ldv, dtype=torch.bfloat16)
    assert L.mb200_gptj_sched_infer(ctypes.byref(m), ptr(x), ptr(logits), ldv, 0, None, None, None, 0, 0, B, S, wsp, n,
                                    None) == 0, L.mb200_last_error()
    return logits


@pytest.mark.parametrize("path", ["gemm", "tile"])
def test_prefill_continuation_and_decode_match_the_oracle(emul, path):
    """A 6-token prefill, a 2-token continuation over the cache, then three decode steps: each call's attentions are
    the oracle's rows for its positions over the keys so far, and the rows of one 11-token call."""
    cfg, w16, x, _ = case(path, "normal", None, False, False, seed=5, B=2)
    x = x[:, :11].contiguous()
    B, S, d = x.shape
    H, hd, S_max = cfg.n_head, cfg.d // cfg.n_head, 16
    params = {k: v.float() for k, v in w16.items()}
    _, _, full_o = oracle_attn_lm(x.float(), params, cfg)
    _, full, _ = run_infer(emul, cfg, w16, x)
    cache = [torch.zeros(cfg.n_layer, B, H, S_max, hd, dtype=torch.bfloat16) for _ in range(2)]
    for p0, p1 in ((0, 6), (6, 8), (8, 9), (9, 10), (10, 11)):
        _, A, _ = run_infer(emul, cfg, w16, x[:, p0:p1].contiguous(), cache=cache, pos0=p0, S_max=S_max)
        assert A.shape == (cfg.n_layer, B, H, p1 - p0, p1)
        check_rows(A, p1)
        for l in range(cfg.n_layer):
            assert rel(A[l], full_o[l][:, :, p0:p1, :p1]) < 2e-2, (p0, l)
            assert rel(A[l], full[l][:, :, p0:p1, :p1]) < 1e-2, (p0, l)


def test_inference_rejects_a_short_ld_attn(emul):
    cfg, w16, x, _ = case("gemm", None, None, False, False)
    keep = []
    m, _ = c_lm_model(cfg, w16, keep, with_grads=False)
    B, S, d = x.shape
    n = emul.mb200_gptj_sched_infer_workspace_bytes(ctypes.byref(m), B, S, S)
    ws, wsp = aligned_ws(n)
    A = [torch.empty(B, cfg.n_head, S, ld8(S), dtype=torch.bfloat16) for _ in range(cfg.n_layer)]
    rc = emul.mb200_gptj_sched_infer_attn(ctypes.byref(m), ptr(x), None, 0, 0, None, 0, ptrs(A), ld8(S) - 8, None, None,
                                          0, 0, B, S, wsp, n, None)
    assert rc != 0 and b"ld_attn" in emul.mb200_last_error()


# ---- the Python surface ----------------------------------------------------------------------------------------------
def test_language_model_returns_attentions_only_when_asked(emul_attn_ops):
    from test_gptj_recompute_cpu import _tiny_lm

    lm, x, labels = _tiny_lm()
    n, H = len(lm.transformer.h), lm.config.num_heads
    B, S, _ = x.shape
    plain = lm(inputs_embeds=x)
    assert set(plain) == {"loss", "logits", "past_key_values", "hidden_states"}
    inf = lm(inputs_embeds=x, output_attentions=True)
    assert len(inf.attentions) == n and all(a.shape == (B, H, S, S) and a.dtype == torch.bfloat16 for a in inf.attentions)
    assert torch.equal(inf.logits, plain.logits)
    with torch.no_grad():  # a loss without backward: the training pass writes them
        tr = lm(inputs_embeds=x, labels=labels, output_attentions=True)
    assert all(torch.equal(a, b) for a, b in zip(tr.attentions, inf.attentions))
    # prefill over a cache, then a host-driven decode step: S_kv grows with the cache
    pre = lm(inputs_embeds=x[:, :7], use_cache=True, output_attentions=True, max_cache_len=16)
    step = lm(inputs_embeds=x[:, 7:8], use_cache=True, past_key_values=pre.past_key_values, output_attentions=True)
    assert step.attentions[0].shape == (B, H, 1, 8)
    for a, b in zip(step.attentions, inf.attentions):
        assert rel(a, b[:, :, 7:8, :8]) < 1e-2


def test_language_model_trains_through_attentions(emul_attn_ops):
    """_LMTrainFn: CE + sum_l <c_l, A_l> gives the oracle's dx; attentions the loss does not read change nothing."""
    from test_gptj_recompute_cpu import _tiny_lm

    lm, x, labels = _tiny_lm()
    B, S, _ = x.shape

    def run(loss_of, **kw):
        xr = x.float().requires_grad_(True)
        out = lm(inputs_embeds=xr, labels=labels, **kw)
        loss_of(out).backward()
        return out, xr.grad

    _, dx_plain = run(lambda o: o.loss)
    out, dx_unused = run(lambda o: o.loss, output_attentions=True, output_hidden_states=True)
    assert "attentions" in out and torch.equal(dx_unused, dx_plain)
    g = torch.Generator().manual_seed(3)
    c = [torch.randn(B, lm.config.num_heads, S, S, generator=g) for _ in range(len(lm.transformer.h))]
    _, dx = run(lambda o: o.loss + sum((ci * a.float()).sum() for ci, a in zip(c, o.attentions)), output_attentions=True)
    w = {"lm." + n: p.detach().float() for n, p in lm.named_parameters()}
    cfg = O.OracleConfig(d=64, n_layer=2, n_head=4, rotary_dim=8, vocab=96, mlp_adapter=None)
    xf = x.float().requires_grad_(True)
    loss, _, attn = oracle_attn_lm(xf, w, cfg, labels=labels)
    (loss + sum((ci * a).sum() for ci, a in zip(c, attn))).backward()
    assert rel(dx, xf.grad) < 3e-2
    assert rel(dx, dx_plain) > 0.1
