"""Training GPT-J's own weights (freeze_lm: false, or any subset) on the CPU build of the schedule, held to the oracle's
autograd.

The backward adds the weight gradients of every LM parameter the mb200_gptj_lm_grads table names to those of the
adapters: dW = dy^T x of each linear from the gradients the dgrad GEMMs read and the activations the forward kept, the
LayerNorm parameter gradients, and the LM head's from the logits gradient. The word embedding's gradient is the input
gradient scattered over the token ids (mb200_embed_grad), whose kernel source runs here on the CPU kernel executor."""
import ctypes
import os
import subprocess

import pytest
import torch

from magma_b200._lib import GptjLayerGradsC, GptjLmGradsC, MB200Error
from oracle import magma_oracle as O
from test_attentions_cpu import attn_weights, oracle_attn_lm
from test_gptj_recompute_cpu import ENTRY, aligned_ws, case
from test_hidden_states_cpu import aux_weights, oracle_lm, ptrs
from test_logits_grad_cpu import BWD_LOGITS, build_logits_emul, grad_of, loss_fn, optr
from test_sched_emul_cpu import FORMS, c_lm_model, ptr, rel

HERE = os.path.dirname(os.path.abspath(__file__))
LAYER_FIELDS = [("ln1_g", "ln_1.weight"), ("ln1_b", "ln_1.bias"), ("w_out", "{attn}.out_proj.weight"),
                ("w_fc_in", "{mlp}.fc_in.weight"), ("b_fc_in", "{mlp}.fc_in.bias"), ("w_fc_out", "{mlp}.fc_out.weight"),
                ("b_fc_out", "{mlp}.fc_out.bias")]
TOP_FIELDS = [("lnf_g", "lm.transformer.ln_f.weight"), ("lnf_b", "lm.transformer.ln_f.bias"),
              ("w_lm", "lm.lm_head.weight"), ("b_lm", "lm.lm_head.bias")]


def build_lm_train_emul():
    """oracle/_build/libsched_emul_lm_train.so: the schedule emulation with the logits-gradient emulations of
    test_logits_grad_cpu.py and tests/embed_grad_emul.cpp."""
    from oracle import build_emul

    base = build_logits_emul()
    out = os.path.join(build_emul.OUT_DIR, "libsched_emul_lm_train.so")
    src = os.path.join(HERE, "embed_grad_emul.cpp")
    deps = [base, src, os.path.join(build_emul.ROOT, "include", "magma_b200.h")]
    if os.path.exists(out) and os.path.getmtime(out) >= max(os.path.getmtime(d) for d in deps):
        return out
    objs = [os.path.join(build_emul.OUT_DIR, os.path.basename(f).rsplit(".", 1)[0] + ".o")
            for f in build_emul.SCHEDULES + [build_emul.EMUL]]
    objs += [os.path.join(build_emul.OUT_DIR, n) for n in ("attention_emul_lg.o", "logits_grad_emul_lg.o")]
    eg = os.path.join(build_emul.OUT_DIR, "embed_grad_emul.o")
    r = subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-Wall", "-c", src, "-o", eg], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    r = subprocess.run(["g++", "-shared", "-o", out, *objs, eg], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return out


@pytest.fixture(scope="module")
def emul():
    from magma_b200 import _lib

    return _lib.configure(ctypes.CDLL(build_lm_train_emul()))


@pytest.fixture
def emul_train_ops(monkeypatch):
    """magma_b200.ops on the emulation above, for the Python training paths."""
    from magma_b200 import _lib, ops

    L = _lib.configure(ctypes.CDLL(build_lm_train_emul()))
    monkeypatch.setattr(_lib, "_lib", L)
    monkeypatch.setattr(ops, "_stream", lambda: None)
    return L


# ---- which LM parameters train --------------------------------------------------------------------------------------
def block_names(cfg, l):
    """{C field: oracle name} of block l's own parameters, q/k/v as the fused 'w_qkv' -> three names."""
    mk = cfg.mlp_adapter["adapter_type"] if cfg.mlp_adapter else None
    ak = cfg.attn_adapter["adapter_type"] if cfg.attn_adapter else None
    p = f"lm.transformer.h.{l}"
    attn = f"{p}.attn" + ("" if ak is None else (".attn_block" if ak == "normal" else ".module"))
    mlp = f"{p}.mlp" + ("" if mk is None else (".0" if mk == "normal" else ".module"))
    out = {f: f"{p}." + n.format(attn=attn[len(p) + 1:], mlp=mlp[len(p) + 1:]) for f, n in LAYER_FIELDS}
    out["w_qkv"] = tuple(f"{attn}.{q}.weight" for q in ("q_proj", "k_proj", "v_proj"))
    return out


def subset(cfg, which):
    """The oracle names of the LM parameters that train in the named choice (the word embedding is not the
    schedule's: see the Python tests)."""
    names = set()
    for l in range(cfg.n_layer):
        for f, n in block_names(cfg, l).items():
            for k in (n if isinstance(n, tuple) else (n,)):
                if which == "all" or (which == "last_block" and l == cfg.n_layer - 1) or \
                        (which == "ln_bias" and (f.startswith("ln1") or f.startswith("b_"))):
                    names.add(k)
    for f, n in TOP_FIELDS:
        if which in ("all", "head") or (which == "ln_bias" and f != "w_lm"):
            names.add(n)
    return names


def attach_lm_grads(m, cfg, w16, train, keep, fill=5.0):
    """Point m.lm_grads at fp32 buffers (filled with `fill`) for the parameters in `train`; returns {name: buffer},
    q/k/v under the tuple of their three names."""
    grads = {}

    def buf(names):
        shape = ((3 * cfg.d, cfg.d) if isinstance(names, tuple) else w16[names].shape)
        grads[names] = torch.full(shape, fill, dtype=torch.float32)
        return grads[names].data_ptr()

    lg = (GptjLayerGradsC * cfg.n_layer)()
    any_block = False
    for l in range(cfg.n_layer):
        for f, n in block_names(cfg, l).items():
            if (n[0] if isinstance(n, tuple) else n) in train:
                setattr(lg[l], f, buf(n))
                any_block = True
    top = GptjLmGradsC()
    for f, n in TOP_FIELDS:
        if n in train:
            setattr(top, f, buf(n))
    if any_block:
        top.layers = ctypes.cast(lg, ctypes.POINTER(GptjLayerGradsC))
    m.lm_grads = ctypes.pointer(top)
    keep += [lg, top]
    return grads


def run_train(L, cfg, w16, x, labels, recompute, train, f=None, dh=None, da=None, chunks=None, accumulate=0,
              scale=1.0, table=True):
    """Training forward, then the _logits backward (which a trainable LM head needs for its combined gradient) with the
    CE gradient scaled by `scale`. table=False leaves m.lm_grads NULL (the frozen LM)."""
    keep = []
    m, grads = c_lm_model(cfg, w16, keep)
    lgrads = attach_lm_grads(m, cfg, w16, train, keep) if table else {}
    B, S, V = x.shape[0], x.shape[1], cfg.vocab
    nbytes, fwd, _ = (getattr(L, fn) for fn in ENTRY[recompute])
    n = nbytes(ctypes.byref(m), B, S)
    ws, wsp = aligned_ws(n)
    ldv = (V + 63) // 64 * 64
    logits = torch.zeros(B * S, ldv, dtype=torch.bfloat16)
    loss = torch.zeros(1, dtype=torch.float32)
    assert fwd(ctypes.byref(m), ptr(x), optr(labels), ptr(logits), ldv, ptr(loss), B, S, wsp, n, None) == 0, \
        L.mb200_last_error()
    G = None
    if f is not None:
        G = grad_of(f, logits[:, :V].reshape(B, S, V)).reshape(B * S, V).to(torch.bfloat16)
    comb = torch.full((B * S, ldv), float("nan"), dtype=torch.bfloat16)
    dx = torch.full_like(x, float("nan"))
    for hi, lo in chunks or [(cfg.n_layer, 0)]:
        rc = getattr(L, BWD_LOGITS[recompute])(ctypes.byref(m), ptr(dx) if lo == 0 else None,
                                               None if dh is None else ptrs(dh), None if da is None else ptrs(da),
                                               (S + 7) // 8 * 8, optr(G), V, ptr(comb), scale if labels is not None else 0.0,
                                               hi, lo, accumulate, B, S, wsp, n, None)
        assert rc == 0, L.mb200_last_error()
    return {"loss": loss, "logits": logits, "dx": dx, **{k: g.clone() for k, g in grads.items()},
            **{k: g.clone() for k, g in lgrads.items()}}


def oracle(cfg, w16, x, labels, train, f=None, ch=None, ca=None, scale=1.0):
    params = {k: v.float().requires_grad_(".adapter" in k or k in train) for k, v in w16.items()}
    xf = x.float().requires_grad_(True)
    S = x.shape[1]
    loss, logits, states = oracle_lm(xf, params, cfg, labels=labels)
    total = scale * loss if labels is not None else 0.0
    if f is not None:
        total = total + f(logits)
    if ch is not None:
        total = total + sum((c.float() * h).sum() for c, h in zip(ch, states) if c is not None)
    if ca is not None:
        attn = oracle_attn_lm(xf, params, cfg)[2]
        total = total + sum((c[..., :S].float() * a).sum() for c, a in zip(ca, attn) if c is not None)
    total.backward()
    want = {k: p.grad for k, p in params.items() if p.requires_grad}
    for k in [k for k in want if k.endswith("q_proj.weight")]:
        trio = tuple(k.replace("q_proj", q) for q in ("q_proj", "k_proj", "v_proj"))
        want[trio] = torch.cat([want.pop(n) for n in trio], 0)
    return xf.grad, want


def check(got, cfg, w16, x, labels, train, tol=3e-2, **kw):  # kw: f, ch, ca, scale of oracle()
    dx_o, want = oracle(cfg, w16, x, labels, train, **kw)
    assert rel(got["dx"], dx_o) < tol
    grads = {k: v for k, v in got.items() if k in want}
    assert set(grads) == set(want)
    bad = {k: round(rel(g, want[k]), 4) for k, g in grads.items() if rel(g, want[k]) > (2 * tol if g.numel() == 1 else tol)}
    assert not bad, bad


# ---- the schedule ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("recompute", [False, True], ids=["stored", "recompute"])
@pytest.mark.parametrize("mlp,attn,mlp_ln,attn_ln", FORMS)
def test_every_lm_gradient_matches_oracle_in_every_adapter_form(emul, recompute, mlp, attn, mlp_ln, attn_ln):
    cfg, w16, x, labels = case("gemm", mlp, attn, mlp_ln, attn_ln)
    train = subset(cfg, "all")
    check(run_train(emul, cfg, w16, x, labels, recompute, train), cfg, w16, x, labels, train)


@pytest.mark.parametrize("which", ["all", "last_block", "ln_bias", "head"])
@pytest.mark.parametrize("recompute", [False, True], ids=["stored", "recompute"])
def test_subsets_with_hidden_attention_and_logits_gradients(emul, which, recompute):
    """Each subset, with gradients on the hidden states, the attentions and the logits in the same backward, in two
    layer chunks, on the fused single-tile attention path."""
    cfg, w16, x, labels = case("tile", "normal", "parallel", True, False, seed=2)
    B, S = labels.shape
    train = subset(cfg, which)
    f, _ = loss_fn("ce_lin", cfg.vocab, B, S, seed=5)
    ch = aux_weights(cfg, x, range(cfg.n_layer + 1))
    ca = attn_weights(cfg, B, S, range(cfg.n_layer), scale=4.0)
    got = run_train(emul, cfg, w16, x, labels, recompute, train, f=f, dh=ch, da=ca, chunks=[(2, 1), (1, 0)])
    check(got, cfg, w16, x, labels, train, tol=5e-2, f=f, ch=ch, ca=ca)


def test_lm_gradients_accumulate_and_recompute_equals_stored(emul):
    """accumulate != 0 adds onto the buffers; the recompute path's weight gradients equal the stored path's bit for bit
    (the 1-D ones are atomically reduced sums, equal to the last bits)."""
    cfg, w16, x, labels = case("gemm", "scaled_parallel", "normal", True, True, seed=3)
    train = subset(cfg, "all")
    g0 = run_train(emul, cfg, w16, x, labels, False, train)
    g1 = run_train(emul, cfg, w16, x, labels, False, train, accumulate=1)
    rc = run_train(emul, cfg, w16, x, labels, True, train)
    for k in g0:
        if k in ("loss", "logits", "dx"):
            continue
        assert torch.allclose(g1[k], g0[k] + 5.0, rtol=1e-4, atol=1e-4), k
        assert torch.allclose(rc[k], g0[k], rtol=1e-5, atol=1e-6), k


@pytest.mark.parametrize("recompute", [False, True], ids=["stored", "recompute"])
def test_all_null_lm_table_gives_the_frozen_lm_bit_for_bit(emul, recompute):
    """A table whose entries are all NULL (it carves the LayerNorm scratch and nothing reads it) gives loss, logits, dx
    and every adapter gradient of the NULL table bit for bit, which is the ctypes mirror's default."""
    cfg, w16, x, labels = case("gemm", "normal", "parallel", True, False, seed=4)
    keep = []
    assert not c_lm_model(cfg, w16, keep)[0].lm_grads
    frozen = run_train(emul, cfg, w16, x, labels, recompute, set(), table=False)
    empty = run_train(emul, cfg, w16, x, labels, recompute, set())
    assert set(frozen) == set(empty) and len(frozen) > 3
    assert not [k for k in frozen if not torch.equal(frozen[k], empty[k])]


@pytest.mark.parametrize("recompute", [False, True], ids=["stored", "recompute"])
def test_trainable_head_under_a_loss_scale(emul, recompute):
    """loss_scale = 0.25 (B200Engine's hint at gradient accumulation 4): the head's gradient is formed as
    (0.25 - 1) * dCE + dCE; dW_lm, db_lm, ln_f and the block gradients match the oracle's of 0.25 * CE."""
    cfg, w16, x, labels = case("gemm", "normal", None, False, False, seed=6)
    train = subset(cfg, "head") | subset(cfg, "last_block")
    got = run_train(emul, cfg, w16, x, labels, recompute, train, scale=0.25)
    check(got, cfg, w16, x, labels, train, scale=0.25)
    full = run_train(emul, cfg, w16, x, labels, recompute, train)
    assert rel(got["lm.lm_head.weight"], 0.25 * full["lm.lm_head.weight"]) < 1e-2


def test_a_trainable_head_needs_the_combined_buffer(emul):
    cfg, w16, x, labels = case("gemm", None, None, False, False)
    keep = []
    m, _ = c_lm_model(cfg, w16, keep)
    attach_lm_grads(m, cfg, w16, subset(cfg, "head"), keep)
    B, S = labels.shape
    n = emul.mb200_gptj_sched_workspace_bytes(ctypes.byref(m), B, S)
    ws, wsp = aligned_ws(n)
    ldv = (cfg.vocab + 63) // 64 * 64
    logits = torch.zeros(B * S, ldv, dtype=torch.bfloat16)
    loss = torch.zeros(1)
    assert emul.mb200_gptj_sched_forward(ctypes.byref(m), ptr(x), ptr(labels), ptr(logits), ldv, ptr(loss), B, S, wsp, n,
                                         None) == 0
    rc = emul.mb200_gptj_sched_backward_range(ctypes.byref(m), None, 1.0, cfg.n_layer, 0, 0, B, S, wsp, n, None)
    assert rc != 0 and b"dlogits_comb" in emul.mb200_last_error()


# ---- the launch trace of the LM-training pass at GPT-J-6B shapes -----------------------------------------------------
# distinct launch configurations (tools/plan_trace.py::config_key) of config 2's training pass with blocks 26, 27, ln_f
# and lm_head trainable that no production pass of tools/plan_trace.py issues; tests/test_lm_train_gpu.py replays each
# against float64. A schedule change that adds or removes one updates the pin on purpose.
LM_TRACE_PINNED = {"stored": 9, "recompute": 9}
# (recompute, loss_scale) of each traced pass: B = 8, S = 128, the recompute one under a 1/8 gradient-accumulation scale
LM_TRACE_PASSES = {"stored": (False, 1.0), "recompute": (True, 0.125)}


def build_trace_emul():
    """oracle/_build/libsched_emul_lm_trace.so: the schedule emulation with tests/lm_train_trace_emul.cpp, which
    records the combine launches while the emulation traces."""
    from oracle import build_emul

    base = build_emul.build()
    out = os.path.join(build_emul.OUT_DIR, "libsched_emul_lm_trace.so")
    src = os.path.join(HERE, "lm_train_trace_emul.cpp")
    if os.path.exists(out) and os.path.getmtime(out) >= max(os.path.getmtime(d) for d in (base, src)):
        return out
    objs = [os.path.join(build_emul.OUT_DIR, os.path.basename(f).rsplit(".", 1)[0] + ".o")
            for f in build_emul.SCHEDULES + [build_emul.EMUL]]
    o = os.path.join(build_emul.OUT_DIR, "lm_train_trace_emul.o")
    r = subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-Wall", "-c", src, "-o", o], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    r = subprocess.run(["g++", "-shared", "-o", out, *objs, o], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return out


def lm_train_records(name):
    """Launch records of a training forward and a _logits backward of GPT-J-6B with config 2's adapters and blocks 26,
    27, ln_f and lm_head trainable, B = 8, S = 128, every pointer resolved to [region, byte offset]."""
    import json
    import sys
    import tempfile

    sys.path.insert(0, os.path.join(HERE, "..", "tools"))
    import plan_trace
    from magma_b200._lib import configure

    recompute, scale = LM_TRACE_PASSES[name]
    B, S = 8, 128
    R = plan_trace.Regions()
    gm, keep = plan_trace.gptj6b(R)
    lg = (GptjLayerGradsC * gm.n_layer)()
    for l in (26, 27):
        for f, _ in GptjLayerGradsC._fields_:
            setattr(lg[l], f, R.new(f"lm.h{l}.g_{f}"))
    top = GptjLmGradsC()
    top.layers = ctypes.cast(lg, ctypes.POINTER(GptjLayerGradsC))
    for f in ("lnf_g", "lnf_b", "w_lm", "b_lm"):
        setattr(top, f, R.new(f"lm.g_{f}"))
    gm.lm_grads = ctypes.pointer(top)
    L = configure(ctypes.CDLL(build_trace_emul()))
    for fn in ("mb200_emul_trace", "mb200_emul_record", "mb200_lm_train_record"):
        getattr(L, fn).argtypes = [ctypes.c_char_p]
    nbytes, fwd, _ = (getattr(L, fn) for fn in ENTRY[recompute])
    with tempfile.TemporaryDirectory() as d:
        paths = [os.path.join(d, n) for n in ("trace", "rec", "rec_lg")]
        L.mb200_emul_trace(paths[0].encode())
        L.mb200_emul_record(paths[1].encode())
        L.mb200_lm_train_record(paths[2].encode())
        try:
            n = nbytes(ctypes.byref(gm), B, S)
            ws = ctypes.c_void_p(R.new("workspace", n))
            plan_trace.check(L, fwd(ctypes.byref(gm), R.new("x"), R.new("labels"), R.new("logits"), plan_trace.LDV,
                                    R.new("loss"), B, S, ws, n, None))
            plan_trace.check(L, getattr(L, BWD_LOGITS[recompute])(ctypes.byref(gm), R.new("dx"), None, None, 0, None, 0,
                                                                  R.new("dlogits_comb"), scale, gm.n_layer, 0, 0, B, S,
                                                                  ws, n, None))
        finally:
            for fn in ("mb200_emul_trace", "mb200_emul_record", "mb200_lm_train_record"):
                getattr(L, fn)(None)
        records = [json.loads(line) for p in paths[1:] for line in open(p)]
    for r in records:
        for k in plan_trace.POINTERS[r["op"]]:
            r[k] = R.resolve(r[k])
    return records


def new_lm_train_configs(name):
    """[(record, launches)] of the configurations of lm_train_records(name) that no production pass issues."""
    import sys

    sys.path.insert(0, os.path.join(HERE, "..", "tools"))
    import plan_trace

    known = set()
    for p in plan_trace.PASSES:
        known.update(plan_trace.distinct_configs(plan_trace.pass_records(p)[1]))
    return [v for k, v in plan_trace.distinct_configs(lm_train_records(name)).items() if k not in known]


@pytest.mark.parametrize("name", list(LM_TRACE_PASSES))
def test_lm_train_trace_is_pinned(name):
    """The new configurations: the wgrads of q/k/v, out_proj, fc_in, fc_out and the LM head (fp32, split-K), the bias
    column sums (the LM head's over the combined buffer's 50304-element rows), the LayerNorm parameter gradients, the
    combine of the CE gradient with itself at scale loss_scale - 1. Every one has a replay in
    tests/test_lm_train_gpu.py."""
    new = new_lm_train_configs(name)
    assert len(new) == LM_TRACE_PINNED[name], [(r["op"], {k: v for k, v in r.items() if not isinstance(v, list)})
                                                 for r, _ in new]
    ops_ = {r["op"] for r, _ in new}
    assert ops_ <= {"gemm", "colsum", "layernorm_param_grad_rows", "logits_grad_combine"}, ops_
    wgrads = {(r["M"], r["N"], r["K"]) for r, _ in new if r["op"] == "gemm" and r["c_dtype"] == 1}
    assert {(12288, 4096, 1024), (4096, 4096, 1024), (16384, 4096, 1024), (4096, 16384, 1024),
            (50258, 4096, 1024)} <= wgrads
    comb = [r for r, _ in new if r["op"] == "logits_grad_combine"]
    scale = LM_TRACE_PASSES[name][1]
    assert [(c["dce"], c["g"], c["alpha"], c["M"], c["V"]) for c in comb] == \
        [(comb[0]["dce"], comb[0]["dce"], scale - 1.0, 1024, 50258)]


# ---- mb200_embed_grad: the kernel source on the CPU kernel executor ---------------------------------------------------
def _embed_case(seed=0, B=3, T=21, d=24, vocab=11):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(-2, vocab + 2, (B, T + 3), generator=g)  # repeats, and ids outside [0, vocab)
    dx = torch.randn(B, T + 5, d, generator=g).to(torch.bfloat16)
    return ids, dx


def test_embed_grad_kernel_source_matches_fp64_and_repeats_bit_for_bit():
    from oracle import build_emul

    kx = ctypes.CDLL(build_emul.build_kernel_exec())
    ids, dx = _embed_case()
    B, T, d, vocab, L = 3, 21, 24, 11, 5
    dy = dx[:, L: L + T]  # rows of stride d inside batches of stride (T + 5) * d
    want = torch.zeros(vocab, d, dtype=torch.float64)
    idc = ids[:, :T].clamp_min(0).where((ids[:, :T] >= 0) & (ids[:, :T] < vocab), torch.zeros_like(ids[:, :T]))
    want.index_add_(0, idc.reshape(-1), dy.double().reshape(-1, d))
    outs = []
    for acc in (0, 0, 1):
        out = torch.full((vocab, d), 0.25, dtype=torch.float32) if acc else torch.full((vocab, d), float("nan"))
        rc = kx.mb200_embed_grad(ctypes.c_void_p(ids.data_ptr()), ctypes.c_int64(ids.stride(0)),
                                 ctypes.c_void_p(dy.data_ptr()), ctypes.c_int64(dy.stride(1)), ctypes.c_int64(dy.stride(0)),
                                 B, T, ctypes.c_void_p(out.data_ptr()), vocab, d, acc, None)
        assert rc == 0
        outs.append(out)
    n_max = int(torch.bincount(idc.reshape(-1)).max())
    assert n_max >= 5  # many repeats per id
    bound = n_max * 2.0**-23 * dy.double().abs().max() * n_max
    assert (outs[0].double() - want).abs().max() <= bound
    assert torch.equal(outs[0], outs[1])
    assert torch.equal(outs[2], (outs[0] + 0.25).float()) or (outs[2].double() - want - 0.25).abs().max() <= bound + 1e-6


def test_embed_grad_emulation_matches_the_kernel_source(emul):
    from oracle import build_emul

    kx = ctypes.CDLL(build_emul.build_kernel_exec())
    ids, dx = _embed_case(seed=1)
    dy = dx[:, 2:23]
    res = []
    for lib in (kx, emul):
        out = torch.empty(11, 24)
        assert lib.mb200_embed_grad(ctypes.c_void_p(ids.data_ptr()), ids.stride(0), ctypes.c_void_p(dy.data_ptr()),
                                    dy.stride(1), dy.stride(0), 3, 21, ctypes.c_void_p(out.data_ptr()), 11, 24, 0,
                                    None) == 0
        res.append(out)
    assert torch.equal(res[0], res[1])


# ---- the Python surface ------------------------------------------------------------------------------------------------
def _lm_and_oracle_weights():
    from test_gptj_recompute_cpu import _tiny_lm

    lm, x, labels = _tiny_lm()
    return lm, x, labels, {"lm." + n: p.detach().float().clone() for n, p in lm.named_parameters()}


def test_mixed_qkv_choice_raises():
    from test_gptj_recompute_cpu import _tiny_lm

    lm, _, _ = _tiny_lm()
    lm.transformer.h[1].attn.q_proj.weight.requires_grad_(True)
    with pytest.raises(MB200Error, match="q_proj, k_proj and v_proj of block 1 must train together"):
        lm.finalize()


def test_memory_check_raises_for_all_of_gpt_j_6b_on_80_gb():
    """18 bytes per trainable parameter: the whole LM (6.05 B parameters, vocabulary 50258) needs ~109 GB, more than an
    80 GB card holds even after its 12.1 GB of bf16 weights are released; the top 2 blocks + ln_f + lm_head fit."""
    from magma_b200.arena import check_fits

    d, dff, V, n_layer = 4096, 16384, 50258, 28
    block = [d, d, 3 * d * d, d * d, dff * d, dff, d * dff, d]
    top = [d, d, V * d, V]
    everything = block * n_layer + top + [V * d]
    n_all = sum(everything)
    assert 6.0e9 < n_all < 6.1e9 and abs(sum(block) - 201.4e6) < 0.1e6
    card = 80e9 - 2 * n_all  # what an 80 GB card can still allocate with the bf16 model on it
    with pytest.raises(MB200Error, match=r"need 10\d{10} bytes"):
        check_fits(everything, 2 * n_all, card)
    part = block * 2 + top
    check_fits(part, 2 * sum(part), card)


def test_language_model_trains_a_subset_and_the_embedding_from_input_ids(emul_train_ops):
    """A bare B200GPTJForCausalLM: block 1 + ln_f + lm_head + wte set to train, finalize(), then a loss through
    input_ids: the oracle's gradients of every trainable tensor; the bf16 module copies are gone and an optimizer step
    reaches the next pass."""
    lm, _, labels, w = _lm_and_oracle_weights()
    names = {n for n, _ in lm.named_parameters() if n.startswith(("transformer.h.1.", "transformer.ln_f.", "lm_head.",
                                                                 "transformer.wte."))}
    for n, p in lm.named_parameters():
        p.requires_grad_(n in names)
    lm.finalize()
    assert all(p.dtype == torch.float32 for n, p in lm.named_parameters() if n in names)
    assert lm.transformer.h[1].attn._fused is None and lm.transformer.h[0].attn._fused is not None
    ids = torch.randint(0, 96, (2, 12), generator=torch.Generator().manual_seed(5))
    ids[0, 3] = ids[1, 7] = ids[0, 9]  # repeated tokens sum their rows
    out = lm(input_ids=ids, labels=labels)
    out.loss.backward()
    params = {k: v.clone().requires_grad_(k[3:] in names) for k, v in w.items()}
    x = params["lm.transformer.wte.weight"][ids]
    cfg = O.OracleConfig(d=64, n_layer=2, n_head=4, rotary_dim=8, vocab=96, mlp_adapter=None)
    oracle_lm(x, params, cfg, labels=labels)[0].backward()
    sd = dict(lm.named_parameters())
    bad = {n: round(rel(sd[n].grad, params["lm." + n].grad), 4) for n in names
           if rel(sd[n].grad, params["lm." + n].grad) > 3e-2}
    assert not bad, bad
    # one optimizer step changes what the next pass computes; frozen weights stay as they were
    frozen = {n: p.detach().clone() for n, p in lm.named_parameters() if n not in names}
    before = lm(input_ids=ids, labels=labels).loss.detach()
    lm._arena.adamw_step(lr=1e-2)
    after = lm(input_ids=ids, labels=labels).loss.detach()
    assert float(after) < float(before)
    assert all(torch.equal(p, frozen[n]) for n, p in lm.named_parameters() if n not in names)


def test_language_model_trains_the_word_embedding_alone(emul_train_ops):
    """Only wte trains: the LM gradient table stays NULL (the frozen LM's backward) and the input gradient, scattered
    over input_ids, is the oracle's wte gradient."""
    lm, _, labels, w = _lm_and_oracle_weights()
    for n, p in lm.named_parameters():
        p.requires_grad_(n == "transformer.wte.weight")
    lm.finalize()
    assert not lm._cmodel_ex()[0].lm_grads
    ids = torch.randint(0, 96, (2, 12), generator=torch.Generator().manual_seed(6))
    ids[1, :4] = ids[0, 2]
    lm(input_ids=ids, labels=labels).loss.backward()
    params = {k: v.clone().requires_grad_(k == "lm.transformer.wte.weight") for k, v in w.items()}
    cfg = O.OracleConfig(d=64, n_layer=2, n_head=4, rotary_dim=8, vocab=96, mlp_adapter=None)
    oracle_lm(params["lm.transformer.wte.weight"][ids], params, cfg, labels=labels)[0].backward()
    got = lm.transformer.wte.weight.grad
    assert rel(got, params["lm.transformer.wte.weight"].grad) < 3e-2
    untouched = torch.ones(96, dtype=torch.bool)
    untouched[ids.reshape(-1)] = False
    assert bool((got[untouched] == 0).all())


def test_frozen_parameter_in_another_dtype_is_refused(emul_train_ops):
    """Only parameters an arena held in fp32 go back to bf16 when they stop training; a frozen one the caller moved to
    fp32 is refused as before."""
    lm, x, labels, _ = _lm_and_oracle_weights()
    lm.transformer.h[0].mlp.fc_in.bias.data = lm.transformer.h[0].mlp.fc_in.bias.data.float()
    with pytest.raises(MB200Error, match="must be bf16"):
        lm(inputs_embeds=x, labels=labels)
    lm, x, labels, _ = _lm_and_oracle_weights()
    p = lm.transformer.h[0].mlp.fc_in.bias
    p.requires_grad_(True)
    lm.finalize()
    assert p.dtype == torch.float32
    p.requires_grad_(False)
    lm.finalize()
    assert p.dtype == torch.bfloat16
    lm(inputs_embeds=x, labels=labels)


def test_magma_freeze_lm_false_trains_every_lm_parameter(emul_train_ops, monkeypatch):
    """Magma with freeze_lm: false: every LM parameter is in the arena, in backward order (LM head first, word
    embedding last); the gradients of the blocks, the head and the word embedding rows of the captions match the
    oracle's."""
    from test_e2e_dryrun_cpu import build, oracle_weights, tiny_cfg

    cfg = tiny_cfg(mlp_adapter={"adapter_type": "normal", "downsample_factor": 4})
    S, B = 16, 2
    w = oracle_weights(cfg)
    model, _ = build(monkeypatch, cfg, w, S, freeze_enc=True, freeze_lm=False)
    lm_names = [n for n, _ in model.named_parameters() if n.startswith("lm.")]
    assert all(dict(model.named_parameters())[n].requires_grad for n in lm_names)
    order = model.arena.names
    assert order[0].startswith(("lm.lm_head.", "lm.transformer.ln_f.")) and \
        order.index("lm.transformer.wte.weight") > max(i for i, n in enumerate(order) if ".transformer.h." in n)
    model.eval()
    images, captions = O.synthetic_batch(cfg, B, S, seed=11)
    with torch.no_grad():
        prefix = O.image_prefix(images.to(torch.bfloat16).float(), w, cfg).to(torch.bfloat16)
    pr = prefix.float().requires_grad_(True)
    model(None, captions, input_embeddings=pr).loss.backward()
    params = {k: v.clone().requires_grad_(k in lm_names) for k, v in w.items()}
    pf = prefix.float().requires_grad_(True)
    _, _, labels = O.magma_forward(None, captions, params, cfg, input_embeddings=pf.detach())
    x = torch.cat([pf, params["lm.transformer.wte.weight"][captions[:, : S - cfg.image_seq_len]]], dim=1)
    oracle_lm(x, params, cfg, labels=labels)[0].backward()
    sd = dict(model.named_parameters())
    bad = {k: round(rel(sd[k].grad, params[k].grad), 4) for k in lm_names if rel(sd[k].grad, params[k].grad) > 5e-2}
    assert not bad, bad
    assert rel(pr.grad, pf.grad) < 5e-2
