"""output_attentions of the GPT-J runtime on the H100.

- The two kernels it adds, held element by element to float64 references with the arguments the schedules issue: the
  single-tile backward with a gradient on P from outside the block (mb200_attn_bwd_tile_dp, the rules of
  tests/test_attention_reference_gpu.py for the tile backward with dP = dO V^T + dP_ext), and the decode step that
  writes its probabilities (mb200_attn_decode_probs: P by the rounding rule, O bit for bit mb200_attn_decode's).
- At a small width through the C ABI: the attentions and the gradients of an auxiliary loss on them against the fp32
  oracle and its autograd, on the tile path (S = 40), the fused forward with the materialised backward (S = 136), and
  with MB200_ATTN_TILE=0 / MB200_ATTN_FLASH=0 (read once per process, so in a child process).
- At full GPT-J-6B size through B200GPTJForCausalLM: stored B = 8, S = 128 and recompute B = 1, S = 2048 (attentions
  equal between the paths bit for bit, a zero attention gradient equal to the plain backward), and a prefill with
  decode steps against a full-sequence call."""
import ctypes
import math
import os
import subprocess
import sys

import pytest
import torch

from _refcheck import SENTINEL, Buf, bf16_rne, bits
from test_attention_reference_gpu import (TINY, U, _acc, _check_bound, _check_rounded, _check_zero, _count, _dev, _draw,
                                          _gen, _inv_rope, _one_launch, _probs, _Qkv, _same, _scores)
from test_attentions_cpu import attn_weights, check, check_rows, ld8, oracle_attn_lm, run_infer, run_train
from test_gptj_recompute_cpu import case
from test_hidden_states_gpu import on_gpu, rel_dev
from test_sched_emul_cpu import rel

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    from magma_b200 import _lib, build

    build.build()
    return _lib.lib()


# ---- A. the tile backward with dP_ext --------------------------------------------------------------------------
def _tile_dp(lib, B, S, H, hd, rot):
    from magma_b200 import ops

    name = f"tile_dp B={B} S={S} H={H} hd={hd} rot={rot}"
    dev, bf = _dev(), torch.bfloat16
    gen = _gen("tile_dp", B, S, H, hd, rot)
    x = _Qkv(gen, B, S, H, hd, "std2")
    ldP = ld8(S)  # the schedules' layout: P and dP_ext both [B, H, S, S rounded up to 8]
    P = torch.empty(B, H, S, ldP, dtype=bf, device=dev)
    ops.attn_fwd_tile(x.view, B, S, H, hd, P=P)
    Ph = P[..., :S].double()
    dOb = Buf((), B * S, H * hd, bf, dev, float("nan"))
    dOb.view.copy_(torch.randn(B * S, H * hd, generator=gen, dtype=torch.float64).to(bf))
    dO = dOb.view.double().unflatten(1, (H, hd)).unflatten(0, (B, S)).permute(0, 2, 1, 3)
    # the gradient on P, NaN in the row padding (not read); as large as dO V^T so both terms show
    dPe = torch.full((B, H, S, ldP), float("nan"), dtype=bf, device=dev)
    dPe[..., :S] = (math.sqrt(hd) * torch.randn(B, H, S, S, generator=gen, dtype=torch.float64)).to(bf).to(dev)
    tab = ops.rope_table(S, rot, 0, device=dev) if rot else None
    inputs = [dOb.storage, P, dPe] + ([tab] if rot else [])
    before = [bits(t) for t in inputs]

    def bwd():
        Db = Buf((), B * S, 3 * H * hd, bf, dev, SENTINEL)
        n0 = _count()
        rc = lib.mb200_attn_bwd_tile_dp(x.view.data_ptr(), x.view.stride(0), dOb.view.data_ptr(), dOb.view.stride(0),
                                        P.data_ptr(), ldP, dPe.data_ptr(), ldP, Db.view.data_ptr(), Db.view.stride(0),
                                        None if tab is None else tab.data_ptr(), rot, B, S, H, hd, ops._stream())
        assert rc == 0, lib.mb200_last_error()
        _one_launch(name, n0)
        return Db

    Db = bwd()
    assert x.unchanged() and all(torch.equal(bits(t), b0) for t, b0 in zip(inputs, before)), f"{name}: input modified"
    assert Db.overwritten() == 0, f"{name}: dqkv written outside its rows"
    vis = torch.ones(S, S, dtype=torch.bool, device=dev).tril()
    dP = dO @ x.v.transpose(-1, -2) + dPe[..., :S].double()
    ddP = _acc(dO, x.v.transpose(-1, -2)) + U * dP.abs()  # + the fp32 addition of dP_ext
    D = (Ph * dP).sum(-1, keepdim=True)
    dD = (Ph * ddP).sum(-1, keepdim=True) + (4 * math.ceil(S / 8) + 2) * U * (Ph * dP.abs()).sum(-1, keepdim=True)
    r = 1.0 / math.sqrt(hd)
    dS = Ph * (dP - D) * r
    one_hot = ((Ph == 1).sum(-1, keepdim=True) == 1) & ((Ph != 0).sum(-1, keepdim=True) == 1)
    ddS = torch.where(one_hot, torch.zeros_like(dS), Ph * (ddP + dD) * r + 5 * U * dS.abs() + TINY)
    dSb = bf16_rne(dS)
    w = _check_rounded(f"{name} dS", dSb, dS, ddS, vis)
    g = Db.view.unflatten(1, (3, H, hd)).unflatten(0, (B, S)).permute(2, 0, 3, 1, 4)
    dq, bq = dSb @ x.k, _acc(dSb, x.k) + w @ x.k.abs()
    dk = dSb.transpose(-1, -2) @ x.q
    bk = _acc(dSb.transpose(-1, -2), x.q) + w.transpose(-1, -2) @ x.q.abs()
    dq, bq = _inv_rope(dq, bq, tab, rot)
    dk, bk = _inv_rope(dk, bk, tab, rot)
    _check_bound(f"{name} dQ", g[0], dq, bq)
    _check_bound(f"{name} dK", g[1], dk, bk)
    _check_bound(f"{name} dV", g[2], Ph.transpose(-1, -2) @ dO, _acc(Ph.transpose(-1, -2), dO))
    assert _same(Db.view, bwd().view), f"{name}: rerun not bit-identical"
    # a zero dP_ext gives mb200_attn_bwd_tile's result bit for bit
    dPe.zero_()
    Dz = bwd()
    D0 = Buf((), B * S, 3 * H * hd, bf, dev, SENTINEL)
    ops.attn_bwd_tile(x.view, dOb.view, P, B, S, H, hd, rope_tab=tab, rot=rot, dqkv=D0.view)
    assert _same(Dz.view, D0.view), f"{name}: zero dP_ext differs from the plain backward"


@pytest.mark.parametrize("hd", [64, 256])
@pytest.mark.parametrize("S", [1, 77, 128])
def test_tile_backward_with_external_dp(lib, S, hd):
    """At the schedule's arguments: fused qkv rows, P and dP_ext at ldP = S rounded up to 8, rotary on 64 dims."""
    _tile_dp(lib, 2, S, 3, hd, 64)


# ---- B. the decode step that writes its probabilities ------------------------------------------------------------
@pytest.mark.parametrize("pos", [0, 263, 2047])
def test_decode_probs(lib, pos):
    from magma_b200 import ops

    B, H, hd, Smax = 4, 16, 256, 2048
    name = f"decode_probs pos={pos}"
    dev, bf = _dev(), torch.bfloat16
    nk = pos + 1
    gen = _gen("decode_probs", pos)
    _, k0, v0 = _draw(gen, B, pos, H, hd, "std2", 0, nk)
    x = _Qkv(gen, B, 1, H, hd, "std2", pos, nk)
    old = []
    for t in (k0, v0):
        c = torch.full((B, H, Smax, hd), float("nan"), dtype=bf, device=dev)
        c[:, :, :pos] = t.permute(0, 2, 1, 3).to(bf).to(dev)
        old.append(c)
    ld = ld8(nk)  # the schedule's row: S_kv = pos + 1 rounded up to 8
    kc, vc = (c.clone() for c in old)
    out = torch.full((B, H * hd), SENTINEL, dtype=bf, device=dev)
    Pb = Buf((B, H), 1, ld, bf, dev, SENTINEL, ld=ld, bstrides=(H * ld, ld))
    n0 = _count()
    rc = lib.mb200_attn_decode_probs(x.view.data_ptr(), x.view.stride(0), kc.data_ptr(), vc.data_ptr(), out.data_ptr(),
                                     H * hd, Pb.storage.data_ptr(), ld, B, H, hd, Smax, pos, ops._stream())
    assert rc == 0, lib.mb200_last_error()
    _one_launch(name, n0)
    assert Pb.overwritten() == 0
    # O and the cache bit for bit what mb200_attn_decode computes
    kc0, vc0 = (c.clone() for c in old)
    out0 = ops.attn_decode(x.view, kc0, vc0, B, H, hd, pos)
    assert _same(out, out0.reshape(out.shape)) and _same(kc, kc0) and _same(vc, vc0)
    # P by the rounding rule against float64, zeros from column pos + 1 on
    k = kc[:, :, :nk].double()
    s, ds = _scores(x.q, k, hd, 5 * U, lane_gamma=(8 * math.ceil(hd / 256) + 5) * U)
    vis = torch.ones(1, nk, dtype=torch.bool, device=dev)
    p, E, flush = _probs(s, ds, vis, math.ceil(nk / 256) + 5 + 8)
    P = Pb.view[..., :nk]
    _check_rounded(f"{name} P", P, p, p * E + TINY, vis, flush)
    _check_zero(f"{name} P columns past pos", Pb.view[..., nk:])
    # O is P V with exactly these probabilities: sequential fp32 accumulation
    Ph = P.double()
    v = vc[:, :, :nk].double()
    _check_bound(f"{name} out", out.unflatten(1, (H, hd))[:, :, None], Ph @ v, nk * U * (Ph @ v.abs()))


# ---- C. small width through the C ABI ----------------------------------------------------------------------------
@pytest.mark.parametrize("recompute", [False, True], ids=["stored", "recompute"])
@pytest.mark.parametrize("path", ["tile", "flash"])
@pytest.mark.parametrize("mlp,attn,mlp_ln,attn_ln", [("normal", "normal", False, False),
                                                     ("parallel", "scaled_parallel", True, True)])
def test_attentions_and_aux_gradients_at_small_width(lib, recompute, path, mlp, attn, mlp_ln, attn_ln):
    cfg, w16, x, labels = case(path, mlp, attn, mlp_ln, attn_ln)
    B, S = labels.shape
    ca = attn_weights(cfg, B, S, range(cfg.n_layer))
    got = on_gpu(run_train, lib, cfg, w16, x, labels, recompute, da=ca)
    check(got, cfg, w16, x, labels, ca)
    other = on_gpu(run_train, lib, cfg, w16, x, labels, not recompute, da=ca)
    assert all(torch.equal(got[f"a{l}"], other[f"a{l}"]) for l in range(cfg.n_layer))
    # a zero attention gradient: the plain backward's dx and loss bit for bit
    zero = on_gpu(run_train, lib, cfg, w16, x, labels, recompute, da=[torch.zeros_like(c) for c in ca])
    plain = on_gpu(run_train, lib, cfg, w16, x, labels, recompute, attn=False)
    assert torch.equal(zero["dx"], plain["dx"]) and torch.equal(zero["loss"], plain["loss"])


@pytest.mark.parametrize("path", ["tile", "flash"])
def test_inference_attentions_at_small_width(lib, path):
    cfg, w16, x, _ = case(path, "normal", "normal", False, False, seed=3)
    B, S, d = x.shape
    _, A, _ = on_gpu(run_infer, lib, cfg, w16, x)
    params = {k: v.float() for k, v in w16.items()}
    _, _, attn_o = oracle_attn_lm(x.float(), params, cfg)
    bad = {l: round(rel(A[l], a), 4) for l, a in enumerate(attn_o) if rel(A[l], a) > 3e-2}
    assert not bad, bad
    check_rows(A, S)
    S_max = S + 8
    cache = [torch.zeros(cfg.n_layer, B, cfg.n_head, S_max, d // cfg.n_head, dtype=torch.bfloat16, device="cuda")
             for _ in range(2)]
    for p0, p1 in ((0, S - 5), (S - 5, S - 3), (S - 3, S - 2), (S - 2, S - 1), (S - 1, S)):
        _, Ap, _ = on_gpu(run_infer, lib, cfg, w16, x[:, p0:p1].contiguous(), cache=cache, pos0=p0, S_max=S_max)
        check_rows(Ap, p1)
        assert max(rel(Ap[l], A[l][:, :, p0:p1, :p1]) for l in range(cfg.n_layer)) < 2e-2, p0


@pytest.mark.parametrize("env", [{"MB200_ATTN_TILE": "0"}, {"MB200_ATTN_TILE": "0", "MB200_ATTN_FLASH": "0"}],
                         ids=["tile0", "tile0-flash0"])
def test_small_width_with_the_fused_kernels_off(env):
    """The same small-width checks on the paths the switches select: the fused forward with the materialised backward
    at S = 40, and batched GEMMs + softmax kernels for every step."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-p", "no:cacheprovider", "-m", "gpu",
                        __file__, "-k", "small_width and not fused_kernels_off"], env=dict(os.environ, **env), cwd=root,
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]


# ---- D. full size: GPT-J-6B through B200GPTJForCausalLM ----------------------------------------------------------
@pytest.fixture(scope="module")
def gptj6b():
    from magma_b200.language_model import get_gptj

    torch.cuda.set_device(0)
    return get_gptj(device="cuda:0").init_weights(seed=0)


@pytest.mark.parametrize("B,S,recompute", [(8, 128, False), (1, 2048, True)], ids=["stored-8x128", "recompute-1x2048"])
def test_gptj6b_attentions(gptj6b, monkeypatch, B, S, recompute):
    from magma_b200 import language_model

    lm = gptj6b
    g = torch.Generator(device="cuda").manual_seed(1)
    x = (0.5 * torch.randn(B, S, lm.config.hidden_size, generator=g, device="cuda")).to(torch.bfloat16)
    labels = torch.randint(0, lm.config.vocab_size, (B, S), generator=g, device="cuda")

    def train(path, attn, aux=None):
        monkeypatch.setattr(language_model, "_use_recompute", lambda *a: path)
        lm._ws.clear()
        xr = x.clone().requires_grad_(True)
        out = lm(inputs_embeds=xr, labels=labels, output_attentions=attn)
        assert lm._workspace_ex(B, S)[1] is path
        (out.loss if aux is None else out.loss + aux(out.attentions)).backward()
        return out, xr.grad

    plain, dx_plain = train(recompute, False)
    assert "attentions" not in plain
    out, dx_zero = train(recompute, True, lambda A: sum((0.0 * a.float()).sum() for a in A))
    assert len(out.attentions) == 28 and out.attentions[0].shape == (B, 16, S, S)
    assert torch.equal(out.loss, plain.loss) and torch.equal(out.logits, plain.logits)
    assert torch.equal(dx_zero, dx_plain)  # a zero attention gradient changes nothing
    for l in (0, 27):
        check_rows(out.attentions[l][:1], S)
    other, _ = train(not recompute, True)
    assert all(torch.equal(a, b) for a, b in zip(out.attentions, other.attentions))
    del other
    with torch.no_grad():
        inf = lm(inputs_embeds=x, output_attentions=True)
    assert max(rel_dev(a, b) for a, b in zip(inf.attentions, out.attentions)) < 1e-2
    # an auxiliary loss on two layers' attentions moves dx, and both paths agree on it bit for bit
    c = {l: torch.randn(B, 16, S, S, generator=g, device="cuda") for l in (3, 20)}
    aux = lambda A: sum((c[l] * A[l].float()).sum() for l in c)  # noqa: E731
    _, dx_aux = train(recompute, True, aux)
    assert rel_dev(dx_aux, dx_plain) > 1e-2
    _, dx_aux_other = train(not recompute, True, aux)
    assert torch.equal(dx_aux, dx_aux_other)
    lm._ws.clear()


def test_gptj6b_prefill_and_decode_attentions_match_a_full_sequence_call(gptj6b):
    lm = gptj6b
    B, S, n_dec = 1, 2044, 4
    g = torch.Generator(device="cuda").manual_seed(2)
    x = (0.5 * torch.randn(B, S + n_dec, lm.config.hidden_size, generator=g, device="cuda")).to(torch.bfloat16)
    with torch.no_grad():
        full = lm(inputs_embeds=x, output_attentions=True).attentions
        out = lm(inputs_embeds=x[:, :S], use_cache=True, output_attentions=True, max_cache_len=S + n_dec)
        parts = [(0, out.attentions)]
        for p in range(S, S + n_dec):
            parts.append((p, lm(inputs_embeds=x[:, p : p + 1], use_cache=True, past_key_values=out.past_key_values,
                                output_attentions=True).attentions))
    for p0, att in parts:
        q = att[0].shape[2]
        assert att[0].shape[-1] == p0 + q
        for l in (0, 13, 27):
            assert rel_dev(att[l], full[l][:, :, p0 : p0 + q, : p0 + q]) < 2e-2, (p0, l)
