"""output_hidden_states of the GPT-J runtime on the H100: the n_layer + 1 hidden states against the fp32 oracle
(rel-Frobenius < 3e-2, the suite's bf16-vs-fp32 bound), gradients of an auxiliary loss on them against the oracle's
autograd, and the paths that do not read them unchanged bit for bit — at a small width through the C ABI, and at full
GPT-J-6B size (28 blocks, d = 4096) through B200GPTJForCausalLM on the stored (B = 8, S = 128) and the recompute
(B = 2, S = 2048) training paths and a KV-cache prefill with decode steps."""
import ctypes

import pytest
import torch

from oracle import magma_oracle as O
from test_gptj_recompute_cpu import case
from test_gptj_recompute_gpu import assert_same
from test_hidden_states_cpu import aux_weights, check_against_oracle, oracle_lm, run_infer, run_train
from test_sched_emul_cpu import rel

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    from magma_b200 import _lib, build

    build.build()
    return _lib.lib()


def moved(v, dev):
    if isinstance(v, torch.Tensor):
        return v.to(dev)
    if isinstance(v, dict):
        return {k: moved(t, dev) for k, t in v.items()}
    if isinstance(v, (list, tuple)):
        return type(v)(moved(t, dev) for t in v)
    return v


def on_gpu(fn, *args, **kw):
    """Run a helper of the CPU tests with its tensors on cuda:0; return its outputs on the CPU for the oracle."""
    with torch.device("cuda:0"):
        return moved(fn(*moved(args, "cuda:0"), **moved(kw, "cuda:0")), "cpu")


# ---- small width, every attention path, through the C ABI ------------------------------------------------------
@pytest.mark.parametrize("recompute", [False, True], ids=["stored", "recompute"])
@pytest.mark.parametrize("path", ["tile", "flash"])
@pytest.mark.parametrize("mlp,attn,mlp_ln,attn_ln", [("normal", None, False, False), ("normal", "normal", False, False),
                                                     ("parallel", "normal", True, True)])
def test_states_and_aux_gradients_at_small_width(lib, recompute, path, mlp, attn, mlp_ln, attn_ln):
    cfg, w16, x, labels = case(path, mlp, attn, mlp_ln, attn_ln)
    c = aux_weights(cfg, x, range(cfg.n_layer + 1))
    got = on_gpu(run_train, lib, cfg, w16, x, labels, recompute, c)
    check_against_oracle(got, cfg, w16, x, labels, c)
    # every hidden-state gradient absent: the plain backward, bit for bit (1-D gradients to their atomic reordering)
    none = on_gpu(run_train, lib, cfg, w16, x, labels, recompute, [None] * (cfg.n_layer + 1))
    plain = on_gpu(run_train, lib, cfg, w16, x, labels, recompute, None)
    assert_same(none, plain)


@pytest.mark.parametrize("path", ["tile", "flash"])
def test_inference_states_prefill_and_decode_at_small_width(lib, path):
    cfg, w16, x, _ = case(path, "normal", "normal", False, False, seed=3)
    logits, states = on_gpu(run_infer, lib, cfg, w16, x)
    params = {k: v.float() for k, v in w16.items()}
    _, _, states_o = oracle_lm(x.float(), params, cfg)
    bad = {l: round(rel(states[l], h), 4) for l, h in enumerate(states_o) if rel(states[l], h) > 3e-2}
    assert not bad, bad
    logits_ref, lnf = on_gpu(run_infer, lib, cfg, w16, x, hidden=False)
    assert torch.equal(logits, logits_ref) and torch.equal(states[-1].reshape(lnf.shape), lnf)
    # prefill of S - 3 positions, then three decode steps, against the slices of the full-sequence call
    B, S, d = x.shape
    S_max = S + 8
    cache = [torch.zeros(cfg.n_layer, B, cfg.n_head, S_max, d // cfg.n_head, dtype=torch.bfloat16, device="cuda")
             for _ in range(2)]
    parts = [on_gpu(run_infer, lib, cfg, w16, x[:, : S - 3].contiguous(), cache=cache, pos0=0, S_max=S_max)[1]]
    for p in range(S - 3, S):
        parts.append(on_gpu(run_infer, lib, cfg, w16, x[:, p : p + 1].contiguous(), cache=cache, pos0=p, S_max=S_max)[1])
    stepped = torch.cat(parts, dim=2)
    bad = {l: round(rel(stepped[l], states[l]), 4) for l in range(cfg.n_layer + 1) if rel(stepped[l], states[l]) > 2e-2}
    assert not bad, bad


# ---- full size: GPT-J-6B through B200GPTJForCausalLM ------------------------------------------------------------
def rel_dev(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-12)).item()


@pytest.fixture(scope="module")
def gptj6b():
    from magma_b200.language_model import get_gptj

    torch.cuda.set_device(0)
    return get_gptj(device="cuda:0").init_weights(seed=0)


@torch.no_grad()
def oracle_states(lm, x):
    """The fp32 oracle's n_layer + 1 states, one block at a time (its weights made fp32 per block) on the GPU."""
    c = lm.config
    cfg = O.OracleConfig(d=c.hidden_size, n_layer=c.num_layers, n_head=c.num_heads, rotary_dim=c.rotary_dim,
                         vocab=lm.lm_head.weight.shape[0], mlp_adapter=None)
    sd = dict(lm.named_parameters())
    h = x.float()
    states = [h]
    with torch.device("cuda:0"):
        positions = torch.arange(x.shape[1])
        for l in range(c.num_layers):
            w = {f"lm.{k}": v.float() for k, v in sd.items() if k.startswith(f"transformer.h.{l}.")}
            h = O.gptj_block(h, w, l, cfg, positions)[0]
            states.append(h)
    states[-1] = O.layer_norm(h, sd["transformer.ln_f.weight"].float(), sd["transformer.ln_f.bias"].float(), cfg.ln_eps)
    return states


def assert_states_close(states, want):
    assert len(states) == len(want) == 29
    bad = {l: round(rel_dev(s, w), 4) for l, (s, w) in enumerate(zip(states, want)) if rel_dev(s, w) > 3e-2}
    assert not bad, bad


def legacy_ln_f_output(lm, x):
    """What output_hidden_states returned before every state was: the inference pass's ln_f output alone."""
    from magma_b200 import ops
    from magma_b200._lib import check, lib as L

    B, S, d = x.shape
    m = lm._cmodel_ex()[0]
    n = L().mb200_gptj_sched_infer_workspace_bytes(ctypes.byref(m), B, S, S)
    ws = torch.empty(n, dtype=torch.uint8, device=x.device)
    hidden = torch.empty(B, S, d, dtype=torch.bfloat16, device=x.device)
    check(L().mb200_gptj_sched_infer(ctypes.byref(m), ops._ptr(x), None, lm.ldv, 0, ops._ptr(hidden), None, None, 0, 0,
                                     B, S, ops._ptr(ws), n, ops._stream()))
    return hidden


@pytest.mark.parametrize("B,S,recompute", [(8, 128, False), (2, 2048, True)], ids=["stored-8x128", "recompute-2x2048"])
def test_gptj6b_hidden_states(gptj6b, monkeypatch, B, S, recompute):
    from magma_b200 import language_model

    lm = gptj6b
    monkeypatch.setattr(language_model, "_use_recompute", lambda *a: recompute)
    lm._ws.clear()
    g = torch.Generator(device="cuda").manual_seed(1)
    x = (0.5 * torch.randn(B, S, lm.config.hidden_size, generator=g, device="cuda")).to(torch.bfloat16)
    labels = torch.randint(0, lm.config.vocab_size, (B, S), generator=g, device="cuda")
    labels[:, :2] = -100

    def train(hidden, aux=None):
        xr = x.clone().requires_grad_(True)
        out = lm(inputs_embeds=xr, labels=labels, output_hidden_states=hidden)
        loss = out.loss if aux is None else out.loss + aux(out.hidden_states)
        loss.backward()
        return out, xr.grad

    plain, dx_plain = train(False)
    assert lm._workspace_ex(B, S)[1] is recompute
    out, dx_unused = train(True)
    # loss, logits and dx bit for bit with and without the states
    assert torch.equal(out.loss, plain.loss) and torch.equal(out.logits, plain.logits)
    assert torch.equal(dx_unused, dx_plain)
    assert_states_close(out.hidden_states, oracle_states(lm, x))
    assert torch.equal(out.hidden_states[0], x)
    # the inference pass: the same states, its ln_f entry bit for bit what the single ln_f output was
    with torch.no_grad():
        inf = lm(inputs_embeds=x, output_hidden_states=True)
        assert torch.equal(inf.hidden_states[-1], legacy_ln_f_output(lm, x))
        assert torch.equal(inf.logits, lm(inputs_embeds=x).logits)
    assert_states_close(inf.hidden_states, out.hidden_states)
    # an auxiliary loss on three states (entry 0, a block output, the ln_f entry) moves dx by exactly its own gradient
    # where it enters, and the stored and recompute paths agree on it
    c = {l: 1e-3 * torch.randn(B, S, lm.config.hidden_size, generator=g, device="cuda") for l in (0, 14, 28)}
    _, dx_aux = train(True, lambda hs: sum((c[l] * hs[l].float()).sum() for l in c))
    assert rel_dev(dx_aux, dx_plain) > 0.1
    monkeypatch.setattr(language_model, "_use_recompute", lambda *a: not recompute)
    lm._ws.clear()
    _, dx_other = train(True, lambda hs: sum((c[l] * hs[l].float()).sum() for l in c))
    assert torch.equal(dx_other, dx_aux)
    lm._ws.clear()


def test_gptj6b_prefill_states_match_a_full_sequence_call(gptj6b):
    """A 2044-token prefill into a KV cache followed by four decode steps returns the states of the new positions,
    equal within tolerance to the matching slices of one 2048-token call."""
    lm = gptj6b
    B, S, n_dec = 1, 2044, 4
    g = torch.Generator(device="cuda").manual_seed(2)
    x = (0.5 * torch.randn(B, S + n_dec, lm.config.hidden_size, generator=g, device="cuda")).to(torch.bfloat16)
    with torch.no_grad():
        full = lm(inputs_embeds=x, output_hidden_states=True).hidden_states
        out = lm(inputs_embeds=x[:, :S], use_cache=True, output_hidden_states=True, max_cache_len=S + n_dec)
        parts = [out.hidden_states]
        for p in range(S, S + n_dec):
            parts.append(lm(inputs_embeds=x[:, p : p + 1], use_cache=True, past_key_values=out.past_key_values,
                            output_hidden_states=True).hidden_states)
    for l in range(len(full)):
        stepped = torch.cat([p[l] for p in parts], dim=1)
        assert rel_dev(stepped, full[l]) < 2e-2, l
