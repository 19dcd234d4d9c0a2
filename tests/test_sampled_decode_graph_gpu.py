"""Sampled decoding (temperature > 0) in the device-resident decode loop: `generate` replays one CUDA graph of the decode
step per token, and the step draws its token with mb200_sample_dev, which reads the Philox offset from the cache
position in device memory (offset = pos - s0 + 1, the step index the host-driven loop passes to mb200_sample).

- The graph-replayed loop emits the same ids as the host-driven loop (MB200_DECODE_GRAPH=0) under the same
  torch.manual_seed, for several (temperature, top_k, top_p), with an EOS that stops generation early, and at B = 1.
- Two calls under different seeds differ.
- A replaced ops.sample is still called once per step (generate keeps the host-driven loop for it).
- mb200_sample_dev at a given position returns the tokens of mb200_sample at offset pos - s0 + 1, on bf16 and fp32
  logits with V not a multiple of 1024, and rejects bad arguments without a launch.

The device comes from MB200_TEST_DEVICE (default cuda:0): tests/test_sampled_decode_graph_twin_cpu.py replays the
kernel-level bodies on the kernel source executed on the CPU (oracle/kernel_host_exec.cpp)."""
import math

import pytest

import test_sampling_reference_gpu as S
from _refcheck import dev as _dev, launches

pytestmark = pytest.mark.gpu

E_SHAPE, E_DTYPE, E_ARG = -1, -2, -7
# (s0, pos): the first decode step (offset 1), a later step of a long prompt, the position before the first step
# (offset 0) and a large position
POSITIONS = ((7, 7), (149, 160), (5, 4), (3, 2**31 - 2))


# ---------------------------------------------------------------------------------------------
# kernel level: mb200_sample_dev against mb200_sample
# ---------------------------------------------------------------------------------------------
def _sample_dev_matches_sample(dtype, V, rows, filters, temps=(0.7, 1.3)):
    """For each (filter, temperature, position): sample_dev on a [rows, V] view with a row stride > V equals sample at
    offset pos - s0 + 1; the logits and the position are left as they were, no token is written past `rows`."""
    import torch

    from magma_b200 import ops

    dev = _dev()
    ld = V + 24
    seed = S.BIG_SEEDS[0]
    int_view = torch.int16 if dtype == torch.bfloat16 else torch.int32
    for ci, (dist, k, p) in enumerate(filters):
        store = torch.full((rows * ld,), math.nan, dtype=dtype, device=dev)
        x = store.view(rows, ld)[:, :V]
        x.copy_(S._logits(dist, rows, V, dtype, S._gen("sample_dev", str(dtype), V, ci)))
        before = store.clone()
        for T in temps:
            for s0, pos in POSITIONS:
                pos_dev = torch.tensor([pos], dtype=torch.int32, device=dev)
                buf = torch.full((rows + 4,), -7, dtype=torch.int64, device=dev)
                n0 = launches()
                ops.sample_dev(x, pos_dev, s0, T, k, p, seed, buf[:rows])
                if dev.type == "cuda":
                    torch.cuda.synchronize()
                assert launches() - n0 == 1, f"{dist} k={k} p={p}: {launches() - n0} launches"
                want = ops.sample(x, T, top_k=k, top_p=p, seed=seed, offset=pos - s0 + 1)
                assert torch.equal(buf[:rows], want), (dist, k, p, T, s0, pos, buf[:rows].tolist(), want.tolist())
                assert bool((buf[rows:] == -7).all()), f"{dist}: tokens written past row {rows}"
                assert int(pos_dev.item()) == pos, "the position was modified"
        assert torch.equal(store.view(int_view), before.view(int_view)), f"{dist}: the logits were modified"


def _argument_checks():
    """Bad arguments return their error code without a launch and write no token; a NULL position is MB200_E_ARG."""
    import torch

    from magma_b200._lib import lib
    from magma_b200 import ops

    dev = _dev()
    x = torch.zeros(2, 64, dtype=torch.bfloat16, device=dev)
    tok = torch.full((4,), -7, dtype=torch.int64, device=dev)
    pos = torch.tensor([9], dtype=torch.int32, device=dev)
    good = dict(code=0, ld=64, R=2, V=64, T=1.0, k=0, p=0.9, pos=pos.data_ptr())
    bad = [("pos_dev=NULL", dict(pos=None), E_ARG), ("rows=0", dict(R=0), E_SHAPE), ("V=0", dict(V=0), E_SHAPE),
           ("ld<V", dict(ld=63), E_SHAPE), ("T=0", dict(T=0.0), E_ARG), ("T=NaN", dict(T=math.nan), E_ARG),
           ("top_k<0", dict(k=-1), E_ARG), ("top_p>1", dict(p=1.5), E_ARG), ("dtype", dict(code=7), E_DTYPE)]
    for name, change, want in bad:
        a = dict(good, **change)
        n0 = launches()
        rc = lib().mb200_sample_dev(x.data_ptr(), a["code"], a["ld"], a["R"], a["V"], a["T"], a["k"], a["p"], 1,
                                    a["pos"], 8, tok.data_ptr(), None, ops._stream())
        if dev.type == "cuda":
            torch.cuda.synchronize()
        assert rc == want, f"{name}: rc {rc}, expected {want}"
        assert launches() == n0, f"{name}: launched"
        assert bool((tok == -7).all()), f"{name}: tokens written"
    assert b"sample_dev" in lib().mb200_last_error()


# (distribution, top_k, top_p), distributions of test_sampling_reference_gpu.py
FILTERS = [("mid", 0, 0.9), ("flat", 0, 0.5), ("peaked", 40, 0.0), ("steps", 40, 0.9), ("mid", 40, 0.9),
           ("flat", 0, 0.0)]


@pytest.mark.parametrize("V", [1031, 50258])
def test_sample_dev_matches_sample_at_the_step_offset(V):
    import torch

    _sample_dev_matches_sample(torch.bfloat16, V, 5, FILTERS)
    _sample_dev_matches_sample(torch.float32, V, 3, FILTERS[::2])


def test_sample_dev_argument_checks_do_not_launch():
    _argument_checks()


# ---------------------------------------------------------------------------------------------
# generate: graph-replayed sampled loop against the host-driven loop
# ---------------------------------------------------------------------------------------------
def _model(seed=9):
    import torch

    from _gpu_util import build_magma_from_weights, gpu_device
    from oracle import magma_oracle as O
    from tools.model_check import small_cfg

    cfg = small_cfg(n_layer=3)
    w16 = {k: v.to(torch.bfloat16).float() for k, v in O.init_weights(cfg, seed=seed).items()}
    model = build_magma_from_weights(w16, cfg, {"mlp": {"adapter_type": "normal", "downsample_factor": 4}}, 32,
                                     gpu_device(), vit_name="clip_vit_sampled_graph_case")
    model.eval()
    return model, cfg


@pytest.fixture(scope="module")
def small_model():
    return _model()


def _prompt(cfg, B, s, seed=3):
    import torch

    g = torch.Generator().manual_seed(seed)
    return (torch.randn(B, s, cfg.d, generator=g) * 0.5).to(torch.bfloat16).to(_dev())


def _generate(monkeypatch, model, emb, graph, torch_seed=0, **kw):
    """sampling.generate(model, emb, decode=False, max_steps=40, **kw) under torch.manual_seed(torch_seed) in the
    host-driven loop or the graph-replayed one. Also returns how often ops.sample_dev was called."""
    import torch

    from magma_b200 import ops, sampling

    calls = [0]
    orig = ops.sample_dev

    def counted(*a, **k):
        calls[0] += 1
        return orig(*a, **k)

    with monkeypatch.context() as m:
        m.setattr(ops, "sample_dev", counted)
        m.setenv("MB200_DECODE_GRAPH", "1" if graph else "0")
        torch.manual_seed(torch_seed)
        out = sampling.generate(model, emb, **dict(dict(max_steps=40, decode=False), **kw)).cpu()
    return out, calls[0]


def _host_and_graph(monkeypatch, model, emb, **kw):
    host, hc = _generate(monkeypatch, model, emb, graph=False, **kw)
    graph, gc = _generate(monkeypatch, model, emb, graph=True, **kw)
    # the graph path calls ops.sample_dev twice (step 1 eagerly, then its capture); the host loop never
    assert hc == 0 and gc == 2, (hc, gc)
    return host, graph


@pytest.mark.parametrize("T,top_k,top_p", [(0.7, 0, 0.9), (1.0, 40, 0.0), (0.5, 40, 0.9), (1.3, 0, 0.0)])
def test_graph_replayed_sampled_decode_emits_the_host_loops_tokens(monkeypatch, small_model, T, top_k, top_p):
    import torch

    model, cfg = small_model
    emb = _prompt(cfg, 4, 7)
    host, graph = _host_and_graph(monkeypatch, model, emb, temperature=T, top_k=top_k, top_p=top_p)
    assert host.shape == (4, 7 + 40) and torch.equal(host, graph), (host[:, 7:].tolist(), graph[:, 7:].tolist())


def test_graph_replayed_sampled_decode_at_batch_one(monkeypatch, small_model):
    import torch

    model, cfg = small_model
    emb = _prompt(cfg, 1, 19, seed=4)
    host, graph = _host_and_graph(monkeypatch, model, emb, temperature=0.7, top_k=0, top_p=0.9)
    assert host.shape == (1, 19 + 40) and torch.equal(host, graph), (host[:, 19:].tolist(), graph[:, 19:].tolist())


def test_graph_replayed_sampled_decode_stops_at_the_same_eos(monkeypatch):
    """An eos_token whose logit is raised so that each row draws it with probability ~0.7 per step: all rows emit it in
    the same step early on, and both loops cut the output at that step (found by the lazy EOS check)."""
    import torch

    model, cfg = _model(seed=11)
    eos = 77
    model.lm.lm_head.bias.data[eos] += math.log(cfg.vocab) + 1.0
    model.lm.invalidate()
    model.lm.attach_arena(model.arena)
    emb = _prompt(cfg, 4, 7, seed=5)
    host, graph = _host_and_graph(monkeypatch, model, emb, temperature=1.0, top_k=0, top_p=0.0, eos_token=eos)
    assert torch.equal(host, graph), (host[:, 7:].tolist(), graph[:, 7:].tolist())
    n = host.shape[1] - 7
    print(f"EOS case: both loops stop after {n} of 40 steps")
    assert n < 40 and bool((host[:, -1] == eos).all()), host[:, 7:].tolist()


def test_graph_replayed_sampled_decode_differs_between_seeds(monkeypatch, small_model):
    """Two calls of the graph-replayed loop under different torch seeds draw different ids; the same seed repeats them.
    (That the offset advances with every replay, not only per call, is what the equality with the host loop, which
    passes the step index, shows.)"""
    import torch

    model, cfg = small_model
    emb = _prompt(cfg, 4, 7)
    kw = dict(temperature=1.3, top_k=0, top_p=0.0)
    a, _ = _generate(monkeypatch, model, emb, graph=True, torch_seed=1, **kw)
    b, _ = _generate(monkeypatch, model, emb, graph=True, torch_seed=2, **kw)
    a2, _ = _generate(monkeypatch, model, emb, graph=True, torch_seed=1, **kw)
    assert torch.equal(a, a2) and not torch.equal(a, b)



def test_a_replaced_sampler_is_called_every_step(monkeypatch, small_model):
    """A caller's replacement of ops.sample (here a counting wrapper of the library's own) is still called once per step
    with the graph enabled: generate keeps the host-driven loop for it, and the ids are those of the graph."""
    import torch

    from magma_b200 import ops, sampling

    model, cfg = small_model
    emb = _prompt(cfg, 4, 7)
    kw = dict(temperature=0.7, top_k=0, top_p=0.9)
    graph, gc = _generate(monkeypatch, model, emb, graph=True, **kw)
    offsets = []
    orig = ops.sample

    def replaced(*a, **k):
        offsets.append(k["offset"])
        return orig(*a, **k)

    monkeypatch.setattr(ops, "sample", replaced)
    monkeypatch.delenv("MB200_DECODE_GRAPH", raising=False)
    torch.manual_seed(0)
    host = sampling.generate(model, emb, max_steps=40, decode=False, **kw).cpu()
    assert offsets == list(range(40)) and gc == 2 and torch.equal(host, graph)
