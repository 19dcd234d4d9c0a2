"""Every distinct launch configuration the production passes issue, replayed on the GPU and held to the float64
references of the element-wise test files.

The launch records come from the product's host schedules run on the CPU emulation (tools/plan_trace.py): GPT-J-6B with
MLP adapters and the frozen ViT-L/14 at B = 8, S = 128 (config 2), GPT-J-6B at B = 8, S = 2048 on the recompute path,
the MAGMA_v2 adapter wiring, the trainable ViT-L/14, a prefill at S = 2048 and decode steps at B = 32. Launches with the
same op, scalars, alignment class and aliasing (tools/plan_trace.py::config_key) are one configuration.

GEMMs are replayed through the C ABI with every recorded scalar, the split-K scratch size included. Each operand sits at
its recorded byte offset mod 256 in NaN-padded storage laid out with the recorded leading dimension and batch strides.
Outputs sit in sentinel-filled storage. An output that aliases an input shares its storage, as the in-place residual
does. A is drawn at unit scale and B at 1 / sqrt(K); the rotary table starts at position 0. The bound is relative, so
neither choice loosens it. Checked: the element-wise bound, the sentinel outside every output, every input byte for byte,
the launch count of the plan the call reports, and that a rerun is bit identical. The float64 reference is computed in
chunks of rows and batches; the peak allocation and the wall time are printed at the end.

The other primitives are replayed at their recorded shape (rows, d, B, S, H, hd, V, ldv, nz, cache length and position,
causal, in place or not) by the checker of tests/test_attention_reference_gpu.py or test_elementwise_reference_gpu.py,
with its own sentinel, input and launch checks; those checkers lay rows out with padded strides of their own. Three
configurations are not replayed: their float64 checkers hold whole [rows, V] or [batch, S, S] tensors, several times the
2 GiB of their inputs, without chunking (TOO_LARGE, pinned by tests/test_production_launches_cpu.py).
"""
import ctypes
import math
import os
import sys
import time

import pytest

from _refcheck import SENTINEL, bits, dev as _dev, launches
import test_attention_reference_gpu as ATT
import test_elementwise_reference_gpu as ELT
from test_gemm_reference_gpu import _check, _reference

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tools"))
import plan_trace  # noqa: E402

pytestmark = pytest.mark.gpu

CHUNK_ELEMS = 1 << 26  # float64 elements of one [rows, N] or [rows, K] reference chunk (512 MiB)


def all_configs():
    """{key: (first record, [passes])} of the distinct launch configurations over every production pass, in issue
    order."""
    out = {}
    for name in plan_trace.PASSES:
        for key, (rec, n) in plan_trace.distinct_configs(plan_trace.pass_records(name)[1]).items():
            out.setdefault(key, (rec, []))[1].append(name)
    return out


def gemm_configs():
    """[(id, record, passes)] of the distinct GEMM configurations."""
    gemms = [(r, p) for r, p in all_configs().values() if r["op"] == "gemm"]
    return [(f"g{i:02d} {describe(r)}", r, p) for i, (r, p) in enumerate(gemms)]


def other_configs():
    """[(id, record, passes)] of the distinct configurations of every other primitive."""
    others = [(r, p) for r, p in all_configs().values() if r["op"] != "gemm"]
    return [(f"o{i:02d} {describe_other(r)}", r, p) for i, (r, p) in enumerate(others)]


def describe_other(r):
    ptrs = plan_trace.POINTERS[r["op"]]
    return r["op"] + " " + " ".join(f"{k}={v}" for k, v in r.items() if k != "op" and k not in ptrs)


def describe(r):
    epi = "+".join(k for k in ("bias", "aux_out", "aux_in", "res1", "res2", "rope_tab") if r[k]) or "plain"
    acts = f" act={r['act']}" * bool(r["act"]) + f" dact={r['dact']}" * bool(r["dact"])
    return (f"M={r['M']} N={r['N']} K={r['K']} nb={r['nb0']}x{r['nb1']} {'MN' if r['a_mn'] else 'K'}"
            f"{'MN' if r['b_mn'] else 'K'} {'f32' if r['c_dtype'] else 'bf16'} {epi}{acts}"
            f"{' static' * bool(r['b_static'])} ws={r['splitk_ws_bytes'] >> 20}M")


CONFIGS = gemm_configs()
OTHERS = other_configs()


def too_large(r):
    """Configurations whose float64 checker would hold several copies of a >= 2 GiB tensor at once."""
    op = r["op"]
    if op == "cross_entropy":
        return r["B"] * r["S"] * r["ldv"] > 1 << 28
    if op == "attn_fwd_flash":
        return r["B"] * r["H"] * r["Sq"] * r["Sk"] > 1 << 28
    if op == "softmax_bwd":
        return r["nz"] * r["Sq"] * r["Sk"] > 1 << 28
    return False


def other_replay(r):
    """The checker call that replays a non-GEMM record at its recorded shape."""
    op = r["op"]
    if op == "layernorm_fwd":
        return lambda: ELT._layernorm(r["rows"], r["d"], "normal")
    if op == "layernorm_bwd":
        return lambda: ELT._layernorm_bwd(r["rows"], r["d"], "normal", r["res"] is not None)
    if op in ("layernorm_param_grad", "layernorm_param_grad_rows"):
        return lambda: ELT._ln_param_grad(r["rows"], r["d"], op.endswith("_rows"), bool(r["accumulate"]))
    if op == "colsum":
        return lambda: ELT.test_colsum(r["rows"], r["cols"], bool(r["accumulate"]))
    if op == "cross_entropy":
        return lambda: ELT._cross_entropy(r["B"], r["S"], r["V"], r["ldv"], in_place=r["dlogits"] == r["logits"],
                                          grad_scale=r["grad_scale"])
    if op == "rope_table":
        return lambda: ELT.test_rope_table(r["S"], r["rot"], r["pos0"])
    if op == "quick_gelu_bwd":
        return lambda: ELT.test_quick_gelu_bwd(r["n"])
    if op == "patchify":
        return lambda: ELT.test_patchify_vit_front_end((r["B"], r["R"], r["P"]))
    if op == "vit_assemble":
        return lambda: ELT.test_vit_assemble((r["B"], r["T"], r["w"]))
    if op in ("attn_fwd_tile", "attn_bwd_tile"):
        return lambda: ATT._tile(r["B"], r["S"], r["H"], r["hd"], r.get("rot", 0))
    if op == "attn_fwd_flash" and r["k"][0] == "kcache":  # prefill: keys and values read from the KV cache
        return lambda: ATT._prefill(r["B"], r["Sq"], r["H"], r["hd"], r["Sk"] - r["Sq"])
    if op == "attn_fwd_flash":
        assert r["Sq"] == r["Sk"]
        return lambda: ATT._flash(r["B"], r["Sq"], r["H"], r["hd"], bool(r["causal"]))
    if op == "kv_append":
        return lambda: ATT._prefill(r["B"], r["S"], r["H"], r["hd"], r["pos0"])
    if op == "attn_decode":
        return lambda: ATT._decode(r["B"], r["H"], r["hd"], r["pos"], Smax=r["Smax"])
    if op == "softmax_bwd":  # the materialised attention backward of a non-causal forward (ViT)
        hd = round(r["scale"] ** -2)
        return lambda: ATT._softmax(r["nz"], r["Sq"], r["Sk"], False, 0, hd=hd)
    raise AssertionError(f"no replay for {op}")


@pytest.mark.parametrize("cid,rec,passes", OTHERS, ids=[c[0] for c in OTHERS])
def test_production_other_launch(budget, cid, rec, passes):
    if too_large(rec):
        pytest.skip("float64 checker does not fit beside its operands (TOO_LARGE)")
    other_replay(rec)()


class Tensor:
    """A [nb1, nb0, rows, cols] strided view at byte offset `off` (mod 256) of a flat storage filled with `fill`."""

    def __init__(self, rows, cols, ld, bs0, bs1, nb0, nb1, dtype, fill, off, dev):
        import torch

        esz = torch.empty((), dtype=dtype).element_size()
        assert off % esz == 0
        e0 = off // esz
        bs0, bs1 = (bs0 if nb0 > 1 else 0), (bs1 if nb1 > 1 else 0)
        size = e0 + (nb0 - 1) * bs0 + (nb1 - 1) * bs1 + (rows - 1) * ld + cols + 64
        self.storage = torch.full((size,), fill, dtype=dtype, device=dev)
        self.view = self.storage.as_strided((nb1, nb0, rows, cols), (bs1, bs0, ld, 1), e0)
        self.fill = fill

    def ptr(self):
        return self.view.data_ptr()

    def outside_untouched(self):
        import torch

        inside = torch.zeros(self.storage.numel(), dtype=torch.bool, device=self.storage.device)
        inside.as_strided(self.view.shape, self.view.stride(), self.view.storage_offset()).fill_(True)
        return bool((self.storage[~inside] == self.fill).all().item())


def _rand_(view, gen, scale):
    import torch

    t = torch.randn(view.shape, generator=gen, device=view.device, dtype=torch.float32) * scale
    view.copy_(t.to(view.dtype))


@pytest.fixture(scope="module")
def budget():
    import torch

    if _dev().type != "cuda":
        yield
        return
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    yield
    print(f"\n[budget] peak allocation {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB, "
          f"wall time {time.perf_counter() - t0:.1f} s for {len(CONFIGS)} GEMM and {len(OTHERS)} other configurations")


@pytest.mark.parametrize("cid,rec,passes", CONFIGS, ids=[c[0] for c in CONFIGS])
def test_production_gemm_launch(budget, cid, rec, passes):
    replay_gemm(cid, rec, passes)


def replay_gemm(cid, r, passes):
    """One GEMM record replayed and checked. The device comes from MB200_TEST_DEVICE (default cuda:0):
    tests/test_production_launches_cpu.py replays the cheap configurations on the CPU emulation of the operator, which has
    no launch plans to count."""
    import torch

    from magma_b200 import ops
    from magma_b200._lib import GemmArgs, lib

    dev = _dev()
    cuda = dev.type == "cuda"
    bf, nan = torch.bfloat16, float("nan")
    M, N, K, nb0, nb1 = r["M"], r["N"], r["K"], r["nb0"], r["nb1"]
    gen = torch.Generator(device=dev).manual_seed(M * 131 + N * 17 + K)
    off = lambda k: r[k][1] % 256  # noqa: E731

    # operands: A [M, K] (MN-major: stored [K, M]), B [N, K] at scale 1 / sqrt(K)
    def operand(name, rows, scale):
        mn = r[name.lower() + "_mn"]
        shape = (K, rows) if mn else (rows, K)
        t = Tensor(*shape, r[name.lower() + "_ld"], r[name.lower() + "_bs0"], r[name.lower() + "_bs1"], nb0, nb1, bf,
                   nan, off(name), dev)
        _rand_(t.view, gen, scale)
        return t, (t.view.transpose(-1, -2) if mn else t.view)

    A, Al = operand("A", M, 1.0)
    B, Bl = operand("B", N, 1.0 / math.sqrt(K))
    f32 = r["c_dtype"] == 1
    cdt = torch.float32 if f32 else bf
    mn_like = lambda dtype, fill, k, ld: Tensor(M, N, ld, r["c_bs0"], r["c_bs1"], nb0, nb1, dtype, fill, off(k), dev)  # noqa: E731
    C = mn_like(cdt, SENTINEL, "C", r["ldc"])
    inputs, outputs = {"A": A, "B": B}, {"C": C}
    if r["bias"]:
        bias = Tensor(1, N, N, 0, 0, 1, 1, bf, nan, off("bias"), dev)
        _rand_(bias.view, gen, 0.5)
        inputs["bias"] = bias
    if r["aux_in"]:
        aux_in = mn_like(bf, nan, "aux_in", r["ldc"])
        _rand_(aux_in.view, gen, 1.5)
        inputs["aux_in"] = aux_in
    for k in ("res1", "res2"):
        if r[k]:
            if r[k] == r["C"]:  # in place: the residual is the output's own storage
                assert r["ld_res"] == r["ldc"] and not f32
                _rand_(C.view, gen, 1.0)
                inputs[k] = C
                continue
            t = mn_like(bf, nan, k, r["ld_res"])
            _rand_(t.view, gen, 1.0)
            inputs[k] = t
    if r["aux_out"]:
        outputs["aux_out"] = mn_like(bf, SENTINEL, "aux_out", r["ldc"])
    tab = None
    if r["rope_tab"]:
        tab = ops.rope_table(r["rope_S"], r["rope_rot"], pos0=0, device=dev)
    ws = torch.full((r["splitk_ws_bytes"] // 4,), nan, dtype=torch.float32, device=dev) if r["splitk_ws"] else None
    res_old = {k: t.view.clone() for k, t in inputs.items() if t is C}

    a = GemmArgs()
    a.M, a.N, a.K, a.nb0, a.nb1, a.c_dtype = M, N, K, nb0, nb1, r["c_dtype"]
    for name, t in (("A", A), ("B", B)):
        o = getattr(a, name)
        o.ptr, o.ld, o.bs0, o.bs1 = t.ptr(), r[name.lower() + "_ld"], r[name.lower() + "_bs0"], r[name.lower() + "_bs1"]
        o.mn_major = r[name.lower() + "_mn"]
    a.B.static_data = r["b_static"]
    a.C, a.ldc, a.c_bs0, a.c_bs1, a.alpha = C.ptr(), r["ldc"], r["c_bs0"], r["c_bs1"], r["alpha"]
    a.act, a.dact, a.accumulate, a.ld_res = r["act"], r["dact"], r["accumulate"], r["ld_res"]
    for k in ("bias", "aux_in", "res1", "res2"):
        setattr(a, k, inputs[k].ptr() if k in inputs else None)
    a.aux_out = outputs["aux_out"].ptr() if "aux_out" in outputs else None
    a.force_bn, a.generic_epilogue = r["force_bn"], r["generic_epilogue"]
    a.rope_mode, a.rope_tab = r["rope_mode"], (tab.data_ptr() if tab is not None else None)
    a.rope_S, a.rope_hd, a.rope_rot, a.rope_ncols = r["rope_S"], r["rope_hd"], r["rope_rot"], r["rope_ncols"]
    a.splitk_ws = ws.data_ptr() if ws is not None else None
    a.splitk_ws_bytes = r["splitk_ws_bytes"]
    assert not r["accumulate"], "an accumulating production GEMM needs its old C drawn before the call"

    L = lib()
    before = {k: bits(t.storage) for k, t in inputs.items() if t is not C}

    def call():
        n0 = launches()
        rc = L.mb200_gemm(ctypes.byref(a), ops._stream())
        assert rc == 0, L.mb200_last_error()
        if not cuda:
            return 0, 1
        torch.cuda.synchronize()
        bn, split = ctypes.c_int32(), ctypes.c_int32()
        L.mb200_gemm_last_plan(ctypes.byref(bn), ctypes.byref(split))
        n = launches() - n0
        assert n == (2 if split.value > 1 else 1), f"{n} launches for a plan of {split.value} K splits"
        return bn.value, split.value

    bn, split = call()
    for k, t in inputs.items():
        if t is not C:
            assert torch.equal(bits(t.storage), before[k]), f"the call modified its input {k}"
    for k, t in outputs.items():
        assert t.outside_untouched(), f"sentinel outside {k} overwritten"

    # float64 reference in chunks of batches x rows
    nbt = nb0 * nb1
    if M * N <= CHUNK_ELEMS and M * K <= CHUNK_ELEMS:
        rows, per = M, max(1, CHUNK_ELEMS // (M * max(N, K)))
    else:
        rows, per = max(1, CHUNK_ELEMS // max(N, K)), 1
    flat = lambda v: v.flatten(0, 1)  # noqa: E731  [nb1, nb0, ...] -> [nb1 * nb0, ...], batch z = z1 * nb0 + z0
    worst, amb_n, total = 0.0, 0, 0
    for z0 in range(0, nbt, per):
        zs = slice(z0, min(nbt, z0 + per))
        for m0 in range(0, M, rows):
            ms = slice(m0, min(M, m0 + rows))
            sub = lambda v: flat(v)[zs, ms]  # noqa: E731
            kw = dict(alpha=r["alpha"], act=r["act"], dact=r["dact"], c_old=None, row0=m0,
                      bias=inputs["bias"].view.reshape(N) if "bias" in inputs else None,
                      aux_in=sub(inputs["aux_in"].view) if "aux_in" in inputs else None,
                      res1=(sub(res_old["res1"]) if "res1" in res_old else sub(inputs["res1"].view)) if "res1" in inputs else None,
                      res2=sub(inputs["res2"].view) if "res2" in inputs else None,
                      rope=(tab, r["rope_mode"], r["rope_S"], r["rope_hd"], r["rope_rot"], r["rope_ncols"]) if tab is not None else None)
            ref, pre, bound, amb = _reference(sub(Al), flat(Bl)[zs], **kw)
            worst = max(worst, _check(f"{cid} out rows {m0}+", sub(C.view), ref, bound, f32, amb, report=False))
            amb_n, total = amb_n + int(amb.sum().item()), total + amb.numel()
            if "aux_out" in outputs:
                worst = max(worst, _check(f"{cid} aux_out rows {m0}+", sub(outputs["aux_out"].view), pre, bound, False,
                                          report=False))
            del ref, pre, bound, amb
    print(f"[ratio] {cid} ({', '.join(passes)}; BN={bn}, {split} K splits): max err/bound {worst:.3f}, "
          f"ambiguous {amb_n} of {total} ({amb_n / total:.3%})")

    first = {k: bits(t.storage) for k, t in outputs.items()}
    for k, t in outputs.items():
        t.storage.fill_(t.fill)
    for k, v in res_old.items():
        C.view.copy_(v)
    if ws is not None:
        ws.fill_(nan)
    assert call() == (bn, split)
    for k, t in outputs.items():
        assert torch.equal(bits(t.storage), first[k]), f"{k}: rerun not bit-identical"
