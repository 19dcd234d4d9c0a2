"""Replay of the DEFAULT paths on the CPU. The GPU parity harness itself (tools/model_check.py groups lm, lm_variants,
vit, resnet, magma, generate — what tests/test_model_gpu.py runs on the GPU), the reference-golden tests of that file and
__graft_entry__.smoke() are executed here on CPU tensors. What runs is the product's own code: its Python, and its
HOST-ONLY C++ schedules (csrc/gptj_sched.cu, csrc/vit_sched.cu — no kernels, no CUDA calls) compiled as plain C++ into
the emulation library, issuing the primitive operators, which are what is emulated (oracle/cabi_emul.cpp). So a change
to anything but a kernel — pointer tables, workspace carving, operand majors and strides, chunked backward, KV-cache
prefill / decode, arena, engine — is caught without a GPU; the kernels themselves are verified by the `-m gpu` tests
only."""
import pytest
import torch


@pytest.fixture
def replay(emul_ops, monkeypatch):
    from magma_b200.magma import Magma

    monkeypatch.setattr(Magma, "_require_cuda", lambda self: None)
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    # the frozen conv trunk replays ~300 launches as one CUDA graph per batch size; "already capturing" = eager launches
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: True)
    return torch.device("cpu")


@pytest.mark.parametrize("group", ["lm", "lm_variants", "vit", "resnet", "magma"])
def test_gpu_parity_harness_replays_on_emulated_kernels(replay, group, capsys):
    from tools import model_check

    assert getattr(model_check, "group_" + group)(replay)
    assert "[FAIL]" not in capsys.readouterr().out




@pytest.mark.parametrize("tag", ["v1_mlp_normal", "v2_mlp_attn_normal", "parallel", "no_adapters"])
def test_reference_goldens_replay_on_emulated_kernels(replay, monkeypatch, golden_dir, tag):
    """The fixtures the REFERENCE ITSELF produced (tests/golden/magma_*.pt: loss, logits, every trainable gradient of
    Magma.forward under four adapter wirings) against this package's Python + host-only schedules on emulated kernels —
    the body of tests/test_model_gpu.py::test_magma_matches_reference_golden, unchanged."""
    import test_model_gpu as G

    monkeypatch.setenv("MB200_TEST_DEVICE", "cpu")
    G.test_magma_matches_reference_golden(golden_dir, tag)


def test_shared_layer_parity_case_replays_at_small_size(replay):
    """The body of tests/test_model_gpu.py::test_config2_full_size_matches_oracle (frozen weights shared across layers,
    per-layer adapters, decided ReLU masks) on emulated kernels at a small size, held to the same bars."""
    import test_model_gpu as G
    from tools.model_check import small_cfg

    r = G._shared_layer_case(replay, small_cfg(n_layer=3, vit_layers=2), B=2, S=32, vit_name="clip_vit_shared_small")
    assert r["dloss"] < 2e-2 and r["logits"] < 3e-2, r
    assert max(r["grads"].values()) < 3e-2, r["grads"]
    assert len(r["grads"]) == 3 * 4 + 4


def test_kv_decode_parity_case_replays_at_small_size(replay):
    """The body of tests/test_model_gpu.py::test_config5_full_size_kv_decode_matches_oracle (cache prefill, then greedy
    single-token steps, teacher-forced against one cache-less oracle forward) on a small geometry with emulated kernels."""
    import test_model_gpu as G
    from tools.model_check import small_cfg

    r = G._kv_decode_case(replay, small_cfg(n_layer=3, vit_layers=2), B=3, n_prompt=5, n_steps=4,
                          vit_name="clip_vit_shared_decode_small")
    assert max(r["logits"]) < 3e-2, r["logits"]
    assert all(r["picks"]), r


def test_reference_assertion_behaviour_replays(replay, monkeypatch):
    import test_model_gpu as G

    monkeypatch.setenv("MB200_TEST_DEVICE", "cpu")
    G.test_magma_forward_asserts_like_the_reference()


def test_generate_harness_and_reference_greedy_golden_replay(replay, monkeypatch, golden_dir, capsys):
    """KV-cache decoding on the CPU: the generate group of the GPU harness (greedy tokens identical to the oracle's, a
    decode step equal to the full forward) and the reference's own greedy-token golden
    (tests/test_model_gpu.py::test_vit_embed_generate_match_reference_golden), through sampling.generate ->
    decode_logits -> the emulated entry points (prefill + per-token decode of csrc/gptj_sched.cu)."""
    import test_model_gpu as G
    from tools import model_check

    assert model_check.group_generate(replay)
    assert "[FAIL]" not in capsys.readouterr().out
    monkeypatch.setenv("MB200_TEST_DEVICE", "cpu")
    G.test_vit_embed_generate_match_reference_golden(golden_dir)


def test_full_smoke_replays_with_decode(replay, capsys):
    import __graft_entry__ as entry

    entry.smoke(_device="cpu")
    assert "smoke OK" in capsys.readouterr().out


def test_generate_works_for_layernorm_and_scaled_adapters(replay, monkeypatch):
    """language_model routes adapters with add_layernorm / adapter_scale through the same schedule for decoding too:
    greedy tokens of the KV-cache loop equal an argmax over full re-forwards of the growing sequence."""
    import test_e2e_dryrun_cpu as E
    from oracle import magma_oracle as O

    mlp = {"adapter_type": "scaled_parallel", "downsample_factor": 4}
    cfg = E.tiny_cfg(mlp_adapter=mlp)
    w = E.oracle_weights(cfg)
    g = torch.Generator().manual_seed(2)
    for l in range(cfg.n_layer):
        pre = f"lm.transformer.h.{l}.mlp"
        for i, j in ((2, 3), (0, 1)):
            for sfx in ("weight", "bias"):
                w[f"{pre}.adapter.{j}.{sfx}"] = w.pop(f"{pre}.adapter.{i}.{sfx}")
        w[f"{pre}.adapter.0.weight"] = (1.0 + 0.1 * torch.randn(cfg.d, generator=g)).to(torch.bfloat16).float()
        w[f"{pre}.adapter.0.bias"] = (0.1 * torch.randn(cfg.d, generator=g)).to(torch.bfloat16).float()
        w[f"{pre}.adapter_scale"] = torch.tensor([0.5 + 0.25 * l])
    model, _ = E.build(monkeypatch, cfg, w, 16, freeze_enc=True, adapter_config={"mlp": dict(mlp, add_layernorm=True)})
    model.eval()
    emb = (torch.randn(2, 5, cfg.d, generator=g) * 0.5).to(torch.bfloat16)
    toks = model.generate(emb, max_steps=6, temperature=0.0, decode=False)
    x = emb
    for i in range(6):   # reference loop without a cache: re-run the whole sequence, take the last position's argmax
        logits = model.lm(inputs_embeds=x).logits[:, -1, :].float()
        nxt = logits.argmax(-1)
        assert torch.equal(toks[:, 5 + i], nxt), i
        x = torch.cat([x, model.lm.transformer.wte(nxt[:, None])], 1)
