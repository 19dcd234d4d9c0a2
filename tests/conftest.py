import os
import sys

import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA (sm_90 / H100) device; run with `-m gpu`")
    config.addinivalue_line("markers", "timeout: per-test time limit (pytest-timeout; ignored when the plugin is absent)")


def _usable_cuda():
    try:
        import torch

        if not torch.cuda.is_available():
            return False
        torch.empty(1, device="cuda").fill_(1.0)  # availability alone is not enough (driver / device mismatch)
        torch.cuda.synchronize()
        return True
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    """`pytest tests` on a box without a usable CUDA device skips the `gpu` tests instead of failing in the driver."""
    gpu_items = [it for it in items if it.get_closest_marker("gpu")]
    if not gpu_items or _usable_cuda():
        return
    skip = pytest.mark.skip(reason="no usable CUDA device (gpu-marked test)")
    for it in gpu_items:
        it.add_marker(skip)


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


def oracle_cfg_from_record(rec):
    from oracle.magma_oracle import OracleConfig

    lm, vit = rec["lm"], rec["vit"]
    ac = rec["adapter_config"] or {}
    return OracleConfig(
        d=lm["n_embd"], n_layer=lm["n_layer"], n_head=lm["n_head"], rotary_dim=lm["rotary_dim"],
        vocab=rec["weights"]["lm.lm_head.weight"].shape[0],
        mlp_adapter=ac.get("mlp"), attn_adapter=ac.get("attention"), image_seq_len=2,
        enc_out_dim=vit["projection_dim"], use_image_embed_layernorm=True, vit_width=vit["hidden_size"],
        vit_layers=vit["num_hidden_layers"], vit_heads=vit["num_attention_heads"], vit_patch=vit["patch_size"],
        vit_image=vit["image_size"], vit_mlp=vit["intermediate_size"], eos_token=rec["eos"], image_token=rec["cls"])


@pytest.fixture
def emul_ops(monkeypatch):
    """Host-side dry run: point magma_b200/ops.py at oracle/cabi_emul.cpp (the CPU emulation of the primitive C-ABI
    operators) for the duration of ONE test, so the Python schedules built on ops.* (image_prefix.py, adapters.py, the
    conv trunk, arena.py) run on CPU tensors and can be held to the oracle. Test infrastructure only: outside this
    fixture `magma_b200._lib.lib()` loads the CUDA library or raises."""
    import ctypes

    from magma_b200 import _lib, ops
    from oracle import build_emul

    L = ctypes.CDLL(build_emul.build())
    L.mb200_last_error.restype = ctypes.c_char_p
    L.mb200_version.restype = ctypes.c_int
    L.mb200_launch_count.restype = ctypes.c_longlong
    for fn in ("mb200_vit_workspace_bytes", "mb200_vit_train_workspace_bytes", "mb200_gptj_sched_infer_workspace_bytes",
               "mb200_gptj_sched_workspace_bytes"):
        getattr(L, fn).restype = ctypes.c_size_t
    monkeypatch.setattr(_lib, "_lib", L)
    monkeypatch.setattr(ops, "_stream", lambda: None)
    return L


@pytest.fixture
def kernel_ops(monkeypatch):
    """magma_b200/ops.py driven by KERNEL SOURCE executed on the CPU (oracle/kernel_host_exec.cpp: the product's .cuh kernel
    fragments compiled as host C++, CUDA thread model emulated) — for the elementwise / reduction operators only; there is
    no GEMM or attention here (wgmma / TMA code cannot run on a CPU)."""
    import ctypes

    from magma_b200 import _lib, ops
    from oracle import build_emul

    L = ctypes.CDLL(build_emul.build_kernel_exec())
    L.mb200_last_error.restype = ctypes.c_char_p
    L.mb200_version.restype = ctypes.c_int
    monkeypatch.setattr(_lib, "_lib", L)
    monkeypatch.setattr(ops, "_stream", lambda: None)
    return L
