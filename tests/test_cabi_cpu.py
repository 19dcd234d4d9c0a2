"""CPU tests: the C-ABI library builds, loads, and exports every symbol include/magma_b200.h declares; the product
path refuses to run without a CUDA sm_90 device (no CPU fallback)."""
import ctypes
import os
import re

import pytest

from conftest import ROOT


@pytest.fixture(scope="module")
def lib():
    from magma_b200 import build, _lib

    build.build()
    return _lib.lib()


def _declared():
    hdr = open(os.path.join(ROOT, "include", "magma_b200.h")).read()
    return sorted(set(re.findall(r"\b(mb200_[a-z0-9_]+)\s*\(", hdr)))


def test_library_exports_every_declared_symbol(lib):
    names = _declared()
    assert len(names) >= 30
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/magma_b200.h but not exported"


def test_python_symbol_table_matches_header():
    from magma_b200 import _lib

    assert sorted(_lib.EXPORTED_SYMBOLS) == _declared()


def test_version_and_error_string(lib):
    assert lib.mb200_version() == 100
    assert isinstance(lib.mb200_last_error(), bytes)


def test_struct_sizes_match_the_c_header():
    """ctypes mirrors must have the C layout (a mismatch would silently corrupt pointers)."""
    import subprocess
    import tempfile

    from magma_b200 import _lib

    src = r'''
#include <stdio.h>
#include "magma_b200.h"
int main(void){printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu\n", sizeof(mb200_operand), sizeof(mb200_gemm_args),
 sizeof(mb200_vit_layer), sizeof(mb200_vit_model), sizeof(mb200_vit_layer_grads), sizeof(mb200_vit_grads),
 sizeof(mb200_adapter_ex), sizeof(mb200_gptj_layer_ex), sizeof(mb200_gptj_model_ex));return 0;}
'''
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "s.c")
        open(c, "w").write(src)
        exe = os.path.join(d, "s")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        sizes = [int(x) for x in subprocess.check_output([exe]).split()]
    want = [ctypes.sizeof(t) for t in (_lib.Operand, _lib.GemmArgs, _lib.VitLayerC, _lib.VitModelC, _lib.VitLayerGradsC,
                                       _lib.VitGradsC, _lib.AdapterExC, _lib.GptjLayerExC, _lib.GptjModelExC)]
    assert sizes == want


def test_no_cpu_fallback(lib):
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from magma_b200 import _lib

    assert lib.mb200_check_device() == -4  # MB200_E_ARCH
    g = _lib.GemmArgs()
    g.M = g.N = g.K = 64
    g.nb0 = g.nb1 = 1
    rc = lib.mb200_gemm(ctypes.byref(g), None)
    assert rc != 0
    assert b"" != lib.mb200_last_error()
    from magma_b200.config import MultimodalConfig
    from magma_b200.magma import Magma

    with pytest.raises(RuntimeError, match="no CPU path"):
        Magma(MultimodalConfig(batch_size=1, train_steps=1), device="cpu")


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    from magma_b200 import _lib

    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", str(tmp_path / "nope.so"))
    with pytest.raises(_lib.MB200Error, match="not found"):
        _lib.lib()


def test_config_loads_reference_style_yaml(tmp_path):
    from magma_b200.config import MultimodalConfig

    y = tmp_path / "c.yml"
    y.write_text("""{
    encoder_name: 'clip_vit_large',
    adapter_config: {"mlp": {"adapter_type": "normal", "downsample_factor": 4}},
    freeze_img_encoder: true, batch_size: 256, train_steps: 150000, lr: 8.0e-4, min_lr: 0.0,
    lr_decay_iters: 300000, use_image_embed_layernorm: true, image_embed_dropout_prob: 0.1, image_size: 224,
    gradient_accumulation_steps: 8, zero_stage: 2, gradient_clipping: 1.0, }""")
    c = MultimodalConfig.from_yml(str(y))
    assert c.adapter_config["mlp"]["downsample_factor"] == 4 and c.image_seq_len == 2
    assert c.lr_at(0) == 0.0 and abs(c.lr_at(100) - 8e-4) < 1e-12 and c.lr_at(300000) == 0.0
    with pytest.raises(TypeError):
        MultimodalConfig(batch_size=1, train_steps=1, dataset_type="new")  # unknown keys rejected like the reference


def test_shipped_and_reference_configs_load():
    """configs/*.yml of this repo and the reference's own MAGMA_v1.yml (stored under tests/golden/) load through the
    same schema (magma/config.py:20-94)."""
    from magma_b200.config import MultimodalConfig

    c = MultimodalConfig.from_yml(os.path.join(ROOT, "configs", "MAGMA_v1_vit.yml"))
    assert c.encoder_name == "clip_vit_large" and c.freeze_img_encoder and c.seq_len == 128
    t = MultimodalConfig.from_yml(os.path.join(ROOT, "configs", "MAGMA_v1_vit_trainable_encoder.yml"))
    assert not t.freeze_img_encoder and t.image_enc_lr == 2.0e-6
    r = MultimodalConfig.from_yml(os.path.join(ROOT, "tests", "golden", "MAGMA_v1.yml"))
    assert r.encoder_name == "clip_resnet_large" and not r.freeze_img_encoder and r.image_enc_lr == 2.0e-6
    assert r.adapter_config == {"mlp": {"adapter_type": "normal", "downsample_factor": 4}}


def test_top_level_exports_mirror_the_reference_package():
    """`from magma import Magma, MultimodalConfig, get_gptj, ...` (magma/__init__.py) works with the package name swapped."""
    import magma_b200
    from magma_b200 import ImageInput, Magma, MultimodalConfig, collate_fn, get_gptj, get_transforms, train_step  # noqa: F401

    for name in ("count_parameters", "is_main", "cycle", "get_tokenizer", "save_model", "load_model", "print_main",
                 "configure_param_groups", "eval_step"):
        assert callable(getattr(magma_b200, name)), name
    with pytest.raises(AttributeError):
        magma_b200.wandb_log  # logging glue is out of scope
