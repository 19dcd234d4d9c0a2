"""Host-side preprocessing (`Magma.preprocess_inputs`, magma/magma.py:176-193): ImageInput and the
CLIP transform are bit-identical to the reference's torchvision pipeline on the golden vectors the reference produced
(oracle/make_golden_preprocess.py)."""
import os

import numpy as np
import pytest
import torch
from PIL import Image

from magma_b200 import transforms as T
from magma_b200.image_input import ImageInput


def _pil(pixels, mode):
    a = pixels.numpy()
    return Image.fromarray(a[:, :, 0] if mode == "L" else a, mode)


def test_clip_preprocess_matches_reference_golden(golden_dir):
    rec = torch.load(os.path.join(golden_dir, "clip_preprocess.pt"), weights_only=False)
    assert len(rec["cases"]) >= 8
    for c in rec["cases"]:
        out = T.clip_preprocess(c["n_px"])(_pil(c["pixels"], c["mode"]))
        assert out.shape == (1, 3, c["n_px"], c["n_px"]) and out.dtype == torch.float32
        assert torch.equal(out, c["out"]), (c["w"], c["h"], c["mode"])
    for c in rec["pad_to_size_tensor"]:
        assert torch.equal(T.pad_to_size_tensor(c["x"], c["size"]), c["out"])


def test_get_transforms_dispatch_and_image_input(tmp_path):
    rng = np.random.default_rng(3)
    img = Image.fromarray(rng.integers(0, 256, (60, 90, 3), dtype=np.uint8), "RGB")
    p = tmp_path / "x.png"
    img.save(p)
    tf = T.get_transforms(256, "clip_vit_large", input_resolution=224)   # "clip" in the name -> CLIP preprocessing
    a = ImageInput(str(p)).get_transformed_image(tf)
    b = ImageInput(img).get_transformed_image(tf)
    assert a.shape == (1, 3, 224, 224) and torch.equal(a, b)
    with pytest.raises(AssertionError):
        T.get_transforms(256, "clip", input_resolution=None)             # transforms.py:71
    with pytest.raises(Exception, match="Could not retrieve image from url"):
        ImageInput("http://127.0.0.1:9/none.png")                        # image_input.py:19-20 (no network here)
    aug = T.get_transforms(64, "nfresnet50")(img)                        # non-CLIP: random-crop augmentation
    assert aug.shape == (1, 3, 64, 64) and 0.0 <= float(aug.min()) and float(aug.max()) <= 1.0
    letter = T.clip_preprocess(48, use_pad=True)(img)
    assert letter.shape == (1, 3, 48, 48)
