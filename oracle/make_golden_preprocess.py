"""TEST INFRASTRUCTURE — golden vectors for the host-side image preprocessing, produced by the
REFERENCE's own magma/transforms.py (loaded from the checkout named by MAGMA_REFERENCE_ROOT; it only needs torchvision +
PIL). Run once; the fixture travels with the repo: tests/golden/clip_preprocess.pt."""
import importlib.util
import os

import numpy as np
import torch
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = [  # (width, height, mode, n_px)
    (50, 37, "RGB", 32), (37, 50, "RGB", 32), (32, 32, "RGB", 32), (20, 90, "RGB", 32), (64, 48, "L", 32),
    (48, 64, "RGBA", 32), (31, 17, "RGB", 32), (100, 75, "RGB", 48), (200, 120, "RGB", 64),
]


def synthetic_image(w, h, mode, seed):
    rng = np.random.default_rng(seed)
    ch = {"RGB": 3, "L": 1, "RGBA": 4}[mode]
    arr = rng.integers(0, 256, (h, w, ch), dtype=np.uint8)
    return arr


def to_pil(arr, mode):
    return Image.fromarray(arr[:, :, 0] if mode == "L" else arr, mode)


def main():
    spec = importlib.util.spec_from_file_location("ref_transforms", os.path.join(os.environ["MAGMA_REFERENCE_ROOT"], "magma",
                                                                              "transforms.py"))
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    rec = {"cases": [], "pad_to_size_tensor": []}
    for i, (w, h, mode, n) in enumerate(CASES):
        arr = synthetic_image(w, h, mode, 100 + i)
        out = ref.clip_preprocess(n)(to_pil(arr, mode))
        rec["cases"].append({"w": w, "h": h, "mode": mode, "n_px": n, "pixels": torch.from_numpy(arr), "out": out})
    g = torch.Generator().manual_seed(0)
    for shape in [(3, 20, 25), (3, 32, 31), (1, 7, 32), (3, 32, 32)]:
        x = torch.randn(*shape, generator=g)
        rec["pad_to_size_tensor"].append({"x": x, "size": 32, "out": ref.pad_to_size_tensor(x, 32)})
    path = os.path.join(ROOT, "tests", "golden", "clip_preprocess.pt")
    torch.save(rec, path)
    print(path, os.path.getsize(path))


if __name__ == "__main__":
    main()
