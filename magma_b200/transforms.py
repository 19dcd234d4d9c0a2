"""Image preprocessing — drop-in for magma/transforms.py (`get_transforms`, `clip_preprocess`, `pad_to_size_tensor`).
Host-side PIL / torch code: nothing here is on the accelerated path, it only has to hand the
encoder the same [1, 3, R, R] tensor the reference does.

`clip_preprocess` is written directly on PIL + torch (resize the short side with bicubic resampling, centre crop or
letterbox, RGB, scale to [0, 1], CLIP mean/std) and is held bit-for-bit to the reference's torchvision pipeline
(magma/transforms.py:139-153) by tests/test_preprocess_cpu.py on fixtures generated from the reference itself. The
random-crop training augmentation for non-CLIP encoders (transforms.py:47-95) is rebuilt on torchvision's primitives
when torchvision is importable."""
import random

import numpy as np
import torch
import torch.nn.functional as F
from PIL import Image, ImageOps

CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)
_BICUBIC = getattr(Image, "Resampling", Image).BICUBIC
_LANCZOS = getattr(Image, "Resampling", Image).LANCZOS  # what PIL.Image.ANTIALIAS named (transforms.py:117)


def maybe_add_batch_dim(t):
    return t.unsqueeze(0) if t.ndim == 3 else t


def _to_unit_tensor(img: Image.Image) -> torch.Tensor:
    """PIL RGB -> float32 [3, H, W] in [0, 1] (what torchvision's ToTensor yields for 8-bit images)."""
    a = np.asarray(img, dtype=np.uint8)
    if a.ndim == 2:
        a = a[:, :, None]
    return torch.from_numpy(a.copy()).permute(2, 0, 1).to(torch.float32).div(255.0)


def _resize_short_side(img: Image.Image, n_px: int) -> Image.Image:
    w, h = img.size
    if (w <= h and w == n_px) or (h <= w and h == n_px):
        return img
    if w < h:
        new_w, new_h = n_px, int(n_px * h / w)
    else:
        new_w, new_h = int(n_px * w / h), n_px
    return img.resize((new_w, new_h), _BICUBIC)


def _center_crop(img: Image.Image, n_px: int) -> Image.Image:
    w, h = img.size
    if w < n_px or h < n_px:  # smaller than the crop: pad symmetrically with black first
        pl, pt = max((n_px - w) // 2, 0), max((n_px - h) // 2, 0)
        pr, pb = max((n_px - w + 1) // 2, 0), max((n_px - h + 1) // 2, 0)
        img = ImageOps.expand(img, (pl, pt, pr, pb))
        w, h = img.size
    top, left = int(round((h - n_px) / 2.0)), int(round((w - n_px) / 2.0))
    return img.crop((left, top, left + n_px, top + n_px))


def pad_img(desired_size):
    """Letterbox: scale the long side to desired_size and paste centred on black (transforms.py:110-128)."""

    def fn(im):
        ratio = float(desired_size) / max(im.size)
        new_size = tuple(int(x * ratio) for x in im.size)
        canvas = Image.new("RGB", (desired_size, desired_size))
        canvas.paste(im.resize(new_size, _LANCZOS),
                     ((desired_size - new_size[0]) // 2, (desired_size - new_size[1]) // 2))
        return canvas

    return fn


def clip_preprocess(n_px, use_pad=False):
    """PIL image -> [1, 3, n_px, n_px] float32, CLIP-normalised (magma/transforms.py:139-153)."""
    mean = torch.tensor(CLIP_MEAN).view(3, 1, 1)
    std = torch.tensor(CLIP_STD).view(3, 1, 1)
    fit = pad_img(n_px) if use_pad else (lambda im: _center_crop(im, n_px))

    def transform(image):
        image = fit(_resize_short_side(image, n_px)).convert("RGB")
        return maybe_add_batch_dim((_to_unit_tensor(image) - mean) / std)

    return transform


def pad_to_size(x, size=256):
    """Pad a PIL image with black up to size x size, centred (transforms.py:8-18)."""
    dw, dh = size - x.size[0], size - x.size[1]
    return ImageOps.expand(x, (dw // 2, dh // 2, dw - dw // 2, dh - dh // 2))


def pad_to_size_tensor(x, size=256):
    """Pad a [c, h, w] tensor up to size on both spatial dims; an odd remainder goes in front (transforms.py:21-40)."""
    pads = []
    for dim in (2, 1):  # F.pad takes the last dimension first
        off = size - x.shape[dim]
        half = max(off // 2, 0)
        pads += [half + (off % 2), half]
    return F.pad(x, pad=(*pads, 0, 0))


class RandCropResize:
    """Random square crop, random resize to [9/8, 12/8] x target, random crop to target — the augmentation of
    arXiv:2102.12092 used for non-CLIP encoders (transforms.py:43-64)."""

    def __init__(self, target_size):
        self.target_size = target_size

    def __call__(self, img):
        from torchvision import transforms as T

        img = pad_to_size(img, self.target_size)
        d_min = min(img.size)
        img = T.RandomCrop(size=d_min)(img)
        t_lo = min(d_min, round(9 / 8 * self.target_size))
        t_hi = min(d_min, round(12 / 8 * self.target_size))
        img = T.Resize(random.randint(t_lo, t_hi + 1))(img)
        if min(img.size) < 256:
            img = T.Resize(256)(img)
        return T.RandomCrop(size=self.target_size)(img)


def get_transforms(image_size, encoder_name, input_resolution=None, use_extra_transforms=False):
    """magma/transforms.py:67-92: CLIP encoders get CLIP's own preprocessing at the encoder's input resolution; other
    encoders the random-crop augmentation at `image_size`."""
    if "clip" in encoder_name:
        assert input_resolution is not None
        return clip_preprocess(input_resolution)
    from torchvision import transforms as T

    steps = [lambda img: img if img.mode == "RGB" else img.convert("RGB"), RandCropResize(image_size),
             T.RandomHorizontalFlip(p=0.5)]
    if use_extra_transforms:
        steps.append(T.ColorJitter(0.1, 0.1, 0.1, 0.05))
    steps += [lambda img: _to_unit_tensor(img), maybe_add_batch_dim]
    return T.Compose(steps)
