"""CPU oracle of the multi-crop augmentation (datasets/build.py:DataAugmentationDINO, utils.py:GaussianBlur/Solarization).

``apply(image, p, size)`` runs one crop's parameter record (esvit_b200.augment.PARAM_FIELDS) through the same Pillow
and torchvision functional calls the reference's transforms make, so the sampled record plus this oracle reproduce the
reference crop.  Nothing here needs the reference tree; ``reference_transform()`` extracts the unmodified reference
class for the fixture generator and bench_augment.py.
"""
from __future__ import annotations

import ast
import hashlib
import os
import random
import types

import numpy as np
import torch
from PIL import Image, ImageFilter, ImageOps
from torchvision import transforms
from torchvision.transforms import functional as F

MEAN = (0.485, 0.456, 0.406)
STD = (0.229, 0.224, 0.225)
_NORMALIZE = transforms.Compose([transforms.ToTensor(), transforms.Normalize(MEAN, STD)])


def apply_u8(image: Image.Image, p, size: int) -> np.ndarray:
    """one crop before ToTensor: uint8 [size, size, 3]"""
    p = [float(v) for v in p]
    top, left, h, w, flip, jitter = (int(v) for v in p[:6])
    perm = [int(v) for v in p[6:10]]
    b, c, s, hue, gray, blur, radius, solar = p[10:18]
    img = F.resized_crop(image, top, left, h, w, [size, size], transforms.InterpolationMode.BICUBIC)  # RandomResizedCrop
    if flip:
        img = F.hflip(img)
    if jitter:  # ColorJitter.forward
        for fn in perm:
            if fn == 0:
                img = F.adjust_brightness(img, b)
            elif fn == 1:
                img = F.adjust_contrast(img, c)
            elif fn == 2:
                img = F.adjust_saturation(img, s)
            else:
                img = F.adjust_hue(img, hue)
    if gray:  # RandomGrayscale
        img = F.rgb_to_grayscale(img, num_output_channels=3)
    if blur:  # utils.GaussianBlur
        img = img.filter(ImageFilter.GaussianBlur(radius=radius))
    if solar:  # utils.Solarization
        img = ImageOps.solarize(img)
    return np.asarray(img, dtype=np.uint8).copy()


def normalize(u8: np.ndarray) -> torch.Tensor:
    """ToTensor + Normalize of a uint8 HWC crop: fp32 [3, S, S]"""
    return _NORMALIZE(Image.fromarray(np.ascontiguousarray(u8), "RGB"))


def digest(u8) -> str:
    """SHA-256 of a uint8 HWC crop's bytes: how the fixture pins every value of a crop without storing it"""
    return hashlib.sha256(np.ascontiguousarray(np.asarray(u8, dtype=np.uint8)).tobytes()).hexdigest()


def apply(image: Image.Image, p, size: int) -> torch.Tensor:
    return normalize(apply_u8(image, p, size))


def synthetic_image(seed: int, height: int, width: int) -> np.ndarray:
    """a photo-like uint8 [H, W, 3] image from integer numpy ops alone: a coarse random grid upsampled by integer
    bilinear interpolation (smooth regions and edges), plus seeded noise, with saturated and grey patches"""
    rng = np.random.default_rng(seed)
    gh, gw = max(2, height // 37), max(2, width // 41)
    grid = rng.integers(0, 256, (gh + 1, gw + 1, 3), dtype=np.int64)
    ys = np.arange(height, dtype=np.int64) * gh * 256 // max(height - 1, 1)
    xs = np.arange(width, dtype=np.int64) * gw * 256 // max(width - 1, 1)
    y0, x0 = np.minimum(ys >> 8, gh - 1), np.minimum(xs >> 8, gw - 1)
    fy, fx = (ys - (y0 << 8))[:, None, None], (xs - (x0 << 8))[None, :, None]
    g00, g01 = grid[y0][:, x0], grid[y0][:, x0 + 1]
    g10, g11 = grid[y0 + 1][:, x0], grid[y0 + 1][:, x0 + 1]
    top = g00 * (256 - fx) + g01 * fx
    bot = g10 * (256 - fx) + g11 * fx
    img = (top * (256 - fy) + bot * fy) >> 16
    img = img + rng.integers(-24, 25, img.shape)
    ph, pw = max(1, height // 6), max(1, width // 6)
    img[:ph, :pw] = img[:ph, :pw, :1]                                   # grey: hue and saturation degenerate
    img[-ph:, -pw:, 0] = 255                                           # saturated red channel
    img[-ph:, :pw] = rng.integers(0, 2, (ph, pw, 1)) * 255              # black / white
    return np.clip(img, 0, 255).astype(np.uint8)


def reference_transform(root: str, global_crops_scale=(0.4, 1.0), local_crops_scale=(0.05, 0.4),
                        local_crops_number=(8,), local_crops_size=(96,)):
    """the unmodified DataAugmentationDINO (datasets/build.py) with utils.GaussianBlur / Solarization, AST-extracted
    from the reference tree at ``root``: datasets/build.py's other imports (TSV datasets, samplers) are not needed"""
    env = {"transforms": transforms, "Image": Image, "ImageFilter": ImageFilter, "ImageOps": ImageOps,
           "random": random, "torch": torch}
    utree = ast.parse(open(os.path.join(root, "utils.py")).read())
    nodes = [n for n in utree.body if isinstance(n, ast.ClassDef) and n.name in ("GaussianBlur", "Solarization")]
    exec(compile(ast.Module(nodes, []), "utils.py", "exec"), env)
    env["utils"] = types.SimpleNamespace(GaussianBlur=env["GaussianBlur"], Solarization=env["Solarization"])
    btree = ast.parse(open(os.path.join(root, "datasets", "build.py")).read())
    nodes = [n for n in btree.body if isinstance(n, ast.ClassDef) and n.name == "DataAugmentationDINO"]
    assert len(nodes) == 1
    exec(compile(ast.Module(nodes, []), "datasets/build.py", "exec"), env)
    return env["DataAugmentationDINO"](global_crops_scale, local_crops_scale, local_crops_number, local_crops_size)
