"""CPU oracle of the evaluation transforms (eval_linear.py: train_transform / val_transform, eval_knn.py: transform).

``apply_eval_u8(image, record)`` runs one evaluation record (esvit_b200.augment.EVAL_FIELDS) through the same Pillow and
torchvision functional calls the reference's transforms make, so the record plus this oracle reproduce the reference
crop; ToTensor + Normalize is oracle.augment.normalize.  ``reference_eval_transforms()`` extracts the unmodified
transforms for the fixture generator and bench_eval.py.
"""
from __future__ import annotations

import ast
import os

import numpy as np
from PIL import Image
from torchvision import transforms
from torchvision.transforms import functional as F


def apply_eval_u8(image: Image.Image, r) -> np.ndarray:
    """one evaluation record before ToTensor: crop the box, resize it to (resize_h, resize_w) with the record's Pillow
    filter (F.resize leaves an image of that size alone, as Resize does), keep the S x S window, flip: uint8 [S, S, 3]"""
    top, left, h, w, rh, rw, oy, ox, S, flip, interp = (int(v) for v in r)
    mode = {2: transforms.InterpolationMode.BILINEAR, 3: transforms.InterpolationMode.BICUBIC}[interp]
    img = F.resized_crop(image, top, left, h, w, [rh, rw], mode)
    img = F.crop(img, oy, ox, S, S)
    if flip:
        img = F.hflip(img)
    return np.asarray(img, dtype=np.uint8).copy()


def reference_eval_transforms(root: str) -> dict:
    """the unmodified evaluation transforms, AST-extracted from the reference tree at ``root``: ``train_transform`` and
    ``val_transform`` from eval_linear() in eval_linear.py, ``transform`` from extract_feature_pipeline() in eval_knn.py
    (the scripts' other imports, models and distributed set-up are not needed)"""
    out = {}
    for script, fn, names in (("eval_linear.py", "eval_linear", ("train_transform", "val_transform")),
                              ("eval_knn.py", "extract_feature_pipeline", ("transform",))):
        tree = ast.parse(open(os.path.join(root, script)).read())
        body = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == fn]
        assert len(body) == 1, (script, fn)
        nodes = [n for n in body[0].body if isinstance(n, ast.Assign) and len(n.targets) == 1
                 and isinstance(n.targets[0], ast.Name) and n.targets[0].id in names]
        assert sorted(n.targets[0].id for n in nodes) == sorted(names), (script, fn)
        env = {"pth_transforms": transforms}
        exec(compile(ast.Module(nodes, []), script, "exec"), env)
        out.update({n: env[n] for n in names})
    return out
