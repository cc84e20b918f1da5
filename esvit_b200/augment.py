"""Device-side multi-crop augmentation: the reference's DataAugmentationDINO (datasets/build.py) on sm_90a kernels.

The reference builds every crop on CPU DataLoader workers in Pillow.  Here the work is split in two:

* in the workers, ``MultiCropParams`` (a drop-in for ``DataAugmentationDINO(...)`` as a Dataset transform) returns the
  decoded image as a uint8 HWC tensor plus a float64 record of every random parameter of every crop, drawn in the
  reference's order from the same torch and Python RNGs (torchvision's own ``get_params`` where one exists);
  ``collate_multicrop`` packs a batch of images of any sizes into one uint8 buffer with 64-bit offsets;
* on the GPU, ``MultiCropAugment`` applies the parameters with kernels that restate Pillow's arithmetic (csrc/augment.cu)
  and returns the ``2 + sum(local_crops_number)`` fp32 ``[B, 3, S, S]`` batches in the reference's collate order.

The evaluation transforms of eval_linear.py and eval_knn.py are split the same way: ``LinearTrainParams`` (the linear
probe's RandomResizedCrop + RandomHorizontalFlip) and ``CenterCropParams`` (Resize(256, bicubic) + CenterCrop(224), the
validation and k-NN transform) draw one record per image on the workers, and ``EvalAugment`` applies a collated batch of
them on the GPU, returning one fp32 ``[B, 3, S, S]`` tensor.

Not differentiable; no host synchronisation.  DESIGN.md §4.7 lists the Pillow arithmetic and its exactness.
"""
from __future__ import annotations

import ctypes
import random
from typing import List, NamedTuple, Optional, Sequence

import numpy as np
import torch
from torchvision import transforms as T

from . import _lib

# one float64 row per crop; the field order is the kernel's (csrc/augment.cu, enum P_*)
PARAM_FIELDS = ("top", "left", "height", "width", "flip", "jitter", "perm0", "perm1", "perm2", "perm3", "brightness",
                "contrast", "saturation", "hue", "grayscale", "blur", "radius", "solarize")
NPARAM = len(PARAM_FIELDS)
_F = {k: i for i, k in enumerate(PARAM_FIELDS)}
NMETA = 9          # int64 per-crop geometry row (csrc/augment.cu, enum M_*)
MAX_SIZE = 241     # largest output side: the colour kernel keeps a crop (3 S^2) and a blur plane (S^2) in shared memory
IMAGENET_MEAN = (0.485, 0.456, 0.406)
IMAGENET_STD = (0.229, 0.224, 0.225)
# one float64 row per image for the evaluation transforms; the field order is the kernels' (csrc/augment.cu, enum R_*):
# crop box, size it is resized to, S x S output window of that resize, flip, Pillow resample code
EVAL_FIELDS = ("top", "left", "height", "width", "resize_h", "resize_w", "win_top", "win_left", "size", "flip",
               "interpolation")
NEVAL = len(EVAL_FIELDS)
_E = {k: i for i, k in enumerate(EVAL_FIELDS)}
NEMETA = 8         # int64 per-image geometry row of the evaluation kernels (csrc/augment.cu, enum E_*)
PIL_BILINEAR, PIL_BICUBIC = 2, 3
_SUPPORT = {PIL_BILINEAR: 1.0, PIL_BICUBIC: 2.0}  # Pillow's filter supports


def _as_u8(image) -> torch.Tensor:
    """a PIL image or uint8 HWC array / tensor as a contiguous uint8 [H, W, 3] tensor"""
    img = torch.from_numpy(np.array(image, dtype=np.uint8, copy=True)) if not isinstance(image, torch.Tensor) else image
    if img.dtype != torch.uint8 or img.dim() != 3 or img.shape[2] != 3:
        raise ValueError(f"expected a uint8 [H, W, 3] RGB image, got {tuple(img.shape)} {img.dtype}")
    if img.shape[0] == 0 or img.shape[1] == 0:
        raise ValueError("empty image")
    return img.contiguous()


def _sizes(local_crops_number, local_crops_size) -> tuple:
    number = [int(n) for n in (local_crops_number if isinstance(local_crops_number, (list, tuple))
                               else [local_crops_number])]
    size = [int(s) for s in (local_crops_size if isinstance(local_crops_size, (list, tuple)) else [local_crops_size])]
    if len(size) != len(number):
        raise ValueError(f"local_crops_size {size} and local_crops_number {number} differ in length")
    return number, size


class MultiCropParams:
    """Worker-side replacement of ``DataAugmentationDINO(global_crops_scale, local_crops_scale, local_crops_number,
    local_crops_size)``: ``__call__(image)`` returns ``(uint8 [H, W, 3] tensor, float64 [ncrops, NPARAM] parameters)``.

    ``image`` is what the reference's loader passes (``Image.open(path).convert('RGB')``) or a uint8 HWC array.
    ``sample(height, width)`` draws the parameters alone, consuming the torch and Python RNGs exactly as the
    reference's transforms do for an image of that size."""

    def __init__(self, global_crops_scale, local_crops_scale, local_crops_number, local_crops_size=96,
                 global_crops_size: int = 224):
        self.local_crops_number, self.local_crops_size = _sizes(local_crops_number, local_crops_size)
        self.global_crops_size = int(global_crops_size)
        self.global_crop = T.RandomResizedCrop(self.global_crops_size, scale=global_crops_scale)
        self.local_crops = [T.RandomResizedCrop(s, scale=local_crops_scale) for s in self.local_crops_size]
        self.jitter = T.ColorJitter(brightness=0.4, contrast=0.4, saturation=0.2, hue=0.1)

    @property
    def sizes(self) -> List[int]:
        """output side of every crop, in the reference's order"""
        out = [self.global_crops_size] * 2
        for n, s in zip(self.local_crops_number, self.local_crops_size):
            out += [s] * n
        return out

    def _crop(self, dims, rrc, blur_p: float, solarize: Optional[float]) -> list:
        # RandomResizedCrop, then flip_and_color_jitter, GaussianBlur(p) and Solarization (utils.py)
        i, j, h, w = T.RandomResizedCrop.get_params(dims, rrc.scale, rrc.ratio)
        flip = bool(torch.rand(1) < 0.5)
        jitter = not bool(0.8 < torch.rand(1))  # RandomApply(p=0.8)
        perm, b, c, s, hue = [0, 1, 2, 3], 1.0, 1.0, 1.0, 0.0
        if jitter:
            fn_idx, b, c, s, hue = T.ColorJitter.get_params(self.jitter.brightness, self.jitter.contrast,
                                                            self.jitter.saturation, self.jitter.hue)
            perm = [int(k) for k in fn_idx]
        gray = bool(torch.rand(1) < 0.2)
        blur = random.random() <= blur_p
        radius = random.uniform(0.1, 2.0) if blur else 0.0
        solar = solarize is not None and random.random() < solarize
        return [i, j, h, w, flip, jitter] + perm + [b, c, s, hue, gray, blur, radius, solar]

    def sample(self, height: int, width: int) -> torch.Tensor:
        dims = torch.empty((3, int(height), int(width)), device="meta")  # get_params reads the size only
        rows = [self._crop(dims, self.global_crop, 1.0, None), self._crop(dims, self.global_crop, 0.1, 0.2)]
        for n, rrc in zip(self.local_crops_number, self.local_crops):
            rows += [self._crop(dims, rrc, 0.5, None) for _ in range(n)]
        return torch.tensor(rows, dtype=torch.float64)

    def __call__(self, image):
        img = _as_u8(image)
        return img, self.sample(img.shape[0], img.shape[1])


class MultiCropBatch(NamedTuple):
    """A collated batch: pixels uint8 [sum H*W*3] (images back to back, HWC), index int64 [B, 3] (byte offset, H, W),
    params float64 [B, ncrops, NPARAM]."""
    pixels: torch.Tensor
    index: torch.Tensor
    params: torch.Tensor

    def pin_memory(self):
        """DataLoader(pin_memory=True) calls this in its pinning thread"""
        return MultiCropBatch(self.pixels.pin_memory(), self.index, self.params.pin_memory())


def collate_multicrop(batch, pin_memory: bool = False):
    """collate_fn for a Dataset whose transform is MultiCropParams, LinearTrainParams or CenterCropParams:
    ``[((image, params), target), ...]`` -> ``(MultiCropBatch, targets)``.  One host -> device copy of ``pixels``
    then carries the step's source images."""
    imgs = [item[0][0] for item in batch]
    params = [item[0][1] for item in batch]
    targets = torch.tensor([int(item[1]) for item in batch], dtype=torch.int64)
    for im in imgs:
        if im.dtype != torch.uint8 or im.dim() != 3 or im.shape[2] != 3 or im.shape[0] == 0 or im.shape[1] == 0:
            raise ValueError(f"expected non-empty uint8 [H, W, 3] images, got {tuple(im.shape)} {im.dtype}")
    nbytes = torch.tensor([im.numel() for im in imgs], dtype=torch.int64)
    index = torch.stack([torch.cumsum(nbytes, 0) - nbytes,
                         torch.tensor([im.shape[0] for im in imgs], dtype=torch.int64),
                         torch.tensor([im.shape[1] for im in imgs], dtype=torch.int64)], 1)
    pixels = torch.empty(int(nbytes.sum()), dtype=torch.uint8, pin_memory=pin_memory)
    for im, off, n in zip(imgs, index[:, 0].tolist(), nbytes.tolist()):
        pixels[off:off + n] = im.reshape(-1)
    par = torch.stack(params).to(torch.float64)
    if pin_memory:
        par = par.pin_memory()
    return MultiCropBatch(pixels, index, par), targets


def _p(t: torch.Tensor):
    return ctypes.c_void_p(t.data_ptr())


def _device_and_norm(mean, std, device):
    """the module's CUDA device and Normalize's fp32 (mean[3], std[3]) on it, as torchvision makes them"""
    dev = torch.device(device if device is not None else "cuda")
    dev = torch.device("cuda", torch.cuda.current_device()) if dev.index is None else dev
    norm = torch.cat([torch.as_tensor(mean, dtype=torch.float32), torch.as_tensor(std, dtype=torch.float32)])
    if norm.numel() != 6:
        raise ValueError("mean and std need three values each")
    return dev, norm.to(dev)


def _validate_pixels(batch, device):
    """checks a collated batch's pixel buffer and image index; returns (pixels, index, params)"""
    if not isinstance(batch, tuple) or len(batch) != 3:
        raise ValueError("expected a MultiCropBatch (pixels, index, params)")
    pixels, index, params = batch
    if not all(isinstance(t, torch.Tensor) for t in batch):
        raise ValueError("MultiCropBatch fields must be tensors")
    if pixels.dtype != torch.uint8 or pixels.dim() != 1 or not pixels.is_contiguous():
        raise ValueError(f"pixels must be a contiguous 1-D uint8 tensor, got {pixels.dtype} {tuple(pixels.shape)}")
    if pixels.is_cuda and pixels.device != device:
        raise ValueError(f"pixels are on {pixels.device}, the module on {device}")
    if index.dtype != torch.int64 or index.dim() != 2 or index.shape[1] != 3 or index.is_cuda:
        raise ValueError("index must be a host int64 [B, 3] tensor (offset, H, W)")
    off, H, W = index[:, 0], index[:, 1], index[:, 2]
    if bool((H < 1).any() or (W < 1).any()):
        raise ValueError("empty image in the batch")
    if bool((off < 0).any() or (off + H * W * 3 > pixels.numel()).any()):
        raise ValueError("an image lies outside the pixel buffer")
    return pixels, index, params


class MultiCropAugment:
    """The device half of DataAugmentationDINO: ``aug(batch)`` -> ``[2 + sum(local_crops_number)]`` fp32
    ``[B, 3, S, S]`` tensors on ``device`` (globals first, then each local group), on the current stream.

    ``out`` (optional): preallocated contiguous fp32 tensors of those shapes that receive the crops.
    Raises ValueError on a malformed batch (dtype, layout, empty image, parameters out of range)."""

    def __init__(self, local_crops_number=(8,), local_crops_size=(96,), global_crops_size: int = 224,
                 mean: Sequence[float] = IMAGENET_MEAN, std: Sequence[float] = IMAGENET_STD, device=None):
        number, size = _sizes(local_crops_number, local_crops_size)
        self.sizes = [int(global_crops_size)] * 2 + [s for n, s in zip(number, size) for _ in range(n)]
        if any(s < 1 or s > MAX_SIZE for s in self.sizes):
            raise ValueError(f"crop sizes must lie in [1, {MAX_SIZE}], got {sorted(set(self.sizes))}")
        self.device, self.norm = _device_and_norm(mean, std, device)

    def _validate(self, batch: MultiCropBatch):
        pixels, index, params = _validate_pixels(batch, self.device)
        B, nc = index.shape[0], len(self.sizes)
        if B < 1 or B * nc > 65535:
            raise ValueError(f"batch of {B} images x {nc} crops is out of range")
        if params.dtype != torch.float64 or tuple(params.shape) != (B, nc, NPARAM) or params.is_cuda:
            raise ValueError(f"params must be a host float64 [{B}, {nc}, {NPARAM}] tensor, got "
                             f"{params.dtype} {tuple(params.shape)} on {params.device}")
        H, W = index[:, 1], index[:, 2]
        p = params
        if not bool(torch.isfinite(p).all()):
            raise ValueError("non-finite parameter")
        ints = p[..., [_F["top"], _F["left"], _F["height"], _F["width"]] + list(range(_F["perm0"], _F["perm3"] + 1))]
        flags = p[..., [_F["flip"], _F["jitter"], _F["grayscale"], _F["blur"], _F["solarize"]]]
        if bool((ints != ints.round()).any()) or bool(((flags != 0) & (flags != 1)).any()):
            raise ValueError("integer or flag parameter out of range")
        top, left, h, w = (p[..., _F[k]] for k in ("top", "left", "height", "width"))
        if bool((top < 0).any() or (left < 0).any() or (h < 1).any() or (w < 1).any()
                or (top + h > H[:, None]).any() or (left + w > W[:, None]).any()):
            raise ValueError("crop box outside its image")
        perm = p[..., _F["perm0"]:_F["perm3"] + 1]
        if bool((perm.sort(-1).values != torch.arange(4, dtype=torch.float64)).any()):
            raise ValueError("jitter order is not a permutation of 0..3")
        fac = p[..., _F["brightness"]:_F["saturation"] + 1]
        hue = p[..., _F["hue"]]
        if bool((fac < 0).any() or (hue.abs() > 0.5).any()):
            raise ValueError("colour jitter factor out of range")
        S = torch.tensor(self.sizes, dtype=torch.float64)
        rad = p[..., _F["radius"]]
        if bool(((p[..., _F["blur"]] == 1) & ((rad <= 0) | (rad > S))).any()):
            raise ValueError("blur radius out of range (0, S]")

    def __call__(self, batch: MultiCropBatch, out: Optional[List[torch.Tensor]] = None) -> List[torch.Tensor]:
        self._validate(batch)
        pixels, index, params = batch
        B, nc, dev = index.shape[0], len(self.sizes), self.device
        if out is None:
            out = [torch.empty((B, 3, s, s), dtype=torch.float32, device=dev) for s in self.sizes]
        elif len(out) != nc or any(not isinstance(o, torch.Tensor) or o.dtype != torch.float32 or o.device != dev
                                   or tuple(o.shape) != (B, 3, s, s) or not o.is_contiguous()
                                   for o, s in zip(out, self.sizes)):
            raise ValueError(f"out must be {nc} contiguous fp32 [B, 3, S, S] tensors on {dev} with S = {self.sizes}")
        # crop c = k * B + b: crops of one output size are contiguous, in the reference's collate order
        P = params.transpose(0, 1).reshape(nc * B, NPARAM).contiguous()
        S = torch.tensor(self.sizes, dtype=torch.int64).repeat_interleave(B)
        b = torch.arange(B, dtype=torch.int64).repeat(nc)
        h, w = P[:, _F["height"]].to(torch.int64), P[:, _F["width"]].to(torch.int64)
        Sd = S.double()
        # Pillow's ksize = ceil(support) * 2 + 1 with support = 2 * max(1, in / out)
        kh = torch.ceil(2.0 * torch.clamp(w.double() / Sd, min=1.0)).to(torch.int64) * 2 + 1
        kv = torch.ceil(2.0 * torch.clamp(h.double() / Sd, min=1.0)).to(torch.int64) * 2 + 1
        tmp_n = h * S * 3
        coef_n = S * (4 + kh + kv)
        base = torch.tensor([o.data_ptr() for o in out], dtype=torch.int64).repeat_interleave(B)
        meta = torch.stack([index[b, 0], index[b, 1], index[b, 2], S, torch.cumsum(tmp_n, 0) - tmp_n,
                            torch.cumsum(coef_n, 0) - coef_n, kh, kv, base + b * 3 * S * S * 4], 1)
        src = pixels.to(dev, non_blocking=True)
        P_d = P.pin_memory().to(dev, non_blocking=True)
        meta_d = meta.pin_memory().to(dev, non_blocking=True)
        tmp = torch.empty(int(tmp_n.sum()), dtype=torch.uint8, device=dev)
        coef = torch.empty(int(coef_n.sum()), dtype=torch.int32, device=dev)
        stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        n = nc * B
        _lib.call("esvit_augment_coeffs", _p(P_d), _p(meta_d), _p(coef), n, max(self.sizes), stream)
        _lib.call("esvit_augment_resize_h", _p(src), _p(P_d), _p(meta_d), _p(coef), _p(tmp), n,
                  int((h * S).max()), stream)
        k = 0
        while k < nc:  # one launch per run of equal output sizes
            e = k
            while e < nc and self.sizes[e] == self.sizes[k]:
                e += 1
            _lib.call("esvit_augment_color", _p(P_d), _p(meta_d), _p(coef), _p(tmp), _p(self.norm), k * B,
                      (e - k) * B, self.sizes[k], stream)
            k = e
        return out


# ---- evaluation transforms (eval_linear.py, eval_knn.py) --------------------------------------------------------------
class LinearTrainParams:
    """Worker-side replacement of eval_linear.py's ``train_transform`` (RandomResizedCrop(size), RandomHorizontalFlip,
    ToTensor, Normalize): ``__call__(image)`` returns ``(uint8 [H, W, 3] tensor, float64 [NEVAL] record)``.

    ``sample(height, width)`` draws the record alone, consuming the torch RNG as the reference's transforms do:
    ``RandomResizedCrop.get_params`` (including its whole-image centre crop after 10 rejected draws), then
    ``torch.rand(1) < 0.5`` for the flip.  The crop box is resized to ``size`` x ``size`` with Pillow's bilinear filter,
    RandomResizedCrop's default."""

    def __init__(self, size: int = 224, scale=(0.08, 1.0), ratio=(3.0 / 4.0, 4.0 / 3.0)):
        self.size, self.scale, self.ratio = int(size), tuple(scale), tuple(ratio)
        if self.size < 1:
            raise ValueError(f"size must be positive, got {size}")

    def sample(self, height: int, width: int) -> torch.Tensor:
        dims = torch.empty((3, int(height), int(width)), device="meta")  # get_params reads the size only
        i, j, h, w = T.RandomResizedCrop.get_params(dims, self.scale, self.ratio)
        flip = bool(torch.rand(1) < 0.5)
        S = self.size
        return torch.tensor([i, j, h, w, S, S, 0, 0, S, flip, PIL_BILINEAR], dtype=torch.float64)

    def __call__(self, image):
        img = _as_u8(image)
        return img, self.sample(img.shape[0], img.shape[1])


class CenterCropParams:
    """Worker-side replacement of eval_linear.py's ``val_transform`` and eval_knn.py's ``transform``
    (Resize(resize, interpolation=3), CenterCrop(crop), ToTensor, Normalize): ``__call__(image)`` returns
    ``(uint8 [H, W, 3] tensor, float64 [NEVAL] record)``.  No RNG.

    ``sample(height, width)`` computes the geometry as torchvision does: the shorter side becomes ``resize`` and the
    longer ``int(resize * long / short)`` (an image of that size already is left alone, which Pillow's bicubic filter
    at scale 1 reproduces exactly), and the window offsets are ``int(round((R - crop) / 2.0))``, rounding half to
    even."""

    def __init__(self, resize: int = 256, crop: int = 224):
        self.resize, self.crop = int(resize), int(crop)
        if not 1 <= self.crop <= self.resize:
            raise ValueError(f"need 1 <= crop <= resize (CenterCrop would pad), got resize {resize}, crop {crop}")

    def sample(self, height: int, width: int) -> torch.Tensor:
        H, W = int(height), int(width)
        short, long = (W, H) if W <= H else (H, W)
        new_long = int(self.resize * long / short)
        rh, rw = (new_long, self.resize) if W <= H else (self.resize, new_long)
        S = self.crop
        oy, ox = int(round((rh - S) / 2.0)), int(round((rw - S) / 2.0))
        return torch.tensor([0, 0, H, W, rh, rw, oy, ox, S, 0, PIL_BICUBIC], dtype=torch.float64)

    def __call__(self, image):
        img = _as_u8(image)
        return img, self.sample(img.shape[0], img.shape[1])


def _first_last_tap(in_size, out_size, o, support):
    """Pillow's precompute_coeffs bounds of output o: (first input index, one past the last), in float64 as Pillow"""
    scale = in_size / out_size
    fs = torch.clamp(scale, min=1.0)
    sup = support * fs
    center = (o + 0.5) * scale
    lo = torch.clamp((center - sup + 0.5).to(torch.int64), min=0)
    hi = torch.minimum((center + sup + 0.5).to(torch.int64), in_size.to(torch.int64))
    return lo, hi


class EvalAugment:
    """The device half of LinearTrainParams / CenterCropParams: ``aug(batch)`` -> fp32 ``[B, 3, S, S]`` on ``device``,
    on the current stream, bit-identical to the reference transform's ToTensor + Normalize output.  Each record carries
    its filter, so one module serves both transforms; every image of a batch must have the same output side S.

    ``out`` (optional): a preallocated contiguous fp32 ``[B, 3, S, S]`` tensor that receives the crops.
    Raises ValueError on a malformed batch (dtype, layout, empty image, non-integer geometry, bad flag or filter, crop
    box outside its image, window outside the resized image)."""

    def __init__(self, mean: Sequence[float] = IMAGENET_MEAN, std: Sequence[float] = IMAGENET_STD, device=None):
        self.device, self.norm = _device_and_norm(mean, std, device)

    def _validate(self, batch: MultiCropBatch) -> int:
        pixels, index, params = _validate_pixels(batch, self.device)
        B = index.shape[0]
        if B < 1 or B > 65535:
            raise ValueError(f"batch of {B} images is out of range")
        if params.dtype != torch.float64 or tuple(params.shape) != (B, NEVAL) or params.is_cuda:
            raise ValueError(f"params must be a host float64 [{B}, {NEVAL}] tensor, got "
                             f"{params.dtype} {tuple(params.shape)} on {params.device}")
        p = params
        if not bool(torch.isfinite(p).all()) or bool((p != p.round()).any()):
            raise ValueError("evaluation records hold integers only")
        if bool((p.abs() >= 2 ** 31).any()):
            raise ValueError("geometry out of the int32 range")
        top, left, h, w, rh, rw, oy, ox, S, flip, interp = p.unbind(1)
        if bool(((flip != 0) & (flip != 1)).any()):
            raise ValueError("flip must be 0 or 1")
        if bool(((interp != PIL_BILINEAR) & (interp != PIL_BICUBIC)).any()):
            raise ValueError(f"interpolation must be {PIL_BILINEAR} (bilinear) or {PIL_BICUBIC} (bicubic)")
        H, W = index[:, 1].double(), index[:, 2].double()
        if bool((top < 0).any() or (left < 0).any() or (h < 1).any() or (w < 1).any()
                or (top + h > H).any() or (left + w > W).any()):
            raise ValueError("crop box outside its image")
        size = int(S[0])
        if bool((S != size).any()) or size < 1 or size * size >= 2 ** 31:
            raise ValueError(f"one output side S per batch with S^2 < 2^31, got {sorted(set(S.tolist()))}")
        if bool((rh < 1).any() or (rw < 1).any() or (oy < 0).any() or (ox < 0).any()
                or (oy + size > rh).any() or (ox + size > rw).any()):
            raise ValueError("output window outside the resized image")
        return size

    def __call__(self, batch: MultiCropBatch, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        S = self._validate(batch)
        pixels, index, params = batch
        B, dev = index.shape[0], self.device
        if out is None:
            out = torch.empty((B, 3, S, S), dtype=torch.float32, device=dev)
        elif (not isinstance(out, torch.Tensor) or out.dtype != torch.float32 or out.device != dev
              or tuple(out.shape) != (B, 3, S, S) or not out.is_contiguous()):
            raise ValueError(f"out must be a contiguous fp32 [{B}, 3, {S}, {S}] tensor on {dev}")
        top, left, h, w, rh, rw, oy, ox, _, _, interp = params.unbind(1)
        support = torch.where(interp == PIL_BICUBIC, _SUPPORT[PIL_BICUBIC], _SUPPORT[PIL_BILINEAR])
        # Pillow's ksize = ceil(support * max(1, in / out)) * 2 + 1
        kh = torch.ceil(support * torch.clamp(w / rw, min=1.0)).to(torch.int64) * 2 + 1
        kv = torch.ceil(support * torch.clamp(h / rh, min=1.0)).to(torch.int64) * 2 + 1
        # the box rows the window's vertical taps read: from the first tap of output oy to the last of oy + S - 1
        y0, _ = _first_last_tap(h, rh, oy, support)
        _, y1 = _first_last_tap(h, rh, oy + (S - 1), support)
        rows = y1 - y0
        tmp_n = rows * S * 3
        coef_n = S * (4 + kh + kv)
        meta = torch.stack([index[:, 0], index[:, 2], y0, rows, torch.cumsum(tmp_n, 0) - tmp_n,
                            torch.cumsum(coef_n, 0) - coef_n, kh, kv], 1)
        src = pixels.to(dev, non_blocking=True)
        rec_d = params.contiguous().pin_memory().to(dev, non_blocking=True)
        meta_d = meta.pin_memory().to(dev, non_blocking=True)
        tmp = torch.empty(int(tmp_n.sum()), dtype=torch.uint8, device=dev)
        coef = torch.empty(int(coef_n.sum()), dtype=torch.int32, device=dev)
        stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        _lib.call("esvit_augment_eval_coeffs", _p(rec_d), _p(meta_d), _p(coef), B, S, stream)
        _lib.call("esvit_augment_eval_resize_h", _p(src), _p(rec_d), _p(meta_d), _p(coef), _p(tmp), B, S,
                  int((rows * S).max()), stream)
        _lib.call("esvit_augment_eval_resize_v", _p(meta_d), _p(coef), _p(tmp), _p(self.norm), _p(out), B, S, stream)
        return out
