"""Refinement driver for the drop-in generator (SURVEY.md row f3): the reference's multi-scale "plug-n-play" refinement
(``saicinpainting/evaluation/refinement.py``) without kornia, on top of the native forward + input-gradient program of
the generator's rear (``lama_b200.engine.generator_rear_with_input_grad``).

What the reference does (refinement.py:86-174, 228-314): build an image / mask pyramid, and at every scale optimise the
feature maps z1, z2 entering the residual blocks (Adam, 15 iterations) so that the down-scaled prediction matches the
previous scale's result inside the (eroded) hole and the input outside.  The optimisation needs dL/dz through the 18
residual blocks, the up-sampling tail and the image-space pyramid operators; the weights are frozen.

Here:
  * rear (residual blocks, ConvTranspose2d / BN / ReLU tail, 7x7 head, sigmoid): ONE native program with a forward and
    an input-gradient part (eval-mode BN folded, ``torch.autograd.Function``), when ``engine.rear_grad_supported``
    holds for the scale's shape; otherwise the module slice ``generator.model[first_block:]`` — native per-block
    gradients (``engine.block_with_input_grad``) with the tail on torch autograd.  LAMA_B200_NATIVE_GRAD=0: torch
    autograd throughout;
  * front (stem + stride-2 convs) under ``no_grad``: the native stage programs;
  * pyramid operators: the three kornia calls restated with torch ops — ``gaussian_blur2d(k=5, sigma=1)`` (reflect
    border, separable normalised Gaussian), ``erosion(mask, 15x15 ellipse)`` (geodesic border: outside counts as +max,
    i.e. the border never erodes) and ``resize(bilinear, align_corners=False)``; pinned against OpenCV in
    ``tests/test_refine_cpu.py`` (``cv2.GaussianBlur`` BORDER_REFLECT_101, ``cv2.erode`` default border).
The reference pipelines the blocks over several GPUs (refinement.py:276-289); batch sharding supersedes that here
(SURVEY.md §8e): one image per GPU, everything on one device.
"""
from __future__ import annotations

import math
import os
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F


# ------------------------------------------------------------------------------------------- pyramid operators
def gaussian_kernel1d(ksize: int = 5, sigma: float = 1.0, device=None, dtype=torch.float32) -> torch.Tensor:
    """Normalised 1-D Gaussian (kornia.filters.get_gaussian_kernel1d == cv2.getGaussianKernel for sigma > 0)."""
    x = torch.arange(ksize, device=device, dtype=torch.float64) - (ksize - 1) / 2.0
    k = torch.exp(-(x * x) / (2.0 * sigma * sigma))
    return (k / k.sum()).to(dtype)


def gaussian_blur2d(x: torch.Tensor, ksize: int = 5, sigma: float = 1.0) -> torch.Tensor:
    """kornia.filters.gaussian_blur2d(x, (k,k), (s,s)) with its default border_type='reflect' (refinement.py:24,55)."""
    c = x.shape[1]
    k = gaussian_kernel1d(ksize, sigma, x.device, x.dtype)
    p = ksize // 2
    x = F.pad(x, (p, p, p, p), mode="reflect")
    x = F.conv2d(x, k.view(1, 1, 1, ksize).expand(c, 1, 1, ksize), groups=c)
    return F.conv2d(x, k.view(1, 1, ksize, 1).expand(c, 1, ksize, 1), groups=c)


def ellipse_kernel(ksize: int = 15) -> np.ndarray:
    """cv2.getStructuringElement(cv2.MORPH_ELLIPSE, (k, k)) restated (refinement.py:139): row i of the inscribed
    ellipse spans |dx| <= round(r * sqrt(1 - (dy / r)^2)) around the centre column, r = k // 2."""
    r = ksize // 2
    out = np.zeros((ksize, ksize), dtype=bool)
    inv_r2 = 1.0 / (r * r) if r else 0.0
    for i in range(ksize):
        dy = i - r
        if abs(dy) <= r:
            dx = int(round(r * math.sqrt(max((r * r - dy * dy) * inv_r2, 0.0))))
            out[i, max(r - dx, 0):min(r + dx + 1, ksize)] = True
    return out


def erosion(mask: torch.Tensor, kernel: torch.Tensor) -> torch.Tensor:
    """kornia.morphology.erosion(mask, kernel) (flat structuring element, border_type='geodesic': pixels outside the
    image never lower the minimum) == cv2.erode with its default border value (refinement.py:69)."""
    kh, kw = kernel.shape
    ph, pw = kh // 2, kw // 2
    big = torch.finfo(mask.dtype).max if mask.dtype.is_floating_point else torch.iinfo(mask.dtype).max
    x = F.pad(mask, (pw, kw - 1 - pw, ph, kh - 1 - ph), mode="constant", value=float(big))
    b, c, h, w = mask.shape
    cols = F.unfold(x.reshape(b * c, 1, h + kh - 1, w + kw - 1), (kh, kw))           # [B*C, kh*kw, H*W]
    sel = kernel.reshape(-1) > 0
    return cols[:, sel].min(dim=1).values.reshape(b, c, h, w)


def pyrdown(im: torch.Tensor, downsize: Optional[Tuple[int, int]] = None) -> torch.Tensor:
    """refinement.py:19-26."""
    if downsize is None:
        downsize = (im.shape[2] // 2, im.shape[3] // 2)
    return F.interpolate(gaussian_blur2d(im), size=downsize, mode="bilinear", align_corners=False)


def pyrdown_mask(mask: torch.Tensor, downsize: Optional[Tuple[int, int]] = None, eps: float = 1e-8,
                 blur_mask: bool = True, round_up: bool = True) -> torch.Tensor:
    """refinement.py:28-64."""
    if downsize is None:
        downsize = (mask.shape[2] // 2, mask.shape[3] // 2)
    if blur_mask:
        mask = gaussian_blur2d(mask)
    mask = F.interpolate(mask, size=downsize, mode="bilinear", align_corners=False)
    thr = eps if round_up else 1.0 - eps
    return (mask >= thr).to(mask.dtype)


def erode_mask(mask: torch.Tensor, ekernel: Optional[torch.Tensor] = None, eps: float = 1e-8) -> torch.Tensor:
    """refinement.py:66-72."""
    if ekernel is None:
        return mask
    return (erosion(mask, ekernel) >= 1.0 - eps).to(mask.dtype)


def l1_loss(pred, pred_downscaled, ref, mask, mask_downscaled, image, on_pred=True):
    """refinement.py:75-84."""
    loss = torch.mean(torch.abs(pred[mask < 1e-8] - image[mask < 1e-8]))
    if on_pred:
        loss = loss + torch.mean(torch.abs(pred_downscaled[mask_downscaled >= 1e-8] - ref[mask_downscaled >= 1e-8]))
    return loss


def image_mask_pyramid(image: torch.Tensor, mask: torch.Tensor, min_side: int, max_scales: int, px_budget: int):
    """refinement.py:176-226 on already un-padded (1,3,h,w) / (1,1,h,w) tensors; lowest resolution first."""
    assert image.shape[0] == 1, "refiner works on only batches of size 1!"
    h, w = image.shape[2:]
    if h * w > px_budget:
        ratio = math.sqrt(px_budget / float(h * w))
        h, w = int(h * ratio), int(w * ratio)
        image = F.interpolate(image, size=(h, w), mode="bilinear", align_corners=False)
        mask = F.interpolate(mask, size=(h, w), mode="bilinear", align_corners=False)
        mask = (mask > 1e-8).to(mask.dtype)
    n_scales = min(1 + int(round(max(0, math.log2(min(h, w) / min_side)))), max_scales)
    images, masks = [image], [mask]
    for _ in range(n_scales - 1):
        images.append(pyrdown(images[-1]))
        masks.append(pyrdown_mask(masks[-1]))
    return images[::-1], masks[::-1]


# ------------------------------------------------------------------------------------------- the refinement loop
def split_generator(model: nn.Sequential):
    """refinement.py:266-289 on one device: (front, rear) — everything before the first residual block, and the rest."""
    from .modules import FFCResnetBlock
    first = next(i for i, m in enumerate(model) if isinstance(m, FFCResnetBlock))
    return model[:first], model[first:]


class NativeRear:
    """``rear((z1, z2))`` for ``infer_scale``: the generator's native rear program where it applies (see
    ``engine.rear_grad_supported``), else the module slice ``generator.model[first_block:]``."""

    def __init__(self, generator, modules: nn.Sequential):
        self.generator, self.modules = generator, modules

    def native_ok(self, z1, z2) -> bool:
        from . import engine as E
        if os.environ.get("LAMA_B200_NATIVE_GRAD", "1") == "0" or not torch.is_grad_enabled() or self.generator.training:
            return False
        if not all(torch.is_tensor(z) and z.is_cuda and z.dtype == torch.float32 for z in (z1, z2)):
            return False
        if any(p.requires_grad for p in self.generator.parameters()):
            return False
        return E.rear_grad_supported(self.generator, tuple(z1.shape), tuple(z2.shape))

    def __call__(self, z):
        z1, z2 = z
        if self.native_ok(z1, z2):
            from . import engine as E
            return E.generator_rear_with_input_grad(self.generator, z1, z2)
        return self.modules(z)


def _pad_to_modulo(t: torch.Tensor, mod: int) -> torch.Tensor:
    """evaluation/data.py:36-40 (reflect padding at the bottom / right)."""
    h, w = t.shape[2:]
    return F.pad(t, (0, (-w) % mod, 0, (-h) % mod), mode="reflect")


def infer_scale(image, mask, front, rear, ref_lower_res, orig_shape, n_iters: int = 15, lr: float = 0.002):
    """refinement.py:86-174 for one scale, single device."""
    dev = image.device
    masked = torch.cat([image * (1 - mask), mask], dim=1)
    mask3 = mask.repeat(1, 3, 1, 1)
    if ref_lower_res is not None:
        ref_lower_res = ref_lower_res.detach().to(dev)
    with torch.no_grad():
        z1, z2 = front(masked)
    ekernel = torch.from_numpy(ellipse_kernel(15)).float().to(dev)
    z1, z2 = z1.detach().clone().requires_grad_(True), z2.detach().clone().requires_grad_(True)
    opt = torch.optim.Adam([z1, z2], lr=lr)
    pred = None
    for it in range(n_iters):
        opt.zero_grad()
        pred = rear((z1, z2))
        if ref_lower_res is None:
            break
        pred_down = pyrdown(pred[:, :, :orig_shape[0], :orig_shape[1]])
        mask_down = pyrdown_mask(mask3[:, :1, :orig_shape[0], :orig_shape[1]], blur_mask=False, round_up=False)
        mask_down = erode_mask(mask_down, ekernel).repeat(1, 3, 1, 1)
        loss = l1_loss(pred, pred_down, ref_lower_res, mask3, mask_down, image, on_pred=True)
        if it < n_iters - 1:
            loss.backward()
            opt.step()
    return (mask3 * pred + (1 - mask3) * image).detach()


def refine_predict(image: torch.Tensor, mask: torch.Tensor, generator, *, modulo: int = 8, n_iters: int = 15,
                   lr: float = 0.002, min_side: int = 512, max_scales: int = 3, px_budget: int = 1800000,
                   device=None) -> torch.Tensor:
    """refinement.py:228-314 for the drop-in generator: ``image`` (1,3,h,w) in [0,1], ``mask`` (1,1,h,w) in {0,1}
    (already un-padded); returns the refined inpainting (1,3,h,w) on the CPU, like the reference."""
    assert not generator.training
    device = device if device is not None else next(generator.parameters()).device
    for p in generator.parameters():
        p.requires_grad_(False)                       # model.freeze(): input gradients only
    front, rear = split_generator(generator.model)
    rear = NativeRear(generator, rear)
    images, masks = image_mask_pyramid(image, mask, min_side, max_scales, px_budget)
    result = None
    for im, mk in zip(images, masks):
        orig = tuple(im.shape[2:])
        im_p, mk_p = _pad_to_modulo(im, modulo).to(device), _pad_to_modulo(mk, modulo).to(device)
        mk_p = (mk_p >= 1e-8).to(mk_p.dtype)
        result = infer_scale(im_p, mk_p, front, rear, result, orig, n_iters, lr)
        result = result[:, :, :orig[0], :orig[1]]
    return result.cpu()
