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


# ------------------------------------------------------------------------------------------- batched refinement
class _StepLane:
    """One refinement step program (``engine.build_refine_program``) for a batch shape and crop, its static inputs,
    Adam over the static z1 / z2 with ``z.grad`` bound to the program's dx outputs, and the CUDA graph of one step
    (rear forward, loss gradient, rear backward, Adam), captured on first use and replayed for every later batch and
    scale of the same shape."""

    def __init__(self, gen, sl, sg, crop, lr: float, device, graphs: bool = True, kind: Optional[str] = None):
        from . import engine as E
        kind = kind if kind is not None else f"generator_refine:{crop[0]}x{crop[1]}"
        with torch.no_grad():
            prog = E.build_module_program(gen, kind, (sl, sg), E.default_math())
        self.ex = E.CudaExecutor(prog, device)
        self.inputs = {k: torch.zeros(v, dtype=torch.float32, device=device) for k, v in prog.inputs.items()}
        self.z = [self.inputs["x0"].requires_grad_(True), self.inputs["x1"].requires_grad_(True)]
        self.z[0].grad, self.z[1].grad = self.ex.outputs["dx0"], self.ex.outputs["dx1"]
        self.opt = torch.optim.Adam(self.z, lr=lr, capturable=True)
        self.graphs, self.graph = graphs, None

    def _step(self):
        self.ex.run(self.inputs, part=0)
        self.ex.run(self.inputs, part=1)
        self.opt.step()

    def run(self, z1, z2, consts, n_steps: int) -> torch.Tensor:
        """Load z1, z2 and the scale's constants, take ``n_steps`` Adam steps from a fresh optimiser state, and return
        the forward of the final z (the executor's own y0 tensor)."""
        with torch.no_grad():
            self.z[0].copy_(z1)
            self.z[1].copy_(z2)
            for k, v in consts.items():
                self.inputs[k].copy_(v)
            for st in self.opt.state.values():          # every batch starts from step 0 with zero moments
                for t in st.values():
                    t.zero_()
        if n_steps > 0 and (self.graph is None or not self.graphs):
            self._step()                                # eager (the first one also creates the Adam state)
            n_steps -= 1
            if self.graphs:
                self.graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(self.graph):
                    self._step()
        for _ in range(n_steps):
            if self.graphs:
                self.graph.replay()
            else:
                self._step()
        return self.ex.run(self.inputs, part=0)["y0"]


class _ForwardLane:
    """The forward-only rear program (``engine.emit_rear_forward``, kind ``generator_rear``) for the lowest scale, where
    the reference takes one forward and no step (refinement.py:150-151: no reference image yet)."""

    graph = None

    def __init__(self, gen, sl, sg, device):
        from . import engine as E
        with torch.no_grad():
            prog = E.build_module_program(gen, "generator_rear", (sl, sg), E.default_math())
        self.ex = E.CudaExecutor(prog, device)

    def run(self, z1, z2, consts, n_steps: int) -> torch.Tensor:
        assert n_steps == 0
        return self.ex.run({"x0": z1.contiguous(), "x1": z2.contiguous()})["y0"]


class BatchedRefiner:
    """refine_predict (evaluation/refinement.py:228-314) for many images: equally sized images are refined together,
    each scale of a batch is one step program whose forward + loss gradient + backward + Adam step is one CUDA graph
    replayed ``n_iters - 1`` times, with no host synchronisation inside a scale.  Images do not interact (eval-mode BN,
    per-plane FFTs, per-image losses, elementwise Adam): each gets the result it would get alone.

        ref = BatchedRefiner(generator.cuda().eval(), max_batch=8)
        outs = ref.inpaint([(img0, mask0), ...])          # HxWx3 / HxW uint8 in, HxWx3 uint8 out

    Images above ``px_budget`` pixels are refined, and returned, at the reduced size, as by the reference.  Groups whose
    scales the native step program does not cover (``engine.refine_supported``: LFU, out_ffc or gated generators,
    bottleneck axes above ``engine.FFT_MAX_LEN``), and every group under LAMA_B200_NATIVE_GRAD=0, run
    ``refine_predict`` image by image.  ``mem_budget``: device bytes the programs of one batch, every scale's, may pool
    (default: 70 % of the free device memory when the group starts).  A group is cut into balanced batches, and the
    programs of one batch size are released before those of another are built, so no more than one batch's programs are
    alive at a time.  An image whose programs alone exceed the budget still runs, at batch 1; if the device cannot hold
    them, the allocation error propagates to the caller.

    ``relu_masks="bits"`` runs the step programs of kind ``generator_refine_bits``: the ReLU masks the backward reads
    are kept as bits instead of the forward activations themselves (``lama_b200.relu_bits``), which cuts a step
    program's storage by about 53 % at large scales, so that 12- and 24-megapixel photos refine at full size on one
    80 GB GPU.  The results are bit-identical to ``"values"``.  This large-photo setting also keeps one scale's program
    alive at a time (a scale's lane releases the previous one; the batch plan still counts every scale) and releases the
    front's (stem and down-sampling) cached stage programs after each scale's front pass, which at 24 MP would otherwise
    hold about 34 GB next to the step programs.  Later batches of the same size build and capture them again.

    ``tail="banded"`` (with ``relu_masks="bits"`` only) runs the step programs of kind ``generator_refine_bits_banded``:
    the full-resolution up-sampling tail and head run in row bands (``lama_b200.banded``), which at 24-50 megapixels
    cuts a step program's storage to less than half the bits program's.  This setting also releases the previous
    scale's lane before the front (stem and down-sampling) runs, and runs the front's stages one at a time, releasing
    each stage's programs after it ran, so that 48-50 megapixel photos refine at full size on one 80 GB GPU.
    The results are bit-identical.  It needs the tensor-core head (split-bf16 arithmetic, ``banded.tail_supported``);
    the constructor raises ``ValueError`` where that does not hold."""

    relu_masks = "values"
    tail = "whole"

    def __init__(self, generator, max_batch: int = 8, *, modulo: int = 8, n_iters: int = 15, lr: float = 0.002,
                 min_side: int = 512, max_scales: int = 3, px_budget: int = 1800000,
                 mem_budget: Optional[int] = None, relu_masks: str = "values", tail: str = "whole"):
        if relu_masks not in ("values", "bits"):
            raise ValueError(f"relu_masks must be 'values' or 'bits', not {relu_masks!r}")
        if tail not in ("whole", "banded"):
            raise ValueError(f"tail must be 'whole' or 'banded', not {tail!r}")
        if tail == "banded" and relu_masks != "bits":
            raise ValueError("tail='banded' needs relu_masks='bits'")
        if tail == "banded":
            from . import engine as E
            from .banded import tail_supported
            if not tail_supported(generator, E.default_math()):
                raise ValueError("tail='banded' needs the tensor-core head: split-bf16 arithmetic (LAMA_B200_MATH), "
                                 "LAMA_B200_HEAD=tc, a head of at most 3 outputs on a multiple of 8 channels")
        self.relu_masks, self.tail = relu_masks, tail
        self.generator = generator.eval()
        self.device = next(generator.parameters()).device
        if self.device.type != "cuda":
            raise RuntimeError("BatchedRefiner needs the generator on a CUDA device (there is no CPU path)")
        for p in generator.parameters():
            p.requires_grad_(False)                     # model.freeze(): input gradients only
        self.max_batch = int(max_batch)
        self.kw = dict(modulo=modulo, n_iters=n_iters, lr=lr, min_side=min_side, max_scales=max_scales,
                       px_budget=px_budget)
        self.mem_budget = mem_budget
        self.front, _ = split_generator(generator.model)
        self._lanes = {}
        self._size = None                               # input size the lanes in _lanes serve
        self._graphs = True

    # -- planning (pure host logic, unit-tested on CPU)
    @staticmethod
    def plan_batches(idx: Sequence[int], per_image_bytes: int, budget: int, max_batch: int) -> List[List[int]]:
        """Balanced batches of ``idx`` (sizes differ by at most one) whose programs (``per_image_bytes`` per image, all
        scales) fit ``budget``; at least one image per batch.  A program of B images pools at most B times the
        one-image program: every buffer, output and workspace scales with B, and tile-blocked buffers round B*H*W up to
        128 pixels once rather than per image."""
        n = len(idx)
        if n == 0:
            return []
        nb = max(1, min(int(max_batch), int(budget) // max(1, int(per_image_bytes))))
        k = -(-n // nb)
        sizes = [n // k + (1 if j < n % k else 0) for j in range(k)]
        starts = [sum(sizes[:j]) for j in range(k)]
        return [list(idx[a:a + m]) for a, m in zip(starts, sizes)]

    def scale_shapes(self, h: int, w: int) -> List[Tuple[Tuple[int, ...], Tuple[int, ...], Tuple[int, int]]]:
        """(z1 shape, z2 shape, crop) of one image per scale of an (h, w) input, lowest resolution first."""
        from . import engine as E
        px = self.kw["px_budget"]
        if h * w > px:
            ratio = math.sqrt(px / float(h * w))
            h, w = int(h * ratio), int(w * ratio)
        n_scales = min(1 + int(round(max(0, math.log2(min(h, w) / self.kw["min_side"])))), self.kw["max_scales"])
        crops = [(h, w)]
        for _ in range(n_scales - 1):
            crops.append((crops[-1][0] // 2, crops[-1][1] // 2))
        lay = E._generator_layout(self.generator)
        if lay is None:
            return []
        blk = lay[2][0].conv1.ffc if lay[2] else None
        f = 2 ** len(lay[1])
        out = []
        for h0, w0 in crops[::-1]:
            m = self.kw["modulo"]
            hp, wp = h0 + (-h0) % m, w0 + (-w0) % m
            cl, cg = (blk.convl2l.in_channels, blk.global_in_num) if blk is not None else (0, 0)
            out.append(((1, cl, hp // f, wp // f), (1, cg, hp // f, wp // f), (h0, w0)))
        return out

    def native_ok(self, h: int, w: int) -> bool:
        """Every scale of an (h, w) input has a native step program (else the group runs ``refine_predict``)."""
        from . import engine as E
        if os.environ.get("LAMA_B200_NATIVE_GRAD", "1") == "0":
            return False
        shapes = self.scale_shapes(h, w)
        return bool(shapes) and all(E.refine_supported(self.generator, sl, sg, crop) for sl, sg, crop in shapes)

    def program_kind(self, scale: int, crop: Tuple[int, int]) -> str:
        """The lowest scale (index 0) runs one forward; every other scale a step program (``relu_masks`` and ``tail``:
        which)."""
        if scale == 0:
            return "generator_rear"
        step = "generator_refine_bits" if self.relu_masks == "bits" else "generator_refine"
        if self.tail == "banded":
            step = "generator_refine_bits_banded"
        return f"{step}:{crop[0]}x{crop[1]}"

    def per_image_bytes(self, h: int, w: int) -> int:
        """Pooled device bytes of the one-image programs of every scale of an (h, w) input (a batch keeps all of them
        alive, so that the next batch of its size reuses their captured graphs)."""
        from . import engine as E
        total = 0
        for s, (sl, sg, crop) in enumerate(self.scale_shapes(h, w)):
            with torch.no_grad():
                prog = E.build_module_program(self.generator, self.program_kind(s, crop), (sl, sg), E.default_math())
            total += E.program_storage_bytes(prog)
        return total

    # -- execution
    def _make_lane(self, kind: str, sl, sg, crop):
        if kind == "generator_rear":
            return _ForwardLane(self.generator, sl, sg, self.device)
        return _StepLane(self.generator, sl, sg, crop, self.kw["lr"], self.device, self._graphs, kind)

    def _lane(self, b: int, scale: int, sl, sg, crop):
        """The lane of scale ``scale`` at batch size ``b``.  Lanes of another batch size are released first: only one
        batch's programs are alive at a time, which is what the batch plan budgets for."""
        key = (b, sl[1:], sg[1:], crop)
        if any(k[0] != b for k in self._lanes) or (self.relu_masks == "bits" and key not in self._lanes):
            self._lanes.clear()
            torch.cuda.empty_cache()
        lane = self._lanes.get(key)
        if lane is None:
            sl, sg = (b,) + tuple(sl[1:]), (b,) + tuple(sg[1:])
            lane = self._make_lane(self.program_kind(scale, crop), sl, sg, crop)
            self._lanes[key] = lane
        return lane

    def _front_stages(self, x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """z1, z2 of the banded setting: the previous scale's lane is released first, then the front's modules run one
        at a time, each stage's cached programs released right after it ran, so that no more than one stage's buffers
        are alive (about 68 GB for all of them at 48 megapixels).  The arithmetic is the cached front's."""
        from . import engine as E
        self._lanes.clear()
        torch.cuda.empty_cache()
        with torch.no_grad():
            for m in self.front:
                x = m(x)
                for sub in m.modules():
                    E.invalidate(sub)
                torch.cuda.empty_cache()
        return x

    def _refine_batch(self, images: List[torch.Tensor], masks: List[torch.Tensor]) -> torch.Tensor:
        """Equally sized (1,3,h,w) / (1,1,h,w) CPU images and masks -> (B,3,h',w') refined results on the device."""
        kw, dev = self.kw, self.device
        pyr = [image_mask_pyramid(im, mk, kw["min_side"], kw["max_scales"], kw["px_budget"])
               for im, mk in zip(images, masks)]
        ekernel = torch.from_numpy(ellipse_kernel(15)).float().to(dev)
        shapes = self.scale_shapes(images[0].shape[2], images[0].shape[3])
        result = None
        for s, (sl, sg, crop) in enumerate(shapes):
            im = torch.cat([_pad_to_modulo(p[0][s], kw["modulo"]) for p in pyr]).to(dev)
            mk = torch.cat([_pad_to_modulo(p[1][s], kw["modulo"]) for p in pyr]).to(dev)
            mk = (mk >= 1e-8).to(mk.dtype)
            x = torch.cat([im * (1 - mk), mk], dim=1)
            if self.tail == "banded":
                z1, z2 = self._front_stages(x)
            else:
                with torch.no_grad():
                    z1, z2 = self.front(x)
            del x
            if self.relu_masks == "bits" and self.tail != "banded":
                # the front's cached stage programs hold full-resolution buffers (about 34 GB for a 24 MP scale); the
                # large-photo setting releases them before the step program of the scale is built
                from . import engine as E
                for m in self.front.modules():
                    E.invalidate(m)
            lane = self._lane(len(images), s, sl, sg, crop)
            h0, w0 = crop
            consts = dict(image=im, mask=mk)
            n_steps = 0
            if result is not None:
                md = pyrdown_mask(mk[:, :, :h0, :w0], blur_mask=False, round_up=False)
                md = erode_mask(md, ekernel)
                n = torch.stack([3 * (mk < 1e-8).sum((1, 2, 3)), 3 * (md >= 1e-8).sum((1, 2, 3))], 1).double()
                inv = torch.where(n > 0, 1.0 / n.clamp_min(1), torch.zeros_like(n)).float()
                consts.update(ref=result, md=md, inv=inv)
                n_steps = kw["n_iters"] - 1
            pred = lane.run(z1, z2, consts, n_steps)
            result = (mk * pred + (1 - mk) * im)[:, :, :h0, :w0]
        return result

    def refine(self, images: Sequence[torch.Tensor], masks: Sequence[torch.Tensor]) -> List[torch.Tensor]:
        """Float entry point: images (3,H,W) in [0,1] and masks (1,H,W) (mask / 255, not thresholded, as the
        reference's dataset delivers them) on the CPU -> refined (3,H',W') float32 CPU tensors in input order."""
        images = [im.float().cpu()[None] for im in images]
        masks = [mk.float().cpu()[None] for mk in masks]
        from .predict import BatchedInpainter
        out: List[Optional[torch.Tensor]] = [None] * len(images)
        for hw, idx in BatchedInpainter.plan([im.shape[2:] for im in images], self.max_batch):
            if not self.native_ok(*hw):
                for i in idx:
                    out[i] = refine_predict(images[i], masks[i], self.generator, device=self.device, **self.kw)[0]
                continue
            if self._size != hw:                   # a new size: the previous size's step programs are done
                self._lanes.clear()
                torch.cuda.empty_cache()
                budget = self.mem_budget
                if budget is None:
                    budget = int(0.7 * torch.cuda.mem_get_info(self.device)[0])
                self._size, self._per_image, self._budget = hw, self.per_image_bytes(*hw), budget
            for part in self.plan_batches(idx, self._per_image, self._budget, self.max_batch):
                res = self._refine_batch([images[i] for i in part], [masks[i] for i in part]).cpu()
                for j, i in enumerate(part):
                    out[i] = res[j]
        return out  # type: ignore[return-value]

    def inpaint(self, items) -> List[np.ndarray]:
        """items: (image HxWx3 uint8 RGB, mask HxW uint8) -> refined images HxWx3 uint8 in input order
        (bin/predict.py:92: ``np.clip(x * 255, 0, 255).astype('uint8')``)."""
        items = list(items)
        for im, mk in items:
            if im.dtype != np.uint8 or mk.dtype != np.uint8 or im.ndim != 3 or im.shape[2] != 3 \
                    or mk.shape != im.shape[:2]:
                raise ValueError("expected (HxWx3 uint8 image, HxW uint8 mask) pairs")
        imgs = [torch.from_numpy(np.ascontiguousarray(im)).permute(2, 0, 1).float() / 255 for im, _ in items]
        msks = [torch.from_numpy(np.ascontiguousarray(mk))[None].float() / 255 for _, mk in items]
        return [to_uint8(r) for r in self.refine(imgs, msks)]


def to_uint8(x: torch.Tensor) -> np.ndarray:
    """(3,H,W) float -> HxWx3 uint8 as bin/predict.py:92 writes it."""
    return np.clip(x.permute(1, 2, 0).numpy() * 255, 0, 255).astype("uint8")
