"""Batched, uint8-in / uint8-out inpainting — the ``bin/predict.py`` path (SURVEY.md row f1) on the native kernels.

The reference loops over the dataset one image at a time: decode -> float32 / 255 -> symmetric padding to a
multiple of 8 -> ``mask > 0`` -> ``img * (1 - mask)`` -> ``cat(mask)`` -> generator -> blend -> crop -> x255 / clip /
``astype(uint8)`` -> write (bin/predict.py:67-95, saicinpainting/evaluation/data.py:11-36,56-81,
saicinpainting/training/trainers/default.py:59-71).  Here everything between "decoded bytes" and "result bytes" is
one CUDA-graph replay: the elementwise work is fused into the first and last kernels of the generator program
(``ffcb_stem_pack_u8`` / ``ffcb_head_gather7_blend_u8``), images of equal size are batched, and host<->device
copies of neighbouring batches overlap the kernels (``lama_b200.serving.GeneratorPipeline``).

    inp = BatchedInpainter(generator.cuda().eval(), max_batch=32)
    outs = inp.inpaint([(img0, mask0), (img1, mask1), ...])      # HxWx3 / HxW uint8 numpy in, HxWx3 uint8 out

    python -m lama_b200.predict --model-dir big-lama --indir images/ --outdir out/     # predict.py's file layout

The model directory may hold an FFC generator (big-lama, lama-fourier) or a LaMa-Regular one (lama-regular,
big-lama-regular: ``pix2pixhd_global``); ``generator_from_config`` builds either.

The arithmetic is the reference's, byte for byte outside the hole and within the generator tolerance (one grey
level where a truncation boundary is crossed) inside it; ``tests/golden/predict_ngf8_3x45x52.npz`` pins it.
There is no CPU path: a generator that is not on a CUDA device, or is outside the native path, is an error.
"""
from __future__ import annotations

import argparse
import gc
import glob
import logging
import os
from collections import OrderedDict
from typing import Dict, Iterable, List, Optional, Sequence, Tuple

import numpy as np
import torch

from .serving import GeneratorPipeline

log = logging.getLogger(__name__)


class BatchedInpainter:
    """Groups equally sized (image, mask) pairs into batches and runs them through u8 generator pipelines.

    One pipeline (program + CUDA graph + staging buffers) is kept per (batch, H0, W0); the least recently used
    one is dropped when more than ``max_pipelines`` shapes are alive (a 512x512 bs32 program holds ~10 GB).

    Batches are sized to fit ``mem_budget``: the device bytes the alive pipelines may pool (default: 70 % of the free
    device memory, plus what this inpainter's own pipelines hold, when a group of equally sized images starts).  A
    group whose ``max_batch`` images fit runs in batches of ``max_batch``; a larger one (big-lama on a 4K photo holds
    ~8 GB per image) is cut into balanced batches of the most images that fit.  Pipelines of another shape are released
    before one that would not fit beside them is built.  An image that alone exceeds the budget still runs at batch 1:
    if it does not fit the device, the allocation error surfaces."""

    def __init__(self, generator, max_batch: int = 32, pad_mod: int = 8, device: Optional[torch.device] = None,
                 max_pipelines: int = 2, depth: int = 2, mem_budget: Optional[int] = None):
        self.generator = generator.eval()
        self.device = device if device is not None else next(generator.parameters()).device
        if self.device.type != "cuda":
            raise RuntimeError("BatchedInpainter needs the generator on a CUDA device (there is no CPU path)")
        self.max_batch, self.pad_mod, self.depth = int(max_batch), int(pad_mod), int(depth)
        self.max_pipelines = max_pipelines
        self.mem_budget = mem_budget
        self._pipes: "OrderedDict[Tuple[int, int, int], _Lane]" = OrderedDict()
        self._per_image: Dict[Tuple[int, int], int] = {}

    # -- planning (pure host logic, unit-tested on CPU)
    @staticmethod
    def plan(sizes: Sequence[Tuple[int, int]], max_batch: int) -> List[Tuple[Tuple[int, int], List[int]]]:
        """Group item indices by (H0, W0), keep first-seen order of the groups, split groups into batches of at
        most ``max_batch``.  Returns [((H0, W0), [indices...]), ...]."""
        groups: "OrderedDict[Tuple[int, int], List[int]]" = OrderedDict()
        for i, hw in enumerate(sizes):
            groups.setdefault((int(hw[0]), int(hw[1])), []).append(i)
        out = []
        for hw, idx in groups.items():
            for k in range(0, len(idx), max_batch):
                out.append((hw, idx[k:k + max_batch]))
        return out

    @staticmethod
    def plan_group(idx: Sequence[int], per_image_bytes: int, budget: int, max_batch: int) -> List[List[int]]:
        """Batches of one group of equally sized images: those of ``plan`` when ``max_batch`` images fit ``budget``,
        else balanced batches of at most ``budget // per_image_bytes`` images (at least one)."""
        from .refine import BatchedRefiner
        if int(budget) // max(1, int(per_image_bytes)) >= max_batch:
            return [list(idx[k:k + max_batch]) for k in range(0, len(idx), max_batch)]
        return BatchedRefiner.plan_batches(idx, per_image_bytes, budget, max_batch)

    def per_image_bytes(self, h0: int, w0: int) -> int:
        """Device bytes of one image's share of a pipeline at (h0, w0): the activations, workspace and outputs of the
        one-image ``generator_u8`` program (``engine.program_storage_bytes``; a program of B images pools at most B
        times this), plus the pipeline's device staging (``depth`` input and output slots, the graph's static input)."""
        key = (int(h0), int(w0))
        if key not in self._per_image:
            from . import engine as E
            metas = (torch.empty(1, h0, w0, 3, dtype=torch.uint8, device="meta"),
                     torch.empty(1, h0, w0, dtype=torch.uint8, device="meta"))
            with torch.no_grad():
                prog = E.build_module_program(self.generator, f"generator_u8:{self.pad_mod}",
                                              tuple(tuple(m.shape) for m in metas), E.default_math())
            staging = (self.depth + 1) * 4 * h0 * w0 + self.depth * 3 * h0 * w0
            self._per_image[key] = E.program_storage_bytes(prog) + staging
        return self._per_image[key]

    def _alive_bytes(self) -> int:
        return sum(lane.bytes for lane in self._pipes.values())

    def _budget(self) -> int:
        if self.mem_budget is not None:
            return int(self.mem_budget)
        return int(0.7 * (torch.cuda.mem_get_info(self.device)[0] + self._alive_bytes()))

    def _release_oldest(self):
        """Close the least recently used lane and free its device memory.  ``_pipes`` must hold the only reference to
        it (``inpaint`` keeps none across ``_lane``), so that its buffers are gone before the next lane allocates."""
        _, old = self._pipes.popitem(last=False)
        old.close()
        del old
        gc.collect()                              # executor / graph objects may sit in reference cycles
        torch.cuda.empty_cache()

    def _lane(self, b: int, h0: int, w0: int, budget: int) -> "_Lane":
        key = (b, h0, w0)
        lane = self._pipes.pop(key, None)
        if lane is None:
            need = b * self.per_image_bytes(h0, w0)
            while self._pipes and (len(self._pipes) >= self.max_pipelines or self._alive_bytes() + need > budget):
                self._release_oldest()
            lane = _Lane(self.generator, b, h0, w0, self.device, self.depth, self.pad_mod)
            lane.bytes = need
        self._pipes[key] = lane
        return lane

    def batches(self, sizes: Sequence[Tuple[int, int]]):
        """Yields ((H0, W0), [indices...], budget): ``plan``'s groups cut by ``plan_group`` under the budget taken
        when each group starts."""
        for hw, idx in self.plan(sizes, max(1, len(sizes))):
            budget = self._budget()
            per = self.per_image_bytes(*hw)
            parts = self.plan_group(idx, per, budget, self.max_batch)
            if budget // per < self.max_batch:
                log.info("%dx%d images: %d per batch at most, batches of %s (one image needs %.2f GB of a %.2f GB "
                         "budget)", hw[0], hw[1], max(1, budget // per), sorted({len(p) for p in parts}, reverse=True),
                         per / 1e9, budget / 1e9)
            for part in parts:
                yield hw, part, budget

    @torch.no_grad()
    def inpaint(self, items: Iterable[Tuple[np.ndarray, np.ndarray]]) -> List[np.ndarray]:
        """items: (image HxWx3 uint8 RGB, mask HxW uint8; any value > 0 marks the hole).  Returns the inpainted
        images (HxWx3 uint8) in input order."""
        items = list(items)
        for im, mk in items:
            if im.dtype != np.uint8 or mk.dtype != np.uint8 or im.ndim != 3 or im.shape[2] != 3 \
                    or mk.shape != im.shape[:2]:
                raise ValueError("expected (HxWx3 uint8 image, HxW uint8 mask) pairs")
        results: List[Optional[np.ndarray]] = [None] * len(items)
        inflight: List[Tuple["_Lane", int, List[int]]] = []

        def collect(upto: int):
            while len(inflight) > upto:
                lane, ticket, idx = inflight.pop(0)
                out = lane.pipe.result(ticket).numpy()
                for j, i in enumerate(idx):
                    results[i] = out[j].copy()

        for (h0, w0), idx, budget in self.batches([im.shape[:2] for im, _ in items]):
            # a partial batch runs at its own size (programs are per shape); full batches share one pipeline
            if inflight and inflight[-1][0].key != (len(idx), h0, w0):
                collect(0)                        # results live in the lane's buffers: drain before switching
            collect(self.depth - 1)
            # no local reference to a lane survives the loop body: a lane _lane releases must be unreachable
            inflight.append(self._submit(self._lane(len(idx), h0, w0, budget), idx, items))
        collect(0)
        return results  # type: ignore[return-value]

    @staticmethod
    def _submit(lane: "_Lane", idx: List[int], items) -> Tuple["_Lane", int, List[int]]:
        img_h, mask_h = lane.stage()
        for j, i in enumerate(idx):
            img_h[j].copy_(torch.from_numpy(np.ascontiguousarray(items[i][0])))
            mask_h[j].copy_(torch.from_numpy(np.ascontiguousarray(items[i][1])))
        return lane, lane.pipe.submit(img_h, mask_h), idx

    def __call__(self, images: np.ndarray, masks: np.ndarray) -> np.ndarray:
        """Equally sized batch: images (B,H,W,3) uint8, masks (B,H,W) uint8 -> (B,H,W,3) uint8."""
        return np.stack(self.inpaint(zip(images, masks)))


class _Lane:
    """One pipeline plus ``depth`` pinned host staging pairs (rotated so a pair is never rewritten while its
    H2D copy may still be in flight)."""

    def __init__(self, generator, b, h0, w0, device, depth, pad_mod):
        self.key = (b, h0, w0)
        self.bytes = 0
        self.pipe = GeneratorPipeline(generator, b, h0, w0, device=device, depth=depth, u8=True, pad_mod=pad_mod)
        self._stage = [(torch.empty((b, h0, w0, 3), dtype=torch.uint8).pin_memory(),
                        torch.empty((b, h0, w0), dtype=torch.uint8).pin_memory()) for _ in range(depth + 1)]
        self._k = 0

    def stage(self):
        pair = self._stage[self._k % len(self._stage)]
        self._k += 1
        return pair

    def close(self):
        """Wait for the pipeline's work and drop its executor from the generator's program cache, so that its buffers
        are freed with the lane."""
        from . import engine as E
        self.pipe.drain()
        E.drop_executor(self.pipe.ex)


# ------------------------------------------------------------------------------- checkpoint / files
def generator_kwargs_from_config(cfg: Dict) -> Dict:
    """``generator:`` section of a training config (configs/training/generator/*.yaml, e.g. big-lama.yaml:26-45)
    -> FFCResNetGenerator kwargs, as make_generator does (saicinpainting/training/modules/__init__.py:7-17)."""
    g = dict(cfg["generator"])
    kind = g.pop("kind")
    if kind != "ffc_resnet":
        raise ValueError(f"generator kind {kind!r} is not the FFC generator")
    return g


def generator_from_config(cfg: Dict):
    """The drop-in generator a training config describes, as make_generator builds it
    (saicinpainting/training/modules/__init__.py:7-17): ``ffc_resnet`` -> FFCResNetGenerator (big-lama, lama-fourier),
    ``pix2pixhd_global`` -> GlobalGenerator (lama-regular, big-lama-regular)."""
    kind = cfg["generator"]["kind"]
    if kind == "ffc_resnet":
        from .modules import FFCResNetGenerator
        return FFCResNetGenerator(**generator_kwargs_from_config(cfg))
    if kind == "pix2pixhd_global":
        from .pix2pixhd import GlobalGenerator
        return GlobalGenerator(**{k: v for k, v in cfg["generator"].items() if k != "kind"})
    raise ValueError(f"generator kind {kind!r} has no drop-in generator (ffc_resnet, pix2pixhd_global)")


def _read_config(model_dir: str) -> Dict:
    import yaml
    with open(os.path.join(model_dir, "config.yaml")) as f:
        return yaml.safe_load(f)


def check_refinable(cfg: Dict) -> None:
    """Refinement optimises the FFC generator's two bottleneck halves (z1, z2; evaluation/refinement.py:128); a
    ``pix2pixhd_global`` generator has one bottleneck tensor, and the reference cannot refine it either."""
    kind = cfg["generator"]["kind"]
    if kind != "ffc_resnet":
        raise ValueError(f"--refine needs an ffc_resnet generator (big-lama, lama-fourier); this model's generator "
                         f"kind is {kind!r}")


def load_generator(model_dir: str, checkpoint: str = "best.ckpt", device: str = "cuda"):
    """Build the drop-in generator from ``<model_dir>/config.yaml`` (``generator_from_config``) and load
    ``<model_dir>/models/<checkpoint>`` (a Lightning checkpoint: generator weights live under the ``generator.``
    prefix of ``state_dict`` — saicinpainting/training/trainers/__init__.py:25-30, bin/predict.py:49-59)."""
    gen = generator_from_config(_read_config(model_dir))
    state = torch.load(os.path.join(model_dir, "models", checkpoint), map_location="cpu", weights_only=False)
    sd = state.get("state_dict", state)
    sd = {k[len("generator."):]: v for k, v in sd.items() if k.startswith("generator.")} or sd
    gen.load_state_dict(sd, strict=True)
    return gen.eval().to(device)


def list_dataset(indir: str, img_suffix: str = ".png") -> List[Tuple[str, str]]:
    """(image file, mask file) pairs as InpaintingDataset finds them (evaluation/data.py:57-61)."""
    masks = sorted(glob.glob(os.path.join(indir, "**", "*mask*.png"), recursive=True))
    return [(m.rsplit("_mask", 1)[0] + img_suffix, m) for m in masks]


def shard_pairs(pairs: Sequence, rank: int, world: int) -> List:
    """Files of one rank when several processes (one per GPU, e.g. under torchrun) share a directory: the path
    shards by image (SURVEY.md §8e), every rank writes its own outputs, no collective is needed.  Interleaved so
    that sorted directories with size-ordered files still balance."""
    assert 0 <= rank < world
    return list(pairs[rank::world])


def predict_directory(inpainter, indir: str, outdir: str, img_suffix: str = ".png",
                      out_ext: str = ".png", chunk: int = 256, rank: int = 0, world: int = 1) -> int:
    """bin/predict.py:63-95 for a whole directory: same file discovery and output naming, batched execution.
    ``inpainter``: a BatchedInpainter or a lama_b200.refine.BatchedRefiner (anything with ``inpaint(items)``)."""
    from PIL import Image
    if not indir.endswith("/"):
        indir += "/"
    pairs = shard_pairs(list_dataset(indir, img_suffix), rank, world)
    for k in range(0, len(pairs), chunk):
        part = pairs[k:k + chunk]
        items = [(np.array(Image.open(i).convert("RGB")), np.array(Image.open(m).convert("L"))) for i, m in part]
        for (_, m), res in zip(part, inpainter.inpaint(items)):
            out = os.path.join(outdir, os.path.splitext(m[len(indir):])[0] + out_ext)
            os.makedirs(os.path.dirname(out) or ".", exist_ok=True)
            Image.fromarray(res).save(out)
    return len(pairs)


def build_parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(
        description="batched LaMa inpainting on the native H100 path",
        epilog="Several GPUs: one process per GPU (python -m torch.distributed.run --nproc-per-node N -m "
               "lama_b200.predict ...), each taking its share of the files.  With --refine this replaces the "
               "reference's refiner.gpu_ids, which splits one image's residual blocks over several GPUs.")
    ap.add_argument("--model-dir", required=True, help="directory with config.yaml and models/<checkpoint>")
    ap.add_argument("--checkpoint", default="best.ckpt")
    ap.add_argument("--indir", required=True)
    ap.add_argument("--outdir", required=True)
    ap.add_argument("--img-suffix", default=".png")
    ap.add_argument("--out-ext", default=".png")
    ap.add_argument("--batch", type=int, default=32,
                    help="images per batch at most; smaller when the programs would not fit device memory")
    ap.add_argument("--pad-mod", type=int, default=8, help="pad to a multiple of this (the refiner's modulo too)")
    # configs/prediction/default.yaml: refine, refiner.{n_iters, lr, min_side, max_scales, px_budget}
    ap.add_argument("--refine", action="store_true",
                    help="multi-scale refinement (evaluation/refinement.py) of every image: lama_b200.refine."
                         "BatchedRefiner; images above --px-budget pixels come out at the reduced size")
    ap.add_argument("--n-iters", type=int, default=15, help="refinement: Adam iterations per scale")
    ap.add_argument("--lr", type=float, default=0.002, help="refinement: Adam learning rate")
    ap.add_argument("--min-side", type=int, default=512, help="refinement: smallest side of the lowest scale")
    ap.add_argument("--max-scales", type=int, default=3, help="refinement: most pyramid scales")
    ap.add_argument("--px-budget", type=int, default=1800000, help="refinement: larger images are resized to this")
    ap.add_argument("--relu-masks", choices=("values", "bits"), default=None,
                    help="refinement: keep the backward's ReLU masks as the forward activations (values, the default) "
                         "or as bits, which needs about half the memory at large scales (same results), e.g. to "
                         "refine 12-24 megapixel photos at full size with a raised --px-budget")
    return ap


def refiner_kwargs(a: argparse.Namespace) -> Dict:
    """Command-line arguments -> lama_b200.refine.BatchedRefiner keyword arguments (``relu_masks`` only when given)."""
    kw = dict(max_batch=a.batch, modulo=a.pad_mod, n_iters=a.n_iters, lr=a.lr, min_side=a.min_side,
              max_scales=a.max_scales, px_budget=a.px_budget)
    if a.relu_masks is not None:
        kw["relu_masks"] = a.relu_masks
    return kw


def main(argv=None):
    a = build_parser().parse_args(argv)
    logging.basicConfig(level=logging.INFO, format="%(message)s")
    # one process per GPU (python -m torch.distributed.run --nproc-per-node N -m lama_b200.predict ...): every rank
    # takes its share of the files; single-process runs see rank 0 of 1
    rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
    device = f"cuda:{os.environ.get('LOCAL_RANK', '0')}"
    if a.refine:
        check_refinable(_read_config(a.model_dir))
    gen = load_generator(a.model_dir, a.checkpoint, device=device)
    if a.refine:
        from .refine import BatchedRefiner
        inpainter = BatchedRefiner(gen, **refiner_kwargs(a))
    else:
        inpainter = BatchedInpainter(gen, max_batch=a.batch, pad_mod=a.pad_mod)
    n = predict_directory(inpainter, a.indir, a.outdir, a.img_suffix, a.out_ext, rank=rank, world=world)
    print(f"[rank {rank}/{world}] inpainted {n} images -> {a.outdir}")


if __name__ == "__main__":
    main()
