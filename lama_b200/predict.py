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

The arithmetic is the reference's, byte for byte outside the hole and within the generator tolerance (one grey
level where a truncation boundary is crossed) inside it; ``tests/golden/predict_ngf8_3x45x52.npz`` pins it.
There is no CPU path: a generator that is not on a CUDA device, or is outside the native path, is an error.
"""
from __future__ import annotations

import argparse
import glob
import os
from collections import OrderedDict
from typing import Dict, Iterable, List, Optional, Sequence, Tuple

import numpy as np
import torch

from .serving import GeneratorPipeline


class BatchedInpainter:
    """Groups equally sized (image, mask) pairs into batches and runs them through u8 generator pipelines.

    One pipeline (program + CUDA graph + staging buffers) is kept per (batch, H0, W0); the least recently used
    one is dropped when more than ``max_pipelines`` shapes are alive (a 512x512 bs32 program holds ~10 GB)."""

    def __init__(self, generator, max_batch: int = 32, pad_mod: int = 8, device: Optional[torch.device] = None,
                 max_pipelines: int = 2, depth: int = 2):
        self.generator = generator.eval()
        self.device = device if device is not None else next(generator.parameters()).device
        if self.device.type != "cuda":
            raise RuntimeError("BatchedInpainter needs the generator on a CUDA device (there is no CPU path)")
        self.max_batch, self.pad_mod, self.depth = int(max_batch), int(pad_mod), int(depth)
        self.max_pipelines = max_pipelines
        self._pipes: "OrderedDict[Tuple[int, int, int], _Lane]" = OrderedDict()

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

    def _lane(self, b: int, h0: int, w0: int) -> "_Lane":
        key = (b, h0, w0)
        lane = self._pipes.pop(key, None)
        if lane is None:
            while len(self._pipes) >= self.max_pipelines:
                _, old = self._pipes.popitem(last=False)
                old.close()
            lane = _Lane(self.generator, b, h0, w0, self.device, self.depth, self.pad_mod)
        self._pipes[key] = lane
        return lane

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

        for (h0, w0), idx in self.plan([im.shape[:2] for im, _ in items], self.max_batch):
            # a partial batch runs at its own size (programs are per shape); full batches share one pipeline
            if inflight and inflight[-1][0].key != (len(idx), h0, w0):
                collect(0)                        # results live in the lane's buffers: drain before switching
            lane = self._lane(len(idx), h0, w0)
            collect(self.depth - 1)
            img_h, mask_h = lane.stage()
            for j, i in enumerate(idx):
                img_h[j].copy_(torch.from_numpy(np.ascontiguousarray(items[i][0])))
                mask_h[j].copy_(torch.from_numpy(np.ascontiguousarray(items[i][1])))
            inflight.append((lane, lane.pipe.submit(img_h, mask_h), idx))
        collect(0)
        return results  # type: ignore[return-value]

    def __call__(self, images: np.ndarray, masks: np.ndarray) -> np.ndarray:
        """Equally sized batch: images (B,H,W,3) uint8, masks (B,H,W) uint8 -> (B,H,W,3) uint8."""
        return np.stack(self.inpaint(zip(images, masks)))


class _Lane:
    """One pipeline plus ``depth`` pinned host staging pairs (rotated so a pair is never rewritten while its
    H2D copy may still be in flight)."""

    def __init__(self, generator, b, h0, w0, device, depth, pad_mod):
        self.key = (b, h0, w0)
        self.pipe = GeneratorPipeline(generator, b, h0, w0, device=device, depth=depth, u8=True, pad_mod=pad_mod)
        self._stage = [(torch.empty((b, h0, w0, 3), dtype=torch.uint8).pin_memory(),
                        torch.empty((b, h0, w0), dtype=torch.uint8).pin_memory()) for _ in range(depth + 1)]
        self._k = 0

    def stage(self):
        pair = self._stage[self._k % len(self._stage)]
        self._k += 1
        return pair

    def close(self):
        self.pipe.drain()


# ------------------------------------------------------------------------------- checkpoint / files
def generator_kwargs_from_config(cfg: Dict) -> Dict:
    """``generator:`` section of a training config (configs/training/generator/*.yaml, e.g. big-lama.yaml:26-45)
    -> FFCResNetGenerator kwargs, as make_generator does (saicinpainting/training/modules/__init__.py:7-17)."""
    g = dict(cfg["generator"])
    kind = g.pop("kind")
    if kind != "ffc_resnet":
        raise ValueError(f"generator kind {kind!r} is not the FFC generator")
    return g


def load_generator(model_dir: str, checkpoint: str = "best.ckpt", device: str = "cuda"):
    """Build the drop-in generator from ``<model_dir>/config.yaml`` and load ``<model_dir>/models/<checkpoint>``
    (a Lightning checkpoint: generator weights live under the ``generator.`` prefix of ``state_dict`` —
    saicinpainting/training/trainers/__init__.py:25-30, bin/predict.py:49-59)."""
    import yaml
    from .modules import FFCResNetGenerator
    with open(os.path.join(model_dir, "config.yaml")) as f:
        cfg = yaml.safe_load(f)
    gen = FFCResNetGenerator(**generator_kwargs_from_config(cfg))
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
                    help="images per batch (with --refine: the most; smaller when the step program would not fit)")
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
    return ap


def refiner_kwargs(a: argparse.Namespace) -> Dict:
    """Command-line arguments -> lama_b200.refine.BatchedRefiner keyword arguments."""
    return dict(max_batch=a.batch, modulo=a.pad_mod, n_iters=a.n_iters, lr=a.lr, min_side=a.min_side,
                max_scales=a.max_scales, px_budget=a.px_budget)


def main(argv=None):
    a = build_parser().parse_args(argv)
    # one process per GPU (python -m torch.distributed.run --nproc-per-node N -m lama_b200.predict ...): every rank
    # takes its share of the files; single-process runs see rank 0 of 1
    rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
    device = f"cuda:{os.environ.get('LOCAL_RANK', '0')}"
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
