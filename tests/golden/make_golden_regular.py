"""Generate the LaMa-Regular golden fixtures in this directory from the UNMODIFIED reference.

Run in the build container only (needs the reference tree, see ``oracle/ref_import.py``):

    python tests/golden/make_golden_regular.py

The reference's ``saicinpainting/training/modules/pix2pixhd.py`` (``GlobalGenerator``, kind ``pix2pixhd_global``:
lama-regular, big-lama-regular) is loaded under a private name, with the stubs and path set-up of
``oracle/ref_import.py``.  As in ``make_golden.py``, parameters come from the seeded factory
``lama_b200.testing.seeded_parameters_`` and the module runs in ``eval()`` under ``no_grad`` on CPU fp32.  Fixtures:

* ``global_ngf8_b2_64x64.npz``         a small generator (ngf 8 -> 64 bottleneck channels, 2 blocks), with its state_dict;
* ``global_ngf8_b2_40x72.npz``         the same weights on a 40x72 image (5x9 bottleneck);
* ``predict_global_ngf8_3x45x52.npz``  the same weights through the predict path's uint8 glue (as predict_ngf8_3x45x52);
* ``regular_state_dict_schema.json``   key -> shape of lama-regular's and big-lama-regular's state_dict.
"""
import importlib.util
import json
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle.ref_import import REFERENCE_ROOT, load_reference_ffc  # noqa: E402
from lama_b200.testing import (BIG_LAMA_REGULAR_KWARGS, LAMA_REGULAR_KWARGS, generator_input,  # noqa: E402
                               seeded_parameters_, small_regular_kwargs, synthetic_image_mask)


def load_reference_pix2pixhd():
    """The unmodified reference ``pix2pixhd.py`` under a private name; its imports of ``base`` / ``ffc`` resolve
    through the reference package, set up by ``load_reference_ffc``."""
    load_reference_ffc()
    spec = importlib.util.spec_from_file_location(
        "_lama_reference_pix2pixhd", os.path.join(REFERENCE_ROOT, "saicinpainting/training/modules/pix2pixhd.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _sd_np(module):
    return {"sd::" + k: v.detach().cpu().numpy() for k, v in module.state_dict().items()
            if not k.endswith("num_batches_tracked")}


def _save(name, **arrays):
    path = os.path.join(HERE, name + ".npz")
    np.savez_compressed(path, **arrays)
    print(f"{name:32s} {os.path.getsize(path) / 1024:8.1f} KiB")


def _predict_fixture(g, name):
    """PNG files -> reference InpaintingDataset (saicinpainting/evaluation/data.py, imported from its file) -> ``g`` ->
    bytes.  DefaultInpaintingTrainingModule.forward and bin/predict.py need pytorch_lightning / hydra to import, so the
    lines of theirs on this path are restated below with their file:line."""
    from PIL import Image
    spec = importlib.util.spec_from_file_location(
        "_ref_eval_data", os.path.join(REFERENCE_ROOT, "saicinpainting/evaluation/data.py"))
    data = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(data)
    rng = np.random.default_rng(7)
    b, h0, w0 = 3, 45, 52
    images = rng.integers(0, 256, size=(b, h0, w0, 3), dtype=np.uint8)
    images[0, :, :, :] = (np.linspace(0, 255, w0)[None, :, None] + np.zeros((h0, 1, 3))).astype(np.uint8)  # ramp
    masks = np.zeros((b, h0, w0), dtype=np.uint8)
    masks[0, 10:30, 12:40] = 255
    masks[1, 30:, 35:] = 255                 # touches the symmetric padding
    masks[1, 5:9, 5:9] = 1                   # "mask > 0" binarisation (predict.py:83)
    masks[2, ::7, ::5] = 128
    with tempfile.TemporaryDirectory() as d:
        for i in range(b):
            Image.fromarray(images[i]).save(os.path.join(d, f"im{i}.png"))
            Image.fromarray(masks[i]).save(os.path.join(d, f"im{i}_mask.png"))
        ds = data.InpaintingDataset(d, img_suffix=".png", pad_out_to_modulo=8)       # default.yaml:8-11
        items = [ds[i] for i in range(len(ds))]
    img = torch.from_numpy(np.stack([it["image"] for it in items]))
    mask = (torch.from_numpy(np.stack([it["mask"] for it in items])) > 0) * 1        # bin/predict.py:83
    unpad = items[0]["unpad_to_size"]
    masked_img = torch.cat([img * (1 - mask), mask], dim=1)                           # trainers/default.py:59,68
    predicted = g(masked_img)                                                         # trainers/default.py:70
    inpainted = mask * predicted + (1 - mask) * img                                   # trainers/default.py:71
    outs = []
    for i in range(b):
        cur = inpainted[i].permute(1, 2, 0).numpy()[:unpad[0], :unpad[1]]            # bin/predict.py:85-91
        outs.append(np.clip(cur * 255, 0, 255).astype("uint8"))                       # bin/predict.py:93
    _save(name, images=images, masks=masks, x=masked_img.numpy(), predicted=predicted.numpy(), out=np.stack(outs))


@torch.no_grad()
def main():
    p2p = load_reference_pix2pixhd()
    torch.set_num_threads(1)
    g = seeded_parameters_(p2p.GlobalGenerator(**small_regular_kwargs(ngf=8, n_blocks=2)).eval(), seed=51, gain=1.0)
    img, mask = synthetic_image_mask(2, 64, seed=5)
    x = generator_input(img, mask)
    _save("global_ngf8_b2_64x64", image=img.numpy(), mask=mask.numpy(), x=x.numpy(), y=g(x).numpy(), **_sd_np(g))
    img, mask = synthetic_image_mask(1, 40, seed=6, width=72)
    x = generator_input(img, mask)
    # same weights as global_ngf8_b2_64x64 (state_dict stored there only)
    _save("global_ngf8_b2_40x72", x=x.numpy(), y=g(x).numpy())
    _predict_fixture(g, "predict_global_ngf8_3x45x52")
    schema = {name: {k: list(v.shape) for k, v in p2p.GlobalGenerator(**kw).state_dict().items()}
              for name, kw in (("lama-regular", LAMA_REGULAR_KWARGS), ("big-lama-regular", BIG_LAMA_REGULAR_KWARGS))}
    path = os.path.join(HERE, "regular_state_dict_schema.json")
    with open(path, "w") as f:
        json.dump(schema, f)
    print(f"{'regular_state_dict_schema':32s} {os.path.getsize(path) / 1024:8.1f} KiB")


if __name__ == "__main__":
    main()
