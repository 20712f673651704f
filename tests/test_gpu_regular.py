"""LaMa-Regular generators (``lama_b200.pix2pixhd.GlobalGenerator``: lama-regular, big-lama-regular) on the GPU.

1. Op by op (``diff_program`` of test_gpu_program_diff.py): every op of the small (ngf 8) program, float and uint8
   variants, and of a program with lama-regular's widths at 64x64 and 48x80 bottleneck planes is judged on the device
   state it read.  This covers the two contractions these models add to ``conv_tc_kernel``: the 512 -> 512 3x3
   reflect contraction in column-halo mode with four N tiles, and the 3x3 stride-2 zero-border contraction as a
   forward layer.
2. The module against the goldens from the unmodified reference, and seeded lama-regular at 512x512 and 1024x768
   (batch 2) against the float64 composition of the same layers, on both arithmetic arms.
3. Batch independence, graph replay = eager bit for bit, a 1024x9216 image (128x1152 bottleneck) natively, and the
   predict command line on a lama-regular model directory.
"""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from conftest import load_golden                     # noqa: E402
from lama_b200 import _lib as L                      # noqa: E402
from lama_b200 import engine as E                    # noqa: E402
from lama_b200 import pix2pixhd as PX                # noqa: E402
from lama_b200.testing import (LAMA_REGULAR_KWARGS, generator_input, seeded_parameters_,  # noqa: E402
                               small_regular_kwargs, synthetic_image_mask)
from test_gpu_program_diff import diff_program       # noqa: E402

DEV = "cuda:0"
MATHS = {"fp32": L.MATH_FP32, "bf16x3": L.MATH_BF16X3}
TIGHT = {"fp32": 5e-5, "bf16x3": 3e-4}               # max-abs vs float64, the bounds big-lama is held to


@pytest.fixture(autouse=True, scope="module")
def _need_gpu():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    L.check(L.get_lib().ffcb_check_device(0), "ffcb_check_device")


@pytest.fixture(autouse=True)
def _strict_env():
    os.environ["LAMA_B200_STRICT"] = "1"
    yield
    os.environ.pop("LAMA_B200_STRICT", None)


@pytest.fixture(params=["fp32", "bf16x3"])
def math_mode(request):
    os.environ["LAMA_B200_MATH"] = request.param
    yield request.param
    os.environ.pop("LAMA_B200_MATH", None)


def _small():
    _, sd = load_golden("global_ngf8_b2_64x64")
    g = PX.GlobalGenerator(**small_regular_kwargs(8, 2))
    g.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=False)
    return g.eval().to(DEV)


def _regular(seed, **over):
    return seeded_parameters_(PX.GlobalGenerator(**dict(LAMA_REGULAR_KWARGS, **over)).eval(), seed, gain=1.0)


def _diff(gen, kind, shapes, feed, math):
    with torch.no_grad():
        prog = E.build_module_program(gen, kind, shapes, MATHS[math])
    assert prog.math == MATHS[math], "the program fell back to the other arithmetic"
    bad = diff_program(prog, feed)
    assert not bad, "ops that disagree with the interpreter:\n" + "\n".join(
        f"  {lab}: {err:.3e} > {tol:g}" for _, lab, err, tol in bad)
    return prog


# ------------------------------------------------------------------------------------------- op by op
@pytest.mark.parametrize("math", ["fp32", "bf16x3"])
def test_small_program_op_by_op(math):
    a, _ = load_golden("global_ngf8_b2_64x64")
    _diff(_small(), "generator", ((2, 4, 64, 64),), {"x0": torch.from_numpy(a["x"])}, math)


def test_small_u8_program_op_by_op():
    a, _ = load_golden("predict_global_ngf8_3x45x52")
    feed = {"img": torch.from_numpy(a["images"]), "mask": torch.from_numpy(a["masks"])}
    _diff(_small(), "generator_u8:8", (a["images"].shape, a["masks"].shape), feed, "bf16x3")


@pytest.mark.parametrize("math", ["fp32", "bf16x3"])
@pytest.mark.parametrize("h,w", [(512, 512), (384, 640)])
def test_lama_regular_program_op_by_op(h, w, math):
    """lama-regular's layers (two of its nine identical blocks) at 64x64 and 48x80 bottleneck planes: the 512-channel
    block contractions (four N tiles) and the stride-2 zero-border downs at every width of the model."""
    g = _regular(3, n_blocks=2).to(DEV)
    img, mask = synthetic_image_mask(1, h, 2, width=w)
    prog = _diff(g, "generator", ((1, 4, h, w),), {"x0": generator_input(img, mask)}, math)
    tags = [op.packed.n_out for op in prog.ops if isinstance(op, E.ConvOp) and op.tag.startswith("block")]
    assert tags == [512] * 4


# ------------------------------------------------------------------------------------------- module level
@pytest.mark.parametrize("name", ["global_ngf8_b2_64x64", "global_ngf8_b2_40x72"])
def test_small_generator_golden(name, math_mode):
    a, _ = load_golden(name)
    g = _small()
    L.get_lib().ffcb_reset_launch_count()
    with torch.no_grad():
        y = g(torch.from_numpy(a["x"]).to(DEV)).cpu().numpy()
    assert L.get_lib().ffcb_launch_count() > 0, "the native program did not run"
    assert float(np.abs(y - a["y"]).max()) < TIGHT[math_mode]


@pytest.mark.parametrize("h,w", [(512, 512), (768, 1024)])
def test_lama_regular_vs_float64(h, w, math_mode):
    """Seeded lama-regular, batch 2, against the float64 composition of the same layers (``self.model`` in float64,
    evaluated on the device)."""
    g = _regular(0).to(DEV)
    img, mask = synthetic_image_mask(2, h, 1, width=w)
    x = generator_input(img, mask).to(DEV)
    with torch.no_grad():
        y = g(x)
        ref = g.double().model(x.double())
    err = float((y.double() - ref).abs().max())
    print(f"lama-regular {h}x{w} bs2 ({math_mode}): max-abs {err:.2e}, output std {float(ref.std()):.3f}")
    assert float(ref.std()) > 0.05, "degenerate (saturated) reference output"
    assert err < TIGHT[math_mode], err


def test_batch_independence_and_graph_replay():
    """bs8 at 512x512: each image equals the same image run in a batch of 2, bit for bit; a CUDA-graph replay of the
    program equals the eager run, bit for bit."""
    g = _regular(1).to(DEV)
    img, mask = synthetic_image_mask(8, 512, 4)
    x = generator_input(img, mask).to(DEV)
    with torch.no_grad():
        y8 = g(x)
        y2 = torch.cat([g(x[i:i + 2].contiguous()) for i in range(0, 8, 2)])
        ex = E.get_executor(g, "generator", (x,))
        graph = E.GraphedProgram(ex)
        yg = graph({"x0": x})["y0"].clone()
    assert torch.equal(y8, y2), "results depend on the batch composition"
    assert torch.equal(yg, y8), "graph replay differs from the eager run"


def test_wide_image_beyond_the_fft_limit():
    """1024x9216 (bottleneck 128x1152, wider than the FFC generator's 1024-point FFT limit) runs natively and
    matches the float64 composition."""
    g = _regular(2).to(DEV)
    img, mask = synthetic_image_mask(1, 1024, 5, width=9216)
    x = generator_input(img, mask).to(DEV)
    assert E.generator_supported(g, x)
    L.get_lib().ffcb_reset_launch_count()
    with torch.no_grad():
        y = g(x)
        assert L.get_lib().ffcb_launch_count() > 0, "the native program did not run"
        E.invalidate(g)
        err = float((y.double() - g.double().model(x.double())).abs().max())
    print(f"lama-regular 1024x9216: max-abs {err:.2e}")
    assert err < 3e-4, err


def test_predict_command_line(tmp_path):
    """``python -m lama_b200.predict`` on a lama-regular model directory (config.yaml + Lightning checkpoint) writes
    the bytes of the reference pipeline (tests/golden/predict_global_ngf8_3x45x52.npz): exact outside the hole,
    within one grey level inside it."""
    import yaml
    from PIL import Image
    from lama_b200 import predict as PR
    a, _ = load_golden("predict_global_ngf8_3x45x52")
    _, sd = load_golden("global_ngf8_b2_64x64")
    model = tmp_path / "lama-regular"
    (model / "models").mkdir(parents=True)
    with open(model / "config.yaml", "w") as f:
        yaml.safe_dump({"generator": dict(kind="pix2pixhd_global", **small_regular_kwargs(8, 2))}, f)
    g = PX.GlobalGenerator(**small_regular_kwargs(8, 2))
    g.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=False)
    torch.save({"state_dict": {"generator." + k: v for k, v in g.state_dict().items()}}, model / "models" / "best.ckpt")
    indir, outdir = tmp_path / "in", tmp_path / "out"
    indir.mkdir()
    for i in range(len(a["images"])):
        Image.fromarray(a["images"][i]).save(indir / f"im{i}.png")
        Image.fromarray(a["masks"][i]).save(indir / f"im{i}_mask.png")
    os.environ["LAMA_B200_MATH"] = "bf16x3"
    try:
        PR.main(["--model-dir", str(model), "--indir", str(indir), "--outdir", str(outdir), "--batch", "2"])
    finally:
        os.environ.pop("LAMA_B200_MATH", None)
    outs = np.stack([np.array(Image.open(outdir / f"im{i}_mask.png")) for i in range(len(a["images"]))])
    hole = a["masks"] > 0
    assert outs.shape == a["out"].shape
    assert np.array_equal(outs[~hole], a["out"][~hole])
    d = np.abs(outs[hole].astype(int) - a["out"][hole].astype(int))
    assert d.max() <= 1 and (d != 0).mean() < 0.05, (int(d.max()), float((d != 0).mean()))
