"""LaMa-Regular generators (``lama_b200.pix2pixhd``, kind ``pix2pixhd_global``) without a GPU: the module surface
against the goldens and the reference's state_dict schema, the generator programs interpreted on the CPU, the pinned
op list and storage, the reference factory after ``patch.install()``, and the predict entry points."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR, ROOT, load_golden
from lama_b200 import _lib as L
from lama_b200 import engine as E
from lama_b200 import pix2pixhd as PX
from lama_b200 import predict as PR
from lama_b200.testing import (BIG_LAMA_REGULAR_KWARGS, LAMA_REGULAR_KWARGS, seeded_parameters_,
                               small_regular_kwargs)
from spec_interp import SpecInterpreter, check_liveness

MATHS = {"fp32": L.MATH_FP32, "bf16x3": L.MATH_BF16X3}


@pytest.fixture(autouse=True)
def _not_strict(monkeypatch):
    monkeypatch.delenv("LAMA_B200_STRICT", raising=False)       # the CPU runs the torch composition


def _small():
    _, sd = load_golden("global_ngf8_b2_64x64")
    g = PX.GlobalGenerator(**small_regular_kwargs(8, 2))
    g.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=False)
    return g.eval()


def _program(gen, kind, shapes, math):
    with torch.no_grad():
        prog = E.build_module_program(gen, kind, shapes, MATHS[math])
    assert prog.math == MATHS[math]
    return prog


# ------------------------------------------------------------------------------------------- module surface
@pytest.mark.parametrize("name", ["global_ngf8_b2_64x64", "global_ngf8_b2_40x72"])
def test_torch_composition_matches_golden(name):
    a, _ = load_golden(name)
    with torch.no_grad():
        y = _small()(torch.from_numpy(a["x"])).numpy()
    assert float(np.abs(y - a["y"]).max()) < 1e-6


@pytest.mark.parametrize("config,kw", [("lama-regular", LAMA_REGULAR_KWARGS),
                                       ("big-lama-regular", BIG_LAMA_REGULAR_KWARGS)])
def test_state_dict_round_trips_against_the_reference_schema(config, kw):
    with open(os.path.join(GOLDEN_DIR, "regular_state_dict_schema.json")) as f:
        schema = json.load(f)[config]
    g = PX.GlobalGenerator(**kw)
    assert {k: list(v.shape) for k, v in g.state_dict().items()} == schema
    # a state_dict with exactly the reference's keys loads strictly, and the drop-in's loads into the reference's shape
    sd = {k: torch.zeros(s, dtype=torch.long if k.endswith("num_batches_tracked") else torch.float32)
          for k, s in schema.items()}
    g.load_state_dict(sd, strict=True)
    assert sorted(g.state_dict()) == sorted(schema)


def test_reference_loads_the_drop_in_state_dict_and_back():
    from oracle import ref_import
    if not ref_import.available():
        pytest.skip("reference tree not present")
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    try:
        from make_golden_regular import load_reference_pix2pixhd
    finally:
        sys.path.pop(0)
    ref = load_reference_pix2pixhd()
    kw = small_regular_kwargs(8, 2)
    mine = seeded_parameters_(PX.GlobalGenerator(**kw).eval(), 1)
    theirs = ref.GlobalGenerator(**kw).eval()
    theirs.load_state_dict(mine.state_dict(), strict=True)
    back = PX.GlobalGenerator(**kw).eval()
    back.load_state_dict(theirs.state_dict(), strict=True)
    x = torch.rand(1, 4, 32, 32, generator=torch.Generator().manual_seed(0))
    with torch.no_grad():
        assert torch.equal(theirs(x), back(x))


def test_options_outside_the_native_path():
    kw = small_regular_kwargs(8, 1)
    x = torch.empty(1, 4, 64, 64, device="meta")
    assert E.generator_supported(PX.GlobalGenerator(**kw), x)
    for over in (dict(norm_layer="in"), dict(padding_type="zero"), dict(padding_type="replicate"), dict(dilation=2),
                 dict(dilated_blocks_n=1), dict(is_resblock_depthwise=True), dict(affine=False),
                 dict(activation=torch.nn.LeakyReLU(0.2)),
                 dict(ffc_positions=[0], ffc_kwargs=dict(ratio_gin=0.75, ratio_gout=0.75, enable_lfu=False))):
        g = PX.GlobalGenerator(**dict(kw, **over))
        assert E._global_layout(g) is None and not E.generator_supported(g, x), over
    for over in (dict(conv_kind="depthwise"), dict(conv_kind="multidilated"),
                 dict(dilation_block_kind="multi", dilated_blocks_n=1)):
        assert PX.reference_only_options(**over)
        with pytest.raises(NotImplementedError):
            PX.GlobalGenerator(**dict(kw, **over))


def test_size_gate():
    g = PX.GlobalGenerator(**LAMA_REGULAR_KWARGS)
    ok = lambda h, w, c=4: E.generator_supported(g, torch.empty(1, c, h, w, device="meta"))  # noqa: E731
    assert ok(512, 512) and ok(16, 16) and ok(1024, 9216) and ok(8200, 8200)    # no FFT: no 1024-point limit
    assert not ok(8, 8) and not ok(512, 516) and not ok(512, 512, c=3)
    assert E.generator_in_channels(g) == 4


# ------------------------------------------------------------------------------------------- programs
@pytest.mark.parametrize("math", ["fp32", "bf16x3"])
@pytest.mark.parametrize("name", ["global_ngf8_b2_64x64", "global_ngf8_b2_40x72"])
def test_generator_program_interpreted(name, math):
    a, _ = load_golden(name)
    prog = _program(_small(), "generator", (a["x"].shape,), math)
    check_liveness(prog)
    y = SpecInterpreter(prog).run({"x0": torch.from_numpy(a["x"])})["y0"].numpy()
    assert float(np.abs(y - a["y"]).max()) < 1e-5


def test_u8_program_interpreted():
    a, _ = load_golden("predict_global_ngf8_3x45x52")
    prog = _program(_small(), "generator_u8:8", (a["images"].shape, a["masks"].shape), "bf16x3")
    out = SpecInterpreter(prog).run({"img": torch.from_numpy(a["images"]),
                                     "mask": torch.from_numpy(a["masks"])})["y0"].numpy()
    hole = a["masks"] > 0
    assert np.array_equal(out[~hole], a["out"][~hole])
    d = np.abs(out[hole].astype(int) - a["out"][hole].astype(int))
    assert d.max() <= 1 and (d != 0).mean() < 0.05


_UP = [(f"convT phase {a}{b}+bn+relu", 0, 1) for a in (0, 1) for b in (0, 1)]
_OPS_TC = ([("StemPackOp", None, None, None), ("ConvOp", "stem 7x7 (windowed)+bn+relu", 0, 1)]
           + [("ConvOp", "down 3x3 s2 (zero border)+bn+relu", 0, 2)] * 3
           + [("ConvOp", "block conv1+bn1+relu", 1, 1), ("ConvOp", "block conv2+bn2 + x", 1, 1)] * 2
           + [("ConvOp",) + u for u in _UP] + [("BorderOp", None, None, None)]
           + [("ConvOp",) + u for u in _UP] + [("BorderOp", None, None, None)]
           + [("ConvOp",) + u for u in _UP] + [("BorderOp", None, None, None)]
           + [("ConvOp", "head 7x7 rows", 1, 1), ("HeadGatherOp", None, None, None)])


def _ops(prog):
    out = []
    for op in prog.ops:
        pk = getattr(op, "packed", None)
        out.append((type(op).__name__, getattr(op, "tag", None), pk.border if pk else None, pk.stride if pk else None))
    return out


def test_op_list_pinned():
    """The ngf 8 program on both arms: op kinds, tags, borders and strides; and the buffer wiring of the bf16x3 arm
    (the blocks run in place on the last down's buffer, one Y per block, pooled)."""
    tc = _program(_small(), "generator", ((2, 4, 64, 64),), "bf16x3")
    assert _ops(tc) == _OPS_TC
    views = [([(t.buf.name, t.c0, t.channels) for t in op.views()[0]],
              [(t.buf.name, t.c0, t.channels, t.phase) for t in op.views()[1]]) for op in tc.ops[2:9]]
    assert views == [([("stem#0", 0, 8)], [("down#2", 0, 16, None)]),
                     ([("down#2", 0, 16)], [("down#3", 0, 32, None)]),
                     ([("down#3", 0, 32)], [("down#4", 0, 64, None)]),
                     ([("down#4", 0, 64)], [("block.y#5", 0, 64, None)]),
                     ([("block.y#5", 0, 64), ("down#4", 0, 64)], [("down#4", 0, 64, None)]),
                     ([("down#4", 0, 64)], [("block.y#6", 0, 64, None)]),
                     ([("block.y#6", 0, 64), ("down#4", 0, 64)], [("down#4", 0, 64, None)])]
    slots = E.assign_storage_slots(tc)
    assert slots["block.y#5"] == slots["block.y#6"]
    assert all(b.fmt == L.BF16X2 and b.pad == 1 for b in tc.bufs if b.name.startswith(("down", "block", "stem#")))
    f32 = _program(_small(), "generator", ((2, 4, 64, 64),), "fp32")
    want = ([("StemOp", None, None, None)] + [t for t in _OPS_TC[2:] if t[0] == "ConvOp" and t[1] != "head 7x7 rows"]
            + [("HeadOp", None, None, None)])
    assert _ops(f32) == want


def test_program_storage_of_lama_regular_at_bs32_512():
    """Device bytes of the lama-regular program at bs32 512x512 (DESIGN.md §6): 7.76 GB on the bf16x3 arm."""
    g = PX.GlobalGenerator(**LAMA_REGULAR_KWARGS).eval()
    assert E.program_storage_bytes(_program(g, "generator", ((32, 4, 512, 512),), "bf16x3")) == 7759511568
    assert E.program_storage_bytes(_program(g, "generator", ((32, 4, 512, 512),), "fp32")) == 4395630608


# ------------------------------------------------------------------------------------------- patch and predict
def test_reference_factory_builds_the_drop_in():
    """In a fresh interpreter with the reference present: after install(), make_generator('pix2pixhd_global') builds
    the drop-in, depthwise convs the reference's class, ResnetBlock stays the reference's; uninstall() restores both
    import sites."""
    from oracle import ref_import
    if not ref_import.available():
        pytest.skip("reference tree not present")
    code = (
        "import sys; sys.path.insert(0, %r); sys.path.append(%r)\n"
        "from oracle import ref_import; ref_import._install_stubs()\n"
        "import lama_b200.patch as p; p.install()\n"
        "from saicinpainting.training.modules import make_generator\n"
        "import saicinpainting.training.modules as pkg\n"
        "import saicinpainting.training.modules.pix2pixhd as p2p\n"
        "from lama_b200 import pix2pixhd as PX\n"
        "from lama_b200.testing import LAMA_REGULAR_KWARGS as KW\n"
        "ref = p2p.GlobalGenerator.reference\n"
        "assert ref.__module__ == 'saicinpainting.training.modules.pix2pixhd'\n"
        "assert type(make_generator(None, kind='pix2pixhd_global', **KW)) is PX.GlobalGenerator\n"
        "assert type(make_generator(None, kind='pix2pixhd_global', **dict(KW, conv_kind='depthwise'))) is ref\n"
        "assert p2p.ResnetBlock is not PX.ResnetBlock\n"
        "p.uninstall()\n"
        "assert pkg.GlobalGenerator is ref and p2p.GlobalGenerator is ref\n"
        "assert type(make_generator(None, kind='pix2pixhd_global', **KW)) is ref\n"
        "print('ok')\n" % (ROOT, ref_import.REFERENCE_ROOT))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "ok" in r.stdout, r.stderr[-2000:]


def _model_dir(tmp_path, kw, kind="pix2pixhd_global", ckpt=True):
    import yaml
    d = tmp_path / "model"
    (d / "models").mkdir(parents=True)
    with open(d / "config.yaml", "w") as f:
        yaml.safe_dump({"generator": dict(kind=kind, **kw), "discriminator": {"kind": "pix2pixhd_nlayer"}}, f)
    g = None
    if ckpt:
        g = seeded_parameters_(PX.GlobalGenerator(**kw).eval(), 3)
        torch.save({"state_dict": {**{"generator." + k: v for k, v in g.state_dict().items()},
                                   "discriminator.model0.0.weight": torch.zeros(1)}}, d / "models" / "best.ckpt")
    return d, g


def test_load_generator_reads_a_regular_model(tmp_path):
    kw = small_regular_kwargs(8, 2)
    d, g = _model_dir(tmp_path, kw)
    g2 = PR.load_generator(str(d), device="cpu")
    assert type(g2) is PX.GlobalGenerator and not g2.training
    for (k, a), (_, b) in zip(g.state_dict().items(), g2.state_dict().items()):
        assert torch.equal(a, b), k
    assert type(PR.generator_from_config({"generator": dict(kind="pix2pixhd_global", **kw)})) is PX.GlobalGenerator
    with pytest.raises(ValueError, match="pix2pixhd_multidilated"):
        PR.generator_from_config({"generator": {"kind": "pix2pixhd_multidilated"}})


def test_refine_with_a_regular_model_raises_before_reading_files(tmp_path):
    d, _ = _model_dir(tmp_path, small_regular_kwargs(8, 2), ckpt=False)
    with pytest.raises(ValueError, match="pix2pixhd_global"):
        PR.main(["--model-dir", str(d), "--indir", str(tmp_path / "missing"), "--outdir", str(tmp_path / "out"),
                 "--refine"])
    assert not (tmp_path / "out").exists()
