"""Host logic of the product (program building, BN folding, weight packing, buffer wiring) checked
on the CPU box: programs built by lama_b200.engine from the drop-in modules are interpreted by
tests/spec_interp.py and compared with the goldens generated from the unmodified reference."""
import numpy as np
import pytest
import torch

from conftest import load_golden
from lama_b200 import _lib as L
from lama_b200 import engine as E
from lama_b200 import modules as M
from lama_b200.testing import small_lama_kwargs
from spec_interp import SpecInterpreter


def _load(module, sd):
    missing, unexpected = module.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=False)
    assert not unexpected and all(k.endswith("num_batches_tracked") for k in missing), (missing, unexpected)
    return module.eval()


def _run(module, kind, tensors):
    shapes = tuple(tuple(t.shape) if torch.is_tensor(t) else None for t in tensors)
    with torch.no_grad():
        prog = E.build_module_program(module, kind, shapes, L.MATH_FP32)
    feed = {f"x{i}": t for i, t in enumerate(t for t in tensors if torch.is_tensor(t))}
    return SpecInterpreter(prog).run(feed), prog


def _close(got, ref, rel=2e-6):
    scale = float(np.abs(ref).max()) or 1.0
    err = float(np.abs(got.numpy() - ref.astype(np.float64)).max())
    assert err <= rel * scale, f"{err:.3e} > {rel:g}*{scale:.3e}"


@pytest.mark.parametrize("name,ci,co", [("fu_c8_16x16", 8, 8), ("fu_c4to6_8x32", 4, 6), ("fu_c16_32x32", 16, 16),
                                        ("fu_c4_15x15", 4, 4), ("fu_c4_6x9", 4, 4)])
def test_fourier_unit_program(name, ci, co):
    a, sd = load_golden(name)
    m = _load(M.FourierUnit(ci, co), sd)
    if not m.native_supported():
        pytest.skip("channel count outside the native path")
    out, _ = _run(m, "fourier_unit", (torch.from_numpy(a["x"]),))
    _close(out["y0"], a["y"])


def test_spectral_transform_program():
    a, sd = load_golden("st_16to24_8x8")
    m = _load(M.SpectralTransform(16, 24, enable_lfu=False), sd)
    assert m.native_supported()
    out, _ = _run(m, "spectral_transform", (torch.from_numpy(a["x"]),))
    _close(out["y0"], a["y"])


@pytest.mark.parametrize("name,ci,co,stride,lfu", [("st_16to16_s2_16x16", 16, 16, 2, False),
                                                    ("st_32to64_s2_12x20", 32, 64, 2, False),
                                                    ("st_32to32_lfu_8x8", 32, 32, 1, True),
                                                    ("st_32to32_s2_lfu_16x16", 32, 32, 2, True)])
def test_spectral_transform_stride2_and_lfu_programs(name, ci, co, stride, lfu):
    """SURVEY.md row f4: AvgPool2d(2,2) + conv1 as one 2x2 stride-2 contraction (ffc.py:122-125, 145); LFU as four
    quadrant FFTs into channel slices of one spectrum, one spectral GEMM, four tiled inverses (ffc.py:148-157)."""
    a, sd = load_golden(name)
    m = _load(M.SpectralTransform(ci, co, stride=stride, enable_lfu=lfu), sd)
    x = torch.from_numpy(a["x"])
    assert m.native_supported(tuple(x.shape[-2:]))
    out, prog = _run(m, "spectral_transform", (x,))
    _close(out["y0"], a["y"])
    assert sum(isinstance(o, E.RfftOp) for o in prog.ops) == (5 if lfu else 1)
    assert sum(isinstance(o, E.IrfftOp) for o in prog.ops) == (5 if lfu else 1)


def test_spectral_pos_encoding_programs():
    """ffc.py:91-95: the two coordinate channels are data independent, so they enter the spectral GEMM as a
    per-position addend (BN scale folded) broadcast over the batch — FourierUnit alone and inside SpectralTransform."""
    a, sd = load_golden("fu_c8_pos_12x16")
    m = _load(M.FourierUnit(8, 8, spectral_pos_encoding=True), sd)
    assert m.native_supported()
    out, prog = _run(m, "fourier_unit", (torch.from_numpy(a["x"]),))
    _close(out["y0"], a["y"])
    assert len(prog.consts) == 1
    a, sd = load_golden("st_16to32_pos_8x8")
    m = _load(M.SpectralTransform(16, 32, enable_lfu=False, spectral_pos_encoding=True), sd)
    out, _ = _run(m, "spectral_transform", (torch.from_numpy(a["x"]),))
    _close(out["y0"], a["y"])


def test_ffc_bn_act_stride2_global_with_lfu_program():
    a, sd = load_golden("ffcbnact_64_s2_lfu_16x16")
    m = _load(M.FFC_BN_ACT(in_channels=64, out_channels=64, kernel_size=3, ratio_gin=0.5, ratio_gout=0.5, stride=2,
                           padding=1, activation_layer=torch.nn.ReLU, enable_lfu=True), sd)
    xl, xg = torch.from_numpy(a["x_l"]), torch.from_numpy(a["x_g"])
    assert m.native_supported() and E.ffc_bn_act_shapes_ok(m, xl, xg)
    out, _ = _run(m, "ffc_bn_act", (xl, xg))
    _close(out["y0"], a["y_l"]); _close(out["y1"], a["y_g"])
    # LFU only type-checks for even square planes (the reference splits rows and columns by h // 2): 12 x 20 -> torch
    assert not E.ffc_bn_act_shapes_ok(m, torch.zeros(1, 32, 12, 20), torch.zeros(1, 32, 12, 20))


def test_resnet_block_with_lfu_program():
    a, sd = load_golden("resblock_64_lfu_8x8")
    m = _load(M.FFCResnetBlock(64, padding_type="reflect", norm_layer=torch.nn.BatchNorm2d,
                               activation_layer=torch.nn.ReLU, ratio_gin=0.5, ratio_gout=0.5, enable_lfu=True), sd)
    assert m.native_supported()
    out, _ = _run(m, "resnet_block", (torch.from_numpy(a["x_l"]), torch.from_numpy(a["x_g"])))
    _close(out["y0"], a["y_l"]); _close(out["y1"], a["y_g"])


@pytest.mark.parametrize("name,kw,has_g", [
    ("ffcbnact_32_k3_075", dict(in_channels=32, out_channels=32, kernel_size=3, ratio_gin=0.75, ratio_gout=0.75,
                                padding=1), True),
    ("ffcbnact_4to8_k7_local", dict(in_channels=4, out_channels=8, kernel_size=7, ratio_gin=0, ratio_gout=0,
                                    padding=0), False),
    ("ffcbnact_16to32_s2_to_global", dict(in_channels=16, out_channels=32, kernel_size=3, ratio_gin=0,
                                          ratio_gout=0.75, stride=2, padding=1), False),
])
def test_ffc_bn_act_program(name, kw, has_g):
    a, sd = load_golden(name)
    m = _load(M.FFC_BN_ACT(activation_layer=torch.nn.ReLU, enable_lfu=False, **kw), sd)
    assert m.native_supported()
    xl = torch.from_numpy(a["x_l"]); xg = torch.from_numpy(a["x_g"]) if has_g else 0
    assert E.ffc_bn_act_shapes_ok(m, xl, xg)
    out, _ = _run(m, "ffc_bn_act", (xl, xg))
    _close(out["y0"], a["y_l"])
    if "y_g" in a:
        _close(out["y1"], a["y_g"])


def test_resnet_block_program():
    a, sd = load_golden("resblock_32_16x16")
    m = _load(M.FFCResnetBlock(32, padding_type="reflect", norm_layer=torch.nn.BatchNorm2d,
                               activation_layer=torch.nn.ReLU, ratio_gin=0.75, ratio_gout=0.75, enable_lfu=False), sd)
    assert m.native_supported()
    out, prog = _run(m, "resnet_block", (torch.from_numpy(a["x_l"]), torch.from_numpy(a["x_g"])))
    _close(out["y0"], a["y_l"]); _close(out["y1"], a["y_g"])
    # two FFC_BN_ACT = 2 x (local conv, conv1, fu conv, global conv) contractions, 2 FFT pairs
    assert sum(isinstance(o, E.ConvOp) for o in prog.ops) == 8
    assert sum(isinstance(o, E.RfftOp) for o in prog.ops) == 2


@pytest.mark.parametrize("name", ["generator_ngf8_b2_64x64", "generator_ngf8_b2_40x72"])
def test_generator_program(name):
    a, _ = load_golden(name)
    _, sd = load_golden("generator_ngf8_b2_64x64")
    g = _load(M.FFCResNetGenerator(**small_lama_kwargs(ngf=8, n_blocks=2)), sd)
    x = torch.from_numpy(a["x"])
    assert E.generator_supported(g, x)
    out, prog = _run(g, "generator", (x,))
    assert float(np.abs(out["y0"].numpy() - a["y"]).max()) < 2e-6
    # residual blocks run in place on one bottleneck buffer: no per-block output allocation
    assert not any(b.name.startswith("block.out") for b in prog.bufs)


def test_generator_with_out_ffc_program():
    """out_ffc=True (ffc.py:356-358): the inline FFCResnetBlock before the head joins the one generator program."""
    a, sd = load_golden("generator_ngf16_outffc_32x32")
    kw = small_lama_kwargs(ngf=16, n_blocks=1, n_downsampling=2)
    kw.update(out_ffc=True, out_ffc_kwargs=dict(ratio_gin=0.5, ratio_gout=0.5, enable_lfu=False))
    g = _load(M.FFCResNetGenerator(**kw), sd)
    x = torch.from_numpy(a["x"])
    assert E.generator_supported(g, x)
    out, prog = _run(g, "generator", (x,))
    assert float(np.abs(out["y0"].numpy() - a["y"]).max()) < 2e-6
    assert sum(isinstance(o, E.RfftOp) for o in prog.ops) == 4          # 1 bottleneck block + the out_ffc block


def test_unsupported_options_are_not_native():
    assert M.FourierUnit(8, 8, spectral_pos_encoding=True).eval().native_supported()        # native since round 2
    assert not M.FourierUnit(8, 8, use_se=True).eval().native_supported()
    assert not M.FourierUnit(8, 8, fft_norm="backward").eval().native_supported()
    assert not M.SpectralTransform(16, 16, enable_lfu=True).eval().native_supported()       # c/4 = 2 channels
    lf = M.SpectralTransform(32, 32, enable_lfu=True).eval()
    assert lf.native_supported() and lf.native_supported((8, 8)) and not lf.native_supported((8, 12))
    assert not M.FFC_BN_ACT(16, 16, 3, 0.5, 0.5, padding=1, enable_lfu=False, gated=True).eval().native_supported()
    assert not M.FFC_BN_ACT(16, 16, 3, 0.5, 0.5, padding=2, dilation=2, enable_lfu=False).eval().native_supported()
    m = M.FFC_BN_ACT(16, 16, 3, 0.5, 0.5, padding=1, enable_lfu=False)
    assert not m.train().native_supported() and m.eval().native_supported()


def test_bf16x3_program_layout_and_semantics():
    """FFCB_MATH_BF16X3 programs: GEMM operands are split-bf16, 3x3 operands carry a reflected ring,
    FFT inputs / spectra leaving the GEMM / the head input stay float32, ring-less producers are
    followed by a BorderOp — and the op list still computes the golden output."""
    a, sd = load_golden("generator_ngf8_b2_64x64")
    g = _load(M.FFCResNetGenerator(**small_lama_kwargs(ngf=8, n_blocks=2)), sd)
    x = torch.from_numpy(a["x"])
    with torch.no_grad():
        prog = E.build_module_program(g, "generator", (tuple(x.shape),), L.MATH_BF16X3)
    assert prog.math == L.MATH_BF16X3 and E.tc_compatible(prog)
    by = {b.name.split("#")[0]: b for b in prog.bufs}
    assert by["stem"].fmt == L.BF16X2 and by["stem"].pad == 1 and by["stem"].reflect_border == 1
    assert by["spectrum"].fmt == L.BF16X2 and by["spectrum"].pad == 0
    assert by["st.u"].fmt == L.BF16X2 and by["st.u"].pad == 0
    assert by["st.t"].fmt == L.F32 and by["spectrum_out"].fmt == L.F32
    up_last = [b for b in prog.bufs if b.name.startswith("up")][-1]
    assert up_last.fmt == L.BF16X2 and up_last.pad == 3       # tensor-core head: 3-pixel reflected ring
    assert isinstance(prog.ops[-1], E.HeadGatherOp) and prog.ops[-2].tag == "head 7x7 rows"
    ops = prog.ops
    assert isinstance(ops[0], E.StemPackOp) and isinstance(ops[1], E.ConvOp) and isinstance(ops[2], E.ConvOp)
    assert ops[1].ins[0].window == 8 and len(ops[1].packed.segs) == 4        # two-row packing: kernel rows (0,1) (2,3) (4,5) (6,-)
    # ring discipline: whenever a contraction reads a ring buffer, every op that touched that buffer since the ring
    # was last complete either was a BorderOp or a whole-plane tensor-core contraction (its epilogue writes the mirrored
    # pixels itself: engine.conv_writes_ring), and no BorderOp is redundant.
    last = {}
    for o in ops:
        if isinstance(o, E.ConvOp):
            for tv in o.ins:
                if tv is not None and tv.buf.reflect_border:
                    assert last.get(tv.buf.name) == "ring ok", f"{o.tag} reads a stale ring of {tv.buf.name}"
        if isinstance(o, E.BorderOp):
            assert last.get(o.view.buf.name) == "write"
            last[o.view.buf.name] = "ring ok"
        else:
            w = getattr(o, "out", None) or getattr(o, "spec", None)
            if isinstance(w, E.TV) and w.buf.reflect_border:
                if E.conv_writes_ring(prog, o):
                    last.setdefault(w.buf.name, "ring ok")       # (a stale ring stays stale until a BorderOp)
                else:
                    last[w.buf.name] = "write"
    n_border = sum(isinstance(o, E.BorderOp) for o in ops)
    assert n_border == 3      # only the 3 up-sampled outputs (written as sub-pixel phases) need the ring kernel
    out = SpecInterpreter(prog).run({"x0": x})
    assert float(np.abs(out["y0"].numpy() - a["y"]).max()) < 2e-6
    # weights of the tensor-core arm: [2][N][Kpad], K padded per segment to 64
    conv = next(o for o in ops if isinstance(o, E.ConvOp))
    ws = conv.packed.split_weights()
    assert ws.dtype == torch.bfloat16 and ws.shape[0] == 2 and ws.shape[2] == 64 * len(conv.packed.segs)
    rec = (ws[0].float() + ws[1].float())[:, :conv.packed.segs[0].nch]
    assert torch.allclose(rec, conv.packed.w_kn.t()[:, :conv.packed.segs[0].nch], rtol=2 ** -15, atol=1e-9)


def test_tc_incompatible_program_downgrades_to_fp32():
    a, sd = load_golden("ffcbnact_4to8_k7_local")
    m = _load(M.FFC_BN_ACT(in_channels=4, out_channels=8, kernel_size=7, ratio_gin=0, ratio_gout=0, padding=0,
                           activation_layer=torch.nn.ReLU, enable_lfu=False), sd)
    with torch.no_grad():
        prog = E.build_module_program(m, "ffc_bn_act", ((1, 4, 22, 22), None), L.MATH_BF16X3)
    assert prog.math == L.MATH_FP32


def test_weights_signature_tracks_changes_cheaply():
    """Programs are rebuilt when weights change: load_state_dict, in-place edits, replaced parameters AND edits
    through ``.data`` (the reference's EMA update, trainers/base.py:40, leaves ``_version`` alone)."""
    m = M.FFC_BN_ACT(16, 16, 3, 0.5, 0.5, padding=1, enable_lfu=False).eval()
    s0 = E._weights_signature(m)
    assert E._weights_signature(m) == s0
    with torch.no_grad():
        m.bn_l.running_mean.add_(1.0)                       # in-place edit bumps the version counter
    s1 = E._weights_signature(m)
    assert s1 != s0
    m.load_state_dict({k: v.clone() for k, v in m.state_dict().items()})
    s2 = E._weights_signature(m)
    assert s2 != s1
    v = m.ffc.convl2l.weight._version
    m.ffc.convl2l.weight.data.mul_(0.999).add_(0.001)       # EMA-style edit: same pointer, same version
    assert m.ffc.convl2l.weight._version == v
    s3 = E._weights_signature(m)
    assert s3 != s2 and s3[:-1] == s2[:-1]                  # only the content checksum moved
    m.ffc.convl2l.weight = torch.nn.Parameter(m.ffc.convl2l.weight.detach().clone() * 2)   # replaced object
    assert E._weights_signature(m) != s3
    big = M.FFCResNetGenerator(**small_lama_kwargs(ngf=8, n_blocks=2)).eval()              # > _SMALL_MODULE tensors
    b0 = E._weights_signature(big)
    big.model[1].ffc.convl2l.weight = torch.nn.Parameter(big.model[1].ffc.convl2l.weight.detach().clone() + 1)
    sigs = [E._weights_signature(big) for _ in range(E._REWALK_EVERY + 1)]
    assert sigs[-1] != b0                                   # at the latest after the periodic re-walk
    E.invalidate(big)
    assert big not in E._PROGRAMS and big not in E._TENSORS


def test_modules_stay_copyable_and_picklable_after_native_use():
    """The executor caches hold ctypes pointers; they live in weak-keyed dictionaries outside the module, so the
    reference's ``copy.deepcopy(self.generator)`` (trainers/base.py:168), ``torch.save(module)`` and pickling keep
    working after a native forward."""
    import copy
    import ctypes
    import io
    import pickle
    g = M.FFCResNetGenerator(**small_lama_kwargs(ngf=8, n_blocks=1)).eval()
    fake = (ctypes.c_void_p(1), ctypes.byref(ctypes.c_int(3)))          # what a CudaExecutor keeps alive
    E._PROGRAMS.setdefault(g, {})[("generator", ((1, 4, 64, 64),), "cuda:0", 1)] = (E._weights_signature(g), fake)
    assert all(isinstance(v, (str, type(None))) for k, v in g.__dict__.items() if k.startswith("_ffcb"))   # plain data only
    g2 = copy.deepcopy(g)
    assert g2 not in E._PROGRAMS
    pickle.loads(pickle.dumps(g))
    buf = io.BytesIO()
    torch.save(g, buf)
    E.invalidate(g)


def test_resnet_block_input_gradient_program_matches_autograd():
    """SURVEY.md row f3: the forward+backward program of FFCResnetBlock (gradients w.r.t. x_l, x_g; eval-mode BN, frozen
    weights) interpreted on the CPU vs torch autograd through the oracle port in float64 — checks the transposed /
    flipped weight packing, the zero-border gradient convolutions + reflect fold, the ReLU masks and that the FFT
    pair is its own adjoint around the spectral GEMM."""
    from oracle import ffc_torch_cpu as otc
    from lama_b200.testing import seeded_parameters_
    blk = seeded_parameters_(M.FFCResnetBlock(64, padding_type="reflect", norm_layer=torch.nn.BatchNorm2d,
                                              activation_layer=torch.nn.ReLU, ratio_gin=0.75, ratio_gout=0.75,
                                              enable_lfu=False).eval(), 3, gain=1.0)
    assert E.block_grad_supported(blk)
    b, cl, cg, h, w = 2, 16, 48, 6, 10
    g = torch.Generator().manual_seed(1)
    xl, xg = torch.randn(b, cl, h, w, generator=g), torch.randn(b, cg, h, w, generator=g)
    gl, gg = torch.randn(b, cl, h, w, generator=g), torch.randn(b, cg, h, w, generator=g)
    with torch.no_grad():
        prog = E.build_module_program(blk, "resnet_block_grad", ((b, cl, h, w), (b, cg, h, w)), L.MATH_FP32)
    out = SpecInterpreter(prog).run(dict(x0=xl, x1=xg, g0=gl, g1=gg))
    sd = {k: v.double() for k, v in blk.state_dict().items()}
    xl64, xg64 = xl.double().requires_grad_(True), xg.double().requires_grad_(True)
    ol, og = otc.ffc_resnet_block(xl64, xg64, sd, "", ratio_gout=0.75)
    ((ol * gl.double()).sum() + (og * gg.double()).sum()).backward()
    _close(out["y0"], (ol.detach() - xl.double()).numpy(), 1e-6)
    _close(out["dx0"], xl64.grad.numpy(), 1e-6)
    _close(out["dx1"], xg64.grad.numpy(), 1e-6)
    assert not E.block_grad_supported(M.FFCResnetBlock(64, padding_type="reflect", norm_layer=torch.nn.BatchNorm2d,
                                                       ratio_gin=0.5, ratio_gout=0.5, enable_lfu=True).eval())


def test_generator_u8_program_matches_reference_predict_bytes():
    """SURVEY.md row f1: the predict-path program (uint8 image + mask in, inpainted uint8 out; decode, symmetric
    modulo padding, mask multiply / concat and blend / crop / x255 fused into the pack and gather kernels)."""
    a, _ = load_golden("predict_ngf8_3x45x52")
    _, sd = load_golden("generator_ngf8_b2_64x64")
    g = _load(M.FFCResNetGenerator(**small_lama_kwargs(ngf=8, n_blocks=2)), sd)
    img, mask = torch.from_numpy(a["images"]), torch.from_numpy(a["masks"])
    with torch.no_grad():
        prog = E.build_module_program(g, "generator_u8:8", (tuple(img.shape), tuple(mask.shape)), L.MATH_BF16X3)
    assert prog.inputs == {"img": (3, 45, 52, 3), "mask": (3, 45, 52)} and prog.outputs == {"y0": (3, 45, 52, 3)}
    assert prog.dtypes == {"img": torch.uint8, "mask": torch.uint8, "y0": torch.uint8}
    assert isinstance(prog.ops[0], E.StemPackU8Op) and isinstance(prog.ops[-1], E.HeadGatherU8Op)
    assert (prog.ops[0].out.buf.H, prog.ops[0].out.buf.W) == (48 + 6, 56 + 8)      # padded to modulo 8, + ring
    # front end alone: bit-exact generator input
    x = SpecInterpreter._u8_front(img, mask, 48, 56)
    assert np.array_equal(x.numpy(), a["x"])
    out = SpecInterpreter(prog).run({"img": img, "mask": mask})["y0"].numpy()
    hole = a["masks"] > 0
    assert out.dtype == np.uint8 and np.array_equal(out[~hole], a["out"][~hole])
    d = np.abs(out[hole].astype(int) - a["out"][hole].astype(int))
    assert d.max() <= 1 and (d != 0).mean() < 0.01
    # the fp32 CUDA-core arm has no uint8 front / back end: asking for it is an error, not a silent detour
    with pytest.raises(ValueError):
        E.build_module_program(g, "generator_u8:8", (tuple(img.shape), tuple(mask.shape)), L.MATH_FP32)


def test_empty_batch_returns_empty_outputs_without_launching():
    """Empty batch -> empty outputs of the right shape: the native entry point takes the output shapes from the
    program of a one-image batch and launches nothing (so this runs on the CPU box)."""
    g = M.FFCResNetGenerator(**small_lama_kwargs(ngf=8, n_blocks=1)).eval()
    (y,) = E.run_module(g, "generator", (torch.empty(0, 4, 64, 48),))
    assert tuple(y.shape) == (0, 3, 64, 48) and y.dtype == torch.float32
    m = M.FFC_BN_ACT(16, 32, 3, 0.5, 0.5, stride=2, padding=1, enable_lfu=False).eval()
    yl, yg = E.run_module(m, "ffc_bn_act", (torch.empty(0, 8, 16, 16), torch.empty(0, 8, 16, 16)))
    assert tuple(yl.shape) == (0, 16, 8, 8) and tuple(yg.shape) == (0, 16, 8, 8)
    # (the torch composition itself cannot serve as the checker here: torch.fft on an empty batch raises an MKL
    #  "inconsistent configuration" error on CPU — the reference has no defined behaviour for B = 0)
    fu = M.FourierUnit(8, 8).eval()
    (yf,) = E.run_module(fu, "fourier_unit", (torch.empty(0, 8, 16, 16),))
    assert tuple(yf.shape) == (0, 8, 16, 16)


def test_storage_slots_never_alias_live_buffers(monkeypatch):
    """engine.assign_storage_slots: buffers share storage only when (a) their storage is byte-identical and (b) the
    last op touching the earlier one comes strictly before the first op touching the later one; constants keep their
    own storage.  big-lama folds onto a dozen slots (bs64 1024x1024 = BASELINE config 4's global batch pools under 80 GB)."""
    from lama_b200.testing import BIG_LAMA_KWARGS
    gen = M.FFCResNetGenerator(**BIG_LAMA_KWARGS).eval()
    with torch.no_grad():
        prog = E.build_module_program(gen, "generator", ((64, 4, 1024, 1024),), L.MATH_BF16X3)
    slots = E.assign_storage_slots(prog)
    first, last = {}, {}
    for i, op in enumerate(prog.ops):
        r, w = op.views()
        for tv in r + w:
            first.setdefault(tv.buf.name, i)
            last[tv.buf.name] = i
    by_slot = {}
    for b in prog.bufs:
        by_slot.setdefault(slots[b.name], []).append(b)
    for members in by_slot.values():
        assert len({E.storage_key(b) for b in members}) == 1
        members = sorted(members, key=lambda b: first[b.name])
        for a, b in zip(members, members[1:]):
            assert last[a.name] < first[b.name], (a.name, b.name)
            assert a.name not in prog.consts and b.name not in prog.consts

    def nbytes(b):
        if b.tile:
            return -(-(b.B * b.H * b.W) // 128) * 128 * b.C * 4
        return b.B * (b.H + 2 * b.pad) * (b.W + 2 * b.pad) * b.C * 4
    pooled = sum(nbytes(m[0]) for m in by_slot.values())
    assert len(by_slot) <= 16 and pooled < 80e9 < sum(nbytes(b) for b in prog.bufs)
    monkeypatch.setenv("LAMA_B200_POOL", "0")
    assert len(set(E.assign_storage_slots(prog).values())) == len(prog.bufs)
