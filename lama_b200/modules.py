"""Drop-in ``nn.Module`` surface of the reference's ``saicinpainting/training/modules/ffc.py``.

Same class names, constructor signatures, sub-module attribute names (hence identical
``state_dict`` keys — ``load_checkpoint`` uses ``strict=False``, trainers/__init__.py:27-28, so
a silent mismatch would go unnoticed) and forward conventions (FFC-family modules take/return
``(x_l, x_g)`` tuples whose empty side is the int ``0``, ffc.py:206,225).

Execution: on a CUDA tensor, in ``eval()`` mode with autograd off and float32 input, every module
runs the hand-written sm_90a kernels of ``libffc_b200.so`` through a cached *program*
(``lama_b200.engine``).  Options no shipped config enables (LFU, gating, SE, positional encoding,
3-D FFT, spatial rescaling, groups, non-ortho norm, non-BatchNorm norms, dilation != 1,
spatial-transform wrappers) and training/autograd run the same maths as a composition of torch
operators on the same device — a *feature* fallback, never a CPU fallback; with
``LAMA_B200_STRICT=1`` (set by the tests and bench) an unexpected fallback raises instead.
On a CUDA tensor the native path raises if the library is missing.
"""
from __future__ import annotations

import os

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import engine as _engine

__all__ = ["FFCSE_block", "FourierUnit", "SpectralTransform", "FFC", "FFC_BN_ACT", "FFCResnetBlock",
           "ConcatTupleLayer", "FFCResNetGenerator", "FFCNLayerDiscriminator", "get_activation"]


def get_activation(kind="tanh"):
    """modules/base.py:43-50 (re-implemented so that importing this module never imports the
    reference package — see the ordering trap in SURVEY.md §8b)."""
    if kind == "tanh":
        return nn.Tanh()
    if kind == "sigmoid":
        return nn.Sigmoid()
    if kind is False:
        return nn.Identity()
    raise ValueError(f"Unknown activation kind {kind}")


def _native_ok(*tensors) -> bool:
    """Fast-path gate shared by all modules: CUDA fp32 tensors, inference, no autograd.  Under ``torch.jit.trace``
    (bin/to_jit.py:55-62) the modules run the reference's torch operator sequence instead, so that the exported
    TorchScript is self-contained (a ctypes call is invisible to the tracer and would be baked in as a constant)."""
    if torch.is_grad_enabled() or torch.jit.is_tracing():
        return False
    for t in tensors:
        if not torch.is_tensor(t):
            continue
        if not (t.is_cuda and t.dtype == torch.float32):
            return False
    return any(torch.is_tensor(t) for t in tensors)


def _generator_grad_native(gen, x) -> bool:
    """Autograd is on, the generator is in eval mode with frozen weights and gets a CUDA float32 input: the native
    path of the whole generator under autograd applies (``LAMA_B200_NATIVE_GRAD=0`` disables it)."""
    return (torch.is_grad_enabled() and not gen.training and not torch.jit.is_tracing() and torch.is_tensor(x)
            and x.is_cuda and x.dtype == torch.float32 and os.environ.get("LAMA_B200_NATIVE_GRAD", "1") != "0"
            and _engine.generator_grad_supported(gen, tuple(x.shape)))


def _generator_grad_forward(gen, x):
    """``gen(x)`` under autograd on the native path: the forward + input-gradient program when x wants a gradient
    (a second forward of the same shape before its backward raises), else the no-grad generator program."""
    if x.requires_grad:
        return _engine.generator_with_input_grad(gen, x)
    return _engine.run_module(gen, "generator", (x,))[0]


def _fallback(why: str):
    if os.environ.get("LAMA_B200_STRICT") == "1" and not torch.jit.is_tracing():
        raise RuntimeError(f"lama_b200: native path unavailable ({why}) and LAMA_B200_STRICT=1")


class _SELayer(nn.Module):
    """squeeze_excitation.py:4-20 (only reachable through use_se=True, off in every shipped config)."""

    def __init__(self, channel, reduction=16):
        super().__init__()
        self.avg_pool = nn.AdaptiveAvgPool2d(1)
        self.fc = nn.Sequential(nn.Linear(channel, channel // reduction, bias=False), nn.ReLU(inplace=True),
                                nn.Linear(channel // reduction, channel, bias=False), nn.Sigmoid())

    def forward(self, x):
        b, c = x.shape[:2]
        return x * self.fc(self.avg_pool(x).view(b, c)).view(b, c, 1, 1).expand_as(x)


class FFCSE_block(nn.Module):
    """ffc.py:16-46 — defined by the reference but unused by shipped configs; torch composition."""

    def __init__(self, channels, ratio_g):
        super().__init__()
        in_cg = int(channels * ratio_g)
        in_cl = channels - in_cg
        r = 16
        self.avgpool = nn.AdaptiveAvgPool2d((1, 1))
        self.conv1 = nn.Conv2d(channels, channels // r, kernel_size=1, bias=True)
        self.relu1 = nn.ReLU(inplace=True)
        self.conv_a2l = None if in_cl == 0 else nn.Conv2d(channels // r, in_cl, kernel_size=1, bias=True)
        self.conv_a2g = None if in_cg == 0 else nn.Conv2d(channels // r, in_cg, kernel_size=1, bias=True)
        self.sigmoid = nn.Sigmoid()

    def forward(self, x):
        id_l, id_g = x if type(x) is tuple else (x, 0)
        pooled = id_l if type(id_g) is int else torch.cat([id_l, id_g], dim=1)
        pooled = self.relu1(self.conv1(self.avgpool(pooled)))
        x_l = 0 if self.conv_a2l is None else id_l * self.sigmoid(self.conv_a2l(pooled))
        x_g = 0 if self.conv_a2g is None else id_g * self.sigmoid(self.conv_a2g(pooled))
        return x_l, x_g


class FourierUnit(nn.Module):
    """ffc.py:49-113.  Native path: rfft2 -> (1x1 conv + folded BN + ReLU) -> irfft2 kernels."""

    def __init__(self, in_channels, out_channels, groups=1, spatial_scale_factor=None,
                 spatial_scale_mode='bilinear', spectral_pos_encoding=False, use_se=False, se_kwargs=None,
                 ffc3d=False, fft_norm='ortho'):
        super().__init__()
        self.groups = groups
        self.conv_layer = nn.Conv2d(in_channels * 2 + (2 if spectral_pos_encoding else 0), out_channels * 2,
                                    kernel_size=1, stride=1, padding=0, groups=groups, bias=False)
        self.bn = nn.BatchNorm2d(out_channels * 2)
        self.relu = nn.ReLU(inplace=True)
        self.use_se = use_se
        if use_se:
            self.se = _SELayer(self.conv_layer.in_channels, **(se_kwargs or {}))
        self.spatial_scale_factor = spatial_scale_factor
        self.spatial_scale_mode = spatial_scale_mode
        self.spectral_pos_encoding = spectral_pos_encoding
        self.ffc3d = ffc3d
        self.fft_norm = fft_norm

    def native_supported(self) -> bool:
        spec_in = self.conv_layer.in_channels - (2 if self.spectral_pos_encoding else 0)
        return (self.groups == 1 and self.spatial_scale_factor is None
                and not self.use_se and not self.ffc3d and self.fft_norm == 'ortho' and not self.training
                and spec_in % 8 == 0 and self.conv_layer.out_channels % 8 == 0
                and _engine.bn_foldable(self.bn))

    def forward(self, x):
        if (_native_ok(x) and self.native_supported() and x.dim() == 4 and _engine.plane_ok(x.shape[-2], x.shape[-1])):
            return _engine.run_module(self, "fourier_unit", (x,))[0]
        _fallback("FourierUnit options / mode")
        return self._torch_forward(x)

    def _torch_forward(self, x):
        """The reference's operator sequence (ffc.py:76-113) for options outside the native path."""
        batch = x.shape[0]
        if self.spatial_scale_factor is not None:
            orig_size = x.shape[-2:]
            x = F.interpolate(x, scale_factor=self.spatial_scale_factor, mode=self.spatial_scale_mode,
                              align_corners=False)
        dims = (-3, -2, -1) if self.ffc3d else (-2, -1)
        spec = torch.fft.rfftn(x, dim=dims, norm=self.fft_norm)
        spec = torch.stack((spec.real, spec.imag), dim=-1).permute(0, 1, 4, 2, 3).contiguous()
        spec = spec.view((batch, -1) + tuple(spec.shape[3:]))
        if self.spectral_pos_encoding:
            h, w = spec.shape[-2:]
            cv = torch.linspace(0, 1, h)[None, None, :, None].expand(batch, 1, h, w).to(spec)
            ch = torch.linspace(0, 1, w)[None, None, None, :].expand(batch, 1, h, w).to(spec)
            spec = torch.cat((cv, ch, spec), dim=1)
        if self.use_se:
            spec = self.se(spec)
        spec = self.relu(self.bn(self.conv_layer(spec)))
        spec = spec.view((batch, -1, 2) + tuple(spec.shape[2:])).permute(0, 1, 3, 4, 2).contiguous()
        spec = torch.complex(spec[..., 0], spec[..., 1])
        out = torch.fft.irfftn(spec, s=x.shape[-3:] if self.ffc3d else x.shape[-2:], dim=dims, norm=self.fft_norm)
        if self.spatial_scale_factor is not None:
            out = F.interpolate(out, size=orig_size, mode=self.spatial_scale_mode, align_corners=False)
        return out


class SpectralTransform(nn.Module):
    """ffc.py:116-163."""

    def __init__(self, in_channels, out_channels, stride=1, groups=1, enable_lfu=True, **fu_kwargs):
        super().__init__()
        self.enable_lfu = enable_lfu
        self.downsample = nn.AvgPool2d(kernel_size=(2, 2), stride=2) if stride == 2 else nn.Identity()
        self.stride = stride
        half = out_channels // 2
        self.conv1 = nn.Sequential(nn.Conv2d(in_channels, half, kernel_size=1, groups=groups, bias=False),
                                   nn.BatchNorm2d(half), nn.ReLU(inplace=True))
        self.fu = FourierUnit(half, half, groups, **fu_kwargs)
        if self.enable_lfu:
            self.lfu = FourierUnit(half, half, groups)
        self.conv2 = nn.Conv2d(half, out_channels, kernel_size=1, groups=groups, bias=False)

    def native_supported(self, hw=None) -> bool:
        """``hw``: spatial size of the input; the LFU branch (ffc.py:148-157) is native for even square planes after the
        optional stride-2 pooling and c % 16 == 0 (quadrant views of c/4 channels), else the torch composition runs."""
        ok = (self.stride in (1, 2) and self.conv1[0].groups == 1 and not self.training
              and self.fu.native_supported() and self.conv1[0].in_channels % 4 == 0
              and self.conv2.out_channels % 4 == 0 and _engine.bn_foldable(self.conv1[1]))
        if ok and self.enable_lfu:
            if hw is None:
                return self.conv1[0].out_channels % 16 == 0 and self.lfu.native_supported()
            ok = _engine.lfu_supported(self, *_engine.st_out_hw(self, *hw))
        return ok

    def forward(self, x):
        if (_native_ok(x) and x.dim() == 4 and self.native_supported(tuple(x.shape[-2:]))
                and _engine.plane_ok(*_engine.st_out_hw(self, *x.shape[-2:]))):
            return _engine.run_module(self, "spectral_transform", (x,))[0]
        _fallback("SpectralTransform options / mode")
        x = self.conv1(self.downsample(x))
        out = self.fu(x)
        if self.enable_lfu:
            n, c, h, w = x.shape
            s = h // 2
            xs = torch.cat(torch.split(x[:, :c // 4], s, dim=-2), dim=1).contiguous()
            xs = torch.cat(torch.split(xs, s, dim=-1), dim=1).contiguous()
            xs = self.lfu(xs).repeat(1, 1, 2, 2).contiguous()
        else:
            xs = 0
        return self.conv2(x + out + xs)


class FFC(nn.Module):
    """ffc.py:166-225."""

    def __init__(self, in_channels, out_channels, kernel_size, ratio_gin, ratio_gout, stride=1, padding=0,
                 dilation=1, groups=1, bias=False, enable_lfu=True, padding_type='reflect', gated=False,
                 **spectral_kwargs):
        super().__init__()
        assert stride == 1 or stride == 2, "Stride should be 1 or 2."
        self.stride = stride
        in_cg = int(in_channels * ratio_gin)
        in_cl = in_channels - in_cg
        out_cg = int(out_channels * ratio_gout)
        out_cl = out_channels - out_cg
        self.ratio_gin = ratio_gin
        self.ratio_gout = ratio_gout
        self.global_in_num = in_cg

        def conv_or_identity(cin, cout):
            if cin == 0 or cout == 0:
                return nn.Identity()
            return nn.Conv2d(cin, cout, kernel_size, stride, padding, dilation, groups, bias,
                             padding_mode=padding_type)

        self.convl2l = conv_or_identity(in_cl, out_cl)
        self.convl2g = conv_or_identity(in_cl, out_cg)
        self.convg2l = conv_or_identity(in_cg, out_cl)
        if in_cg == 0 or out_cg == 0:
            self.convg2g = nn.Identity()
        else:
            self.convg2g = SpectralTransform(in_cg, out_cg, stride, 1 if groups == 1 else groups // 2, enable_lfu,
                                             **spectral_kwargs)
        self.gated = gated
        self.gate = nn.Conv2d(in_channels, 2, 1) if (in_cg != 0 and out_cl != 0 and gated) else nn.Identity()

    def forward(self, x):
        # the native path lives one level up (FFC_BN_ACT fuses BN + activation into these convs);
        # a bare FFC is the torch composition of its (possibly native) children.
        x_l, x_g = x if type(x) is tuple else (x, 0)
        out_xl, out_xg = 0, 0
        if self.gated:
            parts = [x_l] + ([x_g] if torch.is_tensor(x_g) else [])
            gates = torch.sigmoid(self.gate(torch.cat(parts, dim=1)))
            g2l_gate, l2g_gate = gates.chunk(2, dim=1)
        else:
            g2l_gate, l2g_gate = 1, 1
        if self.ratio_gout != 1:
            out_xl = self.convl2l(x_l) + self.convg2l(x_g) * g2l_gate
        if self.ratio_gout != 0:
            out_xg = self.convl2g(x_l) * l2g_gate + self.convg2g(x_g)
        return out_xl, out_xg


class FFC_BN_ACT(nn.Module):
    """ffc.py:228-255.  Native path: one fused program per call (see engine.emit_ffc_bn_act)."""

    def __init__(self, in_channels, out_channels, kernel_size, ratio_gin, ratio_gout, stride=1, padding=0,
                 dilation=1, groups=1, bias=False, norm_layer=nn.BatchNorm2d, activation_layer=nn.Identity,
                 padding_type='reflect', enable_lfu=True, **kwargs):
        super().__init__()
        self.ffc = FFC(in_channels, out_channels, kernel_size, ratio_gin, ratio_gout, stride, padding, dilation,
                       groups, bias, enable_lfu, padding_type=padding_type, **kwargs)
        global_channels = int(out_channels * ratio_gout)
        self.bn_l = (nn.Identity if ratio_gout == 1 else norm_layer)(out_channels - global_channels)
        self.bn_g = (nn.Identity if ratio_gout == 0 else norm_layer)(global_channels)
        self.act_l = (nn.Identity if ratio_gout == 1 else activation_layer)(inplace=True)
        self.act_g = (nn.Identity if ratio_gout == 0 else activation_layer)(inplace=True)

    def native_supported(self) -> bool:
        return _engine.ffc_bn_act_supported(self)

    def forward(self, x):
        x_l, x_g = x if type(x) is tuple else (x, 0)
        if _native_ok(x_l, x_g) and self.native_supported() and _engine.ffc_bn_act_shapes_ok(self, x_l, x_g):
            return _engine.run_module(self, "ffc_bn_act", (x_l, x_g))
        _fallback("FFC_BN_ACT options / mode")
        y_l, y_g = self.ffc(x)
        return self.act_l(self.bn_l(y_l)), self.act_g(self.bn_g(y_g))


class _SpatialTransformUnavailable(nn.Module):
    def __init__(self, *a, **k):
        super().__init__()
        raise NotImplementedError("spatial_transform_kwargs needs kornia (LearnableSpatialTransformWrapper, "
                                  "spatial_transform.py:7-40); no shipped config enables it")


class FFCResnetBlock(nn.Module):
    """ffc.py:258-292."""

    def __init__(self, dim, padding_type, norm_layer, activation_layer=nn.ReLU, dilation=1,
                 spatial_transform_kwargs=None, inline=False, **conv_kwargs):
        super().__init__()
        common = dict(kernel_size=3, padding=dilation, dilation=dilation, norm_layer=norm_layer,
                      activation_layer=activation_layer, padding_type=padding_type)
        self.conv1 = FFC_BN_ACT(dim, dim, **common, **conv_kwargs)
        self.conv2 = FFC_BN_ACT(dim, dim, **common, **conv_kwargs)
        if spatial_transform_kwargs is not None:
            _SpatialTransformUnavailable()
        self.inline = inline

    def native_supported(self) -> bool:
        return (isinstance(self.conv1, FFC_BN_ACT) and isinstance(self.conv2, FFC_BN_ACT)
                and self.conv1.native_supported() and self.conv2.native_supported())

    def _input_grad_native(self, x_l, x_g) -> bool:
        """Autograd is on, the weights are frozen (``model.freeze()``, bin/predict.py:59) and at least one input wants a
        gradient: the native forward + input-gradient program applies (LAMA_B200_NATIVE_GRAD=0 disables it)."""
        if not (torch.is_grad_enabled() and torch.is_tensor(x_l) and torch.is_tensor(x_g) and not self.training
                and not torch.jit.is_tracing() and os.environ.get("LAMA_B200_NATIVE_GRAD", "1") == "1"):
            return False
        if not (x_l.is_cuda and x_g.is_cuda and x_l.dtype == torch.float32 and x_g.dtype == torch.float32
                and (x_l.requires_grad or x_g.requires_grad)):
            return False
        if any(p.requires_grad for p in self.parameters()):
            return False
        if max(x_l.shape[-2:]) > _engine.BLOCK_GRAD_MAX_PLANE:
            return False            # see engine.BLOCK_GRAD_MAX_PLANE: planes the native FFT rejects take torch autograd
        return _engine.block_grad_supported(self) and _engine.ffc_bn_act_shapes_ok(self.conv1, x_l, x_g)

    def forward(self, x):
        if self.inline:
            g = self.conv1.ffc.global_in_num
            x_l, x_g = x[:, :-g], x[:, -g:]
        else:
            x_l, x_g = x if type(x) is tuple else (x, 0)
        if (_native_ok(x_l, x_g) and self.native_supported()
                and _engine.ffc_bn_act_shapes_ok(self.conv1, x_l, x_g)):
            out = _engine.run_module(self, "resnet_block", (x_l, x_g))
        elif self._input_grad_native(x_l, x_g):
            # refinement (evaluation/refinement.py:137-167): frozen weights, gradients w.r.t. the feature maps only
            out = _engine.block_with_input_grad(self, x_l, x_g)
        else:
            _fallback("FFCResnetBlock options / mode")
            y_l, y_g = self.conv2(self.conv1((x_l, x_g)))
            out = (x_l + y_l, x_g + y_g)
        return torch.cat(out, dim=1) if self.inline else out


class ConcatTupleLayer(nn.Module):
    """ffc.py:295-302."""

    def forward(self, x):
        assert isinstance(x, tuple)
        x_l, x_g = x
        assert torch.is_tensor(x_l) or torch.is_tensor(x_g)
        return x_l if not torch.is_tensor(x_g) else torch.cat(x, dim=1)


class FFCResNetGenerator(nn.Module):
    """ffc.py:305-367.  ``self.model`` stays an ``nn.Sequential`` with the reference's stage indices
    (refinement.py:270-289 and predict_inner_features.py:84 slice / iterate it); ``forward`` runs
    the whole stack as one native program when every stage is on the native path."""

    def __init__(self, input_nc, output_nc, ngf=64, n_downsampling=3, n_blocks=9, norm_layer=nn.BatchNorm2d,
                 padding_type='reflect', activation_layer=nn.ReLU, up_norm_layer=nn.BatchNorm2d,
                 up_activation=nn.ReLU(True), init_conv_kwargs={}, downsample_conv_kwargs={},
                 resnet_conv_kwargs={}, spatial_transform_layers=None, spatial_transform_kwargs={},
                 add_out_act=True, max_features=1024, out_ffc=False, out_ffc_kwargs={}):
        assert n_blocks >= 0
        super().__init__()
        # constructor arguments as JSON when they are plain data (default layer classes): lets a torch.jit.trace on
        # CUDA record the native generator call as ONE custom op (lama_b200/ops.py) instead of cuFFT / cuDNN ops
        defaults = (norm_layer is nn.BatchNorm2d and activation_layer is nn.ReLU and up_norm_layer is nn.BatchNorm2d
                    and isinstance(up_activation, nn.ReLU) and spatial_transform_layers is None)
        self._ffcb_spec = None
        if defaults:
            from .ops import spec_of
            self._ffcb_spec = spec_of(dict(
                input_nc=input_nc, output_nc=output_nc, ngf=ngf, n_downsampling=n_downsampling, n_blocks=n_blocks,
                padding_type=padding_type, init_conv_kwargs=init_conv_kwargs,
                downsample_conv_kwargs=downsample_conv_kwargs, resnet_conv_kwargs=resnet_conv_kwargs,
                add_out_act=add_out_act, max_features=max_features, out_ffc=out_ffc, out_ffc_kwargs=out_ffc_kwargs))
        stages = [nn.ReflectionPad2d(3),
                  FFC_BN_ACT(input_nc, ngf, kernel_size=7, padding=0, norm_layer=norm_layer,
                             activation_layer=activation_layer, **init_conv_kwargs)]
        for i in range(n_downsampling):
            mult = 2 ** i
            kw = dict(downsample_conv_kwargs)
            if i == n_downsampling - 1:
                kw['ratio_gout'] = resnet_conv_kwargs.get('ratio_gin', 0)
            stages.append(FFC_BN_ACT(min(max_features, ngf * mult), min(max_features, ngf * mult * 2),
                                     kernel_size=3, stride=2, padding=1, norm_layer=norm_layer,
                                     activation_layer=activation_layer, **kw))
        feats = min(max_features, ngf * 2 ** n_downsampling)
        for i in range(n_blocks):
            if spatial_transform_layers is not None and i in spatial_transform_layers:
                _SpatialTransformUnavailable()
            stages.append(FFCResnetBlock(feats, padding_type=padding_type, activation_layer=activation_layer,
                                         norm_layer=norm_layer, **resnet_conv_kwargs))
        stages.append(ConcatTupleLayer())
        for i in range(n_downsampling):
            mult = 2 ** (n_downsampling - i)
            stages += [nn.ConvTranspose2d(min(max_features, ngf * mult), min(max_features, int(ngf * mult / 2)),
                                          kernel_size=3, stride=2, padding=1, output_padding=1),
                       up_norm_layer(min(max_features, int(ngf * mult / 2))), up_activation]
        if out_ffc:
            stages.append(FFCResnetBlock(ngf, padding_type=padding_type, activation_layer=activation_layer,
                                         norm_layer=norm_layer, inline=True, **out_ffc_kwargs))
        stages += [nn.ReflectionPad2d(3), nn.Conv2d(ngf, output_nc, kernel_size=7, padding=0)]
        if add_out_act:
            stages.append(get_activation('tanh' if add_out_act is True else add_out_act))
        self.model = nn.Sequential(*stages)

    def forward(self, input):
        if _native_ok(input) and not self.training and _engine.generator_supported(self, input):
            return _engine.run_module(self, "generator", (input,))[0]
        if _generator_grad_native(self, input):
            return _generator_grad_forward(self, input)
        if (torch.jit.is_tracing() and self._ffcb_spec is not None and not self.training and torch.is_tensor(input)
                and input.is_cuda and input.dtype == torch.float32 and not torch.is_grad_enabled()
                and os.environ.get("LAMA_B200_TRACE_NATIVE", "1") == "1" and _engine.generator_supported(self, input)):
            # bin/to_jit.py:55-62 on a CUDA box: the traced graph keeps the native kernels as one custom-op node
            from .ops import traced_generator_call
            return traced_generator_call(self, input)
        _fallback("FFCResNetGenerator topology / mode")
        return self.model(input)


class FFCNLayerDiscriminator(nn.Module):
    """ffc.py:370-433 — training-only FFC discriminator (no shipped config uses it).  Kept so that the module
    surface is complete; it is a composition of the drop-in FFC_BN_ACT blocks (LeakyReLU activations keep them
    on the torch path) with the reference's attribute names (model0..modelN) and forward contract
    (final scores, list of intermediate activations)."""

    def __init__(self, input_nc, ndf=64, n_layers=3, norm_layer=nn.BatchNorm2d, max_features=512,
                 init_conv_kwargs={}, conv_kwargs={}):
        super().__init__()
        self.n_layers = n_layers

        def act(inplace=True):
            return nn.LeakyReLU(negative_slope=0.2, inplace=inplace)

        kw, padw = 3, 1
        stages = [[FFC_BN_ACT(input_nc, ndf, kernel_size=kw, padding=padw, norm_layer=norm_layer,
                              activation_layer=act, **init_conv_kwargs)]]
        nf = ndf
        for _ in range(1, n_layers):
            nf_prev, nf = nf, min(nf * 2, max_features)
            stages.append([FFC_BN_ACT(nf_prev, nf, kernel_size=kw, stride=2, padding=padw, norm_layer=norm_layer,
                                      activation_layer=act, **conv_kwargs)])
        nf_prev, nf = nf, min(nf * 2, 512)
        stages.append([FFC_BN_ACT(nf_prev, nf, kernel_size=kw, stride=1, padding=padw, norm_layer=norm_layer,
                                  activation_layer=act, **conv_kwargs), ConcatTupleLayer()])
        stages.append([nn.Conv2d(nf, 1, kernel_size=kw, stride=1, padding=padw)])
        for i, st in enumerate(stages):
            setattr(self, f"model{i}", nn.Sequential(*st))

    def get_all_activations(self, x):
        res = [x]
        for i in range(self.n_layers + 2):
            res.append(getattr(self, f"model{i}")(res[-1]))
        return res[1:]

    def forward(self, x):
        acts = self.get_all_activations(x)
        feats = []
        for out in acts[:-1]:
            if isinstance(out, tuple):
                out = torch.cat(out, dim=1) if torch.is_tensor(out[1]) else out[0]
            feats.append(out)
        return acts[-1], feats
