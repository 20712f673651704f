"""Drop-in ``nn.Module`` surface of the reference's LaMa-Regular generators (``GlobalGenerator`` and its
``ResnetBlock``, ``saicinpainting/training/modules/pix2pixhd.py:30-90, 341-436``): lama-regular and
big-lama-regular (``configs/training/generator/pix2pixhd_global_sigmoid.yaml``, ``big-lama-regular.yaml:3-11``).

Same constructor signatures, the same ``self.model`` ``nn.Sequential`` with the reference's stage indices and the
same attribute tree, hence identical ``state_dict`` keys.

Execution: on a CUDA float32 tensor in ``eval()`` mode with autograd off, ``GlobalGenerator.forward`` runs the whole
stack as one native program (``lama_b200.engine``, kinds ``generator`` / ``generator_u8``) when its layers are the
shipped configuration: plain 3x3 convs (``conv_kind='default'``, dilation 1, groups 1), eval BatchNorm with affine
parameters, reflect padding in the blocks, ReLU activations, no dilated or FFC blocks.  Any other option, training and
autograd run ``self.model`` as it stands (a feature fallback; with ``LAMA_B200_STRICT=1`` an error).

``conv_kind='depthwise'`` / ``'multidilated'`` and ``dilation_block_kind='multi'`` need the reference's own conv
classes, which this module does not import (SURVEY.md §8b); the constructor refuses them, and ``lama_b200.patch``
leaves the reference's class in charge of those configurations.
"""
from __future__ import annotations

import collections
from functools import partial

import torch.nn as nn

from . import engine as _engine
from .modules import (FFCResnetBlock, _fallback, _generator_grad_forward, _generator_grad_native, _native_ok,
                      get_activation)

__all__ = ["ResnetBlock", "GlobalGenerator", "reference_only_options"]


def reference_only_options(conv_kind='default', dilation_block_kind='simple', dilated_blocks_n=0,
                           dilated_blocks_n_start=0, dilated_blocks_n_middle=0, **_ignored) -> bool:
    """GlobalGenerator options that need classes only the reference defines (base.py:21-30: DepthWiseSeperableConv,
    MultidilatedConv; pix2pixhd.py:336-337: MultidilatedResnetBlock)."""
    if isinstance(conv_kind, str) and conv_kind in ('depthwise', 'multidilated'):
        return True
    any_dilated = any(n is not None and n > 0 for n in (dilated_blocks_n, dilated_blocks_n_start,
                                                       dilated_blocks_n_middle))
    return dilation_block_kind != 'simple' and any_dilated


def _conv_ctor(kind):
    """base.py:21-30 for the kinds this module can build."""
    if not isinstance(kind, str):
        return kind
    if kind == 'default':
        return nn.Conv2d
    raise NotImplementedError(f"conv_kind={kind!r} needs the reference's own conv class "
                              "(saicinpainting.training.modules.base.get_conv_block_ctor)")


def _norm_ctor(kind):
    """base.py:33-40."""
    if not isinstance(kind, str):
        return kind
    if kind == 'bn':
        return nn.BatchNorm2d
    if kind == 'in':
        return nn.InstanceNorm2d
    raise ValueError(f'Unknown norm block kind {kind}')


class ResnetBlock(nn.Module):
    """pix2pixhd.py:30-90: ``x + conv_block(x)`` with ``conv_block`` = [pad, conv, norm, act, (dropout), pad, conv,
    norm] — no activation after the sum.  Runs inside the generator program; alone it is the torch composition."""

    def __init__(self, dim, padding_type, norm_layer, activation=nn.ReLU(True), use_dropout=False,
                 conv_kind='default', dilation=1, in_dim=None, groups=1, second_dilation=None):
        super().__init__()
        self.in_dim = in_dim
        self.dim = dim
        if second_dilation is None:
            second_dilation = dilation
        self.conv_block = self.build_conv_block(dim, padding_type, norm_layer, activation, use_dropout,
                                                conv_kind=conv_kind, dilation=dilation, in_dim=in_dim, groups=groups,
                                                second_dilation=second_dilation)
        if self.in_dim is not None:
            self.input_conv = nn.Conv2d(in_dim, dim, 1)
        self.out_channnels = dim          # sic (pix2pixhd.py:45)

    def build_conv_block(self, dim, padding_type, norm_layer, activation, use_dropout, conv_kind='default',
                         dilation=1, in_dim=None, groups=1, second_dilation=1):
        conv_layer = _conv_ctor(conv_kind)

        def pad(d):
            if padding_type == 'reflect':
                return [nn.ReflectionPad2d(d)], 0
            if padding_type == 'replicate':
                return [nn.ReplicationPad2d(d)], 0
            if padding_type == 'zero':
                return [], d
            raise NotImplementedError('padding [%s] is not implemented' % padding_type)

        block, p = pad(dilation)
        block += [conv_layer(dim if in_dim is None else in_dim, dim, kernel_size=3, padding=p, dilation=dilation),
                  norm_layer(dim), activation]
        if use_dropout:
            block += [nn.Dropout(0.5)]
        more, p = pad(second_dilation)
        block += more + [conv_layer(dim, dim, kernel_size=3, padding=p, dilation=second_dilation, groups=groups),
                         norm_layer(dim)]
        return nn.Sequential(*block)

    def forward(self, x):
        x_before = x
        if self.in_dim is not None:
            x = self.input_conv(x)
        return x + self.conv_block(x_before)


class GlobalGenerator(nn.Module):
    """pix2pixhd.py:341-436 (kind ``pix2pixhd_global``).  ``self.model`` keeps the reference's stage indices;
    ``forward`` runs it as one native program when every stage is on the native path (module docstring)."""

    def __init__(self, input_nc, output_nc, ngf=64, n_downsampling=3, n_blocks=9, norm_layer=nn.BatchNorm2d,
                 padding_type='reflect', conv_kind='default', activation=nn.ReLU(True),
                 up_norm_layer=nn.BatchNorm2d, affine=None,
                 up_activation=nn.ReLU(True), dilated_blocks_n=0, dilated_blocks_n_start=0,
                 dilated_blocks_n_middle=0,
                 add_out_act=True,
                 max_features=1024, is_resblock_depthwise=False,
                 ffc_positions=None, ffc_kwargs={}, dilation=1, second_dilation=None,
                 dilation_block_kind='simple', multidilation_kwargs={}):
        assert n_blocks >= 0
        super().__init__()
        if dilation_block_kind not in ('simple', 'multi'):
            raise ValueError(f'dilation_block_kind could not be "{dilation_block_kind}"')
        if reference_only_options(conv_kind, dilation_block_kind, dilated_blocks_n, dilated_blocks_n_start,
                                  dilated_blocks_n_middle):
            raise NotImplementedError("these GlobalGenerator options need the reference's own classes "
                                      f"(conv_kind={conv_kind!r}, dilation_block_kind={dilation_block_kind!r})")
        conv_layer = _conv_ctor(conv_kind)
        norm_layer = _norm_ctor(norm_layer)
        up_norm_layer = _norm_ctor(up_norm_layer)
        if affine is not None:
            norm_layer = partial(norm_layer, affine=affine)
            up_norm_layer = partial(up_norm_layer, affine=affine)
        if ffc_positions is not None:
            ffc_positions = collections.Counter(ffc_positions)

        model = [nn.ReflectionPad2d(3), conv_layer(input_nc, ngf, kernel_size=7, padding=0), norm_layer(ngf),
                 activation]
        for i in range(n_downsampling):
            mult = 2 ** i
            model += [conv_layer(min(max_features, ngf * mult), min(max_features, ngf * mult * 2),
                                 kernel_size=3, stride=2, padding=1),
                      norm_layer(min(max_features, ngf * mult * 2)), activation]
        feats = min(max_features, ngf * 2 ** n_downsampling)
        dil_kw = dict(dim=feats, padding_type=padding_type, activation=activation, norm_layer=norm_layer,
                      conv_kind=conv_kind)

        def dil_blocks(n):          # pix2pixhd.py:328-338, 'simple' kind
            return [ResnetBlock(**dil_kw, dilation=2 ** (i + 1)) for i in range(n)]

        if dilated_blocks_n_start is not None and dilated_blocks_n_start > 0:
            model += dil_blocks(dilated_blocks_n_start)
        for i in range(n_blocks):
            if i == n_blocks // 2 and dilated_blocks_n_middle is not None and dilated_blocks_n_middle > 0:
                model += dil_blocks(dilated_blocks_n_middle)
            if ffc_positions is not None and i in ffc_positions:
                for _ in range(ffc_positions[i]):
                    model += [FFCResnetBlock(feats, padding_type, norm_layer, activation_layer=nn.ReLU, inline=True,
                                             **ffc_kwargs)]
            model += [ResnetBlock(feats, padding_type=padding_type, activation=activation, norm_layer=norm_layer,
                                  conv_kind=conv_kind, groups=feats if is_resblock_depthwise else 1,
                                  dilation=dilation, second_dilation=second_dilation)]
        if dilated_blocks_n is not None and dilated_blocks_n > 0:
            model += dil_blocks(dilated_blocks_n)
        for i in range(n_downsampling):
            mult = 2 ** (n_downsampling - i)
            model += [nn.ConvTranspose2d(min(max_features, ngf * mult), min(max_features, int(ngf * mult / 2)),
                                         kernel_size=3, stride=2, padding=1, output_padding=1),
                      up_norm_layer(min(max_features, int(ngf * mult / 2))), up_activation]
        model += [nn.ReflectionPad2d(3), nn.Conv2d(ngf, output_nc, kernel_size=7, padding=0)]
        if add_out_act:
            model.append(get_activation('tanh' if add_out_act is True else add_out_act))
        self.model = nn.Sequential(*model)

    def forward(self, input):
        if _native_ok(input) and not self.training and _engine.generator_supported(self, input):
            return _engine.run_module(self, "generator", (input,))[0]
        if _generator_grad_native(self, input):
            return _generator_grad_forward(self, input)
        _fallback("GlobalGenerator options / mode")
        return self.model(input)
