"""TEST / BASELINE INFRASTRUCTURE — the reference's CPU path restated with torch-CPU ops.

The reference's FFC path (``/root/reference/saicinpainting/training/modules/ffc.py``) is
pure PyTorch: on CPU every FLOP runs in MKL-FFT / oneDNN / ATen.  The reference tree cannot
travel to the GPU box, so ``bench.py`` times *this* port there as ``cpu_baseline`` (kind
"port") and as the ``--impl reference`` arm: it issues the same torch operator sequence as
the reference modules (one op per reference line, cited below), in fp32, driven by a
``state_dict`` with the reference's key names.  ``tests/test_oracle.py`` pins it against the
goldens generated from the unmodified reference (it must agree to float32 round-off since
the operator sequence is the same).

Never imported by the product path (``lama_b200``).
"""
from __future__ import annotations

import contextlib

import torch
import torch.nn.functional as F

EPS = 1e-5

# Pinned ReLU masks (``pinned_relu_masks``): None, or (site -> mask, set of the sites served)
_PINNED = None
# Masks recorded by ``recorded_relu_masks``: None, or site -> mask
_RECORDED = None


def relu(x, site):
    """The ReLU (in place) after the eval-mode BN whose state-dict prefix is ``site`` (``...bn_l.``, ``...bn_g.``,
    ``...convg2g.conv1.1.``, ``...fu.bn.``, ``model.{i}.`` of an up stage).  Under ``pinned_relu_masks`` it is
    ``x * mask[site]``: linear in x, with the mask given instead of the one x implies."""
    if _PINNED is None:
        y = torch.relu_(x)
        if _RECORDED is not None:
            _RECORDED[site] = (y > 0).detach()
        return y
    masks, served = _PINNED
    if site not in masks:
        raise KeyError(f"no pinned ReLU mask for site {site!r}")
    if tuple(masks[site].shape) != tuple(x.shape):
        raise ValueError(f"the pinned ReLU mask of {site!r} is {tuple(masks[site].shape)}, its input {tuple(x.shape)}")
    served.add(site)
    return x * masks[site]


@contextlib.contextmanager
def recorded_relu_masks():
    """Yield a dict that collects, per site, the mask (output > 0) of every ReLU evaluated inside without pinned masks."""
    global _RECORDED
    prev, _RECORDED = _RECORDED, {}
    try:
        yield _RECORDED
    finally:
        _RECORDED = prev


@contextlib.contextmanager
def pinned_relu_masks(masks):
    """Evaluate every ReLU of the functions below as ``x * masks[site]`` (masks: bool or 0 / 1, of x's NCHW shape).  A
    gradient program is linear once its masks are fixed, so with the masks a device run used, autograd through this
    module differs from that run by round-off alone.  Yields the set of sites served; a site without a mask raises."""
    global _PINNED
    served = set()
    prev, _PINNED = _PINNED, (dict(masks), served)
    try:
        yield served
    finally:
        _PINNED = prev


def _bn(x, sd, p):
    # nn.BatchNorm2d in eval mode (ffc.py:60,131,243-244,353)
    return F.batch_norm(x, sd[p + "running_mean"], sd[p + "running_var"], sd[p + "weight"], sd[p + "bias"],
                        training=False, eps=EPS)


def _conv(x, w, bias=None, stride=1, padding=0, reflect=False, dilation=1):
    if padding and reflect:
        x = F.pad(x, (padding,) * 4, mode="reflect")   # padding_mode='reflect' (ffc.py:189-196)
        padding = 0
    return F.conv2d(x, w, bias, stride=stride, padding=padding, dilation=dilation)


def fourier_unit(x, sd, p=""):
    """ffc.py:76-113, default options."""
    b = x.shape[0]
    f = torch.fft.rfftn(x, dim=(-2, -1), norm="ortho")                         # :86
    f = torch.stack((f.real, f.imag), dim=-1).permute(0, 1, 4, 2, 3).contiguous()   # :87-88
    f = f.view((b, -1) + tuple(f.shape[3:]))                                   # :89
    f = relu(_bn(F.conv2d(f, sd[p + "conv_layer.weight"]), sd, p + "bn."), p + "bn.")   # :100-101
    f = f.view((b, -1, 2) + tuple(f.shape[2:])).permute(0, 1, 3, 4, 2).contiguous()  # :103-104
    f = torch.complex(f[..., 0], f[..., 1])                                    # :105
    return torch.fft.irfftn(f, s=x.shape[-2:], dim=(-2, -1), norm="ortho")      # :108


def spectral_transform(x, sd, p="", stride=1, enable_lfu=False):
    """ffc.py:142-163."""
    if stride == 2:
        x = F.avg_pool2d(x, 2, 2)
    x = relu(_bn(F.conv2d(x, sd[p + "conv1.0.weight"]), sd, p + "conv1.1."), p + "conv1.1.")
    out = fourier_unit(x, sd, p + "fu.")
    if enable_lfu:
        n, c, h, w = x.shape
        s = h // 2
        xs = torch.cat(torch.split(x[:, : c // 4], s, dim=-2), dim=1).contiguous()
        xs = torch.cat(torch.split(xs, s, dim=-1), dim=1).contiguous()
        xs = fourier_unit(xs, sd, p + "lfu.").repeat(1, 1, 2, 2).contiguous()
    else:
        xs = 0
    return F.conv2d(x + out + xs, sd[p + "conv2.weight"])


def ffc_bn_act(x_l, x_g, sd, p, *, ratio_gout, stride=1, padding=0, dilation=1, enable_lfu=False):
    """ffc.py:205-225 (FFC.forward) + :251-255 (FFC_BN_ACT.forward), ReLU activation, not gated."""
    q = p + "ffc."
    kw = dict(stride=stride, padding=padding, reflect=True, dilation=dilation)
    o_l, o_g = 0, 0
    if ratio_gout != 1:
        o_l = _conv(x_l, sd[q + "convl2l.weight"], **kw)
        if (q + "convg2l.weight") in sd:
            o_l = o_l + _conv(x_g, sd[q + "convg2l.weight"], **kw)
        o_l = relu(_bn(o_l, sd, p + "bn_l."), p + "bn_l.")
    if ratio_gout != 0:
        o_g = _conv(x_l, sd[q + "convl2g.weight"], **kw)
        if (q + "convg2g.conv2.weight") in sd:
            o_g = o_g + spectral_transform(x_g, sd, q + "convg2g.", stride=stride, enable_lfu=enable_lfu)
        o_g = relu(_bn(o_g, sd, p + "bn_g."), p + "bn_g.")
    return o_l, o_g


def ffc_resnet_block(x_l, x_g, sd, p, *, ratio_gout=0.75, enable_lfu=False):
    """ffc.py:277-292."""
    kw = dict(ratio_gout=ratio_gout, padding=1, enable_lfu=enable_lfu)
    y_l, y_g = ffc_bn_act(x_l, x_g, sd, p + "conv1.", **kw)
    y_l, y_g = ffc_bn_act(y_l, y_g, sd, p + "conv2.", **kw)
    return x_l + y_l, x_g + y_g


def generator_rear(z1, z2, sd, kw):
    """``generator.model[first_block:]`` composed from the oracle: ffc_resnet_block per block, then ConvTranspose2d +
    eval BN + ReLU per up stage, then reflect pad 3 + 7x7 conv + the head activation (ffc.py:345-363)."""
    nd, nb = kw["n_downsampling"], kw["n_blocks"]
    i = 2 + nd
    z_l, z_g = z1, z2
    for _ in range(nb):
        z_l, z_g = ffc_resnet_block(z_l, z_g, sd, f"model.{i}.", ratio_gout=0.75); i += 1
    h = torch.cat((z_l, z_g), dim=1); i += 1
    for _ in range(nd):
        h = F.conv_transpose2d(h, sd[f"model.{i}.weight"], sd[f"model.{i}.bias"], stride=2, padding=1,
                               output_padding=1)
        h = relu(_bn(h, sd, f"model.{i + 1}."), f"model.{i + 1}."); i += 3
    h = F.conv2d(F.pad(h, (3, 3, 3, 3), mode="reflect"), sd[f"model.{i + 1}.weight"], sd[f"model.{i + 1}.bias"])
    act = kw.get("add_out_act", True)
    if act is True or act == "tanh":
        return torch.tanh(h)
    return torch.sigmoid(h) if act == "sigmoid" else h


@torch.no_grad()
def ffc_resnet_generator(x, sd, *, ngf=64, n_downsampling=3, n_blocks=9, init_conv_kwargs=None,
                         downsample_conv_kwargs=None, resnet_conv_kwargs=None, add_out_act=True,
                         prefix="model.", **_):
    """ffc.py:306-367 with the defaults big-lama uses."""
    init_conv_kwargs = init_conv_kwargs or {}
    downsample_conv_kwargs = downsample_conv_kwargs or {}
    resnet_conv_kwargs = resnet_conv_kwargs or {}
    i = 1
    h = F.pad(x, (3, 3, 3, 3), mode="reflect")
    l, g = ffc_bn_act(h, 0, sd, f"{prefix}{i}.", ratio_gout=init_conv_kwargs.get("ratio_gout", 0)); i += 1
    for d in range(n_downsampling):
        rg = downsample_conv_kwargs.get("ratio_gout", 0)
        if d == n_downsampling - 1:
            rg = resnet_conv_kwargs.get("ratio_gin", 0)
        l, g = ffc_bn_act(l, g, sd, f"{prefix}{i}.", ratio_gout=rg, stride=2, padding=1); i += 1
    for _ in range(n_blocks):
        l, g = ffc_resnet_block(l, g, sd, f"{prefix}{i}.", ratio_gout=resnet_conv_kwargs.get("ratio_gout", 0),
                                enable_lfu=resnet_conv_kwargs.get("enable_lfu", True)); i += 1
    h = torch.cat((l, g), dim=1) if torch.is_tensor(g) else l; i += 1
    for _ in range(n_downsampling):
        h = F.conv_transpose2d(h, sd[f"{prefix}{i}.weight"], sd[f"{prefix}{i}.bias"], stride=2, padding=1,
                               output_padding=1); i += 1
        h = relu(_bn(h, sd, f"{prefix}{i}."), f"{prefix}{i}."); i += 2
    h = F.pad(h, (3, 3, 3, 3), mode="reflect"); i += 1
    h = F.conv2d(h, sd[f"{prefix}{i}.weight"], sd[f"{prefix}{i}.bias"]); i += 1
    if add_out_act:
        h = torch.tanh(h) if add_out_act is True or add_out_act == "tanh" else torch.sigmoid(h)
    return h
