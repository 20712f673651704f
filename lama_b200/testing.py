"""Deterministic model / input factories shared by tests, bench.py and smoke().

No checkpoint exists offline (SURVEY.md headline facts), so parity is established on
seeded random weights.  Default ``BatchNorm2d`` statistics (mean 0, var 1, gamma 1,
beta 0) would hide BN-folding bugs, so every BN is randomised; conv weights are drawn
``N(0, gain^2 / fan_in)`` (gain 0.65: pre-sigmoid std ~1 after all 18 residual blocks)
(PyTorch's default init makes them decay and the parity check trivially easy).

These helpers only touch ``nn.Module`` parameters by *name* and therefore work
identically on the reference classes, the oracle port and the drop-in modules.
"""
import torch
import torch.nn as nn

# configs/training/big-lama.yaml:26-45 (generator block), interpolations resolved.
BIG_LAMA_KWARGS = dict(
    input_nc=4, output_nc=3, ngf=64, n_downsampling=3, n_blocks=18,
    add_out_act="sigmoid",
    init_conv_kwargs=dict(ratio_gin=0, ratio_gout=0, enable_lfu=False),
    downsample_conv_kwargs=dict(ratio_gin=0, ratio_gout=0, enable_lfu=False),
    resnet_conv_kwargs=dict(ratio_gin=0.75, ratio_gout=0.75, enable_lfu=False),
)


# configs/training/generator/pix2pixhd_global_sigmoid.yaml (lama-regular.yaml:29) and big-lama-regular.yaml:3-11:
# GlobalGenerator (lama_b200.pix2pixhd) kwargs.
LAMA_REGULAR_KWARGS = dict(input_nc=4, output_nc=3, ngf=64, n_downsampling=3, n_blocks=9, conv_kind="default",
                           add_out_act="sigmoid")
BIG_LAMA_REGULAR_KWARGS = dict(LAMA_REGULAR_KWARGS, n_blocks=15)


def small_regular_kwargs(ngf=8, n_blocks=2, n_downsampling=3):
    return dict(LAMA_REGULAR_KWARGS, ngf=ngf, n_blocks=n_blocks, n_downsampling=n_downsampling)


def small_lama_kwargs(ngf=8, n_blocks=2, n_downsampling=3):
    kw = {k: (dict(v) if isinstance(v, dict) else v) for k, v in BIG_LAMA_KWARGS.items()}
    kw.update(ngf=ngf, n_blocks=n_blocks, n_downsampling=n_downsampling)
    return kw


@torch.no_grad()
def seeded_parameters_(module: nn.Module, seed: int = 0, gain: float = 0.65) -> nn.Module:
    """Overwrite every parameter / BN buffer of ``module`` from one seeded CPU generator.

    Iteration is over ``named_modules()`` in registration order, which is identical for
    any two module trees with the same ``state_dict`` schema.
    """
    g = torch.Generator(device="cpu").manual_seed(seed)

    def fill(t, values):
        t.copy_(values.to(device=t.device, dtype=t.dtype))

    for _name, m in module.named_modules():
        if isinstance(m, (nn.Conv2d, nn.ConvTranspose2d)):
            w = m.weight
            if isinstance(m, nn.ConvTranspose2d):
                # weight is (C_in, C_out/groups, kh, kw); each output sees ~ C_in*k*k/stride^2 taps
                fan_in = w.shape[0] * w.shape[2] * w.shape[3] / float(m.stride[0] * m.stride[1])
            else:
                fan_in = w.shape[1] * w.shape[2] * w.shape[3]
            fill(w, torch.randn(w.shape, generator=g) * (gain / fan_in ** 0.5))
            if m.bias is not None:
                fill(m.bias, torch.randn(m.bias.shape, generator=g) * 0.1)
        elif isinstance(m, nn.BatchNorm2d):
            c = m.num_features
            fill(m.running_mean, torch.randn(c, generator=g) * 0.1)
            fill(m.running_var, torch.rand(c, generator=g) + 0.5)
            fill(m.weight, torch.rand(c, generator=g) * 0.4 + 0.8)
            fill(m.bias, torch.randn(c, generator=g) * 0.1)
    return module


def synthetic_image_mask(batch: int, size: int, seed: int = 0, width: int = None):
    """``image ~ U[0,1] (B,3,H,W)``, binary mask of seeded rectangles ``(B,1,H,W)`` (BASELINE.md §3)."""
    h, w = size, (width or size)
    g = torch.Generator(device="cpu").manual_seed(1000 + seed)
    image = torch.rand(batch, 3, h, w, generator=g)
    mask = torch.zeros(batch, 1, h, w)
    for b in range(batch):
        for _ in range(3):
            y0 = int(torch.randint(0, max(1, h - h // 4), (1,), generator=g))
            x0 = int(torch.randint(0, max(1, w - w // 4), (1,), generator=g))
            dy = int(torch.randint(max(1, h // 16), max(2, h // 3), (1,), generator=g))
            dx = int(torch.randint(max(1, w // 16), max(2, w // 3), (1,), generator=g))
            mask[b, :, y0:y0 + dy, x0:x0 + dx] = 1.0
    return image, mask


def generator_input(image: torch.Tensor, mask: torch.Tensor) -> torch.Tensor:
    """default.py:59,68 — ``cat([img * (1 - mask), mask], dim=1)``."""
    return torch.cat([image * (1.0 - mask), mask], dim=1)
