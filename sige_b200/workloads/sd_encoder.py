"""The Stable Diffusion VAE encoder (first stage, image -> latent moments) built on the ``sige.nn`` operator surface.

A benchmark / test workload, not part of the operator library, like sd_decoder.py: the GPU machines have no copy of the reference,
so the model whose launches are measured must exist in-tree.  It is written from the architecture of reference
stable-diffusion/ldm/modules/diffusionmodules/sige_model.py (SIGEEncoder, SIGEDownsample) with the SAME module tree and parameter
names, so that ``init_deterministic`` gives both the same weights and their state dicts load into each other.  The resnet and
attention blocks are sd_decoder.py's: the reference uses one class of each for both halves of the autoencoder.

The SDEdit runner encodes every edited image this way: a full pass on the original image (it fills the Scatter* caches and
records every GroupNorm of a sparse block as a per-channel (scale, shift)), ``set_masks``, a sparse pass on the edited image.
``conv_in`` (on the 3-channel image), ``norm_out`` and ``conv_out`` stay dense, as in the reference.  Each downsample is a plain
3x3 stride-2 conv without padding behind a Gather of 6 x 6 tiles; the full pass pads the gathered map by one row and column at the
bottom and right (the reference's asymmetric padding), the sparse pass reads those as the Gather's zero halo.

The output is the 2 * z_channels = 8 channel moments map (mean and log-variance of the latent posterior).  ``quant_conv``, the
diagonal Gaussian posterior and ``scale_factor`` live in the runner, dense, outside the SIGEModel, and are not restated here.

Sizes: ``"full"`` = the first-stage ddconfig of stable-diffusion/configs/sige.yaml (ch 128, mult 1-2-4-4, 2 res blocks, no
attention resolutions), 3 x 512 x 512 -> 8 x 64 x 64; ``"mini"`` = ch 128, mult 1-4, 1 res block (a 512-channel mid block, as at
full size), 3 x 32 x 32 -> 8 x 16 x 16.
"""
from __future__ import annotations

from typing import Tuple

import numpy as np
import torch
from torch import nn
from torch.nn import functional as F

from ..nn import Gather, Scatter, SIGEModel, SIGEModule
from .ddpm import init_deterministic, make_norm, swish
from .sd_decoder import _OTHER_EDITS, SIGEAttnBlock, SIGEResnetBlock, SIZES

IN_CH, Z_CHANNELS = 3, 4
OUT_CH = 2 * Z_CHANNELS
SEED = 37                                  # of init_deterministic: the golden's reference encoder gets the same weights


class SIGEDownsample(SIGEModule):
    """3x3 stride-2 conv without padding on 6 x 6 tiles; the full pass pads (0, 1, 0, 1) itself, as torch has no asymmetric pad."""

    def __init__(self, in_channels: int, block_size: int = 6):
        super().__init__()
        self.conv = nn.Conv2d(in_channels, in_channels, kernel_size=3, stride=2, padding=0)
        self.gather = Gather(self.conv, block_size=block_size)
        self.scatter = Scatter(self.gather)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        x = self.gather(x)
        if self.mode == "full":
            x = F.pad(x, (0, 1, 0, 1), mode="constant", value=0)
        return self.scatter(self.conv(x))


class SIGEEncoder(SIGEModel):
    def __init__(self, *, ch: int, ch_mult: Tuple[int, ...], num_res_blocks: int, resolution: int, in_channels: int = IN_CH,
                 z_channels: int = Z_CHANNELS):
        super().__init__()
        self.ch, self.num_resolutions, self.num_res_blocks, self.resolution = ch, len(ch_mult), num_res_blocks, resolution
        self.in_channels = in_channels
        self.conv_in = nn.Conv2d(in_channels, ch, kernel_size=3, stride=1, padding=1)
        in_ch_mult = (1,) + tuple(ch_mult)
        downs = []
        for level in range(self.num_resolutions):
            down = nn.Module()
            down.block = nn.ModuleList()
            down.attn = nn.ModuleList()                   # no attention resolutions in the SD first stage
            block_in = ch * in_ch_mult[level]
            for _ in range(num_res_blocks):
                down.block.append(SIGEResnetBlock(block_in, ch * ch_mult[level]))
                block_in = ch * ch_mult[level]
            if level != self.num_resolutions - 1:
                down.downsample = SIGEDownsample(block_in)
            downs.append(down)
        self.down = nn.ModuleList(downs)
        self.mid = nn.Module()
        self.mid.block_1 = SIGEResnetBlock(block_in, block_in)
        self.mid.attn_1 = SIGEAttnBlock(block_in)
        self.mid.block_2 = SIGEResnetBlock(block_in, block_in)
        self.norm_out = make_norm(block_in)
        self.conv_out = nn.Conv2d(block_in, 2 * z_channels, kernel_size=3, stride=1, padding=1)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        h = self.conv_in(x)
        for level in range(self.num_resolutions):
            for blk in self.down[level].block:
                h = blk(h)
            if level != self.num_resolutions - 1:
                h = self.down[level].downsample(h)
        h = self.mid.block_1(h)
        h = self.mid.attn_1(h)
        h = self.mid.block_2(h)
        return self.conv_out(swish(self.norm_out(h)))


def build_sd_encoder(size: str = "mini") -> SIGEEncoder:
    return init_deterministic(SIGEEncoder(**SIZES[size]), seed=SEED).eval()


def _image(rng, res: int) -> torch.Tensor:
    return torch.from_numpy(rng.uniform(-1.0, 1.0, size=(1, IN_CH, res, res)).astype(np.float32))


def sd_encoder_inputs(size: str = "mini", seed: int = 4):
    """(x0, x1, mask): the original image in [-1, 1], the edited one and the edit mask.  The mask is sd_decoder_inputs': full:
    BASELINE.json's centred 15 % square of the 512 x 512 image; mini: a 10 x 14 rectangle of the 32 x 32 image.  x1 differs from
    x0 exactly on the pixels the mask sets."""
    res = SIZES[size]["resolution"]
    rng = np.random.default_rng(seed)
    x0 = _image(rng, res)
    mask = torch.zeros(res, res, dtype=torch.bool)
    if size == "full":
        side = int(round((0.15 ** 0.5) * res))
        lo = (res - side) // 2
        mask[lo:lo + side, lo:lo + side] = True
    else:
        mask[9:19, 13:27] = True
    x1 = torch.where(mask, _image(rng, res), x0)
    return x0, x1, mask


def sd_encoder_edits(size: str = "mini", E: int = 3, seed: int = 4):
    """(x0, x1s, masks): E INDEPENDENT EDITS of one image x0 — x1s [E, 3, H, W], masks [E, H, W].  Edit 0 is sd_encoder_inputs'
    (x1, mask); the others are sd_decoder_edits' places: a smaller one, one along the left border, one in the bottom-right corner
    (where the sparse downsamples' zero halo stands in for the full pass's asymmetric pad), cycled for more edits."""
    x0, x1, mask = sd_encoder_inputs(size, seed)
    res = mask.shape[0]
    rng = np.random.default_rng(seed + 1)
    x1s, masks = [x1], [mask]
    for e in range(1, E):
        top, left, h, w = _OTHER_EDITS[(e - 1) % len(_OTHER_EDITS)]
        m = torch.zeros(res, res, dtype=torch.bool)
        y0, x0_ = int(top * res), int(left * res)
        m[y0:y0 + max(1, int(round(h * res))), x0_:x0_ + max(1, int(round(w * res)))] = True
        masks.append(m)
        x1s.append(torch.where(m, _image(rng, res), x0))
    return x0, torch.cat(x1s, 0), torch.stack(masks, 0)


def run_sd_encoder(net, downsample_mask, size: str = "mini", device="cpu", fused=None):
    """Full pass on x0, set_masks with the SDEdit runner's mask pyramid (min_res 4 x 4, dilation 0), sparse pass on x1."""
    x0, x1, mask = (t.to(device) for t in sd_encoder_inputs(size))
    with torch.no_grad():
        net.set_mode("full")
        full0 = net(x0)
        net.set_masks(downsample_mask(mask, min_res=(4, 4), dilation=0))
        net.set_mode("sparse")
        if fused is not None:
            fused(net)
        sparse1 = net(x1)
    return full0, sparse1
