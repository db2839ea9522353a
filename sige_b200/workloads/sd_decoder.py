"""The Stable Diffusion VAE decoder (first stage, latent -> image) built on the ``sige.nn`` operator surface.

A benchmark / test workload, not part of the operator library: the GPU machines have no copy of the reference, so the model whose
launches are measured must exist in-tree.  It is written from the architecture of reference
stable-diffusion/ldm/modules/diffusionmodules/sige_model.py (SIGEDecoder, SIGEResnetBlock, SIGEUpsample) and model.py
(SIGEAttnBlock, my_group_norm) with the SAME module tree and parameter names, so that ``init_deterministic`` gives both the same
weights and their state dicts load into each other.

Per-mode behaviour is the reference's: ``full`` = dense pass that fills the Scatter* caches and records every GroupNorm of a sparse
block as a per-channel (scale, shift); ``sparse`` = the tile-sparse pass, where the Gathers apply them.  ``conv_in`` (on the
4-channel latent), ``norm_out`` and ``conv_out`` stay dense, as in the reference.  The mid block's attention is one head over all
pixels of the latent: in sparse mode the queries are the pixels of the active 4x4 tiles (tile-major, then pixel order), the keys and
values the full k / v maps, pasted together from the cached dense pass and the recomputed tiles.

Sizes: ``"full"`` = the first-stage ddconfig of stable-diffusion/configs/sige.yaml (ch 128, mult 1-2-4-4, 2 res blocks, no
attention resolutions), z 4 x 64 x 64 -> 512 x 512; ``"mini"`` = ch 128, mult 1-4, 1 res block (a 512-channel mid block, as at full
size), z 4 x 16 x 16 -> 32 x 32.
"""
from __future__ import annotations

from typing import Tuple

import numpy as np
import torch
from torch import nn
from torch.nn import functional as F

from ..nn import Gather, Scatter, ScatterGather, ScatterWithBlockResidual, SIGEConv2d, SIGEModel, SIGEModule
from .ddpm import group_norm_folded, init_deterministic, make_norm, swish

SIZES = {
    "mini": dict(ch=128, ch_mult=(1, 4), num_res_blocks=1, resolution=32),
    "full": dict(ch=128, ch_mult=(1, 2, 4, 4), num_res_blocks=2, resolution=512),
}
Z_CHANNELS, OUT_CH = 4, 3


def _folded(x: torch.Tensor, norm: nn.GroupNorm):
    """GroupNorm(x) and its (scale, shift) as [1, C, 1, 1] tensors, the form the reference's blocks hand to their Gathers."""
    y, scale, shift = group_norm_folded(x, norm)
    return y, scale.view(1, -1, 1, 1), shift.view(1, -1, 1, 1)


class SIGEResnetBlock(SIGEModule):
    """norm1-swish-conv1-norm2-swish-conv2 + (1x1 nin_shortcut) residual; 6x6 main tiles, 4x4 shortcut tiles."""

    def __init__(self, in_channels: int, out_channels: int, main_block_size: int = 6, shortcut_block_size: int = 4):
        super().__init__()
        self.in_channels, self.out_channels = in_channels, out_channels
        self.norm1 = make_norm(in_channels)
        self.conv1 = SIGEConv2d(in_channels, out_channels, kernel_size=3, stride=1, padding=1)
        self.norm2 = make_norm(out_channels)
        self.dropout = nn.Dropout(0.0)
        self.conv2 = SIGEConv2d(out_channels, out_channels, kernel_size=3, stride=1, padding=1)
        self.main_gather = Gather(self.conv1, main_block_size, activation_name="swish")
        self.scatter_gather = ScatterGather(self.main_gather, activation_name="swish")
        if in_channels != out_channels:
            self.nin_shortcut = SIGEConv2d(in_channels, out_channels, kernel_size=1, stride=1, padding=0)
            self.shortcut_gather = Gather(self.nin_shortcut, shortcut_block_size)
            self.scatter = ScatterWithBlockResidual(self.main_gather, self.shortcut_gather)
        else:
            self.scatter = Scatter(self.main_gather)
        self.scale1 = self.shift1 = self.scale2 = self.shift2 = None

    def _shortcut(self, x: torch.Tensor) -> torch.Tensor:
        if self.in_channels == self.out_channels:
            return x
        return self.nin_shortcut(self.shortcut_gather(x))

    def forward(self, x: torch.Tensor, temb=None) -> torch.Tensor:
        skip = self._shortcut(x)
        if self.mode == "full":
            h, self.scale1, self.shift1 = _folded(self.main_gather(x), self.norm1)
            h = self.scatter_gather(self.conv1(swish(h)))
            h, self.scale2, self.shift2 = _folded(h, self.norm2)
            h = self.dropout(swish(h))
        elif self.mode in ("sparse", "profile"):
            h = self.scatter_gather(self.conv1(self.main_gather(x, self.scale1, self.shift1)), self.scale2, self.shift2)
        else:
            raise NotImplementedError("Unknown mode [%s]!!!" % self.mode)
        return self.scatter(self.conv2(h), skip)


class SIGEAttnBlock(SIGEModule):
    """Single-head self-attention of the mid block: separate 1x1 q / k / v convs on one gathered stack, k and v pasted into full maps,
    softmax(q k^T / sqrt(C)) v over every pixel, proj_out, and the residual added by out_scatter."""

    def __init__(self, in_channels: int, block_size: int = 4):
        super().__init__()
        self.in_channels, self.block_size = in_channels, block_size
        self.norm = make_norm(in_channels)
        self.q = SIGEConv2d(in_channels, in_channels, kernel_size=1, stride=1, padding=0)
        self.k = SIGEConv2d(in_channels, in_channels, kernel_size=1, stride=1, padding=0)
        self.v = SIGEConv2d(in_channels, in_channels, kernel_size=1, stride=1, padding=0)
        self.proj_out = SIGEConv2d(in_channels, in_channels, kernel_size=1, stride=1, padding=0)
        self.gather = Gather(self.q, block_size=block_size)
        self.k_scatter = Scatter(self.gather)
        self.v_scatter = Scatter(self.gather)
        self.out_scatter = Scatter(self.gather)
        self.scale = self.shift = None

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        sparse = self.mode in ("sparse", "profile")
        if self.mode == "full":
            h, self.scale, self.shift = _folded(self.gather(x), self.norm)
        elif sparse:
            h = self.gather(x, self.scale, self.shift)
        else:
            raise NotImplementedError("Unknown mode [%s]!!!" % self.mode)
        q = self.q(h)
        k = self.k_scatter(self.k(h))
        v = self.v_scatter(self.v(h))
        b = x.size(0)
        c = q.shape[1]
        if sparse:            # [b * tiles, c, bs, bs] -> [b, tiles * bs * bs, c]: tile-major, then pixel order
            q = q.reshape(b, -1, c, self.block_size * self.block_size).permute(0, 1, 3, 2).reshape(b, -1, c)
        else:
            q = q.reshape(b, c, -1).permute(0, 2, 1)
        _, _, hh, ww = k.shape
        w_ = torch.bmm(q, k.reshape(b, c, hh * ww))
        w_ = w_ * (int(c) ** (-0.5))
        w_ = F.softmax(w_, dim=2)
        h = torch.bmm(v.reshape(b, c, hh * ww), w_.permute(0, 2, 1))          # [b, c, queries]
        if sparse:
            bs = self.block_size
            h = h.reshape(b, c, -1, bs, bs).permute(0, 2, 1, 3, 4).reshape(-1, c, bs, bs)
        else:
            h = h.reshape(b, c, hh, ww)
        return self.out_scatter(self.proj_out(h), x)


class SIGEUpsample(SIGEModule):
    """nearest x2 -> 3x3 conv on 6x6 tiles."""

    def __init__(self, in_channels: int, block_size: int = 6):
        super().__init__()
        self.conv = SIGEConv2d(in_channels, in_channels, kernel_size=3, stride=1, padding=1)
        self.gather = Gather(self.conv, block_size=block_size)
        self.scatter = Scatter(self.gather)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        x = F.interpolate(x, scale_factor=2.0, mode="nearest")
        return self.scatter(self.conv(self.gather(x)))


class SIGEDecoder(SIGEModel):
    def __init__(self, *, ch: int, ch_mult: Tuple[int, ...], num_res_blocks: int, resolution: int, z_channels: int = Z_CHANNELS,
                 out_ch: int = OUT_CH):
        super().__init__()
        self.ch, self.num_resolutions, self.num_res_blocks, self.resolution = ch, len(ch_mult), num_res_blocks, resolution
        block_in = ch * ch_mult[-1]
        latent = resolution // 2 ** (self.num_resolutions - 1)
        self.z_shape = (1, z_channels, latent, latent)
        self.conv_in = nn.Conv2d(z_channels, block_in, kernel_size=3, stride=1, padding=1)
        self.mid = nn.Module()
        self.mid.block_1 = SIGEResnetBlock(block_in, block_in)
        self.mid.attn_1 = SIGEAttnBlock(block_in)
        self.mid.block_2 = SIGEResnetBlock(block_in, block_in)
        ups = []
        for level in reversed(range(self.num_resolutions)):
            up = nn.Module()
            up.block = nn.ModuleList()
            up.attn = nn.ModuleList()
            for _ in range(num_res_blocks + 1):
                up.block.append(SIGEResnetBlock(block_in, ch * ch_mult[level]))
                block_in = ch * ch_mult[level]
            if level != 0:
                up.upsample = SIGEUpsample(block_in)
            ups.insert(0, up)
        self.up = nn.ModuleList(ups)
        self.norm_out = make_norm(block_in)
        self.conv_out = nn.Conv2d(block_in, out_ch, kernel_size=3, stride=1, padding=1)

    def forward(self, z: torch.Tensor) -> torch.Tensor:
        h = self.conv_in(z)
        h = self.mid.block_1(h)
        h = self.mid.attn_1(h)
        h = self.mid.block_2(h)
        for level in reversed(range(self.num_resolutions)):
            for blk in self.up[level].block:
                h = blk(h)
            if level != 0:
                h = self.up[level].upsample(h)
        return self.conv_out(swish(self.norm_out(h)))


def build_sd_decoder(size: str = "mini") -> SIGEDecoder:
    return init_deterministic(SIGEDecoder(**SIZES[size]), seed=31).eval()


def sd_decoder_inputs(size: str = "mini", seed: int = 4):
    """(z0, z1, mask): the original latent, the edited one and the edit mask at IMAGE resolution.  full: BASELINE.json's
    centred 15 % square of the 512 x 512 image; mini: a 10 x 14 rectangle of the 32 x 32 image.  z1 differs from z0 on the
    latent pixels the mask touches."""
    cfg = SIZES[size]
    res = cfg["resolution"]
    f = 2 ** (len(cfg["ch_mult"]) - 1)
    rng = np.random.default_rng(seed)
    z0 = torch.from_numpy(rng.standard_normal((1, Z_CHANNELS, res // f, res // f)).astype(np.float32))
    mask = torch.zeros(res, res, dtype=torch.bool)
    if size == "full":
        side = int(round((0.15 ** 0.5) * res))
        lo = (res - side) // 2
        mask[lo:lo + side, lo:lo + side] = True
    else:
        mask[9:19, 13:27] = True
    latent_mask = mask.view(res // f, f, res // f, f).any(3).any(1)
    z1 = z0 + torch.from_numpy(rng.standard_normal(tuple(z0.shape)).astype(np.float32)) * latent_mask
    return z0, z1, mask


def run_sd_decoder(net, downsample_mask, size: str = "mini", device="cpu", fused=None):
    """Full pass on z0, set_masks with the SDEdit runner's mask pyramid (min_res 4 x 4, dilation 0), sparse pass on z1."""
    z0, z1, mask = (t.to(device) for t in sd_decoder_inputs(size))
    with torch.no_grad():
        net.set_mode("full")
        full0 = net(z0)
        net.set_masks(downsample_mask(mask, min_res=(4, 4), dilation=0))
        net.set_mode("sparse")
        if fused is not None:
            fused(net)
        sparse1 = net(z1)
    return full0, sparse1
