"""GauGAN compressed with GAN Compression (the sub-mobile SPADE generator) built on the ``sige.nn`` operator surface.

A benchmark / test workload, not part of the operator library: the GPU machines have no copy of the reference, so the model
whose separable-conv launches are measured must exist in-tree.  It is written from the architecture of reference
gaugan/models/sub_mobile_spade_generators/sige_fused_sub_mobile_spade_generator.py, gaugan/models/sige_normalization.py
(SIGEFusedSubMobileSPADE) and gaugan/models/mobile_modules.py (SIGESeparableConv2d) with the SAME module tree and parameter
names, so that ``init_deterministic`` gives both the same weights and their state dicts load into each other.  The one
substitution: the reference's SynchronizedBatchNorm2d is ``nn.BatchNorm2d`` (same state-dict keys; one process, eval mode).

Per-mode behaviour is the reference's: ``full`` = dense pass that fills the Scatter* caches and records, per separable conv, the
instance-norm statistics as a per-channel (scale, shift); ``sparse`` = the tile-sparse pass that re-uses them.  In sparse mode a
SPADE layer's gamma and beta are each depthwise 3x3 -> x*scale+shift -> 1x1 on the tile stack: what the fused step lowers to
one ``sige_separable_conv`` launch per layer.
"""
from __future__ import annotations

import types
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch
from torch import nn
from torch.nn import functional as F

from ..nn import Gather, Scatter, ScatterGather, ScatterWithBlockResidual, SIGEConv2d, SIGEModel, SIGEModule

# the published GAN Compression GauGAN (Cityscapes) sub-network, and the miniature the tests run
FULL_CONFIG = "32_32_32_48_32_24_24_32"
MINI_CONFIG = "16_16_16_16_16_16_16_16"


def decode_config(config_str: str) -> Dict[str, List[int]]:
    return {"channels": [int(c) for c in config_str.split("_")]}


def instance_norm_fold(x: torch.Tensor, norm: nn.InstanceNorm2d):
    """Instance norm of a batch-1 activation and its per-channel (scale, shift) form: norm(x) == x * scale + shift."""
    assert not norm.track_running_stats
    n, c, h, w = x.shape
    assert n == 1
    var, mean = torch.var_mean(x, unbiased=False, dim=[2, 3], keepdim=True)
    var = torch.sqrt(var + norm.eps)
    x = (x - mean) / var
    scale = 1 / var[0, :, 0, 0]
    shift = -(mean / var)[0, :, 0, 0]
    if norm.affine:
        x = x.view(n, c, h, w)
        x = x * norm.weight.view(1, -1, 1, 1)
        x = x + norm.bias.view(1, -1, 1, 1)
        scale = scale * norm.weight
        shift = shift * norm.weight
        shift = shift + norm.bias
    return x, scale, shift


class SIGESeparableConv2d(SIGEModule):
    """Depthwise k x k (groups = in_channels) -> instance norm -> 1x1.  Sparse mode replaces the norm by the dense pass's
    statistics: x * scale + shift."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, norm_layer=nn.InstanceNorm2d, use_bias=True,
                 scale_factor=1, support_sparse=False):
        super().__init__()
        self.support_sparse = support_sparse
        Conv2d = SIGEConv2d if support_sparse else nn.Conv2d
        self.conv = nn.Sequential(
            Conv2d(in_channels=in_channels, out_channels=in_channels * scale_factor, kernel_size=kernel_size, stride=stride, padding=padding,
                   groups=in_channels, bias=use_bias),
            norm_layer(in_channels * scale_factor),
            Conv2d(in_channels=in_channels * scale_factor, out_channels=out_channels, kernel_size=1, stride=1, bias=use_bias),
        )
        self.scale, self.shift = None, None

    def forward(self, x):
        if self.mode == "full":
            assert x.shape[0] == 1
            x = self.conv[0](x)
            x, self.scale, self.shift = instance_norm_fold(x, self.conv[1])
            return self.conv[2](x)
        if self.mode in ("sparse", "profile"):
            if not self.support_sparse:
                return self.conv(x)
            x = self.conv[0](x)
            x = x * self.scale.view(1, -1, 1, 1) + self.shift.view(1, -1, 1, 1)
            return self.conv[2](x)
        raise NotImplementedError("Unknown mode [%s]!!!" % self.mode)


class SIGEFusedSubMobileSPADE(SIGEModule):
    """SPADE with a parameter-free batch norm of `oc` channels whose gamma / beta come from two separable convs of the shared
    activation.  Its batch norm is folded by the CONSUMER's Gather (scale / shift recorded in the dense pass)."""

    def __init__(self, config_text, norm_nc, nhidden, oc, seg_gather: Optional[Gather] = None, shortcut_conv: Optional[nn.Conv2d] = None,
                 main_block_size: Optional[int] = 6, shortcut_block_size: Optional[int] = 4):
        super().__init__()
        is_shortcut = shortcut_conv is not None
        self.is_shortcut = is_shortcut
        assert config_text == "spadesyncbatch3x3", config_text
        assert norm_nc >= oc
        self.param_free_norm = nn.BatchNorm2d(oc, affine=False)
        block_size = shortcut_block_size if is_shortcut else main_block_size
        self.support_sparse = seg_gather is not None
        self.mlp_gamma = SIGESeparableConv2d(nhidden, oc, kernel_size=3, padding=1, support_sparse=self.support_sparse)
        self.mlp_beta = SIGESeparableConv2d(nhidden, oc, kernel_size=3, padding=1, support_sparse=self.support_sparse)
        if self.support_sparse:
            if is_shortcut:
                self.scatter_gamma = Scatter(seg_gather)
                self.gather_gamma = Gather(shortcut_conv, block_size)
                self.scatter_beta = Scatter(seg_gather)
                self.gather_beta = Gather(shortcut_conv, block_size)
            else:
                self.scatter_gather_gamma = ScatterGather(seg_gather)
                self.scatter_gather_beta = ScatterGather(seg_gather)
        self.scale, self.shift = None, None

    def forward(self, x, actv):
        if self.mode == "full":
            normalized = self.param_free_norm(x)
            var = torch.sqrt(self.param_free_norm.running_var + self.param_free_norm.eps)
            self.scale = 1 / var
            self.shift = -(self.param_free_norm.running_mean / var)
        elif self.mode in ("sparse", "profile"):
            normalized = x
        else:
            raise NotImplementedError("Unknown mode [%s]!!!" % self.mode)
        gamma = self.mlp_gamma(actv)
        beta = self.mlp_beta(actv)
        if self.support_sparse:
            if self.is_shortcut:
                gamma = self.gather_gamma(self.scatter_gamma(gamma))
                beta = self.gather_beta(self.scatter_beta(beta))
            else:
                gamma = self.scatter_gather_gamma(gamma)
                beta = self.scatter_gather_beta(beta)
        return normalized * (1 + gamma) + beta


class SIGEFusedSubMobileSPADEResnetBlock(SIGEModule):
    def __init__(self, fin, fout, ic, opt, config, support_sparse: bool = False):
        super().__init__()
        self.fin, self.fout, self.ic, self.opt, self.config = fin, fout, ic, opt, config
        self.learned_shortcut = fin != fout
        channel, hidden = config["channel"], config["hidden"]
        self.nhidden = hidden
        fmiddle = min(fin, fout)
        main_block_size = opt.main_block_size
        main_support_sparse = support_sparse and main_block_size is not None
        MainConv2d = SIGEConv2d if main_support_sparse else nn.Conv2d

        self.mlp_shared = nn.Sequential(MainConv2d(opt.semantic_nc, hidden * (3 if self.learned_shortcut else 2), kernel_size=3, padding=1), nn.ReLU())
        self.conv_0 = MainConv2d(ic, channel, kernel_size=3, padding=1)
        self.conv_1 = MainConv2d(channel, channel if self.learned_shortcut else ic, kernel_size=3, padding=1)
        if main_support_sparse:
            self.seg_gather = Gather(self.mlp_shared[0], main_block_size)
            self.seg_scatter_gather = ScatterGather(self.seg_gather)
            self.main_gather = Gather(self.conv_0, main_block_size)
            self.main_scatter_gather = ScatterGather(self.main_gather)

        shortcut_block_size = None
        shortcut_support_sparse = False
        if self.learned_shortcut:
            shortcut_block_size = opt.shortcut_block_size
            shortcut_support_sparse = main_support_sparse and shortcut_block_size is not None
            ShortcutConv2d = SIGEConv2d if shortcut_support_sparse else nn.Conv2d
            self.conv_s = ShortcutConv2d(ic, channel, kernel_size=1, bias=False)
            if shortcut_support_sparse:
                self.shortcut_gather = Gather(self.conv_s, shortcut_block_size)
                self.scatter = ScatterWithBlockResidual(self.main_gather, self.shortcut_gather)
            elif main_support_sparse:
                self.scatter = Scatter(self.main_gather)
        elif main_support_sparse:
            self.scatter = Scatter(self.main_gather)
        self.main_support_sparse = main_support_sparse
        self.shortcut_support_sparse = shortcut_support_sparse

        assert "spectral" not in opt.norm_G
        seg_gather = self.seg_gather if main_support_sparse else None
        kw = dict(seg_gather=seg_gather, main_block_size=main_block_size, shortcut_block_size=shortcut_block_size)
        self.norm_0 = SIGEFusedSubMobileSPADE(opt.norm_G, fin, nhidden=hidden, oc=ic, **kw)
        self.norm_1 = SIGEFusedSubMobileSPADE(opt.norm_G, fmiddle, nhidden=hidden, oc=channel, **kw)
        if self.learned_shortcut:
            self.norm_s = SIGEFusedSubMobileSPADE(opt.norm_G, fin, nhidden=hidden, oc=ic, shortcut_conv=self.conv_s, **kw)

    def forward(self, x, seg):
        if self.mode == "full":
            return self.full_forward(x, seg)
        if self.mode in ("sparse", "profile"):
            return self.sparse_forward(x, seg)
        raise NotImplementedError("Unknown mode [%s]!!!" % self.mode)

    def full_forward(self, x, seg):
        sparse, sc_sparse = self.main_support_sparse, self.shortcut_support_sparse
        seg = F.interpolate(seg, size=x.size()[2:], mode="nearest")
        if sparse:
            seg = self.seg_gather(seg)          # records the shape only
        actvs = self.mlp_shared(seg)
        if sparse:
            actvs = self.seg_scatter_gather(actvs)
        if self.learned_shortcut:
            actv_0, actv_1, actv_s = torch.split(actvs, self.nhidden, dim=1)
            x_s = self.shortcut_gather(x) if sc_sparse else x
            x_s = self.conv_s(self.norm_s(x_s, actv_s))
        else:
            actv_0, actv_1 = torch.split(actvs, self.nhidden, dim=1)
            x_s = x
        dx = self.main_gather(x) if sparse else x
        dx = self.conv_0(self.actvn(self.norm_0(dx, actv_0)))
        if sparse:
            dx = self.main_scatter_gather(dx)
        dx = self.conv_1(self.actvn(self.norm_1(dx, actv_1)))
        return self.scatter(dx, x_s) if sparse else x_s + dx

    def sparse_forward(self, x, seg):
        sparse, sc_sparse = self.main_support_sparse, self.shortcut_support_sparse
        seg = F.interpolate(seg, size=x.size()[2:], mode="nearest")
        if sparse:
            seg = self.seg_gather(seg)
        actvs = self.mlp_shared(seg)
        if sparse:
            actvs = self.seg_scatter_gather(actvs)
        if self.learned_shortcut:
            actv_0, actv_1, actv_s = torch.split(actvs, self.nhidden, dim=1)
            if sc_sparse:
                x_s = self.shortcut_gather(x, self.norm_s.scale.view(1, -1, 1, 1), self.norm_s.shift.view(1, -1, 1, 1))
            else:
                x_s = self.norm_s.param_free_norm(x)
            x_s = self.conv_s(self.norm_s(x_s, actv_s))
        else:
            actv_0, actv_1 = torch.split(actvs, self.nhidden, dim=1)
            x_s = x
        if sparse:
            dx = self.main_gather(x, self.norm_0.scale.view(1, -1, 1, 1), self.norm_0.shift.view(1, -1, 1, 1))
        else:
            dx = self.norm_0.param_free_norm(x)
        dx = self.conv_0(self.actvn(self.norm_0(dx, actv_0)))
        if sparse:
            dx = self.main_scatter_gather(dx, self.norm_1.scale.view(1, -1, 1, 1), self.norm_1.shift.view(1, -1, 1, 1))
        else:
            dx = self.norm_1.param_free_norm(dx)
        dx = self.conv_1(self.actvn(self.norm_1(dx, actv_1)))
        return self.scatter(dx, x_s) if sparse else x_s + dx

    def actvn(self, x):
        return F.leaky_relu(x, 2e-1)


class SIGEFusedSubMobileSPADEGenerator(SIGEModel):
    def __init__(self, opt, config, **kwargs):
        super().__init__()
        self.opt, self.config = opt, config
        nf = opt.ngf
        self.sw, self.sh = self.compute_latent_vector_size(opt)
        ch = config["channels"]
        self.fc = nn.Conv2d(opt.semantic_nc, 16 * ch[0], 3, padding=1)
        is_most = opt.num_upsampling_layers == "most"
        n_sparse = opt.num_sparse_layers

        def block(fin, fout, ic, c, mult, level):
            return SIGEFusedSubMobileSPADEResnetBlock(fin, fout, ic, opt, {"channel": c * mult, "hidden": c * 2},
                                                      support_sparse=n_sparse >= level + is_most)

        ic = ch[0] * 16
        self.head_0 = block(16 * nf, 16 * nf, ic, ch[1], 16, 7)
        self.G_middle_0 = block(16 * nf, 16 * nf, ic, ch[2], 16, 6)
        self.G_middle_1 = block(16 * nf, 16 * nf, ic, ch[3], 16, 5)
        self.up_0 = block(16 * nf, 8 * nf, ic, ch[4], 8, 4)
        ic = ch[4] * 8
        self.up_1 = block(8 * nf, 4 * nf, ic, ch[5], 4, 3)
        ic = ch[5] * 4
        self.up_2 = block(4 * nf, 2 * nf, ic, ch[6], 2, 2)
        ic = ch[6] * 2
        self.up_3 = block(2 * nf, 1 * nf, ic, ch[7], 1, 1)
        if opt.num_upsampling_layers == "most":
            raise NotImplementedError
        self.conv_img = nn.Conv2d(ch[7], 3, 3, padding=1)
        self.up = nn.Upsample(scale_factor=2)

    @staticmethod
    def compute_latent_vector_size(opt):
        num_up_layers = {"normal": 5, "more": 6, "most": 7}[opt.num_upsampling_layers]
        sw = opt.crop_size // (2 ** num_up_layers)
        return sw, round(sw / opt.aspect_ratio)

    def forward(self, input):
        seg = input
        x = F.interpolate(seg, size=(self.sh, self.sw))
        x = self.fc(x)
        x = self.head_0(x, seg)
        x = self.up(x)
        x = self.G_middle_0(x, seg)
        if self.opt.num_upsampling_layers in ("more", "most"):
            x = self.up(x)
        x = self.G_middle_1(x, seg)
        x = self.up(x)
        x = self.up_0(x, seg)
        x = self.up(x)
        x = self.up_1(x, seg)
        x = self.up(x)
        x = self.up_2(x, seg)
        x = self.up(x)
        x = self.up_3(x, seg)
        x = self.conv_img(F.leaky_relu(x, 2e-1))
        return torch.tanh(x)


# ------------------------------------------------------------------------------------------------ builders and inputs
def gaugan_gc_opt(size: str = "mini"):
    """The generator options of the full-size GauGAN workload (Cityscapes, 512 x 1024, 5 sparse blocks) and of its miniature
    (ngf 32, 64 x 128, 4 sparse blocks)."""
    if size == "full":
        return types.SimpleNamespace(ngf=64, semantic_nc=36, num_upsampling_layers="more", num_sparse_layers=5, crop_size=1024, aspect_ratio=2.0,
                                     norm_G="spadesyncbatch3x3", main_block_size=6, shortcut_block_size=4)
    return types.SimpleNamespace(ngf=32, semantic_nc=36, num_upsampling_layers="normal", num_sparse_layers=4, crop_size=128, aspect_ratio=2.0,
                                 norm_G="spadesyncbatch3x3", main_block_size=6, shortcut_block_size=4)


def build_gaugan_gc(size: str = "mini", cls=SIGEFusedSubMobileSPADEGenerator) -> nn.Module:
    """`cls` = this file's generator, or the reference's class of the same name (same constructor)."""
    from .ddpm import init_deterministic

    net = cls(gaugan_gc_opt(size), decode_config(FULL_CONFIG if size == "full" else MINI_CONFIG))
    return init_deterministic(net, seed=31).eval()


def gaugan_gc_inputs(size: str = "mini") -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """One-hot 36-channel label maps, original and edited, and the edit mask (mini: 64 x 128; full: 512 x 1024 with a 2.98 % edit):
    the label maps of the full-SPADE GauGAN workload."""
    rng = np.random.default_rng(77)
    H, W = (512, 1024) if size == "full" else (64, 128)
    lab0 = rng.integers(0, 35, size=(H // 8, W // 8)).repeat(8, 0).repeat(8, 1)
    lab1 = lab0.copy()
    if size == "full":
        lab1[200:320, 400:530] = 7                    # 120 x 130 px = 2.98 % of the image
    else:
        lab1[20:30, 70:88] = 7
    mask = torch.from_numpy(lab0 != lab1)

    def onehot(lab):
        t = torch.zeros(1, 36, H, W)
        t.scatter_(1, torch.from_numpy(lab)[None, None].long(), 1.0)
        return t

    return onehot(lab0), onehot(lab1), mask


def gaugan_gc_edits(size: str = "mini", E: int = 3) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """E independent label edits of the workload's scene: the original map [1, 36, H, W], the edited maps [E, 36, H, W] and their
    masks [E, H, W] (the `set_masks` argument of a batch, after the usual pyramid per edit).  Edit 0 is the workload's edit, 1 a
    smaller one elsewhere (`edit_b`), 2 a strip along the image's left border, later ones seeded rectangles of 1 to 3 % of the
    image anywhere."""
    s0, s1, mask = gaugan_gc_inputs(size)
    H, W = int(s0.shape[2]), int(s0.shape[3])
    lab0 = s0.argmax(1)[0]
    maps = [s1[0]]
    for e in range(1, E):
        lab = lab0.clone()
        if e == 1:
            if size == "full":
                lab[360:440, 700:800] = 3
            else:
                lab[40:48, 16:28] = 3
        elif e == 2:
            lab[H // 4:H // 4 + H // 3, 0:W // 12] = 11
        else:
            g = torch.Generator().manual_seed(1000 + e)
            h, w = (int(v) for v in torch.randint(H // 10, H // 5, (2,), generator=g))
            y, x = int(torch.randint(0, H - h + 1, (1,), generator=g)), int(torch.randint(0, W - w + 1, (1,), generator=g))
            lab[y:y + h, x:x + w] = int(torch.randint(0, 35, (1,), generator=g))
        t = torch.zeros(36, H, W)
        t.scatter_(0, lab[None], 1.0)
        maps.append(t)
    s1s = torch.stack(maps, 0)
    return s0, s1s, (s1s != s0).any(1)


def run_gaugan_gc(net: nn.Module, downsample_mask, dilate_mask, device="cpu", fused=None, size: str = "mini"):
    """Dense pass on the original label map, set_masks (the dilated difference-mask pyramid of reference gaugan/runner.py), sparse
    pass on the edited one."""
    s0, s1, mask = (t.to(device) for t in gaugan_gc_inputs(size))
    with torch.no_grad():
        net.set_mode("full")
        full0 = net(s0)
        net.set_masks(downsample_mask(dilate_mask(mask, 1), min_res=(4, 8), dilation=0))
        net.set_mode("sparse")
        if fused is not None:
            fused(net)
        sparse1 = net(s1)
    return full0, sparse1
