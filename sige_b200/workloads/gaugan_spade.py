"""The SPADE GauGAN generator (the full model, not the compressed one) built on the ``sige.nn`` operator surface.

A benchmark / test workload, not part of the operator library: the GPU machines have no copy of the reference, so the model whose
launches are measured must exist in-tree.  It is written from the architecture of reference
gaugan/models/spade_generators/sige_fused_spade_generator.py (SIGEFusedSPADEGenerator, SIGEFusedSPADEResnetBlock) and
gaugan/models/sige_normalization.py (SIGEFusedSPADE) with the SAME module tree and parameter names, so that ``init_deterministic``
gives both the same weights and their state dicts load into each other.  The one substitution: the reference's
SynchronizedBatchNorm2d is ``nn.BatchNorm2d`` (same state-dict keys; one process, eval mode).

Per-mode behaviour is the reference's: ``full`` = dense pass that fills the Scatter* caches and records each SPADE's batch norm as a
per-channel (scale, shift); ``sparse`` = the tile-sparse pass, where the block's Gathers apply that (scale, shift).  A SPADE layer's
gamma and beta are the two channel halves of ONE conv (`mlp_gamma_beta`) of a channel window of the block's shared activation
(`torch.split(actvs, nhidden)`): what the fused step lowers to a strided launch for `mlp_gamma_beta` and a modulated launch, with
gamma / beta windows, for the conv that reads the SPADE.  The label maps are ``gaugan_gc.gaugan_gc_inputs``.
"""
from __future__ import annotations

import types
from typing import Optional

import torch
from torch import nn
from torch.nn import functional as F

from ..nn import Gather, Scatter, ScatterGather, ScatterWithBlockResidual, SIGEConv2d, SIGEModel, SIGEModule


class SIGEFusedSPADE(SIGEModule):
    """normalized * (1 + gamma) + beta, with [gamma | beta] = mlp_gamma_beta(actv) (3x3, 2 * norm_nc outputs).  Its parameter-free
    batch norm is folded by the CONSUMER's Gather in sparse mode (scale / shift recorded in the dense pass)."""

    def __init__(self, config_text, norm_nc, nhidden: int = 128, seg_gather: Optional[Gather] = None, shortcut_conv: Optional[nn.Conv2d] = None,
                 main_block_size: Optional[int] = 6, shortcut_block_size: Optional[int] = 4):
        super().__init__()
        is_shortcut = shortcut_conv is not None
        self.norm_nc = norm_nc
        self.is_shortcut = is_shortcut
        assert config_text in ("spadesyncbatch3x3", "spadebatch3x3"), config_text
        self.param_free_norm = nn.BatchNorm2d(norm_nc, affine=False)
        block_size = shortcut_block_size if is_shortcut else main_block_size
        self.support_sparse = seg_gather is not None
        Conv2d = SIGEConv2d if self.support_sparse else nn.Conv2d
        self.mlp_gamma_beta = Conv2d(nhidden, 2 * norm_nc, kernel_size=3, padding=1)
        if self.support_sparse:
            if is_shortcut:
                self.scatter = Scatter(seg_gather)
                self.gather = Gather(shortcut_conv, block_size)
            else:
                self.scatter_gather = ScatterGather(seg_gather)
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
        gamma_beta = self.mlp_gamma_beta(actv)
        if self.support_sparse:
            gamma_beta = self.gather(self.scatter(gamma_beta)) if self.is_shortcut else self.scatter_gather(gamma_beta)
        gamma, beta = torch.split(gamma_beta, self.norm_nc, dim=1)
        return normalized * (1 + gamma) + beta


class SIGEFusedSPADEResnetBlock(SIGEModule):
    def __init__(self, fin, fout, opt, support_sparse: bool = False):
        super().__init__()
        self.fin, self.fout, self.opt = fin, fout, opt
        self.nhidden = opt.ngf * 2
        self.learned_shortcut = fin != fout
        fmiddle = min(fin, fout)
        main_block_size = opt.main_block_size
        main_support_sparse = support_sparse and main_block_size is not None
        MainConv2d = SIGEConv2d if main_support_sparse else nn.Conv2d

        self.mlp_shared = nn.Sequential(MainConv2d(opt.semantic_nc, self.nhidden * (3 if self.learned_shortcut else 2), kernel_size=3, padding=1), nn.ReLU())
        self.conv_0 = MainConv2d(fin, fmiddle, kernel_size=3, padding=1)
        self.conv_1 = MainConv2d(fmiddle, fout, kernel_size=3, padding=1)
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
            self.conv_s = ShortcutConv2d(fin, fout, kernel_size=1, bias=False)
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
        kw = dict(nhidden=self.nhidden, seg_gather=seg_gather, main_block_size=main_block_size, shortcut_block_size=shortcut_block_size)
        self.norm_0 = SIGEFusedSPADE(opt.norm_G, fin, **kw)
        self.norm_1 = SIGEFusedSPADE(opt.norm_G, fmiddle, **kw)
        if self.learned_shortcut:
            self.norm_s = SIGEFusedSPADE(opt.norm_G, fin, shortcut_conv=self.conv_s, **kw)

    def forward(self, x, seg):
        if self.mode == "full":
            return self._forward(x, seg, sparse_pass=False)
        if self.mode in ("sparse", "profile"):
            return self._forward(x, seg, sparse_pass=True)
        raise NotImplementedError("Unknown mode [%s]!!!" % self.mode)

    def _forward(self, x, seg, sparse_pass: bool):
        """Dense pass: the SPADEs normalise with their batch norms and the Gathers only record shapes.  Sparse pass: the Gathers
        fold each SPADE's batch norm (scale, shift) into the tiles they cut."""
        sparse, sc_sparse = self.main_support_sparse, self.shortcut_support_sparse
        seg = F.interpolate(seg, size=x.size()[2:], mode="nearest")
        if sparse:
            seg = self.seg_gather(seg)
        actvs = self.mlp_shared(seg)
        if sparse:
            actvs = self.seg_scatter_gather(actvs)
        if self.learned_shortcut:
            actv_0, actv_1, actv_s = torch.split(actvs, self.nhidden, dim=1)
            if not sparse_pass:
                x_s = self.shortcut_gather(x) if sc_sparse else x
            elif sc_sparse:
                x_s = self.shortcut_gather(x, self.norm_s.scale.view(1, -1, 1, 1), self.norm_s.shift.view(1, -1, 1, 1))
            else:
                x_s = self.norm_s.param_free_norm(x)
            x_s = self.conv_s(self.norm_s(x_s, actv_s))
        else:
            actv_0, actv_1 = torch.split(actvs, self.nhidden, dim=1)
            x_s = x
        if not sparse_pass:
            dx = self.main_gather(x) if sparse else x
        elif sparse:
            dx = self.main_gather(x, self.norm_0.scale.view(1, -1, 1, 1), self.norm_0.shift.view(1, -1, 1, 1))
        else:
            dx = self.norm_0.param_free_norm(x)
        dx = self.conv_0(self.actvn(self.norm_0(dx, actv_0)))
        if not sparse_pass:
            dx = self.main_scatter_gather(dx) if sparse else dx
        elif sparse:
            dx = self.main_scatter_gather(dx, self.norm_1.scale.view(1, -1, 1, 1), self.norm_1.shift.view(1, -1, 1, 1))
        else:
            dx = self.norm_1.param_free_norm(dx)
        dx = self.conv_1(self.actvn(self.norm_1(dx, actv_1)))
        return self.scatter(dx, x_s) if sparse else x_s + dx

    def actvn(self, x):
        return F.leaky_relu(x, 2e-1)


class SIGEFusedSPADEGenerator(SIGEModel):
    def __init__(self, opt, **kwargs):
        super().__init__()
        self.opt = opt
        nf = opt.ngf
        self.sw, self.sh = self.compute_latent_vector_size(opt)
        self.fc = nn.Conv2d(opt.semantic_nc, 16 * nf, 3, padding=1)
        is_most = opt.num_upsampling_layers == "most"
        n_sparse = opt.num_sparse_layers

        def block(fin, fout, level):
            return SIGEFusedSPADEResnetBlock(fin, fout, opt, support_sparse=n_sparse >= level + is_most)

        self.head_0 = block(16 * nf, 16 * nf, 7)
        self.G_middle_0 = block(16 * nf, 16 * nf, 6)
        self.G_middle_1 = block(16 * nf, 16 * nf, 5)
        self.up_0 = block(16 * nf, 8 * nf, 4)
        self.up_1 = block(8 * nf, 4 * nf, 3)
        self.up_2 = block(4 * nf, 2 * nf, 2)
        self.up_3 = block(2 * nf, 1 * nf, 1)
        final_nc = nf
        if is_most:
            self.up_4 = block(1 * nf, nf // 2, 0)
            final_nc = nf // 2
        self.conv_img = nn.Conv2d(final_nc, 3, 3, padding=1)
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
        if self.opt.num_upsampling_layers == "most":
            x = self.up(x)
            x = self.up_4(x, seg)
        x = self.conv_img(F.leaky_relu(x, 2e-1))
        return torch.tanh(x)


# ------------------------------------------------------------------------------------------------ builders
def gaugan_spade_opt(size: str = "mini"):
    """The generator options of the full-size GauGAN workload (Cityscapes, 512 x 1024, ngf 64, `more` up-sampling layers, 5 sparse
    blocks) and of its miniature (ngf 32, 64 x 128, 4 sparse blocks)."""
    if size == "full":
        return types.SimpleNamespace(ngf=64, semantic_nc=36, num_upsampling_layers="more", num_sparse_layers=5, crop_size=1024, aspect_ratio=2.0,
                                     norm_G="spadesyncbatch3x3", main_block_size=6, shortcut_block_size=4)
    return types.SimpleNamespace(ngf=32, semantic_nc=36, num_upsampling_layers="normal", num_sparse_layers=4, crop_size=128, aspect_ratio=2.0,
                                 norm_G="spadesyncbatch3x3", main_block_size=6, shortcut_block_size=4)


def build_gaugan_spade(size: str = "mini", cls=SIGEFusedSPADEGenerator) -> nn.Module:
    """`cls` = this file's generator, or the reference's class of the same name (same constructor)."""
    from .ddpm import init_deterministic

    return init_deterministic(cls(gaugan_spade_opt(size)), seed=23).eval()
