"""CPU simulator of the launch descriptors of sige_b200.fused — TEST INFRASTRUCTURE.

``sige_b200.fused.Lowering`` turns a traced forward into ``ConvSpec`` / conv_in / tail / attention records and
hands them to an executor.  The product executor (``CudaExecutor``) builds C-ABI descriptors for
libsige_b200.so.  This one interprets the SAME records with plain fp32 torch ops on the CPU, following the
launch contract of include/sige_b200.h (``sige_tile_conv_t``): gather halo tiles from the (virtually
concatenated / upsampled) sources, pre-op, zero outside the image AFTER the pre-op, conv, + bias, fused 1x1
shortcut on flagged tiles / cached residual elsewhere, in-place scatter, extra transformed destinations.

It lets the CPU suite check the tracing + lowering (which launches, which buffers, which folds) against the
reference's golden outputs without a GPU; the kernels themselves are checked on the GPU against the oracle.
"""
from __future__ import annotations

import torch
from torch.nn import functional as F


def _act(z, name):
    return z * torch.sigmoid(z) if name == "swish" else z


class SimExecutor:
    name = "sim"

    def __init__(self):
        self.launches = 0
        self.device = torch.device("cpu")
        self.dtype = torch.float32

    # ------------------------------------------------------------------ fused tile conv
    def prepare_conv(self, fc) -> None:
        s = fc.spec
        # as in the product executor, whether the launch writes its destination's raw tensor is decided when it is prepared: a
        # destination with producer-written views and no raw tensor yet keeps receiving only the views, even when the
        # sparse_update epilogue gives the buffer a raw tensor later; one with neither gets a raw tensor
        write_raw = s.dst is not None and (s.dst.has_raw or not s.aux)

        def run(_stream):
            self.launches += 1
            w = s.weight.clone()
            b = None if s.bias is None else s.bias.clone()
            if s.out_row_scale is not None:
                rows, f = s.out_row_scale
                w[:rows] *= f
                if b is not None:
                    b[:rows] *= f
            k, st, R = s.k, s.stride, s.block
            ro = (R - k) // st + 1
            if s.src_is_stack:
                X = s.srcs[0][0].float()
                M = X.shape[0]
                coords = None if s.idx is None else [(bi, iy, ix) for bi in range(s.B) for (iy, ix) in s.idx.tolist()]
            else:
                parts = [F.interpolate(t.float(), scale_factor=2.0, mode="nearest") if up else t.float() for (t, up) in s.srcs]
                full = parts[0] if len(parts) == 1 else torch.cat(parts, 1)
                B, C, H, W = full.shape
                assert (H, W) == (s.H, s.W) and B == s.B, (s.name, full.shape, s.B, s.H, s.W)
                if s.scale is not None:
                    full = full * (s.scale.view(1, -1, 1, 1) if s.scale.dim() == 1 else s.scale.view(B, -1, 1, 1))
                if s.shift is not None:
                    full = full + (s.shift.view(1, -1, 1, 1) if s.shift.dim() == 1 else s.shift.view(B, -1, 1, 1))
                full = _act(full, s.act)
                P = R + 4
                padded = F.pad(full, (P, P, P, P))                  # zero AFTER the pre-op
                idx = s.idx.tolist()
                tiles, coords = [], []
                if s.tile_img is not None:          # batch of independent edits: tile i belongs to image tile_img[i]
                    assert len(idx) == s.N == s.tile_img.numel()
                    for bi, (iy, ix) in zip(s.tile_img.tolist(), idx):
                        assert 0 <= bi < B
                        tiles.append(padded[bi, :, iy + P:iy + P + R, ix + P:ix + P + R])
                        coords.append((bi, iy, ix))
                else:
                    for bi in range(B):
                        for (iy, ix) in idx:
                            if iy <= -20000:          # SIGE_TILE_NONE padding of a fixed-capacity list: reads zeros, writes nothing
                                tiles.append(torch.zeros_like(padded[0, :, :R, :R]))
                                coords.append(None)
                                continue
                            tiles.append(padded[bi, :, iy + P:iy + P + R, ix + P:ix + P + R])
                            coords.append((bi, iy, ix))
                X = torch.stack(tiles)
                M = X.shape[0]
            out = F.conv2d(X, w, b, stride=st)
            assert out.shape[2] == ro
            fresh = [False] * M
            if s.shortcut is not None:
                sc_tensors, sc_w, sc_b, sc_flags = s.shortcut
                raw = torch.cat([t.float() for t in sc_tensors], 1)
                flags = [1] * s.N if sc_flags is None else sc_flags.tolist()
                assert k == 3 and R == 6 and st == 1
                for m, co_ in enumerate(coords):
                    if co_ is None:
                        continue
                    bi, iy, ix = co_
                    if flags[m % s.N]:
                        fresh[m] = True
                        Pp = 8
                        rp = F.pad(raw[bi:bi + 1], (Pp, Pp, Pp, Pp))
                        centre = rp[:, :, iy + 1 + Pp:iy + 5 + Pp, ix + 1 + Pp:ix + 5 + Pp]
                        out[m] += F.conv2d(centre, sc_w, sc_b)[0]
            if s.dst_stack is not None:
                assert s.residual is None and not s.aux
                s.dst_stack.copy_(out)
                return
            dst = s.dst
            Bd, Cd, Hd, Wd = dst.shape
            res = None if s.residual is None else s.residual.float()
            for m in range(M):
                if coords is not None and coords[m] is None:
                    continue
                bi, iy, ix = coords[m] if coords is not None else (0, 0, 0)
                assert (s.off + iy) >= 0 and (s.off + ix) >= 0
                oy, ox = (s.off + iy) // st, (s.off + ix) // st
                for r in range(ro):
                    for c in range(ro):
                        hh, ww = oy + r, ox + c
                        if not (0 <= hh < Hd and 0 <= ww < Wd):
                            continue
                        v = out[m, :, r, c].clone()
                        if res is not None and not fresh[m]:
                            v = v + res[bi, :, hh, ww]
                        if write_raw:
                            dst.raw[bi, :, hh, ww] = v
                        for (view, sc, sh, act) in s.aux:
                            z = v
                            if sc is not None:
                                z = z * sc
                            if sh is not None:
                                z = z + sh
                            view[bi, :, hh, ww] = _act(z, act)

        fc.launch_fn = run

    # ------------------------------------------------------------------ stem / tail / attention / gather
    def prepare_conv_in(self, rec):
        def run(_stream):
            self.launches += 1
            y = F.conv2d(rec.x.float(), rec.weight.float(), None if rec.bias is None else rec.bias.float(), padding=1)
            B, C, H, W = y.shape
            sel = torch.zeros((B, H, W), dtype=torch.bool)
            if rec.tiles is None:
                sel[:] = True
            else:
                imgs = [None] * rec.tiles.shape[0] if rec.tile_img is None else rec.tile_img.tolist()
                for bi, (iy, ix) in zip(imgs, rec.tiles.tolist()):
                    if iy <= -20000:
                        continue
                    sel[slice(None) if bi is None else bi, max(iy, 0):max(iy + rec.tile_size, 0), max(ix, 0):max(ix + rec.tile_size, 0)] = True
            sel4 = sel[:, None].expand_as(y)
            if rec.out.has_raw:
                rec.out.raw[sel4] = y[sel4].to(rec.out.raw.dtype)
            for (view, sc, sh, act) in rec.aux:
                z = y
                if sc is not None:
                    z = z * sc.view(1, -1, 1, 1)
                if sh is not None:
                    z = z + sh.view(1, -1, 1, 1)
                view[sel4] = _act(z, act)[sel4].to(view.dtype)

        return run

    def prepare_tail(self, x, groups, eps, gamma, beta, act, weight, bias, out):
        def run(_stream):
            self.launches += 3
            z = F.group_norm(x.float(), groups, None if gamma is None else gamma.float(), None if beta is None else beta.float(), eps)
            out.copy_(F.conv2d(_act(z, act), weight.float(), None if bias is None else bias.float(), padding=1))

        return run

    def attention_supported(self, n_tokens, channels):
        return True

    def tail_supported(self, channels, cout):
        return True

    def prepare_attention(self, qkv_tokens, out_tokens, pdl):
        def run(_stream):
            self.launches += 1
            C = qkv_tokens.shape[2] // 3
            q, k, v = qkv_tokens[..., :C].float(), qkv_tokens[..., C:2 * C].float(), qkv_tokens[..., 2 * C:].float()
            att = torch.softmax(q @ k.transpose(1, 2), dim=-1)      # q arrives pre-scaled
            out_tokens.copy_(att @ v)

        return run

    def spade_supported(self, x, gamma, beta):
        return True

    def prepare_spade(self, x, gamma, beta, slope, out):
        def run(_stream):
            self.launches += 1
            # as the kernel: 1 + gamma in fp32, then one fused multiply-add (a single rounding, here of the float64 value)
            z = x.double() * (1 + gamma.float()).double() + beta.double()
            out.copy_(torch.where(z > 0, z, z * float(torch.tensor(slope, dtype=torch.float32))))

        return run

    def sparse_attention_supported(self, head_dim):
        return True

    def prepare_sparse_attention(self, q, k, v, scale, out):
        def run(_stream):
            self.launches += 1
            att = torch.softmax(torch.matmul(q.float(), k.float().transpose(-1, -2)) * scale, dim=-1)       # [bh, n, d] or strided [b, h, n, d]
            out.copy_(torch.matmul(att, v.float()))

        return run

    def gather(self, x, block, idx, scale, shift, act, act_first, up=0):
        if up:
            x = F.interpolate(x.float(), scale_factor=2.0, mode="nearest")
        B, C, H, W = x.shape
        z = x.float()
        if not act_first:
            if scale is not None:
                z = z * scale
            if shift is not None:
                z = z + shift
        z = _act(z, act)
        if act_first:
            if scale is not None:
                z = z * scale
            if shift is not None:
                z = z + shift
        P = max(block) + 4
        padded = F.pad(z, (P, P, P, P))
        tiles = [padded[b, :, iy + P:iy + P + block[0], ix + P:ix + P + block[1]] for b in range(B) for (iy, ix) in idx.tolist()]
        if not tiles:
            return x.new_zeros((0, C, block[0], block[1]))
        return torch.stack(tiles)

    def launch_counter(self):
        return self.launches
