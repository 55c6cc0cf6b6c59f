"""PointGroup's segmentation network on the device, inference only: the voxelisation, the sparse U-Net and the offset
head (PointGroup/model/pointgroup/pointgroup.py, ``PointGroup.forward`` up to ``pt_offsets``).

``PointGroupNet.offsets(level, p2v, feats)`` goes from the first level's sites, each point's site and the point
features to the per-point offsets (N,3) float32.  The level pyramid is built once (``spconv.index``, then six
``spconv.down``); after ``index`` nothing synchronises: every layer runs through ``cg_spconv_conv_dev`` on tables the
forward built itself, so the gather-table check of the public ``spconv.conv`` (one synchronisation per call) is not
needed.  A batched level (``spconv.index_many``, several frames) runs through the same calls, and each frame's offsets
equal its one-frame forward's bit for bit.  The score / proposal branch never runs at inference (``epoch = prepare_epochs - 1``) and is not built.

Wiring, per level with C channels (UBlock):
  blocks: block_reps ResidualBlocks  x + SubM3(BN2 ReLU . SubM3(BN1 ReLU x))      (SubM k1 with bias on x when the
                                                                                    input width differs)
  identity = that output; then, except on the coarsest level:
  conv: BN ReLU SparseConv3d k2 s2 -> the inner UBlock -> deconv: BN ReLU SparseInverseConv3d k2 on the same pairs
  cat(identity, decoder) -> blocks_tail (the first block 2C -> C)
then output_layer (BN, ReLU), Linear m->m, BN, ReLU, Linear m->3 in one kernel per site, gathered to the points.
"""
import numpy as np
import torch

from . import _lib, spconv
from .weights import PG_INPUT_C, PG_LEVELS, pack_pointgroup


def _dev(a, device):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(device)


def _to_device(tree, device):
    if isinstance(tree, dict):
        return {k: _to_device(v, device) for k, v in tree.items()}
    if isinstance(tree, (list, tuple)):
        return type(tree)(_to_device(v, device) for v in tree)
    return _dev(tree, device) if isinstance(tree, np.ndarray) else tree


def pyramid(level):
    """The seven levels of the U-Net from the first: [(Level, down (P,8), up (M,8))] with None tables on the
    coarsest level.  Does not synchronise."""
    out = []
    for _ in range(PG_LEVELS - 1):
        coarse, dn, up = spconv.down(level)
        out.append((level, dn, up))
        level = coarse
    out.append((level, None, None))
    return out


def voxel_mean(level, p2v, feats):
    """pointgroup_ops.voxelization mode 4: (level.rows, C) float32, the mean of each site's point features (N,C)
    float32 (CUDA), summed in ascending point index as the reference's kernel does.  Does not synchronise."""
    ctx = _lib.Context.get(feats.device.index)
    N, C = feats.shape
    out = torch.zeros((level.rows, C), dtype=torch.float32, device=feats.device)
    ctx.call("cg_pointgroup_voxel_mean_dev", ctx.h, feats, N, C, p2v, level.n, level.rows, out)
    return out


class PointGroupNet:
    """The packed weights of one PointGroup checkpoint on one device.  ``sd`` is a state_dict (torch tensors or
    numpy arrays); ``m`` and ``block_reps`` come from the model's config."""

    def __init__(self, sd, m, block_reps, device=None):
        if block_reps not in (1, 2):
            raise NotImplementedError(f"PointGroupNet: block_reps = {block_reps}; the U-Net's tail block i takes "
                                      "(2 - i) * C channels, so only 1 and 2 build")
        self.m, self.block_reps = int(m), int(block_reps)
        self.ctx = _lib.Context.get(device)
        self.device = torch.device("cuda", self.ctx.device)
        self.w = _to_device(pack_pointgroup(sd, self.m, self.block_reps), self.device)

    # -- one convolution through the C entry, on tables this forward built (no check, no synchronisation) --
    def _conv(self, x, nbr, W, n, rows, bn=None, bias=None, residual=None):
        K, Cin, Cout = W.shape
        out = torch.empty((rows, Cout), dtype=torch.float32, device=self.device)
        scale, shift = (None, None) if bn is None else bn
        self.ctx.call("cg_spconv_conv_dev", self.ctx.h, x, Cin, nbr, K, n, rows, W, Cout, scale, shift, bias,
                      residual, out)
        return out

    def _block(self, x, lv, blk):
        nbr, n, rows = lv.nbr, lv.n, lv.rows
        res = x if blk["Wi"] is None else self._conv(x, None, blk["Wi"], n, rows, bias=blk["bi"])
        h = self._conv(x, nbr, blk["W1"], n, rows, bn=blk["bn1"], bias=blk["b1"])
        return self._conv(h, nbr, blk["W2"], n, rows, bn=blk["bn2"], bias=blk["b2"], residual=res)

    def _ublock(self, x, levels, i):
        lv, dn, up = levels[i]
        L = self.w["levels"][i]
        for blk in L["blocks"]:
            x = self._block(x, lv, blk)
        if dn is None:
            return x
        coarse = levels[i + 1][0]
        bn, W, b = L["down"]
        y = self._conv(x, dn, W, coarse.n, coarse.rows, bn=bn, bias=b)
        y = self._ublock(y, levels, i + 1)
        bn, W, b = L["up"]
        d = self._conv(y, up, W, lv.n, lv.rows, bn=bn, bias=b)
        x = torch.cat((x, d), 1)
        for blk in L["tail"]:
            x = self._block(x, lv, blk)
        return x

    def unet(self, levels, vfeats):
        """input_conv and the U-Net: the level-1 features (V,m) before output_layer."""
        lv = levels[0][0]
        W, b = self.w["input"]
        x = self._conv(vfeats, lv.nbr, W, lv.n, lv.rows, bias=b)
        return self._ublock(x, levels, 0)

    def head(self, level, x, p2v):
        """output_layer and the offset head per site, gathered to the points: (N,3) float32."""
        h = self.w["head"]
        N = p2v.shape[0]
        site = torch.empty((level.rows, 3), dtype=torch.float32, device=self.device)
        out = torch.empty((N, 3), dtype=torch.float32, device=self.device)
        self.ctx.call("cg_pointgroup_head_dev", self.ctx.h, x, self.m, level.n, level.rows, h["bn"][0], h["bn"][1],
                      h["W1"], h["b1"], h["W2"], h["b2"], p2v, N, site, out)
        return out

    def offsets(self, level, p2v, feats, levels=None):
        """pt_offsets (N,3) float32 from the first level (``spconv.index`` of the point sites), each point's site
        p2v (N,) int32 and the point features (N,6) float32 (normals, then coordinates).  ``levels`` is the
        pyramid of ``level`` when the caller has built it.  Does not synchronise."""
        if feats.ndim != 2 or feats.shape[1] != PG_INPUT_C or feats.shape[0] != p2v.shape[0]:
            raise ValueError(f"PointGroupNet: feats must be (N, {PG_INPUT_C}) with N = len(p2v), "
                             f"got {tuple(feats.shape)} and {tuple(p2v.shape)}")
        feats = feats.to(device=self.device, dtype=torch.float32).contiguous()
        p2v = p2v.to(device=self.device, dtype=torch.int32).contiguous()
        levels = pyramid(level) if levels is None else levels
        x = self.unet(levels, voxel_mean(level, p2v, feats))
        return self.head(level, x, p2v)
