"""Sparse 3-D convolution on the device (csrc/cg_spconv.cu): the layer types of PointGroup's U-Net with spconv 1.x
semantics -- SubMConv3d k3 and k1, SparseConv3d k2 s2, SparseInverseConv3d k2 -- and the site tables they run on.

A ``Level`` holds a set of distinct sites in ascending (x, y, z) order (z fastest), sized by a row bound ``M``, with
its true count in a device word.  ``index`` synchronises once (it checks the coordinates and sizes the first level by
its site count); ``down`` does not: a coarse level is bounded by min(the finer level's rows, the coarse shape's cells).
``conv`` synchronises once to check that its gather table only names rows of its input.  Weights are spconv's own
layout, (kx, ky, kz, Cin, Cout) or flattened to (K, Cin, Cout).  CUDA tensors in, CUDA tensors out; rows of an output
past the level's count are 0.
"""
import numpy as np
import torch

from . import _lib

MAX_COORD = 1 << 21


class Level:
    """vox (M,3) int32 (the first ``count()`` rows are the sites), n (1,) int32 device word, nbr (M,27) int32 (the
    SubM k3 gather table, k = 9 kx + 3 ky + kz), shape: the spatial shape (3 ints)."""

    def __init__(self, vox, n, nbr, shape):
        self.vox, self.n, self.nbr, self.shape = vox, n, nbr, tuple(int(s) for s in shape)

    @property
    def rows(self):
        return self.vox.shape[0]

    def count(self):
        """Number of sites (synchronises)."""
        return int(self.n.item())


def _i32(*shape, device):
    return torch.empty(shape, dtype=torch.int32, device=device)


def index(coords, shape=None):
    """The level of the distinct sites of ``coords`` (N,3) integers (CUDA tensor), and p2v (N,) int32, each point's
    site.  ``shape`` is the spatial shape (default: the largest coordinate + 1 per axis).  ValueError for a
    coordinate outside [0, min(shape, 2^21)).  The level has exactly as many rows as sites."""
    if not isinstance(coords, torch.Tensor) or not coords.is_cuda:
        raise ValueError("spconv.index: coords must be a CUDA tensor")
    if coords.ndim != 2 or coords.shape[1] != 3 or coords.shape[0] == 0:
        raise ValueError(f"spconv.index: coords must be (N,3) with N >= 1, got {tuple(coords.shape)}")
    c = coords.to(torch.int64)
    lo, hi = c.amin(0).tolist(), c.amax(0).tolist()
    shape = tuple(h + 1 for h in hi) if shape is None else tuple(int(s) for s in shape)
    if min(lo) < 0 or any(h >= s for h, s in zip(hi, shape)) or max(shape) > MAX_COORD:
        raise ValueError(f"spconv.index: coordinates must lie in [0, shape) with shape <= 2^21, got {lo}..{hi}"
                         f" for shape {shape}")
    ctx, c = _lib.inputs(c, dtype=torch.int32)
    N, dev = c.shape[0], c.device
    vox, n, p2v, nbr = _i32(N, 3, device=dev), _i32(1, device=dev), _i32(N, device=dev), _i32(N, 27, device=dev)
    ctx.call("cg_spconv_index_dev", ctx.h, c, N, vox, n, p2v, nbr)
    V = int(n.item())
    return Level(vox[:V].clone(), n, nbr[:V].clone(), shape), p2v


def down(level):
    """The coarser level of SparseConv3d(k2, s2) on ``level``, with its tables: (coarse Level, down (P,8), up (M,8)),
    M = level.rows, P = the coarse level's rows = max(1, min(M, coarse cells)).
    down[p][k] is the child 2 p + (kx, ky, kz) of parent p (k = 4 kx + 2 ky + kz) or -1; up[c][k] is c's parent at
    k = c - 2 parent(c), -1 at the other seven (all eight for a child dropped from an odd axis's last plane)."""
    ctx = _lib.Context.get(level.vox.device.index)
    M, dev = level.rows, level.vox.device
    coarse = tuple((s - 2) // 2 + 1 if s >= 2 else 0 for s in level.shape)
    P = max(1, min(M, int(np.prod(coarse, dtype=np.int64))))
    vox, n, nbr = _i32(P, 3, device=dev), _i32(1, device=dev), _i32(P, 27, device=dev)
    dn, up = _i32(P, 8, device=dev), _i32(M, 8, device=dev)
    ctx.call("cg_spconv_down_dev", ctx.h, level.vox, level.n, M, np.asarray(level.shape, dtype=np.int32), P, vox, n,
             nbr, dn, up)
    return Level(vox, n, nbr, coarse), dn, up


def conv(x, nbr, W, n, bn=None, bias=None, residual=None):
    """One sparse convolution: out (M,Cout) float32, rows r < n[0] =
    (sum_k W[k]^T act(x[nbr[r][k]]) + bias) + residual[r], act = ReLU(BN) when ``bn`` = (scale, shift) is given.
    x (rows,Cin) float32; nbr (M,K) int32 gather table (-1 absent), or None for the 1x1 convolution (M = rows of x);
    W (..., Cin, Cout) with K kernel offsets; n the output level's count word (1,).  bn = (scale (Cin,), shift (Cin,)),
    bias (Cout,), residual (M,Cout).  ValueError for any other shape or for a table entry >= rows of x."""
    Cin, Cout = W.shape[-2], W.shape[-1]
    W = W.reshape(-1, Cin, Cout)
    K = W.shape[0]
    if x.ndim != 2 or x.shape[1] != Cin:
        raise ValueError(f"spconv.conv: x must be (rows, {Cin}), got {tuple(x.shape)}")
    if nbr is None:
        if K != 1:
            raise ValueError("spconv.conv: a 1x1 convolution (nbr=None) takes one kernel offset")
        M = x.shape[0]
    else:
        if nbr.ndim != 2 or nbr.shape[1] != K:
            raise ValueError(f"spconv.conv: nbr must be (M, {K}), got {tuple(nbr.shape)}")
        M = nbr.shape[0]
    scale, shift = (None, None) if bn is None else bn
    for name, a, want in (("scale", scale, (Cin,)), ("shift", shift, (Cin,)), ("bias", bias, (Cout,)),
                          ("residual", residual, (M, Cout)), ("n", n, (1,))):
        if a is not None and tuple(a.shape) != want:
            raise ValueError(f"spconv.conv: {name} must have shape {want}, got {tuple(a.shape)}")
    if nbr is not None and nbr.numel() and int(nbr.max()) >= x.shape[0]:
        raise ValueError(f"spconv.conv: nbr names row {int(nbr.max())} of an input with {x.shape[0]} rows")
    ctx, x, W, scale, shift, bias, residual = _lib.inputs(x, W, scale, shift, bias, residual, dtype=torch.float32)
    dev = x.device
    nbr = None if nbr is None else nbr.to(device=dev, dtype=torch.int32).contiguous()
    n = n.to(device=dev, dtype=torch.int32).contiguous()
    out = torch.zeros((M, Cout), dtype=torch.float32, device=dev)
    ctx.call("cg_spconv_conv_dev", ctx.h, x, Cin, nbr, K, n, M, W, Cout, scale, shift, bias, residual, out)
    return out
