"""Sparse 3-D convolution on the device (csrc/cg_spconv.cu): the layer types of PointGroup's U-Net with spconv 1.x
semantics -- SubMConv3d k3 and k1, SparseConv3d k2 s2, SparseInverseConv3d k2 -- and the site tables they run on.

A ``Level`` holds a set of distinct sites in ascending (x, y, z) order (z fastest), sized by a row bound ``M``, with
its true count in a device word.  ``index`` synchronises once (it checks the coordinates and sizes the first level by
its site count); ``down`` does not: a coarse level is bounded by min(the finer level's rows, the coarse shape's cells).
``conv`` synchronises once to check that its gather table only names rows of its input.

``index_many`` builds one batched level from several frames, each on its own spatial shape: frame b's sites are its
one-frame level's, at rows [base_b, base_b + n_b) (base_b = the sites of the frames before it), and every table entry
of frame b is the one-frame entry plus base_b.  ``down`` takes batched and one-frame levels alike, so a pyramid and a
forward run on either.  The key layout and its width rule are ``key_layout``'s.  Weights are spconv's own
layout, (kx, ky, kz, Cin, Cout) or flattened to (K, Cin, Cout).  CUDA tensors in, CUDA tensors out; rows of an output
past the level's count are 0.
"""
import numpy as np
import torch

from . import _lib

MAX_COORD = 1 << 21


class Level:
    """vox (M,3) int32 (the first ``count()`` rows are the sites), n (1,) int32 device word, nbr (M,27) int32 (the
    SubM k3 gather table, k = 9 kx + 3 ky + kz), shape: the spatial shape (3 ints).  A batched level has shape None,
    ``shapes`` its frames' spatial shapes (B tuples) and ``frame`` (M,) int32, each site's frame."""

    def __init__(self, vox, n, nbr, shape, frame=None, shapes=None):
        self.vox, self.n, self.nbr = vox, n, nbr
        self.shape = None if shape is None else tuple(int(s) for s in shape)
        self.frame = frame
        self.shapes = None if shapes is None else tuple(tuple(int(s) for s in sh) for sh in shapes)

    @property
    def rows(self):
        return self.vox.shape[0]

    def count(self):
        """Number of sites (synchronises)."""
        return int(self.n.item())


def key_layout(shapes):
    """(f, w): the frame bits and the bits per coordinate of a level over the frames' spatial ``shapes`` (B x 3).
    A site (x, y, z) of frame b has the key b << 3w | x << 2w | y << w | z.  One frame: (0, 21), today's layout
    whatever its shape.  B > 1: f = bit_length(B - 1) and w the smallest width with 2^w >= every shape on every axis;
    ValueError when f + 3w > 63 or a shape is outside [1, 2^21]."""
    shapes = [tuple(int(s) for s in sh) for sh in shapes]
    if not shapes or any(len(sh) != 3 or min(sh) < 1 or max(sh) > MAX_COORD for sh in shapes):
        raise ValueError(f"spconv: every frame needs a shape of 3 ints in [1, 2^21], got {shapes}")
    if len(shapes) == 1:
        return 0, 21
    f, w = (len(shapes) - 1).bit_length(), (max(max(sh) for sh in shapes) - 1).bit_length()
    if f + 3 * w > 63:
        raise ValueError(f"spconv: {len(shapes)} frames need {f} frame bits and the largest shape "
                         f"{max(max(sh) for sh in shapes)} needs {w} bits per axis; a key holds f + 3 w <= 63")
    return f, w


def coarse_shape(shape):
    """get_conv_output_size of SparseConv3d(k2, s2) per axis."""
    return tuple((s - 2) // 2 + 1 if s >= 2 else 0 for s in shape)


def down_rows(M, shapes):
    """The row bound of the coarse level of a level with M rows over frames of these spatial shapes:
    max(1, min(M, the coarse shapes' cells summed over the frames))."""
    cells = sum(int(np.prod(coarse_shape(sh), dtype=np.int64)) for sh in shapes)
    return max(1, min(int(M), cells))


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


def index_many(coords, shapes, offsets=None):
    """The batched level of several frames' sites, and p2v (N,) int32, each point's site (a batched row).
    ``coords`` is a list of (N_b,3) integer CUDA tensors, or one (N,3) CUDA tensor of them concatenated with
    ``offsets`` (B + 1 ints, frame b's points at rows [offsets[b], offsets[b + 1])); ``shapes`` the B spatial shapes.
    ValueError for a coordinate outside [0, its frame's shape) or a batch whose keys do not fit (``key_layout``),
    before any launch.  Synchronises once, as ``index``; the level has exactly as many rows as sites."""
    shapes = [tuple(int(s) for s in sh) for sh in shapes]
    if isinstance(coords, (list, tuple)):
        if offsets is not None:
            raise ValueError("spconv.index_many: give offsets only with concatenated coords")
        offsets = np.cumsum([0] + [len(c) for c in coords])
        coords = torch.cat(list(coords)) if coords else None
    if not isinstance(coords, torch.Tensor) or not coords.is_cuda:
        raise ValueError("spconv.index_many: coords must be CUDA tensors")
    offsets = np.asarray(offsets, dtype=np.int64).reshape(-1)
    B = len(shapes)
    if coords.ndim != 2 or coords.shape[1] != 3 or coords.shape[0] == 0:
        raise ValueError(f"spconv.index_many: coords must be (N,3) with N >= 1, got {tuple(coords.shape)}")
    if len(offsets) != B + 1 or offsets[0] != 0 or offsets[-1] != coords.shape[0] or (np.diff(offsets) < 1).any():
        raise ValueError(f"spconv.index_many: {B} frames need B + 1 offsets from 0 to N = {coords.shape[0]}, each "
                         f"frame with a point; got {offsets.tolist()}")
    key_layout(shapes)
    c = coords.to(torch.int64)
    lims = torch.stack([torch.stack([c[a:b].amin(0), c[a:b].amax(0)]) for a, b in zip(offsets[:-1], offsets[1:])])
    lims = lims.cpu().numpy()
    for b, ((lo, hi), sh) in enumerate(zip(lims, shapes)):
        if lo.min() < 0 or (hi >= np.asarray(sh)).any():
            raise ValueError(f"spconv.index_many: frame {b}'s coordinates must lie in [0, shape), got "
                             f"{lo.tolist()}..{hi.tolist()} for shape {sh}")
    ctx, c = _lib.inputs(c, dtype=torch.int32)
    N, dev = c.shape[0], c.device
    vox, n, p2v, nbr = _i32(N, 3, device=dev), _i32(1, device=dev), _i32(N, device=dev), _i32(N, 27, device=dev)
    frame = _i32(N, device=dev)
    ctx.call("cg_spconv_index_many_dev", ctx.h, c, N, B, offsets.astype(np.int32), np.asarray(shapes, dtype=np.int32),
             vox, n, frame, p2v, nbr)
    V = int(n.item())
    return Level(vox[:V].clone(), n, nbr[:V].clone(), None, frame[:V].clone(), shapes), p2v


def down(level):
    """The coarser level of SparseConv3d(k2, s2) on ``level``, with its tables: (coarse Level, down (P,8), up (M,8)),
    M = level.rows, P = the coarse level's rows = ``down_rows`` (max(1, min(M, coarse cells)), the cells summed over
    the frames of a batched level).
    down[p][k] is the child 2 p + (kx, ky, kz) of parent p (k = 4 kx + 2 ky + kz) or -1; up[c][k] is c's parent at
    k = c - 2 parent(c), -1 at the other seven (all eight for a child dropped from an odd axis's last plane).  A batched
    level's children are dropped against their own frame's coarse shape.  Does not synchronise."""
    ctx = _lib.Context.get(level.vox.device.index)
    M, dev = level.rows, level.vox.device
    shapes = [level.shape] if level.frame is None else level.shapes
    P = down_rows(M, shapes)
    vox, n, nbr = _i32(P, 3, device=dev), _i32(1, device=dev), _i32(P, 27, device=dev)
    dn, up = _i32(P, 8, device=dev), _i32(M, 8, device=dev)
    if level.frame is None:
        ctx.call("cg_spconv_down_dev", ctx.h, level.vox, level.n, M, np.asarray(level.shape, dtype=np.int32), P, vox,
                 n, nbr, dn, up)
        return Level(vox, n, nbr, coarse_shape(level.shape)), dn, up
    frame = _i32(P, device=dev)
    ctx.call("cg_spconv_down_many_dev", ctx.h, level.vox, level.frame, level.n, M, len(shapes),
             np.asarray(shapes, dtype=np.int32), P, vox, n, frame, nbr, dn, up)
    return Level(vox, n, nbr, None, frame, [coarse_shape(sh) for sh in shapes]), dn, up


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
