"""PointNet++ sampling/grouping primitives and the PointNet models, with the
names and call signatures of the reference's ``pointnet2.py`` (file:line cited
per function), executing on H100 through libcatgrasp_b200.so.

All tensors are CUDA tensors; indices are returned as int64 like the reference.
"""
import numpy as np
import torch

from . import _lib
from .net import PointNetCls, PointNetSeg  # noqa: F401  (pointnet2.py:275,302)


def _f32(*tensors):
    """(ctx, *tensors): the context of the first tensor's device, and the tensors as contiguous float32 where they are
    (Context.call refuses a CPU tensor, or one on another device, before any launch)."""
    return (_lib.Context.get(tensors[0].device.index), *[None if t is None else t.to(torch.float32).contiguous()
                                                         for t in tensors])


def square_distance(src, dst):
    """pointnet2.py:14-33. src (B,N,3), dst (B,M,3) -> (B,N,M) in the expanded form."""
    ctx, src, dst = _f32(src, dst)
    B, N, _ = src.shape
    M = dst.shape[1]
    out = torch.empty((B, N, M), dtype=torch.float32, device=src.device)
    ctx.call("cg_square_distance_dev", ctx.h, src, dst, B, N, M, out)
    return out


def index_points(points, idx):
    """pointnet2.py:35-51. points (B,N,C), idx (B,S) or (B,S,K) -> (B,S[,K],C)."""
    ctx, points = _f32(points)
    B, N, Cc = points.shape
    shape = list(idx.shape)
    idx32 = idx.reshape(B, -1).to(torch.int32).contiguous()
    S = idx32.shape[1]
    out = torch.empty((B, S, Cc), dtype=torch.float32, device=points.device)
    ctx.call("cg_index_points_dev", ctx.h, points, idx32, B, N, Cc, S, out)
    return out.reshape(shape + [Cc])


def farthest_point_sample(xyz, npoint, start_idx=None):
    """pointnet2.py:54-75. xyz (B,N,3) -> (B,npoint) int64.

    ``start_idx`` (B,) makes the reference's ``torch.randint`` start (:66) explicit;
    when None it is drawn with torch.randint exactly like the reference.
    """
    ctx, xyz = _f32(xyz)
    B, N, _ = xyz.shape
    if start_idx is None:
        start_idx = torch.randint(0, N, (B,), dtype=torch.long).to(xyz.device)
    start = torch.as_tensor(start_idx).to(device=xyz.device, dtype=torch.int32).contiguous()
    out = torch.empty((B, npoint), dtype=torch.int32, device=xyz.device)
    ctx.call("cg_fps_dev", ctx.h, xyz, B, N, int(npoint), start, out)
    return out.long()


def query_ball_point(radius, nsample, xyz, new_xyz):
    """pointnet2.py:78-98. -> (B,S,nsample) int64, nsample smallest in-ball indices, padded with the first."""
    ctx, xyz, new_xyz = _f32(xyz, new_xyz)
    B, N, _ = xyz.shape
    S = new_xyz.shape[1]
    out = torch.empty((B, S, nsample), dtype=torch.int32, device=xyz.device)
    r2 = float(np.float32(radius ** 2))   # torch compares the fp32 tensor against float32(radius**2), :93
    ctx.call("cg_ball_query_dev", ctx.h, r2, int(nsample), xyz, new_xyz, B, N, S, out)
    return out.long()


def sample_and_group(npoint, radius, nsample, xyz, points, returnfps=False, start_idx=None):
    """pointnet2.py:101-129."""
    ctx, xyz, pts = _f32(xyz, points)
    B, N, Cc = xyz.shape
    S = npoint
    fps_idx = farthest_point_sample(xyz, npoint, start_idx=start_idx)
    new_xyz = index_points(xyz, fps_idx)
    idx = query_ball_point(radius, nsample, xyz, new_xyz)
    idx32 = idx.to(torch.int32).contiguous()
    D = 0 if points is None else points.shape[-1]
    new_points = torch.empty((B, S, nsample, 3 + D), dtype=torch.float32, device=xyz.device)
    ctx.call("cg_group_points_dev", ctx.h, xyz, pts, new_xyz, idx32, B, N, D, S, nsample, new_points)
    if returnfps:
        grouped_xyz = index_points(xyz, idx)
        return new_xyz, new_points, grouped_xyz, fps_idx
    return new_xyz, new_points


def sample_and_group_all(xyz, points):
    """pointnet2.py:132-149 (pure views/concat, no kernel needed)."""
    B, N, Cc = xyz.shape
    new_xyz = torch.zeros(B, 1, Cc, device=xyz.device)
    grouped_xyz = xyz.view(B, 1, N, Cc)
    if points is not None:
        new_points = torch.cat([grouped_xyz, points.view(B, 1, N, -1)], dim=-1)
    else:
        new_points = grouped_xyz
    return new_xyz, new_points


# ---------------------------------------------------------------------------------------------------------
# Set-abstraction / feature-propagation modules (the upstream family the reference cites at pointnet2.py:274,304),
# built on the primitives above.  Weights follow the upstream state_dict layout:
#   mlp_convs.{i}.weight (C_out, C_in, 1[, 1]) / .bias,  mlp_bns.{i}.{weight,bias,running_mean,running_var}
class _SharedMLP:
    def __init__(self, state_dict, nlayers, device=None):
        import ctypes as C
        from .weights import fold_mlp
        self.ctx = _lib.Context.get(device)
        Wts, bs = fold_mlp(state_dict, nlayers)
        dims = [Wt.shape[0] for Wt in Wts] + [Wts[-1].shape[1]]
        self.dims = dims
        cdims = (C.c_int * len(dims))(*dims)
        cw = (C.c_void_p * nlayers)(*[w.ctypes.data for w in Wts])
        cb = (C.c_void_p * nlayers)(*[b.ctypes.data for b in bs])
        h = C.c_void_p()
        self.ctx.call("cg_mlp_create", self.ctx.h, nlayers, cdims, cw, cb, C.byref(h))
        self.h = h

    def __del__(self):
        try:
            if getattr(self, "h", None):
                self.ctx.call("cg_mlp_destroy", self.h)
                self.h = None
        except Exception:
            pass


class PointNetSetAbstraction:
    """forward(xyz (B,3,N), points (B,D,N) | None) -> (new_xyz (B,3,S), new_points (B,C_out,S)).

    sample_and_group (pointnet2.py:101-129) / sample_and_group_all (:132-149), then [conv1x1 + BN + ReLU] x L over
    every (group, member) row and a max over the group's nsample members."""

    def __init__(self, npoint, radius, nsample, in_channel, mlp, group_all, state_dict, device=None):
        self.npoint, self.radius, self.nsample, self.group_all = npoint, radius, nsample, group_all
        self.mlp = _SharedMLP(state_dict, len(mlp), device=device)
        assert self.mlp.dims[0] == in_channel and list(self.mlp.dims[1:]) == list(mlp), (self.mlp.dims, in_channel, mlp)

    def forward(self, xyz, points, start_idx=None):
        _, xyz, pts = _f32(xyz.permute(0, 2, 1), None if points is None else points.permute(0, 2, 1))
        if self.group_all:
            new_xyz, new_points = sample_and_group_all(xyz, pts)
        else:
            new_xyz, new_points = sample_and_group(self.npoint, self.radius, self.nsample, xyz, pts, start_idx=start_idx)
        new_points = new_points.to(torch.float32).contiguous()
        B, S, K, Cin = new_points.shape
        out = torch.empty((B, S, self.mlp.dims[-1]), dtype=torch.float32, device=xyz.device)
        self.mlp.ctx.call("cg_group_mlp_max_dev", self.mlp.h, new_points, B * S, K, out)
        return new_xyz.permute(0, 2, 1), out.permute(0, 2, 1)

    __call__ = forward


class PointNetFeaturePropagation:
    """forward(xyz1 (B,3,N), xyz2 (B,3,S), points1 (B,D1,N) | None, points2 (B,D2,S)) -> (B,C_out,N).

    Inverse-distance interpolation of the sparse features onto the dense points over the 3 nearest sparse points
    (square_distance, pointnet2.py:14-33), concatenated behind the skip features, then [conv1 + BN + ReLU] x L."""

    def __init__(self, in_channel, mlp, state_dict, device=None):
        self.mlp = _SharedMLP(state_dict, len(mlp), device=device)
        assert self.mlp.dims[0] == in_channel and list(self.mlp.dims[1:]) == list(mlp), (self.mlp.dims, in_channel, mlp)

    def forward(self, xyz1, xyz2, points1, points2, return_nn=False):
        ctx, x1, x2, p1, p2 = _f32(xyz1.permute(0, 2, 1), xyz2.permute(0, 2, 1),
                                   None if points1 is None else points1.permute(0, 2, 1), points2.permute(0, 2, 1))
        B, N, _ = x1.shape
        S, D2 = p2.shape[1], p2.shape[2]
        D1 = 0 if p1 is None else p1.shape[2]
        idx = w = None
        if S == 1:
            interp = p2.repeat(1, N, 1)
            feat = interp if p1 is None else torch.cat([p1, interp], dim=-1)
        else:
            feat = torch.empty((B, N, D1 + D2), dtype=torch.float32, device=x1.device)
            idx = torch.empty((B, N, 3), dtype=torch.int32, device=x1.device)
            w = torch.empty((B, N, 3), dtype=torch.float32, device=x1.device)
            ctx.call("cg_three_interp_dev", ctx.h, x1, x2, p1, D1, p2, D2, B, N, S, feat, idx, w)
            if S == 2:   # the module family's sort()[:, :, :3] of two columns: two neighbours
                idx, w = idx[:, :, :2], w[:, :, :2]
        feat = feat.contiguous()
        out = torch.empty((B, N, self.mlp.dims[-1]), dtype=torch.float32, device=x1.device)
        self.mlp.ctx.call("cg_shared_mlp_dev", self.mlp.h, feat, B * N, out)
        out = out.permute(0, 2, 1)
        return (out, idx.long(), w) if return_nn else out

    __call__ = forward
