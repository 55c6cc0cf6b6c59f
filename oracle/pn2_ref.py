"""Numpy fp32 restatement of the reference's PointNet++ primitives (pointnet2.py:14-149) -- ORACLE.

The floating-point forms are the reference's: FPS uses the direct form ((dx^2+dy^2)+dz^2) (:71),
the ball query the expanded form -2<s,d> + |s|^2 + |d|^2 (:30-32).  The dot product of the expanded
form is accumulated as fma(sz,dz, fma(sy,dy, sx*dx)) which is what the BLAS sgemm behind
``torch.matmul`` does for K=3 on an FMA machine; tests/golden pins this against the reference itself.

Also the exact fp32 contracts of the feature-propagation kernels (three_nn, three_interp), the FPS launch rule
(fps_config) and a float64 reference of the shared-MLP stacks with an error bound (SharedMLP64).
"""
import numpy as np

from oracle.encoder_ref import FoldedNet, u_bf16x3, u_fp32

f32 = np.float32


def _fma(a, b, c):
    # correctly rounded fp32 fma via float64 (exact product of two fp32 fits in 48 bits; one rounding
    # of the fp64 sum then one to fp32 can double-round only in astronomically rare ties)
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(f32)


def sq_expanded(src, dst):
    """square_distance (:14-33): src (S,3), dst (N,3) -> (S,N) fp32."""
    src = src.astype(f32); dst = dst.astype(f32)
    sx, sy, sz = src[:, 0:1], src[:, 1:2], src[:, 2:3]
    dx, dy, dz = dst[None, :, 0], dst[None, :, 1], dst[None, :, 2]
    dot = _fma(np.broadcast_to(sz, (src.shape[0], dst.shape[0])), np.broadcast_to(dz, (src.shape[0], dst.shape[0])),
               _fma(np.broadcast_to(sy, (src.shape[0], dst.shape[0])), np.broadcast_to(dy, (src.shape[0], dst.shape[0])),
                    (sx * dx).astype(f32)))
    ss = ((sx * sx).astype(f32) + (sy * sy).astype(f32)).astype(f32) + (sz * sz).astype(f32)
    dd = ((dx * dx).astype(f32) + (dy * dy).astype(f32)).astype(f32) + (dz * dz).astype(f32)
    out = (f32(-2.0) * dot).astype(f32)
    out = (out + ss).astype(f32)
    out = (out + dd).astype(f32)
    return out


def square_distance(src, dst):
    return np.stack([sq_expanded(src[b], dst[b]) for b in range(src.shape[0])])


def index_points(points, idx):
    """(:35-51)"""
    B = points.shape[0]
    return np.stack([points[b][idx[b]] for b in range(B)])


def farthest_point_sample(xyz, npoint, start_idx):
    """(:54-75) with an explicit start index per cloud."""
    xyz = xyz.astype(f32)
    B, N, _ = xyz.shape
    centroids = np.zeros((B, npoint), dtype=np.int64)
    for b in range(B):
        distance = np.full((N,), 1e10, dtype=f32)
        farthest = int(start_idx[b])
        P = xyz[b]
        for i in range(npoint):
            centroids[b, i] = farthest
            d = P - P[farthest][None]
            dist = ((d[:, 0] * d[:, 0]).astype(f32) + (d[:, 1] * d[:, 1]).astype(f32)).astype(f32) + (d[:, 2] * d[:, 2]).astype(f32)
            mask = dist < distance
            distance[mask] = dist[mask]
            farthest = int(np.argmax(distance))      # first maximum, like torch.max on CPU
    return centroids


def query_ball_point(radius, nsample, xyz, new_xyz):
    """(:78-98): nsample smallest indices with d2 <= r2 (excluded iff d2 > r2), padded with the first; N if empty."""
    B, N, _ = xyz.shape
    S = new_xyz.shape[1]
    r2 = f32(radius ** 2)
    out = np.zeros((B, S, nsample), dtype=np.int64)
    for b in range(B):
        d = sq_expanded(new_xyz[b], xyz[b])
        for s in range(S):
            inb = np.nonzero(~(d[s] > r2))[0][:nsample]
            row = np.full((nsample,), N if inb.size == 0 else inb[0], dtype=np.int64)
            row[: inb.size] = inb
            out[b, s] = row
    return out


def fps_config(N, max_cluster=16):
    """(cluster size, points per thread) that cg_fps_dev (csrc/cg_pn2.cu) launches for N points: the cheapest cluster
    by its cost model base + 0.025 x points per thread, among the sizes whose points fit 32 per thread of 256; the
    template is the smallest of 4 / 8 / 16 / 32 that holds them.  None when N does not fit."""
    best, cfg = None, None
    for size, base in ((2, 0.70), (4, 0.83), (8, 1.0), (16, 1.45)):
        if size > max_cluster:
            break
        ppt = -(-N // (size * 256))
        if ppt > 32:
            continue
        cost = base + 0.025 * ppt
        if best is None or cost < best:
            best, cfg = cost, (size, next(p for p in (4, 8, 16, 32) if ppt <= p))
    return cfg


def three_nn(xyz1, xyz2):
    """The 3 nearest of the S sparse points xyz2 (B,S,3) for every dense point of xyz1 (B,N,3), as three_nn_kernel
    (csrc/cg_sa.cu) states it: expanded-form fp32 distances (sq_expanded), the first three of a stable ascending sort
    (ties -> lower index), weights (1/(d+1e-8)) / ((r0+r1)+r2) in fp32.  S == 2 keeps two neighbours, normalised
    over two.  Returns idx (B,N,k) int64 and weight (B,N,k) fp32, k = min(S, 3)."""
    B, N, _ = xyz1.shape
    k = min(xyz2.shape[1], 3)
    idx = np.zeros((B, N, k), dtype=np.int64)
    w = np.zeros((B, N, k), dtype=f32)
    for b in range(B):
        d = sq_expanded(xyz1[b], xyz2[b])
        i = np.argsort(d, axis=1, kind="stable")[:, :k]
        r = f32(1.0) / (np.take_along_axis(d, i, 1) + f32(1e-8))
        norm = r[:, 0] + r[:, 1]
        if k == 3:
            norm = norm + r[:, 2]
        idx[b], w[b] = i, r / norm[:, None]
    return idx, w


def three_interp(points1, points2, idx, w):
    """cat([points1, interpolated]) of three_interp_kernel: interpolated = (p0*w0 + p1*w1) + p2*w2 in fp32, every
    product and sum rounded on its own (no fused multiply-add).  points1 (B,N,D1) or None, points2 (B,S,D2)."""
    p = index_points(points2.astype(f32), idx)                 # (B,N,k,D2)
    t = p * w[..., None]
    out = t[:, :, 0] + t[:, :, 1]
    if idx.shape[2] == 3:
        out = out + t[:, :, 2]
    return out if points1 is None else np.concatenate([points1.astype(f32), out], axis=-1)


class SharedMLP64:
    """Float64 reference of a cg_mlp stack (shared 1x1 conv + folded BN + ReLU per layer) with a per-value bound on
    the GPU's error, built from the exact fp32 folded weights the GPU receives (weights.fold_mlp).  The bound follows
    oracle/encoder_ref.py: e_out = |W|^T e_in + u (|W|^T (|x| + e_in) + |b|) per layer, u = u_bf16x3(K) where
    cg_linear_launch puts the layer on tensor cores (engine >= 1, >= 64 rows, K % 64 == 0, C_out >= 64), else
    u_fp32(K).  ReLU and the max over a group's members add no error: a group's bound is its members' largest."""

    def __init__(self, state_dict, nlayers):
        import torch
        from catgrasp_b200.weights import fold_mlp
        Wts, bs = fold_mlp(state_dict, nlayers)
        self.W = [torch.from_numpy(W.astype(np.float64)) for W in Wts]
        self.b = [torch.from_numpy(b.astype(np.float64)) for b in bs]
        self.dims = [W.shape[0] for W in Wts] + [Wts[-1].shape[1]]

    def on_tc(self, engine, rows):
        return [FoldedNet.fc_on_tc(engine, rows, W.shape[0], W.shape[1]) for W in self.W]

    def rows(self, x, engine, rows=None):
        """x (R, dims[0]) -> y (R, dims[-1]) and its bound, both float64 numpy; ``rows`` is the row count of the GPU
        call (it decides tensor cores or FMA), by default R."""
        import torch
        x = torch.as_tensor(np.asarray(x, dtype=np.float64))
        e = torch.zeros_like(x)
        for W, b, tc in zip(self.W, self.b, self.on_tc(engine, x.shape[0] if rows is None else rows)):
            x, e = FoldedNet._lin(x, e, W, b, u_bf16x3(W.shape[0]) if tc else u_fp32(W.shape[0]))
            x = x.clamp_min(0.0)
        return x.numpy(), e.numpy()

    def group_max(self, grouped, engine, rows=None):
        """grouped (G,K,dims[0]) -> max over the K members (G,dims[-1]) and its bound; ``rows`` defaults to G*K."""
        G, K, Cin = grouped.shape
        y, e = self.rows(np.asarray(grouped).reshape(G * K, Cin), engine, G * K if rows is None else rows)
        return y.reshape(G, K, -1).max(1), e.reshape(G, K, -1).max(1)


def sample_and_group(npoint, radius, nsample, xyz, points, start_idx):
    """(:101-129)"""
    fps_idx = farthest_point_sample(xyz, npoint, start_idx)
    new_xyz = index_points(xyz, fps_idx)
    idx = query_ball_point(radius, nsample, xyz, new_xyz)
    grouped_xyz = index_points(xyz, idx)
    grouped_xyz_norm = (grouped_xyz.astype(f32) - new_xyz.astype(f32)[:, :, None, :]).astype(f32)
    if points is not None:
        new_points = np.concatenate([grouped_xyz_norm, index_points(points, idx)], axis=-1)
    else:
        new_points = grouped_xyz_norm
    return new_xyz, new_points, grouped_xyz, fps_idx
