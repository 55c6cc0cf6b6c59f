"""PointGroup's segmentation network in float64 with a propagated error bound, and its host front -- ORACLE, test only.

Restates, independently of catgrasp_b200/pointgroup.py and csrc/cg_spconv.cu:
  * pointgroup_ops ``voxelization_idx`` (sites in first-seen order, each site's points in ascending index) and
    ``voxelization`` mode 4 (out = 0; for each point out = fl(out + fl(fl(1/n) * x)), float32, no FMA);
  * the host front of PointGroupPredictor.predict (predicter.py:234-300) with n_slice_per_side = 1;
  * the network up to ``pt_offsets`` (PointGroup/model/pointgroup/pointgroup.py: input_conv, UBlock of
    [m, ..., 7m], output_layer, offset head), composed from oracle/spconv_ref.conv.

Bound (the rule of spconv_ref.py, per value): every activation carries |device - exact| <= e, where the device works in
fp32 on BN scale / shift and folded head weights that were narrowed from float64.  A BN + ReLU in front of a conv is
applied here, not in spconv_ref.conv, so the narrowing of scale and shift is in its bound (z = s x + t):
    ea = |s| ex (1 + u)^2 + u (1 + u) (|s x| + |t|) + u |z|,  and 0 where z + |s| ex (1 + u)^2 + ... < 0 (ReLU)
The head's first Linear runs on float32 weights rounded from the folded float64 ones, one more u |W|^T |a| + u |b|.
The bound is rigorous and grows by the weights' absolute row sums at every layer, so after the U-Net's ~60 layers in
series it is loose by many orders of magnitude; tests pair it with a relative check against the float64 values.
"""
import numpy as np

from . import spconv_ref as S

U32 = 2.0 ** -24
BN_EPS = 1e-5
LEVELS = 7


# ---------------------------------------------------------------- voxelisation (pointgroup_ops, mode 4)
def voxelization_idx(locs):
    """voxelize_idx for (N,4) int64 locs (batch, x, y, z): (voxel_locs (V,4) int64 in first-seen order, p2v (N,)
    int32, v2p (V, 1 + maxActive) int32: the count, then the site's points in ascending index, 0 padded)."""
    locs = np.asarray(locs, dtype=np.int64)
    _, first, inv = np.unique(locs, axis=0, return_index=True, return_inverse=True)
    inv = inv.reshape(-1)
    order = np.argsort(first, kind="stable")             # unique rows sorted by first appearance
    rank = np.empty_like(order)
    rank[order] = np.arange(len(order))
    p2v = rank[inv]
    V = len(order)
    counts = np.bincount(p2v, minlength=V)
    v2p = np.zeros((V, 1 + int(counts.max())), dtype=np.int32)
    v2p[:, 0] = counts
    pts = np.argsort(p2v, kind="stable")                 # points grouped by site, ascending index within
    start = np.concatenate([[0], np.cumsum(counts)[:-1]])
    slot = np.arange(len(pts)) - start[p2v[pts]]
    v2p[p2v[pts], 1 + slot] = pts
    return locs[first[order]], p2v.astype(np.int32), v2p


def voxelization(feats, v2p):
    """voxelize_fp mode 4 in float32: (V,C)."""
    feats = np.asarray(feats, dtype=np.float32)
    n = v2p[:, 0].astype(np.int64)
    mult = np.where(n > 0, np.float32(1) / np.maximum(n, 1).astype(np.float32), np.float32(1)).astype(np.float32)
    out = np.zeros((len(v2p), feats.shape[1]), dtype=np.float32)
    order = np.argsort(-n, kind="stable")                # sites by count, descending: rank j touches a prefix
    neg = -n[order]
    for j in range(int(n.max()) if len(n) else 0):
        rows = order[:int(np.searchsorted(neg, -j, side="left"))]   # the sites with more than j points
        prod = (mult[rows, None] * feats[v2p[rows, 1 + j]]).astype(np.float32)
        out[rows] = (out[rows] + prod).astype(np.float32)
    return out


# ---------------------------------------------------------------- host front (predicter.py:234-300)
def host_front(cloud_xyz, cloud_normal, downsample_size=0.0005, scale=500, full_scale=128):
    """(xyz_original_all (N,3) float32, locs (N,3) int64, feats (N,6) float32, spatial_shape (3,)), as predict
    builds them with n_slice_per_side = 1.  Down-sampling is oracle.cloud_ref's; the snap is scipy's cKDTree."""
    from scipy.spatial import cKDTree
    from . import cloud_ref
    xyz, nrm = np.asarray(cloud_xyz), np.asarray(cloud_normal)
    x, y = xyz[:, 0], xyz[:, 1]
    xmin, xmax, ymin, ymax = x.min(), x.max(), y.min(), y.max()
    xlen, ylen = (xmax - xmin) / 1, (ymax - ymin) / 1
    keep = (x >= xmin) & (x <= xmin + xlen) & (y >= ymin) & (y <= ymin + ylen)
    xo, no = xyz[keep], nrm[keep]
    down = cloud_ref.voxel_down_sample(np.asarray(xo, np.float64), downsample_size)[0]
    _, idx = cKDTree(xo).query(down)
    xo, no = xo[idx], no[idx]
    s = xo * scale
    s = s - s.min(0)
    locs = s.astype(np.int64)
    shape = np.maximum(locs.max(0) + 1, full_scale)
    feats = np.concatenate([no.astype(np.float32), xo.astype(np.float32)], 1)
    return xo.astype(np.float32), locs, feats, shape


# ---------------------------------------------------------------- network
def _np(sd, k):
    v = sd[k]
    if hasattr(v, "detach"):
        v = v.detach().cpu().numpy()
    return np.asarray(v, dtype=np.float64)


def _bn_act(sd, p, x, ex):
    """ReLU(BN(x)) in float64 and its bound (module docstring)."""
    g, b, mu, var = (_np(sd, p + s) for s in (".weight", ".bias", ".running_mean", ".running_var"))
    s = g / np.sqrt(var + BN_EPS)
    t = b - mu * s
    z = x * s + t
    e = np.abs(s) * ex * (1 + U32) ** 2 + U32 * (1 + U32) * (np.abs(s * x) + np.abs(t)) + U32 * np.abs(z)
    a = np.maximum(z, 0.0)
    ea = np.where(z + e < 0, 0.0, e)
    return a, ea


def _conv(sd, p, x, ex, nbr, K, residual=None, eres=None):
    W = _np(sd, p + ".weight")
    W = W.reshape(K, W.shape[-2], W.shape[-1])
    return S.conv(x, nbr, W, bias=_np(sd, p + ".bias"), residual=residual, ex=ex, eres=eres)


def _resblock(sd, p, x, ex, nbr, cin, cout):
    if cin != cout:
        r, er = _conv(sd, p + "i_branch.0", x, ex, None, 1)
    else:
        r, er = x, ex
    a, ea = _bn_act(sd, p + "conv_branch.0", x, ex)
    h, eh = _conv(sd, p + "conv_branch.2", a, ea, nbr, 27)
    a, ea = _bn_act(sd, p + "conv_branch.3", h, eh)
    return _conv(sd, p + "conv_branch.5", a, ea, nbr, 27, residual=r, eres=er)


def _ublock(sd, p, x, ex, levels, i, m, reps):
    vox, nbr, dn, up = levels[i]
    C = m * (i + 1)
    for j in range(reps):
        x, ex = _resblock(sd, f"{p}blocks.block{j}.", x, ex, nbr, C, C)
    if dn is None:
        return x, ex
    a, ea = _bn_act(sd, p + "conv.0", x, ex)
    y, ey = _conv(sd, p + "conv.2", a, ea, dn, 8)
    y, ey = _ublock(sd, p + "u.", y, ey, levels, i + 1, m, reps)
    a, ea = _bn_act(sd, p + "deconv.0", y, ey)
    d, ed = _conv(sd, p + "deconv.2", a, ea, up, 8)
    x, ex = np.concatenate([x, d], 1), np.concatenate([ex, ed], 1)
    for j in range(reps):
        x, ex = _resblock(sd, f"{p}blocks_tail.block{j}.", x, ex, nbr, C * (2 - j), C)
    return x, ex


def _linear(W, b, a, ea, extra_u):
    """y = a W^T + b (W (out,in) float64) and its bound; extra_u adds u |W|^T |a| + u |b| for rounded weights."""
    Wt, At = W.T, np.abs(W.T)
    y = a @ Wt + b
    mag = (np.abs(a) + ea) @ At + np.abs(b)
    e = ea @ At + (W.shape[1] + 2) * U32 * (1 + 2.0 ** -20) * mag
    if extra_u:
        e += U32 * (1 + U32) * mag
    return y, e


def head(sd, x, ex):
    """output_layer, Linear, BN, ReLU, Linear per row: (y (V,3), bound)."""
    a, ea = _bn_act(sd, "output_layer.0", x, ex)
    g, b, mu, var = (_np(sd, "offset.1" + s) for s in (".weight", ".bias", ".running_mean", ".running_var"))
    s = g / np.sqrt(var + BN_EPS)
    W1 = _np(sd, "offset.0.weight") * s[:, None]
    b1 = (_np(sd, "offset.0.bias") - mu) * s + b
    h, eh = _linear(W1, b1, a, ea, True)
    eh = np.where(h + eh < 0, 0.0, eh)
    h = np.maximum(h, 0.0)
    return _linear(_np(sd, "offset.3.weight"), _np(sd, "offset.3.bias"), h, eh, False)


def levels_of(vox, shape):
    """[(vox, nbr, down, up)] for the seven levels of sites ``vox`` (sorted by key) on ``shape``."""
    out = []
    nbr = S.neighbours(vox)
    for _ in range(LEVELS - 1):
        cvox, cnbr, dn, up, shape = S.down(vox, shape)
        out.append((vox, nbr, dn, up))
        vox, nbr = cvox, cnbr
    out.append((vox, nbr, None, None))
    return out


def forward(sd, m, block_reps, vox, shape, vfeats, p2v):
    """pt_offsets (N,3) float64 and their bound, from the sites ``vox`` (V,3) in any order, the spatial shape, the
    voxel features (V,6) and each point's site p2v (N,).  Also returns the per-site (V,3) values and bound in
    ``vox``'s order."""
    vox = np.asarray(vox, dtype=np.int64)
    order = np.argsort(S.pack(vox), kind="stable")
    rank = np.empty_like(order)
    rank[order] = np.arange(len(order))
    levels = levels_of(vox[order], tuple(int(s) for s in shape))
    x = np.asarray(vfeats, dtype=np.float64)[order]
    y, ey = _conv(sd, "input_conv.0", x, np.zeros_like(x), levels[0][1], 27)
    y, ey = _ublock(sd, "unet.", y, ey, levels, 0, m, block_reps)
    o, eo = head(sd, y, ey)
    o, eo = o[rank], eo[rank]
    p2v = np.asarray(p2v, dtype=np.int64)
    return o[p2v], eo[p2v], o, eo


# ---------------------------------------------------------------- seeded weights
def synthetic_state_dict(key_shapes, seed, offset_scale=3e-3):
    """A PointGroup state_dict (float32 numpy arrays) for ``key_shapes`` [(key, shape)], drawn with numpy's
    RandomState(seed) in key order: conv weights N(0, 1 / (K Cin)) so activations stay O(1) through the levels,
    biases N(0, 0.1), BN weight U(0.5, 1.5), bias N(0, 0.1), running mean N(0, 0.3), running var U(0.5, 2) (positive);
    Linear weights N(0, 1 / in), the last Linear's weight and bias scaled so offsets come out at millimetre scale."""
    rng = np.random.RandomState(seed)
    sd = {}
    for k, shape in key_shapes:
        shape = tuple(int(s) for s in shape)
        if k.endswith("running_var"):
            a = rng.uniform(0.5, 2.0, shape)
        elif k.endswith("running_mean"):
            a = rng.normal(0.0, 0.3, shape)
        elif k.endswith(".weight") and len(shape) == 1:            # BN weight
            a = rng.uniform(0.5, 1.5, shape)
        elif k.endswith(".bias"):
            a = rng.normal(0.0, 0.1, shape)
        elif len(shape) == 5:                                     # spconv (k, k, k, Cin, Cout)
            a = rng.normal(0.0, 1.0, shape) / np.sqrt(np.prod(shape[:4]))
        else:                                                     # Linear (out, in)
            a = rng.normal(0.0, 1.0, shape) / np.sqrt(shape[1])
        if k.startswith("offset.3."):
            a = a * offset_scale
        sd[k] = a.astype(np.float32)
    return sd
